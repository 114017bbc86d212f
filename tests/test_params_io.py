"""Parameters / VerifyingKey (de)serialisation (groth16/src/lib.rs:143-219,258-398): host-side
logic of the product, checked against the oracle's independent ZCash encoders and against the
byte count the reference pins (lib.rs:529: 2136 bytes for its 1-constraint circuit)."""
import random
import struct

import numpy as np
import pytest

from bellman_b200 import params_io
from oracle import o1
from oracle.oracle0 import fields as F

from emulated import worker  # noqa: F401  (the curve / subgroup checks are device code: they run on the emulated library)

R = o1.FR_MODULUS
P = o1.FP_MODULUS


def _params(sizes, seed=1):
    rng = random.Random(seed)
    mk1 = lambda n: o1.g1_fixed_mul(o1.fr_from_ints([rng.randrange(1, R) for _ in range(n)]))
    mk2 = lambda n: o1.g2_fixed_mul(o1.fr_from_ints([rng.randrange(1, R) for _ in range(n)]))
    return dict(vk_g1=mk1(3), vk_g2=mk2(3), ic=mk1(sizes[0]), h=mk1(sizes[1]), l=mk1(sizes[2]), a=mk1(sizes[3]),
                b_g1=mk1(sizes[4]), b_g2=mk2(sizes[5]))


def test_reference_size_and_round_trip(worker):
    # the reference's 1-constraint circuit: ic 2, h 3, l 2, a 3, b_g1 1, b_g2 1  -> 2136 bytes
    p = _params((2, 3, 2, 3, 1, 1))
    data = params_io.write_parameters(p)
    assert len(data) == 2136                                              # groth16/src/lib.rs:529
    q = params_io.read_parameters(data, worker=worker)
    for k in p:
        assert np.array_equal(np.asarray(p[k]).reshape(-1), q[k].reshape(-1)), k
    # encodings agree with the oracle's independent uncompressed encoder
    alpha = o1.g1_to_affine_ints(p["vk_g1"][0:1])[0]
    assert data[:96] == F.g1_uncompressed(alpha)
    beta2 = o1.g2_to_affine_ints(p["vk_g2"][0:1])[0]
    assert data[192:384] == F.g2_uncompressed(beta2)
    assert struct.unpack_from(">I", data, 864)[0] == 2                    # |ic| after the 864-byte key head


def _be48(v):
    return v.to_bytes(48, "big")


def test_rejections(worker):
    p = _params((2, 3, 2, 3, 1, 1), seed=2)
    data = bytearray(params_io.write_parameters(p))
    rd = lambda blob, checked=True: params_io.read_parameters(bytes(blob), checked=checked, worker=worker)
    with pytest.raises(EOFError):
        rd(data[:-5])
    bad = bytearray(data); bad[0] |= 0x80                                  # compressed flag in an uncompressed file
    with pytest.raises(params_io.InvalidData):
        rd(bad)
    bad = bytearray(data); bad[0] |= 0x20                                  # sort flag on an uncompressed point
    with pytest.raises(params_io.InvalidData):
        rd(bad)
    bad = bytearray(data); bad[1:48] = b"\xff" * 47; bad[0] = 0x1f         # x >= p
    with pytest.raises(params_io.InvalidData):
        rd(bad)
    # offsets: vk head 864 bytes, |ic| u32, 2 ic points, then |h| u32 at 864 + 4 + 192
    h0 = 864 + 4 + 2 * 96 + 4
    # a tampered coordinate is off the curve: refused when checked, loaded as-is otherwise (from_uncompressed_unchecked)
    bad = bytearray(data); bad[h0 + 95] ^= 1
    with pytest.raises(params_io.InvalidData, match="not on the curve"):
        rd(bad)
    rd(bad, checked=False)
    # ... but the VerifyingKey is always checked (VerifyingKey::read has no unchecked mode)
    bad = bytearray(data); bad[95] ^= 1
    with pytest.raises(params_io.InvalidData, match="alpha_g1"):
        rd(bad, checked=False)
    # a point of E(Fp) outside the order-r subgroup (the cofactor is ~2^126, so any curve point found by
    # solving for y is outside it with overwhelming probability)
    x = 5
    while True:
        rhs = (x * x * x + 4) % P
        y = pow(rhs, (P + 1) // 4, P)
        if y * y % P == rhs:
            break
        x += 1
    bad = bytearray(data); bad[h0:h0 + 96] = _be48(x) + _be48(y)
    with pytest.raises(params_io.InvalidData, match="subgroup"):
        rd(bad)
    assert np.array_equal(rd(bad, checked=False)["h"][1], p["h"][1])
    # the point at infinity inside a vector or in ic: rejected in BOTH modes (lib.rs:199-207,303-315)
    q = dict(p); q["a"] = p["a"].copy(); q["a"][1] = 0
    blob = params_io.write_parameters(q)
    for checked in (True, False):
        with pytest.raises(params_io.InvalidData, match="infinity"):
            rd(blob, checked)
    q = dict(p); q["ic"] = p["ic"].copy(); q["ic"][0] = 0
    with pytest.raises(params_io.InvalidData, match="infinity"):
        rd(params_io.write_parameters(q), False)
    # ... and accepted for alpha / beta / gamma / delta: the prover reports the subversion CRS itself (prover.rs:320-324)
    q = dict(p); q["vk_g1"] = p["vk_g1"].copy(); q["vk_g1"][2] = 0         # delta_g1 = identity
    got = rd(params_io.write_parameters(q))
    assert not got["vk_g1"][2].any()
    # an infinity flag with anything else set is not an encoding
    blob = bytearray(params_io.write_parameters(q)); d1 = 96 + 96 + 192 + 192
    assert blob[d1] == 0x40
    blob[d1 + 50] = 1
    with pytest.raises(params_io.InvalidData):
        rd(blob)
