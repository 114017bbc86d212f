#!/usr/bin/env python3
"""Generate the BLS12-381 constant headers from first principles.

Writes
  oracle/oracle1/bls_constants.hpp      (u64 limbs, for the CPU oracle)
  bellman_b200/csrc/bls_constants.cuh   (u32 limbs, for the CUDA product code)

Both are derived from the curve parameter z alone (oracle/oracle0/fields.py
self-checks them); the two trees deliberately do not share a header so the
product never includes anything under oracle/.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.oracle0 import fields as F  # noqa: E402

R_MOD, P_MOD = F.FR_MODULUS, F.FP_MODULUS


def limbs(v, n, bits):
    mask = (1 << bits) - 1
    return [(v >> (bits * i)) & mask for i in range(n)]


def carr(v, n, bits):
    w = 16 if bits == 64 else 8
    suffix = "ull" if bits == 64 else "u"
    return "{" + ", ".join(f"0x{x:0{w}x}{suffix}" for x in limbs(v, n, bits)) + "}"


def field_consts(q, nbits_total):
    Rm = (1 << nbits_total) % q
    return dict(
        MOD=q, R=Rm, R2=Rm * Rm % q, R3=Rm * Rm * Rm % q,
        INV64=(-pow(q, -1, 1 << 64)) % (1 << 64),
        INV32=(-pow(q, -1, 1 << 32)) % (1 << 32),
    )


fr = field_consts(R_MOD, 256)
fp = field_consts(P_MOD, 384)
assert fr["INV64"] == 0xFFFFFFFEFFFFFFFF and fp["INV64"] == 0x89F3FFFCFFFCFFFD


def mont(v, c):
    return v * c["R"] % c["MOD"]


# ---- pairing constants: Fp12 = Fp6[w]/(w^2 - v), Fp6 = Fp2[v]/(v^3 - xi), xi = u + 1, so w^6 = xi ----
def fp2_pow(a, e):
    r = (1, 0)
    while e:
        if e & 1:
            r = F.Fp2Ops.mul(r, a)
        a = F.Fp2Ops.mul(a, a)
        e >>= 1
    return r


XI = (1, 1)
# (sum a_k w^k)^(p^m) = sum a_k^(p^m) * xi^(k (p^m - 1) / 6) * w^k: FROB<m>_<k> = xi^(k (p^m - 1) / 6)
FROB = []
for m in (1, 2):
    for k in range(1, 6):
        FROB.append((f"FROB{m}_{k}", fp2_pow(XI, k * (P_MOD ** m - 1) // 6)))
_g1 = dict(FROB)["FROB1_1"]
assert fp2_pow(_g1, 6) == F.Fp2Ops.mul((1, P_MOD - 1), F.Fp2Ops.inv(XI))             # gamma^6 = xi^(p-1) = conj(xi) / xi
assert all(dict(FROB)[f"FROB2_{k}"][1] == 0 for k in range(1, 6))                   # the p^2 coefficients lie in Fp
assert all(dict(FROB)[f"FROB2_{k}"] == F.Fp2Ops.mul(dict(FROB)[f"FROB1_{k}"], (dict(FROB)[f"FROB1_{k}"][0], -dict(FROB)[f"FROB1_{k}"][1] % P_MOD))
           for k in range(1, 6))                                                     # gamma2 = gamma1^(p+1) = norm(gamma1)
assert all(dict(FROB)[f"FROB1_{k}"] == fp2_pow(_g1, k) for k in range(1, 6))
assert (P_MOD - 1) % 6 == 0 and (P_MOD ** 2 - 1) % 6 == 0
# the hard part of the final exponentiation by the x-chain (tower.cuh fp12_final_exp):
# (x - 1)^2 (x + p) (x^2 + p^2 - 1) + 3 = 3 (p^4 - p^2 + 1) / r
_x = F.BLS_X
assert (_x - 1) ** 2 * (_x + P_MOD) * (_x ** 2 + P_MOD ** 2 - 1) + 3 == 3 * (P_MOD ** 4 - P_MOD ** 2 + 1) // R_MOD
assert (P_MOD ** 4 - P_MOD ** 2 + 1) % R_MOD == 0 and -_x == 0xD201000000010000

# ---- decoding compressed points (decode.cu) ----
# square roots: p = 3 mod 4, so sqrt(a) = a^((p+1)/4) in Fp; in Fp2 Algorithm 9 of eprint 2012/685 runs a^((p-3)/4) and
# (1 + alpha)^((p-1)/2) -- the latter exponent is FP_HALF
assert P_MOD % 4 == 3
EXP_SQRT, EXP_SQRT2 = (P_MOD + 1) // 4, (P_MOD - 3) // 4
# subgroup checks of eprint 2021/1130 (proofs for BLS12-381: eprint 2022/352):
#   G1: phi(P) = -[x^2] P  with phi(x, y) = (beta x, y), beta the cube root of unity whose eigenvalue is -x^2
#   G2: psi(P) = [x] P     with psi(x, y) = (conj(x) / xi^((p-1)/3), conj(y) / xi^((p-1)/2))
_w = next(w for w in (pow(g, (P_MOD - 1) // 3, P_MOD) for g in range(2, 100)) if w != 1)


def _mul_int(G, pt, k):                 # [k] pt for an integer k >= 0 WITHOUT reducing k mod r (pt may lie outside G1 / G2)
    acc = None
    while k:
        if k & 1:
            acc = G.add(acc, pt)
        pt = G.add(pt, pt)
        k >>= 1
    return acc


def _phi(pt):
    return (BETA * pt[0] % P_MOD, pt[1])


def _psi(pt):
    (x0, x1), (y0, y1) = pt
    return F.Fp2Ops.mul((x0, -x1 % P_MOD), PSI_X), F.Fp2Ops.mul((y0, -y1 % P_MOD), PSI_Y)


def _g1_fast_check(pt):
    return _phi(pt) == F.G1.neg(_mul_int(F.G1, pt, _x * _x))


def _g2_fast_check(pt):
    return _psi(pt) == F.G2.neg(_mul_int(F.G2, pt, -_x))


def _off_subgroup_point(G, b, make_x, sqrt):
    """the first point of y^2 = x^3 + b over x = make_x(1), make_x(2), ... outside the order-r subgroup"""
    for k in range(1, 1000):
        x = make_x(k)
        if G is F.G1:
            y = sqrt((x * x * x + b) % P_MOD)
        else:
            y = sqrt(F.Fp2Ops.add(F.Fp2Ops.mul(F.Fp2Ops.mul(x, x), x), b))
        if y is not None and G.mul((x, y), R_MOD - 1) != G.neg((x, y)):
            return (x, y)
    raise AssertionError("no point outside the subgroup found")


for BETA in (_w, _w * _w % P_MOD):
    if _g1_fast_check(F.G1_GEN):
        break
assert pow(BETA, 3, P_MOD) == 1 and BETA != 1 and _g1_fast_check(F.G1_GEN)
assert _g1_fast_check(F.G1.mul(F.G1_GEN, 0x1234567))
PSI_X = F.Fp2Ops.inv(fp2_pow(XI, (P_MOD - 1) // 3))
PSI_Y = F.Fp2Ops.inv(fp2_pow(XI, (P_MOD - 1) // 2))
assert _g2_fast_check(F.G2_GEN) and _g2_fast_check(F.G2.mul(F.G2_GEN, 0x7654321))


def _pairing_sqrt(a):
    from oracle.oracle0 import pairing as _PR
    return _PR._fp2_sqrt(a) if isinstance(a, tuple) else _PR._fp_sqrt(a)


_bad1 = _off_subgroup_point(F.G1, F.G1_B, lambda k: k, _pairing_sqrt)
_bad2 = _off_subgroup_point(F.G2, F.G2_B, lambda k: (k, 1), _pairing_sqrt)
assert F.G1.is_on_curve(_bad1) and not _g1_fast_check(_bad1)
assert F.G2.is_on_curve(_bad2) and not _g2_fast_check(_bad2)


def emit(path, bits, ns, guard):
    n_fr, n_fp = 256 // bits, 384 // bits
    macros = []

    def lst(name, v, n):
        if bits == 32:
            macros.append(f"#define BBC_{name}_LIST " + carr(v, n, bits)[1:-1])
    t = "uint64_t" if bits == 64 else "uint32_t"
    L = []
    L.append(f"// GENERATED by tools/gen_constants.py -- do not edit.\n#pragma once\n#include <cstdint>\n")
    L.append(f"namespace {ns} {{\n")
    for name, c, n in (("FR", fr, n_fr), ("FP", fp, n_fp)):
        L.append(f"static constexpr int {name}_LIMBS = {n};")
        for k in ("MOD", "R", "R2", "R3"):
            L.append(f"static constexpr {t} {name}_{k}[{n}] = {carr(c[k], n, bits)};")
            lst(f"{name}_{k}", c[k], n)
        L.append(f"static constexpr {t} {name}_INV = 0x{c['INV64' if bits == 64 else 'INV32']:x}{'ull' if bits == 64 else 'u'};")
        L.append("")
    # Fr domain constants (Montgomery form)
    L.append(f"static constexpr int FR_S = {F.FR_S};")
    L.append(f"static constexpr int FR_NUM_BITS = {F.FR_NUM_BITS};")
    L.append(f"static constexpr {t} FR_GENERATOR_M[{n_fr}] = {carr(mont(F.FR_GENERATOR, fr), n_fr, bits)};")
    L.append(f"static constexpr {t} FR_ROOT_OF_UNITY_M[{n_fr}] = {carr(mont(F.FR_ROOT_OF_UNITY, fr), n_fr, bits)};")
    lst("FR_GENERATOR_M", mont(F.FR_GENERATOR, fr), n_fr)
    lst("FR_ROOT_OF_UNITY_M", mont(F.FR_ROOT_OF_UNITY, fr), n_fr)
    lst("FP_HALF", (P_MOD - 1) // 2, n_fp)
    if bits == 32:      # p^2 as a 2N-limb integer: keeps a0*b0 - a1*b1 non-negative in the lazy Fp2 product
        L.append(f"static constexpr {t} FP_MODSQ[{2 * n_fp}] = {carr(P_MOD * P_MOD, 2 * n_fp, bits)};")
        lst("FP_MODSQ", P_MOD * P_MOD, 2 * n_fp)
    lst("G1_GEN_X_M", mont(F.G1_GEN[0], fp), n_fp)
    lst("G1_GEN_Y_M", mont(F.G1_GEN[1], fp), n_fp)
    lst("G2_GEN_X0_M", mont(F.G2_GEN[0][0], fp), n_fp)
    lst("G2_GEN_X1_M", mont(F.G2_GEN[0][1], fp), n_fp)
    lst("G2_GEN_Y0_M", mont(F.G2_GEN[1][0], fp), n_fp)
    lst("G2_GEN_Y1_M", mont(F.G2_GEN[1][1], fp), n_fp)
    # (p-1)/2 for the lexicographic sign bit of the compressed encoding
    L.append(f"static constexpr {t} FP_HALF[{n_fp}] = {carr((P_MOD - 1) // 2, n_fp, bits)};")
    # curve constants, Montgomery form
    L.append(f"static constexpr {t} G1_B_M[{n_fp}] = {carr(mont(4, fp), n_fp, bits)};")
    L.append(f"static constexpr {t} G1_GEN_X_M[{n_fp}] = {carr(mont(F.G1_GEN[0], fp), n_fp, bits)};")
    L.append(f"static constexpr {t} G1_GEN_Y_M[{n_fp}] = {carr(mont(F.G1_GEN[1], fp), n_fp, bits)};")
    (x0, x1), (y0, y1) = F.G2_GEN
    for nm, v in (("X0", x0), ("X1", x1), ("Y0", y0), ("Y1", y1)):
        L.append(f"static constexpr {t} G2_GEN_{nm}_M[{n_fp}] = {carr(mont(v, fp), n_fp, bits)};")
    if bits == 32:      # pairing (tower.cuh): |x| of the Miller loop and the Frobenius coefficients
        L.append(f"static constexpr uint64_t BLS_X_ABS = 0x{-F.BLS_X:016x}ull;")
        for name, (c0, c1) in FROB:
            if not name.startswith("FROB1"):
                continue                # the p^2 map is two p maps on the device; its coefficients are checked above only
            lst(name + "_C0", mont(c0, fp), n_fp)
            lst(name + "_C1", mont(c1, fp), n_fp)
        # decode.cu: square-root exponents (plain integers), beta and the psi coefficients (Montgomery)
        lst("EXP_SQRT", EXP_SQRT, n_fp)
        lst("EXP_SQRT2", EXP_SQRT2, n_fp)
        lst("BETA_M", mont(BETA, fp), n_fp)
        lst("PSI_X_C0_M", mont(PSI_X[0], fp), n_fp)
        lst("PSI_X_C1_M", mont(PSI_X[1], fp), n_fp)
        lst("PSI_Y_C0_M", mont(PSI_Y[0], fp), n_fp)
        lst("PSI_Y_C1_M", mont(PSI_Y[1], fp), n_fp)
    L.append(f"\n}}  // namespace {ns}\n")
    if macros:
        L.append("// literal limb lists: constexpr arrays are not addressable from device code")
        L.extend(macros)
        L.append("")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write("\n".join(L))
    print("wrote", path)


emit(os.path.join(ROOT, "oracle/oracle1/bls_constants.hpp"), 64, "o1c", "O1")
emit(os.path.join(ROOT, "bellman_b200/csrc/bls_constants.cuh"), 32, "bbc", "BB")
