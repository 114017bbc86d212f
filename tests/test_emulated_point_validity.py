"""Point validity at its edges -- csrc/encoding.cuh through decode.cu, capi.cu and generate.cu -- executed on host
threads (tests/native/).  The test bodies and point families are those of test_gpu_point_validity.py, at the same
sizes."""
import pytest

import test_gpu_point_validity as G
from emulated import worker  # noqa: F401  (the emulated-library fixture)


@pytest.mark.parametrize("group", [1, 2])
def test_emulated_decompress_and_validate(worker, group):
    G.test_decompress_and_validate(worker, group)


@pytest.mark.parametrize("group", [1, 2])
def test_emulated_decompress_edges(worker, group):
    G.test_decompress_edges(worker, group)


def test_emulated_proofs_read(worker):
    G.test_proofs_read(worker)


def test_emulated_queue_bytes_reports_the_index(worker):
    G.test_queue_bytes_reports_the_index(worker)


def test_emulated_params_read_families(worker):
    G.test_params_read_families(worker)


def test_emulated_params_read_edges(worker):
    G.test_params_read_edges(worker)


def test_emulated_params_read_zero_point_without_flag(worker):
    G.test_params_read_zero_point_without_flag(worker)


@pytest.mark.parametrize("first", [0, 63, 64, 65, 199])
def test_emulated_params_read_first_failure(worker, first):
    G.test_params_read_first_failure(worker, first)


def test_emulated_generate_rejects_torsion_generators(worker):
    G.test_generate_rejects_torsion_generators(worker)


@pytest.mark.parametrize("group", [1, 2])
def test_emulated_host_helpers(worker, group):
    G.test_host_helpers(group)


def test_emulated_proofs_write_back(worker):
    G.test_proofs_write_back(worker)
