"""SHA-256 coprocessor traces (`sha256_<call>.bin`, written by a lurk-beta built with integration/rust/trace_export.patch:
one call's inputs and the aux block `synthesize_sha256` allocated).  Every such file under tests/golden/traces/ is replayed
through the oracle's restatement (CPU) and through lurk_sha256_witness_batch (-m gpu) and must match byte for byte: a
reference-written file pins the aux order, today "parity unpinned" (DESIGN.md section 2).  No reference-written file is
committed yet; a synthetic one, written from the oracle at test time, keeps the format, the loader and both replay paths
exercised and pins nothing about the reference."""
import glob
import os
import random

import numpy as np
import pytest

import sha256_gadget_oracle as G
from util import ints, pack

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMMITTED = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "traces", "sha256_*.bin")))


@pytest.fixture(scope="module")
def synthetic(tmp_path_factory, spec):
    import lurk_beta_b200.trace as T
    field, n = 2, 1
    p = spec.FIELD_MODULUS[field]
    rng = random.Random(11)
    inputs = [4, rng.randrange(p)]
    path = str(tmp_path_factory.mktemp("traces") / "sha256_00000.bin")
    T.write_sha256(path, field, n, pack(inputs), pack(G.witness(field, inputs)))
    return path


def _replay_on_oracle(path):
    import lurk_beta_b200.trace as T
    tr = T.read_sha256(path)
    ins = ints(tr.inputs)
    assert tr.aux.size // 32 == G.block_len(tr.field_id, tr.n)
    assert np.array_equal(pack(G.witness(tr.field_id, ins)), tr.aux), "oracle aux differs from the trace"


def _replay_on_gpu(path, L):
    import lurk_beta_b200.trace as T
    tr = T.read_sha256(path)
    got = L.sha256_witness_batch(tr.field_id, tr.n, tr.inputs)
    assert np.array_equal(got, tr.aux), "CUDA aux differs from the trace"


def test_reader_round_trip_and_refusals(synthetic, tmp_path):
    import lurk_beta_b200.trace as T
    tr = T.read_sha256(synthetic)
    assert tr.field_id == 2 and tr.synthetic and tr.n == 1 and tr.inputs.size == 64
    bad = str(tmp_path / "sha256_bad.bin")
    with open(synthetic, "rb") as f, open(bad, "wb") as g:
        g.write(f.read() + b"x")
    with pytest.raises(ValueError):
        T.read_sha256(bad)


def test_synthetic_trace_on_the_oracle(synthetic):
    _replay_on_oracle(synthetic)


@pytest.mark.gpu
def test_synthetic_trace_on_the_gpu(synthetic, L):
    _replay_on_gpu(synthetic, L)


@pytest.mark.parametrize("path", COMMITTED, ids=os.path.basename)
def test_committed_trace_on_the_oracle(path):
    _replay_on_oracle(path)


@pytest.mark.gpu
@pytest.mark.parametrize("path", COMMITTED, ids=os.path.basename)
def test_committed_trace_on_the_gpu(path, L):
    _replay_on_gpu(path, L)
