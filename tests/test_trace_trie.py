"""Trie coprocessor traces (`trie_<call>.bin`, written by a lurk-beta built with integration/rust/trace_export.patch: one
lookup or insert call's inputs and the aux block synthesize_lookup_aux / synthesize_insert_aux allocated).  Every such
file under tests/golden/traces/ is replayed through the oracle's restatement (CPU) and through lurk_trie_witness_batch
(-m gpu) and must match byte for byte: a reference-written file pins the Poseidon aux and to_bits_le_strict order, today
unpinned (DESIGN.md section 2).  No reference-written file is committed yet; a synthetic one, written from the oracle at
test time, keeps the format, the loader and both replay paths exercised and pins nothing about the reference."""
import glob
import os

import numpy as np
import pytest

import trie_gadget_oracle as T
from util import ints, pack

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COMMITTED = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "traces", "trie_*.bin")))


@pytest.fixture(scope="module")
def synthetic(tmp_path_factory):
    import lurk_beta_b200.trace as TR
    field, height = 2, 2
    t = T.SpecTrie(field, height)
    inputs = t.insert_inputs(0o52, 9)
    path = str(tmp_path_factory.mktemp("traces") / "trie_00000.bin")
    TR.write_trie(path, field, T.INSERT, height, pack(inputs), pack(T.witness(field, T.INSERT, inputs)))
    return path


def _replay_on_oracle(path):
    import lurk_beta_b200.trace as TR
    tr = TR.read_trie(path)
    ins = ints(tr.inputs)
    assert len(ins) == T.n_inputs(tr.op, tr.height)
    assert tr.aux.size // 32 == T.block_len(tr.field_id, tr.op, tr.height)
    assert np.array_equal(pack(T.witness(tr.field_id, tr.op, ins)), tr.aux), "oracle aux differs from the trace"
    assert T.check(tr.field_id, tr.op, ints(tr.aux), ins) == []


def _replay_on_gpu(path, L):
    import lurk_beta_b200.trace as TR
    tr = TR.read_trie(path)
    got = L.trie_witness_batch(tr.field_id, tr.op, tr.height, tr.inputs)
    assert np.array_equal(got, tr.aux), "CUDA aux differs from the trace"


def test_reader_round_trip_and_refusals(synthetic, tmp_path):
    import lurk_beta_b200.trace as TR
    tr = TR.read_trie(synthetic)
    assert (tr.field_id, tr.op, tr.height, tr.synthetic) == (2, T.INSERT, 2, True)
    assert tr.inputs.size == 32 * T.n_inputs(T.INSERT, 2)
    bad = str(tmp_path / "trie_bad.bin")
    with open(synthetic, "rb") as f, open(bad, "wb") as g:
        g.write(f.read() + b"x")
    with pytest.raises(ValueError):
        TR.read_trie(bad)


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
