"""The launch-shape model of tests/test_gpu_compress_shapes.py checked without a GPU, for the H100 PCIe (114 SMs) and SXM (132 SMs): the
sizes the GPU tests derive from the SM count straddle every boundary they claim to, and the model's small cases agree with the
formulas of the kernels they restate."""
import pytest

from test_gpu_compress_shapes import (EQ_LOW_MAX, HYPERKZG_EXACT, HYPERKZG_KNOWN_BETA, IPA_LOG_N, KZG_CHUNK, KZG_SEG, Shapes, grid,
                                      kzg_lens, sweeps, tensor_groups)

SMS = [114, 132]


@pytest.mark.parametrize("sms", SMS)
def test_sumcheck_sizes_straddle_the_round_wrap(sms):
    S = Shapes(sms)
    below, at, above = S.sumcheck_sizes()
    assert S.sc_round_sweeps(below, 0) == 1 and S.sc_round_sweeps(at, 0) == 2 and S.sc_round_sweeps(above, 0) >= 3
    assert S.sc_round_sweeps(above, 1) == 2 and S.sc_round_sweeps(at, 1) == 1
    assert above <= 20                                   # the C oracle's budget
    assert S.sc_wrap == {114: 18, 132: 19}[sms]


@pytest.mark.parametrize("sms", SMS)
def test_eq_sizes_reach_every_low_and_the_wrap(sms):
    S = Shapes(sms)
    sizes = S.eq_sizes()
    assert {S.eq_low(l) for l in sizes} == set(range(EQ_LOW_MAX + 1))
    assert [S.eq_sweeps(S.eq_wrap + d) for d in (-1, 0)] == [1, 2] and S.eq_sweeps(S.eq_wrap + 1) >= 3
    assert S.eq_sweeps(24) >= 16 and S.eq_wrap == {114: 20, 132: 21}[sms]
    # below l = 4 one CTA of 128 threads writes 2^l outputs, one thread doing the work
    assert all(S.eq_threads(l) == 128 and S.eq_sweeps(l) == 1 for l in range(EQ_LOW_MAX))


@pytest.mark.parametrize("sms", SMS)
def test_inner_product_and_fold_sizes_straddle_the_caps(sms):
    S = Shapes(sms)
    sizes = S.inner_product_sizes()
    assert S.sc_cap == 1024 * sms
    assert [S.sc_sweeps(n) for n in sizes] == [1, 1, 1, 1, 1, 1, 2, 3, -(-(1 << 22) // S.sc_cap)]
    assert [S.sc_sweeps(h) for h in S.fold_scalar_halves()] == [1, 2]
    assert [S.bases_sweeps(h) for h in S.fold_bases_halves()] == [1, 2]
    assert S.bases_cap == 512 * sms


@pytest.mark.parametrize("sms", SMS)
def test_ipa_sizes_reach_three_tensor_groups_and_the_wrap(sms):
    S = Shapes(sms)
    lo, hi = IPA_LOG_N
    assert S.ipa_reach(lo)["groups"] == 3 and S.ipa_reach(16)["groups"] == 2
    reach = S.ipa_reach(hi)
    assert min(reach["dot"], reach["fold"], reach["weighted"], reach["s"]) >= 2


@pytest.mark.parametrize("sms", SMS)
def test_hyperkzg_sizes_reach_every_level_and_chunk_count(sms):
    S = Shapes(sms)
    assert [S.kzg_levels(l) for l in range(1, 25)] == [0] * 5 + [1] * 5 + [2] * 5 + [3] * 5 + [4] * 4
    assert {S.kzg_levels(l) for l in HYPERKZG_EXACT} == {1, 2, 3}
    chunks = [S.kzg_chunks(l) for l in HYPERKZG_EXACT]
    assert chunks == [1, 1, 1, 2, 8] and (1 << 13) == KZG_CHUNK
    assert [S.kzg_levels(l) for l in HYPERKZG_KNOWN_BETA] == [4, 4]
    big = S.kzg_reach(max(HYPERKZG_KNOWN_BETA))
    assert min(big["sweep0"], big["batch"], big["fold"]) >= 2
    # 2^20, the largest size the older full-chain test reaches, stays inside one sweep of the level-0 sweeps
    assert S.kzg_reach(20)["sweep0"] == 1


@pytest.mark.parametrize("sms", SMS)
def test_batch_eval_size_wraps_the_combine(sms):
    S = Shapes(sms)
    m = S.batch_eval_m()
    assert m == {114: 17, 132: 18}[sms] and S.sc_sweeps(1 << m) == 2 and S.sc_sweeps(1 << (m - 1)) == 1


def test_model_formulas():
    assert grid(0, 256, 4, 132) == 1 and grid(1, 256, 4, 132) == 1 and grid(10 ** 9, 256, 4, 132) == 528
    assert sweeps(528 * 256, 256, 4, 132) == 1 and sweeps(528 * 256 + 1, 256, 4, 132) == 2
    assert [tensor_groups(l) for l in (0, 1, 8, 9, 16, 17, 24, 25, 32)] == [1, 1, 1, 2, 2, 3, 3, 4, 4]
    assert kzg_lens(5) == [32] and kzg_lens(6) == [64, 2] and kzg_lens(11) == [2048, 64, 2] and kzg_lens(21) == [1 << 21, 1 << 16, 2048, 64, 2]
    assert KZG_SEG == 32
