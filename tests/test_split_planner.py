"""Host logic of the tf32x3 engine's balanced split-K planner (csrc/gemm_wgmma.cuh: plan_splitk_balanced), through the
host-only C-ABI entry ta3n_plan_forward_splits.  No GPU: the planner only does arithmetic on shapes."""
import itertools

import pytest

from ta3n_b200 import _lib

BK = 32                     # K slab of the tensor-core kernels (TC_BK)
SHARED_CFG2 = [(2560, 512, 2048)]           # shared layer at cfg2: (Bs+Bt)*T = 2560 rows, 80 tiles of 64 slabs
FWD_BATCH_LIKE = [(2560, 256, 512)] + [(640, 256, 512 * r) for r in (2, 3, 4, 5)]     # short tiles next to long ones


def slabs(k):
    return -(-k // BK)


@pytest.mark.parametrize("shapes", [SHARED_CFG2, FWD_BATCH_LIKE, [(128, 128, 256)], [(4096, 4096, 4096)],
                                    [(640, 256, 1024), (640, 256, 768), (640, 256, 512)]])
def test_split_factors_are_admissible(shapes):
    ks, before, after = _lib.plan_forward_splits(shapes)
    assert len(ks) == len(shapes)
    for (m, n, k), f in zip(shapes, ks):
        assert 1 <= f <= 8
        if f > 1:
            assert slabs(k) // f >= 8, "a split must keep at least 8 slabs (one accumulator chunk) per task"
    # a split is only taken when the model says it pays for the reduce pass
    if any(f > 1 for f in ks):
        assert after + 8.0 < before * 0.92 + 1e-9
    else:
        assert after == before


def test_underfilled_grid_gets_split():
    # 80 tiles on 132 SMs: unsplit, 52 SMs idle and the launch lasts one full tile (64 slabs + overhead)
    ks, before, after = _lib.plan_forward_splits(SHARED_CFG2, sms=132)
    assert before == pytest.approx(68.0)
    assert ks[0] >= 2 and after < 0.8 * before


def test_full_waves_are_left_alone():
    # 1024 equal tiles on 128 SMs: 8 full waves, nothing to balance
    ks, before, after = _lib.plan_forward_splits([(4096, 4096, 1024)], sms=128)
    assert ks == [1] and after == before


def test_scratch_too_small_means_no_split():
    ks, before, after = _lib.plan_forward_splits(SHARED_CFG2, scratch_bytes=4096)
    assert ks == [1] and after == before
    # enough for exactly the partials of the chosen split (k * M * N floats)
    want, _, _ = _lib.plan_forward_splits(SHARED_CFG2)
    m, n, _k = SHARED_CFG2[0]
    ks2, _, _ = _lib.plan_forward_splits(SHARED_CFG2, scratch_bytes=want[0] * m * n * 4)
    assert ks2 == want


def test_deterministic_and_order_independent_makespan():
    a = _lib.plan_forward_splits(FWD_BATCH_LIKE)
    assert a == _lib.plan_forward_splits(FWD_BATCH_LIKE)
    spans = {round(_lib.plan_forward_splits(list(p))[2], 6) for p in itertools.permutations(FWD_BATCH_LIKE[:4])}
    assert len(spans) == 1, "the LPT model sorts the tasks: group order must not change the plan's cost"


def test_bad_arguments_are_rejected():
    with pytest.raises(_lib.Ta3nError):
        _lib.plan_forward_splits([(0, 128, 128)])
    with pytest.raises(_lib.Ta3nError):
        _lib.plan_forward_splits([(128, 128, 128)], sms=0)
