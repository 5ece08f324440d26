"""The byte model's choice of block groups to recompute (simclr_b200/memory.py); no GPU needed."""
from simclr_b200 import memory

CARD = 80e9
ALL = {1, 2, 3, 4}


def test_benchmarked_configuration_recomputes_nothing():
    m = memory.step_model(50, 1, 256, 224)
    assert memory.plan(m, CARD) == frozenset()


def test_resnet50_1x_at_512_per_gpu_fits_without_recomputation():
    # measured on an H100 80GB HBM3 (700 W): 41.3 GiB peak allocated, predicted 41.5 GiB
    m = memory.step_model(50, 1, 512, 224)
    assert memory.plan(m, CARD) == frozenset()
    assert memory.predicted_peak(m, set()) < memory.USABLE_FRACTION * CARD


def test_test_configurations_recompute_nothing():
    for depth, wm, b, s, sk, se in [(18, 1, 32, 64, 0, 0), (50, 1, 16, 64, 0, 0), (50, 1, 8, 64, 0.0625, 0),
                                    (50, 1, 8, 64, 0, 0.25), (18, 1, 8, 32, 0, 0), (50, 2, 32, 224, 0.0625, 0),
                                    (152, 3, 16, 224, 0.0625, 0)]:
        assert memory.plan(memory.step_model(depth, wm, b, s, sk, se), CARD) == frozenset()


def test_target_configurations_fit_with_a_plan():
    for depth, wm, b, sk in [(50, 2, 512, 0.0), (152, 2, 256, 0.0625)]:
        m = memory.step_model(depth, wm, b, 224, sk_ratio=sk)
        p = memory.plan(m, CARD)
        assert p
        assert memory.predicted_peak(m, set()) > memory.USABLE_FRACTION * CARD
        assert memory.predicted_peak(m, p) <= memory.USABLE_FRACTION * CARD < CARD


def test_plan_takes_the_most_bytes_per_flop_first():
    m = memory.step_model(50, 2, 512, 224)
    assert 1 in memory.plan(m, CARD)


def test_recomputation_reduces_the_prediction_monotonically():
    m = memory.step_model(50, 1, 512, 224)
    off, one, every = (memory.predicted_peak(m, r) for r in (set(), {1}, ALL))
    assert off > one > every


def test_finetune_plans_never_name_frozen_groups():
    for ft in range(0, 5):
        m = memory.step_model(152, 3, 2048, 224, sk_ratio=0.0625, train_mode='finetune', fine_tune_after_block=ft)
        p = memory.plan(m, CARD)
        assert not (p & set(range(1, ft + 1))), (ft, p)
        if ft <= 1:
            assert p, ft           # the trained groups do not fit without recomputation at this batch
