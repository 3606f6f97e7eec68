"""Strip planning of sharded frames (zetaray_b200/sharding.py) on CPU: partition properties and optimality. No CUDA and no
product kernels here -- the GPU-side parity of a sharded frame against the unsharded one is tests/test_sharded_1gpu.py (ranks
as threads on one GPU) and tests/test_sharded_gpu.py (NCCL on 2 and 4 GPUs)."""
import importlib.util
import itertools
import os

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


def _sharding():
    # loaded by path: importing the package would load the CUDA library, which these CPU tests do not need
    spec = importlib.util.spec_from_file_location("zr_sharding", os.path.join(os.path.dirname(HERE), "zetaray_b200", "sharding.py"))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


S = _sharding()


def _bottleneck(costs, cuts):
    return max(sum(costs[a:b]) for a, b in zip(cuts, cuts[1:]))


@pytest.mark.parametrize("height", [1080, 2160, 96, 33])
@pytest.mark.parametrize("world", [1, 2, 3, 4, 8])
def test_plan_covers_and_aligns(height, world):
    n = S.StripPlan.num_units(height)
    if world > n:
        pytest.skip("more ranks than 32-row bands")
    rng = np.random.default_rng(height * 31 + world)
    costs = (rng.random(n) * (rng.random(n) > 0.3)).tolist()
    plan = S.StripPlan.balanced(height, world, costs)
    assert plan.world == world and plan.bounds[0] == 0 and plan.bounds[-1] == height
    assert all(b % 32 == 0 for b in plan.bounds[1:-1])
    assert all(b > a for a, b in zip(plan.bounds, plan.bounds[1:]))
    for r in range(world):
        g0, g1 = plan.rows_with_halo(r)
        y0, y1 = plan.rows(r)
        assert g0 == max(0, y0 - 32) and g1 == min(height, y1 + 32)


def test_plan_is_optimal_on_small_cases():
    rng = np.random.default_rng(7)
    for _ in range(40):
        n = int(rng.integers(3, 10))
        world = int(rng.integers(2, min(n, 5) + 1))
        costs = rng.random(n).tolist()
        plan = S.StripPlan.balanced(n * 32, world, costs)
        got = _bottleneck(costs, [b // 32 for b in plan.bounds])
        best = min(_bottleneck(costs, [0, *c, n]) for c in itertools.combinations(range(1, n), world - 1))
        assert got <= best * (1 + 1e-6)


def test_uniform_plan_1080p():
    plan = S.StripPlan.uniform(1080, 8)
    sizes = [b - a for a, b in zip(plan.bounds, plan.bounds[1:])]
    assert sum(sizes) == 1080 and max(sizes) == 160         # 34 bands over 8 ranks: the bottleneck is ceil(34 / 8) = 5 bands
