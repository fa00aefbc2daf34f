"""Host multi-objective geometry and the NumPy EHVI oracle, without a GPU: exactness of the non-dominated partitions on
random fronts, hypervolumes against inclusion-exclusion, the oracle's two EHVI forms, its gradient and a Monte-Carlo
check, and the model stack's plumbing.  The reference's own geometry test cases run in
tests/test_multi_objective_reference.py."""
from itertools import combinations

import numpy as np
import pytest

from tests import ehvi_oracle as eo
from trieste_b200.acquisition.multi_objective import (
    DividedAndConquerNonDominated,
    ExactPartition2dNonDominated,
    Pareto,
    get_reference_point,
    non_dominated,
    prepare_default_non_dominated_partition_bounds,
)


def _front(n, L, seed):
    """n non-dominated points: on the positive orthant of a sphere, jittered outward"""
    rng = np.random.default_rng(seed)
    p = np.abs(rng.standard_normal((n, L)))
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    return non_dominated(p * (1.0 + 0.05 * rng.uniform(size=(n, 1))))[0]


def _dominated_volume_brute(front, ref):
    """inclusion-exclusion over subsets of the front: volume of the union of the boxes [p, ref]"""
    total = 0.0
    for r in range(1, len(front) + 1):
        for sub in combinations(range(len(front)), r):
            corner = np.max(front[list(sub)], axis=0)
            total += (-1) ** (r + 1) * np.prod(np.clip(ref - corner, 0.0, None))
    return total


def test_pareto_and_reference_point_errors():
    with pytest.raises(ValueError):
        Pareto(np.zeros((3,)))
    with pytest.raises(ValueError):
        Pareto(np.zeros((3, 1)))
    with pytest.raises(ValueError):
        Pareto(np.zeros((0, 2))).hypervolume_indicator(np.ones(2))
    p = Pareto(np.array([[1.0, 0.5], [0.7, 0.6]]))
    with pytest.raises(ValueError):
        p.hypervolume_indicator(np.ones(3))
    with pytest.raises(ValueError):
        p.hypervolume_indicator(np.array([0.8, 2.0]))  # below the anti-ideal point
    with pytest.raises(ValueError):
        get_reference_point(np.zeros((0, 2)))


def test_reference_point_is_worst_front_point_plus_twice_range_over_size():
    obs = np.array([[1.0, 0.5], [0.7, 0.6], [0.2, 0.8], [2.0, 2.0]])  # the last row is dominated
    front = obs[:3]
    np.testing.assert_allclose(get_reference_point(obs), front.max(0) + 2.0 * (front.max(0) - front.min(0)) / 3)


# ---- partitions ----
# from five objectives on, fronts of 3-5 points keep the cell count in the hundreds to thousands
@pytest.mark.parametrize("L, n", [(2, 7), (3, 6), (4, 5), (5, 5), (6, 4), (7, 4), (8, 3)])
@pytest.mark.parametrize("seed", [0, 1])
def test_partition_cells_are_disjoint_and_complete(L, n, seed):
    front = _front(n, L, seed)
    ref = front.max(0) + 0.3
    anti = front.min(0) - 0.7
    lower, upper = prepare_default_non_dominated_partition_bounds(ref, front, anti)
    assert np.all(lower <= upper)
    for i in range(len(lower) - 1):  # cell i against every later cell
        ext = np.minimum(upper[i], upper[i + 1:]) - np.maximum(lower[i], lower[i + 1:])
        assert np.all(np.prod(np.clip(ext, 0.0, None), axis=1) < 1e-12), i
    cells = np.sum(np.prod(upper - lower, axis=1))
    dominated = _dominated_volume_brute(front, ref)
    assert cells + dominated == pytest.approx(np.prod(ref - anti), rel=1e-12)
    # no cell reaches into the dominated region: its lower corner is not weakly dominated by a front point
    for lo in lower:
        assert not np.any(np.all(front <= lo + 1e-12, axis=1) & np.all(lo + 1e-12 < ref))


@pytest.mark.parametrize("L, n", [(2, 6), (3, 6), (4, 5), (5, 5), (6, 4), (7, 4), (8, 4)])
def test_hypervolume_indicator_matches_inclusion_exclusion(L, n):
    front = _front(n, L, 3)
    ref = front.max(0) + 0.2
    assert Pareto(front).hypervolume_indicator(ref) == pytest.approx(_dominated_volume_brute(front, ref), rel=1e-12)


def test_partition_defaults_and_errors():
    lo, up = prepare_default_non_dominated_partition_bounds(np.array([1.0, 2.0, 3.0]))
    np.testing.assert_array_equal(lo, [[-1e10] * 3])
    np.testing.assert_array_equal(up, [[1.0, 2.0, 3.0]])
    lo, up = prepare_default_non_dominated_partition_bounds(np.array([1.0, 2.0]), np.zeros((0, 2)), np.array([-1.0, -1.0]))
    np.testing.assert_array_equal(lo, [[-1.0, -1.0]])
    with pytest.raises(ValueError):
        prepare_default_non_dominated_partition_bounds(np.ones((1, 2)))  # reference shape
    with pytest.raises(ValueError):
        prepare_default_non_dominated_partition_bounds(np.array([1.0, -2e10]))  # below the default anti-reference
    with pytest.raises(ValueError):
        prepare_default_non_dominated_partition_bounds(np.array([1.0, 1.0]), np.array([[0.0, -2e10]]))
    with pytest.raises(ValueError):
        prepare_default_non_dominated_partition_bounds(np.array([1.0, 1.0]), np.zeros((0, 2)), np.array([2.0, 0.0]))
    with pytest.raises(ValueError):
        prepare_default_non_dominated_partition_bounds(np.array([1.0, 1.0]), np.array([[0.0, 0.0]]), np.zeros(3))
    with pytest.raises(ValueError):
        prepare_default_non_dominated_partition_bounds(np.array([0.5, 0.5]), np.array([[0.0, 1.0], [1.0, 0.0]]))
    for cls in (ExactPartition2dNonDominated, DividedAndConquerNonDominated):
        with pytest.raises(ValueError, match="dominated"):
            cls(np.array([[0.0, 0.0], [1.0, 1.0]]))


def test_exact_2d_partition_is_the_staircase():
    front = np.array([[0.2, 0.8], [1.0, 0.5], [0.7, 0.6]])
    lower, upper = ExactPartition2dNonDominated(front).partition_bounds(np.array([-1.0, -1.0]), np.array([2.0, 2.0]))
    np.testing.assert_array_equal(lower, [[-1.0, -1.0], [0.2, -1.0], [0.7, -1.0], [1.0, -1.0]])
    np.testing.assert_array_equal(upper, [[0.2, 2.0], [0.7, 0.8], [1.0, 0.6], [2.0, 0.5]])


# ---- the EHVI oracle ----
def _moments(M, L, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    return rng.uniform(-0.5, 1.5, size=(M, L)), scale * rng.uniform(0.01, 0.5, size=(M, L))


@pytest.mark.parametrize("L", [2, 3, 4, 5, 6, 7, 8])
def test_oracle_product_of_sums_equals_literal_form(L):
    # the literal form costs 2^L products per cell: from five objectives on, fronts of four points and fewer candidates
    front = _front(6 if L <= 4 else 4, L, 5)
    lower, upper = prepare_default_non_dominated_partition_bounds(get_reference_point(front), front)
    mean, var = _moments(200 if L <= 4 else 48 if L <= 6 else 8, L, L)
    lit, pos = eo.ehvi_literal(mean, var, lower, upper), eo.ehvi(mean, var, lower, upper)
    np.testing.assert_allclose(pos, lit, rtol=1e-13, atol=1e-300)
    assert np.all(pos > 0)


@pytest.mark.parametrize("L", [2, 3, 4, 5, 6, 7, 8])
def test_oracle_partials_match_central_differences(L):
    front = _front(5 if L <= 5 else 4, L, 7)
    lower, upper = prepare_default_non_dominated_partition_bounds(get_reference_point(front), front)
    mean, var = _moments(50, L, 11)
    dmu, dvar = eo.ehvi_partials(mean, var, lower, upper)
    for l in range(L):
        e = np.zeros(L)
        e[l] = 1.0
        h = 1e-6
        fd_mu = (eo.ehvi(mean + h * e, var, lower, upper) - eo.ehvi(mean - h * e, var, lower, upper)) / (2 * h)
        hv = 1e-6 * var[:, l:l + 1] * e
        fd_var = (eo.ehvi(mean, var + hv, lower, upper) - eo.ehvi(mean, var - hv, lower, upper)) / (2 * hv[:, l])
        np.testing.assert_allclose(dmu[:, l], fd_mu, rtol=1e-6, atol=1e-9)
        np.testing.assert_allclose(dvar[:, l], fd_var, rtol=1e-5, atol=1e-8)


@pytest.mark.parametrize("observations, n_samples, var_scale", [
    ([[0.3, 0.2], [0.2, 0.22], [0.1, 0.25], [0.0, 0.3]], 100_000, 1.0),
    ([[0.3, 0.2], [0.2, 0.22], [0.1, 0.25], [0.0, 0.3]], 200_000, 2.0),
    ([[0.0, 0.0]], 50_000, 1.0),
    ([[2.0, 1.0], [0.8, 3.0]], 50_000, 1.0),
    ([[3.0, 2.0, 1.0], [1.1, 2.0, 3.0]], 100_000, 1.0),
    ([[3.0, 2.0, 1.0, 0.5], [1.1, 2.0, 3.0, 1.0], [2.0, 0.5, 2.0, 2.0]], 100_000, 1.0),
])
def test_oracle_matches_monte_carlo_hypervolume_improvement(observations, n_samples, var_scale):
    """the reference's cases (test_function.py:258-344, rtol 0.01, atol 0.01) plus one with four objectives; candidate
    moments are drawn around the front"""
    obs = np.asarray(observations)
    front = Pareto(obs).front
    lower, upper = prepare_default_non_dominated_partition_bounds(get_reference_point(front), front)
    L = obs.shape[1]
    rng = np.random.default_rng(L)
    mean = obs.mean(0) + rng.uniform(-1.0, 1.0, size=(4, L))
    var = var_scale * rng.uniform(0.2, 1.0, size=(4, L))
    got = eo.ehvi(mean, var, lower, upper)
    mc = [eo.hypervolume_improvement_mc(mean[i], var[i], lower, upper, n_samples, seed=i) for i in range(4)]
    np.testing.assert_allclose(got, mc, rtol=0.01, atol=0.01)


# ---- the model stack (no device: members are stand-ins with the model methods) ----
class _Member:
    def __init__(self, c):
        self.c, self.updates, self.optimized, self.logged = c, [], [], 0

    def predict(self, x):
        x = np.asarray(x)
        return np.full(x.shape[:-1] + (1,), self.c), np.full(x.shape[:-1] + (1,), 10 * self.c)

    def sample(self, x, num_samples):
        return np.full((num_samples,) + np.asarray(x).shape[:-1] + (1,), self.c)

    def log(self, dataset=None):
        self.logged += 1

    def update(self, dataset):
        self.updates.append(np.asarray(dataset.observations))

    def optimize(self, dataset):
        self.optimized.append(np.asarray(dataset.observations))


def test_model_stack_concatenates_and_splits_by_event_size():
    from trieste_b200 import Dataset, ModelStack, TrainableModelStack

    a, b = _Member(1.0), _Member(2.0)
    stack = ModelStack((a, 1), (b, 1))
    m, v = stack.predict(np.zeros((5, 3)))
    np.testing.assert_array_equal(m, np.tile([1.0, 2.0], (5, 1)))
    np.testing.assert_array_equal(v, np.tile([10.0, 20.0], (5, 1)))
    assert stack.sample(np.zeros((4, 3)), 2).shape == (2, 4, 2)
    stack.log()
    assert a.logged == b.logged == 1
    t = TrainableModelStack((a, 1), (b, 2))
    obs = np.arange(12.0).reshape(4, 3)
    t.update(Dataset(np.zeros((4, 2)), obs))
    t.optimize(Dataset(np.zeros((4, 2)), obs))
    np.testing.assert_array_equal(a.updates[0], obs[:, :1])
    np.testing.assert_array_equal(b.updates[0], obs[:, 1:])
    np.testing.assert_array_equal(b.optimized[0], obs[:, 1:])


def test_builder_repr_and_errors_without_a_device():
    from trieste_b200 import Dataset
    from trieste_b200.acquisition import ExpectedHypervolumeImprovement
    from trieste_b200.acquisition.multi_objective import get_reference_point as grp

    assert repr(ExpectedHypervolumeImprovement()) == "ExpectedHypervolumeImprovement(get_reference_point)"
    assert grp is get_reference_point
    assert repr(ExpectedHypervolumeImprovement([1.0, 2.0])).startswith("ExpectedHypervolumeImprovement(array([1., 2.])")
    with pytest.raises(ValueError, match="populated"):
        ExpectedHypervolumeImprovement().prepare_acquisition_function(None, Dataset(np.zeros((0, 2)), np.zeros((0, 2))))
    with pytest.raises(ValueError, match="ModelStack"):
        from trieste_b200.acquisition import expected_hv_improvement

        expected_hv_improvement(object(), (np.zeros((1, 2)), np.ones((1, 2))))
