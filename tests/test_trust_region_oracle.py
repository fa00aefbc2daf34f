"""CPU checks of the box trust regions (trieste tests/unit/acquisition/test_rule.py:576-1800 for Box regions, restated for
this package's stateful rule), the multi-region search space (trieste/space.py:1410-1513) and the host vectorised
L-BFGS with per-problem boxes against SciPy's L-BFGS-B."""
import copy

import numpy as np
import pytest

from oracle import gp_oracle as o
from trieste_b200.acquisition.interface import OBJECTIVE, VectorizedAcquisitionFunctionBuilder
from trieste_b200.acquisition.optimizer import (
    _perform_parallel_continuous_optimization,
)
from trieste_b200.data import Dataset
from trieste_b200.rule import (
    BatchTrustRegionBox,
    DiscreteThompsonSampling,
    EfficientGlobalOptimization,
    SingleObjectiveTrustRegionBox,
    TREGOBox,
    TURBOBox,
    get_unique_points_mask,
)
from trieste_b200.space import Box, TaggedMultiSearchSpace


class _Midpoint:
    """A base rule that returns the centre of the space it is given."""

    def acquire(self, search_space, models, datasets=None):
        return ((search_space.upper + search_space.lower) / 2).reshape(-1, search_space.dimension)


class _Kernel:
    def __init__(self, lengthscales):
        self.lengthscales = np.asarray(lengthscales, dtype=np.float64)


class _Model:
    def __init__(self, lengthscales=1.0):
        self._k = _Kernel(lengthscales)

    def get_kernel(self):
        return self._k


def _ds(X, y):
    return Dataset(np.asarray(X, dtype=np.float64), np.asarray(y, dtype=np.float64))


# ---- TaggedMultiSearchSpace --------------------------------------------------------------------------------------------
def test_multi_search_space_shapes_sampling_and_containment():
    spaces = [Box([0.0, 0.0], [0.1, 0.2]), Box([0.5, 0.5], [1.0, 1.0]), Box([-1.0, 2.0], [-0.5, 3.0])]
    ms = TaggedMultiSearchSpace(spaces, tags=["a", "b", "c"])
    assert ms.subspace_tags == ("a", "b", "c") and ms.dimension == 2
    assert ms.get_subspace("b") is spaces[1]
    np.testing.assert_array_equal(ms.lower, np.stack([s.lower for s in spaces]))
    np.testing.assert_array_equal(ms.upper, np.stack([s.upper for s in spaces]))
    x = ms.sample(500, seed=3)
    assert x.shape == (500, 3, 2)
    for s, sp in enumerate(spaces):
        assert sp.contains(x[:, s]).all()
        np.testing.assert_array_equal(x[:, s], sp.sample(500, seed=3 + s))
    pts = np.array([[0.05, 0.1], [0.7, 0.9], [-0.7, 2.5], [0.3, 0.3], [0.05, 0.9]])
    np.testing.assert_array_equal(ms.contains(pts), [True, True, True, False, False])
    assert TaggedMultiSearchSpace(spaces).subspace_tags == ("0", "1", "2")


def test_multi_search_space_errors():
    with pytest.raises(ValueError, match="At least one subspace"):
        TaggedMultiSearchSpace([])
    with pytest.raises(ValueError, match="same dimension"):
        TaggedMultiSearchSpace([Box([0.0], [1.0]), Box([0.0, 0.0], [1.0, 1.0])])
    with pytest.raises(ValueError, match="Number of tags must match"):
        TaggedMultiSearchSpace([Box([0.0], [1.0])], tags=["a", "b"])
    with pytest.raises(ValueError, match="unique"):
        TaggedMultiSearchSpace([Box([0.0], [1.0]), Box([0.0], [1.0])], tags=["a", "a"])
    with pytest.raises(ValueError, match="does not exist"):
        TaggedMultiSearchSpace([Box([0.0], [1.0])]).get_subspace("x")


# ---- host L-BFGS with per-problem boxes ----------------------------------------------------------------------------
class _ShiftedQuadratics:
    """Column v maximises -|A_v (x - c_v)|^2: a vectorised function [R, V, D] -> [R, V] with its gradient."""

    def __init__(self, centres, scales):
        self.c, self.a = np.asarray(centres), np.asarray(scales)

    def __call__(self, x):
        return -np.sum((self.a * (x - self.c)) ** 2, axis=-1)

    def value_and_gradient(self, x):
        return self(x), -2.0 * self.a**2 * (x - self.c)


def _scipy_column(fn, v, starts, lo, up):
    def vg(xq):
        z = np.broadcast_to(xq[:, None, :], (len(xq), fn.c.shape[0], xq.shape[-1])).copy()
        f, g = fn.value_and_gradient(z)
        return f[:, v], g[:, v]

    return o.scipy_lbfgsb_multistart(vg, starts, lo, up)


@pytest.mark.parametrize("form", ["round_robin", "per_problem"])
def test_host_lbfgs_per_problem_boxes_match_scipy(form):
    rng = np.random.default_rng(0)
    R, V, D, S = 4, 6, 3, 3
    centres = rng.uniform(-0.5, 1.5, size=(V, D))  # some unconstrained minima lie outside their boxes
    fn = _ShiftedQuadratics(centres, rng.uniform(0.5, 2.0, size=(V, D)))
    lo_s = np.array([[0.0, 0.0, 0.0], [0.2, 0.4, 0.1], [0.6, 0.0, 0.45]])
    up_s = np.array([[1.0, 1.0, 1.0], [0.3, 0.5, 0.9], [1.0, 0.05, 0.55]])
    if form == "round_robin":
        lower, upper = lo_s, up_s  # column v in box v mod S
        box_lo = np.broadcast_to(lo_s[np.arange(V) % S], (R, V, D))
        box_up = np.broadcast_to(up_s[np.arange(V) % S], (R, V, D))
    else:
        box_lo = rng.uniform(0.0, 0.5, size=(R, V, D))
        box_up = box_lo + rng.uniform(0.01, 0.5, size=(R, V, D))
        lower, upper = box_lo.reshape(R * V, D), box_up.reshape(R * V, D)
    starts = rng.uniform(-0.2, 1.2, size=(R, V, D))
    ok, fun, x, nfev = _perform_parallel_continuous_optimization(fn, lower, upper, starts, {})
    assert ok.all() and (nfev >= 1).all()
    assert ((x >= box_lo) & (x <= box_up)).all()  # every solution in its own box
    np.testing.assert_allclose(x, np.clip(centres[None], box_lo, box_up), atol=1e-5)
    for r in range(R):
        for v in range(V):
            sok, sf, sx, _ = _scipy_column(fn, v, starts[r, v][None], box_lo[r, v], box_up[r, v])
            assert sok[0]
            np.testing.assert_allclose(x[r, v], sx[0], atol=1e-5)
            np.testing.assert_allclose(fun[r, v], sf[0], rtol=1e-8, atol=1e-9)


def test_host_lbfgs_one_box_is_unchanged_by_the_box_form():
    rng = np.random.default_rng(1)
    fn = _ShiftedQuadratics(rng.uniform(-0.5, 1.5, size=(4, 2)), np.ones((4, 2)))
    starts = rng.uniform(size=(5, 4, 2))
    a = _perform_parallel_continuous_optimization(fn, np.zeros(2), np.ones(2), starts, {})
    b = _perform_parallel_continuous_optimization(fn, np.zeros((1, 2)), np.ones((1, 2)), starts, {})
    for u, w in zip(a, b):
        np.testing.assert_array_equal(u, w)


def test_host_lbfgs_rejects_boxes_that_do_not_divide_the_vectorization():
    fn = _ShiftedQuadratics(np.zeros((4, 2)), np.ones((4, 2)))
    with pytest.raises(ValueError, match="multiple of the number of subspaces"):
        _perform_parallel_continuous_optimization(fn, np.zeros((3, 2)), np.ones((3, 2)), np.zeros((2, 4, 2)), {})


def test_device_route_rejects_per_problem_boxes(monkeypatch):
    class _DeviceQuadratics(_ShiftedQuadratics):
        def maximize_from(self, *args, **kwargs):
            raise AssertionError("per-problem boxes reached the device optimiser")

    monkeypatch.delenv("TB_LBFGS", raising=False)
    fn = _DeviceQuadratics(np.zeros((2, 2)), np.ones((2, 2)))
    with pytest.raises(ValueError, match="TB_LBFGS=host"):
        _perform_parallel_continuous_optimization(fn, np.zeros((6, 2)), np.ones((6, 2)), np.zeros((3, 2, 2)), {})
    monkeypatch.setenv("TB_LBFGS", "host")
    ok, _, x, _ = _perform_parallel_continuous_optimization(fn, np.zeros((6, 2)), np.ones((6, 2)), np.zeros((3, 2, 2)), {})
    assert ok.all()


# ---- regions ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("region", [TREGOBox, SingleObjectiveTrustRegionBox, TURBOBox])
@pytest.mark.parametrize("datasets", [None, {}, {"foo": _ds(np.zeros((1, 1)), np.zeros((1, 1)))}])
def test_regions_raise_for_missing_objective_dataset(region, datasets):
    with pytest.raises(ValueError, match="a single OBJECTIVE dataset must be provided"):
        region(Box([-1.0], [1.0])).update({OBJECTIVE: _Model()}, datasets)


def test_trust_region_box_get_dataset_min_inside_and_outside():
    space = Box([0.0, 0.0], [1.0, 1.0])
    region = SingleObjectiveTrustRegionBox(space, zeta=0.25)
    region.location = np.array([0.5, 0.5])
    region._update_domain()  # eps = 0.25: the region is [0.25, 0.75]^2
    X = np.array([[0.1, 0.1], [0.5, 0.6], [0.7, 0.3], [0.9, 0.9]])
    y = np.array([[-1.0], [0.3], [0.2], [-2.0]])
    x_min, y_min = region.get_dataset_min({OBJECTIVE: _ds(X, y)})
    np.testing.assert_array_equal(x_min, [0.7, 0.3])
    assert y_min == 0.2
    x_out, y_out = region.get_dataset_min({OBJECTIVE: _ds(X[[0, 3]], y[[0, 3]])})  # nothing inside
    assert y_out == np.inf
    x_all, y_all = region.get_values_min(X, y, in_region_only=False)
    np.testing.assert_array_equal(x_all, [0.9, 0.9])
    assert region.get_values_min(X, y, num_query_points=2, in_region_only=True)[1] == 0.2


@pytest.mark.parametrize("zeta", [0.1, 0.5, 0.7])
def test_trust_region_box_initialize(zeta):
    space = Box([0.0, 0.0], [2.0, 1.0])
    region = SingleObjectiveTrustRegionBox(space, zeta=zeta)
    region.initialize(datasets={OBJECTIVE: _ds([[0.5, 0.5]], [[1.0]])}, location_candidate=np.array([1.0, 0.5]))
    np.testing.assert_allclose(region.eps, zeta * np.array([2.0, 1.0]))
    np.testing.assert_allclose(region.lower, np.maximum([0.0, 0.0], [1.0, 0.5] - region.eps))
    np.testing.assert_allclose(region.upper, np.minimum([2.0, 1.0], [1.0, 0.5] + region.eps))
    assert region._y_min == np.inf and not region.requires_initialization


def test_trust_region_box_requires_initialization():
    region = SingleObjectiveTrustRegionBox(Box([0.0], [1.0]), min_eps=0.1)
    assert region.requires_initialization
    region.initialize()
    assert not region.requires_initialization
    region.eps = np.array([0.05])
    assert region.requires_initialization


@pytest.mark.parametrize("success", [True, False])
def test_trust_region_box_update_size(success):
    space = Box([0.0, 0.0], [1.0, 1.0])
    region = SingleObjectiveTrustRegionBox(space, beta=0.7, kappa=0.1)
    region.initialize(location_candidate=np.array([0.5, 0.5]))
    X = np.array([[0.5, 0.5], [0.55, 0.6]])
    region.update(datasets={OBJECTIVE: _ds(X, [[1.0], [0.5]])})  # first update always succeeds
    np.testing.assert_allclose(region.eps, 0.5 / 0.7)
    np.testing.assert_array_equal(region.location, [0.55, 0.6])
    volume = np.prod(region.upper - region.lower)
    y_new = 0.5 - 0.1 * volume - 0.01 if success else 0.5 - 0.1 * volume + 0.01  # kappa * volume is the bar
    region.update(datasets={OBJECTIVE: _ds(np.vstack([X, [[0.4, 0.4]]]), [[1.0], [0.5], [y_new]])})
    np.testing.assert_allclose(region.eps, 0.5 / 0.7 / 0.7 if success else 0.5 / 0.7 * 0.7)
    np.testing.assert_array_equal(region.location, [0.4, 0.4] if success else [0.55, 0.6])
    np.testing.assert_allclose(region.lower, np.maximum(0.0, region.location - region.eps))
    np.testing.assert_allclose(region.upper, np.minimum(1.0, region.location + region.eps))


# ---- TREGO ---------------------------------------------------------------------------------------------------------------
def _trego_region(space, bounds, eps, y_prev, is_global, dataset):
    region = TREGOBox(space, region_index=0)
    region.initialize(datasets={OBJECTIVE: dataset})
    region._eps, region._y_min, region._is_global = eps, y_prev, is_global
    region.lower, region.upper = bounds.lower, bounds.upper
    region.location = (bounds.lower + bounds.upper) / 2
    return region


def _trego_step(region, dataset):
    tr = BatchTrustRegionBox(region, _Midpoint())
    pts = tr.acquire(region.global_search_space, {OBJECTIVE: _Model()}, {OBJECTIVE: dataset})
    return tr.subspaces[0], pts


SPACE = Box([-2.2, -1.0], [1.3, 3.3])
EPS = 0.5 * (SPACE.upper - SPACE.lower) / 10
X2 = np.array([[0.1, 0.2], [-0.1, -0.2]])


def test_trego_starts_global_and_acquires_over_the_global_space():
    tr = BatchTrustRegionBox(TREGOBox(SPACE), _Midpoint())
    pts = tr.acquire(SPACE, {OBJECTIVE: _Model()}, {OBJECTIVE: _ds([[0.0, 0.1]], [[0.012]])})
    region = tr.subspaces[0]
    assert region._is_global and region._y_min == np.inf
    np.testing.assert_array_equal(region.lower, SPACE.lower)
    np.testing.assert_array_equal(region.upper, SPACE.upper)
    np.testing.assert_allclose(pts, [[-0.45, 1.15]])


def test_trego_successful_global_to_global_trust_region_unchanged():
    ds = _ds(X2, [[0.4], [0.3]])
    region, pts = _trego_step(_trego_region(SPACE, SPACE, EPS, 0.4, True, ds), ds)
    np.testing.assert_allclose(region._eps, EPS)
    assert region._is_global
    np.testing.assert_array_equal(region.lower, SPACE.lower)
    np.testing.assert_allclose(pts, [[-0.45, 1.15]])


def test_trego_for_unsuccessful_global_to_local_trust_region_unchanged():
    ds = _ds(X2, [[0.4], [0.5]])
    region0 = _trego_region(SPACE, SPACE, EPS, 0.4, True, ds)
    centre = region0.location.copy()
    region, pts = _trego_step(region0, ds)
    np.testing.assert_allclose(region._eps, EPS)
    assert not region._is_global
    assert (SPACE.lower < region.lower).all() and (region.upper < SPACE.upper).all()
    np.testing.assert_allclose(region.lower, centre - EPS)
    assert SPACE.contains(pts).all()


@pytest.mark.parametrize("y1,grows", [(0.3, True), (0.5, False)])
def test_trego_local_to_global_eps_changes_by_beta(y1, grows):
    ds = _ds(X2, [[0.4], [y1]])
    local = Box(X2[0] - EPS, X2[0] + EPS)
    region, _ = _trego_step(_trego_region(SPACE, local, EPS, 0.4, False, ds), ds)
    np.testing.assert_allclose(region._eps, EPS / 0.7 if grows else EPS * 0.7)
    assert region._is_global
    np.testing.assert_array_equal(region.lower, SPACE.lower)
    np.testing.assert_array_equal(region.upper, SPACE.upper)


def test_trego_always_uses_the_global_dataset():
    space = Box([0.0, 0.0], [1.0, 1.0])
    region = TREGOBox(space)
    region.initialize(location_candidate=np.array([0.5, 0.5]))
    X = np.array([[0.5, 0.5], [1.1, 2.3], [-0.1, -0.2]])  # the best points lie outside the space
    x_min, y_min = region.get_dataset_min({OBJECTIVE: _ds(X, [[0.4], [0.1], [0.2]])})
    np.testing.assert_array_equal(x_min, [1.1, 2.3])
    assert y_min == 0.1


def test_trego_region_deepcopy():
    ds = _ds(X2, [[0.4], [0.5]])
    region = _trego_region(Box([1.2], [3.4]), Box([1.2], [3.4]), np.array([5.6]), 7.8, False, ds)
    c = copy.deepcopy(region)
    np.testing.assert_array_equal(c.lower, region.lower)
    np.testing.assert_array_equal(c._eps, region._eps)
    assert c._y_min == region._y_min and c._is_global == region._is_global


# ---- TuRBO ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize(
    "L_init, L_max, L_min, failure_tolerance, success_tolerance",
    [(-1.0, 0.1, 1.0, 1, 1), (10.0, -1.0, 1.0, 1, 1), (10.0, 1.0, -4.0, 1, 1), (10.0, 1.0, 4.0, -1, 2),
     (10.0, 1.0, 4.0, 1, -1)],
)
def test_turbo_raises_for_invalid_trust_region_params(L_init, L_max, L_min, failure_tolerance, success_tolerance):
    with pytest.raises(ValueError):
        TURBOBox(Box([-1.0], [1.0]), L_init=L_init, L_max=L_max, L_min=L_min, failure_tolerance=failure_tolerance,
                 success_tolerance=success_tolerance)


def test_turbo_heuristics_for_param_init_work(monkeypatch):
    space = Box([-2.0] * 20, [1.0] * 20)
    monkeypatch.setattr(DiscreteThompsonSampling, "acquire", _Midpoint.acquire)
    rule = BatchTrustRegionBox(TURBOBox(space))
    ds = _ds(np.zeros((1, 20)), [[0.0]])
    rule.acquire(space, {OBJECTIVE: _Model()}, {OBJECTIVE: ds})
    region = rule._init_subspaces[0]
    assert region.L_init == 0.8 * 3.0 and region.L_min == 0.5**7 * 3.0 and region.L_max == 1.6 * 3.0
    assert region.failure_tolerance == 20
    assert isinstance(rule._rule, DiscreteThompsonSampling) and rule._rule._num_search_space_samples == 2000
    rule = BatchTrustRegionBox(TURBOBox(space), rule=_Midpoint())
    rule.acquire(space, {OBJECTIVE: _Model()}, {OBJECTIVE: ds})
    assert isinstance(rule._rule, _Midpoint)


def _turbo_region(space, L, failure_counter, success_counter, y_prev, ds, models):
    region = TURBOBox(space)
    region.initialize(models, {OBJECTIVE: ds})
    region.L, region.failure_counter, region.success_counter, region.y_min = L, failure_counter, success_counter, y_prev
    return region


TURBO_SPACE = Box([0.0, 0.0], [1.0, 1.0])
TURBO_DS = _ds([[0.0, 0.0]], [[0.012]])
TURBO_MODELS = {OBJECTIVE: _Model([4.0, 1.0])}


def _turbo_step(region):
    tr = BatchTrustRegionBox(region, _Midpoint())
    tr.acquire(TURBO_SPACE, TURBO_MODELS, {OBJECTIVE: TURBO_DS})
    return tr.subspaces[0]


def test_turbo_doesnt_change_size_unless_needed():
    for failure_counter in (0, 1):
        for success_counter in (0, 1):  # a success, but not enough to grow
            r = _turbo_step(_turbo_region(TURBO_SPACE, 0.8, failure_counter, success_counter, 2.012, TURBO_DS, TURBO_MODELS))
            assert r.L == 0.8 and r.success_counter == success_counter + 1 and r.failure_counter == 0
            np.testing.assert_allclose(r.lower, [0.0, 0.0])
            np.testing.assert_allclose(r.upper, [0.8, 0.2])  # widths 1.6 x 0.4 at lengthscales 4:1, half in the box
    for success_counter in (0, 1, 2):  # a failure, but not enough to shrink
        r = _turbo_step(_turbo_region(TURBO_SPACE, 0.8, 0, success_counter, 0.012, TURBO_DS, TURBO_MODELS))
        assert r.L == 0.8 and r.success_counter == 0 and r.failure_counter == 1
        np.testing.assert_allclose(r.upper, [0.8, 0.2])


def test_turbo_does_change_size_correctly_when_needed():
    r = _turbo_step(_turbo_region(TURBO_SPACE, 0.8, 0, 2, 2.012, TURBO_DS, TURBO_MODELS))  # third success: double
    assert r.L == 1.6 and r.success_counter == 0 and r.failure_counter == 0
    np.testing.assert_allclose(r.upper, [1.0, 0.4])
    r = _turbo_step(_turbo_region(TURBO_SPACE, 0.8, 1, 0, 0.012, TURBO_DS, TURBO_MODELS))  # second failure (D = 2): halve
    assert r.L == 0.4 and r.failure_counter == 0
    np.testing.assert_allclose(r.upper, [0.4, 0.1])
    r = _turbo_step(_turbo_region(TURBO_SPACE, 1.6, 0, 2, 2.012, TURBO_DS, TURBO_MODELS))  # capped at L_max
    assert r.L == 1.6


def test_turbo_restarts_tr_when_too_small():
    region = _turbo_region(TURBO_SPACE, 0.5**7 * 1.0 * 1.5, 1, 0, 0.012, TURBO_DS, TURBO_MODELS)
    r = _turbo_step(region)  # halving drops L below L_min
    assert r.L == r.L_init == 0.8 and r.failure_counter == 0 and r.success_counter == 0


# ---- BatchTrustRegionBox -------------------------------------------------------------------------------------------------
def test_multi_trust_region_box_no_subspace_creates_one_per_query_point():
    space = Box([0.0, 0.0], [1.0, 1.0])
    rule = BatchTrustRegionBox(rule=EfficientGlobalOptimization(_BatchBuilder(), optimizer=_mid_opt, num_query_points=3))
    pts = rule.acquire(space, {OBJECTIVE: _Model()}, {OBJECTIVE: _ds([[0.1, 0.1]], [[0.0]])})
    assert len(rule.subspaces) == 3 and all(type(s) is SingleObjectiveTrustRegionBox for s in rule.subspaces)
    assert [s.region_index for s in rule.subspaces] == [0, 1, 2]
    assert pts.shape == (3, 2)
    for s, region in enumerate(rule.subspaces):
        np.testing.assert_allclose(pts[s], (region.lower + region.upper) / 2)


def test_multi_trust_region_box_single_subspace():
    region = SingleObjectiveTrustRegionBox(Box([0.0], [1.0]))
    rule = BatchTrustRegionBox(region, _Midpoint())
    assert rule._init_subspaces == (region,) and rule._tags == ("0",)


def test_multi_trust_region_box_raises_on_mismatched_global_search_space():
    rule = BatchTrustRegionBox(SingleObjectiveTrustRegionBox(Box([0.0], [1.0])), _Midpoint())
    with pytest.raises(ValueError, match="global search space"):
        rule.acquire(Box([0.0], [2.0]), {OBJECTIVE: _Model()}, {OBJECTIVE: _ds([[0.1]], [[0.0]])})


def test_multi_trust_region_box_leaves_the_callers_regions_alone_and_flattens_per_region_points():
    space = Box([0.0, 0.0], [1.0, 1.0])
    regions = [SingleObjectiveTrustRegionBox(space) for _ in range(3)]
    before = [r.location.copy() for r in regions]

    class _TwoPoints:
        def acquire(self, search_space, models, datasets=None):
            c = (search_space.upper + search_space.lower) / 2
            return np.stack([c, search_space.lower])

    rule = BatchTrustRegionBox(regions, _TwoPoints())
    pts = rule.acquire(space, {OBJECTIVE: _Model()}, {OBJECTIVE: _ds([[0.1, 0.1]], [[0.0]])})
    assert all(np.array_equal(r.location, b) for r, b in zip(regions, before)) and not regions[0]._initialized
    assert rule.subspaces[0] is not regions[0] and len(rule._rules) == 3
    assert pts.shape == (6, 2)  # [q = 2, S = 3, D] flattened
    q = pts.reshape(2, 3, 2)
    for s, region in enumerate(rule.subspaces):
        np.testing.assert_allclose(q[0, s], (region.lower + region.upper) / 2)
        np.testing.assert_allclose(q[1, s], region.lower)


def test_multi_trust_region_box_inits_regions_that_need_it():
    space = Box([0.0], [1.0])
    ds = _ds([[0.5], [0.6], [0.7]], [[0.1], [0.2], [0.3]])
    regions = [SingleObjectiveTrustRegionBox(space, zeta=0.4, min_eps=0.3) for _ in range(3)]
    for i, r in enumerate(regions):
        r.initialize(location_candidate=np.array([0.5 + i * 0.1]))
    regions[0].eps, regions[1].eps, regions[2].eps = np.array([0.45]), np.array([0.25]), np.array([0.42])
    assert [bool(r.requires_initialization) for r in regions] == [False, True, False]
    rule = BatchTrustRegionBox(regions, _Midpoint())
    rule.update_subspaces({OBJECTIVE: _Model()}, {OBJECTIVE: ds})
    s = rule.subspaces
    assert s[0].eps[0] > 0.45 and s[1].eps[0] == 0.4  # a successful step grows region 0; region 1 re-initialises
    assert s[2].eps[0] == 0.4  # region 2 also moved to the best point, 0.5, a duplicate of region 0's centre: re-initialised


def test_multi_trust_region_box_reinitialises_duplicate_centres():
    space = Box([0.0, 0.0], [1.0, 1.0])
    regions = [SingleObjectiveTrustRegionBox(space) for _ in range(3)]
    for i, r in enumerate(regions):  # centres near the best point, all of which contain it
        r.initialize(location_candidate=np.array([0.35 + 0.05 * i, 0.4]))
    rule = BatchTrustRegionBox(regions, _Midpoint())
    ds = _ds([[0.3, 0.3], [0.9, 0.9]], [[0.0], [1.0]])
    rule.acquire(space, {OBJECTIVE: _Model()}, {OBJECTIVE: ds})  # every region moves to the best point: duplicates
    centres = np.stack([r.location for r in rule.subspaces])
    np.testing.assert_array_equal(centres[0], [0.3, 0.3])
    assert not np.array_equal(centres[1], [0.3, 0.3]) and not np.array_equal(centres[2], [0.3, 0.3])
    assert [r.eps[0] for r in rule.subspaces] == [0.5 / 0.7, 0.5, 0.5]  # region 0 grew; 1 and 2 re-initialised
    assert get_unique_points_mask(centres).all()
    np.testing.assert_array_equal(get_unique_points_mask(np.array([[1.0], [2.0], [3.0], [4.0]]), 1.0),
                                  [True, False, True, False])


class _BatchBuilder(VectorizedAcquisitionFunctionBuilder):
    """A stand-in vectorised builder: the function is never evaluated by ``_mid_opt``."""

    def prepare_acquisition_function(self, models, datasets=None):
        return lambda x: np.zeros(x.shape[:-1])

    def update_acquisition_function(self, fn, models, datasets=None):
        return fn


def _mid_opt(space, target):
    """Column v -> centre of subspace v mod S (the round robin of the continuous optimiser)."""
    fn, V = target if isinstance(target, tuple) else (target, 1)
    mids = (space.lower + space.upper) / 2
    return mids[np.arange(V) % len(mids)]
