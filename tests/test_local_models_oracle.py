"""Local models and datasets on the host (no GPU): ``LocalizedTag`` and the tag helpers (trieste utils/misc.py:224-295),
``copy_to_local_models`` / ``with_local_datasets`` (acquisition/utils.py:146-204), the regions' ``select_in_region`` and
filter masks, ``BatchTrustRegionBox.filter_datasets`` and the local-model count check (rule.py:1099-1232, 1364-1435,
1501-1566), and the BO driver's local-dataset bookkeeping (bayesian_optimizer.py:676-840), restating the reference's
unit tests (tests/unit/test_utils.py, acquisition/test_utils.py, acquisition/test_rule.py:1830-1990,
test_bayesian_optimizer.py:250-300) with host stand-ins for the models."""
import copy

import numpy as np
import pytest

from trieste_b200.acquisition.interface import OBJECTIVE
from trieste_b200.acquisition.utils import copy_to_local_models, with_local_datasets
from trieste_b200.bayesian_optimizer import BayesianOptimizer
from trieste_b200.data import Dataset
from trieste_b200.rule import BatchTrustRegionBox, SingleObjectiveTrustRegionBox, TREGOBox
from trieste_b200.space import Box
from trieste_b200.utils import LocalizedTag, get_value_for_tag, ignoring_local_tags


def _ds(x, y):
    return Dataset(np.asarray(x, dtype=np.float64), np.asarray(y, dtype=np.float64))


class _Model:
    """Stands in for a model: records the datasets it is updated with."""

    def __init__(self):
        self.updates = []

    def update(self, dataset):
        self.updates.append(dataset)

    def optimize(self, dataset):
        pass


# ---- tags --------------------------------------------------------------------------------------------------------------
def test_localized_tag():
    tag = LocalizedTag(OBJECTIVE, 2)
    assert tag.is_local and tag.global_tag == OBJECTIVE and tag.local_index == 2
    assert LocalizedTag.from_tag(tag) is tag
    glob = LocalizedTag.from_tag("foo")
    assert glob == LocalizedTag("foo", None) and not glob.is_local and glob.global_tag == "foo"
    assert {tag: 1}[LocalizedTag(OBJECTIVE, 2)] == 1  # frozen dataclass: hashable, equal by value
    with pytest.raises(ValueError, match="local index must be non-negative, got -1"):
        LocalizedTag(OBJECTIVE, -1)


def test_get_value_for_tag_and_ignoring_local_tags():
    mapping = {"a": 1, LocalizedTag("a", 0): 2, "b": 3}
    assert get_value_for_tag(None, "a") == (None, None)
    assert get_value_for_tag({OBJECTIVE: 4}) == (OBJECTIVE, 4)
    assert get_value_for_tag(mapping, LocalizedTag("a", 0), "a") == (LocalizedTag("a", 0), 2)
    assert get_value_for_tag(mapping, LocalizedTag("a", 1), "a") == ("a", 1)
    with pytest.raises(ValueError, match="none of the tags"):
        get_value_for_tag(mapping, "c")
    assert ignoring_local_tags(mapping) == {"a": 1, "b": 3}


# ---- copy_to_local_models / with_local_datasets ------------------------------------------------------------------------
@pytest.mark.parametrize("key", [OBJECTIVE, "foo"])
def test_copy_to_local_models(key):
    model = _Model()
    model.updates.append("x")
    local = copy_to_local_models(model, 3, key=key) if key != OBJECTIVE else copy_to_local_models(model, 3)
    assert list(local) == [LocalizedTag(key, i) for i in range(3)]
    for m in local.values():
        assert m is not model and m.updates == ["x"]
    local[LocalizedTag(key, 0)].updates.append("y")
    assert model.updates == ["x"] and local[LocalizedTag(key, 1)].updates == ["x"]


def test_with_local_datasets_copies_the_global_datasets():
    g = _ds([[0.0], [1.0], [2.0]], [[0.0], [1.0], [2.0]])
    h = _ds([[5.0]], [[5.0]])
    keep = _ds([[9.0]], [[9.0]])
    out = with_local_datasets({OBJECTIVE: g, "h": h, LocalizedTag(OBJECTIVE, 1): keep}, 3)
    assert set(out) == {OBJECTIVE, "h", LocalizedTag(OBJECTIVE, 1), LocalizedTag(OBJECTIVE, 0), LocalizedTag(OBJECTIVE, 2),
                        LocalizedTag("h", 0), LocalizedTag("h", 1), LocalizedTag("h", 2)}
    assert out[LocalizedTag(OBJECTIVE, 0)] is g and out[LocalizedTag(OBJECTIVE, 2)] is g
    assert out[LocalizedTag(OBJECTIVE, 1)] is keep  # an existing local dataset is kept
    assert out[LocalizedTag("h", 2)] is h


def test_with_local_datasets_by_indices():
    g = _ds([[0.0], [1.0], [2.0], [3.0]], [[10.0], [11.0], [12.0], [13.0]])
    out = with_local_datasets({OBJECTIVE: g}, 2, [np.array([0, 2]), np.array([3])])
    np.testing.assert_array_equal(out[LocalizedTag(OBJECTIVE, 0)].query_points, [[0.0], [2.0]])
    np.testing.assert_array_equal(out[LocalizedTag(OBJECTIVE, 0)].observations, [[10.0], [12.0]])
    np.testing.assert_array_equal(out[LocalizedTag(OBJECTIVE, 1)].observations, [[13.0]])
    assert out[OBJECTIVE] is g


def test_with_local_datasets_checks_the_number_of_indices():
    g = _ds([[0.0]], [[0.0]])
    with pytest.raises(ValueError, match="local_dataset_indices should have 3 entries, has 2"):
        with_local_datasets({OBJECTIVE: g}, 3, [np.array([0]), np.array([0])])


def test_deep_copies_of_a_rule_own_their_builders():
    """BatchTrustRegionBox deep-copies its base rule per region: each copy's builder keeps its own state."""
    from trieste_b200.acquisition.interface import SingleModelAcquisitionBuilder
    from trieste_b200.rule import EfficientGlobalOptimization

    class Counting(SingleModelAcquisitionBuilder):
        calls = 0

        def prepare_acquisition_function(self, model, dataset=None):
            self.calls += 1
            return self.calls

    rule = EfficientGlobalOptimization(Counting())
    a, b = copy.deepcopy(rule), copy.deepcopy(rule)
    assert a._builder.prepare_acquisition_function({OBJECTIVE: None}) == 1
    assert a._builder.prepare_acquisition_function({OBJECTIVE: None}) == 2
    assert b._builder.prepare_acquisition_function({OBJECTIVE: None}) == 1
    assert rule._builder.prepare_acquisition_function({OBJECTIVE: None}) == 1


# ---- regions -----------------------------------------------------------------------------------------------------------
def test_select_in_region():
    space = Box([0.0], [1.0])
    mapping = {OBJECTIVE: "g", LocalizedTag(OBJECTIVE, 0): "l0", LocalizedTag(OBJECTIVE, 1): "l1", "c": "gc",
               LocalizedTag("d", 1): "d1"}
    no_index = SingleObjectiveTrustRegionBox(space)
    assert no_index.select_in_region(mapping) == {OBJECTIVE: "g", "c": "gc"}
    r0 = SingleObjectiveTrustRegionBox(space, region_index=0)
    assert r0.select_in_region(mapping) == {LocalizedTag(OBJECTIVE, 0): "l0", "c": "gc"}
    r1 = SingleObjectiveTrustRegionBox(space, region_index=1)
    assert r1.select_in_region(mapping) == {LocalizedTag(OBJECTIVE, 1): "l1", "c": "gc", LocalizedTag("d", 1): "d1"}
    r2 = SingleObjectiveTrustRegionBox(space, region_index=2)
    assert r2.select_in_region(mapping) == {OBJECTIVE: "g", "c": "gc"}
    assert r2.select_in_region(None) is None
    assert r2.select_in_region({LocalizedTag(OBJECTIVE, 0): "l0"}) is None


def test_filter_masks_of_the_regions():
    space = Box([0.0], [3.0])
    region = SingleObjectiveTrustRegionBox(space, zeta=0.1, region_index=1)
    region.initialize(location_candidate=np.array([1.0]))
    datasets = {OBJECTIVE: _ds([[1.0]], [[0.0]]), LocalizedTag(OBJECTIVE, 0): _ds([[1.0]], [[0.0]]),
                LocalizedTag(OBJECTIVE, 1): _ds([[0.5], [1.1], [2.0], [0.9]], [[0.0]] * 4)}
    masks = region.get_datasets_filter_mask(datasets)
    assert list(masks) == [LocalizedTag(OBJECTIVE, 1)]
    np.testing.assert_array_equal(masks[LocalizedTag(OBJECTIVE, 1)], [False, True, False, True])
    trego = TREGOBox(space, region_index=1)
    np.testing.assert_array_equal(trego.get_datasets_filter_mask(datasets)[LocalizedTag(OBJECTIVE, 1)], [True] * 4)
    assert region.get_datasets_filter_mask(None) is None


class _FixedBox(SingleObjectiveTrustRegionBox):
    """A region that stays centred on ``centre`` with half-width ``eps`` (the reference's TestTrustRegionBox)."""

    def __init__(self, centre, space, eps):
        self._centre = np.asarray(centre, dtype=np.float64)
        self._fixed_eps = eps
        super().__init__(space)

    def _init_location(self, location_candidate=None):
        self.location = self._centre.copy()

    def _init_eps(self):
        self.eps = np.full(self._centre.shape, self._fixed_eps)

    def update(self, models=None, datasets=None):
        self._update_domain()


class _PointsInRegion:
    """A base rule that returns q points around the centre of the region it is given."""

    def __init__(self, q):
        self.q = q
        self.seen = []

    def acquire(self, search_space, models, datasets=None):
        self.seen.append((set(models), None if datasets is None else dict(datasets)))
        return search_space.location[None, :] + np.linspace(-0.1, 0.1, self.q)[:, None]


@pytest.mark.parametrize("datasets, exp_num_init_points", [
    ({OBJECTIVE: _ds([[0.0], [1.0], [2.0]], [[1.0]] * 3)}, 1),
    ({OBJECTIVE: _ds([[0.0], [1.0], [0.3], [2.0], [0.7], [1.7]], [[1.0]] * 6)}, 2),
    ({OBJECTIVE: _ds([[-1.0]], [[-1.0]]), LocalizedTag(OBJECTIVE, 0): _ds([[0.0]], [[1.0]]),
      LocalizedTag(OBJECTIVE, 1): _ds([[1.0]], [[1.0]]), LocalizedTag(OBJECTIVE, 2): _ds([[2.0]], [[1.0]])}, 1),
    ({OBJECTIVE: _ds([[-1.0]], [[-1.0]]), LocalizedTag(OBJECTIVE, 0): _ds([[0.0], [1.0]], [[1.0]] * 2),
      LocalizedTag(OBJECTIVE, 1): _ds([[2.0], [1.0]], [[1.0]] * 2), LocalizedTag(OBJECTIVE, 2): _ds([[2.0], [3.0]], [[1.0]] * 2)},
     1),
])
@pytest.mark.parametrize("q", [1, 2])
def test_updated_datasets_are_in_their_regions(datasets, exp_num_init_points, q):
    S = 3
    space = Box([-1.0], [3.0])
    subspaces = [_FixedBox([float(i)], space, 0.4) for i in range(S)]
    models = copy_to_local_models(_Model(), S)
    rule = BatchTrustRegionBox(subspaces, _PointsInRegion(q))
    points = rule.acquire(space, models, datasets)
    assert points.shape == (q * S, 1)
    new = {OBJECTIVE: _ds(points, points ** 2)}
    for s in range(S):  # region s's rows s, s + S, ... (mk_batch_observer on the [q, S, D] batch)
        new[LocalizedTag(OBJECTIVE, s)] = _ds(points[s::S], points[s::S] ** 2)
    updated = {}
    for tag in new:
        _, dataset = get_value_for_tag(datasets, tag, LocalizedTag.from_tag(tag).global_tag)
        updated[tag] = dataset + new[tag]
    filtered = rule.filter_datasets(models, updated)
    for i, subspace in enumerate(rule.subspaces):
        local = filtered[LocalizedTag(OBJECTIVE, i)]
        assert local.query_points.shape[0] == exp_num_init_points + q
        assert np.all(subspace.contains(local.query_points))
    assert filtered[OBJECTIVE].query_points.shape[0] == datasets[OBJECTIVE].query_points.shape[0] + S * q
    np.testing.assert_array_equal(filtered[OBJECTIVE].query_points, updated[OBJECTIVE].query_points)


def test_each_region_acquires_with_its_own_local_model_and_dataset():
    S = 3
    space = Box([-1.0], [3.0])
    rule = BatchTrustRegionBox([_FixedBox([float(i)], space, 0.4) for i in range(S)], _PointsInRegion(1))
    models = copy_to_local_models(_Model(), S)
    datasets = with_local_datasets({OBJECTIVE: _ds([[0.0], [1.0], [2.0]], [[1.0]] * 3)}, S)
    filtered = rule.filter_datasets(models, datasets)
    rule.acquire(space, models, filtered)
    for i, base in enumerate(rule._rules):
        tags, by_tag = base.seen[-1]
        assert tags == {OBJECTIVE}  # local tags remapped to the global tag
        assert by_tag[OBJECTIVE] is filtered[LocalizedTag(OBJECTIVE, i)]


@pytest.mark.parametrize("num_local", [1, 2, 4])
def test_local_model_count_must_match_the_regions(num_local):
    space = Box([0.0], [1.0])
    rule = BatchTrustRegionBox([SingleObjectiveTrustRegionBox(space) for _ in range(3)], _PointsInRegion(1))
    models = copy_to_local_models(_Model(), num_local)
    with pytest.raises(ValueError, match=f"the number of subspaces 3 should be equal to the number of local models "
                                         f"{num_local}"):
        rule.acquire(space, models, {OBJECTIVE: _ds([[0.5]], [[0.0]])})


def test_local_model_count_must_agree_across_tags():
    space = Box([0.0], [1.0])
    rule = BatchTrustRegionBox([SingleObjectiveTrustRegionBox(space) for _ in range(2)], _PointsInRegion(1))
    models = {**copy_to_local_models(_Model(), 2), **copy_to_local_models(_Model(), 1, key="c")}
    with pytest.raises(ValueError, match="The number of local models should be the same for all tags"):
        rule.acquire(space, models, {OBJECTIVE: _ds([[0.5]], [[0.0]])})


def test_an_emptied_local_dataset_keeps_its_previous_points():
    """Deviation (DESIGN.md): a region re-initialised away from all of its points keeps its previous local dataset."""
    space = Box([0.0, 0.0], [1.0, 1.0])
    rule = BatchTrustRegionBox([SingleObjectiveTrustRegionBox(space, zeta=0.05)], _PointsInRegion(1))
    corner = _ds([[0.95, 0.95], [0.97, 0.9]], [[1.0], [2.0]])
    models = copy_to_local_models(_Model(), 1)
    datasets = with_local_datasets({OBJECTIVE: corner}, 1)
    region_ix = LocalizedTag(OBJECTIVE, 0)
    rule.initialize_subspaces(space)
    rule._subspaces = copy.deepcopy(rule._init_subspaces)
    region = rule._subspaces[0]
    region.initialize(location_candidate=np.array([0.96, 0.93]))
    first = rule.filter_datasets(models, datasets)  # the region covers both points
    assert len(first[region_ix]) == 2
    # the region shrinks below its minimum size and re-initialises far from the corner
    region.eps = np.full(2, 1e-3)
    region._init_location = lambda location_candidate=None: setattr(region, "location", np.array([0.1, 0.1]))
    grown = {OBJECTIVE: corner + _ds([[0.9, 0.99]], [[3.0]]), region_ix: first[region_ix] + _ds([[0.9, 0.99]], [[3.0]])}
    second = rule.filter_datasets(models, grown)
    np.testing.assert_allclose(region.location, [0.1, 0.1])
    assert not region.contains(grown[region_ix].query_points).any()
    assert second[region_ix] is first[region_ix]
    assert second[OBJECTIVE] is grown[OBJECTIVE]
    # a dataset that is emptied on the first filtering keeps the points it was given
    fresh = BatchTrustRegionBox([SingleObjectiveTrustRegionBox(space, zeta=0.05)], _PointsInRegion(1))
    fresh.initialize_subspaces(space)
    fresh._subspaces = copy.deepcopy(fresh._init_subspaces)
    fresh._subspaces[0].initialize(location_candidate=np.array([0.1, 0.1]))
    assert fresh.filter_datasets(models, datasets)[region_ix] is datasets[region_ix]


# ---- the BO driver -----------------------------------------------------------------------------------------------------
class _FixedLocalRule:
    """A rule with local datasets that returns the same [q * S, D] points at every step (the reference's
    FixedLocalAcquisitionRule)."""

    def __init__(self, points, num_local_datasets):
        self._points = points
        self._n = num_local_datasets
        self.initialize_subspaces_calls = 0
        self.filter_calls = 0

    @property
    def num_local_datasets(self):
        return self._n

    def initialize_subspaces(self, search_space):
        self.initialize_subspaces_calls += 1

    def filter_datasets(self, models, datasets):
        self.filter_calls += 1
        return datasets

    def acquire(self, search_space, models, datasets=None):
        return self._points


@pytest.mark.parametrize("use_global_model", [True, False])
@pytest.mark.parametrize("use_global_init_dataset", [True, False])
@pytest.mark.parametrize("q", [1, 2])
def test_driver_routes_the_right_dataset_to_each_model(use_global_model, use_global_init_dataset, q):
    S = 4
    if use_global_init_dataset:
        init = {OBJECTIVE: _ds([[0.5], [1.5]], [[0.25], [0.35]])}
    else:
        init = {LocalizedTag(OBJECTIVE, i): _ds([[0.5 + i], [1.5 + i]], [[0.25], [0.35]]) for i in range(S)}
        init[OBJECTIVE] = _ds([[0.5], [1.5]], [[0.25], [0.35]])
    points = np.arange(q * S, dtype=np.float64)[:, None]  # row i belongs to region i mod S
    models = {OBJECTIVE: _Model()} if use_global_model else copy_to_local_models(_Model(), S)
    rule = _FixedLocalRule(points, S)
    result = BayesianOptimizer(lambda x: Dataset(x, x), Box([-1.0], [1.0])).optimize(1, init, models, rule)
    assert result.error is None, result.error
    assert rule.initialize_subspaces_calls == 1 and rule.filter_calls == 2
    final = result.try_get_final_datasets()
    np.testing.assert_array_equal(final[OBJECTIVE].query_points, np.concatenate([init[OBJECTIVE].query_points, points]))
    for i in range(S):
        start = init[OBJECTIVE] if use_global_init_dataset else init[LocalizedTag(OBJECTIVE, i)]
        np.testing.assert_array_equal(final[LocalizedTag(OBJECTIVE, i)].query_points,
                                      np.concatenate([start.query_points, points[i::S]]))
    for tag, model in result.try_get_final_models().items():
        first, last = model.updates  # the initial fit, then the update after the step
        assert first.query_points.shape == init.get(tag, init[OBJECTIVE]).query_points.shape
        assert last is final[tag]
    if use_global_model:
        assert result.try_get_final_dataset() is final[OBJECTIVE]
        assert result.try_get_final_models()[OBJECTIVE] is models[OBJECTIVE]


def test_driver_checks_the_tags():
    bo = BayesianOptimizer(lambda x: x, Box([0.0], [1.0]))
    with pytest.raises(ValueError, match="datasets and models should contain the same keys"):
        bo.optimize(1, {OBJECTIVE: _ds([[0.5]], [[0.0]])}, {"other": _Model()})
    with pytest.raises(ValueError, match="must be populated"):
        bo.optimize(1, {}, {})
    with pytest.raises(ValueError, match="Default acquisition rule EfficientGlobalOptimization requires tag"):
        bo.optimize(1, {"a": _ds([[0.5]], [[0.0]])}, {"a": _Model()})


def test_batch_trust_region_steps_grow_the_global_dataset_by_q_times_s():
    S, q = 3, 2
    space = Box([-1.0], [3.0])
    rule = BatchTrustRegionBox([_FixedBox([float(i)], space, 0.4) for i in range(S)], _PointsInRegion(q))
    init = {OBJECTIVE: _ds([[0.0], [1.0], [2.0]], [[1.0]] * 3)}
    result = BayesianOptimizer(lambda x: x ** 2, space).optimize(3, init, copy_to_local_models(_Model(), S), rule)
    assert result.error is None, result.error
    final = result.try_get_final_datasets()
    assert len(final[OBJECTIVE]) == 3 + 3 * q * S
    for i in range(S):
        model = result.try_get_final_models()[LocalizedTag(OBJECTIVE, i)]
        assert np.all(rule.subspaces[i].contains(model.updates[-1].query_points))
        assert len(model.updates[-1]) == 1 + 3 * q
