"""The reference's own multi-objective geometry tests (tests/unit/acquisition/multi_objective/test_{dominance,pareto,
partition}.py of trieste 4.2.1), run on the NumPy geometry of trieste_b200.acquisition.multi_objective, and the reference's
ModelStack / TrainableModelStack protocol checked against the native stacks.

Everything comes from tests/golden/reference_multi_objective.json, extracted with ``ast`` by
tests/golden/make_multi_objective.py: each reference test's parametrised cases, literal constants, the calls it makes of
the code under test (replayed here in order, a method call on the object the last constructor call returned) and the
literal expectations of its asserts.  The fixture is checked against the digest recorded when it was extracted.  The
HV-Sharpe subset sampling (``sample_diverse_subset``) is out of scope."""
import hashlib
import json
import os

import numpy as np
import pytest

from trieste_b200.acquisition.multi_objective import (
    DividedAndConquerNonDominated,
    ExactPartition2dNonDominated,
    Pareto,
    get_reference_point,
    non_dominated,
    prepare_default_non_dominated_partition_bounds,
)

HERE = os.path.dirname(os.path.abspath(__file__))
FIXTURE = json.load(open(os.path.join(HERE, "golden", "reference_multi_objective.json")))
OUT_OF_SCOPE = "sample_diverse_subset"
FUNCTIONS = {"Pareto": Pareto, "ExactPartition2dNonDominated": ExactPartition2dNonDominated,
             "DividedAndConquerNonDominated": DividedAndConquerNonDominated, "get_reference_point": get_reference_point,
             "prepare_default_non_dominated_partition_bounds": prepare_default_non_dominated_partition_bounds,
             "compiled_non_dominated": non_dominated}


def _cases(group):
    """(test id, case index, environment) for every case of every in-scope reference test of the group"""
    out = []
    for name, t in sorted(FIXTURE[group].items()):
        if OUT_OF_SCOPE in name:
            continue
        for i, case in enumerate(t["params"] or [{}]):
            out.append(pytest.param(name, {**t["constants"], **case}, id=f"{name}[{i}]"))
    return out


def _value(x, env):
    if isinstance(x, dict) and "fill" in x:
        return np.full(x["shape"], x["fill"], dtype=np.float64)
    if isinstance(x, dict) and "expr" in x:
        e = x["expr"]
        if e.startswith("tf.constant(") and e.endswith(")"):
            e = e[len("tf.constant("):-1]
        if e not in env:
            raise KeyError(f"cannot resolve {x['expr']!r}")
        return _value(env[e], env)
    return None if x is None else np.asarray(x, dtype=np.float64)


def _replay(test, env):
    """run the test's calls of the code under test; returns the list of results"""
    results, receiver = [], None
    for c in test["calls"]:
        args = [_value(a, env) for a in c["args"]]
        if c["fn"] in FUNCTIONS:
            r = FUNCTIONS[c["fn"]](*args)
            if c["fn"][0].isupper():
                receiver = r
        else:
            r = getattr(receiver, c["fn"].split(".")[-1])(*args)
        results.append(r)
    return results


def _expected(test, i):
    return np.asarray(test["asserts"][i]["args"][1], dtype=np.float64)


def test_fixture_matches_its_recorded_digest():
    record = json.load(open(os.path.join(HERE, "golden", "reference_multi_objective.sha256.json")))
    got = hashlib.sha256(json.dumps(FIXTURE, sort_keys=True, separators=(",", ":")).encode()).hexdigest()
    assert got == record["sha256"], "tests/golden/reference_multi_objective.json differs from the extraction: re-run make_multi_objective.py"


def test_every_in_scope_reference_test_is_driven():
    for group in ("dominance", "pareto", "partition"):
        for name, t in FIXTURE[group].items():
            if OUT_OF_SCOPE in name:
                continue
            assert t["calls"], f"{group}: {name} records no call of the code under test"
            assert t["raises"] or t["asserts"] or name == "test_dominated_scales_ok", name


def _error_cases():
    return [c for g in ("dominance", "pareto", "partition") for c in _cases(g) if FIXTURE[g][c.values[0]]["raises"]]


@pytest.mark.parametrize("name, env", _error_cases())
def test_reference_error_cases_raise(name, env):
    group = next(k for k in ("dominance", "pareto", "partition") if name in FIXTURE[k])
    with pytest.raises(ValueError):
        _replay(FIXTURE[group][name], env)


@pytest.mark.parametrize("name, env", _cases("dominance"))
def test_reference_dominance_cases(name, env):
    t = FIXTURE["dominance"][name]
    if name == "test_dominated_scales_ok":  # 10,000 random points: every front point is <= some row, the mask selects them
        data = np.random.RandomState(1234).rand(int(env["num_points"]), int(env["num_objectives"]))
        front, mask = non_dominated(data)
        assert all(np.all(np.any(f <= data, axis=1)) for f in front)
        np.testing.assert_array_equal(np.sort(front, axis=0), np.sort(data[mask], axis=0))
        return
    front, mask = _replay(t, env)[0]
    expected_front = _value(env["pareto_set"], env).reshape(-1, front.shape[1])
    np.testing.assert_allclose(np.sort(front, 0), np.sort(expected_front, 0))
    np.testing.assert_array_equal(mask, _value(env["nondominated"], env).astype(bool))


@pytest.mark.parametrize("name, env", [c for c in _cases("pareto") if not FIXTURE["pareto"][c.values[0]]["raises"]])
def test_reference_pareto_cases(name, env):
    t = FIXTURE["pareto"][name]
    got = _replay(t, env)[-1]
    if name == "test_pareto_hypervolume_indicator":
        rtol = t["asserts"][0]["args"][2]
        np.testing.assert_allclose(got, _value(env["expected"], env), rtol=rtol)
    else:
        assert t["asserts"][0]["fn"] == "assert_equal"
        np.testing.assert_array_equal(got, _value(env["expected"], env))


@pytest.mark.parametrize("name, env", [c for c in _cases("partition") if not FIXTURE["partition"][c.values[0]]["raises"]])
def test_reference_partition_cases(name, env):
    t = FIXTURE["partition"][name]
    results = _replay(t, env)
    if name == "test_default_non_dominated_partition_when_no_valid_obs":
        lower, upper = results[0]
        exp = env["expected"]
        np.testing.assert_array_equal(lower, np.asarray(exp[0]))
        np.testing.assert_array_equal(upper, np.asarray(exp[1]))
    elif name in ("test_exact_partition_2d_bounds", "test_divide_conquer_non_dominated_three_dimension_case"):
        part = results[0]
        # the asserts read ._bounds.lower_idx, ._bounds.upper_idx and .front, in that order
        assert [a["args"][0]["expr"].split(".")[-1] for a in t["asserts"]] == ["lower_idx", "upper_idx", "front"]
        np.testing.assert_array_equal(part._lower_idx, _expected(t, 0))
        np.testing.assert_array_equal(part._upper_idx, _expected(t, 1))
        np.testing.assert_allclose(part.front, _expected(t, 2))
    elif name == "test_exact_partition_2d_partition_bounds":
        exp = env["expected"]
        for i in (0, 1):
            np.testing.assert_allclose(results[1 + i][i], np.asarray(exp[i]))
    else:
        raise AssertionError(f"no driver for the reference test {name}")


def _params(fn):
    import inspect

    ps = [p for p in inspect.signature(fn).parameters.values() if p.name != "self"]
    args = [p.name for p in ps if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)]
    return {"args": args, "kwonly": [p.name for p in ps if p.kind == p.KEYWORD_ONLY],
            "with_default": [p.name for p in ps if p.kind in (p.POSITIONAL_ONLY, p.POSITIONAL_OR_KEYWORD)
                             and p.default is not p.empty]}


@pytest.mark.parametrize("cls_name", ["ModelStack", "TrainableModelStack"])
def test_model_stacks_follow_the_reference_protocol(cls_name):
    import trieste_b200 as tb

    protocols = FIXTURE["protocols"]
    cls = getattr(tb, cls_name)
    methods = {}
    for name in [b for b in protocols[cls_name]["bases"] if b in protocols] + [cls_name]:
        methods.update(protocols[name]["methods"])
    assert methods
    for meth, spec in methods.items():
        got = _params(getattr(cls, meth))
        assert got["args"] == spec["args"], (cls_name, meth, got, spec)
        assert got["kwonly"] == spec["kwonly"], (cls_name, meth)
        assert got["with_default"] == spec["with_default"], (cls_name, meth, got, spec)
