"""Extract the literal expectations of the reference's multi-objective geometry tests into a JSON fixture.

    python tests/golden/make_multi_objective.py TRIESTE_CHECKOUT
        (writes tests/golden/reference_multi_objective.json and the digest tests/golden/reference_multi_objective.sha256.json)

The reference's tests/unit/acquisition/multi_objective/test_{dominance,pareto,partition}.py are parsed with ``ast`` (never
imported: they need TensorFlow).  For every test function the fixture records:

  params     the cases of its ``pytest.mark.parametrize`` decorators, one {argument name: value} dict per case
  constants  the literal values assigned to local names in its body (``objectives = tf.constant([...])``)
  asserts    every ``npt.assert_*`` / ``tf.debugging.assert_*`` call: the function name and its arguments, a literal where the
             argument is one, else {"expr": source text}
  calls      every call of the code under test, in source order: the callee's source text and its arguments, as for asserts
             (``Pareto(tf.constant([...]))``, ``partition.partition_bounds(anti, tf.constant(reference))``)
  raises     whether the body expects an exception (``pytest.raises``)

Literals: numbers, strings, None, lists and tuples (as lists), unary minus, ``tf.constant(x)`` as x, and
``tf.zeros(shape=s)`` / ``tf.ones(s)`` as {"fill": 0 or 1, "shape": s}.  The same fixture carries the structural protocol of
the reference's ``ModelStack`` and ``TrainableModelStack`` (models/interfaces.py), in make_protocols.py's format.
tests/test_multi_objective_reference.py drives the geometry and the stack's conformance from it, and checks it against the
digest recorded when it was extracted.
"""
import ast
import hashlib
import importlib.util
import json
import os
import sys

TEST_DIR = "tests/unit/acquisition/multi_objective"
FILES = {"dominance": "test_dominance.py", "pareto": "test_pareto.py", "partition": "test_partition.py"}
PROTOCOL_CLASSES = ["ModelStack", "TrainableModelStack"]


class _NotLiteral(Exception):
    pass


def literal(node):
    if isinstance(node, ast.Constant):
        return node.value
    if isinstance(node, ast.UnaryOp) and isinstance(node.op, ast.USub):
        return -literal(node.operand)
    if isinstance(node, (ast.List, ast.Tuple)):
        return [literal(e) for e in node.elts]
    if isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute):
        name = node.func.attr
        if name in ("constant", "convert_to_tensor") and node.args:
            return literal(node.args[0])
        if name in ("zeros", "ones"):
            shape = node.args[0] if node.args else next(k.value for k in node.keywords if k.arg == "shape")
            return {"fill": 0 if name == "zeros" else 1, "shape": literal(shape)}
        if name == "param":  # pytest.param(*values, id=...)
            return [literal(a) for a in node.args]
    raise _NotLiteral(ast.dump(node))


def _arg(node):
    try:
        return literal(node)
    except _NotLiteral:
        return {"expr": ast.unparse(node)}


def _params(fn):
    cases = [{}]
    for d in fn.decorator_list:
        if not (isinstance(d, ast.Call) and isinstance(d.func, ast.Attribute) and d.func.attr == "parametrize"):
            continue
        names = [n.strip() for n in literal(d.args[0]).split(",")]
        if not isinstance(d.args[1], (ast.List, ast.Tuple)):
            continue  # cases named by a module-level variable (the reference's TF compiler variants): not test data
        rows = []
        for case in d.args[1].elts:
            v = _arg(case)
            rows.append(dict(zip(names, v if len(names) > 1 else [v])))
        cases = [{**c, **r} for c in cases for r in rows]  # stacked decorators: the cross product, as pytest runs them
    return cases if cases != [{}] else []


_NOT_UNDER_TEST = ("tf", "np", "npt", "pytest", "print", "perf_counter", "timedelta", "len", "_COMPILERS")


def _under_test(func):
    root = func
    while isinstance(root, (ast.Attribute, ast.Call, ast.Subscript)):
        root = root.value if not isinstance(root, ast.Call) else root.func
    return not (isinstance(root, ast.Name) and root.id in _NOT_UNDER_TEST)


def _body(fn):
    constants, asserts, calls, raises = {}, [], [], False
    nodes = sorted((n for n in ast.walk(fn) if hasattr(n, "lineno")), key=lambda n: (n.lineno, n.col_offset))
    for node in nodes:
        if isinstance(node, ast.Assign) and len(node.targets) == 1 and isinstance(node.targets[0], ast.Name):
            try:
                constants[node.targets[0].id] = literal(node.value)
            except _NotLiteral:
                pass
        elif isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute):
            if node.func.attr.startswith("assert_"):
                asserts.append({"fn": node.func.attr, "args": [_arg(a) for a in node.args]})
            elif node.func.attr == "raises":
                raises = True
            elif _under_test(node.func):
                calls.append({"fn": ast.unparse(node.func), "args": [_arg(a) for a in node.args]})
        elif isinstance(node, ast.Call) and _under_test(node.func):
            calls.append({"fn": ast.unparse(node.func), "args": [_arg(a) for a in node.args]})
    return constants, asserts, calls, raises


def extract_tests(path):
    tree = ast.parse(open(path).read())
    out = {}
    for node in tree.body:
        if isinstance(node, ast.FunctionDef) and node.name.startswith("test_"):
            constants, asserts, calls, raises = _body(node)
            out[node.name] = {"params": _params(node), "constants": constants, "asserts": asserts, "calls": calls,
                              "raises": raises, "line": node.lineno}
    return out


def build(checkout):
    """``checkout``: the root of a trieste source checkout (the directory holding ``trieste`` and ``tests``)."""
    here = os.path.dirname(os.path.abspath(__file__))
    spec = importlib.util.spec_from_file_location("make_protocols", os.path.join(here, "make_protocols.py"))
    mp = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mp)
    fixture = {key: extract_tests(os.path.join(checkout, TEST_DIR, f)) for key, f in FILES.items()}
    fixture["protocols"] = mp.extract(os.path.join(checkout, "trieste", "models", "interfaces.py"), PROTOCOL_CLASSES)
    return fixture


def digest(fx):
    return hashlib.sha256(json.dumps(fx, sort_keys=True, separators=(",", ":")).encode()).hexdigest()


if __name__ == "__main__":
    checkout = sys.argv[1]
    fx = build(checkout)
    here = os.path.dirname(os.path.abspath(__file__))
    dst = os.path.join(here, "reference_multi_objective.json")
    with open(dst, "w") as f:
        json.dump(fx, f, indent=1, sort_keys=True)
        f.write("\n")
    version = open(os.path.join(checkout, "trieste", "VERSION")).read().strip()
    record = {"reference": f"trieste {version}", "extracted_by": "tests/golden/make_multi_objective.py",
              "canonical_json": "json.dumps(fixture, sort_keys=True, separators=(',', ':'))", "sha256": digest(fx)}
    with open(os.path.join(here, "reference_multi_objective.sha256.json"), "w") as f:
        json.dump(record, f, indent=1)
        f.write("\n")
    print("wrote", dst, {k: sorted(v) for k, v in fx.items()}, file=sys.stderr)
