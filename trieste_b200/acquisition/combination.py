"""Acquisition reducers — mirrors trieste/acquisition/combination.py (Reducer, Sum, Product, Map).

A reducer builds one acquisition function from the functions of several builders, often on different models: for
example ``Product(ExpectedImprovement().using(OBJECTIVE), ProbabilityOfFeasibility(0.5).using("CONSTRAINT"))``.  The
function it returns takes one of two routes, chosen from the built functions:

- **fused**: a ``Sum`` or ``Product`` (or :class:`~trieste_b200.acquisition.function.MakePositive`) of fused single-query
  functions — EI, log-EI, PI / PoF, (negative) LCB, AEI, MES, the feasibility criteria, BALD and predictive variance — on
  at most 8 distinct native models of one device, dtype and input dimension, with at most 8 terms.  It runs on the
  device (``tb_reduce_*``, csrc/reduce.cuh): each distinct model's predict once per chunk, one kernel for the values and
  their gradient, and so has ``value_and_gradient``, ``fused_argmax`` and the device L-BFGS (``maximize_from``).  The
  children's state (EI's eta after an update in place, a feasibility alpha, MES samples) is read at every call.
- **composed**: everything else (nested reducers, :class:`Map` and custom ``_reduce``, plain callables, q-batch children,
  mixed dtypes or devices): the children are evaluated and ``_reduce`` applied to their outputs.  ``Sum``, ``Product``
  and ``MakePositive`` offer ``value_and_gradient`` when every child does: the sum of the gradients, the product rule with
  prefix x suffix products (no division: a zero factor gives a finite gradient) and sigmoid(f) times the gradient.

Deviations from the reference:

- no builders raises ``ValueError`` (the reference raises ``InvalidArgumentError``);
- :class:`Map` and custom ``_reduce`` give values only: the reference differentiates them with TensorFlow's autodiff,
  here ``generate_continuous_optimizer`` raises its "needs value_and_gradient" error for them;
- where autodiff of a product of values would give a NaN gradient (a zero factor times an infinite partial), the
  gradients here take the finite product-rule limit.
"""
from __future__ import annotations

import copy
import ctypes as C
from abc import abstractmethod
from typing import Callable, Optional, Sequence

import numpy as np

from .. import _lib
from .function import _FusedSingleQuery, _to_host
from .interface import AcquisitionFunctionBuilder, AcquisitionFunctionClass

_FUSED_KINDS = frozenset({
    _lib.ACQ_EI, _lib.ACQ_LOG_EI, _lib.ACQ_PBT, _lib.ACQ_NEG_LCB, _lib.ACQ_LCB, _lib.ACQ_AEI, _lib.ACQ_MES,
    _lib.ACQ_FEASIBILITY_BICHON, _lib.ACQ_FEASIBILITY_RANJAN, _lib.ACQ_BALD, _lib.ACQ_PREDICTIVE_VARIANCE,
})
MAX_MODELS = 8  # distinct native models of one fused reduction
MAX_TERMS = 8

REDUCE_SUM, REDUCE_PRODUCT, REDUCE_SOFTPLUS = 0, 1, 2


def _fusable(functions) -> bool:
    """Can ``functions`` be the terms of one fused reduction (see the module docstring)?"""
    if not 1 <= len(functions) <= MAX_TERMS:
        return False
    for f in functions:
        if not isinstance(f, _FusedSingleQuery) or type(f)._native_eval is not _FusedSingleQuery._native_eval:
            return False  # EHVI, HIPPO, penalised and reduced functions run other native objects
        if f._acq not in _FUSED_KINDS:
            return False
    models = {id(f._model): f._model for f in functions}
    if len(models) > MAX_MODELS:
        return False
    first = functions[0]._model
    dim = first.get_internal_data().query_points.shape[-1]
    if any(m.device != first.device or m.dtype != first.dtype or m.get_internal_data().query_points.shape[-1] != dim
           for m in models.values()):
        return False
    samples = {}  # one model holds one set of min-value samples
    for f in functions:
        if f._acq == _lib.ACQ_MES:
            held = samples.setdefault(id(f._model), f._samples)
            if held.shape != f._samples.shape or not np.array_equal(held, f._samples):
                return False
    return True


class reduced_acquisition(_FusedSingleQuery):
    """The fused route: ``op`` (sum, product, softplus) over fused single-query functions on up to 8 distinct native
    models, evaluated by one ``tb_reduce`` object.  Shapes as the reference: ``x [..., 1, D] -> [..., 1]``.  The object
    keeps its children, and with them their models, alive."""

    def __init__(self, op: int, functions):
        self._op = int(op)
        self._functions = tuple(functions)
        members = []
        for f in self._functions:
            if all(f._model is not m for m in members):
                members.append(f._model)
        self._members = tuple(members)
        self._member_of = np.array([next(i for i, m in enumerate(members) if m is f._model) for f in self._functions],
                                   dtype=np.int32)
        self._model = members[0]  # dtype and input checks of the shape handling
        self._param = 0.0
        h = C.c_void_p()
        handles = (C.c_void_p * len(members))(*[m.handle.value for m in members])
        _lib.check(_lib.lib().tb_reduce_create(C.byref(h), handles, len(members)))
        self._h = h

    def __del__(self):
        h = getattr(self, "_h", None)
        if h is not None and h.value:
            try:
                _lib.lib().tb_reduce_destroy(h)
            except Exception:  # pragma: no cover
                pass
            self._h = None

    @property
    def functions(self) -> tuple:
        return self._functions

    def _before_call(self) -> None:
        # the children's current kinds and parameters (an update in place is seen), and the handle state they read
        for f in self._functions:
            f._before_call()
        acq = np.array([f._acq for f in self._functions], dtype=np.int32)
        param = np.array([f._param for f in self._functions], dtype=np.float64)
        alpha = np.array([getattr(f, "_alpha", 0.0) for f in self._functions], dtype=np.float64)  # feasibility only
        _lib.check(_lib.lib().tb_reduce_set_terms(self._h, self._op, len(self._functions), self._member_of.ctypes.data,
                                                  acq.ctypes.data, param.ctypes.data, alpha.ctypes.data))

    def _native_eval(self, px, M, po, pg) -> int:
        return _lib.lib().tb_reduce_eval(self._h, px, M, po, pg)

    def _native_argmax(self, px, M, best, idx) -> int:
        return _lib.lib().tb_reduce_argmax(self._h, px, M, None, best, idx)

    def _native_maximize(self, lo, up, x0, P, *args) -> int:
        return _lib.lib().tb_reduce_maximize(self._h, lo, up, x0, P, *args)


def _same_kind(outputs):
    """The children's outputs as one kind of array: as they are when all are numpy or all torch on one device, else
    host numpy."""
    kinds = {(_lib.is_torch(o), str(getattr(o, "device", ""))) for o in outputs}
    return list(outputs) if len(kinds) == 1 else [np.asarray(_to_host(o)) for o in outputs]


def _softplus(v):
    """log(1 + exp(v)), the reference's form (function.py:1951)"""
    if _lib.is_torch(v):
        import torch

        return torch.log(1 + torch.exp(v))
    return np.log(1 + np.exp(v))


def _sigmoid(v: np.ndarray) -> np.ndarray:
    """d softplus / dv = 1 / (1 + exp(-v)): the finite form of exp(v) / (1 + exp(v))"""
    with np.errstate(over="ignore"):
        return 1.0 / (1.0 + np.exp(-v))


def _product_coefficients(values):
    """d prod / d v_k = prefix_k x suffix_k, no division"""
    T = len(values)
    pre = [None] * T
    acc = np.ones_like(values[0])
    for k in range(T):
        pre[k] = acc
        acc = acc * values[k]
    coef = [None] * T
    acc = np.ones_like(values[0])
    for k in range(T - 1, -1, -1):
        coef[k] = pre[k] * acc
        acc = acc * values[k]
    return coef


class composed_acquisition(AcquisitionFunctionClass):
    """The composed route: ``reduce`` over the outputs of ``functions`` at the same points."""

    def __init__(self, reduce: Callable, functions):
        self._reduce = reduce
        self._functions = tuple(functions)

    @property
    def functions(self) -> tuple:
        return self._functions

    def __call__(self, x):
        return self._reduce(_same_kind([f(x) for f in self._functions]))


class differentiable_composed_acquisition(composed_acquisition):
    """A composed sum, product or softplus over children that all have ``value_and_gradient``: values and gradients
    (host numpy) through the sum rule, the product rule (prefix x suffix) or sigmoid(f)."""

    def __init__(self, op: int, reduce: Callable, functions):
        super().__init__(reduce, functions)
        self._op = op

    def value_and_gradient(self, x):
        pairs = [f.value_and_gradient(x) for f in self._functions]
        vals = [np.asarray(_to_host(v), dtype=np.float64) for v, _ in pairs]
        grads = [np.asarray(_to_host(g), dtype=np.float64) for _, g in pairs]
        if self._op == REDUCE_SOFTPLUS:
            return np.log(1 + np.exp(vals[0])), _sigmoid(vals[0])[..., None] * grads[0]
        if self._op == REDUCE_SUM:
            value, grad = vals[0], grads[0]
            for v, g in zip(vals[1:], grads[1:]):
                value, grad = value + v, grad + g
            return value, grad
        value = vals[0]
        for v in vals[1:]:
            value = value * v
        coef = _product_coefficients(vals)
        grad = coef[0][..., None] * grads[0]
        for c, g in zip(coef[1:], grads[1:]):
            grad = grad + c[..., None] * g
        return value, grad


def reduce_functions(op: Optional[int], reduce: Callable, functions):
    """The function of a reducer over the built ``functions``: the fused route when ``op`` (a sum, product or softplus)
    and the functions allow it, else the composed route, differentiable when ``op`` is set and every child is."""
    if op is not None and _fusable(functions):
        return reduced_acquisition(op, functions)
    if op is not None and all(hasattr(f, "value_and_gradient") for f in functions):
        return differentiable_composed_acquisition(op, reduce, functions)
    return composed_acquisition(reduce, functions)


class Reducer(AcquisitionFunctionBuilder):
    """combination.py:28-118: builds an acquisition function whose output is computed from the outputs of the
    functions of several builders, by :meth:`_reduce`."""

    _op: Optional[int] = None  # the fused / differentiable reduction this class performs, if any

    def __init__(self, *builders: AcquisitionFunctionBuilder):
        if len(builders) == 0:
            raise ValueError("At least one acquisition builder expected, got none.")
        self._acquisitions = builders
        self._function = None

    def __repr__(self) -> str:
        builders = ", ".join(map(repr, self._acquisitions))
        return f"{self.__class__.__name__}({builders})"

    def __deepcopy__(self, memo):  # a copy holds copies of the builders, and no built function (one per trust region)
        new = copy.copy(self)
        new.__dict__.pop("functions", None)
        new._acquisitions = copy.deepcopy(self._acquisitions, memo)
        new._function = None
        return new

    @property
    def acquisitions(self) -> Sequence[AcquisitionFunctionBuilder]:
        """The acquisition function builders specified at class initialisation."""
        return self._acquisitions

    def _op_for(self) -> Optional[int]:
        # a subclass with its own _reduce computes something else than the sum or product it derives from
        return self._op if type(self)._reduce is _REDUCE_OF_OP.get(self._op) else None

    def _build(self):
        self._function = reduce_functions(self._op_for(), self._reduce, self.functions)
        return self._function

    def prepare_acquisition_function(self, models, datasets=None):
        """combination.py:49-72: builds every child's function, keeps them in ``functions`` and reduces them."""
        self.functions = tuple(acq.prepare_acquisition_function(models, datasets=datasets) for acq in self.acquisitions)
        return self._build()

    def update_acquisition_function(self, function, models, datasets=None):
        """combination.py:74-94: updates every child's function with its builder.  When every child was updated in place
        and ``function`` is the one this reducer returned, that same function is returned."""
        functions = tuple(acq.update_acquisition_function(fn, models, datasets=datasets)
                          for fn, acq in zip(self.functions, self.acquisitions))
        unchanged = all(new is old for new, old in zip(functions, self.functions))
        self.functions = functions
        if unchanged and function is self._function and self._function is not None:
            return function
        return self._build()

    @abstractmethod
    def _reduce(self, inputs):
        """The output of the reduced function from the outputs of each child function."""


class Sum(Reducer):
    """combination.py:121-133: the element-wise sum of the children's outputs, in builder order."""

    _op = REDUCE_SUM

    def _reduce(self, inputs):
        out = inputs[0]
        for v in inputs[1:]:
            out = out + v
        return out


class Product(Reducer):
    """combination.py:136-148: the element-wise product of the children's outputs, in builder order."""

    _op = REDUCE_PRODUCT

    def _reduce(self, inputs):
        out = inputs[0]
        for v in inputs[1:]:
            out = out * v
        return out


_REDUCE_OF_OP = {REDUCE_SUM: Sum._reduce, REDUCE_PRODUCT: Product._reduce}


class Map(Reducer):
    """combination.py:151-177: applies ``map_fn`` to the output of one builder's function (values only, see the module
    docstring)."""

    def __init__(self, map_fn: Callable, builder: AcquisitionFunctionBuilder):
        super().__init__(builder)
        self._map_fn = map_fn

    def _reduce(self, inputs):
        if len(inputs) != 1:
            raise ValueError(f"Map reduces exactly one input, got {len(inputs)}")
        return self._map_fn(inputs[0])


__all__ = ["Map", "Product", "Reducer", "Sum"]
