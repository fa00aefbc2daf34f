"""Acquisition-function maximisers — mirrors trieste/acquisition/optimizer.py
(``generate_random_search_optimizer`` :973-1011, ``_get_max_discrete_points`` :124-150,
``sample_from_space`` :196-244, ``generate_initial_points`` :247-341,
``generate_continuous_optimizer`` :344-563, ``batchify_joint`` :897-936,
``automatic_optimizer_selector`` :90-121).

``AcquisitionOptimizer = Callable[[SearchSpace, fn | (fn, V)], points [V, D]]``.

Where the reference multiplexes one SciPy L-BFGS-B run per start through greenlets onto a batched TF
evaluation (:566-745), this module runs ONE multi-start projected L-BFGS over all starts: every
iteration is a single fused value+gradient launch on the GPU for all active starts.  For the fused
single-model functions (EI, log-EI, LCB, PI, AEI, MES) the per-start bookkeeping — two-loop recursion,
line search, convergence tests — runs on the device as well (``tb_acq_maximize``, csrc/lbfgs.cuh; one
warp per start), and so does it for the negated trajectories of continuous Thompson sampling (``tb_rff_maximize``, one
problem per start and trajectory); any other function with a ``value_and_gradient`` method goes through the vectorised
NumPy implementation of the same algorithm below (also selectable with ``TB_LBFGS=host``).  Same
stopping rules as SciPy's defaults (gtol 1e-5 on the projected gradient, ftol 2.2e-9 relative
decrease, maxiter).
"""
from __future__ import annotations

import os
from typing import Callable, Iterator, Optional, Tuple, Union

import numpy as np

from ..space import Box, DiscreteSearchSpace, SearchSpace, TaggedMultiSearchSpace

NUM_SAMPLES_MIN = 5000  # optimizer.py:46-66
NUM_SAMPLES_DIM = 1000
NUM_RUNS_DIM = 10

AcquisitionFunction = Callable
TargetFunc = Union[AcquisitionFunction, Tuple[AcquisitionFunction, int]]


class FailedOptimizationError(Exception):
    """optimizer.py:69-70."""


def _split(target_func: TargetFunc):
    if isinstance(target_func, tuple):
        fn, V = target_func
    else:
        fn, V = target_func, 1
    if V < 0:
        raise ValueError(f"vectorization must be positive, got {V}")
    return fn, V


def _to_numpy(x):
    if type(x).__module__.split(".")[0] == "torch":
        return x.detach().cpu().numpy()
    return np.asarray(x)


def _get_max_discrete_points(points: np.ndarray, target_func: TargetFunc) -> np.ndarray:
    """optimizer.py:124-150: points [M, 1, D] -> best point per vectorised function [V, D];
    first maximal index wins (tf.math.argmax)."""
    fn, V = _split(target_func)
    if V == 1 and hasattr(fn, "fused_argmax"):
        # fused predict + tail + argmax: the M values are never written out
        flat = points[:, 0, :]
        idx, _ = fn.fused_argmax(flat)
        return _to_numpy(flat[idx : idx + 1])
    tiled = np.tile(points, [1, V, 1])
    values = _to_numpy(fn(tiled))
    if values.ndim != 2 or values.shape[-1] != V:
        raise ValueError(
            f"The result of function target_func has shape {values.shape}, however, expected a trailing dimension of size {V}."
        )
    best = np.argmax(values, axis=0)  # [V]
    return np.stack([tiled[best[v], v, :] for v in range(V)], axis=0)


def generate_random_search_optimizer(num_samples: int = NUM_SAMPLES_MIN):
    """optimizer.py:973-1011."""
    if num_samples <= 0:
        raise ValueError(f"num_samples must be positive, got {num_samples}")

    def optimize_random(space: SearchSpace, target_func: TargetFunc) -> np.ndarray:
        points = space.sample(num_samples)[:, None, :]
        return _get_max_discrete_points(points, target_func)

    return optimize_random


def optimize_discrete(space: DiscreteSearchSpace, target_func: TargetFunc) -> np.ndarray:
    """optimizer.py:153-193."""
    return _get_max_discrete_points(space.points[:, None, :], target_func)


def sample_from_space(num_samples: int, batch_size: Optional[int] = None, vectorization: int = 1):
    """optimizer.py:196-244: stream candidate chunks [<= batch_size, D]."""
    if num_samples <= 0:
        raise ValueError(f"num_samples must be positive, got {num_samples}")
    if batch_size is not None and batch_size <= 0:
        raise ValueError(f"batch_size must be positive, got {batch_size}")
    bs = batch_size or num_samples

    def sampler(space: SearchSpace) -> Iterator[np.ndarray]:
        for offset in range(0, num_samples, bs):
            yield space.sample(min(num_samples - offset, bs))

    return sampler


def _tile_samples(samples: np.ndarray, V: int, what: str) -> np.ndarray:
    """Samples [n, D] or, from a multi-region space, [n, S, D] -> [n, V, D]: column v holds a sample of subspace v mod S."""
    if samples.ndim == 3:
        if V % samples.shape[1] != 0:
            raise ValueError(
                f"The vectorization of the target function {V} must be a multiple of the batch shape of {what} "
                f"{samples.shape[1]}."
            )
        return np.tile(samples, [1, V // samples.shape[1], 1])
    if samples.ndim == 2:
        return np.tile(samples[:, None, :], [1, V, 1])
    raise ValueError(f"The {what} must be a tensor of rank 2, got a tensor of rank {samples.ndim}.")


def generate_initial_points(num_initial_points: int, initial_sampler, space: SearchSpace, target_func,
                            vectorization: int = 1) -> np.ndarray:
    """optimizer.py:247-341: running top-k of the acquisition values over the sampler's chunks.
    Returns [num_initial_points, V, D]."""
    from ..sampler import top_k

    top_vals = None  # [V, k]
    top_cands = None  # [V, k, D]
    V = vectorization
    for candidates in initial_sampler(space):
        tiled = _tile_samples(np.asarray(candidates), V, "initial samples")
        values = _to_numpy(target_func(tiled))  # [samples, V]
        if values.ndim != 2 or values.shape[-1] != V:
            raise ValueError(
                f"The result of function target_func has shape {values.shape}, however, expected a trailing dimension of size {V}."
            )
        cand_t = np.transpose(tiled, [1, 0, 2])  # [V, samples, D]
        vals_t = values.T  # [V, samples]
        if top_vals is None:
            all_vals, all_cands = vals_t, cand_t
        else:
            all_cands = np.concatenate([top_cands, cand_t], axis=1)
            all_vals = np.concatenate([top_vals, vals_t], axis=1)
        k = min(num_initial_points, all_vals.shape[-1])
        new_vals, new_cands = [], []
        for v in range(V):
            tv, ti = top_k(np.ascontiguousarray(all_vals[v]), k)  # bitonic top-k on the GPU
            new_vals.append(tv)
            new_cands.append(all_cands[v][ti])
        top_vals, top_cands = np.stack(new_vals), np.stack(new_cands)
    if top_cands is None:
        raise ValueError("No initial point generated!")
    return np.transpose(top_cands, [1, 0, 2])  # [k, V, D]


# ---------------------------------------------------------------------------------------------------
# vectorised projected L-BFGS (replaces greenlets + SciPy L-BFGS-B, optimizer.py:566-745)
# ---------------------------------------------------------------------------------------------------
def _value_and_gradient(fn, x: np.ndarray):
    """x [R, V, D] -> (values [R, V], grads [R, V, D]) of the function to MAXIMISE.  V = 1: an ordinary function
    ``[..., 1, D] -> [..., 1]``; V > 1: a vectorised one, ``[..., V, D] -> [..., V]`` (column v may be a different function,
    e.g. the per-column beta of the multiple-optimism LCB)."""
    if not hasattr(fn, "value_and_gradient"):
        raise NotImplementedError(
            "generate_continuous_optimizer needs an acquisition function with a value_and_gradient method "
            "(the reference differentiates through TensorFlow, optimizer.py:621-629)"
        )
    R, V, D = x.shape
    vals, grads = fn.value_and_gradient(x)
    return _to_numpy(vals).reshape(R, V), _to_numpy(grads).reshape(R, V, D)


def _perform_parallel_continuous_optimization(fn, lower, upper, starting_points: np.ndarray, optimizer_args: dict):
    """Maximise ``fn`` from every start [R, V, D], problem p = (r, v) = r * V + v inside box p mod nbox of ``lower`` /
    ``upper``: one box [D], one box per subspace of a multi-region space [nbox, D] with nbox dividing V (column v searches
    subspace v mod nbox, the reference's round robin, optimizer.py:859-890), or one box per problem [R * V, D].  Returns
    (success [R, V] bool, fun [R, V] (maximised values), x [R, V, D], nfev [R, V]).  The device optimisers take at most
    one box per column, so per-problem boxes need the host implementation (``TB_LBFGS=host``)."""
    m = int(optimizer_args.get("maxcor", 10))
    maxiter = int(optimizer_args.get("maxiter", 15000))
    gtol = float(optimizer_args.get("gtol", 1e-5))
    ftol = float(optimizer_args.get("ftol", 2.220446049250313e-09))
    maxls = int(optimizer_args.get("maxls", 20))

    R, V, D = starting_points.shape
    P = R * V
    boxes = [np.atleast_2d(np.asarray(b, dtype=np.float64)) for b in (lower, upper)]
    nbox = max(len(boxes[0]), len(boxes[1]))
    if V % nbox != 0 and nbox != P:
        raise ValueError(f"The vectorization of the target function {V} must be a multiple of the number of subspaces {nbox}.")
    lo_b, up_b = (np.broadcast_to(b, (nbox, D)) for b in boxes)
    if hasattr(fn, "maximize_from") and os.environ.get("TB_LBFGS", "device") != "host" and m <= 16:
        # the whole multi-start loop runs on the device: tb_acq_maximize for the fused single-model functions (starts
        # [P, D], one box), tb_rff_maximize_boxes for the negated trajectories of continuous Thompson sampling (starts
        # [R, V, D], column v in box v mod nbox)
        if V % nbox != 0:
            raise ValueError(
                f"{nbox} per-problem boxes for {V} columns: the device L-BFGS takes one box per column at most; set "
                "TB_LBFGS=host for one box per problem"
            )
        starts = starting_points.reshape(P, D) if V == 1 else starting_points
        lo_d, up_d = (lo_b[0], up_b[0]) if nbox == 1 else (lo_b, up_b)
        ok, fun, xs, nf = fn.maximize_from(starts, lo_d, up_d, maxcor=m, maxiter=maxiter, maxls=maxls, gtol=gtol, ftol=ftol)
        return ok.reshape(R, V), fun.reshape(R, V), xs.reshape(R, V, D), nf.reshape(R, V)
    box_of = np.arange(P) % nbox
    lower, upper = lo_b[box_of], up_b[box_of]  # [P, D]: the box of every problem
    x = np.clip(starting_points.reshape(P, D).astype(np.float64), lower, upper)

    def evaluate(idx, pts):
        """trial points ``pts`` [n, D] of the problems ``idx`` (flat (run, column) indices) -> (f [n], g [n, D]) of the
        NEGATED function (this routine minimises)"""
        if V == 1:
            v, g = _value_and_gradient(fn, pts.reshape(-1, 1, D))
            return -v.reshape(-1), -g.reshape(-1, D)
        # vectorised function: column v of the input selects the function, so evaluate the full [R, V, D] block with the
        # other problems held at their current iterates and read out the requested entries
        full = x.copy()
        full[idx] = pts
        v, g = _value_and_gradient(fn, full.reshape(R, V, D))
        return -v.reshape(-1)[idx], -g.reshape(-1, D)[idx]

    f, g = evaluate(np.arange(P), x)
    nfev = np.ones(P, dtype=np.int64)
    # shared ring buffer of curvature pairs; a slot with rho == 0 is a no-op for that problem
    S = np.zeros((m, P, D))
    Y = np.zeros((m, P, D))
    rho = np.zeros((m, P))
    gamma = np.ones(P)  # initial Hessian scaling s.y / y.y of the newest stored pair
    npairs = np.zeros(P, dtype=np.int64)
    head = 0
    done = ~np.isfinite(f)
    success = np.zeros(P, dtype=bool)

    def proj_grad(idx, xx, gg):
        return xx - np.clip(xx - gg, lower[idx], upper[idx])

    conv = np.max(np.abs(proj_grad(np.arange(P), x, g)), axis=1) <= gtol
    success |= conv & ~done
    done |= conv

    for it in range(maxiter):
        act = np.nonzero(~done)[0]
        if act.size == 0:
            break
        xa, ga = x[act], g[act]
        # free variables: not pinned at a bound with the gradient pushing outward
        free = ~(((xa <= lower[act]) & (ga > 0)) | ((xa >= upper[act]) & (ga < 0)))
        q = np.where(free, ga, 0.0)
        order = [(head - 1 - i) % m for i in range(m)]  # newest first
        alphas = []
        for slot in order:
            s_, y_ = S[slot, act] * free, Y[slot, act] * free
            a = rho[slot, act] * np.sum(s_ * q, axis=1)
            q = q - a[:, None] * y_
            alphas.append(a)
        r = gamma[act, None] * q
        for i in reversed(range(m)):  # oldest first
            slot = order[i]
            s_, y_ = S[slot, act] * free, Y[slot, act] * free
            beta = rho[slot, act] * np.sum(y_ * r, axis=1)
            r = r + s_ * (alphas[i] - beta)[:, None]
        d = -np.where(free, r, 0.0)
        gd = np.sum(ga * d, axis=1)
        bad = ~(gd < 0)  # not a descent direction: projected steepest descent instead
        if np.any(bad):
            d[bad] = -np.where(free[bad], ga[bad], 0.0)
        t = np.ones(act.size)
        first = npairs[act] == 0  # SciPy-like conservative first step
        nrm = np.sqrt(np.sum(d * d, axis=1))
        t[first] = np.minimum(1.0, 1.0 / np.maximum(nrm[first], 1e-300))

        # projected backtracking (Armijo) line search; each trial = one batched GPU evaluation
        fa = f[act]
        x_new, f_new, g_new = xa.copy(), fa.copy(), ga.copy()
        pending = nrm > 0
        accepted = np.zeros(act.size, dtype=bool)
        for _ls in range(maxls):
            pidx = np.nonzero(pending)[0]
            if pidx.size == 0:
                break
            xt = np.clip(xa[pidx] + t[pidx, None] * d[pidx], lower[act[pidx]], upper[act[pidx]])
            ft, gt = evaluate(act[pidx], xt)
            nfev[act[pidx]] += 1
            step = xt - xa[pidx]
            ok = np.isfinite(ft) & (ft <= fa[pidx] + 1e-4 * np.sum(ga[pidx] * step, axis=1))
            okidx = pidx[ok]
            x_new[okidx], f_new[okidx], g_new[okidx] = xt[ok], ft[ok], gt[ok]
            accepted[okidx] = True
            pending[okidx] = False
            t[pidx[~ok]] *= 0.5
        # a failed line search ends that run unsuccessfully (SciPy: ABNORMAL_TERMINATION_IN_LNSRCH);
        # a zero direction means the projected gradient vanished: converged
        zero_dir = nrm == 0
        success[act[zero_dir]] = True
        done[act[~accepted]] = True

        acc = np.nonzero(accepted)[0]
        ai = act[acc]
        s_new = x_new[acc] - xa[acc]
        y_new = g_new[acc] - ga[acc]
        sy_new = np.sum(s_new * y_new, axis=1)
        yy_new = np.sum(y_new * y_new, axis=1)
        store = sy_new > 1e-10 * yy_new
        S[head], Y[head], rho[head] = 0.0, 0.0, 0.0
        st = ai[store]
        S[head, st], Y[head, st], rho[head, st] = s_new[store], y_new[store], 1.0 / sy_new[store]
        gamma[st] = sy_new[store] / yy_new[store]
        npairs[st] += 1
        head = (head + 1) % m

        f_old = f[ai].copy()
        x[ai], f[ai], g[ai] = x_new[acc], f_new[acc], g_new[acc]
        conv_g = np.max(np.abs(proj_grad(ai, x[ai], g[ai])), axis=1) <= gtol
        conv_f = (f_old - f[ai]) <= ftol * np.maximum(np.maximum(np.abs(f_old), np.abs(f[ai])), 1.0)
        conv = conv_g | conv_f
        success[ai[conv]] = True
        done[ai[conv]] = True

    return success.reshape(R, V), (-f).reshape(R, V), x.reshape(R, V, D), nfev.reshape(R, V)


def generate_continuous_optimizer(num_initial_samples: int = NUM_SAMPLES_MIN, num_optimization_runs: int = 10,
                                  num_recovery_runs: int = 10, optimizer_args: Optional[dict] = None):
    """optimizer.py:344-563 for ``Box`` and ``TaggedMultiSearchSpace`` spaces: best ``num_optimization_runs`` of
    ``num_initial_samples`` random points -> parallel local maximisation -> argmax over runs;
    recovery runs from fresh random starts if every run failed; ``FailedOptimizationError``
    otherwise.  Over a multi-region space of S subspaces, column v of a function vectorised over V (a multiple of S)
    starts from and stays in subspace v mod S."""
    if num_initial_samples <= 0:
        raise ValueError(f"num_initial_samples must be positive, got {num_initial_samples}")
    if num_optimization_runs <= 0:
        raise ValueError(f"num_optimization_runs must be positive, got {num_optimization_runs}")
    if num_initial_samples < num_optimization_runs:
        raise ValueError(
            f"num_initial_samples {num_initial_samples} must be at least num_optimization_runs {num_optimization_runs}"
        )
    if num_recovery_runs < 0:
        raise ValueError(f"num_recovery_runs must be zero or greater, got {num_recovery_runs}")
    args = dict(optimizer_args or {})

    def optimize_continuous(space: SearchSpace, target_func: TargetFunc) -> np.ndarray:
        if not isinstance(space, (Box, TaggedMultiSearchSpace)):
            raise NotImplementedError("generate_continuous_optimizer here supports Box and TaggedMultiSearchSpace search spaces")
        fn, V = _split(target_func)
        initial = generate_initial_points(
            num_optimization_runs, sample_from_space(num_initial_samples), space, fn, vectorization=V
        )  # [runs, V, D]
        success, fun, xs, nfev = _perform_parallel_continuous_optimization(fn, space.lower, space.upper, initial, args)
        ok_any = np.any(success, axis=0)  # [V]
        total_nfev = int(np.max(nfev))
        recovery = 0
        while not np.all(ok_any) and recovery < num_recovery_runs:
            # optimizer.py:462-522: random restarts until some run succeeds for every function
            rnd = _tile_samples(space.sample(1), V, "random samples")
            s2, f2, x2, n2 = _perform_parallel_continuous_optimization(fn, space.lower, space.upper, rnd, args)
            success = np.concatenate([success, s2])
            fun = np.concatenate([fun, f2])
            xs = np.concatenate([xs, x2])
            ok_any = np.any(success, axis=0)
            total_nfev += int(np.max(n2))
            recovery += 1
        if not np.all(ok_any):
            raise FailedOptimizationError(
                f"Acquisition function optimization failed, even after {num_recovery_runs + num_optimization_runs} restarts."
            )
        # optimizer.py:556-559: argmax over the values of ALL runs (``successes`` only decides recovery / failure above);
        # non-finite values never win
        finite = np.where(np.isfinite(fun), fun, -np.inf)
        best = np.argmax(finite, axis=0)  # [V]

        def improvement():
            """optimizer.py:546-549 (evaluated only when asked for: the reference computes it under a summary writer)"""
            init = _to_numpy(fn(initial if V > 1 else initial.reshape(-1, 1, initial.shape[-1]))).reshape(-1, V)
            imp = np.max(finite, axis=0) - np.max(init, axis=0)
            return float(imp[0]) if V == 1 else imp

        optimize_continuous.last_stats = {"spo_af_evaluations": total_nfev, "spo_improvement_on_initial_samples": improvement}
        return np.stack([xs[best[v], v, :] for v in range(V)], axis=0)

    return optimize_continuous


def batchify_joint(batch_size_one_optimizer, batch_size: int):
    """optimizer.py:897-936: optimise q points jointly over ``space ** q``; the function sees
    [..., 1, q*D] reshaped to [..., q, D]."""
    if batch_size <= 0:
        raise ValueError(f"batch_size must be positive, got {batch_size}")

    def optimizer(space: SearchSpace, f: TargetFunc) -> np.ndarray:
        fn, V = _split(f)
        if V != 1:
            raise ValueError("batchify_joint does not support vectorised acquisition functions")
        expanded = space**batch_size

        class _Expanded:
            """``fn`` seen through ``space ** q``: [..., 1, q*D] <-> [..., q, D] (values and, when the function offers
            them, gradients — the reference differentiates through the reshape)."""

            def __call__(self, x):
                x = _to_numpy(x)
                return fn(x.reshape(x.shape[:-2] + (batch_size, -1)))

            if hasattr(fn, "value_and_gradient"):

                def value_and_gradient(self, x):
                    x = _to_numpy(x)
                    val, grad = fn.value_and_gradient(x.reshape(x.shape[:-2] + (batch_size, -1)))
                    return val, _to_numpy(grad).reshape(x.shape)

        target_on_expanded = _Expanded()
        vectorized_points = batch_size_one_optimizer(expanded, target_on_expanded)  # [1, q*D]
        return vectorized_points.reshape(batch_size, -1)

    return optimizer


def batchify_vectorize(batch_size_one_optimizer, batch_size: int):
    """optimizer.py:939-970: for functions whose batch elements can be optimised independently (vectorised functions,
    ``[..., B, D] -> [..., B]``): the batch-size-one optimiser is asked for ``batch_size`` independent maximisers."""
    if batch_size <= 0:
        raise ValueError(f"batch_size must be positive, got {batch_size}")

    def optimizer(space: SearchSpace, f: TargetFunc) -> np.ndarray:
        if isinstance(f, tuple):
            raise ValueError("batchify_vectorize cannot be applied to an already vectorized acquisition function")
        return batch_size_one_optimizer(space, (f, batch_size))

    return optimizer


def automatic_optimizer_selector(space: SearchSpace, target_func: TargetFunc) -> np.ndarray:
    """optimizer.py:90-121."""
    if isinstance(space, DiscreteSearchSpace):
        return optimize_discrete(space, target_func)
    if isinstance(space, (Box, TaggedMultiSearchSpace)):
        num_samples = max(NUM_SAMPLES_MIN, NUM_SAMPLES_DIM * space.dimension)
        num_runs = NUM_RUNS_DIM * space.dimension
        return generate_continuous_optimizer(num_initial_samples=num_samples, num_optimization_runs=num_runs)(space, target_func)
    raise NotImplementedError(f"No optimizer currently supports acquisition function maximisation over search spaces of type {space}.")
