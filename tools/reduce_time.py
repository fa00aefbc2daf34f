"""What the fused route of a reducer saves against the composed route on the same children: Product(EI on an objective
GP, PoF on a constraint GP), both GPs of N points in D dimensions (N in {1024, 4096}, D in {6, 10}).  The composed route
is forced by wrapping the EI child in a plain callable.  Timings, medians of alternated calls after one warm-up each:

  argmax   the first-max over 2^20 uniform candidates: the fused tb_reduce_argmax against the composed route's two
           single-model evaluations, product and host argmax (what _get_max_discrete_points does for a function without
           fused_argmax); beside them the sum of the two members' own unscreened single-model fused argmaxes.
  acquire  a whole generate_continuous_optimizer acquire (initial samples, top-k, L-BFGS): the fused route's device
           L-BFGS (maximize_from) against the composed route's host L-BFGS; the values reached are printed.

The card name, power limit and maximum SM clock are read in the same run and printed with the numbers.

    python tools/reduce_time.py [--reps 5] [--out FILE]     (prints one JSON line per shape)
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

NS, DS, M = (1024, 4096), (6, 10), 1 << 20


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


class _Plain:
    def __init__(self, f):
        self.f = f

    def __call__(self, x):
        return self.f(x)

    def value_and_gradient(self, x):
        return self.f.value_and_gradient(x)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed repeats of each measurement")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()

    import __graft_entry__ as g

    g.build()
    from oracle import gp_oracle as o
    from tests.util import model_pair
    from trieste_b200.acquisition import expected_improvement, probability_below_threshold
    from trieste_b200.acquisition.combination import REDUCE_PRODUCT, Product, reduce_functions, reduced_acquisition
    from trieste_b200.acquisition.optimizer import _get_max_discrete_points, generate_continuous_optimizer
    import trieste_b200 as tb

    info = card()
    med = lambda v: float(np.median(v))  # noqa: E731
    lines = []
    for D in DS:
        space = tb.Box([0.0] * D, [1.0] * D)
        for N in NS:
            o0, n0 = model_pair(lambda x: o.random_fourier_objective(x, seed=2), N, D, seed=0)
            o1, n1 = model_pair(lambda x: o.random_fourier_objective(x, seed=3), N, D, seed=1)
            ei, pof = expected_improvement(n0, o.ei_eta(o0)), probability_below_threshold(n1, 0.0)
            fused = reduced_acquisition(REDUCE_PRODUCT, [ei, pof])
            red = Product(object())
            composed = reduce_functions(REDUCE_PRODUCT, red._reduce, [_Plain(ei), pof])
            assert not isinstance(composed, reduced_acquisition)
            pts = np.random.default_rng(N + D).uniform(size=(M, D))
            os.environ["TB_ARGMAX_SCREEN"] = "0"  # the members' own argmaxes unscreened, as the reduction's

            def singles():
                ei.fused_argmax(pts)
                pof.fused_argmax(pts)

            runs = {"fused": lambda: fused.fused_argmax(pts), "composed": lambda: _get_max_discrete_points(pts[:, None, :], composed),
                    "members": singles}
            times = {k: [] for k in runs}
            for k in runs:
                runs[k]()
            for _ in range(args.reps):
                for k, f in runs.items():
                    t0 = time.perf_counter()
                    f()
                    times[k].append(time.perf_counter() - t0)
            idx_f = fused.fused_argmax(pts)[0]
            idx_c = int(np.argmax(np.asarray(composed(pts[:, None, :]))[:, 0]))
            opt = generate_continuous_optimizer(num_initial_samples=1000, num_optimization_runs=10)
            acq_t = {"fused": [], "composed": []}
            acq_v = {}
            for k, fn in (("fused", fused), ("composed", composed)):
                space._rng = np.random.default_rng(0)
                opt(space, fn)  # warm-up
            for _ in range(args.reps):
                for k, fn in (("fused", fused), ("composed", composed)):
                    space._rng = np.random.default_rng(0)
                    t0 = time.perf_counter()
                    x = opt(space, fn)
                    acq_t[k].append(time.perf_counter() - t0)
                    acq_v[k] = float(np.asarray(fused(np.asarray(x)[:, None, :]))[0, 0])
            line = dict(info, N=N, D=D, M=M, argmax_fused_ms=1e3 * med(times["fused"]),
                        argmax_composed_ms=1e3 * med(times["composed"]), argmax_members_ms=1e3 * med(times["members"]),
                        argmax_same_index=bool(idx_f == idx_c), acquire_fused_ms=1e3 * med(acq_t["fused"]),
                        acquire_composed_ms=1e3 * med(acq_t["composed"]), acquire_value_fused=acq_v["fused"],
                        acquire_value_composed=acq_v["composed"])
            print(json.dumps(line), flush=True)
            lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(x) for x in lines) + "\n")


if __name__ == "__main__":
    main()
