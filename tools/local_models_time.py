"""What the batched local-model route of BatchTrustRegionBox saves: S regions, each with its own local GPR of N points,
maximised in one device L-BFGS over all regions (tb_acq_maximize_models / tb_rff_maximize_models) against the per-region loop
of the existing entries (tb_acq_maximize / tb_rff_maximize_boxes, one region after another).

Shapes: S in {3, 8} SingleObjectiveTrustRegionBox regions (zeta 0.1, random centres), local N in {50, 1000} (Ackley-D data
inside each region), D in {6, 10}; base rules EfficientGlobalOptimization(ExpectedImprovement()) and
EfficientGlobalOptimization(ParallelContinuousThompsonSampling(), num_query_points=2).  Two timings per shape, both medians
of alternated calls after one warm-up each:

  lbfgs    the multi-start L-BFGS alone from the same starts (10 D per column, uniform in each region): one
           _RegionStack.maximize_from against each region's function's maximize_from in turn; the results are checked to
           be bit-identical.
  acquire  the acquisition's optimisation as BatchTrustRegionBox runs it (the automatic continuous optimiser: initial
           samples, top-k and L-BFGS) over the TaggedMultiSearchSpace of the regions with the stacked function, against each
           region's copy of the base rule optimising its own function inside its region.

The card name, power limit and maximum SM clock are read in the same run and printed with the numbers.

    python tools/local_models_time.py [--reps 5] [--out FILE]     (prints one JSON line per shape)
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

SS, NS, DS, KINDS = (3, 8), (50, 1000), (6, 10), ("ei", "pcts")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="timed repeats of each measurement")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()

    import __graft_entry__ as g

    g.build()
    import trieste_b200 as tb
    from trieste_b200.acquisition import ExpectedImprovement, ParallelContinuousThompsonSampling
    from trieste_b200.objectives import ackley
    from trieste_b200.rule import EfficientGlobalOptimization, SingleObjectiveTrustRegionBox, _RegionStack
    from trieste_b200.space import TaggedMultiSearchSpace

    info = card()
    med = lambda v: float(np.median(v))  # noqa: E731
    lines = []
    for D in DS:
        space = tb.Box([0.0] * D, [1.0] * D)
        for S in SS:
            rng = np.random.default_rng(100 * D + S)
            regions = []
            for i in range(S):
                region = SingleObjectiveTrustRegionBox(space, zeta=0.1, region_index=i)
                region.initialize(location_candidate=rng.uniform(0.1, 0.9, size=D))
                regions.append(region)
            lo = np.stack([r.lower for r in regions])
            up = np.stack([r.upper for r in regions])
            for N in NS:
                models, data = [], []
                for r in regions:  # each region's local data lies inside it
                    X = rng.uniform(r.lower, r.upper, size=(N, D))
                    ds = tb.Dataset(X, ackley(X))
                    models.append(tb.GaussianProcessRegression(tb.build_gpr(ds, space)))
                    data.append(ds)
                for kind in KINDS:
                    k = 1 if kind == "ei" else 2
                    rules = [EfficientGlobalOptimization(ExpectedImprovement()) if kind == "ei" else
                             EfficientGlobalOptimization(ParallelContinuousThompsonSampling(), num_query_points=k)
                             for _ in range(S)]
                    fns = [rule._builder.prepare_acquisition_function({"OBJECTIVE": m}, datasets={"OBJECTIVE": d})
                           for rule, m, d in zip(rules, models, data)]
                    if kind == "pcts":
                        for fn in fns:
                            fn(np.zeros((1, k, D)))  # fixes the batch size
                    stack = _RegionStack.of(fns, k)
                    assert stack is not None
                    R = 10 * D
                    starts = rng.uniform(lo, up, size=(R, k, S, D)).reshape(R, k * S, D)  # column v in region v mod S

                    def lbfgs_batched():
                        return stack.maximize_from(starts, lo, up)

                    def lbfgs_loop():
                        outs = []
                        for s, fn in enumerate(fns):
                            x0 = starts[:, s::S] if kind == "pcts" else starts[:, s]
                            outs.append(fn.maximize_from(x0, lo[s], up[s]))
                        return outs

                    b, loop = lbfgs_batched(), lbfgs_loop()
                    for s in range(S):  # the same problems, bit for bit
                        xs = loop[s][2] if kind == "pcts" else loop[s][2][:, None, :]
                        assert np.array_equal(b[2][:, s::S], xs), (D, S, N, kind, s)

                    space_multi = TaggedMultiSearchSpace(regions)

                    def acquire_batched():
                        return rules[0]._base_optimizer(space_multi, (stack, k * S))

                    def acquire_loop():
                        return [rule._optimizer(region, fn) for rule, region, fn in zip(rules, regions, fns)]

                    def timed(f):
                        t0 = time.perf_counter()
                        f()  # every path ends in a device-to-host read of its results
                        return time.perf_counter() - t0

                    row = dict(info, D=D, S=S, N=N, acquisition=kind, k=k, starts_per_column=R)
                    for what, fb, fl in (("lbfgs", lbfgs_batched, lbfgs_loop), ("acquire", acquire_batched, acquire_loop)):
                        timed(fb)
                        timed(fl)
                        tb_, tl = [], []
                        for _ in range(args.reps):
                            tb_.append(timed(fb))
                            tl.append(timed(fl))
                        row.update({f"{what}_batched_s": med(tb_), f"{what}_loop_s": med(tl),
                                    f"{what}_loop_over_batched": med(tl) / med(tb_)})
                    line = json.dumps(row)
                    print(line, flush=True)
                    lines.append(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
