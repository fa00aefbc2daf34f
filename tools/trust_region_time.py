"""What one batch trust-region acquire costs: BatchTrustRegionBox over S in {3, 8} SingleObjectiveTrustRegionBox regions
with EfficientGlobalOptimization(ParallelContinuousThompsonSampling(), num_query_points=S) (one trajectory per region),
D in {6, 20}, N = 1024 training points (Ackley-D data, the model's default decoupled trajectories with 1000 features), the
continuous optimiser with 2000 initial samples and 5 runs per trajectory over the TaggedMultiSearchSpace of the regions.
The device L-BFGS with per-region boxes (tb_rff_maximize_boxes) is timed against the host implementation of the same
algorithm (TB_LBFGS=host): median of the timed acquires after one warm-up each, alternated.  One rule.acquire initialises
the regions; the timed calls then run the base rule over the TaggedMultiSearchSpace of those frozen regions, so every repeat
searches the same boxes (a rule.acquire would first update the regions, and on an unchanged dataset each update is a
failed step that shrinks them).

The card name, power limit and maximum SM clock are read in the same run and printed with the numbers.

    python tools/trust_region_time.py [--reps 3] [--out FILE]     (prints one JSON line per shape)
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

SS, DS, N = (3, 8), (6, 20), 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3, help="timed repeats of each measurement")
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    import torch

    import __graft_entry__ as g

    g.build()
    import trieste_b200 as tb
    from trieste_b200.acquisition import ParallelContinuousThompsonSampling
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.acquisition.optimizer import generate_continuous_optimizer
    from trieste_b200.objectives import ackley
    from trieste_b200.rule import BatchTrustRegionBox, EfficientGlobalOptimization, SingleObjectiveTrustRegionBox
    from trieste_b200.space import TaggedMultiSearchSpace

    info = card()
    med = lambda v: float(np.median(v))  # noqa: E731
    lines = []
    for D in DS:
        rng = np.random.default_rng(D)
        X = rng.uniform(size=(N, D))
        ds = tb.Dataset(X, ackley(X))
        space = tb.Box([0.0] * D, [1.0] * D)
        model = tb.GaussianProcessRegression(tb.build_gpr(ds, space))
        for S in SS:
            opt = generate_continuous_optimizer(num_initial_samples=2000, num_optimization_runs=5)
            base = EfficientGlobalOptimization(ParallelContinuousThompsonSampling(), optimizer=opt, num_query_points=S)
            rule = BatchTrustRegionBox([SingleObjectiveTrustRegionBox(space) for _ in range(S)], base)
            rule.acquire(space, {OBJECTIVE: model}, {OBJECTIVE: ds})  # initialises the regions
            regions = rule.subspaces
            frozen = TaggedMultiSearchSpace(regions)

            def acquire(host: bool):
                if host:
                    os.environ["TB_LBFGS"] = "host"
                try:
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    pts = base.acquire(frozen, {OBJECTIVE: model}, {OBJECTIVE: ds})
                    torch.cuda.synchronize()
                    assert pts.shape == (S, D)
                    assert all(regions[s].contains(pts[s]) for s in range(S))
                    return time.perf_counter() - t0
                finally:
                    os.environ.pop("TB_LBFGS", None)

            acquire(False)
            acquire(True)
            t_dev, t_host = [], []
            for _ in range(args.reps):
                t_dev.append(acquire(False))
                t_host.append(acquire(True))
            row = dict(info, N=N, D=D, S=S, acquire_device_s=med(t_dev), acquire_host_s=med(t_host),
                       acquire_device_all_s=t_dev, acquire_host_all_s=t_host, acquire_host_over_device=med(t_host) / med(t_dev))
            line = json.dumps(row)
            print(line, flush=True)
            lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
