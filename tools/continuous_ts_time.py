"""What continuous Thompson sampling costs, at B in {10, 100} query points, N in {1024, 4096} training points and
D in {6, 10} (Ackley-D data, the model's default decoupled trajectories with 1000 features):

  (a) one EfficientGlobalOptimization(ParallelContinuousThompsonSampling(), num_query_points=B).acquire with the continuous
      optimiser (2000 initial samples, 5 runs per trajectory): the device L-BFGS (tb_rff_maximize) against the host
      implementation of the same algorithm (TB_LBFGS=host), median of the timed acquires after one warm-up each, alternated;
  (b) the paired evaluation of M = 1000 points [M, B, D], each under its own trajectory (tb_rff_eval_paired, one launch),
      against the per-column loop it replaces (B calls of tb_rff_eval, each evaluating all B trajectories), median time,
      alternated, with the two results compared bit for bit.

The card name and power limit are read in the same run and printed with the numbers.

    python tools/continuous_ts_time.py [--reps 3] [--out FILE]     (prints one JSON line per shape)
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

BS, NS, DS, M = (10, 100), (1024, 4096), (6, 10), 1000


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
    from trieste_b200 import _lib
    from trieste_b200.acquisition import ParallelContinuousThompsonSampling
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.acquisition.optimizer import generate_continuous_optimizer
    from trieste_b200.objectives import ackley
    from trieste_b200.rule import EfficientGlobalOptimization

    info = card()
    med = lambda v: float(np.median(v))  # noqa: E731
    lines = []
    for N in NS:
        for D in DS:
            rng = np.random.default_rng(N + D)
            X = rng.uniform(size=(N, D))
            ds = tb.Dataset(X, ackley(X))
            space = tb.Box([0.0] * D, [1.0] * D)
            model = tb.GaussianProcessRegression(tb.build_gpr(ds, space))
            for B in BS:
                opt = generate_continuous_optimizer(num_initial_samples=2000, num_optimization_runs=5)
                rule = EfficientGlobalOptimization(ParallelContinuousThompsonSampling(), optimizer=opt, num_query_points=B)

                def acquire(host: bool):
                    if host:
                        os.environ["TB_LBFGS"] = "host"
                    try:
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        pts = rule.acquire(space, {OBJECTIVE: model}, {OBJECTIVE: ds})
                        torch.cuda.synchronize()
                        assert pts.shape == (B, D)
                        return time.perf_counter() - t0
                    finally:
                        os.environ.pop("TB_LBFGS", None)

                acquire(False)
                acquire(True)
                t_dev, t_host = [], []
                for _ in range(args.reps):
                    t_dev.append(acquire(False))
                    t_host.append(acquire(True))

                # (b) paired evaluation against the per-column loop, on the rule's trajectory
                traj = rule.acquisition_function
                Xq = np.ascontiguousarray(rng.uniform(size=(M, B, D)))
                cols = [np.ascontiguousarray(Xq[:, b, :]) for b in range(B)]

                def paired():
                    out = np.empty((M, B))
                    t0 = time.perf_counter()
                    _lib.check(_lib.lib().tb_rff_eval_paired(traj._h, Xq.ctypes.data, M, B, out.ctypes.data, None))
                    return time.perf_counter() - t0, out

                def per_column():
                    out = np.empty((M, B))
                    tmp = np.empty((M, B))
                    t0 = time.perf_counter()
                    for b in range(B):
                        _lib.check(_lib.lib().tb_rff_eval(traj._h, cols[b].ctypes.data, M, tmp.ctypes.data, None, None))
                        out[:, b] = tmp[:, b]
                    return time.perf_counter() - t0, out

                paired()
                per_column()
                t_pair, t_col = [], []
                for _ in range(args.reps):
                    dt, a = paired()
                    t_pair.append(dt)
                    dt, c = per_column()
                    t_col.append(dt)
                row = dict(info, N=N, D=D, B=B, acquire_device_s=med(t_dev), acquire_host_s=med(t_host),
                           acquire_device_all_s=t_dev, acquire_host_all_s=t_host, acquire_host_over_device=med(t_host) / med(t_dev),
                           eval_points=M, eval_paired_s=med(t_pair), eval_per_column_s=med(t_col),
                           eval_per_column_over_paired=med(t_col) / med(t_pair), eval_bit_identical=bool(np.array_equal(a, c)))
                line = json.dumps(row)
                print(line, flush=True)
                lines.append(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
