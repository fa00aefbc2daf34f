"""What HIPPO's penalty costs on the device: N = 1024 training points, D = 6, DTLZ2 with L = 2 and 3 objectives (one native
GPR per objective), M = 10^6 candidates on the device.

  (a) the fused argmax of the penalised EHVI (hippo_penalized_ehvi.fused_argmax, tb_ehvi_argmax with the penalty set) with
      P = 1, 3 and 15 pending points, against the plain EHVI argmax on the same handle;
  (b) one EfficientGlobalOptimization(HIPPO(), num_query_points=4).acquire over the box with the continuous optimiser: one
      plain EHVI step and three penalised greedy steps, their L-BFGS on the device against the host L-BFGS (TB_LBFGS=host).

(a) is the median over --reps calls of each variant, alternated in one loop; (b) the median of --acquires acquires after one
warm-up each.  The card name, power limit and max SM clock are read in the same run and printed with the numbers.

    python tools/hippo_time.py [--reps 5] [--acquires 3] [--out FILE]     (prints one JSON line)
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

N, D, M = 1024, 6, 1_000_000
PENDING = (1, 3, 15)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def timed(f):
    t0 = time.perf_counter()
    f()  # every ABI call ends in a device synchronise
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--acquires", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import __graft_entry__ as g

    g.build()
    import trieste_b200 as tb
    from trieste_b200.acquisition import HIPPO, ExpectedHypervolumeImprovement, hippo_penalized_ehvi, hippo_penalizer
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.objectives import dtlz2
    from trieste_b200.rule import EfficientGlobalOptimization

    out = {"what": "HIPPO penalised EHVI fused argmax vs plain EHVI / HIPPO q=4 acquire", "N": N, "D": D, "M": M,
           "pending": list(PENDING), "reps": args.reps, "acquires": args.acquires, **card()}
    rng = np.random.default_rng(0)
    X = rng.uniform(size=(N, D))
    space = tb.Box([0.0] * D, [1.0] * D)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    xc = torch.rand(M, D, dtype=torch.float64, device="cuda", generator=gen)
    for L in (2, 3):
        Y = dtlz2(X, L, D)
        members = [tb.GaussianProcessRegression(tb.build_gpr(tb.Dataset(X, Y[:, l:l + 1]), space)) for l in range(L)]
        stack = tb.TrainableModelStack(*[(m, 1) for m in members])
        ds = tb.Dataset(X, Y)
        base = ExpectedHypervolumeImprovement().prepare_acquisition_function(stack, ds)
        row = {"K": int(base.partition_bounds[0].shape[0]), "engines": [m.engine_info()[0] for m in members]}
        variants = {"plain": base}
        for P in PENDING:
            variants[f"P{P}"] = hippo_penalized_ehvi(base, hippo_penalizer(stack, rng.uniform(size=(P, D))))
        for fn in variants.values():
            fn.fused_argmax(xc)
        times = {k: [] for k in variants}
        for _ in range(args.reps):
            for k, fn in variants.items():
                times[k].append(timed(lambda: fn.fused_argmax(xc)))
        for k in variants:
            row[f"fused_argmax_{k}_ms"] = float(np.median(times[k]))
        for mode in ("device", "host"):
            os.environ["TB_LBFGS"] = mode
            rule = EfficientGlobalOptimization(HIPPO(), num_query_points=4)
            rule.acquire(space, {OBJECTIVE: stack}, {OBJECTIVE: ds})
            ts = [timed(lambda: rule.acquire(space, {OBJECTIVE: stack}, {OBJECTIVE: ds})) for _ in range(args.acquires)]
            row[f"acquire_q4_{mode}_lbfgs_ms"] = float(np.median(ts))
        os.environ.pop("TB_LBFGS", None)
        out[f"L{L}"] = row
    line = json.dumps(out)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
