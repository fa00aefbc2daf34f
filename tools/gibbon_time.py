"""What GIBBON costs on the headline workload (N = 4096, D = 10, Ackley-10, 1,216,512 candidates on the device):

  (a) fused argmax of MES, of GIBBON's quality term and of GIBBON with m = 1, 7 and 32 pending points (the same five
      min-value samples throughout): median time per call, the functions alternated call by call;
  (b) one q = 8 EfficientGlobalOptimization.acquire with a random search over the same candidates, GIBBON against
      LocalPenalization and Fantasizer (kriging believer): median of the timed acquires after one warm-up acquire each,
      alternated.

The card name and power limit are read in the same run and printed with the numbers.

    python tools/gibbon_time.py [--reps 7] [--acquires 3] [--out FILE]     (prints one JSON line)
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

N, D, M, Q, S = 4096, 10, 1_216_512, 8, 5
PENDING = (1, 7, 32)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7, help="(a): timed calls of each function")
    ap.add_argument("--acquires", type=int, default=3, help="(b): timed acquires of each rule")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch

    import __graft_entry__ as g

    g.build()
    import trieste_b200 as tb
    from trieste_b200.acquisition import (GIBBON, Fantasizer, GibbonAcquisition, LocalPenalization, gibbon_quality_term,
                                          gibbon_repulsion_term, min_value_entropy_search)
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.objectives import ackley
    from trieste_b200.rule import EfficientGlobalOptimization

    info = card()
    rng = np.random.default_rng(0)
    X = rng.uniform(size=(N, D))
    ds = tb.Dataset(X, ackley(X))
    space = tb.Box([0.0] * D, [1.0] * D)
    model = tb.GaussianProcessRegression(tb.build_gpr(ds, space))
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    xc = torch.rand(M, D, dtype=torch.float64, device="cuda", generator=gen)

    # ---- (a) fused argmax: MES, quality term, GIBBON with m pending points ----
    y = np.asarray(ds.observations)
    samples = y.min() - np.abs(rng.normal(size=(S, 1))) * y.std()
    quality = gibbon_quality_term(model, samples)
    fns = {"mes": min_value_entropy_search(model, samples), "quality": quality}
    for m in PENDING:
        fns[f"gibbon_m{m}"] = GibbonAcquisition(quality, gibbon_repulsion_term(model, space.sample(m, seed=10 + m)))

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn.fused_argmax(xc)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    # the GIBBON functions share the model: each call pushes its own pending set, so alternating them rebuilds W and L_B^-1;
    # time each one in a block of repeats after one warm-up call, and alternate the blocks
    t = {k: [] for k in fns}
    best = {}
    for k, fn in fns.items():
        timed(fn)
    for _ in range(args.reps):
        for k, fn in fns.items():
            timed(fn)  # brings the handle state to this function
            dt, best[k] = timed(fn)
            t[k].append(dt)

    # ---- (b) one q = 8 acquire: GIBBON against LocalPenalization and Fantasizer ----
    def random_search(space_, fn):
        idx, _ = fn.fused_argmax(xc)
        return xc[idx:idx + 1].cpu().numpy()

    rules = {
        "gibbon": EfficientGlobalOptimization(GIBBON(space, seed=0), optimizer=random_search, num_query_points=Q),
        "local_penalization": EfficientGlobalOptimization(LocalPenalization(space), optimizer=random_search, num_query_points=Q),
        "fantasizer": EfficientGlobalOptimization(Fantasizer(), optimizer=random_search, num_query_points=Q),
    }
    times = {k: [] for k in rules}
    batches = {}

    def acquire(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        pts = rules[name].acquire(space, {OBJECTIVE: model}, {OBJECTIVE: ds})
        torch.cuda.synchronize()
        batches[name] = pts
        return time.perf_counter() - t0

    for name in rules:
        acquire(name)
    for _ in range(args.acquires):
        for name in rules:
            times[name].append(acquire(name))
    for name, pts in batches.items():
        assert pts.shape == (Q, D), name

    med = lambda v: float(np.median(v))  # noqa: E731
    row = dict(info, N=N, D=D, candidates=M, samples=S)
    for k, v in t.items():
        row[f"argmax_{k}_s"] = med(v)
        row[f"argmax_{k}_spread"] = [float(min(v)), float(max(v))]
        row[f"argmax_{k}_over_mes"] = med(v) / med(t["mes"])
        row[f"best_{k}"] = [best[k][0], best[k][1]]
    row.update(q=Q, **{f"acquire_{k}_s": med(v) for k, v in times.items()}, **{f"acquire_{k}_all_s": v for k, v in times.items()},
               **{f"distinct_{k}": len({tuple(p) for p in batches[k]}) for k in batches})
    line = json.dumps(row)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
