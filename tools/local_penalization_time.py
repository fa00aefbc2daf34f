"""What local penalisation costs on the headline workload (N = 4096, D = 10, Ackley-10, 1,216,512 candidates on the device):

  (a) EI fused argmax, plain against penalised by P = 7 pending points (soft penaliser): median time per call, the two
      alternated call by call;
  (b) one q = 8 EfficientGlobalOptimization.acquire with a random search over the same candidates, LocalPenalization
      against Fantasizer (kriging believer): median of the timed acquires after one warm-up acquire each, alternated.

The card name and power limit are read in the same run and printed with the numbers.

    python tools/local_penalization_time.py [--reps 7] [--acquires 3] [--out FILE]     (prints one JSON line)
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

N, D, M, P, Q = 4096, 10, 1_216_512, 7, 8


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
    from trieste_b200.acquisition import (ExpectedImprovement, Fantasizer, LocalPenalization, PenalizedAcquisition,
                                          soft_local_penalizer)
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.objectives import ackley
    from trieste_b200.rule import EfficientGlobalOptimization

    info = card()
    rng = np.random.default_rng(0)
    X = rng.uniform(size=(N, D))
    ds = tb.Dataset(X, ackley(X))
    space = tb.Box([0.0] * D, [1.0] * D)
    model = tb.GaussianProcessRegression(tb.build_gpr(ds, space))
    ei = ExpectedImprovement().prepare_acquisition_function(model, ds)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    xc = torch.rand(M, D, dtype=torch.float64, device="cuda", generator=gen)

    # ---- (a) plain against penalised fused argmax ----
    lip = np.concatenate([X, space.sample(500, seed=2)])
    mean, grad = model.mean_gradient(lip)
    L, eta = float(np.linalg.norm(grad, axis=1).max()), float(mean.min())
    pen = PenalizedAcquisition(ei, soft_local_penalizer(model, space.sample(P, seed=3), L, eta))

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn.fused_argmax(xc)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    for fn in (ei, pen, ei, pen):  # warm-up
        timed(fn)
    t_plain, t_pen = [], []
    for _ in range(args.reps):
        t_plain.append(timed(ei)[0])
        t_pen.append(timed(pen)[0])
    best_plain, best_pen = timed(ei)[1], timed(pen)[1]

    # ---- (b) one q = 8 acquire: LocalPenalization against Fantasizer ----
    def random_search(space_, fn):
        idx, _ = fn.fused_argmax(xc)
        return xc[idx:idx + 1].cpu().numpy()

    rules = {
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

    for name in rules:  # warm-up: the Fantasizer builds its second handle here
        acquire(name)
    for _ in range(args.acquires):
        for name in rules:
            times[name].append(acquire(name))
    for name, pts in batches.items():
        assert pts.shape == (Q, D), name

    med = lambda v: float(np.median(v))  # noqa: E731
    row = dict(info, N=N, D=D, candidates=M, pending=P,
               argmax_plain_s=med(t_plain), argmax_penalised_s=med(t_pen),
               argmax_plain_spread=[float(min(t_plain)), float(max(t_plain))],
               argmax_penalised_spread=[float(min(t_pen)), float(max(t_pen))],
               penalised_over_plain=med(t_pen) / med(t_plain),
               best_plain=[best_plain[0], best_plain[1]], best_penalised=[best_pen[0], best_pen[1]],
               q=Q, acquire_lp_s=med(times["local_penalization"]), acquire_fantasizer_s=med(times["fantasizer"]),
               acquire_lp_all_s=times["local_penalization"], acquire_fantasizer_all_s=times["fantasizer"],
               # a pending point whose mean is below eta has a negative radius and barely penalises itself (as in the
               # reference), so a batch may repeat a candidate
               distinct_lp=len({tuple(p) for p in batches["local_penalization"]}),
               distinct_fantasizer=len({tuple(p) for p in batches["fantasizer"]}),
               lipschitz_constant=L, eta=eta)
    line = json.dumps(row)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
