"""What the active-learning acquisitions cost on the headline workload (N = 4096, D = 10, Ackley-10, 1,216,512 candidates on
the device):

  (a) fused argmax of the bichon and ranjan criteria, BALD and the single-query predictive variance against the
      probability below a threshold (PBT, the existing unscreened tail of the same shape): median time per call, the
      functions alternated call by call;
  (b) value + gradient of the q-batch predictive variance against batch Monte-Carlo EI (S = 64 base samples) at equal B
      and q (q = 4 and 8, B * q = 65,536 points): median time per call, alternated.

The card name and power limit are read in the same run and printed with the numbers.

    python tools/active_learning_time.py [--reps 9] [--out FILE]     (prints one JSON line)
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

N, D, M, S, PTS = 4096, 10, 1_216_512, 64, 65_536


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9, help="timed calls of each function")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch

    import __graft_entry__ as g

    g.build()
    import trieste_b200 as tb
    from trieste_b200.acquisition import (BatchMonteCarloExpectedImprovement, bayesian_active_learning_by_disagreement,
                                          bichon_ranjan_criterion, predictive_variance, probability_below_threshold)
    from trieste_b200.objectives import ackley

    info = card()
    rng = np.random.default_rng(0)
    X = rng.uniform(size=(N, D))
    ds = tb.Dataset(X, ackley(X))
    space = tb.Box([0.0] * D, [1.0] * D)
    model = tb.GaussianProcessRegression(tb.build_gpr(ds, space))
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    xc = torch.rand(M, D, dtype=torch.float64, device="cuda", generator=gen)
    T = float(np.median(np.asarray(ds.observations)))

    def timed(call):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        call()
        torch.cuda.synchronize()
        return time.perf_counter() - t0

    # ---- (a) fused argmax against PBT ----
    fns = {
        "pbt": probability_below_threshold(model, T),
        "bichon": bichon_ranjan_criterion(model, T, 1.0, 1),
        "ranjan": bichon_ranjan_criterion(model, T, 1.0, 2),
        "bald": bayesian_active_learning_by_disagreement(model, 1e-6),
        "predictive_variance": predictive_variance(model, 1e-6),
    }
    argmax_t = {k: [] for k in fns}
    for fn in fns.values():
        fn.fused_argmax(xc)
    for _ in range(args.reps):
        for k, fn in fns.items():
            argmax_t[k].append(timed(lambda: fn.fused_argmax(xc)))

    # ---- (b) q-batch value + gradient: predictive variance against batch MC-EI ----
    pv = predictive_variance(model, 1e-6)
    batch_t = {}
    for q in (4, 8):
        xb = xc[:PTS].reshape(PTS // q, q, D)
        mcei = BatchMonteCarloExpectedImprovement(S).prepare_acquisition_function(model, ds)  # its base samples fix q
        pair = {f"pv_q{q}": pv, f"mc_ei_q{q}": mcei}
        for k, fn in pair.items():
            fn.value_and_gradient(xb)
            batch_t[k] = []
        for _ in range(args.reps):
            for k, fn in pair.items():
                batch_t[k].append(timed(lambda: fn.value_and_gradient(xb)))

    med = lambda v: float(np.median(v))  # noqa: E731
    row = dict(info, N=N, D=D, candidates=M, reps=args.reps, engine_digit_products=model.engine_info()[0])
    for k, v in argmax_t.items():
        row[f"argmax_{k}_ms"] = round(1e3 * med(v), 3)
        row[f"argmax_{k}_spread_ms"] = round(1e3 * (max(v) - min(v)), 3)
    for k in fns:
        if k != "pbt":
            row[f"argmax_{k}_over_pbt"] = round(med(argmax_t[k]) / med(argmax_t["pbt"]), 4)
    row.update(batch_points=PTS, mc_ei_samples=S)
    for k, v in batch_t.items():
        row[f"value_grad_{k}_ms"] = round(1e3 * med(v), 3)
    for q in (4, 8):
        row[f"pv_over_mc_ei_q{q}"] = round(med(batch_t[f"pv_q{q}"]) / med(batch_t[f"mc_ei_q{q}"]), 4)
    line = json.dumps(row)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
