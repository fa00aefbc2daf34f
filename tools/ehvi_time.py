"""What expected hypervolume improvement costs on the device: N = 1024 training points, D = 6, DTLZ2 with L = 2 and 3
objectives (one native GPR per objective), M = 10^6 candidates on the device.

  (a) the fused EHVI argmax (tb_ehvi_argmax): the members' K* and variance GEMMs, one EHVI kernel and one fold per chunk;
  (b) the members' predict alone (L x tb_gp_predict into device arrays): (a) - (b) is the EHVI kernel's share;
  (c) the unfused route: L x tb_gp_predict into host arrays over all M, and the NumPy EHVI of tests/ehvi_oracle.py on
      the host over the first 16,384 candidates (over all M its [M, K, L] work does not fit a host's memory in one go);
  (d) one EfficientGlobalOptimization(ExpectedHypervolumeImprovement()).acquire over the box with the continuous
      optimiser, its L-BFGS on the device against the host L-BFGS (TB_LBFGS=host).

(a) and (b) are medians over --reps calls, alternated; (c) is one call; (d) the median of --acquires acquires after one
warm-up each.  The card name and power limit are read in the same run and printed with the numbers.

    python tools/ehvi_time.py [--reps 7] [--acquires 3] [--out FILE]     (prints one JSON line)
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
HOST_M = 16384


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
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--acquires", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import __graft_entry__ as g

    g.build()
    import trieste_b200 as tb
    from tests import ehvi_oracle as eo
    from trieste_b200.acquisition import ExpectedHypervolumeImprovement
    from trieste_b200.acquisition.interface import OBJECTIVE
    from trieste_b200.objectives import dtlz2
    from trieste_b200.rule import EfficientGlobalOptimization

    out = {"what": "EHVI fused argmax / members' predict / unfused route / acquire", "N": N, "D": D, "M": M,
           "reps": args.reps, "acquires": args.acquires, "host_m": HOST_M, **card()}
    rng = np.random.default_rng(0)
    X = rng.uniform(size=(N, D))
    space = tb.Box([0.0] * D, [1.0] * D)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    xc = torch.rand(M, D, dtype=torch.float64, device="cuda", generator=gen)
    xh = xc.cpu().numpy()
    for L in (2, 3):
        Y = dtlz2(X, L, D)
        members = [tb.GaussianProcessRegression(tb.build_gpr(tb.Dataset(X, Y[:, l:l + 1]), space)) for l in range(L)]
        stack = tb.TrainableModelStack(*[(m, 1) for m in members])
        builder = ExpectedHypervolumeImprovement()
        ds = tb.Dataset(X, Y)
        fn = builder.prepare_acquisition_function(stack, ds)
        lower, upper = fn.partition_bounds
        row = {"K": int(lower.shape[0]), "engines": [m.engine_info()[0] for m in members]}
        fn.fused_argmax(xc)
        stack.predict(xc)
        ta, tp = [], []
        for _ in range(args.reps):
            ta.append(timed(lambda: fn.fused_argmax(xc)))
            tp.append(timed(lambda: stack.predict(xc)))
        row["fused_argmax_ms"] = float(np.median(ta))
        row["members_predict_ms"] = float(np.median(tp))

        # unfused route: the members' predict into host arrays over all M, the host EHVI over the first HOST_M candidates
        # (over all M it would take [M, K, L] work on the host; its time per candidate is what the slice shows)
        row["unfused_predict_to_host_ms"] = timed(lambda: stack.predict(xh))
        mean, var = stack.predict(xh[:HOST_M])

        def host_ehvi():
            for c0 in range(0, HOST_M, 512):
                eo.ehvi(mean[c0:c0 + 512], var[c0:c0 + 512], lower, upper)

        row[f"host_ehvi_ms_first_{HOST_M}"] = timed(host_ehvi)
        for mode in ("device", "host"):
            os.environ["TB_LBFGS"] = mode
            rule = EfficientGlobalOptimization(ExpectedHypervolumeImprovement())
            rule.acquire(space, {OBJECTIVE: stack}, {OBJECTIVE: ds})
            ts = [timed(lambda: rule.acquire(space, {OBJECTIVE: stack}, {OBJECTIVE: ds})) for _ in range(args.acquires)]
            row[f"acquire_{mode}_lbfgs_ms"] = float(np.median(ts))
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
