"""What BatchExpectedImprovement costs on the c3 model (Ackley-10, N = 4096, fp64, device-resident q-batches):

  for (q, S) = (3, 100), (8, 512), (8, 2048):
    - q-batches/s of the value (tb_acq_batch_ei) and of the value with gradient (tb_acq_batch_ei_grad);
    - the split between the joint predict (K*, A = Linv K*, joint_kernel: timed as predict_joint of the same batches)
      and the BEI kernels (the rest of the value call);
    - the same batches through BatchMonteCarloExpectedImprovement(512), value and value with gradient.

Times are CUDA events on the current stream around calls that return only once the handle's stream has drained; the
median of --reps calls after one warm-up call.  The card name and power limit are read in the same run.

    python tools/batch_ei_time.py [--reps 5] [--out FILE]     (prints one JSON line)
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np

N, D = 4096, 10
CASES = [(3, 100, 65536), (8, 512, 8192), (8, 2048, 4096)]  # (q, S, q-batches per call)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch

    import trieste_b200 as tb
    from trieste_b200.acquisition import BatchExpectedImprovement, BatchMonteCarloExpectedImprovement
    from trieste_b200.objectives import ackley

    def timed(f):
        f()
        ts = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ts.append(a.elapsed_time(b) / 1e3)
        return float(np.median(ts))

    rng = np.random.default_rng(0)
    X = rng.uniform(size=(N, D))
    ds = tb.Dataset(X, ackley(X))
    model = tb.GaussianProcessRegression(tb.build_gpr(ds, tb.Box([0.0] * D, [1.0] * D)))
    rows = []
    for q, S, B in CASES:
        xd = torch.rand(B, q, D, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(q))
        bei = BatchExpectedImprovement(S, seed=0).prepare_acquisition_function(model, ds)
        mc = BatchMonteCarloExpectedImprovement(512).prepare_acquisition_function(model, ds)
        t_val = timed(lambda: bei(xd))
        t_grad = timed(lambda: bei.value_and_gradient(xd))
        t_joint = timed(lambda: model.predict_joint(xd))
        t_mc = timed(lambda: mc(xd))
        t_mc_grad = timed(lambda: mc.value_and_gradient(xd))
        rows.append({"q": q, "S": S, "batches": B,
                     "bei_value_batches_per_s": B / t_val, "bei_value_grad_batches_per_s": B / t_grad,
                     "bei_value_ms": t_val * 1e3, "joint_predict_ms": t_joint * 1e3,
                     "bei_kernels_ms": (t_val - t_joint) * 1e3,
                     "mc_ei512_value_batches_per_s": B / t_mc, "mc_ei512_value_grad_batches_per_s": B / t_mc_grad})
    line = json.dumps({"tool": "batch_ei_time", "model": f"Ackley-{D} N={N} fp64 engine={model.engine}", **card(),
                       "cases": rows})
    print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
