"""What the screened EI argmax (tb_api.cu, argmax_screened) saves, and what it costs where it cannot prune:

  headline     N = 4096, D = 10, Ackley-10, Matern52, 1,216,512 device candidates (bench.py's headline step)
  c2           N = 1024, D = 6, Hartmann-6, 1,000,000 device candidates (bench.py --config c2)
  adversarial  the headline with eta = 1e8, far above every mean: nothing can be pruned, the call falls back

For each: median time per fused_argmax call with TB_ARGMAX_SCREEN=1 and =0, the two alternated call by call in one
process; the candidates that went through the variance GEMM (profile counters: the survivors padded to whole tiles, plus
the probe's tile) against M; from one profiled screened call (torch.profiler, CUDA activities), the device time of the
fp32 bound pass (mean_bounds_kernel), of the compaction and of the rest (probe, survivors' K* digits and means, GEMM, tail,
folds), the rest and the compaction also per kernel name with their launch counts; and the survivor count of the bound screen (acq(lo) >= tau - margin, lo from tb_gp_mean_bounds) next to the count
the same screen gives on the exact fp64 means (predict), tau being the call's exact best value (EI only).  The card name
and power limit are read in the same run.

    python tools/argmax_screen_time.py [--reps 7] [--out FILE]     (prints one JSON line)
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True).stdout.strip()
    name, power, clock = [s.strip() for s in q.split(",")]
    return {"gpu": name, "power_limit": power, "sm_clock_max": clock}


def kernel_name(key):
    """'void tb::oz5::kstar_digits_kernel<3, 10, 5>(double const*, ...)' -> 'kstar_digits_kernel'; 'Memcpy HtoD (...)' ->
    'Memcpy HtoD'"""
    base = key.split("(")[0].split("<")[0].strip()
    if not base.startswith("void "):
        return base or key
    return base.split()[-1].split("::")[-1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7, help="timed calls of each mode per workload")
    ap.add_argument("--out", default=None, help="also write the JSON line to this file")
    args = ap.parse_args()
    import torch

    import __graft_entry__ as g

    g.build()
    import trieste_b200 as tb
    from trieste_b200 import _lib
    from trieste_b200.acquisition import ExpectedImprovement
    from trieste_b200.acquisition.function import expected_improvement
    from trieste_b200.objectives import ackley, hartmann_6

    lib = _lib.lib()
    info = card()
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)

    def model(obj, N, D):
        X = np.random.default_rng(0).uniform(size=(N, D))
        ds = tb.Dataset(X, obj(X))
        m = tb.GaussianProcessRegression(tb.build_gpr(ds, tb.Box([0.0] * D, [1.0] * D)))
        return m, ExpectedImprovement().prepare_acquisition_function(m, ds)

    m_head, fn_head = model(ackley, 4096, 10)
    m_c2, fn_c2 = model(hartmann_6, 1024, 6)
    x_head = torch.rand(1_216_512, 10, dtype=torch.float64, device="cuda", generator=gen)
    x_c2 = torch.rand(1_000_000, 6, dtype=torch.float64, device="cuda", generator=gen)
    work = {
        "headline": (m_head, fn_head, x_head, 4096),
        "c2": (m_c2, fn_c2, x_c2, 1024),
        "adversarial": (m_head, expected_improvement(m_head, 1e8), x_head, 4096),
    }

    def call(fn, x, mode):
        os.environ["TB_ARGMAX_SCREEN"] = str(mode)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn.fused_argmax(x)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, r

    def survivors(m, fn, x, tau):
        """candidates the screen keeps with the bound pass's lower mean bound, and with the exact fp64 mean (EI, as in
        tb_api.cu: ub = EI(mean, sigma_ub) >= tau - 2^-20 |tau| - 2^-36 sigma_ub, NaN kept)"""
        from scipy.special import ndtr

        M = x.shape[0]
        lo = torch.empty(M, dtype=torch.float64, device="cuda")
        hi = torch.empty_like(lo)
        _lib.check(lib.tb_gp_mean_bounds(m.handle, x.data_ptr(), M, lo.data_ptr(), hi.data_ptr()))
        mu = np.asarray(m.predict(x.cpu().numpy())[0]).reshape(-1)
        eta, sig = fn._param, float(np.sqrt(max(float(m._spec.kernel.variance), 1e-12)))
        thr = tau - (2.0**-20 * abs(tau) + 2.0**-36 * sig)

        def count(mean):
            z = (eta - mean) / sig
            ub = (eta - mean) * ndtr(z) + sig * np.exp(-0.5 * z * z) / np.sqrt(2 * np.pi)
            return int(np.sum(~(ub < thr)))

        return {"bound": count(lo.cpu().numpy()), "exact_mean": count(mu)}

    t = {k: {0: [], 1: []} for k in work}
    best = {k: {} for k in work}
    for k, (_, fn, x, _) in work.items():
        call(fn, x, 0)
        call(fn, x, 1)
    for _ in range(args.reps):
        for k, (_, fn, x, _) in work.items():
            for mode in (1, 0):
                dt, best[k][mode] = call(fn, x, mode)
                t[k][mode].append(dt)

    row = dict(info, reps=args.reps)
    med = lambda v: float(np.median(v))  # noqa: E731
    from torch.profiler import ProfilerActivity, profile

    for k, (m, fn, x, N) in work.items():
        assert best[k][0] == best[k][1], (k, best[k])
        h = m.handle
        lib.tb_gp_profile(h, 1)
        call(fn, x, 1)
        ms, n, fl = C.c_double(), C.c_int64(), C.c_double()
        lib.tb_gp_profile_read(h, C.byref(ms), C.byref(n), C.byref(fl))
        lib.tb_gp_profile(h, 0)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            call(fn, x, 1)
        bound_us = compact_us = rest_us = 0.0
        rest_by_kernel = {}
        for e in prof.key_averages():
            us = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            if us <= 0:
                continue
            if "mean_bounds_kernel" in e.key:
                bound_us += us
                continue
            if "compact_kernel" in e.key:
                compact_us += us
            else:
                rest_us += us
            name = kernel_name(e.key)
            ms, cnt = rest_by_kernel.get(name, (0.0, 0))
            rest_by_kernel[name] = (ms + us / 1e3, cnt + e.count)
        surv = survivors(m, fn, x, best[k][1][1])
        row[k] = {
            "candidates": int(x.shape[0]),
            "screened_s": med(t[k][1]), "screened_spread": [min(t[k][1]), max(t[k][1])],
            "unscreened_s": med(t[k][0]), "unscreened_spread": [min(t[k][0]), max(t[k][0])],
            "speedup": med(t[k][0]) / med(t[k][1]),
            "gemm_candidates": fl.value / float(N) ** 2, "gemm_launches": int(n.value),
            "device_ms": {"bound_pass": bound_us / 1e3, "compaction": compact_us / 1e3, "probe_survivors_rest": rest_us / 1e3},
            "rest_by_kernel": {k: {"ms": v[0], "launches": v[1]} for k, v in sorted(rest_by_kernel.items(), key=lambda kv: -kv[1][0])},
            "survivors": surv,
            "best": list(best[k][1]),
        }
    line = json.dumps(row)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
