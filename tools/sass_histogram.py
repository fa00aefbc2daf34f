"""SASS evidence for the wgmma / TMA kernels: per-kernel mnemonic histogram of the built library.

    python tools/sass_histogram.py > sass_histogram.md

(`cuobjdump -sass` on trieste_b200/libtrieste_b200.so; wgmma.mma_async -> IGMMA, cp.async.bulk -> UBLKCP, mbarrier -> SYNCS,
fp64 mma.sync -> DMMA.)"""
import collections
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "trieste_b200", "libtrieste_b200.so")
WANT = ["dg::digit_gemm_kernel", "oz5::kstar_digits_kernel<3, 10, 5>", "oz5::kstar_digits_kernel<3, 10, 6>", "tb::trigemm_kernel<false, 0>",
        "tb::tail_kernel", "tc_mean_bounds_kernel<3, 10>", "rff_eval_kernel<6, 8>", "joint_kernel<3, 1>", "lbfgs_step_kernel", "kdot_kernel<3, 6, 4>", "grad_kernel<3, 10, 1>", "grad_kernel<3, 10, 8>",
        "fac::chol_syrk_kernel", "fac::kinv_kernel"]
KEY = ["IGMMA", "HGMMA", "UBLKCP", "UTMALDG", "SYNCS", "DMMA", "HMMA", "IMMA", "DFMA", "DADD", "DMUL", "MUFU", "F2F", "I2F", "F2I",
       "LDS", "STS", "LDG", "STG", "LDGSTS", "SHFL", "BAR", "UMOV", "PRMT", "LOP3"]


def demangle(names):
    out = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines()
    return dict(zip(names, out))


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True).stdout
    funcs, cur = collections.OrderedDict(), None
    for ln in sass.splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1)
            funcs[cur] = collections.Counter()
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_]+)", ln)
        if m and cur:
            funcs[cur][m.group(1)] += 1
    names = demangle(list(funcs))
    total = collections.Counter()
    for c in funcs.values():
        total.update(c)
    print("# SASS mnemonic histogram of `trieste_b200/libtrieste_b200.so` (sm_90a)\n")
    print(f"{len(funcs)} kernels; whole library: " + ", ".join(f"{k} {total[k]}" for k in KEY if total[k]) + "\n")
    print("| kernel | instructions | " + " | ".join(KEY[:14]) + " |")
    print("|---|---|" + "---|" * 14)
    for mangled, c in funcs.items():
        d = names[mangled]
        if not any(w in d for w in WANT):
            continue
        short = re.sub(r"\(.*", "", d)
        print(f"| `{short}` | {sum(c.values())} | " + " | ".join(str(c[k]) for k in KEY[:14]) + " |")


if __name__ == "__main__":
    main()
