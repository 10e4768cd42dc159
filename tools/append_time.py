"""Cost of conditioning on new observations by appending to the factor against refactorising the stacked problem.

Config-2 inputs (bench.make_inputs: SE kernel, 1-D x ~ U(0, N/32), sigma^2 = 0.1), N1 = 65536 old observations and
N2 new ones.  Times, with CUDA events on the library stream (median of --reps after one warm-up round):
    append: sb_factor_append on the old factor + sb_factor_set_data on the new handle
    fresh:  sb_factor_create of the stacked problem + sb_factor_set_data
and, from one more append under torch.profiler, the relayout kernel's own time and its HBM rate.  Prints one JSON
line per N2 with the card name and power limit read in the same run.

    python tools/append_time.py [--n1 65536] [--n2 512 4096] [--reps 5] [--trailing 0|1]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK_GBS = 3350.0   # NVIDIA H100 SXM data sheet
NB = 128


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def relayout_bytes(n1, n2):
    """HBM traffic of append_relayout_kernel: old rows [128 j, N1) and N2 rows of V read, ld_j rows written, per
    column of the head."""
    nh = n1 // NB
    np_joint = (n1 + n2 + NB - 1) // NB * NB
    j = np.arange(nh, dtype=np.float64)
    read_l = NB * np.sum(n1 - NB * j)
    read_v = NB * nh * n2
    write = NB * np.sum(np_joint - NB * j)
    return 8.0 * (read_l + read_v + write), 8.0 * read_l, 8.0 * read_v, 8.0 * write


def kernel_ms(prof, needle):
    total = 0.0
    for e in prof.key_averages():
        if needle in e.key:
            total += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
    return total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n1", type=int, default=65536)
    ap.add_argument("--n2", type=int, nargs="+", default=[512, 4096])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--trailing", type=int, default=0)
    args = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile

    import stheno_jl_b200 as sb
    from bench import make_inputs
    from stheno_jl_b200.finite import _noise_struct
    from stheno_jl_b200.gp import spec_dense, spec_symmetric
    lib = sb.lib.load()
    ctx = sb.default_context()
    ctx.set_option("trailing", args.trailing)
    name, power = card()
    n1 = args.n1
    fs = sb.gppp(lambda GP: dict(f=GP(sb.SEKernel())))
    for n2 in args.n2:
        x, y, _ = make_inputs(n1 + n2, 1)
        x1, x2 = x[:n1], x[n1:]
        p1 = sb.posterior(fs(sb.GPPPInput("f", x1), 0.1), y[:n1])
        fx2 = p1(sb.GPPPInput("f", x2), 0.1)
        l2 = fx2.lowered
        cross, full, ns2 = spec_dense(l2, p1.lx), spec_dense(l2, l2), _noise_struct(0.1, n2)
        fj = fs(sb.BlockData(sb.GPPPInput("f", x1), sb.GPPPInput("f", x2)), 0.1)
        spec, nsj = spec_symmetric(fj.lowered), _noise_struct(0.1, n1 + n2)
        delta = np.ascontiguousarray(y - fj.lowered.mean())

        def append():
            h, info = C.c_void_p(), C.c_int64(0)
            sb.lib.check(lib.sb_factor_append(ctx.h, p1.fac.h, C.byref(cross), C.byref(full), C.byref(ns2),
                                              C.byref(h), C.byref(info)), info)
            return h

        def fresh():
            h, info = C.c_void_p(), C.c_int64(0)
            sb.lib.check(lib.sb_factor_create(ctx.h, C.byref(spec), C.byref(nsj), C.byref(h), C.byref(info)), info)
            return h

        t = {"append": [], "append_solve": [], "fresh": [], "fresh_solve": []}
        for rep in range(args.reps + 1):   # the first round warms up every shape
            for key, make in (("append", append), ("fresh", fresh)):
                ctx.mark(0)
                h = make()
                ctx.mark(1)
                sb.lib.check(lib.sb_factor_set_data(ctx.h, h, delta.ctypes.data))
                ctx.mark(2)
                if rep:
                    t[key].append(ctx.elapsed_ms(0, 1))
                    t[key + "_solve"].append(ctx.elapsed_ms(1, 2))
                lib.sb_factor_destroy(h)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            h = append()
            torch.cuda.synchronize()
        lib.sb_factor_destroy(h)
        relay_ms = kernel_ms(prof, "append_relayout")
        nbytes, rl, rv, wr = relayout_bytes(n1, n2)
        med = {k: float(np.median(v)) for k, v in t.items()}
        a, f = med["append"] + med["append_solve"], med["fresh"] + med["fresh_solve"]
        print(json.dumps(dict(
            n1=n1, n2=n2, trailing=args.trailing, reps=args.reps, card=name, power_limit=power,
            append_ms=med["append"], append_set_data_ms=med["append_solve"], append_total_ms=a,
            fresh_ms=med["fresh"], fresh_set_data_ms=med["fresh_solve"], fresh_total_ms=f,
            append_over_fresh=a / f,
            relayout_ms=relay_ms, relayout_gb=nbytes / 1e9,
            relayout_gb_read_L=rl / 1e9, relayout_gb_read_V=rv / 1e9, relayout_gb_written=wr / 1e9,
            relayout_gbs=nbytes / 1e6 / relay_ms if relay_ms > 0 else None,
            relayout_of_hbm_peak=nbytes / 1e6 / relay_ms / HBM_PEAK_GBS if relay_ms > 0 else None,
            all_ms={k: v for k, v in t.items()})), flush=True)
        del p1, fx2, fj


if __name__ == "__main__":
    main()
