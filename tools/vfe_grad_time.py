"""Cost of the elbo gradient against the elbo itself: CUDA-event time of sb_vfe_create and of sb_vfe_grad on the
same handle, at the config-4 shape by default (N = 131072 observations, M = 4096 pseudo-points, SE kernel,
sigma^2 = 0.1, jitter 1e-9).  Prints one JSON line with the card name and power limit read in the same run.

    python tools/vfe_grad_time.py [--n 131072] [--m 4096] [--reps 5] [--trailing 0|1]

Flop model (fp64, tensor-core work only):
    sb_vfe_create: sweep of the N x M block by L_u (N M^2) + D = A A' (2 N M^2) + two M x M Choleskys (2 M^3 / 3)
    sb_vfe_grad:   sweeps of the N x M block by L_u and L_B (2 N M^2) + S = A' E (2 N M^2)
                   + prologue: two identity sweeps (2 M^3) and five M x M products (10 M^3)
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=131072)
    ap.add_argument("--m", type=int, default=4096)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--trailing", type=int, default=0)
    args = ap.parse_args()
    import stheno_jl_b200 as sb
    lib = sb.lib.load()
    ctx = sb.default_context()
    ctx.set_option("trailing", args.trailing)
    n, m = args.n, args.m
    rng = np.random.default_rng(4)
    x = rng.uniform(0, m, n)
    z = np.arange(m) + 0.5
    y = np.sin(x) + 0.3 * rng.standard_normal(n)
    fs = sb.gppp(lambda GP: dict(f=GP(sb.SEKernel())))
    v, fx = sb.VFE(fs(sb.GPPPInput("f", z), 1e-9)), fs(sb.GPPPInput("f", x), 0.1)
    a = sb.finite._VfeInputs(v, fx, y)
    g = [np.zeros(max(2, 2 * s.nterms)) for s in (a.uu, a.xu, a.ffd)] + [np.zeros(m), np.zeros(n)]
    t_create, t_grad = [], []
    for rep in range(args.reps + 1):          # the first round warms up every shape
        ctx.mark(0)
        handle, _, _ = sb.finite._vfe_create(v, fx, y, a)
        ctx.mark(1)
        sb.lib.check(lib.sb_vfe_grad(ctx.h, handle.h, C.byref(a.uu), C.byref(a.xu), C.byref(a.ffd), C.byref(a.nf),
                                     a.delta.ctypes.data, *[b.ctypes.data for b in g]))
        ctx.mark(2)
        if rep:
            t_create.append(ctx.elapsed_ms(0, 1))
            t_grad.append(ctx.elapsed_ms(1, 2))
        del handle
    mc, mg = float(np.median(t_create)), float(np.median(t_grad))
    f_create = 3.0 * n * m * m + 2.0 * m ** 3 / 3
    f_grad = 4.0 * n * m * m + 12.0 * m ** 3
    name, power = card()
    print(json.dumps(dict(
        n=n, m=m, trailing=args.trailing, reps=args.reps, card=name, power_limit=power,
        create_ms=mc, grad_ms=mg, grad_over_create=mg / mc,
        create_tflops=f_create / mc / 1e9, grad_tflops=f_grad / mg / 1e9,
        create_ms_all=t_create, grad_ms_all=t_grad)))


if __name__ == "__main__":
    main()
