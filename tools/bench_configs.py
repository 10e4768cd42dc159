"""BASELINE.json configs 3 and 4 at FULL size on the GPU box (bench.py itself is config 2, the metric's config).

  config 3 (1 GPU):   GPPP f3 = f1 + f2 over BlockData, 3 x 16384 inputs (N = 49152): block cross-cov assembly
                      + joint Cholesky + logpdf + posterior of all three processes at 3 x 1024 points.
  config 4 (2 GPUs):  elbo with M = 4096 pseudo-points, N = 131072 SE kernel: K_uu / K_uf + low-rank Cholesky,
                      approximate-posterior mean / var at 4096 points.  torchrun --nproc-per-node 2 ... --config 4

Parity: config 3 -- residual identity (K + s2 I) alpha = delta on a subset + dmma-vs-ozaki agreement;
config 4 -- the CPU oracle's elbo / dtc at full size (Kuf is 4.3 GB on the host: ~1 min with 64 threads) when
--oracle is given, else cross-check between the two device paths.  One JSON line per config on stdout.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402


def setup():
    import torch
    rank, world, local = (int(os.environ.get(k, d)) for k, d in (("RANK", 0), ("WORLD_SIZE", 1), ("LOCAL_RANK", 0)))
    torch.cuda.set_device(local)
    import stheno_jl_b200 as sb
    from stheno_jl_b200 import lib as sblib
    dist = None
    if world > 1:
        import torch.distributed as dist
        dist.init_process_group(backend="gloo", rank=rank, world_size=world)
        ids = [sblib.nccl_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        ctx = sblib.Context(local, rank, world, ids[0])
    else:
        ctx = sblib.Context(local)
    sblib.set_default_context(ctx)
    return sb, sblib, ctx, dist, rank, world


def timed(fn, reps, sync):
    fn()
    sync()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        sync()
        ts.append(time.perf_counter() - t0)
    return out, min(ts)


def config3(args):
    import torch
    sb, sblib, ctx, dist, rank, world = setup()
    from models import f3_model
    rng = np.random.default_rng(123456)
    nb = args.nb
    xs = [rng.uniform(0, nb / 32, nb) for _ in range(3)]
    xt = [rng.uniform(0, nb / 32, 1024) for _ in range(3)]
    y = np.concatenate([np.sin(v) for v in xs]) + 0.3 * rng.standard_normal(3 * nb)
    f = f3_model(sb)
    names = ["f1", "f2", "f3"]
    obs = sb.BlockData(*[sb.GPPPInput(nm, v) for nm, v in zip(names, xs)])
    tst = sb.BlockData(*[sb.GPPPInput(nm, v) for nm, v in zip(names, xt)])
    res = {}
    for mode, name in ((1, "ozaki"), (0, "dmma")):
        ctx.set_option("trailing", mode)

        def step():
            fx = f(obs, 0.1)
            lp = sb.logpdf(fx, y)
            post = sb.posterior(fx, y)
            m, v = sb.mean_and_var(post, tst)
            return lp, m, v, post
        ctx.timings(reset=True)
        (lp, m, v, post), t = timed(step, 2, torch.cuda.synchronize)
        tm = ctx.timings()
        res[name] = dict(lp=lp, m=m, v=v, t=t, tm=tm, post=post)
    a, b = res["ozaki"], res["dmma"]
    # residual identity on a subset of the training points (zero-mean prior)
    sel = [np.arange(0, nb, 97) for _ in range(3)]
    idx = np.concatenate([s + nb * k for k, s in enumerate(sel)])
    sub = sb.BlockData(*[sb.GPPPInput(nm, x[s]) for nm, x, s in zip(names, xs, sel)])
    alpha = a["post"].alpha
    resid = float(np.max(np.abs(sb.mean(a["post"], sub) - (y[idx] - 0.1 * alpha[idx]))))
    n = 3 * nb
    out = {"config": 3, "workload": f"GPPP f3=f1+f2 (SE + Matern52) over BlockData, 3x{nb} inputs (N={n}) fp64, 1 GPU: "
                                    "block cross-cov assembly + joint Cholesky + logpdf + posterior at 3x1024 points",
           "points_per_s_ozaki": n / a["t"], "s_per_step_ozaki": a["t"], "points_per_s_dmma": n / b["t"], "s_per_step_dmma": b["t"],
           "logpdf_ozaki": a["lp"], "logpdf_dmma": b["lp"], "logpdf_rel_diff": abs(a["lp"] - b["lp"]) / abs(b["lp"]),
           "mean_max_abs_diff": float(np.max(np.abs(a["m"] - b["m"]))), "var_max_rel_diff": float(np.max(np.abs(a["v"] - b["v"]) / np.abs(b["v"]))),
           "residual_identity_max_abs": resid,
           "phases_ms_ozaki": {k: a["tm"][k] / 3 for k in ("assemble_ms", "trailing_ms", "solve_ms", "predict_ms")},
           "n_gpus": world}
    if rank == 0:
        print(json.dumps(out))
    ctx.close()


def config4(args):
    import torch
    sb, sblib, ctx, dist, rank, world = setup()
    rng = np.random.default_rng(123456)
    n, m = args.n4, args.m4
    x = rng.uniform(0, m, n)
    z = np.arange(m) + 0.5
    xs = rng.uniform(0, m, 4096)
    y = np.sin(x) + 0.3 * rng.standard_normal(n)
    f = sb.gppp(lambda GP: dict(f=GP(sb.SEKernel())))

    def sync():
        torch.cuda.synchronize()
        if dist is not None:
            dist.barrier()
    res = {}
    for mode, name in ((1, "ozaki"), (0, "dmma")):
        ctx.set_option("trailing", mode)

        def step():
            fx, fz = f(sb.GPPPInput("f", x), 0.1), f(sb.GPPPInput("f", z), 1e-9)
            ap = sb.approx_posterior(sb.VFE(fz), fx, y)
            mm, vv = sb.mean_and_var(ap, sb.GPPPInput("f", xs))
            return ap.elbo, ap.dtc, mm, vv
        (e, d, mm, vv), t = timed(step, 2, sync)
        res[name] = dict(elbo=e, dtc=d, m=mm, v=vv, t=t)
    a, b = res["ozaki"], res["dmma"]
    out = {"config": 4, "workload": f"elbo(VFE) with M={m} pseudo-points on a unit grid (jitter 1e-9), N={n} SE kernel fp64, "
                                    f"{world} GPU(s): K_uu / K_uf + two MxM Choleskys + approximate-posterior mean/var at 4096 points",
           "points_per_s_ozaki": n / a["t"], "s_per_step_ozaki": a["t"], "points_per_s_dmma": n / b["t"], "s_per_step_dmma": b["t"],
           "elbo_ozaki": a["elbo"], "elbo_dmma": b["elbo"], "dtc_ozaki": a["dtc"],
           "elbo_rel_diff_paths": abs(a["elbo"] - b["elbo"]) / abs(b["elbo"]),
           "mean_max_abs_diff_paths": float(np.max(np.abs(a["m"] - b["m"]))), "n_gpus": world}
    if args.oracle and rank == 0:
        from oracle import stheno_oracle as orc
        import bench
        bench.pin_cpu_threads()
        fo = orc.gppp(lambda GP: dict(f=GP(orc.SEKernel())))
        t0 = time.perf_counter()
        fxo, fzo = fo(orc.GPPPInput("f", x), 0.1), fo(orc.GPPPInput("f", z), 1e-9)
        eo = orc.elbo(orc.VFE(fzo), fxo, y)
        out["oracle_elbo"] = eo
        out["oracle_s"] = time.perf_counter() - t0
        out["elbo_rel_err_vs_oracle"] = abs(a["elbo"] - eo) / abs(eo)
    if rank == 0:
        print(json.dumps(out))
    if dist is not None:
        dist.barrier()
    sblib.set_default_context(None)
    ctx.close()
    if dist is not None:
        dist.destroy_process_group()


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, required=True, choices=[3, 4])
    ap.add_argument("--nb", type=int, default=16384)
    ap.add_argument("--n4", type=int, default=131072)
    ap.add_argument("--m4", type=int, default=4096)
    ap.add_argument("--oracle", action="store_true")
    args = ap.parse_args()
    (config3 if args.config == 3 else config4)(args)
