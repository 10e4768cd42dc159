"""2-rank elbo gradient (run under torch.distributed.run): the observation chunks sharded over the ranks and one
all-reduce of the partial sums must give the single-GPU gradient."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np
import torch
import torch.distributed as dist


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group(backend="gloo", rank=rank, world_size=world)
    import stheno_jl_b200 as sb
    from stheno_jl_b200 import lib as sblib
    from test_gpu_vfe_grad import device_raw
    rng = np.random.default_rng(3)
    n, m = 40000, 200   # 3 chunks of 16384 rows -> uneven split over 2 ranks
    x = rng.uniform(0, 30, n)
    z = np.linspace(0, 30, m)
    y = np.sin(x) + 0.3 * rng.standard_normal(n)
    noise = rng.uniform(0.05, 0.15, n)
    fs = sb.gppp(lambda GP: dict(f=GP(1.2 * sb.with_lengthscale(sb.SEKernel(), 0.9) + 0.3 * sb.Matern32Kernel())))
    fx, fz = fs(sb.GPPPInput("f", x), noise), fs(sb.GPPPInput("f", z), 1e-6)
    one = sblib.Context(local)                      # this rank's GPU on its own
    sblib.set_default_context(one)
    _, e1, g1 = device_raw(sb, sb.VFE(fz), fx, y)
    ids = [sblib.nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx = sblib.Context(local, rank, world, ids[0])
    sblib.set_default_context(ctx)
    _, e2, g2 = device_raw(sb, sb.VFE(fz), fx, y)
    ok = abs(e1 - e2) <= 1e-12 * abs(e1)
    worst = 0.0
    for k in g1:
        ok = ok and np.allclose(g2[k], g1[k], rtol=1e-12, atol=0)
        worst = max(worst, float(np.max(np.abs(g2[k] - g1[k]) / np.maximum(np.abs(g1[k]), 1e-300))))
    t = torch.tensor([0 if ok else 1])
    dist.all_reduce(t)
    if rank == 0:
        print("VFE_GRAD_DIST_OK" if t.item() == 0 else f"VFE_GRAD_DIST_FAIL {e1} {e2} worst rel {worst:.3e}")
    dist.barrier()
    sblib.set_default_context(None)
    ctx.close()
    one.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
