"""2-rank append (run under torch.distributed.run): every rank extends its replicated factor with
sb_factor_append, then the posterior is predicted with the test points sharded over the ranks; both ranks must
match the oracle's posterior of the stacked observations."""
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
    from oracle import stheno_oracle as orc
    ids = [sblib.nccl_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ctx = sblib.Context(local, rank, world, ids[0])
    sblib.set_default_context(ctx)

    rng = np.random.default_rng(8)
    fails = []
    for n1, n2, ns in [(3000, 700, 333), (1100, 200, 77)]:
        x1, x2, xs = rng.uniform(0, 100, n1), rng.uniform(0, 100, n2), rng.uniform(0, 100, ns)
        y1, y2 = np.sin(x1) + 0.3 * rng.standard_normal(n1), np.sin(x2) + 0.3 * rng.standard_normal(n2)
        fs = sb.gppp(lambda GP: dict(f=GP(sb.SEKernel())))
        fo = orc.gppp(lambda GP: dict(f=GP(orc.SEKernel())))
        p1 = sb.posterior(fs(sb.GPPPInput("f", x1), 0.1), y1)
        p12 = sb.posterior(p1(sb.GPPPInput("f", x2), 0.2), y2)
        bo = orc.BlockData(orc.GPPPInput("f", x1), orc.GPPPInput("f", x2))
        po = orc.posterior(fo(bo, np.concatenate([np.full(n1, 0.1), np.full(n2, 0.2)])), np.concatenate([y1, y2]))
        m, v = sb.mean_and_var(p12, sb.GPPPInput("f", xs))
        mo, vo = orc.mean_and_var(po, orc.GPPPInput("f", xs))
        if not (np.allclose(m, mo, rtol=1e-10, atol=1e-11) and np.allclose(v, vo, rtol=1e-9, atol=1e-11)):
            fails.append((n1, n2, float(np.abs(m - mo).max()), float(np.abs(v - vo).max())))
    t = torch.tensor([len(fails)], dtype=torch.int64)
    dist.all_reduce(t)
    if rank == 0:
        print("APPEND_DIST_OK" if t.item() == 0 else f"APPEND_DIST_FAIL {fails}")
    sblib.set_default_context(None)
    ctx.close()
    dist.destroy_process_group()
    sys.exit(0 if t.item() == 0 else 1)


if __name__ == "__main__":
    main()
