"""GPU, 2 ranks over NCCL (needs a machine with >= 2 GPUs; skipped otherwise):
  * slab-sharded marching cubes on the CUDA kernel == the single-GPU mesh, bit for bit (SURVEY.md section 8e, config[4]);
  * one training step per rank on different frames + the single gradient all-reduce: every rank ends with the same
    gradients, equal to the mean of the per-rank ones."""
import os
import socket
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _grid(n):
    ax = np.linspace(-1, 1, n, dtype=np.float32)
    xx, yy, zz = np.meshgrid(ax, ax, ax, indexing="ij")
    return (np.sqrt(xx * xx + yy * yy + zz * zz) - 0.7 + 0.06 * np.sin(5 * xx) * np.cos(3 * zz)).astype(np.float32)


def _worker(rank, world, port, q):
    try:
        sys.path.insert(0, ROOT)
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                          LOCAL_RANK=str(rank))
        import torch.distributed as dist
        from selfreconcode_b200 import parallel, ops
        r, w, local = parallel.init_from_env("nccl")
        dev = torch.device("cuda", local)
        # ---- sharded MC on the CUDA kernel
        for n in (65, 129):
            sdf = torch.from_numpy(_grid(n)).to(dev)
            step, org = (2.0 / n,) * 3, (-1.0 + 1.0 / n,) * 3
            v1, f1 = ops.marching_cubes(sdf, *step, *org, 0.0)
            v, f = parallel.sharded_marching_cubes(sdf, step, org, 0.0, rank, world)
            assert torch.equal(f, f1) and torch.equal(v, v1), "stitched mesh == single-GPU mesh (%d^3)" % n
            v0, f0 = parallel.sharded_marching_cubes(sdf, step, org, 0.0, rank, world, gather_to=0)
            if rank == 0:
                assert torch.equal(f0, f1) and torch.equal(v0, v1)
        # ---- one training step per rank + the gradient all-reduce
        import bench
        sc = bench.build_scene(dev, frame_seed=rank)
        bench.TRAIN_FRAMES, bench.TRAIN_RAYS = 2, 2048
        tr = bench.build_train(sc, dev, rank, world)
        tr["ar"] = parallel.GradAllReduce([q for q in tr["params"]], timed=True)
        tr["opt"].zero_grad(set_to_none=True)
        loss = tr["net"].forward_rays(tr["datas"], tr["bi"], tr["ri"], tr["ci"], tr["init"].clone(), bench.RATIO,
                                      tr["fids"], extra_points=tr["extra"])
        loss.backward()
        tr["net"].propagateTmpPsGrad(tr["fids"], bench.RATIO)
        local_g = [q.grad.detach().clone() if q.grad is not None else torch.zeros_like(q) for q in tr["params"]]
        nbytes = tr["ar"]()
        ms = tr["ar"].collective_ms()
        flat_local = torch.cat([g.reshape(-1) for g in local_g])
        both = [torch.empty_like(flat_local) for _ in range(world)]
        dist.all_gather(both, flat_local)
        mean = sum(both) / world
        flat_red = torch.cat([q.grad.reshape(-1) for q in tr["params"]])
        assert nbytes == 4 * flat_red.numel()
        err = (flat_red - mean).abs().max().item() / max(mean.abs().max().item(), 1e-30)
        assert err < 1e-6, err
        q.put((rank, "ok", "all-reduce %.3f ms for %.1f MB" % (ms, nbytes / 1e6)))
        dist.barrier()
        dist.destroy_process_group()
    except Exception as e:  # surface the failure to the parent
        import traceback
        q.put((rank, "fail", traceback.format_exc()[-1500:]))


def test_two_gpus_nccl():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=900) for _ in range(2))
    for p in procs:
        p.join(timeout=120)
    print(res)
    assert [r[:2] for r in res] == [(0, "ok"), (1, "ok")], res
