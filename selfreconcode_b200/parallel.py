"""One-process-per-GPU data parallelism for the hot path (SURVEY.md section 8e).

The reference has no distributed code at all; this is the native design:

  * training  : frames (and their rays) are sharded across ranks; every rank holds full replicas
                of the three MLPs, the skin volume and the template mesh.  Gradients reach .grad
                from three backward calls per step (network.py:687, train.py:168, network.py:814)
                after one zero_grad, so ONE flat all-reduce (average) of {MLP params, per-frame
                leaf tensors} right after propagateTmpPsGrad covers them all (~15.5 MB over
                NVLink/NVSwitch: tens of microseconds; overlap is a non-goal).
  * rendering : frames are independent -> replicas only, no collective.
  * extraction: the final SDF grid is cut into x-slabs; each rank runs marching cubes on its slab
                plus a two-plane halo and the pieces are stitched into exactly the mesh a single
                GPU would produce (same canonical vertex / face order), with one all-gather of the
                counts and one of the payload.
Collectives go through torch.distributed (NCCL on GPUs; gloo in the CPU tests).
"""
import os

import torch
import torch.distributed as dist


def init_from_env(backend=None):
    """torchrun-style rendezvous (RANK / WORLD_SIZE / LOCAL_RANK / MASTER_*)."""
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = "nccl" if torch.cuda.is_available() else "gloo"
        if backend == "nccl":
            torch.cuda.set_device(local)
            dist.init_process_group(backend, device_id=torch.device("cuda", local))
        else:
            dist.init_process_group(backend)
    return rank, world, local


def shard_frames(frame_ids, rank, world):
    """Contiguous, equal-sized shard of a step's frame ids (the global batch is N*world frames).
    Equal shards make 'mean over frames then mean over ranks' exact (network.py:617,637)."""
    n = len(frame_ids)
    if n % world != 0:
        raise ValueError("global batch of %d frames is not divisible by world size %d" % (n, world))
    per = n // world
    return frame_ids[rank * per:(rank + 1) * per]


class GradAllReduce:
    """Single all-reduce (average) of the gradients of `params` per step (train.py:168-170: after
    propagateTmpPsGrad, before optimizer.step()).

    Flatten: one `torch.cat` into a persistent bucket; NCCL all-reduce over NVLink / NVSwitch; unflatten: one
    fused foreach copy.  Parameters whose .grad is None contribute zeros (a per-frame leaf such as a latent code
    that this rank's frames did not touch) and receive the average.  `last_ms` = device time of the collective
    (CUDA events on the current stream) when `timed`."""

    def __init__(self, params, group=None, timed=False):
        self.params = [p for p in params if p.requires_grad]
        self.group = group
        self.numel = sum(p.numel() for p in self.params)
        self.bucket = None
        self.timed = timed
        self.last_ms = 0.0
        self._ev = None

    def __call__(self):
        if not dist.is_initialized() or dist.get_world_size(self.group) == 1 or not self.params:
            return 0
        dev = self.params[0].device
        world = dist.get_world_size(self.group)
        if self.bucket is None or self.bucket.device != dev:
            self.bucket = torch.empty(self.numel, dtype=torch.float32, device=dev)
        flat = [(p.grad if p.grad is not None else torch.zeros_like(p)).reshape(-1) for p in self.params]
        torch.cat(flat, out=self.bucket)
        if self.timed and dev.type == "cuda":
            if self._ev is None:
                self._ev = (torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
            self._ev[0].record()
        dist.all_reduce(self.bucket, op=dist.ReduceOp.SUM, group=self.group)
        if self.timed and dev.type == "cuda":
            self._ev[1].record()
        self.bucket.div_(world)
        views, o = [], 0
        for p in self.params:
            n = p.numel()
            views.append(self.bucket[o:o + n].view_as(p))
            o += n
        for p in self.params:
            if p.grad is None:
                p.grad = torch.empty_like(p)
        torch._foreach_copy_([p.grad for p in self.params], views)
        return self.numel * 4

    def collective_ms(self):
        """Device time of the last all-reduce (synchronises on its end event)."""
        if self._ev is None:
            return 0.0
        self._ev[1].synchronize()
        return self._ev[0].elapsed_time(self._ev[1])


def slab_range(nx, rank, world):
    """Cells [i0, i1) of the x axis owned by `rank` (nx grid planes -> nx-1 cells)."""
    cells = nx - 1
    base, rem = divmod(cells, world)
    i0 = rank * base + min(rank, rem)
    i1 = i0 + base + (1 if rank < rem else 0)
    return i0, i1


def _default_mc(sdf, step, origin, iso, i_offset):
    from . import ops
    return ops.marching_cubes(sdf, step[0], step[1], step[2], origin[0], origin[1], origin[2], iso,
                              i_offset)


def _default_count(sdf, iso):
    from . import ops
    return ops.marching_cubes_count(sdf, iso)


def sharded_marching_cubes(sdf, step, origin, iso=0.0, rank=0, world=1, group=None, mc_fn=None, count_fn=None,
                           gather_to=None):
    """Marching cubes over x-slabs, stitched to the single-device result.

    `sdf` [nx,ny,nz]: this rank only reads planes [i0, i1+2) of it (its cells plus the halo that
    makes the cells at plane i1 -- owned by the next rank -- valid), so callers may pass a tensor
    whose other planes were never evaluated.  Returns (vertices [V,3], faces [F,3] int64) of the
    WHOLE mesh (on every rank, or only on rank `gather_to`; the others then get empty tensors), in the canonical
    order of the single-device kernel:
      - vertices owned by cells i < i1 of this rank keep their local order;
      - a reference to a vertex owned by a halo cell (plane i1) is rebased onto the next rank's
        first vertices: the halo cells produce the same vertices, in the same order, there.
    ONE emit pass per rank (slab + halo); how many of its vertices / faces belong to the rank's own cells comes
    from a count-only pass over the slab without the halo (classification only, no emission).  The pieces travel
    unpadded: one all-gather of the four counts, then per source rank one broadcast (or one send to `gather_to`)
    of exactly its vertices and faces.
    mc_fn(sdf, step, origin, iso, i_offset) -> (verts, faces) must be deterministic and canonical;
    count_fn(sdf, iso) -> (n_vertices, n_faces) of the same kernel."""
    mc_fn = mc_fn or _default_mc
    nx = sdf.shape[0]
    i0, i1 = slab_range(nx, rank, world)
    last = (rank == world - 1)
    # the slab keeps the GLOBAL x index (i_offset) so positions are bit-identical to one device
    if last or world == 1:
        loc_v, loc_f = mc_fn(sdf[i0:i1 + 1].contiguous(), step, origin, iso, i0)
        V_own, F_own = loc_v.shape[0], loc_f.shape[0]
    else:
        loc_v, loc_f = mc_fn(sdf[i0:i1 + 2].contiguous(), step, origin, iso, i0)  # own cells + halo cells at i1
        if count_fn is None and mc_fn is _default_mc:
            count_fn = _default_count
        if count_fn is not None:
            V_own, F_own = count_fn(sdf[i0:i1 + 1].contiguous(), iso)             # cells i0 .. i1-1
        else:
            ov, of = mc_fn(sdf[i0:i1 + 1].contiguous(), step, origin, iso, i0)
            V_own, F_own = ov.shape[0], of.shape[0]
    faces = loc_f[:F_own]
    verts = loc_v[:V_own]
    if world == 1:
        return verts, faces
    dev = sdf.device
    counts = torch.tensor([V_own, F_own], dtype=torch.int64, device=dev)
    allc = [torch.zeros_like(counts) for _ in range(world)]
    dist.all_gather(allc, counts, group=group)
    allc = torch.stack(allc).cpu()
    voff = torch.cat([torch.zeros(1, dtype=torch.int64), allc[:, 0].cumsum(0)])
    # rebase: own vertices -> voff[rank] + id ; halo vertices -> voff[rank+1] + (id - V_own)
    f = faces.clone()
    halo = f >= V_own
    f = torch.where(f < 0, f, torch.where(halo, f - V_own + int(voff[min(rank + 1, world)]), f + int(voff[rank])))
    verts = verts.contiguous()
    out_v, out_f = [], []
    for r in range(world):
        nv, nf = int(allc[r, 0]), int(allc[r, 1])
        if gather_to is None:
            bv = verts if r == rank else torch.empty((nv, 3), dtype=verts.dtype, device=dev)
            bf = f if r == rank else torch.empty((nf, 3), dtype=torch.int64, device=dev)
            if nv:
                dist.broadcast(bv, src=r, group=group)
            if nf:
                dist.broadcast(bf, src=r, group=group)
            out_v.append(bv)
            out_f.append(bf)
        elif rank == gather_to:
            if r == rank:
                out_v.append(verts)
                out_f.append(f)
            else:
                bv = torch.empty((nv, 3), dtype=verts.dtype, device=dev)
                bf = torch.empty((nf, 3), dtype=torch.int64, device=dev)
                if nv:
                    dist.recv(bv, src=r, group=group)
                if nf:
                    dist.recv(bf, src=r, group=group)
                out_v.append(bv)
                out_f.append(bf)
        elif r == rank:
            if nv:
                dist.send(verts, dst=gather_to, group=group)
            if nf:
                dist.send(f, dst=gather_to, group=group)
    if gather_to is not None and rank != gather_to:
        return verts.new_zeros((0, 3)), f.new_zeros((0, 3))
    return torch.cat(out_v), torch.cat(out_f)
