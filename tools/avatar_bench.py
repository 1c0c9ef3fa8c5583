"""Device time of the textured avatar (selfreconcode_b200.avatar) at a production size: the synthetic body of
tools/uvmap_bench.py (the reference's coarse ladder ending at 225x321x129, simplified to 30 000 faces and unwrapped at
1680^2), a 1680^2 atlas, 120 frames at 1080x1080 in batches of 8 under the synthetic sequence's deformer and camera.
CUDA events per stage and batch (deform, screen + raster, shade, uint8 conversion with readback), summed over the
sequence after one warm-up pass; the one-time mip build; frames/s of render_motion end to end with PNG and video
encoding.  Prints the card and its power limit first, then one JSON line.

    python tools/avatar_bench.py [--frames 120] [--side 1080] [--batch 8]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=120)
    ap.add_argument("--side", type=int, default=1080)
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--faces", type=int, default=30000)
    ap.add_argument("--resolution", type=int, default=1680)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "avatar_bench measures on the GPU"
    import cv2
    from mesh_reg_bench import REF_COARSE, _card
    from test_gpu_avatar import mixed_texture
    from test_gpu_mesh_reg import template
    from test_gpu_mesh_shade import _scene
    from selfreconcode_b200 import avatar, ops, uvmap
    card = _card()
    print(card)
    net, data, cams, _, _, _ = _scene(a.side, a.side, a.frames)
    v, f = template(REF_COARSE)
    V, F, _ = uvmap.simplify(v, f, faces=a.faces)
    vt, ft, _ = uvmap.unwrap(V, F, a.resolution)
    tmp = tempfile.mkdtemp(prefix="avatar_bench_")
    obj = os.path.join(tmp, "uvmap.obj")
    uvmap.write_obj(obj, V, F, vt, ft)
    png = os.path.join(tmp, "texture.png")
    cv2.imwrite(png, mixed_texture(a.resolution))
    av = avatar.TexturedAvatar(obj, png, "cuda")
    Ht, Wt = av.atlas.shape[:2]

    def mips():
        return ops.texture_mips(av.atlas, av.coverage)
    mips()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        mips()
    e1.record()
    torch.cuda.synchronize()
    t_mips = e0.elapsed_time(e1) / 10

    from model.raster import screen_vertices
    B, n, side = a.batch, a.frames, a.side
    bg = torch.randint(0, 256, (B, side, side, 3), dtype=torch.uint8, device="cuda")

    def sequence(times):
        for b in range(0, n, B):
            ids = torch.arange(b, min(b + B, n), device="cuda")
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
            ev[0].record()
            poses, trans, d_cond, _ = data.get_grad_parameters(ids, "cuda")
            verts = avatar.pose_vertices(net, av.V, poses.detach(), trans.detach(), d_cond.detach())
            ev[1].record()
            s = screen_vertices(verts, cams).contiguous()
            p2f, bary, _ = ops.raster_mesh(s, av.faces, side, side)
            ev[2].record()
            out = ops.shade_textured(p2f[..., 0], bary[..., 0, :], s, av.faces, av.ft, av.vt, av.mips, av.levels,
                                     bg[:ids.numel()])
            ev[3].record()
            host = torch.round(out[..., :3].clamp(0., 1.) * 255.).to(torch.uint8).cpu()
            ev[4].record()
            torch.cuda.synchronize()
            for k, name in enumerate(("deform", "screen_raster", "shade", "to_uint8_readback")):
                times[name] = times.get(name, 0.) + ev[k].elapsed_time(ev[k + 1])
        return host
    sequence({})
    stages = {}
    sequence(stages)
    covered = float((ops.raster_mesh(screen_vertices(avatar.pose_vertices(
        net, av.V, *[t.detach() for t in data.get_grad_parameters(torch.arange(1, device="cuda"), "cuda")[:3]]), cams),
        av.faces, side, side)[0] >= 0).float().mean())
    poses = data.poses.detach()[:n]
    trans = data.trans.detach()[:n]
    out_dir = os.path.join(tmp, "motion")
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    avatar.render_motion(net, av, out_dir, poses, trans, cond_frame=0, batch=B)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    px = n * side * side
    res = dict(card=card, frames=n, side=side, batch=B, faces=int(F.shape[0]), atlas=[int(Ht), int(Wt)],
               levels=int(av.levels.shape[0]), mips_ms=round(t_mips, 3),
               stage_ms_per_frame={k: round(t / n, 4) for k, t in stages.items()},
               shade_GBps=round(36. * px / (stages["shade"] * 1e-3) / 1e9, 1), covered_fraction=round(covered, 4),
               frames_per_s_with_encode=round(n / wall, 2))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
