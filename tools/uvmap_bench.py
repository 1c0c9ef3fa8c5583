"""Device time and quality of the template simplification and UV atlas (selfreconcode_b200.uvmap) at infer.py's
settings: the synthetic body SDF (synth.make_sdf) extracted with Seg3dLossless + marching cubes on the reference's
coarse ladder ending at 225x321x129, simplified to 30 000 faces and unwrapped at 1680^2.  CUDA events around each
stage, median of 3 after one warm-up; faces in / out, rounds, charts, utilisation and stretch; the geometric error as
|f| of the SDF network at the simplified vertices and face centroids beside the marching-cubes mesh's own.  Prints the
card and its power limit first, then one JSON line.

    python tools/uvmap_bench.py [--faces 30000] [--resolution 1680]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))


def _timed(fn, reps=3):
    fn()
    torch.cuda.synchronize()
    ts, out = [], None
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        out = fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2], out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--faces", type=int, default=30000)
    ap.add_argument("--resolution", type=int, default=1680)
    ap.add_argument("--padding", type=int, default=4)
    ap.add_argument("--max-angle", type=float, default=60.)
    a = ap.parse_args()
    import helpers as H
    from mesh_reg_bench import REF_COARSE, _card
    from test_gpu_mesh_reg import template
    from test_gpu_mesh_shade import _scene
    from selfreconcode_b200 import uvmap
    card = _card()
    print(card)
    v, f = template(REF_COARSE)
    sdf = _scene(32, 32, 1)[0].sdf

    def err(V, F):
        with torch.no_grad():
            pts = torch.cat([V, V[F].mean(1)]).contiguous()
            s = sdf.forward_fused(pts, H.RATIO, want_grad=False, want_feat=False)[0].view(-1).abs().double()
        nv = V.shape[0]
        q = lambda x: float(torch.quantile(x[:min(x.numel(), 1 << 24)], 0.999))
        return dict(vert_max=float(s[:nv].max()), vert_p999=q(s[:nv]), centroid_max=float(s[nv:].max()),
                    centroid_p999=q(s[nv:]))

    t_simp, (V, F, sinfo) = _timed(lambda: uvmap.simplify(v, f, faces=a.faces))
    t_unwrap, (vt, ft, uinfo) = _timed(lambda: uvmap.unwrap(V, F, a.resolution, a.padding, a.max_angle))
    res = dict(card=card, grid=list(REF_COARSE[-1]), faces_in=sinfo["faces_in"], faces_out=sinfo["faces_out"],
               dropped_faces=sinfo["dropped_faces"], rounds=sinfo["rounds"], stop=sinfo["stop"],
               simplify_ms=round(t_simp, 2), unwrap_ms=round(t_unwrap, 2), charts=uinfo["charts"],
               splits=uinfo["splits"], uv_vertices=vt.shape[0], utilisation=round(uinfo["utilisation"], 4),
               stretch_min=round(uinfo["stretch_min"], 4), stretch_max=round(uinfo["stretch_max"], 4),
               sdf_err_mc=err(v, f[(f >= 0).all(1)]), sdf_err_simplified=err(V, F))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
