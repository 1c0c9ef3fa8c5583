"""Float64 numpy restatement of pytorch3d's vertex normals and HardPhongShader (test infrastructure).

pytorch3d itself is absent, so the shading kernels (csrc/mesh_shade.cu) are pinned to this restatement of its
published rules, the same status the mesh rasteriser has (oracle.raster_mesh):
  * Meshes.verts_normals_packed: face normal (v2-v1) x (v0-v1), summed over incident faces, F.normalize(eps=1e-6);
  * phong_shading + hard_rgb_blend with faces_per_pixel = 1 (pytorch3d/renderer/mesh/shading.py, lighting.py,
    blending.py).  The fragments are taken as given."""
import numpy as np


def _normalize(x, eps=1e-6):
    return x / np.maximum(np.linalg.norm(x, axis=-1, keepdims=True), eps)


def vertex_normals_p3d(verts, faces, unit_faces=False):
    """verts [V,3] or [N,V,3] -> normals of the same shape.  unit_faces=True sums UNIT face normals instead (the
    openmesh rule of utils.compute_vnorms), which is not pytorch3d's rule."""
    v = np.asarray(verts, dtype=np.float64)
    fc = np.asarray(faces, dtype=np.int64)
    single = v.ndim == 2
    v = v[None] if single else v
    out = np.zeros_like(v)
    for n in range(v.shape[0]):
        a, b, c = v[n][fc[:, 0]], v[n][fc[:, 1]], v[n][fc[:, 2]]
        fn = np.cross(c - b, a - b)
        if unit_faces:
            fn = _normalize(fn, 1e-12)
        s = np.zeros_like(v[n])
        for k in range(3):
            np.add.at(s, fc[:, k], fn)
        out[n] = _normalize(s)
    return out[0] if single else out


def shade_phong_p3d(verts, normals, faces, pix_to_face, bary, cam_pos, light_pos, colors=None,
                    light_ambient=(0.5,) * 3, light_diffuse=(0.3,) * 3, light_specular=(0.2,) * 3,
                    mat_ambient=(1.,) * 3, mat_diffuse=(1.,) * 3, mat_specular=(1.,) * 3, shininess=64.,
                    background=(1., 1., 1.), specular=True):
    """verts / normals / colors [N,V,3], faces [F,3], pix_to_face [N,H,W] packed (n*F + f, -1 empty), bary [N,H,W,3],
    cam_pos / light_pos [N,3] -> (images [N,H,W,4] float64, terms dict with per-pixel 'cos' (n.l), 'diffuse' and
    'specular' [N,H,W,3], zero on background).  specular=False drops the specular term (a negative control)."""
    vs = np.asarray(verts, dtype=np.float64)
    nr = np.asarray(normals, dtype=np.float64)
    fc = np.asarray(faces, dtype=np.int64)
    p2f = np.asarray(pix_to_face, dtype=np.int64).reshape(vs.shape[0], *np.shape(pix_to_face)[1:3])
    N, H, W = p2f.shape
    br = np.asarray(bary, dtype=np.float64).reshape(N, H, W, 3)
    F = fc.shape[0]
    col = np.ones_like(vs) if colors is None else np.asarray(colors, dtype=np.float64)
    img = np.zeros((N, H, W, 4))
    img[..., :3] = np.asarray(background, dtype=np.float64)
    terms = {k: np.zeros((N, H, W, 3)) for k in ("diffuse", "specular")}
    terms["cos"] = np.zeros((N, H, W))
    cov = p2f >= 0
    nn, rr, cc = np.nonzero(cov)
    pf = p2f[cov]
    m, f = pf // F, pf % F
    b = br[cov]                                         # [P,3]
    idx = fc[f]                                         # [P,3]

    def interp(attr):
        return (attr[m[:, None], idx] * b[..., None]).sum(1)

    p, nrm, tex = interp(vs), _normalize(interp(nr)), interp(col)
    l = _normalize(np.asarray(light_pos, dtype=np.float64)[nn] - p)
    v = _normalize(np.asarray(cam_pos, dtype=np.float64)[nn] - p)
    cos = (nrm * l).sum(-1)
    diffuse = np.asarray(light_diffuse) * np.maximum(cos, 0.)[:, None]
    r = -l + 2 * cos[:, None] * nrm
    alpha = np.maximum((v * r).sum(-1), 0.) * (cos > 0)
    spec = np.asarray(light_specular) * (alpha ** shininess)[:, None]
    if not specular:
        spec = np.zeros_like(spec)
    rgb = (np.asarray(mat_ambient) * np.asarray(light_ambient) + np.asarray(mat_diffuse) * diffuse) * tex \
        + np.asarray(mat_specular) * spec
    img[nn, rr, cc, :3] = rgb
    img[nn, rr, cc, 3] = 1.
    terms["cos"][nn, rr, cc] = cos
    terms["diffuse"][nn, rr, cc] = diffuse
    terms["specular"][nn, rr, cc] = spec
    return img, terms
