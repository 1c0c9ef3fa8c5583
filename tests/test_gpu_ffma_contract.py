"""GPU: the fused fp32 FFMA field engine (csrc/mlp_core.cuh, csrc/mlp_kernels.cu) against its float64 restatement
(tests/ffma_ref.py, oracle/oracle.py in float64) at every kind of network validate_net accepts, and at batch sizes
that give a CTA one partial tile, several tiles (the weight ring's slot and phase carried across tiles), or none.

  * networks are folded by ops.FusedMLP from seeded weight-normed layers, so the fold kernel is covered too;
  * outputs land in sentinel-filled buffers padded past P: nothing past P may change;
  * bars: elem_err < 1e-4 on every floating-point output, also norm_err < 1e-5 on values (f, offset, D, rgb);
    ReLU networks exclude (and count) points with a unit whose float64 pre-activation is within 1e-5 of 0;
  * invariances, bitwise: a row's arithmetic does not depend on its tile or CTA (permutation, a prefix alone, rerun);
  * argument checks, and the tensor-core engine's refusal of networks with more than one skip layer.

Every measured maximum is printed beside its bar (pytest -s)."""
import ctypes as C

import pytest
import torch

import ffma_ref as R
from helpers import SMPL_PARENTS, elem_err, golden, norm_err
from oracle import oracle as O

pytestmark = pytest.mark.gpu

ELEM, NORM = 1e-4, 1e-5
RELU_MARGIN = 1e-5
NSM = 132
# per point-count kind: T = 3 kernels hold 16 points per tile, T = 0 kernels 64; the last size gives every CTA two
# full tiles and a few CTAs a third
SIZES = {3: (1, 15, 17, 63, 65, 16 * NSM * 2 + 5), 0: (1, 15, 17, 63, 65, 64 * NSM * 2 + 7)}
PAD = 37
SENT = 0x7FA5A5A5            # a NaN bit pattern: any output left unwritten poisons the comparison


def _lib():
    from selfreconcode_b200 import _lib as L
    return L.load()


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _s():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def sentinel(n, dev, dtype=torch.float32):
    return torch.full((int(n) + PAD,), SENT, dtype=torch.int32, device=dev).view(dtype)


def untouched(buf, n):
    """Nothing past the first n elements was written."""
    return bool((buf[n:].view(torch.int32) == SENT).all())


def report(name, got, ref, value, keep=None):
    got, ref = got.detach().double().cpu().numpy(), ref.detach().double().cpu().numpy()
    if keep is not None:
        k = keep.cpu().numpy()
        got, ref = got[k], ref[k]
    if ref.size == 0:
        print("  %-40s (every point excluded)" % name)
        return
    e, n = elem_err(got, ref), norm_err(got, ref)
    print("  %-40s elem %.2e  norm %.2e" % (name, e, n))
    assert e < ELEM, (name, e)
    if value:
        assert n < NORM, (name, n)


# ---------------------------------------------------------------------------------------------------------------------
# networks
# ---------------------------------------------------------------------------------------------------------------------
TARGET = {R.SP: 0.02, R.TANH: 0.8, R.RELU: 4.0, R.NONE: 0.5}   # softplus(beta=100): |100 z| = O(1), mixed


def scaled_layers(ns, inp, skips, hidden, last, seed, dev, last_target=None):
    """Weight-normed layers (v, g, b) whose float64 pre-activations on the sample `inp` have a set spread per
    activation: softplus(beta = 100) units sit where 100 z is O(1), tanh units off their saturated tails."""
    g = torch.Generator().manual_seed(seed)
    h, layers = inp, []
    for l, n in enumerate(ns):
        skip = l in skips
        if skip:
            h = torch.cat([h, inp], 1) * R.INV_SQRT2
        act = hidden if l < len(ns) - 1 else last
        v = torch.randn(n, h.shape[1], generator=g, dtype=torch.float64)
        tgt = TARGET[act] if (l < len(ns) - 1 or last_target is None) else last_target
        z = h @ v.t()
        c = tgt / float(z.std())
        b = 0.3 * tgt * torch.randn(n, generator=g, dtype=torch.float64)
        layers.append(dict(v=v.float().to(dev), g=(c * v.norm(dim=1)).float().to(dev), b=b.float().to(dev),
                           act=act, skip=skip))
        h = R.activation(act, c * z + b)
    return layers


class Net:
    """A folded network and the layer list it was folded from."""

    def __init__(self, layers, d_in, multires, pe_w, dev):
        from selfreconcode_b200 import ops
        self.layers, self.d_in, self.multires, self.pe_w = layers, d_in, multires, list(pe_w)
        self.fused = ops.FusedMLP(d_in, multires, dev).fold(layers, self.pe_w)

    @property
    def desc(self):
        return self.fused.desc


def _sample(n, seed, lo=-1.0, hi=1.0):
    g = torch.Generator().manual_seed(seed)
    return lo + (hi - lo) * torch.rand(n, 3, generator=g)


# name: (widths, multires, skips, hidden act, band-weight ratio)
SDF_GEOMS = {
    "ragged": ([200, 129, 383, 1], 4, {2}, R.SP, 0.6),          # GP 2/2/3/1, kpad 160, 97 slices per tile
    "deep_two_skip": ([64] * 11 + [1], 0, {4, 8}, R.TANH, None),  # 12 layers, multires 0 (kpad 8), two skips
    "one_layer": ([1], 6, set(), R.NONE, None),
    "wide_pe": ([256, 256, 1], 10, set(), R.SP, None),            # tangent x 512 on the top band
    "sp_two_skip": ([64] * 5 + [1], 0, {2, 4}, R.SP, None),       # two skips on a net the tensor-core reverse takes
}


def sdf_net(name, dev):
    if name == "ref_sdf":          # the production network (geometric init, 9 layers, skip at 4), band weights annealed
        from selfreconcode_b200 import synth
        from helpers import sdf_params
        sp = sdf_params(synth.make_sdf())
        layers = [dict(v=v.to(dev), g=g.view(-1).to(dev), b=b.to(dev), act=R.SP if l < len(sp) - 1 else R.NONE,
                       skip=l == 4) for l, (v, g, b) in enumerate(sp)]
        return Net(layers, 39, 6, R.annealing_weights(6, 0.8), dev)
    ns, m, skips, act, ratio = SDF_GEOMS[name]
    pe_w = R.annealing_weights(m, ratio)
    inp = R.embed(_sample(2048, 5), m, pe_w)
    return Net(scaled_layers(ns, inp, skips, act, R.NONE, 17 + len(ns), dev), 3 + 6 * m, m, pe_w, dev)


CONDLEN, NFRAMES = 128, 3


def conds(dev):
    return (0.5 * torch.randn(NFRAMES, CONDLEN, generator=torch.Generator().manual_seed(9))).to(dev)


def translator_net(name, dev):
    """The reference translator (512 x 4 + 3, kpad0 168), a narrow one, or one with a zero output layer (D = LBS(p):
    points can then sit exactly on the skinning grid's voxel faces)."""
    ns = {"translator_ref": [512] * 4 + [3], "translator_300": [300, 3], "zero_offset": [300, 3],
          "translator_9": [64] * 8 + [3]}[name]
    pe_w = R.annealing_weights(6, 0.8)
    cd = conds("cpu").double()
    x = _sample(2048, 6)
    inp = torch.cat([R.embed(x, 6, pe_w), cd[torch.arange(2048) % NFRAMES]], 1)
    layers = scaled_layers(ns, inp, set(), R.RELU, R.NONE, 29 + len(ns), dev, last_target=0.05)
    if name == "zero_offset":
        layers[-1]["g"].zero_()
        layers[-1]["b"].zero_()
    return Net(layers, 39 + CONDLEN, 6, pe_w, dev)


def lbs_setup(dev):
    """Product LbsState and the float64 oracle's inputs from the deform.npz skinning volume, 3 frames."""
    from selfreconcode_b200 import ops
    g = golden("deform.npz")
    Js = torch.from_numpy(g["Js"]).double()
    ipi = O.init_pose_inverse(torch.from_numpy(g["apose"]).double(), Js, SMPL_PARENTS)
    poses, trans = torch.from_numpy(g["poses"]), torch.from_numpy(g["trans"])
    st = ops.LbsState(torch.from_numpy(g["ws"]).to(dev), torch.from_numpy(g["bmin"]), torch.from_numpy(g["bmax"]),
                      Js.float().to(dev), SMPL_PARENTS, ipi.float().to(dev))
    st.set_pose(poses.to(dev), trans.to(dev))
    A, _ = O.bone_transforms(poses.double(), Js, SMPL_PARENTS, ipi.float().double())
    ref = dict(ws=torch.from_numpy(g["ws"]).double().to(dev), bmin=torch.from_numpy(g["bmin"]).double().to(dev),
               bmax=torch.from_numpy(g["bmax"]).double().to(dev), A=A.to(dev), trans=trans.double().to(dev))
    return st, ref


def deform_ref(net, lbs, cd, frame):
    """x -> (D(x), offset(x)) in float64, differentiable; and the ReLU margin of the translator."""
    def fn(x):
        off = R.translator_offset(net.layers, x, 6, net.pe_w, cd, frame)
        p1 = x + off
        if lbs is None:
            return p1
        return O.lbs_forward(lbs["ws"], lbs["bmin"], lbs["bmax"], lbs["A"], lbs["trans"], p1, frame)
    return fn


def relu_keep(net, x, cd, frame):
    _, zs = R.translator_offset(net.layers, x.double(), 6, net.pe_w, cd, frame, with_preacts=True)
    return R.min_relu_margin(net.layers, zs) >= RELU_MARGIN


def lbs_pixel(lbs, p1):
    """float64 grid coordinate (x, y, z order: W, H, D) of deformed points, before the border clamp."""
    size = torch.tensor([lbs["ws"].shape[4], lbs["ws"].shape[3], lbs["ws"].shape[2]], dtype=torch.float64,
                        device=p1.device)
    u = 2.0 * (p1 - lbs["bmin"]) / (lbs["bmax"] - lbs["bmin"]) - 1.0
    return ((u + 1.0) * size - 1.0) / 2.0, size


def lbs_keep(lbs, p1):
    """Points farther than 1e-6 (in space) from every voxel face and border-clamp plane: there D(p) is smooth and
    the corner index is decided by more than rounding."""
    x, size = lbs_pixel(lbs, p1)
    world = (lbs["bmax"] - lbs["bmin"]) / size                      # one pixel, in space
    near_face = ((x - x.round()).abs() * world < 1e-6) & (x > -1.0) & (x < size)
    return ~near_face.any(1), x.clamp(min=0.0).minimum(size - 1).floor().long()


# ---------------------------------------------------------------------------------------------------------------------
# raw launches into sentinel buffers
# ---------------------------------------------------------------------------------------------------------------------
def run_sdf(net, pts, T, nfeat=0):
    lib, dev, P = _lib(), pts.device, pts.shape[0]
    f = sentinel(P, dev)
    g = sentinel(3 * P, dev) if T == 3 else None
    ft = sentinel(nfeat * P, dev) if nfeat else None
    assert lib.sr_sdf_forward(C.byref(net.desc), _p(pts), P, _p(f), _p(g), _p(ft), nfeat, _s()) == 0
    torch.cuda.synchronize()
    assert untouched(f, P) and (g is None or untouched(g, 3 * P)) and (ft is None or untouched(ft, nfeat * P))
    return f[:P], (g[:3 * P].view(P, 3) if g is not None else None), (ft[:nfeat * P].view(P, nfeat) if nfeat else None)


def run_deform(net, lbs, pts, bi, ppf, cd, T):
    lib, dev, P = _lib(), pts.device, pts.shape[0]
    d, off, ci = sentinel(3 * P, dev), sentinel(3 * P, dev), sentinel(3 * P, dev, torch.int32)
    jac = sentinel(9 * P, dev) if T == 3 else None
    assert lib.sr_deform_forward(C.byref(net.desc), C.byref(lbs.params) if lbs is not None else None, _p(pts),
                                 _p(bi), ppf, _p(cd), CONDLEN, P, _p(d), _p(off), _p(jac), _p(ci), _s()) == 0
    torch.cuda.synchronize()
    for b, n in ((d, 3 * P), (off, 3 * P), (ci, 3 * P), (jac, 9 * P)):
        assert b is None or untouched(b, n)
    return (d[:3 * P].view(P, 3), off[:3 * P].view(P, 3), jac[:9 * P].view(P, 3, 3) if T == 3 else None,
            ci[:3 * P].view(P, 3))


def run_render(net, pts, nrm, views, feat):
    lib, dev, P = _lib(), pts.device, pts.shape[0]
    nfeat = feat.shape[1] if feat is not None else 0
    rgb = sentinel(3 * P, dev)
    assert lib.sr_render_forward(C.byref(net.desc), _p(pts), _p(nrm), _p(views), _p(feat), nfeat, P, _p(rgb),
                                 _s()) == 0
    torch.cuda.synchronize()
    assert untouched(rgb, 3 * P)
    return rgb[:3 * P].view(P, 3)


def run_shade(sdf, dnet, lbs, pts, rays, bi, cd):
    lib, dev, P = _lib(), pts.device, pts.shape[0]
    nrm, cr, dp = sentinel(3 * P, dev), sentinel(3 * P, dev), sentinel(3 * P, dev)
    ok = torch.full((P + PAD,), 0xA5, dtype=torch.uint8, device=dev)
    assert lib.sr_shade_geometry(C.byref(sdf.desc), C.byref(dnet.desc) if dnet is not None else None,
                                 C.byref(lbs.params) if lbs is not None else None, _p(pts), _p(rays), _p(bi), _p(cd),
                                 CONDLEN if dnet is not None else 0, P, _p(nrm), _p(cr), None, 0, _p(dp), _p(ok),
                                 _s()) == 0
    torch.cuda.synchronize()
    assert untouched(nrm, 3 * P) and untouched(cr, 3 * P) and untouched(dp, 3 * P) and bool((ok[P:] == 0xA5).all())
    return nrm[:3 * P].view(P, 3), cr[:3 * P].view(P, 3), dp[:3 * P].view(P, 3), ok[:P]


# ---------------------------------------------------------------------------------------------------------------------
# sdf_kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [0, 3])
@pytest.mark.parametrize("name", ["ref_sdf"] + list(SDF_GEOMS))
def test_sdf_forward_matches_fp64(cuda_dev, name, T):
    net = sdf_net(name, cuda_dev)
    pts = _sample(SIZES[T][-1], 100 + T).to(cuda_dev)
    f64, g64, out64 = R.sdf(net.layers, pts, net.multires, net.pe_w, want_grad=T == 3)
    print("sdf_forward %s T=%d" % (name, T))
    for nfeat in ((0, 256) if name == "ref_sdf" else (0,)):
        for P in SIZES[T]:
            f, g, ft = run_sdf(net, pts[:P], T, nfeat)
            tag = "P=%d%s" % (P, " feat" if nfeat else "")
            report("f " + tag, f, f64[:P], True)
            if T == 3:
                report("grad f " + tag, g, g64[:P], False)
            if nfeat:
                report("feat " + tag, ft, out64[:P, 1:], True)


# ---------------------------------------------------------------------------------------------------------------------
# deform_kernel, bone transforms
# ---------------------------------------------------------------------------------------------------------------------
def _deform_points(n, dev, lbs_ref, seed, faces):
    """Points over the skinning box grown by 30 % on every side (border clamp); with `faces`, a quarter of them moved
    onto voxel faces along one axis."""
    lo, hi = lbs_ref["bmin"].float().cpu(), lbs_ref["bmax"].float().cpu()
    ext = hi - lo
    g = torch.Generator().manual_seed(seed)
    x = lo - 0.3 * ext + 1.6 * ext * torch.rand(n, 3, generator=g)
    if faces:
        size = torch.tensor([lbs_ref["ws"].shape[4], lbs_ref["ws"].shape[3], lbs_ref["ws"].shape[2]])
        sel = torch.arange(n) % 4 == 0
        ax = torch.randint(0, 3, (n,), generator=g)
        k = torch.randint(0, 100, (n,), generator=g) % size[ax]
        face = lo[ax] + ext[ax] * (k.float() + 0.5) / size[ax].float()   # pixel coordinate k exactly, in float64
        x[sel, ax[sel]] = face[sel]
    return x.to(dev)


@pytest.mark.parametrize("T", [0, 3])
@pytest.mark.parametrize("name,with_lbs", [("translator_ref", True), ("translator_ref", False),
                                           ("translator_300", True), ("translator_300", False),
                                           ("zero_offset", True)])
def test_deform_forward_matches_fp64(cuda_dev, name, with_lbs, T):
    net = translator_net(name, cuda_dev)
    st, lref = lbs_setup(cuda_dev)
    cd = conds(cuda_dev)
    Pmax = SIZES[T][-1]
    pts = _deform_points(Pmax, cuda_dev, lref, 200 + T, faces=name == "zero_offset")
    bi_all = torch.randint(0, NFRAMES, (Pmax,), generator=torch.Generator().manual_seed(3)).to(cuda_dev)
    print("deform_forward %s lbs=%d T=%d" % (name, with_lbs, T))
    excluded = [0, 0]
    for P in SIZES[T]:
        for mode in ("batch_inds", "pts_per_frame"):
            if mode == "batch_inds":
                bi, ppf, frame = bi_all[:P], 0, bi_all[:P]
            else:
                ppf = -(-P // NFRAMES)
                bi, frame = None, torch.arange(P, device=cuda_dev) // ppf
            x = pts[:P]
            d, off, jac, ci = run_deform(net, st if with_lbs else None, x, bi, ppf, cd, T)
            fn = deform_ref(net, lref if with_lbs else None, cd, frame)
            d64, J64 = R.jacobian(fn, x)
            off64 = R.translator_offset(net.layers, x.double(), 6, net.pe_w, cd, frame)
            keep = relu_keep(net, x, cd, frame)
            smooth = keep.clone()
            if with_lbs:
                lk, ci64 = lbs_keep(lref, x.double() + off64)
                smooth &= lk
                assert torch.equal(ci[smooth].long(), ci64[smooth]), "corner indices"
            excluded[0] += int((~keep).sum())
            excluded[1] += int((keep & ~smooth).sum())
            tag = "P=%d %s" % (P, mode)
            report("D " + tag, d, d64, True, keep)
            report("offset " + tag, off, off64, True, keep)
            if T == 3:
                report("jacobian " + tag, jac, J64, False, smooth)
    total = 2 * sum(SIZES[T])
    print("  excluded: %d points near a ReLU kink, %d more near a voxel face or clamp plane (of %d)"
          % (excluded[0], excluded[1], total))
    assert excluded[0] < 0.01 * total
    if name == "zero_offset":
        assert excluded[1] > total // 8, "the face points must be excluded from the Jacobian"


def test_bone_transforms_match_fp64(cuda_dev):
    """Zero pose (the +1e-8 of batch_rodrigues), rotation angles above pi, the fixture's poses; with and without the
    init-pose inverse."""
    lib = _lib()
    g = golden("deform.npz")
    Js = torch.from_numpy(g["Js"]).double()
    ipi = O.init_pose_inverse(torch.from_numpy(g["apose"]).double(), Js, SMPL_PARENTS).float()
    gen = torch.Generator().manual_seed(4)
    axis = torch.nn.functional.normalize(torch.randn(24, 3, generator=gen, dtype=torch.float64), dim=1)
    big = axis * (3.3 + 2.5 * torch.rand(24, 1, generator=gen, dtype=torch.float64))
    poses = torch.cat([torch.zeros(1, 24, 3, dtype=torch.float64), big[None], torch.from_numpy(g["poses"]).double()])
    F = poses.shape[0]
    parents = torch.as_tensor(SMPL_PARENTS, dtype=torch.int32, device=cuda_dev)
    for name, inv in (("init-pose inverse", ipi), ("rest joints", None)):
        A, pj = sentinel(F * 24 * 16, cuda_dev), sentinel(F * 24 * 3, cuda_dev)
        assert lib.sr_lbs_bone_transforms(_p(poses.float().to(cuda_dev)), _p(Js.float().to(cuda_dev)), _p(parents),
                                          _p(inv.to(cuda_dev) if inv is not None else None), F, _p(A), _p(pj),
                                          _s()) == 0
        torch.cuda.synchronize()
        assert untouched(A, F * 384) and untouched(pj, F * 72)
        A64, posed64 = O.bone_transforms(poses.float().double(), Js.float().double(), SMPL_PARENTS,
                                         inv.double() if inv is not None else None)
        print("bone transforms, %s" % name)
        report("A", A[:F * 384].view(F, 24, 4, 4), A64, True)
        report("posed joints", pj[:F * 72].view(F, 24, 3), posed64, True)


# ---------------------------------------------------------------------------------------------------------------------
# render_kernel
# ---------------------------------------------------------------------------------------------------------------------
RENDER_GEOMS = {"render_ref": ([512] * 4 + [3], 4, 256, 0.8), "render_small": ([128, 3], 0, 0, None)}


def render_net(name, dev):
    ns, m, nfeat, ratio = RENDER_GEOMS[name]
    pe_w = R.annealing_weights(m, ratio)
    g = torch.Generator().manual_seed(12)
    inp = torch.cat([torch.rand(2048, 3, generator=g, dtype=torch.float64), R.embed(torch.randn(2048, 3, generator=g),
                     m, pe_w), torch.randn(2048, 3 + nfeat, generator=g, dtype=torch.float64)], 1)
    layers = scaled_layers(ns, inp, set(), R.RELU, R.TANH, 41 + len(ns), dev)
    return Net(layers, inp.shape[1], m, pe_w, dev), nfeat


def render_inputs(P, nfeat, dev, seed):
    g = torch.Generator().manual_seed(seed)
    pts = torch.rand(P, 3, generator=g)
    nrm = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=1)
    views = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=1)
    feat = torch.randn(P, nfeat, generator=g) if nfeat else None
    return [t.to(dev) if t is not None else None for t in (pts, nrm, views, feat)]


@pytest.mark.parametrize("name", list(RENDER_GEOMS))
def test_render_forward_matches_fp64(cuda_dev, name):
    net, nfeat = render_net(name, cuda_dev)
    pts, nrm, views, feat = render_inputs(SIZES[0][-1], nfeat, cuda_dev, 77)
    rgb64, margin = R.render(net.layers, pts, nrm, views, feat, net.multires, net.pe_w)
    keep = margin >= RELU_MARGIN
    print("render_forward %s: %d of %d points near a ReLU kink excluded" % (name, int((~keep).sum()), keep.numel()))
    assert (~keep).float().mean() < 0.01
    for P in SIZES[0]:
        rgb = run_render(net, pts[:P], nrm[:P], views[:P], feat[:P] if feat is not None else None)
        report("rgb P=%d" % P, rgb, rgb64[:P], True, keep[:P])


# ---------------------------------------------------------------------------------------------------------------------
# shade_kernel
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("pair", ["reference", "ragged"])
def test_shade_geometry_matches_fp64(cuda_dev, pair):
    sdf = sdf_net("ref_sdf" if pair == "reference" else "ragged", cuda_dev)
    dnet = translator_net("translator_ref" if pair == "reference" else "translator_300", cuda_dev)
    st, lref = lbs_setup(cuda_dev)
    if pair != "reference":
        st = lref = None
    cd = conds(cuda_dev)
    Pmax = SIZES[3][-1]
    pts = _sample(Pmax, 300).to(cuda_dev) * 0.8
    rays = torch.nn.functional.normalize(torch.randn(Pmax, 3, generator=torch.Generator().manual_seed(8)), dim=1)
    rays = rays.to(cuda_dev)
    bi = torch.randint(0, NFRAMES, (Pmax,), generator=torch.Generator().manual_seed(2)).to(cuda_dev)
    _, g64, _ = R.sdf(sdf.layers, pts, sdf.multires, sdf.pe_w)
    n64 = g64 / g64.norm(dim=1, keepdim=True)
    fn = deform_ref(dnet, lref, cd, bi)
    d64, J64 = R.jacobian(fn, pts)
    Jinv, ok64 = O.minv3x3(J64)
    cr64 = torch.where(ok64.view(-1, 1), (Jinv @ rays.double().view(-1, 3, 1)).view(-1, 3), rays.double())
    cr64 = cr64 / cr64.norm(dim=1, keepdim=True)
    det = torch.linalg.det(J64)
    keep = relu_keep(dnet, pts, cd, bi)
    if lref is not None:
        off64 = R.translator_offset(dnet.layers, pts.double(), 6, dnet.pe_w, cd, bi)
        keep &= lbs_keep(lref, pts.double() + off64)[0]
    decided = keep & ((det.abs() - 1e-4).abs() > 1e-6)
    print("shade_geometry %s: %d of %d points excluded (ReLU kink / voxel face), %d with |det| at 1e-4"
          % (pair, int((~keep).sum()), Pmax, int((keep & ~decided).sum())))
    for P in SIZES[3]:
        nrm, cr, dp, ok = run_shade(sdf, dnet, st, pts[:P], rays[:P], bi[:P], cd)
        k, kd = keep[:P], decided[:P]
        report("normals P=%d" % P, nrm, n64[:P], False)
        report("D(p) P=%d" % P, dp, d64[:P], True, k)
        assert torch.equal(ok[:P][kd].bool(), ok64[:P][kd]), "inv_ok"
        report("cardinal rays P=%d" % P, cr, cr64[:P], False, kd)


# ---------------------------------------------------------------------------------------------------------------------
# sdf_refine_band (small + indexed engines), sr_sdf_forward_indexed
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["ref_sdf", "ragged", "deep_two_skip"])
def test_refine_band_matches_fp64(cuda_dev, name):
    """Values inside the band are re-evaluated (the first SMALL_CAP listed by the column-split small engine, the rest
    by the persistent one); values outside it are left bit for bit."""
    from selfreconcode_b200 import ops
    net = sdf_net(name, cuda_dev)
    P = SIZES[0][-1]
    pts = _sample(P, 400).to(cuda_dev)
    f64 = R.sdf(net.layers, pts, net.multires, net.pe_w, want_grad=False)[0]
    g = torch.Generator().manual_seed(1)
    start = (f64.float().cpu() + 0.3 * torch.randn(P, generator=g) * f64.abs().mean().float().cpu()).to(cuda_dev)
    center = float(f64.median())
    spread = (start - center).abs().sort().values
    for count in (700, ops.SMALL_CAP + 3000):          # small engine alone; small + indexed
        eps = float(spread[count - 1] + spread[count]) / 2
        v = start.clone()
        ops.sdf_refine_band(net.fused, pts, v, center, eps)
        torch.cuda.synchronize()
        band = (start - center).abs() < eps
        print("refine_band %s: %d values in the band (small-engine cap %d)" % (name, int(band.sum()), ops.SMALL_CAP))
        assert int(band.sum()) == count
        assert torch.equal(v[~band].view(torch.int32), start[~band].view(torch.int32))
        report("refined f (%d listed)" % count, v[band], f64[band], True)


def test_indexed_forward_partial_duplicate_shuffled_list(cuda_dev):
    lib = _lib()
    net = sdf_net("ragged", cuda_dev)
    P = SIZES[0][-1]
    pts = _sample(P, 500).to(cuda_dev)
    f64 = R.sdf(net.layers, pts, net.multires, net.pe_w, want_grad=False)[0]
    g = torch.Generator().manual_seed(5)
    ids = torch.cat([torch.randperm(P, generator=g)[:6000], torch.randint(0, P, (3000,), generator=g)])
    ids = ids[torch.randperm(ids.numel(), generator=g)].int().to(cuda_dev)
    m = 7000
    m_dev = torch.tensor([m], dtype=torch.int32, device=cuda_dev)
    out = sentinel(P, cuda_dev)
    assert lib.sr_sdf_forward_indexed(C.byref(net.desc), _p(pts), P, _p(ids), _p(m_dev), _p(out), _s()) == 0
    torch.cuda.synchronize()
    hit = torch.zeros(P + PAD, dtype=torch.bool, device=cuda_dev)
    hit[ids[:m].long()] = True
    assert bool((out.view(torch.int32)[~hit] == SENT).all()), "only listed ids within m_dev are written"
    print("sdf_forward_indexed: %d listed, %d within m_dev, %d distinct" % (ids.numel(), m, int(hit.sum())))
    report("indexed f", out[:P][hit[:P]], f64[hit[:P]], True)


# ---------------------------------------------------------------------------------------------------------------------
# trace_kernel / trace_rev_kernel against oracle.optimize_surface_ps in float64
# ---------------------------------------------------------------------------------------------------------------------
TRACE_PAIRS = {
    "reference": ("ref_sdf", "translator_ref", True),
    "ragged": ("ragged", "translator_300", False),
    "two_skip_identity": ("deep_two_skip", None, False),
    "deep12_translator9": ("deep_two_skip", "translator_9", False),     # 12 + 9 layers: a 42-step reverse program
}
CAM = (0.0, 0.2, -3.0)
# Each ray passes about 0.03 from its start point (about 0.6 degrees at the camera's distance): the angle term of the
# loss stays away from its kink at 0, where the direction of its gradient is decided by rounding.
ATHR = 3.0


def _trace_setup(pair, dev, n=320, odev="cpu"):
    """pair: a TRACE_PAIRS name or its (sdf, translator or None, with LBS) triple.  The float64 oracle's inputs and
    functions live on `odev`."""
    s_name, d_name, with_lbs = TRACE_PAIRS[pair] if isinstance(pair, str) else pair
    sdf = sdf_net(s_name, dev)
    dnet = translator_net(d_name, dev) if d_name else None
    st, lref = lbs_setup(dev) if with_lbs else (None, None)
    cd = conds(dev)
    x0 = _sample(n, 600, -0.7, 0.7).double().to(odev)
    bi = torch.randint(0, NFRAMES, (n,), generator=torch.Generator().manual_seed(6)).to(odev)
    cam = torch.tensor(CAM, dtype=torch.float64, device=odev)
    lo = {k: v.to(odev) for k, v in lref.items()} if lref is not None else None

    def sdf_fn(p):
        return R.mlp(sdf.layers, R.embed(p, sdf.multires, sdf.pe_w), sdf.d_in)[:, :1]

    def def_fn(p, b):
        p1 = p if dnet is None else p + R.translator_offset(dnet.layers, p, 6, dnet.pe_w, cd.to(odev), b)
        return p1 if lo is None else O.lbs_forward(lo["ws"], lo["bmin"], lo["bmax"], lo["A"], lo["trans"], p1, b)
    with torch.no_grad():
        miss = 0.03 * torch.randn(n, 3, generator=torch.Generator().manual_seed(7), dtype=torch.float64).to(odev)
        rays = torch.nn.functional.normalize(def_fn(x0, bi) + miss - cam, dim=1)
        f0 = sdf_fn(x0).view(-1).abs()
    return sdf, dnet, st, cd, x0, bi, cam, rays, f0, sdf_fn, def_fn


def _oracle_trace(cam, rays, x0, bi, sdf_fn, def_fn, dth, times, eps=(1e-5, 1e-3), with_iters=False):
    """eps: the engine's error bounds on f and on the angle (degrees) that mark a ray decision-sensitive; with_iters
    also returns how many times each ray was updated."""
    sens = dict(eps_f=eps[0], eps_a=eps[1])
    p, conv, iters = O.optimize_surface_ps(cam, rays, x0, bi, sdf_fn, def_fn, dth, ATHR, 3.05, 1.0, times,
                                           sensitivity=sens)
    return (p, conv, sens["sensitive"], iters) if with_iters else (p, conv, sens["sensitive"])


def _split_threshold(cam, rays, x0, bi, sdf_fn, def_fn, f0):
    """A dthreshold that leaves 20-80 % of the rays unconverged after one and after two iterations."""
    for q in (0.3, 0.2, 0.12, 0.06, 0.03, 0.015, 0.007, 0.003, 0.001):
        cand = float(f0.quantile(q))
        fr = [float(_oracle_trace(cam, rays, x0, bi, sdf_fn, def_fn, cand, t)[1].float().mean()) for t in (1, 2)]
        if all(0.2 <= v <= 0.8 for v in fr):
            return cand
    raise AssertionError("no threshold splits the rays")


@pytest.mark.parametrize("pair", list(TRACE_PAIRS))
def test_trace_matches_fp64_oracle(cuda_dev, pair):
    from selfreconcode_b200 import ops
    sdf, dnet, st, cd, x0, bi, cam, rays, f0, sdf_fn, def_fn = _trace_setup(pair, cuda_dev)
    n = x0.shape[0]
    dth = _split_threshold(cam, rays, x0, bi, sdf_fn, def_fn, f0)
    for times in (1, 2):
        po, co, sens = _oracle_trace(cam, rays, x0, bi, sdf_fn, def_fn, dth, times)
        res = {mode: ops.trace_surface_points(sdf.fused.truncated_last(1), dnet.fused if dnet else None, st,
                                              torch.tensor(CAM, device=cuda_dev), rays.float().to(cuda_dev),
                                              x0.float().to(cuda_dev), bi.to(cuda_dev), cd, dth, ATHR, 3.05, 1.0,
                                              times, mode=mode) for mode in ("forward", "reverse")}
        # Ill-conditioned trajectories, excluded and counted like the decision-sensitive rays: the float64 points move
        # by more than a fifth of the bar when every SDF value is off by 2e-6 (relative, or of mean |f|: the size of the
        # engine's measured error on f), or the two fp32 engines (forward- and reverse-mode) end that far apart.  A
        # kernel bug moves most updated rays, so at most 5 % may be excluded.
        rel = lambda a, b: ((a - b).abs() / (b.abs() + b.abs().mean())).amax(1)
        moved = torch.zeros(n, dtype=torch.bool)
        for pert in (lambda p: sdf_fn(p) * (1 + 2e-6), lambda p: sdf_fn(p) + 2e-6 * float(f0.mean())):
            moved |= rel(_oracle_trace(cam, rays, x0, bi, pert, def_fn, dth, times)[0], po) > ELEM / 5
        moved |= rel(res["forward"][0].cpu().double(), res["reverse"][0].cpu().double()) > ELEM / 5
        moved &= ~sens
        assert int(moved.sum()) <= 0.05 * n, int(moved.sum())
        keep = ~sens & ~moved
        for mode, (pt, ct) in res.items():
            mism = int(((ct.cpu() != co) & ~sens).sum())
            print("trace %s times=%d %s: dthreshold %.3g, %d of %d converged, %d sensitive, %d ill-conditioned, "
                  "%d mismatches" % (pair, times, mode, dth, int(co.sum()), n, int(sens.sum()), int(moved.sum()), mism))
            assert 0.2 * n <= int(co.sum()) <= 0.8 * n
            assert keep.float().mean() > 0.9
            assert mism == 0
            report("points", pt.cpu(), po, False, keep)


# ---------------------------------------------------------------------------------------------------------------------
# invariances: a row's arithmetic does not depend on its tile, CTA or launch
# ---------------------------------------------------------------------------------------------------------------------
def _invariant(run, args, P, name):
    """run(*per_point_args) -> tuple of per-point tensors; checks permutation, the first 17 alone, a rerun."""
    perm = torch.randperm(P, generator=torch.Generator().manual_seed(P)).to(args[0].device)
    base = run(*args)
    again = run(*args)
    pm = run(*[a[perm] if a is not None else None for a in args])
    head = run(*[a[:17] if a is not None else None for a in args])
    inv = torch.empty_like(perm)
    inv[perm] = torch.arange(P, device=perm.device)
    for i, b in enumerate(base):
        if b is None:
            continue
        assert torch.equal(b, again[i]), (name, "rerun", i)
        assert torch.equal(b, pm[i][inv]), (name, "permutation", i)
        assert torch.equal(b[:17], head[i]), (name, "prefix", i)


@pytest.mark.parametrize("kernel", ["sdf0", "sdf3", "deform", "render", "shade"])
def test_tile_invariance_bitwise(cuda_dev, kernel):
    st, lref = lbs_setup(cuda_dev)
    cd = conds(cuda_dev)
    if kernel.startswith("sdf"):
        T = int(kernel[3])
        net = sdf_net("ragged", cuda_dev)
        P = SIZES[T][-1]
        _invariant(lambda x: run_sdf(net, x, T)[:2], (_sample(P, 700).to(cuda_dev),), P, kernel)
    elif kernel == "deform":
        net = translator_net("translator_300", cuda_dev)
        P = SIZES[3][-1]
        bi = torch.randint(0, NFRAMES, (P,), generator=torch.Generator().manual_seed(1)).to(cuda_dev)
        _invariant(lambda x, b: run_deform(net, st, x, b, 0, cd, 3), (_deform_points(P, cuda_dev, lref, 9, True), bi),
                   P, kernel)
    elif kernel == "render":
        net, nfeat = render_net("render_ref", cuda_dev)
        P = SIZES[0][-1]
        _invariant(lambda *a: (run_render(net, *a),), tuple(render_inputs(P, nfeat, cuda_dev, 3)), P, kernel)
    else:
        sdf, dnet = sdf_net("ref_sdf", cuda_dev), translator_net("translator_ref", cuda_dev)
        P = SIZES[3][-1]
        g = torch.Generator().manual_seed(2)
        rays = torch.nn.functional.normalize(torch.randn(P, 3, generator=g), dim=1).to(cuda_dev)
        bi = torch.randint(0, NFRAMES, (P,), generator=g).to(cuda_dev)
        _invariant(lambda x, r, b: run_shade(sdf, dnet, st, x, r, b, cd), (_sample(P, 8).to(cuda_dev), rays, bi), P,
                   kernel)


@pytest.mark.parametrize("mode", ["forward", "reverse"])
def test_trace_invariance_bitwise(cuda_dev, mode):
    from selfreconcode_b200 import ops
    sdf, dnet = sdf_net("ragged", cuda_dev), translator_net("translator_300", cuda_dev)
    cd = conds(cuda_dev)
    P = 2 * 64 * NSM + 9
    g = torch.Generator().manual_seed(4)
    x0 = (0.7 * (2 * torch.rand(P, 3, generator=g) - 1)).to(cuda_dev)
    rays = torch.nn.functional.normalize(x0 - torch.tensor(CAM, device=cuda_dev), dim=1)
    bi = torch.randint(0, NFRAMES, (P,), generator=g).to(cuda_dev)
    cam = torch.tensor(CAM, device=cuda_dev)

    def run(x, r, b):
        p, c, cnt = ops.trace_surface_points(sdf.fused, dnet.fused, None, cam, r, x, b, cd, 1e-3, 0.02, 3.05, 1.0, 2,
                                             return_counters=True, mode=mode)
        return p, c
    _invariant(run, (x0, rays, bi), P, "trace " + mode)


# ---------------------------------------------------------------------------------------------------------------------
# argument checks (validation returns before any launch)
# ---------------------------------------------------------------------------------------------------------------------
def test_argument_contract(cuda_dev):
    from selfreconcode_b200 import _lib as L
    lib = _lib()
    base = sdf_net("ragged", cuda_dev)
    pts = torch.zeros(16, 3, device=cuda_dev)
    out = torch.zeros(16 * 512, device=cuda_dev)

    def sdf_rc(desc, nfeat=0):
        return lib.sr_sdf_forward(C.byref(desc), _p(pts), 16, _p(out), _p(out), _p(out) if nfeat else None, nfeat,
                                  _s())

    def mutated(**kw):
        d = L.MlpDesc()
        C.memmove(C.byref(d), C.byref(base.desc), C.sizeof(L.MlpDesc))
        for k, v in kw.items():
            if k.startswith("l"):
                i, field = k[1:].split("_", 1)
                setattr(d.layer[int(i)], field, v)
            else:
                setattr(d, k, v)
        return d
    cases = {
        "kpad 36": (mutated(l0_kpad=36), L.SR_EUNSUPPORTED),
        "npad 640": (mutated(l0_npad=640), L.SR_EUNSUPPORTED),
        "skip at layer 0": (mutated(l0_skip=1), L.SR_EINVAL),
        "0 layers": (mutated(n_layers=0), L.SR_EINVAL),
        "13 layers": (mutated(n_layers=13), L.SR_EINVAL),
        "multires 17": (mutated(multires=17), L.SR_EINVAL),
    }
    # a skip with a 45-wide embedded input (multires 7): wider than the skip stash
    m7 = R.embed(_sample(256, 1), 7, [1.0] * 7)
    wide = Net(scaled_layers([64, 64, 1], m7, {1}, R.SP, R.NONE, 3, cuda_dev), 45, 7, [1.0] * 7, cuda_dev)
    cases["skip with d_in 45"] = (wide.desc, L.SR_EUNSUPPORTED)
    for name, (d, want) in cases.items():
        rc = sdf_rc(d)
        print("  %-20s rc %d (want %d)" % (name, rc, want))
        assert rc == want, name
    # the SDF's feature count must leave column 0 to f
    two = sdf_net("wide_pe", cuda_dev)
    assert lib.sr_sdf_forward(C.byref(two.desc), _p(pts), 16, _p(out), None, _p(out), 1, _s()) == L.SR_EINVAL
    # renderer: at most 8 outputs
    rin = torch.randn(64, 9, dtype=torch.float64)
    r9 = Net(scaled_layers([16, 9], rin, set(), R.RELU, R.TANH, 4, cuda_dev), 9, 0, [], cuda_dev)
    assert lib.sr_render_forward(C.byref(r9.desc), _p(pts), _p(pts), _p(pts), None, 0, 16, _p(out), _s()) == \
        L.SR_EUNSUPPORTED
    # deformer: exactly 3 outputs
    din = torch.randn(64, 39 + CONDLEN, dtype=torch.float64)
    d4 = Net(scaled_layers([32, 4], din, set(), R.RELU, R.NONE, 5, cuda_dev), 39 + CONDLEN, 6, [1.0] * 6, cuda_dev)
    cd = conds(cuda_dev)
    assert lib.sr_deform_forward(C.byref(d4.desc), None, _p(pts), None, 16, _p(cd), CONDLEN, 16, _p(out), None, None,
                                 None, _s()) == L.SR_EINVAL


# ---------------------------------------------------------------------------------------------------------------------
# tensor-core engine: forward sweeps take any skip list, reverse sweeps at most one skip layer
# ---------------------------------------------------------------------------------------------------------------------
def test_tensor_core_two_skip_forward_runs_reverse_refused(cuda_dev):
    from selfreconcode_b200 import ops
    from selfreconcode_b200.train_ops import MlpConfig
    net = sdf_net("sp_two_skip", cuda_dev)
    P = 3000
    pts = _sample(P, 900).to(cuda_dev)
    out = ops.tc_mlp_forward(net.fused, pts)
    f64 = R.sdf(net.layers, pts, net.multires, net.pe_w, want_grad=False)[0]
    print("tensor-core forward, two skips (split-bf16 engine: the elementwise bar only):")
    report("f", out[:, 0], f64, False)
    rays = torch.nn.functional.normalize(torch.randn(P, 3, device=cuda_dev), dim=1)
    with pytest.raises(RuntimeError, match="at most one skip"):
        ops.trace_surface_points(net.fused, None, None, torch.tensor(CAM, device=cuda_dev), rays, pts, None, None,
                                 times=2, mode="tc")
    rnet, nfeat = render_net("render_small", cuda_dev)
    with pytest.raises(RuntimeError, match="at most one skip"):
        ops.shade_and_render_tc(net.fused, None, None, rnet.fused, pts, rays, None, None, nfeat=0)
    with pytest.raises(RuntimeError, match="at most one skip"):
        MlpConfig([R.SP] * 5 + [R.NONE], [l in (2, 4) for l in range(6)], 3, 1)
