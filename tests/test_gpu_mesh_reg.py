"""GPU: the device mesh regularisers (csrc/mesh_reg.cu, ops.mesh_reg_topology / ops.mesh_regularizers) against the
float64 restatement of pytorch3d's rules (tests/mesh_reg_ref.py), and OptimNetwork.forward with positive regulariser
weights with pytorch3d unimportable.

The restatement is fed the device's own fp32 positions.  Bars: topology equal (edge order, face_to_edge, E, P, pair
vertex ids); values |dev - ref| <= 1e-6 |ref| (+1e-12 for values that are 0 in exact arithmetic); gradients
helpers.elem_err < 1e-5; reruns bit-identical."""
import ctypes as C
import sys

import numpy as np
import pytest
import torch

import helpers as H
import mesh_reg_ref as ref
from test_mesh_reg_cpu import edge_case_meshes, jitter

pytestmark = pytest.mark.gpu
DEV = "cuda"
COT = (0.7, -1.3, 2.1)


def template(resolutions):
    """The synthetic SDF's template mesh (fp32 vertices, int64 faces on the device) on a marching-cubes ladder."""
    H.dropin()
    from MCAcc import Seg3dLossless
    from test_gpu_mesh_shade import _scene
    net = _scene(32, 32, 1)[0]
    eng = Seg3dLossless(query_func=None, b_min=[-0.9, -0.9, -0.9], b_max=[0.9, 0.9, 0.9], resolutions=resolutions,
                        align_corners=False, balance_value=0.0, use_cuda_impl=True).to(DEV)
    with torch.no_grad():
        v, f = net.discretizeSDF(H.RATIO, eng, 0.0)
    return v.detach().float().contiguous(), f


def _device(v, f, cot=COT):
    from selfreconcode_b200 import ops
    vs = v.to(DEV).float().detach().clone().requires_grad_(True)
    topo = ops.mesh_reg_topology(f.to(DEV), vs.shape[0])
    r = ops.mesh_regularizers(vs, topo)
    g, = torch.autograd.grad((r * torch.tensor(cot, device=DEV)).sum(), [vs])
    torch.cuda.synchronize()
    return topo, r.detach().cpu().double(), g.cpu().double()


def _check(name, v, f, cot=COT):
    v = torch.as_tensor(v).float().cpu()
    f = torch.as_tensor(f).cpu()
    topo, r, g = _device(v, f, cot)
    topo2, r2, g2 = _device(v, f, cot)
    assert torch.equal(r, r2) and torch.equal(g, g2), "reruns must be bit-identical"
    t = ref.topology(f, v.shape[0])
    assert (topo.E, topo.P) == (t["E"], t["P"]), name
    assert torch.equal(topo.edges.cpu(), t["edges"]) and torch.equal(topo.face_to_edge.cpu(), t["face_to_edge"])
    assert torch.equal(topo.pairs.cpu(), t["pairs"]), name
    rr, gr = ref.values_and_grads(v.double(), f, cot)
    verr = ((r - rr).abs() - 1e-6 * rr.abs()).max().item()
    gerr = H.elem_err(g.numpy(), gr.numpy())
    print("%s: V=%d F=%d E=%d P=%d; values %s (restatement %s); gradient elem_err %.2e"
          % (name, v.shape[0], f.shape[0], topo.E, topo.P, np.array2string(r.numpy(), precision=8),
             np.array2string(rr.numpy(), precision=8), gerr))
    assert verr <= 1e-12, (name, r, rr)
    assert gerr < 1e-5, (name, gerr)
    return r, g


@pytest.mark.parametrize("name", ["tetra", "cube", "grid", "fan3", "fan4", "single", "zero_area", "repeated",
                                  "unreferenced"])
def test_edge_case_meshes(name):
    v, f = edge_case_meshes()[name]
    if name not in ("zero_area", "single"):      # those keep their exact degenerate layout
        v = jitter(v, seed=3)
    if name == "grid":
        v[:, 2] = 0.0                             # jittered in its plane only
    _check(name, v, f)


def test_mc_template_and_term_by_term():
    from test_gpu_mesh_shade import _scene
    _, _, _, TmpVs, Tmpfs, _ = _scene(32, 32, 1)
    v = TmpVs.float().cpu()
    for cot in (COT, (1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)):
        _check("MC_LADDER_65 template, cotangent %s" % (cot,), v, Tmpfs.cpu(), cot)


def test_mc_ladder_257_template():
    from selfreconcode_b200 import synth
    v, f = template(synth.MC_LADDER_257)
    _check("MC_LADDER_257 template", v.cpu(), f.cpu())


def test_invalid_arguments():
    from selfreconcode_b200 import _lib, ops
    lib = _lib.load()
    s = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    buf = torch.zeros(4096, dtype=torch.float64, device=DEV)
    p = C.c_void_p(buf.data_ptr())
    z = C.c_void_p(0)
    good = dict(keys=[p, 2, 4, p, s], runs=[p, 6, p, p, s],
                topo=[p, p, p, p, p, 2, 4, 5, 1, p, p, p, p, s],
                fwd=[p, 4, 5, 1, p, p, p, p, p, p, p, p, s],
                bwd=[p, 4, 5, 1, p, p, p, p, p, p, p, p, p, s])
    fns = dict(keys=lib.sr_mesh_reg_edge_keys, runs=lib.sr_mesh_reg_edge_runs, topo=lib.sr_mesh_reg_topology,
               fwd=lib.sr_mesh_reg_forward, bwd=lib.sr_mesh_reg_backward)
    bad_sizes = dict(keys={1: (0, -1), 2: (0, -1, (1 << 31) + 1)}, runs={1: (0, -1)},
                     topo={5: (0, -1), 6: (0, -1, (1 << 31) + 1), 7: (0, -1, 7), 8: (-1,)},
                     fwd={1: (0, -1), 2: (0, -1), 3: (-1,)}, bwd={1: (0, -1), 2: (0, -1), 3: (-1,)})
    for k, fn in fns.items():     # only argument checks: every call here returns before any launch
        for i, a in enumerate(good[k][:-1]):
            if a is p:
                bad = list(good[k])
                bad[i] = z
                assert fn(*bad) == _lib.SR_EINVAL, (k, i)
        for i, vals in bad_sizes[k].items():
            for x in vals:
                bad = list(good[k])
                bad[i] = x
                assert fn(*bad) == _lib.SR_EINVAL, (k, i, x)
    torch.cuda.synchronize()
    faces = torch.tensor([[0, 1, 2], [0, 2, 3]], device=DEV)
    for bad in (torch.tensor([[0, 1, 4]], device=DEV), torch.tensor([[0, -1, 2]], device=DEV)):
        with pytest.raises(ValueError):
            ops.mesh_reg_topology(bad, 4)
    with pytest.raises(ValueError):
        ops.mesh_reg_topology(faces[:, :2], 4)
    topo = ops.mesh_reg_topology(faces, 4)
    with pytest.raises(ValueError):
        ops.mesh_regularizers(torch.zeros(5, 3, device=DEV), topo)


# ---------------------------------------------------------------------------------------------------------------------
# OptimNetwork.forward end to end
# ---------------------------------------------------------------------------------------------------------------------
WEIGHTS = dict(laplacian_weight=2.0, edge_weight=30.0, norm_weight=0.5)


def _step(monkeypatch, weights, mask_weight=1.0, dc_weight=0.1):
    """One OptimNetwork.forward (then loss.backward) on the point-silhouette test scene; returns (net, info, the
    inner step's TmpVs.grad, [(verts, topo)] of each ops.mesh_regularizers call)."""
    import utils
    from selfreconcode_b200 import ops, synth
    from test_gpu_mesh_shade import _gts, _scene
    Hh = Ww = 128
    net, data, cams, _, _, fids = _scene(Hh, Ww, 3)
    conf = synth.reference_config()
    conf._find('train.coarse.point_render')['radius'] = 0.02
    for lvl in ('loss_coarse', 'loss_medium', 'loss_fine'):
        conf[lvl] = dict(conf[lvl], pc_weight=dict(weight=60., mask_weight=mask_weight, **weights,
                                                   def_consistent=dict(weight=dc_weight, c=0.005)))
    loader = torch.utils.data.DataLoader(list(range(3)), 3)
    net, loader = utils.set_hierarchical_config(conf, 'coarse', net, loader, synth.MC_LADDER_65)
    calls = []
    orig = ops.mesh_regularizers

    def recording(verts, topo):
        calls.append((verts.detach().clone(), topo))
        return orig(verts, topo)
    monkeypatch.setattr(ops, "mesh_regularizers", recording)
    g = torch.Generator().manual_seed(21)
    datas = {'img': (torch.rand(3, Hh, Ww, 3, generator=g) * 2 - 1).to(DEV),
             'mask': _gts(3, Hh, Ww, image=False)['mask']}
    torch.manual_seed(5)
    loss = net.forward(datas, 2048, H.RATIO, fids)
    inner_grad = net.TmpVs.grad.detach().clone()      # before the outer backward adds |f(TmpVs)|'s gradient
    loss.backward()
    torch.cuda.synchronize()
    return net, dict(net.info), inner_grad, calls


@pytest.fixture
def no_pytorch3d(monkeypatch):
    H.dropin()
    monkeypatch.setitem(sys.modules, "pytorch3d", None)        # any pytorch3d import raises
    with pytest.raises(ImportError):
        import pytorch3d  # noqa: F401
    return monkeypatch


def test_forward_step_values(no_pytorch3d):
    net, info, _, calls = _step(no_pytorch3d, WEIGHTS)
    assert len(calls) == 1 and net.mesh_reg_topo is calls[0][1]
    v0 = calls[0][0].cpu()
    rr = ref.regularizers(v0.double(), net.Tmpfs.cpu())
    pc = info['pc_loss']
    got = [pc['lap_loss'], pc['edge_loss'], pc['norm_loss']]
    print("forward step (V=%d): lap / edge / norm %s, restatement %s" % (v0.shape[0], got, rr.tolist()))
    for a, b in zip(got, rr.tolist()):
        assert abs(a - b) <= 1e-6 * abs(b)


def test_forward_step_gradient(no_pytorch3d):
    # mask weight 0 and no deformation-consistency term: the inner step's only gradient is the regularisers'
    net, info, grad, calls = _step(no_pytorch3d, WEIGHTS, mask_weight=0.0, dc_weight=-1.0)
    v0 = calls[0][0].cpu()
    w = (WEIGHTS['laplacian_weight'], WEIGHTS['edge_weight'], WEIGHTS['norm_weight'])
    _, gr = ref.values_and_grads(v0.double(), net.Tmpfs.cpu(), w)
    err = H.elem_err(grad.cpu().numpy(), gr.numpy())
    print("inner-step gradient of the weighted regularisers: elem_err %.2e (max |g| %.2e)" % (err, gr.abs().max()))
    assert gr.abs().max() > 0 and err < 1e-4


def test_negative_weights_build_nothing(no_pytorch3d):
    from selfreconcode_b200 import ops

    def forbidden(*a, **k):
        raise AssertionError("no mesh regulariser topology may be built with every weight <= 0")
    no_pytorch3d.setattr(ops, "mesh_reg_topology", forbidden)
    net, info, _, calls = _step(no_pytorch3d, dict(laplacian_weight=-10., edge_weight=-10., norm_weight=-0.001))
    assert net.mesh_reg_topo is None and not calls
    assert not {'lap_loss', 'edge_loss', 'norm_loss'} & set(info['pc_loss'])
