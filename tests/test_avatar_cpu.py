"""CPU: self-checks of the textured avatar's float64 restatement (tests/avatar_texture_ref.py), argument validation of
selfreconcode_b200.avatar, and the restatement's bone chain against the skinner's own (LBSkinner._chain)."""
import types

import numpy as np
import pytest
import torch

import avatar_texture_ref as ref
import helpers as H


def test_level0_texel_centre_returns_the_texel():
    g = np.random.default_rng(0)
    tex = g.integers(0, 256, (37, 52, 3), dtype=np.uint8)
    lv = ref.mips(tex, np.ones((37, 52), np.uint8))
    i, j = np.meshgrid(np.arange(37), np.arange(52), indexing="ij")
    u, v = (j + 0.5) / 52., 1. - (i + 0.5) / 37.
    got = ref.sample(lv, u, v, np.zeros_like(u))
    assert np.abs(got - tex / 255.).max() < 1e-12


def test_mip_sizes_and_level_table():
    from selfreconcode_b200 import ops
    assert ref.mip_sizes(420, 420)[-4:] == [(7, 7), (4, 4), (2, 2), (1, 1)]
    assert ref.mip_sizes(5, 1) == [(5, 1), (3, 1), (2, 1), (1, 1)]
    t = ops.mip_levels(37, 52).numpy()
    sizes = ref.mip_sizes(37, 52)
    assert [tuple(r[1:]) for r in t] == sizes
    assert list(t[:, 0]) == list(np.cumsum([0] + [h * w for h, w in sizes[:-1]]))


def test_affine_face_footprint_is_its_scale():
    """An orthographic face (equal depths) with an affine UV map: lambda = log2 of the known texels per pixel."""
    Ht = Wt = 1024
    for s in (0.25, 1., 3., 8., 20.):
        xy = np.array([[10., 20.], [60., 25.], [15., 90.]])
        # uv such that one pixel step moves s texels along each screen axis (a scaled rotation of the screen)
        c, sn = np.cos(0.3), np.sin(0.3)
        tex = (xy @ np.array([[c, -sn], [sn, c]]).T) * s
        uv = np.stack([tex[:, 0] / Wt, tex[:, 1] / Ht], 1)
        rho = ref.footprint(xy[None], np.full((1, 3), 1. / 2.5), uv[None], 30., 40., Ht, Wt)
        lam = ref.level_param(rho, 11)
        assert abs(rho[0] - s) < 1e-9
        assert abs(lam[0] - np.clip(np.log2(s), 0, 10)) < 1e-9


def test_weighted_reduction_ignores_uncovered_parents():
    tex = np.zeros((2, 2, 3), np.uint8)
    tex[0, 0] = (200, 100, 50)
    tex[1, 1] = (10, 20, 30)
    cov = np.array([[1, 0], [0, 0]], np.uint8)
    lv = ref.mips(tex, cov)
    assert np.allclose(lv[1][0, 0, :3], np.array([200, 100, 50]) / 255.) and lv[1][0, 0, 3] == 0.25
    # no covered parent: the plain mean
    lv = ref.mips(tex, np.zeros((2, 2), np.uint8))
    assert np.allclose(lv[1][0, 0, :3], np.array([210, 120, 80]) / 255. / 4.) and lv[1][0, 0, 3] == 0.
    # odd sizes: a child with fewer parents averages over those it has
    lv = ref.mips(np.full((3, 3, 3), 90, np.uint8), np.ones((3, 3), np.uint8))
    assert np.allclose(lv[1][..., :3], 90 / 255.) and np.allclose(lv[1][..., 3], 1.)


def _fake_net(frame_num=4):
    return types.SimpleNamespace(dataset=types.SimpleNamespace(frame_num=frame_num, H=8, W=8))


def test_argument_validation(tmp_path):
    from selfreconcode_b200 import avatar
    good_p, good_t = np.zeros((5, 24, 3), np.float32), np.zeros((5, 3), np.float32)
    p, t, y = avatar.motion_args(np.zeros((5, 72)), good_t, np.zeros(5))
    assert tuple(p.shape) == (5, 24, 3) and tuple(t.shape) == (5, 3) and y.dtype == torch.float64
    for bad in (np.zeros((5, 23, 3)), np.zeros((5, 71)), np.zeros((5, 24)), np.zeros(72), np.zeros((0, 72))):
        with pytest.raises(ValueError):
            avatar.motion_args(bad, good_t)
    for bad in (np.zeros((4, 3)), np.zeros((5, 2)), np.zeros(15)):
        with pytest.raises(ValueError):
            avatar.motion_args(good_p, bad)
    with pytest.raises(ValueError):
        avatar.motion_args(good_p, good_t, np.zeros(4))
    net = _fake_net(4)
    for cf in (-1, 4, 100):
        with pytest.raises(ValueError):
            avatar.render_motion(net, None, str(tmp_path / "m"), good_p, good_t, cond_frame=cf)
        with pytest.raises(ValueError):
            avatar.export_avatar(net, None, str(tmp_path / "a.npz"), cond_frame=cf)
    with pytest.raises(ValueError):
        avatar.render_motion(net, None, str(tmp_path / "m"), np.zeros((5, 70)), good_t)
    with pytest.raises(ValueError):
        avatar.render_motion(net, None, str(tmp_path / "m"), good_p, np.zeros((6, 3)))


def test_atlas_validation(tmp_path):
    import cv2
    from selfreconcode_b200 import avatar
    obj = tmp_path / "uvmap.obj"
    obj.write_text("v 0 0 0\nv 1 0 0\nv 0 1 0\nvt 0 0\nvt 1 0\nvt 0 1\nf 1/1 2/2 3/3\n")
    for name, img in (("gray.png", np.zeros((8, 8), np.uint8)), ("rgba.png", np.zeros((8, 8, 4), np.uint8)),
                      ("deep.png", np.zeros((8, 8, 3), np.uint16))):
        cv2.imwrite(str(tmp_path / name), img)
        with pytest.raises(ValueError):
            avatar.TexturedAvatar(str(obj), str(tmp_path / name), device="cpu")
    for arr in (np.zeros((8, 8, 3), np.float32), np.zeros((8, 8, 2), np.uint8), np.zeros((0, 8, 3), np.uint8)):
        with pytest.raises(ValueError):
            avatar.TexturedAvatar(str(obj), arr, device="cpu")
    with pytest.raises(ValueError):
        avatar.TexturedAvatar(str(obj), str(tmp_path / "missing.png"), device="cpu")


def test_rest_inverse_without_init_pose():
    from selfreconcode_b200 import avatar
    Js = torch.arange(72, dtype=torch.float32).view(24, 3) / 50.
    sk = types.SimpleNamespace(init_pose=None, Js=Js)
    inv = avatar.rest_inverse(sk)
    assert np.array_equal(inv[:, :3, :3], np.tile(np.eye(3), (24, 1, 1)))
    assert np.allclose(inv[:, :3, 3], -Js.double().numpy())


def test_bone_chain_matches_the_skinner():
    """The numpy chain the export checks use equals LBSkinner._chain (Rodrigues, parents) on CPU within 1e-6, and
    the skinner's init_pose is the inverse of its rest chain (so A_j = G_j init_pose_j is the skinning transform)."""
    H.dropin()
    from selfreconcode_b200 import avatar, synth
    sk = synth.make_skinner(resolution=(9, 13, 5))
    g = torch.Generator().manual_seed(1)
    poses = 0.3 * torch.randn(4, 24, 3, generator=g)
    got, _ = sk._chain(poses)
    want = ref.bone_chain(poses.numpy(), sk.Js.numpy(), np.asarray([int(p) for p in sk.parents]))
    err = np.abs(got.double().numpy() - want).max()
    print("bone chain: max |err| %.2e" % err)
    assert err <= 1e-6
    inv = avatar.rest_inverse(sk)
    rest = ref.bone_chain(synth.smpl_apose(1).reshape(1, 24, 3), sk.Js.numpy(), np.asarray(sk.parents))[0]
    assert np.abs(rest @ inv - np.eye(4)).max() <= 1e-5
