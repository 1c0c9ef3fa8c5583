"""CPU: the float64 restatement of the texture-atlas rule (tests/texture_ref.py) against closed forms, the frame-id
formula, and the OBJ parser of selfreconcode_b200.texture."""
import numpy as np
import pytest

import texture_ref as ref


# ---- UV raster ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [8, 17, 64])
def test_uv_raster_half_squares(R):
    """Texel (i, j) has u = (j+.5)/R, v = 1-(i+.5)/R: the half-square u + v <= 1 holds j <= i, R(R+1)/2 texels (its
    diagonal texel centres lie exactly on the hypotenuse and count), the other half j >= i; the diagonal goes to the
    lower face id and together they cover every texel once."""
    vt = np.array([[0., 0.], [1., 0.], [0., 1.], [1., 1.]])
    ft = np.array([[0, 1, 2], [1, 3, 2]])
    face, bary, near, overlap = ref.uv_raster(ref.uv_screen(vt, R), ft, R)
    i, j = np.meshgrid(np.arange(R), np.arange(R), indexing="ij")
    assert np.array_equal(face, np.where(j <= i, 0, 1))
    assert (face == 0).sum() == R * (R + 1) // 2 and (face == 1).sum() == R * (R - 1) // 2
    assert np.allclose(bary.sum(-1), 1.) and (bary >= 0).all()
    assert near[i == j].all()                  # the diagonal sits on both faces' shared edge
    # the second face alone covers its closed half, diagonal included
    face2, _, _, _ = ref.uv_raster(ref.uv_screen(vt, R), ft[1:], R)
    assert (face2 == 0).sum() == R * (R + 1) // 2
    # the two halves only touch; a repeated face overlaps its copy on its interior
    assert not overlap.any()
    face3, _, _, overlap3 = ref.uv_raster(ref.uv_screen(vt, R), ft[[0, 0]], R)
    assert np.array_equal(face3, np.where(j <= i, 0, -1)) and np.array_equal(overlap3, j < i)


def test_uv_raster_sub_square_and_degenerate():
    """Half of the square [0, 1/2]^2 at R = 8: n(n+1)/2 texels with n = R/2; a zero-area face covers nothing."""
    R = 8
    vt = np.array([[0., 0.], [.5, 0.], [0., .5], [.25, .25]])
    ft = np.array([[3, 3, 3], [0, 1, 2], [0, 0, 1]])
    face, bary, _, _ = ref.uv_raster(ref.uv_screen(vt, R), ft, R)
    n = R // 2
    assert (face == 1).sum() == n * (n + 1) // 2 and (face == 0).sum() == 0 and (face == 2).sum() == 0
    i, j = np.nonzero(face == 1)
    assert (i >= n).all() and (j < n).all() and ((i - j) >= n).all()
    # barycentrics reproduce the texel centre
    xy = ref.uv_screen(vt, R)
    p = (bary[i, j][:, :, None] * xy[ft[1]][None]).sum(1)
    assert np.abs(p - np.stack([j, i], 1)).max() < 1e-12


# ---- sampling -----------------------------------------------------------------------------------------------------
def test_bilinear_centres_and_clamp():
    img = np.arange(4 * 5 * 3, dtype=np.float64).reshape(4, 5, 3)
    assert np.array_equal(ref.bilinear(img, np.array([[2., 1.]]))[0], img[1, 2])
    np.testing.assert_allclose(ref.bilinear(img, np.array([[2.5, 1.]]))[0], (img[1, 2] + img[1, 3]) / 2)
    np.testing.assert_allclose(ref.bilinear(img, np.array([[2.5, 1.5]]))[0], img[1:3, 2:4].mean((0, 1)))
    # clamp to edge, also far outside
    assert np.array_equal(ref.bilinear(img, np.array([[-0.7, -3.], [40., 2.]])), np.stack([img[0, 0], img[2, 4]]))


# ---- slots --------------------------------------------------------------------------------------------------------
def _run(alphas, colours, S=3, c0=0.5, frames=None):
    st = ref.Slots(1, S, c0)
    frames = frames if frames is not None else list(range(len(alphas)))
    for a, c, f in zip(alphas, colours, frames):
        st.update(np.array([a]), lambda m, c=c: np.array([[c, c, c]]), f)
    return st


def test_slots_first_minimum_and_strict_greater():
    st = _run([0.6, 0.7, 0.55], [0.1, 0.2, 0.3])
    assert st.alpha[:, 0].tolist() == [0.6, 0.7, 0.55] and st.view[:, 0].tolist() == [0, 1, 2]
    st = _run([0.6, 0.7, 0.55, 0.65], [0.1, 0.2, 0.3, 0.4])      # replaces the minimum 0.55 (slot 2)
    assert st.alpha[:, 0].tolist() == [0.6, 0.7, 0.65] and st.view[:, 0].tolist() == [0, 1, 3]
    st = _run([0.6, 0.7, 0.55, 0.65, 0.65], [0] * 5)             # then the minimum 0.6 (slot 0)
    assert st.alpha[:, 0].tolist() == [0.65, 0.7, 0.65] and st.view[:, 0].tolist() == [4, 1, 3]
    st = _run([0.6, 0.7, 0.55, 0.65, 0.65, 0.65], [0] * 6)       # 0.65 > 0.65 is false: no change
    assert st.view[:, 0].tolist() == [4, 1, 3]
    st = _run([0.6, 0.7, 0.55, 0.65, 0.65, 0.9], [0] * 6)        # first of the two minima: slot 0
    assert st.alpha[:, 0].tolist() == [0.9, 0.7, 0.65] and st.view[:, 0].tolist() == [5, 1, 3]
    # alpha == c0 and alpha == 0 (unusable face) never enter
    st = _run([0.5, 0.0], [0.1, 0.2])
    assert (st.view == -1).all() and np.isnan(st.rgb).all()


def test_slots_fill_empty_slots_in_order():
    st = _run([0.9, 0.8], [0.1, 0.2], S=4)
    assert st.view[:, 0].tolist() == [0, 1, -1, -1]


def test_finish_median_counts_and_view():
    st = _run([0.6, 0.7, 0.55], [0.1, 0.5, 0.3])
    med, mf, view, count = ref.finish(st, 3)
    assert count[0] == 3 and mf[0] and view[0] == 1 and np.allclose(med[0], 0.3)    # odd count: the middle value
    st = _run([0.6, 0.7, 0.55, 0.8], [0.1, 0.2, 0.8, 0.4], S=4)
    med, mf, view, count = ref.finish(st, 4)
    assert count[0] == 4 and mf[0] and view[0] == 3 and np.allclose(med[0], 0.3)    # even: mean of 0.2 and 0.4
    med, mf, view, count = ref.finish(st, 5)                                          # min_views cut
    assert count[0] == 4 and not mf[0] and view[0] == -1 and (med[0] == 0).all()
    # partly filled slots: the median of the filled ones only (np.nanmedian), count = filled slots
    st = _run([0.6, 0.9], [0.2, 0.6], S=5)
    med, mf, view, count = ref.finish(st, 2)
    assert count[0] == 2 and mf[0] and view[0] == 1 and np.allclose(med[0], 0.4)
    # ties of the largest alpha: the first slot's frame
    st = _run([0.8, 0.6, 0.8], [0.1, 0.2, 0.3], frames=[7, 8, 9])
    assert ref.finish(st, 1)[2][0] == 7


def test_accumulate_rule_on_one_face():
    """alpha = sum b_i a_v; colour = bilinear(image, sum b_i s_v) / 255; unusable faces never enter."""
    screen = np.array([[1., 1., 2.], [3., 1., 2.], [1., 3., 2.]])
    faces = np.array([[0, 1, 2]])
    img = np.zeros((5, 5, 3), np.uint8)
    img[..., 0] = np.arange(5)[None, :] * 50            # colour = 50 * col in channel 0
    b = np.array([[0.5, 0.25, 0.25], [1., 0., 0.]])
    st = ref.Slots(2, 2, 0.3)
    ref.accumulate(st, np.zeros(2, np.int64), b, screen, faces, np.array([0.4, 0.8, 1.0]), np.array([1]), img, 3)
    np.testing.assert_allclose(st.alpha[0], [0.5 * 0.4 + 0.25 * 0.8 + 0.25, 0.4])
    np.testing.assert_allclose(st.rgb[0, :, 0], [50 * 1.5 / 255., 50 / 255.])
    assert st.view[0].tolist() == [3, 3]
    st2 = ref.Slots(2, 2, 0.3)
    ref.accumulate(st2, np.zeros(2, np.int64), b, screen, faces, np.array([0.4, 0.8, 1.0]), np.array([0]), img, 3)
    assert (st2.view == -1).all()


def test_vertex_in_mask_rounds_half_to_even():
    mask = np.zeros((4, 4), bool)
    mask[2, 2] = True
    s = np.array([[2.5, 2.5], [1.5, 1.5], [2.4, 1.6], [-0.4, 0.], [3.6, 0.]])
    assert ref.vertex_in_mask(s, mask).tolist() == [True, True, True, False, False]


# ---- frame ids ----------------------------------------------------------------------------------------------------
def test_frame_ids():
    from selfreconcode_b200.texture import texture_frame_ids
    assert texture_frame_ids(4, 10).tolist() == [0, 3, 5, 8]
    assert texture_frame_ids(120, 120).tolist() == list(range(120))
    assert texture_frame_ids(1, 7).tolist() == [0]
    ids = texture_frame_ids(120, 263)
    assert np.array_equal(ids, ref.frame_ids(120, 263)) and ids.max() <= 262 and np.all(np.diff(ids) > 0)
    for bad in ((11, 10), (0, 10), (-1, 10)):
        with pytest.raises(ValueError):
            texture_frame_ids(*bad)


# ---- OBJ parser ---------------------------------------------------------------------------------------------------
def _obj(tmp_path, text):
    p = tmp_path / "m.obj"
    p.write_text(text)
    return str(p)


def test_obj_fans_and_vn(tmp_path):
    from selfreconcode_b200.texture import load_obj_uv
    path = _obj(tmp_path, "# quad and pentagon\nmtllib x.mtl\no body\n"
                "v 0 0 0\nv 1 0 0\nv 1 1 0\nv 0 1 0\nv 0.5 2 0 1.0\n"
                "vt 0 0\nvt 1 0\nvt 1 1\nvt 0 1\nvt 0.5 0.5 0\nvn 0 0 1\n"
                "usemtl m\ns off\nf 1/1/1 2/2/1 3/3/1 4/4/1\nf 1/5 2/4 3/3 5/2 4/1\n")
    V, F, vt, ft = load_obj_uv(path)
    assert V.shape == (5, 3) and vt.shape == (5, 2)
    assert V.dtype.is_floating_point and F.dtype == ft.dtype and str(F.dtype) == "torch.int64"
    assert F.tolist() == [[0, 1, 2], [0, 2, 3], [0, 1, 2], [0, 2, 4], [0, 4, 3]]
    assert ft.tolist() == [[0, 1, 2], [0, 2, 3], [4, 3, 2], [4, 2, 1], [4, 1, 0]]
    assert vt[4].tolist() == [0.5, 0.5] and V[4].tolist() == [0.5, 2., 0.]


def test_obj_negative_indices(tmp_path):
    from selfreconcode_b200.texture import load_obj_uv
    path = _obj(tmp_path, "v 0 0 0\nv 1 0 0\nv 0 1 0\nv 1 1 0\nvt 0 0\nvt 1 0\nvt 0 1\n"
                "f -4/-3 -3/-2 -2/-1\nf 2/2 -1/1 3/-1\n")
    _, F, _, ft = load_obj_uv(path)
    assert F.tolist() == [[0, 1, 2], [1, 3, 2]] and ft.tolist() == [[0, 1, 2], [1, 0, 2]]


@pytest.mark.parametrize("face", ["f 1//1 2//1 3//1", "f 1 2 3", "f 1/1 2 3/3", "f 1/1 2/2 9/3", "f 1/1 2/2 3/7",
                                  "f 1/1 2/2"])
def test_obj_rejects(tmp_path, face):
    from selfreconcode_b200.texture import load_obj_uv
    path = _obj(tmp_path, "v 0 0 0\nv 1 0 0\nv 0 1 0\nvt 0 0\nvt 1 0\nvt 0 1\nvn 0 0 1\n" + face + "\n")
    with pytest.raises(ValueError):
        load_obj_uv(path)
