"""CPU: the float64 restatement of pytorch3d's template mesh regularisers (tests/mesh_reg_ref.py) against closed forms,
pair counts of non-manifold edges, degenerate faces and float64 central differences.  Negative controls (L^T for L, the
edge loss over 2E, the 6 unique pairs of a 4-face edge) must fail the same bars.  The meshes here are reused by
tests/test_gpu_mesh_reg.py."""
import math

import numpy as np
import pytest
import torch

import mesh_reg_ref as ref

TETRA_FACES = [[0, 1, 2], [0, 3, 1], [0, 2, 3], [1, 3, 2]]


def tetra(R=1.0):
    v = torch.tensor([[1., 1., 1.], [1., -1., -1.], [-1., 1., -1.], [-1., -1., 1.]], dtype=torch.float64)
    return v * (R / math.sqrt(3.0)), torch.tensor(TETRA_FACES)


def cube():
    v = torch.tensor([[x, y, z] for x in (0., 1.) for y in (0., 1.) for z in (0., 1.)], dtype=torch.float64)
    f = [[0, 1, 3], [0, 3, 2], [4, 6, 7], [4, 7, 5], [0, 4, 5], [0, 5, 1],
         [2, 3, 7], [2, 7, 6], [0, 2, 6], [0, 6, 4], [1, 5, 7], [1, 7, 3]]
    return v, torch.tensor(f)


def grid(n=6):
    """Flat n x n vertex grid, every square split along the same diagonal."""
    v = torch.tensor([[i * 0.3, j * 0.2, 0.0] for j in range(n) for i in range(n)], dtype=torch.float64)
    f = []
    for j in range(n - 1):
        for i in range(n - 1):
            a, b, c, d = j * n + i, j * n + i + 1, (j + 1) * n + i, (j + 1) * n + i + 1
            f += [[a, b, d], [a, d, c]]
    return v, torch.tensor(f)


def fan(m):
    """m triangles sharing the edge (0, 1), wings at distinct angles around it."""
    v = [[0., 0., 0.], [1., 0., 0.]]
    for k in range(m):
        t = 2 * math.pi * k / m + 0.3
        v.append([0.3 + 0.1 * k, math.cos(t), math.sin(t)])
    return torch.tensor(v, dtype=torch.float64), torch.tensor([[0, 1, 2 + k] for k in range(m)])


def single_triangle():
    return torch.tensor([[0., 0., 0.], [1., 0., 0.], [0., 1., 0.]], dtype=torch.float64), torch.tensor([[0, 1, 2]])


def zero_area():
    """Two triangles on the edge (0, 1); the second's third vertex lies on that edge's line (n = 0)."""
    v = torch.tensor([[0., 0., 0.], [1., 0., 0.], [0.3, 1., 0.2], [0.5, 0., 0.]], dtype=torch.float64)
    return v, torch.tensor([[0, 1, 2], [1, 0, 3]])


def repeated_index():
    """The tetrahedron plus a face (0, 0, 1): a self-edge (0, 0) and a fourth and fifth entry on the edge (0, 1)."""
    v, f = tetra(1.0)
    return v, torch.cat([f, torch.tensor([[0, 0, 1]])])


def unreferenced():
    v, f = tetra(1.0)
    return torch.cat([v, torch.tensor([[0.4, -0.7, 2.0]], dtype=torch.float64)]), f


def edge_case_meshes():
    return dict(tetra=tetra(1.3), cube=cube(), grid=grid(), fan3=fan(3), fan4=fan(4), single=single_triangle(),
                zero_area=zero_area(), repeated=repeated_index(), unreferenced=unreferenced())


def jitter(v, seed, scale=0.05):
    g = torch.Generator().manual_seed(seed)
    return v + scale * torch.randn(v.shape, generator=g, dtype=torch.float64)


def lv(v, f, transpose=False):
    edges, _ = ref.packed_edges(f, v.shape[0])
    return torch.sparse.mm(ref.laplacian_matrix(edges, v.shape[0], transpose), v)


def test_tetrahedron_closed_forms():
    R = 1.3
    v, f = tetra(R)
    r = ref.regularizers(v, f)
    a2 = 8.0 / 3.0 * R * R         # squared edge of a regular tetrahedron with circumradius R
    np.testing.assert_allclose(r.numpy(), [4.0 / 3.0 * R, a2, 4.0 / 3.0], rtol=1e-12)
    assert ref.topology(f, 4)["P"] == 6
    # negative control: the edge loss over 2E
    assert abs(ref.regularizers(v, f, half=True)[1].item() - a2) > 1e-3 * a2


def test_cube_normal_consistency():
    v, f = cube()
    t = ref.topology(f, 8)
    assert t["E"] == 18 and t["P"] == 18
    assert abs(ref.regularizers(v, f)[2].item() - 2.0 / 3.0) < 1e-12


def test_flat_grid():
    n = 6
    v, f = grid(n)
    r = ref.regularizers(v, f)
    assert abs(r[2].item()) < 1e-12
    interior = [j * n + i for j in range(1, n - 1) for i in range(1, n - 1)]
    assert lv(v, f)[interior].abs().max().item() < 1e-12
    # negative control: L^T v is not zero next to the boundary
    assert lv(v, f, transpose=True)[interior].abs().max().item() > 1e-3


@pytest.mark.parametrize("m,pairs", [(3, 3), (4, 7)])
def test_non_manifold_edge_pairs(m, pairs):
    v, f = fan(m)
    t = ref.topology(f, v.shape[0])
    assert t["P"] == pairs
    assert t["pairs"][:, :2].tolist() == [[0, 1]] * pairs
    if m == 4:
        # the literal comprehension repeats (e[2], e[1]); the 6 unique pairs are another rule
        _, _, _, up = ref.pair_table(f, v.shape[0], unique_pairs=True)
        assert up.shape[0] == 6
        a = ref.regularizers(v, f)[2].item()
        b = ref.regularizers(v, f, unique_pairs=True)[2].item()
        assert abs(a - b) > 1e-6 * abs(a)


def test_single_triangle():
    v, f = single_triangle()
    assert ref.topology(f, 3)["P"] == 0
    r, g = ref.values_and_grads(v, f, cot=(0.0, 0.0, 1.0))
    assert r[2].item() == 0.0 and g.abs().max().item() == 0.0


def test_zero_area_face():
    v, f = zero_area()
    assert ref.topology(f, 4)["P"] == 1
    assert ref.regularizers(v, f)[2].item() == 1.0      # 1 - 0: the clamp keeps cos at 0


def test_repeated_index_face():
    v, f = repeated_index()
    t = ref.topology(f, 4)
    assert [0, 0] in t["edges"].tolist()
    assert t["P"] == 5 + 7          # five edges with two entries, the edge (0, 1) with four
    L = ref.laplacian_matrix(t["edges"], 4).to_dense()
    assert abs(L[0, 0].item() - (2.0 / 5.0 - 1.0)) < 1e-15     # self-edge counts 2 in A[0,0] and deg(0) = 3 + 2


def test_unreferenced_vertex():
    v, f = unreferenced()
    r, g = ref.values_and_grads(v, f, cot=(1.0, 0.0, 0.0))
    V = v.shape[0]
    np.testing.assert_allclose(lv(v, f)[4].numpy(), -v[4].numpy(), rtol=0, atol=1e-15)
    np.testing.assert_allclose(g[4].numpy(), (v[4] / v[4].norm()).numpy() / V, rtol=1e-12)     # d|-v|/dv / V


@pytest.mark.parametrize("name", ["tetra", "cube", "fan3", "fan4", "repeated", "unreferenced"])
def test_gradients_against_central_differences(name):
    v, f = edge_case_meshes()[name]
    v = jitter(v, seed=len(name))
    cot = (0.7, -1.3, 2.1)
    _, g = ref.values_and_grads(v, f, cot)
    h = 1e-6
    num = torch.zeros_like(v)
    c = torch.tensor(cot, dtype=torch.float64)
    for i in range(v.shape[0]):
        for k in range(3):
            vp, vm = v.clone(), v.clone()
            vp[i, k] += h
            vm[i, k] -= h
            num[i, k] = ((ref.regularizers(vp, f) - ref.regularizers(vm, f)) * c).sum() / (2 * h)
    err = (g - num).abs().max().item() / g.abs().max().item()
    assert err < 1e-7, err
