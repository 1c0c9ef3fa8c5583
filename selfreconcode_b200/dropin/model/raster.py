"""Built-in silhouette rasteriser for the ray seed (SURVEY.md section 8f-1).

`MeshRasterizer` here plays the role pytorch3d's MeshRasterizer plays at model/network.py:864-880 (the object
behind `optNet.maskRender.rasterizer`): it owns `.cameras` and `.raster_settings` and turns the deformed template
into Fragments(pix_to_face, bary_coords, zbuf) -- on one CUDA kernel pair (csrc/raster.cu) instead of the
binned pytorch3d pipeline, and on the camera convention of RectifiedPerspectiveCameras.project directly
(pixel centres at integer (col, row)), so no NDC round trip.  `SilhouetteRenderer` is the minimal
MeshRendererWithFragments: `renderer(verts [N,V,3], faces) -> (hard silhouette [N,H,W,4], fragments)`.
`MeshRenderer` with `HardPhongShader` is the shaded counterpart OptimNetwork.infer renders with (infer.py:80-90):
Phong-lit images of the same fragments (csrc/mesh_shade.cu).  `PointsSilhouetteRenderer` is the soft point-cloud
silhouette of the optimisation step (csrc/points_silhouette.cu), with its gradient."""
import types

import torch

from selfreconcode_b200 import _lib, ops


class RasterSettings:
    def __init__(self, image_size, blur_radius=0., faces_per_pixel=1, perspective_correct=True,
                 clip_barycentric_coords=False, cull_backfaces=False, bin_size=None):
        self.image_size = tuple(image_size)
        self.blur_radius = blur_radius
        self.faces_per_pixel = faces_per_pixel
        self.perspective_correct = perspective_correct
        self.clip_barycentric_coords = clip_barycentric_coords
        self.cull_backfaces = cull_backfaces
        self.bin_size = bin_size
        if blur_radius != 0. or faces_per_pixel != 1 or cull_backfaces or clip_barycentric_coords:
            raise NotImplementedError("the built-in rasteriser implements the settings the optimisation step uses: "
                                      "blur 0, one face per pixel, no culling, unclipped barycentrics")


def screen_vertices(verts, cameras):
    """[N,V,3] world -> (col, row, view-space depth Z) with frame n seen by camera n (CameraMine.py:138-142);
    differentiable.  This is RectifiedPerspectiveCameras' NDC projection with pixel (i, j) centred at
    NDC (1-(2j+1)/W, 1-(2i+1)/H), expressed in pixel units."""
    N = verts.shape[0]
    R, T = cameras.R[:N], cameras.T[:N]
    pc = (verts.unsqueeze(3) * R.unsqueeze(1)).sum(2) + T.view(N, 1, 3)          # p R + T, no GEMM launch
    f, c = cameras.focal_length[:N], cameras.principal_point[:N]
    x = c[:, 0:1] - pc[..., 0] * f[:, 0:1] / pc[..., 2]
    y = c[:, 1:2] - pc[..., 1] * f[:, 1:2] / pc[..., 2]
    return torch.stack([x, y, pc[..., 2]], dim=-1)


class MeshRasterizer:
    def __init__(self, cameras, raster_settings):
        self.cameras = cameras
        self.raster_settings = raster_settings

    def to(self, device):
        if hasattr(self.cameras, "to"):
            self.cameras = self.cameras.to(device)
        return self

    def screen_vertices(self, verts, cameras=None):
        return screen_vertices(verts, cameras if cameras is not None else self.cameras)

    def __call__(self, verts, faces, cameras=None):
        H, W = self.raster_settings.image_size
        with torch.no_grad():
            vs = self.screen_vertices(verts, cameras)
            p2f, bary, zbuf = ops.raster_mesh(vs, faces, H, W)
        return types.SimpleNamespace(pix_to_face=p2f, bary_coords=bary, zbuf=zbuf,
                                     dists=torch.zeros_like(zbuf))


class SilhouetteRenderer:
    """`images, fragments = renderer(verts, faces)`; images[..., 3] is the hard coverage mask."""

    def __init__(self, rasterizer):
        self.rasterizer = rasterizer

    def to(self, device):
        self.rasterizer.to(device)
        return self

    def __call__(self, verts, faces, cameras=None, **kwargs):
        frags = self.rasterizer(verts, faces, cameras)
        cover = (frags.pix_to_face >= 0).float()
        return torch.cat([cover.expand(-1, -1, -1, 3), cover], dim=-1), frags


# ---- soft point silhouette of the optimisation step (model/network.py:495-505, 647-688) --------------------------
# pytorch3d's PointsRasterizer + AlphaCompositor(background_color=None) on the deformed template with unit features,
# restated on the device (csrc/points_silhouette.cu).  Keyword names and defaults are pytorch3d's.

class PointsRasterizationSettings:
    def __init__(self, image_size, radius=0.01, points_per_pixel=8, bin_size=None):
        self.image_size = tuple(image_size)
        self.radius = radius
        self.points_per_pixel = points_per_pixel
        self.bin_size = bin_size          # accepted for pytorch3d compatibility; the device kernel bins by itself


class PointsRasterizer:
    def __init__(self, cameras, raster_settings):
        self.cameras = cameras
        self.raster_settings = raster_settings

    def to(self, device):
        if hasattr(self.cameras, "to"):
            self.cameras = self.cameras.to(device)
        return self


class PointsSilhouetteRenderer:
    """`masks [N,H,W,1] = renderer(verts [N,V,3])`: the soft silhouette of the N frames' points, each seen by its own
    camera, differentiable w.r.t. verts.  Takes the tensor directly (no Pointclouds container): OptimNetwork's
    `takes_tensors` point-renderer protocol."""
    takes_tensors = True

    def __init__(self, rasterizer):
        self.rasterizer = rasterizer

    @property
    def radius(self):
        return self.rasterizer.raster_settings.radius

    def to(self, device):
        self.rasterizer.to(device)
        return self

    def __call__(self, verts, cameras=None):
        s = self.rasterizer.raster_settings
        H, W = s.image_size
        pts = screen_vertices(verts, cameras if cameras is not None else self.rasterizer.cameras)
        return ops.points_silhouette(pts, H, W, s.radius, s.points_per_pixel)


# ---- shaded images of OptimNetwork.infer (model/network.py:318-338; infer.py:90 installs HardPhongShader) ---------
# The classes below take pytorch3d's keyword names and defaults (pytorch3d.renderer PointLights, Materials,
# BlendParams, HardPhongShader); the shading itself is csrc/mesh_shade.cu.  Forward only, one face per pixel.

def _rgb(c, what):
    """A colour argument ((r, g, b),) / (r, g, b) / tensor -> 3 host floats (one colour for every frame)."""
    t = torch.as_tensor(c, dtype=torch.float64).detach().cpu().reshape(-1, 3)
    if not bool((t == t[:1]).all()):
        raise NotImplementedError("%s: one colour for all frames is supported, got %d different ones" % (what, t.shape[0]))
    return tuple(float(x) for x in t[0])


class PointLights:
    def __init__(self, device=None, location=((0., 1., 0.),), ambient_color=((0.5, 0.5, 0.5),),
                 diffuse_color=((0.3, 0.3, 0.3),), specular_color=((0.2, 0.2, 0.2),)):
        self.device = device
        self.location = torch.as_tensor(location, dtype=torch.float32, device=device).reshape(-1, 3)
        self.ambient_color = _rgb(ambient_color, "PointLights.ambient_color")
        self.diffuse_color = _rgb(diffuse_color, "PointLights.diffuse_color")
        self.specular_color = _rgb(specular_color, "PointLights.specular_color")

    def to(self, device):
        self.device = device
        self.location = self.location.to(device)
        return self


class Materials:
    def __init__(self, device=None, ambient_color=((1., 1., 1.),), diffuse_color=((1., 1., 1.),),
                 specular_color=((1., 1., 1.),), shininess=64):
        self.device = device
        self.ambient_color = _rgb(ambient_color, "Materials.ambient_color")
        self.diffuse_color = _rgb(diffuse_color, "Materials.diffuse_color")
        self.specular_color = _rgb(specular_color, "Materials.specular_color")
        s = torch.as_tensor(shininess, dtype=torch.float64).reshape(-1)
        if not bool((s == s[:1]).all()):
            raise NotImplementedError("Materials.shininess: one value for all frames is supported")
        self.shininess = float(s[0])

    def to(self, device):
        self.device = device
        return self


class BlendParams:
    def __init__(self, sigma=1e-4, gamma=1e-4, background_color=(1., 1., 1.)):
        self.sigma = sigma
        self.gamma = gamma
        self.background_color = tuple(float(x) for x in torch.as_tensor(background_color).reshape(3).tolist())


def vertex_face_csr(faces, n_verts):
    """(offsets [V+1], incident face ids) of every vertex, faces ascending per vertex: one stable device sort of the
    face table (optim.vertex_face_pairs) plus a binary search for the offsets (no atomics)."""
    from .optim import vertex_face_pairs
    vid, fid = vertex_face_pairs(faces, n_verts)
    offsets = torch.searchsorted(vid, torch.arange(n_verts + 1, device=vid.device, dtype=vid.dtype))
    return offsets, fid


class HardPhongShader:
    """`images = shader(fragments, verts [N,V,3], faces, ...)`: per-pixel Phong lighting of the interpolated position,
    vertex normal and per-vertex colour (white when none is given), hard blend over the background."""

    def __init__(self, device=None, cameras=None, lights=None, materials=None, blend_params=None):
        self.cameras = cameras
        self.lights = lights if lights is not None else PointLights(device=device)
        self.materials = materials if materials is not None else Materials(device=device)
        self.blend_params = blend_params if blend_params is not None else BlendParams()
        self._csr = None    # (faces, faces._version, V, csr): the CSR is built once per mesh

    def to(self, device):
        if hasattr(self.cameras, "to"):
            self.cameras = self.cameras.to(device)
        self.lights.to(device)
        self.materials.to(device)
        return self

    def csr(self, faces, n_verts):
        c = self._csr
        if c is None or c[0] is not faces or c[1] != faces._version or c[2] != n_verts:
            self._csr = (faces, faces._version, n_verts, vertex_face_csr(faces, n_verts))
        return self._csr[3]

    def params(self, lights, materials, blend_params):
        p = _lib.PhongParams()
        for field, val in (("light_ambient", lights.ambient_color), ("light_diffuse", lights.diffuse_color),
                           ("light_specular", lights.specular_color), ("mat_ambient", materials.ambient_color),
                           ("mat_diffuse", materials.diffuse_color), ("mat_specular", materials.specular_color),
                           ("background", blend_params.background_color)):
            getattr(p, field)[:] = val
        p.shininess = materials.shininess
        return p

    def __call__(self, fragments, verts, faces, cameras=None, lights=None, materials=None, blend_params=None,
                 verts_colors=None, **kwargs):
        cam = cameras if cameras is not None else self.cameras
        if cam is None:
            raise ValueError("HardPhongShader needs cameras (constructor or call argument)")
        lights = lights if lights is not None else self.lights
        materials = materials if materials is not None else self.materials
        blend_params = blend_params if blend_params is not None else self.blend_params
        N, V = verts.shape[0], verts.shape[1]
        with torch.no_grad():
            vs = verts.detach().contiguous().float()
            normals = ops.mesh_vertex_normals(vs, faces, self.csr(faces, V))       # all N frames in one launch
            R, T = cam.R[:N], cam.T[:N]
            cam_pos = -(R * T.view(N, 1, 3)).sum(2)          # cameras.cam_pos(n) for every frame, no host sync
            light_pos = lights.location.to(vs.device).expand(N, 3)
            return ops.shade_phong(vs, normals, faces, fragments.pix_to_face, fragments.bary_coords, cam_pos,
                                   light_pos, self.params(lights, materials, blend_params), colors=verts_colors)


class MeshRenderer:
    """Built-in counterpart of pytorch3d's MeshRendererWithFragments:
    `images [N,H,W,4], fragments = renderer(verts [N,V,3], faces, cameras=None, lights=None)`; `cameras` overrides
    both the rasteriser's and the shader's cameras for this call, `lights` the shader's lights."""

    def __init__(self, rasterizer, shader):
        self.rasterizer = rasterizer
        self.shader = shader

    def to(self, device):
        self.rasterizer.to(device)
        self.shader.to(device)
        return self

    def __call__(self, verts, faces, cameras=None, lights=None, **kwargs):
        frags = self.rasterizer(verts, faces, cameras)
        images = self.shader(frags, verts, faces, cameras=cameras, lights=lights, **kwargs)
        return images, frags
