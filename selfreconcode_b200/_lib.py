"""ctypes binding of libselfrecon_b200.so (the C ABI declared in include/selfrecon_b200.h).

The product path has no CPU fallback: if the library is missing or a CUDA tensor op is asked
for without it, importing / calling raises.  (oracle/ is test infrastructure and is never
imported from here.)
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# SELFRECON_B200_LIB lets tuning scripts A/B differently-built libraries; default = in-tree build
LIB_PATH = os.environ.get("SELFRECON_B200_LIB") or os.path.join(_HERE, "lib", "libselfrecon_b200.so")

SR_OK = 0
SR_EINVAL, SR_EUNSUPPORTED, SR_ECAPACITY = -1, -2, -3
SR_MLP_MAX_LAYERS = 12
SR_ACT_NONE, SR_ACT_SOFTPLUS100, SR_ACT_RELU, SR_ACT_TANH = 0, 1, 2, 3

c_f = C.c_void_p  # all device pointers travel as void*
i64 = C.c_int64
i32 = C.c_int
f32 = C.c_float
stream_t = C.c_void_p


class MlpLayer(C.Structure):
    _fields_ = [("wt", C.c_void_p), ("bias", C.c_void_p), ("k", C.c_int), ("n", C.c_int),
                ("kpad", C.c_int), ("npad", C.c_int), ("act", C.c_int), ("skip", C.c_int),
                ("wb", C.c_void_p)]


class MlpDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int), ("d_in", C.c_int), ("multires", C.c_int),
                ("pe_w", C.c_float * 16), ("layer", MlpLayer * SR_MLP_MAX_LAYERS)]


class LbsParams(C.Structure):
    _fields_ = [("ws_cl", C.c_void_p), ("D", C.c_int), ("H", C.c_int), ("W", C.c_int),
                ("bmin", C.c_float * 3), ("bmax", C.c_float * 3), ("A", C.c_void_p),
                ("trans", C.c_void_p), ("F", C.c_int)]


class TcLayer(C.Structure):
    _fields_ = [("W", C.c_void_p), ("Wb", C.c_void_p), ("bias", C.c_void_p), ("zero_bias", C.c_void_p),
                ("n", C.c_int), ("k", C.c_int), ("act", C.c_int), ("skip", C.c_int)]


class TraceParams(C.Structure):
    _fields_ = [("cam_pos", C.c_float * 3), ("dthreshold", C.c_float), ("athreshold", C.c_float),
                ("w1", C.c_float), ("w2", C.c_float)]


class PhongParams(C.Structure):
    """struct sr_phong_params (light / material colours of sr_shade_phong)."""
    _fields_ = [("light_ambient", C.c_float * 3), ("light_diffuse", C.c_float * 3), ("light_specular", C.c_float * 3),
                ("mat_ambient", C.c_float * 3), ("mat_diffuse", C.c_float * 3), ("mat_specular", C.c_float * 3),
                ("shininess", C.c_float), ("background", C.c_float * 3)]


# name -> (restype, argtypes); every symbol include/selfrecon_b200.h declares
SIGNATURES = {
    "sr_abi_version": (C.c_int, []),
    "sr_build_info": (C.c_char_p, []),
    "sr_minv3x3_f32": (C.c_int, [c_f, c_f, c_f, i64, stream_t]),
    "sr_minv3x3_f64": (C.c_int, [c_f, c_f, c_f, i64, stream_t]),
    "sr_minv3x3_bwd_f32": (C.c_int, [c_f, c_f, c_f, i64, stream_t]),
    "sr_minv3x3_bwd_f64": (C.c_int, [c_f, c_f, c_f, i64, stream_t]),
    "sr_mc_work_bytes": (i64, [i32, i32, i32]),
    "sr_mc_count": (C.c_int, [c_f, i32, i32, i32, f32, c_f, c_f, stream_t]),
    "sr_mc_emit": (C.c_int, [c_f, i32, i32, i32, f32, f32, f32, f32, f32, f32, f32, i32, c_f, c_f, i64,
                             c_f, i64, stream_t]),
    "sr_interp2x3d_fwd_f32": (C.c_int, [c_f, c_f, c_f, i32, i32, i32, i32, f32, stream_t]),
    "sr_interp2x3d_bwd_f32": (C.c_int, [c_f, c_f, i32, i32, i32, i32, stream_t]),
    "sr_interp2x2d_fwd_f32": (C.c_int, [c_f, c_f, c_f, i32, i32, i32, f32, stream_t]),
    "sr_interp2x2d_bwd_f32": (C.c_int, [c_f, c_f, i32, i32, i32, stream_t]),
    "sr_grid_sample3d_fwd_f32": (C.c_int, [c_f, C.POINTER(i64), c_f, c_f, c_f, i32, i32, i32, i32,
                                           i32, i64, stream_t]),
    "sr_grid_sample3d_bwd_f32": (C.c_int, [c_f, C.POINTER(i64), c_f, c_f, c_f, c_f, i32, i32, i32,
                                           i32, i32, i64, stream_t]),
    "sr_grid_sample3d_dbwd_f32": (C.c_int, [c_f, c_f, c_f, C.POINTER(i64), c_f, c_f, c_f, c_f, c_f,
                                            i32, i32, i32, i32, i32, i64, stream_t]),
    "sr_grid_sample3d_fwd_f64": (C.c_int, [c_f, C.POINTER(i64), c_f, c_f, c_f, i32, i32, i32, i32,
                                           i32, i64, stream_t]),
    "sr_grid_sample3d_bwd_f64": (C.c_int, [c_f, C.POINTER(i64), c_f, c_f, c_f, c_f, i32, i32, i32,
                                           i32, i32, i64, stream_t]),
    "sr_grid_sample3d_dbwd_f64": (C.c_int, [c_f, c_f, c_f, C.POINTER(i64), c_f, c_f, c_f, c_f, c_f,
                                            i32, i32, i32, i32, i32, i64, stream_t]),
    "sr_fold_linear": (C.c_int, [c_f, c_f, c_f, i32, i32, i32, i32, c_f, c_f, c_f, stream_t]),
    "sr_sdf_forward": (C.c_int, [C.POINTER(MlpDesc), c_f, i64, c_f, c_f, c_f, i32, stream_t]),
    "sr_lbs_bone_transforms": (C.c_int, [c_f, c_f, c_f, c_f, i32, c_f, c_f, stream_t]),
    "sr_lbs_weights_to_channels_last": (C.c_int, [c_f, c_f, i32, i32, i32, stream_t]),
    "sr_deform_forward": (C.c_int, [C.POINTER(MlpDesc), C.POINTER(LbsParams), c_f, c_f, i64, c_f,
                                    i32, i64, c_f, c_f, c_f, c_f, stream_t]),
    "sr_render_forward": (C.c_int, [C.POINTER(MlpDesc), c_f, c_f, c_f, c_f, i32, i64, c_f,
                                    stream_t]),
    "sr_trace_step": (C.c_int, [C.POINTER(MlpDesc), C.POINTER(MlpDesc), C.POINTER(LbsParams),
                                C.POINTER(TraceParams), c_f, c_f, c_f, c_f, i32, i64, c_f, c_f,
                                c_f, i32, c_f, stream_t]),
    "sr_trace_scratch_bytes": (i64, []),
    "sr_trace_step_rev": (C.c_int, [C.POINTER(MlpDesc), C.POINTER(MlpDesc), C.POINTER(LbsParams),
                                    C.POINTER(TraceParams), c_f, c_f, c_f, c_f, i32, i64, c_f, c_f,
                                    c_f, i32, c_f, c_f, stream_t]),
    "sr_shade_geometry": (C.c_int, [C.POINTER(MlpDesc), C.POINTER(MlpDesc), C.POINTER(LbsParams),
                                    c_f, c_f, c_f, c_f, i32, i64, c_f, c_f, c_f, i32, c_f, c_f,
                                    stream_t]),
    "sr_tc_embed": (C.c_int, [c_f, i64, i32, C.POINTER(f32), i32, c_f, c_f, i64, i32, c_f, i32, c_f, c_f,
                              stream_t]),
    "sr_tc_embed_backward": (C.c_int, [c_f, i64, i32, C.POINTER(f32), i32, c_f, i32, c_f, i32, c_f, stream_t]),
    "sr_tc_act_bytes": (i64, [i64, i32]),
    "sr_tc_weight_bytes": (i64, [i32, i32]),
    "sr_tc_pack_rows": (C.c_int, [c_f, i64, i32, i32, c_f, c_f, stream_t]),
    "sr_tc_pack_weights": (C.c_int, [c_f, i32, i32, i32, c_f, stream_t]),
    "sr_tc_linear": (C.c_int, [c_f, c_f, c_f, i64, i32, i32, i32, i32, i32, c_f, i32, f32, c_f, i32,
                               i32, c_f, i32, i32, i32, c_f, c_f, i32, i32, f32, c_f, stream_t]),
    "sr_tc_trace_mid": (C.c_int, [c_f, c_f, i64, c_f, c_f, c_f, c_f, c_f, C.POINTER(LbsParams),
                                  C.POINTER(TraceParams), i32, c_f, c_f, c_f, i32, c_f, stream_t]),
    "sr_tc_trace_update": (C.c_int, [c_f, c_f, i64, c_f, c_f, i32, c_f, i32, c_f, i32, c_f, i32,
                                     C.POINTER(f32), i32, C.POINTER(f32), c_f, c_f, stream_t]),
    "sr_raster_mesh": (C.c_int, [c_f, c_f, i64, i64, i64, i32, i32, c_f, c_f, c_f, c_f, stream_t]),
    "sr_mesh_vertex_normals": (C.c_int, [c_f, c_f, c_f, c_f, i64, i64, i64, c_f, stream_t]),
    "sr_shade_phong": (C.c_int, [c_f, c_f, c_f, c_f, i64, i64, i64, c_f, c_f, i32, i32, c_f, c_f,
                                 C.POINTER(PhongParams), c_f, stream_t]),
    "sr_points_silhouette_list_capacity": (i64, [i64, i64, i32, i32, f32]),
    "sr_points_silhouette_bin": (C.c_int, [c_f, c_f, i64, i64, i32, i32, f32, c_f, c_f, stream_t]),
    "sr_points_silhouette_forward": (C.c_int, [c_f, c_f, c_f, i64, i64, i32, i32, f32, i32, c_f, c_f, c_f, c_f,
                                               stream_t]),
    "sr_points_silhouette_backward": (C.c_int, [c_f, c_f, c_f, c_f, c_f, i64, i64, i32, i32, f32, c_f, stream_t]),
    "sr_mesh_reg_edge_keys": (C.c_int, [c_f, i64, i64, c_f, stream_t]),
    "sr_mesh_reg_edge_runs": (C.c_int, [c_f, i64, c_f, c_f, stream_t]),
    "sr_mesh_reg_topology": (C.c_int, [c_f, c_f, c_f, c_f, c_f, i64, i64, i64, i64, c_f, c_f, c_f, c_f, stream_t]),
    "sr_mesh_reg_forward": (C.c_int, [c_f, i64, i64, i64, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, stream_t]),
    "sr_mesh_reg_backward": (C.c_int, [c_f, i64, i64, i64, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, stream_t]),
    "sr_texture_accumulate": (C.c_int, [i64, i32, c_f, c_f, c_f, c_f, i64, i64, c_f, c_f, c_f, i32, i32, i32, c_f, c_f,
                                        c_f, c_f, c_f, stream_t]),
    "sr_texture_finish": (C.c_int, [i64, i32, c_f, c_f, c_f, c_f, f32, i32, c_f, c_f, c_f, c_f, stream_t]),
    "sr_texture_mips": (C.c_int, [c_f, c_f, i32, i32, c_f, stream_t]),
    "sr_shade_textured": (C.c_int, [c_f, c_f, i64, i32, i32, c_f, i64, c_f, c_f, i64, c_f, i64, c_f, i32, i32, c_f,
                                    C.POINTER(f32), c_f, stream_t]),
    "sr_simplify_quadrics": (C.c_int, [c_f, c_f, i64, i64, c_f, c_f, c_f, c_f, c_f, c_f, stream_t]),
    "sr_simplify_edge_cost": (C.c_int, [c_f, c_f, c_f, i64, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, stream_t]),
    "sr_simplify_select": (C.c_int, [c_f, i64, i64, c_f, c_f, c_f, c_f, c_f, c_f, stream_t]),
    "sr_simplify_collapse": (C.c_int, [c_f, c_f, i64, i64, c_f, i64, c_f, c_f, c_f, c_f, c_f, c_f, stream_t]),
    "sr_simplify_compact": (C.c_int, [c_f, i64, i64, c_f, c_f, c_f, c_f, c_f, c_f, c_f, c_f, stream_t]),
    "sr_uv_face_adjacency": (C.c_int, [c_f, i64, c_f, c_f, c_f, stream_t]),
    "sr_uv_labels": (C.c_int, [c_f, c_f, i64, c_f, f32, i32, c_f, c_f, c_f, c_f, stream_t]),
    "sr_uv_chart_hook": (C.c_int, [c_f, c_f, i64, c_f, c_f, stream_t]),
    "sr_uv_chart_project": (C.c_int, [c_f, i64, c_f, c_f, c_f, c_f, c_f, stream_t]),
    "sr_uv_place": (C.c_int, [c_f, c_f, i64, c_f, C.c_double, c_f, stream_t]),
    "sr_uv_coverage": (C.c_int, [c_f, c_f, i64, i32, c_f, c_f, stream_t]),
    "sr_lbsw_knn_blend": (C.c_int, [c_f, c_f, i32, i32, C.POINTER(f32), C.POINTER(f32), i32, i32, i32, i32, i32, c_f,
                                    c_f, stream_t]),
    "sr_lbsw_smooth_pass": (C.c_int, [c_f, c_f, i32, i32, i32, i32, f32, stream_t]),
    "sr_lbsw_cut": (C.c_int, [c_f, i64, f32, stream_t]),
    "sr_frames_decode": (C.c_int, [c_f, c_f, c_f, i32, i32, i32, c_f, i64, c_f, c_f, c_f, stream_t]),
    "sr_tc_wgrad_partial_bytes": (i64, [i64, i32, i32, C.POINTER(C.c_int)]),
    "sr_tc_debug_wgrad_desc_swap": (None, [i32]),
    "sr_tc_mlp_forward": (C.c_int, [C.POINTER(TcLayer), i32, c_f, i64, i32, i32, i32, c_f, C.POINTER(C.c_void_p),
                                    C.POINTER(C.c_void_p), c_f, c_f, i32, stream_t]),
    "sr_tc_mlp_backward": (C.c_int, [C.POINTER(TcLayer), i32, i64, i32, i32, i32, c_f, i32, c_f,
                                     C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), c_f, c_f, c_f, c_f, i32,
                                     C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), c_f, c_f, i32, c_f, i32, i32, c_f,
                                     stream_t]),
    "sr_tc_wgrad": (C.c_int, [c_f, i32, c_f, i32, i64, c_f, c_f, i32, i32, i32, stream_t]),
    "sr_tc_colsum": (C.c_int, [c_f, i64, i32, i32, c_f, i32, stream_t]),
    "sr_tc_unpack_rows": (C.c_int, [c_f, i64, i32, i32, c_f, i32, stream_t]),
    "sr_svals3x3_f32": (C.c_int, [c_f, c_f, c_f, i64, stream_t]),
    "sr_svals3x3_bwd_f32": (C.c_int, [c_f, c_f, c_f, c_f, c_f, i64, stream_t]),
    "sr_band_select": (C.c_int, [c_f, i64, f32, f32, c_f, c_f, stream_t]),
    "sr_sdf_small_work_bytes": (i64, [i32]),
    "sr_sdf_forward_small": (C.c_int, [C.POINTER(MlpDesc), c_f, i64, c_f, c_f, c_f, c_f, i32, stream_t]),
    "sr_sdf_forward_indexed": (C.c_int, [C.POINTER(MlpDesc), c_f, i64, c_f, c_f, c_f, stream_t]),
    "sr_tc_shade_point": (C.c_int, [i64, c_f, c_f, c_f, c_f, c_f, C.POINTER(LbsParams), c_f, c_f, c_f, c_f,
                                    stream_t]),
    "sr_tc_shade_point_deformed": (C.c_int, [i64, c_f, c_f, c_f, c_f, c_f, C.POINTER(LbsParams), c_f, c_f, c_f,
                                             c_f, c_f, C.POINTER(f32), stream_t]),
    "sr_tc_render_embed": (C.c_int, [i64, c_f, c_f, c_f, c_f, i32, i32, i32, i32, i32, C.POINTER(f32), c_f,
                                     i32, stream_t]),
    "sr_seg3d_candidates": (C.c_int, [c_f, c_f, c_f, i32, i32, i32, i32, i32, i32, i32, i32, i32,
                                      stream_t]),
    "sr_seg3d_gather": (C.c_int, [c_f, i64, i32, i32, i32, i32, i32, i32, i32, i32, C.POINTER(f32), C.POINTER(f32),
                                  c_f, c_f, c_f, c_f, stream_t]),
    "sr_seg3d_scatter": (C.c_int, [c_f, i64, c_f, c_f, f32, c_f, c_f, i64, c_f, stream_t]),
    "sr_conv_pack": (C.c_int, [c_f, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, i64, i64, c_f,
                               stream_t]),
    "sr_instance_norm_partial_bytes": (i64, [i32, i64, i32]),
    "sr_instance_norm_stats": (C.c_int, [c_f, i32, i64, i32, c_f, c_f, c_f, stream_t]),
    "sr_instance_norm_apply": (C.c_int, [c_f, i32, i64, i32, c_f, c_f, c_f, i32, c_f, stream_t]),
    "sr_normal_unwarp": (C.c_int, [c_f, i32, i32, c_f, c_f, i32, i32, c_f, stream_t]),
}

_lib = None


def load():
    """Loads the library (once) and attaches the prototypes.  Raises if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "selfrecon_b200: %s is missing -- run `python -m selfreconcode_b200.build` "
            "(or __graft_entry__.build()).  There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


_ERR = {SR_EINVAL: "invalid argument", SR_EUNSUPPORTED: "unsupported shape",
        SR_ECAPACITY: "output buffer too small"}


def check(code, what):
    if code == SR_OK:
        return
    if code < 0:
        raise RuntimeError("selfrecon_b200.%s: %s (code %d)" % (what, _ERR.get(code, "error"), code))
    raise RuntimeError("selfrecon_b200.%s: CUDA error %d" % (what, code))
