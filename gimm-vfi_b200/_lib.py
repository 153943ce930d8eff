"""ctypes binding of include/gimmvfi_b200.h.

The product library is ``libgimmvfi_b200.so`` next to this file (built in-tree by
``build.py`` / ``__graft_entry__.build()``).  There is NO fallback: if it is
missing or fails to load, importing the engine raises.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "libgimmvfi_b200.so")


class Problem(C.Structure):
    _fields_ = [
        ("batch", C.c_int32),
        ("height", C.c_int32),
        ("width", C.c_int32),
        ("timesteps", C.c_int32),
        ("ds_factor", C.c_float),
        ("coord_height", C.c_int32),
        ("coord_width", C.c_int32),
    ]


_IO_FIELDS = ["img_xs", "coords", "t", "imgt_pred", "img_warp_4", "flowt0_1", "flowt1_1", "flowt0_4", "flowt1_4",
              "raft_flow", "nflow", "ninrflow", "flowt"]


class IO(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in _IO_FIELDS]


class Clip(C.Structure):
    _fields_ = [("frames", C.c_int32), ("pairs", C.c_int32), ("pair_list", C.c_void_p)]


class Queries(C.Structure):
    _fields_ = [("frames", C.c_int32), ("queries", C.c_int32), ("pair_list", C.c_void_p), ("t", C.c_void_p)]


class FlowInputs(C.Structure):
    _fields_ = [("flows", C.c_void_p), ("feat4", C.c_void_p * 2), ("feat8", C.c_void_p * 2), ("fnet", C.c_void_p * 2)]


class View(C.Structure):
    _fields_ = [
        ("data", C.c_void_p),
        ("n", C.c_int32),
        ("h", C.c_int32),
        ("w", C.c_int32),
        ("c", C.c_int32),
        ("pixel_stride", C.c_int32),
        ("batch_stride", C.c_int64),
    ]


FLOAT32, FLOAT64 = 0, 1   # gimmvfi_tensor4.dtype


class Tensor4(C.Structure):
    """gimmvfi_tensor4: a 4-D strided tensor (sizes and strides in elements)."""
    _fields_ = [("data", C.c_void_p), ("dtype", C.c_int32), ("sizes", C.c_int64 * 4), ("strides", C.c_int64 * 4)]


class Dense(C.Structure):
    """gimmvfi_dense: a dense row-major tensor of up to 5 dimensions."""
    _fields_ = [("data", C.c_void_p), ("dtype", C.c_int32), ("ndim", C.c_int32), ("sizes", C.c_int64 * 5)]


EXPORTS = [
    "gimmvfi_create", "gimmvfi_destroy", "gimmvfi_load_weight", "gimmvfi_finalize_weights", "gimmvfi_plan",
    "gimmvfi_forward", "gimmvfi_last_error", "gimmvfi_last_launches", "gimmvfi_weights_version", "gimmvfi_set_raft_iters", "gimmvfi_set_debug",
    "gimmvfi_get_tap", "gimmvfi_build_info", "gimmvfi_set_profile", "gimmvfi_profile_json",
    "gimmvfi_set_tensor_cores", "gimmvfi_set_cuda_graph", "gimmvfi_graph_replays", "gimmvfi_finalize_weights_gimm", "gimmvfi_finalize_weights_synthesis", "gimmvfi_finalize_weights_f", "gimmvfi_set_flowformer_iters", "gimmvfi_plan_from_flow", "gimmvfi_forward_from_flow", "gimmvfi_gimm_plan", "gimmvfi_gimm_forward", "gimmvfi_frame_cache_bytes", "gimmvfi_set_frame_cache", "gimmvfi_op_conv2d_tc", "gimmvfi_op_conv2d_tc_f16", "gimmvfi_op_conv2d_tc_strided", "gimmvfi_op_frames_u8_to_padded_f32", "gimmvfi_op_pred_to_u8", "gimmvfi_op_softsplat", "gimmvfi_op_softsplat_fused", "gimmvfi_op_backwarp", "gimmvfi_op_layernorm", "gimmvfi_op_window_attention", "gimmvfi_op_global_attention", "gimmvfi_op_patchify", "gimmvfi_op_cost_conv1", "gimmvfi_op_conv7x7_small_cout", "gimmvfi_op_row_softmax", "gimmvfi_op_resize",
    "gimmvfi_op_corr_volume", "gimmvfi_op_corr_volume_tc", "gimmvfi_op_corr_pool", "gimmvfi_op_corr_pool_pyramid", "gimmvfi_op_corr_lookup", "gimmvfi_op_corr_lookup_direct", "gimmvfi_op_conv2d",
    "gimmvfi_instnorm_scratch_floats", "gimmvfi_op_hyponet", "gimmvfi_op_conv2d_halo", "gimmvfi_op_conv2d_wide", "gimmvfi_op_instnorm", "gimmvfi_op_convex_upsample", "gimmvfi_op_pixel_shuffle", "gimmvfi_op_tail_pointwise",
    "gimmvfi_flow_to_image_scratch_floats", "gimmvfi_op_flow_to_image",
    "gimmvfi_finalize_weights_lpips", "gimmvfi_lpips_plan", "gimmvfi_lpips_forward",
    "gimmvfi_finalize_weights_flowformer", "gimmvfi_flowformer_plan", "gimmvfi_flowformer_forward", "gimmvfi_flowformer_forward_ex",
    "gimmvfi_finalize_weights_raft", "gimmvfi_raft_plan", "gimmvfi_raft_forward",
    "gimmvfi_op_softsplat_out", "gimmvfi_op_softsplat_grad",
    "gimmvfi_op_alt_corr_forward", "gimmvfi_op_alt_corr_backward",
    "gimmvfi_op_forward_interpolate",
    "gimmvfi_op_scene_sums", "gimmvfi_op_blend_u8",
    "gimmvfi_set_motion_config",
    "gimmvfi_plan_clip", "gimmvfi_forward_clip",
    "gimmvfi_plan_queries", "gimmvfi_forward_queries", "gimmvfi_set_coord_range",
]


class GimmvfiError(RuntimeError):
    pass


class Lib:
    """Thin typed wrapper over the shared library."""

    def __init__(self, path: str = DEFAULT_LIB):
        if not os.path.exists(path):
            raise ImportError(
                "gimmvfi_b200: native library %s not found — run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU / PyTorch fallback)" % path)
        self.path = path
        self.dll = C.CDLL(path)
        d = self.dll
        vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float
        PV = C.POINTER(View)
        d.gimmvfi_create.argtypes = [i32, C.POINTER(vp)]
        d.gimmvfi_destroy.argtypes = [vp]
        d.gimmvfi_destroy.restype = None
        d.gimmvfi_load_weight.argtypes = [vp, C.c_char_p, vp, C.POINTER(i64), i32]
        d.gimmvfi_finalize_weights.argtypes = [vp]
        d.gimmvfi_plan.argtypes = [vp, C.POINTER(Problem), C.POINTER(C.c_size_t)]
        d.gimmvfi_forward.argtypes = [vp, C.POINTER(Problem), C.POINTER(IO), vp, C.c_size_t, vp]
        d.gimmvfi_plan_clip.argtypes = [vp, C.POINTER(Problem), C.POINTER(Clip), C.POINTER(C.c_size_t)]
        d.gimmvfi_forward_clip.argtypes = [vp, C.POINTER(Problem), C.POINTER(Clip), C.POINTER(IO), vp, C.c_size_t, vp]
        d.gimmvfi_plan_queries.argtypes = [vp, C.POINTER(Problem), C.POINTER(Queries), C.POINTER(C.c_size_t)]
        d.gimmvfi_forward_queries.argtypes = [vp, C.POINTER(Problem), C.POINTER(Queries), C.POINTER(IO), vp, C.c_size_t, vp]
        d.gimmvfi_set_coord_range.argtypes = [vp, C.c_double, C.c_double]
        d.gimmvfi_last_error.argtypes = [vp]
        d.gimmvfi_last_error.restype = C.c_char_p
        d.gimmvfi_last_launches.argtypes = [vp]
        d.gimmvfi_last_launches.restype = i64
        d.gimmvfi_weights_version.argtypes = [vp]
        d.gimmvfi_weights_version.restype = i64
        d.gimmvfi_set_raft_iters.argtypes = [vp, i32]
        d.gimmvfi_set_debug.argtypes = [vp, i32]
        d.gimmvfi_get_tap.argtypes = [vp, C.c_char_p, PV]
        d.gimmvfi_build_info.restype = C.c_char_p
        d.gimmvfi_set_profile.argtypes = [vp, i32]
        d.gimmvfi_set_tensor_cores.argtypes = [vp, i32]
        d.gimmvfi_set_motion_config.argtypes = [vp, i32, i32, f32, f32, i32]
        d.gimmvfi_set_cuda_graph.argtypes = [vp, i32]
        d.gimmvfi_graph_replays.argtypes = [vp]
        d.gimmvfi_graph_replays.restype = i64
        d.gimmvfi_finalize_weights_gimm.argtypes = [vp]
        d.gimmvfi_finalize_weights_synthesis.argtypes = [vp]
        d.gimmvfi_finalize_weights_f.argtypes = [vp]
        d.gimmvfi_set_flowformer_iters.argtypes = [vp, i32]
        d.gimmvfi_plan_from_flow.argtypes = [vp, C.POINTER(Problem), C.POINTER(C.c_size_t)]
        d.gimmvfi_forward_from_flow.argtypes = [vp, C.POINTER(Problem), C.POINTER(IO), C.POINTER(FlowInputs), vp, C.c_size_t, vp]
        d.gimmvfi_gimm_plan.argtypes = [vp, C.POINTER(Problem), C.POINTER(C.c_size_t)]
        d.gimmvfi_finalize_weights_lpips.argtypes = [vp]
        d.gimmvfi_lpips_plan.argtypes = [vp, i32, i32, i32, C.POINTER(C.c_size_t)]
        d.gimmvfi_lpips_forward.argtypes = [vp, vp, vp, i32, i32, i32, i32, vp, vp, vp, C.c_size_t, vp]
        d.gimmvfi_finalize_weights_flowformer.argtypes = [vp]
        d.gimmvfi_flowformer_plan.argtypes = [vp, i32, i32, i32, i32, C.POINTER(C.c_size_t)]
        d.gimmvfi_flowformer_forward.argtypes = [vp, vp, i32, i32, i32, vp, i32, i32, i32, vp, vp, vp, C.c_size_t, vp]
        d.gimmvfi_flowformer_forward_ex.argtypes = [vp, vp, i32, i32, i32, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]
        d.gimmvfi_finalize_weights_raft.argtypes = [vp]
        d.gimmvfi_raft_plan.argtypes = [vp, i32, i32, i32, i32, i32, C.POINTER(C.c_size_t)]
        d.gimmvfi_raft_forward.argtypes = [vp, vp, i32, i32, i32, vp, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, C.c_size_t, vp]
        d.gimmvfi_gimm_forward.argtypes = [vp, C.POINTER(Problem), vp, vp, vp, vp, vp, vp, C.c_size_t, vp]
        d.gimmvfi_frame_cache_bytes.argtypes = [C.POINTER(Problem)]
        d.gimmvfi_frame_cache_bytes.restype = C.c_size_t
        d.gimmvfi_set_frame_cache.argtypes = [vp, vp, C.c_size_t, i32, i32]
        d.gimmvfi_op_conv2d_tc.argtypes = [PV, PV, vp, vp, i32, i32, i32, i32, i32, vp, PV, i32, vp, PV, PV, PV, i32, PV, vp, f32, vp]
        d.gimmvfi_op_conv2d_tc_strided.argtypes = [PV, vp, vp, i32, i32, i32, i32, i32, i32, i32, PV, vp]
        d.gimmvfi_op_conv2d_tc_f16.argtypes = [PV, PV, vp, vp, vp, i32, i32, i32, i32, i32, vp, PV, i32, vp, i32, PV, vp]
        d.gimmvfi_profile_json.argtypes = [vp, vp]
        d.gimmvfi_profile_json.restype = C.c_char_p
        d.gimmvfi_op_softsplat.argtypes = [PV, PV, PV, vp, i32, PV, PV, vp]
        d.gimmvfi_op_softsplat_fused.argtypes = [PV, PV, PV, vp, i32, vp, PV, vp]
        d.gimmvfi_op_backwarp.argtypes = [PV, PV, PV, vp]
        d.gimmvfi_op_resize.argtypes = [PV, PV, f32, f32, vp]
        d.gimmvfi_op_tail_pointwise.argtypes = [i32, PV, PV, PV, f32, f32, i32, i32, i32, vp]
        d.gimmvfi_op_layernorm.argtypes = [PV, vp, vp, f32, PV, f32, i32, vp]
        d.gimmvfi_op_window_attention.argtypes = [PV, PV, PV, PV, i32, i32, vp]
        d.gimmvfi_op_global_attention.argtypes = [PV, PV, PV, PV, i32, vp]
        d.gimmvfi_op_patchify.argtypes = [PV, PV, i32, vp]
        d.gimmvfi_op_cost_conv1.argtypes = [vp, i64, i32, i32, vp, vp, PV, vp]
        d.gimmvfi_op_conv7x7_small_cout.argtypes = [PV, vp, vp, i32, PV, vp]
        d.gimmvfi_op_row_softmax.argtypes = [vp, i64, i64, f32, vp]
        d.gimmvfi_op_corr_volume.argtypes = [PV, PV, vp, vp]
        d.gimmvfi_op_corr_pool.argtypes = [vp, vp, i64, i32, i32, vp]
        d.gimmvfi_op_corr_volume_tc.argtypes = [PV, PV, vp, vp, i32, vp]
        d.gimmvfi_op_corr_pool_pyramid.argtypes = [vp, vp, vp, vp, i64, i32, i32, vp]
        d.gimmvfi_op_corr_lookup.argtypes = [C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(C.c_int32), PV, PV, vp]
        d.gimmvfi_op_corr_lookup_direct.argtypes = [PV, C.POINTER(vp), C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_float, PV, PV, vp]
        d.gimmvfi_op_conv2d.argtypes = [PV, PV, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, i32, i32, vp, PV, PV, vp]
        d.gimmvfi_op_conv2d_halo.argtypes = [PV, vp, vp, vp, i32, i32, i32, vp, PV, i32, vp, i32, i32, PV, vp]
        d.gimmvfi_op_hyponet.argtypes = [vp, PV, vp, PV, i32, vp]
        d.gimmvfi_instnorm_scratch_floats.argtypes = [i32, i32]
        d.gimmvfi_instnorm_scratch_floats.restype = i64
        d.gimmvfi_op_instnorm.argtypes = [PV, i32, vp, PV, vp]
        d.gimmvfi_op_convex_upsample.argtypes = [PV, PV, PV, vp]
        d.gimmvfi_op_pixel_shuffle.argtypes = [PV, PV, i32, vp]
        d.gimmvfi_op_frames_u8_to_padded_f32.argtypes = [vp, i32, i32, i32, vp, i32, i32, i32, i32, vp]
        d.gimmvfi_op_pred_to_u8.argtypes = [vp, i32, i32, i32, vp, i32, i32, i32, i32, i32, vp]
        d.gimmvfi_flow_to_image_scratch_floats.argtypes = [i32, i32]
        d.gimmvfi_flow_to_image_scratch_floats.restype = i64
        d.gimmvfi_op_flow_to_image.argtypes = [vp, i64, i64, i64, i64, i32, i32, i32, C.c_double, C.c_double, i32, vp, vp, vp]
        PT = C.POINTER(Tensor4)
        d.gimmvfi_op_softsplat_out.argtypes = [PT, PT, PT, vp]
        d.gimmvfi_op_softsplat_grad.argtypes = [PT, PT, PT, PT, PT, vp]
        PD = C.POINTER(Dense)
        d.gimmvfi_op_alt_corr_forward.argtypes = [PD, PD, PD, i32, PD, vp]
        d.gimmvfi_op_alt_corr_backward.argtypes = [PD, PD, PD, PD, i32, PD, PD, PD, vp]
        d.gimmvfi_op_forward_interpolate.argtypes = [vp, i32, i32, i32, vp, vp]
        d.gimmvfi_op_scene_sums.argtypes = [vp, vp, i32, i32, i32, vp, vp]
        d.gimmvfi_op_blend_u8.argtypes = [C.POINTER(vp), C.POINTER(i32), i32, i32, i32, i32, i32, vp, i32, i32, i32, vp]

    def build_info(self) -> str:
        return self.dll.gimmvfi_build_info().decode()

    def check(self, rc: int, engine=None):
        if rc != 0:
            msg = self.dll.gimmvfi_last_error(engine).decode(errors="replace")
            raise GimmvfiError(msg)


_default = None


def default_lib() -> Lib:
    global _default
    if _default is None:
        _default = Lib()
    return _default


def view_of(t, channels=None, offset=0) -> View:
    """NHWC fp32 (or, for the half-storage conv op, fp16) torch tensor (n,h,w,C) -> View (optionally a channel slice)."""
    assert t.dim() == 4 and t.is_contiguous() and str(t.dtype) in ("torch.float32", "torch.float16")
    n, h, w, c = t.shape
    cc = c - offset if channels is None else channels
    return View(t.data_ptr() + t.element_size() * offset, n, h, w, cc, c, h * w * c)
