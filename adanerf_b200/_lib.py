"""ctypes binding of libadanerf_b200.so (include/adanerf_b200.h).  Fails loudly when the CUDA
extension is missing -- there is no CPU or PyTorch fallback for the product path."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ADN_LIB_PATH") or os.path.join(_HERE, "libadanerf_b200.so")   # override: A/B builds

STATUS_TEXT = {0: "ok", 1: "invalid argument", 2: "CUDA error", 3: "no usable sm_90 device",
               4: "weights not set", 5: "I/O error", 6: "device watchdog tripped"}


class AdnError(RuntimeError):
    def __init__(self, status, detail=""):
        self.status = status
        super().__init__(f"adanerf_b200 status {status} ({STATUS_TEXT.get(status, '?')}): {detail}")


class Scene(C.Structure):
    _fields_ = [("view_cell_center", C.c_float * 3), ("view_cell_size", C.c_float * 3),
                ("depth_range", C.c_float * 2), ("max_depth", C.c_float), ("fov", C.c_float),
                ("z_near", C.c_float), ("z_far", C.c_float), ("n_freq_pos", C.c_int32), ("n_freq_dir", C.c_int32),
                ("n_freq_pos0", C.c_int32), ("n_freq_dir0", C.c_int32),          # sampling-net encoding (0 = same)
                ("use_ndc", C.c_int32), ("ndc_w", C.c_int32), ("ndc_h", C.c_int32), ("ndc_focal", C.c_float)]


class TensorDesc(C.Structure):
    _fields_ = [("name", C.c_char_p), ("data", C.POINTER(C.c_float)), ("rows", C.c_int64), ("cols", C.c_int64)]


class AuxOutputs(C.Structure):   # adn_aux_outputs: device pointers, any may be NULL
    _fields_ = [("d_weights", C.c_void_p), ("d_alpha", C.c_void_p), ("d_z_vals", C.c_void_p), ("d_depth_map", C.c_void_p),
                ("d_acc_map", C.c_void_p), ("d_disp_map", C.c_void_p), ("d_depth_est", C.c_void_p)]


# adn_budget_reduce_fn: (user, uint64 d_words, n_words, stream) -> 0 on success
BUDGET_REDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p)


class Stats(C.Structure):
    _fields_ = [("n_rays", C.c_int64), ("n_samples", C.c_int64), ("ms_stage", C.c_float * 6),
                ("kernel_launches", C.c_int64)]


# every symbol include/adanerf_b200.h declares (tests/test_abi.py checks the .so exports all of them)
SYMBOLS = [
    "adn_create", "adn_destroy", "adn_strerror", "adn_last_error", "adn_version", "adn_set_weights",
    "adn_create_from_export_dir", "adn_probe_export_dir", "adn_render_camera_surface", "adn_register_host_buffer", "adn_unregister_host_buffer", "adn_net_dims", "adn_net_shape", "adn_set_option", "adn_get_stats", "adn_last_threshold", "adn_set_budget_group", "adn_render_rays", "adn_render_rays_aux", "adn_render_camera",
    "adn_render_camera_rgba8", "adn_render_rays_host", "adn_render_camera_host", "adn_stage0_features",
    "adn_generate_ray_directions", "adn_mlp0_forward", "adn_stage2_sample", "adn_budget_threshold", "adn_stage3_encode",
    "adn_mlp1_forward", "adn_stage5_composite", "adn_stage5_composite_aux", "adn_image_metrics", "adn_sampling_view",
    "adn_image_flip", "adn_image_iwssim", "adn_pdf_sample", "adn_stage5_density_composite", "adn_camera_rays",
    "adn_linear_depths",
]
# every symbol include/adanerf_b200_views.h declares (several cameras in one call; tests/test_views_abi.py checks them)
VIEWS_SYMBOLS = ["adn_render_views_rays", "adn_render_views_camera", "adn_render_views_camera_rgba8"]

_lib = None


def load_library():
    """Loads the in-tree shared library; raises if it has not been built (python __graft_entry__.py)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} not found: build the CUDA extension first "
                          f"(python -c 'import __graft_entry__ as g; g.build()'). There is no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    vp, f32p, i32p, i64 = C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64
    fp = C.POINTER(C.c_float)
    lib.adn_create.argtypes = [C.POINTER(vp), C.POINTER(Scene), C.c_int]
    lib.adn_destroy.argtypes = [vp]
    lib.adn_destroy.restype = None
    lib.adn_strerror.argtypes = [C.c_int]
    lib.adn_strerror.restype = C.c_char_p
    lib.adn_last_error.argtypes = [vp]
    lib.adn_last_error.restype = C.c_char_p
    lib.adn_version.restype = C.c_char_p
    lib.adn_set_weights.argtypes = [vp, C.c_int, C.POINTER(TensorDesc), C.c_int]
    lib.adn_create_from_export_dir.argtypes = [C.POINTER(vp), C.c_char_p, C.c_int, C.POINTER(C.c_float), C.POINTER(C.c_int)]
    lib.adn_probe_export_dir.argtypes = [C.c_char_p, C.POINTER(Scene), C.POINTER(C.c_float), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.adn_set_option.argtypes = [vp, C.c_char_p, i64]
    lib.adn_register_host_buffer.argtypes = [vp, vp, C.c_size_t]
    lib.adn_unregister_host_buffer.argtypes = [vp, vp]
    lib.adn_net_dims.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.adn_net_shape.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    lib.adn_get_stats.argtypes = [vp, C.POINTER(Stats)]
    lib.adn_last_threshold.argtypes = [vp, fp]
    lib.adn_set_budget_group.argtypes = [vp, BUDGET_REDUCE_FN, vp]
    lib.adn_render_rays.argtypes = [vp, fp, fp, f32p, i64, C.c_float, C.c_int, f32p, i32p, f32p, vp]
    lib.adn_render_rays_aux.argtypes = [vp, fp, fp, f32p, i64, C.c_float, C.c_int, f32p, i32p, f32p, C.POINTER(AuxOutputs), vp]
    lib.adn_render_camera.argtypes = [vp, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, f32p, i32p, vp]
    lib.adn_render_camera_rgba8.argtypes = [vp, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, vp, vp]
    lib.adn_render_camera_surface.argtypes = [vp, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, C.c_ulonglong, vp]
    lib.adn_render_views_rays.argtypes = [vp, C.c_int, fp, fp, f32p, i64, C.c_float, C.c_int, f32p, i32p, f32p,
                                          C.POINTER(AuxOutputs), vp]
    lib.adn_render_views_camera.argtypes = [vp, C.c_int, fp, fp, C.c_int, C.c_int, C.c_float, C.c_int, f32p, i32p, vp]
    lib.adn_render_views_camera_rgba8.argtypes = [vp, C.c_int, fp, fp, C.c_int, C.c_int, C.c_float, C.c_int, vp, vp]
    lib.adn_render_rays_host.argtypes = [vp, fp, fp, f32p, i64, C.c_float, C.c_int, f32p, i32p]
    lib.adn_render_camera_host.argtypes = [vp, fp, fp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_int, f32p, i32p]
    lib.adn_stage0_features.argtypes = [vp, fp, fp, f32p, i64, f32p, f32p, f32p, vp]
    lib.adn_generate_ray_directions.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int, f32p, vp]
    lib.adn_mlp0_forward.argtypes = [vp, f32p, i64, f32p, vp]
    lib.adn_stage2_sample.argtypes = [vp, f32p, i64, C.c_float, C.c_int, i32p, i32p, i32p, i32p, f32p, f32p, vp, vp]
    lib.adn_budget_threshold.argtypes = [vp, f32p, i64, C.c_float, C.c_int, i64, f32p, vp]
    lib.adn_sampling_view.argtypes = [vp, f32p, i64, f32p, vp]
    lib.adn_pdf_sample.argtypes = [vp, f32p, i64, C.c_int, C.c_int, i32p, i32p, i32p, f32p]
    lib.adn_stage5_density_composite.argtypes = [vp, f32p, f32p, f32p, i64, C.c_int, f32p, vp, C.POINTER(AuxOutputs)]
    lib.adn_camera_rays.argtypes = [vp, fp, fp, f32p, i64, f32p, f32p, f32p]
    lib.adn_linear_depths.argtypes = [vp, C.c_int, f32p]
    lib.adn_stage3_encode.argtypes = [vp, f32p, f32p, i32p, f32p, i64, f32p, vp]
    lib.adn_mlp1_forward.argtypes = [vp, f32p, i64, f32p, vp]
    lib.adn_stage5_composite.argtypes = [vp, f32p, f32p, f32p, i32p, i32p, i64, C.c_int, f32p, f32p, f32p, vp]
    lib.adn_stage5_composite_aux.argtypes = [vp, f32p, f32p, f32p, i32p, i32p, i64, C.c_int, C.c_int, f32p, vp,
                                             C.POINTER(AuxOutputs), vp]
    lib.adn_image_metrics.argtypes = [vp, f32p, f32p, i64, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double), vp]
    lib.adn_image_flip.argtypes = [vp, f32p, f32p, C.c_int, C.c_int, C.c_double, f32p, C.POINTER(C.c_double)]
    lib.adn_image_iwssim.argtypes = [vp, f32p, f32p, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    for name in SYMBOLS + VIEWS_SYMBOLS:
        fn = getattr(lib, name)
        if fn.restype is C.c_int and name not in ("adn_destroy", "adn_strerror", "adn_last_error", "adn_version"):
            fn.restype = C.c_int
    _lib = lib
    return lib
