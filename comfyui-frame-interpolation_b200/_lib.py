"""ctypes binding of libvfi_b200.so (declared in include/vfi_b200.h).  No fallback: a missing library is an error."""
import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libvfi_b200.so")

# every symbol include/vfi_b200.h declares (tests check the .so exports exactly these)
SYMBOLS = [
    "vfi_last_error", "vfi_version", "vfi_create", "vfi_destroy", "vfi_launch_count", "vfi_set_batch",
    "vfi_rife46_load", "vfi_rife_load", "vfi_rife46_forward", "vfi_rife46_interpolate_host", "vfi_warp_bilinear_border",
    "vfi_softsplat_sum", "vfi_softsplat_weighted", "vfi_costvol_l1", "vfi_corr_dot", "vfi_sepconv", "vfi_adacof", "vfi_edt_pass",
    "vfi_rife46_debug_layer", "vfi_rife46_debug_state", "vfi_rife46_layer_plan", "vfi_sync",
    "vfi_rife_profile", "vfi_rife_profile_read", "vfi_host_copy_frames",
    "vfi_film_load", "vfi_film_forward", "vfi_film_debug_set_ref", "vfi_film_debug_conv", "vfi_film_layer_plan",
    "vfi_film_last_macs", "vfi_film_debug_pack_host", "vfi_film_debug_state", "vfi_film_debug_elem",
    "vfi_sepconv_load", "vfi_sepconv_forward", "vfi_sepconv_debug_set_ref", "vfi_sepconv_debug_pack_host",
    "vfi_sepconv_debug_state", "vfi_sepconv_debug_elem",
    "vfi_flavr_load", "vfi_flavr_forward", "vfi_flavr_debug_set_ref", "vfi_flavr_debug_conv", "vfi_flavr_layer_plan",
    "vfi_flavr_info",
    "vfi_ifrnet_load", "vfi_ifrnet_forward", "vfi_ifrnet_geometry", "vfi_ifrnet_debug_set_ref", "vfi_ifrnet_debug_conv",
    "vfi_ifrnet_layer_plan", "vfi_ifrnet_info", "vfi_streamconv_debug_conv", "vfi_streamconv_plan",
    "vfi_cain_load", "vfi_cain_forward", "vfi_cain_geometry", "vfi_cain_debug_set_ref", "vfi_cain_debug_conv",
    "vfi_cain_layer_plan", "vfi_cain_debug_elem",
    "vfi_ifunet_load", "vfi_ifunet_forward", "vfi_ifunet_geometry", "vfi_ifunet_debug_set_ref", "vfi_ifunet_debug_conv",
    "vfi_ifunet_layer_plan", "vfi_ifunet_debug_elem",
    # GMFSS building blocks (argtypes are set by gmfss.Ops)
    "vfi_gm_conv2d", "vfi_gm_conv2d_packed", "vfi_gm_transpose", "vfi_gm_convt4", "vfi_gm_instance_norm", "vfi_gm_layer_norm", "vfi_gm_softmax_rows", "vfi_gm_gemm", "vfi_gm_window", "vfi_gm_nchw_tokens", "vfi_gm_add_position", "vfi_gm_local_match", "vfi_gm_local_prop", "vfi_gm_convex_up", "vfi_gm_warp_zeros", "vfi_gm_resize", "vfi_gm_metric_input", "vfi_gm_pixel_shuffle2", "vfi_gm_axpby", "vfi_gm_copy_slice",
]

_lib = None


class VfiError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise VfiError(
            f"{LIB_PATH} is missing: build it with `python __graft_entry__.py` (nvcc, sm_90a). "
            "There is no CPU or PyTorch fallback for this path.")
    L = C.CDLL(LIB_PATH)
    vp, i32, i64, f32 = C.c_void_p, C.c_int, C.c_int64, C.c_float
    L.vfi_last_error.restype = C.c_char_p
    L.vfi_version.restype = C.c_char_p
    L.vfi_create.argtypes = [i32, C.POINTER(vp)]
    L.vfi_destroy.argtypes = [vp]
    L.vfi_launch_count.argtypes = [vp]
    L.vfi_launch_count.restype = i64
    L.vfi_set_batch.argtypes = [vp, i32]
    L.vfi_rife46_load.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i32]
    L.vfi_rife_load.argtypes = [vp, i32, C.POINTER(vp), C.POINTER(i64), i32, i32]
    L.vfi_rife46_forward.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, vp, i32, f32, vp, vp]
    L.vfi_rife46_interpolate_host.argtypes = [vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, i32, f32, vp]
    L.vfi_warp_bilinear_border.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp]
    L.vfi_softsplat_sum.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp]
    L.vfi_softsplat_weighted.argtypes = [vp, vp, vp, vp, i32, i32, vp, vp, i32, i32, i32, i32, vp]
    L.vfi_costvol_l1.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp]
    L.vfi_corr_dot.argtypes = [vp, vp, vp, vp, i32, i32, i32, i32, vp]
    L.vfi_sepconv.argtypes = [vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, vp]
    L.vfi_adacof.argtypes = [vp, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, i32, vp]
    L.vfi_edt_pass.argtypes = [vp, vp, vp, i32, i32, i32, f32, vp]
    L.vfi_rife46_debug_layer.argtypes = [vp, i32, i32, vp, vp, vp, i32, i32, i32, i32, vp]
    L.vfi_rife46_debug_state.argtypes = [vp, vp, vp, i32, C.POINTER(i32), C.POINTER(i32)]
    L.vfi_rife46_layer_plan.argtypes = [vp, i32, i32, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32),
                                        C.POINTER(i32), C.POINTER(i64), C.POINTER(i32), C.POINTER(i32)]
    L.vfi_sync.argtypes = [vp]
    L.vfi_rife_profile.argtypes = [vp, i32]
    L.vfi_host_copy_frames.argtypes = [vp, i32, i32, i32, i32, vp, vp, i32]
    L.vfi_rife_profile_read.argtypes = [vp, vp, vp, vp, i32, C.POINTER(i32)]
    L.vfi_film_load.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i32]
    L.vfi_film_forward.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, i32, i32, vp, vp]
    L.vfi_film_debug_set_ref.argtypes = [vp, i32]
    L.vfi_film_debug_conv.argtypes = [vp, i32, i32, vp, i32, vp, i32, vp, i32, i32, i32, i32, i32, vp]
    L.vfi_film_layer_plan.argtypes = [vp, i32, i32] + [C.POINTER(i32)] * 10
    L.vfi_film_last_macs.argtypes = [vp]
    L.vfi_film_debug_pack_host.argtypes = [i32, i32, i32, i32, i32, i32, vp, i32, i32, vp, i64] + [C.POINTER(i32)] * 4
    L.vfi_film_last_macs.restype = i64
    L.vfi_film_debug_state.argtypes = [vp, i32, i32, vp, i32, C.POINTER(i32), C.POINTER(i32)]
    L.vfi_film_debug_elem.argtypes = [vp, i32, vp, i32, vp, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, f32, i32, i32,
                                      vp]
    L.vfi_sepconv_load.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i32]
    L.vfi_sepconv_forward.argtypes = [vp, vp, i32, i32, i32, i32, vp, vp, i32, vp, vp]
    L.vfi_sepconv_debug_set_ref.argtypes = [vp, i32]
    L.vfi_sepconv_debug_state.argtypes = [vp, i32, i32, vp, i32, C.POINTER(i32)]
    L.vfi_sepconv_debug_elem.argtypes = [vp, i32, vp, vp, vp, vp, i32, vp, i32, i32, i32, i32, i32, i32, f32, i32, vp]
    L.vfi_sepconv_debug_pack_host.argtypes = [i32, i32, i32, i32, i32, vp, vp, i64] + [C.POINTER(i32)] * 3
    L.vfi_flavr_load.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i32]
    L.vfi_flavr_forward.argtypes = [vp, vp, i32, i32, i32, i32, vp, i32, vp, vp]
    L.vfi_flavr_debug_set_ref.argtypes = [vp, i32]
    L.vfi_flavr_debug_conv.argtypes = [vp, i32, vp, i32, vp, i32, vp, i32, i32, i32, i32, i32, vp]
    L.vfi_flavr_layer_plan.argtypes = [vp, i32, vp, i32]
    L.vfi_flavr_info.argtypes = [vp, C.POINTER(i32), C.POINTER(i32)]
    f64 = C.c_double
    L.vfi_ifrnet_load.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i32]
    L.vfi_ifrnet_forward.argtypes = [vp, vp, vp, i32, i32, f64, f64, vp, vp]
    L.vfi_ifrnet_geometry.argtypes = [i32, i32, f64, vp, i32]
    L.vfi_ifrnet_debug_set_ref.argtypes = [vp, i32]
    L.vfi_ifrnet_debug_conv.argtypes = [vp, i32, vp, i32, vp, i32, vp, i32, vp, vp, i32, i32, i32, i32, i32, vp]
    L.vfi_ifrnet_layer_plan.argtypes = [vp, i32, vp, i32]
    L.vfi_ifrnet_info.argtypes = [vp, C.POINTER(i32)]
    L.vfi_cain_load.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i32]
    L.vfi_cain_forward.argtypes = [vp, vp, vp, i32, i32, vp, vp]
    L.vfi_cain_geometry.argtypes = [i32, i32, vp, i32]
    L.vfi_cain_debug_set_ref.argtypes = [vp, i32]
    L.vfi_cain_debug_conv.argtypes = [vp, i32, vp, i32, vp, i32, vp, i32, vp, i32, i32, i32, i32, vp]
    L.vfi_cain_layer_plan.argtypes = [vp, i32, vp, i32]
    L.vfi_cain_debug_elem.argtypes = [vp, i32, vp, vp, i32, i32, vp, vp, vp, i32, vp]
    L.vfi_ifunet_load.argtypes = [vp, C.POINTER(vp), C.POINTER(i64), i32, i32]
    L.vfi_ifunet_forward.argtypes = [vp, vp, vp, i32, i32, C.c_double, C.c_double, i32, vp, vp]
    L.vfi_ifunet_geometry.argtypes = [i32, i32, C.c_double, vp, i32]
    L.vfi_ifunet_debug_set_ref.argtypes = [vp, i32]
    L.vfi_ifunet_debug_conv.argtypes = [vp, i32, vp, i32, vp, i32, vp, i32, vp, vp, i32, i32, i32, i32, i32, vp]
    L.vfi_ifunet_layer_plan.argtypes = [vp, i32, vp, i32]
    L.vfi_ifunet_debug_elem.argtypes = [vp, i32, vp, vp, i32, i32, C.c_double, C.c_double, vp, vp, vp, i32, vp]
    L.vfi_streamconv_debug_conv.argtypes = [vp, i32, f32, i32, vp, vp, vp, vp, i32, vp, i32, vp, i32, vp, vp, i32, i32, i32,
                                            i32, i32, i32, vp]
    L.vfi_streamconv_plan.argtypes = [vp, i32, vp, i32]
    for name in SYMBOLS:
        if name not in ("vfi_last_error", "vfi_version", "vfi_launch_count", "vfi_film_last_macs"):
            getattr(L, name).restype = i32
    _lib = L
    return L


def check(rc):
    if rc != 0:
        raise VfiError(f"libvfi_b200 error {rc}: {lib().vfi_last_error().decode()}")
