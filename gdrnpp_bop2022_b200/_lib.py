"""ctypes binding of libgdrn_b200.so (the C ABI declared in include/gdrn_b200.h).

The product path has no CPU fallback: if the shared library is missing or a call fails, we raise.
"""
import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_uint, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgdrn_b200.so")

_lib = None


class GdrnError(RuntimeError):
    pass


class GdrnMaps(ctypes.Structure):
    _fields_ = [
        ("mask", c_void_p),
        ("full_mask", c_void_p),
        ("coor_x", c_void_p),
        ("coor_y", c_void_p),
        ("coor_z", c_void_p),
        ("region", c_void_p),
    ]


_SIGNATURES = {
    "gdrn_last_error": (c_char_p, []),
    "gdrn_version": (c_int, []),
    "gdrn_launch_count": (ctypes.c_longlong, []),
    "gdrn_model_set_profiling": (c_int, [c_void_p, c_int]),
    "gdrn_model_get_profile": (c_int, [c_void_p, c_void_p, c_void_p]),
    "gdrn_model_create": (c_int, [POINTER(c_void_p), c_char_p, c_int, c_int]),
    "gdrn_model_create_ex": (c_int, [POINTER(c_void_p), c_char_p, c_int, c_int, c_int]),
    "gdrn_model_precision": (c_int, [c_void_p]),
    "gdrn_model_destroy": (None, [c_void_p]),
    "gdrn_model_load_tensor": (c_int, [c_void_p, c_char_p, c_void_p, c_int64, c_void_p]),
    "gdrn_model_missing": (c_int, [c_void_p]),
    "gdrn_model_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "gdrn_model_forward": (
        c_int,
        [c_void_p] + [c_void_p] * 8 + [c_int] + [c_void_p] * 3 + [POINTER(GdrnMaps), c_void_p, c_size_t, c_void_p],
    ),
    "gdrn_model_debug_read": (c_int64, [c_void_p, c_char_p, c_int, c_void_p, c_void_p, c_void_p]),
    "gdrn_model_run_stage": (c_int, [c_void_p, c_char_p, c_int] + [c_void_p] * 7 + [POINTER(GdrnMaps), c_void_p, c_size_t,
                                                                                  c_void_p]),
    "gdrn_gemm_bf16": (c_int, [c_void_p] * 6 + [c_int] * 6 + [c_void_p]),
    "gdrn_mlp_fused_x3": (c_int, [c_void_p] * 7 + [ctypes.c_longlong, c_int, c_void_p]),
    "gdrn_dwconv_ln": (c_int, [c_void_p] * 6 + [c_int] * 4 + [c_float, c_int, c_int, c_void_p]),
    "gdrn_gemm_x3": (c_int, [c_void_p] * 6 + [c_int] * 5 + [c_void_p]),
    "gdrn_gemm_x3_ksplit": (c_int, [c_void_p] * 5 + [c_int] * 4 + [c_void_p, c_int, c_void_p]),
    "farthest_point_sampling": (None, [c_void_p, c_void_p, c_int, c_int]),
    "farthest_point_sampling_init_center": (None, [c_void_p, c_void_p, c_int, c_int]),
    "gdrn_fps_set_seed": (None, [c_uint]),
    "gdrn_fps_cuda": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "rv_generate_hypothesis": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p]),
    "rv_voting_for_hypothesis": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_float, c_void_p]),
    "rv_generate_hypothesis_vanishing_point": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_void_p]),
    "rv_voting_for_hypothesis_vanishing_point": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_float, c_void_p]),
    "rv_vote_count": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_float, c_int, c_void_p]),
    "rv_layer_workspace_bytes": (c_size_t, [c_int] * 5),
    "rv_ransac_voting_layer": (c_int, [c_void_p, c_void_p] + [c_int] * 5 + [c_float, c_int, c_int, c_uint] + [c_void_p] * 7
                               + [c_size_t, c_void_p]),
    "nnd_forward_cuda": (c_int, [c_void_p] * 6 + [c_int] * 3 + [c_void_p]),
    "nnd_backward_cuda": (c_int, [c_void_p] * 8 + [c_int] * 3 + [c_void_p]),
    "flow_forward_cuda": (c_int, [c_void_p] * 6 + [c_int] * 3 + [c_void_p]),
    "uncertainty_pnp": (None, [c_void_p] * 6 + [c_int]),
    "upnp_batched": (c_int, [c_void_p] * 6 + [c_int, c_int, c_void_p]),
    "rast_render_depth": (
        c_int,
        [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_float, c_int]
        + [c_void_p] * 4,
    ),
    "rast_scratch_bytes": (c_size_t, [c_int, c_int, c_int]),
    "gdrn_depth_refine_step": (c_int, [c_void_p] * 6 + [c_int, c_int, c_float, c_void_p]),
    "gdrn_depth_refine_step_ex": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 4 + [c_int, c_int, c_float, c_void_p]),
    "gdrn_depth_refine_step_weighted": (c_int, [c_void_p, c_void_p, c_int] + [c_void_p] * 4 + [c_int, c_void_p, c_int, c_int, c_float,
                                                                                          c_void_p]),
    "rast_upload_mesh": (c_int, [c_void_p, c_int, c_void_p, c_int]),
    "rast_mesh_count": (c_int, []),
    "rast_free_meshes": (None, []),
    "rast_render_meshes": (c_int, [c_void_p] * 3 + [c_int] * 3 + [c_float, c_float, c_int] + [c_void_p] * 4),
    "gdrn_pnp_ransac_maps": (c_int, [c_void_p] * 9 + [c_int] * 3 + [c_float, c_float, c_uint] + [c_void_p] * 4),
    "gdrn_pnp_ransac_points": (c_int, [c_void_p] * 4 + [c_int] * 3 + [c_float, c_uint] + [c_void_p] * 4),
    "gdrn_pnp_net_maps": (c_int, [c_void_p] * 10 + [c_int] * 3 + [c_float, c_float, c_int, c_uint] + [c_void_p] * 3),
    "gdrn_pnp_iterative_points": (c_int, [c_void_p] * 5 + [c_int, c_int, c_void_p, c_void_p]),
    "gdrn_xyz_region_targets": (c_int, [c_void_p] * 6 + [c_int] * 4 + [c_void_p] * 5),
    "yolox_postprocess_workspace_bytes": (c_size_t, [c_int, c_int]),
    "yolox_postprocess": (c_int, [c_void_p] + [c_int] * 3 + [c_void_p, c_void_p, c_int, c_float, c_float, c_int, c_int, c_void_p, c_void_p,
                                  c_void_p, c_size_t, c_void_p]),
    "yolox_model_create": (c_int, [POINTER(c_void_p), c_double, c_double] + [c_int] * 5),
    "yolox_model_destroy": (None, [c_void_p]),
    "yolox_model_load_tensor": (c_int, [c_void_p, c_char_p, c_void_p, c_int64, c_void_p]),
    "yolox_model_missing": (c_int, [c_void_p]),
    "yolox_model_num_anchors": (c_int, [c_void_p]),
    "yolox_model_workspace_bytes": (c_size_t, [c_void_p, c_int]),
    "yolox_model_forward": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "yolox_model_set_scales": (c_int, [c_void_p, POINTER(c_double), c_int]),
    "yolox_model_num_anchors_tta": (c_int, [c_void_p]),
    "yolox_model_workspace_bytes_tta": (c_size_t, [c_void_p, c_int]),
    "yolox_model_forward_tta": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_size_t, c_void_p]),
    "yolox_postprocess_single_workspace_bytes": (c_size_t, [c_int] * 3),
    "yolox_postprocess_single": (c_int, [c_void_p] + [c_int] * 3 + [c_float, c_float] + [c_void_p] * 3 + [c_size_t, c_void_p]),
    "gdrn_crop_resize_u8": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p]),
    "gdrn_crop_resize_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "gdrn_roi_setup": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_double, c_int, c_int]
                       + [c_void_p] * 12 + [c_void_p]),
    "gdrn_roi_crop_multi": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                    c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p]),
    "gdrn_vsd_workspace_bytes": (c_size_t, [c_int, c_int]),
    "gdrn_vsd_errors": (c_int, [c_void_p] * 3 + [c_int, c_int] + [c_void_p] * 6 + [c_int, c_void_p, c_int, c_float, c_int,
                                                                                 c_void_p, c_size_t, c_void_p, c_void_p]),
    "gdrn_sym_max_dist": (c_int, [c_void_p] * 9 + [c_int, c_int] + [c_void_p] * 3),
    "gdrn_ad_workspace_bytes": (c_size_t, [c_int, c_int]),
    "gdrn_ad_errors": (c_int, [c_void_p] * 7 + [c_int, c_int, c_void_p, c_size_t, c_void_p, c_void_p]),
    "gdrn_sym_proj_mean": (c_int, [c_void_p] * 9 + [c_int, c_int] + [c_void_p] * 2),
    "gdrn_sym_rt_errors": (c_int, [c_void_p] * 6 + [c_int] + [c_void_p] * 3),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES.keys())


def lib():
    """Load (once) and return the ctypes handle; raises GdrnError when the extension is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GdrnError(
                f"{LIB_PATH} not found: build it with `python -m gdrnpp_bop2022_b200.build` "
                "(there is no CPU fallback for the product path)"
            )
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(h, name)
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def last_error():
    return lib().gdrn_last_error().decode("utf-8", "replace")


def check(rc, what):
    if rc != 0:
        raise GdrnError(f"{what} failed (code {rc}): {last_error()}")


def ptr(t):
    """data pointer of a torch tensor (or None)."""
    if t is None:
        return None
    return c_void_p(t.data_ptr())


def current_stream():
    """Current stream of the CURRENT device (wrappers make their tensors' device current first, see on_device)."""
    import torch

    return c_void_p(torch.cuda.current_stream().cuda_stream)


def on_device(argidx=0):
    """Decorator: run the wrapped call with the CUDA device of positional argument ``argidx`` made current.  The C ABI
    launches on the current device and takes the current stream, so a tensor on cuda:1 must not be processed while
    cuda:0 is current (the kernels' shared-memory opt-in and the SM-count cache are per device too)."""
    import functools

    def deco(fn):
        @functools.wraps(fn)
        def wrapped(*a, **k):
            import torch

            t = a[argidx] if len(a) > argidx else None
            if torch.is_tensor(t) and t.is_cuda:
                with torch.cuda.device(t.device):
                    return fn(*a, **k)
            return fn(*a, **k)

        return wrapped

    return deco
