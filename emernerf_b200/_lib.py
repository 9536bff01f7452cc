"""ctypes binding of libemer_b200.so -- the C-ABI boundary (include/emer_b200.h).

There is no CPU or library fallback: if the shared library cannot be loaded (or built with the
local nvcc) every op raises.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, c_char_p, c_double, c_float, c_int, c_int32, c_int64, c_void_p

from .grid_desc import EmerGridDesc

_LIB = None
_P = c_void_p

# host structs of emer_render_fwd / emer_render_bwd (include/emer_b200.h): field names and order as there
RENDER_IN_PTRS = ("t0", "t1", "sigma", "sigma_s", "sigma_d", "rgb", "rgb_s", "rgb_d", "shadow", "rgb_sky", "dino",
                  "dino_s", "dino_d", "dino_sky", "dino_pe", "fwd_flow", "bwd_flow")
RENDER_OUT_PTRS = ("weights", "trans", "opacity", "depth", "median_depth", "rgb", "shadow_ratio", "dino", "dino_pe_free",
                   "static_opacity", "dynamic_opacity", "static_depth", "dynamic_depth", "static_rgb", "dynamic_rgb",
                   "shadow_reduced_static_rgb", "shadow_only_static_rgb", "shadow", "forward_flow", "backward_flow",
                   "static_dino", "dynamic_dino")
RENDER_GRAD_PTRS = ("g_weights", "g_trans", "g_opacity", "g_depth", "g_rgb", "g_shadow_ratio", "g_dino",
                    "g_dino_pe_free", "d_sigma", "d_sigma_s", "d_sigma_d", "d_rgb", "d_rgb_s", "d_rgb_d", "d_shadow",
                    "d_rgb_sky", "d_dino", "d_dino_s", "d_dino_d", "d_dino_sky", "d_dino_pe")


class EmerRenderIn(ctypes.Structure):
    _fields_ = [(k, _P) for k in RENDER_IN_PTRS] + [("ld_flow", c_int64), ("n_rays", c_int64),
                                                     ("n_samples", c_int32), ("n_dino", c_int32)]


class EmerRenderOut(ctypes.Structure):
    _fields_ = [(k, _P) for k in RENDER_OUT_PTRS]


class EmerRenderGrad(ctypes.Structure):
    _fields_ = [(k, _P) for k in RENDER_GRAD_PTRS]


# host structs of emer_pixel_batch (include/emer_b200.h): field names and order as there
PIXEL_BATCH_IN_PTRS = ("cand", "u_pick", "u_x", "u_y", "i_sel", "i_dy", "i_dx", "images", "sky_masks", "dynamic_masks",
                       "features", "timestamps", "cam_ids", "c2w", "intrinsics")
PIXEL_BATCH_OUT_PTRS = ("img_idx", "cam_idx", "pixels", "sky_masks", "dynamic_masks", "features", "timestamps",
                        "origins", "viewdirs", "norms", "pixel_coords")


class EmerPixelBatchIn(ctypes.Structure):
    _fields_ = [(k, _P) for k in PIXEL_BATCH_IN_PTRS] + [
        ("n_uniform", c_int64), ("n_importance", c_int64), ("height", c_int32), ("width", c_int32),
        ("map_h", c_int32), ("map_w", c_int32), ("map_downscale", c_int32), ("feat_h", c_int32), ("feat_w", c_int32),
        ("feat_c", c_int32), ("feat_scale_y", c_float), ("feat_scale_x", c_float)]


class EmerPixelBatchOut(ctypes.Structure):
    _fields_ = [(k, _P) for k in PIXEL_BATCH_OUT_PTRS]


# host structs of emer_image_rays (include/emer_b200.h): field names and order as there
IMAGE_RAYS_IN_PTRS = ("sky_masks", "dynamic_masks", "features", "timestamps", "cam_ids", "c2w", "intrinsics")
IMAGE_RAYS_OUT_PTRS = ("origins", "viewdirs", "norms", "pixel_coords", "timestamps", "img_idx", "cam_idx", "sky_masks",
                       "dynamic_masks", "features")


class EmerImageRaysIn(ctypes.Structure):
    _fields_ = [(k, _P) for k in IMAGE_RAYS_IN_PTRS] + [
        ("first_image", c_int64), ("n_images", c_int64), ("height", c_int32), ("width", c_int32), ("h", c_int32),
        ("w", c_int32), ("downscale", c_float), ("mask_scale_y", c_float), ("mask_scale_x", c_float),
        ("feat_h", c_int32), ("feat_w", c_int32), ("feat_c", c_int32), ("feat_scale_y", c_float),
        ("feat_scale_x", c_float)]


class EmerImageRaysOut(ctypes.Structure):
    _fields_ = [(k, _P) for k in IMAGE_RAYS_OUT_PTRS]


# host structs of emer_trajectory_rays (include/emer_b200.h): field names and order as there
TRAJECTORY_RAYS_OUT_PTRS = ("origins", "viewdirs", "norms", "pixel_coords", "timestamps", "img_idx", "cam_idx",
                            "sky_masks")


class EmerTrajectoryRaysIn(ctypes.Structure):
    _fields_ = [("c2w", _P), ("intrinsics", _P), ("timestamps", _P), ("n_images", c_int64), ("image_a", c_int64),
                ("image_b", c_int64), ("cam_id", c_int64), ("offset", c_double * 3), ("frac_num", c_int32),
                ("frac_den", c_int32), ("h", c_int32), ("w", c_int32), ("downscale", c_float)]


class EmerTrajectoryRaysOut(ctypes.Structure):
    _fields_ = [(k, _P) for k in TRAJECTORY_RAYS_OUT_PTRS]

# number of kernels this library launched through the C ABI (bench.py reports it as gpu_launches)
LAUNCHES = 0

_SIGNATURES = {
    "emer_grid_fwd": [POINTER(EmerGridDesc), _P, _P, _P, c_int64, _P],
    "emer_grid_bwd": [POINTER(EmerGridDesc), _P, _P, _P, _P, _P, c_int64, _P],
    "emer_grid_indices": [POINTER(EmerGridDesc), _P, _P, c_int64, _P],
    "emer_contract_fwd": [_P, _P, _P, _P, c_int, c_int, c_int, c_int64, _P],
    "emer_contract_bwd": [_P, _P, _P, _P, _P, c_int, c_int, c_int, c_int64, _P],
    "emer_trunc_exp_fwd": [_P, c_int64, _P, c_int64, _P],
    "emer_trunc_exp_bwd": [_P, c_int64, _P, _P, c_int64, _P],
    "emer_linear_fwd": [_P, c_int64, _P, _P, _P, c_int64, c_int64, c_int, c_int, c_int, _P],
    "emer_linear_bwd_data": [_P, c_int64, _P, c_int64, c_int, _P, _P, c_int64, c_int64, c_int, c_int, c_int, _P],
    "emer_linear_bwd_weight": [_P, c_int64, _P, c_int64, _P, c_int64, c_int, _P, _P, c_int64, c_int, c_int, _P],
    "emer_linear_narrow_fwd": [_P, c_int64, _P, _P, _P, c_int64, c_int64, c_int, c_int, c_int, _P],
    "emer_linear_narrow_bwd_data": [_P, c_int64, _P, _P, c_int64, _P, c_int64, c_int, c_int64, c_int, c_int, _P],
    "emer_linear_narrow_bwd_weight": [_P, c_int64, _P, c_int64, _P, _P, c_int64, c_int, c_int, _P],
    "emer_linear_tc_fwd": [_P, c_int64, _P, _P, _P, c_int64, c_int64, c_int, c_int, c_int, _P],
    "emer_linear_tc_bwd_data": [_P, c_int64, _P, c_int64, c_int, _P, _P, c_int64, _P, c_int64, c_int, c_int64, c_int,
                                c_int, c_int, _P],
    "emer_linear_tc_bwd_weight": [_P, c_int64, _P, c_int64, _P, _P, c_int64, c_int, c_int, _P],
    "emer_pdf_resample": [_P, _P, c_int, c_int, _P, c_float, c_float, c_int, _P, _P, _P, c_int64, _P],
    "emer_prop_level": [POINTER(EmerGridDesc), _P, _P, c_int, c_int, _P, c_float, c_float, c_int, _P, _P, _P, c_int, _P,
                        _P, _P, _P, _P, _P, _P, _P, _P, c_int64, _P],
    "emer_prop_level_bwd": [POINTER(EmerGridDesc), _P, _P, _P, c_int, _P, _P, _P, c_int, _P, _P, _P, _P, _P, _P, _P, _P,
                            _P, _P, c_int64, _P],
    "emer_interlevel_loss": [_P, _P, c_int, _P, _P, c_int, c_float, _P, _P, c_int64, _P],
    "emer_field_tail_fwd": [_P, c_int64, c_int, _P, _P, _P, c_int, _P, c_int64, _P, c_int64, c_int, _P],
    "emer_field_tail_bwd": [_P, c_int64, _P, c_int64, c_int, _P, _P, _P, c_int, c_int64, c_int, _P],
    "emer_field_fwd": [_P, c_int64, c_int, _P, _P, _P, _P, c_int, _P, c_int64, _P, _P, c_int64, _P, _P, _P, c_int, _P, _P, _P,
                       _P, _P, _P, c_int64, _P],
    "emer_field_bwd": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, _P, c_int, _P, c_int64, _P, _P, c_int64, _P, _P, _P, _P,
                       _P, _P, c_int64, _P, c_int, c_int64, _P],
    "emer_field_wgrad": [_P, c_int64, c_int, _P, _P, _P, _P, _P, _P, _P, _P, c_int, _P, _P, _P, _P, _P, c_int64, _P, _P,
                         c_int64, _P, _P, c_int64, _P],
    "emer_flow_field_fwd": [_P, c_int64, c_int, _P, _P, _P, _P, c_int, _P, c_int64, _P, _P, c_int64, _P, _P, _P, c_int, _P, _P,
                            _P, _P, _P, _P, c_int64, _P],
    "emer_flow_field_bwd": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int, _P, c_int, _P, c_int64, _P, _P, c_int64, _P, _P, _P,
                            _P, _P, _P, c_int64, _P, _P, c_int, c_int64, _P],
    "emer_flow_warp_fwd": [_P, _P, _P, c_int64, _P, _P, _P, c_int, _P, c_int64, _P],
    "emer_flow_warp_bwd": [_P, _P, _P, c_int64, _P, c_int, _P, _P, c_int64, _P],
    "emer_gen_rays": [_P, _P, _P, _P, _P, c_int, _P, c_int, c_int, _P, _P, _P, _P, _P, c_int64, _P],
    "emer_topk_ratio": [_P, c_int64, _P, c_int64, _P, c_int64, _P, _P, _P],
    "emer_pixel_batch": [POINTER(EmerPixelBatchIn), POINTER(EmerPixelBatchOut), _P],
    "emer_image_rays": [POINTER(EmerImageRaysIn), POINTER(EmerImageRaysOut), _P],
    "emer_trajectory_rays": [POINTER(EmerTrajectoryRaysIn), POINTER(EmerTrajectoryRaysOut), _P],
    "emer_error_map": [_P, _P, _P, c_int64, _P, _P, _P],
    "emer_error_map_normalize": [_P, c_int64, _P, _P],
    "emer_adam_step": [_P, _P, c_int, c_int64, _P, c_float, c_float, c_float, c_float, c_int, _P],
    "emer_composite_fwd": [_P, _P, _P, _P, _P, _P, _P, _P, _P, c_int64, c_int, _P],
    "emer_composite_bwd": [_P, _P, _P, _P, _P, _P, _P, _P, _P, _P, c_int64, c_int, _P],
    "emer_accumulate_fwd": [_P, _P, _P, c_int64, c_int, c_int, _P],
    "emer_accumulate_bwd": [_P, _P, _P, _P, _P, c_int64, c_int, c_int, _P],
    "emer_pointwise_loss_fwd": [c_int, _P, _P, c_int64, c_float, c_float, c_float, c_float, _P, _P, _P],
    "emer_pointwise_loss_bwd": [c_int, _P, _P, c_int64, c_float, c_float, c_float, c_float, _P, _P, _P, _P, _P],
    "emer_ray_loss_fwd": [c_int, _P, _P, _P, c_int64, c_int, c_float, c_float, c_float, c_float, c_float, _P, _P, _P],
    "emer_ray_loss_bwd": [c_int, _P, _P, _P, c_int64, c_int, c_float, c_float, c_float, c_float, c_float, _P, _P, _P,
                          _P],
    "emer_ray_loss_live_fwd": [c_int, _P, _P, _P, c_int64, c_int, _P, c_float, _P, _P, _P],
    "emer_ray_loss_live_bwd": [c_int, _P, _P, _P, c_int64, c_int, _P, c_float, _P, _P, _P, _P],
    "emer_cycle_loss_fwd": [_P, c_int64, _P, c_int64, _P, c_int64, _P, c_int64, c_int64, c_float, _P, _P, _P],
    "emer_cycle_loss_bwd": [_P, c_int64, _P, c_int64, _P, c_int64, _P, c_int64, c_int64, c_float, _P, _P, _P, _P, _P],
    "emer_render_fwd": [POINTER(EmerRenderIn), POINTER(EmerRenderOut), _P],
    "emer_render_bwd": [POINTER(EmerRenderIn), _P, _P, POINTER(EmerRenderGrad), _P],
    "emer_image_metrics": [_P, _P, c_int64, c_int64, c_int, _P, _P, c_int64, _P, c_int64, c_int, _P, _P, _P],
    "emer_depth_rmse": [_P, _P, c_int64, _P, _P, _P],
    "emer_scene_flow_metrics": [_P, _P, c_int64, _P, _P, _P],
    "emer_lidar_flow_accumulate": [_P, c_int64, _P, _P, _P, _P, c_int64, c_float, _P, _P, _P],
    "emer_occ_accumulate": [_P, c_int64, c_int, _P, c_int64, _P, c_int64, c_int, c_float, _P, _P, _P, _P],
    "emer_occ_classify": [_P, c_int64, c_int, _P, c_int64, _P, c_int64, _P, c_int, _P, c_float, _P, _P, _P],
}

EXPORTS = sorted(list(_SIGNATURES) + ["emer_last_error", "emer_version"])


def lib_path() -> str:
    return os.path.join(os.path.dirname(os.path.abspath(__file__)), "lib", "libemer_b200.so")


def load():
    """Load (building first if the .so is absent) and type the library.  Raises on failure."""
    global _LIB
    if _LIB is not None:
        return _LIB
    path = lib_path()
    from .build import build_library

    # (re)build when the library is missing OR stale: build_library() returns at once when build.stamp matches the
    # digest of the sources, so an edited .cu / header can never run as an old binary
    build_library()
    lib = ctypes.CDLL(path)
    for name, argtypes in _SIGNATURES.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = c_int
    lib.emer_last_error.restype = c_char_p
    lib.emer_version.restype = c_int
    _LIB = lib
    return lib


_PROFILE = None      # (predicate(name, args) -> bool, list receiving (name, tag, ev_start, ev_end))


def set_profile(predicate, sink) -> None:
    """bench.py hook: CUDA-event timing of selected launches on the launching stream."""
    global _PROFILE
    _PROFILE = None if predicate is None else (predicate, sink)


def tag_of(name: str, args) -> str:
    """Shape tag of a launch, e.g. ``D3L10F4_N524288`` for grid calls, ``k40_o64_N524288`` for layers."""
    try:
        if name in ("emer_grid_fwd", "emer_grid_bwd"):
            g = args[0]._obj
            n = args[4] if name == "emer_grid_fwd" else args[6]
            extra = ""
            if name == "emer_grid_bwd":
                extra = ("_T" if args[4].value else "") + ("_X" if args[5].value else "")
            return f"D{g.n_dims}L{g.n_levels}F{g.n_feat}_N{n}{extra}"
        if name == "emer_linear_narrow_fwd":
            return f"k{args[7]}_o{args[8]}_N{args[6]}"
        if name == "emer_linear_narrow_bwd_data":
            return f"k{args[9]}_o{args[10]}_N{args[8]}"
        if name == "emer_linear_narrow_bwd_weight":
            return f"k{args[7]}_o{args[8]}_N{args[6]}"
        if name in ("emer_linear_tc_fwd",):
            return f"k{args[7]}_o{args[8]}_N{args[6]}"
        if name in ("emer_linear_tc_bwd_data",):
            return f"k{args[12]}_o{args[13]}_N{args[11]}"
        if name == "emer_linear_fwd":
            return f"k{args[7]}_o{args[8]}_N{args[6]}"
        if name == "emer_linear_bwd_data":
            return f"k{args[9]}_o{args[10]}_N{args[8]}"
        if name == "emer_linear_tc_bwd_weight":
            return f"k{args[7]}_o{args[8]}_N{args[6]}"
        if name == "emer_linear_bwd_weight":
            return f"k{args[10]}_o{args[11]}_N{args[9]}"
        if name == "emer_field_bwd":
            return f"k{args[10]}_f{args[12]}_N{args[27]}"
        if name == "emer_field_wgrad":
            return f"k{args[2]}_f{args[11]}_N{args[23]}"
        if name in ("emer_pointwise_loss_fwd", "emer_pointwise_loss_bwd"):
            return f"kind{args[0]}_N{args[3]}"
        if name in ("emer_ray_loss_fwd", "emer_ray_loss_bwd", "emer_ray_loss_live_fwd", "emer_ray_loss_live_bwd"):
            return f"kind{args[0]}_R{args[4]}_S{args[5]}"
        if name in ("emer_cycle_loss_fwd", "emer_cycle_loss_bwd"):
            return f"N{args[8]}"
        if name == "emer_image_metrics":
            return f"H{args[2]}_W{args[3]}_C{args[4]}_F{args[10]}"
        if name in ("emer_depth_rmse", "emer_scene_flow_metrics"):
            return f"N{args[2]}"
        if name == "emer_lidar_flow_accumulate":
            return f"N{args[6]}" + ("_G" if args[5].value else "")
        if name == "emer_occ_accumulate":
            return f"C{args[2]}_K{args[7]}_N{args[6]}"
        if name == "emer_occ_classify":
            return f"C{args[2]}_K{args[8]}_N{args[6]}"
        if name == "emer_flow_field_fwd":
            return f"k{args[2]}_f{args[7]}_N{args[23]}" + ("" if args[18].value else "_density")
        if name == "emer_flow_field_bwd":
            return f"k{args[10]}_f{args[12]}_N{args[29]}"
        if name in ("emer_flow_warp_fwd", "emer_flow_warp_bwd"):
            return f"N{args[9] if name == 'emer_flow_warp_fwd' else args[8]}"
        if name == "emer_field_fwd":
            return f"k{args[2]}_f{args[7]}_N{args[23]}" + ("_save" if args[19].value else "")
    except Exception:
        pass
    return ""


def algorithmic_bytes(tag: str) -> int:
    """Algorithmic bytes of one grid-forward launch from its tag: N * (L*2^D*F*4 + D*4 + L*F*4)
    (SURVEY.md section 8d)."""
    import re

    m = re.match(r"D(\d+)L(\d+)F(\d+)_N(\d+)", tag)
    d, l, f, n = (int(x) for x in m.groups())
    return n * (l * (2 ** d) * f * 4 + d * 4 + l * f * 4)


# device of the tensors of the op being launched (set by _ops._need_cuda); kernels launch on the CUDA runtime's
# current device, so a call for tensors elsewhere is wrapped in a device guard
DEVICE = None


def call(name: str, *args) -> None:
    if DEVICE is not None:
        import torch

        if DEVICE != torch.cuda.current_device():
            with torch.cuda.device(DEVICE):
                return _call(name, *args)
    return _call(name, *args)


def _call(name: str, *args) -> None:
    global LAUNCHES
    lib = load()
    prof = _PROFILE
    if prof is not None and prof[0](name, args):
        import torch

        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        rc = getattr(lib, name)(*args)
        e1.record()
        prof[1].append((name, tag_of(name, args), e0, e1))
    else:
        rc = getattr(lib, name)(*args)
    LAUNCHES += 1
    if rc != 0:
        raise RuntimeError(f"{name} failed ({rc}): {lib.emer_last_error().decode()}")
