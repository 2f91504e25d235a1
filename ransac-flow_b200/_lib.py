"""ctypes binding of the C ABI in include/ransacflow_b200.h.

There is no Python/CPU fallback: if ``libransacflow_b200.so`` is missing and
cannot be built (nvcc), importing the package raises.  Compute entry points
additionally require CUDA tensors (``need_cuda``)."""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libransacflow_b200.so")

vp, i32, i64, f32, sz = C.c_void_p, C.c_int, C.c_longlong, C.c_float, C.c_size_t

# name -> (restype, argtypes); every symbol declared in include/ransacflow_b200.h
SIGNATURES = {
    "rf_version": (i32, []),
    "rf_source_digest": (C.c_char_p, []),
    "rf_last_error_string": (C.c_char_p, []),
    "rf_launch_count": (C.c_uint64, []),
    "rf_l2norm_f16_nhwc": (i32, [vp, i64, i32, vp, vp, vp]),
    "rf_l2norm_split_nhwc": (i32, [vp, i64, i32, vp, vp, vp, vp, vp]),
    "rf_corr_neigh_pair_split": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp]),
    "rf_corr_mutual_nn_workspace": (sz, [i32, i32, i32, i32]),
    "rf_corr_mutual_nn_launches": (i32, [i32]),
    "rf_corr_mutual_nn": (i32, [vp, i32, vp, i32, i32, vp, vp, vp, vp, sz, i32, vp]),
    "rf_corr_mutual_nn_presplit_workspace": (sz, [i32, i32]),
    "rf_corr_mutual_nn_presplit": (i32, [vp, vp, i32, vp, vp, i32, i32, vp, vp, vp, vp, sz, vp]),
    "rf_ransac_workspace": (sz, [i32]),
    "rf_ransac_homography": (i32, [vp, vp, i32, vp, vp, i32, i32, f32, i32, vp, vp, vp, vp, vp, sz, vp]),
    "rf_ransac_homography_drawn": (i32, [vp, vp, i32, vp, vp, i32, i32, i32, f32, i32, vp, vp, vp, vp, vp, vp, vp, sz, vp]),
    "rf_yfcc_rotation_select": (i32, [vp, vp, vp, vp, i32, vp, vp]),
    "rf_select_copy": (i32, [vp, i32, vp, vp, sz, vp]),
    "rf_homography_dlt": (i32, [vp, vp, i32, vp, vp]),
    "rf_prediction": (i32, [vp, vp, i32, vp, i32, vp, vp]),
    "rf_build_matches": (i32, [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp, i32, vp]),
    "rf_conv2d_nhwc": (i32, [vp, i32, vp, i32, vp, vp, vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, vp]),
    "rf_conv1x1_dual_split": (i32, [vp, vp, i32, vp, vp, i32, i32, i32, vp, vp, i32, i32, vp, vp]),
    "rf_maxpool2d_nhwc": (i32, [vp, i32, vp, i32, i32, i32, i32, vp, vp]),
    "rf_blur_downsample_nhwc": (i32, [vp, i32, vp, i32, i32, vp, vp]),
    "rf_l2norm_nhwc": (i32, [vp, i64, i32, vp, vp, vp]),
    "rf_corr_neigh_nhwc": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, vp]),
    "rf_corr_neigh_pair_nhwc": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, vp, vp]),
    "rf_run_layers": (i32, [vp, i32, vp, i32, vp, i32, vp]),
    "rf_softmax_flow": (i32, [vp, i32, i32, i32, i32, vp, vp]),
    "rf_sigmoid": (i32, [vp, i64, vp, vp]),
    "rf_preproc_u8": (i32, [vp, i64, i32, vp, vp]),
    "rf_resample_u8": (i32, [vp, i32, i32, i32, i32, vp, vp, i32, i32, vp, vp]),
    "rf_lanczos_coeffs_host": (i32, [i32, i32, vp, vp, i32, vp]),
    "rf_bilinear_coeffs_host": (i32, [i32, i32, vp, vp, i32, vp]),
    "rf_bytescale_mask_u8_workspace": (sz, [i32, i32]),
    "rf_bytescale_mask_u8": (i32, [vp, i32, i32, i32, vp, vp, sz, vp]),
    "rf_adaptive_avgpool_split": (i32, [vp, i32, vp, i32, vp, i32, vp, vp]),
    "rf_ppm_concat_split": (i32, [vp, i32, vp, i32, vp, vp, i32, i32, vp, vp]),
    "rf_seg_vote": (i32, [vp, i32, vp, i32, vp, i32, i32, i32, i32, i32, vp, vp, vp, vp]),
    "rf_warp_grid": (i32, [vp, i32, i32, i32, vp, vp]),
    "rf_grid_sample": (i32, [vp, i32, i32, i32, i32, vp, vp, i32, i32, i32, vp, vp, vp]),
    "rf_warp_sample_u8": (i32, [vp, vp, i32, i32, i32, i32, i32, vp, vp]),
    "rf_affine_sample_u8": (i32, [vp, vp, i32, i32, i32, i32, vp, vp]),
    "rf_val_keypoints": (i32, [vp, i32, i32, vp, i32, i32, i32, i32, vp, vp, i32, i32, vp, i32, vp, vp, vp, vp, vp]),
    "rf_upsample_bilinear": (i32, [vp, i32, i32, i32, i32, i32, vp, vp]),
    "rf_compose_fine": (i32, [vp, vp, vp, i32, i32, vp, i32, i32, i32, i32, vp, vp, vp, vp]),
    "rf_compose_fine_ex": (i32, [vp, vp, vp, i32, i32, vp, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp]),
    "rf_fill_nearest_matched_workspace": (sz, [i32, i32]),
    "rf_fill_nearest_matched": (i32, [vp, vp, i32, i32, vp, vp, vp, sz, vp]),
    "rf_remove_small_cc_workspace": (sz, [i32, i32]),
    "rf_remove_small_cc": (i32, [vp, i32, i32, i32, f32, C.c_double, vp, sz, vp]),
    "rf_kitti_region_step_workspace": (sz, [i32, i32]),
    "rf_kitti_region_step": (i32, [vp, vp, vp, vp, i32, i32, vp, vp, i32, i32, vp, vp, sz, vp]),
    "rf_yfcc_matches_workspace": (sz, [i32, i32]),
    "rf_yfcc_matches": (i32, [vp, vp, i32, i32, i32, i32, i32, i32, i32, vp, vp, vp, vp, vp, vp, sz, vp]),
    "rf_essential_ransac_workspace": (sz, [i32]),
    "rf_essential_ransac": (i32, [vp, vp, i32, vp, C.c_double, vp, vp, vp, sz, vp]),
    "rf_recover_pose_workspace": (sz, [i32]),
    "rf_recover_pose": (i32, [vp, vp, i32, vp, vp, vp, vp, sz, vp]),
    "rf_essential_samples": (i32, [vp, vp, vp]),
    "rf_essential_five_point": (i32, [vp, vp, vp, i32, vp, vp, vp]),
    "rf_essential_score": (i32, [vp, vp, i32, vp, i32, C.c_double, vp, vp, vp]),
    "rf_fundamental_8point_workspace": (sz, [i32]),
    "rf_fundamental_8point": (i32, [vp, vp, i32, vp, vp, vp, vp, sz, vp]),
    "rf_fundamental_moments": (i32, [vp, vp, i32, vp, vp, vp, sz, vp]),
}


def _load():
    import importlib.util
    spec = importlib.util.spec_from_file_location("_rf_build", os.path.join(_HERE, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    if not b.is_current():
        # missing, or built from other sources than the ones next to it (a stale git-ignored .so after a pull would be called
        # through newer ctypes signatures): rebuild in-tree if a compiler is present; never fall back to anything else
        try:
            b.build(verbose=False)
        except Exception as e:  # noqa: BLE001
            raise RuntimeError("ransac_flow_b200: CUDA library %s is %s and could not be built (%s). "
                               "There is no CPU fallback; run `python ransac-flow_b200/build.py`."
                               % (LIB_PATH, "stale" if os.path.exists(LIB_PATH) else "missing", e))
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError = header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


class RFError(RuntimeError):
    pass


def check(rc):
    if rc != 0:
        raise RFError(lib.rf_last_error_string().decode())


def need_cuda(*tensors):
    for t in tensors:
        if t is None:
            continue
        if not (isinstance(t, torch.Tensor) and t.is_cuda):
            raise RFError("ransac_flow_b200 runs on CUDA tensors only (got %s); there is no CPU path"
                          % (type(t).__name__ if not isinstance(t, torch.Tensor) else t.device))


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def launch_count():
    return int(lib.rf_launch_count())
