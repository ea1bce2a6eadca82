"""ctypes binding of libpnx.so (C-ABI declared in include/pnx.h).

The library is the product; there is NO fallback: if it is missing (and cannot be built) or an entry
point fails, a RuntimeError is raised.
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libpnx.so")
_lib = None

P = ctypes.c_void_p
I = ctypes.c_int
L = ctypes.c_longlong
F = ctypes.c_float

# name -> argtypes (restype is int unless listed in _RESTYPE)
_SIGS = {
    "pnx_last_error": [],
    "pnx_abi_version": [],
    "pnx_sm_count": [],
    "pnx_scan_u32": [P, I, I, P, P, P, P],
    "pnx_voxelize_bitmap_words": [I, I, I],
    "pnx_scan_blocks": [P, I, P, P, P],
    "pnx_blockcnt_size": [I],
    "pnx_voxelize": [P, I, I, F, F, F, F, I, I, P, P, P, P, P, P, P, I, P, P, P],
    "pnx_voxelize_frames": [P, I, I, F, F, F, F, I, I, P, P, P, P, P, P, P, I, P, P, P, P],
    "pnx_voxelize_frames_scratch": [I],
    "pnx_voxelize_frames_supported": [I, I, I],
    "pnx_bucketize": [P, I, I, P, P, P, P, P, P, P],
    "pnx_bn_finalize": [P, I, P, L, P, P, F, F, P, P, P, P, P, P, P],
    "pnx_bn_eval_affine": [I, P, P, P, P, F, P, P, P],
    "pnx_pfn_mean": [P, P, P, P, I, P, P],
    "pnx_pfn_lin0": [P, P, P, P, P, P, I, F, F, F, F, P, P, P, I, P],
    "pnx_pfn_max0": [P, P, P, I, P, P, P, P],
    "pnx_pfn_lin1": [P, P, P, P, P, I, P, P, P, P, P, I, P],
    "pnx_pfn_max1": [P, P, P, I, P, P, P, P, P],
    "pnx_pfn_backward": [P, P, P, P, P, P, I, I, F, F, F, F] + [P] * 23 + [I, P, P],
    "pnx_tap_gather_sum": [P, L, I, P, I, I, I, P, P],
    "pnx_tap_scatter": [P, I, I, I, P, L, I, I, L, P],
    "pnx_center_loss_task": [P, P, P, P, P, P, P, P, I, I, I, I, I, I, I, I, I, I, I, I, F, F, F, F, F, P, I, P, P],
    "pnx_center_loss_finalize": [P, I, P, P, P, P, P, P],
    "pnx_sites_out_dim": [I, I],
    "pnx_sites_dilate": [P, I, I, I, I, P, P, P, P],
    "pnx_sites_inblock": [P, I, P, P],
    "pnx_sites_coords": [P, P, P, I, I, I, P, I, P],
    "pnx_nbr_table": [P, P, I, P, P, P, I, I, I, I, I, P, P],
    "pnx_scatter_dense": [P, P, P, I, I, I, I, I, P, I, P],
    "pnx_igemm": [P, L, L, I, I, I, P, I, I, P, I, I, I, I, I, I, I, I, I, P, L, I, P, P, I, I, I, I, P, L, I, L, L, I, P, L, P, P, P, P, P, I, I, P],
    "pnx_conv3x3_win": [P, L, I, I, I, I, P, I, I, P, L, P, P, I, I, I, P, L, P, P, P, P, P, I, I, P],
    "pnx_wgrad": [P, L, I, P, L, L, I, I, I, I, P, I, I, I, I, I, I, I, I, I, P, P, I, P],
    "pnx_wgrad_splits": [I, I, I, I, I],
    "pnx_set_deterministic": [I],
    "pnx_bn_apply": [P, L, L, I, P, P, P, L, I, P, L, P],
    "pnx_bn_bwd_reduce": [P, L, P, L, P, L, L, I, P, P, I, P, P, P, P],
    "pnx_bn_bwd_apply": [P, L, P, L, P, L, L, I, P, P, P, P, ctypes.c_double, P, I, P, P, P, L, P, L, I, P],
    "pnx_add_rows": [P, L, P, L, L, I, P],
    "pnx_add_relu": [P, L, P, L, L, I, P, L, P],
    "pnx_relu_bwd": [P, L, P, L, L, I, P, L, I, P],
    # fp32-grade split-rows mode
    "pnx_split_set_pieces": [I],
    "pnx_split_get_pieces": [],
    "pnx_rows_split": [P, L, L, I, P, L, L, P],
    "pnx_rows_merge": [P, L, L, L, I, P, L, I, P],
    "pnx_bn_apply_split": [P, L, L, I, P, P, P, L, L, I, P, L, L, P],
    "pnx_bn_bwd_reduce_split_scratch": [I],
    "pnx_bn_bwd_reduce_split": [P, L, L, P, L, L, P, L, L, I, P, P, I, P, P, P, P, P],
    "pnx_bn_bwd_apply_split": [P, L, L, P, L, L, P, L, L, I, P, P, P, P, ctypes.c_double, I, P, P, P, L, L, P, L, L, P],
    "pnx_add_relu_split": [P, L, L, P, L, L, L, I, P, L, L, P],
    "pnx_relu_bwd_split": [P, L, P, L, L, L, I, P, L, L, P],
    "pnx_pack_weights": [P, I, L, P],
    "pnx_assign_labels": [P, P, I, I, P, P, I, I, ctypes.c_double, ctypes.c_double, ctypes.c_double, ctypes.c_double, I,
                          ctypes.c_double, I, I, I, I, I, P, P, P, P, P, P, P, P],
    # F1: decode + rotated NMS.  common prefix = out, ld, B, H, W, C, offs, osf, vs_x, vs_y, pc_x, pc_y, score_thr, range6, rect
    "pnx_det_keys": [P, L, I, I, I, I, P, F, F, F, F, F, F, P, P, P, P, P],
    "pnx_det_nms": [P, L, I, I, I, I, P, F, F, F, F, F, F, P, P, P, P, P, P, I, I, P, P, P, P],
    "pnx_det_gather": [P, L, I, I, I, I, P, F, F, F, F, F, F, P, P, P, P, P, P, I, I, P, P, P, P],
    "pnx_det_iou_bev_host": [P, P],
    "pnx_aligned_iou3d": [P, P, I, P, P],
    "pnx_aligned_iou3d_host": [P, P],
    "pnx_det_decode_host": [P, L, I, I, I, I, P, F, F, F, F, F, F, P, P, L, P, P, P],
    # double-flip test-time augmentation: point expansion + the F1 entry points on the 4B-frame head output
    "pnx_flip4_points": [P, I, P, P],
    "pnx_det_keys_flip4": [P, L, I, I, I, I, P, F, F, F, F, F, F, P, P, P, P, P],
    "pnx_det_nms_flip4": [P, L, I, I, I, I, P, F, F, F, F, F, F, P, P, P, P, P, P, I, I, P, P, P, P],
    "pnx_det_gather_flip4": [P, L, I, I, I, I, P, F, F, F, F, F, F, P, P, P, P, P, P, I, I, P, P, P, P],
    "pnx_det_decode_flip4_host": [P, L, I, I, I, I, P, F, F, F, F, F, F, P, P, L, P, P, P],
    # global training augmentation (rotation, scaling, translation, flip) of points and raw boxes
    "pnx_global_aug": [P, I, P, I, I, P, P, P, P],
    "pnx_global_aug_host": [P, I, P, I, I, P, P, P],
    # ground-truth database sampling: collision test, scene-point removal and paste
    "pnx_gt_sample_workspace": [I, I, I],
    "pnx_gt_sample": [P, I, P, P, P, I, I, P, P, P, I, P, P, I, P, P, P, P, P, P, P],
    "pnx_gt_sample_host": [P, I, P, P, P, I, I, P, P, P, I, P, P, I, P, P, P, P, P],
    "pnx_points_in_boxes_host": [P, I, I, P, P, I, P],
    "pnx_points_in_boxes": [P, I, I, P, P, I, P, P],
    # multi-sweep accumulation: past sweeps into the key frame, close-point removal, merge
    "pnx_accumulate_sweeps_workspace": [I, I],
    "pnx_accumulate_sweeps": [P, I, P, I, P, I, P, I, P, F, P, P, P, P],
    "pnx_accumulate_sweeps_host": [P, I, P, I, P, I, P, I, P, F, P, P],
    # Waymo-style evaluation: point counts per ground-truth box and the greedy score-ordered match
    "pnx_eval_count_points": [P, L, I, P, P, P, I, I, P, P],
    "pnx_eval_count_points_host": [P, L, I, P, P, P, I, I, P],
    "pnx_eval_match": [P, P, L, P, P, P, P, P, P, I, I, I, P, P, P, P, P],
    "pnx_eval_match_host": [P, P, L, P, P, P, P, P, P, I, I, I, P, P, P, P],
    # the Hungarian mode: feasible pairs, their connected components, the exact assignment per breakdown and cutoff
    "pnx_eval_pairs": [P, P, L, P, P, P, P, P, P, I, I, I, P, P, P, P, P, P, P, P],
    "pnx_eval_pairs_host": [P, P, L, P, P, P, P, P, P, I, I, I, P, P, P, P, P, P, P],
    "pnx_eval_components": [P, P, I, I, I, L, P, P, P, P, P, P, P],
    "pnx_eval_components_host": [P, P, I, I, I, L, P, P, P, P, P, P],
    "pnx_eval_assign_workspace": [L],
    "pnx_eval_assign_warp_pairs": [],
    "pnx_eval_assign": [L, P, P, P, P, P, P, P, P, I, P, P, I, L, L, P, P, P, I, I, P, P, P, P],
    "pnx_eval_assign_host": [L, P, P, P, P, P, P, P, P, I, P, P, I, L, L, P, P, P, I, I, P, P],
    # tracking: the greedy velocity tracker and the CLEAR-MOT frame matching of evaluate_waymo_tracking
    "pnx_track_max_tracks": [],
    "pnx_track_greedy": [P, P, L, P, P, P, P, P, P, I, I, I, P, I, F, I, P, P, P, P, P, P, P],
    "pnx_track_greedy_host": [P, P, L, P, P, P, P, P, P, I, I, I, P, I, F, P, P],
    "pnx_eval_mot_workspace": [I, I, I],
    "pnx_eval_mot": [P, P, L, P, P, P, P, P, P, L, P, P, P, P, P, I, I, I, I, I, I, I, P, P, P, P, P],
    "pnx_eval_mot_host": [P, P, L, P, P, P, P, P, P, L, P, P, P, P, P, I, I, I, I, I, I, I, P, P, P],
    # nuScenes detection score: the centre-distance match, per threshold
    "pnx_eval_match_center": [P, L, P, P, P, P, P, I, I, I, P, I, P, P],
    "pnx_eval_match_center_host": [P, L, P, P, P, P, P, I, I, I, P, I, P],
    # nuScenes tracking: centre-distance pairs and the frame matching of evaluate_nuscenes_tracking
    "pnx_eval_pairs_center": [P, L, P, P, P, P, P, I, I, I, ctypes.c_double, P, P, P, P, P, P],
    "pnx_eval_pairs_center_host": [P, L, P, P, P, P, P, I, I, I, ctypes.c_double, P, P, P, P, P],
    "pnx_eval_mot_center": [P, P, L, P, P, P, P, P, P, L, P, P, P, P, P, I, I, I, I, I, I, I, P, P, P, P, P, P, P],
    "pnx_eval_mot_center_host": [P, P, L, P, P, P, P, P, P, L, P, P, P, P, P, I, I, I, I, I, I, I, P, P, P, P, P],
}
_RESTYPE = {"pnx_last_error": ctypes.c_char_p, "pnx_voxelize_bitmap_words": ctypes.c_size_t,
            "pnx_bn_bwd_reduce_split_scratch": ctypes.c_longlong, "pnx_gt_sample_workspace": ctypes.c_longlong,
            "pnx_accumulate_sweeps_workspace": ctypes.c_longlong, "pnx_eval_assign_workspace": ctypes.c_longlong,
            "pnx_eval_mot_workspace": ctypes.c_longlong,
            "pnx_det_iou_bev_host": ctypes.c_float, "pnx_aligned_iou3d_host": ctypes.c_float}


def exported_symbols():
    """Every symbol include/pnx.h declares (used by the CPU-side load test)."""
    return sorted(_SIGS)


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_SO):
        from . import build as _build  # compiles with nvcc; raises if impossible
        _build.build()
    if not os.path.exists(_SO):
        raise RuntimeError("pillarnext_b200: libpnx.so is missing and could not be built -- no fallback path exists")
    l = ctypes.CDLL(_SO)
    for name, argtypes in _SIGS.items():
        fn = getattr(l, name)  # AttributeError if the .so does not export what the header declares
        fn.argtypes = argtypes
        fn.restype = _RESTYPE.get(name, ctypes.c_int)
    _lib = l
    return l


def check(rc):
    if rc != 0:
        raise RuntimeError("libpnx error %d: %s" % (rc, lib().pnx_last_error().decode()))


def ptr(t):
    if t is None:
        return None
    assert t.is_cuda, "libpnx kernels take device pointers"
    return t.data_ptr()


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def stream():
    """cudaStream_t of torch's current stream (every libpnx launch goes there)."""
    if _raw_stream is not None:
        return _raw_stream(torch.cuda.current_device())
    return torch.cuda.current_stream().cuda_stream


_sm = None


def sm_count():
    global _sm
    if _sm is None:
        _sm = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return _sm
