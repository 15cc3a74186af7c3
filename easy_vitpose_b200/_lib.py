"""ctypes binding of libvitpose_b200.so (C ABI declared in include/vitpose_b200.h).

The library is the product; this module only declares argument types and turns non-zero return codes
into RuntimeError.  A missing library is a hard error: there is no Python / CPU fallback path.
"""
from __future__ import annotations

import ctypes as C
import os

from .build import LIB, build, is_stale

_lib = None


class VpbConfig(C.Structure):
    _fields_ = [("embed_dim", C.c_int32), ("depth", C.c_int32), ("num_heads", C.c_int32),
                ("num_keypoints", C.c_int32), ("max_batch", C.c_int32), ("device", C.c_int32)]


MAX_FRAMES = 64                                       # VPB_MAX_FRAMES: frames with boxes per multi-frame call


class VpbFrame(C.Structure):
    """vpb_frame: one frame of a multi-frame call (vpb_infer_frames and its host forms)."""
    _fields_ = [("data", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32), ("pitch_bytes", C.c_int64),
                ("num_boxes", C.c_int32), ("rotation", C.c_int32)]


ROTATIONS = (0, 90, 180, 270)                         # vpb_frame*.rotation: degrees counter-clockwise, stored frame -> view
YUV_MATRICES = {"bt601": 0, "bt709": 1}              # VPB_YUV_BT601, VPB_YUV_BT709


class VpbFrameNv12(C.Structure):
    """vpb_frame_nv12: one NV12 frame (Y plane + interleaved half-resolution UV plane) of the _nv12 calls."""
    _fields_ = [("y", C.c_void_p), ("y_pitch", C.c_int64), ("uv", C.c_void_p), ("uv_pitch", C.c_int64),
                ("height", C.c_int32), ("width", C.c_int32), ("num_boxes", C.c_int32), ("rotation", C.c_int32)]


YUV_LAYOUTS = {"nv12": 0, "nv21": 1, "i420": 2, "yv12": 3, "yuyv": 4, "uyvy": 5}    # VPB_YUV_NV12 .. VPB_YUV_UYVY
YUV_RANGES = {"limited": 0, "full": 1}               # VPB_YUV_LIMITED, VPB_YUV_FULL


class VpbFrameYuv(C.Structure):
    """vpb_frame_yuv: one YUV frame of the _yuv calls, its planes in the layout's storage order."""
    _fields_ = [("plane", C.c_void_p * 3), ("y_pitch", C.c_int64), ("c_pitch", C.c_int64),
                ("height", C.c_int32), ("width", C.c_int32), ("num_boxes", C.c_int32), ("rotation", C.c_int32)]


MAX_HEADS = 8                                        # VPB_MAX_HEADS: keypoint heads of one engine
MAX_SEGMENTS = 64                                     # VPB_MAX_SEGMENTS: runs of one head per multi-head call
DECODERS = {"classic": 0, "simple": 1}                # VPB_DECODER_CLASSIC, VPB_DECODER_SIMPLE (vpb_create_ex)


class VpbSegment(C.Structure):
    """vpb_segment: `count` consecutive crops of head `head` (vpb_infer_heads)."""
    _fields_ = [("head", C.c_int32), ("count", C.c_int32)]


class VpbOksNmsParams(C.Structure):
    """vpb_oks_nms_params: thr, vis_thr (NaN = None), rescore_vis_thr (NaN = off), soft, max_dets."""
    _fields_ = [("thr", C.c_double), ("vis_thr", C.c_double), ("rescore_vis_thr", C.c_double), ("soft", C.c_int32),
                ("max_dets", C.c_int32)]


class VpbCocoGts(C.Structure):
    """vpb_coco_gts: the ground truths of vpb_coco_eval, CSR by image (device pointers)."""
    _fields_ = [("offsets", C.c_void_p), ("kpts", C.c_void_p), ("area", C.c_void_p), ("bbox", C.c_void_p), ("iscrowd", C.c_void_p),
                ("num_keypoints", C.c_void_p), ("num_images", C.c_int32), ("num_gts", C.c_int32)]


class VpbCocoDets(C.Structure):
    """vpb_coco_dets: the detection frames of vpb_coco_eval (device pointers; keep / keep_counts may be NULL)."""
    _fields_ = [("kpts", C.c_void_p), ("scores", C.c_void_p), ("counts", C.c_void_p), ("frame_image", C.c_void_p), ("keep", C.c_void_p),
                ("keep_counts", C.c_void_p), ("n_rows", C.c_int32), ("num_frames", C.c_int32)]


DRAW_CHANNEL_ORDERS = {"rgb": 0, "bgr": 1}          # VPB_DRAW_RGB, VPB_DRAW_BGR


class VpbCanvas(C.Structure):
    """vpb_canvas: one frame drawn in place by vpb_draw_poses."""
    _fields_ = [("data", C.c_void_p), ("height", C.c_int32), ("width", C.c_int32), ("pitch_bytes", C.c_int64),
                ("num_people", C.c_int32)]


EXPORTS = {
    # name: (restype, argtypes)
    "vpb_last_error": (C.c_char_p, []),
    "vpb_create": (C.c_int, [C.POINTER(VpbConfig), C.POINTER(C.c_void_p)]),
    "vpb_destroy": (None, [C.c_void_p]),
    "vpb_load_tensor": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]),
    "vpb_finalize": (C.c_int, [C.c_void_p]),
    "vpb_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "vpb_forward_features": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "vpb_decode": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vpb_head": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "vpb_flip_back": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "vpb_decode_modes": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_decode_modes_ex": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p]),
    "vpb_infer": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_submit_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32]),
    "vpb_wait_host": (C.c_int, [C.c_void_p, C.c_int32]),
    "vpb_preprocess": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int64, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                 C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_decode_frame": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "vpb_infer_frame": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_frame_status": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "vpb_infer_frame_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_submit_frame_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32]),
    "vpb_infer_frames": (C.c_int, [C.c_void_p, C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_frames_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_submit_frames_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32]),
    "vpb_preprocess_affine": (C.c_int, [C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_affine": (C.c_int, [C.c_void_p, C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
    "vpb_infer_affine_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "vpb_create_heads": (C.c_int, [C.POINTER(VpbConfig), C.c_int32, C.c_void_p, C.c_int32, C.POINTER(C.c_void_p)]),
    "vpb_create_ex": (C.c_int, [C.POINTER(VpbConfig), C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p)]),
    "vpb_infer_heads": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(VpbSegment), C.c_int32, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p]),
    "vpb_infer_frames_heads": (C.c_int, [C.c_void_p, C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p]),
    "vpb_infer_frames_heads_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p]),
    "vpb_infer_affine_heads": (C.c_int, [C.c_void_p, C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                         C.c_void_p, C.c_void_p]),
    "vpb_infer_affine_heads_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrame), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_frames_yuv": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameYuv), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_frames_yuv_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameYuv), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_submit_frames_yuv_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameYuv), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_int32]),
    "vpb_infer_affine_yuv": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameYuv), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                       C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_affine_yuv_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameYuv), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                            C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_frames_heads_yuv": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameYuv), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_frames_heads_yuv_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameYuv), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_affine_heads_yuv": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameYuv), C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_infer_affine_heads_yuv_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameYuv), C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                                  C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_host_alloc": (C.c_void_p, [C.c_int64]),
    "vpb_host_free": (None, [C.c_void_p]),
    "vpb_kernel_launches": (C.c_int, [C.c_void_p, C.c_int32]),
    "vpb_cached_graphs": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "vpb_device_bytes": (C.c_int64, [C.c_void_p]),
    "vpb_set_option": (C.c_int, [C.c_void_p, C.c_char_p, C.c_int32]),
    "vpb_set_flip_test": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]),
    "vpb_set_flip_test_heads": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32]),
    "vpb_profile_classes": (C.c_int, []),
    "vpb_profile_class_name": (C.c_char_p, [C.c_int32]),
    "vpb_profile_collect": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_read_buffer": (C.c_int, [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64]),
    "vpb_gemm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                           C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "vpb_debug_gemm": (C.c_int, [C.c_int32, C.c_void_p]),
    "vpb_expert_gemm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                  C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "vpb_attention": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vpb_qkv_attention": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "vpb_debug_attention": (C.c_int, [C.c_int32]),
    "vpb_layernorm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_void_p]),
    "vpb_draw_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32]),
    "vpb_draw_poses": (C.c_int, [C.POINTER(VpbCanvas), C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32,
                                 C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_float, C.c_void_p, C.c_void_p]),
    "vpb_tracker_create": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32, C.POINTER(C.c_void_p)]),
    "vpb_tracker_destroy": (None, [C.c_void_p]),
    "vpb_tracker_update": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_tracker_reset": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "vpb_tracker_next_id": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64)]),
    "vpb_tracker_set_next_id": (C.c_int, [C.c_void_p, C.c_int64]),
    "vpb_tracker_status": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "vpb_smoother_create": (C.c_int, [C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, C.c_int32,
                                      C.c_int32, C.POINTER(C.c_void_p)]),
    "vpb_smoother_destroy": (None, [C.c_void_p]),
    "vpb_smoother_update": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_smoother_reset": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p]),
    "vpb_smoother_status": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32)]),
    "vpb_oks_nms": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                              C.POINTER(VpbOksNmsParams), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_oks_iou": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_double,
                              C.c_void_p, C.c_void_p, C.c_void_p]),
    "vpb_coco_eval_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "vpb_coco_eval": (C.c_int, [C.c_int32, C.c_void_p, C.POINTER(VpbCocoGts), C.POINTER(VpbCocoDets), C.c_void_p, C.c_int64, C.c_void_p,
                                C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
}

# The NV12 calls: names with a digit, kept apart from EXPORTS, which tests/test_abi.py matches against the header's
# [a-z_] names; tests/test_nv12_oracle.py checks this table against the header's *_nv12* declarations.
EXPORTS_NV12 = {
    "vpb_infer_frames_nv12": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameNv12), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p]),
    "vpb_infer_frames_nv12_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameNv12), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p]),
    "vpb_submit_frames_nv12_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameNv12), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_int32]),
    "vpb_infer_affine_nv12": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameNv12), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                        C.c_void_p, C.c_void_p]),
    "vpb_infer_affine_nv12_host": (C.c_int, [C.c_void_p, C.POINTER(VpbFrameNv12), C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.c_void_p]),
}


def lib():
    """Loads the shared library once.  Raises if it has not been built (python -m easy_vitpose_b200.build)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB) or is_stale():
            try:
                build()                              # nvcc cross-compiles sm_90a anywhere
            except Exception as exc:
                # never load a library older than its sources: its ABI / kernels may no longer match the header and
                # the argtypes below.  VPB_ALLOW_STALE=1 is the explicit escape hatch (e.g. a box without nvcc).
                if not os.path.exists(LIB) or os.environ.get("VPB_ALLOW_STALE", "0") != "1":
                    raise RuntimeError(f"{LIB} is missing or older than its sources and could not be rebuilt ({exc}); build it "
                                       "with `python -m easy_vitpose_b200.build`; there is no fallback implementation") from exc
                import warnings
                warnings.warn(f"loading a STALE {LIB} (VPB_ALLOW_STALE=1): {exc}")
        handle = C.CDLL(LIB)
        for name, (res, args) in {**EXPORTS, **EXPORTS_NV12}.items():
            fn = getattr(handle, name)          # AttributeError here = header and library disagree
            fn.restype = res
            fn.argtypes = args
        _lib = handle
    return _lib


def check(code: int) -> None:
    if code != 0:
        raise RuntimeError(f"vitpose_b200 error {code}: {lib().vpb_last_error().decode()}")


def check_value(code: int) -> None:
    """Like check(), but a bad ARGUMENT (code 1: e.g. a box that is empty after clipping, where the reference raises from
    pad_image / cv2.resize) surfaces as ValueError."""
    if code == 1:
        raise ValueError(lib().vpb_last_error().decode())
    check(code)
