/* vitpose_b200.h -- C ABI of the H100-native ViTPose crop engine (libvitpose_b200.so).
 *
 * One data-parallel hot path of JunkyByte/easy_ViTPose, rebuilt for sm_90a:
 *     crops f32 [B,3,256,192] -> ViT backbone -> TopdownHeatmapSimpleHead -> heatmaps f32 [B,K,64,48]
 *     -> argmax + DARK/UDP refine -> keypoints f32 [B,K,3] rows (y, x, score)
 * Plain pointers and sizes only; no torch types.  Device pointers are CUDA device addresses on the
 * engine's device, `stream` is a cudaStream_t passed as void* (NULL = default stream).  All calls are
 * asynchronous on `stream` unless stated; none of them frees or keeps caller memory.
 * There is no CPU fallback: every entry point fails (non-zero + vpb_last_error()) without an sm_90 (H100) GPU.
 *
 * Concurrency contract.  An engine owns ONE activation workspace, two host-staging slots and its CUDA graphs:
 *   - calls on one engine must come from one host thread at a time (the handle holds no lock);
 *   - calls on the same engine from DIFFERENT streams are safe and are executed one after the other: every entry point
 *     waits (on the device, cudaStreamWaitEvent) for the engine's previous enqueue when the stream changes -- there is no
 *     overlap between two calls of one engine; use one engine per stream (or per GPU) for concurrency;
 *   - the synchronous host calls (vpb_infer_host, vpb_infer_frame_host) use staging slot 0, the same buffers as
 *     vpb_submit_host / vpb_submit_frame_host with slot 0; they are ordered after that slot's last submit and the next
 *     submit(0) is ordered after them;
 *   - if `stream` is being captured by the caller, the engine launches its kernels eagerly into that capture (no nested
 *     graph) and leaves its cross-stream ordering to the caller;
 *   - several engines may share one GPU.  Calls that launch the chained persistent GEMM kernels (option "chain" on, batch >= the
 *     "chain_min_batch" option) are serialised per device across engines and streams (a device-side event wait plus a host mutex
 *     around the enqueue): such a kernel needs all of its CTAs resident at once and must not share the SMs
 *     with a second one.  Another PROCESS running chained launches on the same GPU (MPS) is outside that gate: give chained
 *     engines the GPU to themselves or set option "chain" = 0;
 *   - engines on different devices may live in one process: each entry point makes its engine's device current for the
 *     duration of the call and restores the caller's; `stream` must belong to the engine's device.
 *
 * Each entry point names the reference interface it replaces (paths relative to the reference repo).
 */
#ifndef VITPOSE_B200_H
#define VITPOSE_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VPB_OK 0
#define VPB_ERR_ARG 1      /* bad argument / unsupported configuration / missing weights */
#define VPB_ERR_CUDA 2     /* CUDA runtime or driver error (message in vpb_last_error) */
#define VPB_ERR_STATE 3    /* call order violated (e.g. forward before finalize) */

typedef struct vpb_engine vpb_engine;

/* Model hyper-parameters: easy_ViTPose/configs/ViTPose_common.py:65-195 (embed_dim, depth, num_heads;
 * mlp_ratio 4, qkv_bias, patch 16, img 256x192, 2 deconv layers of 256 filters, 1x1 final conv are fixed
 * on this path) and the per-dataset out_channels (e.g. configs/ViTPose_coco.py:16-18). */
typedef struct vpb_config {
  int32_t embed_dim;      /* 384 / 768 / 1024 / 1280 */
  int32_t depth;          /* 12 / 12 / 24 / 32 */
  int32_t num_heads;      /* 12 / 12 / 16 / 16 */
  int32_t num_keypoints;  /* K = keypoint_head.out_channels, 1..144 */
  int32_t max_batch;      /* workspace is sized for this many crops per call */
  int32_t device;         /* CUDA device ordinal */
} vpb_config;

/* Thread-local description of the last failure in this thread ("" if none). */
const char* vpb_last_error(void);

/* Replaces ViTPose(cfg) construction (easy_ViTPose/vit_models/model.py:10-18; VitInference.__init__,
 * easy_ViTPose/inference.py:156-157): allocates weights arena + workspace on cfg->device. */
int vpb_create(const vpb_config* cfg, vpb_engine** out);
void vpb_destroy(vpb_engine* e);

/* Replaces nn.Module.load_state_dict (easy_ViTPose/inference.py:162-166), one tensor at a time, under the
 * reference's own key names ("backbone.blocks.3.attn.qkv.weight", ...; SURVEY.md section 8b).  `data` is HOST
 * float32, C-contiguous, `numel` elements; "...num_batches_tracked" keys are accepted and ignored. */
int vpb_load_tensor(vpb_engine* e, const char* key, const float* data, int64_t numel);
/* Strict check (every key of the contract loaded exactly once) + one-time packing on the GPU: bf16
 * conversion, q-scale fold into attn.qkv, pos_embed+conv-bias fold, BatchNorm fold into the deconv phases. */
int vpb_finalize(vpb_engine* e);

/* Replaces ViTPose.forward (vit_models/model.py:23-24): d_crops f32 [batch,3,256,192] ->
 * d_heatmaps f32 [batch,K,64,48]. */
int vpb_forward(vpb_engine* e, const float* d_crops, int32_t batch, float* d_heatmaps, void* stream);
/* Replaces ViTPose.forward_features (vit_models/model.py:20-21): -> d_features f32 [batch,D,16,12]. */
int vpb_forward_features(vpb_engine* e, const float* d_crops, int32_t batch, float* d_features, void* stream);

/* Replaces keypoints_from_heatmaps(unbiased=True, use_udp=True) + the (y,x,score) packing of
 * VitInference.postprocess (vit_utils/top_down_eval.py:493-641 branch :586-589; easy_ViTPose/inference.py:187-205).
 * d_heatmaps f32 [n,k,64,48]; d_org_wh i32 [n,2] crop (width,height); d_kpts f32 [n,k,3]; d_idx i32 [n,k] flat
 * argmax or NULL.  wrap_batch selects the reference's "previous map" for max<=0 maps: 0 = one reference call per
 * crop (VitInference), 1 = one reference call on the whole [n,k,H,W] array.  Does not modify d_heatmaps. */
int vpb_decode(const float* d_heatmaps, int32_t n, int32_t k, const int32_t* d_org_wh, float* d_kpts, int32_t* d_idx,
               int32_t wrap_batch, void* stream);

/* Replaces TopdownHeatmapSimpleHead.forward (vit_models/head/topdown_heatmap_simple_head.py:188-193) on its own:
 * d_features f32 [batch,D,16,12] (what vpb_forward_features returns) -> d_heatmaps f32 [batch,K,64,48]. */
int vpb_head(vpb_engine* e, const float* d_features, int32_t batch, float* d_heatmaps, void* stream);
/* Replaces flip_back (vit_utils/post_processing/post_transforms.py:110-147, GaussianHeatmap) plus the optional one-pixel
 * shift of TopdownHeatmapSimpleHead.inference_model (:210-212): d_in / d_out f32 [n,k,64,48] (distinct buffers), d_perm i32 [k]
 * = the keypoint permutation the flip pairs induce (perm[left] = right, perm[right] = left, identity elsewhere). */
int vpb_flip_back(const float* d_in, int32_t n, int32_t k, const int32_t* d_perm, int32_t shift, float* d_out, void* stream);

/* The other modes of keypoints_from_heatmaps (vit_utils/top_down_eval.py:493-641; SURVEY.md section 8 row f4), with the
 * general transform_preds (post_processing/post_transforms.py:150-194).  mode: 0 post_process=None (:598), 1 'default' (+-0.25 px,
 * :617-631), 2 'unbiased' (Gaussian modulation + log + _taylor, :600-607), 3 'megvii' (:573-574,:629-639) -- all use_udp=False --
 * and 4 = use_udp=True DARK (:576-579) with arbitrary centre / scale.  Exactly one of d_cs32 (f32 [n,4]) / d_cs64 (f64 [n,4]) holds
 * (centre_x, centre_y, scale_x, scale_y) per crop: float32 arrays keep numpy's arithmetic in float32, int64 / float64 arrays
 * promote it to float64.  Output layout as vpb_decode: d_kpts f32 [n,k,3] (y, x, score), d_idx i32 [n,k] or NULL.
 * vpb_decode_modes is the kernel = 11 form (every reference config: modulate_kernel=11).  vpb_decode_modes_ex adds
 *   kernel        the `kernel` argument (:499): odd, 1..35 (17 for sigma = 3; 1 only for modes 4-5); used by modes 2-5;
 *   mode 5        use_udp=True with target_type='CombinedTarget' (:580-593): d_heatmaps is f32 [n,3k,64,48], triples of
 *                 (response, offset x, offset y); 2*kernel+1 <= 35; valid_radius = (float)(valid_radius_factor * 64) (:586);
 *                 the (-1,-1) sentinel reads its offsets one row and one pixel before the keypoint's plane, wrapping to the
 *                 last plane of the call for the first keypoint, as numpy's flat index does.  (The reference's own index
 *                 arithmetic (:589) only broadcasts for n = 1; n > 1 here is that formula with the intended shape.)
 * Mode 4 with k = 1 and n > 1: the reference raises (post_dark_udp's `.squeeze()`, :414, drops the k axis of its [n,1,2]
 * offsets); here, as in vpb_decode with wrap_batch = 1 and in the affine calls (a segment of a one-keypoint head), it is the
 * formula with the intended shape: each crop's DARK offset applied to its own keypoint, the max <= 0 sentinel reading the
 * previous crop's map as for any k.  The Python keypoints_from_heatmaps raises ValueError there, as the reference does. */
#define VPB_DECODE_NONE 0
#define VPB_DECODE_DEFAULT 1
#define VPB_DECODE_UNBIASED 2
#define VPB_DECODE_MEGVII 3
#define VPB_DECODE_DARK_UDP 4
#define VPB_DECODE_COMBINED 5
int vpb_decode_modes(const float* d_heatmaps, int32_t n, int32_t k, int32_t mode, const float* d_cs32, const double* d_cs64,
                     float* d_kpts, int32_t* d_idx, void* stream);
int vpb_decode_modes_ex(const float* d_heatmaps, int32_t n, int32_t k, int32_t mode, int32_t kernel, float valid_radius,
                        const float* d_cs32, const double* d_cs64, float* d_kpts, int32_t* d_idx, void* stream);

/* Replaces the model + postprocess part of VitInference._inference_torch (easy_ViTPose/inference.py:320-328)
 * for a whole batch of crops resident on the device.  d_heatmaps may be NULL. */
int vpb_infer(vpb_engine* e, const float* d_crops, const int32_t* d_org_wh, int32_t batch, float* d_kpts,
              int32_t* d_idx, float* d_heatmaps, void* stream);
/* Same with HOST buffers: H2D of crops/org_wh, the path, D2H of keypoints (+idx), then a stream sync --
 * the reference's `.to(device)` ... `.cpu().numpy()` bracket (inference.py:324,327).  Pinned host memory
 * (vpb_host_alloc) makes the copies asynchronous DMA. */
int vpb_infer_host(vpb_engine* e, const float* h_crops, const int32_t* h_org_wh, int32_t batch, float* h_kpts,
                   int32_t* h_idx, void* stream);
/* Pipelined form: vpb_submit_host(slot 0|1) enqueues H2D (engine copy stream), the path and D2H (engine compute stream)
 * and returns; vpb_wait_host(slot) blocks until that slot's keypoints are in h_kpts.  Keeping two slots in flight hides
 * the H2D of batch i+1 under the compute of batch i.  Host buffers must stay valid until the wait (pinned: real overlap). */
int vpb_submit_host(vpb_engine* e, const float* h_crops, const int32_t* h_org_wh, int32_t batch, float* h_kpts,
                    int32_t* h_idx, int32_t slot);
int vpb_wait_host(vpb_engine* e, int32_t slot);
void* vpb_host_alloc(int64_t bytes);   /* cudaHostAlloc; NULL on failure */
void vpb_host_free(void* p);

/* ---- frame-level entry points (SURVEY.md section 8 rows f1, f2): the per-person loop of VitInference.inference
 * (easy_ViTPose/inference.py:258-272) as one batched call.
 *
 * vpb_preprocess replaces, for all n boxes of a frame at once: the +-pad_bbox box padding and clipping (:259-261), the
 * crop (:264), pad_image(crop, 3/4) (vit_utils/inference.py:41-70) and VitInference.pre_img (:314-318: cv2 uint8
 * INTER_LINEAR resize to 192x256, /255, (x-MEAN)/STD in float64, CHW float32).  Bit-exact with cv2 4.13.
 *   d_frame u8 [frame_h, frame_w, 3] RGB, row pitch pitch_bytes (0 = packed);  d_bboxes i32 [n,4] (x0,y0,x1,y1), already
 *   rounded as `res_pd[:, :4].round().astype(int)` (:253);  d_crops f32 [n,3,256,192];  d_org_wh i32 [n,2] padded canvas
 *   (w,h) = what pre_img returns as (org_w, org_h);  d_offs_yx i32 [n,2] = (y0 - top_pad, x0 - left_pad), the offset :270
 *   adds;  d_status i32 [1] or NULL: bit 0 is OR-ed in when a box is empty after clipping (the reference raises there;
 *   the kernel emits a black crop with org_wh = 0). */
int vpb_preprocess(const uint8_t* d_frame, int32_t frame_h, int32_t frame_w, int64_t pitch_bytes, const int32_t* d_bboxes,
                   int32_t n, int32_t pad_bbox, float* d_crops, int32_t* d_org_wh, int32_t* d_offs_yx, int32_t* d_status,
                   void* stream);
/* vpb_decode with the :270 offsets applied in the same kernel: keypoints come out in FRAME pixels. */
int vpb_decode_frame(const float* d_heatmaps, int32_t n, int32_t k, const int32_t* d_org_wh, const int32_t* d_offs_yx,
                     float* d_kpts, int32_t* d_idx, int32_t wrap_batch, void* stream);
/* frame + boxes on the device -> d_kpts f32 [n,K,3] (y, x, score) in frame pixels, d_idx i32 [n,K] or NULL; n <= max_batch.
 * pad_bbox is the reference's 10. */
int vpb_infer_frame(vpb_engine* e, const uint8_t* d_frame, int32_t frame_h, int32_t frame_w, const int32_t* d_bboxes,
                    int32_t n, float* d_kpts, int32_t* d_idx, void* stream);
/* Status of the device-side frame calls since the last query: bit 0 = some box was empty after padding and clipping
 * (the reference raises there: ZeroDivisionError in pad_image / cv2.resize, easy_ViTPose/inference.py:259-265; the
 * device path cannot raise without a sync and decodes such a box from a black crop); bit 1 = vpb_infer_affine got a
 * non-finite matrix entry or a scale <= 0.  Synchronises the device, clears the word. */
int vpb_frame_status(vpb_engine* e, int32_t* h_status);
/* Same with HOST buffers (H2D of the packed uint8 frame + 16 B per box, D2H of the keypoints, stream sync); empty boxes
 * return VPB_ERR_ARG where the reference raises.  The pipelined form shares its slots and vpb_wait_host with vpb_submit_host. */
int vpb_infer_frame_host(vpb_engine* e, const uint8_t* h_frame, int32_t frame_h, int32_t frame_w, const int32_t* h_bboxes,
                         int32_t n, float* h_kpts, int32_t* h_idx, void* stream);
int vpb_submit_frame_host(vpb_engine* e, const uint8_t* h_frame, int32_t frame_h, int32_t frame_w, const int32_t* h_bboxes,
                          int32_t n, float* h_kpts, int32_t* h_idx, int32_t slot);

/* ---- multi-frame entry points: the people of several frames (cameras, video frames, streams) as ONE engine call, so a
 * call of many small frames runs the batch size of their sum.  h_frames is always a HOST array of num_frames entries; the
 * boxes of all frames are concatenated in frame order (frame j owns the next h_frames[j].num_boxes rows), and the outputs
 * [n,K,3] / [n,K] come back in the same order, n = the sum of num_boxes, each keypoint in its own frame's pixels.  The
 * results are bit-identical to one vpb_infer_frame per frame (the forward is batch-invariant, the decode runs per crop).
 * Frames with 0 boxes are skipped and do not count towards VPB_MAX_FRAMES; n = 0 returns VPB_OK and launches nothing.
 * VPB_ERR_ARG: n above the batch limit (max_batch, max_batch / 2 with flip test on), more than VPB_MAX_FRAMES frames with
 * boxes, a negative num_boxes, a frame with boxes whose data is NULL, height or width < 1, or pitch below 3 * width.
 * Flip test (vpb_set_flip_test) applies as for the single-frame calls.
 *
 * Rotated frames (phone footage, portrait-mounted cameras; the reference's `--rotate`, VideoReader's cv2.rotate): every
 * frame struct (vpb_frame, vpb_frame_nv12, vpb_frame_yuv) ends with `rotation`, 0, 90, 180 or 270 degrees counter-clockwise.
 * height, width, the pitches and the planes describe the STORED frame (the decoder's output), and the frame the call sees, its
 * VIEW, is cv2.rotate(stored, code) with code ROTATE_90_COUNTERCLOCKWISE for 90, ROTATE_180 for 180 and ROTATE_90_CLOCKWISE
 * for 270 (the view is width x height for 90 and 270).  Boxes and affine matrices are given in view pixels, box padding,
 * clipping, pad_image, the empty-box status bit and the host forms' empty-box check use the view's size, and keypoints come
 * back in view pixels.  The rotation is folded into the gather's addressing, so a rotated call is bit-identical to the upright
 * call on the rotated copy; YUV taps read the stored pixel's luma and its stored chroma block, which equals converting the
 * stored frame and rotating the result.  Size rules (even sizes for 4:2:0, even width for 4:2:2) apply to the stored frame.
 * Any other value returns VPB_ERR_ARG naming the frame.  Zero-initialise the structs (aggregate initialisation and ctypes
 * do) so that callers written before the field existed keep rotation 0.  The single-frame calls (vpb_infer_frame*,
 * vpb_preprocess) take upright frames; a rotated single frame is a one-entry multi-frame call. */
#define VPB_MAX_FRAMES 64
typedef struct vpb_frame {
  const uint8_t* data;    /* u8 [height, width, 3] RGB, stored; device address (vpb_infer_frames) or host (the _host forms) */
  int32_t height, width;
  int64_t pitch_bytes;    /* row pitch; 0 = packed (3 * width) */
  int32_t num_boxes;      /* this frame's boxes are the next num_boxes rows of the box array (0 allowed) */
  int32_t rotation;       /* 0 | 90 | 180 | 270 degrees counter-clockwise, stored -> view (above) */
} vpb_frame;
/* Device frames and boxes (d_bboxes i32 [n,4], view pixels); boxes empty after clipping to their view set bit 0 of the status
 * word, as vpb_infer_frame does. */
int vpb_infer_frames(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* d_bboxes,
                     float* d_kpts, int32_t* d_idx, void* stream);
/* HOST frames (any pitch; each is staged packed, as stored) and boxes: every box is checked against its own frame's view and
 * an empty one returns VPB_ERR_ARG naming the frame and the box.  Same staging slots, events, concurrency contract and vpb_wait_host as
 * vpb_infer_frame_host / vpb_submit_frame_host; the slot's staging buffer grows to the sum of the frame sizes. */
int vpb_infer_frames_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_bboxes,
                          float* h_kpts, int32_t* h_idx, void* stream);
int vpb_submit_frames_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_bboxes,
                           float* h_kpts, int32_t* h_idx, int32_t slot);     /* completes with vpb_wait_host(slot) */

/* ---- affine top-down crops: the mmpose / HRNet data path of easy_ViTPose/datasets/COCO.py:288-302 (the crop the published
 * COCO AP numbers were measured with) for the people of up to VPB_MAX_FRAMES frames per call.  Frames and their boxes are given
 * as for vpb_infer_frames (vpb_frame.num_boxes = how many of the next matrices belong to that frame; vpb_frame.rotation as
 * there: the matrices map view pixels, and taps outside the view read 0).  Per box:
 *   mats f64 [n,6] = the 2x3 matrix handed to cv2.warpAffine (image -> 192x256 crop), e.g. the UDP matrix
 *   get_warp_matrix(rot, 2c, image_size - 1, s * 200) (vit_utils/post_processing/post_transforms.py:312-340) or the HRNet
 *   get_affine_transform (vit_utils/transform.py:46-75);
 *   cv2.warpAffine(frame, M, (192, 256), INTER_LINEAR) with the constant 0 border, then torchvision ToTensor + Normalize in
 *   float32 (COCO.py:120-123, 300-302): bit-exact with cv2 4.13 and torchvision, singular matrices included.
 * vpb_preprocess_affine (engine-free, like vpb_preprocess): d_crops f32 [n,3,256,192]. */
int vpb_preprocess_affine(const vpb_frame* h_frames, int32_t num_frames, const double* d_mats, float* d_crops, void* stream);
/* The fused gather (the crops are never stored), the engine's forward (cached CUDA graph per batch size) and
 * keypoints_from_heatmaps(heatmaps, c, s * 200, use_udp=True) = vpb_decode_modes mode 4 with d_cs f32 [n,4] (cx, cy, sx, sy) in
 * pixels, as keypoints_from_heatmaps takes them (top_down_eval.py:576-579, one reference call on the whole call's array).
 * d_kpts f32 [n,K,3] (y, x, score), d_idx i32 [n,K] or NULL.  The keypoints are in the coordinates transform_preds gives:
 * view pixels for an unrotated matrix.  The reference's decode has no rotation, and neither has this one: for a rotated
 * matrix they are the reference's values, not the rotated-back positions.  Bit-identical to vpb_preprocess_affine ->
 * vpb_forward -> vpb_decode_modes(mode 4); flip test (vpb_set_flip_test) applies as to the frame calls.
 * VPB_ERR_ARG: n above the batch limit, more than VPB_MAX_FRAMES frames with boxes, a negative num_boxes, a frame with boxes
 * whose data is NULL, height or width < 1 or pitch below 3 * width.  A non-finite matrix entry or a scale <= 0 cannot be
 * returned by the device form without a synchronisation: it sets bit 1 of the status word (vpb_frame_status) instead. */
int vpb_infer_affine(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const double* d_mats, const float* d_cs,
                     float* d_kpts, int32_t* d_idx, void* stream);
/* HOST frames, matrices and centre / scale, staged on slot 0 like vpb_infer_frames_host (synchronous).  A non-finite
 * matrix or centre entry or a scale <= 0 returns VPB_ERR_ARG naming the box. */
int vpb_infer_affine_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const double* h_mats, const float* h_cs,
                          float* h_kpts, int32_t* h_idx, void* stream);

/* ---- NV12 video frames (what NVDEC and ffmpeg's `-pix_fmt nv12` produce): the multi-frame and affine calls read decoder
 * output directly, converting only the pixels the gather taps.  Pixel (x, y) of an even-sized frame takes
 * Y = y[y * y_pitch + x] and the (U, V) pair uv[(y / 2) * uv_pitch + 2 * (x / 2)], uv[... + 1] (nearest chroma, as cv2), then
 * with yy = max(Y - 16, 0) * CY (SHIFT 20, half = 1 << 19):
 *   R = clamp((yy + half + CVR (V - 128)) >> 20), G = clamp((yy + half + CVG (V - 128) + CUG (U - 128)) >> 20),
 *   B = clamp((yy + half + CUB (U - 128)) >> 20) to 0..255;
 *   VPB_YUV_BT601: CY 1220542, CVR 1673527, CVG -852492, CUG -409993, CUB 2116026 = cv2 COLOR_YUV2RGB_NV12, bit for bit;
 *   VPB_YUV_BT709: CY 1220542, CVR 1880097, CVG -558891, CUG -223347, CUB 2214593 (limited-range BT.709, 3-decimal form).
 * The converted taps then go through the RGB arithmetic unchanged, and taps outside the crop or frame read RGB 0, so every
 * call is bit-identical (patch rows, keypoints, argmax, flip test included) to its RGB counterpart on
 * cv2.cvtColor(frame, COLOR_YUV2RGB_NV12) (BT.601) or the formula above (BT.709).  Arguments, errors, status bits, limits,
 * staging slots and graph caches are those of the RGB counterparts, plus `matrix`; VPB_ERR_ARG also for an odd or < 2 height
 * or width, a pitch below width, a NULL plane in a frame with boxes, or an unknown matrix.  The host forms stage each frame
 * packed at 1.5 B per pixel (Y, then UV).  These calls are the NV12, limited-range case of the _yuv calls below, which also
 * take NV21, I420, YV12, YUYV and UYVY frames, full-range YUV, and serve the multi-head engines. */
#define VPB_YUV_BT601 0
#define VPB_YUV_BT709 1
typedef struct vpb_frame_nv12 {
  const uint8_t* y;       /* u8 [height, width] luma; device address or host (the _host forms) */
  int64_t y_pitch;        /* row pitch of y in bytes; 0 = packed (width) */
  const uint8_t* uv;      /* u8 [height / 2, width]: U, V interleaved, one pair per 2x2 block; may be a separate allocation */
  int64_t uv_pitch;       /* row pitch of uv in bytes; 0 = packed (width) */
  int32_t height, width;  /* both even; the stored frame */
  int32_t num_boxes;      /* as vpb_frame.num_boxes */
  int32_t rotation;       /* as vpb_frame.rotation */
} vpb_frame_nv12;
int vpb_infer_frames_nv12(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix,
                          const int32_t* d_bboxes, float* d_kpts, int32_t* d_idx, void* stream);
int vpb_infer_frames_nv12_host(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix,
                               const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, void* stream);
int vpb_submit_frames_nv12_host(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix,
                                const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, int32_t slot);   /* completes with vpb_wait_host(slot) */
int vpb_infer_affine_nv12(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix, const double* d_mats,
                          const float* d_cs, float* d_kpts, int32_t* d_idx, void* stream);
int vpb_infer_affine_nv12_host(vpb_engine* e, const vpb_frame_nv12* h_frames, int32_t num_frames, int32_t matrix, const double* h_mats,
                               const float* h_cs, float* h_kpts, int32_t* h_idx, void* stream);

/* ---- several keypoint heads (datasets) on one backbone: ViTPose+ (model_split.py) and frozen-backbone fine-tunes
 * (train.py --freeze-backbone).  vpb_create_heads makes an engine with num_heads heads of h_keypoints[j] keypoints each
 * (1 <= num_heads <= VPB_MAX_HEADS, 1..144 keypoints; cfg->num_keypoints is ignored) and an expert width P = expert_rows:
 *   P = 0              every head shares the whole backbone (frozen-backbone fine-tunes);
 *   0 < P < D, P % 32  each block's fc2 is a shared part [D-P, 4D] writing columns [0, D-P) plus, per head j, an expert
 *                      [P, 4D] writing columns [D-P, D) -- head j always uses expert j, the pairing model_split.py makes.
 * Any other P returns VPB_ERR_ARG.  The weights load under ViTPose+ key names, so an unsplit ViTPose+ state_dict loads as is:
 * backbone.blocks.{i}.mlp.fc2.{weight,bias} is the shared part, backbone.blocks.{i}.mlp.experts.{j}.{weight,bias} expert j,
 * keypoint_head.* head 0 and associate_keypoint_heads.{j-1}.* head j >= 1; loading is strict as for vpb_create.  Crops of head j
 * give bit-identical results to a single-head engine loaded with model_split.py's checkpoint j.  vpb_create is the
 * num_heads = 1, P = 0 engine.  On a multi-head engine the single-head calls (vpb_infer, vpb_forward, vpb_infer_frames, ...)
 * run every crop through head 0 and return K_0 keypoints per crop, with the single-head launches.  A multi-head call whose
 * crops all use head 0 issues the single-head backbone launches too (head 0's fc2 is the first D rows of the stacked weight);
 * any other call on an engine with P > 0, a single segment of head j != 0 included, runs each block's fc2 as two launches
 * (shared columns, then the grouped expert GEMM), and with option "ln_fused" the LayerNorm after fc2 as a launch of its own; vpb_set_flip_test returns VPB_ERR_STATE (the reference
 * defines flip pairs for COCO only), and the multi-head calls below return VPB_ERR_STATE while flip test set by vpb_set_flip_test is
 * on.  Flip test on a multi-head engine is set with vpb_set_flip_test_heads, which takes a permutation per head. */
#define VPB_MAX_HEADS 8
#define VPB_MAX_SEGMENTS 64
int vpb_create_heads(const vpb_config* cfg, int32_t num_heads, const int32_t* h_keypoints, int32_t expert_rows, vpb_engine** out);
/* A run of `count` consecutive crops of head `head`. */
typedef struct vpb_segment {
  int32_t head, count;
} vpb_segment;
/* Mixed batch: the n crops (n = the sum of the counts, <= max_batch) are the segments h_segs[0 .. num_segs-1] in order (HOST
 * array, num_segs <= VPB_MAX_SEGMENTS; counts of 0 are allowed).  d_crops f32 [n,3,256,192], d_org_wh i32 [n,2] as for vpb_infer;
 * d_kpts f32 [n,K_max,3], d_idx i32 [n,K_max] or NULL, d_heatmaps f32 [n,K_max,64,48] or NULL, K_max = the largest head's K:
 * crop c of head j fills rows / maps 0 .. K_j-1; rows and maps at or beyond K_j are not written.  One backbone pass for all
 * crops (the fc2 expert columns of every segment in one grouped launch), then each segment's head and decode.  Cached CUDA
 * graph per segment list (at most 16, least recently used out first; a list runs eagerly on its first use).
 * VPB_ERR_ARG: a head index out of range, a negative count, more than VPB_MAX_SEGMENTS segments, n above max_batch. */
int vpb_infer_heads(vpb_engine* e, const float* d_crops, const int32_t* d_org_wh, const vpb_segment* h_segs, int32_t num_segs,
                    float* d_kpts, int32_t* d_idx, float* d_heatmaps, void* stream);
/* vpb_infer_frames with a head per frame entry: h_heads i32 [num_frames] (HOST) is the head of every box of that entry (a
 * frame may appear once per head); the segments are the runs of equal head over the entries that have boxes.  Outputs as
 * vpb_infer_heads; the errors of vpb_infer_frames plus a head index out of range.  The _host form stages frames and boxes on
 * slot 0 as vpb_infer_frames_host does and is synchronous. */
int vpb_infer_frames_heads(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_heads, const int32_t* d_bboxes,
                           float* d_kpts, int32_t* d_idx, void* stream);
int vpb_infer_frames_heads_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_heads,
                                const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, void* stream);
/* vpb_infer_affine with a head per frame entry (h_heads as for vpb_infer_frames_heads): frames, matrices d_mats f64 [n,6] and
 * centre / scale d_cs f32 [n,4] as for vpb_infer_affine, in the order of the entries.  Outputs as vpb_infer_heads: d_kpts f32
 * [n,K_max,3], d_idx i32 [n,K_max] or NULL, rows at or beyond K_j not written.  Each segment is decoded as ONE reference call,
 * keypoints_from_heatmaps(c, s * 200, use_udp=True) on that segment's [count, K_j] array (the max <= 0 "previous map" included), so a
 * segment's keypoints equal vpb_infer_affine of a single-head engine on that segment's boxes.  Errors and status bit 1 as for
 * vpb_infer_affine, plus a head index out of range; graphs cached per (segment list, affine).  The _host form stages frames,
 * matrices and centre / scale on slot 0 as vpb_infer_affine_host does, is synchronous and rejects what that call rejects. */
int vpb_infer_affine_heads(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_heads, const double* d_mats,
                           const float* d_cs, float* d_kpts, int32_t* d_idx, void* stream);
int vpb_infer_affine_heads_host(vpb_engine* e, const vpb_frame* h_frames, int32_t num_frames, const int32_t* h_heads,
                                const double* h_mats, const float* h_cs, float* h_kpts, int32_t* h_idx, void* stream);

/* ---- YUV video frames in every 8-bit layout a decoder, camera or capture card delivers: the frame, affine and multi-head
 * calls read them directly and convert only the pixels the gather taps, with nearest chroma as cv2 does.  Each call takes
 * (layout, matrix, range), the same for all frames of the call.  Pixel (x, row) reads
 *   Y                    4:2:0 planar and semi-planar: plane[0][row * y_pitch + x];  4:2:2: the Y byte of pixel x of row `row`
 *   (U, V)               the pair of its chroma block: 2x2 pixels for 4:2:0, 2x1 for 4:2:2
 * and converts it with
 *   VPB_YUV_LIMITED:     the NV12 formula above (SHIFT 20, BT.601 = cv2 COLOR_YUV2RGB_*, BT.709 its 3-decimal form);
 *   VPB_YUV_FULL:        cv2's COLOR_YCrCb2RGB (JPEG range, SHIFT 14, D(s) = (s + 8192) >> 14):
 *                        R = clamp(Y + D(C0 (V - 128))), G = clamp(Y + D(C2 (U - 128) + C1 (V - 128))), B = clamp(Y + D(C3 (U - 128)));
 *                        BT.601 C0..C3 = 22987, -11698, -5636, 29049 (cv2 bit for bit); BT.709 25805, -7668, -3064, 30409.
 * The planes, in the order the layout stores them (unused entries are ignored and may be NULL):
 *   VPB_YUV_NV12  plane[0] Y [h, w], plane[1] UV [h/2, w] (U first)     VPB_YUV_I420  plane[0] Y, plane[1] U [h/2, w/2], plane[2] V
 *   VPB_YUV_NV21  plane[0] Y [h, w], plane[1] VU [h/2, w] (V first)     VPB_YUV_YV12  plane[0] Y, plane[1] V [h/2, w/2], plane[2] U
 *   VPB_YUV_YUYV  plane[0] [h, 2w]: Y0 U Y1 V per pixel pair             VPB_YUV_UYVY  plane[0] [h, 2w]: U Y0 V Y1 per pixel pair
 * y_pitch is plane[0]'s row pitch (0 = packed: w, or 2w for 4:2:2); c_pitch the chroma planes' (0 = packed: w for NV12 / NV21,
 * w/2 for I420 / YV12; unused for 4:2:2).  Every call is bit-identical to its RGB counterpart on the converted frame, as the
 * NV12 calls are, and shares its arguments, errors, status bits, limits, staging slots and graph caches.  VPB_ERR_ARG also for
 * an odd height or width in 4:2:0, an odd width in 4:2:2, a pitch below the row's bytes, a NULL plane the layout uses in a
 * frame with boxes, or an unknown layout, matrix or range.  The host forms stage each frame packed: 1.5 B per pixel for 4:2:0
 * (Y, then the chroma planes), 2 B per pixel for 4:2:2. */
#define VPB_YUV_NV12 0
#define VPB_YUV_NV21 1
#define VPB_YUV_I420 2
#define VPB_YUV_YV12 3
#define VPB_YUV_YUYV 4
#define VPB_YUV_UYVY 5
#define VPB_YUV_LIMITED 0
#define VPB_YUV_FULL 1
typedef struct vpb_frame_yuv {
  const uint8_t* plane[3];  /* in storage order (above); device addresses or host (the _host forms) */
  int64_t y_pitch;          /* row pitch of plane[0] in bytes; 0 = packed */
  int64_t c_pitch;          /* row pitch of the chroma plane(s) in bytes; 0 = packed */
  int32_t height, width;    /* the stored frame */
  int32_t num_boxes;        /* as vpb_frame.num_boxes */
  int32_t rotation;         /* as vpb_frame.rotation */
} vpb_frame_yuv;
int vpb_infer_frames_yuv(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                         int32_t range, const int32_t* d_bboxes, float* d_kpts, int32_t* d_idx, void* stream);
int vpb_infer_frames_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                              int32_t range, const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, void* stream);
int vpb_submit_frames_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                               int32_t range, const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx, int32_t slot);   /* vpb_wait_host(slot) */
int vpb_infer_affine_yuv(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                         int32_t range, const double* d_mats, const float* d_cs, float* d_kpts, int32_t* d_idx, void* stream);
int vpb_infer_affine_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                              int32_t range, const double* h_mats, const float* h_cs, float* h_kpts, int32_t* h_idx, void* stream);
/* the multi-head calls on YUV frames (NV12 included): h_heads, outputs and errors as vpb_infer_frames_heads / vpb_infer_affine_heads */
int vpb_infer_frames_heads_yuv(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                               int32_t range, const int32_t* h_heads, const int32_t* d_bboxes, float* d_kpts, int32_t* d_idx, void* stream);
int vpb_infer_frames_heads_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                                    int32_t range, const int32_t* h_heads, const int32_t* h_bboxes, float* h_kpts, int32_t* h_idx,
                                    void* stream);
int vpb_infer_affine_heads_yuv(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                               int32_t range, const int32_t* h_heads, const double* d_mats, const float* d_cs, float* d_kpts,
                               int32_t* d_idx, void* stream);
int vpb_infer_affine_heads_yuv_host(vpb_engine* e, const vpb_frame_yuv* h_frames, int32_t num_frames, int32_t layout, int32_t matrix,
                                    int32_t range, const int32_t* h_heads, const double* h_mats, const float* h_cs, float* h_kpts,
                                    int32_t* h_idx, void* stream);

/* ---- pose overlay: the pose layer of VitInference.draw() (easy_ViTPose/inference.py:283-312, vit_utils/visualization.py:360-481)
 * for the people of up to VPB_MAX_FRAMES frames in two launches, drawn in place, bit-exact with cv2 4.13.  Per person in order
 * (frame j owns the next h_frames[j].num_people rows of d_kpts, as vpb_infer_frames returns them), the reference's
 * draw_points_and_skeleton:
 *   every limb e (a, b) = h_limbs[2e], h_limbs[2e + 1] whose two scores are > threshold (float compare, as numpy does for
 *   float32 rows): cv2.line(img, (int(x_a), int(y_a)), (int(x_b), int(y_b)), limb colour [idx % num_limb_colors], 2), idx =
 *   d_person_index[p] or, when NULL, the person's position within its frame;
 *   then every keypoint i whose score is > threshold: cv2.circle(img, (int(x), int(y)), radius, point colour [i % num_point_colors], -1).
 * int() truncates toward zero; a coordinate that is not finite or not an int32 is not drawn (the reference raises there).  Later
 * primitives overwrite earlier ones; pixels no primitive covers are not written.  Colours are BGR triples, as the reference holds
 * them: channel_order VPB_DRAW_BGR writes them as given, VPB_DRAW_RGB reversed, which equals the reference's flip -> draw -> flip.
 * radius <= 0 = max(1, min(height, width) / 150) per frame, the reference's rule; at most 1023.
 * d_kpts f32 [n,k,3] (y, x, score) in frame pixels; d_person_index i32 [n] or NULL; h_limbs i32 [num_limbs,2] (HOST), num_limbs
 * <= 128, every index in [0, k); h_point_bgr / h_limb_bgr u8 [count,3] (HOST), 1..64 entries each.  d_workspace: device memory of
 * vpb_draw_workspace_bytes(n, k, num_limbs) bytes, 16-byte aligned, which the call may overwrite until it completes on `stream`.
 * No host synchronisation; the two launches can be captured in a CUDA graph.  Frames with 0 people are skipped and do not count
 * towards VPB_MAX_FRAMES; n = 0 returns VPB_OK and launches nothing.  VPB_ERR_ARG: an unknown channel order, k < 1, a limb index
 * outside [0, k), more than 128 limbs, a colour table of 0 or more than 64 entries, a radius above 1023, more than VPB_MAX_FRAMES
 * frames with people, a negative num_people, a frame with people whose data is NULL, height or width < 1, or pitch below
 * 3 * width, a NULL d_kpts or workspace with n > 0. */
#define VPB_DRAW_RGB 0
#define VPB_DRAW_BGR 1
typedef struct vpb_canvas {
  uint8_t* data;          /* u8 [height, width, 3], device address, drawn in place */
  int32_t height, width;
  int64_t pitch_bytes;    /* row pitch; 0 = packed (3 * width) */
  int32_t num_people;     /* this frame's people are the next num_people rows of d_kpts (0 allowed) */
} vpb_canvas;
int64_t vpb_draw_workspace_bytes(int32_t n, int32_t k, int32_t num_limbs);   /* -1 for a negative n or num_limbs, or k < 1 */
int vpb_draw_poses(const vpb_canvas* h_frames, int32_t num_frames, int32_t channel_order, const float* d_kpts, int32_t k,
                   const int32_t* d_person_index, const int32_t* h_limbs, int32_t num_limbs, const uint8_t* h_point_bgr,
                   int32_t num_point_colors, const uint8_t* h_limb_bgr, int32_t num_limb_colors, int32_t radius, float threshold,
                   void* d_workspace, void* stream);

/* ---- SORT tracker: easy_ViTPose/sort.py's Sort for num_streams video streams, updated in one step on the device.  Stream s
 * is one reference Sort(max_age, min_hits, iou_threshold); one update equals calling the S Sort objects round-robin in one
 * process, and the output equals theirs as float64 values (filterpy 1.4.5's Kalman steps without FMA contraction, scipy's
 * linear_sum_assignment with its tie rule; `lap`'s lapjv may break ties differently and is not followed).  The id counter
 * (KalmanBoxTracker.count) is one per tracker: within an update new tracks take ids in stream order, within a stream in
 * creation order.  Track state stays in device memory between updates.
 * vpb_tracker_update: d_dets f64 [S,VPB_TRACK_MAX,5] (x1, y1, x2, y2, score), stream s's first d_counts[s] rows (i32 [S], DEVICE);
 * outputs d_rows f64 [S,VPB_TRACK_MAX,6] (x1, y1, x2, y2, score, id + 1), stream s's first d_out_counts[s] rows in the reference's
 * order, d_boxes i32 [S,VPB_TRACK_MAX,4] those rows' boxes rounded half to even (the boxes vpb_infer_frames takes, saturated
 * to int32).  Two launches, no host synchronisation, no data-dependent host work: the call can be captured in a CUDA graph.
 * A stream whose count is negative or above VPB_TRACK_MAX, or that has a row with a non-finite value or x2 <= x1 or y2 <= y1,
 * or whose live tracks would exceed VPB_TRACK_MAX, is left unchanged, emits 0 rows and sets a status bit (a reference Sort
 * raises in scipy or carries NaN state there); the other streams are unaffected.
 * vpb_tracker_reset: stream_index's tracks and frame count (-1: every stream), enqueued on `stream`; the id counter carries on,
 * as the reference's VitInference.reset() builds a new Sort but keeps KalmanBoxTracker.count.
 * vpb_tracker_next_id / vpb_tracker_set_next_id: the counter, SYNCHRONOUS (wait for the device).
 * vpb_tracker_status: SYNCHRONOUS; the bits VPB_TRACK_* raised since the last query, then clears them.
 * VPB_ERR_ARG: num_streams outside 1..65535, max_age or min_hits < 0, a non-finite iou_threshold, a bad device, null buffers,
 * a stream_index outside -1..S-1, a negative next id. */
#define VPB_TRACK_MAX 128
#define VPB_TRACK_BAD_ROW 1
#define VPB_TRACK_OVER_CAPACITY 2
typedef struct vpb_tracker vpb_tracker;
int vpb_tracker_create(int32_t num_streams, int32_t max_age, int32_t min_hits, double iou_threshold, int32_t device, vpb_tracker** out);
void vpb_tracker_destroy(vpb_tracker* t);
int vpb_tracker_update(vpb_tracker* t, const double* d_dets, const int32_t* d_counts, double* d_rows, int32_t* d_boxes,
                       int32_t* d_out_counts, void* stream);
int vpb_tracker_reset(vpb_tracker* t, int32_t stream_index, void* stream);
int vpb_tracker_next_id(vpb_tracker* t, int64_t* next_id);
int vpb_tracker_set_next_id(vpb_tracker* t, int64_t next_id);
int vpb_tracker_status(vpb_tracker* t, int32_t* status);

/* ---- One Euro smoother: easy_ViTPose/vit_utils/post_processing/one_euro_filter.py's OneEuroFilter kept per track id, for
 * num_streams video streams in one step on the device.  Per stream there is a map id -> (filter, c_last, u_last); update u
 * (the stream's count of accepted updates, from 0) at clock c with rows (id_i, x_i), x_i the (y, x) columns of a [K,3]
 * keypoint row, does: 1. forget every id absent from more than max_gap updates in a row (max_gap = 0: an id missing once
 * starts again); 2. a known id outputs filter(x_i, t_e), t_e = c - c_last in fps mode (fps > 0; c defaults to u, so t_e
 * counts frames) and (c - c_last) * d_cutoff in realtime mode (fps <= 0; c is the caller's timestamp in seconds, standing in
 * for the reference's time()); 3. a new id builds OneEuroFilter(x_i, dx0, min_cutoff, beta, d_cutoff, fps) and outputs x_i
 * unchanged; 4. every id of the update takes c_last = c, u_last = u.  Outputs equal that composition of the reference class
 * as float64 values: numpy's promotion (the first call's float32 x - x_prev), its evaluation order, no FMA contraction, the
 * x <= 0 mask (-10, NaN not masked), the inf / NaN of t_e = 0.  Filter state stays in device memory between updates.
 * vpb_smoother_create: k 1..144 keypoints; fps <= 0 selects realtime mode; every parameter finite; max_gap >= 0.
 * vpb_smoother_update: d_kpts f32 [n,k,3] (y, x, score), the rows of all streams concatenated stream by stream, stream s
 * holding the next d_counts[s] rows (i32 [S], DEVICE); d_ids i32 [n] each row's track id (frame_inference's keys, the
 * tracker's id + 1); d_clock f64 [S] each stream's clock, NULL in fps mode = the update count (VPB_ERR_ARG in realtime mode);
 * n = the rows d_kpts, d_ids and d_out hold.  Writes the smoothed (y, x), rounded to float32, over d_kpts' first two columns
 * (scores untouched) and, when d_out is not NULL, the float64 result to d_out [n,k,2].  Two launches, no host
 * synchronisation: the call can be captured in a CUDA graph.  A stream whose count is negative or above VPB_SMOOTH_MAX, whose
 * rows would run past n, that names an id twice, or that would hold more than VPB_SMOOTH_MAX ids is left unchanged (its rows
 * are not written, its update count does not advance) and sets a status bit; the other streams are unaffected.
 * vpb_smoother_reset: forget stream_index's filters and update count (-1: every stream), enqueued on `stream`.
 * vpb_smoother_status: SYNCHRONOUS; the bits VPB_SMOOTH_* raised since the last query, then clears them.
 * VPB_ERR_ARG: num_streams outside 1..65535, k outside 1..144, a non-finite parameter, max_gap < 0, a bad device, n < 0, null
 * buffers, a null d_clock in realtime mode, a stream_index outside -1..S-1. */
#define VPB_SMOOTH_MAX 128
#define VPB_SMOOTH_DUPLICATE_ID 1
#define VPB_SMOOTH_OVER_CAPACITY 2
typedef struct vpb_smoother vpb_smoother;
int vpb_smoother_create(int32_t num_streams, int32_t k, double min_cutoff, double beta, double d_cutoff, double fps, double dx0,
                        int32_t max_gap, int32_t device, vpb_smoother** out);
void vpb_smoother_destroy(vpb_smoother* s);
int vpb_smoother_update(vpb_smoother* s, float* d_kpts, int32_t n, const int32_t* d_counts, const int32_t* d_ids,
                        const double* d_clock, double* d_out, void* stream);
int vpb_smoother_reset(vpb_smoother* s, int32_t stream_index, void* stream);
int vpb_smoother_status(vpb_smoother* s, int32_t* status);

/* ---- OKS NMS: easy_ViTPose/vit_utils/post_processing/nms.py's oks_iou, oks_nms and soft_oks_nms, for num_frames frames in
 * one launch (one CTA per frame), with HRNet's evaluation rescoring as an option.  Frame f holds the next d_counts[f] rows
 * (i32 [F], DEVICE) of d_kpts f32 [n_rows,k,3] (y, x, score; the OKS is symmetric in the two coordinates, so the
 * reference's (x, y, score) rows give the same result), d_areas f64 [n_rows] and d_scores f64 [n_rows].  h_sigmas: f64 [k]
 * (HOST, copied into the launch), NULL = the reference's COCO-17 table (k = 17 only).
 * Per frame, as the reference computes it (oracle/oks_nms_oracle.py restates it):
 *   order: scores.argsort()[::-1] with a stable argsort, i.e. descending, NaN above +inf, equal scores later index first;
 *     soft NMS re-sorts the remaining order by the same rule every round (ties then go to the later position);
 *   OKS: float32 dx*dx + dy*dy, then / vars / ((a_g + a_d) / 2 + 2^-52) / 2 in float64, exp, numpy's pairwise sum over the
 *     candidate's keypoints with score > vis_thr (oks_iou's mask quirk keeps the candidate's alone; NaN vis_thr = None, all
 *     keypoints), / count, rounded to float32; 0 with no keypoint.  exp is CUDA's, so an OKS can differ by one float32 ulp;
 *   hard (soft = 0): keep the head, drop the rest whose OKS against it is not <= (float)thr, repeat;
 *   soft (soft = 1): keep the head, scores of the rest *= expf(-(o*o) / (float)thr), re-sort, repeat up to max_dets;
 *   rescore_vis_thr (NaN = off): each row's score becomes float32(mean of its keypoint scores > (float)rescore_vis_thr, 0
 *     when none) * float32(d_scores) before the sort, exactly (HRNet's evaluate).
 * Writes d_keep [n_rows]: over each frame's rows its kept frame-local indices in the reference's order, then -1;
 * d_keep_counts [F]; d_scores_out [n_rows] (may be NULL) the score each row was sorted by.  Rows outside every frame's range
 * are not written.  A frame whose count is above VPB_NMS_MAX_PEOPLE (VPB_NMS_TOO_MANY_PEOPLE), negative or running past
 * n_rows (VPB_NMS_BAD_ROWS) keeps nothing (count 0, -1 over its rows inside the buffer) and ORs its bit into *d_status (i32,
 * DEVICE; the caller clears it); the other frames are unaffected.  No allocation, no host synchronisation: the call can be
 * captured in a CUDA graph.
 * vpb_oks_iou: the OKS matrix of every frame, d_oks f32 [n_rows, VPB_NMS_MAX_PEOPLE]: row r = frame row i, column j < n_f =
 * oks_iou(g = person i, d = person j); other columns are not written.  Same limits and status bits.
 * VPB_ERR_ARG: k outside 1..VPB_NMS_MAX_K, n_rows < 0, num_frames outside 0..65535, null buffers or params, NULL h_sigmas
 * with k != 17, a non-finite sigma or thr, soft not 0 / 1, a soft max_dets outside 0..VPB_NMS_MAX_DETS. */
#define VPB_NMS_MAX_PEOPLE 256
#define VPB_NMS_MAX_K 144
#define VPB_NMS_MAX_DETS 256
#define VPB_NMS_TOO_MANY_PEOPLE 1
#define VPB_NMS_BAD_ROWS 2
typedef struct vpb_oks_nms_params {
  double thr;               /* oks_nms / soft_oks_nms `thr`, used as float32 */
  double vis_thr;           /* oks_iou `vis_thr`, NaN = None */
  double rescore_vis_thr;   /* HRNet's in_vis_thre, NaN = no rescoring */
  int32_t soft;             /* 0: oks_nms, 1: soft_oks_nms */
  int32_t max_dets;         /* soft_oks_nms `max_dets` */
} vpb_oks_nms_params;
int vpb_oks_nms(const float* d_kpts, int32_t n_rows, int32_t k, const int32_t* d_counts, int32_t num_frames, const double* d_areas,
                const double* d_scores, const double* h_sigmas, const vpb_oks_nms_params* params, int32_t* d_keep,
                int32_t* d_keep_counts, double* d_scores_out, int32_t* d_status, void* stream);
int vpb_oks_iou(const float* d_kpts, int32_t n_rows, int32_t k, const int32_t* d_counts, int32_t num_frames, const double* d_areas,
                const double* h_sigmas, double vis_thr, float* d_oks, int32_t* d_status, void* stream);

/* ---- COCO keypoint evaluation: pycocotools' COCOeval(cocoGt, cocoDt, 'keypoints') evaluate(), accumulate() and summarize() for
 * category 1 with Params.setKpParams (maxDets 20, OKS thresholds .5:.05:.95, recall thresholds 0:.01:1, areas all / medium /
 * large), over gts->num_images images in one enqueue (oracle/coco_oks_eval.py restates the algorithm).  All buffers DEVICE.
 * Ground truths, CSR by image in ascending image id (COCOeval's np.unique order): image i holds rows [offsets[i], offsets[i+1])
 * of kpts f64 [num_gts,k,3] (x, y, v), area f64, bbox f64 [num_gts,4] (x, y, w, h), iscrowd i32 and num_keypoints i32.  _ignore
 * is iscrowd != 0, num_keypoints == 0, or area outside the range (pycocotools' _prepare overwrites a gt 'ignore' field).
 * Detections come as frames: frame f holds the next counts[f] rows (the layout vpb_oks_nms reads) of kpts f64 [n_rows,k,2]
 * (x, y) and scores f64 [n_rows], and belongs to image frame_image[f] (0..num_images-1).  With keep (optional, the d_keep /
 * d_keep_counts vpb_oks_nms writes) frame f contributes rows keep[first row + j], j < keep_counts[f], in that order; without
 * it every row.  An image's detections are its frames' rows in frame order, which decides ties among equal scores.  Each
 * detection's area is loadRes's (max x - min x) * (max y - min y).
 * Per image: argsort(-score, kind='mergesort') (descending, stable, NaN last), first 20; computeOks in float64 (the bbox
 * distance for a ground truth with no v > 0); evaluateImg's greedy matching.  accumulate concatenates the images in order and
 * sorts stably by score; summarize takes np.mean over the entries > -1.  Everything but exp follows numpy's order and rounding
 * (pairwise sums, no FMA), so the results equal the numpy statement bit for bit unless CUDA's exp moves an OKS by an ulp across
 * a threshold or another OKS.
 * Writes d_stats f64 [10] (AP, AP50, AP75, AP_medium, AP_large, AR, AR50, AR75, AR_medium, AR_large), d_precision f64
 * [3,10,101] (area, threshold, recall threshold; -1 where an area has no non-ignored ground truth) and d_recall f64 [3,10].
 * An image with more than VPB_COCO_MAX_GTS ground truths (VPB_COCO_TOO_MANY_GTS) or more than VPB_COCO_MAX_ROWS detection rows
 * (VPB_COCO_TOO_MANY_ROWS), a negative count, rows past n_rows, keep counts or entries outside their frame, a frame_image
 * outside 0..num_images-1 or offsets out of order (VPB_COCO_BAD_INPUT) ORs its bit into *d_status (i32; the caller clears it),
 * and every stat is then NaN.  d_workspace: at least vpb_coco_eval_workspace_bytes(num_images, num_frames) bytes (-1 for bad
 * sizes), 256-byte aligned.  No allocation, no host synchronisation: the call can be captured in a CUDA graph.
 * h_sigmas f64 [k] (HOST), NULL = the COCO-17 table (k = 17 only).
 * VPB_ERR_ARG: k outside 1..VPB_COCO_MAX_K, num_images outside 1..VPB_COCO_MAX_IMAGES, a negative size, null buffers, a keep
 * list without keep counts, a short workspace, NULL h_sigmas with k != 17, a non-finite sigma. */
#define VPB_COCO_MAX_GTS 256
#define VPB_COCO_MAX_ROWS 1024
#define VPB_COCO_MAX_K 144
#define VPB_COCO_MAX_IMAGES 1000000
#define VPB_COCO_TOO_MANY_GTS 1
#define VPB_COCO_TOO_MANY_ROWS 2
#define VPB_COCO_BAD_INPUT 4
typedef struct vpb_coco_gts {
  const int32_t* offsets;        /* [num_images + 1] */
  const double* kpts;            /* [num_gts, k, 3] */
  const double* area;            /* [num_gts] */
  const double* bbox;            /* [num_gts, 4] */
  const int32_t* iscrowd;        /* [num_gts] */
  const int32_t* num_keypoints;  /* [num_gts] */
  int32_t num_images;
  int32_t num_gts;
} vpb_coco_gts;
typedef struct vpb_coco_dets {
  const double* kpts;            /* [n_rows, k, 2] */
  const double* scores;          /* [n_rows] */
  const int32_t* counts;         /* [num_frames] */
  const int32_t* frame_image;    /* [num_frames] */
  const int32_t* keep;           /* [n_rows] or NULL */
  const int32_t* keep_counts;    /* [num_frames] or NULL */
  int32_t n_rows;
  int32_t num_frames;
} vpb_coco_dets;
int64_t vpb_coco_eval_workspace_bytes(int32_t num_images, int32_t num_frames);
int vpb_coco_eval(int32_t k, const double* h_sigmas, const vpb_coco_gts* gts, const vpb_coco_dets* dets, void* d_workspace,
                  int64_t workspace_bytes, double* d_stats, double* d_precision, double* d_recall, int32_t* d_status, void* stream);

/* Introspection used by bench.py / tests. */
int vpb_kernel_launches(const vpb_engine* e, int32_t batch);          /* kernels one vpb_infer enqueues */
/* The engine's cached CUDA graphs: mixed = 0 the single-head calls' (one per batch size and decode kind), 1 the multi-head
 * calls' (one per segment list, at most 16).  *entries = layouts seen and kept, *captured = those with a captured graph. */
int vpb_cached_graphs(const vpb_engine* e, int32_t mixed, int32_t* entries, int32_t* captured);
/* Device bytes the engine holds: packed weights, workspace, staging buffers. */
int64_t vpb_device_bytes(const vpb_engine* e);
/* Options (all keep the results bit-identical unless noted): "stop_after", "profile", "pdl", "graph", "ln_fused",
 * "chain" (chained persistent launches, default 0: measured slower on H100), "chain_min_batch" (smallest batch that takes them, default 1),
 * "ln_in_gemm" (LayerNorm + its consumer GEMM as one launch on the unchained path, default 0), "gelu_erf" (fc1 epilogue with
 * erf instead of the fitted tanh form: rounding-level differences), "ln_ctl" (chained launches: counter polls / publishes of
 * the LayerNorm jobs on a control warp, default 1; VPB_LN_CTL), "ln_job_rows" (8 | 16 rows per LayerNorm job, default 16),
 * "resid_rmw" (residual epilogues as load + add + store instead of TMA reduce-add, default 0; VPB_RESID_RMW).
 * "poison" (debug; value != 0) is an action, not a setting: SYNCHRONOUSLY fills every float and bf16 activation and staging
 * buffer with 0xFF bytes (NaN), keeping the cached CUDA graphs, so a test can show that no call uses workspace values it did not
 * write; integer / double buffers, counters and status words are not touched. */
int vpb_set_option(vpb_engine* e, const char* name, int32_t value);
/* Flip test, the test_cfg flip_test=True of every reference config (configs/ViTPose_common.py:91,124,157,190): mmpose's
 * (output + output_flipped) * 0.5, where output_flipped is the model run on flip(crop, dims=[3]) and passed through flip_back
 * (vit_utils/post_processing/post_transforms.py:110-147) and, with shift != 0, the one-pixel shift of
 * TopdownHeatmapSimpleHead.inference_model (vit_models/head/topdown_heatmap_simple_head.py:195-218, shift at :210-212).
 * h_perm i32 [k] (HOST) = the keypoint permutation the flip pairs induce (as for vpb_flip_back); k must equal the engine's K
 * and every entry lie in [0,K), else VPB_ERR_ARG.  h_perm = NULL turns flip test off (the default).
 * While it is on, vpb_infer, vpb_infer_host, vpb_submit_host, vpb_infer_frame, vpb_infer_frame_host, vpb_submit_frame_host and
 * the multi-frame calls (vpb_infer_frames, vpb_infer_frames_host, vpb_submit_frames_host) and the affine calls
 * (vpb_infer_affine, vpb_infer_affine_host) run each crop and its mirror image as one batch of 2 * batch crops (the mirror images are gathered on the fly, never
 * stored), average the maps and decode the averaged maps (wrap_batch = 0); d_heatmaps, when given, receives the averaged
 * maps.  batch must then be <= max_batch / 2.  vpb_forward, vpb_forward_features, vpb_head, vpb_decode* and vpb_flip_back
 * are unaffected.  SYNCHRONOUS: waits for the engine's pending work (which keeps the previous setting), and drops the
 * engine's cached CUDA graphs. */
int vpb_set_flip_test(vpb_engine* e, const int32_t* h_perm, int32_t k, int32_t shift);
/* Flip test for every head of an engine (vpb_create_heads; also valid with one head): h_perms i32 [total] (HOST) = the
 * permutation of every head, concatenated in head order; total must equal the sum of the heads' K_j and every entry of head j
 * lie in [0, K_j), else VPB_ERR_ARG.  h_perms = NULL turns flip test off.  One shift for all heads.  While it is on, the
 * multi-head calls (vpb_infer_heads, vpb_infer_frames_heads, vpb_infer_frames_heads_host, vpb_infer_affine_heads,
 * vpb_infer_affine_heads_host) run the n crops in segment order followed by their n mirror images (the fc2 expert segments of
 * those 2n crops are the segment list twice, runs of one head merged), average each segment's maps with its head's permutation
 * and decode them; the single-head calls run head 0 with head 0's permutation, bit-identical to a head-0 single-head engine with
 * vpb_set_flip_test.  Every keypoint call then takes at most max_batch / 2 crops.  Synchronous like vpb_set_flip_test, and drops
 * both graph caches; this call and vpb_set_flip_test each replace the other's setting. */
int vpb_set_flip_test_heads(vpb_engine* e, const int32_t* h_perms, int32_t total, int32_t shift);
/* With option "profile"=1 every launch is bracketed by a CUDA-event pair on its stream; collect() synchronises,
 * sums elapsed ms and launch counts per kernel class (arrays of vpb_profile_classes() entries) and resets. */
int vpb_profile_classes(void);
const char* vpb_profile_class_name(int32_t cls);
int vpb_profile_collect(vpb_engine* e, float* ms_per_class, int32_t* launches_per_class);
int vpb_read_buffer(vpb_engine* e, const char* name, void* host_dst, int64_t bytes);  /* synchronous debug read */

/* Kernel-level entry points (unit tests / profiling).  All pointers are device pointers.
 * vpb_gemm: out = epilogue(A[M,K] bf16 * W[N,K]^T bf16 + bias);  epilogue ids as in csrc/gemm.cuh (0 bias->bf16, 1 bias+GELU->bf16,
 * 2 implicit-GEMM deconv: aux = H, W, tile rows, (tile cols << 16) | Cin, 4 bias->f32 NCHW: aux0 = channels, aux1 = pixels,
 * 5 f32 out += ...).  d_resid / resid_mod are reserved (pass NULL / 0). */
int vpb_gemm(const void* d_a, const void* d_w, const float* d_bias, void* d_out, int32_t m, int32_t n, int32_t k,
             int32_t epilogue, const float* d_resid, int32_t resid_mod, int32_t aux0, int32_t aux1, int32_t aux2,
             int32_t aux3, void* stream);
/* Debug: limit the GEMM smem ring depth and/or collect per-CTA cycle counters (int64 [grid*8]) for following GEMM launches.
 * Bits 0..7 = the ring depth (0 = the compiled depth; 1 returns VPB_ERR_ARG), bits 8.. = GemmParams::dbg_flags (csrc/gemm.cuh)
 * and the engine's overrides of tile width and residual form.  The depth applies to vpb_gemm, vpb_expert_gemm and the engine's
 * standalone and expert GEMM launches. */
int vpb_debug_gemm(int32_t stages_limit, void* d_counters);
/* The fc2 of a multi-head call on an engine with experts (ViTPose+), by the engine's own launch code: the grouped expert GEMM
 * x[r, D-P + n] += A[r, :] * W[D-P + e*P + n, :]^T + bias[D-P + e*P + n] for every row r of a segment with expert e and n < P, and
 * with shared != 0 first the shared columns x[:, :D-P] += A * W[:D-P]^T + bias[:D-P] over all M rows.  d_a bf16 [M, 4D]; d_w bf16
 * [D-P + num_experts*P, 4D] and d_bias f32 [D-P + num_experts*P] stacked as [shared; expert 0; ...]; d_x f32 [M, D], updated in
 * place.  h_segs i32 [num_segs, 3] (HOST): row_begin, row_end, expert; 1..128 segments in ascending, non-overlapping row order.
 * VPB_ERR_ARG: D not a multiple of 32, P outside 32..D-32 or not a multiple of 32, a segment out of order, empty, past M or with
 * an expert outside [0, num_experts).  Honours vpb_debug_gemm's ring depth. */
int vpb_expert_gemm(const void* d_a, const void* d_w, const float* d_bias, float* d_x, int32_t m, int32_t d, int32_t p,
                    int32_t num_experts, const int32_t* h_segs, int32_t num_segs, int32_t shared, void* stream);
int vpb_attention(const void* d_qkv, int32_t batch, int32_t heads, int32_t head_dim, void* d_out, void* stream);
/* qkv GEMM + attention in one launch: out = attention(xn[batch*192, D] * W[3D, D]^T + bias[3D]), D = heads * head_dim a multiple
 * of 64; bit-identical to vpb_gemm (epilogue 0) followed by vpb_attention.  Both attention entry points fill vpb_debug_gemm's
 * counters when they are set.  Both return VPB_ERR_ARG, before any device work, for a null pointer, head_dim other than 32, 64
 * or 80, batch or heads < 1, or 3 * heads * head_dim, batch * heads or batch * 192 beyond INT32_MAX. */
int vpb_qkv_attention(const void* d_xn, const void* d_w, const float* d_bias, int32_t batch, int32_t heads, int32_t head_dim,
                      void* d_out, void* stream);
/* Debug / measurement switch (process-wide) for the attention kernel.  flags < 0: the defaults (every softmax exponential on
 * the MUFU; VPB_ATT_POLY = 1 in the environment evaluates every 4th one by a polynomial on the FMA pipe instead); otherwise
 * bit 0 = polynomial exponentials, bit 1 = run every block's qkv GEMM and attention as one fused launch, bit 2 = as two launches
 * (neither: the engine's rule; both forms are bit-identical), bits 8.. = cap on the number of CTAs of both attention kernels
 * (0 = one per SM; tests use it to give every CTA several items).  Engines capture CUDA graphs with the setting in effect. */
int vpb_debug_attention(int32_t flags);
int vpb_layernorm(const float* d_x, const float* d_gamma, const float* d_beta, void* d_y, int32_t rows, int32_t dim,
                  float eps, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VITPOSE_B200_H */
