"""Drop-in boundary for easy_ViTPose/inference.py: the torch engine backend re-bound to the H100 engine.

The reference picks its engine in VitInference.__init__ by assigning `self._vit_pose` and
`self._inference = self._inference_torch` (easy_ViTPose/inference.py:156-172); the per-person loop then
calls `self._inference(img_inf)[0]` (:268).  `install()` performs the same two assignments with this
module's backend, so YOLO / SORT / draw and the CLI stay the reference's own code.

`B200PoseBackend` also offers what the reference lists as a TODO (README.md:323): one batched call for
all crops of a frame (`infer_crops`, `inference_batch`), and -- SURVEY.md section 8 rows f1/f2 -- the whole
per-person loop of `VitInference.inference` (:258-272) as ONE engine call on the uint8 frame
(`inference_frame`, and `install(..., batched=True)` which re-binds `VitInference.inference` itself).
"""
from __future__ import annotations

import time
import types

import numpy as np
import torch

from .configs import data_cfg, flip_pairs_for, model_cfg
from .model import ViTPose, _unwrap, state_dict_decoder
from .nms import check as nms_check, oks_nms_device
from .top_down_eval import decode_heatmaps
from .topdown import topdown_args, xywh2cs

__all__ = ["B200PoseBackend", "DeviceTracker", "install", "frame_inference", "frame_draw", "MEAN", "STD"]

MEAN = [0.485, 0.456, 0.406]      # easy_ViTPose/inference.py:32
STD = [0.229, 0.224, 0.225]       # easy_ViTPose/inference.py:33


def pre_img(img: np.ndarray, target_size=(192, 256)):
    """uint8 RGB [h,w,3] -> float32 [1,3,256,192] + (org_h, org_w): bilinear resize, /255, normalise in
    float64, HWC->CHW (easy_ViTPose/inference.py:314-318).  CPU, as in the reference (SURVEY.md section 8 row a1)."""
    import cv2
    org_h, org_w = img.shape[:2]
    x = cv2.resize(img, tuple(target_size), interpolation=cv2.INTER_LINEAR) / 255
    x = ((x - MEAN) / STD).transpose(2, 0, 1)[None].astype(np.float32)
    return x, org_h, org_w


class B200PoseBackend:
    """Owns an H100 `ViTPose` engine and exposes the three methods VitInference's torch backend consists of:
    pre_img (:314-318), _inference (:320-328), postprocess (:187-205)."""

    def __init__(self, model: ViTPose, device: "int | str | None" = None):
        self.model = model.eval()
        if device is not None:
            self.model.to(device)
        self.target_size = data_cfg["image_size"]

    @classmethod
    def from_state_dict(cls, state_dict: dict, size: str, num_keypoints: int, max_batch: int = 64, device=None):
        """A backend for a reference checkpoint ({'state_dict': ...} or the bare dict).  The decoder comes from the keys: a 3x3
        keypoint_head.final_layer.weight and no deconv_layers.* is the simple decoder, anything else the classic head (the
        strict load then reports what does not fit)."""
        state_dict = _unwrap(state_dict)
        m = ViTPose(model_cfg(size, num_keypoints, state_dict_decoder(state_dict)), max_batch=max_batch)
        m.load_state_dict(state_dict)
        return cls(m, device if device is not None else "cuda")

    def pre_img(self, img):
        return pre_img(img, self.target_size)

    @staticmethod
    def postprocess(heatmaps, org_w, org_h):
        """heatmaps [N,K,64,48] (numpy or CUDA tensor) -> float32 [N,K,3] rows (y, x, score).
        Same arguments as VitInference.postprocess; like the reference it treats the array as one call
        (for N=1 -- the only way VitInference uses it -- the two wrap modes coincide)."""
        hm = heatmaps if isinstance(heatmaps, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(heatmaps, np.float32))
        if not hm.is_cuda:
            hm = hm.cuda()
        n = hm.shape[0]
        org = torch.tensor([[int(org_w), int(org_h)]] * n, dtype=torch.int32)
        kp, _ = decode_heatmaps(hm, org, wrap_batch=True)
        return kp.cpu().numpy()

    @torch.no_grad()
    def _inference(self, img: np.ndarray) -> np.ndarray:
        """uint8 RGB crop -> float32 [1,K,3] (y, x, score) in crop pixels; the contract of
        VitInference._inference_torch (:320-328)."""
        x, org_h, org_w = self.pre_img(img)
        kp, _ = self.model.infer_host(x, np.array([[org_w, org_h]], np.int32))
        return kp

    @torch.no_grad()
    def infer_crops(self, crops, org_wh):
        """Pre-normalised crops [B,3,256,192] (CUDA tensor) -> (kpts [B,K,3], idx [B,K]) CUDA tensors."""
        return self.model.infer_crops(crops, org_wh)

    @torch.no_grad()
    def inference_frame(self, img: np.ndarray, bboxes: np.ndarray) -> np.ndarray:
        """uint8 RGB frame [H,W,3] + detector boxes [n,4] (x0,y0,x1,y1; floats are rounded as inference.py:253 does)
        -> float32 [n,K,3] (y, x, score) in frame pixels: inference.py:258-272 for all people in one engine call."""
        return self.model.infer_frame_host(img, bboxes)[0]

    @torch.no_grad()
    def inference_frames(self, imgs: "list[np.ndarray]", bboxes_list: "list[np.ndarray]", rotate=0) -> "list[np.ndarray]":
        """Several uint8 RGB frames (cameras of a rig, frames of a video, several streams) + each frame's boxes -> one
        float32 [n_i,K,3] (y, x, score) per frame, in that frame's pixels: inference_frame for all of them with the people of
        all frames packed into as few engine calls as max_batch allows.  `rotate` (0 | 90 | 180 | 270 degrees
        counter-clockwise, one for all frames or one per frame; the reference's `--rotate`): frames are stored sideways and
        seen as cv2.rotate turns them, boxes and keypoints in the rotated frame's pixels, with no rotated copy made."""
        return self.model.infer_frames_host(imgs, bboxes_list, rotate)[0]

    @torch.no_grad()
    def inference_frames_nv12(self, frames, bboxes_list: "list[np.ndarray]", matrix: str = "bt601", rotate=0) -> "list[np.ndarray]":
        """inference_frames on NV12 video frames (uint8 [3H/2, W] with the planes stacked, or (y, uv) pairs): no RGB conversion."""
        return self.model.infer_frames_nv12_host(frames, bboxes_list, matrix, rotate=rotate)[0]

    @torch.no_grad()
    def inference_frames_heads(self, imgs: "list[np.ndarray]", bboxes_list: "list[np.ndarray]", heads_list, rotate=0) -> "list[np.ndarray]":
        """inference_frames on a multi-head engine (ViTPose(..., heads=...)), with a head index per box (heads_list: per frame
        an int array [n_i], e.g. 0 for people and 3 for animals of a ViTPose+ engine) -> one float32 [n_i,K_max,3] (y, x,
        score) per frame; a box of head j fills rows 0..K_j-1."""
        return self.model.infer_frames_heads_host(imgs, bboxes_list, heads_list, rotate)[0]

    @torch.no_grad()
    def inference_topdown(self, imgs: "list[np.ndarray]", bboxes_list: "list[np.ndarray]", padding: float = 1.25,
                          use_udp: bool = True, rotate=0) -> "list[np.ndarray]":
        """mmpose-style top-down inference: uint8 RGB frames + each frame's person boxes [n_i,4] (x, y, w, h) -> one float32
        [n_i,K,3] (y, x, score) per frame in image pixels.  Each box becomes the reference's centre / scale and warp matrix
        (topdown_args: datasets/COCO.py:318-337, the UDP get_warp_matrix of every config's test_cfg), the crop is
        cv2.warpAffine's, and the keypoints are keypoints_from_heatmaps(c, s, use_udp=True)'s -- all on the device.  `rotate`
        as inference_frames: the boxes and keypoints are in the rotated frame's pixels."""
        args = [topdown_args(b, padding, use_udp) for b in bboxes_list]
        return self.model.infer_affine_host(imgs, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args], rotate)[0]

    @torch.no_grad()
    def inference_topdown_nv12(self, frames, bboxes_list: "list[np.ndarray]", padding: float = 1.25, use_udp: bool = True,
                               matrix: str = "bt601", rotate=0) -> "list[np.ndarray]":
        """inference_topdown on NV12 video frames (uint8 [3H/2, W] with the planes stacked, or (y, uv) pairs)."""
        args = [topdown_args(b, padding, use_udp) for b in bboxes_list]
        return self.model.infer_affine_nv12_host(frames, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args], matrix,
                                                 rotate=rotate)[0]

    @torch.no_grad()
    def inference_topdown_heads(self, imgs: "list[np.ndarray]", bboxes_list: "list[np.ndarray]", heads_list, padding: float = 1.25,
                                use_udp: bool = True, rotate=0) -> "list[np.ndarray]":
        """inference_topdown on a multi-head engine, with a head index per box (heads_list: per frame an int array [n_i]) -> one
        float32 [n_i,K_max,3] (y, x, score) per frame in image pixels; a box of head j fills rows 0..K_j-1.  Flip test, when set
        with ViTPose.set_flip_test_heads, applies with each box's head's pairs."""
        args = [topdown_args(b, padding, use_udp) for b in bboxes_list]
        return self.model.infer_affine_heads_host(imgs, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args], heads_list,
                                                  rotate)[0]

    @torch.no_grad()
    def inference_topdown_eval(self, imgs: "list[np.ndarray]", bboxes_xywh_list: "list[np.ndarray]", box_scores_list,
                               oks_thr: float = 0.9, in_vis_thr: float = 0.2, soft_nms: bool = False, padding: float = 1.25,
                               use_udp: bool = True, rotate=0, evaluator=None, image_ids=None) -> "list[tuple]":
        """The top-down evaluation with detector boxes (HRNet / mmpose's evaluate, the thresholds of datasets/COCO.py:237-241)
        on the device: inference_topdown, then each person's score = box score x mean keypoint score above in_vis_thr, then
        per frame oks_nms (soft_nms: soft_oks_nms, max_dets 20) at oks_thr with the COCO-17 sigmas (the engine must have 17
        keypoints) and area = s[0] * s[1] * 200 * 200 of the box's scale, all in one read-back.  Returns per frame (kept
        keypoints float32 [m,K,3] (y, x, score), their rescored scores float64 [m], their box indices int64 [m]), in the
        reference's order.  Honours the flip test.
        evaluator: a coco_eval.DeviceCocoEval; the kept people and their rescored scores are then appended to it from device
        memory before the read-back, frame j as image image_ids[j] (one COCO image id per frame), the same detections
        `evaluator.add` takes from records built from the returned poses."""
        if not (len(imgs) == len(bboxes_xywh_list) == len(box_scores_list)):
            raise ValueError(f"{len(imgs)} frames, {len(bboxes_xywh_list)} box arrays, {len(box_scores_list)} score arrays")
        if evaluator is not None and (image_ids is None or len(image_ids) != len(imgs)):
            raise ValueError(f"an evaluator needs one image id per frame ({len(imgs)} frames)")
        K = self.model.num_keypoints
        boxes = [np.asarray(b, np.float64).reshape(-1, 4) for b in bboxes_xywh_list]
        scores = [np.asarray(s, np.float64).reshape(-1) for s in box_scores_list]
        for j, (b, s) in enumerate(zip(boxes, scores)):
            if len(b) != len(s):
                raise ValueError(f"frame {j}: {len(b)} boxes and {len(s)} scores")
        counts = [len(b) for b in boxes]
        n, F = sum(counts), len(imgs)
        areas = np.zeros(n, np.float64)
        for r, box in enumerate(b for bb in boxes for b in bb):
            s = xywh2cs(box, padding)[1].astype(np.float64)
            areas[r] = s[0] * s[1] * 200 * 200                   # HRNet's area, from the float64 copy of the scale
        args = [topdown_args(b, padding, use_udp) for b in boxes]
        frames = [im if isinstance(im, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(im)) for im in imgs]
        kps, _ = self.model.infer_affine(frames, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args], rotate=rotate)
        dev = torch.device("cuda", self.model._device)
        kp = torch.cat(kps) if kps else torch.zeros((0, K, 3), dtype=torch.float32, device=dev)
        host = np.concatenate([areas, np.concatenate(scores) if n else np.zeros(0)])
        d = torch.from_numpy(host).to(dev)
        cnt = torch.tensor(counts, dtype=torch.int32).to(dev)
        # one read-back: scores f64 [n] | kpts f32 [n,K,3] | keep i32 [n] | keep_counts i32 [F] | status i32 [1]
        nk = n * K * 3
        back = torch.empty(n + (nk + n + F + 2) // 2, dtype=torch.float64, device=dev)
        bw = back[n:].view(torch.int32)
        oks_nms_device(kp, cnt, d[:n], d[n:], oks_thr, soft=soft_nms, rescore_vis_thr=in_vis_thr,
                             out=(bw[nk:nk + n], bw[nk + n:nk + n + F], back[:n], bw[nk + n + F:nk + n + F + 1].zero_()))
        bw[:nk].view(torch.float32).view(n, K, 3).copy_(kp)
        if evaluator is not None:
            evaluator.add_device(kp, back[:n], cnt, image_ids, keep=bw[nk:nk + n], keep_counts=bw[nk + n:nk + n + F])
        h = back.cpu().numpy()
        hw = h[n:].view(np.int32)
        nms_check(hw[nk + n + F])
        hk = hw[:nk].view(np.float32).reshape(n, K, 3)
        out, r0 = [], 0
        for j, c in enumerate(counts):
            idx = hw[nk + r0:nk + r0 + hw[nk + n + j]].astype(np.int64)
            out.append((hk[r0 + idx].copy(), h[r0 + idx].copy(), idx))
            r0 += c
        return out

    # YUV video frames in any layout ViTPose.infer_frames_yuv takes (layout "i420" | "yv12" | "nv12" | "nv21" | "yuyv" | "uyvy",
    # e.g. ffmpeg's `-pix_fmt yuv420p` output or a V4L2 webcam's YUYV frame), converted on the device only where the gather taps
    @torch.no_grad()
    def inference_frames_yuv(self, frames, bboxes_list: "list[np.ndarray]", layout: str = "i420", matrix: str = "bt601",
                             full_range: bool = False, rotate=0) -> "list[np.ndarray]":
        """inference_frames on YUV video frames: no RGB conversion."""
        return self.model.infer_frames_yuv_host(frames, bboxes_list, layout, matrix, full_range, rotate)[0]

    @torch.no_grad()
    def inference_topdown_yuv(self, frames, bboxes_list: "list[np.ndarray]", padding: float = 1.25, use_udp: bool = True,
                              layout: str = "i420", matrix: str = "bt601", full_range: bool = False, rotate=0) -> "list[np.ndarray]":
        """inference_topdown on YUV video frames."""
        args = [topdown_args(b, padding, use_udp) for b in bboxes_list]
        return self.model.infer_affine_yuv_host(frames, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args], layout, matrix,
                                                full_range, rotate)[0]

    @torch.no_grad()
    def inference_frames_heads_yuv(self, frames, bboxes_list: "list[np.ndarray]", heads_list, layout: str = "i420",
                                   matrix: str = "bt601", full_range: bool = False, rotate=0) -> "list[np.ndarray]":
        """inference_frames_heads on YUV video frames."""
        return self.model.infer_frames_heads_yuv_host(frames, bboxes_list, heads_list, layout, matrix, full_range, rotate)[0]

    @torch.no_grad()
    def inference_topdown_heads_yuv(self, frames, bboxes_list: "list[np.ndarray]", heads_list, padding: float = 1.25,
                                    use_udp: bool = True, layout: str = "i420", matrix: str = "bt601",
                                    full_range: bool = False, rotate=0) -> "list[np.ndarray]":
        """inference_topdown_heads on YUV video frames."""
        args = [topdown_args(b, padding, use_udp) for b in bboxes_list]
        return self.model.infer_affine_heads_yuv_host(frames, [a[0] for a in args], [a[1] for a in args], [a[2] for a in args], heads_list,
                                                      layout, matrix, full_range, rotate)[0]

    def draw_frames(self, imgs: "list[np.ndarray]", kpts_list: "list[np.ndarray]", skeleton, person_index=None,
                    confidence_threshold: float = 0.5, channel_order: str = "rgb", point_colors=None, limb_colors=None) -> "list[np.ndarray]":
        """Host form of draw.draw_poses: uint8 [H,W,3] frames + each frame's float32 [n_i,K,3] (y, x, score) keypoints -> new
        frames with every person's skeleton and keypoints drawn as VitInference.draw() draws them, with one upload, one launch
        and one download.  person_index: None (position within the frame) or per frame a sequence of n_i colour indices
        (draw() uses the tracker ids); colours BGR, None = draw.reference_palettes()."""
        from .draw import draw_poses
        if len(imgs) != len(kpts_list):
            raise ValueError(f"{len(imgs)} frames and {len(kpts_list)} keypoint arrays")
        imgs = [np.ascontiguousarray(im, np.uint8) for im in imgs]
        if any(im.ndim != 3 or im.shape[2] != 3 for im in imgs):
            raise ValueError("frames must be uint8 [H, W, 3]")
        kps = [np.asarray(k, np.float32) for k in kpts_list]
        if any(k.ndim != 3 or k.shape[2] != 3 for k in kps) or len({k.shape[1] for k in kps}) > 1:
            raise ValueError("keypoints must be float32 [n_i, K, 3] with one K for all frames")
        if not imgs:
            return []
        counts = [len(k) for k in kps]
        dev = torch.device("cuda", self.model._device if self.model._device is not None else torch.cuda.current_device())
        sizes = [im.size for im in imgs]
        offs = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
        buf = torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).to(dev)
        frames = [buf[offs[j]:offs[j + 1]].view(im.shape) for j, im in enumerate(imgs)]
        kp = torch.from_numpy(np.concatenate(kps, 0))
        pidx = None if person_index is None else np.concatenate([np.asarray(p, np.int64).reshape(-1) for p in person_index]).astype(np.int32)
        with torch.cuda.device(dev):
            draw_poses(frames, kp.to(dev), counts, skeleton, pidx, point_colors, limb_colors, confidence_threshold, channel_order)
        out = buf.cpu().numpy()
        return [out[offs[j]:offs[j + 1]].reshape(im.shape) for j, im in enumerate(imgs)]

    @torch.no_grad()
    def inference_frames_tracked(self, imgs: "list[np.ndarray]", dets_list, tracker, rotate=0, smoother=None,
                                 clock=None) -> "list[dict]":
        """S streams' `frame_inference` after detection: one frame per stream (uint8 RGB [H,W,3], numpy or CUDA) and its
        detections [n_s, 5] (empty where the detector was skipped, as frame_inference passes them) -> one {id: float32 [K,3]
        (y, x, score)} per stream.  `tracker` (a track.DeviceSort of S streams on the engine's device) is updated once; its
        int32 boxes feed infer_frames on the device, and only the row counts and ids come back before the pose call.  `rotate`:
        each stream's rotation as inference_frames takes it (one for all or one per stream); detections, tracks and keypoints
        are in the rotated frames' pixels.  `smoother` (a smooth.DeviceOneEuro of S streams and the engine's K) smooths every
        person's (y, x) by track id on the device before the read-back; the scores stay as the engine gave them.  `clock`:
        one value per stream for the smoother (realtime mode: seconds, default time.time() for every stream; fps mode:
        default each stream's update count)."""
        if len(imgs) != tracker.num_streams:
            raise ValueError(f"{len(imgs)} frames for a tracker of {tracker.num_streams} streams")
        if smoother is not None and (smoother.num_streams != tracker.num_streams or smoother.num_keypoints != self.model.num_keypoints):
            raise ValueError(f"a smoother of {smoother.num_streams} streams and {smoother.num_keypoints} keypoints for "
                             f"{tracker.num_streams} streams and {self.model.num_keypoints} keypoints")
        dets, counts = tracker.pack(dets_list)
        rows, boxes, out_counts = tracker.update_device(dets, counts)
        n = out_counts.tolist()
        ids = rows[:, :, 5].long().cpu()                     # the rows' id + 1, the keys frame_inference uses (inference.py:249)
        frames = [im if isinstance(im, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(im)) for im in imgs]
        kps, _ = self.model.infer_frames(frames, [boxes[s, :c] for s, c in enumerate(n)], rotate=rotate)
        if smoother is not None:
            dev = rows.device
            kp = torch.cat(kps) if kps else torch.zeros((0, self.model.num_keypoints, 3), dtype=torch.float32, device=dev)
            row_ids = torch.cat([rows[s, :c, 5] for s, c in enumerate(n)]).to(torch.int32)
            if clock is None and smoother.realtime:
                clock = [time.time()] * tracker.num_streams
            clk = None if clock is None else torch.as_tensor(np.asarray(clock, np.float64)).to(dev)
            with torch.cuda.device(dev):
                smoother.update_device(kp, out_counts, row_ids, clk)
            kps = kp.split(n)
        return [dict(zip(ids[s, :c].tolist(), kp.cpu().numpy())) for s, (c, kp) in enumerate(zip(n, kps))]

    @torch.no_grad()
    def inference_batch(self, imgs: "list[np.ndarray]") -> np.ndarray:
        """All person crops of a frame in one engine call -> float32 [n,K,3]."""
        if not imgs:
            return np.zeros((0, self.model.num_keypoints, 3), np.float32)
        pre = [self.pre_img(im) for im in imgs]
        x = np.concatenate([p[0] for p in pre], 0)
        org = np.array([[p[2], p[1]] for p in pre], np.int32)
        out = []
        step = self.model.batch_limit
        for s in range(0, len(imgs), step):
            kp, _ = self.model.infer_host(x[s:s + step], org[s:s + step])
            out.append(kp)
        return np.concatenate(out, 0)


def frame_inference(self, img: np.ndarray) -> dict:
    """`VitInference.inference` (easy_ViTPose/inference.py:214-281) with the per-person loop (:258-272) replaced by one
    engine call on the frame; bound onto the reference object by `install(..., batched=True)`, so `self` is the
    reference's VitInference: its detector (`self.yolo`), SORT tracker, counters and `save_state` fields are used and
    updated exactly as the reference does, which keeps `draw()` (:283-312) and the CLI's JSON writer working.

    Detection cadence (:234-241): the detector runs when there is no tracker, on the first three frames, and every
    `yolo_step`-th frame; rows with confidence <= 0.35 are dropped.  Returns {id: float32 [K,3] (y, x, score)} in frame pixels."""
    detections = np.empty((0, 5))
    results = None
    if self.tracker is None or self.frame_counter < 3 or self.frame_counter % self.yolo_step == 0:
        results = self.yolo(img[..., ::-1], verbose=False, imgsz=self.yolo_size,
                            device=0 if self.device == "cuda" else self.device, classes=self.yolo_classes)[0]
        rows = np.asarray(results.boxes.data.cpu().numpy(), np.float64)
        rows = rows.reshape(-1, rows.shape[-1] if rows.ndim > 1 else 6)
        detections = rows[rows[:, 4] > 0.35, :5].reshape(-1, 5)
    self.frame_counter += 1

    ids = None
    if self.tracker is not None:
        detections = self.tracker.update(detections)
        ids = detections[:, 5].astype(int).tolist()
    bboxes = detections[:, :4].round().astype(int)
    scores = detections[:, 4].tolist()
    if ids is None:
        ids = list(range(len(bboxes)))

    kpts, _ = self._b200.model.infer_frame_host(img, bboxes)            # pad/clip, crop, pad_image, pre_img, model, decode, offsets
    smoother = getattr(self, "_smoother", None)
    if smoother is not None and self.tracker is not None:               # ids are track ids only where there is a tracker
        yx = smoother.update([kpts], [ids], clock=[time.time()] if smoother.realtime else None)[0]
        smoother.check()
        kpts[:, :, :2] = yx
    frame_keypoints = {i: kpts[n] for n, i in enumerate(ids)}
    scores_bbox = {i: sc for i, sc in zip(ids, scores)}

    if self.save_state:
        # the reference pads and clips `bboxes` in place inside its loop (:260-261), so draw() sees the padded boxes
        h, w = img.shape[:2]
        bboxes[:, [0, 2]] = np.clip(bboxes[:, [0, 2]] + [-10, 10], 0, w)
        bboxes[:, [1, 3]] = np.clip(bboxes[:, [1, 3]] + [-10, 10], 0, h)
        self._img = img
        self._yolo_res = results
        self._tracker_res = (bboxes, ids, scores)
        self._keypoints = frame_keypoints
        self._scores_bbox = scores_bbox
    return frame_keypoints


def frame_draw(self, show_yolo=True, show_raw_yolo=False, confidence_threshold=0.5) -> np.ndarray:
    """`VitInference.draw()` (easy_ViTPose/inference.py:283-312) with the pose layer drawn on the device: returns the same
    RGB array.  The box layers, when requested, run first with the reference's own code (ultralytics' `plot()` and
    `draw_bboxes`), as draw() orders them; then every person of `self._keypoints`, in its order and with its key as colour
    index, is drawn with `joints_dict()[self.dataset]['skeleton']` and the palettes draw() passes, in one
    `B200PoseBackend.draw_frames` call.  Bound onto the reference object by `install(..., batched=True)`."""
    import importlib
    img = self._img.copy()
    bboxes, ids, scores = self._tracker_res
    if self._yolo_res is not None and (show_raw_yolo or (self.tracker is None and show_yolo)):
        img = np.array(self._yolo_res.plot())[..., ::-1]
    if show_yolo and self.tracker is not None:
        img = importlib.import_module("easy_ViTPose.vit_utils.inference").draw_bboxes(img, bboxes, ids, scores)
    img = np.ascontiguousarray(img)
    if not self._keypoints:
        return img
    skeleton = importlib.import_module("easy_ViTPose.vit_utils.visualization").joints_dict()[self.dataset]["skeleton"]
    kpts = np.stack([np.asarray(k, np.float32) for k in self._keypoints.values()], 0)
    return self._b200.draw_frames([img], [kpts], skeleton, person_index=[list(self._keypoints.keys())],
                                  confidence_threshold=confidence_threshold)[0]


class DeviceTracker:
    """A one-stream track.DeviceSort behind the reference `Sort` interface: `.update(dets [n, 5])` returns the float64
    [m, 6] array Sort.update returns.  When the reference's sort module is loaded (`easy_ViTPose.sort`), every update starts
    from its `KalmanBoxTracker.count` and writes the next id back, so ids interleave with CPU Sort objects of the same
    process exactly as they do between reference Sorts."""

    def __init__(self, max_age: int = 1, min_hits: int = 3, iou_threshold: float = 0.3, device=None):
        from .track import DeviceSort
        self.max_age, self.min_hits, self.iou_threshold = max_age, min_hits, iou_threshold
        self.sort = DeviceSort(1, max_age, min_hits, iou_threshold, device)

    @staticmethod
    def _counter():
        import sys
        mod = sys.modules.get("easy_ViTPose.sort")
        return getattr(mod, "KalmanBoxTracker", None)

    def update(self, dets=np.empty((0, 5))) -> np.ndarray:
        kbt = self._counter()
        if kbt is not None:
            self.sort.next_id = int(kbt.count)
        rows = self.sort.update([dets])[0]
        self.sort.check()
        if kbt is not None:
            kbt.count = self.sort.next_id
        return rows


def _reference_reset(self):
    """`VitInference.reset()` (easy_ViTPose/inference.py:174-185) with the SORT tracker on the device: the same rule for
    whether there is a tracker and the same parameters.  Bound by `install(..., batched=True, device_tracker=True)`."""
    min_hits = 3 if self.yolo_step == 1 else 1
    use_tracker = self.is_video and not self.single_pose
    self.tracker = DeviceTracker(self.yolo_step, min_hits, 0.3, self._b200.model._device) if use_tracker else None
    self.frame_counter = 0


SMOOTHING_DEFAULTS = dict(min_cutoff=1.7, beta=0.3, d_cutoff=30.0, fps=None, dx0=0.0, max_gap=30)


def _reset_with_smoother(self):
    """The bound `reset()` followed by forgetting the keypoint filters.  Bound by `install(..., smoothing=...)`."""
    self._reset_before_smoothing()
    self._smoother.reset()


def install(vit_inference, max_batch: int = 64, device=None, batched: bool = False, flip_test: bool = False,
            flip_pairs=None, device_tracker: bool = False, smoothing=None) -> B200PoseBackend:
    """Re-bind a constructed reference `VitInference` (torch .pth backend) to the H100 engine: takes the
    weights out of its `_vit_pose` module, then replaces `_vit_pose` and `_inference` exactly where
    easy_ViTPose/inference.py:156-172 set them.  With `batched=True` the object's `inference` method is re-bound to
    `frame_inference` as well (one engine call per frame instead of one per person), and `draw` to `frame_draw` (the pose
    layer of every person in one launch on the device).  With `flip_test=True` every
    keypoint call runs the flip test of the reference configs (test_cfg flip_test=True, shift_heatmap=False), with the
    pairs of `flip_pairs_for(vit_inference.dataset, flip_pairs)`; the engine is then built for 2 * max_batch crops, so
    `max_batch` still counts people per call.  With `batched=True, device_tracker=True` the SORT tracker runs on the device
    too: `vit_inference.tracker` becomes a `DeviceTracker` with the reference's parameters (only where the reference builds a
    Sort) and `reset()` is re-bound to rebuild it.  With `batched=True, smoothing=dict(...)` every frame's keypoints are
    smoothed by track id with the reference's OneEuroFilter, one filter per id, on the device (a one-stream
    `smooth.DeviceOneEuro`; keys min_cutoff, beta, d_cutoff, fps, dx0, max_gap, defaults SMOOTHING_DEFAULTS, `{}` for all of
    them): the returned dict, `_keypoints` and so `draw()` hold the smoothed (y, x) and the engine's scores, with the CPU
    `Sort` or `device_tracker=True`.  Smoothing applies only where the reference has a tracker (video, not single_pose):
    without one the ids are positions in the frame, not people, and the keypoints are left as they are.  With fps=None
    (realtime) each frame's clock is time.time(), as the reference class reads it.  `reset()` also forgets the filters.
    Returns the backend (also stored as `._b200`)."""
    if device_tracker and not batched:
        raise ValueError("device_tracker=True needs batched=True")
    if smoothing is not None:
        if not batched:
            raise ValueError("smoothing needs batched=True")
        unknown = set(smoothing) - set(SMOOTHING_DEFAULTS)
        if unknown:
            raise ValueError(f"unknown smoothing parameters {sorted(unknown)}; expected some of {sorted(SMOOTHING_DEFAULTS)}")
        smoothing = {**SMOOTHING_DEFAULTS, **smoothing}
    pairs = flip_pairs_for(getattr(vit_inference, "dataset", None), flip_pairs) if flip_test else None
    ref = vit_inference._vit_pose
    sd = {k: v.detach().cpu() for k, v in ref.state_dict().items()}
    D = sd["backbone.pos_embed"].shape[2]
    depth = 1 + max(int(k.split(".")[2]) for k in sd if k.startswith("backbone.blocks."))
    heads = int(ref.backbone.blocks[0].attn.num_heads)
    K = sd["keypoint_head.final_layer.weight"].shape[0]
    cfg = model_cfg({384: "s", 768: "b", 1024: "l", 1280: "h"}[D], K)
    cfg["backbone"].update(embed_dim=D, depth=depth, num_heads=heads)
    model = ViTPose(cfg, max_batch=2 * max_batch if flip_test else max_batch)
    model.load_state_dict(sd)
    backend = B200PoseBackend(model, device if device is not None else "cuda")
    if flip_test:
        model.set_flip_test(pairs)
    vit_inference._vit_pose = model
    vit_inference._inference = backend._inference
    vit_inference.postprocess = types.MethodType(lambda self, hm, w, h: backend.postprocess(hm, w, h), vit_inference)
    vit_inference._b200 = backend
    if batched:
        vit_inference.inference = types.MethodType(frame_inference, vit_inference)
        vit_inference.draw = types.MethodType(frame_draw, vit_inference)
    if device_tracker:
        vit_inference.reset = types.MethodType(_reference_reset, vit_inference)
        if vit_inference.tracker is not None:
            vit_inference.tracker = DeviceTracker(vit_inference.tracker.max_age, vit_inference.tracker.min_hits,
                                                  vit_inference.tracker.iou_threshold, model._device)
    if smoothing is not None:
        from .smooth import DeviceOneEuro
        vit_inference._smoother = DeviceOneEuro(1, K, device=model._device, **smoothing)
        vit_inference._reset_before_smoothing = vit_inference.reset
        vit_inference.reset = types.MethodType(_reset_with_smoother, vit_inference)
    return backend
