"""Crop sharding across GPUs: one process per GPU, weights replicated, crops split by index, the only exchange is
the gather of the final keypoint tensors (SURVEY.md section 8e).  The reference has no multi-GPU inference path
(its torch.distributed use is training-only, vit_utils/dist_util.py); this is the data-parallel form its README
lists as future work ("parallel batched inference", README.md:323).

Backend-agnostic host logic (nccl on GPUs, gloo on CPU in the tests): torch.distributed does the plumbing.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

__all__ = ["shard_counts", "shard_range", "gather_keypoints", "infer_sharded", "infer_frame_sharded", "ShardPipeline"]


def shard_counts(n: int, world: int) -> list[int]:
    """Crops per rank: contiguous blocks, the remainder goes to the lowest ranks."""
    base, rem = divmod(n, world)
    return [base + (1 if r < rem else 0) for r in range(world)]


def shard_range(n: int, rank: int, world: int) -> tuple[int, int]:
    counts = shard_counts(n, world)
    lo = sum(counts[:rank])
    return lo, lo + counts[rank]


def gather_keypoints(local: torch.Tensor, n_total: int, group=None) -> torch.Tensor:
    """local [n_local, K, C] on every rank (n_local = shard_counts(n_total, world)[rank]) -> [n_total, K, C] on every
    rank, in crop order.  Equal shards take one all_gather_into_tensor; ragged ones are padded to the largest shard."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    counts = shard_counts(n_total, world)
    if local.shape[0] != counts[rank]:
        raise ValueError(f"rank {rank} holds {local.shape[0]} crops, expected {counts[rank]}")
    tail = tuple(local.shape[1:])
    if len(set(counts)) == 1:
        out = torch.empty((n_total,) + tail, dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(out, local.contiguous(), group=group)
        return out
    cmax = max(counts)
    padded = torch.zeros((cmax,) + tail, dtype=local.dtype, device=local.device)
    padded[: local.shape[0]] = local
    buf = torch.empty((world * cmax,) + tail, dtype=local.dtype, device=local.device)
    dist.all_gather_into_tensor(buf, padded, group=group)
    return torch.cat([buf[r * cmax: r * cmax + counts[r]] for r in range(world)], 0)


@torch.no_grad()
def infer_sharded(model, crops: torch.Tensor, org_wh: torch.Tensor, group=None):
    """Every rank passes the SAME global batch (crops [N,3,256,192], org_wh [N,2]); each runs its own slice through its
    engine and all ranks return the full keypoints [N,K,3] and argmax [N,K]."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n = crops.shape[0]
    lo, hi = shard_range(n, rank, world)
    step = getattr(model, "batch_limit", model.max_batch)      # max_batch // 2 with flip test on
    outs_kp, outs_idx = [], []
    for s in range(lo, hi, step):
        e = min(hi, s + step)
        kp, idx = model.infer_crops(crops[s:e], org_wh[s:e])
        outs_kp.append(kp)
        outs_idx.append(idx)
    if outs_kp:
        kp, idx = torch.cat(outs_kp, 0), torch.cat(outs_idx, 0)
    else:   # more ranks than crops
        dev = torch.device("cuda", torch.cuda.current_device())
        kp = torch.empty((0, model.num_keypoints, 3), dtype=torch.float32, device=dev)
        idx = torch.empty((0, model.num_keypoints), dtype=torch.int32, device=dev)
    return gather_keypoints(kp, n, group), gather_keypoints(idx.unsqueeze(-1), n, group).squeeze(-1)


@torch.no_grad()
def infer_frame_sharded(model, frame: torch.Tensor, bboxes: torch.Tensor, group=None):
    """Frame-level form (SURVEY.md section 8 rows f1/f2 + e): every rank holds the SAME uint8 frame [H,W,3] and the SAME boxes
    [n,4]; the people of the frame are sharded by index, each rank runs its slice through `model.infer_frame` (crop
    pre-processing, model, decode, offsets back to frame pixels on its GPU) and all ranks return the full frame-space
    keypoints [n,K,3] and argmax [n,K] in box order.  The only exchange is the keypoint gather."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    n = bboxes.shape[0]
    lo, hi = shard_range(n, rank, world)
    outs_kp, outs_idx = [], []
    step = getattr(model, "batch_limit", model.max_batch)
    for s in range(lo, hi, step):
        kp, idx = model.infer_frame(frame, bboxes[s:min(hi, s + step)])
        outs_kp.append(kp)
        outs_idx.append(idx)
    if outs_kp:
        kp, idx = torch.cat(outs_kp, 0), torch.cat(outs_idx, 0)
    else:   # more ranks than people
        kp = torch.empty((0, model.num_keypoints, 3), dtype=torch.float32, device=frame.device)
        idx = torch.empty((0, model.num_keypoints), dtype=torch.int32, device=frame.device)
    return gather_keypoints(kp, n, group), gather_keypoints(idx.unsqueeze(-1), n, group).squeeze(-1)


class ShardPipeline:
    """Host crops in -> gathered host keypoints out, `depth` batches in flight per rank (one process per GPU).

    Per submit(): H2D of this rank's pinned crops on a copy stream, the engine on a compute stream, the only exchange of the
    path -- an all_gather of the [B,K,3] keypoints -- on a third stream, then the D2H of the gathered tensor into pinned
    memory.  Nothing blocks the host until wait(); the gather and the copies of batch i run under the compute of batch i+1.
    With world size 1 (or torch.distributed not initialised) the gather is skipped.  Every rank must call submit()/wait()
    the same number of times with the same batch size (the collective is symmetric)."""

    def __init__(self, model, batch: int, depth: int = 2, group=None):
        dev = torch.device("cuda", torch.cuda.current_device())
        self.model, self.batch, self.depth, self.group = model, batch, depth, group
        self.world = dist.get_world_size(group) if dist.is_available() and dist.is_initialized() else 1
        K = model.num_keypoints
        self.s_copy, self.s_comp, self.s_comm = (torch.cuda.Stream(dev) for _ in range(3))
        self.x = [torch.empty((batch, 3, 256, 192), dtype=torch.float32, device=dev) for _ in range(depth)]
        self.org = [torch.empty((batch, 2), dtype=torch.int32, device=dev) for _ in range(depth)]
        self.kp = [torch.empty((batch, K, 3), dtype=torch.float32, device=dev) for _ in range(depth)]
        self.full = [torch.empty((self.world * batch, K, 3), dtype=torch.float32, device=dev) for _ in range(depth)]
        self.host = [torch.empty((self.world * batch, K, 3), dtype=torch.float32).pin_memory() for _ in range(depth)]
        self.ev_h2d = [torch.cuda.Event() for _ in range(depth)]
        self.ev_comp = [torch.cuda.Event() for _ in range(depth)]
        self.ev_done = [torch.cuda.Event() for _ in range(depth)]
        self.used = [False] * depth

    @torch.no_grad()
    def submit(self, slot: int, h_crops: torch.Tensor, h_org_wh: torch.Tensor) -> None:
        """h_crops float32 [B,3,256,192] and h_org_wh int32 [B,2] on the host (pinned for real overlap); they must stay
        unmodified until wait(slot)."""
        if self.used[slot]:
            self.s_copy.wait_event(self.ev_comp[slot])       # the slot's device inputs are free once its compute is done
        with torch.cuda.stream(self.s_copy):
            self.x[slot].copy_(h_crops, non_blocking=True)
            self.org[slot].copy_(h_org_wh, non_blocking=True)
            self.ev_h2d[slot].record(self.s_copy)
        with torch.cuda.stream(self.s_comp):
            self.s_comp.wait_event(self.ev_h2d[slot])
            if self.used[slot]:
                self.s_comp.wait_event(self.ev_done[slot])   # kp[slot] was read by the previous gather
            kp, _ = self.model.infer_crops(self.x[slot], self.org[slot])
            self.kp[slot].copy_(kp)
            self.ev_comp[slot].record(self.s_comp)
        with torch.cuda.stream(self.s_comm):
            self.s_comm.wait_event(self.ev_comp[slot])
            if self.world > 1:
                dist.all_gather_into_tensor(self.full[slot], self.kp[slot], group=self.group)
                self.host[slot].copy_(self.full[slot], non_blocking=True)
            else:
                self.host[slot].copy_(self.kp[slot], non_blocking=True)
            self.ev_done[slot].record(self.s_comm)
        self.used[slot] = True

    def wait(self, slot: int) -> torch.Tensor:
        """Blocks until slot's gathered keypoints [world*B,K,3] are in pinned host memory; the tensor is reused by the
        slot's next submit()."""
        self.ev_done[slot].synchronize()
        return self.host[slot]
