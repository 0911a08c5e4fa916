"""Batch sharding across the GPUs of one box (one process per GPU, torch.distributed / NCCL as plumbing).

The path shards by image (SURVEY.md section 8e): letterbox, convs and NMS are per-image independent, weights are
replicated, and the ONLY exchange is one all-gather of the final padded detections when a single output list is
required.  One subtlety is reproduced: the reference pads every image to the batch-wide canvas
(yolort/models/transform.py:307-314) and rescales boxes with it (yolov5.py:179-181), so every rank letterboxes
its shard to the GLOBAL (Hb, Wb), computed on the host from the image sizes alone -- no collective needed.
"""
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.distributed as dist
from torch import Tensor

from . import _C


def shard_bounds(n_items: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous chunk [lo, hi) of `n_items` owned by `rank`; sizes differ by at most one, earlier ranks larger."""
    base, extra = divmod(n_items, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def global_canvas(sizes: Sequence[Tuple[int, int]], min_size: float, max_size: float, size_divisible: int = 32,
                  fixed_shape: Optional[Tuple[int, int]] = None) -> Tuple[int, int]:
    """(Hb, Wb) of the whole (unsharded) batch; host arithmetic only."""
    _, hw = _C.letterbox_geometry(list(sizes), float(min_size), float(max_size), size_divisible, fixed_shape)
    return hw


def pack_detections(boxes: Tensor, scores: Tensor, labels: Tensor, counts: Optional[Tensor] = None) -> Tensor:
    """[n, D(+1), 6] fp32 rows (x1, y1, x2, y2, score, label) -- the all-gather payload (24 B per detection slot).
    Labels < 2^24 are exact in fp32.  With `counts`, one more row per image carries the detection count in column 0, so
    a single collective moves everything."""
    packed = torch.cat([boxes, scores.unsqueeze(-1), labels.to(torch.float32).unsqueeze(-1)], dim=-1)
    if counts is not None:
        tail = packed.new_zeros((packed.shape[0], 1, 6))
        tail[:, 0, 0] = counts.to(torch.float32)
        packed = torch.cat([packed, tail], dim=1)
    return packed.contiguous()


class DetectionGather:
    """The per-step exchange of a data-parallel serving loop, kept off the compute stream: packing the padded outputs of
    `forward_padded` into the [n, D+1, 6] payload (half a dozen small element-wise launches) and the ONE NCCL all-gather
    both run on a side stream, so the next step's letterbox / convolutions start right after the NMS kernel.

        g = DetectionGather(device)
        for batch in batches:
            g.before_step()                       # the previous pack has finished reading the (reused) output buffers
            out = model.forward_padded(batch)
            gathered = g.launch(out)              # [world, n, D+1, 6]; valid after g.wait() / a stream sync
        g.wait()
    """

    def __init__(self, device: torch.device, group=None):
        self.device, self.group = device, group
        self.world = dist.get_world_size(group)
        self.stream = torch.cuda.Stream(device)
        self._pack_done: Optional[torch.cuda.Event] = None

    def before_step(self) -> None:
        if self._pack_done is not None:
            torch.cuda.current_stream(self.device).wait_event(self._pack_done)

    def launch(self, out) -> Tensor:
        boxes, scores, labels, counts = out[:4]
        self.stream.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(self.stream):
            packed = pack_detections(boxes, scores, labels, counts)
            self._pack_done = torch.cuda.Event()
            self._pack_done.record(self.stream)
            gathered = torch.empty((self.world,) + tuple(packed.shape), dtype=packed.dtype, device=self.device)
            dist.all_gather_into_tensor(gathered, packed, group=self.group)
        return gathered

    def wait(self) -> None:
        torch.cuda.current_stream(self.device).wait_stream(self.stream)


def unpack_detections(packed: Tensor, counts: Tensor) -> List[Dict[str, Tensor]]:
    out = []
    host_counts = counts.to("cpu", torch.int64).tolist()
    for i, c in enumerate(host_counts):
        row = packed[i, :c]
        out.append({"scores": row[:, 4], "labels": row[:, 5].to(torch.int64), "boxes": row[:, :4]})
    return out


def all_gather_detections(packed: Tensor, counts: Tensor, shard_sizes: Sequence[int], group=None) -> Tuple[Tensor, Tensor]:
    """ONE collective over equal-sized buffers: shards are padded to the largest shard and the counts ride in an extra
    row of the payload, so that a single all_gather_into_tensor (NCCL all-gather over NVLink) moves everything;
    returns ([N_total, D, 6], [N_total])."""
    world = dist.get_world_size(group)
    n_max = max(shard_sizes)
    D = packed.shape[1]
    send = packed.new_zeros((n_max, D + 1, 6))
    send[: packed.shape[0], :D] = packed
    send[: counts.shape[0], D, 0] = counts.to(torch.float32)
    recv = packed.new_empty((world * n_max, D + 1, 6))
    dist.all_gather_into_tensor(recv, send, group=group)
    keep = torch.cat([torch.arange(r * n_max, r * n_max + s) for r, s in enumerate(shard_sizes)]).to(recv.device)
    sel = recv[keep]
    return sel[:, :D], sel[:, D, 0].to(torch.int32)


def forward_padded_grow(model, images: List[Tensor], canvas: Tuple[int, int], max_tries: int = 8):
    """`forward_padded` on the shard-local images letterboxed to the GLOBAL canvas, re-run with a larger candidate
    arena until no image overflowed its share (status[1] == 0): nothing is ever truncated or dropped silently.  The
    growth uses the same canvas as the run that overflowed (candidate counts depend on it); a plan whose fused-decode
    arena is fixed falls back to the stored-logits path, whose arena grows."""
    dev = next(model.parameters()).device
    for _ in range(max_tries):
        out = model.forward_padded(images, batch_hw=canvas)
        st = out[4].cpu().tolist()
        if int(st[1]) == 0:
            return out
        arena = _C._arenas.setdefault(dev, _C._NmsArena())
        arena.cap_per_image = max(2 * arena.cap_per_image, int(st[2]))
        arena.ws = None
        plan = model.model.get_plan(len(images), canvas[0], canvas[1])
        if plan.fused_post is not None:      # fixed arena inside the plan: use the growable stand-alone decode
            plan.fused_post = None
    raise _C.NativeLibraryError(f"predict_sharded: candidate arena still overflows after {max_tries} growth steps "
                                f"(needs {int(st[2])} candidates per image)")


def predict_sharded(model, images: List[Tensor], group=None) -> List[Dict[str, Tensor]]:
    """Every rank passes the SAME full list of images (host tensors or tensors on its device); each rank runs
    its contiguous shard on its own GPU and all ranks return the full, ordered detection list."""
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    tr = model.transform
    sizes = [(int(im.shape[-2]), int(im.shape[-1])) for im in images]
    canvas = global_canvas(sizes, tr.min_size, tr.max_size, tr.size_divisible, tr.fixed_shape)
    bounds = [shard_bounds(len(images), r, world) for r in range(world)]
    lo, hi = bounds[rank]
    p = next(model.parameters())
    D = model.model.post_process.detections_per_img
    if hi > lo:
        mine = model.collate_images(images[lo:hi], None)
        boxes, scores, labels, counts, status = forward_padded_grow(model, mine, canvas)
        packed = pack_detections(boxes, scores, labels)
    else:
        packed = torch.zeros((0, D, 6), dtype=torch.float32, device=p.device)
        counts = torch.zeros((0,), dtype=torch.int32, device=p.device)
    all_packed, all_counts = all_gather_detections(packed, counts, [b[1] - b[0] for b in bounds], group)
    return unpack_detections(all_packed, all_counts)
