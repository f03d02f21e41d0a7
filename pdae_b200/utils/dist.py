"""Data-parallel plumbing of the sampling path: contiguous batch shards, one all-gather of results.

The hot path shards over independent images (SURVEY.md section 8e): no collective inside the DDIM loop; the reference
collects results with ``all_gather_object`` of ``.tolist()``-ed images (trainer/base_trainer.py:156-159,
sampler/base_sampler.py:53-56) -- here it is ONE tensor all-gather (NCCL on GPUs, gloo in the CPU tests).
"""
from __future__ import annotations

from typing import List, Tuple

import torch
import torch.distributed as dist


def shard_range(n: int, rank: int, world: int) -> Tuple[int, int]:
    """[start, end) of rank's contiguous shard; like dispatch_num_samples_for_process (sampler/base_sampler.py:40-50)
    every rank gets n // world items and the LAST rank also takes the remainder."""
    per = n // world
    start = rank * per
    end = n if rank == world - 1 else start + per
    return start, end


def all_gather_images(local: torch.Tensor, n_total: int) -> torch.Tensor:
    """Gather per-rank shards (possibly ragged: the last rank may hold the remainder) into [n_total, ...] on every rank
    with a single equal-count all-gather (shards are padded to the largest count)."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return local
    world, rank = dist.get_world_size(), dist.get_rank()
    counts = [shard_range(n_total, r, world) for r in range(world)]
    cmax = max(e - s for s, e in counts)
    pad = local
    if local.shape[0] < cmax:
        pad = torch.cat([local, local.new_zeros((cmax - local.shape[0],) + tuple(local.shape[1:]))], 0)
    out = local.new_empty((world * cmax,) + tuple(local.shape[1:]))
    dist.all_gather_into_tensor(out, pad.contiguous())
    parts: List[torch.Tensor] = [out[r * cmax: r * cmax + (e - s)] for r, (s, e) in enumerate(counts)]
    return torch.cat(parts, 0)


def sharded_autoencode(gd, encoder, decoder, x0_all: torch.Tensor, enc_style: str = "ddim100", dec_style: str = "ddim100",
                       device=None, as_uint8: bool = False) -> torch.Tensor:
    """Autoencode a global batch: every rank runs the hot path on its shard, then one all-gather.
    as_uint8: convert each shard to the reference's wire format first (uint8 NHWC,
    trainer/train_representation_learning.py:173-174) so the gather moves 4x fewer bytes.
    Under torch.use_deterministic_algorithms(True) the deterministic plans are batch-invariant, so the result is bitwise what
    one process returns for the whole of x0_all, whatever the world size."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    s, e = shard_range(x0_all.shape[0], rank, world)
    x = x0_all[s:e]
    if device is not None:
        x = x.to(device)
    if e == s:   # fewer images than ranks: shard_range gives everything to the last rank -- nothing to run here
        rec = x.new_empty((0,) + tuple(x0_all.shape[1:]), dtype=torch.float32)
    else:
        rec = gd.representation_learning_autoencoding(enc_style, dec_style, encoder, decoder, x)
    if as_uint8:
        from ..metric import images_to_uint8
        if rec.shape[0]:
            rec = images_to_uint8(rec)
        else:
            rec = rec.new_empty((0, rec.shape[2], rec.shape[3], rec.shape[1]), dtype=torch.uint8)
    return all_gather_images(rec, x0_all.shape[0])


def allreduce_grads_(params, bucket_bytes: int = 32 << 20) -> float:
    """DDP-equivalent gradient exchange for the trainable parameters (encoder + label_emb, shift_middle_block,
    shift_output_blocks, shift_out; trainer/train_representation_learning.py:44-49 wraps them in DDP): SUM all-reduce of
    every `.grad` in flat buckets, issued asynchronously so bucket k's collective overlaps bucket k+1's packing.
    Returns the factor the caller must fold into the optimizer (`FusedAdamEMA.step(grad_scale=...)`) = 1 / world_size
    -- the mean is never materialised as a separate pass over the gradients."""
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return 1.0
    grads = [p.grad for p in params if p.grad is not None]
    buckets: List[List[torch.Tensor]] = []
    cur: List[torch.Tensor] = []
    size = 0
    for g in grads:
        nb = g.numel() * g.element_size()
        if cur and (size + nb > bucket_bytes or g.dtype != cur[0].dtype):
            buckets.append(cur)
            cur, size = [], 0
        cur.append(g)
        size += nb
    if cur:
        buckets.append(cur)
    pending = []
    for bk in buckets:
        flat = torch.cat([g.reshape(-1) for g in bk])
        pending.append((dist.all_reduce(flat, op=dist.ReduceOp.SUM, async_op=True), flat, bk))
    for work, flat, bk in pending:
        work.wait()
        off = 0
        for g in bk:
            g.copy_(flat[off: off + g.numel()].view_as(g))
            off += g.numel()
    return 1.0 / dist.get_world_size()


class OverlappedGradAllReduce:
    """DDP-equivalent gradient exchange that OVERLAPS with the backward pass (trainer/train_representation_learning.py:29,39
    wraps encoder and decoder in DistributedDataParallel).  Parameters are grouped in the order their gradients become
    ready: the hand-written ShiftUNet backward delivers every decoder gradient at once, then dz flows into the encoder's
    backward -- so the decoder bucket's SUM all-reduce is launched (async, on the process group's own stream) from a
    post-accumulate-grad hook the moment the decoder gradients land and runs while the encoder backward computes.
    `finish()` waits, scatters the reduced values back into `.grad` and returns 1/world for the optimizer to fold in
    (`FusedAdamEMA.step(grad_scale=...)`) -- the mean is never a separate pass."""

    def __init__(self, groups, bucket_bytes: int = 64 << 20):
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.buckets = []          # [params, flat buffer or None, pending count]
        for params in groups:
            cur, size = [], 0
            for p in params:
                if not p.requires_grad:
                    continue
                nb = p.numel() * p.element_size()
                if cur and size + nb > bucket_bytes:
                    self.buckets.append({"params": cur})
                    cur, size = [], 0
                cur.append(p)
                size += nb
            if cur:
                self.buckets.append({"params": cur})
        self._of = {}
        self.handles = []
        for bi, bk in enumerate(self.buckets):
            bk["left"] = len(bk["params"])
            bk["flat"] = None
            for p in bk["params"]:
                self._of[p] = bi
                self.handles.append(p.register_post_accumulate_grad_hook(self._hook))
        self.pending = []

    def _hook(self, p):
        bk = self.buckets[self._of[p]]
        bk["left"] -= 1
        if bk["left"] == 0:
            self._launch(bk)

    def _launch(self, bk):
        if self.world == 1:
            return
        grads = [p.grad for p in bk["params"]]
        n = sum(g.numel() for g in grads)
        if bk["flat"] is None or bk["flat"].numel() != n or bk["flat"].device != grads[0].device:
            bk["flat"] = torch.empty(n, dtype=grads[0].dtype, device=grads[0].device)
        off = 0
        for g in grads:
            bk["flat"][off: off + g.numel()].copy_(g.reshape(-1))
            off += g.numel()
        self.pending.append((dist.all_reduce(bk["flat"], op=dist.ReduceOp.SUM, async_op=True), bk))

    def finish(self) -> float:
        """Call after loss.backward(): waits for every collective and writes the sums back into `.grad`."""
        for work, bk in self.pending:
            work.wait()
            off = 0
            for p in bk["params"]:
                n = p.grad.numel()
                p.grad.copy_(bk["flat"][off: off + n].view_as(p.grad))
                off += n
        self.pending = []
        for bk in self.buckets:
            if bk["left"] != 0 and self.world > 1 and any(p.grad is not None for p in bk["params"]):
                raise RuntimeError("OverlappedGradAllReduce: a bucket received gradients for only some of its parameters; "
                                   "group parameters that are trained together")
            bk["left"] = len(bk["params"])
        return 1.0 / self.world

    def remove(self):
        for h in self.handles:
            h.remove()
        self.handles = []
