# -*- coding: utf-8 -*-
"""Data-parallel plumbing: one process per GPU, NCCL over NVLink.

The reference trains with single-process ``nn.DataParallel`` (bin/train.py:449-454: scatter batch,
replicate params, gather logits on GPU 0, reduce grads).  This build shards the minibatch across
ranks instead; the only exchange on the data path is ONE flat all-reduce of the gradients per step
(8.6 MB fp32 at 64/512).  Each rank computes the mean loss over its own windows, so averaging the
gradients reproduces DataParallel's global mean for equal per-rank batches (SURVEY.md 8e).
Decode needs no collective at all: utterances are split like ``np.array_split`` (bin/decode.py:261).
"""
import numpy as np
import torch
import torch.distributed as dist


class GradAllReduce(object):
    """Average ``.grad`` of every parameter across ranks with a single flat all-reduce."""

    def __init__(self, module, group=None):
        self.module = module
        self.params = [p for p in module.parameters() if p.requires_grad]
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self._flat = None
        if self.world > 1:
            # start from identical weights on every rank (DataParallel replicates rank-0 params)
            for p in self.params:
                dist.broadcast(p.data, src=0, group=group)

    def allreduce(self):
        if self.world == 1:
            return
        live = [p for p in self.params if p.grad is not None]
        flat = getattr(self.module, "_wnb_flat_grad", None)
        if flat is not None and live:
            # the stack path hands autograd views of ONE flat buffer (nets/wavenet.py _StackTrainFn): when every .grad
            # still aliases it, that buffer is the all-reduce message -- no pack / unpack copies, no separate divide
            lo, hi = flat.data_ptr(), flat.data_ptr() + flat.numel() * flat.element_size()
            if all(lo <= p.grad.data_ptr() < hi for p in live):
                dist.all_reduce(flat, op=dist.ReduceOp.AVG, group=self.group)
                return
        n = sum(p.grad.numel() for p in live)
        if self._flat is None or self._flat.numel() != n or self._flat.device != live[0].grad.device:
            self._flat = torch.empty(n, dtype=live[0].grad.dtype, device=live[0].grad.device)
        views, off = [], 0
        for p in live:
            k = p.grad.numel()
            views.append(self._flat[off:off + k].view_as(p.grad))
            off += k
        torch._foreach_copy_(views, [p.grad for p in live])
        dist.all_reduce(self._flat, op=dist.ReduceOp.SUM, group=self.group)
        self._flat.div_(self.world)
        torch._foreach_copy_([p.grad for p in live], views)


def shard_utterances(items, world, rank):
    """bin/decode.py:261-262: ``np.array_split(feat_list, n_gpus)`` -> this rank's slice (order kept)."""
    parts = np.array_split(np.arange(len(items)), world)
    return [items[i] for i in parts[rank]]


def gather_scores(nll, count, group=None):
    """Per-utterance held-out scores (``utils.scoring``) of every rank, concatenated in rank order on every rank.  Each
    rank scored its ``shard_utterances`` share of one list, so the result is in list order and its ``corpus_mean`` is
    bit-identical to scoring the whole list in one process.  Without a process group, returns the arguments."""
    nll, count = np.asarray(nll, dtype=np.float64), np.asarray(count, dtype=np.int64)
    if not dist.is_initialized():
        return nll, count
    parts = [None] * dist.get_world_size(group)
    dist.all_gather_object(parts, (nll, count), group=group)
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
