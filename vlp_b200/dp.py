"""Data-parallel gradient all-reduce for the VLP hot path (SURVEY.md §8e / a19: the path shards by batch; the one collective
is the mean of all gradients per step — `DistributedDataParallel` in the reference, vlp/run_img2txt_dist.py:386).

torch DDP works unchanged on vlp_b200 modules.  This module is the H100-first alternative used by bench.py: the fused
encoder backward already produces each layer group's gradients as ONE contiguous bf16 arena, so the arena itself is handed to
NCCL (`all_reduce`, AVG, asynchronously, the moment the group's backward finishes) while earlier groups are still computing —
no per-parameter bucket copies, no autograd hooks, no graph walk for unused parameters.

What is exposed after backward is only what becomes available last: the arena of the lowest layer group (made ONE layer: group
sizes 1,2,3,3,3 from layer 0 up) and the gradients outside the encoder, reduced in place, tensor by tensor for the large ones (no
flatten / copy-back passes) and as one small flat buffer for the rest, all asynchronous and waited for once.  The largest single
gradient, the [28996,768] word-embedding table tied to the MLM decoder, is one of those large tensors: autograd completes it only when
the embedding lookup's backward, the last of the step, has added its rows to the decoder's contribution.

Contract: gradients are reduced once per backward.  With gradient accumulation (`p.grad` already populated when backward runs) the
arena's in-flight all-reduce would race autograd's `p.grad += arena_view`; that case is detected and the collective is awaited
before the views are handed to autograd (correct, no overlap for those steps).
"""
import os

import torch
import torch.distributed as dist

from . import _lib as L

DEFAULT_GROUPS = (1, 2, 3, 3, 3)
SMALL = 1 << 20          # elements: tensors below this are reduced through one flat buffer


class GradientAllReducer:
    def __init__(self, model, group=None, layer_groups=None, reserved_sms=None):
        """layer_groups: encoder layers per backward call / all-reduce arena, from layer 0 up (default 1,2,3,3,3 scaled to the depth; env
        VLP_DP_GROUPS="a,b,..." overrides).  reserved_sms (default 8, measured +1.8 % at 2 GPUs / env VLP_DP_RESERVED_SMS): while an arena all-reduce is in
        flight the persistent GEMM grids launched after it leave that many SMs to NCCL's CTAs (vlpk_set_reserved_sms)."""
        self.reserved_sms = int(os.environ.get("VLP_DP_RESERVED_SMS", "8")) if reserved_sms is None else int(reserved_sms)
        self.group = group
        self.world = dist.get_world_size(group)
        self.model = model
        self.backend = dist.get_backend(group)
        self.enabled = True                       # False: hooks and finish() do nothing (bench.py measures the step without communication)
        enc = model.bert.encoder
        n = len(enc.layer)
        env = os.environ.get("VLP_DP_GROUPS")
        if env:
            layer_groups = [int(k) for k in env.split(",")]
        if layer_groups is None:
            layer_groups = list(DEFAULT_GROUPS) if n == sum(DEFAULT_GROUPS) else [1] * min(n, 1) + [min(3, n - 1 - s) for s in range(0, max(n - 1, 0), 3)]
            layer_groups = [k for k in layer_groups if k > 0]
        if isinstance(layer_groups, int):
            layer_groups = [min(layer_groups, n - s) for s in range(0, n, layer_groups)]
        if sum(layer_groups) != n:
            raise ValueError(f"layer_groups={layer_groups} must sum to the {n} encoder layers")
        self._saved = (enc.layers_per_call, enc._vlpk_grad_hook)
        enc.layers_per_call = list(layer_groups)
        enc._vlpk_grad_hook = self._on_encoder_grads
        self.enc_params = list(enc.parameters())
        enc_ids = {id(p) for p in self.enc_params}
        self.other = [p for p in model.parameters() if p.requires_grad and id(p) not in enc_ids]
        self._works = []
        self._accumulating = None

    # -- context manager: restores the encoder's previous grouping / hook -------------------------------------------------------
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def close(self):
        enc = self.model.bert.encoder
        if enc._vlpk_grad_hook == self._on_encoder_grads:
            enc.layers_per_call, enc._vlpk_grad_hook = self._saved

    def broadcast_parameters(self, src=0):
        for p in self.model.parameters():
            dist.broadcast(p.data, src=src, group=self.group)

    def _reduce(self, t, async_op):
        if self.backend == "nccl":
            return dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group, async_op=async_op)
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=self.group, async_op=False)   # gloo: no AVG, synchronous
        t.div_(self.world)
        return None

    def _on_encoder_grads(self, arena):
        """Called by EncoderStackFn.backward with the flat gradient arena of one layer group (views of it become .grad)."""
        if not self.enabled:
            return
        if self._accumulating is None:            # once per backward: is autograd going to ADD these views to existing gradients?
            self._accumulating = any(p.grad is not None for p in self.enc_params)
        w = self._reduce(arena, async_op=True)
        if w is not None:
            if self._accumulating:
                w.wait()                          # the reduced values must be in place before autograd's `p.grad += view`
            elif arena.dtype != torch.bfloat16:
                # a group with non-bf16 parameters hands over its fp32 arena, and EncoderStackFn.backward converts the views of the
                # bf16 parameters right after this hook returns, on the current stream: that conversion must read reduced values,
                # so the stream waits for the collective here (no overlap for such groups)
                w.wait()
            else:
                self._works.append(w)
        if self.reserved_sms > 0:
            L.lib().vlpk_set_reserved_sms(self.reserved_sms)

    def finish(self):
        """After loss.backward(): reduce the non-encoder gradients and wait for everything in flight."""
        if not self.enabled:
            return
        grads = [p.grad for p in self.other if p.grad is not None]
        big = [g for g in grads if g.numel() >= SMALL and g.is_contiguous()]
        small = [g for g in grads if not (g.numel() >= SMALL and g.is_contiguous())]
        for g in big:                             # in place, no staging copies
            w = self._reduce(g, async_op=True)
            if w is not None:
                self._works.append(w)
        if small:
            flat = torch._utils._flatten_dense_tensors(small)
            w = self._reduce(flat, async_op=True)
            if w is not None:
                w.wait()
            for g, r in zip(small, torch._utils._unflatten_dense_tensors(flat, small)):
                g.copy_(r)
        for w in self._works:
            w.wait()
        self._works.clear()
        self._accumulating = None
        if self.reserved_sms > 0:
            L.lib().vlpk_set_reserved_sms(0)
