"""Whole-step CUDA-graph replay of the VLP training step (forward + backward through the module surface).

The fused hot path issues ~330 kernel launches per step (12 x BertLayer forward/backward, region projections, embeddings, heads);
driven from Python — torch modules, autograd Functions, ctypes calls — the host needs several milliseconds per step to enqueue them,
so every hiccup (GC, loader work, H2D bookkeeping) can stall the GPU.  `GraphedStep` captures the launch sequence of one step once and
replays it:

    gstep = GraphedStep(model, example_batch, step)      # step(model, batch) -> loss ; must call loss.backward() itself
    for batch in loader:                                  # batch: dict of CUDA tensors (e.g. from staging.BatchStager.get())
        loss = gstep(batch)                               # copies the batch into the captured input buffers, replays the graph
        optimizer.step()                                  # p.grad are the captured (static) gradient tensors, rewritten by each replay

Everything the step launches — libvlpk kernels on the caller's stream and on the library's side stream, programmatic dependent
launches, torch's head / loss kernels, memsets — is captured as is; no kernel is different from the eager path.  Dropout masks stay
fresh because every kernel adds a device-side counter (`ops.set_device_seed_tensor`) to its Philox seed, which is bumped before each
replay.  Shapes are frozen: a batch of another shape needs its own GraphedStep.

Constraints (checked or documented): all parameters' `.grad` are produced by the graph (zero_grad(set_to_none=True) semantics — gradient
accumulation across replays needs an explicit add outside the graph); `step` must not synchronise with the host (no `.item()`).
Data parallelism: `step` may include `dp.GradientAllReducer.finish()` — the arena all-reduces issued from the backward hooks and the
tail reductions are NCCL kernels on torch.distributed's streams and are captured with their stream dependencies like everything
else (every rank must capture and replay in lock-step; pass capture_error_mode="thread_local").
"""
import torch

from . import _lib as L
from . import ops
from .staging import PackedAttentionMask


class GraphedStep:
    def __init__(self, model, example_batch, step, warmup=3, capture_error_mode="global"):
        """capture_error_mode: passed to torch.cuda.graph; use "thread_local" when other threads issue CUDA calls during the capture
        (torch.distributed's NCCL watchdog polling earlier collectives)."""
        self.model = model
        dev = next(model.parameters()).device
        self.static = {}
        for k, v in example_batch.items():
            if isinstance(v, PackedAttentionMask):
                self.static[k] = PackedAttentionMask(v.bits.clone(), v.L)
            elif torch.is_tensor(v) and v.is_cuda:
                self.static[k] = v.clone()
        if ops._seed_dev is None:
            ops.set_device_seed_tensor(torch.zeros(1, dtype=torch.int64, device=dev))
        self._seed = ops._seed_dev
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side):                    # warm-up on a side stream (allocator, lazy library state, cudaFuncSetAttribute)
            for _ in range(max(1, warmup)):
                model.zero_grad(set_to_none=True)
                step(model, self.static)
                self._seed.add_(1)
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        model.zero_grad(set_to_none=True)
        self.graph = torch.cuda.CUDAGraph()
        n0 = L.lib().vlpk_launch_count()
        with torch.cuda.graph(self.graph, capture_error_mode=capture_error_mode):
            self.loss = step(model, self.static)
        self.launches_per_replay = int(L.lib().vlpk_launch_count() - n0)   # libvlpk kernels inside one replay (torch's are extra)
        if self.launches_per_replay <= 0:
            raise RuntimeError("vlp_b200.graph: the captured step launched no libvlpk kernel")
        # the gradient tensors the graph writes; re-attached after every replay so that a training loop's `optimizer.zero_grad()`
        # (set_to_none=True, run_img2txt_dist.py's loop calls it every step) or an interleaved eager step cannot detach them
        self._grads = [(p, p.grad) for p in model.parameters() if p.grad is not None]

    def load(self, batch):
        """Copy a device batch into the captured input buffers (async, on the current stream)."""
        for k, dst in self.static.items():
            src = batch[k]
            if isinstance(dst, PackedAttentionMask):
                if not isinstance(src, PackedAttentionMask):
                    raise RuntimeError(f"vlp_b200.graph: '{k}' was captured as a PackedAttentionMask")
                dst.bits.copy_(src.bits, non_blocking=True)
            elif src.data_ptr() != dst.data_ptr():
                dst.copy_(src, non_blocking=True)

    def __call__(self, batch=None):
        if batch is not None:
            self.load(batch)
        self._seed.add_(1)                               # fresh dropout masks from the frozen launch sequence
        self.graph.replay()
        for p, g in self._grads:
            if p.grad is not g:
                p.grad = g
        return self.loss


class GraphedCall:
    """Capture `fn(*tensors)` (inference: no autograd, no host synchronisation, fixed shapes) once and replay it.

        dec = GraphedCall(lambda *a: decoder(*a, task_idx=None), (vis_feats, vis_pe, input_ids, token_type_ids, position_ids, mask))
        ids, scores = dec(vis_feats2, vis_pe2, input_ids2, ...)        # copies into the captured inputs, replays, returns static outputs

    Written for decode (`BertForSeq2SeqDecoder.forward`, modeling.py:1189-1253 / beam search :1256-1494): with the per-layer K/V caches a
    decode step touches 2 new rows per sequence and is launch-bound (12 layers x 6 launches + head per step, 21 steps); every step has its
    own shapes but the sequence of steps is fixed for a given (batch, lengths), so the whole loop — region projections, 21 cached decode
    steps, greedy arg-max or beam bookkeeping and back-tracking, all on the device — is one graph.  The returned tensors are overwritten by
    the next call; clone what must survive.  Not for `forbid_duplicate_ngrams` (host-side n-gram bookkeeping)."""

    def __init__(self, fn, example_args, warmup=2):
        self.static = tuple(a.clone() if torch.is_tensor(a) else a for a in example_args)
        dev = next(a.device for a in self.static if torch.is_tensor(a))
        cur = torch.cuda.current_stream(dev)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(cur)
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(max(1, warmup)):
                fn(*self.static)
        cur.wait_stream(side)
        torch.cuda.synchronize(dev)
        self.graph = torch.cuda.CUDAGraph()
        n0 = L.lib().vlpk_launch_count()
        with torch.no_grad(), torch.cuda.graph(self.graph):
            self.out = fn(*self.static)
        self.launches_per_replay = int(L.lib().vlpk_launch_count() - n0)

    def __call__(self, *args):
        for dst, src in zip(self.static, args):
            if torch.is_tensor(dst) and src.data_ptr() != dst.data_ptr():
                dst.copy_(src, non_blocking=True)
        self.graph.replay()
        return self.out
