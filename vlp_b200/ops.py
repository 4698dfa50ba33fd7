"""torch.autograd glue between the nn.Module surface (vlp_modules.py) and the C ABI (libvlpk.so).

PyTorch is plumbing here: it owns device memory, streams and the autograd tape.  Every forward/backward
body is one (or a few) calls into the hand-written CUDA library — there is no PyTorch implementation of
these ops anywhere in the package, so a missing library is a hard error.
"""
import ctypes as C
import itertools
import math
import os

import torch

from . import _lib as L

BF16 = torch.bfloat16

# ------------------------------------------------------------------------------------------------
# dropout seeding
# ------------------------------------------------------------------------------------------------
_seed_counter = itertools.count(1)
_seed_dev = None  # optional int64 CUDA tensor: added to the host seed on device (CUDA-graph replays)


def set_device_seed_tensor(t):
    """Register a 1-element int64 CUDA tensor whose value is added to every dropout seed at kernel run time.
    Increment it between CUDA-graph replays to get fresh masks from a frozen launch sequence."""
    global _seed_dev
    _seed_dev = t


SEED_LOG = None  # tests: set to a list to record (kind, seed) of every dropout stream drawn (kind: "encoder", "linear:<site>", "embed")


def next_seed(kind=None):
    seed = (torch.initial_seed() * 1000003 + next(_seed_counter) * 7919) & 0x7FFFFFFFFFFFFFFF
    if SEED_LOG is not None:
        SEED_LOG.append((kind, seed))
    return seed


def dropout_keep_mask(p, seed, site, n):
    """uint8 [n] keep decisions of dropout site `site` under `seed` (vlpk_debug_dropout_mask) — test support."""
    n8 = (n + 7) // 8 * 8
    out = torch.empty(n8, dtype=torch.uint8, device="cuda")
    L.call("vlpk_debug_dropout_mask", _drop(p, seed), site, n8, out.data_ptr(), L.stream())
    return out[:n]


def _drop(p, seed):
    if p <= 0.0 or seed is None:
        return None
    return L.VlpkDropout(float(p), int(seed), None if _seed_dev is None else _seed_dev.data_ptr())


def _bf16c(t):
    """bf16 + contiguous view/copy of a tensor (parameters of a bf16 model pass through untouched)."""
    if t is None:
        return None
    if t.dtype != BF16:
        t = t.to(BF16)
    return t if t.is_contiguous() else t.contiguous()


def _require_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"vlp_b200: {what} must live on a CUDA device (no CPU path exists)")


# ------------------------------------------------------------------------------------------------
# attention mask -> bitmask
# ------------------------------------------------------------------------------------------------
MAX_SEQ = 512  # longest sequence the attention kernels take (4 key tiles of 128)


def key_slots(kv):
    """S = 128 * ceil(kv / 128): key slots of a packed mask row (S / 32 words) and of an attention keep-bit row (S / 8 bytes)."""
    return (kv + 127) // 128 * 128


def kv_slots(Lq, Lkv):
    """VlpkShape.kv_slots for a shape: 0 (the 128-slot layout) when both lengths fit one tile, else key_slots(Lkv).  Raises before any
    launch for lengths the kernels do not take."""
    if not (1 <= Lq and 1 <= Lkv <= MAX_SEQ and Lq <= key_slots(Lkv)):
        raise ValueError(f"vlp_b200: sequence length Lq={Lq} Lkv={Lkv} unsupported (attention takes up to {MAX_SEQ})")
    return 0 if Lq <= 128 and Lkv <= 128 else key_slots(Lkv)


def _check_mask_words(mask_bits, Lkv):
    if mask_bits.shape[-1] * 32 != key_slots(Lkv):
        raise ValueError(f"vlp_b200: packed mask has {mask_bits.shape[-1]} words per row; {key_slots(Lkv) // 32} needed for {Lkv} keys")


def pack_mask(mask, mode="additive"):
    """[B,1,R,KV] / [B,R,KV] additive (0/-10000) or 0/1 mask -> int32 [B,R,S/32] 'attend' bitmask (R may be 1), S = key_slots(KV)."""
    _require_cuda(mask, "attention mask")
    if mask.dim() == 4:
        mask = mask[:, 0]
    if mask.dim() == 2:
        mask = mask[:, None, :]
    mask = mask.contiguous()
    B, R, KV = mask.shape
    dt = {torch.float32: 1, torch.bfloat16: 0, torch.int64: 2}.get(mask.dtype)
    if dt is None:
        mask = mask.float()
        dt = 1
    if KV > MAX_SEQ:
        raise ValueError(f"vlp_b200: attention mask over {KV} keys; the kernels take up to {MAX_SEQ}")
    out = torch.empty(B, R, key_slots(KV) // 32, device=mask.device, dtype=torch.int32)
    L.call("vlpk_mask_pack", mask.data_ptr(), dt, 0 if mode == "additive" else 1, B, R, KV, R * KV, KV, out.data_ptr(), L.stream())
    return out


# ------------------------------------------------------------------------------------------------
# BertLayer stack
# ------------------------------------------------------------------------------------------------
PARAMS_PER_LAYER = 16  # order == _lib.WEIGHT_FIELDS


# Per-layer buffer layouts: [(field, shape)] in allocation order, each field's buffer packed right behind the previous one.  A field
# named None is padding.  vlpk_workspace_bytes states the same sizes on the library side.
def act_layout(B, Lq, H, heads, I, Lkv=None):
    """One layer's activations of B x Lq rows: (bf16 layout, fp32 layout).  Lkv: rows per sequence of "kv", the K | V projections
    that the incremental and cached layers keep apart from qkv; qkv keeps its 3H width there although their kernels store only Q."""
    M = B * Lq
    bf = [("qkv", (M, 3 * H)), ("ctx", (M, H)), ("t1", (M, H)), ("y1", (M, H)), ("u", (M, I)), ("hmid", (M, I)), ("t2", (M, H)),
          ("y", (M, H))]
    if Lkv is not None:
        bf.append(("kv", (B * Lkv, 2 * H)))
    n_lse = B * heads * Lq
    # lse padded up to 4 floats so that the float2 statistics behind it stay 8-byte aligned for odd B * heads * Lq
    return bf, [("lse", (1, n_lse)), (None, (-n_lse % 4,)), ("stats1", (M, 2)), ("stats2", (M, 2))]


def scratch_layout(M, H, I):
    """The bf16 backward scratch of one layer of M rows."""
    return [("dz2", (M, H)), ("dt2", (M, H)), ("du", (M, I)), ("dy1", (M, H)), ("dz1", (M, H)), ("dt1", (M, H)), ("dctx", (M, H)),
            ("dqkv", (M, 3 * H)), ("dx", (M, H))]


def grad_layout(H, I):
    """One layer's fp32 gradient arena: the parameter gradients, q / k / v stacked in wqkv and bqkv."""
    return [("wqkv", (3 * H, H)), ("bqkv", (3 * H,)), ("wo", (H, H)), ("bo", (H,)), ("ln1_g", (H,)), ("ln1_b", (H,)), ("w1", (I, H)),
            ("b1", (I,)), ("w2", (H, I)), ("b2", (H,)), ("ln2_g", (H,)), ("ln2_b", (H,))]


def _layer_sizes(H, I):
    """Element counts of grad_layout's fields, in its order."""
    return [math.prod(shape) for _, shape in grad_layout(H, I)]


def layout_numel(layout):
    return sum(math.prod(shape) for _, shape in layout)


def carve(flat, layout, struct=None):
    """{field: view} of the 1-D tensor flat cut by layout; when struct is given, each field of it is set to its view's pointer."""
    views, off = {}, 0
    for name, shape in layout:
        n = math.prod(shape)
        if name is not None:
            views[name] = flat[off:off + n].view(shape)
            if struct is not None:
                setattr(struct, name, views[name].data_ptr())
        off += n
    return views


def _grad_views(arena, H, I):
    """Views of one layer's fp32 (or converted) arena in the order of WEIGHT_FIELDS (wqkv and bqkv split into q, k, v)."""
    g = carve(arena, grad_layout(H, I))
    return [*g["wqkv"].view(3, H, H), *g["bqkv"].view(3, H)] + [g[n] for n in L.WEIGHT_FIELDS[6:]]


class _Acts:
    """Per-layer activation buffers (one bf16 + one fp32 allocation for the whole stack, each layer's row cut by act_layout)."""

    def __init__(self, n_layers, B, Lq, H, heads, I, device, Lkv=None, drop_bits=False):
        bf, f32 = act_layout(B, Lq, H, heads, I, Lkv)
        self.bf = torch.empty(n_layers, layout_numel(bf), device=device, dtype=BF16)
        self.f32 = torch.empty(n_layers, layout_numel(f32), device=device, dtype=torch.float32)
        self.structs = (L.VlpkLayerActs * n_layers)()
        # training with dropout: 1 bit per attention probability (key_slots(Lq) per query row: the training path has Lkv = Lq),
        # written by the forward attention kernel and re-read by the backward one instead of re-evaluating Philox
        self.bits = torch.empty(n_layers, B * heads * Lq * key_slots(Lq) // 8, device=device, dtype=torch.uint8) if drop_bits else None
        self._views = [{**carve(self.bf[i], bf, self.structs[i]), **carve(self.f32[i], f32, self.structs[i])} for i in range(n_layers)]
        if self.bits is not None:
            for i in range(n_layers):
                self.structs[i].drop_attn = self.bits[i].data_ptr()
        self.y = [v["y"].view(B, Lq, H) for v in self._views]

    def view(self, i, name):
        """Layer i's buffer `name`, shaped as act_layout states it."""
        return self._views[i][name]


def _weight_structs(params, n_layers):
    ws = (L.VlpkLayerWeights * n_layers)()
    for i in range(n_layers):
        for j, name in enumerate(L.WEIGHT_FIELDS):
            setattr(ws[i], name, params[i * PARAMS_PER_LAYER + j].data_ptr())
    return ws


class EncoderStackFn(torch.autograd.Function):
    """n_layers x BertLayer (modeling.py:367-402) in one C call each way.  Returns every layer's output.
    cfg = (n_layers, heads, I, p_attn, p_hidden, training[, grad_hook[, maps]]): maps, when not None, is (row0, views, sink): the forward
    appends every layer's attention probabilities of query rows [row0, L) (attn_probs over the saved qkv and lse; into views[i] when
    views is not None) to the list sink."""

    @staticmethod
    def forward(ctx, hidden, mask_bits, cfg, *params):
        n_layers, heads, I, p_attn, p_hidden, training = cfg[:6]
        _require_cuda(hidden, "hidden_states")
        ctx.set_materialize_grads(False)   # unused layer outputs must arrive as None in backward, not as zero tensors
        x = _bf16c(hidden)
        B, Lq, H = x.shape
        pk = [_bf16c(p) for p in params]
        seed = next_seed("encoder") if (training and (p_attn > 0 or p_hidden > 0)) else None
        slots = kv_slots(Lq, Lq)
        _check_mask_words(mask_bits, Lq)
        acts = _Acts(n_layers, B, Lq, H, heads, I, x.device, drop_bits=seed is not None)
        shape = L.VlpkShape(B, Lq, Lq, H, heads, I, slots)
        ws = _weight_structs(pk, n_layers)
        drop = _drop(max(p_attn, p_hidden), seed)
        L.call("vlpk_encoder_fwd", C.byref(shape), n_layers, ws, x.data_ptr(), mask_bits.data_ptr(), mask_bits.shape[1], acts.structs,
               float(p_attn if training else 0.0), float(p_hidden if training else 0.0), drop, L.stream())
        maps = cfg[7] if len(cfg) > 7 else None     # output_attentions: (row0, per-layer output views or None, list receiving the maps)
        if maps is not None:
            row0, views, sink = maps
            sink.extend(_acts_maps(acts, i, B, Lq, H, heads, mask_bits, row0, None if views is None else views[i]) for i in range(n_layers))
        ctx.cfg = cfg
        ctx.seed = seed
        ctx.acts = acts
        ctx.x = x
        ctx.mask_bits = mask_bits
        ctx.pk = pk
        ctx.param_dtypes = [p.dtype for p in params]
        ctx.mark_non_differentiable(mask_bits)
        outs = tuple(acts.y)
        acts.y = None        # ctx keeps the buffers (acts.bf / raw pointers), not the returned tensor objects: no output -> grad_fn -> ctx ->
        return outs          # output reference cycle, so an un-backpropagated training forward is freed by reference counting

    @staticmethod
    def backward(ctx, *dys):
        n_layers, heads, I, p_attn, p_hidden, training = ctx.cfg[:6]
        grad_hook = ctx.cfg[6] if len(ctx.cfg) > 6 else None      # data parallelism: callable(flat gradient arena) of the owning BertEncoder
        if ctx.acts is None:
            raise RuntimeError("vlp_b200: the fused BertLayer stack frees its activations in backward; a second backward "
                               "(retain_graph=True) is not supported")
        x, acts = ctx.x, ctx.acts
        B, Lq, H = x.shape
        dev = x.device
        if dys[-1] is None:
            dys = list(dys)
            dys[-1] = torch.zeros_like(x)
        dyc = [None if d is None else _bf16c(d) for d in dys]
        dy_ptrs = (C.c_void_p * n_layers)(*[None if d is None else d.data_ptr() for d in dyc])
        grads_l = grad_layout(H, I)
        per_layer = layout_numel(grads_l)
        arena = torch.zeros(n_layers, per_layer, device=dev, dtype=torch.float32)
        gs = (L.VlpkLayerGrads * n_layers)()
        for i in range(n_layers):
            carve(arena[i], grads_l, gs[i])
        scratch_l = scratch_layout(B * Lq, H, I)
        scratch = torch.empty(layout_numel(scratch_l), device=dev, dtype=BF16)
        ws_s = L.VlpkBwdScratch()
        carve(scratch, scratch_l, ws_s)
        dx0 = torch.empty_like(x)
        shape = L.VlpkShape(B, Lq, Lq, H, heads, I, kv_slots(Lq, Lq))
        ws = _weight_structs(ctx.pk, n_layers)
        drop = _drop(max(p_attn, p_hidden), ctx.seed)
        L.call("vlpk_encoder_bwd", C.byref(shape), n_layers, ws, x.data_ptr(), ctx.mask_bits.data_ptr(), ctx.mask_bits.shape[1], acts.structs,
               dy_ptrs, dx0.data_ptr(), gs, C.byref(ws_s), float(p_attn if training else 0.0), float(p_hidden if training else 0.0), drop,
               L.stream())
        # gradient arena -> parameter dtype (one conversion kernel for the whole stack)
        if all(dt == BF16 for dt in ctx.param_dtypes):
            garena = torch.empty(n_layers, per_layer, device=dev, dtype=BF16)
            L.call("vlpk_f32_to_bf16", arena.data_ptr(), garena.data_ptr(), arena.numel(), L.stream())
        else:
            garena = arena
        if grad_hook is not None:
            grad_hook(garena)            # e.g. asynchronous NCCL all-reduce of this group's gradients (dp.GradientAllReducer)
        grads = []
        for i in range(n_layers):
            for v, dt in zip(_grad_views(garena[i], H, I), ctx.param_dtypes[i * PARAMS_PER_LAYER:(i + 1) * PARAMS_PER_LAYER]):
                grads.append(v if v.dtype == dt else v.to(dt))
        ctx.acts = None
        return (dx0, None, None) + tuple(grads)


def encoder_score_fwd(x, shared_bits, query_bits, T, heads, I, params):
    """vlpk_encoder_score_fwd: the teacher-forced scoring pass of the decoder's layer stack, forward only.  x: [B, S + T, H] embeddings
    of S shared rows then T query rows; shared_bits [B, S, S' / 32] / query_bits [B, T, S' / 32]: the packed masks of the shared rows
    and of the query rows over the shared keys (each query row also sees its own key).  params: PARAMS_PER_LAYER per layer.  Returns
    the last layer's output [B, S + T, H] and its _Acts (two buffers used in turn, whatever the depth)."""
    xc = _bf16c(x)
    B, R, H = xc.shape
    S = R - T
    n_layers = len(params) // PARAMS_PER_LAYER
    if not 1 <= T < R:
        raise ValueError(f"vlp_b200: scoring needs 1 <= T < rows, got T={T} of {R} rows")
    slots = kv_slots(S, S)
    for bits, rows in ((shared_bits, S), (query_bits, T)):
        _check_mask_words(bits, S)
        if tuple(bits.shape[:2]) != (B, rows) or bits.dtype != torch.int32 or not bits.is_contiguous():
            raise ValueError(f"vlp_b200: packed scoring mask {tuple(bits.shape)} does not fit B={B}, {rows} rows")
    pk = [_bf16c(p) for p in params]
    acts = _Acts(min(n_layers, 2), B, R, H, heads, I, xc.device)
    structs = (L.VlpkLayerActs * n_layers)(*[acts.structs[i % 2] for i in range(n_layers)])
    shape = L.VlpkShape(B, S, S, H, heads, I, slots)
    L.call("vlpk_encoder_score_fwd", C.byref(shape), int(T), n_layers, _weight_structs(pk, n_layers), xc.data_ptr(), shared_bits.data_ptr(),
           query_bits.data_ptr(), structs, L.stream())
    return acts.y[(n_layers - 1) % 2], acts


def encoder_score_group_fwd(x, prefix, word_bits, query_bits, T, G, heads, I, params):
    """vlpk_encoder_score_group_fwd: the caption matrix's pass of the layer stack, forward only.  x: [B * G, 2T - 1, H] embeddings of
    the (image, caption) pairs, G per image, each its T - 1 words then its T query rows; prefix: one [B, P, 2H] bf16 K | V cache of the
    images' prefix rows per layer; word_bits [B, T - 1, S' / 32] (None when T = 1) / query_bits [B, T, S' / 32]: the packed masks of
    the word and query rows over the keys [prefix | words] (S = P + T - 1), one sequence per image.  params: PARAMS_PER_LAYER per
    layer.  Returns the last layer's output [B * G, 2T - 1, H] and its _Acts (two buffers used in turn, whatever the depth)."""
    xc = _bf16c(x)
    BG, R, H = xc.shape
    n_layers = len(params) // PARAMS_PER_LAYER
    B, P = prefix[0].shape[:2]
    S = P + T - 1
    if R != 2 * T - 1 or G < 1 or B * G != BG or len(prefix) != n_layers:
        raise ValueError(f"vlp_b200: caption-matrix rows {tuple(xc.shape)} do not fit T={T}, G={G}, {B} images and {n_layers} layers")
    for t in prefix:
        if not (t.dtype == BF16 and t.is_contiguous() and tuple(t.shape) == (B, P, 2 * H)):
            raise ValueError(f"vlp_b200: every prefix cache must be a contiguous bf16 [{B}, {P}, {2 * H}] tensor")
    slots = kv_slots(S, S)
    for bits, rows in ((word_bits, T - 1), (query_bits, T)):
        if bits is None and rows == 0:
            continue
        _check_mask_words(bits, S)
        if tuple(bits.shape[:2]) != (B, rows) or bits.dtype != torch.int32 or not bits.is_contiguous():
            raise ValueError(f"vlp_b200: packed caption-matrix mask {tuple(bits.shape)} does not fit {B} images, {rows} rows")
    pk = [_bf16c(p) for p in params]
    acts = _Acts(min(n_layers, 2), BG, R, H, heads, I, xc.device)
    structs = (L.VlpkLayerActs * n_layers)(*[acts.structs[i % 2] for i in range(n_layers)])
    caches = (C.c_void_p * n_layers)(*[t.data_ptr() for t in prefix])
    shape = L.VlpkShape(BG, S, S, H, heads, I, slots)
    L.call("vlpk_encoder_score_group_fwd", C.byref(shape), int(T), int(G), int(P), n_layers, _weight_structs(pk, n_layers), xc.data_ptr(),
           caches, P, L.ptr(word_bits), query_bits.data_ptr(), structs, L.stream())
    return acts.y[(n_layers - 1) % 2], acts


def attn_probs(q, k, lse, mask_bits, row0=0, out=None):
    """Attention probabilities of one layer (vlpk_attn_probs): P[b, h, i - row0, j] = exp(q_i . k_j / 8 + mask_add - lse[b, h, i]) for
    query rows [row0, Lq), fp32, not differentiable — the reference's attention_probs before dropout.
    q: bf16 [B, Lq, heads * 64] and k: bf16 [B, Lkv, heads * 64] views with unit column stride (e.g. slices of the packed qkv
    buffer or of a K/V cache); lse: fp32 [B, heads, Lq] contiguous; mask_bits: the packed mask of the layer's forward.
    out: None (a new [B, heads, Lq - row0, Lkv] tensor) or an fp32 view of that shape with unit column stride, row stride
    ld_p >= Lkv and head stride (Lq - row0) * ld_p; any sequence stride.  Returns out."""
    for t, what in ((q, "attention-map queries"), (k, "attention-map keys"), (lse, "attention logsumexp"), (mask_bits, "attention mask")):
        _require_cuda(t, what)
    if q.dim() != 3 or k.dim() != 3 or q.dtype != BF16 or k.dtype != BF16 or q.stride(2) != 1 or k.stride(2) != 1:
        raise RuntimeError("vlp_b200: attention maps take bf16 [B, L, heads * 64] q / k views with unit column stride")
    B, Lq, H = q.shape
    Lkv = k.shape[1]
    if lse.dim() != 3 or lse.shape[0] != B or lse.shape[2] != Lq or lse.dtype != torch.float32 or not lse.is_contiguous():
        raise RuntimeError("vlp_b200: the attention logsumexp must be a contiguous fp32 [B, heads, Lq] tensor")
    heads = lse.shape[1]
    if k.shape[0] != B or H != heads * 64 or k.shape[2] != H:
        raise RuntimeError(f"vlp_b200: attention-map q {tuple(q.shape)} / k {tuple(k.shape)} do not match {heads} heads of 64")
    if not 0 <= row0 < Lq:
        raise ValueError(f"vlp_b200: attention-map row0={row0} outside [0, {Lq})")
    slots = kv_slots(Lq, Lkv)
    _check_mask_words(mask_bits, Lkv)
    if mask_bits.shape[0] != B or mask_bits.shape[1] not in (1, Lq):
        raise ValueError(f"vlp_b200: packed mask {tuple(mask_bits.shape)} does not fit B={B}, Lq={Lq}")
    rows = Lq - row0
    if out is None:
        out = torch.empty(B, heads, rows, Lkv, device=q.device, dtype=torch.float32)
    elif (out.dtype != torch.float32 or out.shape != (B, heads, rows, Lkv) or out.stride(3) != 1 or out.stride(2) < Lkv
          or out.stride(1) != rows * out.stride(2)):
        raise RuntimeError(f"vlp_b200: attention-map output must be an fp32 [{B}, {heads}, {rows}, {Lkv}] view with unit column "
                           "stride, row stride >= Lkv and head stride rows * row stride")
    L.call("vlpk_attn_probs", B, heads, Lq, Lkv, int(row0), q.data_ptr(), q.stride(1), q.stride(0), k.data_ptr(), k.stride(1), k.stride(0),
           mask_bits.data_ptr(), mask_bits.shape[1], slots, lse.data_ptr(), out.data_ptr(), out.stride(2), out.stride(0) if B > 1 else 0,
           L.stream())
    return out


def _acts_maps(acts, i, B, Lq, H, heads, mask_bits, row0=0, out=None, k=None):
    """attn_probs of layer i of an _Acts: q in place in its qkv buffer (ld 3H, or ld H in the decode layouts that pass k)."""
    qkv = acts.view(i, "qkv")
    lse = acts.view(i, "lse").view(B, heads, Lq)
    if k is None:
        v = qkv.view(B, Lq, 3 * H)
        q, k = v[..., :H], v[..., H:2 * H]
    else:
        q = qkv.view(3, B, Lq, H)[0]
    return attn_probs(q, k, lse, mask_bits, row0, out)


def layer_incremental_fwd(hidden, history, mask_bits, heads, I, params, maps=None):
    """BertLayer.forward with history_states (modeling.py:273-277, 389-390): inference only, q rows = hidden,
    kv rows = cat(history, hidden).  maps: None, or (row0, out) — the layer's attention probabilities of query rows [row0, Lq) are
    written into out (None: a new tensor) and (y, probs) is returned."""
    x = _bf16c(hidden)
    xkv = _bf16c(torch.cat((history.to(x.dtype), x), dim=1))
    B, Lq, H = x.shape
    Lkv = xkv.shape[1]
    slots = kv_slots(Lq, Lkv)
    _check_mask_words(mask_bits, Lkv)
    pk = [_bf16c(p) for p in params]
    acts = _Acts(1, B, Lq, H, heads, I, x.device, Lkv=Lkv)
    shape = L.VlpkShape(B, Lq, Lkv, H, heads, I, slots)
    ws = _weight_structs(pk, 1)
    L.call("vlpk_layer_fwd", C.byref(shape), ws, x.data_ptr(), xkv.data_ptr(), mask_bits.data_ptr(), mask_bits.shape[1], acts.structs, 0.0, 0.0,
           None, 0, L.stream())
    if maps is None:
        return acts.y[0]
    k = acts.view(0, "kv").view(B, Lkv, 2 * H)[..., :H]
    return acts.y[0], _acts_maps(acts, 0, B, Lq, H, heads, mask_bits, maps[0], maps[1], k=k)


# ------------------------------------------------------------------------------------------------
# Linear (+ReLU +dropout): region projections
# ------------------------------------------------------------------------------------------------
class LinearActFn(torch.autograd.Function):
    """y = dropout(relu(x W^T + b)) (modeling.py:1003-1018).  K is zero-padded to a multiple of 8 (TMA strides)."""

    @staticmethod
    def forward(ctx, x, w, b, act, p, training, site):
        _require_cuda(x, "linear input")
        N, K = w.shape
        Kp = (K + 7) // 8 * 8
        x2 = _bf16c(x.reshape(-1, K))
        wc = _bf16c(w)
        if Kp != K:
            x2 = torch.nn.functional.pad(x2, (0, Kp - K))
            wc = torch.nn.functional.pad(wc, (0, Kp - K))
        bc = _bf16c(b)
        M = x2.shape[0]
        y = torch.empty(M, N, device=x.device, dtype=BF16)
        seed = next_seed(f"linear:{site}") if (training and p > 0 and act == 1) else None
        drop = _drop(p, seed)
        L.call("vlpk_linear_fwd", M, N, Kp, x2.data_ptr(), Kp, wc.data_ptr(), Kp, L.ptr(bc), y.data_ptr(), N, act, drop, site, L.stream())
        ctx.save_for_backward(x2, wc, y)
        ctx.meta = (act, p if seed is not None else 0.0, K, Kp, x.shape, w.dtype, None if b is None else b.dtype, x.dtype)
        return y.view(*x.shape[:-1], N)

    @staticmethod
    def backward(ctx, dy):
        x2, wc, y = ctx.saved_tensors
        act, p, K, Kp, xshape, wdt, bdt, xdt = ctx.meta
        M, N = y.shape
        dyc = _bf16c(dy.reshape(M, N))
        need_dx = ctx.needs_input_grad[0]
        dpre = torch.empty(M, N, device=dyc.device, dtype=BF16) if act == 1 else None
        dx = torch.empty(M, Kp, device=dyc.device, dtype=BF16) if need_dx else None
        dw = torch.zeros(N, Kp, device=dyc.device, dtype=torch.float32)
        db = torch.zeros(N, device=dyc.device, dtype=torch.float32) if bdt is not None else None
        L.call("vlpk_linear_bwd", M, N, Kp, x2.data_ptr(), Kp, wc.data_ptr(), Kp, y.data_ptr(), N, dyc.data_ptr(), N, L.ptr(dpre), L.ptr(dx), Kp,
               dw.data_ptr(), Kp, L.ptr(db), act, float(p), L.stream())
        gx = dx[:, :K].reshape(xshape).to(xdt) if need_dx else None
        return gx, dw[:, :K].to(wdt), (db.to(bdt) if db is not None else None), None, None, None, None


# ------------------------------------------------------------------------------------------------
# Embeddings
# ------------------------------------------------------------------------------------------------
class EmbedFn(torch.autograd.Function):
    """BertEmbeddings.forward (modeling.py:217-241)."""

    @staticmethod
    def forward(ctx, vis, vpe, word_w, pos_w, type_w, ln_g, ln_b, ids, tt, pos, vis_input, R, p, training):
        _require_cuda(ids, "input_ids")
        B, Lq = ids.shape
        H = word_w.shape[1]
        visc, vpec = (_bf16c(vis), _bf16c(vpe)) if vis_input else (None, None)
        tabs = [_bf16c(t) for t in (word_w, pos_w, type_w, ln_g, ln_b)]
        ids = ids.contiguous()
        tt = None if tt is None else tt.contiguous()
        pos = None if pos is None else pos.contiguous()
        y = torch.empty(B, Lq, H, device=ids.device, dtype=BF16)
        stats = torch.empty(B * Lq, 2, device=ids.device, dtype=torch.float32)
        seed = next_seed("embed") if (training and p > 0) else None
        drop = _drop(p, seed)
        L.call("vlpk_embed_fwd", B, Lq, H, R, 1 if vis_input else 0, ids.data_ptr(), L.ptr(tt), L.ptr(pos), tabs[0].data_ptr(), tabs[1].data_ptr(),
               tabs[2].data_ptr(), L.ptr(visc), L.ptr(vpec), tabs[3].data_ptr(), tabs[4].data_ptr(), y.data_ptr(), stats.data_ptr(), drop, 1 << 20,
               L.stream())
        ctx.saved = (visc, vpec, tabs, ids, tt, pos, stats)
        ctx.meta = (vis_input, R, p if seed is not None else 0.0, seed, [t.dtype for t in (vis, vpe, word_w, pos_w, type_w, ln_g, ln_b)] if vis_input
                    else [None, None] + [t.dtype for t in (word_w, pos_w, type_w, ln_g, ln_b)])
        return y

    @staticmethod
    def backward(ctx, dy):
        visc, vpec, tabs, ids, tt, pos, stats = ctx.saved
        vis_input, R, p, seed, dts = ctx.meta
        B, Lq = ids.shape
        H = tabs[0].shape[1]
        dev = ids.device
        dyc = _bf16c(dy)
        dz = torch.empty(B, Lq, H, device=dev, dtype=BF16)
        dg = torch.zeros(H, device=dev, dtype=torch.float32)
        db = torch.zeros(H, device=dev, dtype=torch.float32)
        drop = _drop(p, seed)
        L.call("vlpk_embed_bwd", B, Lq, H, R, 1 if vis_input else 0, ids.data_ptr(), L.ptr(tt), L.ptr(pos), tabs[0].data_ptr(), tabs[1].data_ptr(),
               tabs[2].data_ptr(), L.ptr(visc), L.ptr(vpec), tabs[3].data_ptr(), stats.data_ptr(), dyc.data_ptr(), dz.data_ptr(), dg.data_ptr(),
               db.data_ptr(), drop, 1 << 20, L.stream())
        d_vis = dz[:, 1:R + 1] if vis_input else None
        # pre-LN gradient -> tables: region rows feed the projections, the B x (L - R) looked-up rows are scattered by
        # vlpk_embed_tables_bwd (csrc/tables.cu: touched-rows-only word/position scatter, segmented token-type sums)
        V, P, T = tabs[0].shape[0], tabs[1].shape[0], tabs[2].shape[0]
        d_word = torch.empty(V, H, device=dev, dtype=BF16)
        scratch = torch.empty(V, H, device=dev, dtype=torch.float32)
        d_pos = torch.zeros(P, H, device=dev, dtype=torch.float32)
        d_type = torch.zeros(T, H, device=dev, dtype=torch.float32)
        L.call("vlpk_embed_tables_bwd", B, Lq, H, R, 1 if vis_input else 0, ids.data_ptr(), L.ptr(tt), L.ptr(pos), dz.data_ptr(), V, P, T,
               d_word.data_ptr(), scratch.data_ptr(), d_pos.data_ptr(), d_type.data_ptr(), L.stream())
        out = [None if d_vis is None else d_vis.to(dts[0]), None if d_vis is None else d_vis.to(dts[1]), d_word.to(dts[2]), d_pos.to(dts[3]),
               d_type.to(dts[4]), dg.to(dts[5]), db.to(dts[6])]
        return tuple(out) + (None,) * 7


# ------------------------------------------------------------------------------------------------
# masked-LM head tail: tied decoder + bias + per-position cross-entropy (SURVEY.md §8f-3)
# ------------------------------------------------------------------------------------------------
class DecoderCEFn(torch.autograd.Function):
    """loss[r] = CE(h[r] W^T + bias, labels[r]) (modeling.py:478-482 + 1108-1109) without fp32 logits; also returns the bf16
    logits [R,V] (non-differentiable view, kept for `last_prediction_scores`).

    label_smoothing > 0 selects the smoothed loss of crit_mask_lm_smoothed instead (modeling.py:995-999, 1104-1106): per row the
    KL divergence from the target q (q_0 = 0, q_label = 1 - eps, eps / (V - 2) elsewhere) to softmax(logits), with label 0 ignored
    (vlpk_decoder_ce_ls_fwd/bwd).  0 keeps the cross-entropy calls."""

    @staticmethod
    def forward(ctx, h, w, bias, labels, label_smoothing=0.0):
        _require_cuda(h, "decoder input")
        eps = float(label_smoothing)
        ctx.eps = eps
        R, H = h.shape
        V = w.shape[0]
        Vp = (V + 7) // 8 * 8
        hc, wc = _bf16c(h), _bf16c(w)
        bias_pad = torch.zeros(Vp, device=h.device, dtype=BF16)
        bias_pad[:V] = bias
        labels = labels.contiguous()
        logits = torch.empty(R, Vp, device=h.device, dtype=BF16)
        lse = torch.empty(R, device=h.device, dtype=torch.float32)
        loss = torch.empty(R, device=h.device, dtype=torch.float32)
        if eps:
            L.call("vlpk_decoder_ce_ls_fwd", R, V, H, eps, hc.data_ptr(), wc.data_ptr(), bias_pad.data_ptr(), labels.data_ptr(),
                   logits.data_ptr(), lse.data_ptr(), loss.data_ptr(), L.stream())
        else:
            L.call("vlpk_decoder_ce_fwd", R, V, H, hc.data_ptr(), wc.data_ptr(), bias_pad.data_ptr(), labels.data_ptr(), logits.data_ptr(),
                   lse.data_ptr(), loss.data_ptr(), L.stream())
        ctx.save_for_backward(hc, wc, labels, logits, lse)
        ctx.meta = (h.dtype, w.dtype, bias.dtype)
        scores = logits[:, :V]
        ctx.mark_non_differentiable(scores)
        return loss, scores

    @staticmethod
    def backward(ctx, dloss, _dscores):
        hc, wc, labels, logits, lse = ctx.saved_tensors
        hdt, wdt, bdt = ctx.meta
        R, H = hc.shape
        V = wc.shape[0]
        Vp = logits.shape[1]
        dev = hc.device
        dl = dloss.to(torch.float32).contiguous()
        dlogits = torch.empty(R, Vp, device=dev, dtype=BF16)
        dh = torch.zeros(R, H, device=dev, dtype=torch.float32)
        dw = torch.empty(V, H, device=dev, dtype=BF16)
        dbias = torch.zeros(Vp, device=dev, dtype=torch.float32)
        if ctx.eps:
            L.call("vlpk_decoder_ce_ls_bwd", R, V, H, ctx.eps, hc.data_ptr(), wc.data_ptr(), labels.data_ptr(), logits.data_ptr(),
                   lse.data_ptr(), dl.data_ptr(), dlogits.data_ptr(), dh.data_ptr(), dw.data_ptr(), dbias.data_ptr(), L.stream())
        else:
            L.call("vlpk_decoder_ce_bwd", R, V, H, hc.data_ptr(), wc.data_ptr(), labels.data_ptr(), logits.data_ptr(), lse.data_ptr(),
                   dl.data_ptr(), dlogits.data_ptr(), dh.data_ptr(), dw.data_ptr(), dbias.data_ptr(), L.stream())
        return dh.to(hdt), dw.to(wdt), dbias[:V].to(bdt), None, None


def layer_cached_fwd(hidden, kv_cache, pos, mask_bits, heads, I, params, maps=None):
    """BertLayer.forward for decode with a persistent K/V cache (vlpk_layer_cached_fwd): `hidden` [B, Lq, H] are the new rows, `kv_cache`
    [B, rows, 2H] bf16 holds this layer's key | value projections of the `pos` rows already seen; the new rows' K | V are appended at
    [pos, pos + Lq).  Inference only.  maps: as for layer_incremental_fwd (keys read from the cache)."""
    x = _bf16c(hidden)
    B, Lq, H = x.shape
    if not (kv_cache.dtype == BF16 and kv_cache.is_contiguous() and kv_cache.shape[0] == B and kv_cache.shape[2] == 2 * H):
        raise RuntimeError("vlp_b200: kv_cache must be a contiguous bf16 [B, rows, 2H] tensor")
    slots = kv_slots(Lq, pos + Lq)
    _check_mask_words(mask_bits, pos + Lq)
    pk = [_bf16c(p) for p in params]
    acts = _Acts(1, B, Lq, H, heads, I, x.device, Lkv=Lq)            # acts.kv: scratch for the new rows' K | V
    shape = L.VlpkShape(B, Lq, pos + Lq, H, heads, I, slots)
    ws = _weight_structs(pk, 1)
    L.call("vlpk_layer_cached_fwd", C.byref(shape), ws, x.data_ptr(), kv_cache.data_ptr(), kv_cache.shape[1], int(pos), mask_bits.data_ptr(),
           mask_bits.shape[1], acts.structs, 0, L.stream())
    if maps is None:
        return acts.y[0]
    return acts.y[0], _acts_maps(acts, 0, B, Lq, H, heads, mask_bits, maps[0], maps[1], k=kv_cache[:, :pos + Lq, :H])


def layer_cached_group_fwd(hidden, prefix, P, text, slots, G, pos, mask_bits, heads, I, params):
    """vlpk_layer_cached_group_fwd: layer_cached_fwd for the B*G hypotheses `hidden` [B*G, Lq, H] that share, per group of G, one
    image prefix.  Keys [0, P) come from prefix [B, rows >= P, 2H]; key P + j (j < pos) of hypothesis i from text row
    slots[i, j] of text [B*G, T, 2H]; the new rows' K | V are written to text[:, pos:pos + Lq) and are the last keys.  mask_bits:
    one sequence per image.  Inference only."""
    x = _bf16c(hidden)
    BG, Lq, H = x.shape
    if G < 1 or BG % G or prefix.shape[0] * G != BG:
        raise ValueError(f"vlp_b200: {BG} hypotheses are not {prefix.shape[0]} groups of G={G}")
    for t, what in ((prefix, "prefix cache"), (text, "text cache")):
        if not (t.dtype == BF16 and t.is_contiguous() and t.dim() == 3 and t.shape[2] == 2 * H):
            raise RuntimeError(f"vlp_b200: the {what} must be a contiguous bf16 [*, rows, 2H] tensor")
    T = text.shape[1]
    if text.shape[0] != BG or slots.dtype != torch.int32 or not slots.is_contiguous() or tuple(slots.shape) != (BG, T):
        raise RuntimeError("vlp_b200: text cache [B*G, T, 2H] and an int32 slot table [B*G, T] are needed")
    Lkv = P + pos + Lq
    slots_kv = kv_slots(Lq, Lkv)
    _check_mask_words(mask_bits, Lkv)
    pk = [_bf16c(p) for p in params]
    acts = _Acts(1, BG, Lq, H, heads, I, x.device, Lkv=Lq)           # acts.kv: scratch for the new rows' K | V
    shape = L.VlpkShape(BG, Lq, Lkv, H, heads, I, slots_kv)
    ws = _weight_structs(pk, 1)
    L.call("vlpk_layer_cached_group_fwd", C.byref(shape), ws, x.data_ptr(), prefix.data_ptr(), prefix.shape[1], int(P), text.data_ptr(), T,
           slots.data_ptr(), int(G), int(pos), mask_bits.data_ptr(), mask_bits.shape[1], acts.structs, 0, L.stream())
    return acts.y[0]


# ------------------------------------------------------------------------------------------------
# beam search
# ------------------------------------------------------------------------------------------------
def beam_ngram_block(hist_in, hist_out, ptr, wid, f, n, ignore, logp):
    """Duplicate-n-gram blocking of beam frame f >= 1 (vlpk_beam_ngram_block): hist_out [B*K, T_cap] int32 receives the history
    hist_in[parent] + wid of every hypothesis (ptr / wid: int64 [B, K] back pointers and word ids of frame f-1); if f >= n, logp
    (fp32, [B*K, ..., V] with unit stride in V) gets -10000 added in place at each hypothesis' repeated-n-gram completions.
    ignore: int32 device tensor of exempt word ids, or None."""
    for t, what in ((hist_in, "n-gram history"), (hist_out, "n-gram history"), (ptr, "beam back pointers"), (wid, "beam word ids"),
                    (logp, "beam log-probabilities")) + (() if ignore is None else ((ignore, "n-gram ignore set"),)):
        _require_cuda(t, what)
    B, K = wid.shape
    rows, T_cap = hist_out.shape
    V = logp.shape[-1]
    if rows != B * K or hist_out.dtype != torch.int32 or not hist_out.is_contiguous() or hist_in.shape != hist_out.shape \
            or hist_in.dtype != torch.int32 or not hist_in.is_contiguous():
        raise RuntimeError("vlp_b200: n-gram histories must be two contiguous int32 [B*K, T_cap] tensors")
    if ptr.dtype != torch.int64 or wid.dtype != torch.int64 or not (ptr.is_contiguous() and wid.is_contiguous()) or ptr.shape != wid.shape:
        raise RuntimeError("vlp_b200: back pointers and word ids must be contiguous int64 [B, K] tensors")
    lp = logp.view(rows, -1) if logp.dim() != 2 else logp
    if logp.dtype != torch.float32 or lp.stride(1) != 1 or lp.shape[0] != rows:
        raise RuntimeError("vlp_b200: beam log-probabilities must be fp32 [B*K, V] rows with unit column stride")
    if ignore is not None and (ignore.dtype != torch.int32 or ignore.dim() != 1 or not ignore.is_contiguous()):
        raise RuntimeError("vlp_b200: the n-gram ignore set must be a contiguous 1-D int32 tensor of word ids")
    n_ign = 0 if ignore is None else ignore.numel()
    L.call("vlpk_beam_ngram_block", rows, K, int(f), T_cap, int(n), hist_in.data_ptr(), hist_out.data_ptr(), ptr.data_ptr(),
           wid.data_ptr(), ignore.data_ptr() if n_ign else None, n_ign, lp.data_ptr(), lp.stride(0), V, L.stream())


# ------------------------------------------------------------------------------------------------
# top-k / top-p sampling
# ------------------------------------------------------------------------------------------------
SAMPLE_MODES = {"topk": 0, "topp": 1}
MAX_TOPK = 64


def sample_tokens(logits, bias, mode, topk, topp, seed, f, seq, score, finished, live, eos_id, pad_id=0, block_eos=False, ngram=0,
                  ignore=None):
    """One frame of top-k / top-p sampling (vlpk_sample_tokens): for every row of logits ([rows, ..., V], unit stride in V, bf16 or
    fp32, without the head's bias), adds bias ([V], same dtype, or None), blocks the duplicate n-grams of the row's history
    seq[row, :f] when ngram > 0 and [EOS] when block_eos, keeps the top-k words or the top-p nucleus and draws one with the
    Philox uniform keyed by (seed; f, row).  seq: int64 [rows, T] receives column f; score: fp32 [rows, T] or None; finished: int32
    [rows]; live: int32 [1], decremented once per row that draws eos_id.  ignore: int32 device tensor of exempt word ids, or None."""
    tensors = ((logits, "logits"), (seq, "sampled ids"), (finished, "finished flags"), (live, "live-row count"))
    for t, what in tensors + tuple((t, w) for t, w in ((bias, "logit bias"), (score, "scores"), (ignore, "n-gram ignore set"))
                                   if t is not None):
        _require_cuda(t, what)
    if mode not in SAMPLE_MODES:
        raise ValueError(f"vlp_b200: sampling mode must be one of {sorted(SAMPLE_MODES)}, got {mode!r}")
    V = logits.shape[-1]
    lg = logits.reshape(-1, V) if logits.dim() != 2 else logits
    rows = lg.shape[0]
    if logits.dtype not in (BF16, torch.float32) or lg.stride(1) != 1:
        raise RuntimeError("vlp_b200: sampling logits must be bf16 or fp32 [rows, V] with unit column stride")
    if bias is not None and (bias.dtype != logits.dtype or bias.shape != (V,) or not bias.is_contiguous()):
        raise RuntimeError("vlp_b200: the logit bias must be a contiguous [V] tensor of the logits' dtype")
    if seq.dtype != torch.int64 or seq.dim() != 2 or seq.shape[0] != rows or not seq.is_contiguous():
        raise RuntimeError("vlp_b200: sampled ids must be a contiguous int64 [rows, T] tensor")
    if score is not None and (score.dtype != torch.float32 or score.shape != seq.shape or not score.is_contiguous()):
        raise RuntimeError("vlp_b200: sampling scores must be a contiguous fp32 tensor shaped like the ids")
    if finished.dtype != torch.int32 or finished.shape != (rows,) or live.dtype != torch.int32 or live.numel() != 1:
        raise RuntimeError("vlp_b200: finished flags must be int32 [rows] and the live-row count an int32 [1] tensor")
    if ignore is not None and (ignore.dtype != torch.int32 or ignore.dim() != 1 or not ignore.is_contiguous()):
        raise RuntimeError("vlp_b200: the n-gram ignore set must be a contiguous 1-D int32 tensor of word ids")
    n_ign = 0 if ignore is None else ignore.numel()
    L.call("vlpk_sample_tokens", rows, V, lg.data_ptr(), lg.stride(0), L.ptr(bias), int(logits.dtype == torch.float32), SAMPLE_MODES[mode],
           int(topk), float(topp), int(seed) & 0xFFFFFFFFFFFFFFFF, int(f), seq.data_ptr(), seq.shape[1], L.ptr(score), finished.data_ptr(),
           live.data_ptr(), int(eos_id), int(pad_id), int(bool(block_eos)), int(ngram), ignore.data_ptr() if n_ign else None, n_ign,
           L.stream())


# ------------------------------------------------------------------------------------------------
# diverse beam search
# ------------------------------------------------------------------------------------------------
def diverse_beam_step(logits, bias, f, G, penalty, wid, ptr, score, eos, top_w, top_lp, eos_id, block_eos=False, ngram=0, ignore=None,
                      hist_in=None, hist_out=None):
    """The selection of diverse-beam frame f (vlpk_diverse_beam_step): K beams per image in G groups with a Hamming penalty.  logits:
    the head's decoder outputs without its bias, [rows, ..., V] with unit stride in V, bf16 or fp32, rows = B at f = 0 and B*K after;
    bias: [V] of the same dtype, or None.  wid / ptr (int64) and score / eos (fp32): the traces, contiguous [T, B, K]; frame f is
    written and frame f-1 read.  top_w (int32) / top_lp (fp32): contiguous [B*K, K] scratch.  ngram > 0: duplicate-n-gram blocking
    over the int32 [B*K, T_cap] histories hist_in (frame f-1) and hist_out (frame f), two different tensors used in turn; ignore:
    int32 device tensor of exempt word ids, or None.  block_eos: the frame is below min_len."""
    tensors = ((logits, "logits"), (wid, "beam word ids"), (ptr, "beam back pointers"), (score, "beam scores"), (eos, "beam eos flags"),
               (top_w, "top-K scratch"), (top_lp, "top-K scratch"))
    extra = ((bias, "logit bias"), (ignore, "n-gram ignore set"), (hist_in, "n-gram history"), (hist_out, "n-gram history"))
    for t, what in tensors + tuple((t, w) for t, w in extra if t is not None):
        _require_cuda(t, what)
    if wid.dim() != 3 or any(t.shape != wid.shape or not t.is_contiguous() for t in (wid, ptr, score, eos)) \
            or wid.dtype != torch.int64 or ptr.dtype != torch.int64 or score.dtype != torch.float32 or eos.dtype != torch.float32:
        raise RuntimeError("vlp_b200: beam traces must be contiguous [T, B, K] tensors: int64 word ids and pointers, fp32 scores and "
                           "eos flags")
    T, B, K = wid.shape
    if not 0 <= f < T:
        raise ValueError(f"vlp_b200: frame {f} outside the traces' {T} frames")
    V = logits.shape[-1]
    lg = logits.reshape(-1, V) if logits.dim() != 2 else logits
    if logits.dtype not in (BF16, torch.float32) or lg.stride(1) != 1 or lg.shape[0] != (B if f == 0 else B * K):
        raise RuntimeError("vlp_b200: diverse-beam logits must be bf16 or fp32 [rows, V] with unit column stride, rows = B at frame 0 "
                           "and B*K after")
    if bias is not None and (bias.dtype != logits.dtype or bias.shape != (V,) or not bias.is_contiguous()):
        raise RuntimeError("vlp_b200: the logit bias must be a contiguous [V] tensor of the logits' dtype")
    if top_w.dtype != torch.int32 or top_lp.dtype != torch.float32 or top_w.shape != (B * K, K) or top_lp.shape != (B * K, K) \
            or not (top_w.is_contiguous() and top_lp.is_contiguous()):
        raise RuntimeError("vlp_b200: the top-K scratch must be contiguous int32 and fp32 [B*K, K] tensors")
    T_cap = T
    if ngram:
        if hist_in is None or hist_out is None or hist_in.shape != hist_out.shape or hist_out.dim() != 2 or hist_out.shape[0] != B * K \
                or hist_in.dtype != torch.int32 or hist_out.dtype != torch.int32 or not (hist_in.is_contiguous() and hist_out.is_contiguous()):
            raise RuntimeError("vlp_b200: n-gram histories must be two contiguous int32 [B*K, T_cap] tensors")
        T_cap = hist_out.shape[1]
    if ignore is not None and (ignore.dtype != torch.int32 or ignore.dim() != 1 or not ignore.is_contiguous()):
        raise RuntimeError("vlp_b200: the n-gram ignore set must be a contiguous 1-D int32 tensor of word ids")
    n_ign = 0 if ignore is None or not ngram else ignore.numel()
    prev = (wid[f - 1], ptr[f - 1], score[f - 1], eos[f - 1]) if f else (None,) * 4
    L.call("vlpk_diverse_beam_step", B, K, int(G), int(f), V, lg.data_ptr(), lg.stride(0), L.ptr(bias), int(logits.dtype == torch.float32),
           float(penalty), int(eos_id), int(bool(block_eos)), T_cap, int(ngram), L.ptr(hist_in if ngram else None),
           L.ptr(hist_out if ngram else None), ignore.data_ptr() if n_ign else None, n_ign, *(L.ptr(t) for t in prev), top_w.data_ptr(),
           top_lp.data_ptr(), wid[f].data_ptr(), ptr[f].data_ptr(), score[f].data_ptr(), eos[f].data_ptr(), L.stream())


# ------------------------------------------------------------------------------------------------
# constrained beam search
# ------------------------------------------------------------------------------------------------
def constrained_beam_step(logits, bias, f, cons, wid, ptr, score, eos, top_w, top_lp, top_dest, eos_id, block_eos=False, ngram=0, ignore=None,
                          hist_in=None, hist_out=None):
    """The selection of constrained-beam frame f (vlpk_constrained_beam_step): K beams in each of the S = 2^C constraint states of an
    image.  logits: the head's decoder outputs without its bias, [rows, ..., V] with unit stride in V, bf16 or fp32, rows = B at f = 0
    and B*S*K after; bias: [V] of the same dtype, or None.  cons: contiguous int64 [B, C, A, P] constraint table.  wid / ptr (int64)
    and score / eos (fp32): the traces, contiguous [T, B, S*K]; frame f is written and frame f-1 read.  top_w (int32) / top_lp (fp32):
    contiguous [B*S*K, K + C*A] scratch, top_dest (int32) [B*S*K, C*A].  hist_in / hist_out: the int32 [B*S*K, T_cap] histories of
    frames f-1 and f, two different tensors used in turn (needed at f >= 1, whatever ngram).  ngram > 0: duplicate-n-gram blocking;
    ignore: int32 device tensor of exempt word ids, or None.  block_eos: the frame is below min_len."""
    tensors = ((logits, "logits"), (cons, "constraint table"), (wid, "beam word ids"), (ptr, "beam back pointers"), (score, "beam scores"),
               (eos, "beam eos flags"), (top_w, "top-K scratch"), (top_lp, "top-K scratch"), (top_dest, "top-K scratch"))
    extra = ((bias, "logit bias"), (ignore, "n-gram ignore set"), (hist_in, "word history"), (hist_out, "word history"))
    for t, what in tensors + tuple((t, w) for t, w in extra if t is not None):
        _require_cuda(t, what)
    if cons.dim() != 4 or cons.dtype != torch.int64 or not cons.is_contiguous():
        raise RuntimeError("vlp_b200: the constraint table must be a contiguous int64 [B, C, A, P] tensor")
    Bc, C, A, P = cons.shape
    if wid.dim() != 3 or any(t.shape != wid.shape or not t.is_contiguous() for t in (wid, ptr, score, eos)) \
            or wid.dtype != torch.int64 or ptr.dtype != torch.int64 or score.dtype != torch.float32 or eos.dtype != torch.float32:
        raise RuntimeError("vlp_b200: beam traces must be contiguous [T, B, S*K] tensors: int64 word ids and pointers, fp32 scores and "
                           "eos flags")
    T, B, SK = wid.shape
    if Bc != B or C < 1 or SK % (1 << C):
        raise RuntimeError(f"vlp_b200: a constraint table [{Bc}, {C}, ...] does not match traces of {B} images and {SK} slots "
                           "(2^C states of K beams)")
    K = SK >> C
    if not 0 <= f < T:
        raise ValueError(f"vlp_b200: frame {f} outside the traces' {T} frames")
    V = logits.shape[-1]
    lg = logits.reshape(-1, V) if logits.dim() != 2 else logits
    if logits.dtype not in (BF16, torch.float32) or lg.stride(1) != 1 or lg.shape[0] != (B if f == 0 else B * SK):
        raise RuntimeError("vlp_b200: constrained-beam logits must be bf16 or fp32 [rows, V] with unit column stride, rows = B at frame 0 "
                           "and B*S*K after")
    if bias is not None and (bias.dtype != logits.dtype or bias.shape != (V,) or not bias.is_contiguous()):
        raise RuntimeError("vlp_b200: the logit bias must be a contiguous [V] tensor of the logits' dtype")
    W = K + C * A
    if top_w.dtype != torch.int32 or top_lp.dtype != torch.float32 or top_dest.dtype != torch.int32 or top_w.shape != (B * SK, W) \
            or top_lp.shape != (B * SK, W) or top_dest.shape != (B * SK, C * A) \
            or not (top_w.is_contiguous() and top_lp.is_contiguous() and top_dest.is_contiguous()):
        raise RuntimeError("vlp_b200: the top-K scratch must be contiguous int32 / fp32 [B*S*K, K + C*A] and int32 [B*S*K, C*A] tensors")
    T_cap = T
    if hist_out is not None or f:
        if hist_in is None or hist_out is None or hist_in.shape != hist_out.shape or hist_out.dim() != 2 or hist_out.shape[0] != B * SK \
                or hist_in.dtype != torch.int32 or hist_out.dtype != torch.int32 or not (hist_in.is_contiguous() and hist_out.is_contiguous()):
            raise RuntimeError("vlp_b200: word histories must be two contiguous int32 [B*S*K, T_cap] tensors")
        T_cap = hist_out.shape[1]
    if ignore is not None and (ignore.dtype != torch.int32 or ignore.dim() != 1 or not ignore.is_contiguous()):
        raise RuntimeError("vlp_b200: the n-gram ignore set must be a contiguous 1-D int32 tensor of word ids")
    n_ign = 0 if ignore is None or not ngram else ignore.numel()
    prev = (wid[f - 1], ptr[f - 1], score[f - 1], eos[f - 1]) if f else (None,) * 4
    a = L.VlpkConstrainedBeamArgs(B=B, K=K, C=C, A=A, P=P, f=int(f), V=V, logits=lg.data_ptr(), ld=lg.stride(0), bias=L.ptr(bias),
                                  fp32=int(logits.dtype == torch.float32), eos_id=int(eos_id), block_eos=int(bool(block_eos)), T_cap=T_cap,
                                  n=int(ngram), hist_in=L.ptr(hist_in), hist_out=L.ptr(hist_out),
                                  ignore=ignore.data_ptr() if n_ign else None, n_ignore=n_ign, cons=cons.data_ptr(),
                                  prev_wid=L.ptr(prev[0]), prev_ptr=L.ptr(prev[1]), prev_score=L.ptr(prev[2]), prev_eos=L.ptr(prev[3]),
                                  top_w=top_w.data_ptr(), top_lp=top_lp.data_ptr(), top_dest=top_dest.data_ptr(), wid=wid[f].data_ptr(),
                                  ptr=ptr[f].data_ptr(), score=score[f].data_ptr(), eos=eos[f].data_ptr())
    L.call("vlpk_constrained_beam_step", L.C.byref(a), L.stream())
