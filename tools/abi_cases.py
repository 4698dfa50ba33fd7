"""C-ABI call sequences shared by the GPU parity tests and by the CPU marshalling dry-run.

`dry_run()` replaces the library call (`_lib.invoke`, behind `_lib.call`'s deterministic-mode check) by a ctypes conversion of the arguments against the prototypes declared in
vlp_b200/_lib.py (the mirror of include/vlpk.h), so that the host-side marshalling of a GPU test — structs, pointer
arithmetic, argument order and count — is exercised by the `-m "not gpu"` suite without launching anything.  It computes
nothing: buffers keep whatever torch.empty returned.
"""
import contextlib
import ctypes as C
import math

import torch

from tools import kernel_check as kc
from tools import layer_check as lc
from vlp_b200 import _lib as L
from vlp_b200 import ops

BF16 = torch.bfloat16


@contextlib.contextmanager
def dry_run():
    calls = []

    def fake_call(name, *args):
        res, argtypes = L._SIGS[name]
        proto = C.CFUNCTYPE(res, *argtypes)
        proto(lambda *a: 0)(*args)      # raises ctypes.ArgumentError / TypeError on any mismatch
        calls.append(name)

    saved = (L.invoke, L.stream, ops._require_cuda, L._deterministic)
    L.invoke, L.stream, ops._require_cuda = fake_call, (lambda: 0), (lambda t, what: None)
    try:
        yield calls
    finally:
        L.invoke, L.stream, ops._require_cuda, L._deterministic = saved   # the library itself never saw the dry run's mode changes


def _rn(gen, dev, *shape, scale=1.0, shift=0.0):
    return (torch.randn(*shape, generator=gen) * scale + shift).to(dev, BF16)


def layer_params(gen, dev, H, I):
    """One BertLayer's parameters in _lib.WEIGHT_FIELDS order."""
    r = lambda *s, **k: _rn(gen, dev, *s, **k)
    return [r(H, H, scale=.05), r(H, H, scale=.05), r(H, H, scale=.05), r(H, scale=.02), r(H, scale=.02), r(H, scale=.02),
            r(H, H, scale=.05), r(H, scale=.02), r(H, scale=.1, shift=1.0), r(H, scale=.1),
            r(I, H, scale=.05), r(I, scale=.02), r(H, I, scale=.05), r(H, scale=.02), r(H, scale=.1, shift=1.0), r(H, scale=.1)]


def s2s_mask(B, L, n_src, dev):
    """0/1 seq2seq mask (seq2seq_loader.py:291-301): every row sees the source block, target rows see earlier targets."""
    m = torch.zeros(B, L, L, dtype=torch.long)
    m[:, :, :n_src] = 1
    tri = torch.tril(torch.ones(L - n_src, L - n_src, dtype=torch.long))
    m[:, n_src:, n_src:] = tri
    return m.to(dev)


def grad_struct(arena_row, H, I):
    gs = L.VlpkLayerGrads()
    ops.carve(arena_row, ops.grad_layout(H, I), gs)
    return gs


def bwd_scratch(M, H, I, dev):
    layout = ops.scratch_layout(M, H, I)
    buf = torch.empty(ops.layout_numel(layout), device=dev, dtype=BF16)
    st = L.VlpkBwdScratch()
    ops.carve(buf, layout, st)
    return st, buf


def act_view(acts, layer, name, rows, width):
    return acts.view(layer, name).view(rows, width)


def _point(struct, views):
    for n, t in views.items():
        setattr(struct, n, t.data_ptr())


def split_backward_case(dev, B=3, Lq=123, H=128, heads=2, I=512, p=0.1, seed=1234):
    """vlpk_layer_fwd, then the layer backward twice: vlpk_layer_bwd vs vlpk_ffn_bwd + vlpk_mha_bwd (include/vlpk.h)."""
    gen = torch.Generator().manual_seed(0)
    params = layer_params(gen, dev, H, I)
    x = _rn(gen, dev, B, Lq, H)
    dy = _rn(gen, dev, B, Lq, H, scale=.1)
    bits = ops.pack_mask(s2s_mask(B, Lq, max(1, Lq - 21), dev), mode="zero_one")
    M = B * Lq
    acts = ops._Acts(1, B, Lq, H, heads, I, dev)
    shape = L.VlpkShape(B, Lq, Lq, H, heads, I)
    ws = ops._weight_structs(params, 1)
    drop = L.VlpkDropout(p, seed, None)
    L.call("vlpk_layer_fwd", C.byref(shape), ws, x.data_ptr(), None, bits.data_ptr(), bits.shape[1], acts.structs, p, p, drop, 0, L.stream())
    per_layer = sum(ops._layer_sizes(H, I))
    out = {"y": acts.y[0]}
    # (A) composite
    arena_a = torch.zeros(per_layer, device=dev, dtype=torch.float32)
    ga = grad_struct(arena_a, H, I)
    sa, keep_a = bwd_scratch(M, H, I, dev)
    dx_a = torch.empty_like(x)
    L.call("vlpk_layer_bwd", C.byref(shape), ws, x.data_ptr(), bits.data_ptr(), bits.shape[1], acts.structs, dy.data_ptr(), dx_a.data_ptr(),
           C.byref(ga), C.byref(sa), p, p, drop, 0, L.stream())
    # (B) the two halves, own scratch, gradient of y1 handed over in a caller buffer
    arena_b = torch.zeros(per_layer, device=dev, dtype=torch.float32)
    gb = grad_struct(arena_b, H, I)
    sb, keep_b = bwd_scratch(M, H, I, dev)
    dy1 = torch.empty_like(x)
    dx_b = torch.empty_like(x)
    L.call("vlpk_ffn_bwd", C.byref(shape), ws, acts.structs, dy.data_ptr(), dy1.data_ptr(), C.byref(gb), C.byref(sb), p, drop, 0, L.stream())
    L.call("vlpk_mha_bwd", C.byref(shape), ws, x.data_ptr(), bits.data_ptr(), bits.shape[1], acts.structs, dy1.data_ptr(), dx_b.data_ptr(),
           C.byref(gb), C.byref(sb), p, p, drop, 0, L.stream())
    out.update(dx_a=dx_a, dx_b=dx_b, arena_a=arena_a, arena_b=arena_b, dy1=dy1, _keep=(keep_a, keep_b, params, bits, acts))
    return out


def incremental_case(dev, B=2, Lq=2, Lkv=50, H=128, heads=2, I=512):
    """BertAttention with history_states through vlpk_mha_fwd(x_kv) and through the dedicated vlpk_mha_incr_fwd entry point."""
    gen = torch.Generator().manual_seed(1)
    params = layer_params(gen, dev, H, I)
    x_kv = _rn(gen, dev, B, Lkv, H)
    x = x_kv[:, Lkv - Lq:].contiguous()
    mask = torch.ones(B, Lq, Lkv, dtype=torch.long)
    mask[:, 0, Lkv - 1] = 0                                    # first new row does not see the second
    mask[1, :, :5] = 0
    bits = ops.pack_mask(mask.to(dev), mode="zero_one")
    shape = L.VlpkShape(B, Lq, Lkv, H, heads, I)
    ws = ops._weight_structs(params, 1)
    outs = []
    for entry in ("vlpk_mha_fwd", "vlpk_mha_incr_fwd"):
        acts = ops._Acts(1, B, Lq, H, heads, I, dev, Lkv=Lkv)
        if entry == "vlpk_mha_fwd":
            L.call(entry, C.byref(shape), ws, x.data_ptr(), x_kv.data_ptr(), bits.data_ptr(), bits.shape[1], acts.structs, 0.0, 0.0, None, 0,
                   L.stream())
        else:
            L.call(entry, C.byref(shape), ws, x.data_ptr(), x_kv.data_ptr(), bits.data_ptr(), bits.shape[1], acts.structs, 0, L.stream())
        outs.append((act_view(acts, 0, "y1", B * Lq, H), acts))
    return {"y1_mha": outs[0][0], "y1_incr": outs[1][0], "_keep": (outs, params, bits, x_kv)}


# ---- encoder stack and cached decode layer (tests/test_encoder_stack_gpu.py) ------------------------------------------------------
def guarded_acts(n_layers, B, Lq, H, heads, I, dev, drop_bits=False, decode=False, Lkv=None):
    """Per-layer VlpkLayerActs whose every buffer is a NaN-guarded view (tools/kernel_check.guarded) of its ops.act_layout shape.
    Lq: rows per sequence (R = S + T or 2T - 1 for the scoring stacks).  decode: the layout of vlpk_layer_cached_fwd and of the
    re-projecting decode layer (qkv holds Q [B*Lq, H], kv the K | V of Lkv rows per sequence [B*Lkv, 2H]; Lkv defaults to Lq, the
    cached layer's new rows).  drop_bits: attention keep-bits followed by 64 guard bytes of 0xA5.  Returns (structs, [dict of views
    per layer], keep-bit buffer or None)."""
    structs = (L.VlpkLayerActs * n_layers)()
    nb = B * heads * Lq * ops.key_slots(Lq) // 8
    bits = torch.full((n_layers, nb + 64), 0xA5, dtype=torch.uint8, device=dev) if drop_bits else None
    bf, f32 = ops.act_layout(B, Lq, H, heads, I, Lkv=(Lkv or Lq) if decode else None)
    fields = {n: (s, BF16) for n, s in bf} | {n: (s, torch.float32) for n, s in f32 if n is not None}
    if decode:
        # the cached layer stores only Q in qkv: guarding exactly [B*Lq, H] catches a store past Q, which ops' 3H-wide buffer would hide
        fields["qkv"] = ((B * Lq, H), BF16)
    views = []
    for i in range(n_layers):
        v = {n: kc.guarded(*s, dtype=dt, device=dev) for n, (s, dt) in fields.items()}
        _point(structs[i], v)
        structs[i].drop_attn = None if bits is None else bits[i].data_ptr()
        views.append(v)
    return structs, views, bits


def guarded_scratch(M, H, I, dev):
    """VlpkBwdScratch of NaN-guarded views of the ops.scratch_layout shapes: (struct, dict of views)."""
    st, v = L.VlpkBwdScratch(), {n: kc.guarded(*s, device=dev) for n, s in ops.scratch_layout(M, H, I)}
    _point(st, v)
    return st, v


def guarded_grads(priors, H, I, dev):
    """Per-layer VlpkLayerGrads of NaN-guarded fp32 views of the ops.grad_layout shapes (a 1-D gradient as one row) holding the
    given prior contents ([{name: tensor}] per layer).  Returns (structs, [dict of 2-D guarded views per layer])."""
    structs = (L.VlpkLayerGrads * len(priors))()
    views = []
    for i, pr in enumerate(priors):
        v = {}
        for n, s in ops.grad_layout(H, I):
            rows, cols = s if len(s) == 2 else (1, s[0])
            v[n] = kc.guard_fill(kc.guarded(rows, cols, dtype=torch.float32, device=dev), pr[n].reshape(rows, cols))
        _point(structs[i], v)
        views.append(v)
    return structs, views


def stack_inputs(dev, B, Lq, H, I, n_layers, p, mask="s2s", dys_mid=False, seed=0):
    """Inputs of one encoder-stack case: parameters, x, the packed mask, the upstream gradients (dys[n-1], and dys[0] when
    dys_mid), the arena's prior contents and the dropout seed."""
    gen = torch.Generator().manual_seed(seed)
    heads = H // 64
    params = [t for _ in range(n_layers) for t in layer_params(gen, dev, H, I)]
    x = _rn(gen, dev, B * Lq, H)
    if mask == "s2s":
        m = s2s_mask(B, Lq, max(1, Lq - Lq // 5), dev)
    else:
        m = (torch.rand(B, Lq, Lq, generator=gen) < 0.6).long().to(dev)
    bits = ops.pack_mask(m, mode="zero_one")
    dys = [None] * n_layers
    dys[-1] = _rn(gen, dev, B * Lq, H, scale=0.1)
    if dys_mid:
        dys[0] = _rn(gen, dev, B * Lq, H, scale=0.05)
    priors = [{n: torch.randn(s, generator=gen).to(dev) for n, s in lc.grad_shapes(H, I).items()} for _ in range(n_layers)]
    shape = L.VlpkShape(B, Lq, Lq, H, heads, I, ops.kv_slots(Lq, Lq))
    return dict(B=B, Lq=Lq, H=H, I=I, heads=heads, n_layers=n_layers, p=p, params=params, x=x, mask=m, bits=bits, dys=dys,
                priors=priors, shape=shape, ws=ops._weight_structs(params, n_layers), seed=4242 + seed, dev=dev)


def stack_run(c):
    """One encoder step four ways: vlpk_encoder_fwd and a chain of vlpk_layer_fwd(layer_id = i); vlpk_encoder_bwd and a chain of
    vlpk_layer_bwd(layer_id = i), each layer with its own scratch and arena, dy of layer i = dx of layer i + 1 (+ dys[i] rounded to
    bf16).  Both backward runs read the encoder forward's activations.  Every output buffer is NaN-guarded."""
    B, Lq, H, I, heads, n, p, dev = (c[k] for k in ("B", "Lq", "H", "I", "heads", "n_layers", "p", "dev"))
    M = B * Lq
    drop = L.VlpkDropout(p, c["seed"], None) if p > 0 else None
    shape, ws, bits, x = c["shape"], c["ws"], c["bits"], c["x"]
    out = {}
    structs, acts, kbits = guarded_acts(n, B, Lq, H, heads, I, dev, drop_bits=p > 0)
    L.call("vlpk_encoder_fwd", C.byref(shape), n, ws, x.data_ptr(), bits.data_ptr(), bits.shape[1], structs, p, p, drop, L.stream())
    out.update(acts=acts, acts_structs=structs, keep_bits=kbits)
    cstructs, cacts, cbits = guarded_acts(n, B, Lq, H, heads, I, dev, drop_bits=p > 0)
    xin = x
    for i in range(n):
        L.call("vlpk_layer_fwd", C.byref(shape), C.byref(ws[i]), xin.data_ptr(), None, bits.data_ptr(), bits.shape[1], C.byref(cstructs[i]), p,
               p, drop, i, L.stream())
        xin = cacts[i]["y"]
    out.update(chain_acts=cacts, chain_keep_bits=cbits)
    # backward: the encoder
    scr_st, scr = guarded_scratch(M, H, I, dev)
    g_st, grads = guarded_grads(c["priors"], H, I, dev)
    dx0 = kc.guarded(M, H, device=dev)
    dys = (C.c_void_p * n)(*[None if d is None else d.data_ptr() for d in c["dys"]])
    L.call("vlpk_encoder_bwd", C.byref(shape), n, ws, x.data_ptr(), bits.data_ptr(), bits.shape[1], structs, dys, dx0.data_ptr(), g_st,
           C.byref(scr_st), p, p, drop, L.stream())
    out.update(scratch=scr, grads=grads, dx0=dx0)
    # backward: the chain
    cscr, cgrads, cdx, cdy = [None] * n, [None] * n, [None] * n, [None] * n
    dy = c["dys"][n - 1]
    for i in reversed(range(n)):
        st, cscr[i] = guarded_scratch(M, H, I, dev)
        gs, g = guarded_grads([c["priors"][i]], H, I, dev)
        cgrads[i] = g[0]
        cdx[i] = kc.guarded(M, H, device=dev)
        cdy[i] = dy
        xi = x if i == 0 else acts[i - 1]["y"]
        L.call("vlpk_layer_bwd", C.byref(shape), C.byref(ws[i]), xi.data_ptr(), bits.data_ptr(), bits.shape[1], C.byref(structs[i]),
               dy.data_ptr(), cdx[i].data_ptr(), C.byref(gs[0]), C.byref(st), p, p, drop, i, L.stream())
        dy = cdx[i]
        if i > 0 and c["dys"][i - 1] is not None:
            dy = (cdx[i].float() + c["dys"][i - 1].float()).to(BF16)
    out.update(chain_scratch=cscr, chain_grads=cgrads, chain_dx=cdx, chain_dy=cdy)
    return out


def cached_decode_calls(dev, H, B, src, n_steps, cache_rows, seed=0):
    """vlpk_layer_cached_fwd through a decode schedule: a prefix call at pos 0 with Lq = src (its last row the [MASK] row), then
    n_steps calls with Lq = 2 ([word, MASK]) at pos = src - 1, src, ..., each overwriting the previous call's [MASK] row.  The
    cache [B, cache_rows, 2H] starts NaN-filled.  Yields one record per call (taken right after it is enqueued) with the cache
    contents before the call."""
    gen = torch.Generator().manual_seed(seed)
    I, heads = 4 * H, H // 64
    params = layer_params(gen, dev, H, I)
    ws = ops._weight_structs(params, 1)
    cache = torch.empty(B, cache_rows, 2 * H, dtype=BF16, device=dev)
    cache.view(torch.int16).fill_(0x7FA5)
    for pos, Lq in [(0, src)] + [(src - 1 + k, 2) for k in range(n_steps)]:
        Lkv = pos + Lq
        x = _rn(gen, dev, B * Lq, H)
        if pos == 0:
            m = s2s_mask(B, Lq, Lq - 1, dev)
        else:      # row r is position pos + r: it sees every earlier position and itself
            m = torch.tril(torch.ones(Lq, Lkv, dtype=torch.long), diagonal=pos).expand(B, Lq, Lkv).contiguous().to(dev)
        bits = ops.pack_mask(m, mode="zero_one")
        structs, views, _ = guarded_acts(1, B, Lq, H, heads, I, dev, decode=True)
        shape = L.VlpkShape(B, Lq, Lkv, H, heads, I, ops.kv_slots(Lq, Lkv))
        before = cache.clone()
        L.call("vlpk_layer_cached_fwd", C.byref(shape), ws, x.data_ptr(), cache.data_ptr(), cache_rows, pos, bits.data_ptr(), bits.shape[1],
               structs, 0, L.stream())
        yield dict(pos=pos, Lq=Lq, Lkv=Lkv, B=B, H=H, I=I, heads=heads, x=x, mask=m, bits=bits, acts=views[0], before=before, cache=cache,
                   params=params)


# ---- scoring stacks and the re-projecting decode layer (tests/test_score_stack_gpu.py) ----------------------------------------------
def score_masks(kind, B, S, T, gen):
    """0/1 masks (shared [B, S, S], query [B, T, S]) of B sequences of S shared keys and T query rows.
    s2s: vlp_b200.score.layout at in_len = S - T + 1; ragged: the same with the last 3 (b % 5) prefix positions of sequence b padding,
    seen by no row; bernoulli: every bit a coin flip; dead_row: s2s with one query row per sequence seeing no shared key (only
    itself); beyond: Bernoulli(0.8), and score_bits sets every bit past S as well."""
    from vlp_b200 import score
    if kind in ("bernoulli", "beyond"):
        p = 0.5 if kind == "bernoulli" else 0.8
        return (torch.rand(B, S, S, generator=gen) < p).long(), (torch.rand(B, T, S, generator=gen) < p).long()
    in_len = S - T + 1
    _, _, shared_keep, query_keep = score.layout(in_len, T)
    shared, query = shared_keep.long().expand(B, S, S).clone(), query_keep.long().expand(B, T, S).clone()
    for b in range(B):
        if kind == "ragged":
            pad = 3 * (b % 5)
            shared[b, :, in_len - pad:in_len] = 0
            query[b, :, in_len - pad:in_len] = 0
        elif kind == "dead_row":
            query[b, (7 * b + 3) % T] = 0
    return shared, query


def score_bits(m, dev, beyond=False):
    """Packed bits of a 0/1 mask [B, rows, S]; beyond: every bit at key slots [S, key_slots(S)) set too (vlpk_mask_pack never sets
    them), which the kernels must ignore."""
    bits = ops.pack_mask(m.to(dev), "zero_one")
    S = m.shape[2]
    if beyond and S < ops.key_slots(S):
        hi = torch.zeros(bits.shape[2], dtype=torch.int64)
        for j in range(S, ops.key_slots(S)):
            hi[j // 32] |= 1 << (j % 32)
        bits = bits | torch.where(hi >= 2 ** 31, hi - 2 ** 32, hi).to(torch.int32).to(dev)
    return bits


def score_stack_inputs(dev, B, S, T, H, I, n_layers, mask="s2s", seed=0):
    """One vlpk_encoder_score_fwd case: B sequences of R = S + T rows (S shared, then T query rows)."""
    gen = torch.Generator().manual_seed(seed)
    heads, R = H // 64, S + T
    params = [t for _ in range(n_layers) for t in layer_params(gen, dev, H, I)]
    x = _rn(gen, dev, B * R, H)
    shared, query = score_masks(mask, B, S, T, gen)
    return dict(B=B, S=S, T=T, R=R, K=S, H=H, I=I, heads=heads, n_layers=n_layers, params=params, x=x,
                key_bits=score_bits(shared, dev, mask == "beyond"), query_bits=score_bits(query, dev, mask == "beyond"),
                shape=L.VlpkShape(B, S, S, H, heads, I, ops.kv_slots(S, S)), ws=ops._weight_structs(params, n_layers), dev=dev)


def score_stack_run(c, x=None):
    """vlpk_encoder_score_fwd on x (default c["x"]) into per-layer NaN-guarded acts: [dict of views per layer]."""
    x = c["x"] if x is None else x
    structs, views, _ = guarded_acts(c["n_layers"], c["B"], c["R"], c["H"], c["heads"], c["I"], c["dev"])
    L.call("vlpk_encoder_score_fwd", C.byref(c["shape"]), c["T"], c["n_layers"], c["ws"], x.data_ptr(), c["key_bits"].data_ptr(),
           c["query_bits"].data_ptr(), structs, L.stream())
    return views


def score_shared_run(c):
    """vlpk_encoder_fwd over the S shared rows alone under the shared mask into per-layer NaN-guarded acts: [dict of views per layer]."""
    B, S, R, H = c["B"], c["S"], c["R"], c["H"]
    x = c["x"].view(B, R, H)[:, :S].reshape(B * S, H).contiguous()
    structs, views, _ = guarded_acts(c["n_layers"], B, S, H, c["heads"], c["I"], c["dev"])
    bits = c["key_bits"]
    L.call("vlpk_encoder_fwd", C.byref(c["shape"]), c["n_layers"], c["ws"], x.data_ptr(), bits.data_ptr(), bits.shape[1], structs, 0.0, 0.0,
           None, L.stream())
    return views


def group_stack_inputs(dev, images, G, P, T, H, I, n_layers, mask="s2s", seed=0):
    """One vlpk_encoder_score_group_fwd case: images x G pairs of R = 2T - 1 rows (T - 1 words, then T query rows), keys [the image's
    P prefix rows | the pair's words], S = P + T - 1.  Every layer's prefix cache has prefix_rows = P + 3 rows per image, those past
    P NaN."""
    gen = torch.Generator().manual_seed(seed)
    heads, B, R, S = H // 64, images * G, 2 * T - 1, P + T - 1
    params = [t for _ in range(n_layers) for t in layer_params(gen, dev, H, I)]
    x = _rn(gen, dev, B * R, H)
    prefix = []
    for _ in range(n_layers):
        t = torch.full((images, P + 3, 2 * H), float("nan"), dtype=BF16, device=dev)
        t[:, :P] = _rn(gen, dev, images, P, 2 * H)
        prefix.append(t)
    shared, query = score_masks(mask, images, S, T, gen)
    beyond = mask == "beyond"
    return dict(images=images, G=G, P=P, B=B, S=S, T=T, R=R, K=T - 1, H=H, I=I, heads=heads, n_layers=n_layers, params=params, x=x,
                prefix=prefix, key_bits=score_bits(shared[:, P:], dev, beyond) if T > 1 else None, query_bits=score_bits(query, dev, beyond),
                shape=L.VlpkShape(B, S, S, H, heads, I, ops.kv_slots(S, S)), ws=ops._weight_structs(params, n_layers), dev=dev)


def group_stack_run(c, x=None, prefix=None):
    """vlpk_encoder_score_group_fwd on x / prefix (default c's) into per-layer NaN-guarded acts: [dict of views per layer]."""
    x = c["x"] if x is None else x
    prefix = c["prefix"] if prefix is None else prefix
    n = c["n_layers"]
    structs, views, _ = guarded_acts(n, c["B"], c["R"], c["H"], c["heads"], c["I"], c["dev"])
    caches = (C.c_void_p * n)(*[t.data_ptr() for t in prefix])
    L.call("vlpk_encoder_score_group_fwd", C.byref(c["shape"]), c["T"], c["G"], c["P"], n, c["ws"], x.data_ptr(), caches, prefix[0].shape[1],
           L.ptr(c["key_bits"]), c["query_bits"].data_ptr(), structs, L.stream())
    return views


def incr_layer_inputs(dev, B, Lq, Lkv, H, I, mask_rows, seed=0):
    """One re-projecting decode layer case: x_kv [B*Lkv, H] = cat(history, x), x its last Lq rows per sequence.  The mask [B, mask_rows,
    Lkv]: row r sees the positions up to its own, the first 2 (b % 4) of sequence b padding; one row: the last row's."""
    gen = torch.Generator().manual_seed(seed)
    heads = H // 64
    params = layer_params(gen, dev, H, I)
    x_kv = _rn(gen, dev, B * Lkv, H)
    x = x_kv.view(B, Lkv, H)[:, Lkv - Lq:].reshape(B * Lq, H).contiguous()
    m = torch.tril(torch.ones(Lq, Lkv, dtype=torch.long), diagonal=Lkv - Lq).expand(B, Lq, Lkv).clone()
    for b in range(B):
        m[b, :, :2 * (b % 4)] = 0
    m = m[:, Lq - mask_rows:].contiguous()
    return dict(B=B, Lq=Lq, Lkv=Lkv, H=H, I=I, heads=heads, params=params, x=x, x_kv=x_kv, bits=ops.pack_mask(m.to(dev), "zero_one"),
                shape=L.VlpkShape(B, Lq, Lkv, H, heads, I, ops.kv_slots(Lq, Lkv)), ws=ops._weight_structs(params, 1), dev=dev)


def incr_layer_run(c):
    """vlpk_layer_fwd and vlpk_mha_incr_fwd with x_kv, each into its own NaN-guarded acts: (layer views, attention-half views)."""
    out = []
    for entry in ("vlpk_layer_fwd", "vlpk_mha_incr_fwd"):
        structs, views, _ = guarded_acts(1, c["B"], c["Lq"], c["H"], c["heads"], c["I"], c["dev"], decode=True, Lkv=c["Lkv"])
        bits = c["bits"]
        head = (C.byref(c["shape"]), C.byref(c["ws"][0]), c["x"].data_ptr(), c["x_kv"].data_ptr(), bits.data_ptr(), bits.shape[1], structs)
        if entry == "vlpk_layer_fwd":
            L.call(entry, *head, 0.0, 0.0, None, 0, L.stream())
        else:
            L.call(entry, *head, 0, L.stream())
        out.append(views[0])
    return tuple(out)


# ---- fused BertAdam step (tests/test_adam_kernel_gpu.py) ----------------------------------------------------------------------------
ADAM_ROLES = ("param", "grad", "master", "m", "v")
ADAM_HYPER = (1e-3, 0.9, 0.999, 1e-6, 1.0)               # lr, b1, b2, e, max_grad_norm
ADAM_SIZES = (1, 7, 8, 9, 4095, 4096, 4097, 32 * 4096, 33 * 4096 + 5, 2 * 4096 + 3)
ADAM_WDS = (0.0, 0.01, 0.1)                              # per-tensor weight decay, cycled through every table
ADAM_DT = {"bf16": BF16, "fp32": torch.float32}
_ESZ = {BF16: 2, torch.float32: 4}
ADAM_CASES = ([f"sizes-{p}-{g}" for p in ADAM_DT for g in ADAM_DT]
              + [f"align-{r}-bf16-bf16" for r in ADAM_ROLES] + ["align-param-fp32-bf16", "align-grad-bf16-fp32"]
              + ["bert-base", "many-small", "single", "clip", "no-clip", "nonfinite"])


def adam_tensor(gen, dev, n, p_dt=BF16, g_dt=BF16, wd=0.01, g_scale=1e-2, g_norm=None, off=None, bad=None):
    """One tensor of a vlpk_bertadam_step table, each of its buffers a NaN-guarded 1-D view with 16 guard elements behind it.
    `off` {role: element offset of the view in its buffer}; the default is 16 bytes, so the pointer is 16-byte aligned behind a
    front guard.  Gradient, m and v magnitudes spread over three decades inside the tensor, so an error in a small element is not
    hidden by a large one.  g_norm: the gradient is rescaled to that 2-norm (0: all zero); bad: (element, value) written into
    the gradient (inf / NaN)."""
    off = off or {}
    dts = dict(param=p_dt, grad=g_dt, master=torch.float32, m=torch.float32, v=torch.float32)
    t = dict(n=n, p_dt=p_dt, g_dt=g_dt, wd=wd)
    for role in ADAM_ROLES:
        if role == "master" and p_dt != BF16:
            t[role] = None
            continue
        o = off.get(role, 16 // _ESZ[dts[role]])
        t[role] = kc.guarded(1, n, ld=o + n + 16, dtype=dts[role], extra_rows=0, col0=o, device=dev)
    spread = torch.pow(10.0, -3.0 * torch.rand(n, generator=gen, device=dev))
    g = torch.randn(n, generator=gen, device=dev) * spread * g_scale
    if g_norm is not None:
        g = g * (g_norm / g.double().norm().clamp_min(1e-300)).float()
    g = g.to(g_dt)
    if bad is not None:
        g[bad[0]] = bad[1]
    w = torch.randn(n, generator=gen, device=dev) * 0.05
    m = torch.randn(n, generator=gen, device=dev) * 1e-3 * spread
    v = (torch.randn(n, generator=gen, device=dev) * 1e-3).square() * spread
    t["init"] = dict(w=w, g=g, m=m, v=v)
    return t


def adam_case(name, dev, bert_dims=None):
    """(tensors, hyper) of one named case of ADAM_CASES.  bert_dims: the model whose parameter set "bert-base" uses (BERT-base)."""
    import zlib

    from vlp_b200 import synth
    gen = torch.Generator(device=dev).manual_seed(zlib.crc32(name.encode()))
    hyper = ADAM_HYPER
    f32 = torch.float32

    def T(i, n, **kw):
        kw.setdefault("wd", ADAM_WDS[i % 3])
        return adam_tensor(gen, dev, n, **kw)
    kind = name.split("-")
    if kind[0] == "sizes":
        p, g = ADAM_DT[kind[1]], ADAM_DT[kind[2]]
        ts = [T(i, n, p_dt=p, g_dt=g) for i, n in enumerate(ADAM_SIZES)]
    elif kind[0] == "align":         # one role misaligned at a time: each condition of the update kernel's `vec` on its own
        role, p, g = kind[1], ADAM_DT[kind[2]], ADAM_DT[kind[3]]
        fp32_role = role in ("master", "m", "v") or (role == "param" and p == f32) or (role == "grad" and g == f32)
        offs = (1, 2, 3, 1) if fp32_role else (1, 3, 7, 5)
        ts = [T(i, n, p_dt=p, g_dt=g, off={role: o}) for i, (n, o) in enumerate(zip((9, 4097, 2 * 4096 + 3, 33 * 4096 + 5), offs))]
    elif name == "bert-base":        # every parameter of the model, word embedding (5 437 chunks) included: CTAs loop many times
        keys = synth.state_dict_keys(bert_dims or synth.BERT_BASE)
        ts = [T(i, math.prod(shape), wd=0.0 if k in ("b", "g") else 0.01) for i, (_, shape, k) in enumerate(keys)]
    elif name == "many-small":       # 500 tensors of 1-9 elements around 3 large ones: the chunk search crosses many boundaries
        ts, dts = [], [(BF16, BF16), (BF16, f32), (f32, BF16), (f32, f32)]
        for i in range(503):
            n = (5 * 4096 + 77, 3 * 4096, 7 * 4096 + 1)[(i - 100) // 150] if i in (100, 250, 400) else 1 + i % 9
            ts.append(T(i, n, p_dt=dts[i % 4][0], g_dt=dts[i % 4][1]))
    elif name == "single":
        ts = [T(0, 100003, p_dt=BF16, g_dt=f32)]
    elif name in ("clip", "no-clip"):  # 2-norms just above and below max_norm, zero, far above, far below
        mx = hyper[4]
        norms = (mx * (1 + 1e-4), mx * (1 - 1e-4), 0.0, 37.0, 1e-3, mx * (1 + 1e-4), mx * (1 - 1e-4))
        sizes = (4097, 33 * 4096 + 5, 9, 2 * 4096 + 3, 4095, 7, 1)
        ts = [T(i, n, p_dt=(BF16, f32)[i % 2], g_dt=f32, g_norm=gn) for i, (n, gn) in enumerate(zip(sizes, norms))]
        if name == "no-clip":
            hyper = hyper[:4] + (-1.0,)
    elif kind[0] == "nonfinite":     # "nonfinite" and the same table without its inf / NaN ("nonfinite-clean")
        gen.manual_seed(zlib.crc32(b"nonfinite"))
        clean = name == "nonfinite-clean"
        ts = [T(0, 4096, g_scale=10.0), T(1, 5000, g_dt=f32, bad=None if clean else (3000, math.inf)), T(2, 3001, p_dt=f32),
              T(3, 4097, bad=None if clean else (4096, math.nan)), T(4, 777, g_dt=f32, g_scale=1.0)]
    else:
        raise KeyError(name)
    return ts, hyper


def adam_reset(tensors):
    """Put every tensor's initial values back into its buffers (guards untouched)."""
    for t in tensors:
        i = t["init"]
        if t["master"] is not None:
            t["master"][0].copy_(i["w"])
        t["param"][0].copy_(i["w"].to(t["p_dt"]))
        t["grad"][0].copy_(i["g"])
        t["m"][0].copy_(i["m"])
        t["v"][0].copy_(i["v"])


def adam_table(tensors, dev):
    """Host and device descriptor tables (the _TENSOR_DTYPE layout), chunk prefix and a NaN-guarded sums-of-squares buffer."""
    import numpy as np

    from vlp_b200 import optimization as opt_mod
    tab = np.zeros(len(tensors), dtype=opt_mod._TENSOR_DTYPE)
    for i, t in enumerate(tensors):
        tab[i] = (t["param"].data_ptr(), t["grad"].data_ptr(), 0 if t["master"] is None else t["master"].data_ptr(), t["m"].data_ptr(),
                  t["v"].data_ptr(), t["n"], t["wd"], opt_mod._DT[t["p_dt"]], opt_mod._DT[t["g_dt"]], 0)
    prefix = np.zeros(len(tensors) + 1, dtype=np.int32)
    np.cumsum((tab["n"] + kc.ADAM_CHUNK - 1) // kc.ADAM_CHUNK, out=prefix[1:])
    return dict(tab=tab, prefix=prefix, tab_dev=torch.from_numpy(tab.view(np.uint8).copy()).to(dev),
                prefix_dev=torch.from_numpy(prefix.copy()).to(dev),
                sq=kc.guarded(1, len(tensors), ld=len(tensors) + 16, dtype=torch.float32, extra_rows=0, device=dev))


def adam_run(tensors, table, hyper, det=False, reserved_sms=0):
    """Reset the buffers and launch vlpk_bertadam_step once, in the default or the deterministic mode."""
    adam_reset(tensors)
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(det)
    if reserved_sms:
        L.invoke("vlpk_set_reserved_sms", reserved_sms)
    try:
        L.call("vlpk_bertadam_step", table["tab"].ctypes.data, table["tab_dev"].data_ptr(), table["prefix"].ctypes.data,
               table["prefix_dev"].data_ptr(), len(tensors), table["sq"].data_ptr(), *(float(x) for x in hyper), L.stream())
    finally:
        if reserved_sms:
            L.invoke("vlpk_set_reserved_sms", 0)
        torch.use_deterministic_algorithms(before)
