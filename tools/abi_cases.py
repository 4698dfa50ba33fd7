"""C-ABI call sequences shared by the GPU parity tests and by the CPU marshalling dry-run.

`dry_run()` replaces the library call (`_lib.invoke`, behind `_lib.call`'s deterministic-mode check) by a ctypes conversion of the arguments against the prototypes declared in
vlp_b200/_lib.py (the mirror of include/vlpk.h), so that the host-side marshalling of a GPU test — structs, pointer
arithmetic, argument order and count — is exercised by the `-m "not gpu"` suite without launching anything.  It computes
nothing: buffers keep whatever torch.empty returned.
"""
import contextlib
import ctypes as C

import torch

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
    off = 0
    for name, sz in zip(L.GRAD_FIELDS, ops._layer_sizes(H, I)):
        setattr(gs, name, arena_row[off:off + sz].data_ptr())
        off += sz
    assert off == arena_row.numel()
    return gs


def bwd_scratch(M, H, I, dev):
    sizes = {"dz2": M * H, "dt2": M * H, "du": M * I, "dy1": M * H, "dz1": M * H, "dt1": M * H, "dctx": M * H, "dqkv": 3 * M * H, "dx": M * H}
    buf = torch.empty(sum(sizes.values()), device=dev, dtype=BF16)
    st = L.VlpkBwdScratch()
    off = 0
    for name in L.SCRATCH_FIELDS:
        setattr(st, name, buf[off:off + sizes[name]].data_ptr())
        off += sizes[name]
    return st, buf


def act_view(acts, layer, name, rows, width):
    off = 0
    for n, sz in acts.bf_sizes:
        if n == name:
            return acts.bf[layer][off:off + sz].view(rows, width)
        off += sz
    raise KeyError(name)


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
