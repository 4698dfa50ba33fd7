"""The caption matrix on the GPU (BertForSeq2SeqDecoder.score_caption_matrix): the shared-prefix self-key attention kernels bitwise
against the self-key kernels on materialised keys and against fp64 with NaN guard bands; the model bitwise against score_captions on
the explicitly repeated batch where both run the same kernels (S <= 128), within the scoring bound elsewhere and against the golden;
chunkings, C = 1, T = 1, the relaxed head, GraphedCall, deterministic reruns and out-of-range device ids."""
import pytest
import torch

from test_caption_score_gpu import MASKS, TOL, _bits, _bound, _case, _mask
from tools import kernel_check as kc
from vlp_b200 import _lib as L
from vlp_b200 import graph, ops, score

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64


# ---------------------------------------------------------------------------------------------------------------------------
# kernels
# ---------------------------------------------------------------------------------------------------------------------------
def run_group_self(T, P, mask, images=2, G=2, heads=2, seed=0, kind="normal"):
    """Pairs of a T-word caption: T query rows against [P prefix rows | T - 1 word rows] plus each its own key.  The prefix cache has
    rows past P and every pair's text block rows past its words, all NaN: the kernels must read neither."""
    gen = torch.Generator().manual_seed(seed)
    H, B, W = heads * 64, images * G, T - 1
    Lkv = P + W
    scale = {"normal": 1.0, "peaky": 3.0, "common": 0.1}[kind]
    rnd = lambda *s: torch.randn(*s, generator=gen) * scale + (torch.randn(1, 1, s[-1], generator=gen) if kind == "common" else 0.0)
    qkv = rnd(B, T, 3 * H).to(DEV, BF)                                   # query rows: Q | self K | self V
    prefix = torch.full((images, P + 3, 2 * H), float("nan"), dtype=BF, device=DEV)
    prefix[:, :P] = rnd(images, P, 2 * H).to(DEV, BF)
    TT = W + 2
    text = torch.full((B, TT, 2 * H), float("nan"), dtype=BF, device=DEV)
    text[:, :W] = rnd(B, W, 2 * H).to(DEV, BF)
    m = _mask(mask, images, T, Lkv, gen)
    bits = _bits(mask, m)
    slots = 0 if T <= 128 and Lkv <= 128 else ops.key_slots(Lkv)
    q = qkv[..., :H]
    outs = []
    for group in (True, False):
        ld_o = H + 64
        ctx = kc.guarded(B * T, H, ld=ld_o)
        lse = kc.guarded(1, B * heads * T, dtype=F32, extra_rows=1)
        if group:
            L.call("vlpk_attn_core_group_self_fwd", B, G, heads, T, Lkv, P, q.data_ptr(), 3 * H, T * 3 * H, prefix.data_ptr(), P + 3, 2 * H,
                   text.data_ptr(), TT, 2 * H, qkv[..., H:].data_ptr(), qkv[..., 2 * H:].data_ptr(), bits.data_ptr(), slots, ctx.data_ptr(),
                   ld_o, T * ld_o, lse.data_ptr(), L.stream())
        else:                                                             # the same keys materialised per pair
            kv = torch.cat((prefix[:, :P].repeat_interleave(G, 0), text[:, :W]), 1).contiguous()
            L.call("vlpk_attn_core_self_fwd", B, heads, T, Lkv, q.data_ptr(), 3 * H, T * 3 * H, kv.data_ptr(), kv[..., H:].data_ptr(), 2 * H,
                   Lkv * 2 * H, qkv[..., H:].data_ptr(), qkv[..., 2 * H:].data_ptr(), bits.repeat_interleave(G, 0).contiguous().data_ptr(),
                   slots, ctx.data_ptr(), ld_o, T * ld_o, lse.data_ptr(), L.stream())
        torch.cuda.synchronize()
        kc.assert_guard_intact(ctx, "ctx")
        kc.assert_guard_intact(lse, "lse")
        outs.append((ctx.clone(), lse.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])
    ctx, lse = outs[0]
    hv = lambda t: t.reshape(B, -1, heads, 64).permute(0, 2, 1, 3).to(F64)
    keys = torch.cat((prefix[:, :P].repeat_interleave(G, 0), text[:, :W]), 1)
    q64, k64, v64, ks64, vs64 = map(hv, (q, keys[..., :H], keys[..., H:], qkv[..., H:2 * H], qkv[..., 2 * H:]))
    allow = m.to(DEV).bool().repeat_interleave(G, 0)
    s = torch.cat((q64 @ k64.transpose(-1, -2) / 8.0 + (~allow[:, None]).to(F64) * -10000.0, (q64 * ks64).sum(-1, keepdim=True) / 8.0), -1)
    Pm = torch.softmax(s, -1)
    ref = Pm[..., :Lkv] @ v64 + Pm[..., Lkv:] * vs64
    E = Pm[..., :Lkv] @ v64.abs() + Pm[..., Lkv:] * vs64.abs()
    name = f"group self T{T} P{P} h{heads} {mask} {kind}"
    kc.check_attn_block(name + " ctx", hv(ctx.reshape(B, T, H)), ref, E, kc.ATTN_FWD_BLOCK)
    kc.check_lse(name + " lse", lse.reshape(B, heads, T), torch.logsumexp(s, -1))


@pytest.mark.parametrize("P", [1, 102, 128, 129, 256])
@pytest.mark.parametrize("T", [1, 2, 20, 128, 129, 205])
def test_group_self_kernel_lengths(T, P):
    run_group_self(T, P, MASKS[(T + P) % len(MASKS)], seed=T * 1000 + P)


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("heads", [1, 12])
@pytest.mark.parametrize("T,P", [(20, 102), (41, 102)])
def test_group_self_kernel_masks_and_heads(T, P, mask, heads):
    run_group_self(T, P, mask, heads=heads, seed=heads * 10 + MASKS.index(mask))


@pytest.mark.parametrize("kind", ["normal", "peaky", "common"])
def test_group_self_kernel_inputs(kind):
    run_group_self(20, 102, "s2s", images=3, G=3, seed=7, kind=kind)


# ---------------------------------------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------------------------------------
def _shared(name, **kw):
    """A golden case with every caption of the case shared by all its images: (decoder, args, captions [C, T], task_idx)."""
    dec, args, caps, task_idx = _case(name, **kw)
    return dec, args, caps.reshape(-1, caps.shape[-1]), task_idx


def _repeated(args, caps, task_idx):
    """The pairs as score_captions takes them: image b repeated C times, the captions tiled, pair (b, c) at row b * C + c."""
    B, C = args[2].shape[0], caps.shape[0]
    rtask = task_idx.repeat_interleave(C) if torch.is_tensor(task_idx) and task_idx.dim() == 1 else task_idx
    return tuple(a.repeat_interleave(C, 0) for a in args), caps.repeat(B, 1), rtask


def _states(dec, args, caps, task_idx=None, max_rows=None):
    """[B, C, T, H] query-row hidden states of the matrix, chunk by chunk."""
    B, C, T, chunks = score.matrix_query_states(dec, *args, caps, task_idx, max_rows)
    out = None
    for c0, G, h, _, _ in chunks:
        out = torch.empty(B, C, T, h.shape[-1], device=DEV, dtype=h.dtype) if out is None else out
        out[:, c0:c0 + G] = h.reshape(B, G, T, -1)
    return out


@pytest.mark.parametrize("name", ["l123", "l123_relax4", "two_per_image"])
def test_equals_the_repeated_batch_bitwise(name):
    """S = in_len + T - 1 <= 128: the prefix runs single-tile in both, and every kernel sees the same rows and keys."""
    dec, args, caps, task_idx = _shared(name)
    rargs, rcaps, rtask = _repeated(args, caps, task_idx)
    B, C, T = args[2].shape[0], caps.shape[0], caps.shape[1]
    assert args[2].shape[1] + T - 1 <= 128
    with torch.no_grad():
        got = _states(dec, args, caps, task_idx)
        ref = score.query_states(dec, *rargs, rcaps, rtask)[0]
        assert torch.equal(got.reshape(B * C, T, -1), ref)
        lp = dec.score_caption_matrix(*args, caps, task_idx=task_idx)
        assert lp.shape == (B, C, T) and lp.dtype == F32
        assert torch.equal(lp.reshape(B * C, T), dec.score_captions(*rargs, rcaps, task_idx=rtask))


def test_long_case_within_the_scoring_bound(gold):
    """S > 128: the prefix runs single-tile at in_len rows here and KV-tiled at S rows in the repeated batch."""
    dec, args, caps, _ = _shared("l143")
    rargs, rcaps, _ = _repeated(args, caps, None)
    B, C, T = args[2].shape[0], caps.shape[0], caps.shape[1]
    drift = gold["cases"]["l143"]["drift"].reshape(C, T)
    with torch.no_grad():
        got = dec.score_caption_matrix(*args, caps)
        ref = dec.score_captions(*rargs, rcaps).view(B, C, T)
    assert torch.equal(got == 0, ref == 0)
    assert float(((got - ref).abs() / _bound(drift)[None]).max()) <= 1.0


@pytest.mark.parametrize("name", ["l123", "l123_relax4", "l143", "two_per_image"])
def test_diagonal_matches_the_golden(gold, name):
    g = gold["cases"][name]
    dec, args, caps, task_idx = _shared(name)
    B = args[2].shape[0]
    N = caps.shape[0] // B
    with torch.no_grad():
        got = dec.score_caption_matrix(*args, caps, task_idx=task_idx)
    own = got[torch.arange(B, device=DEV).repeat_interleave(N), torch.arange(B * N, device=DEV)].view(g["logp"].shape)
    assert torch.equal((own == 0).cpu(), g["logp"] == 0)
    assert float(((own - g["logp"].to(DEV)).abs() / _bound(g["drift"])).max()) <= 1.0


@pytest.fixture(scope="module")
def gold(golden_dir):
    import os
    return torch.load(os.path.join(golden_dir, "caption_score.pt"), weights_only=False)


def test_chunkings_are_bitwise_equal():
    dec, args, caps, _ = _shared("l123")
    caps = torch.cat((caps, caps.flip(0), caps[:1]), 0)              # C = 7
    B, T = args[2].shape[0], caps.shape[1]
    with torch.no_grad():
        ref = _states(dec, args, caps)
        for per_chunk in (1, 2, 3, 6):                                   # 7 = 3 + 3 + 1, 6 + 1, ...: ragged last chunks
            assert torch.equal(_states(dec, args, caps, max_rows=B * T * per_chunk), ref), per_chunk
        full = dec.score_caption_matrix(*args, caps)
        part = dec.score_caption_matrix(*args, caps, max_rows=B * T * 3)
    assert torch.allclose(full, part, rtol=0, atol=1e-4)


@pytest.mark.parametrize("C,T", [(1, 20), (3, 1)])
def test_one_caption_and_one_word(C, T):
    """The encoder bitwise; the log-probabilities within the scoring bound: at T = 1 the head's torch Linear gets a contiguous
    [rows, 1, H] input here and a strided view in score_captions, and may pick another cuBLAS kernel."""
    dec, args, caps, _ = _shared("l123")
    caps = caps[:C, :T].contiguous()
    rargs, rcaps, _ = _repeated(args, caps, None)
    B = args[2].shape[0]
    with torch.no_grad():
        assert torch.equal(_states(dec, args, caps).reshape(B * C, T, -1), score.query_states(dec, *rargs, rcaps, None)[0])
        got = dec.score_caption_matrix(*args, caps)
        ref = dec.score_captions(*rargs, rcaps)
    assert torch.equal(got.reshape(ref.shape) == 0, ref == 0)
    assert float((got.reshape(ref.shape) - ref).abs().max()) <= TOL


def test_graphed_call_replays_the_python_driven_call():
    dec, args, caps, _ = _shared("two_per_image")
    B, T = args[2].shape[0], caps.shape[1]
    fn = lambda *a: dec.score_caption_matrix(*a[:-1], a[-1], max_rows=B * T * 2)
    with torch.no_grad():
        ref = fn(*args, caps).clone()
        other = caps.flip(1).contiguous()
        ref2 = fn(*args, other).clone()
    g = graph.GraphedCall(fn, args + (caps,))
    assert torch.equal(g(*args, caps), ref)
    assert torch.equal(g(*args, other), ref2)


def test_deterministic_reruns_are_bitwise_equal():
    dec, args, caps, task_idx = _shared("l123_relax4")
    torch.use_deterministic_algorithms(True)
    try:
        with torch.no_grad():
            a = dec.score_caption_matrix(*args, caps, task_idx=task_idx, max_rows=2 * 3 * 20)
            b = dec.score_caption_matrix(*args, caps, task_idx=task_idx, max_rows=2 * 3 * 20)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(a, b)


def test_out_of_range_device_ids_end_the_caption():
    dec, args, caps, _ = _shared("l123")
    V = dec.config.vocab_size
    bad, zero = caps.clone(), caps.clone()
    bad[0, 3], bad[1, 0], bad[2, 2] = V + 5, -7, 2 ** 40
    zero[0, 3], zero[1, 0], zero[2, 2] = 0, 0, 0
    with torch.no_grad():
        a = dec.score_caption_matrix(*args, bad)
        b = dec.score_caption_matrix(*args, zero)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert torch.equal(a[:, 0, 3:], torch.zeros_like(a[:, 0, 3:])) and torch.equal(a[:, 1], torch.zeros_like(a[:, 1]))
