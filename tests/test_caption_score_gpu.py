"""Scoring given captions on the GPU: the self-key attention kernels against fp64 with NaN guard bands, score_captions against the
reference's frame-by-frame golden (tests/golden/caption_score.pt, tools/caption_score_oracle.py), against the decode's own step fed
the words, against the layout as one plain sequence, and against the top-k sampler's scores; bitwise GraphedCall, deterministic and
[B, N, T] reruns; and what an out-of-range device id gives.

Model-level bound per word: max(2 x the reference's own fp32 -> bf16 drift on that word, 2e-2).  The worst share of every bound is
written as JSON to $VLPK_CAPTION_SCORE_REPORT when it is set."""
import json
import os

import pytest
import torch

from tools import abi_cases
from tools import caption_score_bench as csb
from tools import caption_score_oracle as cso
from tools import kernel_check as kc
from vlp_b200 import _lib as L
from vlp_b200 import graph, ops, score
from vlp_b200 import vlp_modules as vm

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64
TOL = 2e-2
WORST = {}


def _note(k, v):
    WORST[k] = max(WORST.get(k, 0.0), float(v))


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("VLPK_CAPTION_SCORE_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(sorted(WORST.items())), f, indent=1)


# ---------------------------------------------------------------------------------------------------------------------------
# kernel
# ---------------------------------------------------------------------------------------------------------------------------
def _mask(kind, B, T, S, gen):
    """0/1 [B, T, S] mask of the query rows over the shared keys."""
    if kind == "all":
        return torch.ones(B, T, S, dtype=torch.long)
    if kind == "s2s":                                              # query row t sees the shared keys before its position
        in_len = max(1, S - T + 1)
        return (torch.arange(S) < (in_len + torch.arange(T)).unsqueeze(1)).long().expand(B, T, S).contiguous()
    if kind == "bernoulli":
        return (torch.rand(B, T, S, generator=gen) < 0.5).long()
    if kind == "dead_row":                                         # some rows see no shared key: only themselves
        m = torch.ones(B, T, S, dtype=torch.long)
        for b in range(B):
            m[b, (7 * b + 3) % T] = 0
        return m
    if kind == "none":                                             # every row sees only itself
        return torch.zeros(B, T, S, dtype=torch.long)
    if kind == "beyond":                                           # Bernoulli here; bits past S are set by _bits
        return (torch.rand(B, T, S, generator=gen) < 0.8).long()
    raise ValueError(kind)


def _bits(kind, m):
    """Packed bits of the 0/1 mask m [B, T, S]; for "beyond", every bit at key slots [S, 128 * ceil(S / 128)) is set too (vlpk_mask_pack
    never sets them): the kernels must ignore them."""
    bits = ops.pack_mask(m.to(DEV), "zero_one")
    S = m.shape[2]
    if kind == "beyond" and S < ops.key_slots(S):
        hi = torch.zeros(bits.shape[2], dtype=torch.int64)
        for j in range(S, ops.key_slots(S)):
            hi[j // 32] |= 1 << (j % 32)
        bits = bits | torch.where(hi >= 2 ** 31, hi - 2 ** 32, hi).to(torch.int32).to(DEV)
    return bits


# the six kinds of test_kernel_edges_gpu.py, with "none" (every row sees only itself) in place of "rows1": the self-key kernels take one
# mask row per query row
MASKS = ["all", "s2s", "bernoulli", "dead_row", "none", "beyond"]


def run_self(B, heads, T, S, mask, seed=0, kind="normal"):
    gen = torch.Generator().manual_seed(seed)
    H = heads * 64
    src = torch.randn(B, S + T, 3 * H, generator=gen)
    if kind == "common":
        src = torch.randn(1, 1, 3 * H, generator=gen) + 0.1 * src
    elif kind == "peaky":
        src = 3.0 * src
    qkv = src.to(DEV, BF)
    q, ks, vs = qkv[:, S:, :H], qkv[:, S:, H:2 * H], qkv[:, S:, 2 * H:]
    k, v = qkv[:, :S, H:2 * H], qkv[:, :S, 2 * H:]
    m = _mask(mask, B, T, S, gen)
    bits = _bits(mask, m)
    ld_o = H + 64
    ctx = kc.guarded(B * T, H, ld=ld_o)
    lse = kc.guarded(1, B * heads * T, dtype=F32, extra_rows=1)
    L.call("vlpk_attn_core_self_fwd", B, heads, T, S, q.data_ptr(), q.stride(1), q.stride(0), k.data_ptr(), v.data_ptr(), k.stride(1),
           k.stride(0), ks.data_ptr(), vs.data_ptr(), bits.data_ptr(), 0 if S <= 128 else ops.key_slots(S), ctx.data_ptr(), ld_o, T * ld_o,
           lse.data_ptr(), L.stream())
    torch.cuda.synchronize()
    kc.assert_guard_intact(ctx, "ctx")
    kc.assert_guard_intact(lse, "lse")
    hv = lambda t: t.reshape(B, -1, heads, 64).permute(0, 2, 1, 3).to(F64)
    q64, k64, v64, ks64, vs64 = map(hv, (q, k, v, ks, vs))
    allow = m.to(DEV).bool()
    s = torch.cat((q64 @ k64.transpose(-1, -2) / 8.0 + (~allow[:, None]).to(F64) * -10000.0, (q64 * ks64).sum(-1, keepdim=True) / 8.0), -1)
    P = torch.softmax(s, -1)
    ref = P[..., :S] @ v64 + P[..., S:] * vs64
    E = P[..., :S] @ v64.abs() + P[..., S:] * vs64.abs()
    got = hv(ctx.reshape(B, T, H))
    e, t = kc.check_attn_block(f"self B{B} h{heads} T{T} S{S} {mask} {kind} ctx", got, ref, E, kc.ATTN_FWD_BLOCK)
    _note("kernel ctx elementwise (share of a E)", e)
    _note("kernel ctx rel-L2 per block / bound", t)
    _note("kernel lse / bound", kc.check_lse(f"self B{B} h{heads} T{T} S{S} {mask} lse", lse.reshape(B, heads, T), torch.logsumexp(s, -1)))


@pytest.mark.parametrize("S", [1, 102, 121, 128, 129, 256, 511])
@pytest.mark.parametrize("T", [1, 17, 20, 128, 129, 205])
def test_self_kernel_lengths(T, S):
    run_self(2, 2, T, S, MASKS[(T + S) % len(MASKS)], seed=T * 1000 + S)


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("heads", [1, 12])
@pytest.mark.parametrize("T,S", [(20, 121), (41, 142)])
def test_self_kernel_masks_and_heads(T, S, mask, heads):
    run_self(2, heads, T, S, mask, seed=heads * 10 + MASKS.index(mask))


@pytest.mark.parametrize("kind", ["normal", "peaky", "common"])
def test_self_kernel_inputs(kind):
    run_self(3, 2, 20, 121, "s2s", seed=7, kind=kind)


# ---------------------------------------------------------------------------------------------------------------------------
# model
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "caption_score.pt"), weights_only=False)


def _case(name, **kw):
    """(decoder, args on the GPU, captions, task_idx) of a golden case."""
    dims, sd, args, caps, task_idx = cso.inputs(name)
    relax = cso.RELAX if task_idx is not None else 0
    cfg = vm.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                        intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                        relax_projection=relax)
    dec = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=cso.MASK_ID, eos_id=cso.EOS_ID, enable_butd=True, len_vis_input=dims.regions, **kw)
    dec.load_state_dict(sd, strict=False)
    dec = dec.to(DEV).bfloat16().eval()
    args = tuple(a.to(DEV).to(BF) if a.is_floating_point() else a.to(DEV) for a in args)
    return dec, args, caps.to(DEV), None if task_idx is None else task_idx.to(DEV)


def _bound(drift):
    return torch.clamp(2 * drift.to(DEV), min=TOL)


def _check(name, got, ref, drift, what):
    err = (got.float() - ref.float().to(DEV)).abs()
    worst = float((err / _bound(drift)).max())
    _note(f"model vs {what} / bound", worst)
    assert worst <= 1.0, f"{name}: |err| {float(err.max()):.3e}, {worst:.2f} x the bound"


def _rows(args, caps):
    """Per-caption image inputs and [rows, T] captions."""
    if caps.dim() == 3:
        N = caps.shape[1]
        return tuple(a.repeat_interleave(N, 0) for a in args), caps.reshape(-1, caps.shape[-1])
    return args, caps


@pytest.mark.parametrize("name", list(cso.CASES))
def test_matches_the_reference_frames(gold, name):
    g = gold["cases"][name]
    dec, args, caps, task_idx = _case(name)
    with torch.no_grad():
        got = dec.score_captions(*args, caps, task_idx=task_idx)
    assert got.shape == caps.shape and got.dtype == F32
    assert torch.equal((got == 0).cpu(), g["logp"] == 0)
    _check(name, got, g["logp"], g["drift"], "golden")


@pytest.mark.parametrize("name", list(cso.CASES))
def test_matches_the_decode_step_and_the_plain_arm(gold, name):
    drift = gold["cases"][name]["drift"]
    dec, args, caps, task_idx = _case(name)
    rargs, rcaps = _rows(args, caps)
    rtask = None if task_idx is None else (task_idx.repeat_interleave(caps.shape[1]) if caps.dim() == 3 else task_idx)
    with torch.no_grad():
        got = dec.score_captions(*args, caps, task_idx=task_idx).reshape(rcaps.shape)
        loop = csb.forced_decode(dec, *rargs, rcaps, rtask)
        plain = csb.plain_arm(dec, *rargs, rcaps, rtask)
    _check(f"{name} vs frame loop", got, loop, drift.reshape(rcaps.shape), "frame loop")
    _check(f"{name} vs plain arm", got, plain, drift.reshape(rcaps.shape), "plain arm")


@pytest.mark.parametrize("name,t0", [("l123", 0), ("l123", 6), ("l143", 30)])
def test_a_query_row_sees_no_word_at_or_after_its_position(name, t0):
    """Changing the words from position t0 on leaves the query rows 0 .. t0 bitwise as they were (every other row's keys are masked
    with an exact zero weight, and the GEMMs and row kernels work row by row) and changes the later ones."""
    dec, args, caps, task_idx = _case(name)
    other = caps.clone()
    other[:, t0:] = (caps[:, t0:] + 7) % 700 + 200
    with torch.no_grad():
        a = score.query_states(dec, *args, caps, task_idx)[0]
        b = score.query_states(dec, *args, other, task_idx)[0]
    assert torch.equal(a[:, :t0 + 1], b[:, :t0 + 1])
    assert not torch.equal(a[:, t0 + 1:], b[:, t0 + 1:])


def test_scores_of_top_k_samples_are_the_samplers_own():
    dec, args, _, _ = _case("l123", sampling_method="topk", topk=5, seed=3)
    with torch.no_grad():
        ids, scores = dec(*args, task_idx=None)
        got = dec.score_captions(*args, ids)
    valid = (ids != 0).cumprod(1).bool()
    assert torch.equal(got[~valid], torch.zeros_like(got[~valid])) and torch.equal(scores[~valid], torch.zeros_like(scores[~valid]))
    err = (got - scores).abs()
    _note("model vs sampler scores / bound", float(err.max()) / TOL)
    assert float(err.max()) <= TOL, float(err.max())
    assert bool((ids == cso.EOS_ID).any()) or bool(valid.all())


def test_graphed_call_replays_the_python_driven_call():
    dec, args, caps, _ = _case("two_per_image")
    with torch.no_grad():
        ref = dec.score_captions(*args, caps).clone()
    g = graph.GraphedCall(lambda *a: dec.score_captions(*a[:-1], a[-1]), args + (caps,))
    assert torch.equal(g(*args, caps), ref)
    other = caps.flip(1)
    with torch.no_grad():
        ref2 = dec.score_captions(*args, other).clone()
    assert torch.equal(g(*args, other), ref2)


def test_deterministic_reruns_are_bitwise_equal():
    dec, args, caps, task_idx = _case("l123_relax4")
    torch.use_deterministic_algorithms(True)
    try:
        with torch.no_grad():
            a = dec.score_captions(*args, caps, task_idx=task_idx)
            b = dec.score_captions(*args, caps, task_idx=task_idx)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(a, b)


def test_several_captions_per_image_equal_the_repeated_batch():
    dec, args, caps, _ = _case("two_per_image")
    rargs, rcaps = _rows(args, caps)
    with torch.no_grad():
        a = dec.score_captions(*args, caps)
        b = dec.score_captions(*rargs, rcaps)
    assert torch.equal(a.reshape(rcaps.shape), b)


def test_out_of_range_device_ids_end_the_caption():
    """An id outside [0, V) on the device reads as 0: the caption ends there, exactly as if it held 0; no out-of-bounds read."""
    dec, args, caps, _ = _case("l123")
    V = dec.config.vocab_size
    bad, zero = caps.clone(), caps.clone()
    bad[0, 3], bad[1, 0], bad[2, 2] = V + 5, -7, 2 ** 40
    zero[0, 3], zero[1, 0], zero[2, 2] = 0, 0, 0
    with torch.no_grad():
        a = dec.score_captions(*args, bad)
        b = dec.score_captions(*args, zero)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert torch.equal(a[0, 3:], torch.zeros_like(a[0, 3:])) and torch.equal(a[1], torch.zeros_like(a[1]))


def test_stack_call_marshals_like_the_dry_run():
    """The same model call under the dry-run and for real issues the same library calls."""
    dec, args, caps, _ = _case("l123")
    n0 = L.lib().vlpk_launch_count()
    with torch.no_grad():
        dec.score_captions(*args, caps)
    torch.cuda.synchronize()
    assert L.lib().vlpk_launch_count() > n0
    with torch.no_grad(), abi_cases.dry_run() as calls:
        dec.score_captions(*args, caps)
    assert "vlpk_encoder_score_fwd" in calls
