"""Scoring given captions (BertForSeq2SeqDecoder.score_captions), host side: the one-pass row layout restated in the fp32 oracle
against the reference's frame-by-frame golden, the layout's positions, token types and visibility against what each reference frame
sees, the C ABI's argument checks, the refusals, and the call sequence under the dry-run."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import vlp_oracle as O
from tools import abi_cases
from tools import caption_score_oracle as cso
from tools import relax_projection_oracle as rpo
from vlp_b200 import _lib, score
from vlp_b200 import vlp_modules as vm


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "caption_score.pt"), weights_only=False)


def _plain_mask(m, in_len, T):
    """[B, S + T, S + T] 0/1 mask of the layout as one plain sequence: shared rows as the layout sees them, query row t over the shared
    columns before its position and over itself."""
    S, _, shared_keep, query_keep = score.layout(in_len, T)
    B = m.shape[0]
    full = torch.zeros(B, S + T, S + T, dtype=m.dtype)
    full[:, :S, :S] = m[:, :S, :S] * shared_keep
    full[:, S:, :S] = m[:, in_len:in_len + T, :S] * query_keep
    full[:, S + torch.arange(T), S + torch.arange(T)] = 1
    return full


def layout_logp(sd, dims, args, caps, task_idx):
    """The scoring layout in the oracle's fp32 arithmetic: one pass of S + T rows under _plain_mask, the head at the query rows."""
    vis, pe, input_ids, tt, pos, m = args
    rows, T = caps.shape
    in_len = input_ids.shape[1]
    S, positions, _, _ = score.layout(in_len, T)
    v, vpe = O.region_projections(sd, vis, pe)
    ids = torch.cat((input_ids, caps[:, :T - 1], torch.full((rows, T), cso.MASK_ID)), dim=1)
    e = O.embeddings(sd, v, vpe, ids, tt[:, positions], pos[:, positions], len_vis_input=dims.regions)
    h = O.encoder(sd, dims.layers, e, O.extended_attention_mask(_plain_mask(m, in_len, T)), dims.heads)[-1][:, S:]
    logits = O.lm_head(sd, h) if task_idx is None else rpo.lm_head(sd, h, cso.RELAX, task_idx)
    logp = F.log_softmax(logits.float(), -1).gather(2, caps.unsqueeze(-1))[..., 0]
    return torch.where((caps != 0).cumprod(1).bool(), logp, torch.zeros_like(logp))


@pytest.mark.parametrize("name", list(cso.CASES))
def test_layout_in_fp32_matches_the_reference_frames(gold, name):
    g = gold["cases"][name]
    dims, sd, args, caps, task_idx = cso.inputs(name)
    assert torch.equal(caps, g["captions"])
    N = cso.CASES[name][2]
    T = caps.shape[-1]
    if N is not None:
        args = tuple(a.repeat_interleave(N, 0) for a in args)
    with torch.no_grad():
        got = layout_logp(sd, dims, args, caps.reshape(-1, T), task_idx).view(caps.shape)
    ref = g["logp"]
    assert torch.equal(got == 0, ref == 0)
    err = (got - ref).abs()
    assert float((err / ref.abs().clamp_min(1.0)).max()) <= 1e-5, float(err.max())
    assert float(g["drift"].max()) < 2e-2            # the golden's bf16 drift stays in the range the GPU bound is written for


@pytest.mark.parametrize("in_len,T", [(102, 1), (102, 20), (102, 21), (6, 8), (102, 41)])
def test_layout_shows_every_frame_what_the_reference_sees(in_len, T):
    """Key by key: frame t's [MASK] row (position p = in_len + t) sees, in the reference, the cached rows at positions [0, p) under
    mask row p and itself; every cached row was computed in its own frame against the rows before it.  The layout must give each
    row the same position, token-type column, and set of (key position, visible) pairs under a seq2seq mask."""
    out_len = in_len + T + 3
    m = abi_cases.s2s_mask(1, out_len, in_len, "cpu")[0]
    tt = torch.tensor([4] * in_len + [5] * (out_len - in_len))
    S, positions, shared_keep, query_keep = score.layout(in_len, T)
    assert S == in_len + T - 1 and positions.tolist() == list(range(S)) + list(range(in_len, in_len + T))
    seen = lambda keys: {(int(k), int(v)) for k, v in keys}
    for r in range(S + T):
        p = int(positions[r])
        if r < S:                                                  # prefix (frame 0) or the word fed at frame p - in_len + 1
            frame_keys = range(in_len) if p < in_len else range(p + 1)
            ref = seen((k, m[p, k]) for k in frame_keys)
            ref_query = seen((k, m[p, k]) for k in range(in_len + 1 if p < in_len else p + 2))   # incl. the frame's [MASK] column
            assert {kv for kv in ref_query if kv[1]} == {kv for kv in ref if kv[1]}          # no row sees its frame's [MASK]
            got = seen((j, m[p, j] * shared_keep[r, j]) for j in range(S) if shared_keep[r, j])
        else:
            t = r - S
            assert p == in_len + t
            # the cached rows [0, p) and the [MASK] row itself (-1: the row's own key, never the word at position p)
            ref = seen((k, m[p, k]) for k in range(p)) | {(-1, int(m[p, p]))}
            got = seen((j, m[p, j] * query_keep[t, j]) for j in range(S) if query_keep[t, j]) | {(-1, 1)}
        assert {kv for kv in got if kv[1]} == {kv for kv in ref if kv[1]}, r
        assert int(tt[p]) == (4 if p < in_len else 5)


# ---------------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------------
_A = 1 << 16                                                   # fake, aligned device addresses: every call below fails validation


def _score_call(shape=None, T=20, n=2, x=_A, sbits=2 * _A, qbits=3 * _A, acts_ptr=4 * _A, alias=False):
    s = shape or dict(B=2, Lq=121, Lkv=121, H=128, heads=2, I=256, kv_slots=0)
    acts = (_lib.VlpkLayerActs * max(n, 1))()
    for i in range(max(n, 1)):
        acts[i] = _lib.VlpkLayerActs(*([acts_ptr + (0 if alias else i) * _A] * len(_lib.ACT_FIELDS)))
    w = (_lib.VlpkLayerWeights * max(n, 1))(*[_lib.VlpkLayerWeights(*([7 * _A] * len(_lib.WEIGHT_FIELDS)))] * max(n, 1))
    return _lib.lib().vlpk_encoder_score_fwd(_lib.VlpkShape(*s.values()), T, n, w, x, sbits, qbits, acts, None)


def _self_call(B=2, heads=2, Lq=20, Lkv=121, kv_slots=0, q=_A, ks=2 * _A, mask=3 * _A):
    return _lib.lib().vlpk_attn_core_self_fwd(B, heads, Lq, Lkv, q, 3 * 128, 0, 4 * _A, 5 * _A, 3 * 128, 0, ks, 6 * _A, mask, kv_slots,
                                              7 * _A, 128, 0, None, None)


def test_abi_rejects_bad_arguments_without_launching():
    lib = _lib.lib()
    for name in ("vlpk_encoder_score_fwd", "vlpk_encoder_score_workspace_bytes", "vlpk_attn_core_self_fwd"):
        assert name in _lib.EXPORTED_SYMBOLS
    before = lib.vlpk_launch_count()
    bad = [dict(T=0), dict(T=513), dict(n=0), dict(x=None), dict(sbits=None), dict(qbits=None), dict(acts_ptr=0), dict(x=_A + 2),
           dict(sbits=2 * _A + 4), dict(alias=True), dict(shape=dict(B=2, Lq=121, Lkv=120, H=128, heads=2, I=256, kv_slots=0)),
           dict(shape=dict(B=2, Lq=130, Lkv=130, H=128, heads=2, I=256, kv_slots=0)),
           dict(shape=dict(B=2, Lq=121, Lkv=121, H=64, heads=1, I=256, kv_slots=0)),
           dict(shape=dict(B=0, Lq=121, Lkv=121, H=128, heads=2, I=256, kv_slots=0))]
    for b in bad:
        assert _score_call(**b) < 0, b
        assert lib.vlpk_last_error()
    for b in [dict(Lq=0), dict(Lq=513), dict(Lkv=0), dict(Lkv=129), dict(Lkv=200, kv_slots=128), dict(q=None), dict(ks=None),
              dict(ks=2 * _A + 4), dict(mask=None), dict(heads=0)]:
        assert _self_call(**b) < 0, b
    assert lib.vlpk_launch_count() == before


def test_workspace_bytes_match_the_python_buffers():
    import ctypes as C
    out = (C.c_size_t * 1)()
    B, S, T, H, heads, I = 3, 121, 20, 128, 2, 256
    assert _lib.lib().vlpk_encoder_score_workspace_bytes(_lib.VlpkShape(B, S, S, H, heads, I, 0), T, out) == 0
    M = B * (S + T)
    lse = math.ceil(B * heads * (S + T) / 4) * 4
    assert out[0] == 2 * M * (8 * H + 2 * I) + 4 * (lse + 4 * M)
    assert _lib.lib().vlpk_encoder_score_workspace_bytes(_lib.VlpkShape(B, S, S, H, heads, I, 0), 0, out) < 0


# ---------------------------------------------------------------------------------------------------------------------------
# model surface
# ---------------------------------------------------------------------------------------------------------------------------
def _tiny(**kw):
    from test_nbest_cpu import _tiny_decoder
    return _tiny_decoder(**kw)


def _refused(model, args, caps, grad=False, **kw):
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="vlp_b200"):
            with torch.set_grad_enabled(grad):
                model.score_captions(*args, caps, **kw)
    assert calls == []


def test_refusals_launch_nothing():
    model, args, T = _tiny()
    B = args[2].shape[0]
    ok = torch.randint(1, 50, (B, T))
    _refused(model, args, ok[:, :0])                                          # T < 1
    _refused(model, args, torch.randint(1, 50, (B, T + 1)))                   # T > out_len - in_len
    _refused(model, args, ok.int())                                           # dtype
    _refused(model, args, ok.float())
    _refused(model, args, ok[:1])                                             # batch
    _refused(model, args, ok.view(B, 1, 1, T))
    _refused(model, args, ok.view(-1))
    _refused(model, args, torch.full((B, T), 1000))                           # CPU ids outside [0, V)
    _refused(model, args, torch.full((B, T), -1))
    _refused(model, args, ok, grad=True)                                      # grad mode with parameters that require grad
    bad = list(args)
    bad[2] = bad[2].int()
    _refused(model, tuple(bad), ok)
    for i, t in ((0, args[0][:, :-1]), (0, args[0][..., :-1]), (0, args[0].long()), (1, args[1][:1]), (1, args[1][..., :-2]),
                 (1, args[1].int()), (5, args[5].to(torch.complex64)), (5, args[5].to(torch.uint8))):
        bad = list(args)                                                      # region inputs and mask of the wrong shape or dtype
        bad[i] = t
        _refused(model, tuple(bad), ok)
    bad = list(args)
    bad[5] = bad[5][:, :-1]
    _refused(model, tuple(bad), ok)
    for p in model.parameters():
        p.requires_grad_(False)
    with abi_cases.dry_run() as calls, torch.enable_grad():
        model.score_captions(*args, ok)                                       # grad mode is fine without trainable parameters
    assert calls


def test_relaxed_head_refuses_a_missing_task_idx():
    from vlp_b200 import synth
    d = synth.TINY
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, relax_projection=4)
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=d.regions).bfloat16().eval()
    _, args, T = _tiny()
    caps = torch.randint(1, 50, (2, T))
    _refused(model, args, caps)
    _refused(model, args, caps, task_idx=torch.tensor([0, 4]))


@pytest.mark.parametrize("N", [None, 3])
def test_call_sequence(N):
    model, args, T = _tiny()
    B = args[2].shape[0]
    caps = torch.randint(1, 50, (B, T) if N is None else (B, N, T))
    with torch.no_grad(), abi_cases.dry_run() as calls:
        out = model.score_captions(*args, caps)
    assert out.shape == caps.shape and out.dtype == torch.float32
    assert calls == ["vlpk_linear_fwd"] * 3 + ["vlpk_embed_fwd", "vlpk_mask_pack", "vlpk_mask_pack", "vlpk_encoder_score_fwd",
                                               "vlpk_decoder_ce_fwd"]
