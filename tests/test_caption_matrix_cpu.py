"""The caption matrix (BertForSeq2SeqDecoder.score_caption_matrix), host side: the matrix layout (prefix once per image, 2T - 1 rows
per pair) restated in the fp32 oracle against the reference's frame-by-frame golden, each pair row's keys against the repeated
batch's layout, the C ABI's argument checks and workspace, the refusals, and the chunked call sequence under the dry-run."""
import ctypes as C
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

from test_caption_score_cpu import _refused, _tiny


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "caption_score.pt"), weights_only=False)


def matrix_logp(sd, dims, args, caps, task_idx):
    """[B, C, T] in the oracle's fp32 arithmetic, laid out as the matrix runs: the prefix rows of each image through every layer
    once under mask[:, :P, :P]; each (image, caption) pair's 2T - 1 rows (words, then [MASK] query rows) per layer against the
    layer's prefix input as history, each row seeing the keys score.layout gives it, a query row also its own key."""
    vis, pe, input_ids, tt, pos, m = args
    B, P = input_ids.shape
    Cn, T = caps.shape
    W, R = T - 1, 2 * T - 1
    S, positions, shared_keep, query_keep = score.layout(P, T)
    v, vpe = O.region_projections(sd, vis, pe)
    pre = O.embeddings(sd, v, vpe, input_ids, tt[:, :P], pos[:, :P], len_vis_input=dims.regions)
    pre_outs = O.encoder(sd, dims.layers, pre, O.extended_attention_mask(m[:, :P, :P]), dims.heads)
    history = [pre] + pre_outs[:-1]                                   # layer i's prefix rows: its input
    rows = positions[P:]
    pc = caps.unsqueeze(0).expand(B, Cn, T).reshape(B * Cn, T)
    ids = torch.cat((pc[:, :W], torch.full((B * Cn, T), cso.MASK_ID)), 1)
    rep = lambda t: t.repeat_interleave(Cn, 0)
    h = O.embeddings(sd, None, None, ids, rep(tt[:, rows]), rep(pos[:, rows]), vis_input=False, len_vis_input=dims.regions)
    keep = torch.zeros(B, R, P + R, dtype=m.dtype)                   # keys [prefix | words | query rows]
    keep[:, :W, :S] = m[:, P:S, :S] * shared_keep[P:]
    keep[:, W:, :S] = m[:, P:P + T, :S] * query_keep
    keep[:, W + torch.arange(T), S + torch.arange(T)] = 1
    ext = O.extended_attention_mask(rep(keep))
    for i in range(dims.layers):
        h = O.bert_layer(sd, i, h, ext, dims.heads, history=rep(history[i]))
    h = h[:, W:]
    tix = None if task_idx is None else rep(task_idx)
    logits = O.lm_head(sd, h) if task_idx is None else rpo.lm_head(sd, h, cso.RELAX, tix)
    logp = F.log_softmax(logits.float(), -1).gather(2, pc.unsqueeze(-1))[..., 0]
    return torch.where((pc != 0).cumprod(1).bool(), logp, torch.zeros_like(logp)).view(B, Cn, T)


@pytest.mark.parametrize("name", list(cso.CASES))
def test_matrix_layout_in_fp32_matches_the_reference_frames(gold, name):
    """The diagonal (each image with its own captions) of the restated matrix against the golden logp."""
    g = gold["cases"][name]
    dims, sd, args, caps, task_idx = cso.inputs(name)
    B, T = args[2].shape[0], caps.shape[-1]
    shared = caps.reshape(-1, T)
    N = shared.shape[0] // B
    with torch.no_grad():
        got = matrix_logp(sd, dims, args, shared, task_idx)
    own = got[torch.arange(B).repeat_interleave(N), torch.arange(B * N)].view(g["logp"].shape)
    ref = g["logp"]
    assert torch.equal(own == 0, ref == 0)
    assert float(((own - ref).abs() / ref.abs().clamp_min(1.0)).max()) <= 1e-5


@pytest.mark.parametrize("in_len,T", [(102, 1), (102, 2), (102, 20), (6, 8), (102, 41)])
def test_every_pair_row_sees_what_the_reference_frame_sees(in_len, T):
    """Key by key under a seq2seq mask: each prefix row and each of a pair's 2T - 1 rows has the decode position and the set of
    visible (key position, mask value) pairs of its reference frame (as test_caption_score_cpu states them for score.layout), over
    the matrix's keys [prefix | the pair's words], key k at position k; a query row's own key is its own [MASK] row (pair row
    T - 1 + t), never the word at its position (pair row t)."""
    out_len = in_len + T + 3
    m = abi_cases.s2s_mask(1, out_len, in_len, "cpu")
    pm, wm, qm = (t[0] for t in score.matrix_masks(m, in_len, T))
    m = m[0]
    S, positions, _, _ = score.layout(in_len, T)
    rows = positions[in_len:]
    vis = lambda mrow: {(k, int(mrow[k])) for k in range(mrow.shape[0]) if mrow[k]}
    for i in range(in_len):                                           # frame 0: the prefix against the prefix
        assert vis(pm[i]) == {(k, int(m[i, k])) for k in range(in_len) if m[i, k]}
    for r in range(2 * T - 1):
        p = int(rows[r])
        if r < T - 1:                                                 # the word at position p, cached at frame p - in_len + 1
            assert p == in_len + r
            assert vis(wm[r]) == {(k, int(m[p, k])) for k in range(p + 1) if m[p, k]}
        else:                                                         # frame t's [MASK] row: the cached rows before p, and itself
            t = r - (T - 1)
            assert p == in_len + t
            if t < T - 1:                                             # the word at position p is pair row t: another key than row r
                assert int(rows[t]) == p and t != r
            assert vis(qm[t]) == {(k, int(m[p, k])) for k in range(p) if m[p, k]}


# ---------------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------------
_A = 1 << 16                                                         # fake, aligned device addresses: every call below fails validation


def _group_call(shape=None, T=20, G=2, P=102, n=2, x=_A, prefix=5 * _A, prefix_rows=102, wbits=2 * _A, qbits=3 * _A, acts_ptr=4 * _A,
                alias=False):
    s = shape or dict(B=4, Lq=121, Lkv=121, H=128, heads=2, I=256, kv_slots=0)
    acts = (_lib.VlpkLayerActs * max(n, 1))()
    for i in range(max(n, 1)):
        acts[i] = _lib.VlpkLayerActs(*([acts_ptr + (0 if alias else i) * _A] * len(_lib.ACT_FIELDS)))
    if alias:
        acts[0].y = x
    w = (_lib.VlpkLayerWeights * max(n, 1))(*[_lib.VlpkLayerWeights(*([7 * _A] * len(_lib.WEIGHT_FIELDS)))] * max(n, 1))
    caches = None if prefix is None else (C.c_void_p * max(n, 1))(*([prefix] * max(n, 1)))
    return _lib.lib().vlpk_encoder_score_group_fwd(_lib.VlpkShape(*s.values()), T, G, P, n, w, x, caches, prefix_rows, wbits, qbits, acts,
                                                   None)


def _core_call(B=4, G=2, heads=2, Lq=20, Lkv=121, P=102, q=_A, prefix=2 * _A, prefix_rows=102, text=3 * _A, T=39, ks=4 * _A, mask=5 * _A,
               kv_slots=0):
    H = heads * 64
    vs = None if ks is None else ks + H * 2
    return _lib.lib().vlpk_attn_core_group_self_fwd(B, G, heads, Lq, Lkv, P, q, 3 * H, 39 * 3 * H, prefix, prefix_rows, 2 * H, text, T, 3 * H,
                                                    ks, vs, mask, kv_slots, 6 * _A, H, 0, None, None)


def test_abi_rejects_bad_arguments_without_launching():
    lib = _lib.lib()
    for name in ("vlpk_encoder_score_group_fwd", "vlpk_encoder_score_group_workspace_bytes", "vlpk_attn_core_group_self_fwd"):
        assert name in _lib.EXPORTED_SYMBOLS
    before = lib.vlpk_launch_count()
    bad = [dict(T=0), dict(T=513), dict(G=3), dict(G=0), dict(P=0), dict(P=103), dict(P=101), dict(prefix_rows=101), dict(n=0),
           dict(x=None), dict(prefix=None), dict(wbits=None), dict(qbits=None), dict(acts_ptr=0), dict(x=_A + 2), dict(wbits=2 * _A + 4),
           dict(prefix=5 * _A + 8), dict(alias=True),
           dict(shape=dict(B=4, Lq=121, Lkv=120, H=128, heads=2, I=256, kv_slots=0)),
           dict(shape=dict(B=4, Lq=130, Lkv=130, H=128, heads=2, I=256, kv_slots=0)),
           dict(shape=dict(B=4, Lq=121, Lkv=121, H=64, heads=1, I=256, kv_slots=0)),
           dict(shape=dict(B=4, Lq=613, Lkv=613, H=128, heads=2, I=256, kv_slots=640), T=512, P=102),
           dict(shape=dict(B=0, Lq=121, Lkv=121, H=128, heads=2, I=256, kv_slots=0))]
    for b in bad:
        assert _group_call(**b) < 0, b
        assert lib.vlpk_last_error()
    for b in [dict(Lq=0), dict(Lq=513), dict(Lkv=0), dict(Lkv=129), dict(Lkv=200, kv_slots=128), dict(G=3), dict(P=0), dict(P=103),
              dict(Lkv=101), dict(T=18), dict(q=None), dict(prefix=None), dict(text=None), dict(text=3 * _A + 8), dict(ks=None),
              dict(ks=4 * _A + 4), dict(mask=None), dict(heads=0)]:
        assert _core_call(**b) < 0, b
    assert lib.vlpk_launch_count() == before


def test_workspace_bytes_match_the_python_buffers():
    from vlp_b200 import ops
    out = (C.c_size_t * 1)()
    B, S, T, H, heads, I = 6, 121, 20, 128, 2, 256
    assert _lib.lib().vlpk_encoder_score_group_workspace_bytes(_lib.VlpkShape(B, S, S, H, heads, I, 0), T, out) == 0
    acts = ops._Acts(1, B, 2 * T - 1, H, heads, I, "cpu")
    assert out[0] == acts.bf[0].numel() * 2 + acts.f32[0].numel() * 4
    M = B * (2 * T - 1)
    assert out[0] == 2 * M * (8 * H + 2 * I) + 4 * (math.ceil(B * heads * (2 * T - 1) / 4) * 4 + 4 * M)
    for t in (0, S + 1):
        assert _lib.lib().vlpk_encoder_score_group_workspace_bytes(_lib.VlpkShape(B, S, S, H, heads, I, 0), t, out) < 0


# ---------------------------------------------------------------------------------------------------------------------------
# model surface
# ---------------------------------------------------------------------------------------------------------------------------
def _matrix_refused(model, args, caps, grad=False, **kw):
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="vlp_b200"):
            with torch.set_grad_enabled(grad):
                model.score_caption_matrix(*args, caps, **kw)
    assert calls == []


def test_refusals_launch_nothing():
    model, args, T = _tiny()
    B = args[2].shape[0]
    ok = torch.randint(1, 50, (3, T))
    _matrix_refused(model, args, ok[:0])                                      # C < 1
    _matrix_refused(model, args, ok[:, :0])                                   # T < 1
    _matrix_refused(model, args, torch.randint(1, 50, (3, T + 1)))            # T > out_len - in_len
    _matrix_refused(model, args, ok.view(3, 1, T))                            # [C, T] only
    _matrix_refused(model, args, ok.view(-1))
    _matrix_refused(model, args, ok.int())                                    # dtype
    _matrix_refused(model, args, torch.full((3, T), 1000))                    # CPU ids outside [0, V)
    _matrix_refused(model, args, torch.full((3, T), -1))
    _matrix_refused(model, args, ok, grad=True)                               # grad mode with parameters that require grad
    for mr in (B * T - 1, 0, 2.0 * B * T, True):
        _matrix_refused(model, args, ok, max_rows=mr)                         # not one caption against every image
    bad = list(args)
    bad[2] = bad[2].int()
    _matrix_refused(model, tuple(bad), ok)
    for i, t in ((0, args[0][:, :-1]), (0, args[0].long()), (1, args[1][:1]), (4, args[4][:, :-1]), (5, args[5][:, :-1]),
                 (5, args[5].to(torch.complex64))):
        bad = list(args)
        bad[i] = t
        _matrix_refused(model, tuple(bad), ok)
    _refused(model, args, ok)                                                 # score_captions still wants [B, T] / [B, N, T]


def test_relaxed_head_refuses_a_missing_task_idx():
    from vlp_b200 import synth
    from vlp_b200 import vlp_modules as vm
    d = synth.TINY
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, relax_projection=4)
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=d.regions).bfloat16().eval()
    _, args, T = _tiny()
    caps = torch.randint(1, 50, (5, T))
    _matrix_refused(model, args, caps)
    _matrix_refused(model, args, caps, task_idx=torch.tensor([0, 4]))


@pytest.mark.parametrize("C,per_chunk", [(5, 2), (5, 5), (1, 1), (4, None)])
def test_call_sequence(C, per_chunk):
    """The prefix once (one cached layer call per layer, one mask), the word and query masks once, then per chunk of captions one
    embedding, one stack call and one head call; chunks of per_chunk captions, the last one ragged."""
    model, args, T = _tiny()
    B = args[2].shape[0]
    caps = torch.randint(1, 50, (C, T))
    with torch.no_grad(), abi_cases.dry_run() as calls:
        out = model.score_caption_matrix(*args, caps, max_rows=None if per_chunk is None else B * T * per_chunk)
    assert out.shape == (B, C, T) and out.dtype == torch.float32
    n_chunks = 1 if per_chunk is None else -(-C // per_chunk)
    layers = len(model.bert.encoder.layer)
    assert calls == (["vlpk_linear_fwd"] * 3 + ["vlpk_embed_fwd", "vlpk_mask_pack"] + ["vlpk_layer_cached_fwd"] * layers
                     + ["vlpk_mask_pack"] * 2 + ["vlpk_embed_fwd", "vlpk_encoder_score_group_fwd", "vlpk_decoder_ce_fwd"] * n_chunks)


def test_one_word_captions_pack_no_word_mask():
    model, args, _ = _tiny()
    with torch.no_grad(), abi_cases.dry_run() as calls:
        out = model.score_caption_matrix(*args, torch.randint(1, 50, (3, 1)))
    assert out.shape == (args[2].shape[0], 3, 1)
    assert calls.count("vlpk_mask_pack") == 2 and calls.count("vlpk_encoder_score_group_fwd") == 1
