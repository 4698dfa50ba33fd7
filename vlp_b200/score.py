"""Scoring given captions under BertForSeq2SeqDecoder: log p(c_t | image, c_<t) of every word in one teacher-forced pass of the
encoder instead of one decode frame per word.

Frame t of the reference's incremental decode (modeling.py:1210-1252) runs a [MASK] row at position p = in_len + t against the
cached rows at positions < p (prefix and the words c_0 .. c_{t-1}) and itself.  The words' keys and values never depend on a [MASK]
row, so one pass over the row layout

    rows [0, in_len)      prefix: [CLS] regions [SEP]        positions 0 .. in_len - 1
    rows [in_len, S)      words c_0 .. c_{T-2}                positions in_len .. S - 1      (S = in_len + T - 1)
    rows [S, S + T)       T query rows ([MASK])               positions in_len .. in_len + T - 1

gives every frame at once: prefix row i sees attention_mask[b, i, :in_len], the word row at position q sees attention_mask[b, q, :q + 1],
and the query row at position p sees attention_mask[b, p, :p] of the S shared rows plus its own key (vlpk_encoder_score_fwd).

This is the decode's computation whenever the prefix rows see no text column and no text row sees a later column, as in the
reference's decoder input (Preprocess4Seq2seqDecoder) and everything synth.py builds.  The condition is not checked on the device:
that would need a host synchronisation.
"""
import torch

from . import ops
from .decode import PAD_ID, expand_task_idx


MASK_DTYPES = (torch.int64, torch.int32, torch.bool, torch.float32, torch.bfloat16, torch.float16)


def layout(in_len, T, device=None):
    """The scoring layout as (S, positions, shared_keep, query_keep), built on `device`: positions [S + T] is the decode position of
    every row; shared_keep [S, S] and query_keep [T, S] are True where a row may see a shared key column, before the attention mask
    applies (prefix rows: the prefix; the word at position q: positions <= q; the query row at position p: positions < p)."""
    S = in_len + T - 1
    j = torch.arange(S, device=device)
    t = torch.arange(T, device=device)
    return S, torch.cat((j, in_len + t)), (j <= j.unsqueeze(1)) | (j < in_len), j < (in_len + t).unsqueeze(1)


def check_score(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids, task_idx):
    """Raises ValueError, before anything is launched, for inputs score_captions does not take."""
    dec.cls.predictions.check_task_idx(task_idx)
    for t, what in ((input_ids, "input_ids"), (token_type_ids, "token_type_ids"), (position_ids, "position_ids"),
                    (caption_ids, "caption_ids")):
        if not torch.is_tensor(t) or t.dtype != torch.int64:
            raise ValueError(f"vlp_b200: score_captions takes int64 {what}, got {getattr(t, 'dtype', type(t).__name__)}")
    if input_ids.dim() != 2:
        raise ValueError(f"vlp_b200: input_ids must be [B, in_len], got {tuple(input_ids.shape)}")
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[-1]
    if token_type_ids.shape != (B, out_len) or position_ids.shape != (B, out_len) or not torch.is_tensor(attention_mask) \
            or attention_mask.shape != (B, out_len, out_len):
        raise ValueError(f"vlp_b200: score_captions needs token_type_ids / position_ids [B, out_len] and attention_mask [B, out_len, out_len] "
                         f"for B={B}")
    if attention_mask.dtype not in MASK_DTYPES:
        raise ValueError(f"vlp_b200: score_captions takes a 0/1 attention_mask of one of {MASK_DTYPES}, got {attention_mask.dtype}")
    R = dec.len_vis_input
    for t, what, width in ((vis_feats, "vis_feats", dec.vis_embed[0].in_features), (vis_pe, "vis_pe", dec.vis_pe_embed[0].in_features)):
        if not torch.is_tensor(t) or not t.is_floating_point() or t.shape != (B, R, width):
            raise ValueError(f"vlp_b200: score_captions needs floating-point {what} [B={B}, {R}, {width}], got "
                             f"{getattr(t, 'dtype', type(t).__name__)} {tuple(getattr(t, 'shape', ()))}")
    if caption_ids.dim() not in (2, 3) or caption_ids.shape[0] != B:
        raise ValueError(f"vlp_b200: caption_ids must be [B, T] or [B, N, T] with B={B}, got {tuple(caption_ids.shape)}")
    T = caption_ids.shape[-1]
    if not 1 <= T <= out_len - in_len or (caption_ids.dim() == 3 and caption_ids.shape[1] < 1):
        raise ValueError(f"vlp_b200: caption length T={T} must lie in [1, out_len - in_len = {out_len - in_len}]")
    V = dec.config.vocab_size
    if not caption_ids.is_cuda and caption_ids.numel():
        lo, hi = int(caption_ids.min()), int(caption_ids.max())
        if lo < 0 or hi >= V:
            raise ValueError(f"vlp_b200: caption ids must lie in [0, {V}), got [{lo}, {hi}]")
    if torch.is_grad_enabled() and any(p.requires_grad for p in dec.parameters()):
        raise ValueError("vlp_b200: score_captions is an inference-only path; wrap it in torch.no_grad()")
    return B, in_len, out_len, T


def score_captions(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids, task_idx=None):
    """fp32 logp shaped like caption_ids: logp[..., t] = log p(c_t | image, c_<t) under the full softmax of the MLM head (bias and
    the relaxed head's task_idx included), the quantity frame t of the decode computes for its [MASK] row when fed c_0 .. c_{t-1}.
    [EOS] is scored like any other word; entries at and after the first 0 are 0.  A device-resident id outside [0, V) is read as 0
    (it ends the caption there); CPU ids are range-checked instead.  No host synchronisation."""
    hidden, cap, task_idx = query_states(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids,
                                         task_idx)
    with torch.no_grad():
        logp = head_logp(dec, hidden, cap, task_idx)
    return logp.view(caption_ids.shape)


def query_states(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids, task_idx=None):
    """The checks and the encoder pass of score_captions: (the T query rows' last hidden states [B * N, T, H], the captions as read
    [B * N, T], task_idx per row)."""
    B, in_len, out_len, T = check_score(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids,
                                        task_idx)
    N = caption_ids.shape[1] if caption_ids.dim() == 3 else 1
    dev = input_ids.device
    V = dec.config.vocab_size
    cap = caption_ids.to(dev).reshape(B * N, T)
    cap = torch.where((cap < 0) | (cap >= V), PAD_ID, cap)
    if N > 1:
        rep = lambda x: x.repeat_interleave(N, 0)
        vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask = map(
            rep, (vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask))
        task_idx = expand_task_idx(task_idx, B, N)
    S, positions, shared_keep, query_keep = layout(in_len, T, dev)
    with torch.no_grad():
        vis, vpe = dec.project_regions(vis_feats, vis_pe)
        ids = torch.cat((input_ids, cap[:, :T - 1], cap[:, :T] * 0 + dec.mask_word_id), dim=1)
        emb = dec.bert.embeddings(vis, vpe, ids, token_type_ids.index_select(1, positions), position_ids.index_select(1, positions),
                                  len_vis_input=dec.len_vis_input)
        m = attention_mask
        shared_bits = ops.pack_mask(m[:, :S, :S] * shared_keep.to(m.dtype), "zero_one")
        query_bits = ops.pack_mask(m[:, in_len:in_len + T, :S] * query_keep.to(m.dtype), "zero_one")
        params = [p for layer in dec.bert.encoder.layer for p in layer.flat_params()]
        cfg = dec.config
        out, _ = ops.encoder_score_fwd(emb, shared_bits, query_bits, T, cfg.num_attention_heads, cfg.intermediate_size, params)
    return out[:, S:], cap, task_idx


def head_logp(dec, hidden, cap, task_idx=None):
    """[rows, T] fp32 log-probabilities of the words cap [rows, T] (ids in [0, V)) under the MLM head at the query rows' last hidden
    states hidden [rows, T, H]: transform, the relaxed head's task slice, and the fused decoder + log-softmax (label 0 and everything
    after the first 0 give 0)."""
    pred = dec.cls.predictions
    h = pred.select_task(pred.transform(hidden.to(pred.decoder.weight.dtype)), task_idx)
    valid = (cap != PAD_ID).cumprod(1).bool()
    labels = torch.where(valid, cap, -1)                          # outside [0, V): the head's ignored position, loss 0
    loss, _ = ops.DecoderCEFn.apply(h.reshape(cap.numel(), -1), pred.decoder.weight, pred.bias, labels.reshape(-1))
    return torch.where(valid, -loss.view(cap.shape), 0.0)
