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

The caption matrix (score_caption_matrix: C shared captions against each of B images) splits the same rows by what they depend on.
The prefix rows depend on the image alone, so they run once per image (prefix_caches: layer by layer, keeping each layer's K | V of
the P = in_len prefix rows in a [B, P, 2H] cache).  Each (image, caption) pair keeps only its 2T - 1 caption rows

    rows [0, T - 1)       words c_0 .. c_{T-2}                positions in_len .. S - 1
    rows [T - 1, 2T - 1)  T query rows ([MASK])               positions in_len .. in_len + T - 1

whose keys are [the image's prefix cache | the pair's words] (vlpk_encoder_score_group_fwd): row for row, key for key, the rows and
visibility of the layout above.  The masks are packed once per image and shared by its pairs.
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


def check_score(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids, task_idx, shared=False):
    """Raises ValueError, before anything is launched, for inputs score_captions (shared: score_caption_matrix, captions [C, T] shared
    by the images) does not take."""
    fn = "score_caption_matrix" if shared else "score_captions"
    dec.cls.predictions.check_task_idx(task_idx)
    for t, what in ((input_ids, "input_ids"), (token_type_ids, "token_type_ids"), (position_ids, "position_ids"),
                    (caption_ids, "caption_ids")):
        if not torch.is_tensor(t) or t.dtype != torch.int64:
            raise ValueError(f"vlp_b200: {fn} takes int64 {what}, got {getattr(t, 'dtype', type(t).__name__)}")
    if input_ids.dim() != 2:
        raise ValueError(f"vlp_b200: input_ids must be [B, in_len], got {tuple(input_ids.shape)}")
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[-1]
    if token_type_ids.shape != (B, out_len) or position_ids.shape != (B, out_len) or not torch.is_tensor(attention_mask) \
            or attention_mask.shape != (B, out_len, out_len):
        raise ValueError(f"vlp_b200: {fn} needs token_type_ids / position_ids [B, out_len] and attention_mask [B, out_len, out_len] "
                         f"for B={B}")
    if attention_mask.dtype not in MASK_DTYPES:
        raise ValueError(f"vlp_b200: {fn} takes a 0/1 attention_mask of one of {MASK_DTYPES}, got {attention_mask.dtype}")
    R = dec.len_vis_input
    for t, what, width in ((vis_feats, "vis_feats", dec.vis_embed[0].in_features), (vis_pe, "vis_pe", dec.vis_pe_embed[0].in_features)):
        if not torch.is_tensor(t) or not t.is_floating_point() or t.shape != (B, R, width):
            raise ValueError(f"vlp_b200: {fn} needs floating-point {what} [B={B}, {R}, {width}], got "
                             f"{getattr(t, 'dtype', type(t).__name__)} {tuple(getattr(t, 'shape', ()))}")
    if shared:
        if caption_ids.dim() != 2 or caption_ids.shape[0] < 1:
            raise ValueError(f"vlp_b200: caption_ids must be [C, T] with C >= 1 captions, got {tuple(caption_ids.shape)}")
    elif caption_ids.dim() not in (2, 3) or caption_ids.shape[0] != B:
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
        raise ValueError(f"vlp_b200: {fn} is an inference-only path; wrap it in torch.no_grad()")
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


MATRIX_MAX_ROWS = 65536
"""Default head rows (B * captions per chunk * T) of one score_caption_matrix chunk.  At BERT-base (H 768, I 3072, V 29 000) a chunk
then holds about 3.8 GB of bf16 logits and 6 GB of encoder activations (two buffers of B * chunk * (2T - 1) rows), about 10 GB in all."""


def matrix_masks(attention_mask, in_len, T):
    """The caption matrix's 0/1 masks, one sequence per image, keys [prefix | the pair's words] (key k at position k): the prefix rows
    [B, P, P], the word rows [B, T - 1, S] and the query rows [B, T, S] (each query row also sees its own key), S = in_len + T - 1;
    the rows of layout's shared and query masks."""
    S, _, shared_keep, query_keep = layout(in_len, T, attention_mask.device)
    m = attention_mask
    return (m[:, :in_len, :in_len], m[:, in_len:S, :S] * shared_keep[in_len:].to(m.dtype),
            m[:, in_len:in_len + T, :S] * query_keep.to(m.dtype))


def prefix_caches(dec, vis, vpe, input_ids, token_type_ids, position_ids, attention_mask):
    """Per-layer K | V caches [B, P, 2H] bf16 of the B images' P = in_len prefix rows (region features already projected): the rows
    run through every layer once, under attention_mask[b, :P, :P] (vlpk_layer_cached_fwd at pos 0)."""
    B, P = input_ids.shape
    cfg = dec.config
    emb = dec.bert.embeddings(vis, vpe, input_ids, token_type_ids[:, :P], position_ids[:, :P], len_vis_input=dec.len_vis_input)
    bits = ops.pack_mask(matrix_masks(attention_mask, P, 1)[0], "zero_one")
    caches, h = [], emb
    for layer in dec.bert.encoder.layer:
        caches.append(torch.empty(B, P, 2 * cfg.hidden_size, device=emb.device, dtype=torch.bfloat16))
        h = ops.layer_cached_fwd(h, caches[-1], 0, bits, cfg.num_attention_heads, cfg.intermediate_size, layer.flat_params())
    return caches


def score_caption_matrix(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids, task_idx=None,
                         max_rows=None):
    """fp32 [B, C, T]: out[b, c, t] = log p(c_t | image b, c_<t) for the C captions caption_ids [C, T] shared by the B images, what
    score_captions gives image b with caption c ([EOS] scored like any word, 0 at and after the first 0, a device id outside [0, V)
    read as 0).  The prefix rows run once per image; each (image, caption) pair adds its 2T - 1 caption rows.  Captions go in chunks
    of max_rows // (B * T) (default MATRIX_MAX_ROWS head rows per chunk) that reuse the prefix caches.  task_idx is per image.  No
    host synchronisation."""
    B, C, T, chunks = matrix_query_states(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids,
                                          task_idx, max_rows)
    out = torch.empty(B, C, T, device=input_ids.device, dtype=torch.float32)
    with torch.no_grad():
        for c0, G, hidden, cap, task in chunks:
            out[:, c0:c0 + G] = head_logp(dec, hidden, cap, task).view(B, G, T)
    return out


def matrix_query_states(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids, task_idx=None,
                        max_rows=None):
    """The checks and the encoder passes of score_caption_matrix: (B, C, T, chunks), the checks done before it returns.  Iterating
    chunks runs the prefix once, then one chunk of G captions at a time and yields (c0, G, the query rows' last hidden states
    [B * G, T, H] of pairs (image i // G, caption c0 + i % G), their captions as read [B * G, T], task_idx per pair)."""
    B, in_len, out_len, T = check_score(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caption_ids,
                                        task_idx, shared=True)
    max_rows = MATRIX_MAX_ROWS if max_rows is None else max_rows
    if isinstance(max_rows, bool) or not isinstance(max_rows, int) or max_rows < B * T:
        raise ValueError(f"vlp_b200: max_rows must be an int >= B * T = {B * T} (one caption against every image), got {max_rows!r}")
    C = caption_ids.shape[0]
    chunk = min(C, max_rows // (B * T))

    def chunks():
        dev = input_ids.device
        V = dec.config.vocab_size
        cap = caption_ids.to(dev)
        cap = torch.where((cap < 0) | (cap >= V), PAD_ID, cap)
        rows = layout(in_len, T, dev)[1][in_len:]                  # a pair's rows: its words, then its query rows
        cfg = dec.config
        params = [p for layer in dec.bert.encoder.layer for p in layer.flat_params()]
        with torch.no_grad():
            vis, vpe = dec.project_regions(vis_feats, vis_pe)
            caches = prefix_caches(dec, vis, vpe, input_ids, token_type_ids, position_ids, attention_mask)
            _, word_mask, query_mask = matrix_masks(attention_mask, in_len, T)
            word_bits = ops.pack_mask(word_mask, "zero_one") if T > 1 else None
            query_bits = ops.pack_mask(query_mask, "zero_one")
            tt, pos = token_type_ids.index_select(1, rows), position_ids.index_select(1, rows)
            for c0 in range(0, C, chunk):
                G = min(chunk, C - c0)
                pc = cap[c0:c0 + G].unsqueeze(0).expand(B, G, T).reshape(B * G, T)
                ids = torch.cat((pc[:, :T - 1], pc * 0 + dec.mask_word_id), dim=1)
                emb = dec.bert.embeddings(None, None, ids, tt.repeat_interleave(G, 0), pos.repeat_interleave(G, 0), vis_input=False,
                                          len_vis_input=dec.len_vis_input)
                y, _ = ops.encoder_score_group_fwd(emb, caches, word_bits, query_bits, T, G, cfg.num_attention_heads,
                                                   cfg.intermediate_size, params)
                yield c0, G, y[:, T - 1:], pc, expand_task_idx(task_idx, B, G)
    return B, C, T, chunks()
