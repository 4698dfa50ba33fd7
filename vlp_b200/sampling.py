"""Top-k and top-p (nucleus) sampling decode for BertForSeq2SeqDecoder, on the device.

`sampling_method="topk"` keeps the `topk` most likely words of every step, `"topp"` the smallest set whose probability reaches
`topp`; one word is drawn from the kept set, renormalised.  The loop is the greedy one (beam size 1, the per-layer K/V caches when
`dec.use_kv_cache`); only the word choice differs: the head's decoder runs without its bias and one vlpk_sample_tokens launch per
step adds the bias, applies the duplicate-n-gram blocking of beam search (`forbid_duplicate_ngrams`, `ngram_size`,
`forbid_ignore_set`) and the `min_len` [EOS] block, selects and draws — no logits leave the device and nothing synchronises with
the host.

Words are ranked by (logit descending, index ascending), so ties are broken towards the lower id: `topk=1` and `topp` -> 0 are the
greedy arg-max.  The uniform of row r at step t comes from a Philox counter keyed by (seed; t, r): a decode is reproducible for a
seed whatever the batch around the row, and the same seed gives the same uniforms to every batch — pass another seed (the `seed`
argument of forward, or `dec.seed`) for independent draws.

Output: (ids, scores), int64 / fp32 [B, out_len - in_len]: the sampled words and their log-probabilities under the full softmax
(and the per-frame attention maps with output_attentions).  With num_return_sequences N > 1: [B, N, out_len - in_len], sample j of
image b drawn as row b * N + j of the batch repeated N times, over one K/V cache of each image's prefix (shared_prefix.py).
A row that draws [EOS] is finished; its later positions hold PAD_ID with score 0.  Outside CUDA-graph capture the loop also stops
once every row is finished: each step copies the device's count of live rows to pinned host memory and the loop reads it once
the copy's event has completed (a non-blocking query, never a synchronisation), so it stops a step or two after the last [EOS].
"""
import torch

from . import ops
from .beam import _ignore_tensor
from .shared_prefix import SharedPrefixCache

SAMPLING_METHODS = ("beam_search", "topk", "topp")
PAD_ID = 0


def check_sampling_args(sampling_method, topk, topp, search_beam_size):
    """Raises ValueError before any launch for a sampling configuration the kernel does not take."""
    if sampling_method not in SAMPLING_METHODS:
        raise ValueError(f"vlp_b200: sampling_method must be one of {', '.join(SAMPLING_METHODS)}, got {sampling_method!r}")
    if sampling_method == "beam_search":
        return
    if int(search_beam_size) != 1:
        raise ValueError(f"vlp_b200: sampling_method={sampling_method!r} needs beam size 1, got {search_beam_size}")
    if sampling_method == "topk":
        if isinstance(topk, bool) or not isinstance(topk, int) or not 1 <= topk <= ops.MAX_TOPK:
            raise ValueError(f"vlp_b200: topk must be an integer in [1, {ops.MAX_TOPK}], got {topk!r}")
    elif isinstance(topp, bool) or not isinstance(topp, (int, float)) or not 0.0 < float(topp) <= 1.0:
        raise ValueError(f"vlp_b200: topp must lie in (0, 1], got {topp!r}")


def sample_decode(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, task_idx=None, seed=None,
                  output_attentions=False):
    """output_attentions: (ids, scores, attentions), attentions as for greedy decode (BertForSeq2SeqDecoder.forward); frames after an
    early stop stay 0."""
    check_sampling_args(dec.sampling_method, dec.topk, dec.topp, dec.search_beam_size)
    if dec.forbid_duplicate_ngrams and int(dec.ngram_size) < 1:
        raise ValueError(f"vlp_b200: forbid_duplicate_ngrams needs ngram_size >= 1 (got {dec.ngram_size})")
    seed = dec.seed if seed is None else seed
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[1]
    T = out_len - in_len
    dev = input_ids.device
    ngram = int(dec.ngram_size) if dec.forbid_duplicate_ngrams else 0
    ignore = _ignore_tensor(dec, dev) if ngram else None
    pred = dec.cls.predictions
    # N > 1: row b * N + j is sample j of image b, drawn exactly as row b * N + j of the batch repeated with repeat_interleave(N)
    N = getattr(dec, "num_return_sequences", 1)
    R = B * N
    ids = torch.full((R, T), PAD_ID, dtype=torch.int64, device=dev)
    scores = torch.zeros(R, T, dtype=torch.float32, device=dev)
    finished = torch.zeros(R, dtype=torch.int32, device=dev)
    live = torch.full((1,), R, dtype=torch.int32, device=dev)
    poll = None
    if dev.type == "cuda" and not torch.cuda.is_current_stream_capturing():
        poll, polled = torch.empty(1, dtype=torch.int32, pin_memory=True), None
    if N > 1:
        caches = SharedPrefixCache(len(dec.bert.encoder.layer), B, N, in_len, T, dec.config.hidden_size, dev)
        if torch.is_tensor(task_idx) and task_idx.dim() == 1 and task_idx.shape[0] == B:
            task_idx = task_idx.repeat_interleave(N)                  # per-sample ids follow their samples (relaxed head)
    else:
        caches = dec.new_kv_caches(B, dev, out_len) if dec.use_kv_cache else None
    maps = dec.new_attention_maps(B, T, out_len, dev) if output_attentions else None
    prev_emb, prev_layers = None, None
    curr_ids = input_ids
    mask_ids = input_ids[:, :1] * 0 + dec.mask_word_id
    next_pos = in_len
    dec.last_decode_steps = 0
    while next_pos < out_len:
        if poll is not None and polled is not None and polled.query():
            if int(poll[0]) == 0:
                break                                                  # every row has drawn [EOS]: the rest stays padding
            polled = None
        cl = curr_ids.shape[1]
        st = next_pos - cl
        x_ids = torch.cat((curr_ids, mask_ids), dim=1)
        extra = {} if maps is None else {"output_attentions": dec.step_maps(maps[:, next_pos - in_len], cl, next_pos + 1)}
        if caches is not None:
            new_emb, last = dec.bert(vis_feats, vis_pe, x_ids, token_type_ids[:, st:next_pos + 1], position_ids[:, st:next_pos + 1],
                                     attention_mask[:, st:next_pos + 1, :next_pos + 1], output_all_encoded_layers=False,
                                     len_vis_input=dec.len_vis_input, kv_caches=caches, cache_pos=st, **extra)[:2]
            new_layers = [last]
        else:
            new_emb, new_layers = dec.bert(vis_feats, vis_pe, x_ids, token_type_ids[:, st:next_pos + 1], position_ids[:, st:next_pos + 1],
                                           attention_mask[:, st:next_pos + 1, :next_pos + 1], prev_embedding=prev_emb,
                                           prev_encoded_layers=prev_layers, output_all_encoded_layers=True, len_vis_input=dec.len_vis_input,
                                           **extra)[:2]
        last = new_layers[-1][:, -1:, :]
        if N > 1 and next_pos == in_len:
            # the prefill ran at B images: its [MASK] row feeds the head at B*N rows, the row count of the repeated batch, and from
            # here on every input is per sample (the attention mask stays per image: the shared cache reads it so).  The rows keep
            # the prefill output's row stride too, as a slice of the repeated batch's output would: the head's GEMMs pick their
            # kernels by shape and strides, and a contiguous copy rounds differently at BERT-base sizes.
            full = last.new_empty(R, in_len + 1, last.shape[2])
            full[:, -1:] = last.repeat_interleave(N, 0)
            last = full[:, -1:]
            token_type_ids, position_ids = token_type_ids.repeat_interleave(N, 0), position_ids.repeat_interleave(N, 0)
            mask_ids = mask_ids.repeat_interleave(N, 0)
        h = pred.select_task(pred.transform(last.to(pred.decoder.weight.dtype)), task_idx)
        logits = pred.decoder(h)                                       # [R, 1, V]; the bias is added inside the sampling kernel
        frame = next_pos - in_len
        ops.sample_tokens(logits, pred.bias.to(logits.dtype), dec.sampling_method, dec.topk, dec.topp, seed, frame, ids, scores, finished,
                          live, dec.eos_id, PAD_ID, block_eos=bool(dec.min_len) and frame + 1 <= dec.min_len, ngram=ngram, ignore=ignore)
        if poll is not None and polled is None:
            poll.copy_(live, non_blocking=True)
            polled = torch.cuda.Event()
            polled.record()
        if caches is None:
            if prev_emb is None:
                prev_emb, prev_layers = new_emb[:, :-1, :], [x[:, :-1, :] for x in new_layers]
            else:
                prev_emb = torch.cat((prev_emb, new_emb[:, :-1, :]), dim=1)
                prev_layers = [torch.cat((a, b[:, :-1, :]), dim=1) for a, b in zip(prev_layers, new_layers)]
        curr_ids = ids[:, frame:frame + 1]
        next_pos += 1
        dec.last_decode_steps += 1
    if N > 1:
        return ids.view(B, N, T), scores.view(B, N, T)
    return (ids, scores) if maps is None else (ids, scores, maps)
