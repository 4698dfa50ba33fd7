"""Beam search for BertForSeq2SeqDecoder (semantics of the reference's modeling.py:1256-1494).

Same algorithm and return format (a `traces` dict of padded tensors: pred_seq, scores, wids, ptrs), with ALL beam
bookkeeping on the device — top-k, back pointers (integer floor division: the reference's `torch.div(k_ids, K)`, :1317, yields
floats on torch >= 1.6 and breaks `gather`, SURVEY.md §2 #7), the per-layer K/V caches reordered by the back pointers, and the final
best-hypothesis selection + back-tracking (:1431-1472) as vectorised tensor ops, and the optional duplicate-n-gram blocking
(`forbid_duplicate_ngrams`, :1375-1428) as one vlpk_beam_ngram_block launch per frame over per-hypothesis word histories held on the
device: no host synchronisation inside or after the loop, so a blocked decode can be captured as a CUDA graph too.
Per-sample `task_idx` (the relaxed MLM head, relax_projection > 1) is expanded to the B*K beam rows with the other inputs; the
reference does not expand it (:1297 vs :1325-1373), so its relaxed beam search only runs at B = 1.
Every step runs the fused layers on the two new rows (token, [MASK]) against the K/V caches (`dec.use_kv_cache`), or — reference
data flow — against the re-encoded prefix.
"""
import math

import torch
import torch.nn.functional as F

from . import ops
from .shared_prefix import SharedPrefixCache


def _expand_beams(x, K):
    """[B, ...] -> [B*K, ...], each item repeated K times consecutively (reference first_expand, :1326-1333)."""
    return x.unsqueeze(1).expand(x.shape[0], K, *x.shape[1:]).reshape(x.shape[0] * K, *x.shape[1:])


def _reorder(x, back_ptrs, B, K):
    """Select, per batch item, the K parent beams named by back_ptrs [B,K] (reference select_beam_items, :1335-1350)."""
    xs = x.view(B, K, *x.shape[1:])
    idx = back_ptrs.view(B, K, *([1] * (x.dim() - 1))).expand(B, K, *x.shape[1:])
    return torch.gather(xs, 1, idx).reshape(x.shape)


def _dup_ngram_candidates(seq, n, ignore):
    """Words that would complete an n-gram already present in seq (reference get_dup_ngram_candidates, :1390-1406).  The rule the
    vlpk_beam_ngram_block kernel implements, kept as the host statement the tests compare against.  As in the reference, the ignore
    test looks at seq[-(n-1):] — all of seq when n = 1 — while each match compares n - 1 words (none when n = 1)."""
    if len(seq) < n:
        return []
    tail = seq[-(n - 1):]
    if ignore and any(t in ignore for t in tail):
        return []
    out = set()
    for i in range(len(seq) - (n - 1)):
        if seq[i:i + n - 1] == seq[len(seq) - (n - 1):] and not (ignore and seq[i + n - 1] in ignore):
            out.add(seq[i + n - 1])
    return sorted(out)


def _ignore_tensor(dec, dev):
    """The decoder's forbid_ignore_set as an int32 device tensor (None when empty), built once per distinct set and device and kept on
    the decoder for its lifetime: the first call (a CUDA graph's warm-up) makes the host-to-device copy, so a capture never does, and
    a graph captured with one set keeps reading a live tensor after decodes with other sets."""
    key = (tuple(sorted(int(w) for w in dec.forbid_ignore_set or ())), str(dev))
    cache = dec.__dict__.setdefault("_ngram_ignore_cache", {})
    if key not in cache:
        cache[key] = torch.tensor(key[0], dtype=torch.int32, device=dev) if key[0] else None
    return cache[key]


def check_ngram_args(dec):
    """Raises before any launch for an n-gram size the blocking rule does not define."""
    if dec.forbid_duplicate_ngrams and dec.search_beam_size > 1 and int(dec.ngram_size) < 1:
        raise ValueError(f"vlp_b200: forbid_duplicate_ngrams needs ngram_size >= 1 (got {dec.ngram_size})")


def beam_search(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, task_idx=None, output_attentions=False):
    """output_attentions: out["attentions"] [B, out_len - in_len, layers, heads, out_len] holds, for frame t of pred_seq, the [MASK]-row
    maps of step t taken from the row its hypothesis continued (beam_maps)."""
    K = dec.search_beam_size
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[1]
    dev = input_ids.device
    prev_emb, prev_layers = None, None
    N = getattr(dec, "num_return_sequences", 1)
    shared = None
    if N > 1:           # the K hypotheses of an image share its prefix K/V; a reorder moves slot-table entries, not cache rows
        caches = shared = SharedPrefixCache(len(dec.bert.encoder.layer), B, K, in_len, out_len - in_len, dec.config.hidden_size, dev)
    else:
        caches = dec.new_kv_caches(B, dev, out_len) if getattr(dec, "use_kv_cache", False) else None
    curr_ids = input_ids
    mask_ids = input_ids[:, :1] * 0 + dec.mask_word_id
    total_scores, beam_eos, step_ids, step_ptrs = [], [], [], []
    if dec.forbid_duplicate_ngrams:
        check_ngram_args(dec)
        ngram, ignore = int(dec.ngram_size), _ignore_tensor(dec, dev)
        hist = [torch.empty(B * K, out_len - in_len, dtype=torch.int32, device=dev) for _ in range(2)]    # word histories, in turn
    # per step t, the [MASK]-row maps of its B*K input rows (step 0: B rows, written at rows b*K)
    maps = dec.new_attention_maps(out_len - in_len, B * K, out_len, dev) if output_attentions else None
    next_pos = in_len
    while next_pos < out_len:
        cl = curr_ids.shape[1]
        st = next_pos - cl
        x_ids = torch.cat((curr_ids, mask_ids), dim=1)
        extra = {}
        if maps is not None:
            buf = maps[next_pos - in_len]
            buf = buf.view(B, K, *buf.shape[1:])[:, 0] if next_pos == in_len else buf
            extra["output_attentions"] = dec.step_maps(buf, cl, next_pos + 1)
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
        scores, _ = dec.cls(new_layers[-1][:, -1:, :], None, task_idx=task_idx)
        logp = F.log_softmax(scores.float(), dim=-1)                      # [B or B*K, 1, V]
        frame = next_pos - in_len
        if dec.forbid_duplicate_ngrams and frame >= 1:
            # history of frame `frame` from the previous frame's words and back pointers; blocks in place once it holds n words
            ops.beam_ngram_block(hist[(frame - 1) % 2], hist[frame % 2], step_ptrs[-1], step_ids[-1], frame, ngram, ignore, logp)
        if dec.min_len and (next_pos - in_len + 1 <= dec.min_len):
            logp[:, :, dec.eos_id] = -10000.0
        kk_scores, kk_ids = torch.topk(logp, k=K)                          # [*, 1, K]
        first = (next_pos == in_len)
        if first:
            k_ids = kk_ids.reshape(B, K)
            back = torch.zeros(B, K, dtype=torch.long, device=dev)
            k_scores = kk_scores.reshape(B, K)
        else:
            kk_scores = kk_scores + beam_eos[-1].reshape(B * K, 1, 1) * -10000.0 + total_scores[-1].reshape(B * K, 1, 1)
            k_scores, flat = torch.topk(kk_scores.reshape(B, K * K), k=K)
            back = torch.div(flat, K, rounding_mode="floor")
            k_ids = torch.gather(kk_ids.reshape(B, K * K), 1, flat)
        step_ptrs.append(back)
        step_ids.append(k_ids)
        beam_eos.append((k_ids == dec.eos_id).float())
        total_scores.append(k_scores)
        if first:
            if shared is not None:
                pass                                                       # the attention mask stays per image, as the shared cache reads it
            elif caches is not None:
                caches = [_expand_beams(c, K).contiguous() for c in caches]
            else:
                prev_emb = _expand_beams(new_emb[:, :-1, :], K)
                prev_layers = [_expand_beams(x[:, :-1, :], K) for x in new_layers]
            token_type_ids, position_ids = _expand_beams(token_type_ids, K), _expand_beams(position_ids, K)
            attention_mask = attention_mask if shared is not None else _expand_beams(attention_mask, K)
            mask_ids = _expand_beams(mask_ids, K)
            if torch.is_tensor(task_idx) and task_idx.dim() == 1 and task_idx.shape[0] == B:
                task_idx = _expand_beams(task_idx, K)                      # per-sample ids follow their beams (relaxed head)
        elif shared is not None:
            shared.reorder((back + torch.arange(B, device=dev).unsqueeze(1) * K).reshape(-1), frame - 1)
        elif caches is not None:
            parent = (back + torch.arange(B, device=dev).unsqueeze(1) * K).reshape(-1)      # beam i continues hypothesis parent[i]
            caches = [c.index_select(0, parent) for c in caches]
        else:
            prev_emb = _reorder(torch.cat((prev_emb, new_emb[:, :-1, :]), dim=1), back, B, K)
            prev_layers = [_reorder(torch.cat((a, b[:, :-1, :]), dim=1), back, B, K) for a, b in zip(prev_layers, new_layers)]
        curr_ids = k_ids.reshape(B * K, 1)
        next_pos += 1

    sc, wi, pt = torch.stack(total_scores), torch.stack(step_ids), torch.stack(step_ptrs)
    out = {"pred_seq": backtrack(sc, wi, pt, dec.eos_id, dec.length_penalty, out_len)}
    if maps is not None:
        out["attentions"] = beam_maps(maps, *best_path(sc, wi, pt, dec.eos_id, dec.length_penalty), pt)
    T = len(total_scores)
    for k, t in (("scores", torch.stack(total_scores)), ("wids", torch.stack(step_ids)), ("ptrs", torch.stack(step_ptrs))):
        padded = t.new_zeros((B, out_len, K))
        padded[:, :T] = t.permute(1, 0, 2)
        out[k] = padded
    if N > 1:
        out["nbest_seq"], out["nbest_scores"] = nbest(sc, wi, pt, dec.eos_id, dec.length_penalty, out_len, N)
    return out


def backtrack(sc, wi, pt, eos_id, length_penalty, out_len):
    """Best-hypothesis selection + back-tracking, same rule as the reference (:1431-1472), vectorised (runs wherever the traces live):
      last[b]   = first frame whose K words are all [EOS] (else the final frame)
      candidate = (word is [EOS], or frame == last[b]) within frames <= last[b]; score + length_penalty * (frame + 1); FIRST maximum wins
    sc [T,B,K] float scores, wi [T,B,K] word ids, pt [T,B,K] back pointers -> pred_seq [B, out_len] (zero padded)."""
    T, B, K = sc.shape
    active, pos = best_path(sc, wi, pt, eos_id, length_penalty)
    pred = torch.zeros(B, out_len, dtype=torch.long, device=sc.device)
    tok = wi.gather(2, pos.unsqueeze(-1)).squeeze(-1)                    # [T,B]
    pred[:, :T] = torch.where(active, tok, torch.zeros_like(tok)).t()
    return pred


def beam_maps(maps, active, pos, pt):
    """Attention maps of the chosen hypotheses: frame t of sample b takes row b*K + pt[t, b, pos[t, b]] of step t — the hypothesis
    that the frame-t word continued, whose [MASK] row predicted it.  maps [T, B*K, ...] per-step maps, active / pos [T,B] of
    best_path, pt [T,B,K] back pointers -> [B, T, ...], zero at frames past the hypothesis' end."""
    T, B, K = pt.shape
    rows = pt.gather(2, pos.unsqueeze(-1)).squeeze(-1) + torch.arange(B, device=pt.device) * K        # [T,B]
    got = maps[torch.arange(T, device=pt.device).unsqueeze(1), rows]                                  # [T,B,...]
    keep = active.view(T, B, *([1] * (got.dim() - 2)))
    return torch.where(keep, got, torch.zeros_like(got)).transpose(0, 1)


def candidate_values(sc, wi, eos_id, length_penalty):
    """The final-selection rule's value of every (frame, beam), [B, T*K] in (frame, beam) order — the reference's loop order: score +
    length_penalty * (frame + 1) for a candidate ([EOS] word, or the last frame, within frames <= last[b]), -inf otherwise."""
    T, B, K = sc.shape
    dev = sc.device
    frames = torch.arange(T, device=dev).view(T, 1)
    all_eos = (wi == eos_id).all(-1)                                      # [T,B]
    last = torch.where(all_eos.any(0), all_eos.float().argmax(0), torch.full((B,), T - 1, device=dev))      # [B]
    cand = (frames <= last.unsqueeze(0)).unsqueeze(-1) & ((wi == eos_id) | (frames == last.unsqueeze(0)).unsqueeze(-1))
    val = torch.where(cand, sc + length_penalty * (frames + 1).unsqueeze(-1).to(sc.dtype), torch.full_like(sc, -math.inf))
    return val.permute(1, 0, 2).reshape(B, T * K)


def nbest(sc, wi, pt, eos_id, length_penalty, out_len, n):
    """The n highest-ranked candidates of the final-selection rule, each back-tracked as backtrack() does its best one: (nbest_seq
    int64 [B, n, out_len] zero padded, nbest_scores [B, n] — the rule's values).  Equal values keep (frame, beam) order, so entry 0
    is backtrack()'s hypothesis; the list is not deduplicated.  Every beam of the last frame is a candidate, so n <= K always fills."""
    T, B, K = sc.shape
    dev = sc.device
    flat = candidate_values(sc, wi, eos_id, length_penalty)
    val, idx = torch.sort(flat, dim=1, descending=True, stable=True)
    val, idx = val[:, :n], idx[:, :n]                                     # [B, n]
    frame, pos = torch.div(idx, K, rounding_mode="floor"), idx % K
    found = torch.isfinite(val)
    toks = [None] * T
    for fid in range(T - 1, -1, -1):                                      # walk the back pointers from `frame` down to 0
        active = found & (fid <= frame)
        toks[fid] = torch.where(active, wi[fid].gather(1, pos), torch.zeros_like(pos))
        pos = torch.where(active & (fid > 0), pt[fid].gather(1, pos), pos)
    seq = torch.zeros(B, n, out_len, dtype=torch.long, device=dev)
    seq[:, :, :T] = torch.stack(toks, dim=-1)
    return seq, val


def best_path(sc, wi, pt, eos_id, length_penalty):
    """The hypothesis backtrack() selects, frame by frame: (active [T,B] — frame t belongs to it —, pos [T,B] — its beam index at
    frame t)."""
    T, B, K = sc.shape
    dev = sc.device
    flat = candidate_values(sc, wi, eos_id, length_penalty)
    best = flat.argmax(-1)                                                # first maximal value
    frame, pos = torch.div(best, K, rounding_mode="floor"), best % K
    found = torch.isfinite(flat.gather(1, best.unsqueeze(1)).squeeze(1))
    bidx = torch.arange(B, device=dev)
    actives, poss = [None] * T, [None] * T
    for fid in range(T - 1, -1, -1):                                      # walk the back pointers from `frame` down to 0
        active = found & (fid <= frame)
        actives[fid], poss[fid] = active, pos
        pos = torch.where(active & (fid > 0), pt[fid, bidx, pos], pos)
    return torch.stack(actives), torch.stack(poss)
