"""Beam search for BertForSeq2SeqDecoder (semantics of the reference's modeling.py:1256-1494).

Same algorithm and return format (a `traces` dict of padded tensors: pred_seq, scores, wids, ptrs), with ALL beam
bookkeeping on the device — top-k, back pointers (integer floor division: the reference's `torch.div(k_ids, K)`, :1317, yields
floats on torch >= 1.6 and breaks `gather`, SURVEY.md §2 #7), the per-layer K/V caches reordered by the back pointers, and the final
best-hypothesis selection + back-tracking (:1431-1472) as vectorised tensor ops, and the optional duplicate-n-gram blocking
(`forbid_duplicate_ngrams`, :1375-1428) as one vlpk_beam_ngram_block launch per frame over per-hypothesis word histories held on the
device: no host synchronisation inside or after the loop, so a blocked decode can be captured as a CUDA graph too.
Per-sample `task_idx` (the relaxed MLM head, relax_projection > 1) is expanded to the B*K beam rows with the other inputs; the
reference does not expand it (:1297 vs :1325-1373), so its relaxed beam search only runs at B = 1.
Diverse beam search (num_beam_groups > 1, diverse_beam_search) runs the same data flow and trace format with its own per-frame selection.
Constrained beam search (constraints, constrained_beam_search) runs it too, over K beams in each of 2^C constraint states.
Every step runs the fused layers on the two new rows (token, [MASK]) through decode.DecodeState, which also expands the history to the
beams after the first step and reorders it by the back pointers after every later one.
"""
import math

import torch
import torch.nn.functional as F

from . import ops
from .decode import (DecodeState, _ignore_tensor, expand_task_idx, new_attention_maps, prompt_constraints, prompt_eos_until, prompt_history,
                     prompt_lengths, with_prompt)


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


def _step_maps(maps, frame, B, W):
    """The buffer of step `frame`'s [MASK]-row maps in maps [T, B*W, ...]: step 0 has B input rows, written at rows b*W; None
    without maps."""
    if maps is None:
        return None
    return maps[frame] if frame else maps[0].view(B, W, *maps.shape[2:])[:, 0]


def _follow_beams(state, frame, ptrs, task_idx):
    """Moves the decode state to frame `frame`'s W beams per image (ptrs [B, W] their back pointers): expands each image's row to
    them after frame 0, per-sample task_idx included, and reorders by the back pointers after every later frame.  Returns task_idx."""
    B, W = ptrs.shape
    if frame == 0:
        state.expand(W)
        return expand_task_idx(task_idx, B, W)                          # per-sample ids follow their beams (relaxed head)
    state.reorder((ptrs + torch.arange(B, device=ptrs.device).unsqueeze(1) * W).reshape(-1))      # beam i continues hypothesis parent[i]
    return task_idx


def _padded_traces(out, sc, wi, pt, out_len):
    """out["scores"], out["wids"], out["ptrs"]: the traces [T, B, W] as [B, out_len, W], zero past frame T."""
    T, B, W = sc.shape
    for k, t in (("scores", sc), ("wids", wi), ("ptrs", pt)):
        padded = t.new_zeros((B, out_len, W))
        padded[:, :T] = t.permute(1, 0, 2)
        out[k] = padded


def beam_search(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, task_idx=None, output_attentions=False,
                prompt=None):
    """output_attentions: out["attentions"] [B, out_len - in_len, layers, heads, out_len] holds, for frame t of pred_seq, the [MASK]-row
    maps of step t taken from the row its hypothesis continued (beam_maps).
    prompt [B, Tp] (Tp >= 1): the search runs out_len - in_len - Tp frames after the prompt's prefill (decode.DecodeState).  Every
    hypothesis' n-gram history starts with its image's prompt (decode.prompt_history: Tp + g entries at frame g, so frame 0 is
    blocked too), [EOS] is blocked while t_b + g + 1 <= min_len, and pred_seq / nbest_seq hold the t_b prompt words before the
    generated ones.  The traces and scores are those of the generated words only."""
    K = dec.search_beam_size
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[1]
    dev = input_ids.device
    N = dec.num_return_sequences
    # N > 1: the K hypotheses of an image share its prefix K/V; a reorder moves slot-table entries, not cache rows
    state = DecodeState(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, K if N > 1 else None, prompt)
    Tp = 0 if prompt is None else prompt.shape[1]
    total_scores, beam_eos, step_ids, step_ptrs = [], [], [], []
    if dec.forbid_duplicate_ngrams:
        ngram, ignore = int(dec.ngram_size), _ignore_tensor(dec, dev)
        hist = [torch.empty(B * K, out_len - in_len, dtype=torch.int32, device=dev) for _ in range(2)]    # word histories, in turn
    # per step t, the [MASK]-row maps of its B*K input rows (step 0: B rows, written at rows b*K)
    maps = new_attention_maps(dec, out_len - in_len, B * K, out_len, dev) if output_attentions else None
    if Tp:
        lens = prompt_lengths(prompt)
        row_lens = lens                                                   # t_b of every row: B rows at frame 0, B*K after
    curr_ids = state.first_ids
    for frame in range(state.frames):
        scores, _ = dec.cls(state.step(curr_ids, _step_maps(maps, frame, B, K)), None, task_idx=task_idx)
        logp = F.log_softmax(scores.float(), dim=-1)                      # [B or B*K, 1, V]
        if Tp:
            if dec.forbid_duplicate_ngrams:
                if frame == 0:
                    # the prompt alone is frame 0's history: one row per image, its own parent, its last entry fed as the word
                    seed = prompt_history(prompt, 1, out_len - in_len)
                    ops.beam_ngram_block(seed, torch.empty_like(seed), torch.zeros(B, 1, dtype=torch.int64, device=dev),
                                         seed[:, Tp - 1:Tp].to(torch.int64), Tp, ngram, ignore, logp)
                    hist[0] = seed.repeat_interleave(K, 0)                # frame 1's parents: each image's rows
                else:
                    ops.beam_ngram_block(hist[(frame - 1) % 2], hist[frame % 2], step_ptrs[-1], step_ids[-1], Tp + frame, ngram, ignore,
                                         logp)
            if dec.min_len:
                block = (row_lens + frame + 1 <= dec.min_len).view(-1, 1)
                logp[:, :, dec.eos_id] = torch.where(block, torch.full_like(logp[:, :, dec.eos_id], -10000.0), logp[:, :, dec.eos_id])
            if frame == 0:
                row_lens = lens.repeat_interleave(K)
        else:
            if dec.forbid_duplicate_ngrams and frame >= 1:
                # history of frame `frame` from the previous frame's words and back pointers; blocks in place once it holds n words
                ops.beam_ngram_block(hist[(frame - 1) % 2], hist[frame % 2], step_ptrs[-1], step_ids[-1], frame, ngram, ignore, logp)
            if dec.min_len and (frame + 1 <= dec.min_len):
                logp[:, :, dec.eos_id] = -10000.0
        kk_scores, kk_ids = torch.topk(logp, k=K)                          # [*, 1, K]
        if frame == 0:
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
        task_idx = _follow_beams(state, frame, back, task_idx)
        curr_ids = k_ids.reshape(B * K, 1)

    sc, wi, pt = torch.stack(total_scores), torch.stack(step_ids), torch.stack(step_ptrs)
    out = {"pred_seq": backtrack(sc, wi, pt, dec.eos_id, dec.length_penalty, out_len)}
    if maps is not None:
        out["attentions"] = beam_maps(maps, *best_path(sc, wi, pt, dec.eos_id, dec.length_penalty), pt)
    _padded_traces(out, sc, wi, pt, out_len)
    if N > 1:
        out["nbest_seq"], out["nbest_scores"] = nbest(sc, wi, pt, dec.eos_id, dec.length_penalty, out_len, N)
    if Tp:
        for k in ("pred_seq", "nbest_seq"):
            if k in out:
                out[k] = with_prompt(prompt, out[k])
    return out


def diverse_beam_search(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, task_idx=None,
                        output_attentions=False, prompt=None):
    """Diverse beam search (Vijayakumar et al., AAAI 2018): the K = dec.search_beam_size beams of an image in G = dec.num_beam_groups
    groups of Kg = K / G.  Every frame, the groups choose in turn; group g extends its own beams and ranks each (parent, word) by its
    beam score minus dec.diversity_penalty times the number of beams of groups < g that chose the word in this frame.  The traces keep
    the unpenalised scores, so the final selection compares the groups on model log-probabilities.  One vlpk_diverse_beam_step per
    frame reads the head's logits (decoder output without the bias) once and writes the frame's traces in place, the n-gram blocking
    and the min_len [EOS] block included; nothing synchronises with the host.

    Output: beam_search's dict (pred_seq, scores, wids, ptrs; attentions, nbest_seq / nbest_scores as there), plus group_seq int64
    [B, G, out_len] and group_scores fp32 [B, G]: the final-selection rule applied to each group's Kg beams alone.
    prompt [B, Tp] (Tp >= 1): as beam_search's, through vlpk_diverse_beam_step_prompt; group_seq holds the prompt words too."""
    K, G = dec.search_beam_size, dec.num_beam_groups
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[1]
    dev = input_ids.device
    N = dec.num_return_sequences
    state = DecodeState(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, K if N > 1 else None, prompt)
    T, Tp = state.frames, state.prefix_len - in_len
    ngram = int(dec.ngram_size) if dec.forbid_duplicate_ngrams else 0
    ignore = _ignore_tensor(dec, dev) if ngram else None
    hist = [torch.empty(B * K, T + Tp, dtype=torch.int32, device=dev) for _ in range(2)] if ngram else [None, None]
    if Tp:
        seed = prompt_history(prompt, 1, T + Tp)
        eos_until = [prompt_eos_until(prompt, 1, dec.min_len), prompt_eos_until(prompt, K, dec.min_len)]
    sc, eos = (torch.zeros(T, B, K, dtype=torch.float32, device=dev) for _ in range(2))
    wi, pt = (torch.zeros(T, B, K, dtype=torch.int64, device=dev) for _ in range(2))
    top_w = torch.empty(B * K, K, dtype=torch.int32, device=dev)
    top_lp = torch.empty(B * K, K, dtype=torch.float32, device=dev)
    pred = dec.cls.predictions
    maps = new_attention_maps(dec, T, B * K, out_len, dev) if output_attentions else None
    curr_ids = state.first_ids
    for frame in range(T):
        h = pred.select_task(pred.transform(state.step(curr_ids, _step_maps(maps, frame, B, K)).to(pred.decoder.weight.dtype)), task_idx)
        logits = pred.decoder(h)                                          # [B or B*K, 1, V]; the kernel adds the bias
        if Tp:
            ops.diverse_beam_step(logits, pred.bias.to(logits.dtype), frame, G, dec.diversity_penalty, wi, pt, sc, eos, top_w, top_lp,
                                  dec.eos_id, ngram=ngram, ignore=ignore, hist_in=seed if frame == 0 else hist[(frame - 1) % 2],
                                  hist_out=hist[frame % 2], prompt=(Tp, eos_until[min(frame, 1)]))
            if frame == 0 and ngram:
                hist[0] = seed.repeat_interleave(K, 0)                    # frame 1's parents: each image's rows
        else:
            ops.diverse_beam_step(logits, pred.bias.to(logits.dtype), frame, G, dec.diversity_penalty, wi, pt, sc, eos, top_w, top_lp,
                                  dec.eos_id, block_eos=bool(dec.min_len) and frame + 1 <= dec.min_len, ngram=ngram, ignore=ignore,
                                  hist_in=hist[(frame - 1) % 2], hist_out=hist[frame % 2])
        task_idx = _follow_beams(state, frame, pt[frame], task_idx)
        curr_ids = wi[frame].reshape(B * K, 1)

    out = {"pred_seq": backtrack(sc, wi, pt, dec.eos_id, dec.length_penalty, out_len)}
    if maps is not None:
        out["attentions"] = beam_maps(maps, *best_path(sc, wi, pt, dec.eos_id, dec.length_penalty), pt)
    _padded_traces(out, sc, wi, pt, out_len)
    if N > 1:
        out["nbest_seq"], out["nbest_scores"] = nbest(sc, wi, pt, dec.eos_id, dec.length_penalty, out_len, N)
    out["group_seq"], out["group_scores"] = group_best(sc, wi, pt, dec.eos_id, dec.length_penalty, out_len, G)
    return _prompted(out, prompt, ("pred_seq", "nbest_seq", "group_seq"))


def _prompted(out, prompt, keys):
    """out with the prompt's words placed before the generated words of every returned caption in keys (decode.with_prompt)."""
    if prompt is not None:
        for k in keys:
            if k in out:
                out[k] = with_prompt(prompt, out[k])
    return out


def constrained_beam_search(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, cons, task_idx=None,
                            output_attentions=False, prompt=None):
    """Constrained beam search (Anderson et al., EMNLP 2017): captions that must contain given words or phrases.  cons: int64 [B, C, A,
    P] on the device, 0-padded: constraint j of image b is met when one of its A alternatives (each a run of up to P word ids) occurs as
    a contiguous run of the generated words; a constraint with no alternative is met from the start.  A hypothesis' state is the set s
    of constraints met so far; each of the S = 2^C states keeps K = dec.search_beam_size beams, slot s*K + k of an image being beam k of
    state s.  Every frame, each (parent, word) pair goes to the state s_parent ∪ {constraints the word completes}, and each state keeps
    its K best pairs (beam search's scores, ties to the lower parent slot, then the lower word); a state with fewer candidates leaves
    empty slots (word 0, pointer 0, score -inf).  One vlpk_constrained_beam_step per frame reads the head's logits once, carries the
    word histories by back pointer and writes the frame's traces in place, the n-gram blocking and the min_len [EOS] block included;
    the S*K hypotheses of an image share one copy of its prefix K/V (per-hypothesis caches with output_attentions, which the shared
    cache does not produce), and nothing synchronises with the host.

    Output: beam_search's dict over the S*K slots (scores, wids, ptrs [B, out_len, S*K]; attentions along pred_seq's path), with
      pred_seq         the accept state's best caption under the final-selection rule (counting live slots only), or, where the accept
                       state has none, the best of the states with the most constraints met (higher value, then lower state);
      constraints_met  bool [B]: the accept state had a candidate;
      state_seq        int64 [B, S, out_len] and state_scores fp32 [B, S]: each state's own best (-inf where it has none);
      nbest_seq / nbest_scores (num_return_sequences N > 1): the accept state's N best.
    prompt [B, Tp] (Tp >= 1): as beam_search's, through vlpk_constrained_beam_step_prompt: a constraint one of whose alternatives the
    prompt contains is met from the start (decode.prompt_constraints: each image starts in its own state), a phrase may begin in the
    prompt and end in the continuation, and constraints_met refers to the whole caption."""
    K, C = dec.search_beam_size, cons.shape[1]
    S = 1 << C
    SK = S * K
    B, in_len = input_ids.shape
    out_len = token_type_ids.shape[1]
    dev = input_ids.device
    N = dec.num_return_sequences
    W = K + C * cons.shape[2]
    # one copy of each image's prefix K/V for its S*K hypotheses; the attention maps come from per-hypothesis caches
    state = DecodeState(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, None if output_attentions else SK,
                        prompt)
    T, Tp = state.frames, state.prefix_len - in_len
    ngram = int(dec.ngram_size) if dec.forbid_duplicate_ngrams else 0
    ignore = _ignore_tensor(dec, dev) if ngram else None
    hist = [torch.empty(B * SK, T + Tp, dtype=torch.int32, device=dev) for _ in range(2)]  # the constraint match reads them always
    if Tp:
        cons = prompt_constraints(cons, prompt)
        seed = prompt_history(prompt, 1, T + Tp)
        eos_until = [prompt_eos_until(prompt, 1, dec.min_len), prompt_eos_until(prompt, SK, dec.min_len)]
    sc, eos = (torch.zeros(T, B, SK, dtype=torch.float32, device=dev) for _ in range(2))
    wi, pt = (torch.zeros(T, B, SK, dtype=torch.int64, device=dev) for _ in range(2))
    top_w = torch.empty(B * SK, W, dtype=torch.int32, device=dev)
    top_lp = torch.empty(B * SK, W, dtype=torch.float32, device=dev)
    top_dest = torch.empty(B * SK, W - K, dtype=torch.int32, device=dev)
    pred = dec.cls.predictions
    maps = new_attention_maps(dec, T, B * SK, out_len, dev) if output_attentions else None
    curr_ids = state.first_ids
    for frame in range(T):
        h = pred.select_task(pred.transform(state.step(curr_ids, _step_maps(maps, frame, B, SK)).to(pred.decoder.weight.dtype)), task_idx)
        logits = pred.decoder(h)                                          # [B or B*S*K, 1, V]; the kernel adds the bias
        if Tp:
            ops.constrained_beam_step(logits, pred.bias.to(logits.dtype), frame, cons, wi, pt, sc, eos, top_w, top_lp, top_dest,
                                      dec.eos_id, ngram=ngram, ignore=ignore, hist_in=seed if frame == 0 else hist[(frame - 1) % 2],
                                      hist_out=hist[frame % 2], prompt=(Tp, eos_until[min(frame, 1)]))
            if frame == 0:
                hist[0] = seed.repeat_interleave(SK, 0)                   # frame 1's parents: each image's rows
        else:
            ops.constrained_beam_step(logits, pred.bias.to(logits.dtype), frame, cons, wi, pt, sc, eos, top_w, top_lp, top_dest,
                                      dec.eos_id, block_eos=bool(dec.min_len) and frame + 1 <= dec.min_len, ngram=ngram, ignore=ignore,
                                      hist_in=hist[(frame - 1) % 2], hist_out=hist[frame % 2])
        task_idx = _follow_beams(state, frame, pt[frame], task_idx)
        curr_ids = wi[frame].reshape(B * SK, 1)

    lp = dec.length_penalty
    paths = [best_path(sc, wi, pt, dec.eos_id, lp, beams=slice(s * K, (s + 1) * K)) for s in range(S)]
    state_seq = torch.stack([_path_tokens(wi, *path, out_len) for path in paths], 1)                    # [B, S, out_len]
    state_scores = torch.stack([candidate_values(sc[:, :, s * K:(s + 1) * K], wi[:, :, s * K:(s + 1) * K], dec.eos_id, lp, live=True)
                                .max(1).values for s in range(S)], 1)                                  # [B, S]
    chosen = state_choice(state_scores)
    bidx = torch.arange(B, device=dev)
    out = {"pred_seq": state_seq[bidx, chosen], "constraints_met": torch.isfinite(state_scores[:, S - 1])}
    if maps is not None:
        active = torch.stack([a for a, _ in paths])[chosen, :, bidx].t()                             # [T, B]: the chosen state's path
        pos = torch.stack([p for _, p in paths])[chosen, :, bidx].t()
        out["attentions"] = beam_maps(maps, active, pos, pt)
    _padded_traces(out, sc, wi, pt, out_len)
    if N > 1:
        out["nbest_seq"], out["nbest_scores"] = nbest(sc, wi, pt, dec.eos_id, lp, out_len, N, beams=slice((S - 1) * K, SK))
    out["state_seq"], out["state_scores"] = state_seq, state_scores
    return _prompted(out, prompt, ("pred_seq", "nbest_seq", "state_seq"))


def state_choice(state_scores):
    """The state pred_seq comes from, [B]: among the states with a candidate (finite value), the most constraints met, then the higher
    value, then the lower state; the accept state S - 1 whenever it has one.  0 where no state has a candidate."""
    B, S = state_scores.shape
    states = torch.arange(S, device=state_scores.device)
    met = sum((states >> j) & 1 for j in range(max(S.bit_length() - 1, 1)))                   # constraints met by each state
    finite = torch.isfinite(state_scores)
    most = torch.where(finite, met, torch.full_like(met, -1)).max(1, keepdim=True).values                    # [B, 1]
    val = torch.where(finite & (met == most), state_scores, torch.full_like(state_scores, -math.inf))
    return val.argmax(1)                                                  # first maximum: the lower state


def _path_tokens(wi, active, pos, out_len):
    """The words of a best_path (active / pos [T, B]) as a zero-padded [B, out_len] sequence."""
    T, B, _ = wi.shape
    seq = torch.zeros(B, out_len, dtype=torch.long, device=wi.device)
    tok = wi.gather(2, pos.unsqueeze(-1)).squeeze(-1)
    seq[:, :T] = torch.where(active, tok, torch.zeros_like(tok)).t()
    return seq


def group_best(sc, wi, pt, eos_id, length_penalty, out_len, G):
    """Each group's best hypothesis under the final-selection rule over its own Kg = K / G beams (a diverse beam search's parents
    stay in their group): (group_seq int64 [B, G, out_len] zero padded, group_scores [B, G] — the rule's values)."""
    T, B, K = sc.shape
    Kg = K // G
    seqs, vals = [], []
    for g in range(G):
        beams = slice(g * Kg, (g + 1) * Kg)
        sg, wg = sc[:, :, beams], wi[:, :, beams]
        pg = pt[:, :, beams] % Kg                                         # the parent's place in the group: ptr - g*Kg (0 at frame 0)
        seqs.append(backtrack(sg, wg, pg, eos_id, length_penalty, out_len))
        vals.append(candidate_values(sg, wg, eos_id, length_penalty).max(1).values)
    return torch.stack(seqs, 1), torch.stack(vals, 1)


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


def candidate_values(sc, wi, eos_id, length_penalty, live=False):
    """The final-selection rule's value of every (frame, beam), [B, T*K] in (frame, beam) order — the reference's loop order: score +
    length_penalty * (frame + 1) for a candidate ([EOS] word, or the last frame, within frames <= last[b]), -inf otherwise.
    live: the beams may hold empty slots (score -inf, constrained beam search); the all-[EOS] test that sets last[b] then counts the
    live slots only, and a frame with no live slot never ends the search."""
    T, B, K = sc.shape
    dev = sc.device
    frames = torch.arange(T, device=dev).view(T, 1)
    if live:
        alive = torch.isfinite(sc)
        all_eos = ((wi == eos_id) | ~alive).all(-1) & alive.any(-1)
    else:
        all_eos = (wi == eos_id).all(-1)                                  # [T,B]
    last = torch.where(all_eos.any(0), all_eos.float().argmax(0), torch.full((B,), T - 1, device=dev))      # [B]
    cand = (frames <= last.unsqueeze(0)).unsqueeze(-1) & ((wi == eos_id) | (frames == last.unsqueeze(0)).unsqueeze(-1))
    val = torch.where(cand, sc + length_penalty * (frames + 1).unsqueeze(-1).to(sc.dtype), torch.full_like(sc, -math.inf))
    return val.permute(1, 0, 2).reshape(B, T * K)


def nbest(sc, wi, pt, eos_id, length_penalty, out_len, n, beams=None):
    """The n highest-ranked candidates of the final-selection rule, each back-tracked as backtrack() does its best one: (nbest_seq
    int64 [B, n, out_len] zero padded, nbest_scores [B, n] — the rule's values).  Equal values keep (frame, beam) order, so entry 0
    is backtrack()'s hypothesis; the list is not deduplicated.  Every beam of the last frame is a candidate, so n <= K always fills.
    beams: a slice of the slots (one state of constrained beam search) whose candidates are ranked, under the live-slot rule of
    candidate_values; the back pointers still run over every slot.  Entries past its live candidates are -inf and zero words."""
    T, B, K = sc.shape
    dev = sc.device
    sel = slice(0, K) if beams is None else beams
    flat = candidate_values(sc[:, :, sel], wi[:, :, sel], eos_id, length_penalty, live=beams is not None)
    Ks = flat.shape[1] // T
    val, idx = torch.sort(flat, dim=1, descending=True, stable=True)
    val, idx = val[:, :n], idx[:, :n]                                     # [B, n]
    frame, pos = torch.div(idx, Ks, rounding_mode="floor"), idx % Ks + sel.start
    found = torch.isfinite(val)
    toks = [None] * T
    for fid in range(T - 1, -1, -1):                                      # walk the back pointers from `frame` down to 0
        active = found & (fid <= frame)
        toks[fid] = torch.where(active, wi[fid].gather(1, pos), torch.zeros_like(pos))
        pos = torch.where(active & (fid > 0), pt[fid].gather(1, pos), pos)
    seq = torch.zeros(B, n, out_len, dtype=torch.long, device=dev)
    seq[:, :, :T] = torch.stack(toks, dim=-1)
    return seq, val


def best_path(sc, wi, pt, eos_id, length_penalty, beams=None):
    """The hypothesis backtrack() selects, frame by frame: (active [T,B] — frame t belongs to it —, pos [T,B] — its beam index at
    frame t).  beams: as nbest's, the best of those slots under the live-slot rule (pos still indexes every slot)."""
    T, B, K = sc.shape
    dev = sc.device
    sel = slice(0, K) if beams is None else beams
    flat = candidate_values(sc[:, :, sel], wi[:, :, sel], eos_id, length_penalty, live=beams is not None)
    Ks = flat.shape[1] // T
    best = flat.argmax(-1)                                                # first maximal value
    frame, pos = torch.div(best, Ks, rounding_mode="floor"), best % Ks + sel.start
    found = torch.isfinite(flat.gather(1, best.unsqueeze(1)).squeeze(1))
    bidx = torch.arange(B, device=dev)
    actives, poss = [None] * T, [None] * T
    for fid in range(T - 1, -1, -1):                                      # walk the back pointers from `frame` down to 0
        active = found & (fid <= frame)
        actives[fid], poss[fid] = active, pos
        pos = torch.where(active & (fid > 0), pt[fid, bidx, pos], pos)
    return torch.stack(actives), torch.stack(poss)
