"""Host statements of constrained beam search (vlpk_constrained_beam_step, beam.constrained_beam_search), in numpy and torch.

  dest         the state a (row, word) pair goes to: the row's state plus every constraint the word completes.
  two_stage    one frame as the kernels run it: each row's completing words (completions) and its top K of the other words, then each
               state's merge over them.
  full_vocab   the same frame over every (parent, word) pair of the vocabulary, with dest taken word by word.
  host_decode  a whole decode: the full-vocabulary rule driving the model's own DecodeState, then the final selection (select).

Slots: image b's hypotheses are [0, S*K), S = 2^C, slot s*K + k is beam k of state s.  Empty slots hold word 0, pointer 0, score -inf.
logp comes from diverse_beam_oracle.frame_logp (log_softmax, n-gram and min_len blocks).  Nothing here calls the kernels or reads
the reference, which has no constrained search."""
import numpy as np
import torch

from tools.diverse_beam_oracle import BLOCK, frame_logp


def alternatives(cons_b):
    """cons_b [C, A, P] (0-padded) -> per constraint, the tuple of its alternatives, each a tuple of word ids (its leading non-zero
    entries); an alternative whose first entry is 0 is absent."""
    out = []
    for c in np.asarray(cons_b):
        alts = []
        for a in c:
            words = []
            for w in a:
                if w == 0:
                    break
                words.append(int(w))
            if words:
                alts.append(tuple(words))
        out.append(tuple(alts))
    return out


def root_state(cons_b):
    """The set of constraints with no alternative (satisfied from the start), as a bit mask."""
    return sum(1 << j for j, alts in enumerate(alternatives(cons_b)) if not alts)


def dest(hist, w, cons_b, s):
    """State of the hypothesis `hist` (its generated words) in state s extended by w: s plus every constraint j one of whose
    alternatives a ends in w with hist ending in a[:-1]."""
    for j, alts in enumerate(alternatives(cons_b)):
        for a in alts:
            if a[-1] == w and len(a) - 1 <= len(hist) and tuple(hist[len(hist) - (len(a) - 1):]) == a[:-1]:
                s |= 1 << j
    return s


def completions(hist, cons_b, s):
    """{word: dest} of the words that move a row in state s to another state (at most C*A of them)."""
    out = {}
    for j, alts in enumerate(alternatives(cons_b)):
        if (s >> j) & 1:
            continue
        for a in alts:
            if len(a) - 1 <= len(hist) and tuple(hist[len(hist) - (len(a) - 1):]) == a[:-1]:
                out[a[-1]] = out.get(a[-1], s) | (1 << j)
    return out


def _rows(B, K, C, first, cons):
    """(image, parent slot, state) of every row of a frame."""
    SK = K << C
    if first:
        return [(b, 0, root_state(cons[b])) for b in range(B)]
    return [(b, p, p // K) for b in range(B) for p in range(SK)]


def _select(cands, K, C):
    """cands: per image, per state, lists of (value, parent, word) -> wid, ptr [S*K] int64, score [S*K], margin: the smallest gap
    between consecutive finite values among each state's K + 1 best, pairs of the same parent excepted (one row's values share its
    logsumexp and score, so every consistent rounding sees their tie and breaks it by word)."""
    S = 1 << C
    wid, ptr, score = np.zeros(S * K, np.int64), np.zeros(S * K, np.int64), np.full(S * K, -np.inf)
    margin = np.inf
    for s in range(S):
        c = sorted((x for x in cands[s] if np.isfinite(x[0])), key=lambda x: (-x[0], x[1], x[2]))
        for r, (v, p, w) in enumerate(c[:K]):
            wid[s * K + r], ptr[s * K + r], score[s * K + r] = w, p, v
        top = c[:K + 1]
        for (v0, p0, _), (v1, p1, _) in zip(top, top[1:]):
            if v0 > v1 or p0 != p1:
                margin = min(margin, float(v0) - float(v1))
    return wid, ptr, score, margin


def _cand(lp, first, prev_score, prev_eos, b, p, dtype):
    if first:
        return lp.astype(dtype)
    return ((lp.astype(dtype) + dtype(prev_eos[b, p]) * dtype(BLOCK)) + dtype(prev_score[b, p])).astype(dtype)


def row_lists(lp, hists, cons, K, C, first, top=None):
    """The rows kernel's outputs: per row, (top-K words, their logp) over the words that keep it in its state, ranked by (logp
    descending, word ascending), and the completing words {word: (logp, dest)}.  top: how many words to rank (default K)."""
    B = cons.shape[0]
    out = []
    for i, (b, p, s) in enumerate(_rows(B, K, C, first, cons)):
        comp = completions(hists[i] if hists is not None else [], cons[b], s)
        order = [w for w in np.lexsort((np.arange(lp.shape[1]), -lp[i])) if int(w) not in comp][:top or K]
        out.append((np.array(order), lp[i, order], {w: (lp[i, w], d) for w, d in comp.items()}))
    return out


def two_stage(lp, hists, prev_score, prev_eos, cons, K, first, dtype=np.float32):
    """lp [rows, V] (rows = B at frame 0, B*S*K after), hists: per row its generated words (None at frame 0), prev_score / prev_eos
    [B, S*K], cons [B, C, A, P] -> wid, ptr [B, S*K] int64, score [B, S*K] dtype, margin [B]."""
    C = cons.shape[1]
    return merge(row_lists(lp.astype(dtype), hists, cons, K, C, first), prev_score, prev_eos, cons, K, first, dtype)


def kernel_lists(top_w, top_lp, top_dest, K):
    """row_lists' format from the rows kernel's scratch (numpy [rows, K + C*A], [rows, K + C*A], [rows, C*A])."""
    return [(tw[:K], tl[:K], {int(w): (l, int(d)) for w, l, d in zip(tw[K:], tl[K:], td) if d >= 0})
            for tw, tl, td in zip(top_w, top_lp, top_dest)]


def merge(lists, prev_score, prev_eos, cons, K, first, dtype=np.float32):
    """Each state's merge over the rows' lists (row_lists or kernel_lists).  Returns two_stage's tuple."""
    B, C = cons.shape[0], cons.shape[1]
    S = 1 << C
    rows = _rows(B, K, C, first, cons)
    cands = [[[] for _ in range(S)] for _ in range(B)]
    for (b, p, s), (tw, tl, comp) in zip(rows, lists):
        for w, l in zip(tw, tl):
            cands[b][s].append((_cand(np.asarray(l), first, prev_score, prev_eos, b, p, dtype), p, int(w)))
        for w, (l, d) in comp.items():
            cands[b][d].append((_cand(np.asarray(l), first, prev_score, prev_eos, b, p, dtype), p, int(w)))
    return _stack([_select(cands[b], K, C) for b in range(B)], dtype)


def full_vocab(lp, hists, prev_score, prev_eos, cons, K, first, dtype=np.float64):
    """The same frame over every (parent, word) pair, each sent to dest(hist, word).  Returns two_stage's tuple."""
    B, C = cons.shape[0], cons.shape[1]
    S = 1 << C
    V = lp.shape[1]
    cands = [[[] for _ in range(S)] for _ in range(B)]
    for i, (b, p, s) in enumerate(_rows(B, K, C, first, cons)):
        hist = hists[i] if hists is not None else []
        vals = _cand(lp[i], first, prev_score, prev_eos, b, p, dtype)
        last = {a[-1] for alts in alternatives(cons[b]) for a in alts}     # only these can complete an alternative
        for w in range(V):
            cands[b][dest(hist, w, cons[b], s) if w in last else s].append((vals[w], p, w))
    return _stack([_select(cands[b], K, C) for b in range(B)], dtype)


def _stack(res, dtype):
    wid, ptr, score, margin = zip(*res)
    return np.stack(wid), np.stack(ptr), np.stack(score).astype(dtype), np.array(margin)


def carry(hists, wid, ptr, K, C, first):
    """The histories of the next frame: slot i continues its parent's words plus its own word (frame 0: the image's empty history)."""
    B, SK = wid.shape
    return [(([] if first else list(hists[b * SK + int(ptr[b, i])])) + [int(wid[b, i])]) for b in range(B) for i in range(SK)]


def select(sc, wi, pt, eos_id, length_penalty, K, C):
    """Final selection on host traces sc / wi / pt [T, B, S*K] (numpy): per state the reference's rule over its K slots, counting live
    slots only in the all-[EOS] test; pred from the accept state if it has a candidate, else from the states with the most constraints
    met (higher value, then lower state).  Returns pred [B, T] (0 padded), state_seq [B, S, T], state_scores [B, S], met [B]."""
    T, B, SK = sc.shape
    S = 1 << C
    state_seq, state_val = np.zeros((B, S, T), np.int64), np.full((B, S), -np.inf)
    for b in range(B):
        for s in range(S):
            sl = slice(s * K, (s + 1) * K)
            live = np.isfinite(sc[:, b, sl])
            all_eos = [(live[t].any() and (wi[t, b, sl][live[t]] == eos_id).all()) for t in range(T)]
            last = all_eos.index(True) if any(all_eos) else T - 1
            best, at = -np.inf, None
            for t in range(last + 1):
                for k in range(K):
                    if wi[t, b, s * K + k] == eos_id or t == last:
                        v = sc[t, b, s * K + k] + length_penalty * (t + 1)
                        if v > best:
                            best, at = v, (t, s * K + k)
            if at is None:
                continue
            state_val[b, s] = best
            t, pos = at
            for fid in range(t, -1, -1):
                state_seq[b, s, fid] = wi[fid, b, pos]
                pos = pt[fid, b, pos] if fid > 0 else pos
    met = np.isfinite(state_val[:, S - 1])
    pred = np.zeros((B, T), np.int64)
    for b in range(B):
        ok = [s for s in range(S) if np.isfinite(state_val[b, s])]
        if ok:
            s = min(ok, key=lambda s: (-bin(s).count("1"), -state_val[b, s], s))
            pred[b] = state_seq[b, s]
    return pred, state_seq, state_val, met


def host_decode(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, cons, task_idx=None, follow=None):
    """The whole decode under the full-vocabulary rule (fp32 logp and scores as the device keeps them), driving the model's own
    DecodeState over one shared prefix cache of S*K hypotheses per image.  cons: int64 [B, C, A, P] (any device).  follow: numpy
    traces (sc, wi, pt) [T, B, S*K] of another decode; each frame is then selected by the rule and continued from those traces, so
    every frame is checked against the same hypotheses.  Returns (sc, wi, pt) numpy [T, B, S*K] of the rule's selections and
    margin [T, B]: each frame's smallest decisive gap per image (_select)."""
    from vlp_b200.beam import _dup_ngram_candidates
    from vlp_b200.decode import DecodeState, expand_task_idx

    cons = np.asarray(cons.cpu() if torch.is_tensor(cons) else cons)
    K, C = dec.search_beam_size, cons.shape[1]
    SK = K << C
    B, in_len = input_ids.shape
    T = token_type_ids.shape[1] - in_len
    dev = input_ids.device
    state = DecodeState(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, SK)
    pred = dec.cls.predictions
    ngram = int(dec.ngram_size) if dec.forbid_duplicate_ngrams else 0
    ignore = set(int(w) for w in dec.forbid_ignore_set or ())
    sc, wi, pt = np.zeros((T, B, SK), np.float32), np.zeros((T, B, SK), np.int64), np.zeros((T, B, SK), np.int64)
    margin = np.zeros((T, B))
    path = (sc, wi, pt) if follow is None else follow
    hists = None
    curr = input_ids
    for f in range(T):
        h = pred.select_task(pred.transform(state.step(curr).to(pred.decoder.weight.dtype)), task_idx)
        logits = pred.decoder(h)
        x = (logits + pred.bias.to(logits.dtype)).float().reshape(logits.shape[0], -1).cpu().numpy()
        blocked = None
        if ngram and f >= ngram:
            blocked = np.zeros(x.shape, bool)
            for i, hist in enumerate(hists):
                blocked[i, _dup_ngram_candidates(hist, ngram, ignore)] = True
        lp = frame_logp(x, blocked, bool(dec.min_len) and f + 1 <= dec.min_len, dec.eos_id, np.float32)
        first = f == 0
        prev = (None, None) if first else (path[0][f - 1], (path[1][f - 1] == dec.eos_id).astype(np.float32))
        wi[f], pt[f], sc[f], margin[f] = full_vocab(lp, hists, *prev, cons, K, first, np.float32)
        w, p = path[1][f], path[2][f]
        hists = carry(hists, w, p, K, C, first)
        if first:
            state.expand(SK)
            task_idx = expand_task_idx(task_idx, B, SK)
        else:
            state.reorder(torch.as_tensor(p + np.arange(B)[:, None] * SK, device=dev).reshape(-1))
        curr = torch.as_tensor(w, device=dev).reshape(B * SK, 1)
    return (sc, wi, pt), margin
