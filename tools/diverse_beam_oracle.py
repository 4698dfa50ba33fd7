"""Host statements of one diverse-beam frame (vlpk_diverse_beam_step), in numpy.

  frame_logp   step 1: logp = x - logsumexp(x), then -10000 at blocked words and logp[eos] = -10000 below min_len.
  two_stage    steps 2-4 as the kernels run them: each row's top K by (logp descending, word ascending) (row_topk), then the
               groups' merge (merge).
  full_vocab   steps 2-4 over every (parent, word) pair of the vocabulary, with no top-K stage.

The two agree exactly (the top-K argument of DESIGN.md §6); two_stage in fp32 is what the device is compared against, with a margin
that says where fp32 rounding could legitimately pick another pair."""
import numpy as np

BLOCK = -10000.0


def frame_logp(x, blocked=None, block_eos=False, eos_id=-1, dtype=np.float32):
    """x [rows, V] logits (already rounded as the head rounds them), blocked [rows, V] bool or None -> logp [rows, V] in dtype."""
    x = np.asarray(x, dtype=dtype)
    mx = x.max(1, keepdims=True)
    lse = np.log(np.exp(x - mx).sum(1, keepdims=True, dtype=dtype)).astype(dtype)
    lp = ((x - mx) - lse).astype(dtype)
    if blocked is not None:
        lp = np.where(blocked, lp + dtype(BLOCK), lp).astype(dtype)
    if block_eos and 0 <= eos_id < lp.shape[1]:
        lp[:, eos_id] = dtype(BLOCK)
    return lp


def _cand(lp_rows, prev_score, prev_eos, first, dtype):
    """cand of every (parent, word): lp at frame 0, (lp + eos * -10000) + score after (the fp32 order of beam search)."""
    if first:
        return lp_rows.astype(dtype)
    return ((lp_rows + (prev_eos.astype(dtype) * dtype(BLOCK))[:, None]) + prev_score.astype(dtype)[:, None]).astype(dtype)


def _merge(parents, words, cands, K, G, lam, dtype):
    """Groups g = 0 .. G-1 over per-group candidate arrays (parents, words, cands of group g), NaN ranked above every number as the
    kernel ranks it -> wid, ptr, score [K], margin: the
    smallest gap between consecutive penalised values among each group's Kg + 1 best.  An exact tie between two words of the same
    parent and penalty does not count: both values come from the same row's logsumexp, parent score and penalty, so any
    implementation that rounds a row consistently sees the same tie and breaks it by word id."""
    Kg = K // G
    wid, ptr, score = np.zeros(K, np.int64), np.zeros(K, np.int64), np.zeros(K, dtype)
    margin = np.inf
    for g in range(G):
        p, w, c = parents(g), words(g), cands(g)
        cnt = np.zeros(len(w), dtype)
        for q in wid[:g * Kg]:
            cnt += (w == q)
        pen = (c - (dtype(lam) * cnt).astype(dtype)).astype(dtype)
        nan = np.isnan(pen)
        order = np.lexsort((w, p, np.where(nan, 0, -pen), ~nan))          # NaN ranks above every number, then ties by (parent, word)
        sel = order[:Kg]
        wid[g * Kg:(g + 1) * Kg], ptr[g * Kg:(g + 1) * Kg], score[g * Kg:(g + 1) * Kg] = w[sel], p[sel], c[sel]
        top = order[:Kg + 1]
        ranked, rp, rc = pen[top].astype(np.float64), p[top], cnt[top]
        gaps = ranked[:-1] - ranked[1:]
        gaps = gaps[(gaps > 0) | (rp[:-1] != rp[1:]) | (rc[:-1] != rc[1:])]
        if len(gaps):
            margin = min(margin, float(gaps.min()))
    return wid, ptr, score, margin


def row_topk(lp, K):
    """Each row's top K (word, logp), ranked by (logp descending, word ascending): (words int [rows, K], logp [rows, K])."""
    rows, V = lp.shape
    words = np.stack([np.lexsort((np.arange(V), -lp[i]))[:K] for i in range(rows)])
    return words, np.take_along_axis(lp, words, 1)


def two_stage(lp, prev_score, prev_eos, K, G, lam, first, dtype=np.float32):
    """lp [B, V] at frame 0 or [B*K, V] after; prev_score / prev_eos [B, K] (unused at frame 0).  Returns wid, ptr [B, K] int64,
    score [B, K] dtype, margin [B]."""
    tw, tl = row_topk(lp.astype(dtype), K)
    return merge(tw, tl, prev_score, prev_eos, K, G, lam, first, dtype)


def merge(tw, tl, prev_score, prev_eos, K, G, lam, first, dtype=np.float32):
    """The groups' merge over the rows' top K (row_topk's words tw and log-probabilities tl, [rows, K]).  Returns two_stage's
    (wid, ptr, score, margin)."""
    B = tw.shape[0] if first else tw.shape[0] // K
    Kg = K // G
    out = [np.zeros((B, K), np.int64), np.zeros((B, K), np.int64), np.zeros((B, K), dtype), np.zeros(B)]
    for b in range(B):
        if first:
            par = lambda g: np.zeros(K, np.int64)
            wrd = lambda g: tw[b]
            cnd = lambda g: tl[b].astype(dtype)
        else:
            rows = lambda g: np.arange(g * Kg, (g + 1) * Kg)
            par = lambda g: np.repeat(rows(g), K)
            wrd = lambda g: tw[b * K + rows(g)].reshape(-1)
            cnd = lambda g: _cand(tl[b * K + rows(g)].astype(dtype), prev_score[b, rows(g)], prev_eos[b, rows(g)], False, dtype).reshape(-1)
        res = _merge(par, wrd, cnd, K, G, lam, dtype)
        for o, r in zip(out, res):
            o[b] = r
    return tuple(out)


def full_vocab(lp, prev_score, prev_eos, K, G, lam, first, dtype=np.float64):
    """The same frame over every (parent, word) pair of the vocabulary.  Returns wid, ptr, score [B, K], margin [B]."""
    lp = lp.astype(dtype)
    V = lp.shape[1]
    B = lp.shape[0] if first else lp.shape[0] // K
    Kg = K // G
    out = [np.zeros((B, K), np.int64), np.zeros((B, K), np.int64), np.zeros((B, K), dtype), np.zeros(B)]
    for b in range(B):
        if first:
            par = lambda g: np.zeros(V, np.int64)
            wrd = lambda g: np.arange(V)
            cnd = lambda g: lp[b]
        else:
            rows = lambda g: np.arange(g * Kg, (g + 1) * Kg)
            par = lambda g: np.repeat(rows(g), V)
            wrd = lambda g: np.tile(np.arange(V), Kg)
            cnd = lambda g: _cand(lp[b * K + rows(g)], prev_score[b, rows(g)], prev_eos[b, rows(g)], False, dtype).reshape(-1)
        res = _merge(par, wrd, cnd, K, G, lam, dtype)
        for o, r in zip(out, res):
            o[b] = r
    return tuple(out)
