"""Exact host statement of the beam selectors' row stage (diverse_beam_rows_kernel, constrained_beam_rows_kernel in csrc/decode.cu) and
of their history carry, in numpy.

Given a row's fp32 logsumexp L, the row stage is exact IEEE arithmetic (the library is built without fast-math):
  x       sampling_oracle.head_x: bf16 logits + bias rounded to bf16, or fp32 logits + bias;
  mx      the largest non-NaN x (an fmaxf fold: exact);
  logp    lp[v] = fl(fl(x[v] - mx) - L), then fl(lp + -10000) at blocked words, then lp[eos] = -10000 under block_eos; every NaN is
          the device's canonical NaN (bits 0x7fffffff);
  top K   words ranked by (order_key(lp) descending, word ascending), order_key being the kernel's map of fp32 bits onto unsigned
          order (NaN above +inf); the constrained kernel's completing words are left out of the ranking and keep their exact lp.
Only L (one expf per word, a fixed-order fp32 sum, one logf) is not restated bit for bit.  recover_lse takes it from the kernel's
own output: L = -lp of an unblocked argmax when the kernel returned one (lp = fl(0 - L) = -L exactly), else the fp32 values within
`lse_tol` of the fp64 logsumexp that reproduce every returned (word, value) bit for bit, nearest first.  Either way the test holds
|L - lse64| <= lse_tol, a bound derived as sampling_oracle derives its sums': each thread sums a chunk of C = ceil(V / 1024) | 1
words, then a 10-level shuffle tree, so the sum of e = exp(x - mx) is within (C + 14) * 2^-24 of its own magnitude; each e carries
expf's 2 ulp and the rounding of x - mx (together (4 + |x - mx|) * 2^-24 relative, plus 2^-148 where e is subnormal); logf adds 1 ulp.

A row with a NaN or +inf x, or whose every x is -inf, has a NaN L: every lp is NaN (but a block_eos [EOS]).

carry states the history carry (carry_history): hist_out[i] = hist_in[(i / width) * width + p] ‖ prev_wid[i], p = prev_ptr[i] (0 at
f = 1); a pointer outside [0, width) gives -1 words and an id outside int32 gives -1.  prompt_carry states the prompted rows'
history (prompt_history): hist_off prompt entries, then the generated words; eos_blocked the prompted rows' [EOS] rule.  The merges
are diverse_beam_oracle.merge and constrained_beam_oracle.merge, fp32-exact already.  Nothing here calls the kernels or reads the
reference."""
import math

import numpy as np

from tools.sampling_oracle import BLOCK, THREADS, U24

CANONICAL_NAN = np.array(0x7FFFFFFF, np.uint32).view(np.float32)
INT32_MIN, INT32_MAX = -(1 << 31), (1 << 31) - 1


def order_key(x):
    """The kernel's order_key of fp32 values: uint32 whose unsigned order is the float order, the canonical NaN above +inf."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32)
    return np.where(u & np.uint32(0x80000000), ~u, u | np.uint32(0x80000000)).astype(np.uint32)


def canonical(x):
    """fp32 copy of x with every NaN the device's canonical NaN."""
    x = np.array(x, dtype=np.float32)
    x[np.isnan(x)] = CANONICAL_NAN
    return x


def nonfinite(x):
    """Whether the row's logsumexp is NaN: a NaN or +inf x, or every x -inf."""
    x = np.asarray(x, dtype=np.float32)
    return bool(np.isnan(x).any() or np.isposinf(x).any() or np.isneginf(x).all())


def _row_max(x):
    ok = x[~np.isnan(x)]
    return np.float32(ok.max()) if ok.size else np.float32(-np.inf)


def row_logp(x, L, blocked=None, block_eos=False, eos_id=-1):
    """The kernel's fp32 logp of one row x [V] under the fp32 logsumexp L (NaN for a non-finite row); blocked: bool [V] or None."""
    x = np.asarray(x, dtype=np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        d = (x - _row_max(x)).astype(np.float32)
        lp = (d - np.float32(L)).astype(np.float32)
        if blocked is not None:
            lp = np.where(blocked, (lp + BLOCK).astype(np.float32), lp)
    if block_eos and 0 <= eos_id < x.size:
        lp[eos_id] = BLOCK
    return canonical(lp)


def rank(lp, K, exclude=()):
    """The first K words of lp [V] by (order_key descending, word ascending), words in `exclude` left out: (words, lp[words])."""
    key = order_key(lp).astype(np.int64)
    if len(exclude):
        key[np.asarray(list(exclude), dtype=np.int64)] = -1
    words = np.lexsort((np.arange(lp.size), -key))[:K]
    return words, lp[words]


def lse_tol(x):
    """(lse64, tol): the fp64 log(sum exp(x - mx)) of a finite row and the bound on the kernel's fp32 L around it."""
    x = np.asarray(x, dtype=np.float32)
    x64 = x.astype(np.float64)
    d = x64 - float(x64.max())
    e = np.exp(d)
    Z = float(e.sum())
    ad = np.where(np.isneginf(d), 0.0, np.abs(d))
    eps = (4.0 + ad) * U24 * e + np.where((e > 0) & (e < 2.0 ** -125), 2.0 ** -148, 0.0)
    C = ((x.size + THREADS - 1) // THREADS) | 1
    rel = (C + 14) * U24 + float(eps.sum()) / Z                      # relative error of the fp32 sum of e
    lse = math.log(Z)
    ulp = float(np.spacing(np.float32(max(lse, 2.0 ** -126))))        # logf's 1 ulp, at the binade of L
    return lse, 1.01 * (-math.log1p(-rel)) + 2.0 * ulp


def _values_at(x, words, L, blocked, block_eos, eos_id):
    """fp32 [len(L), len(words)]: the row's lp at `words` under every fp32 candidate L."""
    x = np.asarray(x, dtype=np.float32)
    d = (x[words] - _row_max(x)).astype(np.float32)
    with np.errstate(invalid="ignore"):
        lp = (d[None, :] - np.asarray(L, dtype=np.float32)[:, None]).astype(np.float32)
        if blocked is not None:
            lp = np.where(blocked[words][None, :], (lp + BLOCK).astype(np.float32), lp)
    if block_eos:
        lp[:, np.asarray(words) == eos_id] = BLOCK
    return lp


def recover_lse(x, words, values, blocked=None, block_eos=False, eos_id=-1, cap=1 << 16):
    """The fp32 L of a finite row x from the kernel's returned pairs (words, values): returns (candidates, lse64, tol).  candidates:
    fp32 [n], the exact L if the kernel returned an unblocked argmax, else every fp32 L within tol of lse64 (the `cap` nearest) that
    reproduces each returned value bit for bit, nearest first; empty if none does."""
    x = np.asarray(x, dtype=np.float32)
    words = np.asarray(words, dtype=np.int64)
    values = np.asarray(values, dtype=np.float32)
    lse, tol = lse_tol(x)
    mx = _row_max(x)
    free = np.ones(x.size, bool) if blocked is None else ~np.asarray(blocked)
    if block_eos and 0 <= eos_id < x.size:
        free[eos_id] = False
    for w, v in zip(words, values):
        if x[w] == mx and free[w]:
            return np.array([-v + np.float32(0.0)], np.float32), lse, tol          # fl(0 - L) = -L; -0 + 0 = +0
    lo = np.float32(max(lse - tol, 0.0))                              # Z >= 1 (the argmax's e is 1), so L >= +0
    b_lo = int(lo.view(np.uint32)) + (float(lo) < lse - tol)
    b_hi = int(np.float32(lse + tol).view(np.uint32))
    while float(np.array(b_hi, np.uint32).view(np.float32)) > lse + tol:
        b_hi -= 1
    mid = int(np.float32(lse).view(np.uint32))                        # the cap nearest: a window of bit patterns around lse64
    c = np.arange(max(b_lo, mid - cap // 2), min(b_hi, mid + cap // 2) + 1, dtype=np.int64)
    if c.size == 0:
        return np.zeros(0, np.float32), lse, tol
    cand = c.astype(np.uint32).view(np.float32)
    cand = cand[np.argsort(np.abs(cand.astype(np.float64) - lse), kind="stable")][:cap]
    got = _values_at(x, words, cand, blocked, block_eos, eos_id)
    ok = (canonical(got).view(np.uint32) == canonical(values).view(np.uint32)[None, :]).all(1)
    return cand[ok], lse, tol


def row_stage(x, K, words, values, blocked=None, block_eos=False, eos_id=-1, exclude=()):
    """The row's restatement matched to the kernel's returned pairs (its top K, plus the constrained kernel's completing words):
    (L, lse64, tol, lp [V], top words [K], top lp [K]).  L is the first recovered candidate whose restated top K equals the kernel's,
    or the nearest one (the comparison then shows the difference); L, lse64 and tol are NaN for a non-finite row."""
    x = np.asarray(x, dtype=np.float32)
    if nonfinite(x):
        lp = row_logp(x, np.nan, blocked, block_eos, eos_id)
        return (np.float32(np.nan), math.nan, math.nan, lp) + rank(lp, K, exclude)
    cands, lse, tol = recover_lse(x, words, values, blocked, block_eos, eos_id)
    want_w = np.asarray(words[:K], dtype=np.int64)
    want_v = canonical(values[:K]).view(np.uint32)
    best = None
    for L in cands[:16]:
        lp = row_logp(x, L, blocked, block_eos, eos_id)
        tw, tl = rank(lp, K, exclude)
        res = (np.float32(L), lse, tol, lp, tw, tl)
        if np.array_equal(tw, want_w) and np.array_equal(tl.view(np.uint32), want_v):
            return res
        best = best or res
    if best is None:                                                  # no candidate: restate at the nearest fp32 to lse64
        L = np.float32(lse)
        lp = row_logp(x, L, blocked, block_eos, eos_id)
        best = (L, lse, tol, lp) + rank(lp, K, exclude)
    return best


def to_word(w):
    """An int64 word id as the kernels read it: ids outside int32 become -1."""
    w = np.asarray(w, dtype=np.int64)
    return np.where((w >= INT32_MIN) & (w <= INT32_MAX), w, -1)


def carry(hist_in, prev_ptr, prev_wid, width, f):
    """hist_out[:, :f] of frame f >= 1: row i continues hist_in[(i // width) * width + p, :f-1], p = prev_ptr[i] (0 at f = 1), with
    -1 words when p lies outside [0, width), then to_word(prev_wid[i]).  hist_in [rows, >= f-1], prev_ptr / prev_wid int64 [rows]."""
    prev_wid = np.asarray(prev_wid, dtype=np.int64).reshape(-1)
    rows = prev_wid.size
    out = np.full((rows, f), -1, dtype=np.int64)
    p = np.zeros(rows, np.int64) if f == 1 else np.asarray(prev_ptr, dtype=np.int64).reshape(-1)
    ok = (p >= 0) & (p < width)
    if f > 1:
        src = (np.arange(rows) // width) * width + np.where(ok, p, 0)
        out[:, :f - 1] = np.where(ok[:, None], np.asarray(hist_in, dtype=np.int64)[src, :f - 1], -1)
    out[:, f - 1] = to_word(prev_wid)
    return out


def prompt_carry(hist_in, prev_ptr, prev_wid, width, f, hist_off):
    """The history of a prompted row at trace frame f, hist_off + f entries: at f = 0 row i is hist_in[i, :hist_off] (one row per
    image, its prompt right-aligned behind -1 entries); at f >= 1 it is carry(..., hist_off + f), so prev_ptr is read whenever
    hist_off + f > 1 (from f = 1 on when hist_off > 0)."""
    if f == 0:
        return np.asarray(hist_in, dtype=np.int64)[:, :hist_off].copy()
    return carry(hist_in, prev_ptr, prev_wid, width, hist_off + f)


def eos_blocked(eos_until, g, rows):
    """bool [rows]: the prompted rows whose [EOS] is blocked at generated word g: g + 1 <= eos_until[i]; none when eos_until is
    None (never blocked, whatever an unprompted call's block_eos would say)."""
    if eos_until is None:
        return np.zeros(rows, bool)
    e = np.asarray(eos_until, dtype=np.int64).reshape(-1)
    assert e.size == rows, (e.size, rows)
    return g + 1 <= e


def ngram_blocked(hists, n, ignore, V):
    """bool [rows, V]: the words the duplicate-n-gram rule blocks for each history (beam._dup_ngram_candidates, ids in [0, V))."""
    from vlp_b200.beam import _dup_ngram_candidates

    out = np.zeros((len(hists), V), bool)
    for i, h in enumerate(hists):
        ws = [w for w in _dup_ngram_candidates([int(t) for t in h], n, set(ignore)) if 0 <= w < V]
        out[i, ws] = True
    return out
