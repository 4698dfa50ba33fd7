"""Host statement of one top-k / top-p sampling frame (vlpk_sample_tokens, sample_kernel in csrc/decode.cu), in numpy.

  philox4x32_10  the counter-based generator of csrc/common.cuh (Philox::gen): key (seed lo32, seed hi32), counter words
                 (ctr_lo lo32, ctr_lo hi32, ctr_hi lo32, ctr_hi hi32), ten rounds; vectorised over arrays of counters.
  uniform        the sampler's draw of row `row` at frame f: u = (Philox(seed; f, row).x >> 8) * 2^-24, in [0, 1 - 2^-24].
  keep_mask      the dropout keep decisions of one site (dropout_keep8): element i keeps iff its 16 bits of
                 Philox(seed; site, i // 8) are >= floor(p * 65536).
  head_x         the kernel's fp32 x of one row: the head's logit (bf16 logits + bias rounded to bf16, or fp32 logits + bias), -10000 added
                 at the words the duplicate-n-gram rule blocks, and x[eos] = -10000 under block_eos.
  frame          the kernel's rule on those x in fp64: words ranked by (x descending, index ascending); top-k keeps the first k, top-p the
                 shortest prefix whose e = exp(x - max x) sum reaches topp * Z; the drawn word is the first kept word in index order whose
                 running e sum exceeds u * (kept e sum).  Two margins say where the kernel's fp32 sums could legitimately decide otherwise.
  select_uniforms  (seed, row) counters of one frame whose uniform satisfies a predicate, so that a test can aim at u = 0, u -> 1 or
                 u * S on a cumulative boundary instead of waiting for them.

The margins are in units of a stated bound on the kernel's fixed-order fp32 sums: each thread sums a chunk of C = ceil(V / 1024) | 1
words, then a shuffle tree (reduction, 10 levels) or scan (at most 12) combines the 1024 chunks, so every partial sum of nonnegative e
is within (C + 14) * 2^-24 of its own magnitude; each e carries expf's error (2 ulp, 4 * 2^-24 relative) and the rounding of x - max x
(|x - max x| * 2^-24 relative), plus 2^-148 absolute where e is subnormal.  Where every e is exactly 0 or 1 the sums are exact integers
and only the products topp * Z and u * S round."""
import math
from collections import namedtuple

import numpy as np

M32 = np.uint64(0xFFFFFFFF)
_MUL0, _MUL1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
_W0, _W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
U24 = 2.0 ** -24
BLOCK = np.float32(-10000.0)
THREADS = 1024                                   # SAMPLE_THREADS: one CTA of 1024 threads per row


def _u64(a):
    return np.asarray(a, dtype=np.uint64) if not isinstance(a, int) else np.asarray(a & 0xFFFFFFFFFFFFFFFF, dtype=np.uint64)


def philox4x32_10(seed, ctr_hi, ctr_lo):
    """uint32 [..., 4]: (x, y, z, w) of Philox4x32-10 keyed by seed at counter (ctr_hi, ctr_lo), broadcast over the arguments."""
    seed, ctr_hi, ctr_lo = np.broadcast_arrays(_u64(seed), _u64(ctr_hi), _u64(ctr_lo))
    k0, k1 = seed & M32, seed >> np.uint64(32)
    c0, c1 = ctr_lo & M32, ctr_lo >> np.uint64(32)
    c2, c3 = ctr_hi & M32, ctr_hi >> np.uint64(32)
    for _ in range(10):
        p0, p1 = _MUL0 * c0, _MUL1 * c2                      # 32 x 32 -> 64 bits: exact in uint64
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32
        k0, k1 = (k0 + _W0) & M32, (k1 + _W1) & M32
    return np.stack([c0, c1, c2, c3], -1).astype(np.uint32)


def uniform(seed, f, rows):
    """fp32 u of rows `rows` (array) at frame f under seed: (Philox(seed; f, row).x >> 8) * 2^-24."""
    x = philox4x32_10(seed, f, rows)[..., 0]
    return ((x >> np.uint32(8)).astype(np.float64) * U24).astype(np.float32)


def keep_mask(p, seed, site, n):
    """uint8 [n] dropout keep decisions of `site` under seed, with thresh16 = floor(fp32(p) * 65536) (make_dropout)."""
    thresh = int(np.float32(p) * np.float32(65536.0))
    r = philox4x32_10(seed, site, np.arange((n + 7) // 8, dtype=np.uint64))
    halves = np.stack([r & np.uint32(0xFFFF), r >> np.uint32(16)], -1).reshape(-1)     # x lo, x hi, y lo, y hi, ...
    return (halves[:n] >= thresh).astype(np.uint8)


def bf16_round(x):
    """fp32 -> nearest bf16 (ties to even), as fp32; finite inputs."""
    b = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    b = (b + np.uint64(0x7FFF) + ((b >> np.uint64(16)) & np.uint64(1))) & np.uint64(0xFFFF0000)
    return b.astype(np.uint32).view(np.float32)


def head_x(logits, bias=None, bf16=True, blocked=None, block_eos=False, eos_id=-1):
    """The kernel's fp32 x of rows `logits` ([..., V] fp32 values of bf16 or fp32 logits; bias [V] likewise, or None)."""
    x = np.asarray(logits, dtype=np.float32)
    if bias is not None:
        x = x + np.asarray(bias, dtype=np.float32)
        if bf16:
            x = bf16_round(x)
    x = np.array(x, dtype=np.float32)
    if blocked is not None:
        x = np.where(blocked, x + BLOCK, x).astype(np.float32)
    if block_eos and 0 <= eos_id < x.shape[-1]:
        x[..., eos_id] = BLOCK
    return x


Frame = namedtuple("Frame", "word kept union plausible score near cut_margin draw_margin d log_z")


def _margin(dist, tol):
    if tol == 0.0:
        return math.inf                                       # exact arithmetic: the comparison itself is exact
    return dist / tol


def frame(x32, mode, k=1, p=1.0, u=0.0):
    """The kernel's rule for one row of fp32 x (finite or -inf, max finite) in fp64.  Returns a Frame:
      word       the drawn word;
      kept       bool [V], the kept set;
      union      bool [V], every word some kept set within the rounding bounds could hold (== kept when the cut is certain);
      plausible  bool [V], the words of union whose cumulative interval lies within the rounding bounds of u * S;
      score      (x - mx) - log Z of word;
      near       whether fp32 rounding could legitimately draw another word: more than one plausible word (a cut or draw margin
                 below 1, or an fp32 e collision of different x at the top-p cut, can make a row near);
      d, log_z   x - mx [V] and log Z, for the score bound."""
    x = np.asarray(x32, dtype=np.float32).reshape(-1)
    assert not np.isnan(x).any() and not np.isposinf(x).any()
    V = x.size
    x64 = x.astype(np.float64)
    mx = x64.max()
    assert np.isfinite(mx)
    d = x64 - mx
    e = np.exp(d)
    C = ((V + THREADS - 1) // THREADS) | 1
    unit = (d == 0) | np.isneginf(d)                          # e exactly 1 or 0 on the device too
    exact = bool(unit.all())
    eps = np.where(unit, 0.0, (4.0 + np.abs(np.where(np.isneginf(d), 0.0, d))) * U24 * e + np.where(e < 2.0 ** -125, 2.0 ** -148, 0.0))
    sum_rel = 0.0 if exact else (C + 14) * U24
    order = np.lexsort((np.arange(V), -x64))
    log_z = math.log(e.sum())
    topp = mode == "topp"
    kept = np.zeros(V, dtype=bool)
    union = np.zeros(V, dtype=bool)
    maybe_out = np.zeros(V, dtype=bool)                       # kept words some kernel-legal kept set leaves out
    cut_margin, collision = math.inf, False
    if not topp:
        kept[order[:min(k, V)]] = True
        union[:] = kept
    else:
        c = np.cumsum(e[order])
        Z = c[-1]
        t = float(np.float32(p)) * Z
        t_round = 0.0 if float(np.float32(t)) == t else U24 * t
        # the kernel compares fp32 masses (each within sum_rel * Z + sum eps of its exact value) with fp32 topp * Z, then counts the
        # ties it needs by one more fp32 subtraction and division
        tol = 2.0 * (sum_rel * Z + eps.sum()) + 3.0 * t_round
        npos = int(np.count_nonzero(e > 0))
        m = max(1, min(V, 1 + int(np.count_nonzero(c < t))))
        m_lo = max(1, min(m, 1 + int(np.count_nonzero(c < t - tol))))
        # at topp = 1 the target is Z itself and the mass of every positive word is summed in Z's own order: that side is exact
        m_hi = m if float(np.float32(p)) == 1.0 else max(m, min(max(npos, 1), 1 + int(np.count_nonzero(c < t + tol))))
        kept[order[:m]] = True
        union[order[:m_hi]] = True
        maybe_out[order[m_lo:m]] = True
        sides = ([t - c[m - 2]] if m >= 2 else []) + ([c[m - 1] - t] if m_hi > m or float(np.float32(p)) < 1.0 else [])
        cut_margin = _margin(min(sides), tol) if sides else math.inf
        if m_lo != m or m_hi != m:
            cut_margin = min(cut_margin, 0.0)
        if m < V:                                             # fp32 e of different x may collide: the kernel then ties them by index
            a, b = order[m - 1], order[m]
            rel = 2.0 * (8.0 + abs(d[a]) + abs(d[b])) * U24
            if x64[a] != x64[b] and e[b] > 0 and e[a] - e[b] <= rel * e[a]:
                collision = True
                union |= e >= e[a] * (1.0 - rel)
                union &= e > 0
                maybe_out |= kept & (e <= e[a] * (1.0 + rel))
    idx = np.flatnonzero(kept)
    cum = np.cumsum(e[idx])
    S = cum[-1]
    uu = float(np.float32(u))
    goal = uu * S
    word = int(idx[min(int(np.searchsorted(cum, goal, side="right")), idx.size - 1)])
    g_round = 0.0 if (exact and float(np.float32(goal)) == goal) else U24 * goal
    tol_d = 2.0 * (sum_rel * S + eps[idx].sum()) + g_round
    inner = cum[(cum > 0) & (cum < S)]
    dist = float(np.abs(inner - goal).min()) if inner.size else math.inf
    draw_margin = math.inf if dist == math.inf else _margin(dist, tol_d)
    # every kept set the kernel may hold lies between order[:m_lo] and union, so its cumulative sums and u * S lie within the uncertain
    # mass mu of union's (plus the rounding bound tol_d): the words whose union interval comes that close to u * S are the plausible
    # draws, and a row is exact when that is the oracle's word alone.  Words of zero weight are never drawn.
    ui = np.flatnonzero(union & (e > 0))
    mu = float(e[union & ~kept].sum() + e[maybe_out].sum())
    ucum = np.cumsum(e[ui])
    ub = ucum - e[ui]
    g_u = uu * ucum[-1]
    slack = tol_d + 2.0 * mu
    plausible = np.zeros(V, dtype=bool)
    plausible[ui[(ub - slack <= g_u) & (g_u < ucum + slack)]] = True
    plausible[word] = True
    near = int(plausible.sum()) > 1
    return Frame(word, kept, union, plausible, float(d[word] - log_z), near, cut_margin, draw_margin, d, log_z)


def select_uniforms(pred, f, rows, seeds):
    """[(seed, row)] of frame f, rows in range(rows) and seed in `seeds`, whose uniform satisfies pred (vectorised over an fp32 array)."""
    hits = []
    r = np.arange(rows, dtype=np.uint64)
    for s in seeds:
        ok = np.flatnonzero(pred(uniform(int(s), f, r)))
        hits += [(int(s), int(i)) for i in ok]
    return hits


def search_seeds(pred, f, row, start, count, want=1, batch=1 << 20):
    """The first `want` seeds in [start, start + count) under which row `row` at frame f draws a uniform satisfying pred."""
    out = []
    for s0 in range(start, start + count, batch):
        s = np.arange(s0, min(s0 + batch, start + count), dtype=np.uint64)
        ok = np.flatnonzero(pred(uniform(s, f, row)))
        out += [int(s[i]) for i in ok[:want - len(out)]]
        if len(out) >= want:
            break
    return out
