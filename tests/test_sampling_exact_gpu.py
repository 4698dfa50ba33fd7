"""GPU: the top-k / top-p sampler (vlpk_sample_tokens) draw by draw against tools/sampling_oracle.py.

Every row's fp32 x is restated on the host (bf16 logits + bias rounded to bf16, or fp32 logits + bias; -10000 at blocked words and at
[EOS] under block_eos) and its uniform recomputed from the host Philox model at the kernel's own (seed; f, row).  A row whose kept set
and draw are further than the oracle's rounding bounds from any boundary must draw the oracle's word exactly; a near row must draw one
of the oracle's plausible words (kept by some kernel-legal cut, with a cumulative interval within the bounds of u * S).  Each case
checks at least min_exact() of its rows exactly.  Every drawn word has positive fp32 weight: its score is finite and lies within
C_SCORE * 2^-23 * (1 + |x - mx| + |log Z|) of the fp64 log-probability.  The dropout keep masks of the device generator are held
bitwise to the same host model, and whole sampling decodes are replayed frame by frame through the oracle."""
import math

import numpy as np
import pytest
import torch

from tools import sampling_oracle as so
from vlp_b200 import beam, ops, synth
from vlp_b200.decode import PAD_ID

from test_nbest_gpu import _args, _decoder

pytestmark = pytest.mark.gpu
DEV = "cuda"
EOS = 102
T_CAP = 4
# Score: |score - ((x - mx) - log Z)| <= C_SCORE * 2^-23 * (1 + |x - mx| + |log Z|): 2x the worst measured on an H100 80GB HBM3
# (1.72), under a ceiling of 8.
C_SCORE = 4.0
SMEM_MAX = 200 * 1024          # SAMPLE_SMEM_MAX


# The share of each case's rows checked exactly (rows with one plausible word), measured on an H100 80GB HBM3 (700 W limit): every case
# not listed here checks all its rows exactly.  The share depends on the inputs and the oracle's bounds only, not on the kernel's draws.
MEASURED_EXACT = {
    "V1023-topk63": 0.9896, "V1023-topp0.999999": 0.9896, "V1023-topp1.0": 0.9896, "V1025-topp0.999999": 0.9896,
    "V1025-topp1.0": 0.9896, "V28996-topp0.9": 0.9375, "V28996-topp0.999999": 0.8125, "V28996-topp1.0": 0.8438,
    "V30522-topp0.9": 0.9062, "V30522-topp0.999999": 0.8750, "V30522-topp1.0": 0.8750, "V3072-topp0.999999": 0.9896,
    "V3073-topp0.9": 0.9896, "V3073-topp0.999999": 0.9792, "V3073-topp1.0": 0.9792, "V49644-topp0.9": 0.8125,
    "V49644-topp0.999999": 0.7500, "V49644-topp1.0": 0.7500, "neginf-torch.float32-V30522-topp0.3": 0.9792,
    "neginf-torch.float32-V30522-topp0.9": 0.8542, "neginf-torch.float32-V30522-topp0.999999": 0.8750,
    "neginf-torch.float32-V30522-topp1.0": 0.8958, "neginf-torch.float32-V3073-topp0.999999": 0.9609,
    "neginf-torch.float32-V3073-topp1.0": 0.9688, "ngram-topk64": 0.9922, "quantised-torch.bfloat16-V30522-topp0.3": 0.9792,
    "quantised-torch.bfloat16-V30522-topp0.9": 0.7083, "quantised-torch.bfloat16-V30522-topp0.999999": 0.5625,
    "quantised-torch.bfloat16-V30522-topp1.0": 0.5625, "quantised-torch.bfloat16-V3073-topp0.9": 0.9531,
    "quantised-torch.bfloat16-V3073-topp0.999999": 0.9375, "quantised-torch.bfloat16-V3073-topp1.0": 0.9375,
    "quantised-torch.float32-V30522-topp0.3": 0.9792, "quantised-torch.float32-V30522-topp0.9": 0.7083,
    "quantised-torch.float32-V30522-topp0.999999": 0.5625, "quantised-torch.float32-V30522-topp1.0": 0.5625,
    "quantised-torch.float32-V3073-topp0.9": 0.9531, "quantised-torch.float32-V3073-topp0.999999": 0.9375,
    "quantised-torch.float32-V3073-topp1.0": 0.9375, "torch.bfloat16-biasFalse-V1025-topp0.9": 0.9922,
    "torch.bfloat16-biasFalse-V3073-topk64": 0.9922, "torch.bfloat16-biasFalse-V3073-topp0.9": 0.9922,
    "torch.bfloat16-biasTrue-V3073-topp0.9": 0.9844}


def min_exact(name):
    """A case must check at least 1 - 2 x its own measured share of near rows exactly."""
    return 1.0 - 2.0 * (1.0 - MEASURED_EXACT.get(name, 1.0))


# seeds >= 2^32 whose uniform at (frame 3, row 0) is exactly 0 and exactly 1/2 (so.search_seeds from 2^32; re-checked below)
SEED_U0, SEED_HALF = 4299676250, 4303814993


def _np(t):
    return t.detach().float().cpu().numpy()


def _run(logits, mode, k=1, p=1.0, seed=0, bias=None, f=0, T=T_CAP, seq=None, finished=None, **kw):
    rows = logits.shape[0]
    seq = torch.full((rows, T), -7, dtype=torch.int64, device=DEV) if seq is None else seq
    score = torch.full((rows, T), 0.125, dtype=torch.float32, device=DEV)
    finished = torch.zeros(rows, dtype=torch.int32, device=DEV) if finished is None else finished
    live = torch.full((1,), rows - int(finished.sum()), dtype=torch.int32, device=DEV)
    ops.sample_tokens(logits, bias, mode, k, p, seed, f, seq, score, finished, live, kw.pop("eos_id", EOS), **kw)
    return seq, score, finished, live


def check_rows(name, x, mode, k, p, seed, f, ids, scores, rows=None, least=None):
    """Hold the draws ids [R] and scores [R] of rows x [R, V] (the kernel's fp32 x) to the oracle; returns the number of rows checked exactly."""
    ids, scores = ids.cpu().numpy(), scores.cpu().numpy().astype(np.float64)
    rows = np.arange(x.shape[0]) if rows is None else rows
    u = so.uniform(seed, f, rows.astype(np.uint64))
    exact = 0
    for i, r in enumerate(rows):
        fr = so.frame(x[i], mode, k, p, float(u[i]))
        w = int(ids[i])
        assert 0 <= w < x.shape[1], (name, r, w)
        if fr.near:
            assert fr.plausible[w], (name, int(r), w, fr.word, float(u[i]), fr.cut_margin, fr.draw_margin)
        else:
            exact += 1
            assert w == fr.word, (name, int(r), w, fr.word, float(u[i]), fr.cut_margin, fr.draw_margin)
        assert math.isfinite(scores[i]), (name, int(r), w, "a drawn word of zero fp32 weight")
        want = float(fr.d[w] - fr.log_z)
        unit = 2.0 ** -23 * (1.0 + abs(float(fr.d[w])) + abs(fr.log_z))
        err = abs(scores[i] - want)
        assert err <= C_SCORE * unit, (name, int(r), scores[i], want, err / unit)
    frac = exact / len(rows)
    print(f"exact {name} {exact}/{len(rows)}")
    assert frac >= (min_exact(name) if least is None else least), (name, frac)
    return exact


def _x(logits, bias, blocked=None, block_eos=False):
    return so.head_x(_np(logits), None if bias is None else _np(bias), logits.dtype == torch.bfloat16, blocked, block_eos, EOS)


def _gen_logits(gen, rows, V, dtype, scale=2.0, quant=None):
    x = torch.randn(rows, V, generator=gen) * scale
    if quant:
        x = torch.round(x / quant) * quant
    return x.to(DEV, dtype)


def _settings():
    return [("topk", k, 1.0) for k in (1, 2, 63, 64)] + [("topp", 64, p) for p in (1e-9, 0.3, 0.9, 0.999999, 1.0)]


def _vmax(T_cap):
    V = 1
    while ((V + 1) + ((V + 1) + 31) // 32 + T_cap) * 4 <= SMEM_MAX:
        V += 1
    return V


VOCABS = [1, 2, 31, 32, 33, 64, 65, 1023, 1024, 1025, 3072, 3073, 28996, 30522, _vmax(T_CAP)]


@pytest.mark.parametrize("V", VOCABS)
def test_draws_equal_the_oracle_across_vocabularies(V):
    gen = torch.Generator().manual_seed(V)
    rows = 96 if V < 20000 else 32
    logits = _gen_logits(gen, rows, V, torch.bfloat16, scale=3.0)
    bias = _gen_logits(gen, 1, V, torch.bfloat16, scale=0.5)[0]
    x = _x(logits, bias)
    seed = (1 << 32) + 977 * V
    for mode, k, p in _settings():
        seq, sc, _, _ = _run(logits, mode, k, p, seed=seed, bias=bias, f=T_CAP - 1)
        check_rows(f"V{V}-{mode}{k if mode == 'topk' else p}", x, mode, k, p, seed, T_CAP - 1, seq[:, -1], sc[:, -1])


def test_the_next_vocabulary_is_refused_before_a_launch():
    V = _vmax(T_CAP) + 1
    logits = torch.zeros(2, V, dtype=torch.bfloat16, device=DEV)
    seq = torch.full((2, T_CAP), -7, dtype=torch.int64, device=DEV)
    with pytest.raises(RuntimeError):
        ops.sample_tokens(logits, None, "topk", 4, 1.0, 0, 0, seq, None, torch.zeros(2, dtype=torch.int32, device=DEV),
                          torch.full((1,), 2, dtype=torch.int32, device=DEV), EOS)
    torch.cuda.synchronize()
    assert bool((seq == -7).all())


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("with_bias", [False, True])
@pytest.mark.parametrize("V", [1025, 3073])
def test_dtypes_bias_and_padded_rows(dtype, with_bias, V):
    """ld > V with NaN in the gap columns: a gap column read would poison the maximum."""
    gen = torch.Generator().manual_seed(V + 7 * with_bias)
    rows, ld = 128, V + 37
    wide = torch.full((rows, ld), float("nan"), dtype=dtype, device=DEV)
    wide[:, :V] = _gen_logits(gen, rows, V, dtype, scale=2.5)
    logits = wide[:, :V]
    bias = _gen_logits(gen, 1, V, dtype, scale=0.5)[0] if with_bias else None
    x = _x(logits, bias)
    seed = 5 + (1 << 40)
    for mode, k, p in (("topk", 64, 1.0), ("topk", 2, 1.0), ("topp", 64, 0.9), ("topp", 64, 0.3)):
        seq, sc, _, _ = _run(logits, mode, k, p, seed=seed, bias=bias, f=2)
        check_rows(f"{dtype}-bias{with_bias}-V{V}-{mode}{k if mode == 'topk' else p}", x, mode, k, p, seed, 2, seq[:, 2], sc[:, 2])
        assert bool((seq[:, [0, 1, 3]] == -7).all()) and bool((sc[:, [0, 1, 3]] == 0.125).all())


def _shape_rows(shape, gen, rows, V, dtype):
    if shape == "quantised":                                        # tie groups of hundreds of words: the cut falls inside one
        return _gen_logits(gen, rows, V, dtype, scale=2.0, quant=1.0)
    if shape == "equal":
        return torch.full((rows, V), 0.75, dtype=dtype, device=DEV)
    if shape == "peaky":                                            # one word at 0, every other e zero or subnormal
        x = -90.0 - 30.0 * torch.rand(rows, V, generator=gen)
        x[torch.arange(rows), torch.randint(0, V, (rows,), generator=gen)] = 0.0
        return x.to(DEV, dtype)
    if shape == "neginf":
        x = torch.randn(rows, V, generator=gen) * 2.0
        x[torch.rand(rows, V, generator=gen) < 0.7] = float("-inf")
        x[:, 5] = 1.0
        return x.to(DEV, dtype)
    raise ValueError(shape)


@pytest.mark.parametrize("shape,dtype", [("quantised", torch.bfloat16), ("quantised", torch.float32), ("equal", torch.bfloat16),
                                         ("peaky", torch.float32), ("peaky", torch.bfloat16), ("neginf", torch.float32)])
@pytest.mark.parametrize("V", [65, 3073, 30522])
def test_row_shapes(shape, dtype, V):
    gen = torch.Generator().manual_seed(V * 3 + len(shape))
    rows = 128 if V < 20000 else 48
    logits = _shape_rows(shape, gen, rows, V, dtype)
    x = _x(logits, None)
    seed = 31337
    for mode, k, p in _settings():
        seq, sc, _, _ = _run(logits, mode, k, p, seed=seed, f=1)
        check_rows(f"{shape}-{dtype}-V{V}-{mode}{k if mode == 'topk' else p}", x, mode, k, p, seed, 1, seq[:, 1], sc[:, 1])


def test_all_but_one_word_blocked():
    """Every word but one is a duplicate-n-gram candidate (n = 1 over a history holding them all) and [EOS] is blocked."""
    V, rows, f = 200, 64, 199
    T = f + 1
    gen = torch.Generator().manual_seed(4)
    logits = _gen_logits(gen, rows, V, torch.bfloat16, scale=3.0)
    free = torch.randint(0, V, (rows,), generator=gen)
    free[free == EOS] = 3
    hist = torch.zeros(rows, T, dtype=torch.int64)
    blocked = np.ones((rows, V), dtype=bool)
    for r in range(rows):
        words = [w for w in range(V) if w != int(free[r])]
        hist[r, :len(words)] = torch.tensor(words)
        hist[r, len(words):f] = words[-1]
        blocked[r] = False
        for w in beam._dup_ngram_candidates(hist[r, :f].tolist(), 1, set()):
            blocked[r, w] = True
    x = _x(logits, None, blocked=blocked, block_eos=True)
    for mode, k, p in (("topk", 64, 1.0), ("topp", 64, 0.9), ("topp", 64, 1.0)):
        seq, sc, _, _ = _run(logits, mode, k, p, seed=9, f=f, T=T, seq=hist.to(DEV).clone(), ngram=1, block_eos=True)
        check_rows(f"blocked-{mode}{p}", x, mode, k, p, 9, f, seq[:, f], sc[:, f])
        if mode == "topk" or p < 1.0:
            assert torch.equal(seq[:, f].cpu(), free)


def test_ngram_histories_outside_int32_and_an_ignore_set():
    V, rows, T, f, n = 300, 128, 24, 20, 2
    gen = torch.Generator().manual_seed(8)
    hist = torch.randint(0, 8, (rows, T), generator=gen)
    hist[::4, 3] = (1 << 40) + 5                                     # outside int32: the kernel reads -1
    hist[1::4, 6] = -(1 << 35)
    logits = _gen_logits(gen, rows, V, torch.float32, scale=1.0)
    logits[:, :8] += 6.0                                             # the history's words are the likely ones
    ign = torch.tensor([2], dtype=torch.int32, device=DEV)
    blocked = np.zeros((rows, V), dtype=bool)
    for r in range(rows):
        h = [w if -2 ** 31 <= w < 2 ** 31 else -1 for w in hist[r, :f].tolist()]
        for w in beam._dup_ngram_candidates(h, n, {2}):
            if 0 <= w < V:
                blocked[r, w] = True
    assert blocked.sum() >= rows
    x = _x(logits, None, blocked=blocked)
    for mode, k, p in (("topk", 64, 1.0), ("topk", 1, 1.0), ("topp", 64, 0.9)):
        seq, sc, _, _ = _run(logits, mode, k, p, seed=12, f=f, T=T, seq=hist.to(DEV).clone(), ngram=n, ignore=ign)
        check_rows(f"ngram-{mode}{k}", x, mode, k, p, 12, f, seq[:, f], sc[:, f])
        assert torch.equal(seq[:, :f].cpu(), hist[:, :f]) and torch.equal(seq[:, f + 1:].cpu(), hist[:, f + 1:])


def test_finished_rows_and_the_live_count():
    V, rows, f = 1000, 512, 2
    gen = torch.Generator().manual_seed(6)
    logits = _gen_logits(gen, rows, V, torch.bfloat16)
    logits[:, EOS] = torch.where(torch.rand(rows, generator=gen) < 0.5, 8.0, -8.0).to(DEV, torch.bfloat16)
    finished = (torch.rand(rows, generator=gen) < 0.25).int().to(DEV)
    fin0 = finished.clone()
    seq, sc, fin, live = _run(logits, "topp", 64, 0.9, seed=4, f=f, finished=finished, pad_id=3)
    done = fin0.bool()
    assert bool((seq[done, f] == 3).all()) and bool((sc[done, f] == 0).all())
    x = _x(logits, None)
    open_rows = torch.nonzero(~done).flatten().cpu().numpy()
    check_rows("finished-topp", x[open_rows], "topp", 64, 0.9, 4, f, seq[~done, f], sc[~done, f], rows=open_rows)
    eos_now = (seq[:, f] == EOS) & ~done
    assert int(eos_now.sum()) > 50
    assert torch.equal(fin.bool(), done | eos_now)
    assert int(live) == rows - int(fin0.sum()) - int(eos_now.sum())
    others = [c for c in range(T_CAP) if c != f]
    assert bool((seq[:, others] == -7).all()) and bool((sc[:, others] == 0.125).all())


# --- adversarial uniforms ----------------------------------------------------------------------------------------------------------
def test_edge_uniforms_on_exact_rows():
    """All-equal rows sum exactly: u = 0 draws the first kept word, u = 1/2 lands exactly on a boundary and draws the word after it."""
    f = 3
    for seed, u in ((SEED_U0, 0.0), (SEED_HALF, 0.5)):
        assert float(so.uniform(seed, f, np.uint64(0))) == u
        for V in (4, 64, 1025):
            logits = torch.zeros(1, V, dtype=torch.float32, device=DEV)
            x = _x(logits, None)
            for mode, k, p in (("topk", 64, 1.0), ("topp", 64, 0.5), ("topp", 64, 1.0)):
                seq, sc, _, _ = _run(logits, mode, k, p, seed=seed, f=f)
                fr = so.frame(x[0], mode, k, p, u)
                assert not fr.near
                assert int(seq[0, f]) == fr.word == (0 if u == 0 else int(fr.kept.sum()) // 2), (V, mode, p)
                check_rows(f"edge-u{u}-V{V}-{mode}{p}", x, mode, k, p, seed, f, seq[:, f], sc[:, f])


def _zero_weight_rows(dtype, V=30522):
    """Chunk 0 (words 0..C-1) holds the maximum, chunk 1 twenty words of e ~ 0.9 * 2^-24 (each below half an ulp of 1) and then kept
    words of zero fp32 weight; every other word has zero weight too.  The chunk's walked sum stays at 1 while the scan's prefix is
    1 + ~9 ulps, so a goal u * S in between (u >= 1 - 2^-20) finds no word whose running sum exceeds it."""
    C = ((V + 1023) // 1024) | 1
    low = float("-inf") if dtype == torch.float32 else -200.0
    x = torch.full((1, V), low)
    x[0, 0] = 0.0
    x[0, C:C + 20] = math.log(0.9 * 2.0 ** -24)
    return x.to(DEV, dtype)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_no_zero_weight_draw_at_the_top_of_the_unit_interval(dtype):
    f = 1
    logits = _zero_weight_rows(dtype)
    x = _x(logits, None)
    seeds = so.search_seeds(lambda a: a >= 1 - 2.0 ** -20, f, 0, 1 << 33, 1 << 26, want=3)
    assert len(seeds) == 3
    for seed in seeds:
        for k in (64, 63, 25):
            seq, sc, _, _ = _run(logits, "topk", k, 1.0, seed=seed, f=f)
            check_rows(f"zero-weight-{dtype}-k{k}", x, "topk", k, 1.0, seed, f, seq[:, f], sc[:, f], least=0.0)
            w = int(seq[0, f])
            assert x[0, w] > -100.0, (seed, k, w)
        seq, sc, _, _ = _run(logits, "topp", 64, 1.0, seed=seed, f=f)
        check_rows(f"zero-weight-{dtype}-topp", x, "topp", 64, 1.0, seed, f, seq[:, f], sc[:, f], least=0.0)


def test_goals_within_rounding_units_of_a_boundary():
    """Rows of one random x; the (seed, row) counters are chosen so that u * S lies within a few rounding units of a cumulative
    boundary of the kept words: those rows are near, and must still draw one of the two words at the boundary."""
    V, f = 1000, 2
    gen = torch.Generator().manual_seed(11)
    logits = _gen_logits(gen, 1, V, torch.float32, scale=1.0)
    x = _x(logits, None)[0]
    for mode, k, p in (("topk", 64, 1.0), ("topp", 64, 0.9)):
        fr = so.frame(x, mode, k, p, 0.5)
        idx = np.flatnonzero(fr.kept)
        cum = np.cumsum(np.exp(fr.d[idx]))
        S = cum[-1]
        inner = cum[:-1]
        tol = 64 * 2.0 ** -24 * S

        def pred(u, inner=inner, S=S, tol=tol):
            g = u.astype(np.float64) * S
            j = np.clip(np.searchsorted(inner, g), 1, inner.size - 1)
            return np.minimum(np.abs(inner[j] - g), np.abs(inner[j - 1] - g)) < tol

        hits = so.select_uniforms(pred, f, 4096, range(1 << 32, (1 << 32) + 64))
        assert len(hits) >= 8
        for seed in sorted({s for s, _ in hits})[:8]:
            rows = max(r for s, r in hits if s == seed) + 1
            lg = logits.expand(rows, V).contiguous()
            seq, sc, _, _ = _run(lg, mode, k, p, seed=seed, f=f)
            check_rows(f"boundary-{mode}", np.broadcast_to(x, (rows, V)), mode, k, p, seed, f, seq[:, f], sc[:, f], least=0.0)


# --- the device generator ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("p", [0.1, 0.5])
@pytest.mark.parametrize("seed", [12345, (1 << 32) + 7, (1 << 63) + 3])
def test_dropout_keep_masks_equal_the_host_philox(p, seed):
    for site in [8 * i + s for i in (0, 3) for s in range(8)] + [1 << 20, (1 << 21) + 1]:
        for n in (13, 1000, 4099):
            got = ops.dropout_keep_mask(p, seed, site, n).cpu().numpy()
            assert np.array_equal(got, so.keep_mask(p, seed, site, n)), (p, seed, site, n)


# --- whole decodes -----------------------------------------------------------------------------------------------------------------
class _Recorder:
    """Wraps ops.sample_tokens: snapshots each call's inputs before it and its column f after it."""

    def __init__(self):
        self.calls, self.inner = [], ops.sample_tokens

    def __call__(self, logits, bias, mode, topk, topp, seed, f, seq, score, finished, live, eos_id, pad_id=0, block_eos=False, ngram=0,
                 ignore=None):
        V = logits.shape[-1]
        rec = dict(logits=logits.reshape(-1, V).clone(), bias=None if bias is None else bias.clone(), mode=mode, k=topk, p=topp,
                   seed=seed, f=f, hist=seq[:, :f].clone(), finished=finished.clone(), eos=eos_id, pad=pad_id, block_eos=block_eos,
                   ngram=ngram, ignore=set() if ignore is None else set(ignore.tolist()))
        self.inner(logits, bias, mode, topk, topp, seed, f, seq, score, finished, live, eos_id, pad_id, block_eos, ngram, ignore)
        rec["ids"], rec["scores"], rec["finished_after"] = seq[:, f].clone(), score[:, f].clone(), finished.clone()
        self.calls.append(rec)


# Decode replays: the share of all open rows over a decode's frames checked exactly (each frame has only a few open rows), at most
# 1 - 2 x the worst measured share of near rows (4 of 246, L = 143 top-p 0.95).
DECODE_MIN_EXACT = 0.96


def _check_decode(rec, name):
    """Every recorded frame's draws against the oracle on the recorded inputs; returns (rows checked exactly, open rows)."""
    assert rec.calls
    exact = total = 0
    for c in rec.calls:
        done = c["finished"].bool().cpu()
        ids = c["ids"].cpu()
        assert bool((ids[done] == c["pad"]).all()) and bool((c["scores"].cpu()[done] == 0).all())
        rows = torch.nonzero(~done).flatten().numpy()
        if rows.size == 0:
            continue
        V = c["logits"].shape[1]
        blocked = np.zeros((rows.size, V), dtype=bool)
        if c["ngram"] and c["f"] >= c["ngram"]:
            for i, r in enumerate(rows):
                for w in beam._dup_ngram_candidates(c["hist"][r].tolist(), c["ngram"], c["ignore"]):
                    if 0 <= w < V:
                        blocked[i, w] = True
        x = so.head_x(_np(c["logits"][rows]), None if c["bias"] is None else _np(c["bias"]), c["logits"].dtype == torch.bfloat16, blocked,
                      c["block_eos"], c["eos"])
        exact += check_rows(f"{name}-f{c['f']}", x, c["mode"], c["k"], c["p"], c["seed"], c["f"], c["ids"][rows], c["scores"][rows],
                            rows=rows, least=0.0)
        total += rows.size
        assert torch.equal(c["finished_after"].bool().cpu(), done | (ids == c["eos"]))
    print(f"exact {name} {exact}/{total} over {len(rec.calls)} frames")
    assert exact >= DECODE_MIN_EXACT * total, (name, exact, total)


DECODES = [dict(sampling_method="topk", topk=64), dict(sampling_method="topp", topp=0.9),
           dict(sampling_method="topk", topk=64, use_kv_cache=False), dict(sampling_method="topp", topp=0.9, use_kv_cache=False),
           dict(sampling_method="topp", topp=0.9, num_return_sequences=3),
           dict(sampling_method="topk", topk=16, forbid_duplicate_ngrams=True, ngram_size=2, forbid_ignore_set={7}, min_len=5),
           dict(sampling_method="topp", topp=0.95, dims="L143")]


@pytest.mark.parametrize("case", DECODES, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_decode_draws_equal_the_oracle(case, monkeypatch):
    """Besides the draws: the decode passes frame f as the call's index, its own seed, mode, k and p, the head's bias, [EOS] blocked
    exactly below min_len, its n-gram settings and padding id, and rows image-major (the N samples of image b are rows b*N .. b*N+N-1,
    which share frame 0's logits, and row r of every call is row r of the returned ids)."""
    import dataclasses
    case = dict(case)
    cache = case.pop("use_kv_cache", True)
    dims = dataclasses.replace(synth.SMALL_L123, text=40) if case.pop("dims", None) == "L143" else synth.SMALL_L123
    seed = (1 << 32) + 19
    model = _decoder(dims, seed=seed, **case)
    model.use_kv_cache = cache
    rec = _Recorder()
    monkeypatch.setattr(ops, "sample_tokens", rec)
    B, N = 6, case.get("num_return_sequences", 1)
    ids, _ = model(*_args(dims, B, seed=3), task_idx=None)
    assert len(rec.calls) == model.last_decode_steps
    flat = ids.reshape(B * N, -1).cpu()
    head_bias = model.cls.predictions.bias
    for f, c in enumerate(rec.calls):
        assert c["f"] == f and c["seed"] == seed and c["mode"] == model.sampling_method
        assert c["k"] == model.topk and c["p"] == model.topp
        assert torch.equal(c["bias"], head_bias.to(c["logits"].dtype))
        assert c["block_eos"] == (bool(model.min_len) and f + 1 <= model.min_len)
        assert c["ngram"] == (model.ngram_size if model.forbid_duplicate_ngrams else 0)
        assert c["ignore"] == (set(model.forbid_ignore_set or ()) if model.forbid_duplicate_ngrams else set())
        assert c["pad"] == PAD_ID and c["eos"] == EOS
        assert c["logits"].shape[0] == B * N and torch.equal(flat[:, f], c["ids"].cpu())
    first = rec.calls[0]["logits"].reshape(B, N, -1)
    assert all(torch.equal(first[:, j], first[:, 0]) for j in range(N))
    _check_decode(rec, "decode-" + "-".join(f"{k}={v}" for k, v in case.items()))
