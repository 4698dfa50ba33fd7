"""GPU: the prompted selectors (vlpk_sample_tokens_prompt, vlpk_diverse_beam_step_prompt, vlpk_constrained_beam_step_prompt) row by
row and frame by frame against the exact host statements: the sampler's draws against tools/sampling_oracle.py on the kernel's own
(seed; g, row) uniform, the beam rows bit for bit against tools/beam_select_oracle.py on each row's own logsumexp, and the frames'
merges against diverse_beam_oracle.merge / constrained_beam_oracle.merge.

A prompted row's history has hist_off prompt entries (right-aligned behind -1 entries), then the generated words: at f = 0 the beam
rows read row b of hist_in ([B, T_cap]), and from f = 1 on the carry runs over hist_off + f entries and follows prev_ptr
(beam_select_oracle.prompt_carry).  [EOS] is blocked per row while g + 1 <= eos_until[row] (beam_select_oracle.eos_blocked), never
when eos_until is NULL.  Cases: every prompt width hist_off in {0, 1, Tp, f} (g = 0 included), ragged prompts with empty ones,
n-grams inside the prompt and across its end, eos_until below, at and above the boundary and NULL, vocabularies from 1 to the
shared-memory limit at a T_cap that includes hist_off, bf16 / fp32, bias, strided logits with NaN past V, finished rows, histories
longer than the CTA with bad pointers, NaN rows; bitwise identities with the unprompted kernels; and whole prompted decodes replayed
frame by frame."""
import numpy as np
import pytest
import torch

from tools import beam_select_oracle as O
from tools import constrained_beam_oracle as CO
from tools import diverse_beam_oracle as DO
from tools import sampling_oracle as SO
from vlp_b200 import _lib as L
from vlp_b200 import decode, ops

from test_beam_select_exact_gpu import (EOS, _bias, _bits, _logits, _nonfinite_rows, _prev, _same, _table, _traces, _vmax,
                                        run_constrained, run_diverse)
from test_beam_select_exact_gpu import _x as _beam_x
from test_sampling_exact_gpu import DECODE_MIN_EXACT, check_rows

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16

# The share of each sampler case's rows checked exactly (rows with one plausible word).  The share depends on the inputs and the
# oracle's bounds only, not on the kernel's draws; printed by check_rows and confirmed on an H100 80GB HBM3 (700 W limit).  Every case
# not listed checks all its rows exactly.
MEASURED_EXACT = {"V1025-bfloat16-bias0-off1-f4-n2-topp": 0.9843, "V1025-bfloat16-bias1-off9-f9-n2-topp": 0.9843,
    "V1025-float32-bias0-off9-f9-n2-topp": 0.9843, "V1025-float32-bias0-off9-f9-n3-topp": 0.9531,
    "V1025-float32-bias1-off6-f9-n3-topp": 0.9843, "V30522-bfloat16-bias0-off0-f4-n1-topp": 0.9166,
    "V30522-bfloat16-bias0-off1-f4-n2-topp": 0.7500, "V30522-bfloat16-bias0-off6-f9-n3-topp": 0.8750,
    "V30522-bfloat16-bias0-off9-f9-n2-topp": 0.9166, "V30522-bfloat16-bias0-off9-f9-n3-topp": 0.8333,
    "V30522-bfloat16-bias1-off0-f4-n1-topp": 0.9583, "V30522-bfloat16-bias1-off1-f4-n2-topp": 0.9583,
    "V30522-bfloat16-bias1-off6-f9-n3-topp": 0.9583, "V30522-bfloat16-bias1-off9-f9-n2-topp": 0.9583,
    "V30522-float32-bias0-off0-f4-n1-topp": 0.9166, "V30522-float32-bias0-off1-f4-n2-topk": 0.9583,
    "V30522-float32-bias0-off1-f4-n2-topk-null": 0.9583, "V30522-float32-bias0-off1-f4-n2-topp": 0.7500,
    "V30522-float32-bias0-off6-f9-n3-topp": 0.8750, "V30522-float32-bias0-off9-f9-n2-topp": 0.9166,
    "V30522-float32-bias0-off9-f9-n3-topp": 0.8333, "V30522-float32-bias1-off0-f4-n1-topp": 0.9583,
    "V30522-float32-bias1-off1-f4-n2-topp": 0.9583, "V30522-float32-bias1-off6-f9-n3-topp": 0.9583,
    "V30522-float32-bias1-off9-f9-n2-topp": 0.9583, "V3073-bfloat16-bias0-off0-f4-n1-topp": 0.9843,
    "V3073-bfloat16-bias0-off6-f9-n3-topp": 0.9843, "V3073-bfloat16-bias0-off9-f9-n2-topp": 0.9843,
    "V3073-bfloat16-bias0-off9-f9-n3-topp": 0.9843, "V3073-bfloat16-bias1-off0-f4-n1-topp": 0.9687,
    "V3073-bfloat16-bias1-off6-f9-n3-topp": 0.9687, "V3073-float32-bias0-off6-f9-n3-topp": 0.9531,
    "V3073-float32-bias0-off9-f9-n2-topp": 0.9375, "V3073-float32-bias1-off0-f4-n1-topp": 0.9687,
    "V3073-float32-bias1-off1-f4-n2-topp": 0.9687, "V3073-float32-bias1-off6-f9-n3-topp": 0.9843,
    "V3073-float32-bias1-off9-f9-n3-topp": 0.9531, "V33-float32-bias0-off6-f9-n3-topk": 0.9843,
    "V33-float32-bias0-off6-f9-n3-topk-null": 0.9843, "V49636-bfloat16-bias0-off0-f4-n1-topp": 0.7916,
    "V49636-bfloat16-bias0-off1-f4-n2-topp": 0.7916, "V49636-bfloat16-bias0-off6-f9-n3-topp": 0.9583,
    "V49636-bfloat16-bias0-off9-f9-n2-topp": 0.8750, "V49636-bfloat16-bias1-off1-f4-n2-topp": 0.8750,
    "V49636-bfloat16-bias1-off9-f9-n2-topp": 0.9583, "V49636-bfloat16-bias1-off9-f9-n3-topp": 0.9166,
    "V49636-float32-bias0-off0-f4-n1-topp": 0.7916, "V49636-float32-bias0-off1-f4-n2-topp": 0.7916,
    "V49636-float32-bias0-off6-f9-n3-topp": 0.9583, "V49636-float32-bias0-off9-f9-n2-topp": 0.8750,
    "V49636-float32-bias1-off1-f4-n2-topp": 0.8750, "V49636-float32-bias1-off9-f9-n2-topp": 0.9583,
    "V49636-float32-bias1-off9-f9-n3-topp": 0.9166, "finished-topp": 0.9946}


def min_exact(name):
    """A case must check at least 1 - 2 x its own measured share of near rows exactly."""
    return 1.0 - 2.0 * (1.0 - MEASURED_EXACT.get(name, 1.0))


def _np(t):
    return t.detach().float().cpu().numpy()


def _eu(vals):
    return None if vals is None else torch.as_tensor(np.asarray(vals), dtype=torch.int32).to(DEV)


def prompt_rows(gen, rows, Tp, alphabet=8):
    """int32 [rows, Tp]: right-aligned prompt histories of t = r % (Tp + 1) words (empty prompts included) behind -1 entries.  The
    words come from a small alphabet, so n-grams repeat inside the prompt and across its end."""
    h = torch.full((rows, Tp), -1, dtype=torch.int32)
    for r in range(rows):
        t = r % (Tp + 1)
        if t:
            h[r, Tp - t:] = torch.randint(0, alphabet, (t,), generator=gen, dtype=torch.int32)
    return h


def eos_pattern(rows, g):
    """eos_until per row: below the block (-2, 0), at g (not blocked) and at g + 1 (blocked: the boundary), and large."""
    return np.array([(-2, 0, g, g + 1, 1000)[r % 5] for r in range(rows)], np.int32)


# ---------------------------------------------------------------------------------------------------------------------------------
# the sampler
# ---------------------------------------------------------------------------------------------------------------------------------
def sampler_inputs(V, dtype, with_bias, hist_off, f, rows, T_cap, seed, dev=DEV, equal=False):
    """Strided logits (NaN past V), bias, and the rows' histories seq0 [rows, T_cap] (hist_off prompt entries, then generated words,
    -7 after).  equal: every row keeps the 8 history words and a random few others at x = 4 exactly (logit 4 - bias, the bias a
    multiple of 1/16), the rest -inf, so that every e is 0 or 1 and the sums are exact; otherwise Gaussian rows."""
    gen = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, V, generator=gen) * 2.0
    x[:, :min(8, V)] += 3.0                                             # the histories' words are the likely ones
    b = torch.randn(V, generator=gen) * 0.5
    if equal:
        b = (torch.round(b * 16) / 16).clamp(-2.0, 2.0)
        keep = torch.rand(rows, V, generator=gen) < 0.005 * torch.rand(rows, 1, generator=gen)
        keep[:, :min(8, V)] = True
        x = torch.where(keep, 4.0 - (b if with_bias else 0.0), torch.tensor(float("-inf")))
    wide = torch.full((rows, V + 37), float("nan"))
    wide[:, :V] = x
    logits = wide.to(dev, dtype)[:, :V]
    bias = b.to(dev, dtype) if with_bias else None
    seq0 = torch.full((rows, T_cap), -7, dtype=torch.int64)
    seq0[:, :hist_off] = prompt_rows(gen, rows, hist_off).long()
    if hist_off >= 6:                                                    # every third prompt ends in a, b, c, a, b, c: its own
        for r in range(1, rows, 3):                                      # n-grams block a for n = 1, 2 and 3
            abc = torch.tensor([0, 1, 2, 4, 5, 6, 7])[torch.randperm(7, generator=gen)[:3]]
            seq0[r, hist_off - 6:hist_off] = abc.repeat(2)
    seq0[:, hist_off:f] = torch.randint(0, 8, (rows, f - hist_off), generator=gen)
    return logits, bias, seq0


def sampler_x(logits, bias, seq0, f, hist_off, n, ignore, eos_until, eos_id):
    """The kernel's fp32 x of every row under the prompted rules: n-gram blocks over seq0[:, :f], [EOS] by eos_blocked at g."""
    rows, V = logits.shape[0], logits.shape[-1]
    blocked = O.ngram_blocked(O.to_word(seq0[:, :f].numpy()), n, ignore, V) if n and f >= n else None
    x = SO.head_x(_np(logits), None if bias is None else _np(bias), logits.dtype == BF, blocked)
    if 0 <= eos_id < V:
        x[O.eos_blocked(eos_until, f - hist_off, rows), eos_id] = SO.BLOCK
    return x


def sample_case(name, logits, bias, mode, k, p, seed, f, hist_off, seq0, eos_until, n=0, ignore=(), finished=None, eos_id=EOS,
                least=None):
    """One prompted sampler launch held to the oracle: draws keyed by (seed; g = f - hist_off, row), finished rows padded, the live
    count, and every other column untouched.  Returns (seq, score, finished, live) on the host."""
    rows = logits.shape[0]
    seq = seq0.to(DEV)
    score = torch.full(seq.shape, 0.125, device=DEV)
    fin = torch.zeros(rows, dtype=torch.int32) if finished is None else finished.clone()
    done = fin.bool()
    live = torch.full((1,), rows - int(fin.sum()), dtype=torch.int32, device=DEV)
    fin = fin.to(DEV)
    ign = torch.tensor(ignore, dtype=torch.int32, device=DEV) if ignore else None
    ops.sample_tokens(logits, bias, mode, k, p, seed, f, seq, score, fin, live, eos_id, pad_id=3, ngram=n, ignore=ign,
                      prompt=(hist_off, _eu(eos_until)))
    torch.cuda.synchronize()
    seq, score, fin, live = seq.cpu(), score.cpu(), fin.cpu(), int(live)
    others = [c for c in range(seq.shape[1]) if c != f]
    assert torch.equal(seq[:, others], seq0[:, others]) and bool((score[:, others] == 0.125).all()), name
    assert bool((seq[done, f] == 3).all()) and bool((score[done, f] == 0).all()), name
    open_rows = torch.nonzero(~done).flatten().numpy()
    if open_rows.size:
        x = sampler_x(logits, bias, seq0, f, hist_off, n, ignore, eos_until, eos_id)
        check_rows(name, x[open_rows], mode, k, p, seed, f - hist_off, seq[open_rows, f], score[open_rows, f], rows=open_rows,
                   least=min_exact(name) if least is None else least)
    eos_now = (seq[:, f] == eos_id) & ~done
    assert torch.equal(fin.bool(), done | eos_now), name
    assert live == rows - int(done.sum()) - int(eos_now.sum()), name
    return seq, score, fin, live


S_TCAP, S_TP = 12, 6
S_CONFIGS = [(0, 4, 1), (1, 4, 2), (S_TP, 9, 3), (9, 9, 2), (9, 9, 3)]    # (hist_off, f, n): hist_off in {0, 1, Tp, f}
S_VOCABS = [1, 33, 1025, 3073, 30522, _vmax(S_TCAP)]
S_MODES = [("topk", 64, 1.0), ("topp", 64, 0.9)]


def sampler_cases(V, dtype, with_bias):
    """(name, hist_off, f, n, ignore, mode, k, p, eos_until, rows, seed, equal) of test_prompted_draws_across_vocabularies.  Top-p
    at V >= 20000 runs on equal-weight rows (sampler_inputs), where Gaussian rows leave many rows near a rounding bound."""
    rows = 64 if V < 20000 else 24
    out = []
    for i, (hist_off, f, n) in enumerate(S_CONFIGS):
        for mode, k, p in S_MODES:
            for eu in ("rows", None) if mode == "topk" else ("rows",):
                name = f"V{V}-{str(dtype)[6:]}-bias{int(with_bias)}-off{hist_off}-f{f}-n{n}-{mode}{'' if eu else '-null'}"
                out.append((name, hist_off, f, n, (3,), mode, k, p, eos_pattern(rows, f - hist_off) if eu else None, rows,
                            (1 << 32) + 977 * V + 31 * i + with_bias, mode == "topp" and V >= 20000))
    return out


@pytest.mark.parametrize("with_bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("V", S_VOCABS)
def test_prompted_draws_across_vocabularies(V, dtype, with_bias):
    eos_id = min(EOS, V - 1)
    for name, hist_off, f, n, ignore, mode, k, p, eu, rows, seed, equal in sampler_cases(V, dtype, with_bias):
        logits, bias, seq0 = sampler_inputs(V, dtype, with_bias, hist_off, f, rows, S_TCAP, seed, equal=equal)
        if hist_off == f and V >= 8:                                     # g = 0: n-grams wholly in the prompt block words
            assert O.ngram_blocked(seq0[:, :f].numpy(), n, ignore, V).any(), name
        sample_case(name, logits, bias, mode, k, p, seed, f, hist_off, seq0, eu, n=n, ignore=ignore, eos_id=eos_id)


def test_prompted_finished_rows_and_the_live_count():
    V, rows, hist_off, f = 1000, 512, 3, 5
    gen = torch.Generator().manual_seed(6)
    logits, _, seq0 = sampler_inputs(V, BF, False, hist_off, f, rows, 8, 6)
    logits[:, EOS] = torch.where(torch.rand(rows, generator=gen) < 0.5, 8.0, -8.0).to(DEV, BF)
    finished = (torch.rand(rows, generator=gen) < 0.25).int()
    eu = eos_pattern(rows, f - hist_off)
    seq, _, fin, _ = sample_case("finished-topp", logits, None, "topp", 64, 0.9, 4, f, hist_off, seq0, eu, n=2, finished=finished)
    blocked = O.eos_blocked(eu, f - hist_off, rows)
    assert not bool((seq[torch.from_numpy(blocked), f] == EOS).any())   # a blocked row never draws [EOS]
    assert int(((seq[:, f] == EOS) & ~finished.bool()).sum()) > 10


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
def test_prompted_draws_equal_the_unprompted_draws_of_the_same_word(dtype):
    """Bitwise, kernel against kernel, on the same logits: with n = 0 the prompted draw at f = Tp + g equals the unprompted draw at
    frame g with block_eos the row's rule under a constant eos_until, whatever Tp; and hist_off = 0 is vlpk_sample_tokens at the same
    f, n-grams included."""
    V, rows, T_cap = 3073, 64, 12
    seed = (1 << 40) + 9

    def run(logits, f, seq0, prompt=None, block_eos=False, n=0):
        seq = seq0.to(DEV)
        score = torch.full(seq.shape, 0.125, device=DEV)
        fin = torch.zeros(rows, dtype=torch.int32, device=DEV)
        live = torch.full((1,), rows, dtype=torch.int32, device=DEV)
        ops.sample_tokens(logits, None, "topp", 64, 0.95, seed, f, seq, score, fin, live, EOS, block_eos=block_eos, ngram=n,
                          prompt=prompt)
        return seq[:, f].cpu(), _bits(score[:, f]), fin.cpu(), int(live)

    for g in (0, 2):
        logits, _, seq0 = sampler_inputs(V, dtype, False, S_TP, S_TP + g, rows, T_cap, 40 + g)
        logits[:, EOS] = 6.0                                             # [EOS] likely: its block shows
        for c in (-1, g, g + 1, 100):
            want = run(logits, g, seq0[:, S_TP:].contiguous(), block_eos=g + 1 <= c)
            for Tp in (S_TP, 2):
                sq = seq0[:, S_TP - Tp:].contiguous()
                got = run(logits, Tp + g, sq, prompt=(Tp, _eu(np.full(rows, c))))
                for a, b in zip(got, want):
                    assert (a == b) if isinstance(a, int) else torch.equal(a, b), (g, c, Tp)
    logits, _, seq0 = sampler_inputs(V, dtype, False, 0, 5, rows, T_cap, 47)
    for c, block in ((None, False), (np.full(rows, 6), True), (np.full(rows, 5), False)):
        got = run(logits, 5, seq0, prompt=(0, _eu(c)), n=2)
        want = run(logits, 5, seq0, block_eos=block, n=2)
        for a, b in zip(got, want):
            assert (a == b) if isinstance(a, int) else torch.equal(a, b), c


# ---------------------------------------------------------------------------------------------------------------------------------
# diverse and constrained rows
# ---------------------------------------------------------------------------------------------------------------------------------
def _per_row(x, K, tw, tl, blocked, beos, comp=None, eos_id=EOS):
    """Each row's top K against the oracle's row restated on the kernel's own logsumexp, with the row's own [EOS] block beos[i];
    returns the oracle's (words, lp, lp rows).  comp: per row, the kernel's completing (words, values), left out of the ranking."""
    ow, ol, lps = [], [], []
    for i in range(x.shape[0]):
        cw, cv = comp[i] if comp else (np.zeros(0, np.int64), np.zeros(0, np.float32))
        words = np.concatenate([tw[i], cw]).astype(np.int64)
        values = np.concatenate([tl[i], cv]).astype(np.float32)
        L_, lse, tol, lp, w, v = O.row_stage(x[i], K, words, values, None if blocked is None else blocked[i], bool(beos[i]), eos_id,
                                             tuple(cw))
        if not O.nonfinite(x[i]):
            assert abs(float(L_) - lse) <= tol, (i, float(L_), lse, tol)
        assert np.array_equal(w, tw[i]), (i, w, tw[i])
        assert np.array_equal(v.view(np.uint32), tl[i].view(np.uint32)), (i, v, tl[i])
        ow.append(w)
        ol.append(v)
        lps.append(lp)
    return np.stack(ow), np.stack(ol), lps


def run_diverse_p(logits, bias, f, B, K, G, lam, prev, n, ignore, hist_in, T_cap, hist_off, eos_until):
    T = T_cap - hist_off
    wi, pt, sc, eo = _traces(T, B, K, f, prev)
    tw = torch.full((B * K, K), -7, dtype=torch.int32, device=DEV)
    tl = torch.full((B * K, K), 0.125, device=DEV)
    hist_out = torch.full((B * K, T_cap), -7, dtype=torch.int32, device=DEV)
    ign = torch.tensor(ignore, dtype=torch.int32, device=DEV) if ignore else None
    ops.diverse_beam_step(logits, bias, f, G, lam, wi, pt, sc, eo, tw, tl, EOS, ngram=n, ignore=ign,
                          hist_in=None if hist_in is None else hist_in.to(DEV), hist_out=hist_out, prompt=(hist_off, _eu(eos_until)))
    torch.cuda.synchronize()
    rows = B if f == 0 else B * K
    assert (wi[f + 1:] == -7).all() and (sc[f + 1:] == 0.125).all()
    return [t[f].cpu() for t in (wi, pt, sc, eo)] + [tw[:rows].cpu(), tl[:rows].cpu(), hist_out.cpu()]


def verify_diverse(out, logits, bias, f, B, K, G, lam, prev, n, ignore, hist_in, hist_off, eos_until, sentinel=True, eos_id=EOS):
    """One prompted diverse frame's outputs against the oracle, bit for bit.  sentinel: hist_out started as -7 (a replayed decode's
    buffers hold earlier frames past hist_off + f)."""
    wid, ptr, score, eos, tw, tl, hist_out = out
    V = logits.shape[-1]
    rows = B if f == 0 else B * K
    hf = hist_off + f
    blocked = None
    if n:
        hists = O.prompt_carry(hist_in.cpu().numpy(), None if f == 0 else prev[1].numpy(), None if f == 0 else prev[0].numpy(), K, f,
                               hist_off)
        if f:
            assert np.array_equal(hist_out[:, :hf].numpy(), hists)
        if sentinel:
            assert (hist_out[:, 0 if f == 0 else hf:] == -7).all()      # frame 0 writes no history
        if hf >= n:
            blocked = O.ngram_blocked(hists, n, ignore, V)
    elif sentinel:
        assert (hist_out == -7).all()
    x = _beam_x(logits.reshape(rows, V), bias)
    ow, ol, _ = _per_row(x, K, tw.numpy(), tl.numpy(), blocked, O.eos_blocked(eos_until, f, rows), eos_id=eos_id)
    ps, pe = (prev[2].numpy(), prev[3].numpy()) if f else (None, None)
    mw, mp, ms, _ = DO.merge(ow, ol, ps, pe, K, G, lam, f == 0)
    assert torch.equal(wid, torch.from_numpy(mw)) and torch.equal(ptr, torch.from_numpy(mp)), (wid, mw, ptr, mp)
    assert torch.equal(_bits(score), _bits(O.canonical(ms))), (score, ms)
    assert torch.equal(eos, (wid == eos_id).float())
    return out


def check_diverse_p(logits, bias, f, B, K, G, lam, prev=None, n=0, ignore=(), hist_in=None, T_cap=8, hist_off=0, eos_until=None):
    out = run_diverse_p(logits, bias, f, B, K, G, lam, prev, n, ignore, hist_in, T_cap, hist_off, eos_until)
    return verify_diverse(out, logits, bias, f, B, K, G, lam, prev, n, ignore, hist_in, hist_off, eos_until)


def run_constrained_p(logits, bias, f, cons, K, prev, n, ignore, hist_in, T_cap, hist_off, eos_until):
    B, C, A, _ = cons.shape
    SK, W = K << C, K + C * A
    wi, pt, sc, eo = _traces(T_cap - hist_off, B, SK, f, prev)
    tw = torch.full((B * SK, W), -7, dtype=torch.int32, device=DEV)
    tl = torch.full((B * SK, W), 0.125, device=DEV)
    td = torch.full((B * SK, C * A), -7, dtype=torch.int32, device=DEV)
    hist_out = torch.full((B * SK, T_cap), -7, dtype=torch.int32, device=DEV)
    ign = torch.tensor(ignore, dtype=torch.int32, device=DEV) if ignore else None
    ops.constrained_beam_step(logits, bias, f, cons.to(DEV), wi, pt, sc, eo, tw, tl, td, EOS, ngram=n, ignore=ign, hist_in=hist_in.to(DEV),
                              hist_out=hist_out, prompt=(hist_off, _eu(eos_until)))
    torch.cuda.synchronize()
    rows = B if f == 0 else B * SK
    assert (wi[f + 1:] == -7).all() and (sc[f + 1:] == 0.125).all()
    return [t[f].cpu() for t in (wi, pt, sc, eo)] + [tw[:rows].cpu(), tl[:rows].cpu(), td[:rows].cpu(), hist_out.cpu()]


def verify_constrained(out, logits, bias, f, cons, K, prev, n, ignore, hist_in, hist_off, eos_until, sentinel=True, eos_id=EOS):
    wid, ptr, score, eos, tw, tl, td, hist_out = out
    B, C, A, _ = cons.shape
    V = logits.shape[-1]
    SK = K << C
    rows = B if f == 0 else B * SK
    hf = hist_off + f
    cn = cons.cpu().numpy()
    hists = O.prompt_carry(hist_in.cpu().numpy(), None if f == 0 else prev[1].numpy(), None if f == 0 else prev[0].numpy(), SK, f,
                           hist_off)
    if f:
        assert np.array_equal(hist_out[:, :hf].numpy(), hists)
    if sentinel:
        assert (hist_out[:, 0 if f == 0 else hf:] == -7).all()
    blocked = O.ngram_blocked(hists, n, ignore, V) if n and hf >= n else None
    tw, tl, td = tw.numpy(), tl.numpy(), td.numpy()
    comp = []
    for i, (b, _, s) in enumerate(CO._rows(B, K, C, f == 0, cn)):
        want = CO.completions([int(w) for w in hists[i]], cn[b], s)     # a phrase may begin in the prompt
        m = len(want)
        assert tw[i, K:K + m].tolist() == list(want) and td[i, :m].tolist() == list(want.values()), (i, want, tw[i, K:], td[i])
        assert (tw[i, K + m:] == -1).all() and (td[i, m:] == -1).all() and np.isneginf(tl[i, K + m:]).all()
        comp.append((tw[i, K:K + m].astype(np.int64), tl[i, K:K + m]))
    x = _beam_x(logits.reshape(rows, V), bias)
    ow, ol, lps = _per_row(x, K, tw[:, :K], tl[:, :K], blocked, O.eos_blocked(eos_until, f, rows), comp, eos_id)
    for i, (cw, cv) in enumerate(comp):
        assert np.array_equal(lps[i][cw].view(np.uint32), cv.view(np.uint32)), i
    lists = [(ow[i], ol[i], {int(w): (lps[i][w], int(d)) for w, d in zip(cw, td[i])}) for i, (cw, _) in enumerate(comp)]
    ps, pe = (prev[2].numpy(), prev[3].numpy()) if f else (None, None)
    mw, mp, ms, _ = CO.merge(lists, ps, pe, cn, K, f == 0)
    assert torch.equal(wid, torch.from_numpy(mw)) and torch.equal(ptr, torch.from_numpy(mp)), (wid, mw, ptr, mp)
    assert torch.equal(_bits(score), _bits(ms.astype(np.float32))), (score, ms)
    assert torch.equal(eos, ((wid == eos_id) & torch.isfinite(score)).float())
    return out


def check_constrained_p(logits, bias, f, cons, K, prev=None, n=0, ignore=(), hist_in=None, T_cap=8, hist_off=0, eos_until=None):
    out = run_constrained_p(logits, bias, f, cons, K, prev, n, ignore, hist_in, T_cap, hist_off, eos_until)
    return verify_constrained(out, logits, bias, f, cons, K, prev, n, ignore, hist_in, hist_off, eos_until)


def _parents(gen, rows, T_cap, hist_off, f, alphabet=12):
    """Frame f's parents [rows, T_cap]: a prompt history in the first hist_off columns, distinct per row (so that following the
    wrong pointer shows), then f - 1 generated words."""
    h = torch.randint(0, alphabet, (rows, T_cap), generator=gen, dtype=torch.int32)
    h[:, :hist_off] = prompt_rows(gen, rows, hist_off, alphabet)
    return h


def repeat_prompts(B, Tp, n, V):
    """int32 [B, Tp] prompt histories whose tails repeat: row r < B - 1 ends in s ‖ w ‖ s (s of n - 1 words, 2n - 1 <= Tp), so the
    duplicate-n-gram rule blocks w from the prompt alone; the last row is empty.  Returns (histories, {row: w})."""
    pool = [w for w in range(min(V, 12)) if w not in (3, EOS)]          # 3: the tests' ignore set
    h = torch.full((B, Tp), -1, dtype=torch.int32)
    blocks = {}
    for r in range(B - 1):
        words = [pool[(r + j) % len(pool)] for j in range(n)]
        tail = words[:n - 1] + [words[-1]] + words[:n - 1]
        h[r, Tp - len(tail):] = torch.tensor(tail, dtype=torch.int32)
        blocks[r] = words[-1]
    return h, blocks


def dominate(logits, blocks):
    """Each row's prompt-blocked word made its unblocked argmax, so that the block moves the row's top K."""
    for r, w in blocks.items():
        logits[r, w] = 30.0
    return logits


def assert_prompt_blocks(hist, n, ignore, V, blocks, logits=None, bias=None):
    """The oracle blocks each row's word w from the prompt alone, and w is that row's unblocked argmax."""
    blocked = O.ngram_blocked(hist.numpy(), n, ignore, V)
    x = None if logits is None else _beam_x(logits, bias)
    for r, w in blocks.items():
        assert blocked[r, w], (r, w, hist[r])
        assert x is None or int(np.argmax(x[r])) == w, (r, w)


def _with_phrase_in_prompt(cons, hist, B, C):
    """Constraint C - 1 of every image also takes the phrase [last prompt word, 2]: it begins in the prompt."""
    cons = cons.clone()
    for b in range(B):
        w = int(hist[b, -1]) if hist.shape[1] else -1
        if w >= 1:
            cons[b, C - 1, 0, :] = 0
            cons[b, C - 1, 0, :2] = torch.tensor([w, 2])
    return cons


P_TCAP, P_TP = 10, 5
P_VMAX = _vmax(P_TCAP)
DIVERSE_P = [(4, 4, 2), (33, 6, 3), (1025, 6, 2), (30522, 48, 4), (P_VMAX, 6, 3)]


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("V,K,G", DIVERSE_P, ids=[f"V{v}-K{k}-G{g}" for v, k, g in DIVERSE_P])
def test_prompted_diverse_rows(V, K, G, dtype):
    """f = 0 on [B, T_cap] prompt histories (n-gram blocks from the prompt alone), f = 1 following non-zero pointers, f = 3; ragged
    eos_until at the boundary; V = K included."""
    gen = torch.Generator().manual_seed(V + K)
    B = 5
    bias = _bias(gen, V, dtype)
    for n in (2, 3):                                                     # frame 0: n-gram blocks from the prompt alone
        h0 = torch.full((B, P_TCAP), -7, dtype=torch.int32)
        h0[:, :P_TP], blocks = repeat_prompts(B, P_TP, n, V)
        logits = dominate(_logits(gen, B, V, K, dtype, ld=V + 37), blocks)
        assert_prompt_blocks(h0[:, :P_TP], n, (3,), V, blocks, logits, bias)
        check_diverse_p(logits, bias, 0, B, K, G, 0.5, n=n, ignore=(3,), hist_in=h0, T_cap=P_TCAP, hist_off=P_TP,
                        eos_until=eos_pattern(B, 0))
    for f in (1, 3):
        prev = _prev(gen, B, K, V)
        prev[1].copy_((torch.arange(K) + 1 + f) % K)                      # every pointer away from the row's own slot
        check_diverse_p(_logits(gen, B * K, V, K, dtype, ld=V + 37), bias, f, B, K, G, 0.75, prev, n=1 + f % 3, ignore=(3,),
                        hist_in=_parents(gen, B * K, P_TCAP, P_TP, f), T_cap=P_TCAP, hist_off=P_TP, eos_until=eos_pattern(B * K, f))


CONSTRAINED_P = [(2, 2, 2, 3, "min"), (4, 1, 4, 2, "min"), (3, 2, 2, 3, 1025), (2, 2, 2, 2, 30522), (4, 2, 2, 3, "max")]


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("K,C,A,P,Vx", CONSTRAINED_P, ids=[f"K{k}-C{c}-A{a}-P{p}-V{v}" for k, c, a, p, v in CONSTRAINED_P])
def test_prompted_constrained_rows(K, C, A, P, Vx, dtype):
    """As the diverse rows, with completions whose phrase begins in the prompt (the -1-padded history read at every frame, n = 0
    too); V = K + C*A included."""
    V = {"min": K + C * A, "max": P_VMAX}.get(Vx, Vx)
    gen = torch.Generator().manual_seed(V * 13 + K)
    B = 4
    alphabet = min(12, V)
    bias = _bias(gen, V, dtype)
    table = _table(gen, B, C, A, P, alphabet=min(12, V - 1))            # ids < V, [EOS] moved up
    for n in (0, 2, 3):                                                  # frame 0: n-gram blocks from the prompt alone (n > 0)
        h0 = torch.full((B, P_TCAP), -7, dtype=torch.int32)
        h0[:, :P_TP], blocks = repeat_prompts(B, P_TP, max(n, 2), V)
        cons = _with_phrase_in_prompt(table, h0[:, :P_TP], B, C)
        logits = dominate(_logits(gen, B, V, K, dtype, alphabet=alphabet), blocks)
        if n:
            assert_prompt_blocks(h0[:, :P_TP], n, (3,), V, blocks, logits, bias)
        out = check_constrained_p(logits, bias, 0, cons, K, n=n, ignore=(3,), hist_in=h0, T_cap=P_TCAP, hist_off=P_TP,
                                  eos_until=eos_pattern(B, 0))
        ends = [b for b in range(B) if int(h0[b, P_TP - 1]) >= 1]
        assert ends and all(2 in out[4][b, K:].tolist() for b in ends)     # [last prompt word, 2] completes across the prompt's end
    SK = K << C
    for f in (1, 3):
        prev = _prev(gen, B, SK, V)
        prev[1].copy_((torch.arange(SK) + 1 + f) % SK)
        check_constrained_p(_logits(gen, B * SK, V, K, dtype, alphabet=alphabet), bias, f, cons, K, prev, n=f % 3, ignore=(3,),
                            hist_in=_parents(gen, B * SK, P_TCAP, P_TP, f, alphabet), T_cap=P_TCAP, hist_off=P_TP,
                            eos_until=eos_pattern(B * SK, f))


def _force_block_eos(monkeypatch):
    """Hand vlpk_constrained_beam_step_prompt args.block_eos = 1, which the ops wrapper refuses to pass beside a prompt."""
    call = L.call

    def forced(name, *args):
        if name == "vlpk_constrained_beam_step_prompt":
            args[0]._obj.block_eos = 1
        return call(name, *args)
    monkeypatch.setattr(L, "call", forced)


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
def test_null_eos_until_never_blocks(dtype, monkeypatch):
    """eos_until NULL: [EOS] is never blocked, in every prompted selector, even with the constrained args' block_eos set.  [EOS] is
    the argmax of every row, so a block would move it out of the top K."""
    V, K, G = 40, 4, 2
    gen = torch.Generator().manual_seed(2)
    B = 3

    def rows(n):
        x = torch.randn(n, V, generator=gen)
        x[:, EOS] = 5.0
        return x.to(DEV, dtype)

    h0 = torch.full((B, P_TCAP), -7, dtype=torch.int32)
    h0[:, :P_TP] = prompt_rows(gen, B, P_TP)
    out = check_diverse_p(rows(B), None, 0, B, K, G, 0.5, n=2, hist_in=h0, T_cap=P_TCAP, hist_off=P_TP)
    assert (out[4][:, 0] == EOS).all()
    _force_block_eos(monkeypatch)
    cons = _table(gen, B, 2, 1, 2)
    out = check_constrained_p(rows(B), None, 0, cons, K, hist_in=h0, T_cap=P_TCAP, hist_off=P_TP)
    assert (out[4][:, 0] == EOS).all()
    SK = K << 2
    prev = _prev(gen, B, SK, V)
    out = check_constrained_p(rows(B * SK), None, 2, cons, K, prev, hist_in=_parents(gen, B * SK, P_TCAP, P_TP, 2), T_cap=P_TCAP,
                              hist_off=P_TP)
    assert (out[4][:, 0] == EOS).all()
    logits, _, seq0 = sampler_inputs(V, dtype, False, 2, 3, 16, 8, 5)
    logits[:, EOS] = 30.0
    seq, _, _, _ = sample_case("null-eos", logits, None, "topk", 1, 1.0, 5, 3, 2, seq0, None)
    assert (seq[:, 3] == EOS).all()


@pytest.mark.parametrize("f", [1, 3])
def test_prompted_rows_equal_the_unprompted_frame(f):
    """Bitwise, kernel against kernel: prompted frame f with hist_off = Tp and a uniform eos_until c equals unprompted frame f + Tp
    with block_eos = (f + 1 <= c), every output and the whole hist_out included; hist_off = 0 equals the unprompted frame f, and
    at f = 0."""
    V, K, G, B, T_cap, Tp = 1025, 6, 3, 3, 12, 4
    gen = torch.Generator().manual_seed(f)
    bias = _bias(gen, V, BF)
    cons = _table(gen, B, 2, 2, 3)
    SK = K << 2
    for c in (f, f + 1):
        for hist_off in (Tp, 0):
            prev = _prev(gen, B, K, V)
            logits = _logits(gen, B * K, V, K, BF)
            logits[:, EOS] = 9.0
            hin = _parents(gen, B * K, T_cap, Tp, f).to(DEV)
            a = run_diverse_p(logits, bias, f, B, K, G, 0.5, prev, 2, (3,), hin, T_cap, hist_off, np.full(B * K, c))
            b = run_diverse(logits, bias, f + hist_off, B, K, G, 0.5, prev, n=2, ignore=(3,), block_eos=f + 1 <= c, hist_in=hin,
                            T_cap=T_cap)
            assert all(_same(x, y) for x, y in zip(a, b)), (c, hist_off)
            cprev = _prev(gen, B, SK, V)
            clog = _logits(gen, B * SK, V, K, BF)
            chin = _parents(gen, B * SK, T_cap, Tp, f).to(DEV)
            a = run_constrained_p(clog, bias, f, cons, K, cprev, 2, (3,), chin, T_cap, hist_off, np.full(B * SK, c))
            b = run_constrained(clog, bias, f + hist_off, cons, K, cprev, n=2, ignore=(3,), block_eos=f + 1 <= c, hist_in=chin,
                                T_cap=T_cap)
            assert all(_same(x, y) for x, y in zip(a, b)), (c, hist_off)
    h0 = torch.full((B, T_cap), -7, dtype=torch.int32, device=DEV)
    logits = _logits(gen, B, V, K, BF)
    a = run_diverse_p(logits, bias, 0, B, K, G, 0.5, None, 2, (), h0, T_cap, 0, None)
    b = run_diverse(logits, bias, 0, B, K, G, 0.5, n=2, T_cap=T_cap)
    assert all(_same(x, y) for x, y in zip(a, b))
    a = run_constrained_p(logits, bias, 0, cons, K, None, 2, (), h0, T_cap, 0, None)
    b = run_constrained(logits, bias, 0, cons, K, n=2, T_cap=T_cap)
    assert all(_same(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("n", [1, 2, 3])
def test_long_prompted_histories_bad_pointers_and_ids_outside_int32(n):
    """hist_off + f = 1080 > 1024: the carry strides past the CTA; back pointers -1, width and 2^40 give -1 words, ids outside int32
    give -1."""
    T_cap, hist_off, f, V, K, G = 1100, 1000, 80, 3073, 4, 2
    gen = torch.Generator().manual_seed(n)
    B = 3
    bad_ptr = [-1, K, 1 << 40]
    bad_wid = [1 << 33, -(1 << 33), 1 << 31, -(1 << 31) - 1, V + 5, -3]
    prev = _prev(gen, B, K, V)
    for j, p in enumerate(bad_ptr):
        prev[1][j % B, (j + 1) % K] = p
    for j, w in enumerate(bad_wid):
        prev[0][(j + 1) % B, j % K] = w
    hin = _parents(gen, B * K, T_cap, hist_off, f, 6)
    check_diverse_p(_logits(gen, B * K, V, K, BF, alphabet=6), None, f, B, K, G, 0.5, prev, n=n, ignore=(0,), hist_in=hin, T_cap=T_cap,
                    hist_off=hist_off, eos_until=eos_pattern(B * K, f))
    C, A, P = 2, 2, 3
    SK = K << C
    cons = _table(gen, B, C, A, P, alphabet=6)
    cprev = _prev(gen, B, SK, V)
    for j, p in enumerate(bad_ptr):
        cprev[1][j % B, (3 * j + 1) % SK] = p if p != K else SK
    for j, w in enumerate(bad_wid):
        cprev[0][(j + 1) % B, (5 * j) % SK] = w
    check_constrained_p(_logits(gen, B * SK, V, K, torch.float32, alphabet=6), None, f, cons, K, cprev, n=n, ignore=(0,),
                        hist_in=_parents(gen, B * SK, T_cap, hist_off, f, 6), T_cap=T_cap, hist_off=hist_off,
                        eos_until=eos_pattern(B * SK, f))


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
def test_prompted_nan_rows(dtype):
    V, K, G, B = 1000, 6, 3, 4
    gen = torch.Generator().manual_seed(17)
    h0 = torch.full((B, P_TCAP), -7, dtype=torch.int32)
    h0[:, :P_TP], blocks = repeat_prompts(B, P_TP, 2, V)              # row 0 (a finite row) has a block from the prompt alone
    l0 = dominate(_nonfinite_rows(gen, B, V, K, dtype), {0: blocks[0]})
    assert_prompt_blocks(h0[:1, :P_TP], 2, (), V, {0: blocks[0]}, l0[:1])
    check_diverse_p(l0, None, 0, B, K, G, 0.5, n=2, hist_in=h0, T_cap=P_TCAP, hist_off=P_TP, eos_until=eos_pattern(B, 0))
    prev = _prev(gen, B, K, V)
    check_diverse_p(_nonfinite_rows(gen, B * K, V, K, dtype), None, 2, B, K, G, 0.5, prev, n=2,
                    hist_in=_parents(gen, B * K, P_TCAP, P_TP, 2),
                    T_cap=P_TCAP, hist_off=P_TP, eos_until=eos_pattern(B * K, 2))
    Kc, C = 4, 2
    SK = Kc << C
    cons = _table(gen, B, C, 2, 2)
    check_constrained_p(dominate(_nonfinite_rows(gen, B, V, Kc, dtype), {0: blocks[0]}), None, 0, cons, Kc, n=2, hist_in=h0,
                        T_cap=P_TCAP, hist_off=P_TP, eos_until=eos_pattern(B, 0))
    cprev = _prev(gen, B, SK, V)
    check_constrained_p(_nonfinite_rows(gen, B * SK, V, Kc, dtype), None, 2, cons, Kc, cprev,
                        hist_in=_parents(gen, B * SK, P_TCAP, P_TP, 2),
                        T_cap=P_TCAP, hist_off=P_TP, eos_until=eos_pattern(B * SK, 2))


# ---------------------------------------------------------------------------------------------------------------------------------
# plain prompted beam search: frame 0's n-gram block
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3])
def test_frame_zero_ngram_block_on_right_aligned_prompts(n):
    """beam_search's frame-0 vlpk_beam_ngram_block call: rows = B, K = 1, f = Tp, each row its own parent and its last prompt entry
    the word, on histories with -1 runs before real words; a row with an empty prompt is left untouched."""
    prompt = torch.tensor([[0, 0, 0, 0, 0], [4, 4, 0, 0, 0], [3, 7, 3, 7, 3], [5, 6, 5, 0, 0], [9, 0, 0, 0, 0]], device=DEV)
    B, Tp = prompt.shape
    V = 40
    seed = decode.prompt_history(prompt, 1, Tp + 4)
    gen = torch.Generator().manual_seed(n)
    logp = torch.randn(B, 1, V, generator=gen).to(DEV)
    ignore = (6,)
    lp = logp.clone()
    out = torch.full_like(seed, -7)
    ops.beam_ngram_block(seed, out, torch.zeros(B, 1, dtype=torch.int64, device=DEV), seed[:, Tp - 1:Tp].to(torch.int64), Tp, n,
                         torch.tensor(ignore, dtype=torch.int32, device=DEV), lp)
    torch.cuda.synchronize()
    blocked = O.ngram_blocked(seed[:, :Tp].cpu().numpy(), n, ignore, V)
    base = logp.cpu().numpy().reshape(B, V)
    want = np.where(blocked, (base + SO.BLOCK).astype(np.float32), base)
    assert np.array_equal(lp.cpu().numpy().reshape(B, V).view(np.uint32), want.view(np.uint32))
    assert torch.equal(lp[0], logp[0])                                   # the empty prompt: nothing blocked
    assert torch.equal(out[:, :Tp], seed[:, :Tp]) and bool((out[:, Tp:] == -7).all())
    assert blocked[1:].any()


# ---------------------------------------------------------------------------------------------------------------------------------
# whole prompted decodes, replayed frame by frame
# ---------------------------------------------------------------------------------------------------------------------------------
class _Recorder:
    """Wraps one ops selector: snapshots each call's inputs before it and its outputs after it."""

    def __init__(self, kind):
        self.kind, self.calls = kind, []
        self.inner = {"sample": ops.sample_tokens, "diverse": ops.diverse_beam_step, "constrained": ops.constrained_beam_step}[kind]

    def __call__(self, *a, **kw):
        return getattr(self, "_" + self.kind)(*a, **kw)

    def _sample(self, logits, bias, mode, topk, topp, seed, f, seq, score, finished, live, eos_id, pad_id=0, block_eos=False, ngram=0,
                ignore=None, prompt=None):
        V = logits.shape[-1]
        rec = dict(logits=logits.reshape(-1, V).clone(), bias=bias.clone(), mode=mode, k=topk, p=topp, seed=seed, f=f,
                   hist=seq[:, :f].cpu(), finished=finished.cpu(), eos=eos_id, pad=pad_id, block_eos=block_eos, ngram=ngram,
                   ignore=() if ignore is None else tuple(ignore.tolist()), hist_off=prompt[0],
                   eos_until=None if prompt[1] is None else prompt[1].cpu())
        self.inner(logits, bias, mode, topk, topp, seed, f, seq, score, finished, live, eos_id, pad_id, block_eos, ngram, ignore, prompt)
        rec.update(ids=seq[:, f].cpu(), scores=score[:, f].cpu(), finished_after=finished.cpu())
        self.calls.append(rec)

    def _beam(self, f, traces, logits, bias, ngram, ignore, hist_in, hist_out, prompt, block_eos, eos_id):
        V = logits.shape[-1]
        return dict(f=f, logits=logits.reshape(-1, V).clone(), bias=bias.clone(), ngram=ngram, block_eos=block_eos, eos=eos_id,
                    ignore=() if ignore is None else tuple(ignore.tolist()), hist_in=None if hist_in is None else hist_in.cpu(),
                    prev=None if f == 0 else [t[f - 1].cpu() for t in traces], hist_off=prompt[0],
                    eos_until=None if prompt[1] is None else prompt[1].cpu())

    def _diverse(self, logits, bias, f, G, penalty, wid, ptr, score, eos, top_w, top_lp, eos_id, block_eos=False, ngram=0, ignore=None,
                 hist_in=None, hist_out=None, prompt=None):
        rec = self._beam(f, (wid, ptr, score, eos), logits, bias, ngram, ignore, hist_in, hist_out, prompt, block_eos, eos_id)
        rec.update(G=G, lam=penalty)
        self.inner(logits, bias, f, G, penalty, wid, ptr, score, eos, top_w, top_lp, eos_id, block_eos, ngram, ignore, hist_in, hist_out,
                   prompt)
        rows = rec["logits"].shape[0]
        rec["out"] = [t[f].cpu() for t in (wid, ptr, score, eos)] + [top_w[:rows].cpu(), top_lp[:rows].cpu(),
                                                                     None if hist_out is None else hist_out.cpu()]
        self.calls.append(rec)

    def _constrained(self, logits, bias, f, cons, wid, ptr, score, eos, top_w, top_lp, top_dest, eos_id, block_eos=False, ngram=0,
                     ignore=None, hist_in=None, hist_out=None, prompt=None):
        rec = self._beam(f, (wid, ptr, score, eos), logits, bias, ngram, ignore, hist_in, hist_out, prompt, block_eos, eos_id)
        rec["cons"] = cons.cpu()
        self.inner(logits, bias, f, cons, wid, ptr, score, eos, top_w, top_lp, top_dest, eos_id, block_eos, ngram, ignore, hist_in,
                   hist_out, prompt)
        rows = rec["logits"].shape[0]
        rec["out"] = [t[f].cpu() for t in (wid, ptr, score, eos)] + [top_w[:rows].cpu(), top_lp[:rows].cpu(), top_dest[:rows].cpu(),
                                                                     hist_out.cpu()]
        self.calls.append(rec)


DECODE_LENS = (0, 2, 5, 3)
DECODE_WORDS = ((), (11, 9), (12, 9, 13, 12, 9), (9, 11, 9))          # repeated tails: frame 0 blocks 13 and 11 from the prompts
PROMPTED_DECODES = {
    "topk": dict(K=1, sampling_method="topk", topk=16, forbid_duplicate_ngrams=True, ngram_size=2, min_len=6),
    "topp-n2": dict(K=1, sampling_method="topp", topp=0.9, num_return_sequences=2, forbid_duplicate_ngrams=True, ngram_size=2,
                    min_len=6),
    "diverse": dict(K=4, num_beam_groups=2, diversity_penalty=0.7, forbid_duplicate_ngrams=True, ngram_size=2, min_len=6),
    "constrained": dict(K=2, constraints=[[20], [[9, 8]]], forbid_duplicate_ngrams=True, ngram_size=2, min_len=6),
}


@pytest.mark.parametrize("mode", list(PROMPTED_DECODES))
def test_prompted_decodes_replay_through_the_oracle(mode, monkeypatch):
    """Every selector call of a ragged prompted decode: hist_off = Tp, the frame index, eos_until = min_len - t_b ([B] at frame 0,
    each image's rows after), frame 0's hist_in = decode.prompt_history(prompt, 1, .), frame 1's parents holding the prompts; and
    each frame against the oracle (beam frames bitwise, the sampler's draws by DECODE_MIN_EXACT)."""
    from tools import prompt_decode_oracle as PO
    from vlp_b200 import synth

    from test_prompt_decode_gpu import _cuda, _decoder
    kw = dict(PROMPTED_DECODES[mode])
    dims = synth.SMALL_L123
    B = len(DECODE_LENS)
    prompt = torch.zeros(B, max(DECODE_LENS), dtype=torch.int64)
    for b, w in enumerate(DECODE_WORDS):
        prompt[b, :len(w)] = torch.tensor(w, dtype=torch.int64)
    prompt = prompt.cuda()
    Tp = prompt.shape[1]
    kind = "sample" if "sampling_method" in kw else "constrained" if "constraints" in kw else "diverse"
    rec = _Recorder(kind)
    monkeypatch.setattr(ops, {"sample": "sample_tokens", "diverse": "diverse_beam_step", "constrained": "constrained_beam_step"}[kind],
                        rec)
    model = _decoder(dims, seed=(1 << 32) + 19, **kw) if kind == "sample" else _decoder(dims, **kw)
    model(*_cuda(PO.decode_inputs(dims, B, 5)), task_idx=None, prompt_ids=prompt)
    assert rec.calls
    min_len = model.min_len
    if kind == "sample":
        N = model.num_return_sequences
        R = B * N
        until = decode.prompt_eos_until(prompt, N, min_len).cpu()
        head = decode.prompt_history(prompt, N, Tp).cpu().long()
        exact = total = 0
        for i, c in enumerate(rec.calls):
            assert c["hist_off"] == Tp and c["f"] == Tp + i and not c["block_eos"] and torch.equal(c["eos_until"], until)
            assert torch.equal(c["hist"][:, :Tp], head)
            done = c["finished"].bool()
            assert bool((c["ids"][done] == c["pad"]).all())
            rows = torch.nonzero(~done).flatten().numpy()
            if rows.size:
                x = sampler_x(c["logits"], c["bias"], c["hist"], c["f"], Tp, c["ngram"], c["ignore"], until.numpy(), c["eos"])
                exact += check_rows(f"decode-{mode}-g{i}", x[rows], c["mode"], c["k"], c["p"], c["seed"], i, c["ids"][rows],
                                    c["scores"][rows], rows=rows, least=0.0)
                total += rows.size
            assert torch.equal(c["finished_after"].bool(), done | (c["ids"] == c["eos"]))
            assert c["logits"].shape[0] == R
        print(f"exact decode-{mode} {exact}/{total} over {len(rec.calls)} frames")
        assert exact >= DECODE_MIN_EXACT * total, (mode, exact, total)
        return
    K = model.search_beam_size
    W = K if kind == "diverse" else K << len(kw["constraints"])
    seed0 = decode.prompt_history(prompt, 1, rec.calls[0]["hist_in"].shape[1]).cpu()
    for i, c in enumerate(rec.calls):
        f = c["f"]
        assert f == i and c["hist_off"] == Tp and not c["block_eos"]
        assert torch.equal(c["eos_until"], decode.prompt_eos_until(prompt, 1 if f == 0 else W, min_len).cpu())
        if f == 0:
            assert torch.equal(c["hist_in"], seed0)
            assert O.ngram_blocked(seed0[:, :Tp].numpy(), c["ngram"], c["ignore"], c["logits"].shape[1]).any()    # blocks from the prompts
        elif f == 1:
            assert torch.equal(c["hist_in"][:, :Tp], decode.prompt_history(prompt, W, Tp).cpu())
        eu = c["eos_until"].numpy()
        if kind == "diverse":
            verify_diverse(c["out"], c["logits"], c["bias"], f, B, K, c["G"], c["lam"], c["prev"], c["ngram"], c["ignore"], c["hist_in"],
                           Tp, eu, sentinel=False, eos_id=c["eos"])
        else:
            verify_constrained(c["out"], c["logits"], c["bias"], f, c["cons"], K, c["prev"], c["ngram"], c["ignore"], c["hist_in"], Tp, eu,
                               sentinel=False, eos_id=c["eos"])
    if kind == "constrained":                                            # the phrase [9, 8] begins in three of the prompts
        assert any((c["out"][6] >= 0).any() for c in rec.calls[:1])
