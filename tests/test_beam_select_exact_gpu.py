"""GPU: bit-exact parity for the diverse and constrained beam selectors (vlpk_diverse_beam_step, vlpk_constrained_beam_step) against
the exact host statement of their row stage (tools/beam_select_oracle.py) on each row's own fp32 logsumexp, and the fp32-exact merges
of tools/diverse_beam_oracle.py and tools/constrained_beam_oracle.py.

Every row and every frame is checked bit for bit, with no filter: each row's top K (words and fp32 values), the constrained rows'
completing words, values and destinations, the carried histories, and the frame's wid / ptr / score / eos, which must equal the
merge over the oracle's own rows.  Each row's recovered logsumexp lies within the stated bound of the fp64 one.  Cases: vocabularies
at the row chunks' edges, V = K and the shared-memory limit (one past it is refused before a launch); Gaussian, quantised, tied,
all-equal, dominant and -inf rows; a blocked word tying [EOS]'s -10000; strided logits with NaN past V and around the bias; bf16 and
fp32; K up to 64 and every group count; constraints up to C = 4 at V = K + C*A; histories longer than the CTA with bad pointers and
ids outside int32; rows whose logsumexp is NaN (NaN ranks first in the diverse merge, deterministically; the constrained merge drops
them); and whole decodes whose head bias holds a NaN."""
import numpy as np
import pytest
import torch

from tools import beam_select_oracle as O
from tools import constrained_beam_oracle as CO
from tools import diverse_beam_oracle as DO
from tools import sampling_oracle as SO
from vlp_b200 import ops

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
EOS = 5
SMEM_MAX = 200 * 1024                                                    # SAMPLE_SMEM_MAX
THREADS = 1024


def _vmax(T_cap):
    V = 1
    while ((V + 1) + ((V + 1) + 31) // 32 + T_cap) * 4 <= SMEM_MAX:
        V += 1
    return V


def _np(t):
    return t.detach().float().cpu().numpy()


def _bits(t):
    """fp32 tensor or array -> int32 bit patterns, so that NaN compares as bits."""
    t = torch.as_tensor(np.ascontiguousarray(t)) if isinstance(t, np.ndarray) else t.detach().cpu().contiguous()
    return t.view(torch.int32)


# ---------------------------------------------------------------------------------------------------------------------------------
# rows
# ---------------------------------------------------------------------------------------------------------------------------------
SHAPES = ["gauss", "quant", "chunk_ties", "equal", "max_last", "dominant", "neginf_k", "neginf_few"]


def _shape_row(shape, gen, V, K, dtype):
    """One fp32 row of logits of the given shape (before rounding to dtype)."""
    x = torch.randn(V, generator=gen) * 2.0
    if shape == "quant":                                                # tie groups that straddle the K boundary
        return torch.round(x * 2) / 2
    if shape == "chunk_ties":                                           # equal values at lo - 1 / lo of adjacent row chunks
        C = ((V + THREADS - 1) // THREADS) | 1
        x = x - 4.0
        for t in range(1, min(THREADS, (V - 1) // C + 1), max(1, THREADS // 64)):
            x[t * C - 1] = x[t * C] = 3.0 + (t % 3)
        return x
    if shape == "equal":
        return torch.full((V,), 0.75)
    if shape == "max_last":
        x[-1] = x.max() + 1.0
        return x
    if shape == "dominant":                                             # L = 0: the argmax's logp is +0
        x = -60.0 - 20.0 * torch.rand(V, generator=gen)
        x[int(torch.randint(0, V, (1,), generator=gen))] = 40.0
        return x
    if shape in ("neginf_k", "neginf_few"):                             # exactly K finite words, or fewer (-inf ties by index)
        keep = K if shape == "neginf_k" else max(1, K // 2)
        out = torch.full((V,), float("-inf"))
        idx = torch.randperm(V, generator=gen)[:min(keep, V)]
        out[idx] = x[idx]
        return out
    return x


def _logits(gen, rows, V, K, dtype, shapes=("gauss",), ld=None, alphabet=12):
    """[rows, V] logits of dtype, row r of shape shapes[r % len]; a view of [rows, ld] with NaN in the columns past V when ld > V.
    The first `alphabet` words (the histories' and constraints' words) are favoured on Gaussian rows, so blocks and completions land
    in the top K."""
    out = torch.stack([_shape_row(shapes[r % len(shapes)], gen, V, K, dtype) for r in range(rows)])
    for r in range(rows):
        if shapes[r % len(shapes)] == "gauss":
            out[r, :min(alphabet, V)] += 4.0
    wide = torch.full((rows, ld or V), float("nan"))
    wide[:, :V] = out
    return wide.to(DEV, dtype)[:, :V]


def _bias(gen, V, dtype, nan_at=None):
    """[V] bias of dtype with NaN on both sides of it in memory (a read past either end shows), and NaN at nan_at."""
    wide = torch.full((V + 2,), float("nan"))
    wide[1:V + 1] = torch.randn(V, generator=gen) * 0.5
    if nan_at is not None:
        wide[1 + nan_at] = float("nan")
    return wide.to(DEV, dtype)[1:V + 1]


def _x(logits, bias):
    return SO.head_x(_np(logits), None if bias is None else _np(bias), logits.dtype == BF)


def _prev(gen, B, W, V, eos_rate=0.2):
    """Frame f-1's traces [B, W]: words, pointers, scores and eos flags (score / eos of a parent enter its candidates)."""
    wid = torch.randint(0, min(V, 12), (B, W), generator=gen)
    ptr = torch.randint(0, W, (B, W), generator=gen)
    score = (-torch.rand(B, W, generator=gen) * 6.0).float()
    eos = (torch.rand(B, W, generator=gen) < eos_rate).float()
    return wid, ptr, score, eos


def _histories(gen, rows, T_cap, f, alphabet=12):
    return torch.randint(0, alphabet, (rows, T_cap), generator=gen, dtype=torch.int32)


# ---------------------------------------------------------------------------------------------------------------------------------
# one frame, run and checked
# ---------------------------------------------------------------------------------------------------------------------------------
def _traces(T, B, W, f, prev):
    wi, pt = (torch.full((T, B, W), -7, dtype=torch.int64) for _ in range(2))
    sc, eo = (torch.full((T, B, W), 0.125) for _ in range(2))
    if f:
        for t, p in zip((wi, pt, sc, eo), prev):
            t[f - 1] = p
    return [t.to(DEV) for t in (wi, pt, sc, eo)]


def _check_rows(x, K, tw, tl, blocked, block_eos, comp=None):
    """Each row's top K against the oracle's row restated on the kernel's own logsumexp; returns the oracle's (words, lp, lp rows).
    comp: per row, the kernel's completing (words, values), left out of the ranking."""
    ow, ol, lps = [], [], []
    for i in range(x.shape[0]):
        cw, cv = comp[i] if comp else (np.zeros(0, np.int64), np.zeros(0, np.float32))
        words = np.concatenate([tw[i], cw]).astype(np.int64)
        values = np.concatenate([tl[i], cv]).astype(np.float32)
        L, lse, tol, lp, w, v = O.row_stage(x[i], K, words, values, None if blocked is None else blocked[i], block_eos, EOS, tuple(cw))
        if not O.nonfinite(x[i]):
            assert abs(float(L) - lse) <= tol, (i, float(L), lse, tol)
        assert np.array_equal(w, tw[i]), (i, w, tw[i])
        assert np.array_equal(v.view(np.uint32), tl[i].view(np.uint32)), (i, v, tl[i])
        ow.append(w)
        ol.append(v)
        lps.append(lp)
    return np.stack(ow), np.stack(ol), lps


def run_diverse(logits, bias, f, B, K, G, lam, prev=None, n=0, ignore=(), block_eos=False, hist_in=None, T_cap=None):
    """One diverse frame on the device; returns its outputs (wid, ptr, score, eos [B, K], top_w, top_lp, hist_out) on the host."""
    T = T_cap or f + 1
    wi, pt, sc, eo = _traces(T, B, K, f, prev)
    tw = torch.full((B * K, K), -7, dtype=torch.int32, device=DEV)
    tl = torch.full((B * K, K), 0.125, device=DEV)
    hist = [torch.full((B * K, T), -7, dtype=torch.int32, device=DEV) for _ in range(2)]
    if hist_in is not None:
        hist[0].copy_(hist_in)
    ign = torch.tensor(ignore, dtype=torch.int32, device=DEV) if ignore else None
    ops.diverse_beam_step(logits, bias, f, G, lam, wi, pt, sc, eo, tw, tl, EOS, block_eos, ngram=n, ignore=ign, hist_in=hist[0],
                          hist_out=hist[1])
    torch.cuda.synchronize()
    rows = B if f == 0 else B * K
    assert (wi[f + 1:] == -7).all() and (sc[f + 1:] == 0.125).all()  # other frames untouched
    if f:
        assert (wi[:f - 1] == -7).all()
    return [t[f].cpu() for t in (wi, pt, sc, eo)] + [tw[:rows].cpu(), tl[:rows].cpu(), hist[1].cpu()]


def check_diverse(logits, bias, f, B, K, G, lam, prev=None, n=0, ignore=(), block_eos=False, hist_in=None, T_cap=None):
    """One diverse frame against the oracle, bit for bit; returns the device outputs."""
    out = run_diverse(logits, bias, f, B, K, G, lam, prev, n, ignore, block_eos, hist_in, T_cap)
    wid, ptr, score, eos, tw, tl, hist_out = out
    V = logits.shape[-1]
    blocked = None
    if n and f >= 1:
        hists = O.carry(hist_in.cpu().numpy(), prev[1].numpy(), prev[0].numpy(), K, f)
        assert np.array_equal(hist_out[:, :f].numpy(), hists)
        assert (hist_out[:, f:] == -7).all()
        if f >= n:
            blocked = O.ngram_blocked(hists, n, ignore, V)
    elif hist_out is not None:
        assert (hist_out == -7).all()                                   # no n-grams: the carry does not run
    x = _x(logits, bias)
    ow, ol, _ = _check_rows(x, K, tw.numpy(), tl.numpy(), blocked, block_eos)
    ps, pe = (prev[2].numpy(), prev[3].numpy()) if f else (None, None)
    mw, mp, ms, _ = DO.merge(ow, ol, ps, pe, K, G, lam, f == 0)
    assert torch.equal(wid, torch.from_numpy(mw)) and torch.equal(ptr, torch.from_numpy(mp)), (wid, mw, ptr, mp)
    assert torch.equal(_bits(score), _bits(O.canonical(ms))), (score, ms)      # the device's arithmetic NaN is canonical
    assert torch.equal(eos, (wid == EOS).float())
    return out


def run_constrained(logits, bias, f, cons, K, prev=None, n=0, ignore=(), block_eos=False, hist_in=None, T_cap=None):
    B, C, A, _ = cons.shape
    SK, W = K << C, K + C * A
    T = T_cap or f + 1
    wi, pt, sc, eo = _traces(T, B, SK, f, prev)
    tw = torch.full((B * SK, W), -7, dtype=torch.int32, device=DEV)
    tl = torch.full((B * SK, W), 0.125, device=DEV)
    td = torch.full((B * SK, C * A), -7, dtype=torch.int32, device=DEV)
    hist = [torch.full((B * SK, T), -7, dtype=torch.int32, device=DEV) for _ in range(2)]
    if hist_in is not None:
        hist[0].copy_(hist_in)
    ign = torch.tensor(ignore, dtype=torch.int32, device=DEV) if ignore else None
    ops.constrained_beam_step(logits, bias, f, cons.to(DEV), wi, pt, sc, eo, tw, tl, td, EOS, block_eos, ngram=n, ignore=ign,
                              hist_in=hist[0], hist_out=hist[1])
    torch.cuda.synchronize()
    rows = B if f == 0 else B * SK
    assert (wi[f + 1:] == -7).all() and (sc[f + 1:] == 0.125).all()
    return [t[f].cpu() for t in (wi, pt, sc, eo)] + [tw[:rows].cpu(), tl[:rows].cpu(), td[:rows].cpu(), hist[1].cpu()]


def check_constrained(logits, bias, f, cons, K, prev=None, n=0, ignore=(), block_eos=False, hist_in=None, T_cap=None):
    out = run_constrained(logits, bias, f, cons, K, prev, n, ignore, block_eos, hist_in, T_cap)
    wid, ptr, score, eos, tw, tl, td, hist_out = out
    B, C, A, _ = cons.shape
    SK = K << C
    V = logits.shape[-1]
    cn = cons.numpy()
    hists, blocked = None, None
    if f >= 1:
        hists = O.carry(hist_in.cpu().numpy(), prev[1].numpy(), prev[0].numpy(), SK, f)
        assert np.array_equal(hist_out[:, :f].numpy(), hists)
        assert (hist_out[:, f:] == -7).all()
        if n and f >= n:
            blocked = O.ngram_blocked(hists, n, ignore, V)
    tw, tl, td = tw.numpy(), tl.numpy(), td.numpy()
    comp = []
    for i, (b, p, s) in enumerate(CO._rows(B, K, C, f == 0, cn)):
        want = CO.completions([] if hists is None else [int(w) for w in hists[i]], cn[b], s)
        m = len(want)
        assert tw[i, K:K + m].tolist() == list(want) and td[i, :m].tolist() == list(want.values()), (i, want, tw[i, K:], td[i])
        assert (tw[i, K + m:] == -1).all() and (td[i, m:] == -1).all() and np.isneginf(tl[i, K + m:]).all()
        comp.append((tw[i, K:K + m].astype(np.int64), tl[i, K:K + m]))
    x = _x(logits, bias)
    ow, ol, lps = _check_rows(x, K, tw[:, :K], tl[:, :K], blocked, block_eos, comp)
    for i, (cw, cv) in enumerate(comp):                                 # a completing word keeps its exact logp
        assert np.array_equal(lps[i][cw].view(np.uint32), cv.view(np.uint32)), i
    lists = [(ow[i], ol[i], {int(w): (lps[i][w], int(d)) for w, d in zip(cw, td[i])}) for i, (cw, _) in enumerate(comp)]
    ps, pe = (prev[2].numpy(), prev[3].numpy()) if f else (None, None)
    mw, mp, ms, _ = CO.merge(lists, ps, pe, cn, K, f == 0)
    assert torch.equal(wid, torch.from_numpy(mw)) and torch.equal(ptr, torch.from_numpy(mp)), (wid, mw, ptr, mp)
    assert torch.equal(_bits(score), _bits(ms.astype(np.float32))), (score, ms)
    assert torch.equal(eos, ((wid == EOS) & torch.isfinite(score)).float())
    return out


def _table(gen, B, C, A, P, alphabet=12):
    """Constraints over the words [1, alphabet) (never [EOS]): alternatives of 1 .. P words, some constraints with fewer."""
    t = torch.zeros(B, C, A, P, dtype=torch.int64)
    for b in range(B):
        for j in range(C):
            for q in range(int(torch.randint(1, A + 1, (1,), generator=gen))):
                L = int(torch.randint(1, P + 1, (1,), generator=gen))
                w = torch.randint(1, alphabet, (L,), generator=gen)
                t[b, j, q, :L] = torch.where(w == EOS, w + 1, w)
    return t


# ---------------------------------------------------------------------------------------------------------------------------------
# vocabularies, beams and groups
# ---------------------------------------------------------------------------------------------------------------------------------
T_CAP = 4
VMAX = _vmax(T_CAP)
DIVERSE_VOCABS = [(1, 1, 1), (6, 6, 3), (63, 63, 63), (64, 64, 2), (33, 2, 2), (33, 6, 6), (1023, 63, 3), (1024, 64, 64),
                  (1025, 48, 2), (3072, 1, 1), (3073, 64, 2), (28996, 6, 3), (30522, 48, 48), (VMAX, 64, 1), (VMAX, 2, 2)]


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("V,K,G", DIVERSE_VOCABS, ids=[f"V{v}-K{k}-G{g}" for v, k, g in DIVERSE_VOCABS])
def test_diverse_vocabularies(V, K, G, dtype):
    gen = torch.Generator().manual_seed(V * 7 + K)
    B = 3
    bias = _bias(gen, V, dtype)
    check_diverse(_logits(gen, B, V, K, dtype), bias, 0, B, K, G, 0.5, T_cap=T_CAP)
    f, n = 2, 2
    prev = _prev(gen, B, K, V)
    hist_in = _histories(gen, B * K, T_CAP, f).to(DEV)
    check_diverse(_logits(gen, B * K, V, K, dtype), bias, f, B, K, G, 0.75, prev, n=n, ignore=(7,), block_eos=True, hist_in=hist_in,
                  T_cap=T_CAP)


CONSTRAINED_VOCABS = [(1, 1, 1, 2), (16, 4, 4, 8), (6, 3, 2, 3), (64, 2, 4, 2), (2, 1, 1, 1), (4, 2, 3, 3)]


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("K,C,A,P", CONSTRAINED_VOCABS, ids=[f"K{k}-C{c}-A{a}-P{p}" for k, c, a, p in CONSTRAINED_VOCABS])
@pytest.mark.parametrize("Vx", ["min", 1025, 3073, 30522, "max"])
def test_constrained_vocabularies(Vx, K, C, A, P, dtype):
    """V = K + C*A exactly ("min"), the row chunks' edges and the shared-memory limit; up to S*K = 256 slots."""
    V = {"min": K + C * A, "max": VMAX}.get(Vx, Vx)
    if K << C > 64 and isinstance(Vx, int) and Vx > 3073:
        pytest.skip("256 rows of a large vocabulary: the V = K + C*A and V_max cases cover the slot count")
    gen = torch.Generator().manual_seed(V * 13 + K + C)
    B = 2
    cons = _table(gen, B, C, A, P, alphabet=min(12, V))
    bias = _bias(gen, V, dtype)
    alphabet = min(12, V)
    check_constrained(_logits(gen, B, V, K, dtype, alphabet=alphabet), bias, 0, cons, K, T_cap=T_CAP)
    SK = K << C
    f = 2
    prev = _prev(gen, B, SK, V)
    hist_in = _histories(gen, B * SK, T_CAP, f, alphabet).to(DEV)
    check_constrained(_logits(gen, B * SK, V, K, dtype, alphabet=alphabet), bias, f, cons, K, prev, n=2 if V > 40 else 0, ignore=(3,),
                      block_eos=V > 40, hist_in=hist_in, T_cap=T_CAP)


def test_one_past_the_shared_memory_limit_is_refused_before_a_launch():
    V, K = VMAX + 1, 4
    logits = torch.zeros(2, V, dtype=BF, device=DEV)
    wi, pt, sc, eo = _traces(T_CAP, 2, K, 0, None)
    tw = torch.full((2 * K, K), -7, dtype=torch.int32, device=DEV)
    tl = torch.full((2 * K, K), 0.125, device=DEV)
    with pytest.raises(RuntimeError):
        ops.diverse_beam_step(logits, None, 0, 2, 0.5, wi, pt, sc, eo, tw, tl, EOS)
    cons = torch.zeros(2, 1, 1, 1, dtype=torch.int64, device=DEV)
    cwi, cpt, csc, ceo = _traces(T_CAP, 2, 2 * K, 0, None)
    ctw = torch.full((4 * K, K + 1), -7, dtype=torch.int32, device=DEV)
    ctl = torch.full((4 * K, K + 1), 0.125, device=DEV)
    ctd = torch.full((4 * K, 1), -7, dtype=torch.int32, device=DEV)
    with pytest.raises(RuntimeError):
        ops.constrained_beam_step(logits, None, 0, cons, cwi, cpt, csc, ceo, ctw, ctl, ctd, EOS)
    torch.cuda.synchronize()
    for t in (wi, pt, tw, cwi, cpt, ctw, ctd):
        assert bool((t == -7).all())
    for t in (sc, eo, tl, csc, ceo, ctl):
        assert bool((t == 0.125).all())


# ---------------------------------------------------------------------------------------------------------------------------------
# row shapes, layouts and dtypes
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("V", [1025, 3073, 30522])
@pytest.mark.parametrize("K,G", [(6, 3), (64, 4)])
def test_row_shapes(K, G, V, dtype):
    """Every shape in one launch: Gaussian, quantised (ties across the K boundary), ties at adjacent chunks' lo - 1 / lo, all equal,
    the max only at V - 1, one dominant word (L = 0), and -inf rows with K or fewer finite words."""
    gen = torch.Generator().manual_seed(V + K)
    B = len(SHAPES)
    check_diverse(_logits(gen, B, V, K, dtype, SHAPES), None, 0, B, K, G, 0.5)
    Bf = max(1, 2 * len(SHAPES) // K)
    prev = _prev(gen, Bf, K, V)
    check_diverse(_logits(gen, Bf * K, V, K, dtype, SHAPES), None, 1, Bf, K, G, 0.3, prev)
    cons = _table(gen, B, 2, 2, 1)
    check_constrained(_logits(gen, B, V, K, dtype, SHAPES), None, 0, cons, K)


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("with_bias", [False, True], ids=["nobias", "bias"])
@pytest.mark.parametrize("V", [1025, 3073])
def test_strided_logits_with_nan_past_the_row(V, with_bias, dtype):
    """ld > V with NaN in the gap columns and on both sides of the bias: a read outside [0, V) would make the row non-finite."""
    gen = torch.Generator().manual_seed(V + with_bias)
    B, K, G = 4, 6, 2
    bias = _bias(gen, V, dtype) if with_bias else None
    check_diverse(_logits(gen, B, V, K, dtype, ld=V + 37), bias, 0, B, K, G, 0.5)
    prev = _prev(gen, B, K, V)
    check_diverse(_logits(gen, B * K, V, K, dtype, ld=V + 37), bias, 1, B, K, G, 0.5, prev)
    cons = _table(gen, B, 2, 2, 2)
    check_constrained(_logits(gen, B, V, K, dtype, ld=V + 37), bias, 0, cons, K)


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
def test_a_blocked_word_ties_the_eos_block(dtype):
    """The dominant word w is blocked (history a, w, a with n = 2) and [EOS] is blocked by min_len: both are exactly -10000
    (fl(fl(0 - L) - 10000), L = 0), and the K = V - 1 cut falls between them, so the lower word id wins."""
    V, K, G, f = 33, 32, 2, 3
    gen = torch.Generator().manual_seed(3)
    B = 2
    a = 9
    logits = -torch.rand(B * K, V, generator=gen) * 2 - 40
    dom = torch.tensor([2 if r % 2 else 20 for r in range(B * K)])        # below and above EOS = 5
    logits[torch.arange(B * K), dom] = 40.0
    hist_in = torch.full((B * K, 4), a, dtype=torch.int32)
    prev = _prev(gen, B, K, V)
    prev[0].fill_(a)
    prev[1].copy_(torch.arange(K).expand(B, K))
    hist_in[:, 1] = dom.int()
    out = check_diverse(logits.to(DEV, dtype), None, f, B, K, G, 0.0, prev, n=2, block_eos=True, hist_in=hist_in.to(DEV), T_cap=4)
    tw, tl = out[4], out[5]
    for r in range(B * K):
        last = tw[r, -1].item()
        assert last == min(int(dom[r]), EOS) and tl[r, -1].item() == -10000.0, (r, tw[r], tl[r])


# ---------------------------------------------------------------------------------------------------------------------------------
# constraints
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
def test_completing_words_at_the_argmax_and_in_the_tie_set(dtype):
    """Constraint 0: word 3 (the argmax of every row); constraint 1: word 7 or the phrase [8, 7]; constraint 2: word 4, tied at the K
    boundary with other words of its row, or (image 1) word 7, so that 7 completes two constraints and its dest is their OR.
    V = K + C*A exactly."""
    K, C, A, P = 6, 3, 2, 2
    V = K + C * A
    B = 2
    cons = torch.zeros(B, C, A, P, dtype=torch.int64)
    cons[:, 0, 0, 0] = 3
    cons[:, 1, 0, 0] = 7
    cons[:, 1, 1, :2] = torch.tensor([8, 7])
    cons[:, 2, 0, 0] = 4
    cons[1, 2, 1, 0] = 7                                                  # image 1: 7 also completes constraint 2
    gen = torch.Generator().manual_seed(11)

    def rows(n):
        x = torch.round(torch.randn(n, V, generator=gen) * 2) / 2
        x[:, 3] = 6.0
        x[:, 4] = x[:, 9] = x[:, 10] = 1.0                             # ties with the constraint word 4
        x[:, 7] = 1.0
        return x.to(DEV, dtype)

    check_constrained(rows(B), None, 0, cons, K)
    SK = K << C
    prev = _prev(gen, B, SK, V)
    prev[0][:, ::2] = 8                                                   # half the slots end in 8: [8, 7] completes too
    hist_in = _histories(gen, B * SK, 4, 2).to(DEV)
    out = check_constrained(rows(B * SK), None, 2, cons, K, prev, hist_in=hist_in, T_cap=4)
    assert (out[6][:, :3] >= 0).any()


# ---------------------------------------------------------------------------------------------------------------------------------
# histories
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,ignore", [(1, (0,)), (2, (4, 9)), (3, ())])
def test_long_histories_bad_pointers_and_ids_outside_int32(n, ignore):
    """T_cap = 1100 and f = 1050: the carry strides past the CTA's 1024 threads.  Back pointers -1, width and 2^40 give -1 words,
    ids outside int32 give -1; the carried rows equal the restatement and the n-gram blocks follow from them."""
    T_cap, f, V, K, G = 1100, 1050, 3073, 4, 2
    gen = torch.Generator().manual_seed(n)
    B = 3
    bad_ptr = [-1, K, 1 << 40]
    bad_wid = [1 << 33, -(1 << 33), 1 << 31, -(1 << 31) - 1, V + 5, -3]
    prev = _prev(gen, B, K, V)
    for j, p in enumerate(bad_ptr):
        prev[1][j % B, (j + 1) % K] = p
    for j, w in enumerate(bad_wid):
        prev[0][(j + 1) % B, j % K] = w
    hist_in = torch.randint(0, 6, (B * K, T_cap), generator=gen, dtype=torch.int32)
    hist_in[::3, 500:700] = torch.randint(-(1 << 31), (1 << 31) - 1, (1, 200), generator=gen, dtype=torch.int32)
    check_diverse(_logits(gen, B * K, V, K, BF, alphabet=6), None, f, B, K, G, 0.5, prev, n=n, ignore=ignore, hist_in=hist_in.to(DEV),
                  T_cap=T_cap)
    C, A, P = 2, 2, 3
    SK = K << C
    cons = _table(gen, B, C, A, P, alphabet=6)
    cprev = _prev(gen, B, SK, V)
    for j, p in enumerate(bad_ptr):
        cprev[1][j % B, (3 * j + 1) % SK] = p if p != K else SK
    for j, w in enumerate(bad_wid):
        cprev[0][(j + 1) % B, (5 * j) % SK] = w
    chist = torch.randint(0, 6, (B * SK, T_cap), generator=gen, dtype=torch.int32)
    check_constrained(_logits(gen, B * SK, V, K, torch.float32, alphabet=6), None, f, cons, K, cprev, n=n, ignore=ignore,
                      hist_in=chist.to(DEV), T_cap=T_cap)


# ---------------------------------------------------------------------------------------------------------------------------------
# rows whose logsumexp is NaN
# ---------------------------------------------------------------------------------------------------------------------------------
def _nonfinite_rows(gen, rows, V, K, dtype):
    """Gaussian rows, one in four with a NaN logit, one with a +inf logit, one all -inf."""
    x = torch.randn(rows, V, generator=gen) * 2
    x[:, :12] += 4
    for r in range(rows):
        kind = r % 4
        if kind == 1:
            x[r, int(torch.randint(0, V, (1,), generator=gen))] = float("nan")
        elif kind == 2:
            x[r, int(torch.randint(0, V, (1,), generator=gen))] = float("inf")
        elif kind == 3:
            x[r] = float("-inf")
    return x.to(DEV, dtype)


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("bias_nan", [False, True], ids=["rows", "bias"])
def test_nan_rows_rank_first_in_the_diverse_merge(bias_nan, dtype):
    """NaN logsumexp rows (NaN / +inf logit, all -inf, or a NaN bias element: every row) give their lowest NaN words with NaN values,
    which rank above every number in the merge, ties by (parent, word); two runs are bitwise equal."""
    V, K, G = 1000, 6, 3
    gen = torch.Generator().manual_seed(17 + bias_nan)
    B = 4
    bias = _bias(gen, V, dtype, nan_at=321 if bias_nan else None)
    l0 = _nonfinite_rows(gen, B, V, K, dtype)
    prev = _prev(gen, B, K, V)
    prev[2][1, 2] = float("nan")                                        # a NaN parent score: all its candidates are NaN
    l1 = _nonfinite_rows(gen, B * K, V, K, dtype)
    outs = []
    for _ in range(2):
        a = check_diverse(l0, bias, 0, B, K, G, 0.5, block_eos=True)
        b = check_diverse(l1, bias, 1, B, K, G, 0.5, prev)
        outs.append(a + b)
    for x, y in zip(*outs):
        assert _same(x, y)
    wid = outs[0][0]
    assert ((wid >= 0) & (wid < V)).all()


@pytest.mark.parametrize("dtype", [BF, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("bias_nan", [False, True], ids=["rows", "bias"])
def test_nan_rows_are_dropped_by_the_constrained_merge(bias_nan, dtype):
    V, K, C, A, P = 1000, 4, 2, 2, 2
    gen = torch.Generator().manual_seed(23 + bias_nan)
    B = 4
    SK = K << C
    cons = _table(gen, B, C, A, P)
    bias = _bias(gen, V, dtype, nan_at=77 if bias_nan else None)
    l0 = _nonfinite_rows(gen, B, V, K, dtype)
    out0 = check_constrained(l0, bias, 0, cons, K)
    prev = _prev(gen, B, SK, V)
    hist_in = _histories(gen, B * SK, 4, 2).to(DEV)
    out1 = check_constrained(_nonfinite_rows(gen, B * SK, V, K, dtype), bias, 2, cons, K, prev, hist_in=hist_in, T_cap=4)
    for wid, ptr, score, _ in (out0[:4], out1[:4]):
        empty = ~torch.isfinite(score)
        assert (wid[empty] == 0).all() and (ptr[empty] == 0).all()
        if bias_nan:
            assert empty.all()
    again = run_constrained(l0, bias, 0, cons, K)
    for x, y in zip(again, out0):
        assert _same(x, y)


# ---------------------------------------------------------------------------------------------------------------------------------
# whole decodes with a NaN in the head bias
# ---------------------------------------------------------------------------------------------------------------------------------
def _nan_bias_decoder(**kw):
    from test_diverse_beam_gpu import _decoder
    from vlp_b200 import synth

    model = _decoder(synth.SMALL_L123, **kw)
    with torch.no_grad():
        model.cls.predictions.bias[321] = float("nan")
    return model


def _same(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32)) if a.dtype == torch.float32 else torch.equal(a, b)


def test_decodes_with_a_nan_in_the_head_bias_complete():
    from test_diverse_beam_gpu import _args
    from vlp_b200 import synth

    dims = synth.SMALL_L123
    B = 3
    args = _args(dims, B, seed=2)
    T = args[3].shape[1] - args[2].shape[1]
    model = _nan_bias_decoder(search_beam_size=6, num_beam_groups=3, diversity_penalty=0.5, forbid_duplicate_ngrams=True, ngram_size=2)
    outs = [model(*args, task_idx=None) for _ in range(2)]
    for k in outs[0]:
        assert _same(outs[0][k], outs[1][k]), k
    wi = outs[0]["wids"][:, :T]
    assert ((wi >= 0) & (wi < dims.vocab)).all() and ((outs[0]["pred_seq"] >= 0) & (outs[0]["pred_seq"] < dims.vocab)).all()
    assert torch.isnan(outs[0]["scores"][:, :T]).all()

    model = _nan_bias_decoder(search_beam_size=3)
    cons = torch.zeros(B, 2, 2, 1, dtype=torch.int64, device=DEV)
    cons[:, :, :, 0] = torch.tensor([[11, 12], [13, 14]], device=DEV)
    outs = [model(*args, task_idx=None, constraints=cons) for _ in range(2)]
    for k in outs[0]:
        assert _same(outs[0][k], outs[1][k]), k
    out = outs[0]
    sc, wi, pt = (out[k][:, :T] for k in ("scores", "wids", "ptrs"))
    assert torch.isneginf(sc).all() and (wi == 0).all() and (pt == 0).all()  # every slot empty from frame 0 on
    assert (out["pred_seq"] == 0).all() and not out["constraints_met"].any()
    assert torch.isneginf(out["state_scores"]).all()
