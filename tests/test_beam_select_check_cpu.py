"""CPU: the exact statement of the beam selectors' row stage (tools/beam_select_oracle.py) on rows built with a known fp32 logsumexp
L: recover_lse finds L (from an unblocked argmax exactly, else as the one fp32 value within the stated bound that reproduces the
returned pairs), the order_key ranking is lexsort's on finite rows and puts NaN first, the history carry treats bad pointers and ids
as the kernels do, and the diverse merge ranks NaN candidates first."""
import numpy as np
import pytest

from tools import beam_select_oracle as O
from tools import diverse_beam_oracle as DO
from tools.sampling_oracle import bf16_round


def _rows(seed, rows, V, bf16):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal((rows, V)) * 1.5).astype(np.float32)
    return bf16_round(x) if bf16 else x


def _kernel_like(x, L, K, blocked=None, block_eos=False, eos=-1):
    """The pairs a kernel with logsumexp L returns for row x: its restated top K."""
    lp = O.row_logp(x, L, blocked, block_eos, eos)
    return O.rank(lp, K)


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("V", [33, 1000, 3073])
def test_an_unblocked_argmax_gives_L_exactly(V, bf16):
    for i, x in enumerate(_rows(V, 8, V, bf16)):
        lse, tol = O.lse_tol(x)
        L = np.float32(lse + (i - 4) * 0.25 * tol)                    # any L within the bound
        w, v = _kernel_like(x, L, 6)
        cands, _, _ = O.recover_lse(x, w, v)
        assert cands.view(np.uint32).tolist() == [np.float32(L).view(np.uint32)]


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("V", [1000, 28996])
def test_a_blocked_argmax_gives_the_one_L_within_the_bound(V, bf16):
    """With the argmax blocked, L comes from the other returned values.  Where the runner-up's lp = fl(d - L) shares L's binade (d =
    -2^-6 here), each fp32 step of L moves it, so exactly one fp32 value within the bound reproduces the pairs; elsewhere the
    candidates include L and any of them restates the same top K."""
    unique = 0
    for i, x in enumerate(_rows(V + 1, 12, V, bf16)):
        top = int(np.argmax(x))
        second = (top + 1) % V
        x[second] = x[top] - np.float32(2.0 ** -6)
        blocked = np.zeros(V, bool)
        blocked[top] = True
        lse, tol = O.lse_tol(x)
        L = np.float32(lse + (i % 7 - 3) * 0.3 * tol)
        w, v = _kernel_like(x, L, 4, blocked)
        cands, _, _ = O.recover_lse(x, w, v, blocked)
        assert np.float32(L).view(np.uint32) in cands.view(np.uint32)
        if np.frexp(v[0])[1] == np.frexp(L)[1]:
            assert cands.view(np.uint32).tolist() == [np.float32(L).view(np.uint32)], (i, cands, L)
            unique += 1
        got = O.row_stage(x, 4, w, v, blocked)
        assert abs(float(got[0]) - lse) <= tol
        assert np.array_equal(got[4], w) and np.array_equal(got[5].view(np.uint32), v.view(np.uint32))
    assert unique >= 9, unique


def test_the_bound_holds_for_a_float32_logsumexp():
    """The bound covers an fp32 evaluation of the same sum in another order (numpy's pairwise sum, expf by float32 exp)."""
    for V in (33, 1025, 30522):
        for x in _rows(V + 2, 4, V, True):
            lse, tol = O.lse_tol(x)
            e = np.exp((x - x.max()).astype(np.float32)).astype(np.float32)
            L32 = np.log(e.sum(dtype=np.float32), dtype=np.float32)
            assert abs(float(L32) - lse) <= tol, (V, float(L32), lse, tol)


def test_order_key_ranks_as_lexsort_on_finite_rows():
    rng = np.random.default_rng(3)
    for V in (7, 64, 1025):
        lp = (np.round(rng.standard_normal(V) * 4) / 4 - 3).astype(np.float32)     # many ties
        lp[rng.random(V) < 0.2] = -np.inf
        lp[rng.random(V) < 0.1] = O.BLOCK
        for K in (1, 5, min(V, 64)):
            w, v = O.rank(lp, K)
            want = np.lexsort((np.arange(V), -lp))[:K]
            assert np.array_equal(w, want) and np.array_equal(v, lp[want])
    keys = O.order_key(np.array([-np.inf, -1.0, -0.0, 0.0, 1e-30, np.inf, np.nan], np.float32))
    assert (np.diff(keys.astype(np.int64)) > 0).all()
    assert O.order_key(O.CANONICAL_NAN) == 0xFFFFFFFF and O.order_key(np.array(-1, np.int32).view(np.float32)) == 0


@pytest.mark.parametrize("kind", ["nan", "posinf", "all_neginf"])
def test_a_non_finite_row_ranks_its_lowest_nan_words(kind):
    V, K, eos = 40, 6, 2
    x = _rows(9, 1, V, False)[0]
    x[{"nan": 17, "posinf": 30, "all_neginf": slice(None)}[kind]] = {"nan": np.nan, "posinf": np.inf, "all_neginf": -np.inf}[kind]
    assert O.nonfinite(x)
    _, _, _, lp, w, v = O.row_stage(x, K, np.zeros(K, np.int64), np.zeros(K, np.float32))
    assert w.tolist() == list(range(K)) and (v.view(np.uint32) == 0x7FFFFFFF).all() and (lp.view(np.uint32) == 0x7FFFFFFF).all()
    _, _, _, lp, w, v = O.row_stage(x, K, np.zeros(K, np.int64), np.zeros(K, np.float32), block_eos=True, eos_id=eos)
    assert w.tolist() == [0, 1, 3, 4, 5, 6] and lp[eos] == O.BLOCK                 # the [EOS] block is a number: it ranks last
    _, _, _, _, w, _ = O.row_stage(x, K, np.zeros(K, np.int64), np.zeros(K, np.float32), exclude=(1, 4))
    assert w.tolist() == [0, 2, 3, 5, 6, 7]


def test_the_carry_treats_bad_pointers_and_ids_as_the_kernels_do():
    width, f = 4, 5
    rng = np.random.default_rng(5)
    hist_in = rng.integers(0, 50, (2 * width, 8))
    ptr = np.array([0, 3, -1, 4, 1 << 40, 2, -(1 << 40), 1])
    wid = np.array([7, 1 << 33, -(1 << 33), -1, (1 << 31) - 1, -(1 << 31), 1 << 31, 9])
    out = O.carry(hist_in, ptr, wid, width, f)
    for i in range(2 * width):
        p = ptr[i]
        want = list(hist_in[(i // width) * width + p, :f - 1]) if 0 <= p < width else [-1] * (f - 1)
        w = wid[i]
        want.append(w if -(1 << 31) <= w < (1 << 31) else -1)
        assert out[i].tolist() == want, i
    first = O.carry(None, None, wid, width, 1)                       # frame 1: no parent words, the pointer is not read
    assert first[:, 0].tolist() == [7, -1, -1, -1, (1 << 31) - 1, -(1 << 31), -1, 9]


def test_the_diverse_merge_ranks_nan_first_by_parent_then_word():
    K, G = 4, 2
    nan = np.float32(np.nan)
    tw = np.array([[5, 6, 7, 8], [1, 2, 3, 4], [9, 10, 11, 12], [13, 14, 15, 16]], np.int64)
    tl = np.array([[-1, -2, nan, -3], [nan, -1, -2, -3], [-1, -2, -3, -4], [nan, nan, nan, nan]], np.float32)
    prev = np.zeros((1, K), np.float32), np.zeros((1, K), np.float32)
    wid, ptr, score, _ = DO.merge(tw, tl, *prev, K, G, 0.5, False)
    assert wid[0].tolist() == [7, 1, 13, 14] and ptr[0].tolist() == [0, 1, 3, 3]
    assert np.isnan(score[0]).all()
    finite = np.nan_to_num(tl, nan=-7.0)                              # finite frames keep lexsort's order
    wid, ptr, _, _ = DO.merge(tw, finite, *prev, K, G, 0.5, False)
    assert wid[0].tolist() == [5, 2, 9, 10] and ptr[0].tolist() == [0, 1, 2, 2]
