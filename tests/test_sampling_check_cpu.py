"""The sampling oracle of tests/test_sampling_exact_gpu.py on the CPU (tools/sampling_oracle.py): its Philox model reproduces the
Random123 known-answer vectors; `frame` agrees with a brute-force statement of the rule (stable sort, cumulative sum, linear scan) on
random, quantised, flat and zero-weight rows; and the exact comparison rejects planted defects of the sampler, several of which the
set-membership and chi-square criteria of tests/test_sampling_gpu.py accept."""
import numpy as np
import pytest
import torch
from scipy import stats

from tools import sampling_oracle as so

ALPHA = 1e-3                   # tests/test_sampling_gpu.py


@pytest.mark.parametrize("ctr,key,want", [
    ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
    ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
    ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0), (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1))])
def test_philox_matches_the_random123_known_answers(ctr, key, want):
    """Random123's kat_vectors for philox4x32_10: counter words (c0, c1, c2, c3) = (ctr_lo lo, ctr_lo hi, ctr_hi lo, ctr_hi hi), key
    words (seed lo, seed hi), as Philox::gen packs them."""
    seed = key[0] | key[1] << 32
    got = so.philox4x32_10(seed, ctr[2] | ctr[3] << 32, ctr[0] | ctr[1] << 32)
    assert tuple(int(v) for v in got) == want
    # vectorised: the same counter among others gives the same words
    many = so.philox4x32_10(seed, ctr[2] | ctr[3] << 32, np.array([ctr[0] | ctr[1] << 32, 5, 6], dtype=np.uint64))
    assert tuple(int(v) for v in many[0]) == want


def test_uniform_and_keep_mask_are_the_stated_bits():
    r = so.philox4x32_10((1 << 32) + 9, 7, np.arange(100, dtype=np.uint64))
    u = so.uniform((1 << 32) + 9, 7, np.arange(100, dtype=np.uint64))
    assert np.array_equal(u.astype(np.float64), (r[:, 0] >> 8).astype(np.float64) * 2.0 ** -24)
    m = so.keep_mask(0.1, 3, 17, 21)
    r = so.philox4x32_10(3, 17, np.arange(3, dtype=np.uint64))
    thresh = int(np.float32(0.1) * 65536)
    for i in range(21):
        word = int(r[i // 8, (i % 8) // 2])
        assert m[i] == (((word >> (16 * (i % 2))) & 0xFFFF) >= thresh)


def test_bf16_round_is_torchs():
    x = (np.random.default_rng(0).standard_normal(10000) * 10.0).astype(np.float32)
    x[:3] = [1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, -(1.0 + 2.0 ** -8)]     # ties to even
    assert np.array_equal(so.bf16_round(x), torch.from_numpy(x).bfloat16().float().numpy())


# --- the rule, brute force, with planted defects -----------------------------------------------------------------------------------
DEFECTS = ["tie_off_by_one", "nucleus_short", "nucleus_long", "nucleus_gt", "rank_walk", "bias_fp32", "philox_swap", "u_from_y",
           "u_23bits"]


def _uniforms(seed, f, rows, defect=None):
    if defect == "philox_swap":
        r = so.philox4x32_10(seed, rows, f)
    else:
        r = so.philox4x32_10(seed, f, rows)
    if defect == "u_from_y":
        return ((r[..., 1] >> 8).astype(np.float64) * 2.0 ** -24).astype(np.float32)
    if defect == "u_23bits":                                    # `r.x >> 9` at the same scale: 23 random bits, u in [0, 1/2)
        return ((r[..., 0] >> 9).astype(np.float64) * 2.0 ** -24).astype(np.float32)
    return ((r[..., 0] >> 8).astype(np.float64) * 2.0 ** -24).astype(np.float32)


def _rule(x32, mode, k, p, u, defect=None, scan=False):
    """The sampling rule in fp64 for one row and an array of uniforms, optionally with a planted defect.  scan=True states the cut and
    the draw as linear scans (the brute force); otherwise the draw is a search over the same cumulative sums."""
    x = np.asarray(x32, dtype=np.float32).astype(np.float64)
    V = x.size
    e = np.exp(x - x.max())
    order = np.argsort(-x, kind="stable")
    if mode == "topk":
        m = min(k, V)
    else:
        c = np.cumsum(e[order])
        t = float(np.float32(p)) * c[-1]
        m = 1
        if scan:
            while m < V and (c[m - 1] <= t if defect == "nucleus_gt" else c[m - 1] < t):
                m += 1
        else:
            m = max(1, min(V, 1 + int(np.count_nonzero(c <= t if defect == "nucleus_gt" else c < t))))
        if defect == "nucleus_short":
            m = max(1, m - 1)
        if defect == "nucleus_long":
            m = min(V, m + 1)
    if defect == "tie_off_by_one" and m < V and x[order[m]] == x[order[m - 1]]:
        m += 1
    walk = order[:m] if defect == "rank_walk" else np.sort(order[:m])
    w = e[walk]
    cum = np.cumsum(w)
    u = np.atleast_1d(np.asarray(u, dtype=np.float32)).astype(np.float64)
    if scan:
        out = []
        for g in u * cum[-1]:
            acc, pick = 0.0, walk[np.flatnonzero(w > 0)[-1]]
            for v, wv in zip(walk, w):
                acc += wv
                if g < acc:
                    pick = v
                    break
            out.append(int(pick))
        return np.array(out)
    return walk[np.minimum(np.searchsorted(cum, u * cum[-1], side="right"), m - 1)]


def _rows(gen, kind, R, V):
    if kind == "normal":
        return (gen.standard_normal((R, V)) * 3.0).astype(np.float32)
    if kind == "quantised":                                      # tie groups across many chunks
        return np.round(gen.standard_normal((R, V)) * 2.0).astype(np.float32)
    if kind == "equal":
        return np.full((R, V), 0.5, dtype=np.float32)
    if kind == "zero_weight":                                    # kept words of zero weight: -inf and e < 2^-1074 in fp64 too
        x = np.where(gen.random((R, V)) < 0.6, -np.inf, gen.standard_normal((R, V))).astype(np.float32)
        x[:, gen.integers(0, V)] = 2.0
        x[:, :V // 3] = np.where(gen.random((R, V // 3)) < 0.5, np.float32(-800.0), x[:, :V // 3])
        return x
    raise ValueError(kind)


SETTINGS = [("topk", 1, 1.0), ("topk", 2, 1.0), ("topk", 64, 1.0), ("topk", 64, 1.0), ("topp", 64, 1e-9), ("topp", 64, 0.3),
            ("topp", 64, 0.9), ("topp", 64, 1.0)]


@pytest.mark.parametrize("kind", ["normal", "quantised", "equal", "zero_weight"])
@pytest.mark.parametrize("V", [1, 2, 5, 33, 1025, 3073, 50000])
def test_frame_equals_the_brute_force_rule(kind, V):
    gen = np.random.default_rng(V + len(kind))
    R = 3 if V >= 3073 else 12
    x = _rows(gen, kind, R, V)
    for mode, k, p in SETTINGS + [("topk", V + 5 if V < 60 else 64, 1.0)]:
        u = so.uniform((1 << 32) + V, 5, np.arange(R, dtype=np.uint64))
        for r in range(R):
            fr = so.frame(x[r], mode, k, p, float(u[r]))
            want = int(_rule(x[r], mode, k, p, u[r], scan=V <= 3073)[0])
            assert fr.word == want, (kind, V, mode, k, p, r)
            assert fr.plausible[fr.word] and fr.union[fr.kept].all()
            assert np.isfinite(fr.score) and fr.score <= 0.0


def _suite():
    """(x rows, setting, uniforms) on which the exact comparison runs: bf16 logits + bias, quantised rows, flat rows."""
    gen = np.random.default_rng(2)
    out = []
    for V in (40, 1000, 3073):
        logits = so.bf16_round((gen.standard_normal((48, V)) * 3.0).astype(np.float32))
        bias = so.bf16_round((gen.standard_normal(V) * 0.5).astype(np.float32))
        out.append((logits, bias, V))
        out.append((so.bf16_round(np.round(gen.standard_normal((48, V)) * 2.0).astype(np.float32)), bias * 0, V))
        out.append((np.full((8, V), 0.5, dtype=np.float32), bias * 0, V))
    return out


def _mismatches(defect):
    seed, f = (1 << 32) + 3, 2
    bad = exact = 0
    for logits, bias, V in _suite():
        x = so.head_x(logits, bias, bf16=True)
        xm = so.head_x(logits, bias, bf16=defect != "bias_fp32")
        rows = np.arange(x.shape[0], dtype=np.uint64)
        u, um = _uniforms(seed, f, rows), _uniforms(seed, f, rows, defect)
        for mode, k, p in SETTINGS + [("topp", 64, 0.5), ("topk", 63, 1.0)]:
            for r in range(x.shape[0]):
                fr = so.frame(x[r], mode, k, p, float(u[r]))
                if fr.near:
                    continue
                exact += 1
                bad += int(_rule(xm[r], mode, k, p, um[r], defect)[0]) != fr.word
    return bad, exact


def test_the_brute_force_rule_is_the_oracle_on_the_defect_suite():
    assert _mismatches(None)[0] == 0


@pytest.mark.parametrize("defect", DEFECTS)
def test_exact_comparison_rejects_planted_defects(defect):
    bad, exact = _mismatches(defect)
    assert exact > 1000 and bad > 0, (defect, bad, exact)


# --- what the criteria of tests/test_sampling_gpu.py accept ------------------------------------------------------------------------
def _ranks(x):
    order = np.argsort(-x, kind="stable")
    ranks = np.empty(x.size, dtype=np.int64)
    ranks[order] = np.arange(x.size)
    return ranks, order


def _membership_accepts(defect):
    """test_draws_lie_in_the_top_k_set_and_nucleus on rows of its kind (fewer of them): ranks < k, mass before < p + 1e-5."""
    for V in (37, 1000):
        gen = torch.Generator().manual_seed(7 + V)
        logits = (torch.randn(64, V, generator=gen) * 3.0).bfloat16().float().numpy()
        bias = (torch.randn(1, V, generator=gen) * 0.5).bfloat16().float().numpy()[0]
        x = so.head_x(logits, bias, bf16=True)
        xm = so.head_x(logits, bias, bf16=defect != "bias_fp32")
        for seed in (1, 2):
            um = _uniforms(seed, 0, np.arange(64, dtype=np.uint64), defect)
            for r in range(64):
                ranks, order = _ranks(x[r].astype(np.float64))
                pr = np.exp(x[r] - x[r].max()).astype(np.float64)
                pr /= pr.sum()
                before = np.empty(V)
                before[order] = np.cumsum(pr[order]) - pr[order]
                for k in (2, 8, 64):
                    if ranks[int(_rule(xm[r], "topk", k, 1.0, um[r], defect)[0])] >= min(k, V):
                        return False
                for p in (0.3, 0.9, 1.0):
                    if before[int(_rule(xm[r], "topp", 64, p, um[r], defect)[0])] >= p + 1e-5:
                        return False
    return True


def _chi_square_accepts(defect, mode, k, p):
    """test_draws_follow_the_renormalised_distribution: 2^16 draws of one V = 1000 row, chi-square at ALPHA."""
    N, V = 1 << 16, 1000
    gen = torch.Generator().manual_seed(k * 100 + int(p * 10))
    row = torch.randn(V, generator=gen, dtype=torch.float64) * (1.0 if mode == "topk" else 2.0)
    x = row.float().numpy()
    ids = _rule(x, mode, k, p, _uniforms(2024, 0, np.arange(N, dtype=np.uint64), defect), defect)
    xd = x.astype(np.float64)
    ranks, order = _ranks(xd)
    pr = np.exp(xd - xd.max())
    pr /= pr.sum()
    before = np.empty(V)
    before[order] = np.cumsum(pr[order]) - pr[order]
    keep = ranks < k if mode == "topk" else before < p
    counts = np.bincount(ids, minlength=V).astype(np.float64)
    if counts[~keep].sum() != 0:
        return False
    exp = pr[keep] / pr[keep].sum() * N
    obs = counts[keep]
    small = exp < 5
    if small.any():
        exp = np.concatenate([exp[~small], [exp[small].sum()]])
        obs = np.concatenate([obs[~small], [obs[small].sum()]])
    return stats.chisquare(obs, exp * (obs.sum() / exp.sum())).pvalue > ALPHA


CHI_CASES = [("topk", 2, 1.0), ("topk", 8, 1.0), ("topk", 64, 1.0), ("topp", 1, 0.5), ("topp", 1, 0.9), ("topp", 1, 1.0)]
# the defects both criteria of tests/test_sampling_gpu.py accept on their own inputs: each keeps every draw in the kept set and leaves
# the distribution of one row alone (or changes it below what 2^16 draws resolve); only the exact comparison above rejects them
PASS_OLD = ["nucleus_gt", "rank_walk", "bias_fp32", "philox_swap", "u_from_y"]


@pytest.mark.parametrize("defect", PASS_OLD)
def test_the_set_and_chi_square_criteria_accept_these_defects(defect):
    assert _membership_accepts(defect)
    assert all(_chi_square_accepts(defect, *c) for c in CHI_CASES)


def test_the_criteria_accept_the_correct_rule():
    assert _membership_accepts(None)
    assert all(_chi_square_accepts(None, *c) for c in CHI_CASES)
