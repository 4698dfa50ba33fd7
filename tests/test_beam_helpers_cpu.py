"""Host-side pieces of the beam search (vlp_b200/beam.py, semantics of the reference's modeling.py:1390-1406, 1431-1472) that need
no GPU: the duplicate-n-gram candidate rule, integer back pointers and the back-tracking.  Expansion to the beams and re-ordering by
back pointers: test_decode_state_cpu.py."""
import torch

from vlp_b200 import beam


def test_dup_ngram_candidates_match_reference_rule():
    # trigram blocking: the last two words (7, 8) occurred before followed by 9 and by 4
    seq = [7, 8, 9, 1, 7, 8, 4, 7, 8]
    assert beam._dup_ngram_candidates(seq, 3, None) == [4, 9]
    assert beam._dup_ngram_candidates([1, 2], 3, None) == []
    assert beam._dup_ngram_candidates(seq, 3, {8}) == []          # tail contains an ignored word
    assert beam._dup_ngram_candidates(seq, 3, {9}) == [4]         # completion word ignored


def test_floor_division_back_pointers():
    """The reference's torch.div(k_ids, K) (modeling.py:1317) yields floats on torch >= 1.6; the rewrite must produce integer parents."""
    K = 4
    flat = torch.tensor([[0, 5, 7, 15]])
    back = torch.div(flat, K, rounding_mode="floor")
    assert back.dtype == torch.int64 and back.tolist() == [[0, 1, 1, 3]]


def _reference_backtrack(scores, wids_list, ptrs, eos_id, length_penalty):
    """The reference's host loop for one batch item (modeling.py:1431-1472), restated."""
    import math
    last = len(scores) - 1
    for i, w in enumerate(wids_list):
        if all(x == eos_id for x in w):
            last = i
            break
    best, frame, pos = -math.inf, -1, -1
    for fid in range(last + 1):
        for i, w in enumerate(wids_list[fid]):
            if w == eos_id or fid == last:
                s = scores[fid][i] + length_penalty * (fid + 1)
                if s > best:
                    best, frame, pos = s, fid, i
    if frame == -1:
        return [0]
    seq = [wids_list[frame][pos]]
    for fid in range(frame, 0, -1):
        pos = ptrs[fid][pos]
        seq.append(wids_list[fid - 1][pos])
    return seq[::-1]


def test_vectorised_backtracking_equals_the_reference_host_loop():
    import torch
    g = torch.Generator().manual_seed(0)
    EOS = 7
    for trial in range(40):
        T, B, K = int(torch.randint(1, 9, (1,), generator=g)), 5, int(torch.randint(1, 5, (1,), generator=g))
        wi = torch.randint(5, 12, (T, B, K), generator=g)              # [EOS] = 7 appears often
        if trial % 3 == 0:
            wi[T // 2, 1] = EOS                                        # an all-[EOS] frame stops the search early
        sc = torch.randn(T, B, K, generator=g).round(decimals=1)       # coarse values: ties are exercised (first maximum must win)
        pt = torch.randint(0, K, (T, B, K), generator=g)
        lp = float(torch.randint(0, 3, (1,), generator=g)) * 0.5
        got = beam.backtrack(sc, wi, pt, EOS, lp, 12)
        for b in range(B):
            want = _reference_backtrack(sc[:, b].tolist(), wi[:, b].tolist(), pt[:, b].tolist(), EOS, lp)
            assert got[b, :len(want)].tolist() == want and int(got[b, len(want):].abs().sum()) == 0, (trial, b)
