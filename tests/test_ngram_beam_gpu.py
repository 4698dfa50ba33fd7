"""GPU: duplicate-n-gram blocking in beam search (vlpk_beam_ngram_block, vlp_b200/beam.py; the reference's forbid_duplicate_ngrams,
modeling.py:1375-1428).
 (1) the kernel against beam._dup_ngram_candidates at 1-500 hypotheses, histories of 1-409 words, n = 1-4, ignore sets of 0 / 1 / 64
     words, V = 1000 / 28996 with NaN guard columns, word ids >= V and < 0 and back pointers outside [0, K): blocked entries are bitwise
     x + (-10000), everything else untouched (ids outside [0, V) are never blocked), hist_out is the parent's history plus the new word
     (-1 words for a bad parent), and a second run is bitwise identical;
 (2) blocked beam decodes, with and without the K/V caches, against the reference's traces (tests/golden/ngram_beam.pt), exact where
     the decisions agree; the same inputs unblocked decode differently; with min_len = 5 and without it (case c) both follow the
     reference, and the [EOS] fill changes the words;
 (3) a blocked decode captured by GraphedCall replays to the Python-driven traces, bitwise, for the captured and for new inputs;
 (4) under torch.use_deterministic_algorithms(True) two blocked decodes are identical."""
import os

import pytest
import torch

from tools import ngram_beam_oracle as NBO
from vlp_b200 import beam, graph, ops, synth
from vlp_b200 import vlp_modules as vm

from test_decode_gpu import MARGIN, _first_diff
from test_parity_gpu import TOL_HID, make_config, rel

pytestmark = pytest.mark.gpu
DEV = "cuda"


# ---------------------------------------------------------------------------------------------------------------------------------
# (1) the kernel
# ---------------------------------------------------------------------------------------------------------------------------------
def _histories(gen, rows, f, alphabet):
    h = torch.randint(0, alphabet, (rows, f), generator=gen, dtype=torch.int32)
    for r in range(0, rows, 4):                                      # long constant runs in every fourth row
        if f > 4:
            a = int(torch.randint(0, f - 1, (1,), generator=gen))
            h[r, a:] = h[r, a]
    return h


def _nan_pattern(shape):
    bits = torch.arange(shape[0] * shape[1], dtype=torch.int32).reshape(shape) % 4096 | 0x7FC00000
    return bits.view(torch.float32)


@pytest.mark.parametrize("V", [1000, 28996])
@pytest.mark.parametrize("n_ignore", [0, 1, 64])
def test_kernel_matches_the_rule(V, n_ignore):
    gen = torch.Generator().manual_seed(V + n_ignore)
    T_cap = 409
    ld = V + 37
    for (B, K) in ((1, 1), (100, 5)):
        rows = B * K
        for f in (1, 2, 3, 20, 31, 32, 33, 64, 409):
            for n in (1, 2, 3, 4):
                alphabet = 4 if (f + n) % 2 else 13
                ignore = [] if n_ignore == 0 else [int(torch.randint(0, alphabet, (1,), generator=gen))]    # one id that occurs
                ignore = sorted(set(ignore + torch.randint(0, V, (n_ignore - 1,), generator=gen).tolist())) if n_ignore > 1 else ignore
                ign_dev = torch.tensor(ignore, dtype=torch.int32, device=DEV) if ignore else None
                prev = torch.full((rows, T_cap), -7, dtype=torch.int32)
                if f > 1:
                    prev[:, :f - 1] = _histories(gen, rows, f - 1, alphabet)
                ptr = torch.randint(0, K, (B, K), generator=gen)
                wid = torch.randint(0, alphabet, (B, K), generator=gen)
                if B > 1:                                                  # device data the host cannot check
                    wid[1, :2] = torch.tensor([V, -3])                      # ids outside [0, V): kept in the history, never blocked
                    wid[2, 0] = V + 5
                    ptr[3, 0], ptr[4, 1] = K, -1                            # bad back pointers: a history of -1 words
                    if f > 3:
                        prev[5 * K:6 * K, :f - 1:3] = V + 2                # ids >= V and < 0 inside histories
                        prev[6 * K:7 * K, 1:f - 1:2] = -4
                x = torch.randn(rows, ld, generator=gen)
                x[:, V:] = _nan_pattern((rows, ld - V))
                ok = ((ptr >= 0) & (ptr < K)).reshape(-1)
                parent = (ptr.clamp(0, K - 1) + torch.arange(B).unsqueeze(1) * K).reshape(-1)
                want_h = torch.full((rows, T_cap), 12345, dtype=torch.int32)
                want_h[:, :f - 1] = torch.where(ok.unsqueeze(1), prev.index_select(0, parent)[:, :f - 1], -1)
                want_h[:, f - 1] = wid.reshape(-1).to(torch.int32)
                want = x.clone()
                if f >= n:
                    for i in range(rows):
                        c = [w for w in beam._dup_ngram_candidates(want_h[i, :f].tolist(), n, set(ignore) if ignore else None) if 0 <= w < V]
                        if c:
                            want[i, c] = want[i, c] + (-10000.0)
                outs = []
                for _ in range(2):
                    h_in, h_out = prev.to(DEV), torch.full((rows, T_cap), 12345, dtype=torch.int32, device=DEV)
                    lp = x.to(DEV)
                    ops.beam_ngram_block(h_in, h_out, ptr.to(DEV), wid.to(DEV), f, n, ign_dev, lp[:, :V])
                    outs.append((h_out.cpu(), lp.cpu()))
                for h, lp in outs:
                    assert torch.equal(h, want_h), (rows, f, n)
                    assert torch.equal(lp.view(torch.int32), want.view(torch.int32)), (rows, f, n, ignore)


# ---------------------------------------------------------------------------------------------------------------------------------
# (2) decode against the reference
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "ngram_beam.pt"))


def _decoder(dims, weights_seed, K, forbid=True, n=3, ignore=None, min_len=0, length_penalty=0.5, state_dict=None):
    model = vm.BertForSeq2SeqDecoder(make_config(dims), mask_word_id=103, eos_id=NBO.EOS_ID, search_beam_size=K, enable_butd=True,
                                     len_vis_input=dims.regions, length_penalty=length_penalty, forbid_duplicate_ngrams=forbid,
                                     forbid_ignore_set=set(ignore) if ignore else None, ngram_size=n, min_len=min_len)
    model.load_state_dict(state_dict if state_dict is not None else synth.make_state_dict(dims, weights_seed), strict=False)
    return model.cuda().bfloat16().eval()


def _dev(args):
    vis, pe, input_ids, tt, pos, mask = args
    return (vis.cuda().bfloat16(), pe.cuda().bfloat16(), input_ids.cuda(), tt.cuda(), pos.cuda(), mask.cuda())


def _case_decoder(name, case, forbid=True, min_len=None):
    """The case's decoder: its weights (with the case's [EOS] bias), n-gram settings and min_len (unless given)."""
    dims, sd, _ = NBO.case_inputs(name)
    return _decoder(dims, case["weights_seed"], case["K"], forbid=forbid, n=case["ngram_size"], ignore=case["ignore"],
                    min_len=case["min_len"] if min_len is None else min_len, length_penalty=case["length_penalty"], state_dict=sd)


def _check_traces(name, tr, ref, K, T, B):
    """Our traces vs the reference's: exact up to the first differing decision, which must sit at a near-tie among the reference's
    K + 1 best candidates of that frame (the K chosen and the best one left out), with our K hypothesis scores matching its K."""
    assert tr["pred_seq"].shape == ref["pred_seq"].shape
    for b in range(B):
        t = _first_diff(tr["wids"][b].cpu().reshape(1, -1), ref["wids"][b].reshape(1, -1))
        n_same = T if t is None else t // K
        assert n_same >= 1
        assert rel(tr["scores"][b, :n_same].float(), ref["scores"][b, :n_same]) < TOL_HID
        if t is None:
            assert torch.equal(tr["ptrs"][b].cpu(), ref["ptrs"][b]) and torch.equal(tr["pred_seq"][b].cpu(), ref["pred_seq"][b])
        else:
            fr = t // K
            assert torch.equal(tr["ptrs"][b, :fr].cpu(), ref["ptrs"][b, :fr])
            gs = ref["scores"][b, fr].sort(descending=True).values
            pool = ref["cand_scores"][b, fr]                                 # the K chosen + the best unchosen candidate
            gaps = (pool[:-1] - pool[1:]).abs()
            ours = tr["scores"][b, fr].float().cpu().sort(descending=True).values
            assert float(gaps.min()) < MARGIN and float((ours - gs).abs().max()) < 2 * MARGIN, \
                f"case {name} sample {b}: decisions differ at frame {fr} without a near-tie: reference {gs.tolist()} ours {ours.tolist()}"
            print(f"case {name} sample {b}: first differing word at frame {fr}; reference frame scores {gs.tolist()} (near-tie)")


@pytest.mark.parametrize("name", list(NBO.CASES))
def test_blocked_beam_search_matches_reference_traces(golden, name):
    case = golden["cases"][name]
    args = _dev(NBO.case_inputs(name)[2])
    outs = []
    for use_cache in (True, False):
        model = _case_decoder(name, case)
        model.use_kv_cache = use_cache
        outs.append(model(*args, task_idx=None))
    tr, tr_re = outs
    for k in ("pred_seq", "wids", "ptrs"):
        assert torch.equal(tr[k], tr_re[k]), k                               # K/V caches do not change a single decision
    _check_traces(name, tr, case, case["K"], NBO.n_frames(name), case["B"])


def test_min_len_fill_decides_words_like_the_reference(golden):
    """Case c: with min_len = 5 no beam takes [EOS] in frames 0-4; without it the beams do, in the reference's traces and in ours,
    and both runs follow the reference's.  The [EOS] fill comes after the blocking (modeling.py:1300-1303) and both are live."""
    name = "c"
    case = golden["cases"][name]
    args = _dev(NBO.case_inputs(name)[2])
    K, T, B, m = case["K"], NBO.n_frames(name), case["B"], case["min_len"]
    with_fill = _case_decoder(name, case)(*args, task_idx=None)
    free = _case_decoder(name, case, min_len=0)(*args, task_idx=None)
    assert not bool((with_fill["wids"][:, :m] == NBO.EOS_ID).any())
    assert bool((free["wids"][:, :m] == NBO.EOS_ID).any())
    _check_traces(name + " without min_len", free, case["no_min_len"], K, T, B)
    assert bool((case["wids"][:, :T] == NBO.EOS_ID).any())                 # [EOS] enters the histories after min_len ...
    assert case["blocked_pairs"] > 0                                        # ... and the blocking is live in the same run


def test_blocking_changes_the_traces(golden):
    """The path is live: unblocked, the same inputs decode differently in at least one case (and blocked decodes follow the golden)."""
    differs = []
    for name in NBO.CASES:
        case = golden["cases"][name]
        args = _dev(NBO.case_inputs(name)[2])
        on = _case_decoder(name, case)(*args, task_idx=None)
        off = _case_decoder(name, case, forbid=False)(*args, task_idx=None)
        differs.append(not torch.equal(on["wids"], off["wids"]))
    assert any(differs), differs


# ---------------------------------------------------------------------------------------------------------------------------------
# (3) graph capture, (4) deterministic mode
# ---------------------------------------------------------------------------------------------------------------------------------
def _small_args(seed):
    import test_decode_gpu as td
    return _dev(td._inputs(synth.SMALL_L123, 3, seed))


@pytest.mark.parametrize("n,ignore", [(3, None), (2, [7, 117])])
def test_graphed_blocked_decode_equals_python_driven_decode(n, ignore):
    model = _decoder(synth.SMALL_L123, NBO.WEIGHTS_SEED, 3, n=n, ignore=ignore)
    a0, a1 = _small_args(5), _small_args(6)
    g = graph.GraphedCall(lambda *a: model(*a, task_idx=None), a0)          # capture fails on any host synchronisation
    assert g.launches_per_replay > 100
    for a in (a1, a0):
        want = model(*a, task_idx=None)
        got = g(*a)
        for k in ("pred_seq", "wids", "ptrs", "scores"):
            assert torch.equal(got[k], want[k]), k
    unblocked = _decoder(synth.SMALL_L123, NBO.WEIGHTS_SEED, 3, forbid=False)(*a0, task_idx=None)
    assert not torch.equal(unblocked["wids"], g(*a0)["wids"])               # the captured graph blocks


def test_blocked_decodes_are_identical_in_deterministic_mode():
    before = torch.are_deterministic_algorithms_enabled()
    cublas = os.environ.get("CUBLAS_WORKSPACE_CONFIG")
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    torch.use_deterministic_algorithms(True)
    try:
        model = _decoder(synth.SMALL_L123, NBO.WEIGHTS_SEED, 3, n=2, ignore=[540])
        a = _small_args(7)
        r1, r2 = model(*a, task_idx=None), model(*a, task_idx=None)
        for k in ("pred_seq", "wids", "ptrs", "scores"):
            assert torch.equal(r1[k], r2[k]), k
    finally:
        torch.use_deterministic_algorithms(before)
        if cublas is None:
            os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
        else:
            os.environ["CUBLAS_WORKSPACE_CONFIG"] = cublas
