"""Duplicate-n-gram blocking in beam search (vlp_b200/beam.py, csrc/decode.cu; the reference's forbid_duplicate_ngrams,
modeling.py:1375-1428), host side: the reference golden (tools/ngram_beam_oracle.py) against the candidate rule, a step-by-step model of
the vlpk_beam_ngram_block kernel against the rule, the ABI's argument checks and the launches of a blocked decode under the dry-run."""
import os
import random

import pytest
import torch

from tools import abi_cases
from tools import ngram_beam_oracle as NBO
from vlp_b200 import _lib, synth
from vlp_b200 import beam
from vlp_b200 import vlp_modules as vm


def kernel_model(hist_in, ptr, wid, f, n, ignore, V):
    """vlpk_beam_ngram_block restated step by step (one CTA per row): history update, tail ignore test, match scan into a V-bit
    bitmap (duplicates collapse), then one write per set bit.  Returns (hist_out rows, {row: sorted blocked words})."""
    rows = len(wid)                                                 # ptr[i]: absolute parent row (b*K + back pointer)
    hist_out, blocked = [], {}
    for i in range(rows):
        seq = list(hist_in[ptr[i]][:f - 1]) if f > 1 else []
        seq.append(wid[i])
        hist_out.append(seq)
        if f < n:
            continue
        m = n - 1
        t0 = f - m
        if ignore and any(w in ignore for w in seq[(0 if m == 0 else t0):f]):
            continue
        bits = [0] * ((V + 31) // 32)
        for s in range(t0):
            if all(seq[s + j] == seq[t0 + j] for j in range(m)):
                w = seq[s + m]
                if 0 <= w < V and not (ignore and w in ignore):
                    bits[w >> 5] |= 1 << (w & 31)
        words = [j * 32 + b for j, x in enumerate(bits) for b in range(32) if x >> b & 1]
        if words:
            blocked[i] = words
    return hist_out, blocked


def _histories(case, T):
    """Per frame f (1..T-1) and row i = b*K + k: the history hist_f[i] (f words) the golden's traces imply."""
    B, K = case["B"], case["K"]
    wids, ptrs = case["wids"], case["ptrs"]
    hist = {1: [[int(wids[b, 0, k])] for b in range(B) for k in range(K)]}
    for f in range(2, T):
        hist[f] = [hist[f - 1][b * K + int(ptrs[b, f - 1, k])] + [int(wids[b, f - 1, k])] for b in range(B) for k in range(K)]
    return hist


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, "ngram_beam.pt"))


@pytest.mark.parametrize("name", list(NBO.CASES))
def test_golden_traces_follow_the_rule(golden, name):
    """Every hypothesis of the reference's traces, rebuilt from wids / ptrs: the words the reference blocked at each frame are exactly
    the candidate sets of beam._dup_ngram_candidates (and of the kernel model), and no chosen word extends its parent with a blocked
    word (there is always another finite choice: V = 1000 > K)."""
    case = golden["cases"][name]
    n, K, B = case["ngram_size"], case["K"], case["B"]
    ignore = set(case["ignore"]) if case["ignore"] else None
    T = NBO.n_frames(name)
    hist = _histories(case, T)
    want = {}
    for f, i, w in case["blocked"].tolist():
        want.setdefault((f, i), []).append(w)
    got = {}
    for f in range(n, T):
        for i, seq in enumerate(hist[f]):
            c = beam._dup_ngram_candidates(seq, n, ignore)
            if c:
                got[(f, i)] = c
    assert got == {k: sorted(v) for k, v in want.items()}
    assert len(got) == case["blocked_pairs"] > 0
    for f in range(max(n, 1), T):                  # kernel model on the golden's own histories
        ptr = [b * K + int(case["ptrs"][b, f - 1, k]) for b in range(B) for k in range(K)]
        wid = [int(case["wids"][b, f - 1, k]) for b in range(B) for k in range(K)]
        prev = hist[f - 1] if f > 1 else [[]] * (B * K)
        h, blk = kernel_model(prev, ptr, wid, f, n, ignore, 1000)
        assert h == hist[f]
        assert blk == {i: got[(f, i)] for (ff, i) in got if ff == f}
    for f in range(n, T):
        for b in range(B):
            for k in range(K):
                parent = b * K + int(case["ptrs"][b, f, k])
                assert int(case["wids"][b, f, k]) not in got.get((f, parent), []), (name, f, b, k)


@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_kernel_model_equals_the_rule_on_random_histories(n):
    """The kernel's history update + dedup'd candidate write equals beam._dup_ngram_candidates on random histories: small alphabets
    and constant runs (dense matches), ignore sets that hit tails and completions, lengths up to 409 (L = 512)."""
    rng = random.Random(n)
    V = 50
    for trial in range(60):
        f = rng.choice([1, 2, 3, n, n + 1, 20, 31, 32, 33, 64, 409])
        rows = rng.choice([1, 3, 6])
        alphabet = rng.choice([2, 3, 5, V + 3])                    # V + 3: some ids fall outside [0, V) and are never blocked
        prev = []
        for _ in range(rows):
            seq = [rng.randrange(alphabet) for _ in range(f - 1)]
            if f > 8 and rng.random() < 0.3:
                a = rng.randrange(f - 1)
                seq[a:] = [seq[a]] * (f - 1 - a)                    # a long constant run
            prev.append(seq)
        ptr = [rng.randrange(rows) for _ in range(rows)]
        wid = [rng.randrange(alphabet) for _ in range(rows)]
        ignore = rng.choice([None, {0}, set(range(1, V, 3)), {rng.randrange(alphabet)}])
        h, blk = kernel_model(prev, ptr, wid, f, n, ignore, V)
        for i in range(rows):
            assert h[i] == prev[ptr[i]][:f - 1] + [wid[i]]
            want = [w for w in beam._dup_ngram_candidates(h[i], n, ignore) if 0 <= w < V]
            assert blk.get(i, []) == want, (trial, i, h[i], n, ignore)


def test_rule_keeps_the_reference_reading_of_n_equal_1():
    """n = 1: the reference compares no words (every position matches) and its ignore test covers the whole sequence."""
    assert beam._dup_ngram_candidates([4, 2, 4], 1, None) == [2, 4]
    assert beam._dup_ngram_candidates([4, 2, 4], 1, {2}) == []
    assert beam._dup_ngram_candidates([4, 2, 4], 1, {7}) == [2, 4]


def test_abi_rejects_bad_arguments_without_launching():
    lib = _lib.lib()
    P = 4096                                                        # never dereferenced: every call below fails validation first
    good = dict(rows=6, K=3, f=4, T_cap=21, n=3, hist_in=P, hist_out=2 * P, ptr=P, wid=P, ignore=None, n_ignore=0, logp=P, ld=1000,
                V=1000, stream=None)
    order = list(good)

    def call(**kw):
        a = dict(good, **kw)
        return lib.vlpk_beam_ngram_block(*[a[k] for k in order])

    for bad in (dict(n=0), dict(n=-2), dict(f=0), dict(f=22), dict(ld=999), dict(hist_in=2 * P), dict(hist_out=None), dict(wid=None),
                dict(ptr=None), dict(hist_in=None), dict(logp=None), dict(n_ignore=2), dict(n_ignore=-1), dict(rows=7), dict(K=0),
                dict(V=0), dict(V=400000, ld=400000)):
        assert call(**bad) < 0, bad
        assert _lib.lib().vlpk_last_error()
    before = lib.vlpk_launch_count()
    assert call(rows=0) == 0                                        # nothing to do: accepted, no launch
    assert lib.vlpk_launch_count() == before


def _tiny_decoder(K, **kw):
    d = synth.TINY
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, search_beam_size=K, enable_butd=True, len_vis_input=d.regions,
                                     **kw).bfloat16().eval()
    B, R, L = 2, d.regions, d.seq_len
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    args = (torch.randn(B, R, d.vis_dim).bfloat16(), torch.randn(B, R, d.pe_dim).bfloat16(), input_ids, tt, pos, mask)
    return model, args, L - R - 2


@pytest.mark.parametrize("n", [1, 3])
def test_blocked_beam_decode_marshalling_dry_run(n):
    """A blocked beam decode marshals one vlpk_beam_ngram_block per frame f >= 1, whatever n is: every call carries the histories one
    frame forward, and the calls at f >= n also block.  No other call changes; unblocked, the decode marshals no such call."""
    model, args, frames = _tiny_decoder(3, ngram_size=n, forbid_ignore_set={7, 9})
    with abi_cases.dry_run() as plain:
        model(*args, task_idx=None)
    assert "vlpk_beam_ngram_block" not in plain
    model.forbid_duplicate_ngrams = True
    with abi_cases.dry_run() as calls:
        tr = model(*args, task_idx=None)
    assert tr["wids"].shape[2] == 3
    assert calls.count("vlpk_beam_ngram_block") == frames - 1
    assert [c for c in calls if c != "vlpk_beam_ngram_block"] == plain
    assert list(model._ngram_ignore_cache) == [((7, 9), "cpu")]
    model.forbid_ignore_set = {5}                                   # another set gets its own entry; the first one stays alive
    with abi_cases.dry_run():
        model(*args, task_idx=None)
    assert list(model._ngram_ignore_cache) == [((7, 9), "cpu"), ((5,), "cpu")]


def test_ngram_size_below_one_raises_before_any_launch():
    model, args, _ = _tiny_decoder(3, forbid_duplicate_ngrams=True, ngram_size=0)
    with abi_cases.dry_run() as calls, pytest.raises(ValueError, match="ngram_size"):
        model(*args, task_idx=None)
    assert calls == []


def test_ops_wrapper_rejects_host_tensors_and_wrong_ignore_dtype():
    from vlp_b200 import ops
    B, K, T = 2, 3, 8
    h_in, h_out = torch.zeros(B * K, T, dtype=torch.int32), torch.zeros(B * K, T, dtype=torch.int32)
    ptr, wid, logp = torch.zeros(B, K, dtype=torch.int64), torch.zeros(B, K, dtype=torch.int64), torch.zeros(B * K, 1, 50)
    with pytest.raises(RuntimeError, match="CUDA"):                 # host memory is never handed to the kernel
        ops.beam_ngram_block(h_in, h_out, ptr, wid, 3, 3, None, logp)
    with abi_cases.dry_run() as calls:                              # (device checks off) the ignore set must be int32 ids
        with pytest.raises(RuntimeError, match="int32"):
            ops.beam_ngram_block(h_in, h_out, ptr, wid, 3, 3, torch.tensor([4, 5]), logp)
        ops.beam_ngram_block(h_in, h_out, ptr, wid, 3, 3, torch.tensor([4, 5], dtype=torch.int32), logp)
    assert calls == ["vlpk_beam_ngram_block"]
