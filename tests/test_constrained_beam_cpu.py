"""CPU: constrained beam search (`constraints`): the two-stage selection rule against the full-vocabulary statement, hand-worked
destinations, the C ABI's and the ops wrapper's refusals, the refused settings in check_decode, the model and on the command line,
and the dry-run call sequences, with and without constraints."""
import argparse

import numpy as np
import pytest
import torch

from tools import abi_cases
from tools import constrained_beam_oracle as O
from vlp_b200 import _lib, beam, decode, decode_args, ops

from test_diverse_beam_cpu import _tiny_decoder


# ---------------------------------------------------------------------------------------------------------------------------
# the rule
# ---------------------------------------------------------------------------------------------------------------------------
def test_dest_by_hand():
    cons = np.zeros((3, 2, 3), np.int64)
    cons[0, 0, :2] = (5, 6)             # constraint 0: "5 6" or "9"
    cons[0, 1, :1] = 9
    cons[1, 0, :1] = 6                  # constraint 1: "6"
    # constraint 2 has no alternative: met from the start
    assert O.root_state(cons) == 0b100
    assert O.dest([], 6, cons, 0b100) == 0b110                  # "6" alone meets constraint 1, not the phrase "5 6"
    assert O.dest([5], 6, cons, 0b100) == 0b111                 # one word completes two constraints at once
    assert O.dest([5, 7], 6, cons, 0b100) == 0b110              # the phrase must be contiguous
    assert O.dest([1, 2], 9, cons, 0b100) == 0b101
    assert O.dest([5], 7, cons, 0b100) == 0b100
    assert O.dest([5], 6, cons, 0b111) == 0b111                 # met constraints stay met
    assert O.completions([5], cons, 0b100) == {6: 0b111, 9: 0b101}
    assert O.completions([5], cons, 0b110) == {6: 0b111, 9: 0b111}
    assert O.completions([5], cons, 0b111) == {}
    assert O.alternatives(cons) == [((5, 6), (9,)), ((6,),), ()]


def _random_frame(rng, B, K, C, first, V=40):
    """Random constraints (phrases, alternatives, overlaps, empty constraints), histories that end in phrase prefixes, logp and traces
    with empty slots."""
    A, P = 3, 3
    S = 1 << C
    cons = np.zeros((B, C, A, P), np.int64)
    for b in range(B):
        for j in range(C):
            for q in range(rng.integers(0 if j == C - 1 and b == 0 else 1, A + 1)):
                L = rng.integers(1, P + 1)
                cons[b, j, q, :L] = rng.integers(1, 12, L)         # a small alphabet: alternatives overlap and share last words
    rows = B if first else B * S * K
    lp = rng.standard_normal((rows, V)).astype(np.float32) * 2
    lp[:, :12] += 2
    lp = (lp - np.log(np.exp(lp).sum(1, keepdims=True))).astype(np.float32)
    hists, prev_score, prev_eos = None, None, None
    if not first:
        hists = [list(rng.integers(1, 12, 3)) for _ in range(rows)]
        for i, h in enumerate(hists):                              # a phrase prefix at the end of some histories
            alt = cons[i // (S * K), rng.integers(C), 0]
            n = int((alt != 0).sum())
            if n > 1 and rng.random() < 0.5:
                h[-(n - 1):] = list(alt[:n - 1])
        prev_score = (-rng.random((B, S * K)) * 5).astype(np.float32)
        prev_score[rng.random((B, S * K)) < 0.3] = -np.inf        # empty slots
        prev_eos = (rng.random((B, S * K)) < 0.1).astype(np.float32)
    return lp, hists, prev_score, prev_eos, cons


def test_two_stage_rule_equals_the_full_vocabulary_rule():
    rng = np.random.default_rng(0)
    frames = 0
    for C in (1, 2, 3):
        for K in (1, 2, 4):
            for first in (True, False):
                for _ in range(6):
                    lp, hists, ps, pe, cons = _random_frame(rng, 2, K, C, first)
                    a = O.two_stage(lp, hists, ps, pe, cons, K, first, np.float64)
                    b = O.full_vocab(lp, hists, ps, pe, cons, K, first, np.float64)
                    for x, y in zip(a[:3], b[:3]):
                        np.testing.assert_array_equal(x, y)
                    frames += 1
    assert frames == 108


def test_states_keep_their_own_parents_and_empty_slots():
    rng = np.random.default_rng(1)
    for _ in range(20):
        K, C = 3, 2
        lp, hists, ps, pe, cons = _random_frame(rng, 2, K, C, False)
        wid, ptr, score, _ = O.two_stage(lp, hists, ps, pe, cons, K, False)
        for b in range(2):
            for slot in range(4 * K):
                if np.isfinite(score[b, slot]):                    # a state's parents lie in its subsets
                    s, sp = slot // K, ptr[b, slot] // K
                    assert sp & s == sp and np.isfinite(ps[b, ptr[b, slot]])
                else:
                    assert wid[b, slot] == 0 and ptr[b, slot] == 0
    lp, _, _, _, cons = _random_frame(rng, 1, 2, 2, True)          # frame 0: only the root state and one-word completions
    _, _, score, _ = O.two_stage(lp, None, None, None, cons, 2, True)
    root = O.root_state(cons[0])
    assert np.isfinite(score[0, 2 * root:2 * root + 2]).all()
    assert all(s & root == root for s in range(4) if np.isfinite(score[0, 2 * s]))


def test_live_slot_rule_in_the_final_selection():
    """candidate_values / best_path / nbest with beams: empty slots never end a state's search nor become candidates; without beams the
    rule is today's."""
    T, B, K = 4, 1, 2
    ninf = -float("inf")
    sc = torch.tensor([[[-1.0, -2.0, -1.5, ninf]], [[-2.0, -3.0, -2.5, ninf]], [[-3.0, -4.0, -3.5, -3.6]], [[-4.0, -5.0, -4.5, -4.6]]])
    wi = torch.tensor([[[4, 5, 6, 0]], [[7, 8, 9, 0]], [[3, 4, 3, 3]], [[1, 1, 1, 1]]])
    pt = torch.tensor([[[0, 0, 0, 0]], [[0, 1, 2, 0]], [[0, 1, 2, 2]], [[0, 1, 2, 3]]])
    eos = 3
    # state 1 (slots 2, 3): frame 0 has one live slot; frame 2 has both slots [EOS], which ends its search there
    v = beam.candidate_values(sc[:, :, 2:], wi[:, :, 2:], eos, 0.0, live=True)
    assert torch.isfinite(v).sum() == 2 and v.max() == -3.5
    active, pos = beam.best_path(sc, wi, pt, eos, 0.0, beams=slice(2, 4))
    assert pos[:3, 0].tolist() == [2, 2, 2] and active[:, 0].tolist() == [True, True, True, False]
    seq, val = beam.nbest(sc, wi, pt, eos, 0.0, 6, 2, beams=slice(2, 4))
    assert torch.equal(val[0], torch.tensor([-3.5, -3.6])) and seq[0, 1, :3].tolist() == [6, 9, 3]
    for f in (beam.candidate_values,):                            # the default is today's rule, bit for bit
        assert torch.equal(f(sc[:, :, :2], wi[:, :, :2], eos, 1.0), f(sc[:, :, :2], wi[:, :, :2], eos, 1.0, live=False))
    assert torch.equal(beam.state_choice(torch.tensor([[-1.0, -2.0, ninf, -9.0], [-1.0, -2.0, -3.0, ninf], [-1.0, ninf, ninf, ninf],
                                                       [-5.0, -2.0, -2.0, ninf]])), torch.tensor([3, 1, 0, 1]))


def test_host_selection_agrees_with_the_torch_selection():
    rng = np.random.default_rng(2)
    T, B, K, C = 5, 3, 2, 2
    sc = np.cumsum(-rng.random((T, B, 4 * K)), 0).astype(np.float32)
    sc[rng.random(sc.shape) < 0.3] = -np.inf
    wi = rng.integers(1, 6, (T, B, 4 * K))
    pt = rng.integers(0, 4 * K, (T, B, 4 * K))
    pt[0] = 0
    pred, state_seq, state_val, met = O.select(sc, wi, pt, 3, 0.5, K, C)
    t = lambda a: torch.from_numpy(np.asarray(a))
    for s in range(4):
        active, pos = beam.best_path(t(sc), t(wi), t(pt), 3, 0.5, beams=slice(s * K, (s + 1) * K))
        assert torch.equal(beam._path_tokens(t(wi), active, pos, T), t(state_seq[:, s]))
    vals = torch.stack([beam.candidate_values(t(sc[:, :, s * K:(s + 1) * K]), t(wi[:, :, s * K:(s + 1) * K]), 3, 0.5, live=True)
                        .max(1).values for s in range(4)], 1)
    assert torch.equal(vals, t(state_val).float())
    assert torch.equal(t(state_seq)[torch.arange(B), beam.state_choice(vals)], t(pred))


# ---------------------------------------------------------------------------------------------------------------------------
# C ABI and ops
# ---------------------------------------------------------------------------------------------------------------------------
_A = 1 << 16


def _abi_call(**over):
    a = dict(B=2, K=6, C=2, A=2, P=3, f=2, V=1000, logits=_A, ld=1000, bias=None, fp32=0, eos_id=102, block_eos=0, T_cap=20, n=3,
             hist_in=2 * _A, hist_out=3 * _A, ignore=None, n_ignore=0, cons=14 * _A, prev_wid=4 * _A, prev_ptr=5 * _A, prev_score=6 * _A,
             prev_eos=7 * _A, top_w=8 * _A, top_lp=9 * _A, top_dest=15 * _A, wid=10 * _A, ptr=11 * _A, score=12 * _A, eos=13 * _A)
    a.update(over)
    s = abi_cases.constrained_beam_args(**a)
    return _lib.lib().vlpk_constrained_beam_step(_lib.C.byref(s), None)


BAD_ABI = [dict(C=0), dict(C=5), dict(A=0), dict(A=5), dict(P=0), dict(P=9), dict(K=0), dict(K=65, C=1), dict(K=17, C=4),
           dict(K=33, C=3), dict(B=-1), dict(V=9), dict(ld=999), dict(fp32=2), dict(f=20), dict(f=-1), dict(T_cap=0), dict(n=-1),
           dict(n_ignore=2), dict(logits=None), dict(cons=None), dict(top_w=None), dict(top_lp=None), dict(top_dest=None), dict(wid=None),
           dict(ptr=None), dict(score=None), dict(eos=None), dict(prev_score=None), dict(prev_eos=None), dict(prev_wid=None),
           dict(hist_out=None), dict(hist_in=None), dict(prev_ptr=None), dict(hist_in=3 * _A), dict(V=60000, ld=60000),
           dict(T_cap=60000, f=3), dict(n=0, hist_out=None)]


def test_abi_refuses_bad_arguments_without_launching():
    lib = _lib.lib()
    assert "vlpk_constrained_beam_step" in _lib.EXPORTED_SYMBOLS
    before = lib.vlpk_launch_count()
    for bad in BAD_ABI:
        assert _abi_call(**bad) < 0, bad
        assert lib.vlpk_last_error()
    assert lib.vlpk_constrained_beam_step(None, None) < 0
    for ok in (dict(K=16, C=4, A=4, P=8), dict(K=64, C=1, A=4), dict(K=64, C=2, A=4), dict(K=32, C=3)):
        assert _abi_call(B=0, **ok) == 0                            # the stated limits: accepted (nothing to do, no launch)
    assert _abi_call(B=0, f=0, prev_score=None, prev_eos=None, prev_wid=None, prev_ptr=None, hist_in=None, hist_out=None) == 0
    assert _abi_call(B=0, f=1, hist_in=None, prev_ptr=None) == 0
    assert lib.vlpk_launch_count() == before


def _op_tensors(B=2, K=2, C=2, A=2, P=3, T=5, V=50):
    SK = K << C
    return dict(logits=torch.zeros(B * SK, 1, V, dtype=torch.bfloat16), bias=torch.zeros(V, dtype=torch.bfloat16),
                cons=torch.zeros(B, C, A, P, dtype=torch.int64), wid=torch.zeros(T, B, SK, dtype=torch.int64),
                ptr=torch.zeros(T, B, SK, dtype=torch.int64), score=torch.zeros(T, B, SK), eos=torch.zeros(T, B, SK),
                top_w=torch.zeros(B * SK, K + C * A, dtype=torch.int32), top_lp=torch.zeros(B * SK, K + C * A),
                top_dest=torch.zeros(B * SK, C * A, dtype=torch.int32),
                hist=[torch.zeros(B * SK, T, dtype=torch.int32) for _ in range(2)])


def _op(t, f, **over):
    t = {**t, **over}
    return ops.constrained_beam_step(t["logits"], t["bias"], f, t["cons"], t["wid"], t["ptr"], t["score"], t["eos"], t["top_w"],
                                     t["top_lp"], t["top_dest"], 102, hist_in=t["hist"][0], hist_out=t["hist"][1],
                                     ngram=t.get("ngram", 0), ignore=t.get("ignore"))


def test_ops_wrapper_checks_tensors():
    t = _op_tensors()
    with pytest.raises(RuntimeError, match="CUDA"):
        _op(t, 1)
    with abi_cases.dry_run() as calls:
        with pytest.raises(RuntimeError, match="traces"):
            _op(t, 1, ptr=t["ptr"].int())
        with pytest.raises(RuntimeError, match="constraint table"):
            _op(t, 1, cons=t["cons"].int())
        with pytest.raises(RuntimeError, match="does not match"):
            _op(t, 1, cons=torch.zeros(2, 4, 2, 3, dtype=torch.int64))
        with pytest.raises(RuntimeError, match="rows = B at frame 0"):
            _op(t, 0)
        with pytest.raises(RuntimeError, match="bias"):
            _op(t, 1, bias=t["bias"].float())
        with pytest.raises(RuntimeError, match="scratch"):
            _op(t, 1, top_dest=t["top_dest"][:, :2])
        with pytest.raises(RuntimeError, match="histories"):
            _op(t, 1, hist=[None, None])
        with pytest.raises(ValueError, match="frame"):
            _op(t, 5)
        _op(t, 1, ngram=2, ignore=torch.tensor([4], dtype=torch.int32))
        _op(t, 0, logits=t["logits"][:2], hist=[None, None])
    assert calls == ["vlpk_constrained_beam_step"] * 2


# ---------------------------------------------------------------------------------------------------------------------------
# refused settings: check_decode, model, forward and command line
# ---------------------------------------------------------------------------------------------------------------------------
CONS = [[[5, 6], 9], [7]]


def test_constraint_table():
    t = decode.constraint_table(CONS)
    assert t.shape == (1, 2, 2, 2) and t[0].tolist() == [[[5, 6], [9, 0]], [[7, 0], [0, 0]]]
    assert decode.constraint_table([[], [3]])[0, 0].eq(0).all()
    for bad in ([], "dog", [["dog"]], [5], [[[]]], [[True]], [[1.5]]):
        with pytest.raises(ValueError, match="vlp_b200"):
            decode.constraint_table(bad)


BAD = [dict(sampling_method="topk", topk=4), dict(sampling_method="topp", topp=0.9), dict(K=4, num_beam_groups=2),
       dict(K=4, num_return_sequences=5), dict(K=1, num_return_sequences=2)]


@pytest.mark.parametrize("bad", BAD, ids=lambda b: "-".join(f"{k}={v}" for k, v in b.items()))
def test_check_decode_and_constructor_refuse(bad):
    kw = dict(bad)
    K = kw.pop("K", 1)
    meth = kw.pop("sampling_method", "beam_search")
    with pytest.raises(ValueError, match="vlp_b200"):
        decode.check_decode(meth, kw.pop("topk", 1), kw.pop("topp", 1.0), K, constraints=True, **kw)
    with pytest.raises(ValueError, match="vlp_b200"):
        _tiny_decoder(K=bad.get("K", 1), constraints=CONS, **{k: v for k, v in bad.items() if k != "K"})


BAD_TABLES = [dict(C=5), dict(A=5), dict(P=9), dict(K=17, C=4), dict(K=65, C=1), dict(ids=(-1,)), dict(ids=(1000,)), dict(gap=True),
              dict(long=True), dict(dtype=torch.int32), dict(images=3)]


def _table(C=2, A=2, P=3, ids=(), gap=False, long=False, dtype=torch.int64, images=2, K=None):
    t = torch.zeros(images, C, A, P, dtype=torch.int64)
    t[:, :, 0, 0] = 7
    for i, w in enumerate(ids):
        t[0, 0, 1, i] = w
    if gap:
        t[0, 1, 1, 1] = 5
    if long:
        t[0, 1, 1, :] = 5
    return t.to(dtype)


@pytest.mark.parametrize("bad", BAD_TABLES, ids=lambda b: "-".join(f"{k}={v}" for k, v in b.items()))
def test_forward_refuses_before_any_launch(bad):
    K = bad.get("K", 2)
    model, args, frames = _tiny_decoder(K=K)
    P = frames + 1 if bad.get("long") else bad.get("P", 3)
    cons = _table(**{**bad, "P": P})
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="vlp_b200"):
            model(*args, constraints=cons)
    assert calls == []


@pytest.mark.parametrize("setting", ["nokv", "sampling", "groups"])
def test_forward_refuses_settings_that_do_not_combine(setting):
    model, args, _ = _tiny_decoder(K=4, constraints=CONS)
    if setting == "nokv":
        model.use_kv_cache = False
    elif setting == "sampling":
        model.sampling_method, model.search_beam_size, model.topk = "topk", 1, 3
    else:
        model.num_beam_groups = 2
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="vlp_b200"):
            model(*args)
    assert calls == []


def _parser():
    return decode_args.add_decode_args(argparse.ArgumentParser())


@pytest.mark.parametrize("argv", [["--constraints", "dog,|cat"], ["--constraints", "dog||cat"], ["--constraints", "a|b|c|d|e"],
                                  ["--constraints", "a,b,c,d,e"], ["--constraints", "dog", "--sampling_method", "topk", "--topk", "3"],
                                  ["--constraints", "dog", "--beam_size", "4", "--num_beam_groups", "2"]])
def test_cli_refuses(argv):
    with pytest.raises(SystemExit) as e:
        decode_args.parse_decode_args(_parser(), argv)
    assert e.value.code == 2


class _Tok:
    """A wordpiece tokenizer stand-in: 'frisbee' splits into two pieces."""
    vocab = {"dog": 11, "dogs": 12, "fr": 13, "##is": 14, "##bee": 15}

    def tokenize(self, text):
        return ["fr", "##is", "##bee"] if text == "frisbee" else [text]

    def convert_tokens_to_ids(self, toks):
        return [self.vocab[t] for t in toks]


def test_cli_passes_the_constraints_on():
    args = decode_args.parse_decode_args(_parser(), ["--beam_size", "3", "--constraints", "dog,dogs|frisbee"])
    assert args.constraints == [["dog", "dogs"], ["frisbee"]]
    with pytest.raises(ValueError, match="tokenizer"):
        decode_args.decoder_kwargs(args)
    kw = decode_args.decoder_kwargs(args, _Tok())
    assert kw["constraints"] == [[[11], [12]], [[13, 14, 15]]]
    model, _, _ = _tiny_decoder(K=kw.pop("search_beam_size"), **kw)
    assert model.constraints[0].tolist() == [[[11, 0, 0], [12, 0, 0]], [[13, 14, 15], [0, 0, 0]]]
    assert "constraints" not in decode_args.decoder_kwargs(decode_args.parse_decode_args(_parser(), ["--beam_size", "3"]))


# ---------------------------------------------------------------------------------------------------------------------------
# call sequences
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(K=3, constraints=CONS), dict(K=1, constraints=[[4]]),
                                dict(K=2, constraints=[[3], [4, [5, 6]], [7]], forbid_duplicate_ngrams=True, forbid_ignore_set={7},
                                     ngram_size=2, min_len=2),
                                dict(K=4, constraints=CONS, num_return_sequences=3, length_penalty=0.5)])
def test_constrained_decode_call_sequence(kw):
    model, args, frames = _tiny_decoder(**kw)
    cons = model.constraints
    model.constraints = None
    model.num_return_sequences = max(2, kw.get("num_return_sequences", 1)) if kw["K"] > 1 else 1
    with abi_cases.dry_run() as plain:
        model(*args)                                                    # beam search on the shared prefix cache, at K beams
    model.num_return_sequences = kw.get("num_return_sequences", 1)
    model.constraints = cons
    with abi_cases.dry_run() as calls:
        out = model(*args)
    assert calls.count("vlpk_constrained_beam_step") == frames
    assert "vlpk_beam_ngram_block" not in calls
    layer_calls = lambda cs: [c for c in cs if c not in ("vlpk_constrained_beam_step", "vlpk_beam_ngram_block")]
    if kw["K"] > 1:
        assert layer_calls(calls) == layer_calls(plain)                 # the same shared-cache encoder steps as n-best beam search
    B, out_len, K, S = args[2].shape[0], args[3].shape[1], kw["K"], 1 << cons.shape[1]
    keys = {"pred_seq", "scores", "wids", "ptrs", "constraints_met", "state_seq", "state_scores"}
    if kw.get("num_return_sequences", 1) > 1:
        keys |= {"nbest_seq", "nbest_scores"}
    assert set(out) == keys
    assert out["state_seq"].shape == (B, S, out_len) and out["state_scores"].shape == (B, S)
    assert out["constraints_met"].shape == (B,) and out["constraints_met"].dtype == torch.bool
    assert out["scores"].shape == (B, out_len, S * K)
    # a per-call table overrides the constructor's
    with abi_cases.dry_run() as calls:
        model(*args, constraints=torch.tensor([[[[9, 0]]]] * B))
    assert calls.count("vlpk_constrained_beam_step") == frames


def test_no_constraints_keeps_todays_beam_search():
    model, args, frames = _tiny_decoder(K=4, forbid_duplicate_ngrams=True, ngram_size=2)
    with abi_cases.dry_run() as before:
        out = model(*args)
    assert "vlpk_constrained_beam_step" not in before
    assert before.count("vlpk_beam_ngram_block") == frames - 1
    assert set(out) == {"pred_seq", "scores", "wids", "ptrs"}
    model.constraints = decode.constraint_table(CONS)
    model.constraints = None                                            # set and cleared: today's calls again
    with abi_cases.dry_run() as after:
        model(*args)
    assert after == before
