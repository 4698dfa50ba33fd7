"""Diverse beam search (`num_beam_groups`, `diversity_penalty`), host side: the two-stage selection rule (row top K, then the
groups' merge) against a full-vocabulary statement of the frame, the C ABI's argument checks, the refused model and command-line
combinations, the per-group final selection, and the call sequences under the dry-run."""
import argparse

import numpy as np
import pytest
import torch

from tools import abi_cases
from tools import diverse_beam_oracle as O
from vlp_b200 import _lib, beam, decode, decode_args, ops, synth
from vlp_b200 import vlp_modules as vm


# ---------------------------------------------------------------------------------------------------------------------------
# the selection rule: the row top K hold every pair a group can keep
# ---------------------------------------------------------------------------------------------------------------------------
def _random_frame(rng, K, G, lam, first):
    """Coarse logits (many exact ties), -10000 blocks, finished beams, min_len; returns (lp, prev_score, prev_eos)."""
    B = int(rng.integers(1, 3))
    V = int(rng.integers(K, K + 40))
    rows = B if first else B * K
    step = [0.25, 0.5, 1.0][int(rng.integers(3))]
    x = np.round(rng.normal(0, 2, (rows, V)) / step) * step
    if rng.random() < 0.3:
        x[:, : V // 2] = x[:, :1]                                       # a long run of equal logits
    blocked = rng.random((rows, V)) < [0.0, 0.05, 0.5][int(rng.integers(3))]
    eos = int(rng.integers(V))
    lp = O.frame_logp(x, blocked, block_eos=rng.random() < 0.3, eos_id=eos, dtype=np.float64)
    prev_score = np.round(rng.normal(-5, 3, (B, K)) * 4) / 4
    prev_eos = (rng.random((B, K)) < 0.3).astype(np.float64)
    return lp, prev_score, prev_eos


def test_two_stage_rule_equals_the_full_vocabulary_rule():
    rng = np.random.default_rng(7)
    cases = 0
    for K in (2, 3, 4, 6, 8, 12, 16, 32, 64):
        groups = [g for g in range(1, K + 1) if K % g == 0]
        for G in groups:
            for lam in (0.0, 0.3, 5.0):
                for first in (True, False):
                    if G == 1 and lam > 0:
                        continue
                    reps = 2 if K <= 16 else 1
                    for _ in range(reps):
                        lp, ps, pe = _random_frame(rng, K, G, lam, first)
                        got = O.two_stage(lp, ps, pe, K, G, lam, first, dtype=np.float64)
                        want = O.full_vocab(lp, ps, pe, K, G, lam, first)
                        for a, b in zip(got[:3], want[:3]):
                            np.testing.assert_array_equal(a, b, err_msg=f"K={K} G={G} lam={lam} first={first}")
                        cases += 1
    assert cases >= 200


def test_groups_keep_their_own_parents_and_a_large_penalty_keeps_words_apart():
    rng = np.random.default_rng(3)
    K, G = 6, 3
    lp, ps, pe = _random_frame(rng, K, G, 1000.0, False)
    pe[:] = 0
    wid, ptr, _, _ = O.two_stage(lp, ps, pe, K, G, 1000.0, False, dtype=np.float64)
    Kg = K // G
    for g in range(G):
        assert ((ptr[:, g * Kg:(g + 1) * Kg] >= g * Kg) & (ptr[:, g * Kg:(g + 1) * Kg] < (g + 1) * Kg)).all()
    for b in range(wid.shape[0]):
        for g in range(1, G):                                           # no earlier group's word, V is large enough for that
            assert not set(wid[b, g * Kg:(g + 1) * Kg]) & set(wid[b, :g * Kg])


def test_zero_penalty_groups_are_beam_search_at_kg():
    """lambda = 0 at frame 0: every group draws the same Kg best words of the image's row."""
    rng = np.random.default_rng(11)
    lp, ps, pe = _random_frame(rng, 6, 3, 0.0, True)
    wid, ptr, score, _ = O.two_stage(lp, ps, pe, 6, 3, 0.0, True, dtype=np.float64)
    np.testing.assert_array_equal(wid[:, 0:2], wid[:, 2:4])
    np.testing.assert_array_equal(wid[:, 0:2], wid[:, 4:6])
    assert (ptr == 0).all()


# ---------------------------------------------------------------------------------------------------------------------------
# per-group final selection
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("lp", [0.0, 1.0])
def test_group_best_back_tracks_each_groups_beams(lp):
    rng = torch.Generator().manual_seed(2)
    eos = 3
    for trial in range(30):
        T, B, G, Kg = 1 + trial % 7, 2, [2, 3][trial % 2], [1, 2, 3][trial % 3]
        K = G * Kg
        sc = torch.randint(-8, 1, (T, B, K), generator=rng).float() * 0.5
        wi = torch.where(torch.rand(T, B, K, generator=rng) < 0.3, torch.full((T, B, K), eos), torch.randint(4, 9, (T, B, K), generator=rng))
        pt = (torch.arange(K) // Kg * Kg).expand(T, B, K) + torch.randint(0, Kg, (T, B, K), generator=rng)
        pt[0] = 0
        seq, val = beam.group_best(sc, wi, pt, eos, lp, T + 3, G)
        assert seq.shape == (B, G, T + 3) and val.shape == (B, G)
        for g in range(G):
            s = slice(g * Kg, (g + 1) * Kg)
            want = beam.backtrack(sc[:, :, s], wi[:, :, s], (pt[:, :, s] - g * Kg).clamp(min=0), eos, lp, T + 3)
            assert torch.equal(seq[:, g], want)
            assert torch.equal(val[:, g], beam.candidate_values(sc[:, :, s], wi[:, :, s], eos, lp).max(1).values)


# ---------------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------------
_A = 1 << 16                                                   # fake, aligned device addresses: every call below fails validation


def _abi_call(**over):
    a = dict(B=2, K=6, G=3, f=2, V=1000, logits=_A, ld=1000, bias=None, fp32=0, lam=0.5, eos_id=102, block_eos=0, T_cap=20, n=3,
             hist_in=2 * _A, hist_out=3 * _A, ignore=None, n_ignore=0, prev_wid=4 * _A, prev_ptr=5 * _A, prev_score=6 * _A,
             prev_eos=7 * _A, top_w=8 * _A, top_lp=9 * _A, wid=10 * _A, ptr=11 * _A, score=12 * _A, eos=13 * _A, stream=None)
    a.update(over)
    return _lib.lib().vlpk_diverse_beam_step(*a.values())


BAD_ABI = [dict(K=0), dict(K=65, G=5), dict(K=128, G=2), dict(G=4), dict(G=0), dict(G=-3), dict(B=-1), dict(V=5), dict(ld=999),
           dict(fp32=2), dict(lam=-0.5), dict(lam=float("nan")), dict(lam=float("inf")), dict(f=20), dict(f=-1), dict(T_cap=0),
           dict(n=-1), dict(n_ignore=2), dict(logits=None), dict(top_w=None), dict(top_lp=None), dict(wid=None), dict(ptr=None),
           dict(score=None), dict(eos=None), dict(prev_score=None), dict(prev_eos=None), dict(hist_out=None), dict(prev_wid=None),
           dict(hist_in=None), dict(prev_ptr=None), dict(hist_in=3 * _A), dict(V=60000, ld=60000), dict(T_cap=60000, f=3)]


def test_abi_refuses_bad_arguments_without_launching():
    lib = _lib.lib()
    assert "vlpk_diverse_beam_step" in _lib.EXPORTED_SYMBOLS
    before = lib.vlpk_launch_count()
    for bad in BAD_ABI:
        assert _abi_call(**bad) < 0, bad
        assert lib.vlpk_last_error()
    assert _abi_call(B=0) == 0                                          # nothing to do: accepted, no launch
    assert _abi_call(B=0, f=0, prev_score=None, prev_eos=None, prev_wid=None, prev_ptr=None, hist_in=None, hist_out=None) == 0
    assert _abi_call(B=0, f=1, hist_in=None, prev_ptr=None) == 0        # frame 1 reads no earlier history
    assert _abi_call(B=0, n=0, hist_in=None, hist_out=None, prev_wid=None, prev_ptr=None) == 0
    assert lib.vlpk_launch_count() == before


def test_ops_wrapper_checks_tensors():
    B, K, T, V = 2, 4, 5, 50
    logits = torch.zeros(B * K, 1, V, dtype=torch.bfloat16)
    wi, pt = torch.zeros(T, B, K, dtype=torch.int64), torch.zeros(T, B, K, dtype=torch.int64)
    sc, eo = torch.zeros(T, B, K), torch.zeros(T, B, K)
    tw, tl = torch.zeros(B * K, K, dtype=torch.int32), torch.zeros(B * K, K)
    bias = torch.zeros(V, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="CUDA"):                     # host memory is never handed to the kernel
        ops.diverse_beam_step(logits, bias, 1, 2, 0.5, wi, pt, sc, eo, tw, tl, 102)
    with abi_cases.dry_run() as calls:
        with pytest.raises(RuntimeError, match="traces"):
            ops.diverse_beam_step(logits, bias, 1, 2, 0.5, wi, pt.int(), sc, eo, tw, tl, 102)
        with pytest.raises(RuntimeError, match="rows = B at frame 0"):
            ops.diverse_beam_step(logits, bias, 0, 2, 0.5, wi, pt, sc, eo, tw, tl, 102)
        with pytest.raises(RuntimeError, match="bias"):
            ops.diverse_beam_step(logits, bias.float(), 1, 2, 0.5, wi, pt, sc, eo, tw, tl, 102)
        with pytest.raises(RuntimeError, match="scratch"):
            ops.diverse_beam_step(logits, bias, 1, 2, 0.5, wi, pt, sc, eo, tw[:, :2], tl, 102)
        with pytest.raises(RuntimeError, match="histories"):
            ops.diverse_beam_step(logits, bias, 1, 2, 0.5, wi, pt, sc, eo, tw, tl, 102, ngram=2)
        with pytest.raises(ValueError, match="frame"):
            ops.diverse_beam_step(logits, bias, T, 2, 0.5, wi, pt, sc, eo, tw, tl, 102)
        hist = [torch.zeros(B * K, T, dtype=torch.int32) for _ in range(2)]
        ops.diverse_beam_step(logits, bias, 1, 2, 0.5, wi, pt, sc, eo, tw, tl, 102, ngram=2, ignore=torch.tensor([4], dtype=torch.int32),
                              hist_in=hist[0], hist_out=hist[1])
        ops.diverse_beam_step(logits[:B], None, 0, 2, 0.0, wi, pt, sc, eo, tw, tl, 102)
    assert calls == ["vlpk_diverse_beam_step"] * 2


# ---------------------------------------------------------------------------------------------------------------------------
# refused combinations: check_decode, model and command line
# ---------------------------------------------------------------------------------------------------------------------------
def _tiny_decoder(K=1, **kw):
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


BAD = [dict(K=4, num_beam_groups=0), dict(K=4, num_beam_groups=-2), dict(K=4, num_beam_groups=2.0), dict(K=4, num_beam_groups=True),
       dict(K=1, num_beam_groups=2, sampling_method="topk", topk=4), dict(K=1, num_beam_groups=2, sampling_method="topp", topp=0.9),
       dict(K=1, num_beam_groups=2), dict(K=6, num_beam_groups=4), dict(K=66, num_beam_groups=2), dict(K=128, num_beam_groups=64),
       dict(K=4, num_beam_groups=2, diversity_penalty=-0.1), dict(K=4, num_beam_groups=2, diversity_penalty=float("nan")),
       dict(K=4, num_beam_groups=2, diversity_penalty=float("inf")), dict(K=4, num_beam_groups=2, diversity_penalty="0.5"),
       dict(K=4, diversity_penalty=0.5), dict(K=1, diversity_penalty=1.0)]
_ID = lambda b: "-".join(f"{k}={v}" for k, v in b.items())


@pytest.mark.parametrize("bad", BAD, ids=_ID)
def test_check_decode_and_constructor_refuse(bad):
    kw = dict(bad)
    K = kw.pop("K")
    meth = kw.pop("sampling_method", "beam_search")
    with pytest.raises(ValueError, match="vlp_b200"):
        decode.check_decode(meth, kw.pop("topk", 1), kw.pop("topp", 1.0), K, **kw)
    with pytest.raises(ValueError, match="vlp_b200"):
        _tiny_decoder(**bad)


@pytest.mark.parametrize("bad", BAD, ids=_ID)
def test_forward_refuses_before_any_launch(bad):
    model, args, _ = _tiny_decoder(K=4, num_beam_groups=2, diversity_penalty=0.5)
    model.num_beam_groups, model.diversity_penalty = 1, 0.0
    for k, v in bad.items():
        setattr(model, "search_beam_size" if k == "K" else k, v)
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="vlp_b200"):
            model(*args)
    assert calls == []


def test_accepted_settings():
    for K, G, lam in ((2, 2, 0.0), (6, 3, 0.5), (64, 64, 2), (64, 2, 0.0), (5, 1, 0.0)):
        decode.check_decode("beam_search", 1, 1.0, K, num_beam_groups=G, diversity_penalty=lam)
    model, _, _ = _tiny_decoder(K=6, num_beam_groups=3, diversity_penalty=0.5)
    assert (model.num_beam_groups, model.diversity_penalty) == (3, 0.5)
    model, _, _ = _tiny_decoder(K=3)
    assert (model.num_beam_groups, model.diversity_penalty) == (1, 0.0)


def _parser():
    return decode_args.add_decode_args(argparse.ArgumentParser())


@pytest.mark.parametrize("argv", [["--num_beam_groups", "0", "--beam_size", "4"], ["--num_beam_groups", "2"],
                                  ["--num_beam_groups", "4", "--beam_size", "6"], ["--num_beam_groups", "2", "--beam_size", "66"],
                                  ["--num_beam_groups", "2", "--beam_size", "1", "--sampling_method", "topk", "--topk", "4"],
                                  ["--num_beam_groups", "2", "--beam_size", "4", "--diversity_penalty", "-1"],
                                  ["--num_beam_groups", "2", "--beam_size", "4", "--diversity_penalty", "nan"],
                                  ["--beam_size", "4", "--diversity_penalty", "0.5"]])
def test_cli_refuses(argv):
    with pytest.raises(SystemExit) as e:
        decode_args.parse_decode_args(_parser(), argv)
    assert e.value.code == 2
    with pytest.raises(ValueError, match="vlp_b200"):
        decode_args.check_decode_args(_parser().parse_args(argv))


def test_cli_passes_the_settings_on():
    kw = decode_args.decoder_kwargs(decode_args.parse_decode_args(_parser(), ["--beam_size", "6", "--num_beam_groups", "3",
                                                                               "--diversity_penalty", "0.5"]))
    assert (kw["search_beam_size"], kw["num_beam_groups"], kw["diversity_penalty"]) == (6, 3, 0.5)
    model, _, _ = _tiny_decoder(K=kw.pop("search_beam_size"), **kw)
    assert (model.num_beam_groups, model.diversity_penalty) == (3, 0.5)
    kw = decode_args.decoder_kwargs(decode_args.parse_decode_args(_parser(), ["--beam_size", "4", "--num_beam_groups", "2"]))
    assert kw["num_beam_groups"] == 2 and "diversity_penalty" not in kw
    kw = decode_args.decoder_kwargs(decode_args.parse_decode_args(_parser(), ["--beam_size", "4"]))
    assert "num_beam_groups" not in kw and "diversity_penalty" not in kw


# ---------------------------------------------------------------------------------------------------------------------------
# call sequences
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(K=4, num_beam_groups=2, diversity_penalty=0.5),
                                dict(K=6, num_beam_groups=3, diversity_penalty=1.0, forbid_duplicate_ngrams=True, forbid_ignore_set={7},
                                     ngram_size=2, min_len=2),
                                dict(K=6, num_beam_groups=2, num_return_sequences=3),
                                dict(K=4, num_beam_groups=4, diversity_penalty=0.3, forbid_duplicate_ngrams=True, ngram_size=1)])
def test_diverse_decode_call_sequence(kw):
    model, args, frames = _tiny_decoder(**kw)
    with abi_cases.dry_run() as plain:
        model.num_beam_groups, model.diversity_penalty = 1, 0.0
        model(*args)                                                    # today's beam search at the same K
    model.num_beam_groups, model.diversity_penalty = kw["num_beam_groups"], kw.get("diversity_penalty", 0.0)
    with abi_cases.dry_run() as calls:
        out = model(*args)
    assert calls.count("vlpk_diverse_beam_step") == frames
    assert "vlpk_beam_ngram_block" not in calls
    layer_calls = lambda cs: [c for c in cs if c not in ("vlpk_diverse_beam_step", "vlpk_beam_ngram_block")]
    assert layer_calls(calls) == layer_calls(plain)                     # the same encoder steps as beam search
    B, out_len, K, G = args[2].shape[0], args[3].shape[1], kw["K"], kw["num_beam_groups"]
    keys = {"pred_seq", "scores", "wids", "ptrs", "group_seq", "group_scores"}
    if kw.get("num_return_sequences", 1) > 1:
        keys |= {"nbest_seq", "nbest_scores"}
    assert set(out) == keys
    assert out["group_seq"].shape == (B, G, out_len) and out["group_seq"].dtype == torch.int64
    assert out["group_scores"].shape == (B, G) and out["group_scores"].dtype == torch.float32
    assert out["scores"].shape == (B, out_len, K)


def test_one_group_keeps_todays_beam_search():
    model, args, frames = _tiny_decoder(K=4, forbid_duplicate_ngrams=True, ngram_size=2)
    with abi_cases.dry_run() as calls:
        out = model(*args)
    assert "vlpk_diverse_beam_step" not in calls
    assert calls.count("vlpk_beam_ngram_block") == frames - 1
    assert "group_seq" not in out
