"""CPU: prompted captions (`prompt_ids`, `--prompt`): the refusals of the model and the command line, the column layout of the step-0
prefill against a host restatement of its rules, the prompt-seeded n-gram history against the rule on the whole caption, the
caption assembly, the dry-run call sequences with and without a prompt, and the oracle's inputs against the stored golden."""
import argparse
import os

import numpy as np
import pytest
import torch

from tools import abi_cases
from tools import prompt_decode_oracle as PO
from vlp_b200 import decode, decode_args
from vlp_b200.beam import _dup_ngram_candidates

from test_diverse_beam_cpu import _tiny_decoder

PROMPT = torch.tensor([[11, 12, 13], [21, 0, 0]])


# ---------------------------------------------------------------------------------------------------------------------------
# refusals
# ---------------------------------------------------------------------------------------------------------------------------
def _bad_prompt(kind, frames):
    return {"vocab": torch.tensor([[11, 1000]]), "negative": torch.tensor([[11, -3]]), "eos": torch.tensor([[11, 102]]),
            "mask": torch.tensor([[103, 0]]), "gap": torch.tensor([[11, 0, 12], [4, 5, 6]]), "rows": torch.ones(3, 2, dtype=torch.int64),
            "long": torch.ones(1, frames, dtype=torch.int64), "dtype": torch.tensor([[11.0, 12.0]]), "dim": torch.tensor([11, 12]),
            "list": [11, 12]}[kind]


@pytest.mark.parametrize("kind", ["vocab", "negative", "eos", "mask", "gap", "rows", "long", "dtype", "dim", "list"])
@pytest.mark.parametrize("K", [1, 3])
def test_forward_refuses_bad_prompts_before_any_launch(kind, K):
    model, args, frames = _tiny_decoder(K=K)
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="vlp_b200"):
            model(*args, prompt_ids=_bad_prompt(kind, frames))
    assert calls == []


@pytest.mark.parametrize("setting", ["nokv", "attentions"])
def test_forward_refuses_settings_that_do_not_take_a_prompt(setting):
    model, args, _ = _tiny_decoder(K=4)
    kw = {}
    if setting == "nokv":
        model.use_kv_cache = False
    else:
        kw["output_attentions"] = True
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="vlp_b200"):
            model(*args, prompt_ids=PROMPT, **kw)
    assert calls == []


def test_constructor_refuses():
    with pytest.raises(ValueError, match="list of word ids"):
        _tiny_decoder(K=2, prompt="a photo of")


def _parser():
    return decode_args.add_decode_args(argparse.ArgumentParser())


class _Tok:
    """A wordpiece tokenizer stand-in: 'close-up' splits into three pieces."""
    vocab = {"a": 31, "close": 32, "-": 33, "up": 34, "of": 35}

    def tokenize(self, text):
        return [p for w in text.split() for p in (["close", "-", "up"] if w == "close-up" else [w])]

    def convert_tokens_to_ids(self, toks):
        return [self.vocab[t] for t in toks]


def test_cli_parses_and_tokenizes_the_prompt():
    args = decode_args.parse_decode_args(_parser(), ["--beam_size", "3", "--prompt", "a close-up of"])
    assert args.prompt == "a close-up of"
    with pytest.raises(ValueError, match="tokenizer"):
        decode_args.decoder_kwargs(args)
    kw = decode_args.decoder_kwargs(args, _Tok())
    assert kw["prompt"] == [31, 32, 33, 34, 35]
    model, _, _ = _tiny_decoder(K=kw.pop("search_beam_size"), **kw)
    assert model.prompt.tolist() == [[31, 32, 33, 34, 35]]
    assert "prompt" not in decode_args.decoder_kwargs(decode_args.parse_decode_args(_parser(), ["--beam_size", "3"]))


@pytest.mark.parametrize("argv", [["--prompt", "a", "--sampling_method", "topk", "--topk", "3"],
                                  ["--prompt", "a", "--beam_size", "4", "--num_beam_groups", "2"],
                                  ["--prompt", "a", "--beam_size", "2", "--constraints", "dog"]])
def test_cli_takes_the_prompt_in_every_mode(argv):
    assert decode_args.parse_decode_args(_parser(), argv).prompt == "a"


# ---------------------------------------------------------------------------------------------------------------------------
# the constrained start state
# ---------------------------------------------------------------------------------------------------------------------------
def test_constrained_start_state_against_brute_force():
    """prompt_constraints zeroes exactly the constraints one of whose alternatives is a contiguous run of the image's prompt words."""
    from tools import constrained_beam_oracle as CO
    rng = np.random.default_rng(7)
    for trial in range(300):
        B, C, A, P, Tp = 3, int(rng.integers(1, 4)), int(rng.integers(1, 4)), int(rng.integers(1, 4)), int(rng.integers(1, 6))
        cons = torch.zeros(B, C, A, P, dtype=torch.int64)
        for b in range(B):
            for j in range(C):
                for q in range(int(rng.integers(0, A + 1))):
                    n = int(rng.integers(1, P + 1))
                    cons[b, j, q, :n] = torch.as_tensor(rng.integers(1, 5, n))
        prompt = torch.zeros(B, Tp, dtype=torch.int64)
        for b in range(B):
            t = int(rng.integers(0, Tp + 1))
            prompt[b, :t] = torch.as_tensor(rng.integers(1, 5, t))
        got = decode.prompt_constraints(cons, prompt)
        for b in range(B):
            words = [w for w in prompt[b].tolist() if w]
            for j, alts in enumerate(CO.alternatives(cons[b].numpy())):
                met = any(tuple(words[s:s + len(a)]) == a for a in alts for s in range(len(words) - len(a) + 1))
                assert torch.equal(got[b, j], torch.zeros_like(cons[b, j]) if met else cons[b, j]), (trial, b, j, words, alts)


# ---------------------------------------------------------------------------------------------------------------------------
# the layout
# ---------------------------------------------------------------------------------------------------------------------------
def _host_columns(t, Tp, in_len, out_len):
    """Host restatement of the gap layout for one image with t prompt words: (position of each column, gap flag of each column)."""
    pos, gap = [], []
    for c in range(out_len):
        if c < in_len + t:
            pos.append(c), gap.append(False)                          # prefix, then the prompt words at their own positions
        elif c < in_len + Tp:
            pos.append(c), gap.append(True)                           # the padding columns of a shorter prompt
        else:
            pos.append(c - (Tp - t)), gap.append(False)               # [MASK] and later words continue right after the prompt
    return pos, gap


def _inputs(B, in_len, out_len, seed=0):
    g = torch.Generator().manual_seed(seed)
    tt = torch.randint(0, 6, (B, out_len), generator=g)
    pos = torch.randint(0, 500, (B, out_len), generator=g)
    mask = torch.randint(0, 2, (B, out_len, out_len), generator=g)
    return tt, pos, mask


@pytest.mark.parametrize("lens", [(3, 0), (2, 2), (1, 3, 0, 2)])
def test_column_layout_against_host_rules(lens):
    in_len, out_len, Tp = 5, 14, max(lens)
    B = len(lens)
    prompt = torch.zeros(B, Tp, dtype=torch.int64)
    for b, t in enumerate(lens):
        prompt[b, :t] = torch.arange(1, t + 1) + 40
    tt, pos, mask = _inputs(B, in_len, out_len)
    dec = type("D", (), {"mask_word_id": 103, "use_kv_cache": False})()
    state = decode.DecodeState(dec, None, None, torch.ones(B, in_len, dtype=torch.int64), tt, pos, mask, prompt=prompt)
    assert state.frames == out_len - in_len - Tp and state.next_pos == in_len + Tp
    assert torch.equal(state.first_ids[:, in_len:], prompt)
    for b, t in enumerate(lens):
        hp, hg = _host_columns(t, Tp, in_len, out_len)
        assert state.position_ids[b].tolist() == [int(pos[b, p]) for p in hp]
        assert state.token_type_ids[b].tolist() == [int(tt[b, p]) for p in hp]
        for q in range(out_len):
            for k in range(out_len):
                want = 0 if hg[k] else int(mask[b, hp[q], hp[k]])
                assert int(state.attention_mask[b, q, k]) == want, (b, q, k)
        # the visible columns, in order, are positions 0, 1, 2, ...: what the reference's decode of the same words sees
        visible = [p for p, g in zip(hp, hg) if not g]
        assert visible == list(range(len(visible)))


def test_no_prompt_keeps_the_callers_tensors():
    tt, pos, mask = _inputs(2, 5, 12)
    dec = type("D", (), {"mask_word_id": 103, "use_kv_cache": False})()
    ids = torch.ones(2, 5, dtype=torch.int64)
    state = decode.DecodeState(dec, None, None, ids, tt, pos, mask)
    assert state.first_ids is ids and state.token_type_ids is tt and state.position_ids is pos and state.attention_mask is mask
    assert state.frames == 7 and state.prefix_len == 5


def test_with_prompt_places_the_prompt_before_the_words():
    seq = torch.tensor([[5, 6, 7, 0, 0, 0], [8, 9, 10, 0, 0, 0]])
    assert decode.with_prompt(PROMPT, seq).tolist() == [[11, 12, 13, 5, 6, 7], [21, 8, 9, 10, 0, 0]]
    sc = torch.tensor([[1.0, 2.0, 3.0, 0, 0, 0], [4.0, 5.0, 6.0, 0, 0, 0]])
    assert decode.with_prompt(PROMPT, sc, fill=0).tolist() == [[0, 0, 0, 1, 2, 3], [0, 4, 5, 6, 0, 0]]
    nb = torch.stack([seq, seq + 1], 1)                                  # [B, N, L]
    assert decode.with_prompt(PROMPT, nb)[1, 1].tolist() == [21, 9, 10, 11, 1, 1]


# ---------------------------------------------------------------------------------------------------------------------------
# the rules on the whole caption
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 2, 3, 4])
def test_prompt_history_blocks_the_ngrams_of_the_whole_caption(n):
    """The right-aligned history (Tp - t_b entries of -1, the prompt, then the generated words) gives, among real words, exactly
    the candidates of the reference's rule on prompt + continuation, for every t_b, continuation length and ignore set."""
    rng = np.random.default_rng(n)
    Tp = 5
    for trial in range(400):
        t = int(rng.integers(0, Tp + 1))
        prompt = torch.zeros(1, Tp, dtype=torch.int64)
        prompt[0, :t] = torch.as_tensor(rng.integers(1, 5, t))
        gen = [int(w) for w in rng.integers(1, 5, int(rng.integers(0, 6)))]
        ignore = {int(rng.integers(1, 5))} if trial % 3 == 0 else None
        hist = decode.prompt_history(prompt, 1, Tp + 8)[0, :Tp].tolist() + gen
        caption = prompt[0, :t].tolist() + gen
        got = [w for w in _dup_ngram_candidates(hist, n, ignore) if w >= 0]
        assert got == _dup_ngram_candidates(caption, n, ignore), (hist, caption)


def test_prompt_history_layout():
    h = decode.prompt_history(PROMPT, 2, 6)
    assert h.dtype == torch.int32 and h.shape == (4, 6)
    assert h[:, :3].tolist() == [[11, 12, 13]] * 2 + [[-1, -1, 21]] * 2


# ---------------------------------------------------------------------------------------------------------------------------
# call sequences
# ---------------------------------------------------------------------------------------------------------------------------
def _layer_calls(calls):
    return [c for c in calls if c != "vlpk_beam_ngram_block"]


@pytest.mark.parametrize("kw", [dict(K=1), dict(K=3, forbid_duplicate_ngrams=True, ngram_size=2, min_len=3),
                                dict(K=3, num_return_sequences=2, length_penalty=0.5)])
def test_prompted_decode_call_sequence(kw):
    model, args, frames = _tiny_decoder(**kw)
    B, out_len = args[2].shape[0], args[3].shape[1]
    with abi_cases.dry_run() as plain:
        before = model(*args)
    with abi_cases.dry_run() as empty:
        model(*args, prompt_ids=torch.zeros(B, 0, dtype=torch.int64))
    assert empty == plain                                                  # width 0: today's decode
    with abi_cases.dry_run() as calls:
        out = model(*args, prompt_ids=PROMPT)
    Tp = PROMPT.shape[1]
    if kw.get("forbid_duplicate_ngrams"):
        assert calls.count("vlpk_beam_ngram_block") == frames - Tp          # every frame, the first one included, sees the prompt
        assert plain.count("vlpk_beam_ngram_block") == frames - 1
    # Tp fewer frames, each with the layer calls of one of today's later frames (the prefill's calls are those of today's)
    per_frame = (len(_layer_calls(plain)) - len(_layer_calls(calls))) // Tp
    assert len(_layer_calls(calls)) == len(_layer_calls(plain)) - Tp * per_frame and per_frame > 0
    if kw["K"] == 1:
        ids, scores = out
        assert ids.shape == before[0].shape and scores.shape == before[1].shape
        assert ids[:, :1].tolist() == [[11], [21]] and ids[0, :3].tolist() == [11, 12, 13]
        assert float(scores[:, :1].abs().sum()) == 0.0
    else:
        assert set(out) == set(before) and all(out[k].shape == before[k].shape for k in out)
        assert out["pred_seq"].shape == (B, out_len)
        assert out["pred_seq"][0, :3].tolist() == [11, 12, 13] and out["pred_seq"][1, 0] == 21
        assert bool((out["scores"][:, frames - Tp:] == 0).all())            # traces index the frames actually run
        if "nbest_seq" in out:
            assert out["nbest_seq"][:, :, 0].tolist() == [[11, 11], [21, 21]]


def test_shared_prompt_from_the_constructor_and_override():
    model, args, _ = _tiny_decoder(K=1, prompt=[31, 32])
    with abi_cases.dry_run():
        ids, _ = model(*args)
        assert ids[:, :2].tolist() == [[31, 32], [31, 32]]
        ids, _ = model(*args, prompt_ids=torch.tensor([[41]]))
        assert ids[:, :1].tolist() == [[41], [41]]


# ---------------------------------------------------------------------------------------------------------------------------
# the oracle
# ---------------------------------------------------------------------------------------------------------------------------
def test_oracle_inputs_match_the_golden(golden_dir):
    gold = torch.load(os.path.join(golden_dir, "prompt_decode.pt"))
    assert set(gold["cases"]) == set(PO.CASES)
    for name, case in gold["cases"].items():
        dims, mode, B, t, seed, relaxed = PO.CASES[name]
        _, _, _, prompt, task_idx = PO.case_inputs(name)
        assert torch.equal(case["prompt"], prompt) and case["t"] == t and case["mode"] == mode and case["relaxed"] == relaxed
        assert bool(((prompt >= 1) & (prompt < dims.vocab) & (prompt != PO.EOS_ID) & (prompt != PO.MASK_ID)).all())
        frames = dims.seq_len - dims.regions - 2 - t                     # the reference generates T - t words after the prompt
        if mode == "greedy":
            assert case["ids"].shape == (B, frames) and case["gaps"].shape == (B, frames)
        else:
            assert case["pred_seq"].shape == (B, dims.seq_len) and case["cand_scores"].shape == (B, frames, PO.K + 1)
            assert bool((case["wids"][:, frames:] == 0).all())
