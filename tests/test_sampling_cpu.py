"""Top-k / top-p sampling decode (vlp_b200/decode.py, vlpk_sample_tokens in csrc/decode.cu), host side: argument validation at the
C ABI, the Python API and the command line (nothing is launched for a refused combination), and the launches of a sampling decode
under the dry-run."""
import argparse

import pytest
import torch

from tools import abi_cases
from vlp_b200 import _lib, decode_args, ops, synth
from vlp_b200 import vlp_modules as vm


def _abi_call(**over):
    a = dict(rows=4, V=1000, logits=1, ld=1000, bias=None, fp32=0, mode=0, topk=8, topp=0.9, seed=1, f=0, seq=1, T_cap=20, score=None,
             finished=1, live=1, eos_id=102, pad_id=0, block_eos=0, n=0, ignore=None, n_ignore=0, stream=None)
    a.update(over)
    return _lib.lib().vlpk_sample_tokens(*a.values())


def test_abi_refuses_bad_arguments_without_launching():
    lib = _lib.lib()
    before = lib.vlpk_launch_count()
    for bad in (dict(mode=2), dict(mode=-1), dict(topk=0), dict(topk=65), dict(mode=1, topp=0.0), dict(mode=1, topp=1.5),
                dict(mode=1, topp=float("nan")), dict(ld=999), dict(V=0), dict(f=20), dict(f=-1), dict(T_cap=0), dict(logits=None),
                dict(seq=None), dict(finished=None), dict(live=None), dict(n_ignore=1), dict(n=-1), dict(fp32=2),
                dict(V=60000, ld=60000)):
        assert _abi_call(**bad) < 0, bad
        assert lib.vlpk_last_error()
    assert _abi_call(rows=0) == 0                                    # nothing to do: accepted, no launch
    assert _abi_call(rows=0, mode=0, topk=64) == 0 and _abi_call(rows=0, mode=1, topp=1.0, topk=0) == 0    # topk unused by top-p
    assert lib.vlpk_launch_count() == before


def _tiny_decoder(**kw):
    d = synth.TINY
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=d.regions, **kw).bfloat16().eval()
    B, R, L = 2, d.regions, d.seq_len
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    args = (torch.randn(B, R, d.vis_dim).bfloat16(), torch.randn(B, R, d.pe_dim).bfloat16(), input_ids, tt, pos, mask)
    return model, args, L - R - 2


BAD_API = [dict(sampling_method="topk", topk=0), dict(sampling_method="topk", topk=65), dict(sampling_method="topk", topk=2.0),
           dict(sampling_method="topk", topk=True), dict(sampling_method="topp", topp=0.0), dict(sampling_method="topp", topp=1.01),
           dict(sampling_method="topp", topp=-0.5), dict(sampling_method="topp", topp=float("nan")),
           dict(sampling_method="topk", topk=4, search_beam_size=3), dict(sampling_method="topp", topp=0.9, search_beam_size=2),
           dict(sampling_method="greedy")]


@pytest.mark.parametrize("bad", BAD_API, ids=lambda b: "-".join(f"{k}={v}" for k, v in b.items()))
def test_api_refuses_bad_combinations_before_any_launch(bad):
    with pytest.raises(ValueError, match="vlp_b200"):
        _tiny_decoder(**bad)
    model, args, _ = _tiny_decoder(sampling_method="topk", topk=4)   # set after construction: forward refuses before any launch
    for k, v in bad.items():
        setattr(model, k, v)
    with abi_cases.dry_run() as calls, pytest.raises(ValueError, match="vlp_b200"):
        model(*args, task_idx=None)
    assert calls == []


def test_beam_search_defaults_are_unchanged():
    model, _, _ = _tiny_decoder()
    assert (model.sampling_method, model.search_beam_size) == ("beam_search", 1)
    model, _, _ = _tiny_decoder(search_beam_size=3, topk=0, topp=5.0)    # unused sampling options are not checked for beam search
    assert model.sampling_method == "beam_search"


@pytest.mark.parametrize("method,extra", [("topk", dict(topk=8)), ("topp", dict(topp=0.9))])
@pytest.mark.parametrize("ngram", [False, True])
def test_sampling_decode_marshalling_dry_run(method, extra, ngram):
    """One vlpk_sample_tokens per frame replaces the greedy arg-max; n-gram blocking is inside it (no vlpk_beam_ngram_block); the
    layer calls are the greedy decode's."""
    model, args, frames = _tiny_decoder(forbid_duplicate_ngrams=ngram, forbid_ignore_set={7}, ngram_size=2, min_len=2)
    with abi_cases.dry_run() as greedy:
        model(*args, task_idx=None)
    model.sampling_method = method
    for k, v in extra.items():
        setattr(model, k, v)
    with abi_cases.dry_run() as calls:
        ids, scores = model(*args, task_idx=None, seed=5)
    assert ids.shape == (2, frames) and ids.dtype == torch.int64 and scores.dtype == torch.float32
    assert calls.count("vlpk_sample_tokens") == frames and model.last_decode_steps == frames
    assert [c for c in calls if c != "vlpk_sample_tokens"] == greedy
    assert "vlpk_beam_ngram_block" not in calls


def test_ops_wrapper_checks_tensors():
    V, rows, T = 50, 3, 6
    logits, seq = torch.zeros(rows, 1, V, dtype=torch.bfloat16), torch.zeros(rows, T, dtype=torch.int64)
    fin, live = torch.zeros(rows, dtype=torch.int32), torch.ones(1, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):                  # host memory is never handed to the kernel
        ops.sample_tokens(logits, None, "topk", 4, 1.0, 0, 0, seq, None, fin, live, 102)
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="mode"):
            ops.sample_tokens(logits, None, "nucleus", 4, 1.0, 0, 0, seq, None, fin, live, 102)
        with pytest.raises(RuntimeError, match="bias"):
            ops.sample_tokens(logits, torch.zeros(V), "topk", 4, 1.0, 0, 0, seq, None, fin, live, 102)
        with pytest.raises(RuntimeError, match="bf16 or fp32"):
            ops.sample_tokens(logits.half(), None, "topk", 4, 1.0, 0, 0, seq, None, fin, live, 102)
        with pytest.raises(RuntimeError, match="int64"):
            ops.sample_tokens(logits, None, "topk", 4, 1.0, 0, 0, seq.int(), None, fin, live, 102)
        with pytest.raises(RuntimeError, match="int32"):
            ops.sample_tokens(logits, None, "topk", 4, 1.0, 0, 0, seq, None, fin, live, 102, ngram=3, ignore=torch.tensor([4]))
        ops.sample_tokens(logits, torch.zeros(V, dtype=torch.bfloat16), "topp", 4, 0.5, 2 ** 64 - 1, 5, seq, torch.zeros(rows, T), fin, live,
                          102, ngram=3, ignore=torch.tensor([4], dtype=torch.int32))
    assert calls == ["vlpk_sample_tokens"]


def _parser(**defaults):
    p = argparse.ArgumentParser()
    if defaults:
        p.add_argument("--seed", type=int, default=defaults["seed"])   # a script's own --seed stays
    return decode_args.add_decode_args(p)


def test_cli_flags_build_decoder_kwargs():
    args = decode_args.parse_decode_args(_parser(), ["--sampling_method", "topp", "--topp", "0.9", "--seed", "7",
                                                     "--forbid_duplicate_ngrams", "--forbid_ignore_word", "a|b", "--min_len", "3"])

    class Tok:
        def convert_tokens_to_ids(self, toks):
            return [{"a": 11, "b": 12}[t] for t in toks]

    kw = decode_args.decoder_kwargs(args, Tok())
    assert kw == dict(search_beam_size=1, length_penalty=0, forbid_duplicate_ngrams=True, forbid_ignore_set={11, 12}, ngram_size=3,
                      min_len=3, sampling_method="topp", topk=1, topp=0.9, seed=7)
    model, _, _ = _tiny_decoder(**{k: v for k, v in kw.items()})
    assert (model.sampling_method, model.topp, model.seed) == ("topp", 0.9, 7)
    assert decode_args.parse_decode_args(_parser(seed=99), []).seed == 99
    kw = decode_args.decoder_kwargs(decode_args.parse_decode_args(_parser(), ["--beam_size", "5"]))
    assert (kw["sampling_method"], kw["search_beam_size"]) == ("beam_search", 5)


@pytest.mark.parametrize("argv", [["--sampling_method", "topk", "--topk", "0"], ["--sampling_method", "topk", "--topk", "65"],
                                  ["--sampling_method", "topp", "--topp", "0"], ["--sampling_method", "topp", "--topp", "1.5"],
                                  ["--sampling_method", "topk", "--topk", "5", "--beam_size", "3"], ["--sampling_method", "nucleus"],
                                  ["--sampling_method", "topk", "--forbid_duplicate_ngrams", "--ngram_size", "0"]])
def test_cli_refuses_bad_combinations(argv, capsys):
    with pytest.raises(SystemExit) as e:
        decode_args.parse_decode_args(_parser(), argv)
    assert e.value.code == 2
    assert "error" in capsys.readouterr().err
