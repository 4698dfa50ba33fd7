"""The decode step data flow (vlp_b200/decode.py DecodeState) and the decode refusals (check_decode), host side: per frame, the layer
call and its rows, query length, key length and cache position for each of the three histories, derived from the positions rather
than recorded; the rows after expand; reorder against a plain gather; and the refusal matrix of the constructor, forward and the
command line."""
import argparse
import contextlib

import pytest
import torch

from tools import abi_cases
from vlp_b200 import _lib, decode_args, synth
from vlp_b200 import vlp_modules as vm
from vlp_b200.decode import DecodeState

LAYER_CALLS = ("vlpk_encoder_fwd", "vlpk_layer_fwd", "vlpk_layer_cached_fwd", "vlpk_layer_cached_group_fwd")


@pytest.fixture
def tiny():
    """make(K=1, **decoder kwargs) -> (decoder, the six inputs of its forward, frames decoded)."""
    d = synth.TINY
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)
    B, R, L = 2, d.regions, d.seq_len
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    vis, pe = torch.randn(B, R, d.vis_dim).bfloat16(), torch.randn(B, R, d.pe_dim).bfloat16()

    def make(K=1, **kw):
        model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, search_beam_size=K, enable_butd=True, len_vis_input=R,
                                         **kw).bfloat16().eval()
        return model, (vis, pe, input_ids, tt, pos, mask), L - R - 2
    return make


@contextlib.contextmanager
def _layer_calls():
    """The dry-run's layer calls as (name, rows, Lq, Lkv, cache position) plus, for the group call, (P, G)."""
    with abi_cases.dry_run():
        calls, fake = [], _lib.invoke

        def record(name, *args):
            if name in LAYER_CALLS:
                s = args[0]._obj
                extra = {"vlpk_layer_cached_fwd": (args[5],), "vlpk_layer_cached_group_fwd": (args[10], args[5], args[9])}.get(name, ())
                calls.append((name, s.B, s.Lq, s.Lkv) + extra)
            return fake(name, *args)
        _lib.invoke = record
        yield calls


def _expected(history, B, G, in_len, frames, layers):
    """Frame 0 runs [input | MASK] at one row per image from position 0; frame f >= 1 runs (word, MASK) at positions
    in_len + f - 1, in_len + f, over keys [0, in_len + f] (the previous [MASK] row's K | V is overwritten), at B*G rows."""
    out = [{"cache": ("vlpk_layer_cached_fwd", B, in_len + 1, in_len + 1, 0),
            "shared": ("vlpk_layer_cached_fwd", B, in_len + 1, in_len + 1, 0),
            "reference": ("vlpk_encoder_fwd", B, in_len + 1, in_len + 1)}[history]] * (1 if history == "reference" else layers)
    for f in range(1, frames):
        pos, Lkv = in_len + f - 1, in_len + f + 1
        call = {"cache": ("vlpk_layer_cached_fwd", B * G, 2, Lkv, pos),
                "shared": ("vlpk_layer_cached_group_fwd", B * G, 2, Lkv, pos - in_len, in_len, G),
                "reference": ("vlpk_layer_fwd", B * G, 2, Lkv)}[history]
        out += [call] * layers
    return out


@pytest.mark.parametrize("kw,history,G", [
    (dict(), "cache", 1), (dict(), "reference", 1),                                            # greedy
    (dict(K=3), "cache", 3), (dict(K=3), "reference", 3),                                      # beam search
    (dict(sampling_method="topk", topk=4), "cache", 1), (dict(sampling_method="topp", topp=0.9), "reference", 1),
    (dict(K=3, num_return_sequences=2), "shared", 3), (dict(sampling_method="topk", topk=4, num_return_sequences=3), "shared", 3)])
def test_layer_calls_per_frame(tiny, kw, history, G):
    model, args, frames = tiny(**kw)
    model.use_kv_cache = history != "reference"
    with _layer_calls() as calls:
        model(*args)
    B, in_len = args[2].shape
    assert calls == _expected(history, B, G, in_len, frames, model.config.num_hidden_layers)


def _state(model, args, shared_prefix=None):
    """A DecodeState of forward's inputs, the regions projected as forward projects them."""
    with torch.no_grad(), abi_cases.dry_run():
        vis, pe = model.project_regions(args[0], args[1])
    return DecodeState(model, vis, pe, *args[2:], shared_prefix=shared_prefix)


@pytest.mark.parametrize("history", ["cache", "reference", "shared"])
def test_rows_after_expand(tiny, history):
    model, args, _ = tiny(K=3, num_return_sequences=2 if history == "shared" else 1)
    model.use_kv_cache = history != "reference"
    B, G = args[2].shape[0], 3
    state = _state(model, args, G if history == "shared" else None)
    with torch.no_grad(), abi_cases.dry_run():
        state.step(args[2])
    state.expand(G)
    assert state.token_type_ids.shape[0] == state.position_ids.shape[0] == state.mask_ids.shape[0] == B * G
    if history == "shared":                                   # G hypotheses per image already; the mask is read per image
        assert state.attention_mask.shape[0] == B and state.caches.B == B and state.caches.G == G
    elif history == "cache":
        assert state.attention_mask.shape[0] == B * G and all(c.shape[0] == B * G and c.is_contiguous() for c in state.caches)
    else:
        assert state.attention_mask.shape[0] == B * G
        assert state.prev_emb.shape[0] == B * G and all(x.shape[0] == B * G for x in state.prev_layers)
    with torch.no_grad(), abi_cases.dry_run() as calls:
        state.step(torch.zeros(B * G, 1, dtype=torch.long))
    assert calls


def test_expand_repeats_each_item_consecutively(tiny):
    model, args, _ = tiny(K=2)
    state = _state(model, args)
    state.caches = [torch.arange(6).view(3, 2)]
    state.expand(2)
    assert state.caches[0].tolist() == [[0, 1], [0, 1], [2, 3], [2, 3], [4, 5], [4, 5]]


def test_reorder_follows_back_pointers_per_batch_item(tiny):
    """The beam reorder of the contiguous caches and of the re-encoded history."""
    model, args, _ = tiny(K=3)
    B, K = 2, 3
    x = torch.arange(B * K * 4, dtype=torch.float32).view(B * K, 2, 2)
    back = torch.tensor([[2, 0, 0], [1, 1, 2]])
    for history in ("cache", "reference"):
        state = _state(model, args)
        if history == "cache":
            state.caches = [x, x + 100]
        else:
            state.caches, state.prev_emb, state.prev_layers = None, x, [x + 100]
        state.reorder((back + torch.arange(B).unsqueeze(1) * K).reshape(-1))
        ys = state.caches if history == "cache" else [state.prev_emb] + state.prev_layers
        for y, src in zip(ys, (x, x + 100)):
            xs = src.view(B, K, 2, 2)
            for b in range(B):
                for k in range(K):
                    assert torch.equal(y.view(B, K, 2, 2)[b, k], xs[b, back[b, k]]), history


def test_shared_reorder_gathers_the_slot_table(tiny):
    model, args, frames = tiny(K=3, num_return_sequences=2)
    B, G = args[2].shape[0], 3
    state = _state(model, args, G)
    gen = torch.Generator().manual_seed(0)
    with torch.no_grad(), abi_cases.dry_run():
        state.step(args[2])
        state.expand(G)
        for f in range(1, frames):
            state.step(torch.zeros(B * G, 1, dtype=torch.long))
            parent = [b * G + int(torch.randint(G, (1,), generator=gen)) for b in range(B) for _ in range(G)]
            slots = state.caches.slots.tolist()
            for i in range(B * G):
                slots[i][f - 1] = i * frames + f - 1           # the word each hypothesis has just written, in its own row
            state.reorder(torch.tensor(parent))
            assert state.caches.slots.tolist() == [slots[p] for p in parent]


# ---------------------------------------------------------------------------------------------------------------------------
# refusals: the same settings at the constructor, at forward (set after construction) and on the command line
# ---------------------------------------------------------------------------------------------------------------------------
NG0 = dict(forbid_duplicate_ngrams=True, ngram_size=0)
# settings, refused by (constructor, forward, command line)
MATRIX = [
    (dict(sampling_method="nucleus"), (True, True, True)),
    (dict(sampling_method="topk", topk=0), (True, True, True)),
    (dict(sampling_method="topk", topk=65), (True, True, True)),
    (dict(sampling_method="topp", topp=1.5), (True, True, True)),
    (dict(sampling_method="topk", topk=4, beam_size=3), (True, True, True)),
    (dict(**NG0), (False, False, True)),                      # greedy ignores the n-gram settings; the command line does not
    (dict(beam_size=3, **NG0), (False, True, True)),
    (dict(sampling_method="topk", topk=4, **NG0), (False, True, True)),
    (dict(sampling_method="topp", topp=0.9, **NG0), (False, True, True)),
    (dict(num_return_sequences=2), (True, True, True)),
    (dict(num_return_sequences=0, beam_size=3), (True, True, True)),
    (dict(num_return_sequences=4, beam_size=3), (True, True, True)),
    (dict(num_return_sequences=3, beam_size=3, **dict(forbid_duplicate_ngrams=True, ngram_size=2)), (False, False, False)),
    (dict(num_return_sequences=2, sampling_method="topk", topk=4), (False, False, False)),
]


def _ctor_kw(s):
    kw = {("search_beam_size" if k == "beam_size" else k): v for k, v in s.items()}
    return kw.pop("search_beam_size", 1), kw


def _argv(s):
    argv = []
    for k, v in s.items():
        argv += [f"--{k}"] if v is True else [f"--{k}", str(v)]
    return argv


def _case_id(x):
    return "-".join(f"{k}={v}" for k, v in x.items()) if isinstance(x, dict) else None


@pytest.mark.parametrize("settings,refused", MATRIX, ids=_case_id)
def test_refusal_matrix(tiny, settings, refused):
    by_ctor, by_forward, by_cli = refused
    K, kw = _ctor_kw(settings)
    if by_ctor:
        with pytest.raises(ValueError, match="vlp_b200"):
            tiny(K=K, **kw)
    model, args, _ = tiny()
    model.search_beam_size = K
    for k, v in kw.items():
        setattr(model, k, v)
    with abi_cases.dry_run() as calls:
        if by_forward:
            with pytest.raises(ValueError, match="vlp_b200"):
                model(*args)
        else:
            model(*args)
    assert (calls == []) == by_forward
    if not by_ctor:
        tiny(K=K, **kw)
    parser = decode_args.add_decode_args(argparse.ArgumentParser())
    if by_cli:
        with pytest.raises(SystemExit) as e:
            decode_args.parse_decode_args(parser, _argv(settings))
        assert e.value.code == 2
        ns = argparse.Namespace(**{**vars(parser.parse_args([])), **settings})
        with pytest.raises(ValueError, match="vlp_b200"):
            decode_args.check_decode_args(ns)
    else:
        decode_args.parse_decode_args(parser, _argv(settings))


@pytest.mark.parametrize("kw,over", [(dict(K=3, num_return_sequences=2), dict(use_kv_cache=False)),
                                     (dict(K=3, num_return_sequences=2), dict(output_attentions=True)),
                                     (dict(sampling_method="topk", topk=4, num_return_sequences=2), dict(use_kv_cache=False)),
                                     (dict(sampling_method="topk", topk=4, num_return_sequences=2), dict(output_attentions=True))])
def test_forward_refuses_settings_of_the_call(tiny, kw, over):
    model, args, _ = tiny(**kw)
    model.use_kv_cache = over.get("use_kv_cache", True)
    with abi_cases.dry_run() as calls, pytest.raises(ValueError, match="vlp_b200"):
        model(*args, output_attentions=over.get("output_attentions", False))
    assert calls == []
