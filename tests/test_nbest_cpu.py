"""Several captions per image (`num_return_sequences` N > 1) over one K/V cache of the image prefix, host side: the C ABI's argument
checks, the refused model and command-line combinations, the n-best selection against a plain restatement of the final-selection
rule, the slot-table bookkeeping against today's expand + index_select cache chain, and the call sequences under the dry-run."""
import argparse
import math
import random

import pytest
import torch

from tools import abi_cases
from vlp_b200 import _lib, beam, decode_args, synth
from vlp_b200 import vlp_modules as vm
from vlp_b200.shared_prefix import SharedPrefixCache

# ---------------------------------------------------------------------------------------------------------------------------
# C ABI
# ---------------------------------------------------------------------------------------------------------------------------
_A = 1 << 16                                                   # fake, aligned device addresses: every call below fails validation


def _group_call(shape=None, **over):
    a = dict(x=_A, prefix=2 * _A, prefix_rows=11, P=10, text=3 * _A, T=8, slots=4 * _A, G=3, pos=3, mask=5 * _A, mask_rows=2)
    a.update(over)
    s = shape or dict(B=6, Lq=2, Lkv=a["P"] + a["pos"] + 2, H=128, heads=2, I=256, kv_slots=0)
    acts = _lib.VlpkLayerActs(*([6 * _A] * len(_lib.ACT_FIELDS)))
    w = _lib.VlpkLayerWeights(*([7 * _A] * len(_lib.WEIGHT_FIELDS)))
    return _lib.lib().vlpk_layer_cached_group_fwd(_lib.VlpkShape(*s.values()), w, a["x"], a["prefix"], a["prefix_rows"], a["P"], a["text"],
                                                  a["T"], a["slots"], a["G"], a["pos"], a["mask"], a["mask_rows"], acts, 0, None)


BAD_ABI = [dict(G=4), dict(G=0), dict(G=-3), dict(P=12), dict(P=0), dict(pos=7), dict(pos=-1), dict(x=None), dict(prefix=None),
           dict(text=None), dict(slots=None), dict(mask=None), dict(prefix=2 * _A + 8), dict(text=3 * _A + 8), dict(x=_A + 2),
           dict(slots=4 * _A + 2), dict(mask=5 * _A + 4), dict(mask_rows=3), dict(mask_rows=0)]


def test_abi_rejects_bad_arguments_without_launching():
    lib = _lib.lib()
    assert "vlpk_layer_cached_group_fwd" in _lib.EXPORTED_SYMBOLS
    before = lib.vlpk_launch_count()
    for bad in BAD_ABI:
        assert _group_call(**bad) < 0, bad
        assert lib.vlpk_last_error()
    # Lkv must be P + pos + Lq, and at most 512
    assert _group_call(shape=dict(B=6, Lq=2, Lkv=16, H=128, heads=2, I=256, kv_slots=0)) < 0
    assert _group_call(shape=dict(B=6, Lq=2, Lkv=600, H=128, heads=2, I=256, kv_slots=640), P=500, prefix_rows=501, pos=98, T=100) < 0
    assert _group_call(shape=dict(B=6, Lq=2, Lkv=15, H=100, heads=2, I=256, kv_slots=0)) < 0           # head_dim must be 64
    assert lib.vlpk_launch_count() == before


# ---------------------------------------------------------------------------------------------------------------------------
# refused combinations: model and command line
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


BAD_CTOR = [dict(num_return_sequences=0), dict(num_return_sequences=-1), dict(num_return_sequences=1.5), dict(num_return_sequences=True),
            dict(K=3, num_return_sequences=4), dict(K=1, num_return_sequences=2)]


@pytest.mark.parametrize("bad", BAD_CTOR, ids=lambda b: "-".join(f"{k}={v}" for k, v in b.items()))
def test_constructor_refuses(bad):
    with pytest.raises(ValueError, match="vlp_b200"):
        _tiny_decoder(**bad)


def _refused_forward(model, args, **kw):
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="vlp_b200"):
            model(*args, **kw)
    assert calls == []


def test_forward_refuses_before_any_launch():
    model, args, _ = _tiny_decoder(K=3, num_return_sequences=2)
    _refused_forward(model, args, output_attentions=True)
    model.use_kv_cache = False
    _refused_forward(model, args)
    model.use_kv_cache = True
    model.num_return_sequences = 4                             # N > K
    _refused_forward(model, args)
    model.num_return_sequences = 0
    _refused_forward(model, args)
    model.search_beam_size, model.num_return_sequences = 1, 2  # greedy, and the reference's sample_mode="sample"
    _refused_forward(model, args)
    _refused_forward(model, args, sample_mode="sample")
    model, args, _ = _tiny_decoder(sampling_method="topk", topk=4, num_return_sequences=3)
    _refused_forward(model, args, output_attentions=True)
    model.use_kv_cache = False
    _refused_forward(model, args)


def _parser():
    return decode_args.add_decode_args(argparse.ArgumentParser())


@pytest.mark.parametrize("argv", [["--num_return_sequences", "0"], ["--num_return_sequences", "4", "--beam_size", "3"],
                                  ["--num_return_sequences", "2"], ["--num_return_sequences", "-2", "--sampling_method", "topk"]])
def test_cli_refuses(argv):
    with pytest.raises(SystemExit) as e:
        decode_args.parse_decode_args(_parser(), argv)
    assert e.value.code == 2
    with pytest.raises(ValueError, match="vlp_b200"):
        decode_args.check_decode_args(_parser().parse_args(argv))


def test_cli_passes_the_count_on():
    kw = decode_args.decoder_kwargs(decode_args.parse_decode_args(_parser(), ["--beam_size", "5", "--num_return_sequences", "3"]))
    assert (kw["search_beam_size"], kw["num_return_sequences"]) == (5, 3)
    kw = decode_args.decoder_kwargs(decode_args.parse_decode_args(_parser(), ["--sampling_method", "topk", "--topk", "8",
                                                                               "--num_return_sequences", "5"]))
    assert kw["num_return_sequences"] == 5
    model, _, _ = _tiny_decoder(K=kw.pop("search_beam_size"), **kw)
    assert model.num_return_sequences == 5
    assert "num_return_sequences" not in decode_args.decoder_kwargs(decode_args.parse_decode_args(_parser(), []))


# ---------------------------------------------------------------------------------------------------------------------------
# n-best selection
# ---------------------------------------------------------------------------------------------------------------------------
def _plain_nbest(sc, wi, pt, eos, lp, n, out_len):
    """The final-selection rule as plain loops: candidates in (frame, beam) order, stable sort by value, each back-tracked."""
    T, B, K = sc.shape
    seqs, vals = [], []
    for b in range(B):
        last = next((f for f in range(T) if all(int(wi[f, b, k]) == eos for k in range(K))), T - 1)
        cands = []
        for f in range(last + 1):
            for k in range(K):
                if int(wi[f, b, k]) == eos or f == last:
                    v = (sc[f, b, k] + torch.tensor(lp * (f + 1), dtype=torch.float32)).item()     # fp32, as the device computes it
                    cands.append((v, f, k))
        cands.sort(key=lambda c: -c[0])                        # stable: equal values keep (frame, beam) order
        rows, vs = [], []
        for v, f, k in cands[:n]:
            seq, pos = [0] * out_len, k
            for g in range(f, -1, -1):
                seq[g] = int(wi[g, b, pos])
                pos = int(pt[g, b, pos]) if g > 0 else pos
            rows.append(seq)
            vs.append(v)
        seqs.append(rows)
        vals.append(vs)
    return torch.tensor(seqs), torch.tensor(vals)


@pytest.mark.parametrize("lp", [0.0, 0.5, -1.0])
def test_nbest_matches_the_plain_rule(lp):
    rng = torch.Generator().manual_seed(5)
    eos = 3
    for trial in range(40):
        T, B, K = int(torch.randint(1, 9, (1,), generator=rng)), int(torch.randint(1, 4, (1,), generator=rng)), [2, 3, 5][trial % 3]
        out_len = T + 4
        sc = torch.randint(-6, 1, (T, B, K), generator=rng).float() * 0.5          # coarse values: many exact ties
        p_eos = [0.0, 0.3, 0.9][trial % 3]
        wi = torch.where(torch.rand(T, B, K, generator=rng) < p_eos, torch.full((T, B, K), eos),
                         torch.randint(4, 9, (T, B, K), generator=rng))
        if trial % 5 == 0 and T > 2:
            wi[T // 2, 0] = eos                                # a whole frame of [EOS] ends that sample early
        pt = torch.randint(0, K, (T, B, K), generator=rng)
        for n in range(1, K + 1):
            seq, val = beam.nbest(sc, wi, pt, eos, lp, out_len, n)
            want_seq, want_val = _plain_nbest(sc, wi, pt, eos, lp, n, out_len)
            assert seq.shape == (B, n, out_len) and val.shape == (B, n)
            assert torch.equal(seq, want_seq), (trial, n)
            assert torch.equal(val, want_val), (trial, n)
            assert torch.equal(seq[:, 0], beam.backtrack(sc, wi, pt, eos, lp, out_len))


# ---------------------------------------------------------------------------------------------------------------------------
# slot table: the rows every hypothesis reads, against today's contiguous per-hypothesis caches
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_slot_table_selects_the_rows_of_the_contiguous_cache_chain(seed):
    rnd = random.Random(seed)
    B, G, P, T = rnd.choice([1, 2, 3]), rnd.choice([1, 2, 3, 5]), rnd.choice([1, 4]), rnd.choice([2, 3, 7, 12])
    cache = SharedPrefixCache(1, B, G, P, T, 64, "cpu")
    # today's path: each hypothesis owns a contiguous cache, expanded from its image after step 0 and index_selected every step;
    # a row is named by who computed it: ("p", image, r) for the prefix, ("t", i, f) for hypothesis i's row at text position f
    contig = [[("p", i // G, r) for r in range(P)] for i in range(B * G)]
    written, read = {}, {}                                  # text row -> steps (pos) that wrote / read it
    for pos in range(T - 1):                                # the step feeding frame pos's word, Lq = 2 (word, [MASK])
        for i in range(B * G):
            new = [("t", i, pos), ("t", i, pos + 1)]
            for f in (pos, pos + 1):
                written.setdefault(i * T + f, []).append(pos)
            # what the group kernel reads: the image prefix, slot rows for frames < pos, then its own new rows
            got = [("p", i // G, r) for r in range(P)]
            for j in range(pos):
                row = int(cache.slots[i, j])
                read.setdefault(row, []).append(pos)
                got.append(("t", row // T, row % T))
            assert got + new == contig[i] + new, (pos, i)
            contig[i] = contig[i] + new
        parent = [b * G + rnd.randrange(G) for b in range(B) for _ in range(G)]
        contig = [contig[p][:P + pos + 1] for p in parent]  # the [MASK] row is dropped: the next step overwrites it
        cache.reorder(torch.tensor(parent), pos)
    for row, steps in read.items():                         # write-before-read: no row changes once a descendant could read it
        assert max(written[row]) < min(steps), row


# ---------------------------------------------------------------------------------------------------------------------------
# call sequences
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(K=3, num_return_sequences=2), dict(K=3, num_return_sequences=3),
                                dict(sampling_method="topk", topk=4, num_return_sequences=2),
                                dict(sampling_method="topp", topp=0.9, num_return_sequences=5)])
def test_group_decode_call_sequence(kw):
    model, args, steps = _tiny_decoder(**kw)
    layers = model.config.num_hidden_layers
    N = kw["num_return_sequences"]
    with abi_cases.dry_run() as calls:
        out = model(*args)
    cached = [c for c in calls if c in ("vlpk_layer_cached_fwd", "vlpk_layer_cached_group_fwd", "vlpk_layer_fwd", "vlpk_encoder_fwd")]
    assert cached == ["vlpk_layer_cached_fwd"] * layers + ["vlpk_layer_cached_group_fwd"] * (layers * (steps - 1))
    B, out_len = args[2].shape[0], args[3].shape[1]
    if "K" in kw:
        assert set(out) == {"pred_seq", "scores", "wids", "ptrs", "nbest_seq", "nbest_scores"}
        assert out["nbest_seq"].shape == (B, N, out_len) and out["nbest_scores"].shape == (B, N)
    else:
        assert out[0].shape == (B, N, steps) and out[1].shape == (B, N, steps)


@pytest.mark.parametrize("kw", [dict(K=3), dict(sampling_method="topk", topk=4), dict(K=1)])
def test_single_caption_decode_keeps_its_calls(kw):
    model, args, steps = _tiny_decoder(**kw)
    with abi_cases.dry_run() as calls:
        model(*args)
    assert calls.count("vlpk_layer_cached_fwd") == steps * model.config.num_hidden_layers
    assert "vlpk_layer_cached_group_fwd" not in calls
