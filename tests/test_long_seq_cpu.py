"""CPU: the host side of sequences longer than one 128-row tile (L in (128, 512]) — VlpkShape.kv_slots, argument checks that run
before any launch, buffer sizes, and the marshalling of a full L = 143 training step and a cached decode (tools/abi_cases.dry_run)."""
import ctypes as C

import pytest
import torch

from tools import abi_cases
from vlp_b200 import _lib, ops, synth
from vlp_b200 import vlp_modules as vm


def _shape(B, Lq, Lkv, slots, H=128, heads=2, I=512):
    return _lib.VlpkShape(B, Lq, Lkv, H, heads, I, slots)


def test_kv_slots_rule():
    assert [ops.kv_slots(L, L) for L in (1, 123, 128, 129, 143, 256, 257, 384, 385, 512)] == [0, 0, 0, 256, 256, 256, 384, 384, 512, 512]
    assert ops.kv_slots(2, 300) == 384 and ops.kv_slots(2, 100) == 0
    assert _lib.VlpkShape(1, 2, 3, 128, 2, 512).kv_slots == 0          # the six-field form keeps the 128-slot layout
    for Lq, Lkv in ((513, 513), (1, 513), (0, 5)):
        with pytest.raises(ValueError, match="sequence length"):
            ops.kv_slots(Lq, Lkv)


@pytest.mark.parametrize("L", [143, 512])
def test_workspace_bytes_match_acts(L):
    out = (C.c_size_t * 3)()
    shape = _shape(2, L, L, ops.kv_slots(L, L))
    assert _lib.lib().vlpk_workspace_bytes(C.byref(shape), out) == 0
    a = ops._Acts(1, 2, L, 128, 2, 512, "cpu", drop_bits=True)
    assert out[0] == a.bf.numel() * 2 + a.f32.numel() * 4
    assert a.bits.shape[1] == 2 * 2 * L * ops.key_slots(L) // 8


@pytest.mark.parametrize("Lq,Lkv,slots", [(129, 129, 0), (129, 129, 128), (200, 200, 384), (200, 200, 640), (513, 513, 640),
                                          (300, 129, 256), (143, 143, 255)])
def test_shape_rejects_slots_that_disagree(Lq, Lkv, slots):
    out = (C.c_size_t * 3)()
    n0 = _lib.lib().vlpk_launch_count()
    assert _lib.lib().vlpk_workspace_bytes(C.byref(_shape(2, Lq, Lkv, slots)), out) < 0
    assert b"sequence length" in _lib.lib().vlpk_last_error()
    # the layer entry points check the shape first, so null pointers are never reached
    assert _lib.lib().vlpk_layer_fwd(C.byref(_shape(2, Lq, Lkv, slots)), None, None, None, None, 1, None, 0.0, 0.0, None, 0, None) < 0
    assert _lib.lib().vlpk_launch_count() == n0


def test_wide_entry_points_are_declared_and_exported():
    for name in ("vlpk_attn_core_fwd_wide", "vlpk_attn_core_bwd_wide"):
        assert name in _lib.EXPORTED_SYMBOLS and hasattr(_lib.lib(), name)
    assert _lib.lib().vlpk_debug_set_option(b"attn_tiled", 0) == 0


def test_mask_pack_over_512_keys_raises_before_launch():
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError):
            ops.pack_mask(torch.ones(1, 1, 513, dtype=torch.long), "zero_one")
    assert calls == []


def _config(dims, max_pos=None):
    return vm.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                         intermediate_size=dims.inter, type_vocab_size=dims.type_vocab,
                         max_position_embeddings=dims.max_pos if max_pos is None else max_pos)


def _dims(L):
    return synth.VlpDims(vocab=1000, hidden=128, layers=2, heads=2, inter=512, regions=100, text=L - 103)


def _step(model, b):
    out = model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None,
                b["is_next"], masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"], drop_worst_ratio=0.0)
    sum(l.float().sum() for l in out).backward()


def test_dry_run_training_step_at_143():
    d = _dims(143)
    model = vm.BertForPreTrainingLossMask(_config(d), enable_butd=True, len_vis_input=d.regions).bfloat16().train()
    b = synth.make_batch(d, 2, seed=1, mode="mix", ragged=True)
    with abi_cases.dry_run() as calls:
        _step(model, b)
    assert "vlpk_mask_pack" in calls and "vlpk_encoder_fwd" in calls and "vlpk_encoder_bwd" in calls


def test_dry_run_cached_greedy_decode_to_length_143():
    d = _dims(143)
    model = vm.BertForSeq2SeqDecoder(_config(d), mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=d.regions).bfloat16().eval()
    B, R, L = 1, d.regions, d.seq_len
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.ones(B, L, L, dtype=torch.long)
    vis = torch.zeros(B, R, d.vis_dim)
    pe = torch.zeros(B, R, d.pe_dim)
    sizes = []
    new = model.new_kv_caches
    model.new_kv_caches = lambda batch, device, rows=128: (sizes.append(rows), new(batch, device, rows))[1]
    with abi_cases.dry_run() as calls:
        model(vis.bfloat16(), pe.bfloat16(), input_ids, tt, pos, mask)
    assert sizes == [L]                                                  # caches sized from the output length, not 128
    assert calls.count("vlpk_layer_cached_fwd") == d.layers * (L - R - 2)


def test_python_surface_raises_for_long_sequences():
    d = _dims(143)
    b = synth.make_batch(d, 1, seed=1)
    model = vm.BertForPreTrainingLossMask(_config(d, max_pos=140), enable_butd=True, len_vis_input=d.regions).bfloat16()
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="max_position_embeddings"):
            _step(model, b)
    assert calls == []
    d = _dims(515)
    b = synth.make_batch(d, 1, seed=1)
    model = vm.BertForPreTrainingLossMask(_config(d, max_pos=1024), enable_butd=True, len_vis_input=d.regions).bfloat16()
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="512"):
            _step(model, b)
    assert calls == []


# ---- oracle vs the reference above one tile ----------------------------------------------------------------------------------------
def _rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def long_gold(golden_dir):
    import os
    return torch.load(os.path.join(golden_dir, "long_seq.pt"))


@pytest.mark.parametrize("name", ["l143_mix_ragged", "l256_s2s", "l512_bi"])
def test_oracle_matches_reference_golden_above_one_tile(name, long_gold):
    """The fp32 oracle (oracle/vlp_oracle.py), which the GPU tests compare with, against the unmodified reference at L = 143 / 256 / 512:
    losses, activation samples (rel-L2 <= 1e-5) and every parameter gradient (rel-L2 <= 1e-4)."""
    from oracle import vlp_oracle as O
    from tools import long_seq_oracle as LSO
    g = long_gold["cases"][name]
    dims, sd, batch = LSO.inputs(name)
    for k, v in sd.items():
        if k != "cls.predictions.decoder.weight":
            v.requires_grad_(True)
    losses, aux = O.pretraining_loss(sd, dims, batch, return_all=True)
    sum(l.sum() for l in losses).backward()
    for got, ref in zip(losses, g["losses"]):
        assert abs(float(got.detach()) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref)))
    assert _rel(LSO.sample(aux["embedding"]), g["embedding"]) < 1e-5
    assert len(aux["layers"]) == len(g["layers"])
    for got, ref in zip(aux["layers"], g["layers"]):
        assert _rel(LSO.sample(got), ref) < 1e-5
    assert _rel(LSO.sample(aux["logits"]), g["logits"]) < 1e-5
    assert _rel(LSO.sample(aux["pooled"]), g["pooled"]) < 1e-5
    scale = max(float(fp["full"].norm()) if "full" in fp else fp["norm"] for fp in g["grads"].values())
    n = 0
    for k, fp in g["grads"].items():
        got = sd[k].grad
        assert got is not None, k
        if "full" in fp:
            if fp["full"].norm() <= 1e-7 * scale:           # zero in exact arithmetic (key bias): round-off level only
                assert got.norm() <= 1e-7 * scale, k
            else:
                assert _rel(got, fp["full"]) < 1e-4, k
        else:
            assert abs(got.norm().item() - fp["norm"]) <= 1e-4 * fp["norm"] + 1e-12, k
            assert _rel(LSO.sample(got, LSO.GRAD_SAMPLES), fp["sample"]) < 1e-4, k
        n += 1
    assert n >= 40


def test_oracle_greedy_decode_matches_reference_golden_at_143(long_gold):
    from oracle import vlp_oracle as O
    from tools import long_seq_oracle as LSO
    g = long_gold["greedy"]
    dims, sd, args = LSO.decode_inputs(g["B"], g["seed"])
    with torch.no_grad():
        ids, scores = O.greedy_decode(sd, dims, *args, mask_word_id=103)
    assert torch.equal(ids, g["ids"])
    assert _rel(scores, g["scores"]) < 1e-5
