"""Several captions per image in one packed pass (captions_per_image), host side: the packed layout is exact (the packed oracle pass
equals the flattened pairs in float64), the oracle matches the unmodified reference's stored outputs, the packed mask and the
masked-position map, every refusal, and the marshalling of a grouped step."""
import os

import pytest
import torch

from tools import grouped_captions_oracle as GO
from vlp_b200 import staging, synth
from vlp_b200 import vlp_modules as vm


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def _leaf_sd(name, dtype):
    dims, sd, batch, G, dw, eps = GO.inputs(name)
    sd = {k: v.to(dtype).requires_grad_(True) for k, v in sd.items()}
    batch = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
    return dims, sd, batch, G, dw, eps


@pytest.mark.parametrize("name", ["h128_b3g5", "h128_b3g5_dw02_ls01"])
def test_packed_pass_equals_flattened_pairs_float64(name):
    """One packed pass per image gives the loss and every parameter gradient of the B * G separate pairs (dropout off)."""
    dims, sd, batch, G, dw, eps = _leaf_sd(name, torch.float64)
    out = []
    for fn in (GO.pair_loss, GO.packed_loss):
        for v in sd.values():
            v.grad = None
        loss, aux = fn(sd, dims, batch, G, dw, eps, return_all=True)
        loss.backward()
        out.append((loss.detach(), aux, {k: v.grad.clone() for k, v in sd.items() if v.grad is not None}))
    (l0, a0, g0), (l1, a1, g1) = out
    assert abs(float(l1) - float(l0)) <= 1e-10 * abs(float(l0))
    assert g0.keys() == g1.keys()
    for k in g0:
        scale = max(float(g0[k].norm()), 1e-30)
        assert float((g1[k] - g0[k]).norm()) <= 1e-10 * scale or k.endswith("key.bias"), k
    for x0, x1 in zip(a0["layers"], a1["layers"]):
        assert rel(GO.unpack(x1, dims, G), x0) < 1e-12
    assert rel(a1["logits"], a0["logits"]) < 1e-12


@pytest.mark.parametrize("name", list(GO.CASES))
def test_oracle_matches_reference_golden(name, golden_dir):
    """The oracle on the flattened pairs, and the packed oracle pass, against the reference's stored outputs (test_oracle.py's
    bounds: 1e-5 on losses and activations, 1e-4 on gradients)."""
    gold = torch.load(os.path.join(golden_dir, "grouped_captions.pt"))["cases"][name]
    dims, sd, batch, G, dw, eps = _leaf_sd(name, torch.float32)
    if dims.hidden > 128:
        torch.set_num_threads(max(torch.get_num_threads(), 8))
    loss, aux = GO.packed_loss(sd, dims, batch, G, dw, eps, return_all=True)
    assert abs(float(loss) - float(gold["losses"][0])) <= 1e-5 * max(1.0, abs(float(gold["losses"][0])))
    assert rel(GO.LS.sample(GO.unpack(aux["embedding"], dims, G)), gold["embedding"]) < 1e-5
    for got, ref in zip(aux["layers"], gold["layers"]):
        assert rel(GO.LS.sample(GO.unpack(got, dims, G)), ref) < 1e-5
    assert rel(GO.LS.sample(aux["logits"]), gold["logits"]) < 1e-5
    loss.backward()
    scale = max(float(v.grad.norm()) for v in sd.values() if v.grad is not None)
    for k, fp in gold["grads"].items():
        g = sd[k].grad
        ref_norm = float(fp["full"].norm()) if "full" in fp else fp["norm"]
        if ref_norm <= 1e-7 * scale:              # key.bias: exactly 0 in exact arithmetic, round-off on both sides
            assert g.norm() <= 1e-7 * scale, k
        elif "full" in fp:
            assert rel(g, fp["full"]) < 1e-4, k
        else:
            assert abs(g.norm().item() - fp["norm"]) <= 1e-4 * fp["norm"] + 1e-12, k
            assert rel(g.flatten()[GO.LS.sample_idx(g.numel(), GO.LS.GRAD_SAMPLES)], fp["sample"]) < 1e-4, k


@pytest.mark.parametrize("G", [1, 2, 5, 19])
def test_packed_mask_restates_each_pair(G):
    """Caption g's block (prefix + its text rows and keys) is that pair's loader mask; cross-caption blocks are zero; padding rows see
    the prefix only."""
    d = synth.SMALL_L123
    P, T, Lp = GO.geometry(d, G)
    len_b = torch.tensor([(3 * i) % T for i in range(2 * G)])
    m = GO.packed_mask(len_b, G, d.regions, d.seq_len)
    assert m.shape == (2, Lp, Lp)
    for b in range(2):
        for g in range(G):
            rows = torch.cat([torch.arange(P), P + g * T + torch.arange(T)])
            want = synth.attention_mask(d, int(len_b[b * G + g]), "s2s")
            assert torch.equal(m[b][rows][:, rows], want)
            for h in range(G):
                if h != g:
                    assert not m[b, P + g * T:P + (g + 1) * T, P + h * T:P + (h + 1) * T].any()
            nt = min(int(len_b[b * G + g]) + 1, T)
            pad = m[b, P + g * T + nt:P + (g + 1) * T]
            assert (pad[:, :P] == 1).all() and not pad[:, P:].any()
        assert (m[b, :P, :P] == 1).all() and not m[b, :P, P:].any()


def _cfg(d, drop=0.0):
    return vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                         type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=drop,
                         attention_probs_dropout_prob=drop)


def _grouped(G=5, B=2, d=synth.SMALL_L123, tasks="img2txt"):
    model = vm.BertForPreTrainingLossMask(_cfg(d), enable_butd=True, len_vis_input=d.regions, tasks=tasks).bfloat16().train()
    batch = synth.make_batch(d, B * G, seed=7, mode="s2s", ragged=True)
    batch["img"], batch["vis_pe"] = batch["img"][::G].bfloat16(), batch["vis_pe"][::G].bfloat16()
    len_b = (batch["input_mask"].diagonal(dim1=1, dim2=2).sum(-1) - d.regions - 3).to(torch.int32)
    _, T, Lp = GO.geometry(d, G)
    mask = staging.GroupedCaptionMask(torch.zeros(B, Lp, (Lp + 127) // 128 * 4, dtype=torch.int32), G, T, d.regions, d.seq_len)
    return model, batch, mask, len_b


def _call(model, b, mask, **kw):
    return model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], mask, b["masked_ids"], None, b["is_next"],
                 masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"], drop_worst_ratio=0.0, **kw)


def test_packed_rows_and_masked_position_map():
    """The module's packed ids / types / positions and masked rows equal the oracle's restatement."""
    G = 5
    model, b, mask, _ = _grouped(G)
    d = synth.SMALL_L123
    P, T, Lp = GO.geometry(d, G)
    ids, tt, pos, flat = model._pack_captions(b["img"], b["input_ids"], b["segment_ids"], mask, b["masked_pos"], G, None, False, False)
    src = GO.packed_rows(d, G)
    for img in range(2):
        for k, (g, r) in enumerate(src):
            assert ids[img, k] == b["input_ids"][img * G + g, r] and tt[img, k] == b["segment_ids"][img * G + g, r]
            assert pos[img, k] == r
    want = GO.masked_rows(b["masked_pos"], G, P, T) + (torch.arange(2 * G) // G * Lp).unsqueeze(1)
    assert torch.equal(flat, want)
    mp = torch.tensor([[0, 50, P, P + 3], [P - 1, P + T - 1, 1, P]] * G)
    got = GO.masked_rows(mp, G, P, T)
    assert got[1].tolist() == [P - 1, P + T + T - 1, 1, P + T]      # pair 1 is caption 1 of image 0
    assert torch.equal(got[G], mp[G])                                 # pair G is caption 0 of image 1


def _refused(fn, match):
    from tools import abi_cases
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match=match):
            fn()
    assert calls == []


def test_refusals_before_any_launch():
    G = 5
    model, b, mask, _ = _grouped(G)
    _refused(lambda: _call(model, b, mask, captions_per_image=G, mask_image_regions=True), "mask_image_regions")
    _refused(lambda: _call(model, b, b["input_mask"], captions_per_image=G), "GroupedCaptionMask")
    _refused(lambda: _call(model, b, mask, captions_per_image=2), "groups 5 captions")
    _refused(lambda: _call(model, b, mask), "groups 5 captions")
    odd = dict(b, input_ids=b["input_ids"][:-1])
    _refused(lambda: _call(model, odd, mask, captions_per_image=G), "whole images")
    more = dict(b, img=b["img"].repeat(2, 1, 1))
    _refused(lambda: _call(model, more, mask, captions_per_image=G), "vis_feats has 4 rows")
    _refused(lambda: _call(model, b, mask, captions_per_image=G, vqa_inference=True), "VQA")
    vqa, bv, mv, _ = _grouped(G, tasks="vqa2")
    _refused(lambda: _call(vqa, bv, mv, captions_per_image=G), "VQA")
    with pytest.raises(ValueError, match="pack to 522 rows"):
        staging.GroupedCaptionMask.check(20, 100, 123)
    assert staging.GroupedCaptionMask.check(19, 100, 123) == (21, 501)
    too_long = staging.GroupedCaptionMask(mask.bits, 20, 21, 100, 123)
    _refused(lambda: _call(model, b, too_long, captions_per_image=20), "pack to 522 rows")
    bi = synth.make_batch(synth.SMALL_L123, 4, seed=3, mode="bi")["input_mask"]
    with pytest.raises(ValueError, match="bidirectional"):
        staging.GroupedCaptionMask.from_pair_masks(bi, 2, 100)


def test_grouped_step_marshalling_dry_run():
    """A grouped training step with the library call replaced by prototype conversion: region projections on B images, one packed
    embedding and encoder pass, the head over the B * G pairs; the mask from len_b in one vlpk_mask_synth_grouped."""
    from tools import abi_cases
    G = 5
    model, b, _, len_b = _grouped(G)
    with abi_cases.dry_run() as calls:
        mask = staging.GroupedCaptionMask.synthesize(len_b, G, 100, 123)
        out = _call(model, b, mask, captions_per_image=G)
        sum(l.float().sum() for l in out).backward()
    assert mask.bits.shape == (2, 207, 8)
    assert calls == ["vlpk_mask_synth_grouped"] + ["vlpk_linear_fwd"] * 3 + ["vlpk_embed_fwd", "vlpk_encoder_fwd", "vlpk_decoder_ce_fwd",
                     "vlpk_decoder_ce_bwd", "vlpk_encoder_bwd", "vlpk_f32_to_bf16", "vlpk_embed_bwd", "vlpk_embed_tables_bwd"] + \
        ["vlpk_linear_bwd"] * 3
    assert model.last_prediction_scores.shape == (2 * G, 3, synth.SMALL_L123.vocab)
    for n, p in model.named_parameters():
        if p.grad is not None:
            assert p.grad.shape == p.shape, n


def test_positions_not_packed_length_meet_max_position_embeddings():
    """Packed rows keep their pair's positions, all below L: a table of L positions serves L' = 207 rows, and a shorter one is refused
    at L before any launch."""
    from tools import abi_cases
    import dataclasses
    G = 5
    for max_pos, ok in ((123, True), (122, False)):
        d = dataclasses.replace(synth.SMALL_L123, max_pos=max_pos)
        model = vm.BertForPreTrainingLossMask(_cfg(d), enable_butd=True, len_vis_input=d.regions).bfloat16().train()
        _, b, _, len_b = _grouped(G)
        if ok:
            with abi_cases.dry_run() as calls:
                _call(model, b, staging.GroupedCaptionMask.synthesize(len_b, G, 100, 123), captions_per_image=G)
            assert "vlpk_encoder_fwd" in calls
        else:
            mask = staging.GroupedCaptionMask(torch.zeros(2, 207, 8, dtype=torch.int32), G, 21, 100, 123)
            _refused(lambda: _call(model, b, mask, captions_per_image=G), "max_position_embeddings 122")
