"""Region masking (mask_image_regions=True, --vis_mask_prob) and the drop-worst normalisation on the plain path, host side: the oracle
against the unmodified reference's stored outputs, the synthesised loader mask against a restatement of the loader, the module's
pretext loss against the oracle's, describe_mask's refusal of a matrix with blocked region columns, and the marshalling of a
region-masked step."""
import os

import pytest
import torch

from oracle import vlp_oracle as O
from tools import abi_cases
from tools import label_smoothing_oracle as LS
from tools import region_masking_oracle as RM
from vlp_b200 import staging, synth
from vlp_b200 import vlp_modules as vm


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def _leaf(sd, dtype=torch.float32):
    sd = {k: v.to(dtype) for k, v in sd.items()}
    sd["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]
    for k, v in sd.items():
        if k != "cls.predictions.decoder.weight":
            v.requires_grad_(True)
    return sd


@pytest.mark.parametrize("name", list(RM.CASES))
def test_oracle_matches_reference_golden(name, golden_dir):
    """oracle/vlp_oracle.pretraining_loss(mask_image_regions=...) against the reference's stored outputs, test_oracle.py's bounds:
    1e-5 on losses and activations, 1e-4 on gradients."""
    gold = torch.load(os.path.join(golden_dir, "region_masking.pt"))["cases"][name]
    dims, sd, batch, tasks, mir, dw = RM.inputs(name)
    if dims.hidden > 128:
        torch.set_num_threads(max(torch.get_num_threads(), 8))
    sd = _leaf(sd)
    losses, aux = O.pretraining_loss(sd, dims, batch, tasks=tasks, drop_worst_ratio=dw, return_all=True, mask_image_regions=mir)
    for got, ref in zip(losses, gold["losses"]):
        assert abs(float(got) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref))), (float(got), float(ref))
    assert (float(losses[1]) > 0) == mir
    assert rel(LS.sample(aux["embedding"]), gold["embedding"]) < 1e-5
    for got, ref in zip(aux["layers"], gold["layers"]):
        assert rel(LS.sample(got), ref) < 1e-5
    if tasks != "vqa2":
        assert rel(LS.sample(aux["logits"]), gold["logits"]) < 1e-5
    assert rel(aux["pooled"], gold["pooled"]) < 1e-5
    sum(l.sum() for l in losses).backward()
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
            assert rel(g.flatten()[LS.sample_idx(g.numel(), LS.GRAD_SAMPLES)], fp["sample"]) < 1e-4, k


def test_golden_drift_is_stored_and_the_pretext_bound_follows_it(golden_dir):
    """The reference's own fp32 -> bf16 drift is stored with every case; the GPU bound of the pretext loss is derived from it."""
    cases = torch.load(os.path.join(golden_dir, "region_masking.pt"))["cases"]
    for name, gold in cases.items():
        _, _, _, _, mir, _ = RM.inputs(name)
        d = gold["drift"]
        assert set(d["grads"]) == set(gold["grads"]) and len(d["layers"]) == len(gold["layers"])
        assert RM.loss_bound(gold, 1) >= RM.LOSS_FLOOR
        if mir:
            assert d["losses"][1] > 0                 # the bf16 run really moved the pretext loss


def test_synth_default_is_unchanged_and_region_draws_follow_the_loader():
    d = synth.SMALL_L123
    plain = synth.make_batch(d, 6, seed=9, mode="mix", ragged=True)
    assert plain["vis_masked_pos"].shape == (6, 0)
    assert torch.equal(plain["input_mask"], synth.make_batch(d, 6, seed=9, mode="mix", ragged=True, vis_mask_prob=0.0)["input_mask"])
    for p, n in ((0.25, 25), (0.15, 15), (0.999, 99)):
        b = synth.make_batch(d, 6, seed=9, mode="mix", ragged=True, vis_mask_prob=p)
        for k in synth.make_batch(d, 1).keys():
            if k not in ("vis_masked_pos", "input_mask"):
                assert torch.equal(b[k], plain[k]), k
        vm_ = b["vis_masked_pos"]
        assert vm_.shape == (6, n) and vm_.dtype == torch.long
        assert int(vm_.min()) >= 1 and int(vm_.max()) <= d.regions
        assert all(len(set(r.tolist())) == n for r in vm_)


def _loader_mask(d, n_tokens, mode, vis_masked_pos):
    """seq2seq_loader.py:291-304 for one sample, statement by statement."""
    max_len, len_a = d.seq_len, d.regions
    len_b = n_tokens - len_a - 3
    n_pad = max_len - n_tokens
    input_mask = torch.zeros(max_len, max_len, dtype=torch.long)
    second_st, second_end = len_a + 2, len_a + len_b + 3
    if mode == "s2s":
        input_mask[:, :len_a + 2].fill_(1)
        tril = torch.tril(torch.ones(max_len, max_len, dtype=torch.long))
        input_mask[second_st:second_end, second_st:second_end].copy_(tril[:second_end - second_st, :second_end - second_st])
    else:
        input_mask = torch.tensor([1] * n_tokens + [0] * n_pad, dtype=torch.long).unsqueeze(0).expand(max_len, max_len).clone()
    if len(vis_masked_pos):
        input_mask[:, vis_masked_pos].fill_(0)
    return input_mask


@pytest.mark.parametrize("dims", [synth.SMALL_L123, synth.TINY])
@pytest.mark.parametrize("p", [0.0, 0.25])
def test_synthesised_loader_mask_restates_the_loader(dims, p):
    """The loader's region 'blocking' (:303-304) fills the copy an index array returns, so its matrix is the plain one — as here."""
    b = synth.make_batch(dims, 8, seed=4, mode="mix", ragged=True, vis_mask_prob=p)
    assert b["vis_masked_pos"].shape[1] == int(dims.regions * p)
    import numpy as np
    for i in range(8):
        n_tokens = int((b["input_ids"][i] != 0).sum())
        mode = "s2s" if int(b["task_idx"][i]) == 3 else "bi"
        pos = b["vis_masked_pos"][i].numpy().astype(np.int64)     # np.random.choice(...) + 1 in the loader
        assert torch.equal(b["input_mask"][i], _loader_mask(dims, n_tokens, mode, pos)), i
    plain = synth.make_batch(dims, 8, seed=4, mode="mix", ragged=True)
    assert torch.equal(b["input_mask"], plain["input_mask"])


def test_module_pretext_matches_oracle_float64():
    """BertForPreTrainingLossMask._loss_tail's pretext (modeling.py:1113-1131), which evaluates in fp32 whatever the input dtype,
    against oracle.region_pretext_loss in float64: the loss and its gradients into the projected features, the projected position
    encodings and the pooled output, within fp32 round-off."""
    d = synth.SMALL_L123
    model = vm.BertForPreTrainingLossMask(vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers,
                                                        num_attention_heads=d.heads, intermediate_size=d.inter),
                                          enable_butd=True, len_vis_input=d.regions)
    g = torch.Generator().manual_seed(3)
    B, H = 3, d.hidden
    pos = synth.make_batch(d, B, seed=5, vis_mask_prob=0.25)["vis_masked_pos"]
    pos[0, :2] = torch.tensor([1, d.regions])                 # the first and the last region
    x = [(torch.randn(B, d.regions, H, generator=g, dtype=torch.float64) * s).requires_grad_(True) for s in (0.3, 0.3)]
    pooled = torch.randn(B, H, generator=g, dtype=torch.float64).tanh().requires_grad_(True)
    outs = []
    for fn in (lambda v, pe, po: model._loss_tail(torch.zeros(1, dtype=torch.float64), None, po, v, pe, pos, True, None)[1],
               lambda v, pe, po: O.region_pretext_loss(v, pe, po, pos)):
        loss = fn(x[0], x[1], pooled)
        grads = torch.autograd.grad(loss, [x[0], x[1], pooled])
        outs.append((loss.detach(), grads))
    (l0, g0), (l1, g1) = outs
    assert abs(float(l0) - float(l1)) <= 1e-6 * abs(float(l1))
    for a, b_, nm in zip(g0, g1, ("vis", "vpe", "pooled")):
        assert float((a.double() - b_).abs().max()) <= 1e-5 * float(b_.abs().max()), nm
    rows = torch.zeros(B, d.regions, dtype=torch.bool)
    rows.scatter_(1, pos - 1, True)
    assert bool((g1[0][~rows] == 0).all()) and bool((g1[0][rows].abs().sum(-1) > 0).all())   # only the masked rows get a gradient


def test_masked_regions_change_only_the_pretext_float64():
    """Oracle, float64: new input features at the masked regions leave the embedding output, every layer and the masked-LM loss
    exactly as they were, and move the pretext loss."""
    dims, sd, batch, tasks, mir, dw = RM.inputs("l123_s2s_vm25")
    sd = {k: v.double() for k, v in sd.items()}
    sd["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]
    b0 = {k: (v.double() if v.is_floating_point() else v) for k, v in batch.items()}
    b1 = dict(b0, img=b0["img"].clone(), vis_pe=b0["vis_pe"].clone())
    for i in range(b1["img"].shape[0]):
        r = b1["vis_masked_pos"][i] - 1
        b1["img"][i, r] = b1["img"][i, r].flip(0) + 0.5
        b1["vis_pe"][i, r] = -b1["vis_pe"][i, r]
    with torch.no_grad():
        (m0, p0, _), a0 = O.pretraining_loss(sd, dims, b0, return_all=True, mask_image_regions=True)
        (m1, p1, _), a1 = O.pretraining_loss(sd, dims, b1, return_all=True, mask_image_regions=True)
    assert torch.equal(a0["embedding"], a1["embedding"]) and all(torch.equal(x, y) for x, y in zip(a0["layers"], a1["layers"]))
    assert torch.equal(m0, m1) and abs(float(p1) - float(p0)) > 1e-3


def blocked(batch):
    """The batch's loader matrices with the key columns of its masked regions blocked — what seq2seq_loader.py:303-304 means to
    build ("block the masked visual feature")."""
    m = batch["input_mask"].clone()
    for i, pos in enumerate(batch["vis_masked_pos"]):
        m[i][:, pos] = 0
    return m


def test_describe_mask_refuses_a_matrix_with_blocked_regions():
    """describe_mask returns (len_b, mode) only for a matrix it reproduces exactly.  With blocked region columns the diagonal is
    short by the masked regions and the old reading returned a wrong len_b (and may call a pair bidirectional); such a matrix is
    refused, also through GroupedCaptionMask.from_pair_masks, before any launch."""
    for d in (synth.SMALL_L123, synth.TINY, synth.BERT_BASE):
        b = synth.make_batch(d, 8, seed=6, mode="mix", ragged=True, vis_mask_prob=0.25)
        len_b, s2s = staging.describe_mask(b["input_mask"], d.regions)
        assert torch.equal(staging.loader_mask(len_b, s2s, d.regions, d.seq_len).long(), b["input_mask"])
        assert torch.equal(s2s.long(), (b["task_idx"] == 3).long())
        with pytest.raises(ValueError, match="blocked region columns"):
            staging.describe_mask(blocked(b), d.regions)
        one = b["input_mask"].clone()
        one[5, :, 3] = 0                                      # one blocked region in one sample
        with pytest.raises(ValueError, match=r"sample\(s\) \[5\]"):
            staging.describe_mask(one, d.regions)
    d = synth.SMALL_L123
    b = synth.make_batch(d, 4, seed=6, mode="s2s", ragged=True, vis_mask_prob=0.25)
    with abi_cases.dry_run() as calls:
        with pytest.raises(ValueError, match="blocked region columns"):
            staging.GroupedCaptionMask.from_pair_masks(blocked(b), 2, d.regions)
    assert calls == []


def _cfg(d, drop=0.0):
    return vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                         type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=drop,
                         attention_probs_dropout_prob=drop)


@pytest.mark.parametrize("tasks", ["img2txt", "vqa2"])
def test_region_masked_step_marshalling_dry_run(tasks):
    """A region-masked training step with the library call replaced by prototype conversion: the same launches as the unmasked step
    (the zeroing and the pretext are torch ops around them), every gradient of its parameter's shape."""
    d = synth.SMALL_L123
    model = vm.BertForPreTrainingLossMask(_cfg(d, 0.1), enable_butd=True, len_vis_input=d.regions, tasks=tasks).bfloat16().train()
    seqs = []
    for p in (0.0, 0.25):
        b = synth.make_batch(d, 3, seed=8, mode="bi" if tasks == "vqa2" else "s2s", tasks=tasks, vis_mask_prob=p)
        model.zero_grad(set_to_none=True)
        with abi_cases.dry_run() as calls:
            out = model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"],
                        b["ans_labels"] if tasks == "vqa2" else None, b["is_next"], masked_pos=b["masked_pos"],
                        masked_weights=b["masked_weights"], task_idx=b["task_idx"], vis_masked_pos=b["vis_masked_pos"],
                        mask_image_regions=p > 0, drop_worst_ratio=0.2)
            sum(l.float().sum() for l in out).backward()
        seqs.append(list(calls))
        for n, prm in model.named_parameters():
            if prm.grad is not None:
                assert prm.grad.shape == prm.shape, n
    assert seqs[0] == seqs[1]
    assert seqs[1].count("vlpk_linear_fwd") == 3 and seqs[1].count("vlpk_linear_bwd") == 3 and "vlpk_embed_bwd" in seqs[1]
