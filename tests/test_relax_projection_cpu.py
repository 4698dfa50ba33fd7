"""Relaxed per-task MLM head projection (config.relax_projection = n > 1, modeling.py:420-482, from_pretrained :704-732) without a GPU:
the oracle (tools/relax_projection_oracle.py) against the unmodified reference's stored outputs (tests/golden/relax_projection.pt), the
state_dict contract, from_pretrained's relaxed <-> plain remaps bit for bit, the task select against the reference's indexing, the
C-ABI call sequence of a relaxed training step and the task_idx checks."""
import os

import pytest
import torch

from oracle import make_golden as mg
from tools import relax_projection_oracle as RPO
from vlp_b200 import synth
from vlp_b200 import vlp_modules as vm

HEAD = RPO.HEAD


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "relax_projection.pt"))


def make_config(d, relax=0, label_smoothing=None):
    return vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                         type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, relax_projection=relax,
                         label_smoothing=label_smoothing)


# ---- oracle vs the reference ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(RPO.CASES))
def test_oracle_matches_reference_golden_with_relaxed_head(name, gold):
    g = gold["cases"][name]
    dims, sd, batch, n, eps = RPO.inputs(name)
    assert g["relax_projection"] == n and g["label_smoothing"] == eps
    assert set(batch["task_idx"].tolist()) == {0, 3}                     # both task slices are selected, 1 and 2 never
    for k, v in sd.items():
        if k != "cls.predictions.decoder.weight":
            v.requires_grad_(True)
    losses, aux = RPO.pretraining_loss(sd, dims, batch, n, eps, return_all=True)
    sum(l.sum() for l in losses).backward()
    for got, ref in zip(losses, g["losses"]):
        assert abs(float(got.detach()) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref)))
    assert rel(RPO.sample(aux["embedding"]), g["embedding"]) < 1e-5
    assert len(aux["layers"]) == len(g["layers"])
    for got, ref in zip(aux["layers"], g["layers"]):
        assert rel(RPO.sample(got), ref) < 1e-5
    assert rel(RPO.sample(aux["logits"]), g["logits"]) < 1e-5
    assert rel(RPO.sample(aux["pooled"]), g["pooled"]) < 1e-5
    scale = max(float(fp["full"].norm()) if "full" in fp else fp["norm"] for fp in g["grads"].values())
    for k, fp in g["grads"].items():
        got = sd[k].grad
        assert got is not None, k
        if "full" in fp:
            if fp["full"].norm() <= 1e-7 * scale:           # zero in exact arithmetic (key bias): round-off level only
                assert got.norm() <= 1e-7 * scale, k
            else:
                assert rel(got, fp["full"]) < 1e-4, k
        else:
            assert abs(got.norm().item() - fp["norm"]) <= 1e-4 * fp["norm"] + 1e-12, k
            assert rel(RPO.sample(got, RPO.GRAD_SAMPLES), fp["sample"]) < 1e-4, k
    H = dims.hidden
    for k in ("dense.weight", "dense.bias", "LayerNorm.weight", "LayerNorm.bias"):
        ref, got = g["grads"][HEAD + k]["full"], sd[HEAD + k].grad
        assert ref.shape[0] == n * H
        for s in range(n):
            r, o = ref[s * H:(s + 1) * H], got[s * H:(s + 1) * H]
            if k.startswith("LayerNorm") and s in (1, 2):
                # never selected: the LayerNorm's affine parameters of these slices reach no output
                assert float(r.abs().max()) == 0.0 and float(o.abs().max()) == 0.0, (k, s)
            else:
                # slices 1 and 2 of dense receive gradient through the LayerNorm statistics only
                assert float(r.norm()) > 0 and rel(o, r) < 1e-4, (k, s, rel(o, r))


def test_relaxed_head_differs_from_each_plain_slice(gold):
    """The golden really exercises per-sample selection: the loss differs from the one every sample would get on slice 0 or 3 alone."""
    name = "l123_mix_relax4"
    dims, sd, batch, n, eps = RPO.inputs(name)
    with torch.no_grad():
        mixed = float(RPO.pretraining_loss(sd, dims, batch, n, eps)[0])
        assert abs(mixed - float(gold["cases"][name]["losses"][0])) < 1e-5
        for t in (0, 3):
            b = dict(batch, task_idx=torch.full_like(batch["task_idx"], t))
            assert abs(float(RPO.pretraining_loss(sd, dims, b, n, eps)[0]) - mixed) > 1e-4


# ---- module surface ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(RPO.CASES))
def test_relaxed_state_dict_matches_reference(name, gold):
    g = gold["cases"][name]
    dims, sd, _, n, eps = RPO.inputs(name)
    model = vm.BertForPreTrainingLossMask(make_config(dims, n, eps), enable_butd=True, len_vis_input=dims.regions)
    assert {k: tuple(v.shape) for k, v in model.state_dict().items()} == g["state_dict_shapes"]
    res = model.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys and set(res.missing_keys) <= {"crit_mask_lm_smoothed.one_hot"}
    assert model.cls.predictions.relax_projection == n


def test_select_task_is_the_reference_indexing():
    """select_task == view(B, P, n, H)[arange(B), :, task_idx, :] bit for bit (fp32 and bf16; [B], 0-d and int ids); its gradient is the
    upstream gradient in the selected slice and exactly 0 elsewhere."""
    d = synth.TINY
    head = vm.BertLMPredictionHead(make_config(d, 4), torch.nn.Parameter(torch.zeros(d.vocab, d.hidden)))
    gen = torch.Generator().manual_seed(3)
    B, P, H = 5, 3, d.hidden
    for dtype in (torch.float32, torch.bfloat16):
        x = torch.randn(B, P, 4 * H, generator=gen).to(dtype).requires_grad_(True)
        t = torch.tensor([3, 0, 2, 1, 3])
        for ids in (t, torch.tensor(2), 1):
            want = x.view(B, P, 4, H)[torch.arange(B), :, ids, :]
            got = head.select_task(x, ids)
            assert got.shape == (B, P, H) and torch.equal(got, want)
        dy = torch.randn(B, P, H, generator=gen).to(dtype)
        (gx,) = torch.autograd.grad(head.select_task(x, t), x, dy)
        gx = gx.view(B, P, 4, H)
        for b in range(B):
            for s in range(4):
                assert torch.equal(gx[b, :, s], dy[b] if s == int(t[b]) else torch.zeros_like(dy[b]))
    plain = vm.BertLMPredictionHead(make_config(d), torch.nn.Parameter(torch.zeros(d.vocab, d.hidden)))
    x = torch.randn(2, 3, H)
    assert plain.relax_projection == 0 and plain.select_task(x, None) is x


def test_invalid_task_idx_raises_before_anything_runs():
    d = synth.TINY
    head = vm.BertLMPredictionHead(make_config(d, 4), torch.nn.Parameter(torch.zeros(d.vocab, d.hidden)))
    x = torch.randn(2, 3, 4 * d.hidden)
    for bad in (None, torch.tensor([0, 4]), torch.tensor([-1, 3]), 4, -1, torch.tensor([0.0, 1.0]), True, "3"):
        with pytest.raises(ValueError):
            head.select_task(x, bad)
    with pytest.raises(ValueError):
        head.select_task(x, torch.tensor([0, 1, 2]))                     # three ids for a batch of two
    # the model forwards check before the first library call: no CUDA tensor is needed to hit the ValueError
    model = vm.BertForPreTrainingLossMask(make_config(d, 4), enable_butd=True, len_vis_input=d.regions)
    b = synth.make_batch(d, 2, seed=1)
    for bad in (None, torch.tensor([3, 4])):
        with pytest.raises(ValueError):
            model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None, b["is_next"],
                  masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=bad, drop_worst_ratio=0.0)
    dec = vm.BertForSeq2SeqDecoder(make_config(d, 4), mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=d.regions)
    args = RPO.decode_inputs(d, 2, 1)
    for bad in (None, torch.tensor([0, 7])):
        with pytest.raises(ValueError):
            dec(*args, task_idx=bad)


def test_unsupported_configs_still_raise_and_relax_is_accepted():
    with pytest.raises(NotImplementedError):
        vm.BertLayer(vm.BertConfig(100, hidden_size=128, num_attention_heads=2, intermediate_size=512, hidden_act="relu", relax_projection=4))
    vm.BertLayer(vm.BertConfig(100, hidden_size=128, num_attention_heads=2, intermediate_size=512, relax_projection=4))


# ---- from_pretrained -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(RPO.FROM_PRETRAINED))
def test_from_pretrained_relax_remaps_match_reference(case, tmp_path, gold):
    """Compared parameter by parameter, bit for bit, with the unmodified reference's from_pretrained on the same checkpoint."""
    write, sds, kw = RPO.from_pretrained_checkpoints()
    ckpt, extra = RPO.FROM_PRETRAINED[case]
    write(str(tmp_path))
    mine = vm.BertForPreTrainingLossMask.from_pretrained(str(tmp_path), state_dict={k: v.clone() for k, v in sds[ckpt].items()}, **kw,
                                                         **extra)
    want = gold["from_pretrained"]["digests"][case]
    a = mine.state_dict()
    assert set(a.keys()) == set(want.keys())
    for k in a:
        assert mg.tensor_digest(a[k]) == want[k], k
    H = a["bert.embeddings.word_embeddings.weight"].shape[1]
    src = sds[ckpt][HEAD + "dense.weight"]
    if case == "plain_to_relax4":
        assert torch.equal(a[HEAD + "dense.weight"], src.repeat(4, 1))
    else:
        s = 3 if "task3" in case else 0
        assert torch.equal(a[HEAD + "dense.weight"], src[s * H:(s + 1) * H])


def test_from_pretrained_task_idx_zero_behaves_like_unset(tmp_path, gold):
    """The reference sets config.task_idx only for a truthy kwarg (modeling.py:622-623): task_idx=0 keeps slice 0 through the default."""
    write, sds, kw = RPO.from_pretrained_checkpoints()
    write(str(tmp_path))
    mine = vm.BertForPreTrainingLossMask.from_pretrained(str(tmp_path), state_dict={k: v.clone() for k, v in sds["relax4"].items()},
                                                         relax_projection=0, task_idx=0, **kw)
    assert mine.config.task_idx is None
    want = gold["from_pretrained"]["digests"]["relax4_to_plain_unset"]
    assert all(mg.tensor_digest(v) == want[k] for k, v in mine.state_dict().items())


def test_from_pretrained_relax_mismatch_raises(tmp_path, gold):
    assert gold["from_pretrained"]["mismatch"]["raised"] == "AssertionError"      # the reference asserts; here it is a ValueError
    write, sds, kw = RPO.from_pretrained_checkpoints()
    ckpt, extra = RPO.MISMATCH
    write(str(tmp_path))
    with pytest.raises(ValueError, match="relax_projection"):
        vm.BertForPreTrainingLossMask.from_pretrained(str(tmp_path), state_dict={k: v.clone() for k, v in sds[ckpt].items()}, **kw, **extra)


# ---- C ABI ---------------------------------------------------------------------------------------------------------------------
def _dry_run_step(relax, eps=None):
    from tools import abi_cases
    d = synth.TINY
    model = vm.BertForPreTrainingLossMask(make_config(d, relax, eps), enable_butd=True, len_vis_input=d.regions).bfloat16().train()
    b = synth.make_batch(d, 3, seed=1503, mode="mix")
    with abi_cases.dry_run() as calls:
        out = model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None,
                    b["is_next"], masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"],
                    vis_masked_pos=b["vis_masked_pos"], mask_image_regions=False, drop_worst_ratio=0.0)
        sum(l.float().sum() for l in out).backward()
    for n, p in model.named_parameters():
        if not n.startswith("bert.pooler."):
            assert p.grad is not None and p.grad.shape == p.shape and p.grad.dtype == p.dtype, n
    return calls


@pytest.mark.parametrize("eps", [None, 0.1])
def test_relaxed_training_step_makes_the_plain_library_calls(eps):
    """The relaxed head is a PyTorch-side change: a relaxed training step calls the library exactly as the plain step does."""
    plain = _dry_run_step(0, eps)
    assert ("vlpk_decoder_ce_ls_fwd" if eps else "vlpk_decoder_ce_fwd") in plain
    assert _dry_run_step(4, eps) == plain


def test_relaxed_beam_search_marshalling_dry_run():
    """Beam search with a per-sample task_idx at B = 2 (the reference only runs B = 1): task_idx follows the beams."""
    from tools import abi_cases
    d = synth.TINY
    model = vm.BertForSeq2SeqDecoder(make_config(d, 4), mask_word_id=103, eos_id=102, search_beam_size=3, enable_butd=True,
                                     len_vis_input=d.regions).bfloat16().eval()
    vis, pe, input_ids, tt, pos, mask = RPO.decode_inputs(d, 2, 4)
    seen = []
    model.cls.predictions.register_forward_hook(lambda m, i, o: seen.append(tuple(o.shape)))
    with abi_cases.dry_run():
        tr = model(vis.bfloat16(), pe.bfloat16(), input_ids, tt, pos, mask, task_idx=torch.tensor([3, 0]))
    assert tr["wids"].shape == (2, d.seq_len, 3)
    assert seen[0][0] == 2 and all(s[0] == 6 for s in seen[1:])
