"""Label-smoothed masked-LM loss (config.label_smoothing, crit_mask_lm_smoothed = LabelSmoothingLoss, modeling.py:995-999, 1104-1106)
without a GPU: the oracle (tools/label_smoothing_oracle.py) against the reference's stored outputs (tests/golden/label_smoothing.pt), a model of the smoothed row
kernels' reduction order (csrc/head.cu, decoder_ce_*_kernel<true>) against the reference's kl_div formula, the state_dict contract,
the C-ABI marshalling of a training step and the argument checks of vlpk_decoder_ce_ls_fwd/bwd."""
import json
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import make_golden as mg
from oracle import vlp_oracle as O
from tools import label_smoothing_oracle as LSO
from vlp_b200 import _lib, synth
from vlp_b200 import vlp_modules as vm


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "label_smoothing.pt"))["cases"]


def make_config(d, label_smoothing=None, drop=0.1):
    return vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                         type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=drop,
                         attention_probs_dropout_prob=drop, label_smoothing=label_smoothing)


# ---- oracle vs the reference ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(LSO.CASES))
def test_oracle_matches_reference_golden_with_label_smoothing(name, gold):
    g = gold[name]
    dims, sd, batch, eps = LSO.inputs(name)
    assert g["label_smoothing"] == eps
    b, j = LSO.ZERO_LABEL
    assert batch["masked_ids"][b, j] == 0 and batch["masked_weights"][b, j] == 1
    for k, v in sd.items():
        if k != "cls.predictions.decoder.weight":
            v.requires_grad_(True)
    losses, aux = LSO.pretraining_loss(sd, dims, batch, eps, return_all=True)
    sum(l.sum() for l in losses).backward()
    for got, ref in zip(losses, g["losses"]):
        assert abs(float(got.detach()) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref)))
    assert rel(LSO.sample(aux["embedding"]), g["embedding"]) < 1e-5
    assert len(aux["layers"]) == len(g["layers"])
    for got, ref in zip(aux["layers"], g["layers"]):
        assert rel(LSO.sample(got), ref) < 1e-5
    assert rel(LSO.sample(aux["logits"]), g["logits"]) < 1e-5
    assert rel(LSO.sample(aux["pooled"]), g["pooled"]) < 1e-5
    scale = max(float(fp["full"].norm()) if "full" in fp else fp["norm"] for fp in g["grads"].values())
    n = 0
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
            assert rel(LSO.sample(got, LSO.GRAD_SAMPLES), fp["sample"]) < 1e-4, k
        n += 1
    assert n >= 40


def test_smoothed_loss_differs_from_cross_entropy_and_ignores_label_zero(gold):
    """The golden really exercises the smoothed loss: it differs from the cross-entropy on the same inputs, and the forced label-0
    position changes the loss only through the denominator of loss_mask_and_normalize."""
    name = "l123_mix_ls01"
    dims, sd, batch, eps = LSO.inputs(name)
    with torch.no_grad():
        ce = float(O.pretraining_loss(sd, dims, batch)[0])
        ls = float(LSO.pretraining_loss(sd, dims, batch, eps)[0])
        assert abs(ls - float(gold[name]["losses"][0])) < 1e-5 and abs(ls - ce) > 1e-3
        b, j = LSO.ZERO_LABEL
        unweighted = {k: v.clone() for k, v in batch.items()}
        unweighted["masked_weights"][b, j] = 0
        n = float(batch["masked_weights"].sum())
        assert abs(float(LSO.pretraining_loss(sd, dims, unweighted, eps)[0]) * (n - 1) - ls * n) < 1e-4


def test_label_smoothing_module_matches_the_dense_kl_div():
    """vlp_modules.LabelSmoothingLoss (closed form, the torch comparison arm) vs the reference's dense-target kl_div, forward and
    gradient, and the buffer of the reference (loss.py:29-31)."""
    gen = torch.Generator().manual_seed(4)
    for V, eps in ((29, 0.1), (1003, 0.1), (1003, 1.0)):
        crit = vm.LabelSmoothingLoss(eps, V, ignore_index=0, reduction="none")
        assert crit.one_hot.shape == (1, V) and float(crit.one_hot[0, 0]) == 0.0
        assert torch.equal(crit.one_hot[0, 1:], torch.full((V - 1,), eps / (V - 2)))
        x = (torch.randn(3, 4, V, generator=gen) * 3).requires_grad_(True)
        t = torch.randint(1, V, (3, 4), generator=gen)
        t[0, 1], t[2, 3] = 0, V - 1
        crit(F.log_softmax(x, -1), t).sum().backward()
        got = x.grad.clone()
        x.grad = None
        loss = crit(F.log_softmax(x, -1), t)
        ref = LSO.label_smoothing_loss(F.log_softmax(x, -1), t, eps, V)
        ref.sum().backward()
        assert loss.shape == (3, 4) and float(loss[0, 1].detach()) == 0.0
        assert torch.allclose(loss, ref, atol=2e-5, rtol=1e-5)
        assert torch.allclose(got, x.grad, atol=1e-6)
    with pytest.raises(ValueError):
        vm.LabelSmoothingLoss(0.0, 100)
    with pytest.raises(ValueError):
        vm.LabelSmoothingLoss(1.5, 100)
    with pytest.raises(ValueError):
        vm.LabelSmoothingLoss(0.1, 2)


# ---- model of the smoothed row kernels -----------------------------------------------------------------------------------------
def _online_merge(m, s, m2, s2):            # head.cu online_merge
    mn = max(m, m2)
    return mn, s * math.exp(m - mn) + s2 * math.exp(m2 - mn)


def _smoothing_constants(V, eps):           # head.cu smoothing(): double on the host, rounded to fp32
    e = float(np.float32(eps))
    c, s = 1.0 - e, e / (V - 2)
    k = (c * math.log(c) if c > 0 else 0.0) + (V - 2) * s * math.log(s)
    return np.float32(c), np.float32(s), np.float32(k)


def _smoothed_fwd_row(x, V, y, eps, THREADS=256):
    """decoder_ce_fwd_kernel<true> for one row x (fp32 values of bf16 logits, length Vp): per-thread 8-column stripes with stride
    8 * THREADS (online max / sum, and the fp32 stripe sum added to the thread's S), a butterfly over each warp, then thread 0 merges
    the warps in order.  Returns (lse, loss, columns visited)."""
    f32 = np.float32
    seen = np.zeros(V, dtype=np.int64)
    ms, ss, zs = [], [], []
    for tid in range(THREADS):
        m, s, z = -3.0e38, 0.0, f32(0)
        for c in range(tid * 8, V, THREADS * 8):
            cols = [c + j for j in range(8) if c + j < V]
            seen[cols] += 1
            v = [float(x[k]) for k in cols]
            cm = max(v)
            m, s = _online_merge(m, s, cm, sum(math.exp(a - cm) for a in v))
            cz = f32(0)
            for k in cols:
                cz = f32(cz + f32(x[k]))
            z = f32(z + cz)
        ms.append(m)
        ss.append(s)
        zs.append(z)
    warp_z = []
    for w in range(THREADS // 32):
        lane = list(zs[32 * w:32 * w + 32])
        for o in (16, 8, 4, 2, 1):
            lane = [f32(lane[i] + lane[i ^ o]) for i in range(32)]
        warp_z.append(lane[0])
    M, S = ms[0], ss[0]
    for m2, s2 in zip(ms[1:], ss[1:]):
        M, S = _online_merge(M, S, m2, s2)
    lse = f32(M + math.log(S))
    Z = warp_z[0]
    for v in warp_z[1:]:
        Z = f32(Z + v)
    if not (0 < y < V):
        return lse, f32(0), seen
    c, s, k = _smoothing_constants(V, eps)
    xt, x0 = f32(x[y]), f32(x[0])
    return lse, f32(k + lse - c * xt - s * (Z - x0 - xt)), seen


@pytest.mark.parametrize("eps", [0.1, 1.0])
@pytest.mark.parametrize("V", [29, 1003, 8 * 256 + 5])
def test_smoothed_decoder_row_model_matches_kl_div(V, eps):
    gen = torch.Generator().manual_seed(V)
    Vp = (V + 7) // 8 * 8
    R = 6
    logits = torch.zeros(R, Vp)
    logits[:, :V] = (torch.randn(R, V, generator=gen) * 3 + 0.5).bfloat16().float()
    labels = torch.randint(1, V, (R,), generator=gen)
    labels[1], labels[2], labels[3], labels[4] = 0, -100, V - 1, V       # ignore index, ignored, last column, out of range
    dloss = torch.rand(R, generator=gen)
    x = logits.numpy()
    lse, loss = torch.zeros(R), torch.zeros(R)
    for r in range(R):
        l, lo, seen = _smoothed_fwd_row(x[r], V, int(labels[r]), eps)
        lse[r], loss[r] = float(l), float(lo)
        assert (seen == 1).all()                                  # every column < V exactly once, no pad column
    # reference (loss.py:28-48 on the fp32 log-softmax); labels outside [0, V) are ignored like label 0
    ref_labels = torch.where((labels >= 0) & (labels < V), labels, torch.zeros_like(labels))
    xr = logits[:, :V].clone().requires_grad_(True)
    ref = LSO.label_smoothing_loss(F.log_softmax(xr, -1).unsqueeze(0), ref_labels.unsqueeze(0), eps, V)[0]
    assert torch.allclose(lse, torch.logsumexp(logits[:, :V], -1), atol=1e-5)
    assert torch.allclose(loss, ref.detach(), atol=1e-4), (loss, ref)
    assert float(loss[1]) == 0.0 and float(loss[2]) == 0.0 and float(loss[4]) == 0.0
    # backward model (decoder_ce_bwd_kernel<true>): (exp(x - lse) - q) * dloss, q_0 = 0, q_label = c, q_v = s otherwise; zero in
    # the pad columns and for ignored rows
    c, s, _ = _smoothing_constants(V, eps)
    live = (labels > 0) & (labels < V)
    q = torch.full((R, Vp), float(s))
    q[:, 0] = 0
    q[:, V:] = 0
    q[torch.arange(R)[live], labels[live]] = float(c)
    p = torch.exp(logits - lse[:, None])
    p[:, V:] = 0
    d = (p - q) * (dloss * live)[:, None]
    (ref * dloss).sum().backward()
    assert torch.allclose(d[:, :V], xr.grad, atol=1e-5)
    assert float(d[:, V:].abs().sum()) == 0 and float(d[~live].abs().sum()) == 0
    assert float(d[0, 0]) == pytest.approx(float(p[0, 0] * dloss[0]), rel=1e-6)      # column 0: softmax only, q_0 = 0


# ---- state_dict contract -------------------------------------------------------------------------------------------------------
def _reference_style_state_dict(dims, eps, gold_case):
    """A state dict as the reference model with label smoothing saves it: the parameters plus its one_hot buffer (loss.py:29-31),
    whose bytes are those the reference produced."""
    sd = {k: v.clone() for k, v in synth.make_state_dict(dims, 0).items()}
    one_hot = torch.full((dims.vocab,), eps / (dims.vocab - 2))
    one_hot[0] = 0
    sd["crit_mask_lm_smoothed.one_hot"] = one_hot.unsqueeze(0)
    assert mg.tensor_digest(sd["crit_mask_lm_smoothed.one_hot"]) == gold_case["one_hot"]
    return sd


def test_state_dict_keys_match_reference_with_label_smoothing(gold):
    for name in ("l123_mix_ls01", "l123_v28996_ls01"):
        g = gold[name]
        dims, _, _, eps = LSO.inputs(name)
        model = vm.BertForPreTrainingLossMask(make_config(dims, eps), enable_butd=True, len_vis_input=dims.regions)
        sd = model.state_dict()
        assert set(sd.keys()) == set(g["state_dict_keys"])
        assert sd["crit_mask_lm_smoothed.one_hot"].shape == (1, dims.vocab)
        assert mg.tensor_digest(sd["crit_mask_lm_smoothed.one_hot"]) == g["one_hot"]
        res = model.load_state_dict(_reference_style_state_dict(dims, eps, g), strict=True)
        assert not res.missing_keys and not res.unexpected_keys
    plain = vm.BertForPreTrainingLossMask(make_config(synth.SMALL_L123), enable_butd=True, len_vis_input=synth.SMALL_L123.regions)
    assert plain.crit_mask_lm_smoothed is None and "crit_mask_lm_smoothed.one_hot" not in plain.state_dict()


def test_from_pretrained_with_label_smoothing(tmp_path, gold):
    """run_img2txt_dist.py --label_smoothing 0.1 passes label_smoothing= to from_pretrained (:328, 351)."""
    name = "l123_mix_ls01"
    g = gold[name]
    dims, _, _, eps = LSO.inputs(name)
    cfg = {"vocab_size": dims.vocab, "hidden_size": dims.hidden, "num_hidden_layers": dims.layers, "num_attention_heads": dims.heads,
           "intermediate_size": dims.inter, "hidden_act": "gelu", "hidden_dropout_prob": 0.1, "attention_probs_dropout_prob": 0.1,
           "max_position_embeddings": dims.max_pos, "type_vocab_size": dims.type_vocab, "initializer_range": 0.02}
    (tmp_path / "bert_config.json").write_text(json.dumps(cfg))
    sd = synth.make_state_dict(dims, 0)
    model = vm.BertForPreTrainingLossMask.from_pretrained(str(tmp_path), state_dict={k: v.clone() for k, v in sd.items()}, label_smoothing=eps,
                                                          enable_butd=True, len_vis_input=dims.regions, tasks="img2txt")
    assert model.config.label_smoothing == eps and model.crit_mask_lm_smoothed is not None
    assert set(model.state_dict().keys()) == set(g["state_dict_keys"])
    assert model.missing_keys == ["crit_mask_lm_smoothed.one_hot"]           # a BERT checkpoint has no buffer; it keeps its init
    assert mg.tensor_digest(model.state_dict()["crit_mask_lm_smoothed.one_hot"]) == g["one_hot"]
    res = model.load_state_dict(_reference_style_state_dict(dims, eps, g), strict=True)
    assert not res.missing_keys and not res.unexpected_keys


# ---- C ABI ---------------------------------------------------------------------------------------------------------------------
def test_training_step_with_label_smoothing_marshalling_dry_run():
    """A bf16 training step with label_smoothing = 0.1 under the prototype-conversion dry-run: the smoothed pair replaces the
    cross-entropy pair and nothing else changes."""
    from tools import abi_cases
    d = synth.TINY
    model = vm.BertForPreTrainingLossMask(make_config(d, 0.1), enable_butd=True, len_vis_input=d.regions).bfloat16().train()
    assert model.fused_mlm_head is True
    b = synth.make_batch(d, 2, seed=1)
    with abi_cases.dry_run() as calls:
        out = model(b["img"].bfloat16(), b["vis_pe"].bfloat16(), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None,
                    b["is_next"], masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"],
                    vis_masked_pos=b["vis_masked_pos"], mask_image_regions=False, drop_worst_ratio=0.0)
        sum(l.float().sum() for l in out).backward()
    assert calls == ["vlpk_linear_fwd"] * 3 + ["vlpk_embed_fwd", "vlpk_mask_pack", "vlpk_encoder_fwd", "vlpk_decoder_ce_ls_fwd",
                                               "vlpk_decoder_ce_ls_bwd", "vlpk_encoder_bwd", "vlpk_f32_to_bf16", "vlpk_embed_bwd",
                                               "vlpk_embed_tables_bwd"] + ["vlpk_linear_bwd"] * 3
    for n, p in model.named_parameters():
        if not n.startswith("bert.pooler."):
            assert p.grad is not None and p.grad.shape == p.shape and p.grad.dtype == p.dtype, n


def test_label_smoothing_entry_points_reject_bad_arguments():
    """eps outside (0, 1] or V < 3: rc < 0 before anything is launched (the pointers are never dereferenced)."""
    lib = _lib.lib()
    ok = [4096 * i for i in range(1, 13)]

    def fwd(V, eps):
        return lib.vlpk_decoder_ce_ls_fwd(4, V, 128, eps, *ok[:7], None)

    def bwd(V, eps):
        return lib.vlpk_decoder_ce_ls_bwd(4, V, 128, eps, *ok[:10], None)

    for V, eps in ((100, 0.0), (100, -0.1), (100, 1.0000001), (100, 2.0), (100, float("nan")), (2, 0.1), (0, 0.1)):
        assert fwd(V, eps) < 0 and b"label smoothing" in lib.vlpk_last_error(), (V, eps)
        assert bwd(V, eps) < 0 and b"label smoothing" in lib.vlpk_last_error(), (V, eps)
    assert lib.vlpk_decoder_ce_ls_fwd(4, 100, 100, 0.1, *ok[:7], None) < 0        # the shared checks still apply (H % 64)
    assert lib.vlpk_decoder_ce_ls_bwd(4, 100, 128, 0.1, ok[0], ok[1], ok[2], ok[3] + 2, *ok[4:10], None) < 0   # misaligned logits
