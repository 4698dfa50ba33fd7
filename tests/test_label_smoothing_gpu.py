"""GPU: the label-smoothed masked-LM head (vlpk_decoder_ce_ls_fwd/bwd, csrc/head.cu decoder_ce_*_kernel<true>) and the model with
config.label_smoothing set.

Kernel level, as in test_kernel_edges_gpu.test_decoder_ce_head_gemms: every output sits in a NaN guard band; lse, loss and dlogits
are held to an fp64 evaluation on the kernel's OWN bf16 logits, dh / dW / dbias to the existing GEMM and column-sum bounds on the
kernel's own dlogits, and dh must be bitwise identical run to run.  Model level: against the unmodified reference's outputs
(tests/golden/label_smoothing.pt) with the tolerances of test_parity_gpu.py, against the torch evaluation of the head on identical
weights, and under CUDA-graph replay.

VLPK_LS_CHECK_REPORT=<path> writes the worst error / bound of the kernel-level checks as JSON."""
import json
import math
import os

import pytest
import torch

from tools import kernel_check as kc
from tools import label_smoothing_oracle as LSO
from vlp_b200 import _lib as L
from vlp_b200 import graph, ops, synth
from vlp_b200 import vlp_modules as vm

pytestmark = pytest.mark.gpu

DEV = "cuda"
BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64

# Bounds of the row kernels, >= 2x the worst value measured on the H100 (see DESIGN.md §6)
LOSS_TOL = 2e-5               # |loss - ref| and |lse - ref| <= LOSS_TOL * (1 + |ref|)
DLOGITS_A = 2.0 ** -16        # |dlogits - ref| <= 2^-8 |ref| + DLOGITS_A * max |ref| (per row)
TOL_HID, TOL_GRAD, TOL_LOSS = 3e-2, 5e-2, 5e-3
WORST = {}


def _note(family, ratio):
    WORST[family] = max(WORST.get(family, 0.0), ratio)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("VLPK_LS_CHECK_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(sorted(WORST.items())), f, indent=1)


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def cosine(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm() + 1e-30)).item()


# ---- kernel level --------------------------------------------------------------------------------------------------------------
def _smoothed_ref(x, labels, eps, dloss):
    """fp64 loss, lse and dlogits of the smoothed loss on logits x [R, V] (the kernel's own bf16 values)."""
    R, V = x.shape
    x = x.to(F64)
    e = float(torch.tensor(eps, dtype=F32))                  # the fp32 value the kernel receives
    c, s = 1.0 - e, e / (V - 2)
    K = (c * math.log(c) if c > 0 else 0.0) + (V - 2) * s * math.log(s)
    lse = torch.logsumexp(x, -1)
    live = (labels > 0) & (labels < V)
    t = torch.where(live, labels, torch.zeros_like(labels))
    xt = x.gather(1, t[:, None])[:, 0]
    loss = torch.where(live, K + lse - c * xt - s * (x.sum(-1) - x[:, 0] - xt), torch.zeros_like(lse))
    q = torch.full_like(x, s)
    q[:, 0] = 0
    q[torch.arange(R, device=x.device)[live], t[live]] = c
    d = (torch.exp(x - lse[:, None]) - q) * (dloss.to(F64) * live)[:, None]
    return lse, loss, d, live


@pytest.mark.parametrize("eps", [0.1, 1.0])
@pytest.mark.parametrize("R,V,H", [(6, 1003, 128), (192, 28996, 768)])
def test_smoothed_head_kernels(R, V, H, eps):
    torch.manual_seed(R + V)
    Vp = (V + 7) // 8 * 8
    h = torch.randn(R, H, device=DEV).to(BF)
    w = (torch.randn(V, H, device=DEV) * 0.05).to(BF)
    bias_pad = torch.zeros(Vp, device=DEV, dtype=BF)
    bias_pad[:V] = (torch.randn(V, device=DEV) * 0.1).to(BF)
    labels = torch.randint(1, V, (R,), device=DEV)
    labels[::7] = -1                                          # ignored position
    labels[1], labels[2] = 0, V - 1                           # the ignore index of the smoothed loss; the last column
    logits = kc.guarded(R, Vp)
    lse = kc.guarded(R, 1, dtype=F32)
    loss = kc.guarded(R, 1, dtype=F32)
    L.call("vlpk_decoder_ce_ls_fwd", R, V, H, eps, h.data_ptr(), w.data_ptr(), bias_pad.data_ptr(), labels.data_ptr(), logits.data_ptr(),
           lse.data_ptr(), loss.data_ptr(), L.stream())
    torch.cuda.synchronize()
    for t, nm in ((logits, "logits"), (lse, "lse"), (loss, "loss")):
        kc.assert_guard_intact(t, nm)
    w_pad = torch.cat([w, torch.zeros(Vp - V, H, device=DEV, dtype=BF)])
    acc, E = kc.gemm_ref(h, w_pad)
    ref, Er = kc.epilogue_ref(0, acc, E, bias=bias_pad)["d0"]
    kc.check_gemm("smoothed head logits", logits, ref, Er)
    dloss = torch.rand(R, device=DEV) + 0.5
    x = logits[:, :V].clone()
    lse_ref, loss_ref, d_ref, live = _smoothed_ref(x, labels, eps, dloss)
    for nm, got, want in (("lse", lse[:, 0], lse_ref), ("loss", loss[:, 0], loss_ref)):
        err = (got.to(F64) - want).abs()
        ratio = float((err / (LOSS_TOL * (1 + want.abs()))).max())
        _note(f"{nm}", ratio)
        assert ratio <= 1.0, (nm, float(err.max()))
    assert bool((loss[~live, 0] == 0).all())

    def bwd():
        dlogits = kc.guarded(R, Vp)
        dh = kc.guarded(R, H, dtype=F32)
        kc.guard_fill(dh, torch.zeros(R, H, device=DEV))
        dw = kc.guarded(V, H)
        dbias = kc.guarded(Vp, 1, dtype=F32)
        kc.guard_fill(dbias, torch.zeros(Vp, 1, device=DEV))
        L.call("vlpk_decoder_ce_ls_bwd", R, V, H, eps, h.data_ptr(), w.data_ptr(), labels.data_ptr(), logits.data_ptr(), lse.data_ptr(),
               dloss.data_ptr(), dlogits.data_ptr(), dh.data_ptr(), dw.data_ptr(), dbias.data_ptr(), L.stream())
        torch.cuda.synchronize()
        return dlogits, dh, dw, dbias

    dlogits, dh, dw, dbias = bwd()
    for t, nm in ((dlogits, "dlogits"), (dh, "dh"), (dw, "dW"), (dbias, "dbias")):
        kc.assert_guard_intact(t, nm)
    assert bool((dlogits[:, V:] == 0).all()) and bool((dlogits[~live] == 0).all())
    scale = d_ref.abs().amax(1, keepdim=True).expand_as(d_ref)
    _note("dlogits elementwise", kc.check_elementwise("smoothed dlogits", dlogits[:, :V], d_ref, scale, kc.R_BF16, DLOGITS_A,
                                                      where=lambda i, j: f"row {i} col {j} (label {int(labels[i])})"))
    d = dlogits[:, :V]
    acc, E = kc.gemm_ref(d, w.t())
    kc.check_gemm("smoothed head dh", dh, acc, E)
    acc, E = kc.gemm_ref(d.t(), h.t())
    kc.check_gemm("smoothed head dW", dw, acc, E)
    kc.check_colsum("smoothed head dbias", dbias[:, 0], dlogits)
    _, dh2, dw2, _ = bwd()
    assert torch.equal(dh, dh2), "smoothed head dh differs between two identical calls"
    assert torch.equal(dw, dw2)


# ---- model level ---------------------------------------------------------------------------------------------------------------
def _config(dims, eps, drop=0.0):
    return vm.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                         intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                         hidden_dropout_prob=drop, attention_probs_dropout_prob=drop, label_smoothing=eps)


def _model(dims, eps, sd, drop=0.0):
    model = vm.BertForPreTrainingLossMask(_config(dims, eps, drop), enable_butd=True, len_vis_input=dims.regions)
    model.load_state_dict(sd, strict=False)
    return model.cuda().bfloat16()


def _run(model, b):
    return model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None, b["is_next"],
                 masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"],
                 vis_masked_pos=b["vis_masked_pos"], mask_image_regions=False, drop_worst_ratio=0.0)


def _dev(batch):
    b = {k: v.cuda() for k, v in batch.items()}
    b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()
    return b


def _reference_bf16_drift(name):
    """The reference algorithm's own fp32 -> bf16 gradient drift on this case (oracle run twice on the host CPU), per parameter."""
    out = []
    for dtype in (torch.float32, torch.bfloat16):
        dims, sd, batch, eps = LSO.inputs(name)
        sd = {k: v.to(dtype) for k, v in sd.items()}
        sd["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]
        for k, v in sd.items():
            if k != "cls.predictions.decoder.weight":
                v.requires_grad_(True)
        batch = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
        LSO.pretraining_loss(sd, dims, batch, eps)[0].float().backward()
        out.append(sd)
    a, b = out
    return {k: rel(b[k].grad, a[k].grad) for k in a if a[k].grad is not None and k != "cls.predictions.decoder.weight"
            and float(a[k].grad.norm()) > 0}


@pytest.mark.parametrize("name", ["l123_mix_ls01", "l123_v28996_ls01"])
def test_model_with_label_smoothing_matches_reference_golden(name, golden_dir):
    from test_parity_gpu import compare_grads
    gold = torch.load(os.path.join(golden_dir, "label_smoothing.pt"))["cases"][name]
    dims, sd, batch, eps = LSO.inputs(name)
    model = _model(dims, eps, sd).eval()
    assert model.fused_mlm_head
    losses = _run(model, _dev(batch))
    for got, ref in zip(losses, gold["losses"]):
        assert abs(float(got) - float(ref)) <= TOL_LOSS * max(1.0, abs(float(ref))), (float(got), float(ref))
    assert rel(LSO.sample(model.last_prediction_scores.float().cpu()), gold["logits"]) < TOL_HID
    sum(l.sum() for l in losses).backward()
    worst = compare_grads(model, gold["grads"], drift_fn=lambda: _reference_bf16_drift(name),
                          sample_idx_fn=lambda n: LSO.sample_idx(n, LSO.GRAD_SAMPLES))
    print(f"{name}: loss {float(losses[0]):.6f} reference {float(gold['losses'][0]):.6f}; worst grad rel-L2 {worst:.3e}")


def test_fused_smoothed_head_matches_torch_head():
    """fused_mlm_head True (vlpk_decoder_ce_ls_*) vs False (crit_mask_lm_smoothed on the fp32 log-softmax, modeling.py:1104-1106)
    on identical weights and inputs, a weighted label-0 position included."""
    dims, sd, batch, eps = LSO.inputs("l123_mix_ls01")
    b = _dev(batch)
    outs = []
    for fused in (False, True):
        model = _model(dims, eps, sd).eval()
        model.fused_mlm_head = fused
        losses = _run(model, b)
        sum(l.float().sum() for l in losses).backward()
        torch.cuda.synchronize()
        outs.append((float(losses[0]), {n: p.grad.detach().float().cpu() for n, p in model.named_parameters() if p.grad is not None},
                     model.last_prediction_scores.detach().float().cpu()))
    (l0, g0, s0), (l1, g1, s1) = outs
    assert abs(l0 - l1) < 2e-2 and rel(s1, s0) < 1e-2
    assert set(g0) == set(g1)
    for n in g0:
        if "attention.self.key.bias" in n:       # exactly 0 in exact arithmetic: rounding noise on both paths
            continue
        if float(g0[n].norm()) > 0:
            assert rel(g1[n], g0[n]) < 5e-2, n
            assert cosine(g1[n], g0[n]) > 0.999, n


def test_graphed_step_with_label_smoothing_equals_python_driven_step():
    """GraphedStep replay of a training step with label smoothing on equals the Python-driven step on a new batch."""
    d = synth.SMALL_L123
    sd = synth.make_state_dict(d, 0)
    model = _model(d, 0.1, sd).train()
    b0 = _dev(synth.make_batch(d, 4, seed=11, mode="mix", ragged=True))
    b1 = _dev(synth.make_batch(d, 4, seed=12, mode="mix", ragged=True))

    def step(m, b):
        out = _run(m, b)
        loss = out[0] + out[1] + out[2]
        loss.backward()
        return loss

    def grads():
        return {n: p.grad.detach().float().clone() for n, p in model.named_parameters() if p.grad is not None}

    try:
        model.zero_grad(set_to_none=True)
        want_loss = float(step(model, b1))
        want = grads()
        g = graph.GraphedStep(model, b0, step)
        assert g.launches_per_replay > 20
        loss = g(b1)
        got = grads()
        assert abs(float(loss) - want_loss) < 1e-6
        assert set(got) == set(want)
        for n in want:
            err = float((got[n] - want[n]).norm() / (want[n].norm() + 1e-30))
            assert err < 2e-3, (n, err)
        model.zero_grad(set_to_none=True)
        plain = float(step(_model(d, None, sd).train(), b1))
        assert abs(plain - want_loss) > 1e-3                  # the replayed step really is the smoothed one
    finally:
        ops.set_device_seed_tensor(None)
