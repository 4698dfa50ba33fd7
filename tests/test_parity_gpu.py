"""Parity tests proper (GPU): the sm_90a path behind the reference's Python surface vs (a) the reference's own
outputs stored under tests/golden/ and (b) the fp32 oracle run live on the host CPU.

Stated tolerance for bf16 kernels vs the fp32 reference (BASELINE.md §3 / SURVEY.md §8c, derived from the reference's
own fp32->bf16 self-drift): hidden states / logits rel-L2 <= 3e-2, loss abs diff <= 5e-3 (relative 5e-3 for the
3129-way VQA loss whose magnitude is ~2e3), parameter gradients rel-L2 <= 5e-2 and cosine >= 0.999.
"""
import os

import pytest
import torch

from oracle import make_golden as mg
from oracle import vlp_oracle as O
from vlp_b200 import synth
from vlp_b200 import vlp_modules as vm

pytestmark = pytest.mark.gpu

TOL_HID, TOL_GRAD, TOL_LOSS = 3e-2, 5e-2, 5e-3


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def cosine(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return (a @ b / (a.norm() * b.norm() + 1e-30)).item()


def make_config(d, drop=0.0):
    return vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                         type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=drop,
                         attention_probs_dropout_prob=drop)


def build(dims, tasks, dtype=torch.bfloat16, drop=0.0, sd_seed=0):
    model = vm.BertForPreTrainingLossMask(make_config(dims, drop), enable_butd=True, len_vis_input=dims.regions, tasks=tasks)
    model.load_state_dict(synth.make_state_dict(dims, sd_seed, tasks))
    return model.to("cuda", dtype)


def run_model(model, batch, tasks, dtype=torch.bfloat16):
    b = {k: v.cuda() for k, v in batch.items()}
    ans = b["ans_labels"] if tasks == "vqa2" else None
    return model(b["img"].to(dtype), b["vis_pe"].to(dtype), b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], ans, b["is_next"],
                 masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"], vis_masked_pos=b["vis_masked_pos"],
                 mask_image_regions=False, drop_worst_ratio=0.0)


def reference_bf16_drift(name):
    """The reference algorithm's own fp32 -> bf16 drift on the same inputs (oracle run twice on the host CPU): per-parameter
    gradient rel-L2.  BASELINE.md §3: the kernels' error must stay within 2x of it where it exceeds the flat tolerance."""
    dims, B, seed, mode, ragged, tasks = mg.CASES[name]
    out = []
    for dtype in (torch.float32, torch.bfloat16):
        sd = {k: v.to(dtype) for k, v in synth.make_state_dict(dims, 0, tasks).items()}
        sd["cls.predictions.decoder.weight"] = sd["bert.embeddings.word_embeddings.weight"]
        for k, v in sd.items():
            if k != "cls.predictions.decoder.weight":
                v.requires_grad_(True)
        batch = synth.make_batch(dims, B, seed=seed, mode=mode, ragged=ragged, tasks=tasks)
        batch = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
        losses = O.pretraining_loss(sd, dims, batch, tasks=tasks)
        sum(l.float().sum() for l in losses).backward()
        out.append(sd)
    a, b = out
    return {k: rel(b[k].grad, a[k].grad) for k in a if a[k].grad is not None and k != "cls.predictions.decoder.weight"
            and float(a[k].grad.norm()) > 0}


def check_loss(got, ref):
    got, ref = float(got), float(ref)
    assert abs(got - ref) <= TOL_LOSS * max(1.0, abs(ref)), (got, ref)


def compare_grads(model, ref, drift_fn=None, sample_idx_fn=None):
    """Every parameter gradient of `model` against `ref[name]` = {"full": tensor} or a fingerprint {"sample": values[, "sample_idx"]}.
    Criterion (BASELINE.md §3): rel-L2 <= 5e-2 and cosine >= 0.999; a tensor may exceed that flat bound only where the reference's
    OWN fp32 -> bf16 drift on the same inputs (drift_fn() -> {name: rel-L2}) is itself above 2.5e-2 — i.e. where bf16 storage alone
    already consumes the budget — and then must stay within 2x that drift.  Returns the worst rel-L2 seen; asserts with the list of
    offending tensors."""
    drift = None
    worst, bad, relaxed = 0.0, [], []
    for k, p in model.named_parameters():
        fp = ref.get(k)
        if fp is None:
            continue
        assert p.grad is not None, k
        if k.endswith("attention.self.key.bias"):
            # softmax is invariant to a per-query constant, so d(loss)/d(key.bias) is exactly 0 in exact arithmetic: the
            # reference holds fp32 round-off (~1e-9), here it is bf16 round-off.  Compare against the scale of the
            # sibling query.bias gradient instead of a relative error on noise.
            sfp = ref[k.replace("key.bias", "query.bias")]
            sib = float(sfp["full"].norm()) if "full" in sfp else float(sfp["norm"])
            own = float(fp["full"].norm()) if "full" in fp else float(fp["norm"])
            assert own < 1e-3 * sib
            assert p.grad.float().norm().item() < 5e-2 * sib + 1e-6, (k, p.grad.float().norm().item(), sib)
            continue
        if "full" in fp:
            refv = fp["full"]
            if refv.norm() == 0:
                assert float(p.grad.float().norm()) == 0.0, k
                continue
            r, c = rel(p.grad, refv), cosine(p.grad, refv)
        else:
            flat = p.grad.detach().float().cpu().flatten()
            idx = fp["sample_idx"] if "sample_idx" in fp else sample_idx_fn(flat.numel())
            got = flat[idx]
            r, c = rel(got, fp["sample"]), cosine(got, fp["sample"])
            if "norm" in fp and fp["norm"] > 0:
                assert abs(float(flat.norm()) / fp["norm"] - 1.0) < TOL_GRAD, (k, float(flat.norm()), fp["norm"])
        worst = max(worst, r)
        if r < 0.0447 and c > 0.999:                       # flat criterion (cos >= 0.999 <=> rel <= 0.0447 for orthogonal error)
            continue
        if drift is None:
            drift = drift_fn() if drift_fn is not None else {}
        dk = drift.get(k, 0.0)
        tol = 2.0 * dk if dk > 0.5 * TOL_GRAD else TOL_GRAD
        if r < tol and c > 1.0 - tol * tol:
            relaxed.append((k, round(r, 4), round(dk, 4)))
        else:
            bad.append((k, round(r, 4), round(c, 5), round(dk, 4)))
    if relaxed:
        print("gradients admitted through the 2x-reference-drift clause:", relaxed)
    assert not bad, f"{len(bad)} gradient(s) out of tolerance: {bad[:12]}"
    return worst


@pytest.mark.parametrize("name", list(mg.CASES))
def test_model_matches_reference_golden(name, golden_dir):
    """Forward activations, losses and every parameter gradient vs the UNMODIFIED reference's stored outputs."""
    dims, B, seed, mode, ragged, tasks = mg.CASES[name]
    gold = torch.load(os.path.join(golden_dir, name + ".pt"))
    batch = synth.make_batch(dims, B, seed=seed, mode=mode, ragged=ragged, tasks=tasks)
    model = build(dims, tasks).eval()
    cap = {}
    model.bert.embeddings.register_forward_hook(lambda m, i, o: cap.__setitem__("embedding", o.detach()))
    losses = run_model(model, batch, tasks)
    for got, ref in zip(losses, gold["losses"]):
        check_loss(got, ref)
    assert rel(cap["embedding"], gold["embedding"]) < TOL_HID
    if tasks != "vqa2":
        assert rel(model.last_prediction_scores, gold["logits"]) < TOL_HID
    sum(l.sum() for l in losses).backward()
    worst = compare_grads(model, gold["grads"], drift_fn=lambda: reference_bf16_drift(name))
    # per-layer outputs (second forward with output_all_encoded_layers=True through BertModel)
    b = {k: v.cuda() for k, v in batch.items()}
    with torch.no_grad():
        v, pe = model.project_regions(b["img"].bfloat16(), b["vis_pe"].bfloat16())
        layers, pooled = model.bert(v, pe, b["input_ids"], b["segment_ids"], b["input_mask"], output_all_encoded_layers=True,
                                    len_vis_input=dims.regions)
    assert len(layers) == dims.layers
    for got, ref in zip(layers, gold["layers"]):
        assert rel(got, ref) < TOL_HID
    assert rel(pooled, gold["pooled"]) < TOL_HID
    print(f"{name}: worst grad rel-L2 {worst:.3e}")


@pytest.mark.parametrize("name", list(mg.BIG_CASES))
def test_full_size_matches_reference_golden(name, golden_dir):
    """BASELINE.json configs[1] (12-layer BERT-base, B = 64, s2s) and configs[3] (VQA, B = 128, bidirectional) NUMERICALLY: losses,
    samples of the last hidden state / MLM logits and every parameter gradient vs fingerprints of the unmodified reference's fp32
    run at that size (oracle/make_golden.py BIG_CASES), with the reference's own bf16 drift stored beside them."""
    dims, B, seed, mode, ragged, tasks = mg.BIG_CASES[name]
    gold = torch.load(os.path.join(golden_dir, name + ".pt"))
    batch = synth.make_batch(dims, B, seed=seed, mode=mode, ragged=ragged, tasks=tasks)
    model = build(dims, tasks).eval()
    cap = {}
    model.bert.encoder.register_forward_hook(lambda m, i, o: cap.__setitem__("hidden", o[-1].detach().float().cpu().flatten()))
    losses = run_model(model, batch, tasks)
    for got, ref in zip(losses, gold["losses"]):
        check_loss(got, ref)
    hid = cap["hidden"]
    assert rel(hid[mg.big_sample_idx(hid.numel(), 8192)], gold["hidden"]) < max(TOL_HID, 2.0 * gold["hidden_drift"])
    if tasks != "vqa2":
        lg = model.last_prediction_scores.detach().float().cpu().flatten()
        assert rel(lg[mg.big_sample_idx(lg.numel(), 8192)], gold["logits"]) < TOL_HID
    sum(l.sum() for l in losses).backward()
    worst = compare_grads(model, gold["grads"], drift_fn=lambda: gold["drift"], sample_idx_fn=mg.big_sample_idx)
    print(f"{name}: worst grad rel-L2 {worst:.3e} (reference bf16 drift: hidden {gold['hidden_drift']:.3e})")


def test_fp32_parameter_model_is_supported():
    """The reference's default recipes keep fp32 parameters (SURVEY.md §2.1): casts happen at the op boundary and gradients
    come back in fp32."""
    dims = synth.SMALL_L123
    batch = synth.make_batch(dims, 2, seed=5)
    model = build(dims, "img2txt", dtype=torch.float32).eval()
    losses = run_model(model, batch, "img2txt", dtype=torch.float32)
    sd = synth.make_state_dict(dims, 0)
    ref = O.pretraining_loss(sd, dims, batch)
    check_loss(losses[0], ref[0])
    losses[0].backward()
    g = model.bert.encoder.layer[0].attention.self.query.weight.grad
    assert g is not None and g.dtype == torch.float32 and torch.isfinite(g).all()


def test_bert_base_layer_shapes_vs_oracle():
    """Real BERT-base width (H=768, 12 heads, I=3072, L=123) for two layers: exercises the production tile shapes
    (N=2304 / 3072 GEMMs, 12 heads) against the oracle computed live on the host."""
    dims = synth.VlpDims(vocab=2000, layers=2)
    batch = synth.make_batch(dims, 3, seed=11, mode="mix", ragged=True)
    sd = synth.make_state_dict(dims, 1)
    model = vm.BertForPreTrainingLossMask(make_config(dims), enable_butd=True, len_vis_input=dims.regions)
    model.load_state_dict(sd)
    model = model.cuda().bfloat16().eval()
    losses = run_model(model, batch, "img2txt")
    for v in sd.values():
        v.requires_grad_(False)
    names = ["bert.encoder.layer.0.attention.self.key.weight", "bert.encoder.layer.1.output.dense.weight", "vis_embed.0.weight",
             "bert.encoder.layer.0.intermediate.dense.bias", "bert.embeddings.LayerNorm.weight", "vis_pe_embed.0.weight"]
    for n in names:
        sd[n].requires_grad_(True)
    ref_losses, aux = O.pretraining_loss(sd, dims, batch, return_all=True)
    check_loss(losses[0], ref_losses[0])
    assert rel(model.last_prediction_scores, aux["logits"]) < TOL_HID
    losses[0].backward()
    ref_losses[0].backward()
    got = dict(model.named_parameters())
    for n in names:
        r, c = rel(got[n].grad, sd[n].grad), cosine(got[n].grad, sd[n].grad)
        assert r < TOL_GRAD and c > 0.999, (n, r, c)


def test_dropout_training_step_is_finite_and_consistent():
    """p = 0.1 (the reference's training setting): forward and backward regenerate the same Philox masks; loss finite,
    gradients finite, and two runs with the same seed are bit-identical while a different seed differs."""
    from vlp_b200 import ops
    dims = synth.SMALL_L123
    batch = synth.make_batch(dims, 4, seed=21)
    outs = []
    for seed in (7, 7, 8):
        torch.manual_seed(seed)
        ops._seed_counter = __import__("itertools").count(1)
        model = build(dims, "img2txt", drop=0.1).train()
        loss = run_model(model, batch, "img2txt")[0]
        loss.backward()
        g = model.bert.encoder.layer[0].output.dense.weight.grad.float().clone()
        assert torch.isfinite(loss).all() and torch.isfinite(g).all()
        outs.append((float(loss), g))
    assert outs[0][0] == outs[1][0] and torch.equal(outs[0][1], outs[1][1])
    assert outs[0][0] != outs[2][0]
    # expectation check: dropout-scaled training loss stays close to the eval loss
    model = build(dims, "img2txt", drop=0.0).eval()
    ev = float(run_model(model, batch, "img2txt")[0])
    assert abs(outs[0][0] - ev) < 0.5


def test_full_size_properties_bert_base_b64():
    """BASELINE.json configs[1] size (BERT-base, B=64, L=123) through size-independent properties, since the CPU oracle
    would take minutes here: (1) batch independence — sample i's hidden state is the same computed alone or inside the
    batch of 64 (up to bf16 tile-order effects), (2) mask semantics — s2s image rows are invariant to the text tokens,
    (3) gradient linearity — grad(2*loss) == 2*grad(loss)."""
    dims = synth.BERT_BASE
    B = 64
    torch.manual_seed(0)
    model = vm.BertForPreTrainingLossMask(make_config(dims), enable_butd=True, len_vis_input=dims.regions).cuda().bfloat16().eval()
    batch = synth.make_batch(dims, B, seed=31)
    b = {k: v.cuda() for k, v in batch.items()}

    def hidden(sl):
        with torch.no_grad():
            v, pe = model.project_regions(b["img"][sl].bfloat16(), b["vis_pe"][sl].bfloat16())
            seq, _ = model.bert(v, pe, b["input_ids"][sl], b["segment_ids"][sl], b["input_mask"][sl], output_all_encoded_layers=False,
                                len_vis_input=dims.regions)
        return seq.float()

    full = hidden(slice(0, B))
    one = hidden(slice(5, 6))
    assert rel(one[0], full[5]) < 1e-2
    ids2 = b["input_ids"].clone()
    ids2[:, dims.regions + 2:dims.regions + 2 + dims.text] = 1234
    saved = b["input_ids"]
    b["input_ids"] = ids2
    alt = hidden(slice(0, 4))
    b["input_ids"] = saved
    R = dims.regions
    assert rel(alt[:, :R + 2], full[:4, :R + 2]) < 1e-6          # image/CLS/SEP rows cannot see the text under the s2s mask
    assert rel(alt[:, R + 2:], full[:4, R + 2:]) > 1e-3
    model.train(False)
    grads = []
    for scale in (1.0, 2.0):
        model.zero_grad(set_to_none=True)
        loss = run_model(model, {k: v[:8] for k, v in batch.items()}, "img2txt")[0] * scale
        loss.backward()
        grads.append(model.bert.encoder.layer[3].intermediate.dense.weight.grad.float().clone())
    assert rel(grads[1], 2 * grads[0]) < 2e-2
