"""GPU: region masking (mask_image_regions=True, --vis_mask_prob) and drop-worst on the plain path, through the module surface.

Against the unmodified reference's stored outputs (tests/golden/region_masking.pt, tools/region_masking_oracle.py) with the
criterion of test_parity_gpu.py; the pretext loss, a log-softmax over dot products of projected features, is held to the larger of
BASELINE.md §3's loss bound and twice the reference's own fp32 -> bf16 drift (region_masking_oracle.loss_bound).  With dropout 0.1
the kernels' keep masks are replayed into the oracle (test_dropout_parity_gpu.py's criterion).  Exact properties: new input
features at the masked regions change the embedding output, every encoder layer's output and the masked-LM loss by nothing; a
GraphedStep takes vis_masked_pos as a captured input; deterministic steps are bitwise reproducible; the grouped BatchStager refuses a loader
matrix with blocked region columns before any launch."""
import itertools
import os

import pytest
import torch

from oracle import vlp_oracle as O
from tools import label_smoothing_oracle as LS
from tools import region_masking_oracle as RM
from vlp_b200 import _lib as L
from vlp_b200 import graph, ops, staging, synth

from test_dropout_parity_gpu import P, _provider
from test_parity_gpu import TOL_HID, build, compare_grads, rel

pytestmark = pytest.mark.gpu


def _dev(batch):
    b = {k: v.cuda() for k, v in batch.items()}
    b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()
    return b


def _run(model, b, tasks, mir, dw):
    return model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"],
                 b["ans_labels"] if tasks == "vqa2" else None, b["is_next"], masked_pos=b["masked_pos"],
                 masked_weights=b["masked_weights"], task_idx=b["task_idx"], vis_masked_pos=b["vis_masked_pos"],
                 mask_image_regions=mir, drop_worst_ratio=dw)


@pytest.fixture
def deterministic():
    before = torch.are_deterministic_algorithms_enabled()
    cublas = os.environ.get("CUBLAS_WORKSPACE_CONFIG")
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(before)
    if cublas is None:
        os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
    else:
        os.environ["CUBLAS_WORKSPACE_CONFIG"] = cublas
    ops.set_device_seed_tensor(None)
    L.call("vlpk_debug_set_option", b"wgrad_stream", 0 if os.environ.get("VLPK_WGRAD_STREAM", "1").startswith("0") else 1)


@pytest.mark.parametrize("name", list(RM.CASES))
def test_model_matches_reference_golden(name, golden_dir):
    gold = torch.load(os.path.join(golden_dir, "region_masking.pt"))["cases"][name]
    dims, sd, batch, tasks, mir, dw = RM.inputs(name)
    model = build(dims, tasks).eval()
    cap = {}
    model.bert.embeddings.register_forward_hook(lambda m, i, o: cap.__setitem__("embedding", o.detach()))
    model.bert.pooler.register_forward_hook(lambda m, i, o: cap.__setitem__("pooled", o.detach()))
    losses = _run(model, _dev(batch), tasks, mir, dw)
    for i, (got, ref) in enumerate(zip(losses, gold["losses"])):
        assert abs(float(got) - float(ref)) <= RM.loss_bound(gold, i), (i, float(got), float(ref), RM.loss_bound(gold, i))
    assert (float(losses[1]) != 0) == mir
    assert rel(LS.sample(cap["embedding"].float().cpu()), gold["embedding"]) < max(TOL_HID, 2 * gold["drift"]["embedding"])
    assert rel(cap["pooled"], gold["pooled"]) < max(TOL_HID, 2 * gold["drift"]["pooled"])
    if tasks != "vqa2":
        assert rel(LS.sample(model.last_prediction_scores.float().cpu()), gold["logits"]) < max(TOL_HID, 2 * gold["drift"]["logits"])
    sum(l.float().sum() for l in losses).backward()
    worst = compare_grads(model, gold["grads"], drift_fn=lambda: gold["drift"]["grads"],
                          sample_idx_fn=lambda n: LS.sample_idx(n, LS.GRAD_SAMPLES))
    print(f"{name}: losses {[round(float(l), 5) for l in losses]} reference {[round(float(l), 5) for l in gold['losses']]}; "
          f"worst grad rel-L2 {worst:.3e}")


@pytest.mark.parametrize("name", ["l123_s2s_vm25_dw02", "l123_bi_vqa_vm25"])
def test_training_mode_dropout_matches_oracle_with_replayed_masks(name, golden_dir):
    """Dropout 0.1 on every site with the kernels' keep masks replayed into the fp32 oracle: loss, logits and every gradient."""
    dims, sd, batch, tasks, mir, dw = RM.inputs(name)
    B = batch["img"].shape[0]
    torch.manual_seed(1234)
    model = build(dims, tasks, drop=P).train()
    ops.SEED_LOG = []
    try:
        losses = _run(model, _dev(batch), tasks, mir, dw)
        sum(l.float().sum() for l in losses).backward()
        torch.cuda.synchronize()
        seeds = dict(ops.SEED_LOG)
    finally:
        ops.SEED_LOG = None

    def oracle(dtype):
        ref_sd = {k: v.to(dtype) for k, v in synth.make_state_dict(dims, 0, tasks).items()}
        ref_sd["cls.predictions.decoder.weight"] = ref_sd["bert.embeddings.word_embeddings.weight"]
        for k, v in ref_sd.items():
            if k != "cls.predictions.decoder.weight":
                v.requires_grad_(True)
        b = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
        O.MASK_PROVIDER = _provider(seeds, dims, B)[0]
        try:
            out = O.pretraining_loss(ref_sd, dims, b, tasks=tasks, drop_worst_ratio=dw, p_hidden=P, p_attn=P, training=True,
                                     return_all=True, mask_image_regions=mir)
            sum(l.float().sum() for l in out[0]).backward()
        finally:
            O.MASK_PROVIDER = None
        return out, ref_sd

    (ref_losses, aux), ref_sd = oracle(torch.float32)
    gold = torch.load(os.path.join(golden_dir, "region_masking.pt"))["cases"][name]
    for i, (got, ref) in enumerate(zip(losses, ref_losses)):
        assert abs(float(got) - float(ref)) <= RM.loss_bound(gold, i), (i, float(got), float(ref))
    if tasks != "vqa2":
        assert rel(model.last_prediction_scores, aux["logits"]) < TOL_HID
    ref_grads = {k: {"full": v.grad} for k, v in ref_sd.items() if v.grad is not None}

    def drift():
        _, lo = oracle(torch.bfloat16)
        return {k: rel(lo[k].grad, g["full"]) for k, g in ref_grads.items() if lo[k].grad is not None and float(g["full"].norm()) > 0}

    worst = compare_grads(model, ref_grads, drift_fn=drift)
    print(f"{name} dropout {P}: worst grad rel-L2 {worst:.3e}")


def _small(tasks="img2txt", drop=0.0):
    dims = synth.SMALL_L123
    torch.manual_seed(0)
    return build(dims, tasks, drop=drop).train(), dims


def test_masked_region_features_change_only_the_pretext(deterministic):
    """New input features at the masked regions: embedding output, every layer's output and masked-LM loss bitwise unchanged, the
    pretext loss moved; the gradient reaching the projected features and position encodings at the masked rows is the pretext's,
    bit for bit, and the masked-LM loss sends none there."""
    model, dims = _small()
    dims, sd, batch, tasks, mir, dw = RM.inputs("l123_s2s_vm25")
    b0 = _dev(batch)
    b1 = dict(b0, img=b0["img"].clone(), vis_pe=b0["vis_pe"].clone())
    for i in range(b1["img"].shape[0]):
        r = b1["vis_masked_pos"][i] - 1
        b1["img"][i, r] = b1["img"][i, r].flip(0) + 0.5
        b1["vis_pe"][i, r] = -b1["vis_pe"][i, r]
    outs = []
    stack = ops.EncoderStackFn.apply
    for b in (b0, b1):
        cap = {"layers": []}

        def record(*a):
            out = stack(*a)
            cap["layers"].extend(o.detach().clone() for o in out)
            return out

        h = model.bert.embeddings.register_forward_hook(lambda m, i, o: cap.__setitem__("emb", o.detach().clone()))
        ops.EncoderStackFn.apply = record
        try:
            with torch.no_grad():
                losses = _run(model, b, tasks, True, 0.0)
        finally:
            ops.EncoderStackFn.apply = stack
            h.remove()
        outs.append((cap, [l.clone() for l in losses]))
    (c0, l0), (c1, l1) = outs
    assert len(c0["layers"]) == dims.layers
    assert torch.equal(c0["emb"], c1["emb"]) and all(torch.equal(x, y) for x, y in zip(c0["layers"], c1["layers"]))
    assert torch.equal(l0[0], l1[0]) and abs(float(l1[1]) - float(l0[1])) > 1e-3

    # gradient at the projection outputs: at the masked rows the pretext's alone (the zeroing passes nothing back); elsewhere both
    # losses reach them, the pretext through the pooled output
    grads = {}
    orig = ops.LinearActFn.apply

    def spy(*a):
        y = orig(*a)
        if y.requires_grad:
            y.register_hook(lambda g, site=a[-1]: grads.__setitem__(site, g.detach().float().clone()))
        return y

    got = []
    ops.LinearActFn.apply = spy
    try:
        for pick in (lambda l: l[0] + l[1], lambda l: l[1], lambda l: l[0]):
            model.zero_grad(set_to_none=True)
            grads.clear()
            pick(_run(model, b0, tasks, True, 0.0)).float().sum().backward()
            got.append(dict(grads))
    finally:
        ops.LinearActFn.apply = orig
    both, pre, mlm = got
    rows = torch.zeros(b0["img"].shape[:2], dtype=torch.bool, device="cuda")
    rows.scatter_(1, b0["vis_masked_pos"] - 1, True)
    for site in ((1 << 21) + 1, (1 << 21) + 2):
        assert torch.equal(both[site][rows], pre[site][rows]), site
        assert float(mlm[site][rows].abs().sum()) == 0, site
        assert float(pre[site][rows].abs().sum(-1).amin()) > 0, site       # every masked row gets a gradient
        assert float(mlm[site][~rows].abs().sum()) > 0 and float(pre[site][~rows].abs().sum()) > 0, site


def test_graphed_step_takes_vis_masked_pos_as_an_input(deterministic):
    """A GraphedStep captured on one region-masked batch and fed batches with other masked regions equals the Python-driven step on
    each, bit for bit: the positions are read at replay, not frozen at capture."""
    model, dims = _small()
    bs = [_dev(synth.make_batch(dims, 4, seed=s, mode="mix", ragged=True, vis_mask_prob=0.25)) for s in (40, 41, 42)]
    assert not torch.equal(bs[1]["vis_masked_pos"], bs[2]["vis_masked_pos"])

    def step(m, b):
        out = _run(m, b, "img2txt", True, 0.2)
        loss = out[0] + out[1] + out[2]
        loss.backward()
        return loss

    def grads():
        return {n: p.grad.detach().clone() for n, p in model.named_parameters() if p.grad is not None}

    g = graph.GraphedStep(model, bs[0], step)
    replayed = []
    for b in bs[1:]:
        loss = g(b).clone()
        torch.cuda.synchronize()
        replayed.append((loss, grads()))
    for b, (loss, gr) in zip(bs[1:], replayed):
        model.zero_grad(set_to_none=True)
        want = step(model, b).detach()
        torch.cuda.synchronize()
        assert torch.equal(loss, want), (float(loss), float(want))
        w = grads()
        assert w.keys() == gr.keys()
        assert [n for n in w if not torch.equal(w[n], gr[n])] == []
    assert not torch.equal(replayed[0][0], replayed[1][0])


@pytest.mark.parametrize("tasks", ["img2txt", "vqa2"])
def test_deterministic_region_masked_steps_are_bitwise_equal(deterministic, tasks):
    """Dropout 0.1, region masking and drop-worst: two steps from the same seeds give the same bits."""
    res = []
    for _ in range(2):
        ops._seed_counter = itertools.count(1)
        model, dims = _small(tasks, drop=0.1)
        b = _dev(synth.make_batch(dims, 4, seed=43, mode="bi" if tasks == "vqa2" else "mix", ragged=True, tasks=tasks,
                                  vis_mask_prob=0.25))
        out = _run(model, b, tasks, True, 0.2)
        sum(l.float().sum() for l in out).backward()
        torch.cuda.synchronize()
        res.append(([l.detach().clone() for l in out], {n: p.grad.clone() for n, p in model.named_parameters() if p.grad is not None}))
    (l0, g0), (l1, g1) = res
    assert all(torch.equal(a, b) for a, b in zip(l0, l1))
    assert g0.keys() == g1.keys() and [n for n in g0 if not torch.equal(g0[n], g1[n])] == []


def test_grouped_stager_refuses_a_matrix_with_blocked_regions():
    d = synth.SMALL_L123
    b = synth.make_batch(d, 4, seed=6, mode="s2s", ragged=True, vis_mask_prob=0.25)
    m = b["input_mask"].clone()
    for i, pos in enumerate(b["vis_masked_pos"]):
        m[i][:, pos] = 0
    stager = staging.BatchStager("cuda", d.regions, d.seq_len, captions_per_image=2)
    n0 = L.lib().vlpk_launch_count()
    with pytest.raises(ValueError, match="blocked region columns"):
        stager.put(dict(b, input_mask=m, img=b["img"][::2], vis_pe=b["vis_pe"][::2]))
    assert L.lib().vlpk_launch_count() == n0
    stager.put(dict(b, img=b["img"][::2], vis_pe=b["vis_pe"][::2]))       # the loader's own matrix is accepted
    staged = stager.get()
    assert isinstance(staged["input_mask"], staging.GroupedCaptionMask)
    torch.cuda.synchronize()
