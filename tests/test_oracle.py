"""The oracle (oracle/vlp_oracle.py) against the reference's own outputs.

tests/golden/*.pt were produced by oracle/make_golden.py running the UNMODIFIED reference on CPU; inputs and
weights are regenerated here from vlp_b200/synth.py seeds.  fp32 vs fp32 on the same machine class, so
the tolerance is tight (different op order only): rel-L2 <= 1e-5 on activations, 1e-4 on gradients.
"""
import os

import pytest
import torch

from oracle import make_golden as mg
from oracle import vlp_oracle as O
from vlp_b200 import synth


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


def oracle_run(name, with_grad=True):
    dims, B, seed, mode, ragged, tasks = mg.CASES[name]
    sd = synth.make_state_dict(dims, seed=0, tasks=tasks)
    for k, v in sd.items():
        if k != "cls.predictions.decoder.weight":   # tied to word_embeddings (same tensor object)
            v.requires_grad_(with_grad)
    batch = synth.make_batch(dims, B, seed=seed, mode=mode, ragged=ragged, tasks=tasks)
    losses, aux = O.pretraining_loss(sd, dims, batch, tasks=tasks, return_all=True)
    if with_grad:
        sum(l.sum() for l in losses).backward()
    return sd, losses, aux


@pytest.mark.parametrize("name", list(mg.CASES))
def test_oracle_matches_reference_golden(name, golden_dir):
    gold = torch.load(os.path.join(golden_dir, name + ".pt"))
    sd, losses, aux = oracle_run(name)
    for got, ref in zip(losses, gold["losses"]):
        assert abs(float(got) - float(ref)) <= 1e-5 * max(1.0, abs(float(ref)))
    assert rel(aux["embedding"], gold["embedding"]) < 1e-5
    for got, ref in zip(aux["layers"], gold["layers"]):
        assert rel(got, ref) < 1e-5
    assert rel(aux["logits"], gold["logits"]) < 1e-5
    assert rel(aux["pooled"], gold["pooled"]) < 1e-5
    n = 0
    # Some gradients are zero in exact arithmetic (the key bias: softmax ignores a per-row constant) and hold only fp32 round-off,
    # whose pattern depends on the host's vector units; those must stay at round-off level relative to the gradient scale.
    scale = max(float(fp["full"].norm()) if "full" in fp else fp["norm"] for fp in gold["grads"].values())
    for k, fp in gold["grads"].items():
        g = sd[k].grad
        assert g is not None, k
        if "full" in fp:
            if fp["full"].norm() == 0:
                assert g.norm() == 0, k
            elif fp["full"].norm() <= 1e-7 * scale:
                assert g.norm() <= 1e-7 * scale, k
            else:
                assert rel(g, fp["full"]) < 1e-4, k
        else:
            assert abs(g.norm().item() - fp["norm"]) <= 1e-4 * fp["norm"] + 1e-12, k
            assert rel(g.flatten()[fp["sample_idx"]], fp["sample"]) < 1e-4, k
        n += 1
    assert n >= 40


def test_oracle_greedy_decode_matches_reference_golden(golden_dir):
    gold = torch.load(os.path.join(golden_dir, "decode_greedy.pt"))
    dims = synth.SMALL_L123
    sd = synth.make_state_dict(dims, seed=0)
    B, R, L = 2, dims.regions, dims.seq_len
    g = torch.Generator().manual_seed(gold["seed"])
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    vis = torch.randn(B, R, dims.vis_dim, generator=g).clamp_min(0)
    pe = torch.randn(B, R, dims.pe_dim, generator=g)
    with torch.no_grad():
        ids, scores = O.greedy_decode(sd, dims, vis, pe, input_ids, tt, pos, mask, mask_word_id=103)
    assert torch.equal(ids, gold["ids"])
    assert rel(scores, gold["scores"]) < 1e-5


def test_oracle_matches_reference_loss_on_another_seed(golden_dir):
    """One more case with fresh seeds (weights 3, ragged mixed-mask batch 99) vs the reference's stored loss
    (oracle/make_golden.py run_mix_seed3)."""
    gold = torch.load(os.path.join(golden_dir, "mix_seed3.pt"))
    dims = synth.SMALL_L123
    sd = synth.make_state_dict(dims, seed=3)
    batch = synth.make_batch(dims, 3, seed=99, mode="mix", ragged=True)
    with torch.no_grad():
        got = O.pretraining_loss(sd, dims, batch)
    assert abs(float(got[0]) - float(gold["loss"])) < 1e-5


def _run_bertadam_oracle():
    from oracle import bertadam_oracle as bo
    params, wds, grads = bo.case()
    ps = [p.clone() for p in params]
    ms = [torch.zeros_like(p) for p in ps]
    vs = [torch.zeros_like(p) for p in ps]
    out = []
    for t in range(bo.CASE_STEPS):
        gs = [g.clone() for g in grads[t]]
        lrs = [bo.step(p, g, m, v, t, weight_decay=wd, **bo.CASE_HYPER) for p, g, m, v, wd in zip(ps, gs, ms, vs, wds)]
        out.append({"p": [p.clone() for p in ps], "m": [m.clone() for m in ms], "v": [v.clone() for v in vs], "grad_after": gs, "lr": lrs})
    return out


def test_bertadam_oracle_matches_reference_golden(golden_dir):
    """oracle/bertadam_oracle.py vs the reference's own BertAdam (optimization.py:112-182) — parameters, both moments, the
    in-place clipped gradients and the schedule, three steps, eight tensors straddling the clip threshold."""
    from oracle import bertadam_oracle as bo
    gold = torch.load(os.path.join(golden_dir, "bertadam.pt"))
    mine = _run_bertadam_oracle()
    assert len(gold["steps"]) == bo.CASE_STEPS
    for t, (a, b) in enumerate(zip(mine, gold["steps"])):
        for key in ("p", "m", "v", "grad_after"):
            for i, (x, y) in enumerate(zip(a[key], b[key])):
                # sums of opposite-signed terms can cancel, so the bound is a few ulp of the tensor's scale, not of each element
                # (the 1-ulp source: modern torch evaluates the clip coefficient in fp32, this restatement — like torch 1.1 — in double)
                err, scale = float((x - y).abs().max()), float(y.abs().max())
                assert err <= 1e-6 * scale, (t, key, i, err, scale)
    # schedule: get_lr() before step t reports lr * schedule((t)/t_total) for t >= 1 ([0] before any state exists)
    h = bo.CASE_HYPER
    assert gold["steps"][0]["get_lr_before"] == [0]
    for t in (1, 2):
        ref_lrs = gold["steps"][t]["get_lr_before"]
        assert all(abs(l - bo.lr_at(t, h["lr"], h["warmup"], h["t_total"], h["schedule"])) < 1e-12 for l in ref_lrs)
    # clipping really happened for some tensors and not for others
    _, _, grads = bo.case()
    scaled = [not torch.equal(g0, g1) for g0, g1 in zip(grads[0], gold["steps"][0]["grad_after"])]
    assert any(scaled) and not all(scaled)


def test_bertadam_oracle_per_parameter_schedule_matches_reference_golden(golden_dir):
    """oracle/bertadam_oracle.run_skip vs the reference's BertAdam on skip_case(): three groups (two schedules, two lrs, with and
    without decay) and two tensors that miss gradients, whose own step counts — and so learning rates — lag their group's."""
    from oracle import bertadam_oracle as bo
    gold = torch.load(os.path.join(golden_dir, "bertadam_skip.pt"))
    params, grads = bo.skip_case()
    mine = bo.run_skip(params, grads)
    assert len(gold["steps"]) == bo.SKIP_STEPS
    for t, (a, b) in enumerate(zip(mine, gold["steps"])):
        assert a["step"] == b["step"], t
        for key in ("p", "m", "v"):
            for i, (x, y) in enumerate(zip(a[key], b[key])):
                if y is None:
                    assert x is None, (t, key, i)
                    continue
                err, scale = float((x - y).abs().max()), float(y.abs().max())
                assert err <= 1e-6 * scale, (t, key, i, err, scale)
    # the lagging tensors are what the case is about: tensor 1 has no state before step 2 and sits at its own step 0 (lr 0 under
    # warmup) on that step, while its group has moved on
    assert gold["steps"][2]["step"][1] == 1 and gold["steps"][2]["step"][0] == 3
    assert torch.equal(gold["steps"][2]["p"][1], params[1])
    assert gold["steps"][2]["step"][2] == 2 and gold["steps"][4]["step"][2] == 4


def test_bertadam_schedules():
    from oracle import bertadam_oracle as bo
    assert bo.schedule_value("warmup_linear", 0.05, 0.1) == 0.5
    assert abs(bo.schedule_value("warmup_linear", 0.55, 0.1) - 0.5) < 1e-12
    assert bo.schedule_value("warmup_linear", 1.5, 0.1) == 0
    assert bo.schedule_value("warmup_constant", 0.5, 0.1) == 1.0
    assert abs(bo.schedule_value("warmup_cosine", 0.5, 0.1) - 0.5) < 1e-12
    assert bo.lr_at(7, 1e-3) == 1e-3
