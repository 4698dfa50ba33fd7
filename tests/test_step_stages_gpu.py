"""GPU: stage-local checks of the training step around the encoder stack (tools/step_check.py) on real `model(...)` steps: the region
projections, the embedding, the masked-LM tail with drop-worst, and the exact composition invariants, each against fp64 of the
step's own recorded inputs.  At the production width (H = 768, B = 64, L = 123) and at H = 128, with and without region masking,
label smoothing, a relaxed head and VQA, with dropout 0.1, in default and deterministic mode.

VLPK_STEP_CHECK_REPORT=<path> writes the worst share of each bound as JSON."""
import dataclasses
import json
import os

import pytest
import torch

from tools import step_check as sc
from vlp_b200 import ops, synth
from vlp_b200 import vlp_modules as vm

pytestmark = pytest.mark.gpu
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("VLPK_STEP_CHECK_REPORT")
    if path:
        with open(path, "w") as f:
            json.dump(dict(sorted(WORST.items())), f, indent=1)


def _model(dims, tasks, drop, ls=None, relax=0):
    cfg = vm.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                        intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                        hidden_dropout_prob=drop, attention_probs_dropout_prob=drop, label_smoothing=ls, relax_projection=relax)
    torch.manual_seed(0)
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=dims.regions, tasks=tasks)
    own = model.state_dict()
    model.load_state_dict({k: v for k, v in synth.make_state_dict(dims, 0, tasks).items() if own[k].shape == v.shape}, strict=False)
    return model.cuda().bfloat16().train()


SMALL = synth.SMALL_L123
BASE2 = dataclasses.replace(synth.BERT_BASE, layers=2)
# name: (dims, B, mode, tasks, vis_mask_prob, drop_worst_ratio, label_smoothing, relax_projection)
CASES = {
    "h128_s2s_vm25_dw02": (SMALL, 6, "s2s", "img2txt", 0.25, 0.2, None, 0),
    "h128_mix_plain": (SMALL, 6, "mix", "img2txt", 0.0, 0.0, None, 0),
    "h128_mix_ls01_vm25": (SMALL, 5, "mix", "img2txt", 0.25, 0.2, 0.1, 0),
    "h128_s2s_relax2": (SMALL, 4, "s2s", "img2txt", 0.0, 0.0, None, 2),
    "h128_bi_vqa_vm25": (SMALL, 4, "bi", "vqa2", 0.25, 0.0, None, 0),
    "h768_b64_s2s_vm25_dw02": (BASE2, 64, "s2s", "img2txt", 0.25, 0.2, None, 0),
    "h768_b64_s2s_plain": (BASE2, 64, "s2s", "img2txt", 0.0, 0.0, None, 0),
}


def run_case(name, deterministic=False):
    dims, B, mode, tasks, vmp, dw, ls, relax = CASES[name]
    model = _model(dims, tasks, 0.1, ls, relax)
    batch = synth.make_batch(dims, B, seed=300 + len(name), mode=mode, ragged=True, tasks=tasks, vis_mask_prob=vmp)
    if dw > 0:
        batch["masked_weights"][1] = 0                 # a sample whose weights are all zero
    if relax:
        batch["task_idx"] = torch.arange(B) % relax
    b = {k: v.cuda() for k, v in batch.items()}
    b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()
    with sc.Recorder(model) as rec:
        losses = model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"],
                       b["ans_labels"] if tasks == "vqa2" else None, b["is_next"], masked_pos=b["masked_pos"],
                       masked_weights=b["masked_weights"], task_idx=b["task_idx"], vis_masked_pos=b["vis_masked_pos"],
                       mask_image_regions=vmp > 0, drop_worst_ratio=dw)
        sum(l.float().sum() for l in losses).backward()
        torch.cuda.synchronize()
    assert set(rec.lin) == set(sc.SITES) and rec.emb and rec.enc_in is not None
    assert rec.emb["dvis"] is not None and rec.lin[(1 << 21) + 2]["x"].shape[-1] == 1607
    shares = sc.check_step(rec, model, b, tasks, dw, losses)
    for k, v in shares.items():
        key = f"{k}" + (" (deterministic)" if deterministic else "")
        WORST[key] = max(WORST.get(key, 0.0), v)
    return shares


@pytest.mark.parametrize("name", list(CASES))
def test_step_stages(name):
    shares = run_case(name)
    assert all(v <= 1.0 for v in shares.values())
    assert any(k.startswith("projection vis_pe_embed.0") for k in shares) and "embedding dz (vis)" in shares
    if CASES[name][3] != "vqa2":
        assert "drop-worst dloss" in shares and "encoder top dy" in shares


@pytest.mark.parametrize("name", ["h128_s2s_vm25_dw02", "h128_bi_vqa_vm25"])
def test_step_stages_deterministic(name):
    before = torch.are_deterministic_algorithms_enabled()
    cublas = os.environ.get("CUBLAS_WORKSPACE_CONFIG")
    os.environ["CUBLAS_WORKSPACE_CONFIG"] = ":4096:8"
    torch.use_deterministic_algorithms(True)
    try:
        run_case(name, deterministic=True)
    finally:
        torch.use_deterministic_algorithms(before)
        if cublas is None:
            os.environ.pop("CUBLAS_WORKSPACE_CONFIG", None)
        else:
            os.environ["CUBLAS_WORKSPACE_CONFIG"] = cublas
        ops.set_device_seed_tensor(None)
