"""ORACLE SUPPORT for region masking (--vis_mask_prob, run_img2txt_dist.py: mask_image_regions = vis_mask_prob > 0) and for the
drop-worst normalisation (--max_drop_worst_ratio) on the plain path.  Test infrastructure, not product code: only tests/ import it.

Region masking in BertForPreTrainingLossMask.forward (modeling.py:1033-1143): the projected features and position encodings of
the masked regions enter the embedding as zeros (:1050-1057) and a "Selfie-like" pretext loss scores each masked region's
unmasked position encoding plus the pooled output against the unmasked features of every masked region of its sample
(:1113-1131).  The loader draws the masked regions (seq2seq_loader.py:267-269) and leaves the attention mask plain (its column
blocking at :303-304 fills a copy): vlp_b200/synth.make_batch(vis_mask_prob=...) restates that;
oracle/vlp_oracle.pretraining_loss(mask_image_regions=True) the forward.

* CASES / inputs(): the seeded cases, regenerated from vlp_b200/synth.py.
* `python -O tools/region_masking_oracle.py` runs the UNMODIFIED reference (imported through oracle/ref_shim.py, checkout at
  $VLP_REFERENCE_ROOT; its uint8 masked_fill mask is accepted through ref_shim.bool_masked_fill) and writes
  tests/golden/region_masking.pt: per case the three losses, evenly spaced samples of the embedding output, every layer output
  and the MLM logits, the pooled output, a fingerprint of every parameter gradient, and the reference's OWN fp32 -> bf16 drift
  of each (a second run with the model and inputs cast to bfloat16 on the CPU).
"""
import dataclasses
import os
import subprocess
import sys

if __debug__ and __name__ == "__main__":
    sys.exit(subprocess.call([sys.executable, "-O"] + sys.argv))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402

from tools import label_smoothing_oracle as LS  # noqa: E402
from vlp_b200 import synth  # noqa: E402

# name: (dims, batch, seed, mode, ragged, tasks, vis_mask_prob, drop_worst_ratio)
CASES = {
    "l123_s2s_vm25": (synth.SMALL_L123, 3, 1501, "s2s", True, "img2txt", 0.25, 0.0),
    "l123_s2s_vm25_dw02": (synth.SMALL_L123, 5, 1502, "s2s", True, "img2txt", 0.25, 0.2),
    "l123_bi_vqa_vm25": (synth.SMALL_L123, 3, 1503, "bi", False, "vqa2", 0.25, 0.0),
    "h768_v28996_s2s_vm25": (dataclasses.replace(synth.BERT_BASE, layers=2), 2, 1504, "s2s", True, "img2txt", 0.25, 0.0),
    "l123_mix_dw02": (synth.SMALL_L123, 5, 1505, "mix", True, "img2txt", 0.0, 0.2),
}
# Loss bound of a bf16 run against these outputs: BASELINE.md §3's 5e-3 x max(1, |ref|), and for the pretext loss twice the
# reference's own fp32 -> bf16 drift of it where that is larger.  The pretext loss is a log-softmax over dot products of H-wide
# projected features (|logit| in the tens at H = 768), so bf16 storage of its inputs alone moves it by 2.6e-2 at H = 768 (1.6e-2 on the H = 128 VQA
# case), past the floor.
LOSS_FLOOR = 5e-3


def loss_bound(gold, i):
    """Allowed |loss_i - reference| of a bf16 run on a case of tests/golden/region_masking.pt (its record `gold`).  Only the pretext
    loss (i = 1) takes the drift clause; the masked-LM and VQA losses keep BASELINE.md §3's bound."""
    floor = LOSS_FLOOR * max(1.0, abs(float(gold["losses"][i])))
    return max(floor, 2.0 * gold["drift"]["losses"][i]) if i == 1 else floor


# every drop-worst case holds a sample whose masked-LM weights are all zero: its loss is 0, so it is always kept, and it adds nothing
# to the denominator
ZERO_WEIGHT_SAMPLE = 1


def inputs(name):
    """(dims, state dict, batch, tasks, mask_image_regions, drop_worst_ratio) of CASES[name]."""
    dims, B, seed, mode, ragged, tasks, vmp, dw = CASES[name]
    sd = synth.make_state_dict(dims, seed=0, tasks=tasks)
    batch = synth.make_batch(dims, B, seed=seed, mode=mode, ragged=ragged, tasks=tasks, vis_mask_prob=vmp)
    if dw > 0:
        batch["masked_weights"][ZERO_WEIGHT_SAMPLE] = 0
    return dims, sd, batch, tasks, vmp > 0, dw


def run_reference(name, dtype=torch.float32):
    from oracle import ref_shim
    dims, sd, batch, tasks, mir, dw = inputs(name)
    model = ref_shim.build_reference_model(dims, sd, tasks=tasks).eval()
    if dtype != torch.float32:
        model = model.to(dtype)
        batch = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
    cap = {"layers": []}
    hooks = [model.bert.embeddings.register_forward_hook(lambda m, i, o: cap.__setitem__("embedding", o.detach().float())),
             model.cls.predictions.register_forward_hook(lambda m, i, o: cap.__setitem__("logits", o.detach().float())),
             model.bert.pooler.register_forward_hook(lambda m, i, o: cap.__setitem__("pooled", o.detach().float()))]
    for lyr in model.bert.encoder.layer:
        hooks.append(lyr.register_forward_hook(lambda m, i, o: cap["layers"].append(o.detach().float())))
    ans = batch["ans_labels"] if tasks == "vqa2" else None
    with ref_shim.bool_masked_fill():
        losses = model(batch["img"], batch["vis_pe"], batch["input_ids"], batch["segment_ids"], batch["input_mask"], batch["masked_ids"],
                       ans, batch["is_next"], masked_pos=batch["masked_pos"], masked_weights=batch["masked_weights"],
                       task_idx=batch["task_idx"], vis_masked_pos=batch["vis_masked_pos"], mask_image_regions=mir, drop_worst_ratio=dw)
    sum(l.float().sum() for l in losses).backward()
    for h in hooks:
        h.remove()
    grads = {k: LS.grad_fingerprint(p.grad.float()) for k, p in model.named_parameters() if p.grad is not None}
    out = {"losses": [l.detach().float().clone() for l in losses], "embedding": LS.sample(cap["embedding"]),
           "layers": [LS.sample(x) for x in cap["layers"]], "pooled": cap["pooled"].clone(), "grads": grads}
    if tasks != "vqa2":
        out["logits"] = LS.sample(cap["logits"])
    return out


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / (b.norm() + 1e-30)).item()


def drift(ref, low):
    """The reference's own fp32 -> bf16 drift: |loss difference| per loss, rel-L2 per activation sample and per gradient."""
    out = {"losses": [abs(float(a) - float(b)) for a, b in zip(low["losses"], ref["losses"])],
           "embedding": _rel(low["embedding"], ref["embedding"]), "pooled": _rel(low["pooled"], ref["pooled"]),
           "layers": [_rel(a, b) for a, b in zip(low["layers"], ref["layers"])], "grads": {}}
    if "logits" in ref:
        out["logits"] = _rel(low["logits"], ref["logits"])
    for k, f in ref["grads"].items():
        a, b = (low["grads"][k]["full"], f["full"]) if "full" in f else (low["grads"][k]["sample"], f["sample"])
        out["grads"][k] = _rel(a, b)
    return out


if __name__ == "__main__":
    torch.set_num_threads(8)
    cases = {}
    for name in CASES:
        ref = run_reference(name)
        ref["drift"] = drift(ref, run_reference(name, torch.bfloat16))
        cases[name] = ref
        print(name, [float(l) for l in ref["losses"]], "bf16 loss drift", ref["drift"]["losses"], "grads", len(ref["grads"]),
              "max grad drift", max(ref["drift"]["grads"].values()))
    out = {"case": "region_masking", "cases": cases, "torch": str(torch.__version__), "reference_commit": "74c4d85"}
    path = os.path.join(ROOT, "tests", "golden", "region_masking.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes")
