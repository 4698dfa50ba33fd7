"""ORACLE SUPPORT for the label-smoothed masked-LM loss (--label_smoothing, run_img2txt_dist.py:78): crit_mask_lm_smoothed =
LabelSmoothingLoss (loss.py:12-48), built at modeling.py:995-999 and applied at :1104-1106.  Test infrastructure, not product code:
only tests/ import it.

* label_smoothing_loss / pretraining_loss: the fp32 restatement, on top of oracle/vlp_oracle.py (same logits, same
  loss_mask_and_normalize), one op per reference op.
* CASES / inputs(): the seeded cases, regenerated from vlp_b200/synth.py.
* `python -O tools/label_smoothing_oracle.py` runs the UNMODIFIED reference (imported through oracle/ref_shim.py, checkout at
  $VLP_REFERENCE_ROOT) with config.label_smoothing set and writes tests/golden/label_smoothing.pt: per case the losses, evenly
  spaced samples (sample_idx()) of the embedding output, every layer output, the MLM logits and the pooled output, a fingerprint
  of every parameter gradient (the full tensor when it has at most GRAD_SAMPLES elements, otherwise norm, sum and GRAD_SAMPLES
  samples), the reference model's state_dict keys and the SHA-256 digest of its crit_mask_lm_smoothed.one_hot buffer.
  (-O strips the reference's `assert len_vis_input == 100`, modeling.py:231, which the 4-region case trips.)
"""
import dataclasses
import os
import pickle
import subprocess
import sys
import tempfile

if __debug__ and __name__ == "__main__":
    sys.exit(subprocess.call([sys.executable, "-O"] + sys.argv))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from oracle import make_golden as mg  # noqa: E402
from oracle import vlp_oracle as O  # noqa: E402
from vlp_b200 import synth  # noqa: E402

# name: (dims, batch, seed, mode, ragged, label_smoothing).  In every case one weighted label is forced to 0, the ignore index of the
# smoothed loss: that position adds 0 to the loss but still counts in the denominator of loss_mask_and_normalize.
CASES = {
    "l123_mix_ls01": (synth.SMALL_L123, 4, 1401, "mix", True, 0.1),
    "l123_v28996_ls01": (dataclasses.replace(synth.SMALL_L123, vocab=28996), 2, 1402, "s2s", True, 0.1),
    "tiny_ls1": (synth.TINY, 2, 1403, "s2s", False, 1.0),
}
ZERO_LABEL = (1, 0)          # (sample, prediction slot) whose label is set to 0 with its weight left at 1
ACT_SAMPLES = 1024
GRAD_SAMPLES = 256


def inputs(name):
    """(dims, state dict, batch, label_smoothing) of CASES[name]."""
    dims, B, seed, mode, ragged, eps = CASES[name]
    sd = synth.make_state_dict(dims, seed=0)
    batch = synth.make_batch(dims, B, seed=seed, mode=mode, ragged=ragged)
    b, j = ZERO_LABEL
    assert batch["masked_weights"][b, j] == 1
    batch["masked_ids"][b, j] = 0
    return dims, sd, batch, eps


def label_smoothing_loss(log_probs, target, label_smoothing, vocab, ignore_index=0):
    """LabelSmoothingLoss(label_smoothing, vocab, ignore_index=0, reduction='none') (loss.py:19-48): a dense target row per position
    — eps / (vocab - 2) everywhere, 0 at the ignore index, 1 - eps at the label, all zero for a position whose label is the ignore
    index — and the per-position sum of kl_div(log_probs, target)."""
    smooth = torch.full((vocab,), label_smoothing / (vocab - 2))
    smooth[ignore_index] = 0
    B, P = target.shape
    t = target.reshape(-1)
    q = smooth.unsqueeze(0).repeat(t.numel(), 1)
    q.scatter_(1, t.unsqueeze(1), 1.0 - label_smoothing)
    q.masked_fill_((t == ignore_index).unsqueeze(1), 0)
    return F.kl_div(log_probs.reshape(-1, vocab), q, reduction="none").view(B, P, -1).sum(2)


def pretraining_loss(sd, dims, batch, label_smoothing, drop_worst_ratio=0.0, return_all=False):
    """BertForPreTrainingLossMask.forward (img2txt) with crit_mask_lm_smoothed on the fp32 log-softmax of the logits
    (modeling.py:1104-1106) in place of crit_mask_lm; everything up to the logits is oracle/vlp_oracle.pretraining_loss."""
    _, aux = O.pretraining_loss(sd, dims, batch, return_all=True)
    logits = aux["logits"]
    ls = label_smoothing_loss(F.log_softmax(logits.float(), dim=-1), batch["masked_ids"], label_smoothing, logits.size(-1))
    mlm = O.loss_mask_and_normalize(ls.float(), batch["masked_weights"], drop_worst_ratio)
    losses = (mlm, mlm.new_zeros(1), mlm.new_zeros(1))
    return (losses, aux) if return_all else losses


def sample_idx(numel, n=ACT_SAMPLES):
    """Indices of the stored samples of a flattened tensor (evenly spaced, integer arithmetic)."""
    return mg.big_sample_idx(numel, n)


def sample(t, n=ACT_SAMPLES):
    flat = t.detach().flatten()
    return flat[sample_idx(flat.numel(), n)].clone()


def grad_fingerprint(g):
    if g.numel() <= GRAD_SAMPLES:
        return {"full": g.detach().clone()}
    return {"norm": g.norm().item(), "sum": g.double().sum().item(), "sample": sample(g, GRAD_SAMPLES)}


def build_reference(dims, state_dict, label_smoothing):
    """The reference's BertForPreTrainingLossMask (enable_butd=True) built from a BertConfig with label_smoothing set, so that its own
    constructor creates crit_mask_lm_smoothed (modeling.py:995-999), with `state_dict` loaded; the one_hot buffer keeps its
    construction value.  modeling.py:1008-1014 reads detectron_weights/fc7_{w,b}.pkl from the CWD: synthetic pickles are provided
    in a scratch directory and overwritten by the load."""
    import numpy as np
    from oracle import ref_shim
    m = ref_shim.import_reference_modeling()
    cfg = m.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                       intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                       hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, label_smoothing=label_smoothing)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.makedirs(os.path.join(tmp, "detectron_weights"))
        pickle.dump(np.zeros((2048, 2048), np.float32), open(os.path.join(tmp, "detectron_weights", "fc7_w.pkl"), "wb"))
        pickle.dump(np.zeros((2048,), np.float32), open(os.path.join(tmp, "detectron_weights", "fc7_b.pkl"), "wb"))
        os.chdir(tmp)
        try:
            torch.manual_seed(0)
            model = m.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=dims.regions, tasks="img2txt")
        finally:
            os.chdir(cwd)
    missing, unexpected = model.load_state_dict({k: v.clone() for k, v in state_dict.items()}, strict=False)
    if unexpected or list(missing) != ["crit_mask_lm_smoothed.one_hot"]:     # explicit raise: run under `python -O`
        raise RuntimeError(f"reference state_dict mismatch: missing={missing} unexpected={unexpected}")
    return model


def run_reference(name):
    dims, sd, batch, eps = inputs(name)
    model = build_reference(dims, sd, eps).eval()
    cap = {"layers": []}
    hooks = [model.bert.embeddings.register_forward_hook(lambda m, i, o: cap.__setitem__("embedding", o.detach().clone())),
             model.cls.predictions.register_forward_hook(lambda m, i, o: cap.__setitem__("logits", o.detach().clone())),
             model.bert.pooler.register_forward_hook(lambda m, i, o: cap.__setitem__("pooled", o.detach().clone()))]
    for lyr in model.bert.encoder.layer:
        hooks.append(lyr.register_forward_hook(lambda m, i, o: cap["layers"].append(o.detach().clone())))
    losses = model(batch["img"], batch["vis_pe"], batch["input_ids"], batch["segment_ids"], batch["input_mask"], batch["masked_ids"], None,
                   batch["is_next"], masked_pos=batch["masked_pos"], masked_weights=batch["masked_weights"], task_idx=batch["task_idx"],
                   vis_masked_pos=batch["vis_masked_pos"], mask_image_regions=False, drop_worst_ratio=0.0)
    sum(l.sum() for l in losses).backward()
    for h in hooks:
        h.remove()
    grads = {k: grad_fingerprint(p.grad) for k, p in model.named_parameters() if p.grad is not None}
    print(name, [float(l) for l in losses], "grads", len(grads))
    return {"losses": [l.detach().clone() for l in losses], "label_smoothing": eps, "embedding": sample(cap["embedding"]),
            "layers": [sample(x) for x in cap["layers"]], "logits": sample(cap["logits"]), "pooled": sample(cap["pooled"]), "grads": grads,
            "state_dict_keys": sorted(model.state_dict().keys()),
            "one_hot": mg.tensor_digest(model.crit_mask_lm_smoothed.one_hot)}


if __name__ == "__main__":
    torch.set_num_threads(8)
    out = {"case": "label_smoothing", "cases": {n: run_reference(n) for n in CASES}, "torch": str(torch.__version__),
           "reference_commit": "74c4d85"}
    path = os.path.join(ROOT, "tests", "golden", "label_smoothing.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes")
