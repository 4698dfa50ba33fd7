"""ORACLE SUPPORT for the relaxed per-task MLM head projection (--relax_projection, run_img2txt_dist.py:183-185, 314): the transform
becomes Linear(H, nH) -> GELU -> LayerNorm(nH) and each sample keeps the H-wide slice named by its task_idx (modeling.py:420-482), and
from_pretrained converts the head between relaxed and plain layouts (:704-732).  Test infrastructure, not product code: only tests/
import it.

* relaxed_state_dict / inputs(): the seeded cases, regenerated from vlp_b200/synth.py plus a seeded [nH, H] transform.
* lm_head / pretraining_loss: the fp32 restatement of the relaxed head (built from oracle/vlp_oracle.py's linear, gelu and
  layer_norm, one op per reference op) and of the training loss around it; with label smoothing the loss is
  tools/label_smoothing_oracle.label_smoothing_loss.
* `python -O tools/relax_projection_oracle.py` runs the UNMODIFIED reference (imported through oracle/ref_shim.py, checkout at
  $VLP_REFERENCE_ROOT) and writes tests/golden/relax_projection.pt:
  - per training case: the losses, evenly spaced samples of the embedding output, every layer output, the MLM logits and the pooled
    output, every parameter gradient (full when it has at most GRAD_SAMPLES elements and for every cls.predictions.transform.*
    tensor, otherwise norm, sum and GRAD_SAMPLES samples), and the reference model's state_dict keys and shapes;
  - "from_pretrained": SHA-256 digests of every tensor the reference's from_pretrained loads for a relaxed checkpoint into a plain
    model with task_idx=3 and with task_idx unset, and for a plain checkpoint into a relaxed model; and the exception the reference
    raises for a relax-2 checkpoint into a relax-4 model (probed in a child process WITHOUT -O, since that check is an assert);
  - "decode": greedy ids / scores / top-1 minus top-2 logit margins of a plain decoder loaded from a relaxed checkpoint with
    task_idx=3 and of a relaxed decoder with per-sample task ids, and the beam-search traces (K = 3, B = 1) of the relaxed decoder
    (torch.div patched to floor semantics, as in oracle/make_golden.run_decode_beam).
  (-O strips the reference's `assert len_vis_input == 100`, modeling.py:231, which the 4-region case trips.)
"""
import json
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
from tools import label_smoothing_oracle as LSO  # noqa: E402
from vlp_b200 import synth  # noqa: E402

RELAX = 4
# name: (dims, batch, seed, mode, ragged, relax_projection, label_smoothing).  Mixed s2s / bi batches: both task ids (3 and 0) occur.
CASES = {
    "l123_mix_relax4": (synth.SMALL_L123, 4, 1501, "mix", True, RELAX, None),
    "tiny_relax4_ls01": (synth.TINY, 3, 1503, "mix", False, RELAX, 0.1),
}
ACT_SAMPLES = 1024
GRAD_SAMPLES = 256
HEAD = "cls.predictions.transform."
DECODE_SEED, BEAM_SEED = 79, 80
DECODE_TASKS = (3, 0)          # per-sample task ids of the relaxed greedy decode (s2s, bidirectional)
BEAM_K, BEAM_TASK, LENGTH_PENALTY = 3, 3, 0.5


def relaxed_state_dict(sd, hidden, n, seed=1500):
    """`sd` with its MLM head transform replaced by a seeded relaxed one: dense [nH, H] + [nH], LayerNorm [nH] (the slices differ)."""
    g = torch.Generator().manual_seed(seed)
    out = {k: v.clone() for k, v in sd.items()}
    out["cls.predictions.decoder.weight"] = out["bert.embeddings.word_embeddings.weight"]
    out[HEAD + "dense.weight"] = torch.randn(n * hidden, hidden, generator=g) * 0.02
    out[HEAD + "dense.bias"] = 0.02 * torch.randn(n * hidden, generator=g)
    out[HEAD + "LayerNorm.weight"] = 1.0 + 0.05 * torch.randn(n * hidden, generator=g)
    out[HEAD + "LayerNorm.bias"] = 0.02 * torch.randn(n * hidden, generator=g)
    return out


def inputs(name):
    """(dims, state dict, batch, relax_projection, label_smoothing) of CASES[name]."""
    dims, B, seed, mode, ragged, n, eps = CASES[name]
    sd = relaxed_state_dict(synth.make_state_dict(dims, seed=0), dims.hidden, n)
    batch = synth.make_batch(dims, B, seed=seed, mode=mode, ragged=ragged)
    return dims, sd, batch, n, eps


def lm_head(sd, x, relax_projection, task_idx):
    """modeling.py:420-435 (transform, [nH, H] dense and a LayerNorm over nH) + :471-476 (sample b keeps slice task_idx[b]) +
    :478-482 (tied decoder + bias)."""
    t = O.layer_norm(O.gelu(O.linear(x, sd, HEAD + "dense")), sd[HEAD + "LayerNorm.weight"], sd[HEAD + "LayerNorm.bias"])
    if relax_projection > 1:
        B, P = t.shape[0], t.shape[1]
        t = t.view(B, P, relax_projection, -1)[torch.arange(B), :, task_idx, :]
    return F.linear(t, sd["bert.embeddings.word_embeddings.weight"]) + sd["cls.predictions.bias"]


def pretraining_loss(sd, dims, batch, relax_projection, label_smoothing=None, return_all=False):
    """BertForPreTrainingLossMask.forward (img2txt, eval, drop_worst_ratio 0, modeling.py:1033-1111) with the relaxed head: the
    oracle's region projections, embeddings and encoder, then lm_head above with the batch's task_idx, then
    crit_mask_lm (or crit_mask_lm_smoothed on the fp32 log-softmax) and loss_mask_and_normalize."""
    vis, vpe = O.region_projections(sd, batch["img"], batch["vis_pe"])
    ext = O.extended_attention_mask(batch["input_mask"], dtype=vis.dtype)
    emb = O.embeddings(sd, vis, vpe, batch["input_ids"], batch["segment_ids"], len_vis_input=dims.regions)
    outs = O.encoder(sd, dims.layers, emb, ext, dims.heads)
    seq = outs[-1]
    pos = batch["masked_pos"]
    gathered = torch.gather(seq, 1, pos.unsqueeze(2).expand(-1, -1, seq.size(-1)))
    logits = lm_head(sd, gathered, relax_projection, batch["task_idx"])
    if label_smoothing:
        per = LSO.label_smoothing_loss(F.log_softmax(logits.float(), dim=-1), batch["masked_ids"], label_smoothing, logits.size(-1))
    else:
        per = F.cross_entropy(logits.transpose(1, 2).float(), batch["masked_ids"], reduction="none")
    mlm = O.loss_mask_and_normalize(per.float(), batch["masked_weights"], 0.0)
    losses = (mlm, mlm.new_zeros(1), mlm.new_zeros(1))
    if return_all:
        return losses, {"embedding": emb, "layers": outs, "logits": logits, "pooled": O.pooler(sd, seq)}
    return losses


def sample(t, n=ACT_SAMPLES):
    flat = t.detach().flatten()
    return flat[mg.big_sample_idx(flat.numel(), n)].clone()


def grad_fingerprint(name, g):
    if g.numel() <= GRAD_SAMPLES or name.startswith(HEAD):
        return {"full": g.detach().clone()}
    return {"norm": g.norm().item(), "sum": g.double().sum().item(), "sample": sample(g, GRAD_SAMPLES)}


def decode_inputs(dims, B, seed):
    """Decoder inputs as decode_img2txt.py / Preprocess4Seq2seqDecoder build them (same layout as oracle/make_golden.run_decode)."""
    R, L = dims.regions, dims.seq_len
    g = torch.Generator().manual_seed(seed)
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    token_type_ids = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    position_ids = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    vis = torch.randn(B, R, dims.vis_dim, generator=g).clamp_min(0)
    pe = torch.randn(B, R, dims.pe_dim, generator=g)
    return vis, pe, input_ids, token_type_ids, position_ids, mask


def checkpoint_config(dims):
    return {"vocab_size": dims.vocab, "hidden_size": dims.hidden, "num_hidden_layers": dims.layers, "num_attention_heads": dims.heads,
            "intermediate_size": dims.inter, "hidden_act": "gelu", "hidden_dropout_prob": 0.1, "attention_probs_dropout_prob": 0.1,
            "max_position_embeddings": dims.max_pos, "type_vocab_size": dims.type_vocab, "initializer_range": 0.02}


def write_checkpoint_dir(path, cfg):
    """bert_config.json plus the synthetic detectron_weights/fc7_{w,b}.pkl the reference reads from the CWD (modeling.py:1008-1014)."""
    import numpy as np
    with open(os.path.join(path, "bert_config.json"), "w") as f:
        f.write(json.dumps(cfg))
    os.makedirs(os.path.join(path, "detectron_weights"), exist_ok=True)
    with open(os.path.join(path, "detectron_weights", "fc7_w.pkl"), "wb") as f:
        pickle.dump(np.zeros((2048, 2048), np.float32), f)
    with open(os.path.join(path, "detectron_weights", "fc7_b.pkl"), "wb") as f:
        pickle.dump(np.zeros((2048,), np.float32), f)


def from_pretrained_checkpoints():
    """The checkpoints of the from_pretrained cases: oracle/make_golden.from_pretrained_case() (TF-era names, 2 -> 6 segment types,
    64 -> 128 positions) as is ("plain") and with a relaxed head of 4 or 2 slices.  Returns (writer, {name: state_dict}, kwargs)."""
    write, sd, kw = mg.from_pretrained_case()
    H = sd["bert.embeddings.word_embeddings.weight"].shape[1]
    sds = {"plain": sd, "relax4": relaxed_state_dict(sd, H, 4, seed=1510), "relax2": relaxed_state_dict(sd, H, 2, seed=1511)}
    return write, sds, kw


# (checkpoint, from_pretrained kwargs) of each remap case
FROM_PRETRAINED = {
    "relax4_to_plain_task3": ("relax4", dict(relax_projection=0, task_idx=3)),
    "relax4_to_plain_unset": ("relax4", dict(relax_projection=0)),
    "plain_to_relax4": ("plain", dict(relax_projection=4)),
}
MISMATCH = ("relax2", dict(relax_projection=4))


def _in_dir(tmp, fn):
    cwd = os.getcwd()
    os.chdir(tmp)
    try:
        return fn()
    finally:
        os.chdir(cwd)


def _reference_from_pretrained(m, cls, ckpt, extra, **kw):
    write, sds, base_kw = from_pretrained_checkpoints()
    with tempfile.TemporaryDirectory() as tmp:
        write(tmp)
        return _in_dir(tmp, lambda: getattr(m, cls).from_pretrained(tmp, state_dict={k: v.clone() for k, v in sds[ckpt].items()},
                                                                    fp32_embedding=False, **base_kw, **extra, **kw))


def mismatch_probe():
    """Run in a child process without -O: what the reference's from_pretrained raises for a relax-2 checkpoint into a relax-4 model."""
    from oracle import ref_shim
    m = ref_shim.import_reference_modeling()
    ckpt, extra = MISMATCH
    try:
        _reference_from_pretrained(m, "BertForPreTrainingLossMask", ckpt, extra)
        out = {"raised": None}
    except Exception as e:  # noqa: BLE001 — the type is the record
        out = {"raised": type(e).__name__, "message": str(e)}
    print("PROBE " + json.dumps(out))


def run_from_pretrained():
    from oracle import ref_shim
    m = ref_shim.import_reference_modeling()
    out = {}
    for name, (ckpt, extra) in FROM_PRETRAINED.items():
        ref = _reference_from_pretrained(m, "BertForPreTrainingLossMask", ckpt, extra)
        out[name] = {k: mg.tensor_digest(v) for k, v in ref.state_dict().items()}
        print(name, tuple(ref.state_dict()[HEAD + "dense.weight"].shape))
    env = dict(os.environ)
    res = subprocess.run([sys.executable, "-c", "from tools import relax_projection_oracle as R; R.mismatch_probe()"], cwd=ROOT, env=env,
                         capture_output=True, text=True, check=True)
    probe = json.loads([ln for ln in res.stdout.splitlines() if ln.startswith("PROBE ")][-1][len("PROBE "):])
    print("relax2 -> relax4:", probe)
    return {"digests": out, "mismatch": probe}


def build_reference(dims, state_dict, relax_projection=0, label_smoothing=None, decoder=False, **kw):
    """The reference's BertForPreTrainingLossMask / BertForSeq2SeqDecoder (enable_butd=True) from a BertConfig with relax_projection
    (and label_smoothing) set, with `state_dict` loaded (the smoothed loss's one_hot buffer keeps its construction value)."""
    from oracle import ref_shim
    m = ref_shim.import_reference_modeling()
    cfg = m.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                       intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                       hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1, relax_projection=relax_projection,
                       label_smoothing=label_smoothing)
    with tempfile.TemporaryDirectory() as tmp:
        write_checkpoint_dir(tmp, {})
        torch.manual_seed(0)
        if decoder:
            model = _in_dir(tmp, lambda: m.BertForSeq2SeqDecoder(cfg, **kw))
        else:
            model = _in_dir(tmp, lambda: m.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=dims.regions, tasks="img2txt"))
    missing, unexpected = model.load_state_dict({k: v.clone() for k, v in state_dict.items()}, strict=False)
    if unexpected or [k for k in missing if k != "crit_mask_lm_smoothed.one_hot"]:      # explicit raise: run under `python -O`
        raise RuntimeError(f"reference state_dict mismatch: missing={missing} unexpected={unexpected}")
    return model


def run_reference(name):
    dims, sd, batch, n, eps = inputs(name)
    model = build_reference(dims, sd, n, eps).eval()
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
    grads = {k: grad_fingerprint(k, p.grad) for k, p in model.named_parameters() if p.grad is not None}
    print(name, "task ids", batch["task_idx"].tolist(), [float(l) for l in losses], "grads", len(grads))
    return {"losses": [l.detach().clone() for l in losses], "relax_projection": n, "label_smoothing": eps,
            "embedding": sample(cap["embedding"]), "layers": [sample(x) for x in cap["layers"]], "logits": sample(cap["logits"]),
            "pooled": sample(cap["pooled"]), "grads": grads,
            "state_dict_shapes": {k: tuple(v.shape) for k, v in model.state_dict().items()}}


def _greedy(model, args, task_idx):
    gaps = []

    def hook(m, i, o):
        top2 = torch.topk(o.detach(), 2, dim=-1).values
        gaps.append(top2[..., 0] - top2[..., 1])
    h = model.cls.predictions.register_forward_hook(hook)
    try:
        with torch.no_grad():
            ids, scores = model(*args, task_idx=task_idx, sample_mode="greedy")
    finally:
        h.remove()
    return {"ids": ids.clone(), "scores": scores.clone(), "gaps": torch.cat(gaps, dim=1)}


def run_decode():
    from oracle import ref_shim
    m = ref_shim.import_reference_modeling()
    dims = synth.SMALL_L123
    sd = relaxed_state_dict(synth.make_state_dict(dims, seed=0), dims.hidden, RELAX)
    dec_kw = dict(mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=dims.regions)
    args = decode_inputs(dims, len(DECODE_TASKS), DECODE_SEED)
    out = {"seed": DECODE_SEED, "tasks": DECODE_TASKS}
    # decode_img2txt.py:161-168: a plain decoder built from a relaxed checkpoint with task_idx=3
    with tempfile.TemporaryDirectory() as tmp:
        write_checkpoint_dir(tmp, checkpoint_config(dims))
        plain = _in_dir(tmp, lambda: m.BertForSeq2SeqDecoder.from_pretrained(tmp, state_dict={k: v.clone() for k, v in sd.items()},
                                                                            relax_projection=0, task_idx=3, search_beam_size=1, **dec_kw))
    out["greedy_plain_task3"] = _greedy(plain.eval(), args, None)
    relaxed = build_reference(dims, sd, RELAX, decoder=True, search_beam_size=1, **dec_kw).eval()
    out["greedy_relax4"] = _greedy(relaxed, args, torch.tensor(DECODE_TASKS))
    beam = build_reference(dims, sd, RELAX, decoder=True, search_beam_size=BEAM_K, length_penalty=LENGTH_PENALTY, **dec_kw).eval()
    orig_div = torch.div

    def floor_div(a, b, *args, **kw):
        if not args and not kw and torch.is_tensor(a) and not a.is_floating_point():
            return orig_div(a, b, rounding_mode="floor")
        return orig_div(a, b, *args, **kw)
    torch.div = floor_div
    try:
        with torch.no_grad():
            traces = beam(*decode_inputs(dims, 1, BEAM_SEED), task_idx=torch.tensor([BEAM_TASK]))
    finally:
        torch.div = orig_div
    out["beam_relax4"] = {"seed": BEAM_SEED, "K": BEAM_K, "task": BEAM_TASK, "length_penalty": LENGTH_PENALTY,
                          **{k: v.clone() for k, v in traces.items()}}
    for k in ("greedy_plain_task3", "greedy_relax4"):
        print(k, out[k]["ids"].tolist())
    print("beam_relax4", out["beam_relax4"]["pred_seq"][0].tolist())
    return out


if __name__ == "__main__":
    torch.set_num_threads(8)
    out = {"case": "relax_projection", "cases": {n: run_reference(n) for n in CASES}, "from_pretrained": run_from_pretrained(),
           "decode": run_decode(), "torch": str(torch.__version__), "reference_commit": "74c4d85"}
    path = os.path.join(ROOT, "tests", "golden", "relax_projection.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes")
