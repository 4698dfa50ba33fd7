"""ORACLE SUPPORT for several captions per image in one packed pass (BertForPreTrainingLossMask(..., captions_per_image=G)).
Test infrastructure, not product code: only tests/ import it.

* CASES / inputs(): B images x G seq2seq captions, regenerated from vlp_b200/synth.py.  Pair p = b * G + g is a full loader sample
  (seq2seq_loader.py:229-359); the G pairs of image b share its region features.
* pair_batch(): the flattened B * G pairs as the reference trains on them, one L-row sample each.
* packed_mask() / packed_rows() / masked_rows(): the packed layout restated on the host: image b's sequence of L' = P + G * T rows (P =
  len_a + 2, T = L - P), its [B, L', L'] 0/1 mask (seq2seq_loader.py:291-298 per caption, no caption sees another's text), the source
  (pair, row) of every packed row and the packed row of every masked position.
* packed_loss(): the packed pass on oracle/vlp_oracle.py's embeddings / encoder / lm_head with explicit positions and the packed mask.
  With dropout off it equals pair_loss() on the flattened pairs in exact arithmetic (tests/test_grouped_captions_cpu.py, float64).
* `python -O tools/grouped_captions_oracle.py` runs the UNMODIFIED reference (imported through oracle/ref_shim.py, checkout at
  $VLP_REFERENCE_ROOT) on the flattened pairs, dropout off, and writes tests/golden/grouped_captions.pt in the format of
  label_smoothing.pt: per case the losses, samples of the embedding output, every layer output and the MLM logits, and a
  fingerprint of every parameter gradient.
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
import torch.nn.functional as F  # noqa: E402

from oracle import vlp_oracle as O  # noqa: E402
from tools import label_smoothing_oracle as LS  # noqa: E402
from vlp_b200 import synth  # noqa: E402

BASE768 = dataclasses.replace(synth.SMALL_L123, vocab=28996, hidden=768, heads=12, inter=3072)
# name: (dims, images B, captions per image G, seed, drop_worst_ratio, label_smoothing)
CASES = {
    "h128_b3g5": (synth.SMALL_L123, 3, 5, 2101, 0.0, None),
    "h128_b3g5_dw02_ls01": (synth.SMALL_L123, 3, 5, 2102, 0.2, 0.1),
    "h128_b1g19": (synth.SMALL_L123, 1, 19, 2103, 0.0, None),
    "h768_b4g5": (BASE768, 4, 5, 2104, 0.0, None),
}


def inputs(name):
    """(dims, state dict, grouped batch, G, drop_worst_ratio, label_smoothing).  The grouped batch holds the B * G pairs' text fields
    and "len_b" (int32 [B * G]), and B rows of "img" / "vis_pe"."""
    dims, B, G, seed, dw, eps = CASES[name]
    sd = synth.make_state_dict(dims, seed=0)
    batch = synth.make_batch(dims, B * G, seed=seed, mode="s2s", ragged=True)
    batch["img"], batch["vis_pe"] = batch["img"][::G].clone(), batch["vis_pe"][::G].clone()
    batch["len_b"] = (batch["input_mask"].diagonal(dim1=1, dim2=2).sum(-1) - dims.regions - 3).to(torch.int32)
    return dims, sd, batch, G, dw, eps


def pair_batch(batch, G):
    """The flattened pairs: every pair with its image's features, as the reference loader would give them."""
    out = {k: v for k, v in batch.items() if k != "len_b"}
    out["img"] = batch["img"].repeat_interleave(G, 0)
    out["vis_pe"] = batch["vis_pe"].repeat_interleave(G, 0)
    return out


def geometry(dims, G):
    """(P, T, L') of G captions per image."""
    P = dims.regions + 2
    T = dims.seq_len - P
    return P, T, P + G * T


def packed_rows(dims, G):
    """[L'] (caption g, row of pair b * G + g) behind every packed row of image b: the prefix comes from caption 0."""
    P, T, Lp = geometry(dims, G)
    return [(0, k) if k < P else ((k - P) // T, P + (k - P) % T) for k in range(Lp)]


def packed_mask(len_b, G, len_a, L):
    """int64 [B, L', L'] 0/1 mask of B images x G seq2seq captions (len_b [B * G] text tokens per pair)."""
    P = len_a + 2
    T = L - P
    Lp = P + G * T
    B = len(len_b) // G
    m = torch.zeros(B, Lp, Lp, dtype=torch.long)
    m[:, :, :P] = 1
    for b in range(B):
        for g in range(G):
            nt = min(int(len_b[b * G + g]) + 1, T)            # text rows incl. [SEP] (seq2seq_loader.py:296-298: st .. en)
            o = P + g * T
            m[b, o:o + nt, o:o + nt] = torch.tril(torch.ones(nt, nt, dtype=torch.long))
    return m


def masked_rows(masked_pos, G, P, T):
    """Packed row (within the image) of every masked position: p >= P of pair (b, g) -> P + g * T + (p - P); p < P stays."""
    g = (torch.arange(masked_pos.size(0)) % G).unsqueeze(1)
    return torch.where(masked_pos >= P, masked_pos + g * T, masked_pos)


def _mlm(sd, gathered, batch, dw, eps):
    logits = O.lm_head(sd, gathered)
    if eps:
        per = LS.label_smoothing_loss(F.log_softmax(logits.float(), dim=-1), batch["masked_ids"], eps, logits.size(-1))
    else:
        per = F.cross_entropy(logits.transpose(1, 2).float(), batch["masked_ids"], reduction="none")
    return O.loss_mask_and_normalize(per, batch["masked_weights"], dw), logits


def pair_loss(sd, dims, batch, G, dw=0.0, eps=None, return_all=False):
    """The reference's step on the flattened pairs (oracle/vlp_oracle.pretraining_loss, with the smoothed loss when eps is set)."""
    pb = pair_batch(batch, G)
    vis, vpe = O.region_projections(sd, pb["img"], pb["vis_pe"])
    ext = O.extended_attention_mask(pb["input_mask"], dtype=vis.dtype)
    emb = O.embeddings(sd, vis, vpe, pb["input_ids"], pb["segment_ids"], len_vis_input=dims.regions)
    outs = O.encoder(sd, dims.layers, emb, ext, dims.heads)
    seq = outs[-1]
    gathered = torch.gather(seq, 1, pb["masked_pos"].unsqueeze(2).expand(-1, -1, seq.size(-1)))
    loss, logits = _mlm(sd, gathered, pb, dw, eps)
    return (loss, {"embedding": emb, "layers": outs, "logits": logits}) if return_all else loss


def unpack(x, dims, G):
    """[B, L', ...] packed rows -> [B * G, L, ...] per pair: every pair's prefix is its image's, its text rows its own."""
    P, T, Lp = geometry(dims, G)
    B = x.size(0)
    rows = torch.cat([torch.arange(P).repeat(G, 1), P + torch.arange(G).unsqueeze(1) * T + torch.arange(T)], 1)     # [G, L]
    return x[:, rows.flatten()].reshape(B * G, dims.seq_len, *x.shape[2:])


def packed_loss(sd, dims, batch, G, dw=0.0, eps=None, return_all=False, p=0.0, training=False):
    """The packed pass: region projections once per image, one [B, L'] sequence per image with explicit positions, the packed mask.
    p / training: dropout on every site, as oracle/vlp_oracle.py applies it (O.MASK_PROVIDER supplies the keep masks of a replay):
    region projections over the B images, embeddings, attention probabilities and hidden states over the [B, L'] rows."""
    P, T, Lp = geometry(dims, G)
    N = batch["input_ids"].size(0)
    B = N // G
    src = packed_rows(dims, G)
    pick = torch.tensor([g * dims.seq_len + r for g, r in src])
    ids = batch["input_ids"].reshape(B, -1)[:, pick]
    tt = batch["segment_ids"].reshape(B, -1)[:, pick]
    pos = torch.tensor([r for _, r in src]).unsqueeze(0).expand(B, Lp)
    vis, vpe = O.region_projections(sd, batch["img"], batch["vis_pe"], p, training)
    ext = O.extended_attention_mask(packed_mask(batch["len_b"], G, dims.regions, dims.seq_len), dtype=vis.dtype)
    emb = O.embeddings(sd, vis, vpe, ids, tt, position_ids=pos, len_vis_input=dims.regions, p=p, training=training)
    outs = O.encoder(sd, dims.layers, emb, ext, dims.heads, p_hidden=p, p_attn=p, training=training)
    seq = outs[-1]
    rows = masked_rows(batch["masked_pos"], G, P, T) + (torch.arange(N) // G * Lp).unsqueeze(1)
    gathered = seq.reshape(B * Lp, -1)[rows]
    loss, logits = _mlm(sd, gathered, batch, dw, eps)
    return (loss, {"embedding": emb, "layers": outs, "logits": logits}) if return_all else loss


def run_reference(name):
    """The unmodified reference on the flattened pairs of CASES[name], dropout off (eval)."""
    from oracle import ref_shim
    dims, sd, batch, G, dw, eps = inputs(name)
    pb = pair_batch(batch, G)
    model = (LS.build_reference(dims, sd, eps) if eps else ref_shim.build_reference_model(dims, sd)).eval()
    cap = {"layers": []}
    hooks = [model.bert.embeddings.register_forward_hook(lambda m, i, o: cap.__setitem__("embedding", o.detach().clone())),
             model.cls.predictions.register_forward_hook(lambda m, i, o: cap.__setitem__("logits", o.detach().clone()))]
    for lyr in model.bert.encoder.layer:
        hooks.append(lyr.register_forward_hook(lambda m, i, o: cap["layers"].append(o.detach().clone())))
    losses = model(pb["img"], pb["vis_pe"], pb["input_ids"], pb["segment_ids"], pb["input_mask"], pb["masked_ids"], None, pb["is_next"],
                   masked_pos=pb["masked_pos"], masked_weights=pb["masked_weights"], task_idx=pb["task_idx"],
                   vis_masked_pos=pb["vis_masked_pos"], mask_image_regions=False, drop_worst_ratio=dw)
    sum(l.sum() for l in losses).backward()
    for h in hooks:
        h.remove()
    grads = {k: LS.grad_fingerprint(p.grad) for k, p in model.named_parameters() if p.grad is not None}
    print(name, [float(l) for l in losses], "grads", len(grads))
    return {"losses": [l.detach().clone() for l in losses], "G": G, "drop_worst_ratio": dw, "label_smoothing": eps,
            "embedding": LS.sample(cap["embedding"]), "layers": [LS.sample(x) for x in cap["layers"]], "logits": LS.sample(cap["logits"]),
            "grads": grads}


if __name__ == "__main__":
    torch.set_num_threads(16)
    out = {"case": "grouped_captions", "cases": {n: run_reference(n) for n in CASES}, "torch": str(torch.__version__),
           "reference_commit": "74c4d85"}
    path = os.path.join(ROOT, "tests", "golden", "grouped_captions.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes")
