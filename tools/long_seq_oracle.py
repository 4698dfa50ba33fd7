"""ORACLE SUPPORT for sequences longer than one 128-row tile: L = max_len_b + len_vis_input + 3 (run_img2txt_dist.py:193) and
L = max_tgt_length + len_vis_input + 3 (decode_img2txt.py:127) above 128.  Test infrastructure, not product code: only tests/ import it.

* CASES / inputs(): the seeded training cases (2 layers, H = 128, 100 regions), regenerated from vlp_b200/synth.py.
* decode_inputs(): the decode inputs at max_tgt_length 40 (L = 143), laid out as oracle/make_golden.py does at L = 123.
* `python tools/long_seq_oracle.py` runs the UNMODIFIED reference (imported through oracle/ref_shim.py, checkout at $VLP_REFERENCE_ROOT)
  and writes tests/golden/long_seq.pt: per training case the losses, evenly spaced samples of the embedding output, every layer
  output, the MLM logits and the pooled output, and a fingerprint of every parameter gradient (the full tensor when it has at most
  GRAD_SAMPLES elements, otherwise norm, sum and GRAD_SAMPLES samples); the greedy ids and scores of BertForSeq2SeqDecoder; and the
  beam-search (K = 3, B = 1) traces, with torch.div patched to floor division for integer operands as in oracle/make_golden.py.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402

from oracle import make_golden as mg  # noqa: E402
from vlp_b200 import synth  # noqa: E402

# name: (L, batch, seed, mode, ragged)
CASES = {
    "l143_mix_ragged": (143, 3, 1431, "mix", True),
    "l256_s2s": (256, 2, 2561, "s2s", False),
    "l512_bi": (512, 2, 5121, "bi", False),
}
DECODE_L = 143            # max_tgt_length 40
ACT_SAMPLES = 1024
GRAD_SAMPLES = 256


def dims_for(L):
    return synth.VlpDims(vocab=1000, hidden=128, layers=2, heads=2, inter=512, regions=100, text=L - 103)


def inputs(name):
    """(dims, state dict, batch) of CASES[name]."""
    L, B, seed, mode, ragged = CASES[name]
    dims = dims_for(L)
    return dims, synth.make_state_dict(dims, seed=0), synth.make_batch(dims, B, seed=seed, mode=mode, ragged=ragged)


def decode_inputs(B, seed):
    """(dims, state dict, (vis, vis_pe, input_ids, token_type_ids, position_ids, mask)) at L = DECODE_L."""
    dims = dims_for(DECODE_L)
    R, L = dims.regions, dims.seq_len
    g = torch.Generator().manual_seed(seed)
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    vis = torch.randn(B, R, dims.vis_dim, generator=g).clamp_min(0)
    pe = torch.randn(B, R, dims.pe_dim, generator=g)
    return dims, synth.make_state_dict(dims, seed=0), (vis, pe, input_ids, tt, pos, mask)


def sample(t, n=ACT_SAMPLES):
    flat = t.detach().flatten()
    return flat[mg.big_sample_idx(flat.numel(), n)].clone()


def grad_fingerprint(g):
    if g.numel() <= GRAD_SAMPLES:
        return {"full": g.detach().clone()}
    return {"norm": g.norm().item(), "sum": g.double().sum().item(), "sample": sample(g, GRAD_SAMPLES)}


def run_training(name):
    from oracle import ref_shim
    dims, sd, batch = inputs(name)
    model = ref_shim.build_reference_model(dims, sd).eval()
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
    return {"losses": [l.detach().clone() for l in losses], "embedding": sample(cap["embedding"]), "layers": [sample(x) for x in cap["layers"]],
            "logits": sample(cap["logits"]), "pooled": sample(cap["pooled"]), "grads": grads}


def run_greedy(B=2, seed=143):
    from oracle import ref_shim
    dims, sd, args = decode_inputs(B, seed)
    model = ref_shim.build_reference_model(dims, sd, decoder=True, mask_word_id=103, eos_id=102, search_beam_size=1).eval()
    with torch.no_grad():
        ids, scores = model(*args, task_idx=None, sample_mode="greedy")
    print("greedy ids", ids[0].tolist())
    return {"ids": ids, "scores": scores, "seed": seed, "B": B}


def run_beam(B=1, K=3, seed=144, length_penalty=0.5):
    from oracle import ref_shim
    dims, sd, args = decode_inputs(B, seed)
    model = ref_shim.build_reference_model(dims, sd, decoder=True, mask_word_id=103, eos_id=102, search_beam_size=K,
                                           length_penalty=length_penalty).eval()
    orig_div = torch.div

    def floor_div(a, b, *rest, **kw):
        if not rest and not kw and torch.is_tensor(a) and not a.is_floating_point():
            return orig_div(a, b, rounding_mode="floor")
        return orig_div(a, b, *rest, **kw)

    torch.div = floor_div
    try:
        with torch.no_grad():
            traces = model(*args, task_idx=None)
    finally:
        torch.div = orig_div
    print("beam pred_seq", traces["pred_seq"][0].tolist())
    return {"seed": seed, "B": B, "K": K, "length_penalty": length_penalty,
            **{k: (v.clone() if torch.is_tensor(v) else v) for k, v in traces.items()}}


if __name__ == "__main__":
    torch.set_num_threads(8)
    out = {"case": "long_seq", "cases": {n: run_training(n) for n in CASES}, "greedy": run_greedy(), "beam": run_beam(),
           "torch": str(torch.__version__), "reference_commit": "74c4d85"}
    path = os.path.join(ROOT, "tests", "golden", "long_seq.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes")
