"""ORACLE SUPPORT for attention maps (BertModel / BertLayer output_attentions, the decoders' per-word maps).  Test infrastructure, not
product code: only tests/ import it.

`python -O tools/attention_maps_oracle.py` runs the UNMODIFIED reference (imported through oracle/ref_shim.py, checkout at
$VLP_REFERENCE_ROOT) on the CPU with a forward hook on every layer's attention.self.dropout — the hook a reference user writes to read
attention_probs (modeling.py:283-295); eval mode, so what the hook receives is the softmax itself — and writes
tests/golden/attention_maps.pt:

* ENCODER cases (2 layers, H = 128): the training forward's maps per layer.  Stored as SAMPLE_ROWS whole query rows per (sequence,
  head), rows drawn by a seeded generator (`rows` [B, heads, SAMPLE_ROWS]), plus `drift` per layer: the rel-L2 between the same
  rows of a second reference run with the model and inputs cast to bfloat16 — the reference algorithm's own fp32 -> bf16 drift.
  "bernoulli" replaces the loader's mask by a Bernoulli(0.6) 0/1 mask with one fully masked query row per sequence (row
  DEAD_ROW[b]); its rows always include that row.
* DECODE cases (L = 123): per step, the [MASK] row (the last query row) of every layer, over keys [0, out_len) (zero beyond the step's
  keys): "greedy" (B = 2) `maps` [B, T, layers, heads, out_len]; "beam" (K = 3, B = 1) `step_maps` [T, B*K, layers, heads, out_len]
  (step 0: the B rows at b*K) with the traces, and `chosen` [B, T, layers, heads, out_len]: frame t of pred_seq takes the row its
  hypothesis continued, found by walking the reference's back pointers as its own back-tracking does (modeling.py:1431-1472).
  Beam search runs with integer torch.div floor-patched (:1317) and Tensor.cuda the identity, as tools/ngram_beam_oracle.py does.
"""
import os
import subprocess
import sys

if __debug__ and __name__ == "__main__":
    sys.exit(subprocess.call([sys.executable, "-O"] + sys.argv))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402

from vlp_b200 import synth  # noqa: E402

SAMPLE_ROWS = 16
ROW_SEED = 4321
# name: (sequence length, batch, batch seed, loader mask mode, ragged, Bernoulli mask seed or None)
ENCODER_CASES = {
    "l123_mix": (123, 2, 1236, "mix", True, None),
    "l143_mix": (143, 2, 1431, "mix", True, None),
    "bernoulli": (123, 2, 1237, "s2s", False, 99),
}
DEAD_ROW = (17, 118)
GREEDY = dict(B=2, seed=77)
BEAM = dict(B=1, K=3, seed=78, length_penalty=0.5)
EOS_ID = 102


def dims_for(L):
    return synth.SMALL_L123 if L == 123 else synth.VlpDims(vocab=1000, hidden=128, layers=2, heads=2, inter=512, regions=100, text=L - 103)


def encoder_inputs(name):
    """(dims, state dict, batch) of ENCODER_CASES[name]; batch["input_mask"] is the [B, L, L] 0/1 mask the model attends with."""
    L, B, seed, mode, ragged, bern = ENCODER_CASES[name]
    dims = dims_for(L)
    batch = synth.make_batch(dims, B, seed=seed, mode=mode, ragged=ragged)
    if bern is not None:
        g = torch.Generator().manual_seed(bern)
        m = (torch.rand(B, L, L, generator=g) < 0.6).long()
        for b in range(B):
            m[b, DEAD_ROW[b]] = 0
        batch["input_mask"] = m
    return dims, synth.make_state_dict(dims, seed=0), batch


def sample_rows(B, heads, L, name):
    """[B, heads, SAMPLE_ROWS] query rows stored for a case (seeded; the Bernoulli case always keeps its fully masked rows)."""
    g = torch.Generator().manual_seed(ROW_SEED + sum(map(ord, name)))
    rows = torch.stack([torch.stack([torch.randperm(L, generator=g)[:SAMPLE_ROWS] for _ in range(heads)]) for _ in range(B)])
    if ENCODER_CASES[name][5] is not None:
        for b in range(B):
            rows[b, :, 0] = DEAD_ROW[b]
    return rows.sort(-1).values


def decode_inputs(B, seed):
    """(dims, state dict, (vis, vis_pe, input_ids, token_type_ids, position_ids, mask)) of the L = 123 decode cases."""
    dims = synth.SMALL_L123
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


def _hooked(model):
    """Forward hooks on every layer's attention.self.dropout; returns (captured list of attention_probs in call order, handles)."""
    cap = []
    hs = [lyr.attention.self.dropout.register_forward_hook(lambda m, i, o: cap.append(i[0].detach().float().clone()))
          for lyr in model.bert.encoder.layer]
    return cap, hs


def run_encoder(name, dtype=torch.float32):
    from oracle import ref_shim
    dims, sd, batch = encoder_inputs(name)
    model = ref_shim.build_reference_model(dims, sd).eval()
    if dtype != torch.float32:
        model = model.to(dtype)
        batch = {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in batch.items()}
    cap, hs = _hooked(model)
    with torch.no_grad():
        model(batch["img"], batch["vis_pe"], batch["input_ids"], batch["segment_ids"], batch["input_mask"], batch["masked_ids"], None,
              batch["is_next"], masked_pos=batch["masked_pos"], masked_weights=batch["masked_weights"], task_idx=batch["task_idx"],
              vis_masked_pos=batch["vis_masked_pos"], mask_image_regions=False, drop_worst_ratio=0.0)
    for h in hs:
        h.remove()
    if len(cap) != dims.layers:
        raise RuntimeError(f"{name}: {len(cap)} hook calls for {dims.layers} layers")
    B, heads, L, _ = cap[0].shape
    rows = sample_rows(B, heads, L, name)
    idx = rows.unsqueeze(-1).expand(B, heads, SAMPLE_ROWS, L)
    return rows, [p.gather(2, idx) for p in cap]


def encoder_case(name):
    rows, maps = run_encoder(name)
    _, low = run_encoder(name, torch.bfloat16)
    drift = [((lo.double() - m.double()).norm() / m.double().norm()).item() for lo, m in zip(low, maps)]
    L, B, seed, mode, ragged, bern = ENCODER_CASES[name]
    print(f"{name}: rows {tuple(rows.shape)} drift {drift}")
    return {"L": L, "B": B, "seed": seed, "mode": mode, "ragged": ragged, "bernoulli_seed": bern, "rows": rows, "maps": maps,
            "drift": drift}


def _step_rows(cap, n_layers, out_len):
    """Hook captures of one decode run -> per step [rows, layers, heads, out_len]: each layer's last query row, zero-padded."""
    if len(cap) % n_layers:
        raise RuntimeError(f"{len(cap)} hook calls for {n_layers} layers")
    steps = []
    for s in range(0, len(cap), n_layers):
        per = []
        for p in cap[s:s + n_layers]:
            row = torch.zeros(p.shape[0], p.shape[1], out_len)
            row[..., :p.shape[-1]] = p[:, :, -1]
            per.append(row)
        steps.append(torch.stack(per, 1))
    return steps


def greedy_case():
    from oracle import ref_shim
    dims, sd, args = decode_inputs(GREEDY["B"], GREEDY["seed"])
    model = ref_shim.build_reference_model(dims, sd, decoder=True, mask_word_id=103, eos_id=EOS_ID, search_beam_size=1).eval()
    cap, hs = _hooked(model)
    with torch.no_grad():
        ids, scores = model(*args, task_idx=None, sample_mode="greedy")
    for h in hs:
        h.remove()
    steps = _step_rows(cap, dims.layers, dims.seq_len)
    if len(steps) != ids.shape[1]:
        raise RuntimeError(f"greedy: {len(steps)} steps for {ids.shape[1]} words")
    print("greedy ids", ids[0].tolist())
    return {**GREEDY, "ids": ids.clone(), "scores": scores.clone(), "maps": torch.stack(steps, 1)}


def chosen_maps(step_maps, traces, K, length_penalty):
    """Restatement of the reference's back-tracking (modeling.py:1431-1472) over its traces, recording for every frame the step row
    whose [MASK] row predicted the chosen word: frame t of beam k continued row b*K + ptrs[b, t, k]."""
    wids, ptrs, scores = traces["wids"], traces["ptrs"], traces["scores"]
    T = step_maps.shape[0]
    B = wids.shape[0]
    out = torch.zeros(B, T, *step_maps.shape[2:])
    for b in range(B):
        last = T - 1
        for t in range(T):
            if all(int(w) == EOS_ID for w in wids[b, t]):
                last = t
                break
        best, pos = None, None
        for t in range(last + 1):
            for k in range(K):
                if int(wids[b, t, k]) == EOS_ID or t == last:
                    s = float(scores[b, t, k]) + length_penalty * (t + 1)
                    if best is None or s > best:
                        best, pos = s, (t, k)
        t, k = pos
        while t >= 0:
            out[b, t] = step_maps[t, b * K + (int(ptrs[b, t, k]) if t > 0 else 0)]
            k = int(ptrs[b, t, k])
            t -= 1
    return out


def beam_case():
    from oracle import ref_shim
    B, K = BEAM["B"], BEAM["K"]
    dims, sd, args = decode_inputs(B, BEAM["seed"])
    model = ref_shim.build_reference_model(dims, sd, decoder=True, mask_word_id=103, eos_id=EOS_ID, search_beam_size=K,
                                           length_penalty=BEAM["length_penalty"]).eval()
    orig_div, orig_cuda = torch.div, torch.Tensor.cuda

    def floor_div(a, b, *rest, **kw):
        if not rest and not kw and torch.is_tensor(a) and not a.is_floating_point():
            return orig_div(a, b, rounding_mode="floor")
        return orig_div(a, b, *rest, **kw)

    cap, hs = _hooked(model)
    torch.div, torch.Tensor.cuda = floor_div, (lambda t, *a, **kw: t)
    try:
        with torch.no_grad():
            traces = model(*args, task_idx=None)
    finally:
        torch.div, torch.Tensor.cuda = orig_div, orig_cuda
        for h in hs:
            h.remove()
    traces = {k: v.clone() for k, v in traces.items()}
    steps = _step_rows(cap, dims.layers, dims.seq_len)
    T = dims.seq_len - dims.regions - 2
    if len(steps) != T:
        raise RuntimeError(f"beam: {len(steps)} steps for {T} frames")
    step_maps = torch.zeros(T, B * K, *steps[0].shape[1:])
    step_maps[0, ::K] = steps[0]
    for t in range(1, T):
        step_maps[t] = steps[t]
    print("beam pred_seq", traces["pred_seq"][0].tolist())
    return {**BEAM, **traces, "step_maps": step_maps, "chosen": chosen_maps(step_maps, traces, K, BEAM["length_penalty"])}


if __name__ == "__main__":
    torch.set_num_threads(8)
    out = {"case": "attention_maps", "sample_rows": SAMPLE_ROWS, "dead_rows": DEAD_ROW,
           "encoder": {n: encoder_case(n) for n in ENCODER_CASES}, "greedy": greedy_case(), "beam": beam_case(),
           "torch": str(torch.__version__), "reference_commit": "74c4d85"}
    path = os.path.join(ROOT, "tests", "golden", "attention_maps.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes")
