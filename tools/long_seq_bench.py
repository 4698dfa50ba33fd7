"""Long-sequence measurements (L > 128): the attention kernels alone and graphed BERT-base training steps.

* attention fwd / bwd (12 heads, dropout 0.1, loader s2s mask) at L in {123, 143, 256, 512} with B * L held near 7 872 tokens
  (B = 64, 55, 31, 15); at L = 123 both the single-tile kernels and the KV-tiled ones (option "attn_tiled").  Median CUDA-event time of
  back-to-back launches over rotating buffers, and TFLOP/s from the algorithmic FLOPs (4 B h L^2 64 forward, 10 B h L^2 64 backward;
  the tiled backward's recompute is not counted);
* torch.nn.functional.scaled_dot_product_attention forward + backward on the same bf16 inputs and additive mask (no dropout), as a
  reference point;
* graphed BERT-base training steps (vlp_b200.graph.GraphedStep, dropout 0.1) at L = 143 / B = 64 and L = 256 / B = 32, samples/s.

Prints the card name and power limit and writes one JSON line per measurement to --out (default results/long_seq_h100.json).
python tools/long_seq_bench.py [--out PATH]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from vlp_b200 import _lib as L  # noqa: E402
from vlp_b200 import ops, synth  # noqa: E402

DEV, BF = "cuda", torch.bfloat16
HEADS, HD = 12, 64


def timed(fn, nset, reps=20, rounds=7):
    """Median microseconds per call of fn(i) over `rounds` windows of `reps` back-to-back calls (after a warm-up of every buffer set)."""
    for i in range(nset):
        fn(i)
    torch.cuda.synchronize()
    ts = []
    for _ in range(rounds):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for r in range(reps):
            fn(r % nset)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / reps)
    ts.sort()
    return ts[len(ts) // 2]


def s2s_mask(B, Lq):
    n_src = Lq - 21
    m = torch.zeros(B, Lq, Lq, device=DEV, dtype=torch.int64)
    m[:, :, :n_src] = 1
    m[:, n_src:, n_src:] = torch.tril(torch.ones(21, 21, device=DEV, dtype=torch.int64))
    return m


def attention(Lq, B, tiled):
    H = HEADS * HD
    nset = 4
    torch.manual_seed(0)
    qkv = [torch.randn(B, Lq, 3 * H, device=DEV).to(BF) for _ in range(nset)]
    dctx = [torch.randn(B, Lq, H, device=DEV).to(BF) for _ in range(nset)]
    ctx = [torch.zeros(B, Lq, H, device=DEV, dtype=BF) for _ in range(nset)]
    dqkv = [torch.zeros(B, Lq, 3 * H, device=DEV, dtype=BF) for _ in range(nset)]
    lse = [torch.zeros(B, HEADS, Lq, device=DEV) for _ in range(nset)]
    mask = s2s_mask(B, Lq)
    bits = ops.pack_mask(mask, "zero_one")
    slots = ops.kv_slots(Lq, Lq)
    drop = L.VlpkDropout(0.1, 99, None)
    L.call("vlpk_debug_set_option", b"attn_tiled", 1 if tiled else 0)

    def fwd(i):
        q = qkv[i]
        L.call("vlpk_attn_core_fwd_wide", B, HEADS, Lq, Lq, q.data_ptr(), 3 * H, q[..., H:].data_ptr(), q[..., 2 * H:].data_ptr(), 3 * H,
               bits.data_ptr(), Lq, ctx[i].data_ptr(), H, lse[i].data_ptr(), drop, 3, slots, L.stream())

    def bwd(i):
        q = qkv[i]
        L.call("vlpk_attn_core_bwd_wide", B, HEADS, Lq, q.data_ptr(), q[..., H:].data_ptr(), q[..., 2 * H:].data_ptr(), 3 * H, bits.data_ptr(),
               Lq, ctx[i].data_ptr(), dctx[i].data_ptr(), H, lse[i].data_ptr(), dqkv[i].data_ptr(), dqkv[i][..., H:].data_ptr(),
               dqkv[i][..., 2 * H:].data_ptr(), 3 * H, drop, 3, slots, L.stream())

    try:
        t_f, t_b = timed(fwd, nset), timed(bwd, nset)
    finally:
        L.call("vlpk_debug_set_option", b"attn_tiled", 0)
    flops = B * HEADS * Lq * Lq * HD
    out = [{"what": "attn_fwd", "kernels": "tiled" if tiled or Lq > 128 else "single_tile", "L": Lq, "B": B, "us": t_f,
            "tflops": 4 * flops / t_f / 1e6},
           {"what": "attn_bwd", "kernels": "tiled" if tiled or Lq > 128 else "single_tile", "L": Lq, "B": B, "us": t_b,
            "tflops": 10 * flops / t_b / 1e6}]
    # SDPA forward + backward on the same bf16 inputs and additive mask, no dropout
    add = ((1 - mask.to(BF)) * -10000.0)[:, None]
    qs = [t.view(B, Lq, 3, HEADS, HD).permute(2, 0, 3, 1, 4) for t in qkv]
    leaves = [[x.detach().clone().requires_grad_(True) for x in (s[0], s[1], s[2])] for s in qs]
    gos = [d.view(B, Lq, HEADS, HD).transpose(1, 2) for d in dctx]

    def sdpa(i):
        q, k, v = leaves[i]
        o = F.scaled_dot_product_attention(q, k, v, attn_mask=add)
        torch.autograd.grad(o, (q, k, v), gos[i])

    t_s = timed(sdpa, nset)
    out.append({"what": "sdpa_fwd_bwd", "L": Lq, "B": B, "us": t_s, "tflops": 14 * flops / t_s / 1e6})
    return out


def graphed_steps(Lq, B, steps=20):
    from vlp_b200 import graph
    from vlp_b200 import vlp_modules as vm
    d = synth.VlpDims(text=Lq - 103)
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions).cuda().bfloat16().train()
    host = synth.make_batch(d, B, seed=1, mode="mix", ragged=True)
    b = {k: v.cuda() for k, v in host.items()}
    b["img"], b["vis_pe"] = b["img"].bfloat16(), b["vis_pe"].bfloat16()

    def step(m, x):
        out = m(x["img"], x["vis_pe"], x["input_ids"], x["segment_ids"], x["input_mask"], x["masked_ids"], None, x["is_next"],
                masked_pos=x["masked_pos"], masked_weights=x["masked_weights"], task_idx=x["task_idx"], drop_worst_ratio=0.0)
        loss = out[0] + out[1] + out[2]
        loss.backward()
        return loss

    g = graph.GraphedStep(model, b, step)
    for _ in range(3):
        g()
    torch.cuda.synchronize()
    ts = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            g()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) / steps)
    ts.sort()
    ops.set_device_seed_tensor(None)
    ms = ts[len(ts) // 2]
    return {"what": "graphed_bert_base_step", "L": Lq, "B": B, "ms": ms, "samples_per_s": B / ms * 1e3}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "results", "long_seq_h100.json"))
    a = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("card:", card)
    rows = []
    for Lq, B, tiled in ((123, 64, False), (123, 64, True), (143, 55, False), (256, 31, False), (512, 15, False)):
        rows += attention(Lq, B, tiled)
    rows.append(graphed_steps(143, 64))
    rows.append(graphed_steps(256, 32))
    with open(a.out, "w") as f:
        for r in rows:
            r["card"] = card
            print(json.dumps(r))
            f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
