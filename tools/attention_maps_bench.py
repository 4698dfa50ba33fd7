"""Cost of attention maps on the GPU: the vlpk_attn_probs kernel per layer, and greedy / beam-3 decode with and without maps.

    python tools/attention_maps_bench.py [--out results/attention_maps_h100.json]

Kernel: B = 64 sequences x 12 heads, L = 123 / 256 / 512 (encoder layout, q and k in place in a packed [B*L, 3H] projection), CUDA
events around ITERS launches after a warm-up; reported as us per layer, GB/s of fp32 P written, and that rate over the data sheet's
3.35 TB/s of HBM3 (the kernel is bound by the write of P: B * heads * L^2 * 4 bytes, against 2 * B * L * 2H bytes of q / k read).
Decode: BERT-base decoder, 100 regions, max_tgt_length 20 (out_len 122), B = 100, greedy and beam 3, with and without maps, Python-
driven and as one GraphedCall replay; median of REPS timed calls.  Prints one JSON object with the card's name and power limit."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402

from vlp_b200 import graph, ops, synth  # noqa: E402
from vlp_b200 import vlp_modules as vm  # noqa: E402

HBM = 3.35e12
ITERS = 200
REPS = 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip()


def kernel_case(L, B=64, heads=12):
    H = heads * 64
    g = torch.Generator(device="cuda").manual_seed(L)
    qkv = torch.randn(B, L, 3 * H, device="cuda", generator=g).bfloat16()
    m = torch.ones(B, L, L, dtype=torch.long, device="cuda")
    bits = ops.pack_mask(m, "zero_one")
    lse = torch.empty(B, heads, L, device="cuda")
    ctx = torch.empty(B * L, H, device="cuda", dtype=torch.bfloat16)
    from vlp_b200 import _lib as Lb
    Lb.call("vlpk_attn_core_fwd_wide", B, heads, L, L, qkv.data_ptr(), 3 * H, qkv[..., H:].data_ptr(), qkv[..., 2 * H:].data_ptr(), 3 * H,
            bits.data_ptr(), L, ctx.data_ptr(), H, lse.data_ptr(), None, 0, ops.kv_slots(L, L), Lb.stream())
    out = torch.empty(B, heads, L, L, device="cuda")
    q, k = qkv[..., :H], qkv[..., H:2 * H]
    for _ in range(10):
        ops.attn_probs(q, k, lse, bits, 0, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        ops.attn_probs(q, k, lse, bits, 0, out)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / ITERS
    written = 4.0 * B * heads * L * L
    return {"L": L, "B": B, "heads": heads, "us": round(us, 2), "GB_s_written": round(written / us / 1e3, 1),
            "hbm_share": round(written / (us * 1e-6) / HBM, 3)}


def decode_cases(B=100):
    d = synth.BERT_BASE
    L = d.regions + 2 + 20
    dims = synth.VlpDims(vocab=d.vocab, hidden=d.hidden, layers=d.layers, heads=d.heads, inter=d.inter, regions=d.regions, text=L - d.regions)
    cfg = vm.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                        intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    R = dims.regions
    g = torch.Generator().manual_seed(0)
    ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    args = (torch.randn(B, R, dims.vis_dim, generator=g).clamp_min(0).cuda().bfloat16(), torch.randn(B, R, dims.pe_dim, generator=g).cuda().bfloat16(),
            ids.cuda(), tt.cuda(), pos.cuda(), mask.cuda())
    res = {}
    for K in (1, 3):
        model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, search_beam_size=K, enable_butd=True, len_vis_input=R)
        model.load_state_dict(synth.make_state_dict(dims, 0), strict=False)
        model = model.cuda().bfloat16().eval()
        for maps in (False, True):
            fn = (lambda *a, m=maps, mod=model: mod(*a, task_idx=None, output_attentions=m))
            gc = graph.GraphedCall(fn, args)
            for how, call in (("python", lambda: fn(*args)), ("graph", lambda: gc(*args))):
                call()
                ts = []
                for _ in range(REPS):
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    call()
                    e1.record()
                    torch.cuda.synchronize()
                    ts.append(e0.elapsed_time(e1))
                res[f"{'greedy' if K == 1 else 'beam3'} {'maps' if maps else 'plain'} {how} ms"] = round(statistics.median(ts), 2)
            del gc
        del model
        torch.cuda.empty_cache()
    return {"B": B, "out_len": L, **res}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card(), "kernel": [kernel_case(L) for L in (123, 256, 512)], "decode": decode_cases()}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
