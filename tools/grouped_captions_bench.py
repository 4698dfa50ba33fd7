"""Several captions per image in one packed pass (captions_per_image = G) against today's one-sequence-per-pair step.

    python tools/grouped_captions_bench.py [--out results/grouped_captions_h100.json] [--steps 30]

BERT-base bf16 caption step (100 regions, L = 123, dropout 0.1, drop_worst_ratio 0, forward + backward, optimizer excluded), each arm a
vlp_b200.graph.GraphedStep replay on a synthetic seq2seq batch with ragged captions.  Two comparisons:
  320 pairs per step: today's step on 320 pairs against 64 images x G = 5 (the same number of pairs);
  64 images per step: today's step on 64 pairs (one caption per image) against 64 images x G = 5.
The arms of a comparison alternate replay by replay in one loop; each replay is timed with CUDA events.  Reported per arm: pairs/s
from the median step time, p5 / p50 / p95 step time, and peak allocated memory of the arm's capture and replays.  A separate
torch.profiler run of the grouped step (not part of the timings) gives the attention kernels' share of its device time.  The card's
name, power limit and SM clock are queried in the same run."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402

from tools import grouped_captions_oracle as GO  # noqa: E402
from vlp_b200 import graph, ops, staging, synth  # noqa: E402
from vlp_b200 import vlp_modules as vm  # noqa: E402

G = 5


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def build():
    d = synth.BERT_BASE
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos, hidden_dropout_prob=0.1, attention_probs_dropout_prob=0.1)
    torch.manual_seed(0)
    model = vm.BertForPreTrainingLossMask(cfg, enable_butd=True, len_vis_input=d.regions)
    return model.to("cuda", torch.bfloat16).train(), d


def batch(d, images, g, seed):
    """Device batch of `images` x g pairs: g = 1 is today's format (tensor mask synthesised per pair), g > 1 the grouped one."""
    h = synth.make_batch(d, images * g, seed=seed, mode="s2s", ragged=True)
    b = {k: v.cuda() for k, v in h.items()}
    b["img"], b["vis_pe"] = b["img"][::g].bfloat16().contiguous(), b["vis_pe"][::g].bfloat16().contiguous()
    len_b = (h["input_mask"].diagonal(dim1=1, dim2=2).sum(-1) - d.regions - 3).to(torch.int32).cuda()
    if g > 1:
        b["input_mask"] = staging.GroupedCaptionMask.synthesize(len_b, g, d.regions, d.seq_len)
    else:
        b["input_mask"] = staging.PackedAttentionMask.synthesize(len_b, torch.ones_like(len_b), d.regions, d.seq_len)
    return b


def step(g):
    def body(model, b):
        out = model(b["img"], b["vis_pe"], b["input_ids"], b["segment_ids"], b["input_mask"], b["masked_ids"], None, b["is_next"],
                    masked_pos=b["masked_pos"], masked_weights=b["masked_weights"], task_idx=b["task_idx"], drop_worst_ratio=0.0,
                    captions_per_image=g)
        loss = out[0] + out[1] + out[2]
        loss.backward()
        return loss
    return body


def pct(v, q):
    v = sorted(v)
    return v[min(len(v) - 1, int(round(q * (len(v) - 1))))]


def compare(model, d, arms, steps):
    """arms: [(name, images, g)], alternating replays."""
    graphs, times, peaks, pairs = {}, {}, {}, {}
    for name, images, g in arms:
        torch.cuda.reset_peak_memory_stats()
        b = batch(d, images, g, seed=7)
        graphs[name] = graph.GraphedStep(model, b, step(g))
        graphs[name]()
        torch.cuda.synchronize()
        peaks[name] = torch.cuda.max_memory_allocated() / 2**30
        times[name], pairs[name] = [], images * g
        model.zero_grad(set_to_none=True)
        graphs[name].loss = None
    for _ in range(steps):
        for name, _, _ in arms:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            graphs[name]()
            e1.record()
            e1.synchronize()
            times[name].append(e0.elapsed_time(e1))
    out = {}
    for name, _, _ in arms:
        t = times[name]
        out[name] = {"pairs": pairs[name], "pairs_per_s": round(pairs[name] / (pct(t, 0.5) / 1e3), 1), "ms_p5": round(pct(t, 0.05), 3),
                     "ms_p50": round(pct(t, 0.5), 3), "ms_p95": round(pct(t, 0.95), 3), "peak_alloc_gib": round(peaks[name], 2)}
    del graphs
    torch.cuda.empty_cache()
    return out


def attention_share(model, d, images, g, out_dir):
    """Device time of the attention kernels over all kernels of one grouped step (torch.profiler, separate run)."""
    from torch.profiler import ProfilerActivity, profile
    b = batch(d, images, g, seed=9)
    body = step(g)
    for _ in range(2):
        model.zero_grad(set_to_none=True)
        body(model, b)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        model.zero_grad(set_to_none=True)
        body(model, b)
        torch.cuda.synchronize()
    total, attn, names = 0.0, 0.0, {}
    for e in prof.key_averages():
        t = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
        if t <= 0:
            continue
        total += t
        if "attn" in e.key.lower() or "mha" in e.key.lower():
            attn += t
            names[e.key[:80]] = round(t / 1e3, 3)
    if out_dir:
        prof.export_chrome_trace(os.path.join(out_dir, "grouped_captions_trace.json"))
    return {"images": images, "G": g, "attention_ms": round(attn / 1e3, 3), "all_kernels_ms": round(total / 1e3, 3),
            "attention_share": round(attn / max(total, 1e-9), 4), "attention_kernels_ms": names}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--trace_dir", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "grouped_captions_bench needs a GPU"
    model, d = build()
    P, T, Lp = GO.geometry(d, G)
    res = {"card": card(), "geometry": {"L": d.seq_len, "prefix": P, "text": T, "G": G, "packed_len": Lp}, "steps": args.steps,
           "320_pairs": compare(model, d, [("today_b320", 320, 1), ("grouped_64x5", 64, G)], args.steps),
           "64_images": compare(model, d, [("today_b64", 64, 1), ("grouped_64x5", 64, G)], args.steps)}
    ops.set_device_seed_tensor(None)
    res["profile"] = attention_share(model, d, 64, G, args.trace_dir)
    res["card_after"] = card()
    s = json.dumps(res, indent=1)
    print(s)
    if args.out:
        with open(args.out, "w") as f:
            f.write(s + "\n")


if __name__ == "__main__":
    main()
