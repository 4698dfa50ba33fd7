"""Cost of several captions per image over one K/V cache of the image prefix (num_return_sequences N > 1) against today's decodes.

    python tools/nbest_bench.py [--out results/nbest_h100.json]

BERT-base bf16 decoder, B = 100 images, 100 regions, max_tgt_length 20 (out_len 122).  Arms, each Python-driven and as one GraphedCall
replay:
  beam K (K = 3, 5): today's K-beam (N = 1: per-hypothesis caches, expanded after step 0 and index_selected every frame) against the
                     N = K beam on the shared prefix cache, whose pred_seq is bitwise the same (checked here);
  top-k sampling:    N = 5 samples per image against today's sampler on the batch repeated 5 times (same draws, checked here).
The arms of a pair alternate inside one loop; each figure is the median of REPS calls timed with CUDA events after a warm-up call.
Peak allocated memory is that of one Python-driven call.  Prints one JSON object, with the card's name, power limit and SM clock
queried in the same run."""
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

from vlp_b200 import graph, synth  # noqa: E402
from vlp_b200 import vlp_modules as vm  # noqa: E402

REPS = 7


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip()


def inputs(B, L, R, dims, rep=1):
    g = torch.Generator().manual_seed(0)
    ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    args = (torch.randn(B, R, dims.vis_dim, generator=g).clamp_min(0).bfloat16(), torch.randn(B, R, dims.pe_dim, generator=g).bfloat16(),
            ids, tt, pos, mask)
    return tuple(a.repeat_interleave(rep, 0).cuda() for a in args)


def timed(call):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def peak_mb(call):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    call()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)


def compare(arms):
    """arms: {name: (fn, args)} -> {name: {python ms, graph ms, peak MB}}, arms alternating inside each repetition."""
    out = {n: {"peak_MB": peak_mb(lambda f=f, a=a: f(*a))} for n, (f, a) in arms.items()}
    for how in ("python", "graph"):
        calls = {}
        for n, (f, a) in arms.items():
            calls[n] = (lambda f=f, a=a: f(*a)) if how == "python" else (lambda g=graph.GraphedCall(f, a), a=a: g(*a))
            calls[n]()                                         # warm-up (and capture)
        ts = {n: [] for n in arms}
        for _ in range(REPS):
            for n, c in calls.items():
                ts[n].append(timed(c))
        for n in arms:
            out[n][f"{how}_ms"] = round(statistics.median(ts[n]), 2)
        del calls
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--B", type=int, default=100)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    d = synth.BERT_BASE
    R, B = d.regions, a.B
    L = R + 2 + 20
    dims = synth.VlpDims(vocab=d.vocab, hidden=d.hidden, layers=d.layers, heads=d.heads, inter=d.inter, regions=R, text=L - R)
    cfg = vm.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                        intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    sd = synth.make_state_dict(dims, 0)

    def decoder(**kw):
        m = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=R, **kw)
        m.load_state_dict(sd, strict=False)
        return m.cuda().bfloat16().eval()

    res = {"card (name, power limit, SM clock, max SM clock)": card(), "B": B, "out_len": L}
    args = inputs(B, L, R, dims)
    for K in (3, 5):
        one, grp = decoder(search_beam_size=K), decoder(search_beam_size=K, num_return_sequences=K)
        assert torch.equal(one(*args, task_idx=None)["pred_seq"], grp(*args, task_idx=None)["pred_seq"])
        res[f"beam{K}"] = compare({"N=1": (lambda *x, m=one: m(*x, task_idx=None), args),
                                   f"N={K}": (lambda *x, m=grp: m(*x, task_idx=None), args)})
        del one, grp
        torch.cuda.empty_cache()
    N = 5
    rep = inputs(B, L, R, dims, rep=N)
    one, grp = decoder(sampling_method="topk", topk=8, seed=1), decoder(sampling_method="topk", topk=8, seed=1, num_return_sequences=N)
    assert torch.equal(one(*rep, task_idx=None)[0], grp(*args, task_idx=None)[0].reshape(B * N, -1))
    res["topk8 x5"] = compare({"repeated batch": (lambda *x, m=one: m(*x, task_idx=None), rep),
                               f"N={N}": (lambda *x, m=grp: m(*x, task_idx=None), args)})
    res["card after (name, power limit, SM clock, max SM clock)"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
