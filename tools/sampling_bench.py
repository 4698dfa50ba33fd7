"""Decode throughput with top-k / top-p sampling at BERT-base size (100 regions + 21 decode steps, V = 28 996).

For each batch size: tokens/s of greedy, top-k (k = 1, 8, 64) and top-p (p = 0.9) decodes, Python-driven with the K/V caches;
the same sampling decodes with the word choice done in torch instead (bias add, sort / top-k, softmax, multinomial, and a read
of the finished count on the host every step, as a loop that stops on [EOS] without the device-side count needs); and the
time of one vlpk_sample_tokens launch against one decode step.  Decode times: CUDA events around whole decodes, 3 after 2 warm-ups,
the arms alternating over 5 rounds; the median of the 15.  Kernel times: CUDA events around 200 back-to-back launches on the decoder's own logits.

    python tools/sampling_bench.py [batch ...]          (default 32 128)
"""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vlp_b200 import ops, synth
from vlp_b200 import vlp_modules as vm

EOS = 102
ROUNDS = 5
MODES = [("greedy", "beam_search", {}), ("topk k=1", "topk", dict(topk=1)), ("topk k=8", "topk", dict(topk=8)),
         ("topk k=64", "topk", dict(topk=64)), ("topp p=0.9", "topp", dict(topp=0.9))]


def torch_sample_tokens(logits, bias, mode, topk, topp, seed, f, seq, score, finished, live, eos_id, pad_id=0, block_eos=False, ngram=0,
                        ignore=None):
    """The word choice in torch (no n-gram blocking), for comparison: same arguments and outputs as ops.sample_tokens."""
    x = (logits.reshape(seq.shape[0], -1) + bias).float()
    if block_eos:
        x[:, eos_id] = -10000.0
    if mode == "topk":
        vals, idx = torch.topk(x, topk, dim=-1)
    else:
        vals, idx = torch.sort(x, dim=-1, descending=True)
        pr = torch.softmax(vals, -1)
        drop = (torch.cumsum(pr, -1) - pr) >= topp
        vals = vals.masked_fill(drop, -float("inf"))
    pick = idx.gather(1, torch.multinomial(torch.softmax(vals, -1), 1))[:, 0]
    done = finished.bool()
    seq[:, f] = torch.where(done, torch.full_like(pick, pad_id), pick)
    score[:, f] = torch.where(done, torch.zeros_like(score[:, f]), torch.log_softmax(x, -1).gather(1, pick[:, None])[:, 0])
    newly = (~done) & (pick == eos_id)
    finished |= newly.int()
    live -= newly.sum().int()
    live.item()                                                       # the host reads the finished count: one round trip per step


def time_decode(model, args, reps=3):
    for _ in range(2):
        model(*args, task_idx=None)
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        model(*args, task_idx=None)
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return ts


def time_kernel(fn, n=200):
    for _ in range(5):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n * 1e3                             # us per launch


def main():
    batches = [int(a) for a in sys.argv[1:]] or [32, 128]
    d = synth.BERT_BASE
    R, Ln = d.regions, d.seq_len
    steps = Ln - R - 2
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(f"GPU: {torch.cuda.get_device_name()} | nvidia-smi: {smi}")
    print(f"BERT-base decoder (12 layers, H = 768, V = {d.vocab}), {R} regions, {steps} decode steps, K/V caches, Python-driven")
    cfg = vm.BertConfig(d.vocab, hidden_size=d.hidden, num_hidden_layers=d.layers, num_attention_heads=d.heads, intermediate_size=d.inter,
                        type_vocab_size=d.type_vocab, max_position_embeddings=d.max_pos)
    torch.manual_seed(0)
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=EOS, enable_butd=True, len_vis_input=R).cuda().bfloat16().eval()
    for B in batches:
        g = torch.Generator().manual_seed(B)
        input_ids = torch.tensor([[101] + [100] * R + [102]] * B).cuda()
        tt = torch.tensor([[4] * (R + 2) + [5] * (Ln - R - 2)] * B).cuda()
        pos = torch.arange(Ln).unsqueeze(0).expand(B, Ln).contiguous().cuda()
        mask = torch.zeros(B, Ln, Ln, dtype=torch.long)
        mask[:, :, :R + 2] = 1
        mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(Ln - R - 2, Ln - R - 2, dtype=torch.long))
        args = (torch.randn(B, R, d.vis_dim, generator=g).clamp_min(0).cuda().bfloat16(), torch.randn(B, R, d.pe_dim, generator=g).cuda().bfloat16(),
                input_ids, tt, pos, mask.cuda())
        print(f"\nbatch {B}")
        runs = {}                                                      # the arms alternate, ROUNDS times: host noise hits them alike
        for _ in range(ROUNDS):
            for name, method, kw in MODES:
                for arm in (("device", "torch") if method != "beam_search" and kw.get("topk") != 1 else ("device",)):
                    model.sampling_method, model.topk, model.topp = method, kw.get("topk", 1), kw.get("topp", 1.0)
                    saved = ops.sample_tokens
                    if arm == "torch":
                        ops.sample_tokens = torch_sample_tokens
                    try:
                        runs.setdefault((name, arm), []).extend(time_decode(model, args))
                    finally:
                        ops.sample_tokens = saved
        times = {k: sorted(v)[len(v) // 2] for k, v in runs.items()}
        for name, method, kw in MODES:
            t = times[(name, "device")]
            line = f"  {name:12s} device {t:8.2f} ms {B * steps / t * 1e3:9.0f} tokens/s"
            if (name, "torch") in times:
                tt = times[(name, "torch")]
                line += f" | torch word choice {tt:8.2f} ms {B * steps / tt * 1e3:9.0f} tokens/s | device / torch time {t / tt:.2f}"
            print(line)
        times["greedy"] = times[("greedy", "device")]
        # one launch against one decode step, on the decoder's logits of this batch
        pred = model.cls.predictions
        with torch.no_grad():
            h = torch.randn(B, 1, d.hidden, generator=g).cuda().bfloat16()
            logits = pred.decoder(pred.transform(h))
        seq = torch.zeros(B, steps, dtype=torch.int64, device="cuda")
        sc = torch.zeros(B, steps, dtype=torch.float32, device="cuda")
        fin = torch.zeros(B, dtype=torch.int32, device="cuda")
        live = torch.full((1,), B, dtype=torch.int32, device="cuda")
        step_ms = times["greedy"] / steps
        for name, method, kw in MODES[1:]:
            us = time_kernel(lambda: ops.sample_tokens(logits, pred.bias, method, kw.get("topk", 1), kw.get("topp", 1.0), 1, 3, seq, sc, fin,
                                                       live, EOS))
            ut = time_kernel(lambda: torch_sample_tokens(logits, pred.bias, method, kw.get("topk", 1), kw.get("topp", 1.0), 1, 3, seq, sc,
                                                         fin, live, EOS), n=50)
            print(f"  {name:12s} vlpk_sample_tokens {us:7.1f} us per step = {us / 1e3 / step_ms * 100:5.2f} % of a greedy decode step "
                  f"({step_ms * 1e3:7.1f} us); torch word choice {ut:7.1f} us")


if __name__ == "__main__":
    main()
