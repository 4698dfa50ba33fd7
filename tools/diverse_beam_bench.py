"""Cost of diverse beam search (num_beam_groups G > 1) against today's beam search, and of its per-frame selection.

    python tools/diverse_beam_bench.py [--out results/diverse_beam_h100.json]

BERT-base bf16 decoder, B = 100 images, 100 regions, max_tgt_length 20 (out_len 122).  Arms, each Python-driven and as one GraphedCall
replay, alternating inside one loop (tools/nbest_bench.py's compare): today's beam search at K = 6, and diverse beam search at K = 6
with G = 2, 3 and 6 (lambda = 0.5).  Each figure is the median of REPS calls timed with CUDA events after a warm-up call; peak
allocated memory is that of one Python-driven call.  Also printed: the mean number of distinct group_seq captions per image.

Per-frame selection at B*K = 600 rows and V = 28 996, each the median over REPS windows of ITERS back-to-back calls timed with CUDA
events: today's log_softmax in fp32 over the head's output + topk(K) + the finished/total add + topk over K*K, against one
vlpk_diverse_beam_step on the head's decoder output without its bias.  Prints one JSON object, with the card's name, power limit
and SM clock queried in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from tools.nbest_bench import card, compare, inputs  # noqa: E402
from vlp_b200 import ops, synth  # noqa: E402
from vlp_b200 import vlp_modules as vm  # noqa: E402

REPS, ITERS = 7, 50
K, LAM = 6, 0.5


def window(fn):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ITERS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / ITERS


def selection(B, V):
    """Per-frame selection time, microseconds, at frame 1 (B*K rows)."""
    gen = torch.Generator(device="cuda").manual_seed(0)
    rows = B * K
    logits = torch.randn(rows, 1, V, generator=gen, device="cuda").bfloat16()
    bias = (torch.randn(V, generator=gen, device="cuda") * 0.1).bfloat16()
    scores = logits + bias                                        # today's head output, bias included
    total = torch.randn(B, K, device="cuda")
    eos = torch.zeros(B, K, device="cuda")

    def today():
        logp = F.log_softmax(scores.float(), dim=-1)
        kk_scores, kk_ids = torch.topk(logp, k=K)
        kk_scores = kk_scores + eos.reshape(rows, 1, 1) * -10000.0 + total.reshape(rows, 1, 1)
        k_scores, flat = torch.topk(kk_scores.reshape(B, K * K), k=K)
        return torch.gather(kk_ids.reshape(B, K * K), 1, flat)

    wi, pt = (torch.zeros(2, B, K, dtype=torch.int64, device="cuda") for _ in range(2))
    sc, eo = (torch.zeros(2, B, K, device="cuda") for _ in range(2))
    tw, tl = torch.empty(rows, K, dtype=torch.int32, device="cuda"), torch.empty(rows, K, device="cuda")
    arms = {"today (log_softmax + 2 topk)": today}
    for G in (2, 3, 6):
        arms[f"diverse_beam_step G={G}"] = lambda G=G: ops.diverse_beam_step(logits, bias, 1, G, LAM, wi, pt, sc, eo, tw, tl, 102)
    for fn in arms.values():
        fn()
    ts = {n: [] for n in arms}
    for _ in range(REPS):
        for n, fn in arms.items():
            ts[n].append(window(fn))
    return {n: round(statistics.median(t), 1) for n, t in ts.items()}


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
        m = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=R, search_beam_size=K, **kw)
        m.load_state_dict(sd, strict=False)
        return m.cuda().bfloat16().eval()

    res = {"card (name, power limit, SM clock, max SM clock)": card(), "B": B, "out_len": L, "K": K, "diversity_penalty": LAM,
           "selection_us at B*K = %d rows, V = %d" % (B * K, dims.vocab): selection(B, dims.vocab)}
    args = inputs(B, L, R, dims)
    models = {"beam K=6": decoder()}
    for G in (2, 3, 6):
        models[f"diverse G={G}"] = decoder(num_beam_groups=G, diversity_penalty=LAM)
    distinct = {}
    for n, m in models.items():
        if m.num_beam_groups > 1:
            gs = m(*args, task_idx=None)["group_seq"]
            distinct[n] = round(sum(len({tuple(r.tolist()) for r in gs[b]}) for b in range(B)) / B, 2)
    res["distinct group_seq captions per image (mean)"] = distinct
    res["decode"] = compare({n: (lambda *x, m=m: m(*x, task_idx=None), args) for n, m in models.items()})
    res["card after (name, power limit, SM clock, max SM clock)"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
