"""Cost of constrained beam search (constraints) against today's beam search, and of its per-frame selection.

    python tools/constrained_beam_bench.py [--out results/constrained_beam_h100.json]

BERT-base bf16 decoder, B = 100 images, 100 regions, max_tgt_length 20 (out_len 122), K = 6 beams per state.  Arms, each Python-driven
and as one GraphedCall replay, alternating inside one loop (tools/nbest_bench.py's compare): today's beam search at K = 6, and
constrained beam search with C = 1, 2 and 3 one-word constraints shared by every image (S*K = 12, 24 and 48 hypotheses per image).
Each figure is the median of REPS calls timed with CUDA events after a warm-up call; peak allocated memory is that of one
Python-driven call.  Also reported: the share of images whose caption meets every constraint (constraints_met).

Per-frame selection at frame 1 (B*S*K rows, V = 28 996), each the median over REPS windows of ITERS back-to-back calls timed with
CUDA events: a torch statement of the rule (log_softmax in fp32 over the head's output, the parent scores added, each (row, word)'s
destination state as an int8 mask, one topk per state over the image's rows) against one vlpk_constrained_beam_step on the head's
decoder output without its bias.  Prints one JSON object, with the card's name, power limit and SM clock queried in the same run."""
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

from tools.diverse_beam_bench import window  # noqa: E402
from tools.nbest_bench import REPS, card, compare, inputs  # noqa: E402
from vlp_b200 import ops, synth  # noqa: E402
from vlp_b200 import vlp_modules as vm  # noqa: E402

K = 6
WORDS = (2100, 3100, 4100)                                         # constraint j: word WORDS[j]


def table(B, C):
    return torch.tensor(WORDS[:C], dtype=torch.int64).view(1, C, 1, 1).expand(B, C, 1, 1).contiguous()


def selection(B, V, C):
    """Per-frame selection time, microseconds, at frame 1 (B*S*K rows)."""
    S = 1 << C
    SK = S * K
    rows = B * SK
    gen = torch.Generator(device="cuda").manual_seed(C)
    logits = torch.randn(rows, 1, V, generator=gen, device="cuda").bfloat16()
    bias = (torch.randn(V, generator=gen, device="cuda") * 0.1).bfloat16()
    scores = logits + bias                                         # the head's output, bias included
    cons = table(B, C).cuda()
    wi, pt = (torch.zeros(2, B, SK, dtype=torch.int64, device="cuda") for _ in range(2))
    sc, eo = (torch.zeros(2, B, SK, device="cuda") for _ in range(2))
    sc[0] = torch.randn(B, SK, generator=gen, device="cuda")
    W = K + C
    tw, tl = torch.empty(rows, W, dtype=torch.int32, device="cuda"), torch.empty(rows, W, device="cuda")
    td = torch.empty(rows, C, dtype=torch.int32, device="cuda")
    hist = [torch.zeros(rows, 2, dtype=torch.int32, device="cuda") for _ in range(2)]
    state = (torch.arange(SK, device="cuda") // K).repeat(B).to(torch.int8)
    words = torch.tensor(WORDS[:C], device="cuda")
    bits = (1 << torch.arange(C, device="cuda")).to(torch.int8)

    def torch_rule():
        logp = F.log_softmax(scores.float(), dim=-1).view(rows, V)
        cand = logp + eo[0].reshape(rows, 1) * -10000.0 + sc[0].reshape(rows, 1)
        dest = state.view(rows, 1).expand(rows, V).clone()
        dest[:, words] |= bits                                     # one-word constraints complete wherever their word is chosen
        out = []
        for s in range(S):
            v = torch.where(dest == s, cand, torch.full_like(cand, -float("inf"))).view(B, SK * V)
            out.append(torch.topk(v, K))
        return out

    arms = {"torch (log_softmax + masks + per-state topk)": torch_rule,
            "constrained_beam_step": lambda: ops.constrained_beam_step(logits, bias, 1, cons, wi, pt, sc, eo, tw, tl, td, 102,
                                                                       hist_in=hist[0], hist_out=hist[1])}
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

    res = {"card (name, power limit, SM clock, max SM clock)": card(), "B": B, "out_len": L, "K": K,
           "constraints": {f"C={C}": [[w] for w in WORDS[:C]] for C in (1, 2, 3)}}
    res["selection_us at frame 1, V = %d" % dims.vocab] = {f"C={C} ({B * (K << C)} rows)": selection(B, dims.vocab, C)
                                                           for C in (1, 2, 3)}
    args = inputs(B, L, R, dims)
    models = {"beam K=6": decoder()}
    for C in (1, 2, 3):
        models[f"constrained C={C}"] = decoder(constraints=[[w] for w in WORDS[:C]])
    res["constraints_met rate"] = {n: round(float(m(*args, task_idx=None)["constraints_met"].float().mean()), 3)
                                   for n, m in models.items() if m.constraints is not None}
    res["decode"] = compare({n: (lambda *x, m=m: m(*x, task_idx=None), args) for n, m in models.items()})
    res["card after (name, power limit, SM clock, max SM clock)"] = card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
