"""Cost of prompted captions (prompt_ids): decodes that continue given caption beginnings against the unprompted decode.

    python tools/prompt_decode_bench.py [--out results/prompt_decode_h100.json]

BERT-base bf16 decoder, B = 32 images, 100 regions, max_tgt_length 20 (out_len 122).  For greedy decode and beam search (K = 5), the arms
Tp = 0 (no prompt), a uniform prompt of Tp = 4 and of Tp = 8 words, and a ragged batch of width 8 (t_b = b mod 9) alternate inside one
loop, each Python-driven and as one GraphedCall replay; each figure is the median of REPS calls timed with CUDA events after a warm-up
call (nbest_bench.compare).  `prefill_ms` is the step-0 prefill alone (DecodeState.step on [CLS] regions [SEP] prompt [MASK] and
the head), timed the same way, and `prefill_share` its share of the Python-driven greedy decode.  Prints one JSON object, with the
card's name, power limit and SM clock queried in the same run."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402

from tools.nbest_bench import REPS, card, compare, inputs, timed  # noqa: E402
from vlp_b200 import synth  # noqa: E402
from vlp_b200 import vlp_modules as vm  # noqa: E402
from vlp_b200.decode import DecodeState  # noqa: E402


def prompts(B, dev):
    """{arm: prompt_ids or None}: none, uniform 4 and 8 words, ragged t_b = b mod 9 at width 8."""
    g = torch.Generator().manual_seed(1)
    words = torch.randint(1000, 20000, (B, 8), generator=g)
    ragged = words.clone()
    for b in range(B):
        ragged[b, b % 9:] = 0
    return {"Tp=0": None, "Tp=4": words[:, :4].to(dev), "Tp=8": words.to(dev), "ragged(Tp=8)": ragged.to(dev)}


def prefill_ms(model, args, prompt):
    """Median time of the step-0 prefill and the head at B images."""
    def call():
        state = DecodeState(model, *model.project_regions(*args[:2]), *args[2:], prompt=prompt)
        model.cls(state.step(state.first_ids), None)
    with torch.no_grad():
        call()
        return round(statistics.median(timed(call) for _ in range(REPS)), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--B", type=int, default=32)
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
    args = inputs(B, L, R, dims)
    arms = prompts(B, args[0].device)
    res = {"card (name, power limit, SM clock, max SM clock)": card(), "B": B, "out_len": L, "frames": {n: L - R - 2 - (0 if p is None else
                                                                                                              p.shape[1])
                                                                                                     for n, p in arms.items()}}
    for mode, K in (("greedy", 1), ("beam5", 5)):
        m = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=R, search_beam_size=K)
        m.load_state_dict(sd, strict=False)
        m = m.cuda().bfloat16().eval()
        res[mode] = compare({n: ((lambda *x, m=m: m(*x[:6], task_idx=None)) if p is None else
                                 (lambda *x, m=m: m(*x[:6], task_idx=None, prompt_ids=x[6])), args if p is None else args + (p,))
                             for n, p in arms.items()})
        if K == 1:
            for n, p in arms.items():
                res[mode][n]["prefill_ms"] = prefill_ms(m, args, p)
                res[mode][n]["prefill_share"] = round(res[mode][n]["prefill_ms"] / res[mode][n]["python_ms"], 3)
        del m
        torch.cuda.empty_cache()
    res["card after"] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
