"""Cost of the caption matrix (BertForSeq2SeqDecoder.score_caption_matrix) against score_captions on the repeated batch.

    python tools/caption_matrix_bench.py [--out results/caption_matrix_h100.json]

BERT-base bf16 decoder, B = 100 images, 100 regions (in_len 102), out_len in_len + T + 2 (112 and 124), C shared
captions for C in {5, 100, 1000} and T in {8, 20}.  Arms:
  matrix:    score_caption_matrix, the prefix once per image, 2T - 1 rows per (image, caption) pair;
  repeated:  score_captions on the batch repeated per caption (in_len + 2T - 1 rows per pair), in chunks of the same captions per
             call as the matrix's chunks, so that both arms run the head over the same rows per call.
Each arm runs Python-driven and as one GraphedCall replay; the arms alternate inside each repetition, each figure is the median of
REPS calls timed with CUDA events after a warm-up call, with the peak allocated memory of one call.  Prints one JSON object, with the
card's name, power limit and SM clock queried before and after in the same run, and the largest |difference| of the two arms'
log-probabilities."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402

from vlp_b200 import score  # noqa: E402


def repeated_arm(dec, args, caps, max_rows):
    """[B, C, T]: score_captions on the image inputs repeated per caption, chunk by chunk as score_caption_matrix chunks."""
    B, (C, T) = args[2].shape[0], caps.shape
    G = min(C, max_rows // (B * T))
    out = torch.empty(B, C, T, device=caps.device, dtype=torch.float32)
    rep = tuple(a.repeat_interleave(G, 0) for a in args)
    for c0 in range(0, C, G):
        g = min(G, C - c0)
        a = rep if g == G else tuple(x.repeat_interleave(g, 0) for x in args)
        out[:, c0:c0 + g] = dec.score_captions(*a, caps[c0:c0 + g].unsqueeze(0).expand(B, g, T).reshape(B * g, T)).view(B, g, T)
    return out


def main():
    from tools import nbest_bench as nb
    from vlp_b200 import synth
    from vlp_b200 import vlp_modules as vm
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--B", type=int, default=100)
    ap.add_argument("--C", type=int, nargs="+", default=[5, 100, 1000])
    ap.add_argument("--T", type=int, nargs="+", default=[8, 20])
    a = ap.parse_args()
    torch.cuda.set_device(0)
    d = synth.BERT_BASE
    R, B = d.regions, a.B
    res = {"card before (name, power limit, SM clock, max SM clock)": nb.card(), "images": B, "max_rows": score.MATRIX_MAX_ROWS,
           "cases": []}
    for T in a.T:
        L = R + 2 + T + 2
        dims = synth.VlpDims(vocab=d.vocab, hidden=d.hidden, layers=d.layers, heads=d.heads, inter=d.inter, regions=R, text=L - R)
        cfg = vm.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                            intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                            hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
        dec = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=R)
        dec.load_state_dict(synth.make_state_dict(dims, 0), strict=False)
        dec = dec.cuda().bfloat16().eval()
        args = nb.inputs(B, L, R, dims)
        for C in a.C:
            g = torch.Generator().manual_seed(C * 100 + T)
            caps = torch.randint(1000, dims.vocab, (C, T), generator=g).cuda()
            mr = score.MATRIX_MAX_ROWS
            case = {"C": C, "T": T, "out_len": L, "captions per chunk": min(C, mr // (B * T)),
                    "encoder rows per pair (matrix, repeated)": [2 * T - 1 + (R + 2) / C, R + 2 + 2 * T - 1]}
            with torch.no_grad():
                m = dec.score_caption_matrix(*args, caps)
                r = repeated_arm(dec, args, caps, mr)
                case["max |logp matrix - repeated|"] = float((m - r).abs().max())
                del m, r
            arms = {"matrix": (lambda *x: dec.score_caption_matrix(*x[:-1], x[-1]), args + (caps,)),
                    "repeated": (lambda *x: repeated_arm(dec, x[:-1], x[-1], mr), args + (caps,))}
            with torch.no_grad():
                case["arms"] = nb.compare(arms)
            res["cases"].append(case)
            print(json.dumps(case), flush=True)
            torch.cuda.empty_cache()
        del dec
    res["card after (name, power limit, SM clock, max SM clock)"] = nb.card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
