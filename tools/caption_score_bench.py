"""Cost of scoring given captions (BertForSeq2SeqDecoder.score_captions) against the two other ways to get the same numbers.

    python tools/caption_score_bench.py [--out results/caption_score_h100.json]

BERT-base bf16 decoder, B = 100 images x 5 captions of T = 20 words, 100 regions, out_len 122 (in_len 102).  Arms:
  score:        score_captions, one teacher-forced pass of S + T = 141 rows per caption (vlpk_encoder_score_fwd);
  plain:        the same layout as one plain sequence of S + T rows with a materialised [S + T, S + T] mask through vlpk_encoder_fwd
                (the KV-tiled kernels, since 141 > 128) — forced_decode's and this arm's helpers are the test references too;
  frame loop:   the decode's own step (DecodeState with per-caption K/V caches), T frames with forced ids.
Each arm runs Python-driven and as one GraphedCall replay; the arms alternate inside each repetition, each figure is the median of
REPS calls timed with CUDA events after a warm-up call.  Prints one JSON object, with the card's name, power limit and SM clock
queried in the same run, and the largest |difference| of each arm's log-probabilities from the score arm's."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from vlp_b200 import score  # noqa: E402
from vlp_b200.decode import DecodeState  # noqa: E402


def forced_decode(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caps, task_idx=None):
    """The decode's step (DecodeState, per-caption K/V caches) fed caps [rows, T] frame by frame: [rows, T] log_softmax at c_t of every
    frame's [MASK] row, 0 at and after the first 0.  The image inputs have one row per caption."""
    T = caps.shape[1]
    with torch.no_grad():
        v, pe = dec.project_regions(vis_feats, vis_pe)
        state = DecodeState(dec, v, pe, input_ids, token_type_ids, position_ids, attention_mask)
        curr, out = input_ids, []
        for t in range(T):
            scores, _ = dec.cls(state.step(curr), None, task_idx=task_idx)
            out.append(F.log_softmax(scores[:, 0].float(), -1).gather(1, caps[:, t:t + 1]))
            curr = caps[:, t:t + 1]
        logp = torch.cat(out, 1)
    return torch.where((caps != 0).cumprod(1).bool(), logp, 0.0)


def plain_arm(dec, vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask, caps, task_idx=None):
    """The scoring layout as one plain sequence of S + T rows: a materialised mask (shared rows as score_captions sees them, query row t
    over the shared columns before its position and over itself) through BertEncoder (vlpk_encoder_fwd), then the same head."""
    rows, T = caps.shape
    in_len = input_ids.shape[1]
    dev = input_ids.device
    S, positions, shared_keep, query_keep = score.layout(in_len, T, dev)
    m = attention_mask
    full = torch.zeros(rows, S + T, S + T, dtype=m.dtype, device=dev)
    full[:, :S, :S] = m[:, :S, :S] * shared_keep.to(m.dtype)
    full[:, S:, :S] = m[:, in_len:in_len + T, :S] * query_keep.to(m.dtype)
    full[:, S:, S:] = torch.eye(T, dtype=m.dtype, device=dev)
    with torch.no_grad():
        v, pe = dec.project_regions(vis_feats, vis_pe)
        ids = torch.cat((input_ids, caps[:, :T - 1], caps * 0 + dec.mask_word_id), dim=1)
        emb = dec.bert.embeddings(v, pe, ids, token_type_ids.index_select(1, positions), position_ids.index_select(1, positions),
                                  len_vis_input=dec.len_vis_input)
        ext = dec.bert.get_extended_attention_mask(ids, None, full)
        h = dec.bert.encoder(emb, ext, output_all_encoded_layers=False)[-1][:, S:]
        return score.head_logp(dec, h, caps, task_idx)


def main():
    from tools import nbest_bench as nb
    from vlp_b200 import graph, synth
    from vlp_b200 import vlp_modules as vm
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--B", type=int, default=100)
    ap.add_argument("--N", type=int, default=5)
    ap.add_argument("--T", type=int, default=20)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    d = synth.BERT_BASE
    R, B, N, T = d.regions, a.B, a.N, a.T
    L = R + 2 + 20
    dims = synth.VlpDims(vocab=d.vocab, hidden=d.hidden, layers=d.layers, heads=d.heads, inter=d.inter, regions=R, text=L - R)
    cfg = vm.BertConfig(dims.vocab, hidden_size=dims.hidden, num_hidden_layers=dims.layers, num_attention_heads=dims.heads,
                        intermediate_size=dims.inter, type_vocab_size=dims.type_vocab, max_position_embeddings=dims.max_pos,
                        hidden_dropout_prob=0.0, attention_probs_dropout_prob=0.0)
    dec = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=102, enable_butd=True, len_vis_input=R)
    dec.load_state_dict(synth.make_state_dict(dims, 0), strict=False)
    dec = dec.cuda().bfloat16().eval()
    args = nb.inputs(B, L, R, dims)
    g = torch.Generator().manual_seed(5)
    caps = torch.randint(1000, dims.vocab, (B, N, T), generator=g).cuda()
    rep = tuple(x.repeat_interleave(N, 0) for x in args)
    flat = caps.view(B * N, T)
    res = {"card (name, power limit, SM clock, max SM clock)": nb.card(), "images": B, "captions per image": N, "T": T, "out_len": L}
    with torch.no_grad():
        ref = dec.score_captions(*args, caps).view(B * N, T)
        res["max |logp - score| (plain, frame loop)"] = [float((plain_arm(dec, *rep, flat) - ref).abs().max()),
                                                         float((forced_decode(dec, *rep, flat) - ref).abs().max())]
        res["mean logp per word (score)"] = float(ref.mean())
    arms = {"score": (lambda *x: dec.score_captions(*x[:-1], x[-1]), args + (caps,)),
            "plain": (lambda *x: plain_arm(dec, *x), rep + (flat,)),
            "frame loop": (lambda *x: forced_decode(dec, *x), rep + (flat,))}
    with torch.no_grad():
        res["arms"] = nb.compare(arms)
    res["card after (name, power limit, SM clock, max SM clock)"] = nb.card()
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
