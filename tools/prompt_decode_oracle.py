"""ORACLE SUPPORT for prompted captions (BertForSeq2SeqDecoder.forward's prompt_ids).  Test infrastructure, not product code: only tests/
import it.

The reference has no prompt, but for a prompt of the same length t for every image its own decode gives the answer: the prompt appended
to input_ids ([CLS] regions [SEP] prompt), with token_type_ids, position_ids and the attention mask unchanged (they already cover every
position up to out_len), runs the prompt through the first step's prefill and generates out_len - in_len - t words.  A prompted decode
with n-gram blocking off and min_len 0 returns the prompt followed by exactly those words.

* CASES / case_inputs(): the seeded cases, regenerated from vlp_b200/synth.py (inputs laid out as oracle/make_golden.run_decode does).
* `python -O tools/prompt_decode_oracle.py` runs the UNMODIFIED reference's BertForSeq2SeqDecoder.forward / beam_search (imported
  through oracle/ref_shim.py, checkout at $VLP_REFERENCE_ROOT) on the CPU and writes tests/golden/prompt_decode.pt.  Per case: the
  prompt [B, t], and for greedy decode the reference's ids / scores of the generated words and every frame's top-1 minus top-2 logit
  margin (`gaps`); for beam search its traces (pred_seq, scores, wids, ptrs) and the K + 1 best candidate scores of every frame's
  selection (`cand_scores`).  Beam search runs with torch.div patched to floor semantics for integer operands (:1317, as in
  oracle/make_golden.run_decode_beam), restored afterwards.
"""
import os
import subprocess
import sys

if __debug__ and __name__ == "__main__":
    sys.exit(subprocess.call([sys.executable, "-O"] + sys.argv))

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import torch  # noqa: E402

from vlp_b200 import synth  # noqa: E402

MASK_ID, EOS_ID = 103, 102
K = 3
LENGTH_PENALTY = 0.5
RELAX_TASKS = (3, 0)            # per-sample task ids of the relaxed case (s2s, bidirectional)
# 2-layer decoder at BERT-base width and vocabulary
WIDE = synth.VlpDims(vocab=28996, hidden=768, layers=2, heads=12, inter=3072, regions=100, text=20)
# name: (dims, mode "greedy" / "beam", batch, prompt length t, input seed, relaxed head)
CASES = {
    "greedy_h128": (synth.SMALL_L123, "greedy", 2, 3, 77, False),
    "beam_h128": (synth.SMALL_L123, "beam", 2, 3, 78, False),
    "greedy_h768": (WIDE, "greedy", 2, 4, 81, False),
    "beam_h768": (WIDE, "beam", 2, 2, 82, False),
    "greedy_relax4": (synth.SMALL_L123, "greedy", 2, 2, 79, True),
}


def decode_inputs(dims, B, seed):
    """(vis, vis_pe, input_ids, token_type_ids, position_ids, mask), fp32 / int64 on the CPU, as decode_img2txt.py builds them."""
    R, L = dims.regions, dims.seq_len
    g = torch.Generator().manual_seed(seed)
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    vis = torch.randn(B, R, dims.vis_dim, generator=g).clamp_min(0)
    pe = torch.randn(B, R, dims.pe_dim, generator=g)
    return vis, pe, input_ids, tt, pos, mask


def prompt_words(dims, B, t, seed):
    """A seeded prompt [B, t] of word ids in [200, vocab): no padding, [EOS], [MASK] or the input's special ids."""
    g = torch.Generator().manual_seed(seed + 1000)
    return torch.randint(200, dims.vocab, (B, t), generator=g, dtype=torch.int64)


def case_inputs(name):
    """(dims, state dict, decoder inputs, prompt, task_idx) of CASES[name]."""
    dims, _, B, t, seed, relaxed = CASES[name]
    sd = synth.make_state_dict(dims, seed=0)
    task_idx = None
    if relaxed:
        from tools import relax_projection_oracle as rpo
        sd = rpo.relaxed_state_dict(sd, dims.hidden, rpo.RELAX)
        task_idx = torch.tensor(RELAX_TASKS)
    return dims, sd, decode_inputs(dims, B, seed), prompt_words(dims, B, t, seed), task_idx


def _reference(name, **kw):
    from oracle import ref_shim
    dims, sd, _, _, _ = case_inputs(name)
    if CASES[name][5]:
        from tools import relax_projection_oracle as rpo
        return rpo.build_reference(dims, sd, rpo.RELAX, decoder=True, mask_word_id=MASK_ID, eos_id=EOS_ID, enable_butd=True,
                                   len_vis_input=dims.regions, **kw).eval()
    return ref_shim.build_reference_model(dims, sd, decoder=True, mask_word_id=MASK_ID, eos_id=EOS_ID, **kw).eval()


def run_case(name):
    dims, mode, B, t, seed, relaxed = CASES[name]
    _, _, args, prompt, task_idx = case_inputs(name)
    vis, pe, input_ids, tt, pos, mask = args
    ref_args = (vis, pe, torch.cat((input_ids, prompt), dim=1), tt, pos, mask)
    out = {"mode": mode, "B": B, "t": t, "seed": seed, "relaxed": relaxed, "prompt": prompt, "hidden": dims.hidden, "vocab": dims.vocab}
    if mode == "greedy":
        model = _reference(name, search_beam_size=1)
        gaps = []

        def hook(m, i, o):
            top2 = torch.topk(o.detach(), 2, dim=-1).values
            gaps.append(top2[..., 0] - top2[..., 1])
        h = model.cls.predictions.register_forward_hook(hook)
        try:
            with torch.no_grad():
                ids, scores = model(*ref_args, task_idx=task_idx, sample_mode="greedy")
        finally:
            h.remove()
        out.update(ids=ids.clone(), scores=scores.clone(), gaps=torch.cat(gaps, dim=1))
        print(f"{name}: prompt {prompt[0].tolist()} ids {ids[0].tolist()}")
        return out
    model = _reference(name, search_beam_size=K, length_penalty=LENGTH_PENALTY)
    orig_div, orig_topk = torch.div, torch.topk
    cands, frames = [], dims.seq_len - dims.regions - 2 - t

    def floor_div(a, b, *rest, **kw):
        if not rest and not kw and torch.is_tensor(a) and not a.is_floating_point():
            return orig_div(a, b, rounding_mode="floor")
        return orig_div(a, b, *rest, **kw)

    def topk(x, k, *a, **kw):              # :1304 on [B, 1, V] scores at frame 0; :1316 on [B, K*K] after
        if (not cands and x.dim() == 3) or x.dim() == 2:
            cands.append(orig_topk(x.reshape(B, -1), K + 1).values)
        return orig_topk(x, k, *a, **kw)

    torch.div, torch.topk = floor_div, topk
    try:
        with torch.no_grad():
            traces = model(*ref_args, task_idx=task_idx)
    finally:
        torch.div, torch.topk = orig_div, orig_topk
    if len(cands) != frames:                # explicit raise: this module runs under `python -O`
        raise RuntimeError(f"case {name}: {len(cands)} beam selections recorded for {frames} frames")
    out.update(K=K, length_penalty=LENGTH_PENALTY, cand_scores=torch.stack(cands, dim=1).clone(),
               **{k: v.clone() for k, v in traces.items()})
    print(f"{name}: prompt {prompt[0].tolist()} pred_seq {traces['pred_seq'][0].tolist()}")
    return out


if __name__ == "__main__":
    torch.set_num_threads(8)
    out = {"case": "prompt_decode", "cases": {n: run_case(n) for n in CASES}, "torch": str(torch.__version__)}
    path = os.path.join(ROOT, "tests", "golden", "prompt_decode.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes")
