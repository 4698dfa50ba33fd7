"""ORACLE SUPPORT for scoring given captions (BertForSeq2SeqDecoder.score_captions).  Test infrastructure, not product code: only
tests/ import it.

`python -O tools/caption_score_oracle.py` runs the UNMODIFIED reference (imported through oracle/ref_shim.py, checkout at
$VLP_REFERENCE_ROOT) on the CPU.  It drives the reference's BertModelIncr and cls frame by frame exactly as its
BertForSeq2SeqDecoder.forward does (modeling.py:1189-1252), but feeds the given word c_t instead of the arg-max and records
log_softmax(prediction_scores)[c_t] of every frame.  It writes tests/golden/caption_score.pt, per case:
  `captions` int64 [B, T] or [B, N, T] (0-padded after [EOS]), `task_idx`, `logp` fp32 shaped like captions (0 at and after the first
  0), and `drift`: |logp of a second run with the model and inputs in bfloat16 - logp|, per word — the reference's own fp32 -> bf16
  drift.
Cases: "l123" (L = 123, seq2seq mask, B = 3, ragged captions with [EOS] and 0-padding), "l123_relax4" (the same with
relax_projection 4 and per-sample task ids), "l143" (out_len 143, T = 41: the tiled kernels) and "two_per_image" (B = 2 images, N = 2
captions each).
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
import torch.nn.functional as F  # noqa: E402

from tools import relax_projection_oracle as rpo  # noqa: E402
from vlp_b200 import synth  # noqa: E402

MASK_ID, EOS_ID = 103, 102
RELAX = 4
# name: (out_len, images B, captions per image N (None: [B, T]), caption lengths (None: no [EOS], full T), T, relax tasks, seed)
CASES = {
    "l123": (123, 3, None, (20, 12, 5), 20, None, 2101),
    "l123_relax4": (123, 3, None, (20, 9, 14), 20, (3, 0, 3), 2102),
    "l143": (143, 2, None, (None, 23), 41, None, 2103),
    "two_per_image": (123, 2, 2, (17, 6, 21, 10), 21, None, 2104),
}


def dims_for(out_len):
    return synth.SMALL_L123 if out_len == 123 else synth.VlpDims(vocab=1000, hidden=128, layers=2, heads=2, inter=512, regions=100,
                                                                  text=out_len - 103)


def captions(name):
    """int64 captions of a case: words in [200, 1000), [EOS] closing each caption of the given length (a length None has no [EOS]
    and fills all T words), 0 after it."""
    out_len, B, N, lens, T, _, seed = CASES[name]
    g = torch.Generator().manual_seed(seed)
    c = torch.randint(200, 1000, (len(lens), T), generator=g)
    for i, n in enumerate(lens):
        if n is not None:
            c[i, n - 1] = EOS_ID
            c[i, n:] = 0
    return c if N is None else c.view(B, N, T)


def inputs(name):
    """(dims, state dict, decoder args, captions, task_idx) of a case."""
    out_len, B, N, lens, T, tasks, seed = CASES[name]
    dims = dims_for(out_len)
    sd = synth.make_state_dict(dims, seed=0)
    if tasks is not None:
        sd = rpo.relaxed_state_dict(sd, dims.hidden, RELAX)
    return dims, sd, rpo.decode_inputs(dims, B, seed), captions(name), None if tasks is None else torch.tensor(tasks)


def forced_decode(model, args, caps, task_idx):
    """The reference decode loop (modeling.py:1189-1252) fed the caption's words: [rows, T] log_softmax at c_t of every frame."""
    vis_feats, vis_pe, input_ids, token_type_ids, position_ids, attention_mask = args
    vis_feats = model.vis_embed(vis_feats)
    vis_pe = model.vis_pe_embed(vis_pe)
    T = caps.shape[1]
    prev_embedding = prev_encoded_layers = None
    curr_ids = input_ids
    mask_ids = input_ids[:, :1] * 0 + model.mask_word_id
    next_pos = input_ids.shape[1]
    out = []
    for t in range(T):
        start_pos = next_pos - curr_ids.shape[1]
        new_embedding, new_encoded_layers, _ = model.bert(
            vis_feats, vis_pe, torch.cat((curr_ids, mask_ids), dim=1), token_type_ids[:, start_pos:next_pos + 1],
            position_ids[:, start_pos:next_pos + 1], attention_mask[:, start_pos:next_pos + 1, :next_pos + 1], prev_embedding=prev_embedding,
            prev_encoded_layers=prev_encoded_layers, output_all_encoded_layers=True, len_vis_input=model.len_vis_input)
        prediction_scores, _ = model.cls(new_encoded_layers[-1][:, -1:, :], None, task_idx=task_idx)
        out.append(F.log_softmax(prediction_scores[:, 0].float(), dim=-1).gather(1, caps[:, t:t + 1]))
        if prev_embedding is None:
            prev_embedding = new_embedding[:, :-1, :]
            prev_encoded_layers = [x[:, :-1, :] for x in new_encoded_layers]
        else:
            prev_embedding = torch.cat((prev_embedding, new_embedding[:, :-1, :]), dim=1)
            prev_encoded_layers = [torch.cat((a, b[:, :-1, :]), dim=1) for a, b in zip(prev_encoded_layers, new_encoded_layers)]
        curr_ids = caps[:, t:t + 1]
        next_pos += 1
    logp = torch.cat(out, dim=1)
    return torch.where((caps != 0).cumprod(1).bool(), logp, torch.zeros_like(logp))


def run(name, dtype=torch.float32):
    dims, sd, args, caps, task_idx = inputs(name)
    N = CASES[name][2]
    B, T = caps.shape[0], caps.shape[-1]
    if N is not None:                       # N captions per image: the image inputs repeated per caption
        args = tuple(a.repeat_interleave(N, 0) for a in args)
        task_idx = None if task_idx is None else task_idx.repeat_interleave(N)
    model = rpo.build_reference(dims, sd, RELAX if task_idx is not None else 0, decoder=True, mask_word_id=MASK_ID, eos_id=EOS_ID,
                                enable_butd=True, len_vis_input=dims.regions, search_beam_size=1).eval()
    if dtype != torch.float32:
        model = model.to(dtype)
        args = tuple(a.to(dtype) if a.is_floating_point() else a for a in args)
    with torch.no_grad():
        logp = forced_decode(model, args, caps.reshape(-1, T), task_idx)
    return logp.view(caps.shape)


def case(name):
    logp = run(name)
    drift = (run(name, torch.bfloat16) - logp).abs()
    _, _, _, caps, task_idx = inputs(name)
    print(f"{name}: captions {tuple(caps.shape)} logp sum {float(logp.sum()):.4f} max drift {float(drift.max()):.3e}")
    return {"out_len": CASES[name][0], "seed": CASES[name][6], "captions": caps, "task_idx": task_idx, "logp": logp, "drift": drift}


if __name__ == "__main__":
    torch.set_num_threads(8)
    out = {"case": "caption_score", "mask_id": MASK_ID, "eos_id": EOS_ID, "relax_projection": RELAX,
           "cases": {n: case(n) for n in CASES}, "torch": str(torch.__version__), "reference_commit": "74c4d85"}
    path = os.path.join(ROOT, "tests", "golden", "caption_score.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes")
