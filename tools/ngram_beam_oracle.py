"""ORACLE SUPPORT for duplicate-n-gram blocking in beam search (decode_img2txt.py --forbid_duplicate_ngrams, --forbid_ignore_word,
--ngram_size, --min_len; modeling.py:1256-1494).  Test infrastructure, not product code: only tests/ import it.

* CASES / case_inputs(): the seeded decode cases, regenerated from vlp_b200/synth.py (the L = 123 inputs are laid out as
  oracle/make_golden.run_decode_beam does, with the weights of synth seed WEIGHTS_SEED; case "e" uses
  tools/long_seq_oracle.decode_inputs at max_tgt_length 40, L = 143).
* `python -O tools/ngram_beam_oracle.py` runs the UNMODIFIED reference's beam_search (imported through oracle/ref_shim.py, checkout at
  $VLP_REFERENCE_ROOT) on the CPU and writes tests/golden/ngram_beam.pt.  Two torch-2 breakages are patched for the run only and
  restored afterwards: torch.div with integer operands gets floor semantics (:1317, as in make_golden.run_decode_beam), and
  Tensor.cuda is the identity (:1426, the forbidden-word mask is moved to the GPU).  Per case it stores the settings, the traces
  (pred_seq, scores, wids, ptrs), the K + 1 best candidate scores of every frame's selection (`cand_scores`) and `blocked`: every (frame, hypothesis row, word) the reference's forbidden-word mask marked,
  read from the mask itself; the frame is the one whose log-probabilities the mask is added to.  `blocked_pairs` counts the
  (frame, hypothesis) pairs with a non-empty candidate set; the tool refuses a case in which it is 0.
  Case "b"'s ignore set is the word the same inputs' UNBLOCKED reference beam search chooses most often (smallest id on a tie).
  Case "c" (min_len = 5) raises the decoder bias of [EOS] by EOS_BIAS, so that without min_len the beams take [EOS] within the first
  five frames; the tool refuses it unless its traces differ from the same run with min_len = 0, and stores that run too
  ("no_min_len"), so the [EOS] fill is shown to decide words.
"""
import collections
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

SEED = 78                 # oracle/make_golden.run_decode_beam's inputs
LONG_SEED = 145
# synth.make_state_dict seeds.  Seed 0 at L = 123 decodes 21 frames without a repeated trigram (nothing to block), seed 2 repeats.
WEIGHTS_SEED = 2
LONG_WEIGHTS_SEED = 0
K = 3
LENGTH_PENALTY = 0.5
EOS_ID = 102
EOS_BIAS = 1.0
# name: (long sequence, batch, ngram_size, min_len, ignore = "most frequent unblocked word" or None, added [EOS] decoder bias)
CASES = {
    "a": (False, 2, 3, 0, None, 0.0),
    "b": (False, 2, 2, 0, "most_frequent", 0.0),
    "c": (False, 2, 3, 5, None, EOS_BIAS),
    "d": (False, 2, 1, 0, None, 0.0),
    "e": (True, 2, 3, 0, None, 0.0),
}


def case_inputs(name):
    """(dims, state dict, (vis, vis_pe, input_ids, token_type_ids, position_ids, mask)) of CASES[name], fp32 on the CPU."""
    long_seq, B = CASES[name][:2]
    eos_bias = CASES[name][5]
    if long_seq:
        from tools import long_seq_oracle as lso
        dims, _, args = lso.decode_inputs(B, LONG_SEED)
        return dims, _with_eos_bias(synth.make_state_dict(dims, seed=LONG_WEIGHTS_SEED), eos_bias), args
    dims = synth.SMALL_L123
    R, L = dims.regions, dims.seq_len
    g = torch.Generator().manual_seed(SEED)
    input_ids = torch.tensor([[101] + [100] * R + [102]] * B)
    tt = torch.tensor([[4] * (R + 2) + [5] * (L - R - 2)] * B)
    pos = torch.arange(L).unsqueeze(0).expand(B, L).contiguous()
    mask = torch.zeros(B, L, L, dtype=torch.long)
    mask[:, :, :R + 2] = 1
    mask[:, R + 2:, R + 2:] = torch.tril(torch.ones(L - R - 2, L - R - 2, dtype=torch.long))
    vis = torch.randn(B, R, dims.vis_dim, generator=g).clamp_min(0)
    pe = torch.randn(B, R, dims.pe_dim, generator=g)
    return dims, _with_eos_bias(synth.make_state_dict(dims, seed=WEIGHTS_SEED), eos_bias), (vis, pe, input_ids, tt, pos, mask)


def _with_eos_bias(sd, eos_bias):
    if eos_bias:
        sd = dict(sd)
        bias = sd["cls.predictions.bias"].clone()
        bias[EOS_ID] += eos_bias
        sd["cls.predictions.bias"] = bias
    return sd


def n_frames(name):
    """Beam frames of a case: output length minus the input length ([CLS] + regions + [SEP])."""
    dims = case_inputs(name)[0]
    return dims.seq_len - dims.regions - 2


def most_frequent_word(wids):
    """The word id occurring most often in a [B, T, K] trace (smallest id on a tie)."""
    counts = collections.Counter(wids.flatten().tolist())
    return min(counts, key=lambda w: (-counts[w], w))


def run_reference(name, forbid, ignore=None, min_len=None):
    """The reference's beam search on case `name` (min_len: the case's unless given); returns (traces, blocked [N, 3] int64
    (frame, row, word)).  traces["cand_scores"] [B, T, K + 1]: per frame the K + 1 best scores of the pool the frame's K hypotheses
    were chosen from (the word scores at frame 0, the K·K extended hypothesis scores after), so that a decision that differs can be
    checked for a near-tie with the best candidate that was NOT chosen."""
    from oracle import ref_shim
    long_seq, B, n, case_min_len = CASES[name][:4]
    min_len = case_min_len if min_len is None else min_len
    dims, sd, args = case_inputs(name)
    model = ref_shim.build_reference_model(dims, sd, decoder=True, mask_word_id=103, eos_id=EOS_ID, search_beam_size=K,
                                           length_penalty=LENGTH_PENALTY, forbid_duplicate_ngrams=forbid,
                                           forbid_ignore_set=ignore, ngram_size=n, min_len=min_len).eval()
    orig_div, orig_cuda, orig_lsm, orig_topk = torch.div, torch.Tensor.cuda, torch.nn.functional.log_softmax, torch.topk
    frames, blocked, cands = [0], [], []

    def topk(x, k, *a, **kw):              # :1304 on [B, 1, V] scores at frame 0; :1316 on [B, K*K] after
        if (frames[0] == 1 and x.dim() == 3) or x.dim() == 2:
            cands.append(orig_topk(x.reshape(B, -1), K + 1).values)
        return orig_topk(x, k, *a, **kw)

    def floor_div(a, b, *rest, **kw):
        if not rest and not kw and torch.is_tensor(a) and not a.is_floating_point():
            return orig_div(a, b, rounding_mode="floor")
        return orig_div(a, b, *rest, **kw)

    def log_softmax(*a, **kw):             # once per frame (:1298)
        frames[0] += 1
        return orig_lsm(*a, **kw)

    def cuda_identity(t, *a, **kw):        # only the forbidden-word mask is moved (:1426); it is added to the NEXT frame's scores
        if frames[0] >= n_frames(name):    # the mask built after the last frame is never applied
            return t
        m = t.reshape(t.shape[0], -1)
        for row, word in (m != 0).nonzero().tolist():
            blocked.append((frames[0], row, word))
        return t

    torch.div, torch.Tensor.cuda, torch.nn.functional.log_softmax, torch.topk = floor_div, cuda_identity, log_softmax, topk
    try:
        with torch.no_grad():
            traces = model(*args, task_idx=None)
    finally:
        torch.div, torch.Tensor.cuda, torch.nn.functional.log_softmax, torch.topk = orig_div, orig_cuda, orig_lsm, orig_topk
    if len(cands) != n_frames(name):
        raise RuntimeError(f"case {name}: {len(cands)} beam selections recorded for {n_frames(name)} frames")
    traces["cand_scores"] = torch.stack(cands, dim=1).clone()
    if frames[0] != n_frames(name):
        raise RuntimeError(f"case {name}: {frames[0]} log_softmax calls for {n_frames(name)} frames; the frame numbering would be wrong")
    return {k: v.clone() for k, v in traces.items()}, torch.tensor(blocked, dtype=torch.int64).reshape(-1, 3)


def run_case(name):
    long_seq, B, n, min_len, ignore_rule, eos_bias = CASES[name]
    ignore = None
    if ignore_rule == "most_frequent":
        plain, _ = run_reference(name, forbid=False)
        ignore = [most_frequent_word(plain["wids"][:, :n_frames(name)])]
    traces, blocked = run_reference(name, forbid=True, ignore=set(ignore) if ignore else None)
    pairs = len({(f, r) for f, r, _ in blocked.tolist()})
    if pairs == 0:                         # explicit raise: this module runs under `python -O`
        raise RuntimeError(f"case {name}: the reference blocked nothing; the case does not exercise n-gram blocking")
    extra = {}
    if min_len:
        free, _ = run_reference(name, forbid=True, ignore=set(ignore) if ignore else None, min_len=0)
        if torch.equal(free["wids"], traces["wids"]):
            raise RuntimeError(f"case {name}: min_len = {min_len} changes no decision; the case does not exercise the [EOS] fill")
        if not bool((free["wids"][:, :min_len] == EOS_ID).any()):
            raise RuntimeError(f"case {name}: without min_len no beam takes [EOS] in the first {min_len} frames")
        extra["no_min_len"] = {k: free[k] for k in ("pred_seq", "scores", "wids", "ptrs", "cand_scores")}
    print(f"case {name}: n={n} min_len={min_len} ignore={ignore} blocked (frame, hypothesis) pairs {pairs}, words {blocked.shape[0]}; "
          f"pred_seq {traces['pred_seq'][0].tolist()}")
    return {"long_seq": long_seq, "B": B, "K": K, "ngram_size": n, "min_len": min_len, "ignore": ignore, "length_penalty": LENGTH_PENALTY,
            "seed": LONG_SEED if long_seq else SEED, "weights_seed": LONG_WEIGHTS_SEED if long_seq else WEIGHTS_SEED, "eos_bias": eos_bias,
            "blocked": blocked, "blocked_pairs": pairs, **traces, **extra}


if __name__ == "__main__":
    torch.set_num_threads(8)
    out = {"case": "ngram_beam", "cases": {n: run_case(n) for n in CASES}, "torch": str(torch.__version__), "reference_commit": "74c4d85"}
    path = os.path.join(ROOT, "tests", "golden", "ngram_beam.pt")
    torch.save(out, path)
    print(path, os.path.getsize(path), "bytes")
