"""GPU: prompted captions (`prompt_ids`).
 (1) the reference's own decode with the prompt appended to input_ids (tests/golden/prompt_decode.pt): greedy and beam search at H = 128
     and H = 768 (V = 28 996) and a relaxed head, EXACT-OR-EXPLAINED as the unprompted decode goldens are compared;
 (2) width 0 is today's decode, bitwise, in every mode;
 (3) teacher forcing: today's greedy captions, their first t_b words given back as ragged prompts, continue as they did;
 (4) each image of a ragged batch equals that image decoded alone at its own width;
 (5) the n-gram blocking and min_len on prompt + continuation, against the host rule on the whole caption;
 (6) GraphedCall captures a prompted decode; replays with other prompt words and lengths equal the eager decodes bitwise."""
import os

import pytest
import torch

from tools import prompt_decode_oracle as PO
from tools import relax_projection_oracle as RPO
from vlp_b200 import graph, synth
from vlp_b200 import vlp_modules as vm
from vlp_b200.beam import _dup_ngram_candidates

from test_parity_gpu import TOL_HID, make_config, rel

pytestmark = pytest.mark.gpu
MARGIN = 4e-2          # ~ 2 bf16 ulps at |logit| ~ 4
EOS, MASK = PO.EOS_ID, PO.MASK_ID


def _decoder(dims, K=1, relax=0, sd=None, **kw):
    cfg = make_config(dims)
    if relax:
        cfg.relax_projection = relax
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=MASK, eos_id=EOS, search_beam_size=K, enable_butd=True, len_vis_input=dims.regions,
                                     **kw)
    res = model.load_state_dict(synth.make_state_dict(dims, 0) if sd is None else sd, strict=False)
    assert not res.unexpected_keys
    return model.cuda().bfloat16().eval()


def _cuda(args):
    vis, pe, input_ids, tt, pos, mask = args
    return (vis.cuda().bfloat16(), pe.cuda().bfloat16(), input_ids.cuda(), tt.cuda(), pos.cuda(), mask.cuda())


def _first_diff(a, b):
    d = (a != b).nonzero()
    return None if d.numel() == 0 else int(d[:, -1].min())


def _gaps_hook(model, store):
    def hook(m, i, o):
        top2 = torch.topk(o.detach().float(), 2, dim=-1).values
        store.append((top2[..., 0] - top2[..., 1]).cpu())
    return model.cls.predictions.register_forward_hook(hook)


# ---------------------------------------------------------------------------------------------------------------------------
# (1) reference goldens
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "prompt_decode.pt"))


@pytest.mark.parametrize("name", list(PO.CASES))
def test_prompted_decode_matches_the_reference(name, gold):
    ref = gold["cases"][name]
    dims, sd, args, prompt, task_idx = PO.case_inputs(name)
    t = ref["t"]
    relax = RPO.RELAX if ref["relaxed"] else 0
    K = PO.K if ref["mode"] == "beam" else 1
    model = _decoder(dims, K=K, relax=relax, sd=sd, length_penalty=PO.LENGTH_PENALTY if K > 1 else 1.0)
    out = model(*_cuda(args), task_idx=None if task_idx is None else task_idx.cuda(), prompt_ids=prompt.cuda())
    frames = ref["cand_scores"].shape[1] if K > 1 else ref["ids"].shape[1]
    if K == 1:
        ids, scores = (x.cpu() for x in out)
        assert torch.equal(ids[:, :t], prompt) and float(scores[:, :t].float().abs().sum()) == 0.0
        gen, gsc = ids[:, t:t + frames], scores[:, t:t + frames].float()
        for b in range(ids.shape[0]):
            d = _first_diff(gen[b:b + 1], ref["ids"][b:b + 1])
            n_same = frames if d is None else d
            assert rel(gsc[b, :n_same], ref["scores"][b, :n_same]) < TOL_HID
            if d is not None:
                assert float(ref["gaps"][b, d]) < MARGIN, f"{name} sample {b}: id differs at frame {d}, margin {float(ref['gaps'][b, d]):.3f}"
                print(f"{name} sample {b}: first id flip at frame {d}, reference margin {float(ref['gaps'][b, d]):.4f}")
        return
    assert torch.equal(out["pred_seq"][:, :t].cpu(), prompt)
    for b in range(prompt.shape[0]):
        d = _first_diff(out["wids"][b, :frames].cpu().reshape(1, -1), ref["wids"][b, :frames].reshape(1, -1))
        n_same = frames if d is None else d // K
        assert rel(out["scores"][b, :n_same].float().cpu(), ref["scores"][b, :n_same]) < TOL_HID
        if d is None:
            assert torch.equal(out["ptrs"][b].cpu(), ref["ptrs"][b])
            assert torch.equal(out["pred_seq"][b, t:].cpu(), ref["pred_seq"][b, :dims.seq_len - t])
        else:
            cs = ref["cand_scores"][b, d // K]
            gap = float((cs[:-1] - cs[1:]).abs().min())
            assert gap < MARGIN, f"{name} sample {b}: decisions differ at frame {d // K} without a near-tie ({cs.tolist()})"
            print(f"{name} sample {b}: first differing word at frame {d // K}, near-tie {gap:.4f}")


# ---------------------------------------------------------------------------------------------------------------------------
# (2) width 0
# ---------------------------------------------------------------------------------------------------------------------------
MODES = {"greedy": dict(K=1), "topk": dict(K=1, sampling_method="topk", topk=8, forbid_duplicate_ngrams=True, ngram_size=2),
         "topp": dict(K=1, sampling_method="topp", topp=0.9), "topp_n3": dict(K=1, sampling_method="topp", topp=0.9, num_return_sequences=3),
         "beam_nbest": dict(K=4, num_return_sequences=3, forbid_duplicate_ngrams=True, ngram_size=2, min_len=3, length_penalty=0.5),
         "diverse": dict(K=4, num_beam_groups=2, diversity_penalty=0.7),
         "constrained": dict(K=2, constraints=[[5], [[7, 8]]])}


@pytest.mark.parametrize("mode", list(MODES))
def test_width_zero_is_todays_decode_bitwise(mode):
    dims = synth.SMALL_L123
    args = _cuda(PO.decode_inputs(dims, 3, 5))
    model = _decoder(dims, **MODES[mode])
    a = model(*args, task_idx=None)
    b = model(*args, task_idx=None, prompt_ids=torch.zeros(3, 0, dtype=torch.int64, device="cuda"))
    if isinstance(a, dict):
        assert set(a) == set(b) and all(torch.equal(a[k], b[k]) for k in a)
    else:
        assert all(torch.equal(x, y) for x, y in zip(a, b))


# ---------------------------------------------------------------------------------------------------------------------------
# (3) teacher forcing and (4) ragged batches
# ---------------------------------------------------------------------------------------------------------------------------
LENS = (0, 2, 5, 3)


def _ragged(ids, lens):
    Tp = max(lens)
    p = torch.zeros(len(lens), Tp, dtype=torch.int64, device=ids.device)
    for b, t in enumerate(lens):
        p[b, :t] = ids[b, :t]
    return p


def test_teacher_forced_prompts_continue_todays_captions():
    """The prefill of t_b given words must leave the decode where today's steps left it after choosing those words."""
    dims = synth.SMALL_L123
    args = _cuda(PO.decode_inputs(dims, len(LENS), 11))
    model = _decoder(dims)
    gaps = []
    h = _gaps_hook(model, gaps)
    try:
        ids0, sc0 = model(*args, task_idx=None)
    finally:
        h.remove()
    gaps = torch.cat(gaps, dim=1)                                         # [B, T] the arg-max margin of every frame
    Tp = max(LENS)
    # a prompt never holds [EOS]: the seeded captions must not take it within their first t_b words
    assert all(EOS not in ids0[b, :t].tolist() and MASK not in ids0[b, :t].tolist() for b, t in enumerate(LENS))
    ids, sc = model(*args, task_idx=None, prompt_ids=_ragged(ids0, LENS))
    T = ids0.shape[1]
    flips = 0
    for b, t in enumerate(LENS):
        assert torch.equal(ids[b, :t], ids0[b, :t])
        n = T - Tp
        d = _first_diff(ids[b:b + 1, t:t + n].cpu(), ids0[b:b + 1, t:t + n].cpu())
        n_same = n if d is None else d
        assert rel(sc[b, t:t + n_same].float(), sc0[b, t:t + n_same].float()) < TOL_HID
        if d is not None:
            flips += 1
            assert float(gaps[b, t + d]) < MARGIN, f"sample {b}: differs at word {t + d}, margin {float(gaps[b, t + d]):.3f}"
        assert bool((ids[b, t + n:] == 0).all())
    print(f"teacher forcing: {flips} of {len(LENS)} captions flip at a near-tie")


@pytest.mark.parametrize("K", [1, 3])
def test_each_image_of_a_ragged_batch_equals_it_decoded_alone(K):
    dims = synth.SMALL_L123
    args = _cuda(PO.decode_inputs(dims, len(LENS), 12))
    model = _decoder(dims, K=K, forbid_duplicate_ngrams=K > 1, ngram_size=2, min_len=4 if K > 1 else 0)
    g = torch.Generator().manual_seed(3)
    words = torch.randint(200, dims.vocab, (len(LENS), max(LENS)), generator=g).cuda()
    prompt = _ragged(words, LENS)
    out = model(*args, task_idx=None, prompt_ids=prompt)
    T, Tp = dims.seq_len - dims.regions - 2, max(LENS)
    bitwise = True
    for b, t in enumerate(LENS):
        one = tuple(a[b:b + 1] for a in args)
        alone = model(*one, task_idx=None, prompt_ids=prompt[b:b + 1, :t])
        n = T - Tp                                                        # the words the ragged batch generates for every image
        if K == 1:
            assert torch.equal(out[0][b, :t + n], alone[0][0, :t + n])
            assert rel(out[1][b, :t + n].float(), alone[1][0, :t + n].float()) < TOL_HID
            bitwise &= torch.equal(out[1][b, :t + n], alone[1][0, :t + n])
        else:
            # beams that hold the same words tie on their scores, and a rounding difference may pick the other parent of a tie:
            # the words and the scores of every slot are compared, and the back pointers only reported
            assert torch.equal(out["wids"][b, :n], alone["wids"][0, :n])
            assert rel(out["scores"][b, :n], alone["scores"][0, :n]) < TOL_HID
            bitwise &= torch.equal(out["scores"][b, :n], alone["scores"][0, :n]) and torch.equal(out["ptrs"][b, :n], alone["ptrs"][0, :n])
    print(f"ragged batch K={K}: scores bitwise equal to the images decoded alone: {bitwise}")


# ---------------------------------------------------------------------------------------------------------------------------
# (5) the rules on the whole caption
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2, 3])
def test_beam_ngram_blocking_sees_the_prompt(n):
    """Every generated word of every hypothesis is checked against the rule on its whole caption (prompt + its words): no beam ever
    repeats an n-gram of prompt + continuation, including n-grams of the prompt alone and n-grams that span its end."""
    dims = synth.SMALL_L123
    args = _cuda(PO.decode_inputs(dims, len(LENS), 13))
    K = 3
    model = _decoder(dims, K=K, forbid_duplicate_ngrams=True, ngram_size=n)
    plain = _decoder(dims, K=K)
    base = plain(*args, task_idx=None)
    # prompts that end in an n-gram prefix the unblocked search would complete: the first words the plain search chose, repeated
    words = base["pred_seq"][:, :max(LENS)]
    prompt = _ragged(torch.cat((words, words), 1), LENS)
    out = model(*args, task_idx=None, prompt_ids=prompt)
    wi, pt = out["wids"].cpu(), out["ptrs"].cpu()
    frames = dims.seq_len - dims.regions - 2 - max(LENS)
    checked = 0
    for b, t in enumerate(LENS):
        p = prompt[b, :t].tolist()
        hists = [[] for _ in range(K)]
        for f in range(frames):
            new = []
            for k in range(K):
                parent = hists[int(pt[b, f, k])] if f else []
                w = int(wi[b, f, k])
                if out["scores"][b, f, k] > -5000:                   # a hypothesis still alive (not pushed below by a block)
                    assert w not in _dup_ngram_candidates(p + parent, n, None), (b, f, k, p + parent, w)
                    checked += 1
                new.append(parent + [w])
            hists = new
    assert checked > 0


@pytest.mark.parametrize("kw", [dict(K=3), dict(K=1, sampling_method="topk", topk=8), dict(K=4, num_beam_groups=2, diversity_penalty=0.5),
                                dict(K=2, constraints=[[301]])], ids=["beam", "topk", "diverse", "constrained"])
def test_min_len_counts_the_prompt(kw):
    """With [EOS] made the most likely word, each image's first [EOS] comes at the first frame g with t_b + g + 1 > min_len."""
    dims = synth.SMALL_L123
    sd = synth.make_state_dict(dims, 0)
    sd["cls.predictions.bias"] = sd["cls.predictions.bias"].clone()
    sd["cls.predictions.bias"][EOS] += 30.0
    min_len = 6
    args = _cuda(PO.decode_inputs(dims, len(LENS), 14))
    model = _decoder(dims, sd=sd, min_len=min_len, seed=2, **kw)
    prompt = _ragged(torch.randint(200, dims.vocab, (len(LENS), max(LENS)), generator=torch.Generator().manual_seed(5)).cuda(), LENS)
    out = model(*args, task_idx=None, prompt_ids=prompt)
    for b, t in enumerate(LENS):
        if isinstance(out, dict):
            first = (out["wids"][b] == EOS).any(-1).nonzero().flatten().tolist()
        else:
            first = [g for g in range(out[0].shape[1] - t) if int(out[0][b, t + g]) == EOS]
        assert first and first[0] == max(min_len - t, 0), (b, t, first[:3])


# ---------------------------------------------------------------------------------------------------------------------------
# (6) graph capture
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kw", [dict(K=1), dict(K=3, num_return_sequences=2, forbid_duplicate_ngrams=True, ngram_size=2, min_len=5)],
                         ids=["greedy", "beam"])
def test_graphed_prompted_decode_equals_eager(kw):
    dims = synth.SMALL_L123
    args = _cuda(PO.decode_inputs(dims, len(LENS), 15))
    model = _decoder(dims, **kw)
    g = torch.Generator().manual_seed(4)
    p1 = _ragged(torch.randint(200, dims.vocab, (4, 5), generator=g).cuda(), LENS)
    p2 = _ragged(torch.randint(200, dims.vocab, (4, 5), generator=g).cuda(), (5, 0, 1, 4))
    call = graph.GraphedCall(lambda *x: model(*x[:6], task_idx=None, prompt_ids=x[6]), args + (p1,))
    for p in (p2, p1):
        eager = model(*args, task_idx=None, prompt_ids=p)
        out = call(*args, p)
        if isinstance(eager, dict):
            assert set(out) == set(eager) and all(torch.equal(out[k], eager[k]) for k in eager)
        else:
            assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
        seq = out["pred_seq"] if isinstance(out, dict) else out[0]
        assert torch.equal(torch.where(p != 0, seq[:, :5], p), p)          # each caption starts with its own prompt words


# ---------------------------------------------------------------------------------------------------------------------------
# (7) the prompted selectors: sampling, diverse and constrained beam search
# ---------------------------------------------------------------------------------------------------------------------------
def _host_histories(out_w, out_p, frames, K):
    """Per (image, frame, slot): the slot's generated words up to and including that frame, back-tracked through the pointers."""
    B = out_w.shape[0]
    res = [[None] * frames for _ in range(B)]
    for b in range(B):
        hists = None
        for f in range(frames):
            hists = [(hists[int(out_p[b, f, k])] if f else []) + [int(out_w[b, f, k])] for k in range(out_w.shape[2])]
            res[b][f] = hists
    return res


def test_constraint_met_inside_the_prompt_and_completed_across_its_end():
    """Image 0's prompt holds constraint 0's word and ends with the first word of constraint 1's phrase; image 1's prompt holds
    neither.  At frame 0 image 0 starts in state {0}: no slot of a state without constraint 0 is filled, and the slots of the
    accept state hold exactly the phrase's second word.  Image 1 starts in the root state and can reach no two-constraint state."""
    dims = synth.SMALL_L123
    args = _cuda(PO.decode_inputs(dims, 2, 16))
    w0, p1, p2 = 301, 302, 303
    model = _decoder(dims, K=2, constraints=[[w0], [[p1, p2]]])
    prompt = torch.tensor([[w0, 500, p1], [500, 501, 0]], device="cuda")
    out = model(*args, task_idx=None, prompt_ids=prompt)
    K = 2
    sc0, wi0 = out["scores"][:, 0].view(2, 4, K), out["wids"][:, 0].view(2, 4, K)
    assert bool(torch.isinf(sc0[0, 0]).all() and torch.isinf(sc0[0, 2]).all())          # states without constraint 0: empty
    assert bool(torch.isfinite(sc0[0, 3, 0])) and int(wi0[0, 3, 0]) == p2 and bool(torch.isinf(sc0[0, 3, 1]))
    assert bool(torch.isfinite(sc0[0, 1]).all())
    assert bool(torch.isfinite(sc0[1, 0]).all()) and bool(torch.isinf(sc0[1, 3]).all())
    assert bool(out["constraints_met"][0])
    assert out["pred_seq"][0, :3].tolist() == [w0, 500, p1] and out["pred_seq"][1, :2].tolist() == [500, 501]


FAVOURED = 250        # a word the head's bias makes the most likely everywhere: only the n-gram rule keeps it from repeating


@pytest.mark.parametrize("kw", [dict(K=3), dict(K=1, sampling_method="topk", topk=8),
                                dict(K=1, sampling_method="topp", topp=0.95, num_return_sequences=2),
                                dict(K=4, num_beam_groups=2, diversity_penalty=0.5),
                                dict(K=2, constraints=[[301], [[302, 303]]])],
                         ids=["beam", "topk", "topp_n2", "diverse", "constrained"])
def test_prompted_selectors_block_ngrams_of_the_whole_caption_and_count_min_len(kw):
    """Every word a prompted selector keeps is checked against the host rule on the whole caption (prompt + its words): no live
    hypothesis or sample repeats a bigram, and none ends before min_len words of caption.  The prompts are the favoured word
    repeated: the bigram (w, w) is in every prompt of two words or more, so the rule blocks w after w in the continuation."""
    dims = synth.SMALL_L123
    args = _cuda(PO.decode_inputs(dims, len(LENS), 17))
    sd = synth.make_state_dict(dims, 0)
    sd["cls.predictions.bias"] = sd["cls.predictions.bias"].clone()
    sd["cls.predictions.bias"][FAVOURED] += 12.0
    model = _decoder(dims, sd=sd, forbid_duplicate_ngrams=True, ngram_size=2, min_len=6, seed=3, **kw)
    prompt = _ragged(torch.full((len(LENS), max(LENS)), FAVOURED, device="cuda"), LENS)
    out = model(*args, task_idx=None, prompt_ids=prompt)
    frames = dims.seq_len - dims.regions - 2 - max(LENS)
    checked = 0
    if isinstance(out, tuple):                                            # sampling: [B, (N,) T]
        ids = out[0].view(len(LENS), -1, out[0].shape[-1]).cpu()
        for b, t in enumerate(LENS):
            for seq in ids[b].tolist():
                assert seq[:t] == prompt[b, :t].tolist()
                cap = seq[:t]
                assert t < 2 or seq[t] != FAVOURED, (b, seq[:t + 1])               # frame 0 sees the prompt's (w, w)
                for w in seq[t:t + frames]:
                    if w == 0:
                        break
                    assert w not in _dup_ngram_candidates(cap, 2, None), (b, cap, w)
                    assert w != EOS or len(cap) + 1 > 6, (b, cap)
                    cap.append(w)
                    checked += 1
                    if w == EOS:
                        break
    else:
        wi, pt, sc = out["wids"].cpu(), out["ptrs"].cpu(), out["scores"].cpu()
        hists = _host_histories(wi, pt, frames, wi.shape[2])
        for b, t in enumerate(LENS):
            p = prompt[b, :t].tolist()
            for f in range(frames):
                for k in range(wi.shape[2]):
                    if not bool(torch.isfinite(sc[b, f, k])) or sc[b, f, k] < -5000:
                        continue
                    h = hists[b][f][k]
                    assert h[-1] not in _dup_ngram_candidates(p + h[:-1], 2, None), (b, f, k, p + h)
                    assert t < 2 or f > 0 or h[-1] != FAVOURED, (b, k)         # frame 0 sees the prompt's (w, w)
                    assert h[-1] != EOS or t + f + 1 > 6, (b, f, k)
                    checked += 1
    assert checked > 0


@pytest.mark.parametrize("kw", [dict(K=1, sampling_method="topk", topk=8, forbid_duplicate_ngrams=True, ngram_size=2, min_len=4),
                                dict(K=4, num_beam_groups=2, diversity_penalty=0.5, forbid_duplicate_ngrams=True, ngram_size=2),
                                dict(K=2, constraints=[[301], [[302, 303]]], min_len=3)],
                         ids=["topk", "diverse", "constrained"])
def test_graphed_prompted_selectors_equal_eager(kw):
    dims = synth.SMALL_L123
    args = _cuda(PO.decode_inputs(dims, len(LENS), 18))
    model = _decoder(dims, seed=5, **kw)
    g = torch.Generator().manual_seed(9)
    p1 = _ragged(torch.randint(200, dims.vocab, (4, 5), generator=g).cuda(), LENS)
    p2 = _ragged(torch.randint(200, dims.vocab, (4, 5), generator=g).cuda(), (5, 0, 1, 4))
    call = graph.GraphedCall(lambda *x: model(*x[:6], task_idx=None, prompt_ids=x[6]), args + (p1,))
    for p in (p2, p1):
        eager = model(*args, task_idx=None, prompt_ids=p)
        out = call(*args, p)
        if isinstance(eager, dict):
            assert set(out) == set(eager) and all(torch.equal(out[k], eager[k]) for k in eager)
        else:
            assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])


def test_sampled_prompt_keeps_the_draws_of_each_generated_word():
    """With a prompt of width Tp, generated word g of row r is drawn with the uniform of (seed; g, r): a row whose prompt is empty
    draws the unprompted decode's words while its history matches (top-k = 1 would hide the draw; k = 8 does not)."""
    dims = synth.SMALL_L123
    args = _cuda(PO.decode_inputs(dims, 2, 19))
    model = _decoder(dims, sampling_method="topk", topk=8, seed=11)
    plain, _ = model(*args, task_idx=None)
    prompt = torch.tensor([[0, 0], [333, 334]], device="cuda")
    ids, _ = model(*args, task_idx=None, prompt_ids=prompt)
    n = plain.shape[1] - 2
    d = _first_diff(ids[:1, :n].cpu(), plain[:1, :n].cpu())
    assert d is None or d >= 3, f"row 0 differs from its unprompted draws at word {d}"
