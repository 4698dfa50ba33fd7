"""GPU: constrained beam search (`constraints`).
 (1) the kernels: vlpk_constrained_beam_step against the numpy statement of the frame (tools/constrained_beam_oracle.py) on random
     bf16 and fp32 logits, over phrases, alternatives, n-gram blocking with an ignore set, min_len and empty slots, at the stated
     limits of K; reruns are bitwise equal and the carried histories are bitwise vlpk_beam_ngram_block's;
 (2) constraints that are all empty: the accept state is today's beam search;
 (3) one-word constraints with room for all of them: every caption meets them;
 (4) the whole decode against the oracle's host decode (the full-vocabulary rule driving the model's own DecodeState);
 (5) every composing option completes, state_seq is each state's back-track, and a GraphedCall replay equals the Python-driven
     decode."""
import numpy as np
import pytest
import torch

from tools import constrained_beam_oracle as O
from vlp_b200 import graph, ops, synth

from test_diverse_beam_gpu import _args, _decoder, _traces

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
EOS = 102


def _random_table(gen, B, C, A, P, lo=1, hi=12):
    """Constraints over a small alphabet [lo, hi): alternatives of 1 .. P words, some constraints with fewer alternatives."""
    t = torch.zeros(B, C, A, P, dtype=torch.int64)
    for b in range(B):
        for j in range(C):
            for q in range(int(torch.randint(1, A + 1, (1,), generator=gen))):
                L = int(torch.randint(1, P + 1, (1,), generator=gen))
                t[b, j, q, :L] = torch.randint(lo, hi, (L,), generator=gen)
    return t


# ---------------------------------------------------------------------------------------------------------------------------------
# (1) the kernels
# ---------------------------------------------------------------------------------------------------------------------------------
KERNEL_CASES = [dict(C=1, A=2, P=2, K=64, n=2, ignore=(7,), min_len=0), dict(C=2, A=3, P=3, K=4, n=0, ignore=(), min_len=1),
                dict(C=3, A=2, P=1, K=6, n=3, ignore=(), min_len=2), dict(C=4, A=4, P=8, K=16, n=1, ignore=(3, 9), min_len=0),
                dict(C=2, A=4, P=2, K=64, n=2, ignore=(), min_len=0), dict(C=3, A=1, P=4, K=32, n=0, ignore=(), min_len=0)]
PARAMS = [(c, fp32, V) for c in KERNEL_CASES for fp32 in (False, True) for V in (37, 1000, 28996) if V >= c["K"] + c["C"] * c["A"]]


@pytest.mark.parametrize("case,fp32,V", PARAMS,
                         ids=[f"C{c['C']}-A{c['A']}-P{c['P']}-K{c['K']}-n{c['n']}-{'fp32' if f else 'bf16'}-V{V}" for c, f, V in PARAMS])
def test_kernel_matches_the_oracle(case, fp32, V):
    C, A, P, K, n, min_len = case["C"], case["A"], case["P"], case["K"], case["n"], case["min_len"]
    SK = K << C
    B, frames, eos = 2, 3, 5
    gen = torch.Generator(device=DEV).manual_seed(V + K + C + int(fp32))
    cons = _random_table(torch.Generator().manual_seed(V + C), B, C, A, P)
    cons_d = cons.to(DEV)
    dt = torch.float32 if fp32 else BF
    T = frames + 1
    wi, pt = (torch.zeros(T, B, SK, dtype=torch.int64, device=DEV) for _ in range(2))
    sc, eo = (torch.zeros(T, B, SK, device=DEV) for _ in range(2))
    W = K + C * A
    top_w, top_lp = torch.empty(B * SK, W, dtype=torch.int32, device=DEV), torch.empty(B * SK, W, device=DEV)
    top_dest = torch.empty(B * SK, C * A, dtype=torch.int32, device=DEV)
    hist = [torch.full((B * SK, T), -7, dtype=torch.int32, device=DEV) for _ in range(2)]
    ref = [h.clone() for h in hist]
    ign = torch.tensor(case["ignore"], dtype=torch.int32, device=DEV) if case["ignore"] else None
    bias = (torch.randn(V, generator=gen, device=DEV) * 0.5).to(dt)
    hists = None
    rows_checked = rows_total = 0
    for f in range(frames):
        rows = B if f == 0 else B * SK
        logits = torch.randn(rows, V, generator=gen, device=DEV) * 3
        logits[:, :12] += 6                                              # the constraints' alphabet: completions happen
        logits[:, eos] += 4
        logits = logits.to(dt)
        block_eos = bool(min_len) and f + 1 <= min_len
        ops.constrained_beam_step(logits.unsqueeze(1), bias, f, cons_d, wi, pt, sc, eo, top_w, top_lp, top_dest, eos, block_eos,
                                  ngram=n, ignore=ign, hist_in=hist[(f - 1) % 2], hist_out=hist[f % 2])
        blocked = None
        if f >= 1:                                                       # the history carry is beam_ngram_block's, n-grams or not
            lp_blk = torch.zeros(rows, V, device=DEV)
            ops.beam_ngram_block(ref[(f - 1) % 2], ref[f % 2], pt[f - 1], wi[f - 1], f, max(n, 1), ign, lp_blk)
            assert torch.equal(hist[f % 2][:, :f], ref[f % 2][:, :f]), f
            if n and f >= n:
                blocked = (lp_blk < -1).cpu().numpy()
            hists = [list(r) for r in ref[f % 2][:, :f].cpu().tolist()]
        x = (logits + bias).float().cpu().numpy()
        lp = O.frame_logp(x, blocked, block_eos, eos)
        prev = (sc[f - 1].cpu().numpy(), eo[f - 1].cpu().numpy()) if f else (None, None)
        gw, gp, gs, ge = (t[f].cpu() for t in (wi, pt, sc, eo))
        # the row stage: the completing words exactly; the top K wherever no two of its K + 1 best lie within fp32 rounding
        kl = O.kernel_lists(top_w[:rows].cpu().numpy(), top_lp[:rows].cpu().numpy(), top_dest[:rows].cpu().numpy(), K)
        ol = O.row_lists(lp, hists, cons.numpy(), K, C, f == 0, top=K + 1)
        for i, ((kw, kv, kc), (ow, ov, oc)) in enumerate(zip(kl, ol)):
            assert {w: d for w, (_, d) in kc.items()} == {w: d for w, (_, d) in oc.items()}, (f, i)
            for w, (l, _) in kc.items():
                assert l == pytest.approx(float(lp[i, w]), rel=1e-6, abs=1e-4)
            gaps = ov[:-1].astype(np.float64) - ov[1:]
            near = 8 * np.finfo(np.float32).eps * np.maximum(np.abs(ov[:-1]), 1)
            xs = x[i, ow]
            if ((gaps > near) | ((gaps == 0) & (xs[:-1] == xs[1:]))).all():
                rows_checked += 1
                np.testing.assert_array_equal(kw, ow[:K])
                np.testing.assert_allclose(kv, ov[:K], rtol=1e-6, atol=1e-4)
        rows_total += rows
        # the merge: exactly the oracle's merge over the kernel's own row lists
        mw, mp, ms, _ = O.merge(kl, *prev, cons.numpy(), K, f == 0)
        assert torch.equal(gw, torch.from_numpy(mw)) and torch.equal(gp, torch.from_numpy(mp)), f
        assert torch.equal(gs, torch.from_numpy(ms)), f
        # the whole frame against the oracle, wherever its margin at the selection boundary exceeds 1e-3
        ow, op, osc, margin = O.two_stage(lp, hists, *prev, cons.numpy(), K, f == 0)
        ok = torch.from_numpy(margin > 1e-3)
        assert torch.equal(gw[ok], torch.from_numpy(ow)[ok]), f
        assert torch.equal(gp[ok], torch.from_numpy(op)[ok]), f
        torch.testing.assert_close(gs[ok], torch.from_numpy(osc)[ok], rtol=1e-6, atol=1e-4)
        assert torch.equal(ge, ((gw == eos) & torch.isfinite(gs)).float())
        empty = ~torch.isfinite(gs)
        assert (gw[empty] == 0).all() and (gp[empty] == 0).all()
    assert rows_checked * 4 >= rows_total, (rows_checked, rows_total)


def test_kernel_is_bitwise_reproducible():
    B, K, C, A, P, V = 3, 6, 3, 2, 2, 28996
    SK = K << C
    cons = _random_table(torch.Generator().manual_seed(0), B, C, A, P).to(DEV)
    outs = []
    for _ in range(2):
        wi, pt = (torch.zeros(2, B, SK, dtype=torch.int64, device=DEV) for _ in range(2))
        sc, eo = (torch.zeros(2, B, SK, device=DEV) for _ in range(2))
        tw, tl = torch.empty(B * SK, K + C * A, dtype=torch.int32, device=DEV), torch.empty(B * SK, K + C * A, device=DEV)
        td = torch.empty(B * SK, C * A, dtype=torch.int32, device=DEV)
        hist = [torch.zeros(B * SK, 2, dtype=torch.int32, device=DEV) for _ in range(2)]
        gen = torch.Generator(device=DEV).manual_seed(1)
        l0 = torch.randn(B, V, generator=gen, device=DEV).to(BF)
        l1 = torch.randn(B * SK, V, generator=gen, device=DEV).to(BF)
        l0[:, :12] += 3
        l1[:, :12] += 3
        ops.constrained_beam_step(l0, None, 0, cons, wi, pt, sc, eo, tw, tl, td, EOS, hist_in=hist[1], hist_out=hist[0])
        ops.constrained_beam_step(l1, None, 1, cons, wi, pt, sc, eo, tw, tl, td, EOS, hist_in=hist[0], hist_out=hist[1])
        outs.append((wi, pt, sc, eo, tw, tl, td, hist[1]))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------------------
# (2) - (5) decodes
# ---------------------------------------------------------------------------------------------------------------------------------
def _check_states(out, model, cons, T):
    """state_seq / state_scores / pred_seq / constraints_met against the oracle's final selection over the decode's own traces."""
    sc, wi, pt = (t.cpu().numpy() for t in _traces(out, T))
    K, C = model.search_beam_size, cons.shape[1]
    pred, state_seq, state_val, met = O.select(sc, wi, pt, EOS, model.length_penalty, K, C)
    assert np.array_equal(out["state_seq"][:, :, :T].cpu().numpy(), state_seq)
    assert (out["state_seq"][:, :, T:] == 0).all() and (out["pred_seq"][:, T:] == 0).all()
    np.testing.assert_array_equal(out["state_scores"].cpu().numpy(), state_val.astype(np.float32))
    assert np.array_equal(out["pred_seq"][:, :T].cpu().numpy(), pred)
    assert np.array_equal(out["constraints_met"].cpu().numpy(), met)


def test_empty_constraints_are_todays_beam_search():
    dims = synth.SMALL_L123
    B, K = 8, 4
    args = _args(dims, B, seed=3)
    T = args[3].shape[1] - args[2].shape[1]
    model = _decoder(dims, search_beam_size=K)
    plain = model(*args, task_idx=None)
    cons = torch.zeros(B, 1, 1, 1, dtype=torch.int64, device=DEV)       # one constraint without alternatives: met from the start
    out = model(*args, task_idx=None, constraints=cons)
    sc, wi, pt = _traces(out, T)
    assert not torch.isfinite(sc[:, :, :K]).any()                       # state 0 is never reached
    psc, pwi, ppt = _traces(plain, T)
    # images where no tie between two parents (exact at the -10000 scale of finished hypotheses) or near-tie flips the selection:
    # torch.topk breaks ties in its own order, the kernels by the lower parent, then the lower word
    same = (pwi == wi[:, :, K:]).all(2).all(0) & (ppt[1:] == pt[1:, :, K:] - K).all(2).all(0)
    assert int(same.sum()) >= B // 2, same
    assert torch.equal(out["pred_seq"][same], plain["pred_seq"][same])
    torch.testing.assert_close(sc[:, same, K:], psc[:, same], rtol=1e-5, atol=1e-4)
    assert out["constraints_met"].all()
    _check_states(out, model, cons, T)


def test_one_word_constraints_are_always_met():
    dims = synth.SMALL_L123
    B, K, C = 6, 3, 3
    args = _args(dims, B, seed=5)
    T = args[3].shape[1] - args[2].shape[1]
    assert T >= C + 1
    gen = torch.Generator().manual_seed(5)
    cons = torch.zeros(B, C, 2, 1, dtype=torch.int64)
    cons[:, :, :, 0] = torch.randint(200, 900, (B, C, 2), generator=gen)  # unlikely words, two alternatives each
    cons[0, 1, 1] = 0
    model = _decoder(dims, search_beam_size=K)
    out = model(*args, task_idx=None, constraints=cons.to(DEV))
    assert out["constraints_met"].all()
    for b in range(B):
        words = out["pred_seq"][b].tolist()
        for j in range(C):
            assert any(int(w) in words for w in cons[b, j, :, 0] if w), (b, j, words)
    _check_states(out, model, cons, T)


@pytest.mark.parametrize("kw,C", [(dict(search_beam_size=2), 2), (dict(search_beam_size=3, forbid_duplicate_ngrams=True, ngram_size=2,
                                                                         forbid_ignore_set={7}, length_penalty=0.5), 1)],
                         ids=["K2-C2", "K3-C1-ngram"])
def test_decode_matches_the_oracle_host_decode(kw, C):
    """Every frame of the decode against the full-vocabulary rule on the model's own logits: the oracle's host decode follows the
    device's traces and selects each frame anew, which must equal the device's wherever the oracle's smallest gap at a selection
    boundary exceeds 5e-5 (fp32 rounding of logsumexp cannot reorder the pairs).  [EOS] is blocked throughout, since finished
    hypotheses tie exactly at the -10000 scale."""
    dims = synth.SMALL_L123
    B = 3
    args = _args(dims, B, seed=11 + C)
    T = args[3].shape[1] - args[2].shape[1]
    model = _decoder(dims, min_len=T, **kw)
    first = model(*args, task_idx=None)["wids"][:, 0, 0]               # beam search's first words: a constraint met early
    cons = _random_table(torch.Generator().manual_seed(C), B, C, 2, 2, lo=990, hi=1000)
    cons[:, 0, 0, 0] = first.cpu()
    cons[:, 0, 0, 1:] = 0
    out = model(*args, task_idx=None, constraints=cons.to(DEV))
    _check_states(out, model, cons, T)
    dev = tuple(t.cpu().numpy() for t in _traces(out, T))
    with torch.no_grad():
        (sc, wi, pt), margin = O.host_decode(model, *model.project_regions(args[0], args[1]), *args[2:], cons, follow=dev)
    ok = margin > 5e-5                                                   # [T, B]
    assert ok.mean() >= 0.5, ok
    np.testing.assert_array_equal(dev[1][ok], wi[ok])
    np.testing.assert_array_equal(dev[2][ok], pt[ok])
    np.testing.assert_allclose(dev[0][ok], sc[ok], rtol=1e-5, atol=1e-4)


DECODE_CASES = [dict(K=3, C=2, forbid_duplicate_ngrams=True, ngram_size=2, forbid_ignore_set={7, 11}, min_len=4, length_penalty=0.5),
                dict(K=4, C=1, N=3), dict(K=2, C=3, attn=True), dict(K=2, C=2, relax=4, length_penalty=-1.0),
                dict(K=4, C=4, P=3)]


@pytest.mark.parametrize("case", DECODE_CASES, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_decode_completes_with_every_option(case):
    case = dict(case)
    K, C, P = case.pop("K"), case.pop("C"), case.pop("P", 2)
    N, attn, relax = case.pop("N", 1), case.pop("attn", False), case.pop("relax", 0)
    dims = synth.SMALL_L123
    B = 5
    args = _args(dims, B, seed=K + C)
    task_idx = torch.tensor([0, 3, 1, 2, 3], device=DEV) if relax else None
    model = _decoder(dims, relax=relax, search_beam_size=K, **case)
    cons = _random_table(torch.Generator().manual_seed(K * C), B, C, 2, P, lo=100, hi=110).to(DEV)
    out = model(*args, task_idx=task_idx, output_attentions=attn, constraints=cons)
    out_len = args[3].shape[1]
    T = out_len - args[2].shape[1]
    S = 1 << C
    assert out["state_seq"].shape == (B, S, out_len) and out["scores"].shape == (B, out_len, S * K)
    _check_states(out, model, cons, T)
    if attn:
        assert out["attentions"].shape == (B, T, dims.layers, dims.heads, out_len)
        assert torch.isfinite(out["attentions"]).all()
    if N > 1:
        model.num_return_sequences = N
        many = model(*args, task_idx=task_idx, constraints=cons)
        for k in ("scores", "wids", "ptrs", "pred_seq", "state_seq", "state_scores"):
            assert torch.equal(many[k], out[k]), k
        assert many["nbest_seq"].shape == (B, N, out_len)
        met = out["constraints_met"]
        assert torch.equal(many["nbest_seq"][met, 0], out["pred_seq"][met])
    again = model(*args, task_idx=task_idx, output_attentions=attn, constraints=cons)
    for k in out:
        assert torch.equal(again[k], out[k]), k


def test_graphed_call_equals_the_python_driven_decode():
    dims = synth.SMALL_L123
    args = _args(dims, 4, seed=6)
    model = _decoder(dims, search_beam_size=3, forbid_duplicate_ngrams=True, ngram_size=2, min_len=2,
                     constraints=[[[104, 105], 106], [107]])
    eager = model(*args, task_idx=None)
    g = graph.GraphedCall(lambda *x: model(*x, task_idx=None), args)
    out = g(*args)
    assert set(out) == set(eager)
    for k in eager:
        assert torch.equal(out[k], eager[k]), k
    cons = _random_table(torch.Generator().manual_seed(9), 4, 2, 2, 2, lo=100, hi=110).to(DEV)
    eager = model(*args, task_idx=None, constraints=cons)
    g = graph.GraphedCall(lambda *x: model(*x[:-1], task_idx=None, constraints=x[-1]), args + (cons,))
    args2 = _args(dims, 4, seed=7)
    cons2 = _random_table(torch.Generator().manual_seed(10), 4, 2, 2, 2, lo=100, hi=110).to(DEV)
    eager2 = model(*args2, task_idx=None, constraints=cons2)
    out2 = g(*args2, cons2)
    for k in eager2:
        assert torch.equal(out2[k], eager2[k]), k
    out = g(*args, cons)
    for k in eager:
        assert torch.equal(out[k], eager[k]), k
