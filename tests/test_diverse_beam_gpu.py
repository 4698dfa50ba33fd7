"""GPU: diverse beam search (`num_beam_groups` G > 1, `diversity_penalty` lambda).
 (1) the kernels: vlpk_diverse_beam_step against the numpy statement of the frame (tools/diverse_beam_oracle.py) on random bf16 and
     fp32 logits, with n-gram blocking over an ignore set and the min_len [EOS] block; its histories are bitwise
     vlpk_beam_ngram_block's;
 (2) decodes: lambda = 0 makes every group a copy of group 0, which is today's beam search at K / G beams; a large lambda keeps the
     groups' words apart; reruns are bitwise equal; every composing option completes; group_seq is each group's back-track;
     the shared prefix cache (num_return_sequences > 1) gives bitwise the traces of N = 1; a GraphedCall replay equals the
     Python-driven decode."""
import dataclasses

import pytest
import torch

from tools import diverse_beam_oracle as O
from tools import relax_projection_oracle as RPO
from vlp_b200 import beam, graph, ops, synth
from vlp_b200 import vlp_modules as vm

from test_decode_gpu import _inputs
from test_parity_gpu import make_config

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
EOS = 102


# ---------------------------------------------------------------------------------------------------------------------------------
# (1) the kernels
# ---------------------------------------------------------------------------------------------------------------------------------
KERNEL_CASES = [dict(K=6, G=3, lam=0.5, n=2, ignore=(7, 11), min_len=2), dict(K=4, G=2, lam=0.0, n=0, ignore=(), min_len=0),
                dict(K=8, G=8, lam=2.0, n=1, ignore=(3,), min_len=1), dict(K=32, G=4, lam=0.3, n=3, ignore=(), min_len=3),
                dict(K=64, G=2, lam=5.0, n=2, ignore=(5, 9), min_len=0), dict(K=48, G=1, lam=0.0, n=2, ignore=(), min_len=0)]


@pytest.mark.parametrize("V", [37, 1000, 28996])
@pytest.mark.parametrize("fp32", [False, True], ids=["bf16", "fp32"])
@pytest.mark.parametrize("case", KERNEL_CASES, ids=lambda c: f"K{c['K']}-G{c['G']}-n{c['n']}")
def test_kernel_matches_the_oracle(case, fp32, V):
    K, G, lam, n, min_len = case["K"], case["G"], case["lam"], case["n"], case["min_len"]
    if K > V:
        pytest.skip("the beam is wider than the vocabulary")
    B, frames = 3, 6
    eos = 5
    gen = torch.Generator(device=DEV).manual_seed(V + K + int(fp32))
    dt = torch.float32 if fp32 else BF
    T = frames + 1
    wi, pt = (torch.zeros(T, B, K, dtype=torch.int64, device=DEV) for _ in range(2))
    sc, eo = (torch.zeros(T, B, K, device=DEV) for _ in range(2))
    top_w, top_lp = torch.empty(B * K, K, dtype=torch.int32, device=DEV), torch.empty(B * K, K, device=DEV)
    hist = [torch.full((B * K, T), -7, dtype=torch.int32, device=DEV) for _ in range(2)]
    ref = [h.clone() for h in hist]
    ign = torch.tensor(case["ignore"], dtype=torch.int32, device=DEV) if case["ignore"] else None
    bias = (torch.randn(V, generator=gen, device=DEV) * 0.5).to(dt)
    rows_checked = rows_total = 0
    for f in range(frames):
        rows = B if f == 0 else B * K
        logits = torch.randn(rows, V, generator=gen, device=DEV) * 3
        logits[:, :12] += 6                                              # a small alphabet, so that n-grams repeat
        logits[:, eos] += 4
        logits = logits.to(dt)
        block_eos = bool(min_len) and f + 1 <= min_len
        ops.diverse_beam_step(logits.unsqueeze(1), bias, f, G, lam, wi, pt, sc, eo, top_w, top_lp, eos, block_eos, ngram=n, ignore=ign,
                              hist_in=hist[(f - 1) % 2], hist_out=hist[f % 2])
        blocked = None
        if n and f >= 1:
            lp_blk = torch.zeros(rows, V, device=DEV)
            ops.beam_ngram_block(ref[(f - 1) % 2], ref[f % 2], pt[f - 1], wi[f - 1], f, n, ign, lp_blk)
            assert torch.equal(hist[f % 2][:, :f], ref[f % 2][:, :f]), f
            blocked = (lp_blk < -1).cpu().numpy()
        x = (logits + bias).float().cpu().numpy()                        # the head's rounding: decoder(h) + bias in its dtype
        lp = O.frame_logp(x, blocked, block_eos, eos)
        prev = (sc[f - 1].cpu().numpy(), eo[f - 1].cpu().numpy()) if f else (None, None)
        gw, gp, gs, ge = (t[f].cpu() for t in (wi, pt, sc, eo))
        # the row stage: each row's top K against the oracle's, wherever no two of its K + 1 best lie within a few fp32 rounding
        # steps of each other (a tie of equal logits is broken by word id on both sides: one row shares one logsumexp)
        tw, tl = top_w[:rows].cpu(), top_lp[:rows].cpu()
        ow, ol = (torch.from_numpy(a) for a in O.row_topk(lp, K + 1))
        gaps = ol[:, :-1].double() - ol[:, 1:].double()
        near = 8 * torch.finfo(torch.float32).eps * ol[:, :-1].double().abs().clamp(min=1)
        xs = torch.from_numpy(x).gather(1, ow)
        clear = ((gaps > near) | ((gaps == 0) & (xs[:, :-1] == xs[:, 1:]))).all(1)
        rows_checked += int(clear.sum())
        rows_total += rows
        assert torch.equal(tw[clear].long(), ow[clear, :K]), f
        torch.testing.assert_close(tl[clear], ol[clear, :K], rtol=1e-6, atol=1e-4)
        # the merge: exactly the oracle's merge over the kernel's own row top K
        mw, mp, ms, _ = O.merge(tw.numpy(), tl.numpy(), *prev, K, G, lam, f == 0)
        assert torch.equal(gw, torch.from_numpy(mw)) and torch.equal(gp, torch.from_numpy(mp)), f
        assert torch.equal(gs, torch.from_numpy(ms)), f
        # the whole frame against the oracle, wherever its margin at the selection boundary exceeds 1e-3
        ow, op, osc, margin = O.two_stage(lp, *prev, K, G, lam, f == 0)
        ok = torch.from_numpy(margin > 1e-3)
        assert torch.equal(gw[ok], torch.from_numpy(ow)[ok]), f
        assert torch.equal(gp[ok], torch.from_numpy(op)[ok]), f
        torch.testing.assert_close(gs[ok], torch.from_numpy(osc)[ok], rtol=1e-6, atol=1e-4)
        assert torch.equal(ge, (gw == eos).float())
        if f == 0:
            assert (gp == 0).all()
        else:                                                            # every group extends its own beams
            Kg = K // G
            assert ((gp // Kg) == (torch.arange(K) // Kg)).all()
    assert rows_checked * 4 >= rows_total, (rows_checked, rows_total)


def test_kernel_is_bitwise_reproducible():
    B, K, G, V = 4, 6, 3, 28996
    gen = torch.Generator(device=DEV).manual_seed(1)
    outs = []
    for _ in range(2):
        wi, pt = (torch.zeros(2, B, K, dtype=torch.int64, device=DEV) for _ in range(2))
        sc, eo = (torch.zeros(2, B, K, device=DEV) for _ in range(2))
        tw, tl = torch.empty(B * K, K, dtype=torch.int32, device=DEV), torch.empty(B * K, K, device=DEV)
        gen.manual_seed(1)
        l0 = torch.randn(B, V, generator=gen, device=DEV).to(BF)
        l1 = torch.randn(B * K, V, generator=gen, device=DEV).to(BF)
        ops.diverse_beam_step(l0, None, 0, G, 0.7, wi, pt, sc, eo, tw, tl, EOS)
        ops.diverse_beam_step(l1, None, 1, G, 0.7, wi, pt, sc, eo, tw, tl, EOS)
        outs.append((wi, pt, sc, eo, tw, tl))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------------------------------
# (2) decodes
# ---------------------------------------------------------------------------------------------------------------------------------
def _decoder(dims, relax=0, **kw):
    cfg = make_config(dims)
    if relax:
        cfg.relax_projection = relax
    model = vm.BertForSeq2SeqDecoder(cfg, mask_word_id=103, eos_id=EOS, enable_butd=True, len_vis_input=dims.regions, **kw)
    sd = synth.make_state_dict(dims, 0)
    model.load_state_dict(RPO.relaxed_state_dict(sd, dims.hidden, relax) if relax else sd, strict=False)
    return model.cuda().bfloat16().eval()


def _args(dims, B, seed=0):
    vis, pe, input_ids, tt, pos, mask = _inputs(dims, B, seed)
    return (vis.cuda().bfloat16(), pe.cuda().bfloat16(), input_ids.cuda(), tt.cuda(), pos.cuda(), mask.cuda())


def _traces(out, T):
    return tuple(out[k][:, :T].permute(1, 0, 2) for k in ("scores", "wids", "ptrs"))


def _check_groups(out, model, T):
    """group_seq / group_scores are each group's final selection over its own beams, and pred_seq the selection over all beams."""
    sc, wi, pt = _traces(out, T)
    K, G = model.search_beam_size, model.num_beam_groups
    Kg = K // G
    out_len = out["pred_seq"].shape[1]
    assert torch.equal(out["pred_seq"], beam.backtrack(sc, wi, pt, EOS, model.length_penalty, out_len))
    for g in range(G):
        s = slice(g * Kg, (g + 1) * Kg)
        pg = pt[:, :, s]
        assert ((pg[1:] >= g * Kg) & (pg[1:] < (g + 1) * Kg)).all()
        pg = pg - g * Kg
        pg[0] = 0
        assert torch.equal(out["group_seq"][:, g], beam.backtrack(sc[:, :, s], wi[:, :, s], pg, EOS, model.length_penalty, out_len))
        want = beam.candidate_values(sc[:, :, s], wi[:, :, s], EOS, model.length_penalty).max(1).values
        assert torch.equal(out["group_scores"][:, g], want)


def test_zero_penalty_groups_copy_group_zero_which_is_beam_search():
    dims = synth.SMALL_L123
    B, K, G = 8, 6, 3
    Kg = K // G
    args = _args(dims, B, seed=3)
    T = args[3].shape[1] - args[2].shape[1]
    model = _decoder(dims, search_beam_size=K, num_beam_groups=G, diversity_penalty=0.0)
    out = model(*args, task_idx=None)
    sc, wi, pt = _traces(out, T)
    for g in range(1, G):
        s = slice(g * Kg, (g + 1) * Kg)
        assert torch.equal(sc[:, :, s], sc[:, :, :Kg]) and torch.equal(wi[:, :, s], wi[:, :, :Kg])
        assert torch.equal(pt[1:, :, s] - g * Kg, pt[1:, :, :Kg])
        assert torch.equal(out["group_seq"][:, g], out["group_seq"][:, 0])
    plain = _decoder(dims, search_beam_size=Kg)(*args, task_idx=None)
    psc, pwi, _ = _traces(plain, T)
    same = (pwi == wi[:, :, :Kg]).all(2).all(0)                          # images without a near-tie flip between the two selections
    assert int(same.sum()) >= B * 3 // 4, same
    assert torch.equal(out["group_seq"][same, 0], plain["pred_seq"][same])
    torch.testing.assert_close(sc[:, same, :Kg], psc[:, same], rtol=1e-5, atol=1e-4)


def test_large_penalty_keeps_the_groups_words_apart():
    dims = synth.SMALL_L123
    B, K, G = 5, 6, 3
    Kg = K // G
    args = _args(dims, B, seed=4)
    T = args[3].shape[1] - args[2].shape[1]
    model = _decoder(dims, search_beam_size=K, num_beam_groups=G, diversity_penalty=1000.0, min_len=T)
    out = model(*args, task_idx=None)
    wi = out["wids"][:, :T].cpu()
    for b in range(B):
        for t in range(T):
            seen = set()
            for g in range(G):
                words = set(wi[b, t, g * Kg:(g + 1) * Kg].tolist())
                assert not words & seen, (b, t, g)
                seen |= words
    _check_groups(out, model, T)
    assert any(len({tuple(out["group_seq"][b, g].tolist()) for g in range(G)}) == G for b in range(B))


LONG = dataclasses.replace(synth.SMALL_L123, text=60)                    # 102 + 60 rows: the tiled attention kernels from frame ~26 on
DECODE_CASES = [
    dict(K=6, G=3, lam=0.5, forbid_duplicate_ngrams=True, ngram_size=2, forbid_ignore_set={7, 11}, min_len=4, length_penalty=0.5),
    dict(K=4, G=2, lam=1.0, N=3),
    dict(K=6, G=2, lam=0.5, attn=True),
    dict(K=4, G=4, lam=0.3, relax=4, length_penalty=-1.0),
    dict(K=4, G=2, lam=0.5, nokv=True, forbid_duplicate_ngrams=True, ngram_size=3),
    dict(K=4, G=2, lam=0.5, N=2, dims="long", forbid_duplicate_ngrams=True, ngram_size=2, min_len=3),
    dict(K=6, G=3, lam=0.8, dims="base", forbid_duplicate_ngrams=True, ngram_size=3, forbid_ignore_set={1012}, N=2)]


@pytest.mark.parametrize("case", DECODE_CASES, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_decode_completes_with_every_option(case):
    case = dict(case)
    K, G, lam = case.pop("K"), case.pop("G"), case.pop("lam")
    N, attn, nokv, relax = case.pop("N", 1), case.pop("attn", False), case.pop("nokv", False), case.pop("relax", 0)
    dims = {"long": LONG, "base": synth.BERT_BASE, None: synth.SMALL_L123}[case.pop("dims", None)]
    B = 2 if dims is synth.BERT_BASE else 5
    args = _args(dims, B, seed=K + G)
    task_idx = torch.tensor([0, 3, 1, 2, 3], device=DEV) if relax else None
    model = _decoder(dims, relax=relax, search_beam_size=K, num_beam_groups=G, diversity_penalty=lam, **case)
    model.use_kv_cache = not nokv
    out = model(*args, task_idx=task_idx, output_attentions=attn)
    out_len = args[3].shape[1]
    T = out_len - args[2].shape[1]
    assert out["group_seq"].shape == (B, G, out_len) and out["group_scores"].shape == (B, G)
    assert torch.isfinite(out["group_scores"]).all()
    _check_groups(out, model, T)
    if attn:
        assert out["attentions"].shape == (B, T, dims.layers, dims.heads, out_len)
        assert torch.isfinite(out["attentions"]).all()
    if N > 1:                                                            # the shared prefix cache: bitwise the N = 1 traces
        model.num_return_sequences = N
        many = model(*args, task_idx=task_idx)
        for k in ("scores", "wids", "ptrs", "pred_seq", "group_seq", "group_scores"):
            assert torch.equal(many[k], out[k]), k
        assert many["nbest_seq"].shape == (B, N, out_len)
        assert torch.equal(many["nbest_seq"][:, 0], out["pred_seq"])
    again = model(*args, task_idx=task_idx)
    for k in ("scores", "wids", "ptrs", "group_seq"):
        assert torch.equal(again[k], out[k]), k


@pytest.mark.parametrize("kw", [dict(search_beam_size=6, num_beam_groups=3, diversity_penalty=0.5, forbid_duplicate_ngrams=True,
                                     ngram_size=2, forbid_ignore_set={7}, min_len=3),
                                dict(search_beam_size=4, num_beam_groups=2, diversity_penalty=1.0, num_return_sequences=4)],
                         ids=["ngram", "nbest"])
def test_graphed_call_equals_the_python_driven_decode(kw):
    dims = synth.SMALL_L123
    args = _args(dims, 4, seed=6)
    model = _decoder(dims, **kw)
    eager = model(*args, task_idx=None)
    g = graph.GraphedCall(lambda *x: model(*x, task_idx=None), args)
    out = g(*args)
    assert set(out) == set(eager)
    for k in eager:
        assert torch.equal(out[k], eager[k]), k
    args2 = _args(dims, 4, seed=7)
    eager2 = model(*args2, task_idx=None)
    out2 = g(*args2)
    for k in eager2:
        assert torch.equal(out2[k], eager2[k]), k
