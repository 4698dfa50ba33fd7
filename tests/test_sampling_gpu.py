"""GPU: top-k / top-p sampling (vlpk_sample_tokens, vlp_b200/decode.py).
 (1) the kernel: topk = 1 and topp -> 0 are the first arg-max of the head's logits (bias added in the logits' dtype), ties included, at
     ragged vocabularies up to 30 522; every draw lies in the torch-computed top-k set / nucleus (words ranked by logit, then id) and its
     score is the full log-softmax; 2^16 draws per case pass a chi-square test against the renormalised torch distribution at
     ALPHA; draws depend on (seed, frame, row) only; n-gram blocking follows beam._dup_ngram_candidates and the [EOS] block holds;
     finished rows write padding and the live count drops once per [EOS];
 (2) the decode: topk = 1 / tiny topp equal the greedy decode, and with n-gram blocking (and min_len) beam search at beam size 1;
     a decode whose rows all draw [EOS] stops early; decodes are reproducible per seed; a GraphedCall capture replays the eager decode."""
import pytest
import torch
from scipy import stats

from vlp_b200 import beam, graph, ops, synth

from test_decode_gpu import _decoder, _inputs

pytestmark = pytest.mark.gpu
DEV = "cuda"
ALPHA = 1e-3           # chi-square significance level: a correct sampler fails one case in a thousand (the draws are seeded: fixed outcome)
EOS = 102


def _run(logits, mode, k=1, p=1.0, seed=0, bias=None, f=0, T=4, seq=None, finished=None, **kw):
    rows = logits.shape[0]
    seq = torch.full((rows, T), -1, dtype=torch.int64, device=DEV) if seq is None else seq
    score = torch.zeros(rows, T, dtype=torch.float32, device=DEV)
    finished = torch.zeros(rows, dtype=torch.int32, device=DEV) if finished is None else finished
    live = torch.full((1,), rows - int(finished.sum()), dtype=torch.int32, device=DEV)
    ops.sample_tokens(logits, bias, mode, k, p, seed, f, seq, score, finished, live, kw.pop("eos_id", EOS), **kw)
    return seq[:, f], score[:, f], finished, live


def _head_logits(logits, bias):
    """The head's logits: decoder output + bias in the logits' dtype, as fp64."""
    return (logits if bias is None else logits + bias).double()


def _ranks(x):
    """rank[r, v]: position of word v in row r's order (logit descending, id ascending)."""
    order = torch.sort(x, dim=1, descending=True, stable=True).indices
    return torch.empty_like(order).scatter_(1, order, torch.arange(x.shape[1], device=x.device).expand_as(order)), order


def _mass_before(x):
    """Probability mass of the words ranked before each word."""
    ranks, order = _ranks(x)
    pr = torch.softmax(x, dim=1).gather(1, order)
    before = torch.cumsum(pr, 1) - pr
    return before.gather(1, ranks)


def _rand_logits(gen, rows, V, dtype, scale=2.0, quant=None):
    x = torch.randn(rows, V, generator=gen) * scale
    if quant:
        x = torch.round(x / quant) * quant                          # many exact ties, at the maximum too
    return x.to(DEV, dtype)


VOCABS = [1, 7, 31, 1000, 1023, 28996, 30522]


@pytest.mark.parametrize("V", VOCABS)
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_topk1_and_tiny_topp_are_first_argmax(V, dtype):
    gen = torch.Generator().manual_seed(V)
    for quant in (None, 0.5):
        logits = _rand_logits(gen, 300, V, dtype, quant=quant)
        bias = _rand_logits(gen, 1, V, dtype, scale=0.5, quant=quant)[0]
        want = torch.argmax(_head_logits(logits, bias), dim=1)          # first maximal index
        for seed in (0, 12345):
            assert torch.equal(_run(logits, "topk", k=1, bias=bias, seed=seed)[0], want)
            assert torch.equal(_run(logits, "topp", p=1e-9, bias=bias, seed=seed)[0], want)


@pytest.mark.parametrize("V", [37, 1000, 28996])
def test_draws_lie_in_the_top_k_set_and_nucleus(V):
    gen = torch.Generator().manual_seed(7 + V)
    logits = _rand_logits(gen, 512, V, torch.bfloat16, scale=3.0)
    bias = _rand_logits(gen, 1, V, torch.bfloat16, scale=0.5)[0]
    x = _head_logits(logits, bias)
    ranks, _ = _ranks(x)
    before = _mass_before(x)
    logp = torch.log_softmax(x, dim=1)
    for seed in (1, 2, 3):
        for k in (2, 8, 64):
            ids, sc, _, _ = _run(logits, "topk", k=k, bias=bias, seed=seed)
            assert int(ranks.gather(1, ids[:, None]).max()) < min(k, V)
            assert torch.allclose(sc.double(), logp.gather(1, ids[:, None])[:, 0], rtol=1e-4, atol=1e-4)
        for p in (0.3, 0.9, 1.0):
            ids, sc, _, _ = _run(logits, "topp", p=p, bias=bias, seed=seed)
            assert float(before.gather(1, ids[:, None]).max()) < p + 1e-5       # the mass ranked before a kept word is below p
            assert torch.allclose(sc.double(), logp.gather(1, ids[:, None])[:, 0], rtol=1e-4, atol=1e-4)


def _expected(x, mode, k, p):
    """Renormalised kept distribution of one row x [V] (fp64)."""
    ranks, _ = _ranks(x[None])
    ranks = ranks[0]
    pr = torch.softmax(x, 0)
    keep = ranks < k if mode == "topk" else _mass_before(x[None])[0] < p
    q = torch.where(keep, pr, torch.zeros_like(pr))
    return q / q.sum(), keep


@pytest.mark.parametrize("mode,k,p", [("topk", 2, 1.0), ("topk", 8, 1.0), ("topk", 64, 1.0), ("topp", 1, 0.5), ("topp", 1, 0.9),
                                      ("topp", 1, 1.0)])
def test_draws_follow_the_renormalised_distribution(mode, k, p):
    N, V = 1 << 16, 1000
    gen = torch.Generator().manual_seed(k * 100 + int(p * 10))
    row = torch.randn(V, generator=gen, dtype=torch.float64) * (1.0 if mode == "topk" else 2.0)
    logits = row.float().to(DEV).expand(N, V).contiguous()           # every row the same logits, its own uniform
    ids = _run(logits, mode, k=k, p=p, seed=2024)[0]
    q, keep = _expected(row.float().double().to(DEV), mode, k, p)
    counts = torch.bincount(ids, minlength=V).double()
    assert float(counts[~keep].sum()) == 0.0
    exp = q[keep] * N
    obs = counts[keep]
    small = exp < 5                                                   # pool the rare words into one bin
    if bool(small.any()):
        exp = torch.cat((exp[~small], exp[small].sum()[None]))
        obs = torch.cat((obs[~small], obs[small].sum()[None]))
    pval = stats.chisquare(obs.cpu().numpy(), exp.cpu().numpy() * (float(obs.sum()) / float(exp.sum()))).pvalue
    assert pval > ALPHA, f"chi-square p = {pval:.2e} over {len(exp)} bins"


def test_draws_depend_on_seed_frame_and_row_only():
    gen = torch.Generator().manual_seed(3)
    logits = _rand_logits(gen, 64, 28996, torch.bfloat16, scale=3.0)
    for mode in ("topk", "topp"):
        a = _run(logits, mode, k=64, p=0.9, seed=77, f=2)
        b = _run(logits, mode, k=64, p=0.9, seed=77, f=2)
        assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])    # bitwise, run to run
        c = _run(logits[:8].clone(), mode, k=64, p=0.9, seed=77, f=2)  # the same rows in a smaller batch
        assert torch.equal(a[0][:8], c[0]) and torch.equal(a[1][:8], c[1])
        assert not torch.equal(a[0], _run(logits, mode, k=64, p=0.9, seed=78, f=2)[0])
        assert not torch.equal(a[0], _run(logits, mode, k=64, p=0.9, seed=77, f=1)[0])


@pytest.mark.parametrize("n", [1, 2, 3])
@pytest.mark.parametrize("n_ignore", [0, 1])
def test_ngram_blocking_and_eos_block_compose(n, n_ignore):
    """topk = 1 under blocking is the arg-max of the logits with -10000 at beam._dup_ngram_candidates of the history; with a high
    logit on every candidate, top-k = 64 / top-p = 0.9 never draw one."""
    gen = torch.Generator().manual_seed(n * 10 + n_ignore)
    rows, V, T, f = 200, 1000, 40, 30
    hist = torch.randint(0, 6, (rows, T), generator=gen)
    hist[::3, :] = 5 - hist[::3, :] // 2
    ignore = [3] if n_ignore else []
    cands = [beam._dup_ngram_candidates(hist[r, :f].tolist(), n, set(ignore)) for r in range(rows)]
    assert sum(map(len, cands)) >= 5                                   # (an ignored word in the tail unblocks a row: few at n = 1)
    logits = _rand_logits(gen, rows, V, torch.bfloat16)
    boosted = logits.clone()
    for r, c in enumerate(cands):
        if c:
            boosted[r, c] += 20.0
    ign = torch.tensor(ignore, dtype=torch.int32, device=DEV) if ignore else None
    x = boosted.double()
    for r, c in enumerate(cands):
        if c:
            x[r, c] = (boosted[r, c].float() + -10000.0).double()
    want = torch.argmax(x, 1)
    ids = _run(boosted, "topk", k=1, f=f, T=T, seq=hist.to(DEV).clone(), ngram=n, ignore=ign)[0]
    assert torch.equal(ids, want)
    for mode in ("topk", "topp"):
        for seed in range(5):
            ids = _run(boosted, mode, k=64, p=0.9, seed=seed, f=f, T=T, seq=hist.to(DEV).clone(), ngram=n, ignore=ign)[0].cpu()
            assert not any(int(ids[r]) in c for r, c in enumerate(cands))
    # [EOS] below min_len: never drawn even when it is the arg-max
    eos_top = logits.clone()
    eos_top[:, EOS] = 50.0
    assert not bool((_run(eos_top, "topk", k=1, block_eos=True)[0] == EOS).any())
    assert bool((_run(eos_top, "topk", k=1)[0] == EOS).all())


def test_finished_rows_pad_and_live_count():
    gen = torch.Generator().manual_seed(5)
    rows, V, T = 64, 1000, 6
    logits = _rand_logits(gen, rows, V, torch.bfloat16)
    logits[::2, EOS] = 60.0                                           # even rows draw [EOS]
    seq = torch.full((rows, T), -1, dtype=torch.int64, device=DEV)
    ids, sc, fin, live = _run(logits, "topp", p=0.9, seq=seq, f=0, T=T)
    assert bool((ids[::2] == EOS).all()) and not bool((ids[1::2] == EOS).any())
    assert torch.equal(fin.cpu(), (torch.arange(rows) % 2 == 0).int()) and int(live) == rows // 2
    ids2, sc2, fin2, live2 = _run(logits, "topp", p=0.9, seq=seq, f=1, T=T, finished=fin, pad_id=0)
    assert bool((ids2[::2] == 0).all()) and bool((sc2[::2] == 0).all()) and bool((sc2[1::2] < 0).all())
    assert int(live2) == rows // 2 - int((ids2[1::2] == EOS).sum())


# ---------------------------------------------------------------------------------------------------------------------------------
# (2) the decode
# ---------------------------------------------------------------------------------------------------------------------------------
def _args(dims, B, seed=0):
    vis, pe, input_ids, tt, pos, mask = _inputs(dims, B, seed)
    return (vis.cuda().bfloat16(), pe.cuda().bfloat16(), input_ids.cuda(), tt.cuda(), pos.cuda(), mask.cuda())


def _pad_after_eos(ids):
    out = ids.clone()
    after = (torch.cumsum((ids == EOS).int(), 1) - (ids == EOS).int()) > 0
    out[after] = 0
    return out


@pytest.mark.parametrize("cache", [True, False])
def test_degenerate_sampling_decodes_equal_greedy(cache):
    dims = synth.SMALL_L123
    args = _args(dims, 8)
    model = _decoder(dims)
    model.use_kv_cache = cache
    greedy, _ = model(*args, task_idx=None, sample_mode="greedy")
    for method, kw in (("topk", dict(topk=1)), ("topp", dict(topp=1e-9))):
        model.sampling_method = method
        for k, v in kw.items():
            setattr(model, k, v)
        ids, scores = model(*args, task_idx=None, seed=11)
        assert torch.equal(ids, _pad_after_eos(greedy))
        assert bool((scores <= 0).all())
        model.sampling_method = "beam_search"


@pytest.mark.parametrize("n,min_len", [(1, 0), (2, 0), (3, 4)])
def test_blocked_top1_decode_equals_beam_size_one(n, min_len):
    dims = synth.SMALL_L123
    args = _args(dims, 8, seed=3)
    model = _decoder(dims, forbid_duplicate_ngrams=True, ngram_size=n, min_len=min_len)
    with torch.no_grad():
        vis, pe = model.project_regions(args[0], args[1])
        want = beam.beam_search(model, vis, pe, *args[2:], task_idx=None)["pred_seq"]
    T = args[3].shape[1] - args[2].shape[1]
    model.sampling_method, model.topk = "topk", 1
    ids, _ = model(*args, task_idx=None)
    assert torch.equal(ids, want[:, :T])
    model.forbid_duplicate_ngrams = False
    plain, _ = model(*args, task_idx=None)
    if n == 1:
        assert not torch.equal(plain, ids)                            # the greedy decode repeats words; the blocked one does not
    for r in range(ids.shape[0]):
        seq = [w for w in ids[r].tolist()]
        seq = seq[:seq.index(EOS) + 1] if EOS in seq else seq
        assert all(seq[t] not in beam._dup_ngram_candidates(seq[:t], n, set()) for t in range(len(seq)))


def test_all_finished_decode_stops_early_and_pads():
    dims = synth.SMALL_L123
    args = _args(dims, 8)
    model = _decoder(dims, sampling_method="topp", topp=0.9)
    with torch.no_grad():
        model.cls.predictions.bias[EOS] += 60.0                       # every row draws [EOS] at the first step
    ids, scores = model(*args, task_idx=None, seed=1)
    T = ids.shape[1]
    assert bool((ids[:, 0] == EOS).all()) and bool((ids[:, 1:] == 0).all()) and bool((scores[:, 1:] == 0).all())
    assert model.last_decode_steps < T, f"{model.last_decode_steps} of {T} steps ran"


def test_sampling_decode_is_reproducible_and_graph_capturable():
    dims = synth.SMALL_L123
    args = _args(dims, 8, seed=4)
    model = _decoder(dims, sampling_method="topk", topk=64, seed=9)
    a = model(*args, task_idx=None)
    b = model(*args, task_idx=None)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    assert not torch.equal(a[0], model(*args, task_idx=None, seed=10)[0])
    model.sampling_method, model.topp = "topp", 0.9
    eager = model(*args, task_idx=None)
    g = graph.GraphedCall(lambda *x: model(*x, task_idx=None), args)
    out = g(*args)
    assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
