"""GPU: several captions per image over one K/V cache of the image prefix (`num_return_sequences` N > 1).
 (1) the kernel: vlpk_layer_cached_group_fwd is bitwise vlpk_layer_cached_fwd on each hypothesis' materialised contiguous cache — the
     layer output and the appended K|V rows — for groups, prefixes, positions and key counts on both sides of 128 (up to 512), with
     slot tables from random back-pointer chains and three kinds of masks; the prefix and the text rows it must not write stay
     bitwise unchanged inside NaN guard bands;
 (2) beam search: the traces and pred_seq are bitwise those of the N = 1 decode, and every n-best row is the back-track of its
     candidate under the final-selection rule (n-gram blocking with an ignore set, min_len, length penalties, a relaxed head with
     per-sample task_idx, an output long enough for the tiled kernel);
 (3) sampling: ids and scores are bitwise today's sampler on the batch repeated with repeat_interleave(N);
 (4) GraphedCall replays equal the Python-driven decodes."""
import dataclasses
import random

import pytest
import torch

from tools import abi_cases
from tools import relax_projection_oracle as RPO
from vlp_b200 import graph, ops, synth
from vlp_b200 import vlp_modules as vm

from test_decode_gpu import _inputs
from test_nbest_cpu import _plain_nbest
from test_parity_gpu import make_config

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
EOS = 102
PAD = 64                       # guard band, elements (a multiple of 8 keeps the 16-byte alignment)


# ---------------------------------------------------------------------------------------------------------------------------------
# (1) the kernel
# ---------------------------------------------------------------------------------------------------------------------------------
def _banded(n, gen):
    """A random bf16 tensor of n elements inside NaN guard bands: (the whole buffer, the inner view)."""
    buf = torch.full((n + 2 * PAD,), float("nan"), device=DEV, dtype=BF)
    buf[PAD:PAD + n] = torch.randn(n, generator=gen, device=DEV).to(BF)
    return buf, buf[PAD:PAD + n]


def _chain_slots(BG, G, T, pos, rnd):
    """A slot table after `pos` beam reorders with random parents inside each image's group (SharedPrefixCache.reorder)."""
    own = (torch.arange(BG, dtype=torch.int32) * T).unsqueeze(1) + torch.arange(T, dtype=torch.int32)
    slots = own.clone()
    for f in range(pos):
        parent = torch.tensor([i // G * G + rnd.randrange(G) for i in range(BG)])
        slots[:, f] = own[:, f]
        slots = slots.index_select(0, parent)
    return slots


def _mask(kind, images, Lq, P, pos, gen):
    Lkv = P + pos + Lq
    m = torch.zeros(images, Lq, Lkv, dtype=torch.long)
    m[:, :, :P] = 1
    for q in range(Lq):
        m[:, q, P:P + pos + q + 1] = 1                          # the decode's s2s rows: every earlier word and itself
    if kind == "zeroed_prefix":
        m[:, :, torch.randperm(P, generator=gen)[:max(1, P // 3)]] = 0
    elif kind == "bernoulli":
        m = (torch.rand(images, Lq, Lkv, generator=gen) < 0.6).long()
    return m.to(DEV)


def _kernel_case(images, G, P, pos, Lq, H, heads, kind, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    cgen = torch.Generator().manual_seed(seed)
    rnd = random.Random(seed)
    I = 4 * H
    BG, T = images * G, pos + Lq + 2
    Lkv = P + pos + Lq
    params = abi_cases.layer_params(cgen, DEV, H, I)
    pre_buf, prefix = _banded(images * (P + 3) * 2 * H, gen)
    prefix = prefix.view(images, P + 3, 2 * H)
    txt_buf, text = _banded(BG * T * 2 * H, gen)
    text = text.view(BG, T, 2 * H)
    text[:, pos:pos + Lq] = float("nan")                         # rows the call must write
    slots = _chain_slots(BG, G, T, pos, rnd).to(DEV)
    x = torch.randn(BG, Lq, H, generator=gen, device=DEV).to(BF)
    m = _mask(kind, images, Lq, P, pos, cgen)
    bits = ops.pack_mask((1 - m) * -10000.0, "additive")
    # the contiguous caches today's decode would hold: prefix rows, then the slot rows, then room for the new rows (NaN past Lkv)
    cache = torch.full((BG, Lkv + 5, 2 * H), float("nan"), device=DEV, dtype=BF)
    cache[:, :P] = prefix[torch.arange(BG, device=DEV) // G, :P]
    if pos:
        cache[:, P:P + pos] = text.reshape(BG * T, 2 * H)[slots[:, :pos].long()]
    pre0, txt0 = pre_buf.clone(), txt_buf.clone()
    want = ops.layer_cached_fwd(x, cache, P + pos, bits.repeat_interleave(G, 0), heads, I, params)
    got = ops.layer_cached_group_fwd(x, prefix, P, text, slots, G, pos, bits, heads, I, params)
    torch.cuda.synchronize()
    assert torch.equal(got, want)
    assert torch.equal(text[:, pos:pos + Lq], cache[:, P + pos:P + pos + Lq])
    same = torch.ones(T, dtype=torch.bool)
    same[pos:pos + Lq] = False
    inner = txt_buf[PAD:-PAD].view(BG, T, 2 * H)
    assert torch.equal(inner[:, same].view(torch.int16), txt0[PAD:-PAD].view(BG, T, 2 * H)[:, same].view(torch.int16))
    assert torch.equal(pre_buf.view(torch.int16), pre0.view(torch.int16))     # prefix and its bands
    assert bool(txt_buf[:PAD].isnan().all()) and bool(txt_buf[-PAD:].isnan().all())


def _kernel_cases():
    rnd = random.Random(1)
    cases = []
    for G in (1, 2, 3, 5, 8):
        for images in (1, 3, 37):
            for P in (1, 7, 102):
                pos, Lq = rnd.choice((0, 1, 5, 20)), rnd.choice((1, 2))
                cases.append((images, G, P, pos, Lq, 128, 2, rnd.choice(("s2s", "zeroed_prefix", "bernoulli"))))
    # BERT-base heads, and key counts on both sides of 128 and up to 512 (the tiled kernel, tiles with and without a prefix box)
    cases += [(3, 5, 102, 20, 2, 768, 12, "s2s"), (2, 3, 102, 24, 2, 768, 12, "s2s"), (2, 3, 102, 25, 2, 768, 12, "zeroed_prefix"),
              (2, 2, 126, 0, 2, 128, 2, "s2s"), (2, 2, 126, 1, 2, 128, 2, "bernoulli"), (1, 3, 102, 300, 2, 128, 2, "s2s"),
              (3, 2, 200, 100, 1, 128, 2, "bernoulli"), (2, 5, 1, 509, 2, 128, 2, "s2s"), (2, 2, 400, 110, 2, 768, 12, "zeroed_prefix")]
    return cases


@pytest.mark.parametrize("case", _kernel_cases(), ids=lambda c: "img{}-G{}-P{}-pos{}-Lq{}-H{}-{}".format(*c[:6], c[7]))
def test_group_layer_is_bitwise_the_contiguous_cache_layer(case):
    _kernel_case(*case, seed=sum(v * 31 ** i for i, v in enumerate(case[:6])) % 65521)


# ---------------------------------------------------------------------------------------------------------------------------------
# (2) beam search, (3) sampling, (4) graphs
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


LONG = dataclasses.replace(synth.SMALL_L123, text=60)          # 102 + 60 + ... rows: the tiled kernel from frame ~26 on
BEAM_CASES = [dict(K=K, N=N) for K in (2, 3, 5) for N in sorted({2, K})] + [
    dict(K=3, N=3, forbid_duplicate_ngrams=True, ngram_size=2, forbid_ignore_set={7, 11}, min_len=4, length_penalty=0.5),
    dict(K=4, N=2, length_penalty=-1.0, min_len=2),
    dict(K=3, N=2, relax=4),
    dict(K=3, N=3, dims="long", length_penalty=0.5)]


@pytest.mark.parametrize("case", BEAM_CASES, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_beam_nbest(case):
    case = dict(case)
    K, N = case.pop("K"), case.pop("N")
    dims = LONG if case.pop("dims", None) == "long" else synth.SMALL_L123
    relax = case.pop("relax", 0)
    B = 5
    args = _args(dims, B, seed=K + N)
    task_idx = torch.tensor([0, 3, 1, 2, 3], device=DEV) if relax else None
    model = _decoder(dims, relax=relax, search_beam_size=K, **case)
    one = model(*args, task_idx=task_idx)
    model.num_return_sequences = N
    tr = model(*args, task_idx=task_idx)
    for k in ("scores", "wids", "ptrs", "pred_seq"):
        assert torch.equal(tr[k], one[k]), k
    out_len = args[3].shape[1]
    T = out_len - args[2].shape[1]
    sc, wi, pt = (tr[k][:, :T].permute(1, 0, 2).cpu() for k in ("scores", "wids", "ptrs"))
    want_seq, want_val = _plain_nbest(sc, wi, pt, EOS, model.length_penalty, N, out_len)
    assert torch.equal(tr["nbest_seq"].cpu(), want_seq)
    assert torch.equal(tr["nbest_scores"].cpu(), want_val)
    assert torch.equal(tr["nbest_seq"][:, 0], tr["pred_seq"])


SAMPLE_CASES = [dict(sampling_method=m, N=N, **kw) for m, kw in (("topk", dict(topk=8)), ("topp", dict(topp=0.9))) for N in (2, 5)] + [
    dict(sampling_method="topk", topk=16, N=3, forbid_duplicate_ngrams=True, ngram_size=2, forbid_ignore_set={7}, min_len=5),
    dict(sampling_method="topp", topp=0.95, N=2, dims="long")]


@pytest.mark.parametrize("case", SAMPLE_CASES, ids=lambda c: "-".join(f"{k}={v}" for k, v in c.items()))
def test_sampling_equals_the_repeated_batch(case):
    case = dict(case)
    N = case.pop("N")
    dims = LONG if case.pop("dims", None) == "long" else synth.SMALL_L123
    B = 6
    args = _args(dims, B, seed=N)
    model = _decoder(dims, seed=17, **case)
    rep = tuple(a.repeat_interleave(N, 0) for a in args)
    ids1, sc1 = model(*rep, task_idx=None)
    model.num_return_sequences = N
    ids, sc = model(*args, task_idx=None)
    assert ids.shape == (B, N, ids1.shape[1])
    assert torch.equal(ids.reshape(B * N, -1), ids1) and torch.equal(sc.reshape(B * N, -1), sc1)


def test_sampling_early_stop_equals_the_repeated_batch():
    dims = synth.SMALL_L123
    B, N = 4, 3
    args = _args(dims, B, seed=2)
    model = _decoder(dims, sampling_method="topk", topk=4, seed=3)
    model.cls.predictions.bias.data[EOS] = 30.0                   # every row draws [EOS] at once: the loop stops early
    rep = tuple(a.repeat_interleave(N, 0) for a in args)
    ids1, sc1 = model(*rep, task_idx=None)
    steps1 = model.last_decode_steps
    model.num_return_sequences = N
    ids, sc = model(*args, task_idx=None)
    assert model.last_decode_steps == steps1 < ids.shape[-1]
    assert torch.equal(ids.reshape(B * N, -1), ids1) and torch.equal(sc.reshape(B * N, -1), sc1)


def test_samples_of_an_image_differ():
    dims = synth.SMALL_L123
    model = _decoder(dims, sampling_method="topk", topk=64, seed=5, num_return_sequences=5)
    ids, _ = model(*_args(dims, 4, seed=1), task_idx=None)
    for b in range(ids.shape[0]):
        assert any(not torch.equal(ids[b, 0], ids[b, j]) for j in range(1, 5)), b


@pytest.mark.parametrize("kw", [dict(search_beam_size=3, num_return_sequences=3),
                                dict(sampling_method="topk", topk=8, num_return_sequences=4)],
                         ids=["beam", "topk"])
def test_graphed_call_equals_the_python_driven_decode(kw):
    dims = synth.SMALL_L123
    args = _args(dims, 4, seed=6)
    model = _decoder(dims, seed=21, **kw)
    eager = model(*args, task_idx=None)
    g = graph.GraphedCall(lambda *x: model(*x, task_idx=None), args)
    out = g(*args)
    if isinstance(eager, dict):
        assert set(out) == set(eager)
        for k in eager:
            assert torch.equal(out[k], eager[k]), k
    else:
        assert torch.equal(out[0], eager[0]) and torch.equal(out[1], eager[1])
