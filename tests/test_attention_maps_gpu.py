"""GPU: attention maps (vlpk_attn_probs and output_attentions through BertLayer, BertEncoder, BertModel and the decoders).

Kernel level: every map is checked against fp64 softmax(QK^T / 8 + mask) of the kernel's own bf16 q and k, elementwise and per row
sum, inside a NaN guard band (tools/kernel_check.py): columns [Lkv, ld_p), rows outside [row0, Lq) and everything around the view
must stay bit-identical.  Bounds (the worst measured ratio is recorded in DESIGN.md §6):
  |P - P_ref| <= P_ref * PROB_REL_BOUND * (2^-16 |q_i| . |k_j| / 8 + ATTN_LSE (1 + |lse_i|) + 2^-10 [row fully masked] + 2^-21)
      the fp32 score (GEMM_A per unit of |q||k|), the forward's logsumexp (ATTN_LSE), and in a fully masked row the fp32 rounding
      of the -10000 offset (ulp 2^-10 at |s| ~ 1.4e4 in the log2 domain); PROB_REL_BOUND = 4, ceiling 8;
  |sum_j P_ij - 1| <= ROW_SUM_BOUND * ATTN_LSE (1 + |lse_i|), ROW_SUM_BOUND = 5 (ceiling 8): a row sums to 1 as closely as the forward's
      logsumexp is known; in a fully masked row (lse ~ -10000, held by fp32 to 2^-11) within DEAD_ROW_SUM = 2^-8 (ceiling 2^-7).
Model level: against tests/golden/attention_maps.pt (tools/attention_maps_oracle.py, the unmodified reference with forward hooks on
attention.self.dropout) at rel-L2 <= 3e-2 per layer, or 2x the reference's own fp32 -> bf16 drift where that is above 2.5e-2; the three
BertLayer paths agree; decode with K/V caches matches the re-projection path, beam maps gathered through the back pointers included;
GraphedCall replays and deterministic reruns are bitwise equal; and requesting maps leaves the loss, every gradient and every decoded
id bitwise unchanged."""
import itertools
import os

import pytest
import torch

from tools import abi_cases
from tools import attention_maps_oracle as amo
from tools import kernel_check as kc
from vlp_b200 import _lib as L
from vlp_b200 import beam, graph, ops, synth
from vlp_b200 import vlp_modules as vm

from test_parity_gpu import TOL_HID, make_config, rel

pytestmark = pytest.mark.gpu
DEV = "cuda"
BF = torch.bfloat16
F64 = torch.float64
PROB_REL_BOUND = 4.0
ROW_SUM_BOUND = 5.0
DEAD_ROW_SUM = 2.0 ** -8   # also the row-sum bound of the model-level maps, whose rows include fully masked ones
PATH_REL = 1e-2            # rel-L2 between two paths that compute the same map from bf16 projections of different GEMMs
WORST = {}
MASKS = ["all", "s2s", "bernoulli", "dead_row", "rows1", "beyond"]
KINDS = ["normal", "peaky", "common"]


def _note(k, v):
    WORST[k] = max(WORST.get(k, 0.0), v)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    path = os.environ.get("VLPK_ATTN_MAPS_REPORT")
    if path:
        import json
        with open(path, "w") as f:
            json.dump(dict(sorted(WORST.items())), f, indent=1)


def _mask(kind, B, Lq, Lkv, gen):
    """0/1 [B, rows, Lkv] mask (rows = 1 for "rows1") and, for "beyond", the extra bits past Lkv the kernels must ignore."""
    if kind == "all":
        m = torch.ones(B, Lq, Lkv, dtype=torch.long)
    elif kind == "s2s":
        m = abi_cases.s2s_mask(B, Lq, max(1, Lq - Lq // 5), "cpu") if Lq == Lkv else torch.tril(
            torch.ones(Lq, Lkv, dtype=torch.long), diagonal=Lkv - Lq).expand(B, Lq, Lkv).contiguous()
    elif kind == "bernoulli":
        m = (torch.rand(B, Lq, Lkv, generator=gen) < 0.5).long()
    elif kind == "dead_row":
        m = torch.ones(B, Lq, Lkv, dtype=torch.long)
        for b in range(B):
            m[b, (7 * b + 3) % Lq] = 0
    elif kind == "rows1":
        m = (torch.rand(B, 1, Lkv, generator=gen) < 0.7).long()
        m[:, 0, 0] = 1
    else:
        m = (torch.rand(B, Lq, Lkv, generator=gen) < 0.8).long()
    bits = ops.pack_mask(m.to(DEV), mode="zero_one")
    if kind == "beyond":
        S = ops.key_slots(Lkv)
        hi = torch.zeros(S // 32, dtype=torch.int64)
        for j in range(Lkv, S):
            hi[j // 32] |= 1 << (j % 32)
        bits = bits | torch.where(hi >= 2 ** 31, hi - 2 ** 32, hi).to(torch.int32).to(DEV)
    return bits


def _inputs(kind, B, L, width, gen):
    if kind == "normal":
        t = torch.randn(B, L, width, generator=gen)
    elif kind == "peaky":
        t = 3.0 * torch.randn(B, L, width, generator=gen)
    else:
        t = torch.randn(1, 1, width, generator=gen) + 0.1 * torch.randn(B, L, width, generator=gen)
    return t.to(DEV, BF)


def run_probs(B, heads, Lq, Lkv, mask, kind, row0=0, spare_rows=0, seed=0, odd_ld=False):
    """Forward attention (for the kernel's own lse), then vlpk_attn_probs into a guarded buffer; checked against fp64."""
    gen = torch.Generator().manual_seed(seed)
    H = heads * 64
    bits = _mask(mask, B, Lq, Lkv, gen)
    slots = ops.kv_slots(Lq, Lkv)
    if Lq == Lkv and not spare_rows:                 # encoder layout: q, k, v in place in the packed [B, L, 3H] projection
        qkv = _inputs(kind, B, Lq, 3 * H, gen)
        q, k = qkv[..., :H], qkv[..., H:2 * H]
        kv, ld_kv = qkv[..., H:], 3 * H
    else:                                            # decode layout: q [B, Lq, H], K|V cache [B, Lkv + spare, 2H]
        q = _inputs(kind, B, Lq, H, gen)
        cache = _inputs("peaky" if kind == "peaky" else "normal", B, Lkv + spare_rows, 2 * H, gen)
        k = cache[:, :Lkv, :H]
        kv, ld_kv = cache[:, :Lkv].contiguous(), 2 * H   # the forward kernel takes no sequence stride; its lse does not depend on it
    ctx = torch.empty(B * Lq, H, device=DEV, dtype=BF)
    lse = torch.empty(B, heads, Lq, device=DEV, dtype=torch.float32)
    L.call("vlpk_attn_core_fwd_wide", B, heads, Lq, Lkv, q.data_ptr(), q.stride(1), kv.data_ptr(), kv[..., H:].data_ptr(), ld_kv,
           bits.data_ptr(), bits.shape[1], ctx.data_ptr(), H, lse.data_ptr(), None, 0, slots, L.stream())
    rows = Lq - row0
    ld = Lkv + (3 if odd_ld else 8)
    P = kc.guarded(B * heads * rows, Lkv, ld=ld, dtype=torch.float32, extra_rows=2)
    out = P.as_strided((B, heads, rows, Lkv), (heads * rows * ld, rows * ld, ld, 1))
    ops.attn_probs(q, k, lse, bits, row0, out)
    torch.cuda.synchronize()
    kc.assert_guard_intact(P, f"probs B{B} h{heads} Lq{Lq} Lkv{Lkv} {mask} row0={row0}")
    got = out.double()
    qh = q.unflatten(2, (heads, 64)).permute(0, 2, 1, 3).to(F64)
    kh = k.unflatten(2, (heads, 64)).permute(0, 2, 1, 3).to(F64)
    allow = kc.bits_to_allow(bits, Lq, Lkv)
    s = qh @ kh.transpose(-1, -2) / 8.0 + (~allow[:, None]).to(F64) * -10000.0
    ref = torch.softmax(s, -1)[:, :, row0:]
    E = (qh.abs() @ kh.abs().transpose(-1, -2) / 8.0)[:, :, row0:]
    lse_ref = torch.logsumexp(s, -1)[:, :, row0:]
    dead = (~allow).all(-1)[:, None, row0:, None].to(F64)
    bound = ref * PROB_REL_BOUND * (2.0 ** -16 * E + kc.ATTN_LSE * (1 + lse_ref.abs().unsqueeze(-1)) + dead * 2.0 ** -10 + 2.0 ** -21) \
        + 2.0 ** -120                                # below fp32's normal range ex2.approx.ftz flushes to 0
    err = (got - ref).abs()
    assert torch.isfinite(got).all()
    ratio = float((err / (bound + 1e-300)).max())
    _note("elementwise / bound", ratio / PROB_REL_BOUND)
    if ratio > 1.0:
        i = (err - bound).flatten().argmax()
        raise AssertionError(f"probs Lq{Lq} Lkv{Lkv} {mask} {kind}: |err| {float(err.flatten()[i]):.3e} > bound {float(bound.flatten()[i]):.3e}")
    rs_err = (got.sum(-1) - 1).abs()
    rs_bound = torch.where(dead[..., 0] > 0, torch.full_like(rs_err, DEAD_ROW_SUM), ROW_SUM_BOUND * kc.ATTN_LSE * (1 + lse_ref.abs()))
    rs = float((rs_err / rs_bound).max())
    _note("row sum / bound", rs)
    assert rs <= 1.0, f"row sums off by {rs:.3f} x their bound"
    return got, ref


LS = list(range(1, 129)) + [129, 143, 256, 257, 511, 512]


@pytest.mark.parametrize("L_", LS)
def test_probs_lengths(L_):
    i = LS.index(L_)
    run_probs(2, 1 if i % 2 else 12, L_, L_, MASKS[i % 6], KINDS[i % 3], seed=i, odd_ld=bool(i % 3 == 1))


@pytest.mark.parametrize("mask", MASKS)
@pytest.mark.parametrize("heads", [1, 12])
@pytest.mark.parametrize("L_", [64, 123, 128, 143, 256, 512])
def test_probs_masks_and_heads(L_, heads, mask):
    got, ref = run_probs(2, heads, L_, L_, mask, KINDS[(L_ + heads) % 3], seed=L_ * 7 + heads)
    if mask == "dead_row":     # the -10000 offset shifts every score of the row equally: the row is the unmasked softmax, not 0 or NaN
        r = 3
        assert float((got[0, :, r].sum(-1) - 1).abs().max()) < DEAD_ROW_SUM and float(got[0, :, r].min()) > 0.0


@pytest.mark.parametrize("Lq,Lkv,spare", [(1, 1, 0), (1, 128, 5), (2, 104, 19), (2, 123, 0), (5, 128, 0), (64, 128, 7), (2, 143, 3),
                                          (2, 300, 12), (1, 512, 0)])
@pytest.mark.parametrize("mask", ["bernoulli", "rows1", "beyond", "s2s"])
def test_probs_decode_shapes(Lq, Lkv, spare, mask):
    run_probs(3, 2, Lq, Lkv, mask, "normal" if Lq != 5 else "peaky", row0=Lq - 1, spare_rows=spare, seed=Lq * 1000 + Lkv, odd_ld=True)


@pytest.mark.parametrize("Lq,row0", [(123, 0), (123, 122), (123, 64), (143, 130), (256, 1), (512, 384), (103, 102)])
def test_probs_row_ranges(Lq, row0):
    full, _ = run_probs(2, 2, Lq, Lq, "s2s", "normal", seed=Lq + 1)
    part, _ = run_probs(2, 2, Lq, Lq, "s2s", "normal", row0=row0, seed=Lq + 1)
    assert torch.equal(full[:, :, row0:], part)


def test_probs_production_size():
    run_probs(64, 12, 123, 123, "s2s", "normal", seed=5)


# ---- model level ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gold(golden_dir):
    return torch.load(os.path.join(golden_dir, "attention_maps.pt"))


def _pretrain_model(dims, drop=0.0):
    model = vm.BertForPreTrainingLossMask(make_config(dims, drop), enable_butd=True, len_vis_input=dims.regions)
    model.load_state_dict(synth.make_state_dict(dims, 0), strict=False)
    return model.cuda().bfloat16()


def _encoder_maps(model, batch, **kw):
    b = {k: v.cuda() for k, v in batch.items()}
    vis, pe = model.project_regions(b["img"].bfloat16(), b["vis_pe"].bfloat16())
    return model.bert(vis, pe, b["input_ids"], b["segment_ids"], b["input_mask"], output_all_encoded_layers=False,
                      len_vis_input=model.len_vis_input, output_attentions=True, **kw)


def _bound(drift):
    return TOL_HID if drift <= 2.5e-2 else 2 * drift


@pytest.mark.parametrize("name", list(amo.ENCODER_CASES))
@pytest.mark.parametrize("layers_per_call", [None, 1])
def test_encoder_maps_match_reference(gold, name, layers_per_call):
    g = gold["encoder"][name]
    dims, _, batch = amo.encoder_inputs(name)
    model = _pretrain_model(dims).eval()
    model.bert.encoder.layers_per_call = layers_per_call
    with torch.no_grad():
        seq, pooled, att = _encoder_maps(model, batch)
    assert len(att) == dims.layers
    rows = g["rows"].to(DEV)
    for l, (m, ref) in enumerate(zip(att, g["maps"])):
        assert m.dtype == torch.float32 and m.shape == (g["B"], dims.heads, g["L"], g["L"]) and not m.requires_grad
        got = m.gather(2, rows.unsqueeze(-1).expand(*rows.shape, g["L"]))
        r = rel(got, ref)
        _note(f"golden {name} rel-L2", r)
        assert r <= _bound(g["drift"][l]), f"{name} layer {l}: rel-L2 {r:.3e}"
        assert float((got.sum(-1) - 1).abs().max()) < DEAD_ROW_SUM
    if name == "bernoulli":       # the fully masked rows: the softmax of the unmasked scores, as the reference's additive mask gives
        for b, r in enumerate(amo.DEAD_ROW):
            assert float(att[0][b, :, r].min()) > 0.0


def test_maps_in_train_mode_leave_the_step_bitwise_unchanged(monkeypatch):
    dims = synth.SMALL_L123
    batch = synth.make_batch(dims, 3, seed=11, mode="mix", ragged=True)
    model = _pretrain_model(dims, drop=0.1).train()
    b = {k: v.cuda() for k, v in batch.items()}

    def step(maps):
        monkeypatch.setattr(ops, "_seed_counter", itertools.count(1))
        model.zero_grad(set_to_none=True)
        vis, pe = model.project_regions(b["img"].bfloat16(), b["vis_pe"].bfloat16())
        out = model.bert(vis, pe, b["input_ids"], b["segment_ids"], b["input_mask"], output_all_encoded_layers=True,
                         len_vis_input=dims.regions, output_attentions=maps)
        loss = sum((x.float() * (i + 1)).square().mean() for i, x in enumerate(out[0])) + out[1].float().sum()
        loss.backward()
        return loss.detach(), {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}, (out[2] if maps else None)

    l0, g0, _ = step(False)
    l1, g1, att = step(True)
    assert torch.equal(l0, l1)
    assert g0.keys() == g1.keys() and all(torch.equal(g0[k], g1[k]) for k in g0)
    for m in att:   # pre-dropout probabilities: rows sum to 1 although the step ran with attention dropout
        assert float((m.sum(-1) - 1).abs().max()) < ROW_SUM_BOUND


def test_maps_are_bitwise_reproducible_in_deterministic_mode():
    dims = synth.SMALL_L123
    batch = synth.make_batch(dims, 2, seed=12, mode="s2s")
    model = _pretrain_model(dims).eval()
    before = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        with torch.no_grad():
            a = _encoder_maps(model, batch)[2]
            b = _encoder_maps(model, batch)[2]
    finally:
        torch.use_deterministic_algorithms(before)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_the_three_layer_paths_agree():
    dims = synth.SMALL_L123
    model = _pretrain_model(dims).eval()
    layer = model.bert.encoder.layer[0]
    B, Lq, H, p = 2, 123, dims.hidden, 101
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(B, Lq, H, generator=gen).to(DEV, BF)
    m = abi_cases.s2s_mask(B, Lq, p, "cpu")
    ext = (1.0 - m[:, None].to(DEV, BF)) * -10000.0
    with torch.no_grad():
        y, plain = layer(x, ext, output_attentions=True)
        y2, hist = layer(x[:, p:], ext[:, :, p:], history_states=x[:, :p], output_attentions=True)
        cache = torch.empty(B, Lq + 4, 2 * H, device=DEV, dtype=BF)
        layer(x[:, :p], ext[:, :, :p, :p], kv_cache=cache, cache_pos=0)
        y3, cached = layer(x[:, p:], ext[:, :, p:], kv_cache=cache, cache_pos=p, output_attentions=True)
        y4, rows = layer(x[:, p:], ext[:, :, p:], history_states=x[:, :p], output_attentions=(Lq - p - 1, None))
    assert plain.shape == (B, dims.heads, Lq, Lq) and hist.shape == cached.shape == (B, dims.heads, Lq - p, Lq)
    for nm, got in (("history", hist), ("kv_cache", cached)):
        r = rel(got, plain[:, :, p:])
        _note(f"path {nm} rel-L2", r)
        assert r <= PATH_REL, f"{nm}: {r:.3e}"
    assert torch.equal(rows, hist[:, :, -1:])


# ---- decode -----------------------------------------------------------------------------------------------------------------------
def _decoder(K=1, **kw):
    dims = synth.SMALL_L123
    model = vm.BertForSeq2SeqDecoder(make_config(dims), mask_word_id=103, eos_id=amo.EOS_ID, search_beam_size=K, enable_butd=True,
                                     len_vis_input=dims.regions, **kw)
    model.load_state_dict(synth.make_state_dict(dims, 0), strict=False)
    return model.cuda().bfloat16().eval()


def _dargs(B, seed):
    vis, pe, ids, tt, pos, mask = amo.decode_inputs(B, seed)[2]
    return (vis.cuda().bfloat16(), pe.cuda().bfloat16(), ids.cuda(), tt.cuda(), pos.cuda(), mask.cuda())


def _check_decode_maps(att, ids_len, in_len, out_len):
    """zero beyond the keys each frame could see; every run frame's rows sum to 1"""
    T = att.shape[1]
    for t in range(T):
        if in_len + t + 1 < out_len:
            assert float(att[:, t, ..., in_len + t + 1:].abs().max()) == 0.0
    if ids_len:
        assert float((att[:, :ids_len].sum(-1) - 1).abs().max()) < DEAD_ROW_SUM


def test_greedy_maps_cache_reprojection_reference(gold):
    g = gold["greedy"]
    model = _decoder()
    args = _dargs(g["B"], g["seed"])
    ids0, sc0 = model(*args, task_idx=None)
    ids, sc, att = model(*args, task_idx=None, output_attentions=True)
    assert torch.equal(ids0, ids) and torch.equal(sc0, sc)
    dims = synth.SMALL_L123
    in_len, out_len = dims.regions + 2, dims.seq_len
    assert att.shape == (g["B"], out_len - in_len, dims.layers, dims.heads, out_len)
    _check_decode_maps(att, ids.shape[1], in_len, out_len)
    model.use_kv_cache = False
    ids_r, _, att_r = model(*args, task_idx=None, output_attentions=True)
    assert torch.equal(ids, ids_r)
    r = rel(att, att_r)
    _note("greedy cache vs reprojection rel-L2", r)
    assert r <= PATH_REL
    n = ids.shape[1]
    d = (ids.cpu() != g["ids"]).nonzero()
    if d.numel():
        n = int(d[:, 1].min())                   # a flipped word (test_decode_gpu explains those) changes every later prefix
    assert n >= 1
    r = rel(att[:, :n], g["maps"][:, :n])
    _note("greedy golden rel-L2", r)
    assert r <= TOL_HID, f"greedy maps vs reference: {r:.3e}"


@pytest.mark.parametrize("cache", [True, False])
def test_beam_maps_follow_the_back_pointers(gold, cache):
    g = gold["beam"]
    model = _decoder(K=g["K"], length_penalty=g["length_penalty"])
    model.use_kv_cache = cache
    args = _dargs(g["B"], g["seed"])
    plain = model(*args, task_idx=None)
    out = model(*args, task_idx=None, output_attentions=True)
    for k in ("pred_seq", "scores", "wids", "ptrs"):
        assert torch.equal(plain[k], out[k]), k
    att = out["attentions"]
    T = att.shape[1]
    if torch.equal(out["pred_seq"].cpu(), g["pred_seq"]):
        r = rel(att, g["chosen"])
    else:
        # a near-tie decided differently (test_decode_gpu explains those): up to the first frame whose words or pointers differ every
        # hypothesis has the reference's history, so frame t of OUR chosen hypothesis is row rows[t] of the reference's step t
        K = g["K"]
        wi, pt = out["wids"][:, :T].cpu(), out["ptrs"][:, :T].cpu()
        d = ((wi != g["wids"][:, :T]) | (pt != g["ptrs"][:, :T])).any(-1).any(0).nonzero()
        n = int(d[0, 0]) if d.numel() else T
        assert n >= 1
        active, pos = beam.best_path(out["scores"][:, :T].permute(1, 0, 2).float().cpu(), wi.permute(1, 0, 2), pt.permute(1, 0, 2),
                                     amo.EOS_ID, g["length_penalty"])
        rows = pt.permute(1, 0, 2).gather(2, pos.unsqueeze(-1)).squeeze(-1)[:n, 0]
        ref = torch.stack([g["step_maps"][t, int(rows[t])] * active[t, 0] for t in range(n)])
        r = rel(att[0, :n], ref)
    _note("beam golden rel-L2", r)
    assert r <= TOL_HID, f"beam maps vs reference: {r:.3e}"
    if cache:
        model.use_kv_cache = False
        att_r = model(*args, task_idx=None, output_attentions=True)["attentions"]
        assert rel(att, att_r) <= PATH_REL


def test_graphed_decodes_with_maps_replay_the_python_driven_decode():
    for K in (1, 3):
        model = _decoder(K=K)
        a0, a1 = _dargs(2, 5), _dargs(2, 6)
        gc = graph.GraphedCall(lambda *a: model(*a, task_idx=None, output_attentions=True), a0)
        for a in (a0, a1):
            ref = model(*a, task_idx=None, output_attentions=True)
            got = gc(*a)
            if K == 1:
                assert all(torch.equal(x, y) for x, y in zip(got, ref))
            else:
                assert all(torch.equal(got[k], ref[k]) for k in ref)


@pytest.mark.parametrize("method", ["topk", "topp"])
def test_sampling_maps(method):
    model = _decoder(sampling_method=method, topk=5, topp=0.9, seed=3)
    args = _dargs(2, 7)
    ids0, sc0 = model(*args, task_idx=None)
    ids, sc, att = model(*args, task_idx=None, output_attentions=True)
    assert torch.equal(ids0, ids) and torch.equal(sc0, sc)
    steps = model.last_decode_steps
    if steps < att.shape[1]:
        assert float(att[:, steps:].abs().max()) == 0.0
    dims = synth.SMALL_L123
    _check_decode_maps(att, steps, dims.regions + 2, dims.seq_len)
