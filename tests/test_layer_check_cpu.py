"""The stage references of tools/layer_check.py are right and the stage checks bite, on the CPU.

The references chained in fp64 agree with torch autograd through the oracle's bert_layer (float64, the same keep-masks), so the
suite does not encode the same mistake as the kernels (dz2 versus dt2 as LN2's residual gradient, a dropout scale, a transposed
operand).  The stage checks reject defects of the composite entry points that the model-level criterion (rel-L2 <= 5e-2 and cosine
>= 0.999 per parameter gradient) lets through, and the GPU module's call sequences marshal against the C prototypes."""
import ctypes as C

import pytest
import torch

from oracle import vlp_oracle as O
from tools import abi_cases
from tools import kernel_check as kc
from tools import layer_check as lc
from vlp_b200 import _lib as L

F64 = torch.float64
BF = torch.bfloat16
ORACLE_NAMES = ["attention.self.query.weight", "attention.self.key.weight", "attention.self.value.weight", "attention.self.query.bias",
                "attention.self.key.bias", "attention.self.value.bias", "attention.output.dense.weight", "attention.output.dense.bias",
                "attention.output.LayerNorm.weight", "attention.output.LayerNorm.bias", "intermediate.dense.weight", "intermediate.dense.bias",
                "output.dense.weight", "output.dense.bias", "output.LayerNorm.weight", "output.LayerNorm.bias"]


def _model_level_passes(got, ref):
    """The model-level parity criterion of one parameter gradient: rel-L2 <= 5e-2 and cosine >= 0.999."""
    g, r = got.to(F64).flatten(), ref.to(F64).flatten()
    return float((g - r).norm() / r.norm()) <= 5e-2 and float(g @ r / (g.norm() * r.norm())) >= 0.999


def _case(B, Lq, H, I, p, seed, n_src):
    gen = torch.Generator().manual_seed(seed)
    heads = H // 64
    w = lc.weights([t.to(F64) for t in abi_cases.layer_params(gen, "cpu", H, I)])
    x = torch.randn(B * Lq, H, generator=gen, dtype=F64)
    dy = torch.randn(B * Lq, H, generator=gen, dtype=F64) * 0.1
    allow = abi_cases.s2s_mask(B, Lq, n_src, "cpu").bool()
    keep = {}
    if p > 0:
        keep = {"attn": (torch.rand(B, heads, Lq, Lq, generator=gen) >= p).to(torch.uint8),
                "hid1": (torch.rand(B * Lq, H, generator=gen) >= p).to(torch.uint8),
                "hid2": (torch.rand(B * Lq, H, generator=gen) >= p).to(torch.uint8)}
    prior = {n: torch.randn(s, generator=gen, dtype=F64) for n, s in lc.grad_shapes(H, I).items()}
    return dict(B=B, Lq=Lq, H=H, I=I, heads=heads, p=p, w=w, x=x, dy=dy, allow=allow, keep=keep, prior=prior)


@pytest.mark.parametrize("p", [0.1, 0.0])
def test_stage_references_match_autograd_through_oracle_layer(p):
    c = _case(2, 9, 128, 512, p, 3, 6)
    B, Lq, H, heads = c["B"], c["Lq"], c["H"], c["heads"]
    A, S, G = lc.reference_layer(c["w"], c["x"], c["allow"], c["keep"], p, B, Lq, heads, c["dy"], c["prior"])
    pre = "bert.encoder.layer.0."
    sd = {pre + n: c["w"][f].clone().requires_grad_(True) for n, f in zip(ORACLE_NAMES, L.WEIGHT_FIELDS)}
    x = c["x"].view(B, Lq, H).clone().requires_grad_(True)
    ext = (1.0 - c["allow"][:, None].to(F64)) * -10000.0
    sites = {("attn", 0): c["keep"].get("attn"), ("hid1", 0): c["keep"].get("hid1"), ("hid2", 0): c["keep"].get("hid2")}
    O.MASK_PROVIDER = lambda site, shape: None if sites.get(site) is None else sites[site].view(shape)
    try:
        y = O.bert_layer(sd, 0, x, ext, heads, p_hidden=p, p_attn=p, training=True)
    finally:
        O.MASK_PROVIDER = None
    y.backward(c["dy"].view(B, Lq, H))
    close = dict(rtol=1e-9, atol=1e-11)
    torch.testing.assert_close(A["y"], y.detach().view(B * Lq, H), **close)
    torch.testing.assert_close(S["dx"], x.grad.view(B * Lq, H), **close)
    g = {f: sd[pre + n].grad for n, f in zip(ORACLE_NAMES, L.WEIGHT_FIELDS)}
    auto = {"wqkv": torch.cat((g["wq"], g["wk"], g["wv"])), "bqkv": torch.cat((g["bq"], g["bk"], g["bv"])), "wo": g["wo"], "bo": g["bo"],
            "ln1_g": g["ln1_g"], "ln1_b": g["ln1_b"], "w1": g["w1"], "b1": g["b1"], "w2": g["w2"], "b2": g["b2"], "ln2_g": g["ln2_g"],
            "ln2_b": g["ln2_b"]}
    for n in L.GRAD_FIELDS:
        torch.testing.assert_close(G[n] - c["prior"][n], auto[n], **close, msg=lambda m: f"d{n}: {m}")


def test_rejects_wgrad_tile_missing_one_of_six_k_slices():
    """dWo [768, 768] over 7 872 tokens split six ways: one 128 x 128 tile without one slice is ~1/6 off in 1 of 36 tiles, about
    0.03 globally.  The upstream gradient is correlated with the layer input, as a training gradient is, so that the six slices add
    up coherently."""
    gen = torch.Generator().manual_seed(5)
    M, H = 7872, 768
    ctx = torch.randn(M, H, generator=gen).to(BF)
    dt1 = (ctx.float() @ (torch.randn(H, H, generator=gen) * H ** -0.5) + 0.5 * torch.randn(M, H, generator=gen)).to(BF)
    prior = torch.randn(H, H, generator=gen)
    G = {"wo": ("gemm", *lc.ref_wgrad(dt1, ctx, prior))}
    good = prior + dt1.float().t() @ ctx.float()
    lc.check_arena("layer 2", {"wo": good}, G, lc.Worst())
    bad = good.clone()
    ks = slice(3 * (M // 6), 4 * (M // 6))
    bad[256:384, 640:768] -= dt1[ks, 256:384].float().t() @ ctx[ks, 640:768].float()
    assert _model_level_passes(bad - prior, G["wo"][1] - prior.double())
    with pytest.raises(kc.CheckError, match=r"layer 2 bwd5: dwo: .*tile m=2 n=5"):
        lc.check_arena("layer 2", {"wo": bad}, G, lc.Worst())


def test_rejects_layer_input_of_the_previous_layer_in_wgrad():
    """Layer 1's dWqkv taken from layer 0's input x instead of its own input y0.  Where neighbouring layers' inputs differ by ~2 %
    (a residual stream deep in the stack) the model-level criterion passes it; stage bwd7 does not."""
    gen = torch.Generator().manual_seed(6)
    M, H = 1968, 768
    x0 = torch.randn(M, H, generator=gen)
    y0 = (x0 + 0.02 * torch.randn(M, H, generator=gen)).to(BF)
    x0 = x0.to(BF)
    dqkv = (y0.float() @ (torch.randn(H, 3 * H, generator=gen) * H ** -0.5) + 0.5 * torch.randn(M, 3 * H, generator=gen)).to(BF)
    prior = torch.randn(3 * H, H, generator=gen)
    G = {"wqkv": ("gemm", *lc.ref_wgrad(dqkv, y0, prior))}
    lc.check_arena("layer 1", {"wqkv": prior + dqkv.float().t() @ y0.float()}, G, lc.Worst())
    bad = prior + dqkv.float().t() @ x0.float()
    assert _model_level_passes(bad - prior, G["wqkv"][1] - prior.double())
    with pytest.raises(kc.CheckError, match=r"layer 1 bwd7: dwqkv"):
        lc.check_arena("layer 1", {"wqkv": bad}, G, lc.Worst())


def _rounded(t):
    """What a correct kernel stores: the exact value rounded once to bf16."""
    return t.to(BF)


def test_rejects_dt2_for_dz2_as_the_residual_gradient():
    """dy1 = du W1 + dt2 instead of + dz2.  At p = 0.01 the defect changes dy1 and every gradient below it by ~3 % (the
    model-level criterion passes all of them); stage bwd3 rejects it.  At p = 0.1 it is ~11 %, which the model level sees too."""
    c = _case(2, 123, 768, 3072, 0.01, 7, 102)
    w, B, Lq, heads, p = c["w"], c["B"], c["Lq"], c["heads"], c["p"]
    A, S, _ = lc.reference_layer(w, c["x"], c["allow"], c["keep"], p, B, Lq, heads, c["dy"], c["prior"])
    Sk = {k: _rounded(v) for k, v in S.items()}
    bad = _rounded(lc.ref_linear(Sk["du"], w["w1"].t(), epi=lc.ADD, aux=Sk["dt2"])["d0"][0])

    def below(dy1):     # what dy1 feeds: LN1 backward, Wo, attention, Wqkv
        l1 = kc.ln_bwd_ref(A["t1"], c["x"], w["ln1_g"], A["stats1"], dy1, c["keep"]["hid1"], p)
        dt1 = l1["dt"][0]
        q, k, v = lc._split(A["qkv"], B, Lq, heads)
        a = kc.attn_bwd_ref(q, k, v, c["allow"], kc.heads_view(dt1 @ w["wo"], B, Lq, heads), c["keep"]["attn"], p)
        dqkv = torch.cat([lc._merge(a[n]) for n in ("dq", "dk", "dv")], 1)
        return {"dy1": dy1.to(F64), "wo": dt1.t() @ A["ctx"], "bo": dt1.sum(0), "ln1_g": l1["dgamma"].sum(0), "ln1_b": l1["dbeta"].sum(0),
                "wqkv": dqkv.t() @ c["x"], "bqkv": dqkv.sum(0), "dx": dqkv @ lc._wqkv(w) + l1["dz"][0]}

    good_g, bad_g = below(S["dy1"]), below(bad)
    for n in good_g:
        assert _model_level_passes(bad_g[n], good_g[n]), n
    R, _ = lc.layer_bwd_refs(w, c["x"], c["allow"], A, c["dy"], Sk, c["prior"], c["keep"], p, B, Lq, heads)
    good = _rounded(lc.ref_linear(Sk["du"], w["w1"].t(), epi=lc.ADD, aux=Sk["dz2"])["d0"][0])
    lc.check_gemm_stage(lc.Worst(), "layer 0 bwd3 dy1: dy1", good, R["dy1"])
    with pytest.raises(kc.CheckError, match=r"layer 0 bwd3 dy1: dy1"):
        lc.check_gemm_stage(lc.Worst(), "layer 0 bwd3 dy1: dy1", bad, R["dy1"])


CALL_CASES = [dict(B=2, Lq=123, H=768, I=3072, n_layers=3, p=0.1), dict(B=4, Lq=143, H=128, I=512, n_layers=2, p=0.1, dys_mid=True),
              dict(B=2, Lq=512, H=128, I=512, n_layers=2, p=0.0), dict(B=1, Lq=1, H=128, I=512, n_layers=2, p=0.1, mask="bernoulli")]


@pytest.mark.parametrize("case", CALL_CASES, ids=["production", "over-tile-dys", "widest", "small-m-bernoulli"])
def test_encoder_stack_call_sequences_marshal(case):
    with abi_cases.dry_run() as calls:
        c = abi_cases.stack_inputs("cpu", **case)
        r = abi_cases.stack_run(c)
    n = case["n_layers"]
    assert calls.count("vlpk_encoder_fwd") == 1 and calls.count("vlpk_encoder_bwd") == 1
    assert calls.count("vlpk_layer_fwd") == n and calls.count("vlpk_layer_bwd") == n
    assert len(r["acts"]) == n and len(r["chain_scratch"]) == n and r["chain_dy"][n - 1] is c["dys"][n - 1]


@pytest.mark.parametrize("H,src,n_steps", [(768, 100, 3), (128, 126, 5), (128, 506, 6)])
def test_cached_decode_call_sequences_marshal(H, src, n_steps):
    with abi_cases.dry_run() as calls:
        recs = list(abi_cases.cached_decode_calls("cpu", H, 6, src, n_steps, src + n_steps + 5))
    assert calls.count("vlpk_layer_cached_fwd") == n_steps + 1
    assert [(r["pos"], r["Lq"], r["Lkv"]) for r in recs] == [(0, src, src)] + [(src - 1 + k, 2, src + 1 + k) for k in range(n_steps)]
