"""The tile-local checker (tools/kernel_check.py) is sensitive: it accepts a correctly rounded result at the production shape and
rejects each defect a tiled kernel typically has, including defects the global rel-L2 of tools/bringup.py lets through."""
import pytest
import torch

from tools import abi_cases, bringup
from tools import kernel_check as kc

BF = torch.bfloat16
M, N, K = 7872, 2304, 768     # the packed QKV projection of one training step (B = 64 x L = 123 rows, 3 x 768 outputs)


def _rounded_gemm(A, B, bias=None):
    """What a correct kernel returns: fp32 accumulation of the bf16 inputs (+ bias), rounded once to bf16."""
    acc = A.float() @ B.float().t()
    if bias is not None:
        acc = acc + bias.float()
    return acc.to(BF)


@pytest.fixture(scope="module")
def qkv():
    """x [M, K] and the three [768, 768] projections of one abi_cases layer stacked as a 3-segment B operand, with their biases."""
    gen = torch.Generator().manual_seed(7)
    p = abi_cases.layer_params(gen, "cpu", K, 4 * K)
    x = abi_cases._rn(gen, "cpu", M, K)
    Bw = torch.cat(p[0:3])
    bias = torch.cat(p[3:6])
    got = _rounded_gemm(x, Bw, bias)
    acc, E = kc.gemm_ref(x, Bw)
    ref, E = kc.epilogue_ref(0, acc, E, bias=bias)["d0"]
    return dict(x=x, B=Bw, bias=bias, got=got, ref=ref, E=E)


def test_accepts_correctly_rounded_result(qkv):
    e, t = kc.check_gemm("qkv", qkv["got"], qkv["ref"], qkv["E"])
    assert e <= 1.0 and t <= 1.0


def test_rejects_zeroed_box_that_global_metric_passes(qkv):
    got = qkv["got"].clone()
    got[64 * 37:64 * 38, 64 * 21:64 * 22] = 0          # one 64 x 64 TMA store box never written
    assert bringup.rel(got, qkv["ref"]) < 2e-2          # the bring-up metric would have passed this
    with pytest.raises(kc.CheckError, match=r"tile m=18 n=10"):
        kc.check_gemm("qkv", got, qkv["ref"], qkv["E"])


def test_rejects_missing_k_block(qkv):
    x, Bw = qkv["x"], qkv["B"]
    tm, tn, kb = 40, 7, 5
    rows, cols, ks = slice(tm * 128, tm * 128 + 128), slice(tn * 128, tn * 128 + 128), slice(kb * 64, kb * 64 + 64)
    acc = x.float() @ Bw.float().t() + qkv["bias"].float()
    acc[rows, cols] -= x[rows, ks].float() @ Bw[cols, ks].float().t()
    with pytest.raises(kc.CheckError, match=rf"tile m={tm} n={tn}"):
        kc.check_gemm("qkv", acc.to(BF), qkv["ref"], qkv["E"])


def test_rejects_shifted_ragged_last_tile(qkv):
    got = qkv["got"].clone()
    last = (M // 128) * 128                              # 7808: the last M tile holds 64 real rows
    got[last + 1:] = got[last:M - 1].clone()
    with pytest.raises(kc.CheckError, match=r"tile m=61"):
        kc.check_gemm("qkv", got, qkv["ref"], qkv["E"])


def test_rejects_bias_from_neighbouring_segment(qkv):
    x, Bw, bias = qkv["x"], qkv["B"], qkv["bias"]
    wrong = bias.clone()
    wrong[768:896] = bias[0:128]                        # first 128-column block of the key segment reads the query bias
    with pytest.raises(kc.CheckError, match=r"n=6"):
        kc.check_gemm("qkv", _rounded_gemm(x, Bw, wrong), qkv["ref"], qkv["E"])


def test_rejects_shifted_dropout_keep_mask():
    gen = torch.Generator().manual_seed(3)
    m, n, k, p = 520, 776, 256, 0.1
    A = torch.randn(m, k, generator=gen).to(BF)
    Bw = (torch.randn(n, k, generator=gen) * 0.05).to(BF)
    bias = (torch.randn(n, generator=gen) * 0.02).to(BF)
    keep = (torch.rand(m * n, generator=gen) >= p).to(torch.uint8)
    acc, E = kc.gemm_ref(A, Bw)
    ref, Er = kc.epilogue_ref(2, acc, E, bias=bias, keep=keep.view(m, n), scale=1 / (1 - p))["d0"]

    def run(kmask):
        return (torch.relu(A.float() @ Bw.float().t() + bias.float()) * kmask.view(m, n).float() * (1 / (1 - p))).to(BF)

    kc.check_gemm("relu+dropout", run(keep), ref, Er)
    with pytest.raises(kc.CheckError):
        kc.check_gemm("relu+dropout", run(torch.roll(keep, 1)), ref, Er)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_guard_band_detects_one_overwritten_element(dtype):
    v = kc.guarded(65, 136, ld=136 + 64, dtype=dtype, extra_rows=3, col0=8, device="cpu")
    v.copy_(torch.randn(65, 136).to(dtype))
    kc.assert_guard_intact(v)
    v._guard[0][66 * 200 + 150] = 0                       # one element of the tail rows
    with pytest.raises(kc.CheckError, match="1 guard element"):
        kc.assert_guard_intact(v)
    v2 = kc.guarded(65, 136, ld=136 + 64, dtype=dtype, extra_rows=3, col0=8, device="cpu")
    v2.fill_(1)
    v2._guard[0][5 * 200 + 3] = 0                         # one element left of the view (the 16-byte offset)
    with pytest.raises(kc.CheckError):
        kc.assert_guard_intact(v2)


def test_unwritten_element_stays_nan_and_fails():
    v = kc.guarded(130, 136, device="cpu")
    ref = torch.randn(130, 136, dtype=torch.float64)
    v.copy_(ref.to(BF))
    v[129, 135] = float("nan")                           # as if the kernel skipped it
    with pytest.raises(kc.CheckError, match="row 129 col 135"):
        kc.check_gemm("d", v, ref, ref.abs())


def _attn_case(B=4, heads=2, L=123, seed=0):
    gen = torch.Generator().manual_seed(seed)
    q, k, v, dO = (torch.randn(B, heads, L, 64, generator=gen).to(BF) for _ in range(4))
    allow = abi_cases.s2s_mask(B, L, 102, "cpu").bool()
    ref = kc.attn_bwd_ref(q, k, v, allow, dO)
    # what a correct kernel returns: fp32 math on the same bf16 inputs, outputs rounded to bf16
    qf, kf, vf = (t.float().requires_grad_(True) for t in (q, k, v))
    s = qf @ kf.transpose(-1, -2) / 8.0 + (~allow[:, None]).float() * -10000.0
    ctx = torch.softmax(s, -1) @ vf
    ctx.backward(dO.float())
    got = {"ctx": ctx.detach().to(BF), "lse": torch.logsumexp(s, -1).detach(), "dq": qf.grad.to(BF), "dk": kf.grad.to(BF), "dv": vf.grad.to(BF)}
    return ref, got


def test_attention_accepts_and_rejects_wrong_half_block():
    ref, got = _attn_case()
    f = ref["fwd"]
    kc.check_attn_block("ctx", got["ctx"], f["ctx"], f["E"], kc.ATTN_FWD_BLOCK)
    kc.check_lse("lse", got["lse"], f["lse"])
    for nm in ("dq", "dk", "dv"):
        kc.check_attn_block(nm, got[nm], ref[nm], ref["E_" + nm], kc.ATTN_BWD_BLOCK, conditioned=True)
    # warpgroup 1 of block (b=2, h=1) gets its 59 real query rows 5 % wrong: under 3e-2 globally at production size, not per block
    bad = got["dq"].clone()
    bad[2, 1, 64:] = (bad[2, 1, 64:].float() * 1.05).to(BF)
    with pytest.raises(kc.CheckError, match=r"b=2 h=1"):
        kc.check_attn_block("dq", bad, ref["dq"], ref["E_dq"], kc.ATTN_BWD_BLOCK, conditioned=True)
    bad = got["ctx"].clone()
    bad[1, 0, 64:] = bad[0, 0, 64:]                       # the second half of one block's context taken from another sequence
    with pytest.raises(kc.CheckError, match=r"b=1 h=0"):
        kc.check_attn_block("ctx", bad, f["ctx"], f["E"], kc.ATTN_FWD_BLOCK)


# ---- row kernels -------------------------------------------------------------------------------------------------------------
F64 = torch.float64


def test_ln_refs_match_autograd():
    gen = torch.Generator().manual_seed(11)
    Mr, H, p = 6, 24, 0.25
    t, res, dy = (torch.randn(Mr, H, generator=gen, dtype=F64) for _ in range(3))
    g, b = torch.randn(H, generator=gen, dtype=F64), torch.randn(H, generator=gen, dtype=F64)
    keep = (torch.rand(Mr, H, generator=gen) >= p).to(torch.uint8)
    for kp, pp, r_ in ((keep, p, res), (None, 0.0, None)):
        ta, ga, ba = t.clone().requires_grad_(True), g.clone().requires_grad_(True), b.clone().requires_grad_(True)
        z = ta * (1.0 if kp is None else kp.to(F64) / (1 - pp)) + (0.0 if r_ is None else r_)
        y = torch.nn.functional.layer_norm(z, (H,), ga, ba, kc.LN_EPS)
        y.backward(dy)
        ref = kc.ln_ref(t, r_, g, b, kp, pp)
        torch.testing.assert_close(ref["y"][0], y.detach(), rtol=1e-12, atol=1e-12)
        stats = torch.stack((ref["mean"], ref["rstd"]), -1)
        r = kc.ln_bwd_ref(t, r_, g, stats, dy, kp, pp)
        torch.testing.assert_close(r["dt"][0], ta.grad, rtol=1e-10, atol=1e-12)
        torch.testing.assert_close(r["dgamma"].sum(0), ga.grad, rtol=1e-10, atol=1e-12)
        torch.testing.assert_close(r["dbeta"].sum(0), ba.grad, rtol=1e-10, atol=1e-12)
        torch.testing.assert_close(r["dbias"].sum(0), ta.grad.sum(0), rtol=1e-10, atol=1e-12)


def test_embed_refs_match_autograd():
    gen = torch.Generator().manual_seed(12)
    B, Lq, H, R, V, P, T, p = 3, 7, 16, 2, 11, 9, 3, 0.2
    word, posw, typew = (torch.randn(n, H, generator=gen, dtype=F64) for n in (V, P, T))
    vis, vpe = torch.randn(B, R, H, generator=gen, dtype=F64), torch.randn(B, R, H, generator=gen, dtype=F64)
    g, b = torch.randn(H, generator=gen, dtype=F64), torch.randn(H, generator=gen, dtype=F64)
    ids, tt = torch.randint(0, V, (B, Lq), generator=gen), torch.randint(0, T, (B, Lq), generator=gen)
    pos = torch.stack([torch.randperm(Lq, generator=gen) for _ in range(B)])
    keep = (torch.rand(B, Lq, H, generator=gen) >= p).to(torch.uint8)
    dy = torch.randn(B, Lq, H, generator=gen, dtype=F64)
    z = kc.embed_z(ids, word, posw, typew, tt=tt, pos=pos, vis=vis, vpe=vpe, R=R)
    for bb in range(B):
        for l in range(Lq):
            src = vis[bb, l - 1] + vpe[bb, l - 1] if 1 <= l <= R else word[ids[bb, l]] + posw[pos[bb, l]]
            torch.testing.assert_close(z[bb, l], src + typew[tt[bb, l]], rtol=0, atol=0)
    za, ga, ba = z.clone().requires_grad_(True), g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    y = torch.nn.functional.layer_norm(za, (H,), ga, ba, kc.LN_EPS) * keep.to(F64) / (1 - p)
    y.backward(dy)
    ref = kc.embed_ref(z, g, b, keep, p)
    torch.testing.assert_close(ref["y"][0], y.detach(), rtol=1e-12, atol=1e-12)
    r = kc.embed_bwd_ref(z, g, torch.stack((ref["mean"], ref["rstd"]), -1), dy, keep, p)
    torch.testing.assert_close(r["dz"][0], za.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(r["dgamma"].reshape(-1, H).sum(0), ga.grad, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(r["dbeta"].reshape(-1, H).sum(0), ba.grad, rtol=1e-10, atol=1e-12)


def test_ce_ref_matches_autograd():
    gen = torch.Generator().manual_seed(13)
    R, V = 8, 37
    x = (torch.randn(R, V, generator=gen, dtype=F64) * 3).requires_grad_(True)
    labels = torch.tensor([0, V - 1, -1, -100, V, 5, 17, 36])
    dloss = torch.rand(R, generator=gen, dtype=F64) + 0.5
    live = (labels >= 0) & (labels < V)
    loss = torch.nn.functional.cross_entropy(x, torch.where(live, labels, torch.zeros_like(labels)), reduction="none") * live
    (loss * dloss).sum().backward()
    ref = kc.ce_ref(x.detach(), labels, dloss)
    torch.testing.assert_close(ref["loss"], loss.detach(), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["lse"], torch.logsumexp(x.detach(), -1), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(ref["dlogits"], x.grad, rtol=1e-12, atol=1e-12)
    assert bool((ref["dlogits"][~live] == 0).all()) and bool((ref["E"][~live] == 0).all())


def _kernel_like_ln(t, res, g, b, dy, keep, p, two_pass=True):
    """What a correct row kernel returns: fp32 arithmetic on the bf16 inputs, bf16 outputs, fp32 statistics and column sums."""
    z = t.float() * (1.0 if keep is None else keep.float() * torch.tensor(1 / (1 - p), dtype=torch.float32)) + res.float()
    mean = z.mean(-1, keepdim=True)
    var = (z - mean).pow(2).mean(-1, keepdim=True) if two_pass else z.pow(2).mean(-1, keepdim=True) - mean * mean
    rstd = torch.rsqrt(var + kc.LN_EPS)
    xh = (z - mean) * rstd
    y = xh * g.float() + b.float()
    gy = dy.float() * g.float()
    dz = rstd * (gy - gy.mean(-1, keepdim=True) - xh * (gy * xh).mean(-1, keepdim=True))
    dt = dz * (1.0 if keep is None else keep.float() / (1 - p))
    return {"y": y.to(BF), "stats": torch.cat((mean, rstd), -1), "dz": dz.to(BF), "dt": dt.to(BF), "dt32": dt,
            "dgamma": (dy.float() * xh).sum(0), "dbeta": dy.float().sum(0), "dbias": dt.sum(0)}


@pytest.fixture(scope="module")
def ln_prod():
    """LayerNorm + residual + dropout at the production shape (B 64 x L 123 rows, H 768); dy rows of varied magnitude."""
    gen = torch.Generator().manual_seed(14)
    Mr, H, p = 7872, 768, 0.1
    t, res = torch.randn(Mr, H, generator=gen).to(BF), torch.randn(Mr, H, generator=gen).to(BF)
    g, b = (1 + 0.1 * torch.randn(H, generator=gen)).to(BF), (0.1 * torch.randn(H, generator=gen)).to(BF)
    scale = 0.5 + torch.rand(Mr, 1, generator=gen)
    scale[-1] = 0.5
    dy = (torch.randn(Mr, H, generator=gen) * scale).to(BF)
    keep = (torch.rand(Mr, H, generator=gen) >= p).to(torch.uint8)
    got = _kernel_like_ln(t, res, g, b, dy, keep, p)
    ref = kc.ln_ref(t, res, g, b, keep, p)
    bwd = kc.ln_bwd_ref(t, res, g, got["stats"], dy, keep, p)
    return dict(t=t, res=res, g=g, b=b, dy=dy, keep=keep, p=p, got=got, ref=ref, bwd=bwd)


def test_row_checks_accept_correctly_rounded_result(ln_prod):
    got, ref, bwd = ln_prod["got"], ln_prod["ref"], ln_prod["bwd"]
    assert kc.check_rows("y", got["y"], *ref["y"]) <= 1.0
    assert kc.check_ln_stats("ln", got["stats"], ref["mean"], ref["rstd"], ref["z"]) <= 1.0
    for o in ("dz", "dt"):
        assert kc.check_rows(o, got[o], *bwd[o]) <= 1.0
    prior = torch.randn(768, generator=torch.Generator().manual_seed(1))
    for o in ("dgamma", "dbeta", "dbias"):
        assert kc.check_sum_onto(o, prior + got[o], prior, bwd[o]) <= 1.0


def test_row_check_rejects_one_zeroed_row(ln_prod):
    bad = ln_prod["got"]["dz"].clone()
    bad[-1] = 0                                           # the last row never written
    assert bringup.rel(bad, ln_prod["bwd"]["dz"][0]) < 1e-2
    with pytest.raises(kc.CheckError, match=r"row 7871 "):
        kc.check_rows("dz", bad, *ln_prod["bwd"]["dz"])


def test_row_check_rejects_dt_without_dropout_scale():
    gen = torch.Generator().manual_seed(15)
    Mr, H, p = 7872, 768, 0.008
    t, res, dy = (torch.randn(Mr, H, generator=gen).to(BF) for _ in range(3))
    g, b = (1 + 0.1 * torch.randn(H, generator=gen)).to(BF), (0.1 * torch.randn(H, generator=gen)).to(BF)
    keep = (torch.rand(Mr, H, generator=gen) >= p).to(torch.uint8)
    got = _kernel_like_ln(t, res, g, b, dy, keep, p)
    bwd = kc.ln_bwd_ref(t, res, g, got["stats"], dy, keep, p)
    kc.check_rows("dt", got["dt"], *bwd["dt"])
    bad = (got["dz"].float() * keep.float()).to(BF)       # keep * dz: the 1 / (1 - p) forgotten
    assert bringup.rel(bad, bwd["dt"][0]) < 1e-2
    with pytest.raises(kc.CheckError, match="dt"):
        kc.check_rows("dt", bad, *bwd["dt"])


def test_stats_check_rejects_single_pass_variance():
    gen = torch.Generator().manual_seed(16)
    Mr, H = 7872, 768
    t = torch.randn(Mr, H, generator=gen).to(BF)
    sign = torch.randint(0, 2, (Mr, 1), generator=gen) * 2 - 1
    res = (torch.randn(Mr, H, generator=gen) + 64 * 2 ** 0.5 * sign).to(BF)        # |mean| ~ 64 sigma
    g, b = (1 + 0.1 * torch.randn(H, generator=gen)).to(BF), (0.1 * torch.randn(H, generator=gen)).to(BF)
    dy = torch.randn(Mr, H, generator=gen).to(BF)
    ref = kc.ln_ref(t, res, g, b)
    good = _kernel_like_ln(t, res, g, b, dy, None, 0.0)
    kc.check_ln_stats("two-pass", good["stats"], ref["mean"], ref["rstd"], ref["z"])
    bad = _kernel_like_ln(t, res, g, b, dy, None, 0.0, two_pass=False)
    assert bringup.rel(bad["y"], ref["y"][0]) < 1e-2
    with pytest.raises(kc.CheckError, match="rstd"):
        kc.check_ln_stats("single-pass", bad["stats"], ref["mean"], ref["rstd"], ref["z"])


def test_sum_check_rejects_column_off_by_one_lane_in_ragged_chunk():
    """H = 1000: the last chunk holds 232 columns (lanes 0..28).  dgamma of column 996 (lane 28) taken from column 988 (lane 27)."""
    gen = torch.Generator().manual_seed(17)
    Mr, H = 7872, 1000
    t, res = torch.randn(Mr, H, generator=gen).to(BF), torch.randn(Mr, H, generator=gen).to(BF)
    g, b = torch.ones(H).to(BF), torch.zeros(H).to(BF)
    ref = kc.ln_ref(t, res, g, b)
    dy = (ref["xhat"] + 0.1 * torch.randn(Mr, H, generator=gen, dtype=F64)).to(BF)   # an upstream gradient correlated with the output
    got = _kernel_like_ln(t, res, g, b, dy, None, 0.0)
    bwd = kc.ln_bwd_ref(t, res, g, got["stats"], dy)
    prior = torch.randn(H, generator=gen)
    dg = prior + got["dgamma"]
    kc.check_sum_onto("dgamma", dg, prior, bwd["dgamma"])
    bad = dg.clone()
    bad[996] = prior[996] + got["dgamma"][988]
    assert bringup.rel(bad, prior.double() + bwd["dgamma"].sum(0)) < 1e-2
    with pytest.raises(kc.CheckError, match=r"column 996 \(chunk 3, lane 28\)"):
        kc.check_sum_onto("dgamma", bad, prior, bwd["dgamma"])


def test_ce_check_accepts_rounded_rows_and_rejects_shifted_one_hot():
    gen = torch.Generator().manual_seed(18)
    R, V = 192, 28996
    x = (torch.randn(R, V, generator=gen) * 1.4)
    x[::4] *= 20                                          # peaky rows: |logit| ~ 30, a few columns decide lse
    x = x.to(BF)
    labels = torch.randint(0, V, (R,), generator=gen)
    labels[:5] = torch.tensor([V - 1, 0, -1, -100, V])
    labels[4::8] = x[4::8].float().argmax(-1)             # peaky rows whose label holds nearly all the probability
    dloss = torch.rand(R, generator=gen) + 0.5
    live = (labels >= 0) & (labels < V)
    lse = torch.logsumexp(x.float(), -1)
    t = torch.where(live, labels, torch.zeros_like(labels))
    loss = torch.where(live, lse - x.float().gather(1, t[:, None])[:, 0], torch.zeros_like(lse))
    onehot = torch.zeros(R, V)
    onehot[torch.arange(R)[live], t[live]] = 1
    d = (torch.exp(x.float() - lse[:, None]) - onehot) * (dloss * live)[:, None]
    ref = kc.ce_ref(x, labels, dloss)
    kc.check_ce_rows("ce", lse, loss, d.to(BF), ref, labels)
    shifted = torch.zeros(R, V)
    shifted[torch.arange(R)[live], (t[live] + 1) % V] = 1
    bad = ((torch.exp(x.float() - lse[:, None]) - shifted) * (dloss * live)[:, None]).to(BF)
    with pytest.raises(kc.CheckError, match="dlogits"):
        kc.check_ce_rows("ce", lse, loss, bad, ref, labels)


def test_bits_to_allow_ignores_bits_beyond_lkv_and_broadcasts():
    bits = torch.zeros(2, 1, 4, dtype=torch.int32)
    bits[:, 0, 0] = 0b1011
    bits[:, 0, 3] = -1                                     # bits 96..127 set: beyond Lkv = 70
    allow = kc.bits_to_allow(bits, 5, 70)
    assert allow.shape == (2, 5, 70)
    assert allow[:, :, :4].tolist() == [[[True, True, False, True]] * 5] * 2
    assert not allow[:, :, 4:].any()
