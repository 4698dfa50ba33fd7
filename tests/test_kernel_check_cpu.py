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


def test_bits_to_allow_ignores_bits_beyond_lkv_and_broadcasts():
    bits = torch.zeros(2, 1, 4, dtype=torch.int32)
    bits[:, 0, 0] = 0b1011
    bits[:, 0, 3] = -1                                     # bits 96..127 set: beyond Lkv = 70
    allow = kc.bits_to_allow(bits, 5, 70)
    assert allow.shape == (2, 5, 70)
    assert allow[:, :, :4].tolist() == [[[True, True, False, True]] * 5] * 2
    assert not allow[:, :, 4:].any()
