"""GPU bring-up harness: runs each kernel family in its own subprocess (a device trap must not take the
other checks down), compares with plain PyTorch fp32 math, and prints one report per case.

    python tools/bringup.py            # run everything
    python tools/bringup.py gemm_kk    # one case in-process
"""
import math
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from vlp_b200 import _lib as L

DEV = "cuda"
BF = torch.bfloat16


def rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def report(name, got, ref, tol=2e-2):
    r = rel(got, ref)
    bad = not (r < tol) or not torch.isfinite(got.float()).all().item()
    print(f"  {name:32s} rel_l2={r:.3e} max_abs={(got.float() - ref.float()).abs().max().item():.3e} {'FAIL' if bad else 'ok'}")
    return not bad


def gemm(M, N, K, A, B, a_mn=0, b_mn=0, bias=None, epi=0, aux=None, splits=1, bn=0, out_f32=False, D1=None, D0=None):
    if D0 is None:
        D0 = torch.zeros(M, N, device=DEV, dtype=torch.float32 if out_f32 else BF)
    L.call("vlpk_gemm", M, N, K, a_mn, A.data_ptr(), A.stride(0), b_mn, B.data_ptr(), B.stride(0), L.ptr(bias), D0.data_ptr(),
           D0.stride(0), L.ptr(D1), D1.stride(0) if D1 is not None else 0, L.ptr(aux), aux.stride(0) if aux is not None else 0,
           epi, splits, bn, L.stream())
    return D0


def case_gemm_kk():
    ok = True
    torch.manual_seed(0)
    for (M, N, K, bn) in [(128, 128, 64, 128), (300, 256, 192, 128), (300, 256, 192, 0), (1000, 768, 768, 0), (7872, 2304, 768, 0)]:
        A = torch.randn(M, K, device=DEV).to(BF)
        B = torch.randn(N, K, device=DEV).to(BF)
        bias = torch.randn(N, device=DEV).to(BF)
        ref = A.float() @ B.float().t() + bias.float()
        D = gemm(M, N, K, A, B, bias=bias, bn=bn)
        torch.cuda.synchronize()
        ok &= report(f"kk M{M} N{N} K{K} bn{bn}", D, ref)
    # K tail (1608 -> partial k-block, zero filled)
    M, N, K = 640, 768, 1608
    A = torch.randn(M, K, device=DEV).to(BF); B = torch.randn(N, K, device=DEV).to(BF)
    ok &= report("kk K=1608 tail", gemm(M, N, K, A, B), A.float() @ B.float().t())
    return ok


def case_gemm_epi():
    ok = True
    torch.manual_seed(1)
    M, N, K = 520, 512, 256
    A = torch.randn(M, K, device=DEV).to(BF) * 0.5
    B = torch.randn(N, K, device=DEV).to(BF) * 0.1
    bias = torch.randn(N, device=DEV).to(BF)
    u_ref = A.float() @ B.float().t() + bias.float()
    D1 = torch.zeros(M, N, device=DEV, dtype=BF)
    U = gemm(M, N, K, A, B, bias=bias, epi=1, D1=D1)
    torch.cuda.synchronize()
    gp_ref = 0.5 * (1 + torch.erf(u_ref / math.sqrt(2))) + u_ref * torch.exp(-0.5 * u_ref * u_ref) / math.sqrt(2 * math.pi)
    ok &= report("gelu: gelu'(u)", U, gp_ref)
    ok &= report("gelu: gelu(u)", D1, torch.nn.functional.gelu(u_ref))
    R = gemm(M, N, K, A, B, bias=bias, epi=2)
    ok &= report("relu", R, torch.relu(u_ref))
    return ok


def case_gemm_dgrad():
    torch.manual_seed(2)

    def run():
        ok = True
        for (M, N, K, bn) in [(300, 256, 128, 128), (300, 512, 320, 0), (1000, 768, 3072, 0)]:
            # D[M,N] = A[M,K] B[N,K]^T with B stored as [K,N] row-major (MN-major)
            A = torch.randn(M, K, device=DEV).to(BF)
            Bs = (torch.randn(K, N, device=DEV) * 0.1).to(BF)
            ref = A.float() @ Bs.float()
            ok &= report(f"dgrad M{M} N{N} K{K} bn{bn}", gemm(M, N, K, A, Bs, b_mn=1, bn=bn), ref)
        M, N, K = 300, 256, 192
        A = torch.randn(M, K, device=DEV).to(BF); Bs = (torch.randn(K, N, device=DEV) * 0.1).to(BF)
        aux = torch.randn(M, N, device=DEV).to(BF)
        ref = A.float() @ Bs.float()
        ok &= report("dgrad +aux", gemm(M, N, K, A, Bs, b_mn=1, epi=3, aux=aux), ref + aux.float())
        ok &= report("dgrad *aux", gemm(M, N, K, A, Bs, b_mn=1, epi=4, aux=aux), ref * aux.float())
        return ok

    return run()


def case_gemm_wgrad():
    torch.manual_seed(3)

    def run():
        ok = True
        for (T, Nf, Kf, splits, bn) in [(128, 128, 128, 1, 128), (500, 256, 384, 1, 128), (500, 256, 512, 3, 0), (7872, 768, 768, 8, 0),
                                        (640, 768, 1608, 2, 0)]:
            dY = (torch.randn(T, Nf, device=DEV) * 0.1).to(BF)
            X = torch.randn(T, Kf, device=DEV).to(BF)
            ref = dY.float().t() @ X.float()
            D = gemm(Nf, Kf, T, dY, X, a_mn=1, b_mn=1, epi=6, splits=splits, bn=bn, out_f32=True)
            ok &= report(f"wgrad T{T} N{Nf} K{Kf} s{splits} bn{bn}", D, ref)
        return ok

    return run()


def _mask_bits(mask01):
    B, R, KV = mask01.shape
    out = torch.zeros(B, R, 4, device=DEV, dtype=torch.int32)
    m = mask01.contiguous()
    L.call("vlpk_mask_pack", m.data_ptr(), 2, 1, B, R, KV, m.stride(0), m.stride(1), out.data_ptr(), L.stream())
    return out


def _attn_ref(q, k, v, mask01):
    # q,k,v [B,h,L,64] fp32; reference semantics modeling.py:279-298 (dropout off)
    s = q @ k.transpose(-1, -2) / 8.0 + (1.0 - mask01[:, None].float()) * -10000.0
    p = torch.softmax(s, -1)
    return p @ v


def case_attn():
    ok = True
    torch.manual_seed(4)
    B, heads, Lq, H = 3, 2, 123, 128
    qkv = torch.randn(B, Lq, 3 * H, device=DEV).to(BF)
    mask = torch.zeros(B, Lq, Lq, device=DEV, dtype=torch.int64)
    mask[:, :, :102] = 1
    mask[:, 102:, 102:] = torch.tril(torch.ones(21, 21, device=DEV, dtype=torch.int64))
    mask[1, :, 5:9] = 0
    bits = _mask_bits(mask)
    # check the packer itself
    ref_bits = torch.zeros(B, Lq, 4, dtype=torch.int64)
    mc = mask.cpu()
    for j in range(Lq):
        ref_bits[:, :, j // 32] |= mc[:, :, j] << (j % 32)
    ref_bits = ref_bits.to(torch.int32)  # wrap
    ok &= bool((bits.cpu() == ref_bits).all())
    print("  mask_pack", "ok" if ok else "FAIL")
    ctx = torch.zeros(B, Lq, H, device=DEV, dtype=BF)
    lse = torch.zeros(B, heads, Lq, device=DEV)
    q, k, v = qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:]
    L.call("vlpk_attn_core_fwd", B, heads, Lq, Lq, q.data_ptr(), 3 * H, k.data_ptr(), v.data_ptr(), 3 * H, bits.data_ptr(), Lq,
           ctx.data_ptr(), H, lse.data_ptr(), None, 0, L.stream())
    torch.cuda.synchronize()

    def heads_view(t):
        return t.float().view(B, Lq, heads, 64).permute(0, 2, 1, 3)

    qf, kf, vf = (heads_view(t).clone().requires_grad_(True) for t in (q, k, v))
    ref = _attn_ref(qf, kf, vf, mask)
    ref_ctx = ref.permute(0, 2, 1, 3).reshape(B, Lq, H)
    ok &= report("attn fwd ctx", ctx, ref_ctx)
    s = qf @ kf.transpose(-1, -2) / 8.0 + (1.0 - mask[:, None].float()) * -10000.0
    ok &= report("attn fwd lse", lse, torch.logsumexp(s, -1), tol=1e-3)
    # backward
    dctx = torch.randn(B, Lq, H, device=DEV).to(BF)
    dqkv = torch.zeros(B, Lq, 3 * H, device=DEV, dtype=BF)
    L.call("vlpk_attn_core_bwd", B, heads, Lq, q.data_ptr(), k.data_ptr(), v.data_ptr(), 3 * H, bits.data_ptr(), Lq, ctx.data_ptr(),
           dctx.data_ptr(), H, lse.data_ptr(), dqkv.data_ptr(), dqkv[..., H:].data_ptr(), dqkv[..., 2 * H:].data_ptr(), 3 * H, None, 0,
           L.stream())
    torch.cuda.synchronize()
    ref_ctx.backward(dctx.float())
    for nm, t, g in (("dq", dqkv[..., :H], qf.grad), ("dk", dqkv[..., H:2 * H], kf.grad), ("dv", dqkv[..., 2 * H:], vf.grad)):
        ok &= report(f"attn bwd {nm}", t, g.permute(0, 2, 1, 3).reshape(B, Lq, H), tol=3e-2)
    # incremental shape: Lq=2, Lkv=104, broadcast row mask
    Lq2, Lkv2 = 2, 104
    q2 = torch.randn(B, Lq2, H, device=DEV).to(BF)
    kv2 = torch.randn(B, Lkv2, 2 * H, device=DEV).to(BF)
    m2 = torch.ones(B, Lq2, Lkv2, device=DEV, dtype=torch.int64)
    m2[:, 0, -1] = 0
    bits2 = _mask_bits(m2)
    ctx2 = torch.zeros(B, Lq2, H, device=DEV, dtype=BF)
    L.call("vlpk_attn_core_fwd", B, heads, Lq2, Lkv2, q2.data_ptr(), H, kv2.data_ptr(), kv2[..., H:].data_ptr(), 2 * H, bits2.data_ptr(),
           Lq2, ctx2.data_ptr(), H, None, None, 0, L.stream())
    torch.cuda.synchronize()
    qf2 = q2.float().view(B, Lq2, heads, 64).permute(0, 2, 1, 3)
    kf2 = kv2[..., :H].float().reshape(B, Lkv2, heads, 64).permute(0, 2, 1, 3)
    vf2 = kv2[..., H:].float().reshape(B, Lkv2, heads, 64).permute(0, 2, 1, 3)
    ok &= report("attn fwd incr (2x104)", ctx2, _attn_ref(qf2, kf2, vf2, m2).permute(0, 2, 1, 3).reshape(B, Lq2, H))
    return ok


def case_attn_full():
    """Production item count (B = 64 x 12 heads = 768 (sequence, head) items -> every persistent CTA walks 2-3 items) with per-sample
    mixed seq2seq / bidirectional masks and ragged lengths; forward and backward against fp32 torch on the same bf16 inputs, then the
    same with attention dropout 0.1, the keep-mask replayed from the kernels' Philox stream (vlpk_debug_dropout_mask)."""
    from vlp_b200 import ops
    ok = True
    torch.manual_seed(12)
    B, heads, Lq, H = 64, 12, 123, 768
    qkv = torch.randn(B, Lq, 3 * H, device=DEV).to(BF)
    mask = torch.zeros(B, Lq, Lq, device=DEV, dtype=torch.int64)
    for b in range(B):
        n_tok = 102 + 1 + int(torch.randint(8, 21, (1,)))
        if b % 4 == 3:
            mask[b, :, :n_tok] = 1
        else:
            mask[b, :, :102] = 1
            mask[b, 102:n_tok, 102:n_tok] = torch.tril(torch.ones(n_tok - 102, n_tok - 102, device=DEV, dtype=torch.int64))
    bits = _mask_bits(mask)
    q, k, v = qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:]

    def heads_view(t):
        return t.float().view(B, Lq, heads, 64).permute(0, 2, 1, 3)

    for p_drop in (0.0, 0.1):
        ctx = torch.zeros(B, Lq, H, device=DEV, dtype=BF)
        lse = torch.zeros(B, heads, Lq, device=DEV)
        seed, site = 4242, 5
        drop = L.VlpkDropout(p_drop, seed, None) if p_drop > 0 else None
        L.call("vlpk_attn_core_fwd", B, heads, Lq, Lq, q.data_ptr(), 3 * H, k.data_ptr(), v.data_ptr(), 3 * H, bits.data_ptr(), Lq,
               ctx.data_ptr(), H, lse.data_ptr(), drop, site, L.stream())
        dctx = torch.randn(B, Lq, H, device=DEV).to(BF)
        dqkv = torch.zeros(B, Lq, 3 * H, device=DEV, dtype=BF)
        L.call("vlpk_attn_core_bwd", B, heads, Lq, q.data_ptr(), k.data_ptr(), v.data_ptr(), 3 * H, bits.data_ptr(), Lq, ctx.data_ptr(),
               dctx.data_ptr(), H, lse.data_ptr(), dqkv.data_ptr(), dqkv[..., H:].data_ptr(), dqkv[..., 2 * H:].data_ptr(), 3 * H, drop, site,
               L.stream())
        torch.cuda.synchronize()
        qf, kf, vf = (heads_view(t).clone().requires_grad_(True) for t in (q, k, v))
        s = qf @ kf.transpose(-1, -2) / 8.0 + (1.0 - mask[:, None].float()) * -10000.0
        pr = torch.softmax(s, -1)
        if p_drop > 0:
            keep = ops.dropout_keep_mask(p_drop, seed, site, B * heads * Lq * 128).view(B, heads, Lq, 128)[..., :Lq].float()
            pr = pr * keep / (1.0 - p_drop)
        ref_ctx = (pr @ vf).permute(0, 2, 1, 3).reshape(B, Lq, H)
        tag = f"p={p_drop}"
        ok &= report(f"attn full fwd ctx {tag}", ctx, ref_ctx)
        ok &= report(f"attn full fwd lse {tag}", lse, torch.logsumexp(s, -1), tol=1e-3)
        ref_ctx.backward(dctx.float())
        for nm, t, g in (("dq", dqkv[..., :H], qf.grad), ("dk", dqkv[..., H:2 * H], kf.grad), ("dv", dqkv[..., 2 * H:], vf.grad)):
            ok &= report(f"attn full bwd {nm} {tag}", t, g.permute(0, 2, 1, 3).reshape(B, Lq, H), tol=3e-2)
    return ok


def case_attn_common_mode():
    """Numerical stress for the attention backward: keys / values / queries dominated by a component shared by all rows
    (VLP's 100 near-identical region rows at initialisation) and a gradient that enters at two rows only (the VQA head).
    The softmax-backward row term must cancel that common mode; compared with fp32 autograd on the same bf16 inputs."""
    ok = True
    torch.manual_seed(9)
    B, heads, Lq, H = 2, 2, 123, 128
    common = torch.randn(1, 1, 3 * H, device=DEV)
    qkv = (common * 1.0 + 0.1 * torch.randn(B, Lq, 3 * H, device=DEV)).to(BF)
    mask = torch.ones(B, Lq, Lq, device=DEV, dtype=torch.int64)
    bits = _mask_bits(mask)
    ctx = torch.zeros(B, Lq, H, device=DEV, dtype=BF)
    lse = torch.zeros(B, heads, Lq, device=DEV)
    q, k, v = qkv[..., :H], qkv[..., H:2 * H], qkv[..., 2 * H:]
    L.call("vlpk_attn_core_fwd", B, heads, Lq, Lq, q.data_ptr(), 3 * H, k.data_ptr(), v.data_ptr(), 3 * H, bits.data_ptr(), Lq,
           ctx.data_ptr(), H, lse.data_ptr(), None, 0, L.stream())

    def heads_view(t):
        return t.float().view(B, Lq, heads, 64).permute(0, 2, 1, 3)

    qf, kf, vf = (heads_view(t).clone().requires_grad_(True) for t in (q, k, v))
    ref_ctx = _attn_ref(qf, kf, vf, mask).permute(0, 2, 1, 3).reshape(B, Lq, H)
    ok &= report("common-mode fwd ctx", ctx, ref_ctx)
    dctx = torch.zeros(B, Lq, H, device=DEV)
    dctx[:, 0] = torch.randn(B, H, device=DEV)
    dctx[:, 101] = torch.randn(B, H, device=DEV)
    dctx = dctx.to(BF)
    dqkv = torch.zeros(B, Lq, 3 * H, device=DEV, dtype=BF)
    L.call("vlpk_attn_core_bwd", B, heads, Lq, q.data_ptr(), k.data_ptr(), v.data_ptr(), 3 * H, bits.data_ptr(), Lq, ctx.data_ptr(),
           dctx.data_ptr(), H, lse.data_ptr(), dqkv.data_ptr(), dqkv[..., H:].data_ptr(), dqkv[..., 2 * H:].data_ptr(), 3 * H, None, 0,
           L.stream())
    torch.cuda.synchronize()
    ref_ctx.backward(dctx.float())
    for nm, t, g in (("dq", dqkv[..., :H], qf.grad), ("dk", dqkv[..., H:2 * H], kf.grad), ("dv", dqkv[..., 2 * H:], vf.grad)):
        ok &= report(f"common-mode bwd {nm}", t, g.permute(0, 2, 1, 3).reshape(B, Lq, H), tol=3e-2)
    return ok


def case_rowops():
    ok = True
    torch.manual_seed(5)
    for H in (768, 128):
        M = 1000
        t = torch.randn(M, H, device=DEV).to(BF); res = torch.randn(M, H, device=DEV).to(BF)
        g = (1 + 0.1 * torch.randn(H, device=DEV)).to(BF); b = (0.1 * torch.randn(H, device=DEV)).to(BF)
        y = torch.zeros(M, H, device=DEV, dtype=BF); stats = torch.zeros(M, 2, device=DEV)
        L.call("vlpk_ln_res_drop_fwd", M, H, t.data_ptr(), res.data_ptr(), g.data_ptr(), b.data_ptr(), y.data_ptr(), stats.data_ptr(), None, 0,
               L.stream())
        tf, rf = t.float().requires_grad_(True), res.float().requires_grad_(True)
        gf, bf_ = g.float().requires_grad_(True), b.float().requires_grad_(True)
        ref = torch.nn.functional.layer_norm(tf + rf, (H,), gf, bf_, 1e-5)
        ok &= report(f"ln fwd H{H}", y, ref, tol=1e-2)
        dy = torch.randn(M, H, device=DEV).to(BF)
        dz = torch.zeros(M, H, device=DEV, dtype=BF)
        dg = torch.zeros(H, device=DEV); db = torch.zeros(H, device=DEV); dbias = torch.zeros(H, device=DEV)
        L.call("vlpk_ln_res_drop_bwd", M, H, t.data_ptr(), res.data_ptr(), g.data_ptr(), stats.data_ptr(), dy.data_ptr(), dz.data_ptr(), None,
               dg.data_ptr(), db.data_ptr(), dbias.data_ptr(), None, 0, L.stream())
        ref.backward(dy.float())
        ok &= report(f"ln bwd dz H{H}", dz, tf.grad, tol=1e-2)
        ok &= report(f"ln bwd dgamma H{H}", dg, gf.grad, tol=1e-2)
        ok &= report(f"ln bwd dbeta H{H}", db, bf_.grad, tol=1e-2)
        ok &= report(f"ln bwd dbias H{H}", dbias, tf.grad.sum(0), tol=1e-2)
    # dropout consistency: fwd then bwd regenerate the same mask
    M, H, p = 512, 768, 0.1
    t = torch.ones(M, H, device=DEV).to(BF); res = torch.zeros(M, H, device=DEV).to(BF)
    g = torch.ones(H, device=DEV).to(BF); b = torch.zeros(H, device=DEV).to(BF)
    y = torch.zeros(M, H, device=DEV, dtype=BF); stats = torch.zeros(M, 2, device=DEV)
    dr = L.VlpkDropout(p, 1234, None)
    L.call("vlpk_ln_res_drop_fwd", M, H, t.data_ptr(), res.data_ptr(), g.data_ptr(), b.data_ptr(), y.data_ptr(), stats.data_ptr(), dr, 7, L.stream())
    torch.cuda.synchronize()
    frac = (y.float() < 0).float().mean().item()  # dropped elements sit below the row mean -> negative after LN
    print(f"  dropout drop fraction {frac:.4f} (target {p})")
    ok &= abs(frac - p) < 0.01
    x = torch.randn(1000, 3072, device=DEV).to(BF)
    cs = torch.zeros(3072, device=DEV)
    L.call("vlpk_colsum", x.data_ptr(), 3072, 1000, 3072, cs.data_ptr(), L.stream())
    ok &= report("colsum", cs, x.float().sum(0), tol=1e-3)
    xf = torch.randn(100003, device=DEV)
    yb = torch.zeros(100003, device=DEV, dtype=BF)
    L.call("vlpk_f32_to_bf16", xf.data_ptr(), yb.data_ptr(), xf.numel(), L.stream())
    ok &= report("f32->bf16", yb, xf.to(BF), tol=1e-6)
    return ok


def case_perf():
    return _perf(True)


def _perf(extras):
    """Quick device-time numbers for the hot shapes (CUDA events, L2-sized rotation not applied: indicative only)."""
    torch.manual_seed(6)
    M = 7872

    def timeit(fn, flops, name, iters=20):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(iters):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / iters
        print(f"  {name:36s} {ms * 1e3:9.1f} us  {flops / ms / 1e9:8.1f} TFLOP/s")

    for (N, K, bn) in [(2304, 768, 0), (768, 768, 0), (3072, 768, 0), (768, 3072, 0), (768, 768, 128), (3072, 768, 128)]:
        A = torch.randn(M, K, device=DEV).to(BF); B = torch.randn(N, K, device=DEV).to(BF); D = torch.zeros(M, N, device=DEV, dtype=BF)
        timeit(lambda: gemm(M, N, K, A, B, bn=bn, D0=D), 2.0 * M * N * K, f"fwd  {M}x{N}x{K} bn{bn}")
        if extras:
            timeit(lambda: torch.matmul(A, B.t(), out=D), 2.0 * M * N * K, f"cublas {M}x{N}x{K}")
    for (N, K) in [(3072, 768), (768, 3072)]:
        A = torch.randn(M, K, device=DEV).to(BF); Bs = torch.randn(K, N, device=DEV).to(BF); D = torch.zeros(M, N, device=DEV, dtype=BF)
        timeit(lambda: gemm(M, N, K, A, Bs, b_mn=1, D0=D), 2.0 * M * N * K, f"dgrad {M}x{N}x{K}")
    for (Nf, Kf, s) in [(768, 768, 0), (768, 3072, 0), (3072, 768, 0), (2304, 768, 0)]:
        dY = torch.randn(M, Nf, device=DEV).to(BF); X = torch.randn(M, Kf, device=DEV).to(BF); D = torch.zeros(Nf, Kf, device=DEV)
        timeit(lambda: gemm(Nf, Kf, M, dY, X, a_mn=1, b_mn=1, epi=6, splits=s, out_f32=True, D0=D), 2.0 * M * Nf * Kf, f"wgrad {Nf}x{Kf}x{M} s{s}")
    if not extras:
        return True
    B, heads, Lq, H = 64, 12, 123, 768
    qkv = torch.randn(B, Lq, 3 * H, device=DEV).to(BF)
    bits = torch.full((B, Lq, 4), -1, device=DEV, dtype=torch.int32)
    ctx = torch.zeros(B, Lq, H, device=DEV, dtype=BF); lse = torch.zeros(B, heads, Lq, device=DEV)
    dqkv = torch.zeros_like(qkv); dctx = torch.randn(B, Lq, H, device=DEV).to(BF)
    fl = 4.0 * B * heads * Lq * Lq * 64
    timeit(lambda: L.call("vlpk_attn_core_fwd", B, heads, Lq, Lq, qkv.data_ptr(), 3 * H, qkv[..., H:].data_ptr(), qkv[..., 2 * H:].data_ptr(), 3 * H,
                          bits.data_ptr(), Lq, ctx.data_ptr(), H, lse.data_ptr(), None, 0, L.stream()), fl, "attn fwd B64")
    timeit(lambda: L.call("vlpk_attn_core_bwd", B, heads, Lq, qkv.data_ptr(), qkv[..., H:].data_ptr(), qkv[..., 2 * H:].data_ptr(), 3 * H,
                          bits.data_ptr(), Lq, ctx.data_ptr(), dctx.data_ptr(), H, lse.data_ptr(), dqkv.data_ptr(), dqkv[..., H:].data_ptr(),
                          dqkv[..., 2 * H:].data_ptr(), 3 * H, None, 0, L.stream()), 2.5 * fl, "attn bwd B64")
    t = torch.randn(M, H, device=DEV).to(BF); res = torch.randn(M, H, device=DEV).to(BF)
    g = torch.ones(H, device=DEV).to(BF); b = torch.zeros(H, device=DEV).to(BF)
    y = torch.zeros(M, H, device=DEV, dtype=BF); stats = torch.zeros(M, 2, device=DEV)
    dr = L.VlpkDropout(0.1, 1, None)
    timeit(lambda: L.call("vlpk_ln_res_drop_fwd", M, H, t.data_ptr(), res.data_ptr(), g.data_ptr(), b.data_ptr(), y.data_ptr(), stats.data_ptr(), dr, 7,
                          L.stream()), 3.0 * M * H * 2 * 1e3 / 1e0, "ln fwd (col = GB/s x1e-3... bytes)")
    return True


CASES = {"gemm_kk": case_gemm_kk, "gemm_epi": case_gemm_epi, "gemm_dgrad": case_gemm_dgrad, "gemm_wgrad": case_gemm_wgrad,
         "attn": case_attn, "attn_full": case_attn_full, "attn_common_mode": case_attn_common_mode, "rowops": case_rowops, "perf": case_perf}

if __name__ == "__main__":
    if len(sys.argv) > 1:
        name = sys.argv[1]
        print(f"== {name}")
        ok = CASES[name]()
        torch.cuda.synchronize()
        print(f"== {name}: {'PASS' if ok else 'FAIL'}")
        sys.exit(0 if ok else 1)
    for name in CASES:
        t0 = time.time()
        try:
            r = subprocess.run(["timeout", "180", sys.executable, __file__, name], capture_output=True, text=True)
            out = r.stdout + ("\n[stderr]\n" + r.stderr[-3000:] if r.returncode != 0 else "")
            rc = r.returncode
        except Exception as e:  # pragma: no cover
            out, rc = repr(e), -1
        print(f"{out}\n[{name}] rc={rc} {time.time() - t0:.1f}s\n", flush=True)
