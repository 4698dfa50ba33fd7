"""Per-shape comparison of vlpk::gemm_kernel with cuBLAS (torch.matmul / F.linear) on the 12 hot GEMM shapes of one BertLayer at
B = 64 (M = 7872 token rows): 4 forward, 4 dgrad, 4 wgrad.  Same box, same clocks, CUDA events on the launch stream.
  "stream" (the figure that matters inside a training step): 16 launches back to back over 4 rotating operand sets (> L2 together for
           the large shapes), time / 16 — the host runs ahead, so this is device time per launch including launch gaps, not host latency;
  "cold"   : one launch after a 512 MB buffer was rewritten, event to event — INCLUDES the host's launch latency (ours: ctypes + tensor-map
           encoding ~ 8 us, cuBLAS ~ 4 us), kept for continuity with the first table of this round.
Prints a markdown table (and writes it to the optional path argument).

    python tools/gemm_vs_cublas.py [out.md]
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F

from vlp_b200 import _lib as L

DEV, BF = "cuda", torch.bfloat16
M = 7872
H, I = 768, 3072


def timeit(fn, flush, iters=15):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        if flush is not None:
            flush.zero_()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def stream_time(fns, reps=16, iters=7):
    """median over `iters` of (time of `reps` back-to-back launches cycling through fns) / reps, in us"""
    for f in fns:
        f()
    torch.cuda.synchronize()
    ts = []
    for _ in range(iters):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for r in range(reps):
            fns[r % len(fns)]()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3 / reps)
    ts.sort()
    return ts[len(ts) // 2]


def vgemm(Mg, N, K, A, B, a_mn=0, b_mn=0, bias=None, epi=0, aux=None, splits=1, bn=0, D0=None, D1=None):
    L.call("vlpk_gemm", Mg, N, K, a_mn, A.data_ptr(), A.stride(0), b_mn, B.data_ptr(), B.stride(0), L.ptr(bias), D0.data_ptr(), D0.stride(0),
           L.ptr(D1), D1.stride(0) if D1 is not None else 0, L.ptr(aux), aux.stride(0) if aux is not None else 0, epi, splits, bn, L.stream())


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    torch.manual_seed(0)
    flush = torch.empty(512 * 1024 * 1024 // 4, device=DEV, dtype=torch.float32)
    rows = []
    # (name, kind, N_out, K_in, epilogue)  forward: y[M,N] = x[M,K] W[N,K]^T + b
    fwd = [("fwd QKV", 3 * H, H, 0), ("fwd attn-out", H, H, 0), ("fwd FFN-up+GELU", I, H, 1), ("fwd FFN-down", H, I, 0)]
    NS = 4
    for name, N, K, epi in fwd:
        xs = [torch.randn(M, K, device=DEV).to(BF) for _ in range(NS)]
        x = xs[0]
        w = (torch.randn(N, K, device=DEV) * 0.05).to(BF)
        b = torch.randn(N, device=DEV).to(BF)
        ys = [torch.empty(M, N, device=DEV, dtype=BF) for _ in range(NS)]
        y = ys[0]
        y1s = [torch.empty(M, N, device=DEV, dtype=BF) if epi == 1 else None for _ in range(NS)]
        y1 = y1s[0]
        ours = lambda: vgemm(M, N, K, x, w, bias=b, epi=epi, D0=y, D1=y1)
        ref = lambda: F.linear(x, w, b)
        ours_s = [(lambda i=i: vgemm(M, N, K, xs[i], w, bias=b, epi=epi, D0=ys[i], D1=y1s[i])) for i in range(NS)]
        ref_s = [(lambda i=i: F.linear(xs[i], w, b)) for i in range(NS)]
        rows.append((name, M, N, K, 2.0 * M * N * K, [timeit(ours, flush), timeit(ref, flush), stream_time(ours_s), stream_time(ref_s)],
                     "cuBLAS: linear+bias" + (" (no GELU, one output)" if epi == 1 else "")))
    # dgrad: dx[M,K] = dy[M,N] W[N,K]  (ours: contraction over N with W read MN-major)
    dg = [("dgrad dU (x gelu')", H, I, 4), ("dgrad dy1 (+res)", I, H, 3), ("dgrad dx (+res)", 3 * H, H, 3), ("dgrad dctx", H, H, 0)]
    for name, N, K, epi in dg:
        dys = [torch.randn(M, N, device=DEV).to(BF) for _ in range(NS)]
        dy = dys[0]
        w = (torch.randn(N, K, device=DEV) * 0.05).to(BF)
        auxs = [torch.randn(M, K, device=DEV).to(BF) if epi in (3, 4) else None for _ in range(NS)]
        aux = auxs[0]
        dxs = [torch.empty(M, K, device=DEV, dtype=BF) for _ in range(NS)]
        dx = dxs[0]
        ours = lambda: vgemm(M, K, N, dy, w, b_mn=1, epi=epi, aux=aux, D0=dx)
        ref = lambda: torch.matmul(dy, w)
        ours_s = [(lambda i=i: vgemm(M, K, N, dys[i], w, b_mn=1, epi=epi, aux=auxs[i], D0=dxs[i])) for i in range(NS)]
        ref_s = [(lambda i=i: torch.matmul(dys[i], w)) for i in range(NS)]
        rows.append((name, M, K, N, 2.0 * M * N * K, [timeit(ours, flush), timeit(ref, flush), stream_time(ours_s), stream_time(ref_s)],
                     "cuBLAS: plain matmul (no fused add / mul)"))
    # wgrad: dw[N,K] = dy[M,N]^T x[M,K]   (ours: split-K, fp32 TMA reduce-add into a pre-zeroed buffer)
    wg = [("wgrad Wqkv", 3 * H, H), ("wgrad Wo", H, H), ("wgrad W1", I, H), ("wgrad W2", H, I)]
    for name, N, K in wg:
        dys = [torch.randn(M, N, device=DEV).to(BF) for _ in range(NS)]
        xs = [torch.randn(M, K, device=DEV).to(BF) for _ in range(NS)]
        dy, x = dys[0], xs[0]
        dw = torch.zeros(N, K, device=DEV, dtype=torch.float32)
        ours = lambda: vgemm(N, K, M, dy, x, a_mn=1, b_mn=1, epi=6, splits=0, D0=dw)
        ref = lambda: torch.matmul(dy.t(), x)
        ours_s = [(lambda i=i: vgemm(N, K, M, dys[i], xs[i], a_mn=1, b_mn=1, epi=6, splits=0, D0=dw)) for i in range(NS)]
        ref_s = [(lambda i=i: torch.matmul(dys[i].t(), xs[i])) for i in range(NS)]
        rows.append((name, N, K, M, 2.0 * M * N * K, [timeit(ours, flush), timeit(ref, flush), stream_time(ours_s), stream_time(ref_s)],
                     "ours: fp32 reduce-add output; cuBLAS: bf16 output"))
    lines = ["# r02 — vlpk::gemm_kernel vs cuBLAS on the hot shapes of one BertLayer (B = 64, M = 7872)", "",
             f"device: {torch.cuda.get_device_name(0)}; torch {torch.__version__}; CUDA events; stream = 16 back-to-back launches over 4 operand sets / 16 "
             "(device time per launch); cold = single launch after a 512 MB rewrite (includes host launch latency)", "",
             "| GEMM | M x N x K | ours stream us | cuBLAS stream us | ours TF/s | cuBLAS TF/s | ours/cuBLAS (stream) | ours cold us | cuBLAS cold us | note |",
             "|---|---|---|---|---|---|---|---|---|---|"]
    tot = [0.0, 0.0, 0.0, 0.0]
    for name, m, n, k, fl, t, note in rows:
        for i in range(4):
            tot[i] += t[i]
        lines.append(f"| {name} | {m} x {n} x {k} | {t[2]:.1f} | {t[3]:.1f} | {fl / t[2] / 1e6:.0f} | {fl / t[3] / 1e6:.0f} | {t[3] / t[2]:.2f} | {t[0]:.1f} | {t[1]:.1f} | {note} |")
    flops = sum(r[4] for r in rows)
    lines.append(f"| **sum (one layer fwd+bwd)** | | {tot[2]:.1f} | {tot[3]:.1f} | {flops / tot[2] / 1e6:.0f} | {flops / tot[3] / 1e6:.0f} | {tot[3] / tot[2]:.2f} | {tot[0]:.1f} | {tot[1]:.1f} | |")
    text = "\n".join(lines) + "\n"
    if out_path:
        os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
        open(out_path, "w").write(text)
    print(text)


if __name__ == "__main__":
    main()
