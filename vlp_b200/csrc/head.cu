// vlp_b200 — masked-LM head tail (SURVEY.md §8f-3): cls.predictions.decoder (weight tied to the word embeddings, output-only
// bias; modeling.py:465-482) followed by the per-position cross-entropy of crit_mask_lm (modeling.py:1108-1109).
//
// The reference materialises fp32 logits [B*P, 28996] and runs softmax / NLL as separate passes; through torch on this stack
// the three GEMMs additionally fall on legacy 2-byte-aligned kernels because 28996 is not a multiple of 8.  Here:
//   forward : logits (bf16, leading dimension padded to a multiple of 8) from the wgmma GEMM with the bias in its epilogue —
//             the decoder weight is read in place, its 4 missing rows are zero-filled by TMA — then ONE pass per row for the
//             online log-sum-exp and the loss;
//   backward: dlogits = (softmax - onehot) * dloss in one pass (bf16), bias gradient by column sums, dh by a split-K GEMM over the
//             vocabulary (fp32 reduce-add) and dW written directly as bf16 by a GEMM with both operands read MN-major.
// HBM-bound row kernels: a row is 58 KB of bf16, read once (forward) / read once + written once (backward).
#include "head.cuh"

#include "gemm.cuh"
#include "host.cuh"
#include "rowops.cuh"

namespace vlpk {
namespace {

constexpr int CE_THREADS = 256;

__device__ __forceinline__ void online_merge(float& m, float& s, float m2, float s2) {
  const float mn = fmaxf(m, m2);
  s = s * __expf(m - mn) + s2 * __expf(m2 - mn);
  m = mn;
}

// One CTA per row: lse = log sum_v exp(x_v), loss = lse - x_label.
__global__ void __launch_bounds__(CE_THREADS) decoder_ce_fwd_kernel(const __nv_bfloat16* __restrict__ logits, int V, int Vp,
                                                                     const long long* __restrict__ labels, float* __restrict__ lse,
                                                                     float* __restrict__ loss) {
  __shared__ float s_m[CE_THREADS / 32], s_s[CE_THREADS / 32];
  const int r = blockIdx.x;
  const __nv_bfloat16* row = logits + static_cast<long long>(r) * Vp;
  float m = -3.0e38f, s = 0.f;
  for (int c = threadIdx.x * 8; c < V; c += CE_THREADS * 8) {
    const uint4 u = *reinterpret_cast<const uint4*>(row + c);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
    float x[8];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      x[2 * j] = f.x;
      x[2 * j + 1] = f.y;
    }
    float cm = -3.0e38f;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (c + j < V) cm = fmaxf(cm, x[j]);
    float cs = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j)
      if (c + j < V) cs += __expf(x[j] - cm);
    online_merge(m, s, cm, cs);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
    online_merge(m, s, m2, s2);
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
    s_m[warp] = m;
    s_s[warp] = s;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float M = s_m[0], S = s_s[0];
    for (int i = 1; i < CE_THREADS / 32; ++i) online_merge(M, S, s_m[i], s_s[i]);
    const float l = M + logf(S);
    lse[r] = l;
    const long long y = labels[r];
    loss[r] = (y >= 0 && y < V) ? l - __bfloat162float(row[y]) : 0.f;
  }
}

// grid (R, column slabs): dlogits = (exp(x - lse) - [v == label]) * dloss, zero in the pad columns and for ignored rows.
__global__ void __launch_bounds__(CE_THREADS) decoder_ce_bwd_kernel(const __nv_bfloat16* __restrict__ logits, int V, int Vp,
                                                                     const long long* __restrict__ labels, const float* __restrict__ lse,
                                                                     const float* __restrict__ dloss, __nv_bfloat16* __restrict__ dlogits) {
  const int r = blockIdx.x;
  const int c = (blockIdx.y * CE_THREADS + threadIdx.x) * 8;
  if (c >= Vp) return;
  const long long y = labels[r];
  const bool live = (y >= 0 && y < V);
  const float g = live ? dloss[r] : 0.f;
  const float l = lse[r];
  const long long off = static_cast<long long>(r) * Vp + c;
  const uint4 u = *reinterpret_cast<const uint4*>(logits + off);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
  float d[8];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    d[2 * j] = f.x;
    d[2 * j + 1] = f.y;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int v = c + j;
    const float p = (v < V) ? __expf(d[j] - l) : 0.f;
    d[j] = (p - ((live && v == y) ? 1.f : 0.f)) * g;
  }
  *reinterpret_cast<uint4*>(dlogits + off) =
      make_uint4(pack_bf16x2(d[0], d[1]), pack_bf16x2(d[2], d[3]), pack_bf16x2(d[4], d[5]), pack_bf16x2(d[6], d[7]));
}

int check(const DecoderCeArgs& a, bool bwd) {
  VLPK_CHECK_ARG(a.R > 0 && a.V > 0 && a.H > 0 && a.H % 64 == 0, "decoder_ce: R=%d V=%d H=%d (H must be a multiple of 64)", a.R, a.V, a.H);
  VLPK_CHECK_ARG(a.h && a.w && a.labels && a.logits && a.lse, "decoder_ce: null pointer");
  if (!bwd) VLPK_CHECK_ARG(a.bias_pad && a.loss, "decoder_ce_fwd: null pointer");
  if (bwd) VLPK_CHECK_ARG(a.dloss && a.dlogits && a.dh && a.dw && a.dbias, "decoder_ce_bwd: null pointer");
  VLPK_CHECK_ARG((reinterpret_cast<uintptr_t>(a.logits) & 15u) == 0 && (reinterpret_cast<uintptr_t>(a.dlogits) & 15u) == 0,
                 "decoder_ce: logits buffers must be 16-byte aligned");
  return 0;
}

}  // namespace

int launch_decoder_ce_fwd(const DecoderCeArgs& a, cudaStream_t s) {
  VLPK_TRY(check(a, false));
  const int Vp = (a.V + 7) / 8 * 8;
  GemmDesc g;  // logits[R,Vp] = h[R,H] W[V,H]^T + bias   (rows V..Vp-1 of W do not exist: zero-filled by TMA)
  g.M = a.R; g.N = Vp; g.K = a.H;
  g.A = a.h; g.lda = a.H;
  g.B[0] = a.w; g.ldb = a.H; g.nseg = 1; g.b_rows = a.V;
  g.bias[0] = static_cast<const __nv_bfloat16*>(a.bias_pad);
  g.D0 = a.logits; g.ldd0 = Vp;
  g.epi = EPI_STORE;
  VLPK_TRY(launch_gemm(g, s));
  LaunchScope scope(CAT_MISC, 2.0 * a.R * Vp, s);
  decoder_ce_fwd_kernel<<<a.R, CE_THREADS, 0, s>>>(static_cast<const __nv_bfloat16*>(a.logits), a.V, Vp, a.labels, a.lse, a.loss);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

int launch_decoder_ce_bwd(const DecoderCeArgs& a, cudaStream_t s) {
  VLPK_TRY(check(a, true));
  const int Vp = (a.V + 7) / 8 * 8;
  {
    LaunchScope scope(CAT_MISC, 4.0 * a.R * Vp, s);
    dim3 grid(a.R, (Vp / 8 + CE_THREADS - 1) / CE_THREADS);
    decoder_ce_bwd_kernel<<<grid, CE_THREADS, 0, s>>>(static_cast<const __nv_bfloat16*>(a.logits), a.V, Vp, a.labels, a.lse, a.dloss,
                                                     static_cast<__nv_bfloat16*>(a.dlogits));
    VLPK_CUDA(cudaGetLastError());
  }
  VLPK_TRY(launch_colsum(a.dlogits, Vp, a.R, Vp, a.dbias, s));  // d bias = column sums of dlogits
  {
    GemmDesc g;  // dh[R,H] (fp32 +=) = dlogits[R,Vp] W[V,H]: contraction over the vocabulary, split-K
    g.M = a.R; g.N = a.H; g.K = Vp;
    g.A = a.dlogits; g.lda = Vp;
    g.b_mn = true; g.B[0] = a.w; g.ldb = a.H; g.nseg = 1; g.b_rows = a.V;
    g.D0 = a.dh; g.ldd0 = a.H;
    g.epi = EPI_REDUCE_F32;
    g.splits = 0;
    int bn = 0;
    VLPK_TRY(plan_gemm(g, &bn, &g.splits));
    if (g.splits > 1) {
      // dh feeds every activation gradient of the backward pass, so its sum must not depend on the order in which the splits
      // finish: each split adds into its own zeroed slice and the slices are summed in a fixed order
      const long long n = static_cast<long long>(a.R) * a.H;
      float* part = scratch_f32(SCRATCH_SPLITK, static_cast<size_t>(n) * g.splits, s);
      if (part == nullptr) return -1;
      VLPK_CUDA(cudaMemsetAsync(part, 0, static_cast<size_t>(n) * g.splits * sizeof(float), s));
      g.D0 = part;
      g.split_stride = n;
      VLPK_TRY(launch_gemm(g, s));
      VLPK_TRY(launch_sum_parts(part, g.splits, n, a.dh, s));
    } else {
      VLPK_TRY(launch_gemm(g, s));
    }
  }
  GemmDesc g;  // dW[V,H] (bf16) = dlogits^T h: both operands read MN-major, K = R fits one or a few k-blocks, direct store
  g.M = a.V; g.N = a.H; g.K = a.R;
  g.a_mn = true; g.A = a.dlogits; g.lda = Vp;
  g.b_mn = true; g.B[0] = a.h; g.ldb = a.H; g.nseg = 1;
  g.D0 = a.dw; g.ldd0 = a.H;
  g.epi = EPI_STORE;
  return launch_gemm(g, s);
}

}  // namespace vlpk
