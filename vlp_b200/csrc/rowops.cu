// vlp_b200 — HBM-bound row kernels of the VLP hot path (warp-per-row, 16-byte vector access,
// fp32 statistics through __shfl_xor_sync).  No tensor cores here by design: these are pure
// bandwidth kernels and their roofline is HBM GB/s (SURVEY.md §8d).
//
//   ln_res_drop_fwd/bwd : y = LN(dropout(t) + res)           BertSelfOutput / BertOutput, modeling.py:313-317, 353-357
//   embed_fwd/bwd       : y = dropout(LN(word|vis + pos|vis_pe + type))      BertEmbeddings, modeling.py:217-241
//   mask_pack           : additive/0-1 attention mask -> 128-bit row bitmask  get_extended_attention_mask, modeling.py:807-833
//   colsum              : bias gradients
//   f32_to_bf16         : gradient arena conversion
#include "rowops.cuh"

#include <cstdlib>
#include "host.cuh"

namespace vlpk {

static constexpr int MAXCH = 4;  // up to 4 x (32 lanes x 8 elems) = 1024 columns per row; kernels are templated on
                                 // NCH = ceil(H / 256) so that per-row state stays in registers without padding to the maximum

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ void load8(const __nv_bfloat16* p, float (&f)[8]) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 x = unpack_bf16x2(w[j]);
    f[2 * j] = x.x;
    f[2 * j + 1] = x.y;
  }
}
__device__ __forceinline__ void store8(__nv_bfloat16* p, const float (&f)[8]) {
  uint4 u;
  u.x = pack_bf16x2(f[0], f[1]);
  u.y = pack_bf16x2(f[2], f[3]);
  u.z = pack_bf16x2(f[4], f[5]);
  u.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(p) = u;
}

// mean / rstd of a row distributed as z[i][0..7] over the warp (two-pass, fp32)
template <int NCH>
__device__ __forceinline__ void row_stats(const float (&z)[NCH][8], const bool (&ok)[NCH], int H, float eps,
                                          float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i)
    if (ok[i]) {
#pragma unroll
      for (int j = 0; j < 8; ++j) s += z[i][j];
    }
  mean = warp_sum(s) / H;
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < NCH; ++i)
    if (ok[i]) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = z[i][j] - mean;
        v += d * d;
      }
    }
  rstd = rsqrtf(warp_sum(v) / H + eps);
}

// ------------------------------------------------------------------------------------------------
// LN + residual + dropout
// ------------------------------------------------------------------------------------------------
template <int NCH>
__global__ void __launch_bounds__(256) ln_res_drop_fwd_kernel(LnArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const uint64_t dseed = drop_seed(a.drop);
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const long long rowi = static_cast<long long>(blockIdx.x) * wpb + (threadIdx.x >> 5);
  if (rowi >= a.M) return;
  float z[NCH][8];
  bool ok[NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int col = (lane + 32 * i) * 8;
    ok[i] = col < a.H;
    if (ok[i]) {
      float t[8];
      load8(a.t + rowi * a.H + col, t);
      uint32_t keep = 0xFFu;
      if (a.drop.p > 0.f) keep = dropout_keep8(dseed, a.drop.site, (rowi * a.H + col) >> 3, a.drop.thresh16);
      float r[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (a.res != nullptr) load8(a.res + rowi * a.H + col, r);
#pragma unroll
      for (int j = 0; j < 8; ++j) z[i][j] = (((keep >> j) & 1u) ? t[j] * a.drop.scale : 0.f) + r[j];
    }
  }
  float mean, rstd;
  row_stats(z, ok, a.H, a.eps, mean, rstd);
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int col = (lane + 32 * i) * 8;
    if (ok[i]) {
      float g[8], be[8], y[8];
      load8(a.gamma + col, g);
      load8(a.beta + col, be);
#pragma unroll
      for (int j = 0; j < 8; ++j) y[j] = (z[i][j] - mean) * rstd * g[j] + be[j];
      store8(a.y + rowi * a.H + col, y);
    }
  }
  if (lane == 0 && a.stats != nullptr) a.stats[rowi] = make_float2(mean, rstd);
}

// Backward.  One 16-warp block per SM; each warp walks rows (grid-stride) and keeps its dgamma / dbeta / dbias partial sums
// in a private slice of shared memory (float4 read-modify-write, lane-interleaved so every access is conflict free) instead
// of 72+ accumulator registers per thread: ~90 registers/thread -> 16 resident warps/SM with 9 independent 16-byte loads in
// flight per lane, which is what an HBM-bound kernel needs.  One smem reduction + one fp32 atomicAdd per column per block.
static constexpr int LNB_WARPS = 16;

// index of (chunk i, lane l, element j) of a per-warp [NCH*256] accumulator: two float4 halves, lanes adjacent
__device__ __forceinline__ int lnb_idx(int i, int half, int lane) { return ((i * 2 + half) * 32 + lane) * 4; }

template <int NCH>
__global__ void __launch_bounds__(LNB_WARPS * 32, 1) ln_res_drop_bwd_kernel(LnArgs a) {
  pdl_launch_dependents();
  pdl_wait();
  const uint64_t dseed = drop_seed(a.drop);
  extern __shared__ float s_ln[];       // [LNB_WARPS][3][NCH*256] accumulators, then gamma [NCH*256]
  constexpr int W = NCH * 256;
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  float* sg = s_ln + (wib * 3 + 0) * W;
  float* sb = s_ln + (wib * 3 + 1) * W;
  float* st = s_ln + (wib * 3 + 2) * W;
  float* s_gamma = s_ln + LNB_WARPS * 3 * W;
  bool ok[NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    ok[i] = (lane + 32 * i) * 8 < a.H;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(sg + lnb_idx(i, h, lane)) = z4;
      *reinterpret_cast<float4*>(sb + lnb_idx(i, h, lane)) = z4;
      *reinterpret_cast<float4*>(st + lnb_idx(i, h, lane)) = z4;
    }
  }
  if (wib == 0) {
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      float g[8] = {0, 0, 0, 0, 0, 0, 0, 0};
      if (ok[i]) load8(a.gamma + (lane + 32 * i) * 8, g);
      *reinterpret_cast<float4*>(s_gamma + lnb_idx(i, 0, lane)) = make_float4(g[0], g[1], g[2], g[3]);
      *reinterpret_cast<float4*>(s_gamma + lnb_idx(i, 1, lane)) = make_float4(g[4], g[5], g[6], g[7]);
    }
  }
  __syncthreads();

  for (long long rowi = static_cast<long long>(blockIdx.x) * LNB_WARPS + wib; rowi < a.M;
       rowi += static_cast<long long>(gridDim.x) * LNB_WARPS) {
    const float2 stt = a.stats[rowi];
    const float mean = stt.x, rstd = stt.y;
    float xh[NCH][8], gy[NCH][8];
    uint32_t keepm[NCH];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int col = (lane + 32 * i) * 8;
      keepm[i] = 0xFFu;
      if (ok[i]) {
        float t[8], r[8] = {0, 0, 0, 0, 0, 0, 0, 0}, dy[8];
        load8(a.t + rowi * a.H + col, t);
        if (a.res != nullptr) load8(a.res + rowi * a.H + col, r);
        load8(a.dy + rowi * a.H + col, dy);
        if (a.drop.p > 0.f) keepm[i] = dropout_keep8(dseed, a.drop.site, (rowi * a.H + col) >> 3, a.drop.thresh16);
        float g[8];
        {
          const float4 g0 = *reinterpret_cast<const float4*>(s_gamma + lnb_idx(i, 0, lane));
          const float4 g1 = *reinterpret_cast<const float4*>(s_gamma + lnb_idx(i, 1, lane));
          g[0] = g0.x; g[1] = g0.y; g[2] = g0.z; g[3] = g0.w; g[4] = g1.x; g[5] = g1.y; g[6] = g1.z; g[7] = g1.w;
        }
        float pg[8], pb[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float zz = (((keepm[i] >> j) & 1u) ? t[j] * a.drop.scale : 0.f) + r[j];
          xh[i][j] = (zz - mean) * rstd;
          gy[i][j] = dy[j] * g[j];
          s1 += gy[i][j];
          s2 += gy[i][j] * xh[i][j];
          pg[j] = dy[j] * xh[i][j];
          pb[j] = dy[j];
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          float4* pgs = reinterpret_cast<float4*>(sg + lnb_idx(i, h, lane));
          float4* pbs = reinterpret_cast<float4*>(sb + lnb_idx(i, h, lane));
          float4 vg = *pgs, vb = *pbs;
          vg.x += pg[4 * h]; vg.y += pg[4 * h + 1]; vg.z += pg[4 * h + 2]; vg.w += pg[4 * h + 3];
          vb.x += pb[4 * h]; vb.y += pb[4 * h + 1]; vb.z += pb[4 * h + 2]; vb.w += pb[4 * h + 3];
          *pgs = vg;
          *pbs = vb;
        }
      }
    }
    const float c1 = warp_sum(s1) / a.H, c2 = warp_sum(s2) / a.H;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int col = (lane + 32 * i) * 8;
      if (ok[i]) {
        float dz[8], dt[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          dz[j] = rstd * (gy[i][j] - c1 - xh[i][j] * c2);
          dt[j] = ((keepm[i] >> j) & 1u) ? dz[j] * a.drop.scale : 0.f;
        }
        if (a.dz != nullptr) store8(a.dz + rowi * a.H + col, dz);
        if (a.dt != nullptr) store8(a.dt + rowi * a.H + col, dt);
        if (a.dbias != nullptr) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float4* pts = reinterpret_cast<float4*>(st + lnb_idx(i, h, lane));
            float4 vt = *pts;
            vt.x += dt[4 * h]; vt.y += dt[4 * h + 1]; vt.z += dt[4 * h + 2]; vt.w += dt[4 * h + 3];
            *pts = vt;
          }
        }
      }
    }
  }
  __syncthreads();
  // fold the 16 per-warp partials; column c lives at lnb_idx(c / 256, (c % 8) / 4, (c % 256) / 8) + c % 4
  for (int c = threadIdx.x; c < a.H; c += blockDim.x) {
    const int idx = lnb_idx(c >> 8, (c & 7) >> 2, (c & 255) >> 3) + (c & 3);
    float vg = 0.f, vb = 0.f, vt = 0.f;
#pragma unroll 4
    for (int w = 0; w < LNB_WARPS; ++w) {
      vg += s_ln[(w * 3 + 0) * W + idx];
      vb += s_ln[(w * 3 + 1) * W + idx];
      vt += s_ln[(w * 3 + 2) * W + idx];
    }
    if (a.dgamma != nullptr) atomicAdd(a.dgamma + c, vg);
    if (a.dbeta != nullptr) atomicAdd(a.dbeta + c, vb);
    if (a.dbias != nullptr) atomicAdd(a.dbias + c, vt);
  }
}

#define VLPK_DISPATCH_NCH(H, ...)                  \
  do {                                             \
    const int _nch = ((H) + 255) / 256;            \
    if (_nch == 1) { constexpr int NCH = 1; __VA_ARGS__; }      \
    else if (_nch == 2) { constexpr int NCH = 2; __VA_ARGS__; } \
    else if (_nch == 3) { constexpr int NCH = 3; __VA_ARGS__; } \
    else { constexpr int NCH = 4; __VA_ARGS__; }   \
  } while (0)

// every bf16 row pointer is read / written with 16-byte vectors, stats as float2: misalignment must be an argument error,
// not a device fault (null = absent)
static inline bool misaligned(const void* p, unsigned mask) { return (reinterpret_cast<uintptr_t>(p) & mask) != 0; }

static int check_ln(const LnArgs& a) {
  VLPK_CHECK_ARG(a.M > 0 && a.H > 0 && a.H % 8 == 0 && a.H <= MAXCH * 256, "layernorm: H=%d must be a multiple of 8 and <= %d",
                 a.H, MAXCH * 256);
  VLPK_CHECK_ARG(!(misaligned(a.t, 15) || misaligned(a.res, 15) || misaligned(a.gamma, 15) || misaligned(a.beta, 15) || misaligned(a.y, 15) ||
                   misaligned(a.dy, 15) || misaligned(a.dz, 15) || misaligned(a.dt, 15) || misaligned(a.stats, 7) ||
                   misaligned(a.dgamma, 3) || misaligned(a.dbeta, 3) || misaligned(a.dbias, 3)),
                 "layernorm: bf16 buffers must be 16-byte aligned (stats 8, fp32 accumulators 4)");
  return 0;
}

int launch_ln_res_drop_fwd(const LnArgs& a, cudaStream_t s) {
  VLPK_TRY(check_ln(a));
  const int wpb = 8;
  const long long grid = (a.M + wpb - 1) / wpb;
  LaunchScope scope(CAT_LN_FWD, 2.0 * a.M * a.H * (a.res ? 3 : 2) + 8.0 * a.M, s);
  VLPK_DISPATCH_NCH(a.H, VLPK_CUDA(launch_ex(ln_res_drop_fwd_kernel<NCH>, dim3(static_cast<unsigned>(grid)), dim3(wpb * 32), 0, s, 1, a)));
  return 0;
}

int launch_ln_res_drop_bwd(const LnArgs& a, cudaStream_t s) {
  VLPK_TRY(check_ln(a));
  VLPK_CHECK_ARG(a.dy != nullptr && a.stats != nullptr, "layernorm bwd: missing dy / stats");
  const int nch = (a.H + 255) / 256;
  long long grid = (a.M + LNB_WARPS - 1) / LNB_WARPS;
  if (grid > num_sms()) grid = num_sms();
  const size_t smem = static_cast<size_t>(LNB_WARPS * 3 + 1) * nch * 256 * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    VLPK_CUDA(cudaFuncSetAttribute(ln_res_drop_bwd_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (LNB_WARPS * 3 + 1) * 1 * 1024));
    VLPK_CUDA(cudaFuncSetAttribute(ln_res_drop_bwd_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (LNB_WARPS * 3 + 1) * 2 * 1024));
    VLPK_CUDA(cudaFuncSetAttribute(ln_res_drop_bwd_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (LNB_WARPS * 3 + 1) * 3 * 1024));
    VLPK_CUDA(cudaFuncSetAttribute(ln_res_drop_bwd_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (LNB_WARPS * 3 + 1) * 4 * 1024));
    attr_set = true;
  }
  LaunchScope scope(CAT_LN_BWD, 2.0 * a.M * a.H * ((a.res ? 3 : 2) + (a.dz ? 1 : 0) + (a.dt ? 1 : 0)) + 8.0 * a.M, s);
  VLPK_DISPATCH_NCH(a.H, VLPK_CUDA(launch_ex(ln_res_drop_bwd_kernel<NCH>, dim3(static_cast<unsigned>(grid)), dim3(LNB_WARPS * 32), smem, s, 1, a)));
  return 0;
}

// ------------------------------------------------------------------------------------------------
// Embeddings: gather + region splice + LN + dropout
// ------------------------------------------------------------------------------------------------
template <int NCH>
__device__ __forceinline__ void embed_row_z(const EmbedArgs& a, long long rowi, int lane, float (&z)[NCH][8], bool (&ok)[NCH]) {
  const int b = static_cast<int>(rowi / a.L), l = static_cast<int>(rowi % a.L);
  const bool vis = a.vis_input && l >= 1 && l <= a.R;
  const long long wid = a.ids[rowi];
  const long long pid = a.pos != nullptr ? a.pos[rowi] : l;
  const long long tid = a.tt != nullptr ? a.tt[rowi] : 0;
  const __nv_bfloat16* wsrc = vis ? a.vis + (static_cast<long long>(b) * a.R + (l - 1)) * a.H : a.word + wid * a.H;
  const __nv_bfloat16* psrc = vis ? a.vpe + (static_cast<long long>(b) * a.R + (l - 1)) * a.H : a.posw + pid * a.H;
  const __nv_bfloat16* tsrc = a.typew + tid * a.H;
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int col = (lane + 32 * i) * 8;
    ok[i] = col < a.H;
    if (ok[i]) {
      float w[8], p[8], t[8];
      load8(wsrc + col, w);
      load8(psrc + col, p);
      load8(tsrc + col, t);
#pragma unroll
      for (int j = 0; j < 8; ++j) z[i][j] = w[j] + p[j] + t[j];
    }
  }
}

template <int NCH>
__global__ void __launch_bounds__(256) embed_fwd_kernel(EmbedArgs a) {
  const uint64_t dseed = drop_seed(a.drop);
  const int lane = threadIdx.x & 31;
  const int wpb = blockDim.x >> 5;
  const long long rowi = static_cast<long long>(blockIdx.x) * wpb + (threadIdx.x >> 5);
  const long long M = static_cast<long long>(a.B) * a.L;
  if (rowi >= M) return;
  float z[NCH][8];
  bool ok[NCH];
  embed_row_z(a, rowi, lane, z, ok);
  float mean, rstd;
  row_stats(z, ok, a.H, a.eps, mean, rstd);
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    const int col = (lane + 32 * i) * 8;
    if (ok[i]) {
      float g[8], be[8], y[8];
      load8(a.gamma + col, g);
      load8(a.beta + col, be);
      uint32_t keep = 0xFFu;
      if (a.drop.p > 0.f) keep = dropout_keep8(dseed, a.drop.site, (rowi * a.H + col) >> 3, a.drop.thresh16);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float v = (z[i][j] - mean) * rstd * g[j] + be[j];
        y[j] = ((keep >> j) & 1u) ? v * a.drop.scale : 0.f;
      }
      store8(a.y + rowi * a.H + col, y);
    }
  }
  if (lane == 0 && a.stats != nullptr) a.stats[rowi] = make_float2(mean, rstd);
}

template <int NCH>
__global__ void __launch_bounds__(256) embed_bwd_kernel(EmbedArgs a) {
  const uint64_t dseed = drop_seed(a.drop);
  extern __shared__ float s_red[];  // [wpb][2][H]
  const int lane = threadIdx.x & 31;
  const int wib = threadIdx.x >> 5;
  const int wpb = blockDim.x >> 5;
  const long long M = static_cast<long long>(a.B) * a.L;
  float ag[NCH][8], ab[NCH][8], g[NCH][8];
  bool okc[NCH];
#pragma unroll
  for (int i = 0; i < NCH; ++i) {
    okc[i] = (lane + 32 * i) * 8 < a.H;
    if (okc[i]) load8(a.gamma + (lane + 32 * i) * 8, g[i]);
#pragma unroll
    for (int j = 0; j < 8; ++j) ag[i][j] = ab[i][j] = 0.f;
  }
  for (long long rowi = static_cast<long long>(blockIdx.x) * wpb + wib; rowi < M;
       rowi += static_cast<long long>(gridDim.x) * wpb) {
    float z[NCH][8];
    bool ok[NCH];
    embed_row_z(a, rowi, lane, z, ok);
    const float2 st = a.stats[rowi];
    const float mean = st.x, rstd = st.y;
    float gy[NCH][8];
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int col = (lane + 32 * i) * 8;
      if (ok[i]) {
        float dy[8];
        load8(a.dy + rowi * a.H + col, dy);
        uint32_t keep = 0xFFu;
        if (a.drop.p > 0.f) keep = dropout_keep8(dseed, a.drop.site, (rowi * a.H + col) >> 3, a.drop.thresh16);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float d = ((keep >> j) & 1u) ? dy[j] * a.drop.scale : 0.f;  // grad wrt LN output
          z[i][j] = (z[i][j] - mean) * rstd;                                // x-hat
          gy[i][j] = d * g[i][j];
          s1 += gy[i][j];
          s2 += gy[i][j] * z[i][j];
          ag[i][j] += d * z[i][j];
          ab[i][j] += d;
        }
      }
    }
    const float c1 = warp_sum(s1) / a.H, c2 = warp_sum(s2) / a.H;
#pragma unroll
    for (int i = 0; i < NCH; ++i) {
      const int col = (lane + 32 * i) * 8;
      if (ok[i]) {
        float dz[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) dz[j] = rstd * (gy[i][j] - c1 - z[i][j] * c2);
        store8(a.dz + rowi * a.H + col, dz);
      }
    }
  }
  float* sg = s_red + (wib * 2 + 0) * a.H;
  float* sb = s_red + (wib * 2 + 1) * a.H;
#pragma unroll
  for (int i = 0; i < NCH; ++i)
    if (okc[i]) {
      const int col = (lane + 32 * i) * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        sg[col + j] = ag[i][j];
        sb[col + j] = ab[i][j];
      }
    }
  __syncthreads();
  for (int c = threadIdx.x; c < a.H; c += blockDim.x) {
    float vg = 0.f, vb = 0.f;
    for (int w = 0; w < wpb; ++w) {
      vg += s_red[(w * 2 + 0) * a.H + c];
      vb += s_red[(w * 2 + 1) * a.H + c];
    }
    atomicAdd(a.dgamma + c, vg);
    atomicAdd(a.dbeta + c, vb);
  }
}

static int check_embed(const EmbedArgs& a) {
  VLPK_CHECK_ARG(a.B > 0 && a.L > 0 && a.H > 0 && a.H % 8 == 0 && a.H <= MAXCH * 256, "embed: bad shape B=%d L=%d H=%d", a.B,
                 a.L, a.H);
  VLPK_CHECK_ARG(!a.vis_input || (a.vis != nullptr && a.vpe != nullptr && a.R + 1 <= a.L), "embed: vis_input needs vis/vpe and R+1<=L");
  VLPK_CHECK_ARG(!(misaligned(a.word, 15) || misaligned(a.posw, 15) || misaligned(a.typew, 15) || misaligned(a.vis, 15) || misaligned(a.vpe, 15) ||
                   misaligned(a.gamma, 15) || misaligned(a.beta, 15) || misaligned(a.y, 15) || misaligned(a.dy, 15) || misaligned(a.dz, 15) ||
                   misaligned(a.stats, 7) || misaligned(a.ids, 7) || misaligned(a.tt, 7) || misaligned(a.pos, 7)),
                 "embed: bf16 buffers must be 16-byte aligned (ids / stats 8)");
  return 0;
}

int launch_embed_fwd(const EmbedArgs& a, cudaStream_t s) {
  VLPK_TRY(check_embed(a));
  const int wpb = 8;
  const long long M = static_cast<long long>(a.B) * a.L;
  LaunchScope scope(CAT_EMBED, 2.0 * M * a.H * 4, s);
  VLPK_DISPATCH_NCH(a.H, embed_fwd_kernel<NCH><<<static_cast<unsigned>((M + wpb - 1) / wpb), wpb * 32, 0, s>>>(a));
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

int launch_embed_bwd(const EmbedArgs& a, cudaStream_t s) {
  VLPK_TRY(check_embed(a));
  VLPK_CHECK_ARG(a.dy && a.dz && a.stats && a.dgamma && a.dbeta, "embed bwd: missing buffers");
  const int wpb = 8;
  const long long M = static_cast<long long>(a.B) * a.L;
  long long grid = (M + wpb - 1) / wpb;
  const long long cap = static_cast<long long>(num_sms()) * 4;
  if (grid > cap) grid = cap;
  const size_t smem = static_cast<size_t>(wpb) * 2 * a.H * sizeof(float);
  static bool attr_set = false;
  if (!attr_set) {
    VLPK_CUDA(cudaFuncSetAttribute(embed_bwd_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 1024 * 4));
    VLPK_CUDA(cudaFuncSetAttribute(embed_bwd_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 1024 * 4));
    VLPK_CUDA(cudaFuncSetAttribute(embed_bwd_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 1024 * 4));
    VLPK_CUDA(cudaFuncSetAttribute(embed_bwd_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * 2 * 1024 * 4));
    attr_set = true;
  }
  LaunchScope scope(CAT_EMBED, 2.0 * M * a.H * 5, s);
  VLPK_DISPATCH_NCH(a.H, embed_bwd_kernel<NCH><<<static_cast<unsigned>(grid), wpb * 32, smem, s>>>(a));
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// mask pack
// ------------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ bool mask_attend(T v, int mode);
template <>
__device__ __forceinline__ bool mask_attend<float>(float v, int mode) { return mode == MASK_ADDITIVE ? v > -5000.f : v != 0.f; }
template <>
__device__ __forceinline__ bool mask_attend<__nv_bfloat16>(__nv_bfloat16 v, int mode) {
  return mask_attend<float>(__bfloat162float(v), mode);
}
template <>
__device__ __forceinline__ bool mask_attend<long long>(long long v, int mode) { return v != 0; }

// One warp per mask row: lane j tests elements j, j+32, j+64, j+96 (coalesced 256-byte requests for int64 masks) and the four
// words come from __ballot_sync.  (Round 1 walked a whole 984-byte row per thread: 49 us for the [64,123,123] int64 mask.)
template <typename T>
__global__ void __launch_bounds__(256) mask_pack_kernel(const T* __restrict__ m, long long sb, long long sr, int B, int rows, int kv,
                                                              int mode, uint32_t* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (idx >= static_cast<long long>(B) * rows) return;  // warp-uniform
  const int lane = threadIdx.x & 31;
  const int b = static_cast<int>(idx / rows), r = static_cast<int>(idx % rows);
  const T* p = m + b * sb + r * sr;
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = lane + 32 * i;
    const bool on = (j < kv) && mask_attend<T>(p[j], mode);
    w[i] = __ballot_sync(0xffffffffu, on);
  }
  if (lane == 0) reinterpret_cast<uint4*>(out)[idx] = make_uint4(w[0], w[1], w[2], w[3]);
}

int launch_mask_pack(const void* mask, int dtype, int mode, int B, int rows, int kv, long long stride_b, long long stride_r,
                     uint32_t* out, cudaStream_t s) {
  VLPK_CHECK_ARG(B > 0 && rows > 0 && kv > 0 && kv <= 128, "mask_pack: kv=%d must be in [1,128]", kv);
  VLPK_CHECK_ARG(!misaligned(out, 15), "mask_pack: the bitmask buffer must be 16-byte aligned");
  const long long n = static_cast<long long>(B) * rows;
  const unsigned gridw = static_cast<unsigned>((n + 7) / 8);
  LaunchScope scope(CAT_MISC, 0.0, s);
  switch (dtype) {
    case VLPK_DT_F32: mask_pack_kernel<float><<<gridw, 256, 0, s>>>(static_cast<const float*>(mask), stride_b, stride_r, B, rows, kv, mode, out); break;
    case VLPK_DT_BF16: mask_pack_kernel<__nv_bfloat16><<<gridw, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(mask), stride_b, stride_r, B, rows, kv, mode, out); break;
    case VLPK_DT_I64: mask_pack_kernel<long long><<<gridw, 256, 0, s>>>(static_cast<const long long*>(mask), stride_b, stride_r, B, rows, kv, mode, out); break;
    default: set_error("mask_pack: unsupported dtype %d", dtype); return -1;
  }
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

// Device-side synthesis of the loader's self-attention mask (vlp/seq2seq_loader.py:291-301), straight into the packed form: the
// reference builds a [L,L] int64 matrix per sample on a CPU worker and ships 121 KB per sample to the GPU; here three integers per
// sample do.  len_a = region tokens, len_b = text tokens, st = len_a + 2, en = len_a + len_b + 3 (= tokens incl. [CLS] / 2 x [SEP]):
//   s2s : every row attends to columns [0, st); rows in [st, en) additionally to columns [st, row]   (causal over the text)
//   bi  : every row attends to columns [0, en)
__global__ void __launch_bounds__(256) mask_synth_kernel(const int* __restrict__ len_b, const int* __restrict__ mode, int len_a, int B, int L,
                                                          uint32_t* __restrict__ out) {
  const long long idx = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (idx >= static_cast<long long>(B) * L) return;  // warp-uniform
  const int lane = threadIdx.x & 31;
  const int b = static_cast<int>(idx / L), r = static_cast<int>(idx % L);
  const int st = len_a + 2, en = min(len_a + len_b[b] + 3, L);
  const bool s2s = mode[b] != 0;
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int j = lane + 32 * i;
    bool on;
    if (s2s) on = (j < st) || (r >= st && r < en && j >= st && j <= r);
    else on = j < en;
    w[i] = __ballot_sync(0xffffffffu, on && j < L);
  }
  if (lane == 0) reinterpret_cast<uint4*>(out)[idx] = make_uint4(w[0], w[1], w[2], w[3]);
}

int launch_mask_synth(const int* len_b, const int* mode, int len_a, int B, int L, uint32_t* out, cudaStream_t s) {
  VLPK_CHECK_ARG(len_b != nullptr && mode != nullptr && out != nullptr, "mask_synth: null pointer");
  VLPK_CHECK_ARG(B > 0 && L > 0 && L <= 128 && len_a >= 0 && len_a + 3 <= L, "mask_synth: B=%d L=%d len_a=%d", B, L, len_a);
  VLPK_CHECK_ARG(!misaligned(out, 15), "mask_synth: the bitmask buffer must be 16-byte aligned");
  const long long n = static_cast<long long>(B) * L;
  LaunchScope scope(CAT_MISC, 0.0, s);
  mask_synth_kernel<<<static_cast<unsigned>((n + 7) / 8), 256, 0, s>>>(len_b, mode, len_a, B, L, out);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

// ------------------------------------------------------------------------------------------------
// column sums (bias gradients) and fp32 -> bf16 conversion
// ------------------------------------------------------------------------------------------------
// Block = 8 column-groups (8 columns = 16 bytes each) x 32 row-lanes over a [COLSUM_ROWS x 64] slab: every 128-byte
// line is consumed whole by 8 adjacent threads, each thread keeps 8 independent 16-byte loads in flight, and the
// 32 row-lane partials are folded through shared memory before one atomicAdd per column per block.
static constexpr int COLSUM_ROWS = 256;
__global__ void __launch_bounds__(256) colsum_kernel(const __nv_bfloat16* __restrict__ x, long long ld, long long M, int N,
                                                      float* __restrict__ out) {
  __shared__ float s_part[32][65];
  const int cg = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int col = blockIdx.x * 64 + cg * 8;
  const long long r0 = static_cast<long long>(blockIdx.y) * COLSUM_ROWS;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (col < N) {
#pragma unroll
    for (int i = 0; i < COLSUM_ROWS / 32; ++i) {
      const long long r = r0 + rl + 32 * i;
      if (r < M) {
        float v[8];
        load8(x + r * ld + col, v);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] += v[j];
      }
    }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) s_part[rl][cg * 8 + j] = acc[j];
  __syncthreads();
  if (threadIdx.x < 64) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) t += s_part[i][threadIdx.x];
    const int c = blockIdx.x * 64 + threadIdx.x;
    if (c < N) atomicAdd(out + c, t);
  }
}

int launch_colsum(const void* x, long long ld, long long M, int N, float* out, cudaStream_t s) {
  VLPK_CHECK_ARG(N % 8 == 0 && ld % 8 == 0, "colsum: N=%d ld=%lld must be multiples of 8", N, ld);
  VLPK_CHECK_ARG(M > 0 && !misaligned(x, 15) && !misaligned(out, 3), "colsum: M=%lld, x must be 16-byte aligned", M);
  dim3 grid((N + 63) / 64, static_cast<unsigned>((M + COLSUM_ROWS - 1) / COLSUM_ROWS));
  LaunchScope scope(CAT_MISC, 2.0 * M * N, s);
  colsum_kernel<<<grid, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(x), ld, M, N, out);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

// out[i] += sum over p of part[p * n + i], added in the order p = 0, 1, ... : the fixed-order second stage of a reduction
// whose first stage wrote one partial per CTA (attention bias gradients) or per split (split-K), so that the result does not
// depend on the order in which those CTAs finish.
__global__ void __launch_bounds__(256) sum_parts_kernel(const float* __restrict__ part, int parts, long long n, float* __restrict__ out) {
  for (long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += static_cast<long long>(gridDim.x) * blockDim.x) {
    float t = 0.f;
    for (int p = 0; p < parts; ++p) t += part[p * n + i];
    out[i] += t;
  }
}

int launch_sum_parts(const float* part, int parts, long long n, float* out, cudaStream_t s) {
  VLPK_CHECK_ARG(part != nullptr && out != nullptr && parts >= 1 && n >= 1, "sum_parts: parts=%d n=%lld", parts, n);
  long long blocks = (n + 255) / 256;
  if (blocks > 4LL * num_sms()) blocks = 4LL * num_sms();
  LaunchScope scope(CAT_MISC, 4.0 * n * (parts + 2), s);
  sum_parts_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(part, parts, n, out);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

// Test support: the keep-decisions the kernels take for dropout site `site` under `seed`, element by element (1 = keep), produced by
// the same dropout_keep8() every fused epilogue / row kernel calls — tests feed these masks to the fp32 oracle to check the
// dropout-on (training) configuration numerically.
__global__ void __launch_bounds__(256) dropout_mask_kernel(DropoutCfg d, long long n8, unsigned char* __restrict__ out) {
  const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n8) return;
  const uint32_t keep = dropout_keep8(drop_seed(d), d.site, static_cast<uint64_t>(i), d.thresh16);
  uint2 v;
  v.x = (keep & 1u) | ((keep >> 1 & 1u) << 8) | ((keep >> 2 & 1u) << 16) | ((keep >> 3 & 1u) << 24);
  v.y = (keep >> 4 & 1u) | ((keep >> 5 & 1u) << 8) | ((keep >> 6 & 1u) << 16) | ((keep >> 7 & 1u) << 24);
  reinterpret_cast<uint2*>(out)[i] = v;
}

int launch_dropout_mask(const DropoutCfg& d, long long n, unsigned char* out, cudaStream_t s) {
  VLPK_CHECK_ARG(n > 0 && n % 8 == 0 && !misaligned(out, 7), "dropout_mask: n=%lld must be a positive multiple of 8, out 8-byte aligned", n);
  VLPK_CHECK_ARG(d.p > 0.f && d.p < 1.f, "dropout_mask: p=%g out of (0,1)", d.p);
  const long long n8 = n / 8;
  dropout_mask_kernel<<<static_cast<unsigned>((n8 + 255) / 256), 256, 0, s>>>(d, n8, out);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

__global__ void __launch_bounds__(256) f32_to_bf16_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ y, long long n) {
  const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const float4 a = __ldg(reinterpret_cast<const float4*>(x + i));
    const float4 b = __ldg(reinterpret_cast<const float4*>(x + i + 4));
    uint4 u;
    u.x = pack_bf16x2(a.x, a.y);
    u.y = pack_bf16x2(a.z, a.w);
    u.z = pack_bf16x2(b.x, b.y);
    u.w = pack_bf16x2(b.z, b.w);
    *reinterpret_cast<uint4*>(y + i) = u;
  } else {
    for (long long k = i; k < n; ++k) y[k] = __float2bfloat16_rn(x[k]);
  }
}

int launch_f32_to_bf16(const float* x, void* y, long long n, cudaStream_t s) {
  if (n <= 0) return 0;
  VLPK_CHECK_ARG((reinterpret_cast<uintptr_t>(x) & 15u) == 0 && (reinterpret_cast<uintptr_t>(y) & 15u) == 0,
                 "f32_to_bf16: pointers must be 16-byte aligned");
  const long long nthreads = (n + 7) / 8;
  LaunchScope scope(CAT_MISC, 6.0 * n, s);
  f32_to_bf16_kernel<<<static_cast<unsigned>((nthreads + 255) / 256), 256, 0, s>>>(x, static_cast<__nv_bfloat16*>(y), n);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace vlpk
