// vlp_b200 — masked-softmax attention core for VLP's [image-region | text-token] sequence (L <= 128).
//
// Reference semantics (pytorch_pretrained_bert/modeling.py:279-302):
//   S = Q K^T / sqrt(64) + mask_add ; P = softmax(S) ; P = dropout(P) ; ctx = P V
// where mask_add is 0 / -10000 (modeling.py:832).  One whole sequence (123 -> 128 rows) is a single
// 128-row tile, so S and P live only in registers / shared memory: the reference's
// [B,12,L,L] score tensor (written + read ~6x per layer, SURVEY.md §8a a5) never touches HBM.
//
// One CTA per (head, batch), two warpgroups: warpgroup g owns query rows [64 g, 64 g + 64) and all 128 key columns, so
// every row reduction stays inside a quad of threads (wgmma accumulator layout, see wgmma.cuh).
//   fwd : TMA Q,K,V -> S=QK^T (wgmma, registers) -> scale+bitmask+softmax in registers -> Philox dropout
//         -> P (bf16, registers) -> O=PV (wgmma with A from registers, V read MN-major straight from its [kv,d] tile)
//         -> O/rowsum -> TMA store.  Saves only logsumexp per row for backward.
//   bwd : recompute S,P from Q,K + logsumexp; dP=dO V^T; dS=P*(dP-delta)/8; dV=P^T dO; dK=dS^T Q; dQ=dS K
//         — five wgmma chains, all operands fed from the same TMA tiles via K-major / MN-major descriptors.
#include "attn.cuh"
#include "host.cuh"
#include "rowops.cuh"

namespace vlpk {

static constexpr int HD = 64;         // head dim (VLP/BERT-base: 768/12)
static constexpr int TL = 128;        // tile rows (max sequence length)
static constexpr int TILE_B = TL * 128;  // bytes of one [128 x 64] bf16 tile
static constexpr float LOG2E = 1.4426950408889634f;
static constexpr float LN2 = 0.6931471805599453f;
static constexpr int ATT_THREADS = 256;

struct AttnTmaps {
  CUtensorMap q, k, v, o;         // fwd: o = ctx ; bwd: o = dO (load)
  CUtensorMap dq, dk, dv;         // bwd outputs
};

struct AttnArgs {
  int B, heads, Lq, Lkv;
  const uint32_t* mask_bits;  // [B, mask_rows, 4] ; bit j of row i set = attend to kv position j
  int mask_rows;              // Lq, or 1 when the mask broadcasts over query rows
  float* lse;                 // [B, heads, Lq] natural-log logsumexp of the scaled+masked scores
  const __nv_bfloat16* o_ptr;   // bwd: forward output ctx [B, Lq, ld_o] (for delta)
  const __nv_bfloat16* do_ptr;  // bwd: dO, same layout
  long long ld_o;
  DropoutCfg drop;
  unsigned char* keep_out;  // fwd, optional: packed dropout keep-decisions, 16 bytes per (sequence, head, query row)
  float* dbias_part;  // bwd, optional: [B][3 * heads * 64] fp32 per-sequence column sums of dQ | dK | dV (q/k/v bias gradients)
};

// bf16 pair (columns col, col + 1) into a [rows x 64] bf16 tile stored with the 128-byte swizzle of the TMA boxes
__device__ __forceinline__ void sw_write_pair(uint8_t* tile, int row, int col, uint32_t v) {
  *reinterpret_cast<uint32_t*>(tile + row * 128 + (((col >> 3) ^ (row & 7)) << 4) + (col & 7) * 2) = v;
}

// Per-thread view of one warpgroup's accumulator rows: element i of an m64nN fragment lies in row fr + 8 * ((i >> 1) & 1) of
// the warpgroup's 64 rows and column 8 * (i >> 2) + fc + (i & 1).
struct Frag {
  int fr, fc;
  __device__ __forceinline__ Frag() {
    const int t = threadIdx.x & 127, lane = threadIdx.x & 31;
    fr = (t >> 5) * 16 + (lane >> 2);
    fc = (lane & 3) * 2;
  }
};

__device__ __forceinline__ float quad_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  return fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}

// Keep-decisions of the 128 key columns of query rows r (h = 0) and r + 8 (h = 1): word w bit j = column 32 w + j, i.e. byte g of
// word w = dropout_keep8(seed, site, (row_elem0 + 32 w + 8 g) / 8).  The four threads of a quad each evaluate one word per row
// (or read the forward's bytes) and exchange them.
__device__ __forceinline__ void attn_keep_words(const DropoutCfg& d, uint64_t dseed, const uint64_t (&row_elem0)[2], uint32_t (&kw)[2][4]) {
  const int lane = threadIdx.x & 31, qi = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    uint32_t mine = 0xFFFFFFFFu;
    if (d.p > 0.f) {
      if (d.bits != nullptr) {
        mine = __ldg(reinterpret_cast<const uint32_t*>(d.bits + (row_elem0[h] >> 3)) + qi);
      } else {
        mine = 0;
#pragma unroll
        for (int g = 0; g < 4; ++g) mine |= dropout_keep8(dseed, d.site, (row_elem0[h] + qi * 32 + g * 8) >> 3, d.thresh16) << (8 * g);
      }
    }
#pragma unroll
    for (int w = 0; w < 4; ++w) kw[h][w] = __shfl_sync(0xffffffffu, mine, (lane & ~3) | w);
  }
}

// Scaled + masked score in the log2 domain: bit set -> attend (add 0) ; bit clear -> add -10000 (reference additive mask) ;
// col >= Lkv -> -inf.
__device__ __forceinline__ float score(float s, const uint32_t (&mw)[4], int col, int Lkv) {
  const float x = s * (0.125f * LOG2E) + (((mw[col >> 5] >> (col & 31)) & 1u) ? 0.f : -10000.0f * LOG2E);
  return col < Lkv ? x : -INFINITY;
}

__device__ __forceinline__ void load_mask_words(const AttnArgs& a, int b, int row, uint32_t (&mw)[4]) {
  const int mr = (a.mask_rows == 1) ? 0 : min(row, a.mask_rows - 1);
  const uint4 m4 = __ldg(reinterpret_cast<const uint4*>(a.mask_bits + (static_cast<size_t>(b) * a.mask_rows + mr) * 4));
  mw[0] = m4.x; mw[1] = m4.y; mw[2] = m4.z; mw[3] = m4.w;
}

// ------------------------------------------------------------------------------------------------
// forward  (256 threads, 48 KB smem: Q | K | V; the Q tile is reused as output staging)
// ------------------------------------------------------------------------------------------------
struct FwdSmem {
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = TILE_B;
  static constexpr int OFF_V = 2 * TILE_B;
  static constexpr int OFF_BAR = 3 * TILE_B;
  static constexpr int TOTAL = OFF_BAR + 16;
  static constexpr int DYN = TOTAL + 1024;
};

__global__ void __launch_bounds__(ATT_THREADS, 2) attn_fwd_kernel(const __grid_constant__ AttnTmaps tm, const AttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem + FwdSmem::OFF_Q;
  uint8_t* sK = smem + FwdSmem::OFF_K;
  uint8_t* sV = smem + FwdSmem::OFF_V;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FwdSmem::OFF_BAR);
  uint64_t* bar_qk = &bars[0];
  uint64_t* bar_v = &bars[1];

  pdl_launch_dependents();
  const int h = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x, wg = tid >> 7;
  const Frag f;
  const int qi = tid & 3;

  if (tid == 0) {
    tma_prefetch_desc(&tm.q);
    tma_prefetch_desc(&tm.k);
    tma_prefetch_desc(&tm.v);
    tma_prefetch_desc(&tm.o);
    mbar_init(bar_qk, 1);
    mbar_init(bar_v, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar_qk, 2 * TILE_B);
    tma_load_3d(sQ, &tm.q, bar_qk, h * HD, 0, b);
    tma_load_3d(sK, &tm.k, bar_qk, h * HD, 0, b);
    mbar_arrive_expect_tx(bar_v, TILE_B);
    tma_load_3d(sV, &tm.v, bar_v, h * HD, 0, b);
  }

  const int row[2] = {wg * 64 + f.fr, wg * 64 + f.fr + 8};
  uint32_t mw[2][4];
  uint64_t row_elem0[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    load_mask_words(a, b, row[hh], mw[hh]);
    row_elem0[hh] = ((static_cast<uint64_t>(b) * a.heads + h) * a.Lq + min(row[hh], a.Lq - 1)) * TL;
  }

  // S = Q K^T for this warpgroup's 64 query rows
  float s[64];
  mbar_wait(bar_qk, 0);
  {
    const uint32_t q0 = smem_u32(sQ) + wg * 8192, k0 = smem_u32(sK);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k)
      wgmma_m64n128k16_ss<0, 0>(s, wgmma_desc_sw128(q0 + k * 32, 16, 1024), wgmma_desc_sw128(k0 + k * 32, 16, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
  }
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int hh = (i >> 1) & 1;
    s[i] = score(s[i], mw[hh], 8 * (i >> 2) + f.fc + (i & 1), a.Lkv);
    mx[hh] = fmaxf(mx[hh], s[i]);
  }
  mx[0] = quad_max(mx[0]);  // Lkv >= 1 guarantees a finite maximum
  mx[1] = quad_max(mx[1]);
  uint32_t kw[2][4];  // evaluated here rather than up front: keeps them out of the registers live across the S = QK^T wgmma
  attn_keep_words(a.drop, drop_seed(a.drop), row_elem0, kw);
  if (a.keep_out != nullptr) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      if (row[hh] < a.Lq) reinterpret_cast<uint32_t*>(a.keep_out + (row_elem0[hh] >> 3))[qi] = kw[hh][qi];
  }
  // exponentiate, dropout, pack P (bf16) straight into the A fragments of P V
  float rsum[2] = {0.f, 0.f}, lsum[2] = {0.f, 0.f};
  uint32_t pa[8][4];
#pragma unroll
  for (int i = 0; i < 64; i += 2) {
    const int hh = (i >> 1) & 1, col = 8 * (i >> 2) + f.fc;
    const float x0 = fast_ex2(s[i] - mx[hh]), x1 = fast_ex2(s[i + 1] - mx[hh]);
    lsum[hh] += x0 + x1;                                   // exact sum -> logsumexp (backward recomputes P from it)
    const float e0 = bf16_round(x0), e1 = bf16_round(x1);  // the tensor core sees bf16 P: normalise O by the sum of
    rsum[hh] += e0 + e1;                                   // exactly those values
    const uint32_t keep = kw[hh][col >> 5] >> (col & 31);
    const float p0 = (keep & 1u) ? e0 * a.drop.scale : 0.f;
    const float p1 = (keep & 2u) ? e1 * a.drop.scale : 0.f;
    pa[i >> 3][(i >> 1) & 3] = pack_bf16x2(p0, p1);
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    rsum[hh] = quad_sum(rsum[hh]);
    lsum[hh] = quad_sum(lsum[hh]);
    if (qi == 0 && a.lse != nullptr && row[hh] < a.Lq)
      a.lse[(static_cast<size_t>(b) * a.heads + h) * a.Lq + row[hh]] = (mx[hh] + log2f(lsum[hh])) * LN2;
  }
  // O = P V
  float o[32];
  mbar_wait(bar_v, 0);
  {
    const uint32_t v0 = smem_u32(sV);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TL / 16; ++k) wgmma_m64n64k16_rs<1>(o, pa[k], wgmma_desc_sw128(v0 + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(o);
  }
  // O / rowsum -> bf16 -> this warpgroup's half of the (dead) Q tile -> one TMA store of the whole tile
  const float inv[2] = {1.0f / rsum[0], 1.0f / rsum[1]};
  uint8_t* stg = sQ + wg * 8192;
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int hh = (i >> 1) & 1;
    sw_write_pair(stg, f.fr + 8 * hh, 8 * (i >> 2) + f.fc, pack_bf16x2(o[i] * inv[hh], o[i + 1] * inv[hh]));
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    tma_store_3d(&tm.o, sQ, h * HD, 0, b);
    tma_store_commit();
    tma_store_wait<0>();
  }
}

// ------------------------------------------------------------------------------------------------
// backward  (256 threads, 96 KB smem: Q | K | V | dO | a [128 x 128] bf16 buffer holding P (for dV) and then dS (for dK))
// ------------------------------------------------------------------------------------------------
struct BwdSmem {
  static constexpr int OFF_Q = 0;            // later dQ staging
  static constexpr int OFF_K = TILE_B;       // later dK staging
  static constexpr int OFF_V = 2 * TILE_B;   // later dV staging
  static constexpr int OFF_DO = 3 * TILE_B;
  static constexpr int OFF_PD = 4 * TILE_B;  // 2 atoms of [128 q x 64 kv]: P, then dS
  static constexpr int OFF_BAR = 6 * TILE_B;
  static constexpr int TOTAL = OFF_BAR + 16;
  static constexpr int DYN = TOTAL + 1024;
};

__global__ void __launch_bounds__(ATT_THREADS, 1) attn_bwd_kernel(const __grid_constant__ AttnTmaps tm, const AttnArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem + BwdSmem::OFF_Q;
  uint8_t* sK = smem + BwdSmem::OFF_K;
  uint8_t* sV = smem + BwdSmem::OFF_V;
  uint8_t* sdO = smem + BwdSmem::OFF_DO;
  uint8_t* sPD = smem + BwdSmem::OFF_PD;
  uint64_t* bar_in = reinterpret_cast<uint64_t*>(smem + BwdSmem::OFF_BAR);

  pdl_launch_dependents();
  const int h = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x, wg = tid >> 7;
  const Frag f;

  if (tid == 0) {
    tma_prefetch_desc(&tm.q);
    tma_prefetch_desc(&tm.k);
    tma_prefetch_desc(&tm.v);
    tma_prefetch_desc(&tm.o);
    mbar_init(bar_in, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (tid == 0) {
    mbar_arrive_expect_tx(bar_in, 4 * TILE_B);
    tma_load_3d(sQ, &tm.q, bar_in, h * HD, 0, b);
    tma_load_3d(sK, &tm.k, bar_in, h * HD, 0, b);
    tma_load_3d(sV, &tm.v, bar_in, h * HD, 0, b);
    tma_load_3d(sdO, &tm.o, bar_in, h * HD, 0, b);
  }

  const int row[2] = {wg * 64 + f.fr, wg * 64 + f.fr + 8};
  uint32_t mw[2][4];
  uint64_t row_elem0[2];
  float lse2[2];
  bool row_ok[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    load_mask_words(a, b, row[hh], mw[hh]);
    row_elem0[hh] = ((static_cast<uint64_t>(b) * a.heads + h) * a.Lq + min(row[hh], a.Lq - 1)) * TL;
    row_ok[hh] = row[hh] < a.Lq;
    lse2[hh] = row_ok[hh] ? a.lse[(static_cast<size_t>(b) * a.heads + h) * a.Lq + row[hh]] * LOG2E : 0.f;
  }
  uint32_t kw[2][4];  // dropout keep mask of this thread's rows (forward's bytes when available, else Philox evaluated once)
  attn_keep_words(a.drop, drop_seed(a.drop), row_elem0, kw);

  // S = Q K^T and dP = dO V^T for this warpgroup's 64 query rows
  float s[64], dp[64];
  mbar_wait(bar_in, 0);
  {
    const uint32_t q0 = smem_u32(sQ) + wg * 8192, k0 = smem_u32(sK), do0 = smem_u32(sdO) + wg * 8192, v0 = smem_u32(sV);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < HD / 16; ++k)
      wgmma_m64n128k16_ss<0, 0>(s, wgmma_desc_sw128(q0 + k * 32, 16, 1024), wgmma_desc_sw128(k0 + k * 32, 16, 1024), k > 0 ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < HD / 16; ++k)
      wgmma_m64n128k16_ss<0, 0>(dp, wgmma_desc_sw128(do0 + k * 32, 16, 1024), wgmma_desc_sw128(v0 + k * 32, 16, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(s);
    reg_fence(dp);
  }
  // P (recomputed from the logsumexp; 0 for columns >= Lkv and rows >= Lq) and the dropout-masked dP.
  // delta_r = sum_j P_rj dP_rj with the SAME recomputed P that dS multiplies with, so that sum_j dS_rj = 0 holds to fp32
  // round-off.  (The usual shortcut delta = dO . O inherits the bf16 rounding of O; when keys / values share a large common
  // component — VLP's 100 near-identical region rows at initialisation — that error is amplified by |mean| / |spread| and
  // reached 10-20 % in dQ/dK on the VQA parity case.)
  float delta[2] = {0.f, 0.f};
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int hh = (i >> 1) & 1, col = 8 * (i >> 2) + f.fc + (i & 1);
    const float p = row_ok[hh] ? fast_ex2(score(s[i], mw[hh], col, a.Lkv) - lse2[hh]) : 0.f;
    const bool kp = (kw[hh][col >> 5] >> (col & 31)) & 1u;
    const float dpm = kp ? dp[i] * a.drop.scale : 0.f;
    delta[hh] = fmaf(p, dpm, delta[hh]);
    s[i] = p;
    dp[i] = dpm;
  }
  delta[0] = quad_sum(delta[0]);
  delta[1] = quad_sum(delta[1]);
  uint32_t dsa[8][4];  // dS (bf16) as the A fragments of dQ = dS K
#pragma unroll
  for (int i = 0; i < 64; i += 2) {
    const int hh = (i >> 1) & 1, col = 8 * (i >> 2) + f.fc;
    const uint32_t keep = kw[hh][col >> 5] >> (col & 31);
    const float p0 = (keep & 1u) ? s[i] * a.drop.scale : 0.f, p1 = (keep & 2u) ? s[i + 1] * a.drop.scale : 0.f;
    sw_write_pair(sPD + (col >> 6) * TILE_B, row[hh], col & 63, pack_bf16x2(p0, p1));
    dsa[i >> 3][(i >> 1) & 3] = pack_bf16x2(s[i] * (dp[i] - delta[hh]) * 0.125f, s[i + 1] * (dp[i + 1] - delta[hh]) * 0.125f);
  }
  fence_proxy_async_smem();
  __syncthreads();

  // dV[kv, d] = sum_q Pd[q, kv] dO[q, d] for kv rows [64 wg, 64 wg + 64): A = Pd^T (MN-major), B = dO (MN-major)
  float dv[32];
  {
    const uint32_t p0 = smem_u32(sPD) + wg * TILE_B, do0 = smem_u32(sdO);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TL / 16; ++k)
      wgmma_m64n64k16_ss<1, 1>(dv, wgmma_desc_sw128(p0 + k * 2048, 8192, 1024), wgmma_desc_sw128(do0 + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dv);
  }
  __syncthreads();  // both warpgroups have read P: the buffer can take dS
#pragma unroll
  for (int c = 0; c < 8; ++c)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int hh = e & 1, col = 16 * c + 8 * (e >> 1) + f.fc;
      sw_write_pair(sPD + (col >> 6) * TILE_B, row[hh], col & 63, dsa[c][e]);
    }
  fence_proxy_async_smem();
  __syncthreads();

  // dK[kv, d] = sum_q dS[q, kv] Q[q, d]  (A = dS^T from shared memory) ; dQ[q, d] = sum_kv dS[q, kv] K[kv, d]  (A = dS registers)
  float dk[32], dq[32];
  {
    const uint32_t p0 = smem_u32(sPD) + wg * TILE_B, q0 = smem_u32(sQ), k0 = smem_u32(sK);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < TL / 16; ++k)
      wgmma_m64n64k16_ss<1, 1>(dk, wgmma_desc_sw128(p0 + k * 2048, 8192, 1024), wgmma_desc_sw128(q0 + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
#pragma unroll
    for (int k = 0; k < TL / 16; ++k) wgmma_m64n64k16_rs<1>(dq, dsa[k], wgmma_desc_sw128(k0 + k * 2048, 8192, 1024), k > 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(dk);
    reg_fence(dq);
  }
  __syncthreads();  // every wgmma has read Q / K / V: reuse them as output staging
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int r = wg * 64 + f.fr + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + f.fc;
    sw_write_pair(sQ, r, col, pack_bf16x2(dq[i], dq[i + 1]));
    sw_write_pair(sK, r, col, pack_bf16x2(dk[i], dk[i + 1]));
    sw_write_pair(sV, r, col, pack_bf16x2(dv[i], dv[i + 1]));
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    tma_store_3d(&tm.dq, sQ, h * HD, 0, b);
    tma_store_3d(&tm.dk, sK, h * HD, 0, b);
    tma_store_3d(&tm.dv, sV, h * HD, 0, b);
    tma_store_commit();
  }
  if (a.dbias_part != nullptr && tid < 192) {
    // this sequence's share of the q/k/v bias gradients = column sums of the staged dQ / dK / dV tiles (rows >= L are exactly
    // zero); written, not added, so that launch_sum_parts can add the sequences in a fixed order
    const int o = tid >> 6, c = tid & 63;
    const uint8_t* stg = (o == 0) ? sQ : (o == 1 ? sK : sV);
    float acc = 0.f;
#pragma unroll 8
    for (int r = 0; r < TL; ++r)
      acc += __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(stg + r * 128 + (((c >> 3) ^ (r & 7)) << 4) + (c & 7) * 2));
    a.dbias_part[static_cast<size_t>(b) * 3 * a.heads * HD + o * a.heads * HD + h * HD + c] = acc;
  }
  if (tid == 0) tma_store_wait<0>();
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
static int make_seq_tmap(CUtensorMap* out, const void* base, int width, int L, int B, int64_t ld, int64_t batch_stride = 0) {
  uint64_t dims[3] = {static_cast<uint64_t>(width), static_cast<uint64_t>(L), static_cast<uint64_t>(B)};
  uint64_t strides[2] = {static_cast<uint64_t>(ld) * 2,
                         batch_stride > 0 ? static_cast<uint64_t>(batch_stride) * 2 : static_cast<uint64_t>(ld) * 2 * static_cast<uint64_t>(L)};
  uint32_t box[3] = {HD, TL, 1};
  return make_tmap(out, TM_BF16, 3, base, dims, strides, box);
}

static int check_common(const AttnDesc& d) {
  VLPK_CHECK_ARG(d.head_dim == HD, "attention: head_dim %d unsupported (only 64)", d.head_dim);
  VLPK_CHECK_ARG(d.Lq >= 1 && d.Lq <= TL && d.Lkv >= 1 && d.Lkv <= TL, "attention: Lq=%d Lkv=%d must be in [1,128]",
                 d.Lq, d.Lkv);
  VLPK_CHECK_ARG(d.B >= 1 && d.heads >= 1, "attention: B=%d heads=%d", d.B, d.heads);
  VLPK_CHECK_ARG(d.mask_bits != nullptr && (d.mask_rows == 1 || d.mask_rows == d.Lq), "attention: mask rows %d",
                 d.mask_rows);
  return 0;
}

int launch_attn_fwd(const AttnDesc& d, cudaStream_t stream) {
  VLPK_TRY(check_common(d));
  const int width = d.heads * HD;
  AttnTmaps tm;
  memset(&tm, 0, sizeof(tm));
  VLPK_TRY(make_seq_tmap(&tm.q, d.q, width, d.Lq, d.B, d.ld_q));
  VLPK_TRY(make_seq_tmap(&tm.k, d.k, width, d.Lkv, d.B, d.ld_kv, d.kv_batch_stride));
  VLPK_TRY(make_seq_tmap(&tm.v, d.v, width, d.Lkv, d.B, d.ld_kv, d.kv_batch_stride));
  VLPK_TRY(make_seq_tmap(&tm.o, d.o, width, d.Lq, d.B, d.ld_o));
  tm.dq = tm.dk = tm.dv = tm.o;
  AttnArgs a;
  a.B = d.B; a.heads = d.heads; a.Lq = d.Lq; a.Lkv = d.Lkv;
  a.mask_bits = d.mask_bits; a.mask_rows = d.mask_rows;
  a.lse = d.lse; a.o_ptr = nullptr; a.do_ptr = nullptr; a.ld_o = d.ld_o;
  a.drop = d.drop;
  a.keep_out = d.keep_out;
  a.dbias_part = nullptr;
  static bool attr_set = false;
  if (!attr_set) {
    VLPK_CUDA(cudaFuncSetAttribute(attn_fwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FwdSmem::DYN));
    attr_set = true;
  }
  LaunchScope scope(CAT_ATTN_FWD, 4.0 * d.B * d.heads * d.Lq * d.Lkv * HD, stream);
  VLPK_CUDA(launch_ex(attn_fwd_kernel, dim3(d.heads, d.B), dim3(ATT_THREADS), FwdSmem::DYN, stream, 1, tm, a));
  return 0;
}

int launch_attn_bwd(const AttnDesc& d, cudaStream_t stream) {
  VLPK_TRY(check_common(d));
  VLPK_CHECK_ARG(d.Lq == d.Lkv, "attention bwd: Lq must equal Lkv (training path)");
  VLPK_CHECK_ARG(d.lse != nullptr && d.d_o != nullptr && d.dq && d.dk && d.dv, "attention bwd: missing buffers");
  const int width = d.heads * HD;
  AttnTmaps tm;
  memset(&tm, 0, sizeof(tm));
  VLPK_TRY(make_seq_tmap(&tm.q, d.q, width, d.Lq, d.B, d.ld_q));
  VLPK_TRY(make_seq_tmap(&tm.k, d.k, width, d.Lkv, d.B, d.ld_kv));
  VLPK_TRY(make_seq_tmap(&tm.v, d.v, width, d.Lkv, d.B, d.ld_kv));
  VLPK_TRY(make_seq_tmap(&tm.o, d.d_o, width, d.Lq, d.B, d.ld_o));
  VLPK_TRY(make_seq_tmap(&tm.dq, d.dq, width, d.Lq, d.B, d.ld_dqkv));
  VLPK_TRY(make_seq_tmap(&tm.dk, d.dk, width, d.Lkv, d.B, d.ld_dqkv));
  VLPK_TRY(make_seq_tmap(&tm.dv, d.dv, width, d.Lkv, d.B, d.ld_dqkv));
  AttnArgs a;
  a.B = d.B; a.heads = d.heads; a.Lq = d.Lq; a.Lkv = d.Lkv;
  a.mask_bits = d.mask_bits; a.mask_rows = d.mask_rows;
  a.lse = d.lse;
  a.o_ptr = reinterpret_cast<const __nv_bfloat16*>(d.o);
  a.do_ptr = reinterpret_cast<const __nv_bfloat16*>(d.d_o);
  a.ld_o = d.ld_o;
  a.drop = d.drop;
  a.keep_out = nullptr;
  a.dbias_part = nullptr;
  const long long nbias = 3LL * d.heads * HD;
  if (d.dbias != nullptr) {
    a.dbias_part = scratch_f32(SCRATCH_ATTN_DBIAS, static_cast<size_t>(d.B) * nbias, stream);
    if (a.dbias_part == nullptr) return -1;
  }
  static bool attr_set = false;
  if (!attr_set) {
    VLPK_CUDA(cudaFuncSetAttribute(attn_bwd_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BwdSmem::DYN));
    attr_set = true;
  }
  {
    LaunchScope scope(CAT_ATTN_BWD, 10.0 * d.B * d.heads * d.Lq * d.Lkv * HD, stream);
    VLPK_CUDA(launch_ex(attn_bwd_kernel, dim3(d.heads, d.B), dim3(ATT_THREADS), BwdSmem::DYN, stream, 1, tm, a));
  }
  if (d.dbias != nullptr) VLPK_TRY(launch_sum_parts(a.dbias_part, d.B, nbias, d.dbias, stream));
  return 0;
}

}  // namespace vlpk
