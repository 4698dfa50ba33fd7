// vlp_b200 — masked-softmax attention core for VLP's [image-region | text-token] sequence: single-tile kernels for L <= 128, KV-tiled ones up to 512.
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
// shared-prefix K/V (vlpk_layer_cached_group_fwd, vlpk_encoder_score_group_fwd): hypothesis b of image b / G reads key r < P from
// the image's prefix cache (a TMA box, like a contiguous cache), key r = P + j from text row slots[b, j] when j < pos and from its
// own row b * T + j otherwise.  T is the text rows per hypothesis: the decode's text cache rows, or, for the caption matrix (pos = 0),
// the 2 t - 1 rows of a pair of a t-word caption in the layer's packed qkv.
// The text rows are gathered into the same 128B-swizzled tile slots a TMA box of the contiguous cache fills, and slots past Lkv
// are zeroed as TMA's out-of-bounds fill zeroes them: the tiles, and so every instruction after the load, are those of
// the contiguous cache.  A slot entry outside the text tensor is clamped into it (wrong numbers, never an out-of-bounds read).
// ------------------------------------------------------------------------------------------------
struct GroupKv {
  const __nv_bfloat16* text;  // [B, T, ld]: K | V rows, V at column H
  const int* slots;           // [B, T]; not read when pos = 0
  long long ld;
  int H, G, P, pos, T;
  long long text_rows;        // B * T
};

// Key rows [max(P, k0), k0 + 128) of a K tile and its V tile, for hypothesis b and head h.  Called by all threads after the tile's
// TMA box (if any) has landed; the caller fences and synchronises before the tiles are read.
__device__ __forceinline__ void group_fill(uint8_t* sK, uint8_t* sV, const GroupKv& g, int b, int h, int k0, int Lkv) {
  for (int i = threadIdx.x; i < TL * 8; i += ATT_THREADS) {
    const int r = i >> 3, c = i & 7, key = k0 + r;
    if (key < g.P) continue;
    uint4 kx = make_uint4(0u, 0u, 0u, 0u), vx = kx;
    if (key < Lkv) {
      const int j = key - g.P;
      long long row = static_cast<long long>(b) * g.T + j;
      if (j < g.pos) row = min(max(static_cast<long long>(__ldg(g.slots + static_cast<long long>(b) * g.T + j)), 0ll), g.text_rows - 1);
      const __nv_bfloat16* src = g.text + row * g.ld + h * HD + c * 8;
      kx = __ldg(reinterpret_cast<const uint4*>(src));
      vx = __ldg(reinterpret_cast<const uint4*>(src + g.H));
    }
    const int off = r * 128 + ((c ^ (r & 7)) << 4);
    *reinterpret_cast<uint4*>(sK + off) = kx;
    *reinterpret_cast<uint4*>(sV + off) = vx;
  }
}

// ------------------------------------------------------------------------------------------------
// per-row self key (vlpk_encoder_score_fwd): query row i of sequence b also attends to one extra key, its own (k_i, v_i), which no
// mask hides.  Its score q_i . k_i / 8 joins the row's maximum and sums after the shared keys (the O accumulator and sums rescaled to
// the new maximum), and p_self v_i joins O, so the softmax runs over [shared keys | self] and the saved logsumexp includes the self
// term.  Row i reads k / v at k + b * bstride + i * ld (the same for v); rows past Lq read row Lq - 1 (never stored).
// ------------------------------------------------------------------------------------------------
struct SelfKv {
  const __nv_bfloat16* k;
  const __nv_bfloat16* v;
  long long ld, bstride;
};

// This thread's two rows' self scores in the log2 domain (scaled, unmasked): q_i . k_i with q from the swizzled Q tile (local rows
// lr[hh]) and k from global memory; each thread of a quad takes 16 of the 64 dimensions.
__device__ __forceinline__ void self_scores(const uint8_t* sQ, const SelfKv& sk, int b, int h, const int (&lr)[2], const int (&row)[2],
                                            int Lq, float (&ss)[2]) {
  const int qi = threadIdx.x & 3;
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const __nv_bfloat16* kp = sk.k + b * sk.bstride + static_cast<long long>(min(row[hh], Lq - 1)) * sk.ld + h * HD;
    float acc = 0.f;
#pragma unroll
    for (int c = 2 * qi; c < 2 * qi + 2; ++c) {
      const uint4 q4 = *reinterpret_cast<const uint4*>(sQ + lr[hh] * 128 + ((c ^ (lr[hh] & 7)) << 4));
      const uint4 k4 = __ldg(reinterpret_cast<const uint4*>(kp + c * 8));
      const uint32_t qw[4] = {q4.x, q4.y, q4.z, q4.w}, kw[4] = {k4.x, k4.y, k4.z, k4.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 a = unpack_bf16x2(qw[j]), k2 = unpack_bf16x2(kw[j]);
        acc = fmaf(a.x, k2.x, fmaf(a.y, k2.y, acc));
      }
    }
    ss[hh] = quad_sum(acc) * (0.125f * LOG2E);
  }
}

// Folds the self key into a finished row (quad-reduced mx / lsum / rsum, unnormalised o) as one more online-softmax step.
__device__ __forceinline__ void fold_self(const SelfKv& sk, const Frag& f, int b, int h, const int (&row)[2], int Lq, const float (&ss)[2],
                                          float (&mx)[2], float (&lsum)[2], float (&rsum)[2], float (&o)[32]) {
  float alpha[2], es[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    const float mnew = fmaxf(mx[hh], ss[hh]);
    alpha[hh] = fast_ex2(mx[hh] - mnew);
    const float x = fast_ex2(ss[hh] - mnew);
    es[hh] = bf16_round(x);  // the self term enters O and the normalising sum as the bf16 value the shared keys' P would be
    lsum[hh] = lsum[hh] * alpha[hh] + x;
    rsum[hh] = rsum[hh] * alpha[hh] + es[hh];
    mx[hh] = mnew;
  }
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int hh = (i >> 1) & 1, col = 8 * (i >> 2) + f.fc;
    const __nv_bfloat16* vp = sk.v + b * sk.bstride + static_cast<long long>(min(row[hh], Lq - 1)) * sk.ld + h * HD + col;
    const float2 v2 = unpack_bf16x2(__ldg(reinterpret_cast<const uint32_t*>(vp)));
    o[i] = fmaf(es[hh], v2.x, o[i] * alpha[hh]);
    o[i + 1] = fmaf(es[hh], v2.y, o[i + 1] * alpha[hh]);
  }
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

// GROUP: K/V from a shared prefix + text rows (GroupKv); grid (G * heads, images), so the G hypotheses of an image and head run
// next to each other and read its prefix box from L2.  Otherwise grid (heads, B) and K/V from tm.k / tm.v.
// SELF: every query row also attends to its own key (SelfKv), folded in after the shared keys; no dropout.  With GROUP, b (the
// hypothesis) selects the query, output, lse and self rows, the image the prefix box and the mask rows.
template <bool GROUP, bool SELF>
__device__ __forceinline__ void attn_fwd_body(const AttnTmaps& tm, const AttnArgs a, const GroupKv g, const SelfKv sk) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem + FwdSmem::OFF_Q;
  uint8_t* sK = smem + FwdSmem::OFF_K;
  uint8_t* sV = smem + FwdSmem::OFF_V;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FwdSmem::OFF_BAR);
  uint64_t* bar_qk = &bars[0];
  uint64_t* bar_v = &bars[1];

  pdl_launch_dependents();
  const int h = GROUP ? blockIdx.x / g.G : blockIdx.x;
  const int b = GROUP ? blockIdx.y * g.G + blockIdx.x % g.G : blockIdx.y;
  const int kb = GROUP ? blockIdx.y : b;  // sequence of the K/V boxes and of the mask rows
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
    tma_load_3d(sK, &tm.k, bar_qk, h * HD, 0, kb);
    mbar_arrive_expect_tx(bar_v, TILE_B);
    tma_load_3d(sV, &tm.v, bar_v, h * HD, 0, kb);
  }

  const int row[2] = {wg * 64 + f.fr, wg * 64 + f.fr + 8};
  uint32_t mw[2][4];
  uint64_t row_elem0[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    load_mask_words(a, kb, row[hh], mw[hh]);
    row_elem0[hh] = ((static_cast<uint64_t>(b) * a.heads + h) * a.Lq + min(row[hh], a.Lq - 1)) * TL;
  }
  if constexpr (GROUP) {  // text rows over the prefix box's out-of-bounds rows
    mbar_wait(bar_qk, 0);
    mbar_wait(bar_v, 0);
    group_fill(sK, sV, g, b, h, 0, a.Lkv);
    fence_proxy_async_smem();
    __syncthreads();
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
    if (!SELF && qi == 0 && a.lse != nullptr && row[hh] < a.Lq)
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
  if constexpr (SELF) {  // this warpgroup's Q rows are still in its half of the Q tile: staging below overwrites them
    float ss[2];
    self_scores(sQ, sk, b, h, row, row, a.Lq, ss);
    fold_self(sk, f, b, h, row, a.Lq, ss, mx, lsum, rsum, o);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      if (qi == 0 && a.lse != nullptr && row[hh] < a.Lq)
        a.lse[(static_cast<size_t>(b) * a.heads + h) * a.Lq + row[hh]] = (mx[hh] + log2f(lsum[hh])) * LN2;
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

__global__ void __launch_bounds__(ATT_THREADS, 2) attn_fwd_kernel(const __grid_constant__ AttnTmaps tm, const AttnArgs a) {
  attn_fwd_body<false, false>(tm, a, GroupKv{}, SelfKv{});
}

__global__ void __launch_bounds__(ATT_THREADS, 2) attn_fwd_group_kernel(const __grid_constant__ AttnTmaps tm, const AttnArgs a,
                                                                         const GroupKv g) {
  attn_fwd_body<true, false>(tm, a, g, SelfKv{});
}

__global__ void __launch_bounds__(ATT_THREADS, 2) attn_fwd_self_kernel(const __grid_constant__ AttnTmaps tm, const AttnArgs a,
                                                                        const SelfKv sk) {
  attn_fwd_body<false, true>(tm, a, GroupKv{}, sk);
}

__global__ void __launch_bounds__(ATT_THREADS, 2) attn_fwd_group_self_kernel(const __grid_constant__ AttnTmaps tm, const AttnArgs a,
                                                                              const GroupKv g, const SelfKv sk) {
  attn_fwd_body<true, true>(tm, a, g, sk);
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
// tiled kernels: sequences longer than one tile (Lq or Lkv in (128, 512]), or any length under the "attn_tiled" test option.
// Key slots S = 128 * ceil(Lkv / 128): a mask row has S / 32 words, a keep-bit row S / 8 bytes, and the dropout element of
// (b, h, q, key) is ((b * heads + h) * Lq + q) * S + key.  For Lkv <= 128 that is the single-tile kernels' layout.
//   fwd     : CTA per (head, sequence, 128-row q tile); K/V tiles stream through a two-stage TMA ring; online softmax in the log2
//             domain, O rescaled in registers.  Same per-element semantics as attn_fwd_kernel.
//   bwd dq  : CTA per (head, sequence, q tile); pass 1 over the KV tiles: delta_r = sum_j P_rj dP_rj from the recomputed P (as
//             attn_bwd_kernel); pass 2: dS and dQ = dS K / 8 in registers.  Writes dQ, delta and the dQ column sums.
//   bwd dkv : CTA per (head, sequence, kv tile); loops over the q tiles: P from lse, dS with delta, dV += P^T dO, dK += dS^T Q in
//             registers.  Writes dK, dV and their column sums.
// No floating-point atomics: every output element and every bias partial is written by exactly one CTA.  Recompute cost: QK^T runs
// 3x and dO V^T 3x (2 in the dq kernel, 1 in the dkv kernel) against 1x each in the single-tile backward.
// ------------------------------------------------------------------------------------------------
static constexpr int MAX_SLOTS = 512;
static bool g_attn_tiled = false;  // test option "attn_tiled": the tiled kernels at every length

void set_attn_tiled(bool on) { g_attn_tiled = on; }

struct AttnTiledArgs {
  int B, heads, Lq, Lkv;
  int slots;                  // S: key slots per query row
  int tiles;                  // bwd: bias partials per sequence (= q tiles = kv tiles)
  const uint32_t* mask_bits;  // [B, mask_rows, S / 32]
  int mask_rows;
  float* lse;                 // [B, heads, Lq]
  float* delta;               // bwd: [B, heads, Lq], written by the dq kernel, read by the dkv kernel
  DropoutCfg drop;
  unsigned char* keep_out;    // fwd, optional: S / 8 bytes per (sequence, head, query row)
  float* dbias_part;          // bwd, optional: [B * tiles][3 * heads * 64] column sums of dQ | dK | dV per (sequence, tile)
};

// The 4 mask words of key tile kt for query row `row`.
__device__ __forceinline__ void load_mask_tile(const AttnTiledArgs& a, int b, int row, int kt, uint32_t (&mw)[4]) {
  const int mr = (a.mask_rows == 1) ? 0 : min(row, a.mask_rows - 1);
  const uint4 m4 = __ldg(reinterpret_cast<const uint4*>(a.mask_bits + (static_cast<size_t>(b) * a.mask_rows + mr) * (a.slots >> 5)) + kt);
  mw[0] = m4.x; mw[1] = m4.y; mw[2] = m4.z; mw[3] = m4.w;
}

__device__ __forceinline__ uint64_t tiled_row_elem0(const AttnTiledArgs& a, int b, int h, int row) {
  return ((static_cast<uint64_t>(b) * a.heads + h) * a.Lq + min(row, a.Lq - 1)) * a.slots;
}

// this thread's column of the bias partial: column sums of a staged [128 x 64] bf16 tile (rows past the sequence are zero)
__device__ __forceinline__ float staged_colsum(const uint8_t* stg, int c) {
  float acc = 0.f;
#pragma unroll 8
  for (int r = 0; r < TL; ++r)
    acc += __bfloat162float(*reinterpret_cast<const __nv_bfloat16*>(stg + r * 128 + (((c >> 3) ^ (r & 7)) << 4) + (c & 7) * 2));
  return acc;
}

struct FwdTiledSmem {
  static constexpr int OFF_Q = 0;        // later output staging
  static constexpr int OFF_KV = TILE_B;  // 2 stages of K | V
  static constexpr int OFF_BAR = 5 * TILE_B;
  static constexpr int TOTAL = OFF_BAR + 24;
  static constexpr int DYN = TOTAL + 1024;
};

// One CTA per SM: the running O (32 registers) stays live beside S and P, which does not fit the 128 registers of two CTAs.
// GROUP: as attn_fwd_body; a key tile that starts at or past the prefix gets no TMA box (its barrier is arrived on without bytes).
// SELF: as attn_fwd_body.
template <bool GROUP, bool SELF>
__device__ __forceinline__ void attn_fwd_tiled_body(const AttnTmaps& tm, const AttnTiledArgs a, const GroupKv g, const SelfKv sk) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem + FwdTiledSmem::OFF_Q;
  uint8_t* sKV = smem + FwdTiledSmem::OFF_KV;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + FwdTiledSmem::OFF_BAR);  // [0] Q, [1 + s] K|V stage s

  pdl_launch_dependents();
  const int h = GROUP ? blockIdx.x / g.G : blockIdx.x;
  const int b = GROUP ? blockIdx.y * g.G + blockIdx.x % g.G : blockIdx.y;
  const int kb = GROUP ? blockIdx.y : b;  // sequence of the K/V boxes and of the mask rows
  const int q0 = blockIdx.z * TL;
  const int tid = threadIdx.x, wg = tid >> 7;
  const Frag f;
  const int qi = tid & 3;
  const int nkt = (a.Lkv + TL - 1) / TL;

  if (tid == 0) {
    tma_prefetch_desc(&tm.q);
    tma_prefetch_desc(&tm.k);
    tma_prefetch_desc(&tm.v);
    tma_prefetch_desc(&tm.o);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bars[0], TILE_B);
    tma_load_3d(sQ, &tm.q, &bars[0], h * HD, q0, b);
    for (int kt = 0; kt < 2 && kt < nkt; ++kt) {
      if (GROUP && kt * TL >= g.P) {
        mbar_arrive(&bars[1 + kt]);
        continue;
      }
      mbar_arrive_expect_tx(&bars[1 + kt], 2 * TILE_B);
      tma_load_3d(sKV + kt * 2 * TILE_B, &tm.k, &bars[1 + kt], h * HD, kt * TL, kb);
      tma_load_3d(sKV + kt * 2 * TILE_B + TILE_B, &tm.v, &bars[1 + kt], h * HD, kt * TL, kb);
    }
  }

  const int row[2] = {q0 + wg * 64 + f.fr, q0 + wg * 64 + f.fr + 8};
  uint64_t row_elem0[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) row_elem0[hh] = tiled_row_elem0(a, b, h, row[hh]);
  const uint64_t dseed = drop_seed(a.drop);

  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float mx[2] = {-INFINITY, -INFINITY}, rsum[2] = {0.f, 0.f}, lsum[2] = {0.f, 0.f};  // lsum / rsum: this thread's columns only
  mbar_wait(&bars[0], 0);
  for (int kt = 0; kt < nkt; ++kt) {
    const int st = kt & 1;
    uint8_t* sK = sKV + st * 2 * TILE_B;
    uint8_t* sV = sK + TILE_B;
    uint32_t mw[2][4];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) load_mask_tile(a, kb, row[hh], kt, mw[hh]);
    float s[64];
    mbar_wait(&bars[1 + st], (kt >> 1) & 1);
    if constexpr (GROUP) {
      group_fill(sK, sV, g, b, h, kt * TL, a.Lkv);
      fence_proxy_async_smem();
      __syncthreads();
    }
    {
      const uint32_t qa = smem_u32(sQ) + wg * 8192, k0 = smem_u32(sK);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < HD / 16; ++k)
        wgmma_m64n128k16_ss<0, 0>(s, wgmma_desc_sw128(qa + k * 32, 16, 1024), wgmma_desc_sw128(k0 + k * 32, 16, 1024), k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
    }
    const int lkv = a.Lkv - kt * TL;  // >= 1: column 0 of every tile is a real key, so the tile maximum is finite
    float tmx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int hh = (i >> 1) & 1;
      s[i] = score(s[i], mw[hh], 8 * (i >> 2) + f.fc + (i & 1), lkv);
      tmx[hh] = fmaxf(tmx[hh], s[i]);
    }
    float alpha[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const float mnew = fmaxf(mx[hh], quad_max(tmx[hh]));
      alpha[hh] = fast_ex2(mx[hh] - mnew);  // 0 on the first tile (mx = -inf)
      mx[hh] = mnew;
      lsum[hh] *= alpha[hh];
      rsum[hh] *= alpha[hh];
    }
    uint32_t kw[2][4];
    const uint64_t tile_elem0[2] = {row_elem0[0] + kt * TL, row_elem0[1] + kt * TL};
    attn_keep_words(a.drop, dseed, tile_elem0, kw);
    if (a.keep_out != nullptr) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh)
        if (row[hh] < a.Lq) reinterpret_cast<uint32_t*>(a.keep_out + (tile_elem0[hh] >> 3))[qi] = kw[hh][qi];
    }
    uint32_t pa[8][4];
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int hh = (i >> 1) & 1, col = 8 * (i >> 2) + f.fc;
      const float x0 = fast_ex2(s[i] - mx[hh]), x1 = fast_ex2(s[i + 1] - mx[hh]);
      lsum[hh] += x0 + x1;
      const float e0 = bf16_round(x0), e1 = bf16_round(x1);
      rsum[hh] += e0 + e1;
      const uint32_t keep = kw[hh][col >> 5] >> (col & 31);
      const float p0 = (keep & 1u) ? e0 * a.drop.scale : 0.f;
      const float p1 = (keep & 2u) ? e1 * a.drop.scale : 0.f;
      pa[i >> 3][(i >> 1) & 3] = pack_bf16x2(p0, p1);
    }
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
    {
      const uint32_t v0 = smem_u32(sV);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TL / 16; ++k) wgmma_m64n64k16_rs<1>(o, pa[k], wgmma_desc_sw128(v0 + k * 2048, 8192, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(o);
    }
    __syncthreads();  // both warpgroups are done with stage st
    if (tid == 0 && kt + 2 < nkt) {
      if (GROUP && (kt + 2) * TL >= g.P) {
        mbar_arrive(&bars[1 + st]);
      } else {
        mbar_arrive_expect_tx(&bars[1 + st], 2 * TILE_B);
        tma_load_3d(sK, &tm.k, &bars[1 + st], h * HD, (kt + 2) * TL, kb);
        tma_load_3d(sV, &tm.v, &bars[1 + st], h * HD, (kt + 2) * TL, kb);
      }
    }
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    rsum[hh] = quad_sum(rsum[hh]);
    lsum[hh] = quad_sum(lsum[hh]);
    if (!SELF && qi == 0 && a.lse != nullptr && row[hh] < a.Lq)
      a.lse[(static_cast<size_t>(b) * a.heads + h) * a.Lq + row[hh]] = (mx[hh] + log2f(lsum[hh])) * LN2;
  }
  if constexpr (SELF) {
    const int lr[2] = {wg * 64 + f.fr, wg * 64 + f.fr + 8};
    float ss[2];
    self_scores(sQ, sk, b, h, lr, row, a.Lq, ss);
    fold_self(sk, f, b, h, row, a.Lq, ss, mx, lsum, rsum, o);
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      if (qi == 0 && a.lse != nullptr && row[hh] < a.Lq)
        a.lse[(static_cast<size_t>(b) * a.heads + h) * a.Lq + row[hh]] = (mx[hh] + log2f(lsum[hh])) * LN2;
  }
  const float inv[2] = {1.0f / rsum[0], 1.0f / rsum[1]};
  uint8_t* stg = sQ + wg * 8192;  // this warpgroup's own Q rows: only its own S = QK^T read them
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int hh = (i >> 1) & 1;
    sw_write_pair(stg, f.fr + 8 * hh, 8 * (i >> 2) + f.fc, pack_bf16x2(o[i] * inv[hh], o[i + 1] * inv[hh]));
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    tma_store_3d(&tm.o, sQ, h * HD, q0, b);
    tma_store_commit();
    tma_store_wait<0>();
  }
}

__global__ void __launch_bounds__(ATT_THREADS, 1) attn_fwd_tiled_kernel(const __grid_constant__ AttnTmaps tm, const AttnTiledArgs a) {
  attn_fwd_tiled_body<false, false>(tm, a, GroupKv{}, SelfKv{});
}

__global__ void __launch_bounds__(ATT_THREADS, 1) attn_fwd_group_tiled_kernel(const __grid_constant__ AttnTmaps tm, const AttnTiledArgs a,
                                                                               const GroupKv g) {
  attn_fwd_tiled_body<true, false>(tm, a, g, SelfKv{});
}

__global__ void __launch_bounds__(ATT_THREADS, 1) attn_fwd_self_tiled_kernel(const __grid_constant__ AttnTmaps tm, const AttnTiledArgs a,
                                                                              const SelfKv sk) {
  attn_fwd_tiled_body<false, true>(tm, a, GroupKv{}, sk);
}

__global__ void __launch_bounds__(ATT_THREADS, 1) attn_fwd_group_self_tiled_kernel(const __grid_constant__ AttnTmaps tm, const AttnTiledArgs a,
                                                                                    const GroupKv g, const SelfKv sk) {
  attn_fwd_tiled_body<true, true>(tm, a, g, sk);
}

// P (recomputed from the logsumexp; 0 for keys >= Lkv and rows >= Lq) and the dropout-masked dP of one 64 x 128 (q, key) block,
// in place of the S = QK^T and dP = dO V^T accumulators.
__device__ __forceinline__ void tiled_p_dp(const AttnTiledArgs& a, const Frag& f, float (&s)[64], float (&dp)[64], const uint32_t (&mw)[2][4],
                                           const uint32_t (&kw)[2][4], const float (&lse2)[2], const bool (&row_ok)[2], int lkv) {
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int hh = (i >> 1) & 1, col = 8 * (i >> 2) + f.fc + (i & 1);
    s[i] = row_ok[hh] ? fast_ex2(score(s[i], mw[hh], col, lkv) - lse2[hh]) : 0.f;
    dp[i] = ((kw[hh][col >> 5] >> (col & 31)) & 1u) ? dp[i] * a.drop.scale : 0.f;
  }
}

// S = Q K^T and dP = dO V^T for one warpgroup's 64 query rows against one 128-key tile
__device__ __forceinline__ void tiled_s_dp(uint32_t qa, uint32_t doa, uint32_t k0, uint32_t v0, float (&s)[64], float (&dp)[64]) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < HD / 16; ++k)
    wgmma_m64n128k16_ss<0, 0>(s, wgmma_desc_sw128(qa + k * 32, 16, 1024), wgmma_desc_sw128(k0 + k * 32, 16, 1024), k > 0 ? 1u : 0u);
#pragma unroll
  for (int k = 0; k < HD / 16; ++k)
    wgmma_m64n128k16_ss<0, 0>(dp, wgmma_desc_sw128(doa + k * 32, 16, 1024), wgmma_desc_sw128(v0 + k * 32, 16, 1024), k > 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();
  reg_fence(s);
  reg_fence(dp);
}

struct BwdDqSmem {
  static constexpr int OFF_Q = 0;  // later dQ staging
  static constexpr int OFF_DO = TILE_B;
  static constexpr int OFF_KV = 2 * TILE_B;  // 2 stages of K | V
  static constexpr int OFF_BAR = 6 * TILE_B;
  static constexpr int TOTAL = OFF_BAR + 24;
  static constexpr int DYN = TOTAL + 1024;
};

__global__ void __launch_bounds__(ATT_THREADS, 1) attn_bwd_dq_tiled_kernel(const __grid_constant__ AttnTmaps tm, const AttnTiledArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem + BwdDqSmem::OFF_Q;
  uint8_t* sdO = smem + BwdDqSmem::OFF_DO;
  uint8_t* sKV = smem + BwdDqSmem::OFF_KV;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + BwdDqSmem::OFF_BAR);  // [0] Q | dO, [1 + s] K|V stage s

  pdl_launch_dependents();
  const int h = blockIdx.x, b = blockIdx.y, qt = blockIdx.z, q0 = qt * TL;
  const int tid = threadIdx.x, wg = tid >> 7;
  const Frag f;
  const int nkt = (a.Lkv + TL - 1) / TL;
  const int nload = 2 * nkt;  // the KV tiles stream through the ring twice: delta pass, then dQ pass

  if (tid == 0) {
    tma_prefetch_desc(&tm.q);
    tma_prefetch_desc(&tm.k);
    tma_prefetch_desc(&tm.v);
    tma_prefetch_desc(&tm.o);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bars[0], 2 * TILE_B);
    tma_load_3d(sQ, &tm.q, &bars[0], h * HD, q0, b);
    tma_load_3d(sdO, &tm.o, &bars[0], h * HD, q0, b);
    for (int i = 0; i < 2; ++i) {
      mbar_arrive_expect_tx(&bars[1 + i], 2 * TILE_B);
      tma_load_3d(sKV + i * 2 * TILE_B, &tm.k, &bars[1 + i], h * HD, (i % nkt) * TL, b);
      tma_load_3d(sKV + i * 2 * TILE_B + TILE_B, &tm.v, &bars[1 + i], h * HD, (i % nkt) * TL, b);
    }
  }

  const int row[2] = {q0 + wg * 64 + f.fr, q0 + wg * 64 + f.fr + 8};
  uint64_t row_elem0[2];
  float lse2[2];
  bool row_ok[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    row_elem0[hh] = tiled_row_elem0(a, b, h, row[hh]);
    row_ok[hh] = row[hh] < a.Lq;
    lse2[hh] = row_ok[hh] ? a.lse[(static_cast<size_t>(b) * a.heads + h) * a.Lq + row[hh]] * LOG2E : 0.f;
  }
  const uint64_t dseed = drop_seed(a.drop);
  const uint32_t qa = smem_u32(sQ) + wg * 8192, doa = smem_u32(sdO) + wg * 8192;

  float delta[2] = {0.f, 0.f};
  float dq[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dq[i] = 0.f;
  mbar_wait(&bars[0], 0);
  for (int it = 0; it < nload; ++it) {
    const int st = it & 1, kt = it % nkt;
    uint8_t* sK = sKV + st * 2 * TILE_B;
    uint8_t* sV = sK + TILE_B;
    uint32_t mw[2][4], kw[2][4];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) load_mask_tile(a, b, row[hh], kt, mw[hh]);
    const uint64_t tile_elem0[2] = {row_elem0[0] + kt * TL, row_elem0[1] + kt * TL};
    attn_keep_words(a.drop, dseed, tile_elem0, kw);
    float s[64], dp[64];
    mbar_wait(&bars[1 + st], (it >> 1) & 1);
    tiled_s_dp(qa, doa, smem_u32(sK), smem_u32(sV), s, dp);
    tiled_p_dp(a, f, s, dp, mw, kw, lse2, row_ok, a.Lkv - kt * TL);
    if (it < nkt) {
#pragma unroll
      for (int i = 0; i < 64; ++i) delta[(i >> 1) & 1] = fmaf(s[i], dp[i], delta[(i >> 1) & 1]);
      if (it == nkt - 1) {
        delta[0] = quad_sum(delta[0]);
        delta[1] = quad_sum(delta[1]);
        if ((tid & 3) == 0) {
#pragma unroll
          for (int hh = 0; hh < 2; ++hh)
            if (row_ok[hh]) a.delta[(static_cast<size_t>(b) * a.heads + h) * a.Lq + row[hh]] = delta[hh];
        }
      }
    } else {
      uint32_t dsa[8][4];
#pragma unroll
      for (int i = 0; i < 64; i += 2) {
        const int hh = (i >> 1) & 1;
        dsa[i >> 3][(i >> 1) & 3] = pack_bf16x2(s[i] * (dp[i] - delta[hh]) * 0.125f, s[i + 1] * (dp[i + 1] - delta[hh]) * 0.125f);
      }
      const uint32_t k0 = smem_u32(sK);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TL / 16; ++k) wgmma_m64n64k16_rs<1>(dq, dsa[k], wgmma_desc_sw128(k0 + k * 2048, 8192, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(dq);
    }
    __syncthreads();  // both warpgroups are done with stage st
    if (tid == 0 && it + 2 < nload) {
      const int nt = (it + 2) % nkt;
      mbar_arrive_expect_tx(&bars[1 + st], 2 * TILE_B);
      tma_load_3d(sK, &tm.k, &bars[1 + st], h * HD, nt * TL, b);
      tma_load_3d(sV, &tm.v, &bars[1 + st], h * HD, nt * TL, b);
    }
  }
  uint8_t* stg = sQ + wg * 8192;  // this warpgroup's own Q rows
#pragma unroll
  for (int i = 0; i < 32; i += 2) sw_write_pair(stg, f.fr + 8 * ((i >> 1) & 1), 8 * (i >> 2) + f.fc, pack_bf16x2(dq[i], dq[i + 1]));
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    tma_store_3d(&tm.dq, sQ, h * HD, q0, b);
    tma_store_commit();
  }
  if (a.dbias_part != nullptr && tid < HD)
    a.dbias_part[(static_cast<size_t>(b) * a.tiles + qt) * 3 * a.heads * HD + h * HD + tid] = staged_colsum(sQ, tid);
  if (tid == 0) tma_store_wait<0>();
}

struct BwdDkvSmem {
  static constexpr int OFF_K = 0;        // later dK staging
  static constexpr int OFF_V = TILE_B;   // later dV staging
  static constexpr int OFF_QD = 2 * TILE_B;  // 2 stages of Q | dO
  static constexpr int OFF_P = 6 * TILE_B;   // 2 atoms of [128 q x 64 kv]: dropout-masked P
  static constexpr int OFF_DS = 8 * TILE_B;  // 2 atoms of [128 q x 64 kv]: dS
  static constexpr int OFF_BAR = 10 * TILE_B;
  static constexpr int TOTAL = OFF_BAR + 24;
  static constexpr int DYN = TOTAL + 1024;
};

__global__ void __launch_bounds__(ATT_THREADS, 1) attn_bwd_dkv_tiled_kernel(const __grid_constant__ AttnTmaps tm, const AttnTiledArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sK = smem + BwdDkvSmem::OFF_K;
  uint8_t* sV = smem + BwdDkvSmem::OFF_V;
  uint8_t* sQD = smem + BwdDkvSmem::OFF_QD;
  uint8_t* sP = smem + BwdDkvSmem::OFF_P;
  uint8_t* sDS = smem + BwdDkvSmem::OFF_DS;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + BwdDkvSmem::OFF_BAR);  // [0] K | V, [1 + s] Q|dO stage s

  pdl_launch_dependents();
  const int h = blockIdx.x, b = blockIdx.y, kt = blockIdx.z, kv0 = kt * TL;
  const int tid = threadIdx.x, wg = tid >> 7;
  const Frag f;
  const int nqt = (a.Lq + TL - 1) / TL;
  const int lkv = a.Lkv - kv0;

  if (tid == 0) {
    tma_prefetch_desc(&tm.q);
    tma_prefetch_desc(&tm.k);
    tma_prefetch_desc(&tm.v);
    tma_prefetch_desc(&tm.o);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // also orders the reads of delta after the dq kernel
  if (tid == 0) {
    mbar_arrive_expect_tx(&bars[0], 2 * TILE_B);
    tma_load_3d(sK, &tm.k, &bars[0], h * HD, kv0, b);
    tma_load_3d(sV, &tm.v, &bars[0], h * HD, kv0, b);
    for (int i = 0; i < 2 && i < nqt; ++i) {
      mbar_arrive_expect_tx(&bars[1 + i], 2 * TILE_B);
      tma_load_3d(sQD + i * 2 * TILE_B, &tm.q, &bars[1 + i], h * HD, i * TL, b);
      tma_load_3d(sQD + i * 2 * TILE_B + TILE_B, &tm.o, &bars[1 + i], h * HD, i * TL, b);
    }
  }
  const uint64_t dseed = drop_seed(a.drop);

  float dk[32], dv[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) dk[i] = dv[i] = 0.f;
  mbar_wait(&bars[0], 0);
  for (int qt = 0; qt < nqt; ++qt) {
    const int st = qt & 1;
    uint8_t* sQ = sQD + st * 2 * TILE_B;
    uint8_t* sdO = sQ + TILE_B;
    const int rl[2] = {wg * 64 + f.fr, wg * 64 + f.fr + 8};  // rows within the q tile
    const int row[2] = {qt * TL + rl[0], qt * TL + rl[1]};
    uint32_t mw[2][4], kw[2][4];
    float lse2[2], delta[2];
    bool row_ok[2];
    uint64_t tile_elem0[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      load_mask_tile(a, b, row[hh], kt, mw[hh]);
      tile_elem0[hh] = tiled_row_elem0(a, b, h, row[hh]) + kv0;
      row_ok[hh] = row[hh] < a.Lq;
      const size_t li = (static_cast<size_t>(b) * a.heads + h) * a.Lq + row[hh];
      lse2[hh] = row_ok[hh] ? a.lse[li] * LOG2E : 0.f;
      delta[hh] = row_ok[hh] ? a.delta[li] : 0.f;
    }
    attn_keep_words(a.drop, dseed, tile_elem0, kw);
    float s[64], dp[64];
    mbar_wait(&bars[1 + st], (qt >> 1) & 1);
    tiled_s_dp(smem_u32(sQ) + wg * 8192, smem_u32(sdO) + wg * 8192, smem_u32(sK), smem_u32(sV), s, dp);
    tiled_p_dp(a, f, s, dp, mw, kw, lse2, row_ok, lkv);
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int hh = (i >> 1) & 1, col = 8 * (i >> 2) + f.fc;
      const uint32_t keep = kw[hh][col >> 5] >> (col & 31);
      const float p0 = (keep & 1u) ? s[i] * a.drop.scale : 0.f, p1 = (keep & 2u) ? s[i + 1] * a.drop.scale : 0.f;
      sw_write_pair(sP + (col >> 6) * TILE_B, rl[hh], col & 63, pack_bf16x2(p0, p1));
      sw_write_pair(sDS + (col >> 6) * TILE_B, rl[hh], col & 63,
                    pack_bf16x2(s[i] * (dp[i] - delta[hh]) * 0.125f, s[i + 1] * (dp[i + 1] - delta[hh]) * 0.125f));
    }
    fence_proxy_async_smem();
    __syncthreads();
    // dV[kv, d] += sum_q Pd[q, kv] dO[q, d] and dK[kv, d] += sum_q dS[q, kv] Q[q, d] for kv rows [64 wg, 64 wg + 64)
    {
      const uint32_t p0 = smem_u32(sP) + wg * TILE_B, ds0 = smem_u32(sDS) + wg * TILE_B, do0 = smem_u32(sdO), q0 = smem_u32(sQ);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TL / 16; ++k)
        wgmma_m64n64k16_ss<1, 1>(dv, wgmma_desc_sw128(p0 + k * 2048, 8192, 1024), wgmma_desc_sw128(do0 + k * 2048, 8192, 1024), 1u);
#pragma unroll
      for (int k = 0; k < TL / 16; ++k)
        wgmma_m64n64k16_ss<1, 1>(dk, wgmma_desc_sw128(ds0 + k * 2048, 8192, 1024), wgmma_desc_sw128(q0 + k * 2048, 8192, 1024), 1u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(dv);
      reg_fence(dk);
    }
    __syncthreads();  // P / dS buffers and stage st are free
    if (tid == 0 && qt + 2 < nqt) {
      mbar_arrive_expect_tx(&bars[1 + st], 2 * TILE_B);
      tma_load_3d(sQ, &tm.q, &bars[1 + st], h * HD, (qt + 2) * TL, b);
      tma_load_3d(sdO, &tm.o, &bars[1 + st], h * HD, (qt + 2) * TL, b);
    }
  }
  // every wgmma has read K / V: reuse them as output staging
#pragma unroll
  for (int i = 0; i < 32; i += 2) {
    const int r = wg * 64 + f.fr + 8 * ((i >> 1) & 1), col = 8 * (i >> 2) + f.fc;
    sw_write_pair(sK, r, col, pack_bf16x2(dk[i], dk[i + 1]));
    sw_write_pair(sV, r, col, pack_bf16x2(dv[i], dv[i + 1]));
  }
  fence_proxy_async_smem();
  __syncthreads();
  if (tid == 0) {
    tma_store_3d(&tm.dk, sK, h * HD, kv0, b);
    tma_store_3d(&tm.dv, sV, h * HD, kv0, b);
    tma_store_commit();
  }
  if (a.dbias_part != nullptr && tid < 2 * HD) {
    const int o = 1 + (tid >> 6), c = tid & 63;
    a.dbias_part[(static_cast<size_t>(b) * a.tiles + kt) * 3 * a.heads * HD + o * a.heads * HD + h * HD + c] =
        staged_colsum(o == 1 ? sK : sV, c);
  }
  if (tid == 0) tma_store_wait<0>();
}

// ------------------------------------------------------------------------------------------------
// attention probabilities (opt-in, vlpk_attn_probs): P[b, h, i, j] = exp(s_ij - lse_i), recomputed from Q, K and the logsumexp the
// forward kernels save, so that those kernels stay as they are and one kernel serves every forward path (single-tile, tiled,
// re-projected prefix, K/V cache).  CTA per (head, sequence, 128-row query tile from row0); K tiles stream through a two-stage TMA
// ring; S = QK^T as in the forward, the same score() (scale, additive -10000 mask, key slots), then exp2(s - lse2) stored as fp32
// straight from the accumulator registers: a quad of threads writes 8 consecutive columns (32 bytes) of a row.
// ------------------------------------------------------------------------------------------------
struct ProbsArgs {
  AttnTiledArgs t;      // B, heads, Lq, Lkv, slots, mask_bits, mask_rows, lse (the mask loader's view)
  int row0;             // first query row written
  float* p;             // [B, heads, Lq - row0, ld_p], sequences p_bstride floats apart
  long long ld_p, p_bstride;
  int vec2;             // p and ld_p allow 8-byte stores
};

struct ProbsSmem {
  static constexpr int OFF_Q = 0;
  static constexpr int OFF_K = TILE_B;  // 2 stages of K
  static constexpr int OFF_BAR = 3 * TILE_B;
  static constexpr int TOTAL = OFF_BAR + 24;
  static constexpr int DYN = TOTAL + 1024;
};

__global__ void __launch_bounds__(ATT_THREADS, 2) attn_probs_kernel(const __grid_constant__ AttnTmaps tm, const ProbsArgs a) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem + ProbsSmem::OFF_Q;
  uint8_t* sK = smem + ProbsSmem::OFF_K;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + ProbsSmem::OFF_BAR);  // [0] Q, [1 + s] K stage s

  pdl_launch_dependents();
  const int h = blockIdx.x, b = blockIdx.y, q0 = a.row0 + blockIdx.z * TL;
  const int tid = threadIdx.x, wg = tid >> 7;
  const Frag f;
  const int nkt = (a.t.Lkv + TL - 1) / TL;

  if (tid == 0) {
    tma_prefetch_desc(&tm.q);
    tma_prefetch_desc(&tm.k);
    for (int i = 0; i < 3; ++i) mbar_init(&bars[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();
  if (tid == 0) {
    mbar_arrive_expect_tx(&bars[0], TILE_B);
    tma_load_3d(sQ, &tm.q, &bars[0], h * HD, q0, b);
    for (int kt = 0; kt < 2 && kt < nkt; ++kt) {
      mbar_arrive_expect_tx(&bars[1 + kt], TILE_B);
      tma_load_3d(sK + kt * TILE_B, &tm.k, &bars[1 + kt], h * HD, kt * TL, b);
    }
  }

  const int row[2] = {q0 + wg * 64 + f.fr, q0 + wg * 64 + f.fr + 8};
  float lse2[2];
  bool row_ok[2];
  float* prow[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    row_ok[hh] = row[hh] < a.t.Lq;
    lse2[hh] = row_ok[hh] ? a.t.lse[(static_cast<size_t>(b) * a.t.heads + h) * a.t.Lq + row[hh]] * LOG2E : 0.f;
    prow[hh] = a.p + b * a.p_bstride + (static_cast<long long>(h) * (a.t.Lq - a.row0) + (row[hh] - a.row0)) * a.ld_p;
  }
  mbar_wait(&bars[0], 0);
  for (int kt = 0; kt < nkt; ++kt) {
    const int st = kt & 1;
    uint8_t* sKs = sK + st * TILE_B;
    uint32_t mw[2][4];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) load_mask_tile(a.t, b, row[hh], kt, mw[hh]);
    float s[64];
    mbar_wait(&bars[1 + st], (kt >> 1) & 1);
    {
      const uint32_t qa = smem_u32(sQ) + wg * 8192, k0 = smem_u32(sKs);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < HD / 16; ++k)
        wgmma_m64n128k16_ss<0, 0>(s, wgmma_desc_sw128(qa + k * 32, 16, 1024), wgmma_desc_sw128(k0 + k * 32, 16, 1024), k > 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<0>();
      reg_fence(s);
    }
    __syncthreads();  // both warpgroups are done with stage st
    if (tid == 0 && kt + 2 < nkt) {
      mbar_arrive_expect_tx(&bars[1 + st], TILE_B);
      tma_load_3d(sKs, &tm.k, &bars[1 + st], h * HD, (kt + 2) * TL, b);
    }
    const int lkv = a.t.Lkv - kt * TL;
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int hh = (i >> 1) & 1, col = 8 * (i >> 2) + f.fc;
      if (!row_ok[hh] || col >= lkv) continue;
      const float p0 = fast_ex2(score(s[i], mw[hh], col, lkv) - lse2[hh]);
      const float p1 = fast_ex2(score(s[i + 1], mw[hh], col + 1, lkv) - lse2[hh]);
      float* dst = prow[hh] + kt * TL + col;
      if (col + 1 < lkv && a.vec2) {
        *reinterpret_cast<float2*>(dst) = make_float2(p0, p1);
      } else {
        dst[0] = p0;
        if (col + 1 < lkv) dst[1] = p1;
      }
    }
  }
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
  if (d.kv_slots == 0) {
    VLPK_CHECK_ARG(d.Lq >= 1 && d.Lq <= TL && d.Lkv >= 1 && d.Lkv <= TL, "attention: Lq=%d Lkv=%d must be in [1,128]",
                   d.Lq, d.Lkv);
  } else {
    VLPK_CHECK_ARG(d.Lkv >= 1 && d.Lkv <= MAX_SLOTS && d.kv_slots == (d.Lkv + TL - 1) / TL * TL && d.Lq >= 1 && d.Lq <= d.kv_slots,
                   "attention: Lq=%d Lkv=%d kv_slots=%d (needs Lkv in [1,512], kv_slots = 128 * ceil(Lkv / 128), Lq in [1,kv_slots])",
                   d.Lq, d.Lkv, d.kv_slots);
  }
  VLPK_CHECK_ARG(d.B >= 1 && d.heads >= 1, "attention: B=%d heads=%d", d.B, d.heads);
  VLPK_CHECK_ARG(d.mask_bits != nullptr && (d.mask_rows == 1 || d.mask_rows == d.Lq), "attention: mask rows %d",
                 d.mask_rows);
  return 0;
}

static bool use_tiled(const AttnDesc& d) { return g_attn_tiled || d.Lq > TL || d.Lkv > TL; }

static AttnTiledArgs tiled_args(const AttnDesc& d) {
  AttnTiledArgs a;
  a.B = d.B; a.heads = d.heads; a.Lq = d.Lq; a.Lkv = d.Lkv;
  a.slots = d.kv_slots != 0 ? d.kv_slots : TL;
  a.tiles = (d.Lq + TL - 1) / TL;
  a.mask_bits = d.mask_bits; a.mask_rows = d.mask_rows;
  a.lse = d.lse; a.delta = nullptr;
  a.drop = d.drop;
  a.keep_out = nullptr;
  a.dbias_part = nullptr;
  return a;
}

// Launches Kernel with ATT_THREADS threads and `smem` bytes of dynamic shared memory, raising its limit to `smem` on the first launch.
// The flag is per kernel (a template argument), not per kernel type: kernels of one signature need different limits.
template <auto Kernel, typename... Args>
static int launch_attn_kernel(dim3 grid, int smem, cudaStream_t stream, const Args&... args) {
  static bool attr_set = false;
  if (!attr_set) {
    VLPK_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr_set = true;
  }
  VLPK_CUDA(launch_ex(Kernel, grid, dim3(ATT_THREADS), smem, stream, 1, args...));
  return 0;
}

static int launch_attn_bwd_tiled(const AttnDesc& d, const AttnTmaps& tm, cudaStream_t stream) {
  AttnTiledArgs a = tiled_args(d);
  const long long nbias = 3LL * d.heads * HD;
  a.delta = scratch_f32(SCRATCH_ATTN_DELTA, static_cast<size_t>(d.B) * d.heads * d.Lq, stream);
  if (a.delta == nullptr) return -1;
  if (d.dbias != nullptr) {
    a.dbias_part = scratch_f32(SCRATCH_ATTN_DBIAS, static_cast<size_t>(d.B) * a.tiles * nbias, stream);
    if (a.dbias_part == nullptr) return -1;
  }
  const double flops = 10.0 * d.B * d.heads * d.Lq * d.Lkv * HD;  // algorithmic: the recomputed products are not counted
  {
    LaunchScope scope(CAT_ATTN_BWD, 0.4 * flops, stream);
    VLPK_TRY(launch_attn_kernel<attn_bwd_dq_tiled_kernel>(dim3(d.heads, d.B, a.tiles), BwdDqSmem::DYN, stream, tm, a));
  }
  {
    LaunchScope scope(CAT_ATTN_BWD, 0.6 * flops, stream);
    VLPK_TRY(launch_attn_kernel<attn_bwd_dkv_tiled_kernel>(dim3(d.heads, d.B, (d.Lkv + TL - 1) / TL), BwdDkvSmem::DYN, stream, tm, a));
  }
  if (d.dbias != nullptr) VLPK_TRY(launch_sum_parts(a.dbias_part, d.B * a.tiles, nbias, d.dbias, stream));
  return 0;
}

// Tensor maps of a forward over contiguous K/V: Q / ctx and K / V with their row and sequence strides.
static int fwd_tmaps(const AttnDesc& d, AttnTmaps* tm) {
  const int width = d.heads * HD;
  memset(tm, 0, sizeof(*tm));
  VLPK_TRY(make_seq_tmap(&tm->q, d.q, width, d.Lq, d.B, d.ld_q, d.q_batch_stride));
  VLPK_TRY(make_seq_tmap(&tm->k, d.k, width, d.Lkv, d.B, d.ld_kv, d.kv_batch_stride));
  VLPK_TRY(make_seq_tmap(&tm->v, d.v, width, d.Lkv, d.B, d.ld_kv, d.kv_batch_stride));
  VLPK_TRY(make_seq_tmap(&tm->o, d.o, width, d.Lq, d.B, d.ld_o, d.o_batch_stride));
  tm->dq = tm->dk = tm->dv = tm->o;
  return 0;
}

// Arguments of the single-tile forward kernels.
static AttnArgs fwd_args(const AttnDesc& d) {
  AttnArgs a;
  a.B = d.B; a.heads = d.heads; a.Lq = d.Lq; a.Lkv = d.Lkv;
  a.mask_bits = d.mask_bits; a.mask_rows = d.mask_rows;
  a.lse = d.lse; a.o_ptr = nullptr; a.do_ptr = nullptr; a.ld_o = d.ld_o;
  a.drop = d.drop;
  a.keep_out = d.keep_out;
  a.dbias_part = nullptr;
  return a;
}

// Tensor maps and loader arguments of a shared-prefix forward: Q / ctx of the d.B hypotheses with their strides, K / V boxes over
// the P prefix rows of each image, text rows gd.ld_text (0: d.ld_kv) elements apart.
static int group_setup(const AttnDesc& d, const AttnGroupKv& gd, AttnTmaps* tm, GroupKv* g) {
  VLPK_CHECK_ARG(gd.G >= 1 && d.B % gd.G == 0, "attention group: %d hypotheses are not whole groups of G=%d", d.B, gd.G);
  VLPK_CHECK_ARG(gd.prefix != nullptr && gd.text != nullptr && (gd.slots != nullptr || gd.pos == 0), "attention group: null pointer");
  const int width = d.heads * HD, images = d.B / gd.G;
  const int64_t ld_text = gd.ld_text != 0 ? gd.ld_text : d.ld_kv;
  VLPK_CHECK_ARG((reinterpret_cast<uintptr_t>(gd.text) & 15u) == 0 && ld_text % 8 == 0 && ld_text >= 2 * width,
                 "attention group: text rows need 16-byte alignment and K | V in each row (ld=%lld)", static_cast<long long>(ld_text));
  memset(tm, 0, sizeof(*tm));
  VLPK_TRY(make_seq_tmap(&tm->q, d.q, width, d.Lq, d.B, d.ld_q, d.q_batch_stride));
  VLPK_TRY(make_seq_tmap(&tm->k, gd.prefix, width, gd.P, images, d.ld_kv, static_cast<int64_t>(gd.prefix_rows) * d.ld_kv));
  VLPK_TRY(make_seq_tmap(&tm->v, static_cast<const __nv_bfloat16*>(gd.prefix) + width, width, gd.P, images, d.ld_kv,
                         static_cast<int64_t>(gd.prefix_rows) * d.ld_kv));
  VLPK_TRY(make_seq_tmap(&tm->o, d.o, width, d.Lq, d.B, d.ld_o, d.o_batch_stride));
  tm->dq = tm->dk = tm->dv = tm->o;
  g->text = static_cast<const __nv_bfloat16*>(gd.text);
  g->slots = gd.slots;
  g->ld = ld_text;
  g->H = width; g->G = gd.G; g->P = gd.P; g->pos = gd.pos; g->T = gd.T;
  g->text_rows = static_cast<long long>(d.B) * gd.T;
  return 0;
}

// Shape, mask and self-row rules of the self-key forwards (contiguous or shared-prefix K/V).
static int check_self(const AttnDesc& d, const AttnSelfKv& sd) {
  VLPK_CHECK_ARG(d.head_dim == HD, "attention self: head_dim %d unsupported (only 64)", d.head_dim);
  VLPK_CHECK_ARG(d.B >= 1 && d.heads >= 1 && d.Lq >= 1 && d.Lq <= MAX_SLOTS && d.Lkv >= 1 && d.Lkv <= MAX_SLOTS,
                 "attention self: B=%d heads=%d Lq=%d Lkv=%d (lengths in [1,512])", d.B, d.heads, d.Lq, d.Lkv);
  VLPK_CHECK_ARG(d.kv_slots == 0 ? d.Lkv <= TL : d.kv_slots == (d.Lkv + TL - 1) / TL * TL,
                 "attention self: kv_slots=%d for Lkv=%d (0 needs Lkv <= 128, else 128 * ceil(Lkv / 128))", d.kv_slots, d.Lkv);
  VLPK_CHECK_ARG(d.mask_bits != nullptr && d.mask_rows == d.Lq, "attention self: one mask row per query row needed (%d for Lq=%d)",
                 d.mask_rows, d.Lq);
  VLPK_CHECK_ARG(d.q && d.o && sd.k && sd.v, "attention self: null pointer");
  VLPK_CHECK_ARG(d.drop.p == 0.f && d.keep_out == nullptr, "attention self: forward only, without dropout");
  const auto a16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0; };
  VLPK_CHECK_ARG(a16(sd.k) && a16(sd.v) && sd.ld % 8 == 0 && sd.batch_stride % 8 == 0 && sd.ld >= d.heads * HD,
                 "attention self: self keys / values need 16-byte rows (ld=%lld, batch stride=%lld)", static_cast<long long>(sd.ld),
                 static_cast<long long>(sd.batch_stride));
  return 0;
}

static SelfKv self_kv(const AttnDesc& d, const AttnSelfKv& sd) {
  SelfKv sk;
  sk.k = static_cast<const __nv_bfloat16*>(sd.k);
  sk.v = static_cast<const __nv_bfloat16*>(sd.v);
  sk.ld = sd.ld;
  sk.bstride = sd.batch_stride != 0 ? sd.batch_stride : static_cast<int64_t>(d.Lq) * sd.ld;
  return sk;
}

int launch_attn_fwd(const AttnDesc& d, const AttnGroupKv* gd, const AttnSelfKv* sd, cudaStream_t stream) {
  // Each key source keeps its own rules: check_self takes lengths check_common refuses, and the two group rules differ.
  if (sd == nullptr) VLPK_TRY(check_common(d));
  else VLPK_TRY(check_self(d, *sd));
  AttnTmaps tm;
  GroupKv g{};
  if (gd == nullptr) {
    if (sd != nullptr) VLPK_CHECK_ARG(d.k && d.v, "attention self: null pointer");
    VLPK_TRY(fwd_tmaps(d, &tm));
  } else {
    if (sd == nullptr)
      VLPK_CHECK_ARG(gd->P >= 1 && gd->P <= gd->prefix_rows && gd->pos >= 0 && gd->pos + d.Lq <= gd->T && gd->P + gd->pos + d.Lq == d.Lkv,
                     "attention group: P=%d (prefix rows %d) pos=%d Lq=%d T=%d Lkv=%d", gd->P, gd->prefix_rows, gd->pos, d.Lq, gd->T, d.Lkv);
    else
      VLPK_CHECK_ARG(gd->P >= 1 && gd->P <= gd->prefix_rows && gd->pos >= 0 && gd->P + gd->pos <= d.Lkv && d.Lkv - gd->P <= gd->T,
                     "attention group self: P=%d (prefix rows %d) pos=%d Lkv=%d T=%d (needs P + pos <= Lkv <= P + T)", gd->P, gd->prefix_rows,
                     gd->pos, d.Lkv, gd->T);
    VLPK_TRY(group_setup(d, *gd, &tm, &g));
  }
  const SelfKv sk = sd != nullptr ? self_kv(d, *sd) : SelfKv{};
  unsigned char* keep_out = gd != nullptr ? nullptr : d.keep_out;  // with a self key d.keep_out is null: check_self refuses it
  const int G = gd != nullptr ? gd->G : 1;
  const bool tiled = use_tiled(d);
  const dim3 grid(G * d.heads, d.B / G, tiled ? (d.Lq + TL - 1) / TL : 1);
  LaunchScope scope(CAT_ATTN_FWD, 4.0 * d.B * d.heads * d.Lq * (d.Lkv + (sd != nullptr ? 1 : 0)) * HD, stream);
  if (tiled) {
    AttnTiledArgs a = tiled_args(d);
    a.keep_out = keep_out;
    constexpr int smem = FwdTiledSmem::DYN;
    if (gd != nullptr && sd != nullptr) return launch_attn_kernel<attn_fwd_group_self_tiled_kernel>(grid, smem, stream, tm, a, g, sk);
    if (gd != nullptr) return launch_attn_kernel<attn_fwd_group_tiled_kernel>(grid, smem, stream, tm, a, g);
    if (sd != nullptr) return launch_attn_kernel<attn_fwd_self_tiled_kernel>(grid, smem, stream, tm, a, sk);
    return launch_attn_kernel<attn_fwd_tiled_kernel>(grid, smem, stream, tm, a);
  }
  AttnArgs a = fwd_args(d);
  a.keep_out = keep_out;
  constexpr int smem = FwdSmem::DYN;
  if (gd != nullptr && sd != nullptr) return launch_attn_kernel<attn_fwd_group_self_kernel>(grid, smem, stream, tm, a, g, sk);
  if (gd != nullptr) return launch_attn_kernel<attn_fwd_group_kernel>(grid, smem, stream, tm, a, g);
  if (sd != nullptr) return launch_attn_kernel<attn_fwd_self_kernel>(grid, smem, stream, tm, a, sk);
  return launch_attn_kernel<attn_fwd_kernel>(grid, smem, stream, tm, a);
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
  if (use_tiled(d)) return launch_attn_bwd_tiled(d, tm, stream);
  AttnArgs a = fwd_args(d);
  a.o_ptr = reinterpret_cast<const __nv_bfloat16*>(d.o);
  a.do_ptr = reinterpret_cast<const __nv_bfloat16*>(d.d_o);
  a.keep_out = nullptr;
  const long long nbias = 3LL * d.heads * HD;
  if (d.dbias != nullptr) {
    a.dbias_part = scratch_f32(SCRATCH_ATTN_DBIAS, static_cast<size_t>(d.B) * nbias, stream);
    if (a.dbias_part == nullptr) return -1;
  }
  {
    LaunchScope scope(CAT_ATTN_BWD, 10.0 * d.B * d.heads * d.Lq * d.Lkv * HD, stream);
    VLPK_TRY(launch_attn_kernel<attn_bwd_kernel>(dim3(d.heads, d.B), BwdSmem::DYN, stream, tm, a));
  }
  if (d.dbias != nullptr) VLPK_TRY(launch_sum_parts(a.dbias_part, d.B, nbias, d.dbias, stream));
  return 0;
}

int launch_attn_probs(const AttnDesc& d, int64_t q_batch_stride, int row0, float* p, int64_t ld_p, int64_t p_batch_stride,
                      cudaStream_t stream) {
  VLPK_TRY(check_common(d));
  VLPK_CHECK_ARG(d.q != nullptr && d.k != nullptr && d.lse != nullptr && p != nullptr, "attn_probs: null pointer");
  VLPK_CHECK_ARG(row0 >= 0 && row0 < d.Lq, "attn_probs: row0=%d outside [0, Lq=%d)", row0, d.Lq);
  VLPK_CHECK_ARG(ld_p >= d.Lkv, "attn_probs: ld_p=%lld < Lkv=%d", static_cast<long long>(ld_p), d.Lkv);
  const int64_t rows = d.Lq - row0;
  const int64_t pbs = p_batch_stride != 0 ? p_batch_stride : d.heads * rows * ld_p;
  VLPK_CHECK_ARG(pbs >= d.heads * rows * ld_p || d.B == 1, "attn_probs: p batch stride %lld overlaps the %d x %lld x %lld block of a sequence",
                 static_cast<long long>(pbs), d.heads, static_cast<long long>(rows), static_cast<long long>(ld_p));
  // TMA: 16-byte aligned bases and row / sequence strides; checked here so that a bad stride is an argument error on any machine
  const auto a16 = [](const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15u) == 0; };
  VLPK_CHECK_ARG(a16(d.q) && a16(d.k) && d.ld_q % 8 == 0 && d.ld_kv % 8 == 0 && q_batch_stride % 8 == 0 && d.kv_batch_stride % 8 == 0,
                 "attn_probs: q / k pointers and strides must be 16-byte multiples (ld_q=%lld ld_k=%lld q_bstride=%lld k_bstride=%lld)",
                 static_cast<long long>(d.ld_q), static_cast<long long>(d.ld_kv), static_cast<long long>(q_batch_stride),
                 static_cast<long long>(d.kv_batch_stride));
  const int width = d.heads * HD;
  VLPK_CHECK_ARG(d.ld_q >= width && d.ld_kv >= width, "attn_probs: ld_q=%lld / ld_k=%lld below heads * 64 = %d",
                 static_cast<long long>(d.ld_q), static_cast<long long>(d.ld_kv), width);
  AttnTmaps tm;
  memset(&tm, 0, sizeof(tm));
  VLPK_TRY(make_seq_tmap(&tm.q, d.q, width, d.Lq, d.B, d.ld_q, q_batch_stride));
  VLPK_TRY(make_seq_tmap(&tm.k, d.k, width, d.Lkv, d.B, d.ld_kv, d.kv_batch_stride));
  tm.v = tm.o = tm.dq = tm.dk = tm.dv = tm.q;
  ProbsArgs a;
  a.t = tiled_args(d);
  a.row0 = row0;
  a.p = p;
  a.ld_p = ld_p;
  a.p_bstride = pbs;
  a.vec2 = (reinterpret_cast<uintptr_t>(p) & 7u) == 0 && ld_p % 2 == 0 && pbs % 2 == 0;
  // bandwidth kernel: fp32 P written, Q / K / lse read
  const double bytes = 4.0 * d.B * d.heads * rows * d.Lkv + 2.0 * d.B * width * (rows + d.Lkv) + 4.0 * d.B * d.heads * rows;
  LaunchScope scope(CAT_MISC, bytes, stream);
  return launch_attn_kernel<attn_probs_kernel>(dim3(d.heads, d.B, (rows + TL - 1) / TL), ProbsSmem::DYN, stream, tm, a);
}

}  // namespace vlpk
