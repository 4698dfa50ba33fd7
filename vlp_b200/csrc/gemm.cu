// vlp_b200 — persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   D[M,N] = epilogue( sum_k A[m,k] * B[n,k] )         bf16 operands, fp32 accumulation in registers
//
// Every dense contraction on the VLP hot path goes through this one kernel family
// (SURVEY.md §8a a1,a2,a5,a6,a8,a9,a18 / Appendix B):
//   forward  Linear      : A = activations [M,K] (K-major),  B = weight [N,K] (K-major)
//   dgrad    dX = dY W   : A = dY [M,N'] (K-major),          B = weight [N',K'] read MN-major (no transpose copy)
//   wgrad    dW = dY^T X : A = dY read MN-major, B = X read MN-major, split-K, fp32 TMA reduce-add
//
// Structure (384 threads per CTA, one CTA per SM, 128 x 128 output tiles, two in flight):
//   warpgroup 0     TMA producer   : one elected lane of warp 0 issues cp.async.bulk.tensor into a 128B-swizzled smem ring
//                                    (STAGES deep), tile after tile in the CTA's work order.
//   warpgroups 1,2  MMA + epilogue : ping-pong consumers.  Consumer c takes every other tile of the CTA's work sequence and
//                                    owns all 128 rows of it: two wgmma m64n128k16 per k16 step (rows 0-63 and 64-127 of the
//                                    A stage) into a 2 x 64 register accumulator, one wgmma group kept in flight across
//                                    k-blocks, then the fused pointwise op -> swizzled smem staging -> TMA store (or TMA
//                                    reduce-add for split-K weight gradients).  One consumer's epilogue runs while the other
//                                    consumer's mainloop keeps the tensor pipe busy.
// Each ring stage is read by exactly one consumer.  The producer signals a stage on the full barrier of the consumer whose
// tile it belongs to (one set of full barriers per consumer), so each consumer waits only on phases of its own k-blocks and
// can never mistake a phase of the other consumer's k-blocks for one of its own.  A consumer steps its ring position over
// the k-blocks of the other consumer's tiles.
// Aux epilogues (ADD / MUL / DRELU): while a tile's first wgmma group runs, the consumer's store thread loads the tile's
// [128 x 128] aux block by TMA into the consumer's four staging boxes, in the swizzled layout of the output boxes.  Each
// thread then reads its aux pair from the very place it writes its output pair, so the epilogue has no global loads to wait
// on; per-thread 4-byte loads from global memory left the dgrad through GELU at about half the rate of a plain store.
// Registers: a 12-warp block is capped at 168 per thread, too few for a 128-register accumulator plus an epilogue.  The
// producer warpgroup gives registers back (setmaxnreg 24) and the consumers take them (setmaxnreg 240):
// 128 x 24 + 256 x 240 = 64 512 of the 65 536-register file.  ptxas allocates the consumer code under the 240 only if
// that code contains no trap, so the consumers use the flagging mbar_wait_flag and trap after their loop.
// Tiles are 128 wide only: a 256-wide tile would need a 256-register accumulator per consumer thread.
#include "gemm.cuh"

#include <cstdlib>

#include "host.cuh"
#include "rowops.cuh"

namespace vlpk {

static constexpr int BM = 128;  // rows per tile (one consumer warpgroup: two m64 wgmma row halves)
static constexpr int BK = 64;   // k-block: 64 bf16 = one 128-byte swizzle span
static constexpr int NUM_THREADS = 384;
static constexpr int PRODUCER_REGS = 24;
static constexpr int CONSUMER_REGS = 240;
static constexpr int STG_BYTES = 64 * 128;  // one staging box: 64 rows x 128 bytes
static constexpr int STG_PER_CONSUMER = 4;  // staging boxes per consumer warpgroup (a 4-deep store ring; GELU: 2 pairs)
static constexpr int SMEM_MAX = 232448;     // 227 KB: the per-block opt-in limit of sm_90
static constexpr int BN = 128;              // tile columns (see above)

struct GemmTmaps {
  CUtensorMap a;
  CUtensorMap b[3];
  CUtensorMap d0;
  CUtensorMap d1;
  CUtensorMap aux;  // EPI_ADD / EPI_MUL / EPI_DRELU: the [M,N] side input, read in the output's 64 x 64 boxes
};

struct GemmArgs {
  int M, N, K;
  int b_seg_rows;
  int splits;
  int split_slices;  // EPI_REDUCE_F32: split s reduce-adds into slice s of the 3-D output map (else all into slice 0)
  const __nv_bfloat16* bias[3];
  float relu_scale;
  DropoutCfg drop;
  float* colsum;  // optional [N] fp32: += column sums of the (bf16-rounded) output tile, i.e. the bias gradient of a dgrad output
};

template <int STAGES>
struct SmemLayout {
  static constexpr int A_BYTES = BM * BK * 2;  // 16 KB
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int OFF_STG = STAGES * STAGE_BYTES;  // STG_PER_CONSUMER staging boxes per consumer warpgroup
  static constexpr int OFF_BAR = OFF_STG + 2 * STG_PER_CONSUMER * STG_BYTES;
  static constexpr int NUM_BARS = 3 * STAGES + 2;  // full (one set per consumer) + empty + one aux-tile barrier per consumer
  static constexpr int TOTAL = OFF_BAR + NUM_BARS * 8;
  static constexpr int DYN_BYTES = TOTAL + 1024;  // slack for manual 1024-byte alignment
  static_assert(DYN_BYTES <= SMEM_MAX, "shared memory budget exceeded");
};

struct StageCount {
  // everything left of the 227 KB after the staging boxes, barriers and alignment slack
  static constexpr int value = (SMEM_MAX - 1024 - 2 * STG_PER_CONSUMER * STG_BYTES - 256) / (BM * BK * 2 + BN * BK * 2);
};

__device__ __forceinline__ void wg_bar_sync(int cw) {
  asm volatile("bar.sync %0, 128;" ::"r"(cw + 1) : "memory");
}

template <bool A_MN, bool B_MN, int EPI>
__global__ void __launch_bounds__(NUM_THREADS, 1)
gemm_kernel(const __grid_constant__ GemmTmaps tm, const GemmArgs args) {
  constexpr int STAGES = StageCount::value;
  using L = SmemLayout<STAGES>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));

  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t* full_bar = bars;                // TMA -> consumer c: full_bar[c * STAGES + stage]
  uint64_t* empty_bar = bars + 2 * STAGES;  // consumer -> TMA (one arrival per warp of the consuming warpgroup)
  uint64_t* aux_bar = bars + 3 * STAGES;    // aux tile -> consumer c: aux_bar[c]
  constexpr bool HAS_AUX = (EPI == EPI_ADD || EPI == EPI_MUL || EPI == EPI_DRELU);

  pdl_launch_dependents();  // the next kernel may be scheduled as SMs free up; it blocks in its own pdl_wait()
  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);  // warp-uniform as far as the compiler can tell
  const int lane = threadIdx.x & 31;

  const int num_m = (args.M + BM - 1) / BM;
  const int num_n = (args.N + BN - 1) / BN;
  const int total_kb = (args.K + BK - 1) / BK;
  const int kb_per = (total_kb + args.splits - 1) / args.splits;
  const int num_work = num_m * num_n * args.splits;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm.a);
    tma_prefetch_desc(&tm.b[0]);
    tma_prefetch_desc(&tm.d0);
    if (HAS_AUX) tma_prefetch_desc(&tm.aux);
    for (int i = 0; i < 2 * STAGES; ++i) mbar_init(&full_bar[i], 1);
    for (int i = 0; i < STAGES; ++i) mbar_init(&empty_bar[i], 4);
    for (int i = 0; i < 2; ++i) mbar_init(&aux_bar[i], 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // barrier init and descriptor prefetch above overlap the previous kernel's tail

  if (wg == 0) {
    // ===================================== TMA producer ========================================
    setmaxnreg_dec<PRODUCER_REGS>();
    if (threadIdx.x < 32) {
      // The whole warp walks the loop (warp-uniform state); one elected lane issues.
      int stage = 0;
      uint32_t phase = 0;
      int item = 0;  // index in this CTA's work sequence: even items go to consumer 0, odd ones to consumer 1
      for (int w = blockIdx.x; w < num_work; w += gridDim.x, ++item) {
        uint64_t* fb = full_bar + (item & 1) * STAGES;
        const int n_blk = w % num_n;
        const int m_blk = (w / num_n) % num_m;
        const int split = w / (num_n * num_m);
        const int kb0 = split * kb_per;
        const int kb1 = min(total_kb, kb0 + kb_per);
        const int m0 = m_blk * BM;
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          if (elect_one()) {
            uint8_t* sA = smem + stage * L::STAGE_BYTES;
            uint8_t* sB = sA + L::A_BYTES;
            mbar_arrive_expect_tx(&fb[stage], L::STAGE_BYTES);
            if (!A_MN) {
              tma_load_2d(sA, &tm.a, &fb[stage], kb * BK, m0);
            } else {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(sA + j * 8192, &tm.a, &fb[stage], m0 + j * 64, kb * BK);
            }
            if (!B_MN) {
              const int n0 = n_blk * BN;
              const int seg = n0 / args.b_seg_rows;
              tma_load_2d(sB, &tm.b[seg], &fb[stage], kb * BK, n0 - seg * args.b_seg_rows);
            } else {
              const int k0 = kb * BK;
              const int seg = k0 / args.b_seg_rows;
#pragma unroll
              for (int j = 0; j < BN / 64; ++j)
                tma_load_2d(sB + j * 8192, &tm.b[seg], &fb[stage], n_blk * BN + j * 64, k0 - seg * args.b_seg_rows);
            }
          }
          __syncwarp();
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
  } else {
    // ================================== MMA + epilogue ==========================================
    setmaxnreg_inc<CONSUMER_REGS>();
    const int cw = wg - 1;                         // consumer index: items cw, cw + 2, ... of this CTA's work sequence
    const int t = threadIdx.x - 128 * wg;          // 0..127
    const int fr = (t >> 5) * 16 + (lane >> 2);    // first accumulator row of this thread in each 64-row half (second: fr + 8)
    const int fc = (lane & 3) * 2;                 // first accumulator column within each 8-column group
    const bool store_thread = (t == 0);
    const uint64_t dseed = drop_seed(args.drop);
    // bias exists only for forward Linears (B read K-major, segments tile N)
    constexpr bool HAS_BIAS = !B_MN && (EPI == EPI_STORE || EPI == EPI_GELU || EPI == EPI_RELU);
    uint8_t* stg_base = smem + L::OFF_STG + cw * STG_PER_CONSUMER * STG_BYTES;
    // A rows 64 h .. 64 h + 63 of a stage: 64 rows x 128 B (K-major) or the h-th 64-wide M box (MN-major) — 8 KB apart
    const uint32_t a_base = smem_u32(smem);
    const uint32_t b_base = smem_u32(smem) + L::A_BYTES;
    uint64_t* fb = full_bar + cw * STAGES;
    int stage = 0;        // ring stage of the next k-block, counted over both consumers' k-blocks
    uint32_t phases = 0;  // bit s: parity of this consumer's next wait on fb[s]
    uint32_t box_seq = 0;
    uint32_t aux_phase = 0;  // parity of this consumer's next wait on aux_bar[cw]
    bool timed_out = false;  // a full-barrier wait gave up: trap after the loop (see mbar_wait_flag)
    float acc[2][BN / 2];  // rows 0-63 and 64-127 of the tile
    // Defined here so that the accumulator is live only in the consumer branch (reg_fence reads it before the first wgmma,
    // whose accumulate flag is 0): otherwise it would be live from kernel entry, under the producer's register count.
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[0][i] = acc[1][i] = 0.f;
    for (int w = blockIdx.x + cw * gridDim.x; w < num_work; w += 2 * gridDim.x) {
      const int w_other = w - static_cast<int>(gridDim.x);
      if (w_other >= static_cast<int>(blockIdx.x)) {
        // step over the k-blocks of the other consumer's tile, which precedes this one in the ring
        const int split_o = w_other / (num_n * num_m);
        const int kb0_o = split_o * kb_per;
        stage = (stage + min(total_kb, kb0_o + kb_per) - kb0_o) % STAGES;
      }
      const int n_blk = w % num_n;
      const int m_blk = (w / num_n) % num_m;
      const int split = w / (num_n * num_m);
      const int kb0 = split * kb_per;
      const int kb1 = min(total_kb, kb0 + kb_per);
      const int n0 = n_blk * BN;

      // One wgmma group stays in flight: a stage is released once the group after the one that read it has been issued.
      int prev_stage = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait_flag(&fb[stage], (phases >> stage) & 1u, timed_out);
        phases ^= 1u << stage;
        const uint32_t sa = a_base + stage * L::STAGE_BYTES;
        const uint32_t sb = b_base + stage * L::STAGE_BYTES;
        reg_fence(acc[0]);
        reg_fence(acc[1]);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t bdesc = B_MN ? wgmma_desc_sw128(sb + k * 2048, 8192, 1024) : wgmma_desc_sw128(sb + k * 32, 16, 1024);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const uint32_t sah = sa + h * 8192;
            const uint64_t adesc = A_MN ? wgmma_desc_sw128(sah + k * 2048, 8192, 1024) : wgmma_desc_sw128(sah + k * 32, 16, 1024);
            wgmma_m64n128k16_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc[h], adesc, bdesc, (kb > kb0 || k > 0) ? 1u : 0u);
          }
        }
        wgmma_commit();
        if (HAS_AUX && kb == kb0) {
          // The epilogue's aux tile goes into this consumer's four staging boxes, in the swizzled layout of the output boxes, while
          // the tile's first wgmma group runs: the epilogue then reads it from shared memory instead of from global memory.
          static_assert(STG_PER_CONSUMER == 2 * (BN / 64), "one staging box per aux box of a tile");
          wg_bar_sync(cw);  // every thread of this consumer is done with the previous tile's staging boxes (colsum reads)
          if (store_thread) {
            tma_store_wait_read<0>();
            fence_proxy_async_smem();
            mbar_arrive_expect_tx(&aux_bar[cw], STG_PER_CONSUMER * STG_BYTES);
#pragma unroll
            for (int b = 0; b < STG_PER_CONSUMER; ++b)
              tma_load_2d(stg_base + b * STG_BYTES, &tm.aux, &aux_bar[cw], n0 + (b & 1) * 64, m_blk * BM + (b >> 1) * 64);
          }
        }
        wgmma_wait<1>();
        reg_fence(acc[0]);
        reg_fence(acc[1]);
        if (kb > kb0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);  // this warp's share of the previous slot has been read
        prev_stage = stage;
        if (++stage == STAGES) stage = 0;
      }
      wgmma_wait<0>();
      reg_fence(acc[0]);
      reg_fence(acc[1]);
      if (lane == 0) mbar_arrive(&empty_bar[prev_stage]);

      // ---- epilogue, one 64-row half h at a time: accumulator element acc[h][i] of this thread sits at row
      //      64 h + fr + 8 * ((i >> 1) & 1), column 8 * (i >> 2) + fc + (i & 1)
      if (EPI == EPI_REDUCE_F32) {
        // fp32 staging: 32 columns = 128 bytes per row; one TMA reduce-add box per 64 rows x 32 columns.
        constexpr int NBOX = BN / 32;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m0 = m_blk * BM + h * 64;
#pragma unroll
          for (int c = 0; c < NBOX; ++c) {
            uint8_t* stg = stg_base + (box_seq % STG_PER_CONSUMER) * STG_BYTES;
            if (store_thread) tma_store_wait_read<STG_PER_CONSUMER - 1>();
            wg_bar_sync(cw);
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const int i = c * 16 + 2 * j;
              const int r = fr + 8 * (j & 1), col = 8 * (j >> 1) + fc;
              *reinterpret_cast<float2*>(stg + r * 128 + (((col >> 2) ^ (r & 7)) << 4) + (col & 3) * 4) = make_float2(acc[h][i], acc[h][i + 1]);
            }
            fence_proxy_async_smem();
            wg_bar_sync(cw);
            if (store_thread) {
              tma_reduce_add_3d(&tm.d0, stg, n0 + c * 32, m0, args.split_slices ? split : 0);
              tma_store_commit();
            }
            ++box_seq;
          }
        }
      } else {
        // bf16 staging: 64 columns = 128 bytes per row; one TMA store box per 64 rows x 64 columns.  GELU stores two outputs
        // per box position, from a pair of staging boxes; its two pairs alternate like the single boxes of the other epilogues.
        constexpr int NBOX = BN / 64;
        if (HAS_AUX) {
          mbar_wait_flag(&aux_bar[cw], aux_phase, timed_out);
          aux_phase ^= 1u;
        }
        const __nv_bfloat16* bp = nullptr;
        int bias_off = 0;
        if (HAS_BIAS) {
          const int seg = n0 / args.b_seg_rows;
          bp = args.bias[seg];
          bias_off = seg * args.b_seg_rows;
        }
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int m0 = m_blk * BM + h * 64;
          // Each half recomputes its column offsets, bias addresses and dropout seed: shared by both halves, they would
          // stay live through the first half's epilogue next to the 128-register accumulator and spill.
          int nh = n0;
          const __nv_bfloat16* bph = bp;
          uint64_t dsh = dseed;
          asm volatile("" : "+r"(nh), "+l"(bph), "+l"(dsh));
#pragma unroll
          for (int c = 0; c < NBOX; ++c) {
            uint8_t* stg = (EPI == EPI_GELU) ? stg_base + (box_seq & 1u) * 2 * STG_BYTES : stg_base + (box_seq % STG_PER_CONSUMER) * STG_BYTES;
            uint8_t* stg_g = stg + STG_BYTES;  // EPI_GELU: gelu(u) next to gelu'(u)
            if (store_thread) {
              if (EPI == EPI_GELU) tma_store_wait_read<STG_PER_CONSUMER / 2 - 1>(); else tma_store_wait_read<STG_PER_CONSUMER - 1>();
            }
            wg_bar_sync(cw);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const int i = c * 32 + 2 * j;
              const int r = fr + 8 * (j & 1), col = 8 * (j >> 1) + fc;
              const int n = nh + c * 64 + col;
              const long long m = m0 + r;
              const int so = r * 128 + (((col >> 3) ^ (r & 7)) << 4) + (col & 7) * 2;
              float v0 = acc[h][i], v1 = acc[h][i + 1];
              if (HAS_BIAS) {
                if (bph != nullptr && n < args.N) {
                  const float2 bb = unpack_bf16x2(__ldg(reinterpret_cast<const unsigned int*>(bph + n - bias_off)));
                  v0 += bb.x;
                  v1 += bb.y;
                }
              }
              if (EPI == EPI_GELU) {
                float g0, d0, g1, d1;
                gelu_and_grad(v0, g0, d0);
                gelu_and_grad(v1, g1, d1);
                *reinterpret_cast<uint32_t*>(stg + so) = pack_bf16x2(d0, d1);    // gelu'(u): all backward needs from the pre-activation
                *reinterpret_cast<uint32_t*>(stg_g + so) = pack_bf16x2(g0, g1);  // gelu(u)
                continue;
              }
              if (EPI == EPI_RELU) {
                uint32_t keep = 0xFFu;
                if (args.drop.p > 0.f)
                  keep = dropout_keep8(dsh, args.drop.site, (static_cast<uint64_t>(m) * args.N + (n - fc)) >> 3, args.drop.thresh16);
                v0 = fmaxf(v0, 0.f);
                v1 = fmaxf(v1, 0.f);
                v0 = ((keep >> fc) & 1u) ? v0 * args.drop.scale : 0.f;
                v1 = ((keep >> (fc + 1)) & 1u) ? v1 * args.drop.scale : 0.f;
              } else if (EPI == EPI_ADD || EPI == EPI_MUL || EPI == EPI_DRELU) {
                // this thread's aux pair, at the place its output pair goes (TMA zero-filled it beyond M and N)
                const float2 x = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(stg + so));
                if (EPI == EPI_ADD) {
                  v0 += x.x;
                  v1 += x.y;
                } else if (EPI == EPI_MUL) {
                  v0 *= x.x;
                  v1 *= x.y;
                } else {
                  v0 = x.x > 0.f ? v0 * args.relu_scale : 0.f;
                  v1 = x.y > 0.f ? v1 * args.relu_scale : 0.f;
                }
              }
              *reinterpret_cast<uint32_t*>(stg + so) = pack_bf16x2(v0, v1);
            }
            fence_proxy_async_smem();
            wg_bar_sync(cw);
            if (store_thread) {
              tma_store_2d(&tm.d0, stg, nh + c * 64, m0);
              if (EPI == EPI_GELU) tma_store_2d(&tm.d1, stg_g, nh + c * 64, m0);
              tma_store_commit();
            }
            if (EPI != EPI_GELU && args.colsum != nullptr) {
              // bias gradient = column sums of this output: fold the staged [64 x 64] bf16 box (rows beyond M are zero).
              // Two threads per column take 32 rows each; the box is not overwritten before the barrier STG_PER_CONSUMER boxes on.
              const int col = t & 63, r0 = (t >> 6) * 32;
              float acc_c = 0.f;
#pragma unroll 8
              for (int rr = r0; rr < r0 + 32; ++rr) {
                const __nv_bfloat16 v = *reinterpret_cast<const __nv_bfloat16*>(stg + rr * 128 + (((col >> 3) ^ (rr & 7)) << 4) + (col & 7) * 2);
                acc_c += __bfloat162float(v);
              }
              if (nh + c * 64 + col < args.N) atomicAdd(args.colsum + nh + c * 64 + col, acc_c);
            }
            ++box_seq;
          }
        }
      }
    }
    if (store_thread) tma_store_wait<0>();
    if (timed_out) __trap();
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
template <bool A_MN, bool B_MN, int EPI>
static int launch_inst(const GemmTmaps& tm, const GemmArgs& args, int num_work, cudaStream_t stream) {
  constexpr int STAGES = StageCount::value;
  using L = SmemLayout<STAGES>;
  auto kfn = gemm_kernel<A_MN, B_MN, EPI>;
  static bool attr_set = false;  // benign race: idempotent
  if (!attr_set) {
    VLPK_CUDA(cudaFuncSetAttribute(kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, L::DYN_BYTES));
    attr_set = true;
  }
  const int max_ctas = gemm_sms();
  const int ctas = num_work < max_ctas ? num_work : max_ctas;
  LaunchScope scope(A_MN ? CAT_GEMM_WGRAD : (B_MN ? CAT_GEMM_DGRAD : CAT_GEMM_FWD), 2.0 * args.M * args.N * args.K, stream);
  VLPK_CUDA(launch_ex(kfn, dim3(ctas), dim3(NUM_THREADS), L::DYN_BYTES, stream, 1, tm, args));
  return 0;
}

static int dispatch(const GemmDesc& g, const GemmTmaps& tm, const GemmArgs& args, int num_work, cudaStream_t s) {
  if (!g.a_mn && !g.b_mn) {
    switch (g.epi) {
      case EPI_STORE: return launch_inst<false, false, EPI_STORE>(tm, args, num_work, s);
      case EPI_GELU: return launch_inst<false, false, EPI_GELU>(tm, args, num_work, s);
      case EPI_RELU: return launch_inst<false, false, EPI_RELU>(tm, args, num_work, s);
      default: break;
    }
  } else if (!g.a_mn && g.b_mn) {
    switch (g.epi) {
      case EPI_STORE: return launch_inst<false, true, EPI_STORE>(tm, args, num_work, s);
      case EPI_ADD: return launch_inst<false, true, EPI_ADD>(tm, args, num_work, s);
      case EPI_MUL: return launch_inst<false, true, EPI_MUL>(tm, args, num_work, s);
      case EPI_DRELU: return launch_inst<false, true, EPI_DRELU>(tm, args, num_work, s);
      case EPI_REDUCE_F32: return launch_inst<false, true, EPI_REDUCE_F32>(tm, args, num_work, s);  // split-K dgrad (MLM head)
      default: break;
    }
  } else if (g.a_mn && g.b_mn) {
    if (g.epi == EPI_REDUCE_F32) return launch_inst<true, true, EPI_REDUCE_F32>(tm, args, num_work, s);
    if (g.epi == EPI_STORE) return launch_inst<true, true, EPI_STORE>(tm, args, num_work, s);        // bf16 wgrad, no split-K
  }
  set_error("gemm: unsupported (a_mn=%d, b_mn=%d, epi=%d) combination", (int)g.a_mn, (int)g.b_mn, g.epi);
  return -1;
}

// Cost model used to pick split-K: rounds of the persistent loop x per-tile cost, where the mainloop cost per k-block is
// proportional to the operand bytes each SM pulls from L2 (128 rows of A + BN rows of B) and the epilogue cost to the BN
// columns each CTA drains.
static double tile_cost(int M, int N, int total_kb, int splits, bool reduce) {
  const int num_m = (M + BM - 1) / BM;
  const int num_n = (N + BN - 1) / BN;
  const long long tiles = static_cast<long long>(num_m) * num_n * splits;
  // deterministic mode: the split count decides how a weight gradient is summed, so it must not follow vlpk_set_reserved_sms
  const int slots = deterministic() ? num_sms() : gemm_sms();
  const long long rounds = (tiles + slots - 1) / slots;
  const int kb_per = (total_kb + splits - 1) / splits;
  const double mainloop = kb_per * (128.0 + double(BN));
  const double epi = (reduce ? 3.0 : 1.5) * BN;
  return rounds * (mainloop + epi + 60.0);
}

// Tile N (always BN) and split-K for one GEMM (pure host logic; exposed to the CPU tests as vlpk_debug_plan_gemm).
int plan_gemm(const GemmDesc& g, int* bn_out, int* splits_out) {
  const int seg_rows = g.nseg > 1 ? g.b_seg_rows : (g.b_mn ? g.K : g.N);
  const int total_kb = (g.K + BK - 1) / BK;
  const bool reduce = (g.epi == EPI_REDUCE_F32);
  VLPK_CHECK_ARG(g.bn == 0 || g.bn == BN, "gemm: no valid tile configuration (bn=%d; tiles are %d wide)", g.bn, BN);
  VLPK_CHECK_ARG(g.nseg == 1 || seg_rows % (g.b_mn ? BK : BN) == 0, "gemm: segment rows %d not tile aligned", seg_rows);
  int splits = 1;
  if (reduce) {
    const int max_s = total_kb / 8 > 0 ? total_kb / 8 : 1;
    if (g.splits > 0) {
      splits = g.splits < max_s ? g.splits : max_s;
    } else {
      double best = 1e300;
      for (int s = 1; s <= max_s; ++s) {
        const double c = tile_cost(g.M, g.N, total_kb, s, reduce);
        if (c < best) {
          best = c;
          splits = s;
        }
      }
    }
  }
  if (splits > total_kb) splits = total_kb;
  {
    const int kb_per = (total_kb + splits - 1) / splits;
    splits = (total_kb + kb_per - 1) / kb_per;  // no empty splits
  }
  *bn_out = BN;
  *splits_out = splits;
  return 0;
}

int launch_gemm(const GemmDesc& g, cudaStream_t stream) {
  VLPK_CHECK_ARG(g.M > 0 && g.N > 0 && g.K > 0, "gemm: empty problem M=%d N=%d K=%d", g.M, g.N, g.K);
  VLPK_CHECK_ARG(g.N % 8 == 0, "gemm: N=%d must be a multiple of 8", g.N);
  VLPK_CHECK_ARG(g.nseg >= 1 && g.nseg <= 3, "gemm: nseg=%d", g.nseg);
  const int seg_rows = g.nseg > 1 ? g.b_seg_rows : (g.b_mn ? g.K : g.N);
  const bool reduce = (g.epi == EPI_REDUCE_F32);
  VLPK_CHECK_ARG(g.splits <= 1 || reduce, "gemm: split-K needs EPI_REDUCE_F32");
  VLPK_CHECK_ARG(g.b_rows == 0 || (g.nseg == 1 && g.b_rows <= (g.b_mn ? g.K : g.N)), "gemm: b_rows=%d needs a single B segment", g.b_rows);

  // ---- choose tile N and split-K
  int bn = BN, splits = 1;
  VLPK_TRY(plan_gemm(g, &bn, &splits));

  GemmTmaps tm;
  memset(&tm, 0, sizeof(tm));
  if (!g.a_mn) {
    VLPK_TRY(make_tmap_2d(&tm.a, TM_BF16, g.A, g.K, g.M, g.lda, BK, BM));
  } else {
    VLPK_TRY(make_tmap_2d(&tm.a, TM_BF16, g.A, g.M, g.K, g.lda, 64, BK));
  }
  for (int s = 0; s < g.nseg; ++s) {
    if (!g.b_mn) {
      const int rows = g.nseg > 1 ? seg_rows : (g.b_rows > 0 ? g.b_rows : g.N);
      VLPK_TRY(make_tmap_2d(&tm.b[s], TM_BF16, g.B[s], g.K, rows, g.ldb, BK, bn));
    } else {
      const int rows = g.nseg > 1 ? seg_rows : (g.b_rows > 0 ? g.b_rows : g.K);
      VLPK_TRY(make_tmap_2d(&tm.b[s], TM_BF16, g.B[s], g.N, rows, g.ldb, 64, BK));
    }
  }
  for (int s = g.nseg; s < 3; ++s) tm.b[s] = tm.b[0];
  if (reduce) {
    // 3-D map [slices][M][N]: one slice, or one per split when the caller sums the splits itself
    VLPK_CHECK_ARG(g.split_stride == 0 || (g.split_stride % 4 == 0 && g.split_stride >= static_cast<int64_t>(g.M) * g.ldd0),
                   "gemm: split_stride %lld must be a multiple of 4 and cover M x ldd0", (long long)g.split_stride);
    const uint64_t dims[3] = {static_cast<uint64_t>(g.N), static_cast<uint64_t>(g.M), static_cast<uint64_t>(g.split_stride ? splits : 1)};
    const uint64_t strides[2] = {static_cast<uint64_t>(g.ldd0) * 4,
                                 static_cast<uint64_t>(g.split_stride ? g.split_stride : static_cast<int64_t>(g.M) * g.ldd0) * 4};
    const uint32_t box[3] = {32, 64, 1};
    VLPK_TRY(make_tmap(&tm.d0, TM_F32, 3, g.D0, dims, strides, box));
    tm.d1 = tm.d0;
  } else {
    VLPK_TRY(make_tmap_2d(&tm.d0, TM_BF16, g.D0, g.N, g.M, g.ldd0, 64, 64));
    if (g.epi == EPI_GELU) {
      VLPK_CHECK_ARG(g.D1 != nullptr, "gemm: EPI_GELU needs D1");
      VLPK_TRY(make_tmap_2d(&tm.d1, TM_BF16, g.D1, g.N, g.M, g.ldd1, 64, 64));
    } else {
      tm.d1 = tm.d0;
    }
  }
  VLPK_CHECK_ARG(g.colsum == nullptr || (!reduce && g.epi != EPI_GELU), "gemm: colsum fusion is for single-output bf16 epilogues");
  if (g.epi == EPI_ADD || g.epi == EPI_MUL || g.epi == EPI_DRELU) {
    VLPK_CHECK_ARG(g.aux != nullptr && (g.ld_aux % 8) == 0 && (reinterpret_cast<uintptr_t>(g.aux) & 15u) == 0,
                   "gemm: aux must be 16-byte aligned with ld %% 8 == 0");
    VLPK_TRY(make_tmap_2d(&tm.aux, TM_BF16, g.aux, g.N, g.M, g.ld_aux, 64, 64));
  } else {
    tm.aux = tm.d0;
  }

  GemmArgs a;
  a.M = g.M;
  a.N = g.N;
  a.K = g.K;
  a.b_seg_rows = seg_rows;
  a.splits = splits;
  a.split_slices = (reduce && g.split_stride > 0) ? 1 : 0;
  for (int s = 0; s < 3; ++s) a.bias[s] = (s < g.nseg) ? g.bias[s] : nullptr;
  a.relu_scale = g.relu_scale;
  a.colsum = g.colsum;
  a.drop = g.drop;

  const int num_m = (g.M + BM - 1) / BM;
  const int num_n = (g.N + bn - 1) / bn;
  const int num_work = num_m * num_n * splits;
  return dispatch(g, tm, a, num_work, stream);
}

int launch_gemm_split_slices(GemmDesc g, int slot, cudaStream_t stream) {
  VLPK_CHECK_ARG(g.epi == EPI_REDUCE_F32 && g.split_stride == 0, "gemm: split slices are for EPI_REDUCE_F32 into one D0");
  int bn = 0, splits = 1;
  VLPK_TRY(plan_gemm(g, &bn, &splits));
  if (splits == 1) return launch_gemm(g, stream);  // one reduce-add per element: already order-free
  VLPK_CHECK_ARG(g.ldd0 == g.N, "gemm: split slices need a dense D0 (ldd0 %lld != N %d)", (long long)g.ldd0, g.N);
  const long long n = static_cast<long long>(g.M) * g.N;
  float* part = scratch_f32(slot, static_cast<size_t>(n) * splits, stream);
  if (part == nullptr) return -1;
  VLPK_CUDA(cudaMemsetAsync(part, 0, static_cast<size_t>(n) * splits * sizeof(float), stream));
  float* out = static_cast<float*>(g.D0);
  g.D0 = part;
  g.splits = splits;
  g.split_stride = n;
  VLPK_TRY(launch_gemm(g, stream));
  return launch_sum_parts(part, splits, n, out, stream);
}

}  // namespace vlpk
