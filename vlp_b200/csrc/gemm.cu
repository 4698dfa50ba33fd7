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
// Structure (288 threads per CTA, one CTA per SM, one 128 x 128 output tile at a time):
//   warp 8          TMA producer   : one elected lane issues cp.async.bulk.tensor into a 128B-swizzled smem ring (STAGES deep)
//   warpgroups 0,1  MMA + epilogue : each owns 64 rows of the tile: wgmma m64n128k16 (x4 per 64-wide k-block) into a register
//                                    accumulator, then the fused pointwise op -> swizzled smem staging -> TMA store (or TMA
//                                    reduce-add for split-K weight gradients).  While one warpgroup drains its epilogue the
//                                    producer keeps filling the ring for the next tile.
// Tiles are 128 wide only: a 256-wide tile needs a 128-register accumulator per thread, and a 9-warp (or 12-warp) block is
// capped at 168 registers, so its epilogues spill.
#include "gemm.cuh"

#include <cstdlib>

#include "host.cuh"

namespace vlpk {

static constexpr int BM = 128;  // rows per CTA tile (two warpgroups x 64)
static constexpr int BK = 64;   // k-block: 64 bf16 = one 128-byte swizzle span
static constexpr int NUM_THREADS = 288;
static constexpr int STG_BYTES = 64 * 128;  // one staging box: 64 rows x 128 bytes
static constexpr int SMEM_MAX = 232448;     // 227 KB: the per-block opt-in limit of sm_90
static constexpr int BN = 128;              // tile columns (see above)

struct GemmTmaps {
  CUtensorMap a;
  CUtensorMap b[3];
  CUtensorMap d0;
  CUtensorMap d1;
};

struct GemmArgs {
  int M, N, K;
  int b_seg_rows;
  int splits;
  int split_slices;  // EPI_REDUCE_F32: split s reduce-adds into slice s of the 3-D output map (else all into slice 0)
  const __nv_bfloat16* bias[3];
  const __nv_bfloat16* aux;
  long long ld_aux;
  float relu_scale;
  DropoutCfg drop;
  float* colsum;  // optional [N] fp32: += column sums of the (bf16-rounded) output tile, i.e. the bias gradient of a dgrad output
};

template <int STAGES>
struct SmemLayout {
  static constexpr int A_BYTES = BM * BK * 2;  // 16 KB
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int OFF_STG = STAGES * STAGE_BYTES;  // 4 staging boxes (2 per MMA warpgroup)
  static constexpr int OFF_BAR = OFF_STG + 4 * STG_BYTES;
  static constexpr int NUM_BARS = 2 * STAGES;
  static constexpr int TOTAL = OFF_BAR + NUM_BARS * 8;
  static constexpr int DYN_BYTES = TOTAL + 1024;  // slack for manual 1024-byte alignment
  static_assert(DYN_BYTES <= SMEM_MAX, "shared memory budget exceeded");
};

struct StageCount {
  // everything left of the 227 KB after the 4 staging boxes, barriers and alignment slack
  static constexpr int value = (SMEM_MAX - 1024 - 4 * STG_BYTES - 256) / (BM * BK * 2 + BN * BK * 2);
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
  uint64_t* full_bar = bars;            // TMA -> MMA
  uint64_t* empty_bar = bars + STAGES;  // MMA -> TMA (one arrival per MMA warp)

  pdl_launch_dependents();  // the next kernel may be scheduled as SMs free up; it blocks in its own pdl_wait()
  const int wg = threadIdx.x >> 7;
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
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);
    }
    fence_mbar_init();
  }
  __syncthreads();
  pdl_wait();  // barrier init and descriptor prefetch above overlap the previous kernel's tail

  if (wg == 2) {
    // ===================================== TMA producer ========================================
    {
      // The whole warp walks the loop (warp-uniform state); one elected lane issues.
      int stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
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
            mbar_arrive_expect_tx(&full_bar[stage], L::STAGE_BYTES);
            if (!A_MN) {
              tma_load_2d(sA, &tm.a, &full_bar[stage], kb * BK, m0);
            } else {
#pragma unroll
              for (int j = 0; j < BM / 64; ++j) tma_load_2d(sA + j * 8192, &tm.a, &full_bar[stage], m0 + j * 64, kb * BK);
            }
            if (!B_MN) {
              const int n0 = n_blk * BN;
              const int seg = n0 / args.b_seg_rows;
              tma_load_2d(sB, &tm.b[seg], &full_bar[stage], kb * BK, n0 - seg * args.b_seg_rows);
            } else {
              const int k0 = kb * BK;
              const int seg = k0 / args.b_seg_rows;
#pragma unroll
              for (int j = 0; j < BN / 64; ++j)
                tma_load_2d(sB + j * 8192, &tm.b[seg], &full_bar[stage], n_blk * BN + j * 64, k0 - seg * args.b_seg_rows);
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
    const int cw = wg;                             // rows [64 cw, 64 cw + 64) of every tile
    const int t = threadIdx.x - 128 * wg;          // 0..127
    const int fr = (t >> 5) * 16 + (lane >> 2);    // first accumulator row of this thread (second: fr + 8)
    const int fc = (lane & 3) * 2;                 // first accumulator column within each 8-column group
    const bool store_thread = (t == 0);
    const uint64_t dseed = drop_seed(args.drop);
    // bias exists only for forward Linears (B read K-major, segments tile N)
    constexpr bool HAS_BIAS = !B_MN && (EPI == EPI_STORE || EPI == EPI_GELU || EPI == EPI_RELU);
    uint8_t* stg0 = smem + L::OFF_STG + cw * 2 * STG_BYTES;
    uint8_t* stg1 = stg0 + STG_BYTES;
    // A rows of this warpgroup: 64 rows x 128 B (K-major) or the second 64-wide M box (MN-major) — 8 KB further either way
    const uint32_t a_base = smem_u32(smem) + cw * 8192;
    const uint32_t b_base = smem_u32(smem) + L::A_BYTES;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t box_seq = 0;
    float acc[BN / 2];
    for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
      const int n_blk = w % num_n;
      const int m_blk = (w / num_n) % num_m;
      const int split = w / (num_n * num_m);
      const int kb0 = split * kb_per;
      const int kb1 = min(total_kb, kb0 + kb_per);
      const int n0 = n_blk * BN;
      const int m0 = m_blk * BM + cw * 64;

      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = a_base + stage * L::STAGE_BYTES;
        const uint32_t sb = b_base + stage * L::STAGE_BYTES;
        reg_fence(acc);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k) {
          const uint64_t adesc = A_MN ? wgmma_desc_sw128(sa + k * 2048, 8192, 1024) : wgmma_desc_sw128(sa + k * 32, 16, 1024);
          const uint64_t bdesc = B_MN ? wgmma_desc_sw128(sb + k * 2048, 8192, 1024) : wgmma_desc_sw128(sb + k * 32, 16, 1024);
          wgmma_m64n128k16_ss<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, adesc, bdesc, (kb > kb0 || k > 0) ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        reg_fence(acc);
        if (lane == 0) mbar_arrive(&empty_bar[stage]);  // this warp's share of the slot has been read
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1u;
        }
      }

      // ---- epilogue: accumulator element i of this thread sits at row fr + 8 * ((i >> 1) & 1), column 8 * (i >> 2) + fc + (i & 1)
      if (EPI == EPI_REDUCE_F32) {
        // fp32 staging: 32 columns = 128 bytes per row; one TMA reduce-add box per 32 columns.
        constexpr int NBOX = BN / 32;
#pragma unroll
        for (int c = 0; c < NBOX; ++c) {
          uint8_t* stg = (box_seq & 1u) ? stg1 : stg0;
          if (store_thread) tma_store_wait_read<1>();
          wg_bar_sync(cw);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int i = c * 16 + 2 * j;
            const int r = fr + 8 * (j & 1), col = 8 * (j >> 1) + fc;
            *reinterpret_cast<float2*>(stg + r * 128 + (((col >> 2) ^ (r & 7)) << 4) + (col & 3) * 4) = make_float2(acc[i], acc[i + 1]);
          }
          fence_proxy_async_smem();
          wg_bar_sync(cw);
          if (store_thread) {
            tma_reduce_add_3d(&tm.d0, stg, n0 + c * 32, m0, args.split_slices ? split : 0);
            tma_store_commit();
          }
          ++box_seq;
        }
      } else {
        // bf16 staging: 64 columns = 128 bytes per row; one TMA store box per 64 columns.
        constexpr int NBOX = BN / 64;
        const __nv_bfloat16* bp = nullptr;
        int bias_off = 0;
        if (HAS_BIAS) {
          const int seg = n0 / args.b_seg_rows;
          bp = args.bias[seg];
          bias_off = seg * args.b_seg_rows;
        }
#pragma unroll
        for (int c = 0; c < NBOX; ++c) {
          uint8_t* stg = (EPI == EPI_GELU) ? stg0 : ((box_seq & 1u) ? stg1 : stg0);
          if (store_thread) {
            if (EPI == EPI_GELU) tma_store_wait_read<0>(); else tma_store_wait_read<1>();
          }
          wg_bar_sync(cw);
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int i = c * 32 + 2 * j;
            const int r = fr + 8 * (j & 1), col = 8 * (j >> 1) + fc;
            const int n = n0 + c * 64 + col;
            const long long m = m0 + r;
            float v0 = acc[i], v1 = acc[i + 1];
            if (HAS_BIAS) {
              if (bp != nullptr && n < args.N) {
                const float2 bb = unpack_bf16x2(__ldg(reinterpret_cast<const unsigned int*>(bp + n - bias_off)));
                v0 += bb.x;
                v1 += bb.y;
              }
            }
            const int so = r * 128 + (((col >> 3) ^ (r & 7)) << 4) + (col & 7) * 2;
            if (EPI == EPI_GELU) {
              float g0, d0, g1, d1;
              gelu_and_grad(v0, g0, d0);
              gelu_and_grad(v1, g1, d1);
              *reinterpret_cast<uint32_t*>(stg0 + so) = pack_bf16x2(d0, d1);  // gelu'(u): all backward needs from the pre-activation
              *reinterpret_cast<uint32_t*>(stg1 + so) = pack_bf16x2(g0, g1);  // gelu(u)
              continue;
            }
            if (EPI == EPI_RELU) {
              uint32_t keep = 0xFFu;
              if (args.drop.p > 0.f)
                keep = dropout_keep8(dseed, args.drop.site, (static_cast<uint64_t>(m) * args.N + (n - fc)) >> 3, args.drop.thresh16);
              v0 = fmaxf(v0, 0.f);
              v1 = fmaxf(v1, 0.f);
              v0 = ((keep >> fc) & 1u) ? v0 * args.drop.scale : 0.f;
              v1 = ((keep >> (fc + 1)) & 1u) ? v1 * args.drop.scale : 0.f;
            } else if (EPI == EPI_ADD || EPI == EPI_MUL || EPI == EPI_DRELU) {
              float2 x = make_float2(0.f, 0.f);
              if (m < args.M && n < args.N) x = unpack_bf16x2(__ldg(reinterpret_cast<const unsigned int*>(args.aux + m * args.ld_aux + n)));
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
            tma_store_2d(&tm.d0, stg, n0 + c * 64, m0);
            if (EPI == EPI_GELU) tma_store_2d(&tm.d1, stg1, n0 + c * 64, m0);
            tma_store_commit();
          }
          if (EPI != EPI_GELU && args.colsum != nullptr) {
            // bias gradient = column sums of this output: fold the staged [64 x 64] bf16 box (rows beyond M are zero).
            // Two threads per column take 32 rows each; the buffer is not overwritten before the next-but-one barrier.
            const int col = t & 63, r0 = (t >> 6) * 32;
            float acc_c = 0.f;
#pragma unroll 8
            for (int rr = r0; rr < r0 + 32; ++rr) {
              const __nv_bfloat16 v = *reinterpret_cast<const __nv_bfloat16*>(stg + rr * 128 + (((col >> 3) ^ (rr & 7)) << 4) + (col & 7) * 2);
              acc_c += __bfloat162float(v);
            }
            if (n0 + c * 64 + col < args.N) atomicAdd(args.colsum + n0 + c * 64 + col, acc_c);
          }
          ++box_seq;
        }
      }
    }
    if (store_thread) tma_store_wait<0>();
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
  const int slots = gemm_sms();
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
  }

  GemmArgs a;
  a.M = g.M;
  a.N = g.N;
  a.K = g.K;
  a.b_seg_rows = seg_rows;
  a.splits = splits;
  a.split_slices = (reduce && g.split_stride > 0) ? 1 : 0;
  for (int s = 0; s < 3; ++s) a.bias[s] = (s < g.nseg) ? g.bias[s] : nullptr;
  a.aux = g.aux;
  a.ld_aux = g.ld_aux;
  a.relu_scale = g.relu_scale;
  a.colsum = g.colsum;
  a.drop = g.drop;

  const int num_m = (g.M + BM - 1) / BM;
  const int num_n = (g.N + bn - 1) / bn;
  const int num_work = num_m * num_n * splits;
  return dispatch(g, tm, a, num_work, stream);
}

}  // namespace vlpk
