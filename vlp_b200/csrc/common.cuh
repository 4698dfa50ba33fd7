// vlp_b200 — sm_90a device-side primitives shared by every kernel in this library.
//
// Thin inline-PTX wrappers for the Hopper async machinery (mbarrier, TMA, wgmma),
// the wgmma shared-memory descriptor builder, a counter-based Philox RNG for
// regenerable dropout masks, and small bf16 pack helpers.  Nothing here is a translation of
// reference code: the reference (LuoweiZhou/VLP) has no native code at all (SURVEY.md §2.1).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "wgmma.cuh"

namespace vlpk {

// ----------------------------------------------------------------------------------------------
// address helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31u; }

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a protocol bug must surface as a trap (=> CUDA error the host reports), never as a
// hung GPU.  2^28 polls of a HW-sleeping try_wait is many seconds — far beyond any legitimate wait.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 28)) { __trap(); }
  }
}
// The same bounded spin for code that must not contain a trap: a trap inside a setmaxnreg.inc region makes ptxas
// allocate that region under the launch register count.  A timeout sets `timed_out`, after which every later wait
// returns at once; the caller traps once it has left the region.
__device__ __forceinline__ void mbar_wait_flag(uint64_t* bar, uint32_t parity, bool& timed_out) {
  uint32_t spins = 0;
  while (!timed_out && !mbar_try_wait(bar, parity)) {
    if (++spins > (1u << 28)) timed_out = true;
  }
}

// ----------------------------------------------------------------------------------------------
// Programmatic dependent launch: a kernel launched with the programmatic-stream-serialization attribute may start while
// its predecessor drains; everything that touches the predecessor's output must come after pdl_wait() (which returns once
// the prerequisite grid has completed and its memory is visible).  Both are no-ops for ordinary launches.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// TMA (cp.async.bulk.tensor)
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* m, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* m, const void* src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_reduce_add_3d(const CUtensorMap* m, const void* src, int c0, int c1, int c2) {
  asm volatile("cp.reduce.async.bulk.tensor.3d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3, %4}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void tma_store_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void tma_store_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma (warpgroup MMA) issue / completion
// ----------------------------------------------------------------------------------------------
// Orders this warpgroup's register accesses before the wgmma that follow (required before the first wgmma that reads or
// accumulates into registers written by ordinary instructions).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Register reallocation between warpgroups: every warp of the warpgroup executes it, and the block's producer / consumer
// counts must fit the register file together.
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(N)); }
template <uint32_t N>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(N)); }
// Keeps the compiler from moving accesses of an accumulator across wgmma_fence / wgmma_wait.
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ----------------------------------------------------------------------------------------------
// wgmma shared-memory matrix descriptor (PTX ISA "Matrix Descriptor Format" for wgmma), 128-byte swizzle:
//   start address >>4 : bits [0,14)   leading byte offset >>4 : bits [16,30)   stride byte offset >>4 : bits [32,46)
//   swizzle mode (1 = 128B) : bits [62,64)
// K-major operand (rows of 64 bf16 = 128 B):  SBO = 1024 (8-row group), LBO unused;  +32 B per K = 16 step.
// MN-major operand ([k][64 mn] boxes of 8 KB): SBO = 1024 (8-k group), LBO = 8192 (next 64-wide MN box);  +2048 B per K = 16.
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t wgmma_desc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= 1ull << 62;
  return d;
}

// ----------------------------------------------------------------------------------------------
// bf16 helpers
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}
__device__ __forceinline__ float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// erf-GELU of the reference (pytorch_pretrained_bert/modeling.py:62-67): gelu(x) = x * 0.5 * (1 + erf(x / sqrt 2)), and its
// derivative gelu'(x) = Phi(x) + x * phi(x).  erf is evaluated with Abramowitz-Stegun 7.1.26 (|abs err| <= 1.5e-7, i.e.
// below fp32 round-off of the surrounding arithmetic and 4 orders below bf16 resolution); it shares one exp(-x^2/2) with
// the density term, so the pair costs one MUFU.EX2 + one MUFU.RCP + ~12 FMAs.  (This is the erf form, not the tanh
// approximation the reference explicitly does not use.)
// MUFU approximations without the IEEE slow paths the libm-style calls carry (rcp.rn / exp2f expand to a guarded
// subroutine call per element, which made the GELU epilogue instruction-bound).  ~1 ulp-level error (2^-22 relative).
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float fast_rcp(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void gelu_and_grad(float x, float& g, float& d) {
  const float ax = fabsf(x);
  const float e = fast_ex2(-0.72134752044448170f * x * x);  // exp(-x^2 / 2)
  const float t = fast_rcp(fmaf(0.3275911f * 0.70710678118654752f, ax, 1.0f));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  const float erf_abs = fmaf(-poly, e, 1.0f);        // erf(|x|/sqrt2)
  const float cdf = 0.5f * (1.0f + copysignf(erf_abs, x));
  g = x * cdf;
  d = fmaf(x * 0.3989422804014327f, e, cdf);
}

// ----------------------------------------------------------------------------------------------
// Philox4x32-10: counter-based RNG so backward can regenerate forward's dropout mask from
// (seed, site-offset, element index) without storing it (SURVEY.md §7 "Dropout parity").
// ----------------------------------------------------------------------------------------------
struct Philox {
  __device__ __forceinline__ static uint4 gen(uint64_t seed, uint64_t ctr_hi, uint64_t ctr_lo) {
    uint32_t k0 = static_cast<uint32_t>(seed), k1 = static_cast<uint32_t>(seed >> 32);
    uint4 c = make_uint4(static_cast<uint32_t>(ctr_lo), static_cast<uint32_t>(ctr_lo >> 32),
                         static_cast<uint32_t>(ctr_hi), static_cast<uint32_t>(ctr_hi >> 32));
#pragma unroll
    for (int i = 0; i < 10; ++i) {
      const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
      const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
      c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
      k0 += 0x9E3779B9u;
      k1 += 0xBB67AE85u;
    }
    return c;
  }
};
// Dropout keep-decision for 8 consecutive elements starting at element index `idx8*8` of site `site`.
// Returns an 8-bit mask (bit i set = keep).  16 random bits per element, threshold = p * 65536.
__device__ __forceinline__ uint32_t dropout_keep8(uint64_t seed, uint64_t site, uint64_t idx8, uint32_t thresh16) {
  const uint4 r = Philox::gen(seed, site, idx8);
  uint32_t m = 0;
  m |= ((r.x & 0xFFFFu) >= thresh16) ? 1u : 0u;
  m |= ((r.x >> 16) >= thresh16) ? 2u : 0u;
  m |= ((r.y & 0xFFFFu) >= thresh16) ? 4u : 0u;
  m |= ((r.y >> 16) >= thresh16) ? 8u : 0u;
  m |= ((r.z & 0xFFFFu) >= thresh16) ? 16u : 0u;
  m |= ((r.z >> 16) >= thresh16) ? 32u : 0u;
  m |= ((r.w & 0xFFFFu) >= thresh16) ? 64u : 0u;
  m |= ((r.w >> 16) >= thresh16) ? 128u : 0u;
  return m;
}

struct DropoutCfg {
  float p;            // drop probability (0 => disabled)
  float scale;        // 1/(1-p)
  uint32_t thresh16;  // floor(p * 65536)
  uint64_t seed;
  uint64_t site;  // distinguishes (layer, site) streams
  const unsigned long long* seed_ptr;  // optional device-side counter added to seed (CUDA-graph replays)
  const unsigned char* bits;  // optional (attention backward): forward's keep-decisions of this site, bits[i] = dropout_keep8(seed,
                              // site, i), read back instead of re-evaluating Philox (the kernel is instruction-issue bound)
};

__device__ __forceinline__ uint64_t drop_seed(const DropoutCfg& d) {
  return (d.p > 0.f && d.seed_ptr != nullptr) ? d.seed + *d.seed_ptr : d.seed;
}

__host__ inline DropoutCfg make_dropout(float p, uint64_t seed, uint64_t site,
                                        const unsigned long long* seed_ptr = nullptr) {
  DropoutCfg d;
  d.bits = nullptr;
  d.seed_ptr = seed_ptr;
  d.p = p;
  d.scale = p > 0.f ? 1.0f / (1.0f - p) : 1.0f;
  d.thresh16 = static_cast<uint32_t>(p * 65536.0f);
  d.seed = seed;
  d.site = site;
  return d;
}

}  // namespace vlpk
