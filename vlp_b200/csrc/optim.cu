// vlp_b200 — BertAdam.step (pytorch_pretrained_bert/optimization.py:112-182) for ALL parameters in two launches.
//
// The reference walks ~400 parameter tensors in Python; for each: clip_grad_norm_(p, max_grad_norm) (a norm kernel, a host
// read-back and a scale), then five elementwise kernels (m, v, update, decay, apply).  Here the host uploads one descriptor
// table per step and two HBM-bound kernels do the rest with no host synchronisation:
//   1. adam_sqnorm_kernel : per-tensor sum of squared gradients (fp32 partials, one atomicAdd per 4096-element chunk);
//   2. adam_update_kernel : per-tensor clip factor min(1, max_norm / (||g|| + 1e-6)) (torch clip_grad_norm_ semantics),
//                           m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; u = m / (sqrt(v) + e) + wd p ; p -= lr u
//                           — no bias correction, decoupled weight decay (optimization.py:150-172).
// Parameters may be bf16 (then an fp32 master copy carries the arithmetic and the bf16 parameter is its rounding) or fp32.
// Deterministic mode: step 1 writes one partial per chunk and a third kernel adds each tensor's partials in a fixed order.
// Work decomposition: chunk c -> tensor t by binary search in an exclusive prefix of per-tensor chunk counts, so tensors of
// any size mix (a 28996x768 embedding next to 768-element biases) and the grid is sized from the SM count.
// Algorithmic HBM bytes per element: gradient read twice (2 x 2 B bf16) + master/m/v read+write (24 B) + parameter write (2 B).
#include "optim.cuh"

#include "host.cuh"

namespace vlpk {
namespace {

constexpr int ADAM_THREADS = 256;

__device__ __forceinline__ int find_tensor(const int* __restrict__ prefix, int n_tensors, int chunk) {
  int lo = 0, hi = n_tensors;  // prefix[lo] <= chunk < prefix[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (__ldg(prefix + mid) <= chunk) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ float load1(const void* p, int dtype, long long i) {
  return dtype == VLPK_BF16 ? __bfloat162float(static_cast<const __nv_bfloat16*>(p)[i]) : static_cast<const float*>(p)[i];
}

// 8 consecutive elements starting at element i (16-byte aligned address for bf16, 32-byte span for fp32)
__device__ __forceinline__ void load8(const void* p, int dtype, long long i, float (&out)[8]) {
  if (dtype == VLPK_BF16) {
    const uint4 u = *reinterpret_cast<const uint4*>(static_cast<const __nv_bfloat16*>(p) + i);
    const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 f = unpack_bf16x2(w[j]);
      out[2 * j] = f.x;
      out[2 * j + 1] = f.y;
    }
  } else {
    const float4 a = *reinterpret_cast<const float4*>(static_cast<const float*>(p) + i);
    const float4 b = *reinterpret_cast<const float4*>(static_cast<const float*>(p) + i + 4);
    out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w;
    out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
  }
}

__device__ __forceinline__ void load8_f32(const float* p, long long i, float (&out)[8]) {
  const float4 a = *reinterpret_cast<const float4*>(p + i);
  const float4 b = *reinterpret_cast<const float4*>(p + i + 4);
  out[0] = a.x; out[1] = a.y; out[2] = a.z; out[3] = a.w;
  out[4] = b.x; out[5] = b.y; out[6] = b.z; out[7] = b.w;
}

__device__ __forceinline__ void store8_f32(float* p, long long i, const float (&v)[8]) {
  *reinterpret_cast<float4*>(p + i) = make_float4(v[0], v[1], v[2], v[3]);
  *reinterpret_cast<float4*>(p + i + 4) = make_float4(v[4], v[5], v[6], v[7]);
}

__device__ __forceinline__ void store8_bf16(__nv_bfloat16* p, long long i, const float (&v)[8]) {
  *reinterpret_cast<uint4*>(p + i) =
      make_uint4(pack_bf16x2(v[0], v[1]), pack_bf16x2(v[2], v[3]), pack_bf16x2(v[4], v[5]), pack_bf16x2(v[6], v[7]));
}

__device__ __forceinline__ bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ORDERED (deterministic mode): chunk c writes its sum to sq[c] instead of adding it to sq[tensor].
template <bool ORDERED>
__global__ void __launch_bounds__(ADAM_THREADS)
adam_sqnorm_kernel(const VlpkAdamTensor* __restrict__ T, const int* __restrict__ prefix, int n_tensors, int n_chunks,
                   float* __restrict__ sq) {
  __shared__ float s_part[ADAM_THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const int t = find_tensor(prefix, n_tensors, c);
    const void* __restrict__ g = T[t].grad;
    const int gdt = T[t].grad_dtype;
    const long long n = T[t].n;
    const long long base = static_cast<long long>(c - __ldg(prefix + t)) * ADAM_CHUNK;
    const int cnt = static_cast<int>(n - base < ADAM_CHUNK ? n - base : ADAM_CHUNK);
    float acc = 0.f;
    if (aligned16(g)) {
      for (int i = threadIdx.x * 8; i < cnt; i += ADAM_THREADS * 8) {
        if (i + 8 <= cnt) {
          float v[8];
          load8(g, gdt, base + i, v);
#pragma unroll
          for (int j = 0; j < 8; ++j) acc = fmaf(v[j], v[j], acc);
        } else {
          for (int k = i; k < cnt; ++k) {
            const float x = load1(g, gdt, base + k);
            acc = fmaf(x, x, acc);
          }
        }
      }
    } else {
      for (int i = threadIdx.x; i < cnt; i += ADAM_THREADS) {
        const float x = load1(g, gdt, base + i);
        acc = fmaf(x, x, acc);
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) s_part[warp] = acc;
    __syncthreads();
    if (warp == 0) {
      float tot = lane < ADAM_THREADS / 32 ? s_part[lane] : 0.f;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
      if (lane == 0) {
        if constexpr (ORDERED) sq[c] = tot;
        else atomicAdd(sq + t, tot);
      }
    }
    __syncthreads();  // s_part is reused by the next chunk
  }
}

// sq[t] = sum of tensor t's chunk partials: one warp per tensor, lane l adds chunks l, l + 32, ... in turn, then a fixed butterfly.
__global__ void __launch_bounds__(ADAM_THREADS)
adam_sqnorm_sum_kernel(const int* __restrict__ prefix, int n_tensors, const float* __restrict__ part, float* __restrict__ sq) {
  const int t = blockIdx.x * (ADAM_THREADS / 32) + (threadIdx.x >> 5);
  if (t >= n_tensors) return;
  const int lane = threadIdx.x & 31;
  float acc = 0.f;
  for (int c = __ldg(prefix + t) + lane; c < __ldg(prefix + t + 1); c += 32) acc += part[c];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if (lane == 0) sq[t] = acc;
}

__device__ __forceinline__ void adam_elem(float g, float& m, float& v, float& p, float coef, float wd, const AdamHyper& h) {
  g *= coef;
  m = fmaf(h.omb1, g, m * h.b1);
  v = fmaf(h.omb2 * g, g, v * h.b2);
  float u = m / (sqrtf(v) + h.eps);
  if (wd > 0.f) u = fmaf(wd, p, u);
  p -= h.lr * u;
}

__global__ void __launch_bounds__(ADAM_THREADS)
adam_update_kernel(const VlpkAdamTensor* __restrict__ T, const int* __restrict__ prefix, int n_tensors, int n_chunks,
                   const float* __restrict__ sq, AdamHyper h) {
  for (int c = blockIdx.x; c < n_chunks; c += gridDim.x) {
    const int t = find_tensor(prefix, n_tensors, c);
    const VlpkAdamTensor d = T[t];
    const long long base = static_cast<long long>(c - __ldg(prefix + t)) * ADAM_CHUNK;
    const int cnt = static_cast<int>(d.n - base < ADAM_CHUNK ? d.n - base : ADAM_CHUNK);
    float coef = 1.f;
    if (h.max_grad_norm > 0.f) {  // torch.nn.utils.clip_grad_norm_ on this single tensor (optimization.py:145-146)
      const float cc = h.max_grad_norm / (sqrtf(sq[t]) + 1e-6f);
      coef = cc < 1.f ? cc : 1.f;
    }
    const bool p_bf16 = (d.param_dtype == VLPK_BF16);
    float* const w32 = p_bf16 ? d.master : static_cast<float*>(d.param);  // fp32 copy that carries the arithmetic
    __nv_bfloat16* const w16 = p_bf16 ? static_cast<__nv_bfloat16*>(d.param) : nullptr;
    const bool vec = aligned16(d.grad) && aligned16(d.param) && aligned16(d.m) && aligned16(d.v) && aligned16(w32);
    if (vec) {
      for (int i = threadIdx.x * 8; i < cnt; i += ADAM_THREADS * 8) {
        const long long e = base + i;
        if (i + 8 <= cnt) {
          float g[8], m[8], v[8], p[8];
          load8(d.grad, d.grad_dtype, e, g);
          load8_f32(d.m, e, m);
          load8_f32(d.v, e, v);
          load8_f32(w32, e, p);
#pragma unroll
          for (int j = 0; j < 8; ++j) adam_elem(g[j], m[j], v[j], p[j], coef, d.weight_decay, h);
          store8_f32(d.m, e, m);
          store8_f32(d.v, e, v);
          store8_f32(w32, e, p);
          if (w16 != nullptr) store8_bf16(w16, e, p);
        } else {
          for (int k = i; k < cnt; ++k) {
            const long long ek = base + k;
            float m = d.m[ek], v = d.v[ek], p = w32[ek];
            adam_elem(load1(d.grad, d.grad_dtype, ek), m, v, p, coef, d.weight_decay, h);
            d.m[ek] = m; d.v[ek] = v; w32[ek] = p;
            if (w16 != nullptr) w16[ek] = __float2bfloat16_rn(p);
          }
        }
      }
    } else {
      for (int i = threadIdx.x; i < cnt; i += ADAM_THREADS) {
        const long long e = base + i;
        float m = d.m[e], v = d.v[e], p = w32[e];
        adam_elem(load1(d.grad, d.grad_dtype, e), m, v, p, coef, d.weight_decay, h);
        d.m[e] = m; d.v[e] = v; w32[e] = p;
        if (w16 != nullptr) w16[e] = __float2bfloat16_rn(p);
      }
    }
  }
}

}  // namespace

int launch_bertadam(const VlpkAdamTensor* th, const VlpkAdamTensor* td, const int32_t* ph, const int32_t* pd, int n_tensors,
                    float* sqnorm_dev, const AdamHyper& h, cudaStream_t s) {
  VLPK_CHECK_ARG(n_tensors > 0 && th && td && ph && pd && sqnorm_dev, "bertadam: null table / no tensors");
  VLPK_CHECK_ARG(ph[0] == 0, "bertadam: chunk prefix must start at 0");
  double bytes = 0.0;
  for (int t = 0; t < n_tensors; ++t) {
    const VlpkAdamTensor& d = th[t];
    VLPK_CHECK_ARG(d.n > 0, "bertadam: tensor %d is empty (drop it from the table)", t);
    VLPK_CHECK_ARG(d.param && d.grad && d.m && d.v, "bertadam: tensor %d has a null pointer", t);
    VLPK_CHECK_ARG((d.param_dtype == VLPK_BF16 || d.param_dtype == VLPK_F32) && (d.grad_dtype == VLPK_BF16 || d.grad_dtype == VLPK_F32),
                   "bertadam: tensor %d: parameters and gradients must be bf16 or fp32", t);
    VLPK_CHECK_ARG(d.param_dtype == VLPK_F32 || d.master != nullptr, "bertadam: tensor %d is bf16 and needs an fp32 master copy", t);
    VLPK_CHECK_ARG(d.weight_decay >= 0.f, "bertadam: tensor %d: negative weight decay", t);
    const long long chunks = (d.n + ADAM_CHUNK - 1) / ADAM_CHUNK;
    VLPK_CHECK_ARG(static_cast<long long>(ph[t + 1]) - ph[t] == chunks, "bertadam: chunk prefix of tensor %d is %d, expected %lld", t,
                   ph[t + 1] - ph[t], chunks);
    bytes += static_cast<double>(d.n) * (2.0 * (d.grad_dtype == VLPK_BF16 ? 2 : 4) + 24.0 + (d.param_dtype == VLPK_BF16 ? 2 : 0));
  }
  const int n_chunks = ph[n_tensors];
  const int grid = n_chunks < num_sms() * 8 ? n_chunks : num_sms() * 8;
  VLPK_CUDA(cudaMemsetAsync(sqnorm_dev, 0, sizeof(float) * n_tensors, s));
  if (h.max_grad_norm > 0.f && !deterministic()) {
    LaunchScope scope(CAT_MISC, 0.0, s);
    adam_sqnorm_kernel<false><<<grid, ADAM_THREADS, 0, s>>>(td, pd, n_tensors, n_chunks, sqnorm_dev);
    VLPK_CUDA(cudaGetLastError());
  } else if (h.max_grad_norm > 0.f) {
    float* part = scratch_f32(SCRATCH_ORDERED, static_cast<size_t>(n_chunks), s);
    if (part == nullptr) return -1;
    {
      LaunchScope scope(CAT_MISC, 0.0, s);
      adam_sqnorm_kernel<true><<<grid, ADAM_THREADS, 0, s>>>(td, pd, n_tensors, n_chunks, part);
      VLPK_CUDA(cudaGetLastError());
    }
    LaunchScope scope(CAT_MISC, 0.0, s);
    adam_sqnorm_sum_kernel<<<(n_tensors + ADAM_THREADS / 32 - 1) / (ADAM_THREADS / 32), ADAM_THREADS, 0, s>>>(pd, n_tensors, part, sqnorm_dev);
    VLPK_CUDA(cudaGetLastError());
  }
  {
    LaunchScope scope(CAT_MISC, bytes, s);
    adam_update_kernel<<<grid, ADAM_THREADS, 0, s>>>(td, pd, n_tensors, n_chunks, sqnorm_dev, h);
    VLPK_CUDA(cudaGetLastError());
  }
  return 0;
}

}  // namespace vlpk
