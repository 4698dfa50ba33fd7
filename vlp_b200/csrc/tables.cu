// vlp_b200 — scatter of BertEmbeddings' pre-LayerNorm gradient into the word / position / token-type tables
// (autograd backward of the three nn.Embedding lookups, modeling.py:217-241).
//
// In the round-1 profile this glue, done with torch ops, cost ~215 us of a 7.2 ms step: a dense fp32 zero-fill of the
// [28996,768] word table (89 MB), its conversion to bf16, and an index_add of all B*L rows into the 6-row token-type table
// (7 872 x 768 atomics onto 6 x 768 addresses).  Only B x 23 rows of the word / position tables are ever looked up
// (the 100 region rows are spliced in from the projections), so:
//   word : memset the bf16 gradient (44 MB), then three tiny launches over the looked-up rows only — zero their fp32
//          scratch rows, atomically accumulate (duplicates such as [CLS]/[SEP] collide here, in fp32), convert to bf16;
//   pos  : fp32 atomics from the same rows;
//   type : a segmented column sum — each thread keeps one accumulator per token type (<= 8) — one atomic per
//          (type, column, 256-row slab) instead of one per element.
// Deterministic mode (vlpk_set_deterministic) replaces every atomic: the (id, row) and (position, row) pairs are stable-sorted by
// key on the device (CUB radix sort), one warp per run of equal keys sums the run's rows in row order and writes the table row once;
// the token-type sums write one partial per slab, which are then added in slab order.
#include "tables.cuh"

#include <cub/device/device_radix_sort.cuh>

#include "host.cuh"
#include "rowops.cuh"

namespace vlpk {
namespace {

constexpr int TT_MAX = 8;
constexpr int SLAB = 256;

__device__ __forceinline__ void ld8(const __nv_bfloat16* p, float (&v)[8]) {
  const uint4 u = *reinterpret_cast<const uint4*>(p);
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 f = unpack_bf16x2(w[j]);
    v[2 * j] = f.x;
    v[2 * j + 1] = f.y;
  }
}

// entry e -> (sample, position) of the e-th row that reads the word / position tables
__device__ __forceinline__ long long table_row(const TableGradArgs& a, long long e) {
  const int n_tab = a.vis_input ? a.L - a.R : a.L;
  const long long b = e / n_tab;
  const int k = static_cast<int>(e % n_tab);
  const int l = a.vis_input ? (k == 0 ? 0 : a.R + k) : k;
  return b * a.L + l;
}

// PHASE 0: zero the scratch rows; 1: accumulate; 2: scratch -> bf16.  One warp per looked-up row.
template <int PHASE>
__global__ void __launch_bounds__(256) word_pos_kernel(TableGradArgs a, long long n_entries) {
  const long long e = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (e >= n_entries) return;
  const int lane = threadIdx.x & 31;
  const long long row = table_row(a, e);
  const long long id = a.ids[row];
  const bool id_ok = (id >= 0 && id < a.V);
  long long p = (a.pos != nullptr) ? a.pos[row] : (row % a.L);
  const bool p_ok = (p >= 0 && p < a.P);
  for (int c = lane * 8; c < a.H; c += 256) {
    if (PHASE == 0) {
      if (id_ok) {
        float* d = a.scratch + id * a.H + c;
        *reinterpret_cast<float4*>(d) = make_float4(0.f, 0.f, 0.f, 0.f);
        *reinterpret_cast<float4*>(d + 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    } else if (PHASE == 1) {
      float v[8];
      ld8(a.dz + row * a.H + c, v);
      if (id_ok) {
#pragma unroll
        for (int j = 0; j < 8; ++j) atomicAdd(a.scratch + id * a.H + c + j, v[j]);
      }
      if (p_ok) {
#pragma unroll
        for (int j = 0; j < 8; ++j) atomicAdd(a.d_pos + p * a.H + c + j, v[j]);
      }
    } else {
      if (id_ok) {
        const float* sp = a.scratch + id * a.H + c;
        const float4 x = *reinterpret_cast<const float4*>(sp), y = *reinterpret_cast<const float4*>(sp + 4);
        *reinterpret_cast<uint4*>(a.d_word + id * a.H + c) =
            make_uint4(pack_bf16x2(x.x, x.y), pack_bf16x2(x.z, x.w), pack_bf16x2(y.x, y.y), pack_bf16x2(y.z, y.w));
      }
    }
  }
}

// d_type[t, :] += sum over the rows of this 256-row slab whose token type is t.  Block: 8 column groups x 32 row lanes.
// ORDERED (deterministic mode): the sums go to part[(slab * T + t) * H + c] instead.
template <bool ORDERED>
__global__ void __launch_bounds__(256) type_grad_kernel(TableGradArgs a, float* __restrict__ part) {
  __shared__ float s_part[32][65];
  const int cgp = threadIdx.x & 7, rl = threadIdx.x >> 3;
  const int col = blockIdx.x * 64 + cgp * 8;
  const long long M = static_cast<long long>(a.B) * a.L;
  const long long r0 = static_cast<long long>(blockIdx.y) * SLAB;
  float acc[TT_MAX][8];
#pragma unroll
  for (int t = 0; t < TT_MAX; ++t)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[t][j] = 0.f;
  if (col < a.H) {
#pragma unroll
    for (int i = 0; i < SLAB / 32; ++i) {
      const long long r = r0 + rl + 32 * i;
      if (r < M) {
        float v[8];
        ld8(a.dz + r * a.H + col, v);
        const int ty = (a.tt != nullptr) ? static_cast<int>(a.tt[r]) : 0;
#pragma unroll
        for (int t = 0; t < TT_MAX; ++t) {
          const float sel = (ty == t) ? 1.f : 0.f;
#pragma unroll
          for (int j = 0; j < 8; ++j) acc[t][j] = fmaf(sel, v[j], acc[t][j]);
        }
      }
    }
  }
#pragma unroll
  for (int t = 0; t < TT_MAX; ++t) {
    if (t < a.T) {  // uniform across the block
#pragma unroll
      for (int j = 0; j < 8; ++j) s_part[rl][cgp * 8 + j] = acc[t][j];
      __syncthreads();
      if (threadIdx.x < 64) {
        float tot = 0.f;
#pragma unroll
        for (int i = 0; i < 32; ++i) tot += s_part[i][threadIdx.x];
        const int c = blockIdx.x * 64 + threadIdx.x;
        if constexpr (ORDERED) {
          if (c < a.H) part[(static_cast<long long>(blockIdx.y) * a.T + t) * a.H + c] = tot;
        } else {
          if (c < a.H && tot != 0.f) atomicAdd(a.d_type + static_cast<long long>(t) * a.H + c, tot);
        }
      }
      __syncthreads();
    }
  }
}

// ---- deterministic mode: sorted segmented scatter ----------------------------------------------------------------------------
// Sort inputs: word key, position key and source row of every entry.  Keys outside the table become V resp. P and sort last.
__global__ void __launch_bounds__(256) table_keys_kernel(TableGradArgs a, long long n, int* __restrict__ wk, int* __restrict__ pk,
                                                           int* __restrict__ rows) {
  const long long e = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const long long row = table_row(a, e);
  const long long id = a.ids[row];
  const long long p = (a.pos != nullptr) ? a.pos[row] : (row % a.L);
  wk[e] = (id >= 0 && id < a.V) ? static_cast<int>(id) : a.V;
  pk[e] = (p >= 0 && p < a.P) ? static_cast<int>(p) : a.P;
  rows[e] = static_cast<int>(row);
}

enum { RUN_WORD_STORE = 0, RUN_F32_ADD = 2 };

// One warp per sorted position that starts a run of equal keys: sums src[row] over the run in sorted order (= ascending
// row order: the sort is stable and its input was in row order) and updates table row `key` once.
//   RUN_WORD_STORE: bf16 dst[key] = sum        RUN_F32_ADD: fp32 dst[key] += each row in turn
template <int MODE>
__global__ void __launch_bounds__(256) sorted_run_sum_kernel(const int* __restrict__ keys, const int* __restrict__ rows, long long n, int n_keys,
                                                               const __nv_bfloat16* __restrict__ src, int H, void* dst) {
  const long long i = static_cast<long long>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (i >= n) return;
  const int key = keys[i];
  if (key >= n_keys || (i > 0 && keys[i - 1] == key)) return;
  const int lane = threadIdx.x & 31;
  for (int c = lane * 8; c < H; c += 256) {
    float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    float* d32 = static_cast<float*>(dst) + static_cast<long long>(key) * H + c;
    if (MODE == RUN_F32_ADD) {
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] = d32[j];
    }
    for (long long r = i; r < n && keys[r] == key; ++r) {
      float v[8];
      ld8(src + static_cast<long long>(rows[r]) * H + c, v);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += v[j];
    }
    if (MODE == RUN_F32_ADD) {
#pragma unroll
      for (int j = 0; j < 8; ++j) d32[j] = acc[j];
    } else {
      __nv_bfloat16* d16 = static_cast<__nv_bfloat16*>(dst) + static_cast<long long>(key) * H + c;
      *reinterpret_cast<uint4*>(d16) =
          make_uint4(pack_bf16x2(acc[0], acc[1]), pack_bf16x2(acc[2], acc[3]), pack_bf16x2(acc[4], acc[5]), pack_bf16x2(acc[6], acc[7]));
    }
  }
}

inline int key_bits(int n_keys) {  // radix-sort bits for keys in [0, n_keys]
  int b = 1;
  while (b < 31 && (1LL << b) <= n_keys) ++b;
  return b;
}

// The sort buffers of n entries in scratch slot SCRATCH_SORT: word / position keys and rows, their sorted copies, CUB temporaries.
struct SortBufs {
  int *wk, *pk, *rows, *wk_s, *wrow_s, *pk_s, *prow_s;
  void* temp;
  size_t temp_bytes;
};

int sort_bufs(long long n, int V, int P, cudaStream_t s, SortBufs* b) {
  VLPK_CHECK_ARG(n < (1LL << 30), "table scatter: %lld entries exceed the deterministic sort's int32 indices", n);
  size_t tw = 0, tp = 0;
  VLPK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tw, static_cast<const int*>(nullptr), static_cast<int*>(nullptr),
                                            static_cast<const int*>(nullptr), static_cast<int*>(nullptr), static_cast<int>(n), 0, key_bits(V), s));
  VLPK_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, tp, static_cast<const int*>(nullptr), static_cast<int*>(nullptr),
                                            static_cast<const int*>(nullptr), static_cast<int*>(nullptr), static_cast<int>(n), 0, key_bits(P), s));
  b->temp_bytes = tw > tp ? tw : tp;
  const size_t na = (static_cast<size_t>(n) + 63) / 64 * 64;  // 256-byte aligned arrays
  float* base = scratch_f32(SCRATCH_SORT, 7 * na + (b->temp_bytes + 3) / 4, s);
  if (base == nullptr) return -1;
  int* p = reinterpret_cast<int*>(base);
  int** arr[7] = {&b->wk, &b->pk, &b->rows, &b->wk_s, &b->wrow_s, &b->pk_s, &b->prow_s};
  for (int k = 0; k < 7; ++k) *arr[k] = p + k * na;
  b->temp = p + 7 * na;
  return 0;
}

// Sort by word key and by position key and apply the runs.
int sorted_scatter(const SortBufs& b, long long n, int H, int V, int P, const __nv_bfloat16* src, __nv_bfloat16* d_word, float* d_pos,
                   cudaStream_t s) {
  size_t tb = b.temp_bytes;
  VLPK_CUDA(cub::DeviceRadixSort::SortPairs(b.temp, tb, b.wk, b.wk_s, b.rows, b.wrow_s, static_cast<int>(n), 0, key_bits(V), s));
  const unsigned grid = static_cast<unsigned>((n + 7) / 8);
  {
    LaunchScope scope(CAT_EMBED, 0.0, s);
    sorted_run_sum_kernel<RUN_WORD_STORE><<<grid, 256, 0, s>>>(b.wk_s, b.wrow_s, n, V, src, H, d_word);
    VLPK_CUDA(cudaGetLastError());
  }
  tb = b.temp_bytes;
  VLPK_CUDA(cub::DeviceRadixSort::SortPairs(b.temp, tb, b.pk, b.pk_s, b.rows, b.prow_s, static_cast<int>(n), 0, key_bits(P), s));
  LaunchScope scope(CAT_EMBED, 0.0, s);
  sorted_run_sum_kernel<RUN_F32_ADD><<<grid, 256, 0, s>>>(b.pk_s, b.prow_s, n, P, src, H, d_pos);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

int launch_embed_tables_bwd(const TableGradArgs& a, cudaStream_t s) {
  VLPK_CHECK_ARG(a.B > 0 && a.L > 0 && a.H > 0 && a.H % 8 == 0, "embed_tables_bwd: B=%d L=%d H=%d (H must be a multiple of 8)", a.B, a.L, a.H);
  VLPK_CHECK_ARG(a.V > 0 && a.P > 0 && a.T > 0 && a.T <= TT_MAX, "embed_tables_bwd: V=%d P=%d T=%d (at most %d token types)", a.V, a.P, a.T, TT_MAX);
  VLPK_CHECK_ARG(!a.vis_input || (a.R > 0 && a.R < a.L), "embed_tables_bwd: R=%d regions do not fit L=%d", a.R, a.L);
  VLPK_CHECK_ARG(a.ids && a.dz && a.d_type && a.d_word && a.scratch && a.d_pos, "embed_tables_bwd: null pointer");
  VLPK_CHECK_ARG(((reinterpret_cast<uintptr_t>(a.dz) | reinterpret_cast<uintptr_t>(a.d_word) | reinterpret_cast<uintptr_t>(a.scratch)) & 15u) == 0,
                 "embed_tables_bwd: dz / d_word / scratch must be 16-byte aligned");
  const long long M = static_cast<long long>(a.B) * a.L;
  const long long n_entries = static_cast<long long>(a.B) * (a.vis_input ? a.L - a.R : a.L);
  const unsigned grid = static_cast<unsigned>((n_entries + 7) / 8);
  VLPK_CUDA(cudaMemsetAsync(a.d_word, 0, static_cast<size_t>(a.V) * a.H * 2, s));
  if (deterministic()) {
    SortBufs b;
    VLPK_TRY(sort_bufs(n_entries, a.V, a.P, s, &b));
    {
      LaunchScope scope(CAT_EMBED, 0.0, s);
      table_keys_kernel<<<static_cast<unsigned>((n_entries + 255) / 256), 256, 0, s>>>(a, n_entries, b.wk, b.pk, b.rows);
      VLPK_CUDA(cudaGetLastError());
    }
    VLPK_TRY(sorted_scatter(b, n_entries, a.H, a.V, a.P, a.dz, a.d_word, a.d_pos, s));
    const unsigned slabs = static_cast<unsigned>((M + SLAB - 1) / SLAB);
    float* part = scratch_f32(SCRATCH_ORDERED, static_cast<size_t>(slabs) * a.T * a.H, s);
    if (part == nullptr) return -1;
    {
      LaunchScope scope(CAT_EMBED, 2.0 * M * a.H, s);
      type_grad_kernel<true><<<dim3((a.H + 63) / 64, slabs), 256, 0, s>>>(a, part);
      VLPK_CUDA(cudaGetLastError());
    }
    return launch_sum_parts(part, static_cast<int>(slabs), static_cast<long long>(a.T) * a.H, a.d_type, s);
  }
  {
    LaunchScope scope(CAT_EMBED, 0.0, s);
    word_pos_kernel<0><<<grid, 256, 0, s>>>(a, n_entries);
    VLPK_CUDA(cudaGetLastError());
  }
  {
    LaunchScope scope(CAT_EMBED, 0.0, s);
    word_pos_kernel<1><<<grid, 256, 0, s>>>(a, n_entries);
    VLPK_CUDA(cudaGetLastError());
  }
  {
    LaunchScope scope(CAT_EMBED, 2.0 * a.V * a.H, s);
    word_pos_kernel<2><<<grid, 256, 0, s>>>(a, n_entries);
    VLPK_CUDA(cudaGetLastError());
  }
  LaunchScope scope(CAT_EMBED, 2.0 * M * a.H, s);
  type_grad_kernel<false><<<dim3((a.H + 63) / 64, static_cast<unsigned>((M + SLAB - 1) / SLAB)), 256, 0, s>>>(a, nullptr);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace vlpk
