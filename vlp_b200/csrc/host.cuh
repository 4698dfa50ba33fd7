// vlp_b200 — host-side utilities: error channel, TMA descriptor encode, device properties.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <utility>

namespace vlpk {

// Thread-local last-error text surfaced through vlpk_last_error() (include/vlpk.h).
void set_error(const char* fmt, ...);
const char* get_error();

#define VLPK_CHECK_ARG(cond, ...)          \
  do {                                     \
    if (!(cond)) {                         \
      ::vlpk::set_error(__VA_ARGS__);      \
      return -1;                           \
    }                                      \
  } while (0)

#define VLPK_CUDA(expr)                                                                        \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess) {                                                                   \
      ::vlpk::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return static_cast<int>(_e);                                                             \
    }                                                                                          \
  } while (0)

#define VLPK_TRY(expr)        \
  do {                        \
    int _rc = (expr);         \
    if (_rc != 0) return _rc; \
  } while (0)

enum TmapDtype { TM_BF16 = 0, TM_F32 = 1 };

// Encode a tiled tensor map with 128-byte swizzle over a row-major tensor of `rank` dims.
// dims[0] is the contiguous dimension.  strides_bytes[i] is the byte stride of dims[i+1].
// Out-of-bounds box elements are zero-filled on load and clipped on store.
int make_tmap(CUtensorMap* out, TmapDtype dt, int rank, const void* base, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box);

inline int make_tmap_2d(CUtensorMap* out, TmapDtype dt, const void* base, uint64_t inner, uint64_t outer,
                        uint64_t ld_elems, uint32_t box_inner, uint32_t box_outer) {
  const uint64_t es = (dt == TM_BF16) ? 2 : 4;
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {ld_elems * es};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap(out, dt, 2, base, dims, strides, box);
}

// Library-owned fp32 device scratch for the ordered reductions, one buffer per slot and device.  Grow-only, and a buffer is
// never freed, so CUDA graphs captured earlier keep valid pointers; growing is refused (nullptr, error set) while `s` is being
// captured — the first call of a shape must run outside capture, as a graph's warm-up does.
enum ScratchSlot { SCRATCH_ATTN_DBIAS = 0, SCRATCH_SPLITK = 1, SCRATCH_SLOTS = 2 };
float* scratch_f32(int slot, size_t n, cudaStream_t s);

int num_sms();
// SMs available to the persistent GEMM grids: num_sms() minus what vlpk_set_reserved_sms put aside (default 0), at least 1.
int gemm_sms();
void set_reserved_sms(int n);

// Launch with optional cluster dimension and programmatic dependent launch (VLPK_PDL=0 disables the latter).
bool pdl_enabled();
template <typename... KArgs, typename... Args>
inline cudaError_t launch_ex(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, int cluster_x, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster_x > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster_x;
    attr[n].val.clusterDim.y = 1;
    attr[n].val.clusterDim.z = 1;
    ++n;
  }
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

// ---- launch accounting + optional per-kernel-family timing (CUDA events on the launch stream) ----
enum KernelCat { CAT_GEMM_FWD = 0, CAT_GEMM_DGRAD, CAT_GEMM_WGRAD, CAT_ATTN_FWD, CAT_ATTN_BWD, CAT_LN_FWD, CAT_LN_BWD, CAT_EMBED,
                 CAT_MISC, CAT_COUNT };
void prof_enable(bool on);
void prof_reset();
// Sums over all launches recorded since the last reset (synchronises the recorded events).
int prof_get(int cat, double* ms, double* work, long long* launches);
long long launch_count();
// RAII: counts one kernel launch; when profiling is enabled brackets it with events.  `work` = algorithmic FLOPs
// (tensor-bound kernels) or algorithmic HBM bytes (bandwidth-bound kernels) of this launch.
struct LaunchScope {
  LaunchScope(int cat, double work, cudaStream_t s);
  ~LaunchScope();
  int idx_;
  cudaStream_t s_;
};

}  // namespace vlpk
