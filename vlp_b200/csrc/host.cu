// vlp_b200 — host-side utilities (see host.cuh).
#include "host.cuh"

#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <vector>

namespace vlpk {

static thread_local char g_err[1024] = {0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
const char* get_error() { return g_err; }

// cuTensorMapEncodeTiled is a driver-API symbol.  Resolve it through the runtime so that the
// library has no link-time dependency on libcuda (the build container has no driver installed).
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn resolve_encode() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess) {
      fn = reinterpret_cast<EncodeTiledFn>(p);
    }
  });
  return fn;
}

int make_tmap(CUtensorMap* out, TmapDtype dt, int rank, const void* base, const uint64_t* dims,
              const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn fn = resolve_encode();
  VLPK_CHECK_ARG(fn != nullptr, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  VLPK_CHECK_ARG((reinterpret_cast<uintptr_t>(base) & 15u) == 0, "TMA base %p not 16-byte aligned", base);
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    estr[i] = 1;
    VLPK_CHECK_ARG(box[i] >= 1 && box[i] <= 256, "TMA box dim %d = %u out of range", i, box[i]);
  }
  for (int i = 0; i + 1 < rank; ++i) {
    gstr[i] = strides_bytes[i];
    VLPK_CHECK_ARG((strides_bytes[i] & 15u) == 0, "TMA stride %llu of dim %d not a multiple of 16 bytes",
                   (unsigned long long)strides_bytes[i], i + 1);
  }
  const CUtensorMapDataType cdt = (dt == TM_BF16) ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32;
  CUresult r = fn(out, cdt, static_cast<cuuint32_t>(rank), const_cast<void*>(base), gdim, gstr, bx, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d) rank=%d dims=[%llu,%llu,%llu] box=[%u,%u,%u]", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
              (unsigned long long)(rank > 2 ? dims[2] : 0), box[0], rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0);
    return -2;
  }
  return 0;
}

float* scratch_f32(int slot, size_t n, cudaStream_t s) {
  struct Buf {
    int dev, slot;
    float* p;
    size_t n;
  };
  static std::mutex mu;
  static std::vector<Buf> bufs;  // superseded buffers stay allocated (graphs may still reference them)
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    set_error("scratch: no CUDA device");
    return nullptr;
  }
  std::lock_guard<std::mutex> lk(mu);
  Buf* best = nullptr;
  for (auto& b : bufs)
    if (b.dev == dev && b.slot == slot && (best == nullptr || b.n > best->n)) best = &b;
  if (best != nullptr && best->n >= n) return best->p;
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(s, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
    set_error("scratch: %zu floats needed for slot %d while a CUDA graph is being captured; run the step once before capturing", n, slot);
    return nullptr;
  }
  float* p = nullptr;
  const size_t want = best != nullptr && 2 * best->n > n ? 2 * best->n : n;
  if (cudaMalloc(&p, want * sizeof(float)) != cudaSuccess) {
    set_error("scratch: cudaMalloc of %zu floats failed", want);
    return nullptr;
  }
  bufs.push_back(Buf{dev, slot, p, want});
  return p;
}

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("VLPK_PDL");
    v = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;  // no device visible (host-only planning): an H100 SXM
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  }
  return n;
}

// SMs the persistent GEMM grids may occupy.  A data-parallel caller can reserve some for a concurrently running collective
// (vlpk_set_reserved_sms): a persistent grid sized for all SMs would otherwise leave its last CTAs waiting behind the
// collective's CTAs and finish a full tile-loop late.
static int g_reserved_sms = 0;
void set_reserved_sms(int n) { g_reserved_sms = n > 0 ? n : 0; }
int gemm_sms() {
  const int n = num_sms() - g_reserved_sms;
  return n < 1 ? 1 : n;
}

static bool g_deterministic = false;
bool deterministic() { return g_deterministic; }
void set_deterministic(bool on) { g_deterministic = on; }

// ------------------------------------------------------------------------------------------------
// launch accounting / profiling
// ------------------------------------------------------------------------------------------------
struct ProfRec {
  int cat;
  double work;
  cudaEvent_t e0, e1;
};
static std::mutex g_prof_mu;
static bool g_prof_on = false;
static std::vector<ProfRec> g_recs;
static std::vector<cudaEvent_t> g_event_pool;
static std::atomic<long long> g_launches{0};

void prof_enable(bool on) { g_prof_on = on; }
long long launch_count() { return g_launches.load(); }

void prof_reset() {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  for (auto& r : g_recs) {
    g_event_pool.push_back(r.e0);
    g_event_pool.push_back(r.e1);
  }
  g_recs.clear();
}

static cudaEvent_t get_event() {
  if (!g_event_pool.empty()) {
    cudaEvent_t e = g_event_pool.back();
    g_event_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}

LaunchScope::LaunchScope(int cat, double work, cudaStream_t s) : idx_(-1), s_(s) {
  g_launches.fetch_add(1);
  if (!g_prof_on) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  ProfRec r;
  r.cat = cat;
  r.work = work;
  r.e0 = get_event();
  r.e1 = get_event();
  cudaEventRecord(r.e0, s);
  idx_ = static_cast<int>(g_recs.size());
  g_recs.push_back(r);
}
LaunchScope::~LaunchScope() {
  if (idx_ < 0) return;
  std::lock_guard<std::mutex> lk(g_prof_mu);
  cudaEventRecord(g_recs[idx_].e1, s_);
}

int prof_get(int cat, double* ms, double* work, long long* launches) {
  std::lock_guard<std::mutex> lk(g_prof_mu);
  double tms = 0, tw = 0;
  long long n = 0;
  for (auto& r : g_recs) {
    if (r.cat != cat) continue;
    VLPK_CUDA(cudaEventSynchronize(r.e1));
    float f = 0.f;
    VLPK_CUDA(cudaEventElapsedTime(&f, r.e0, r.e1));
    tms += f;
    tw += r.work;
    ++n;
  }
  *ms = tms;
  *work = tw;
  *launches = n;
  return 0;
}

}  // namespace vlpk
