// vlp_b200 — duplicate-n-gram blocking for beam search (the reference's forbid_duplicate_ngrams, modeling.py:1375-1428, and its
// get_dup_ngram_candidates, :1391-1406), on the device so that a blocked decode needs no host synchronisation and can be captured
// in a CUDA graph.
//
// One launch per beam frame f >= 1, one CTA per hypothesis row i = b*K + k:
//   history  hist_out[i, :f-1] = hist_in[b*K + ptr[i], :f-1],  hist_out[i, f-1] = wid[i]        (the reference's partial_seqs)
//   blocking (f >= n) seq = hist_out[i, :f], tail = seq[-(n-1):] (the whole of seq when n = 1, as in the reference);
//            no candidates if a tail word is ignored, else w = seq[s+n-1] for every s <= f-n with seq[s:s+n-1] == tail, unless w
//            is ignored; logp[i, w] += -10000 once per distinct candidate.
// The history row lives in shared memory, so its length is bounded by shared memory and not by the CTA's threads.  Candidates are
// collected in a V-bit shared bitmap (integer atomicOr: the set does not depend on scheduling) and each set bit is applied by one
// thread with one fp32 add, so every (row, word) is written at most once and the result is bitwise reproducible.  Word ids outside
// [0, V) never become candidates; a back pointer outside [0, K) gives a history of -1 words (never a candidate, never matching a
// real tail).
#include "decode.cuh"

#include <climits>

#include "host.cuh"

namespace vlpk {
namespace {

constexpr int NGRAM_THREADS = 256;
constexpr size_t NGRAM_SMEM_MAX = 48 * 1024;

__device__ __forceinline__ bool is_ignored(int w, const int* ignore, int n_ignore) {
  for (int j = 0; j < n_ignore; ++j)
    if (__ldg(ignore + j) == w) return true;
  return false;
}

// The candidates of history seq[0:f], f >= n, as set bits of `bits` ([ceil(V/32)] words, cleared here).  seq must be complete in
// shared memory before the call (the first barrier here orders it).  Returns, uniformly across the CTA, whether any bit was set.
__device__ bool ngram_candidates(const int* seq, int f, int n, int V, const int* ignore, int n_ignore, unsigned* bits) {
  const int tid = threadIdx.x;
  const int nwords = (V + 31) >> 5;
  for (int j = tid; j < nwords; j += blockDim.x) bits[j] = 0u;
  __syncthreads();

  const int m = n - 1;                                             // words matched before a candidate
  const int t0 = f - m;                                            // start of the tail
  if (n_ignore > 0) {
    int hit = 0;
    for (int t = (m == 0 ? 0 : t0) + tid; t < f; t += blockDim.x) hit |= is_ignored(seq[t], ignore, n_ignore);
    if (__syncthreads_or(hit)) return false;
  }
  int found = 0;
  for (int s = tid; s < t0; s += blockDim.x) {                     // s <= f - n
    bool match = true;
    for (int j = 0; j < m && match; ++j) match = seq[s + j] == seq[t0 + j];
    if (!match) continue;
    const int w = seq[s + m];
    if (w < 0 || w >= V) continue;
    if (n_ignore > 0 && is_ignored(w, ignore, n_ignore)) continue;
    atomicOr(bits + (w >> 5), 1u << (w & 31));
    found = 1;
  }
  return __syncthreads_or(found) != 0;
}

__global__ void __launch_bounds__(NGRAM_THREADS) beam_ngram_block_kernel(NgramBlockArgs a) {
  extern __shared__ int smem[];
  int* seq = smem;                                                 // [T_cap] this row's history
  unsigned* bits = reinterpret_cast<unsigned*>(smem + a.T_cap);   // [ceil(V/32)] candidate words
  const int i = blockIdx.x;
  const int f = a.f;
  const int tid = threadIdx.x;

  // history of frame f: the parent's f-1 words, then this frame's word
  const long long p = f > 1 ? a.ptr[i] : 0;
  const bool parent_ok = p >= 0 && p < a.K;
  const int* src = a.hist_in + (static_cast<size_t>(i / a.K) * a.K + (parent_ok ? p : 0)) * a.T_cap;
  int* dst = a.hist_out + static_cast<size_t>(i) * a.T_cap;
  for (int t = tid; t < f - 1; t += blockDim.x) {
    const int w = parent_ok ? src[t] : -1;
    seq[t] = w;
    dst[t] = w;
  }
  if (tid == 0) {
    const long long w64 = a.wid[i];
    const int w = (w64 >= INT_MIN && w64 <= INT_MAX) ? static_cast<int>(w64) : -1;
    seq[f - 1] = w;
    dst[f - 1] = w;
  }
  if (f < a.n) return;                                             // uniform: too short for an n-gram

  if (!ngram_candidates(seq, f, a.n, a.V, a.ignore, a.n_ignore, bits)) return;      // no candidate: the row is not touched

  float* row = a.logp + static_cast<size_t>(i) * a.ld;
  const int nwords = (a.V + 31) >> 5;
  for (int j = tid; j < nwords; j += blockDim.x) {
    unsigned w = bits[j];
    while (w) {
      const int b = __ffs(w) - 1;
      w &= w - 1;
      row[j * 32 + b] += -10000.0f;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Top-k / top-p sampling of one decode frame f, one CTA of SAMPLE_THREADS per row:
//   x[v]   = logits[row, v] + bias[v], rounded to the logits' dtype (bit for bit the head's `decoder(h) + bias`), plus -10000 at
//            the words the duplicate-n-gram rule above blocks for history seq[row, :f] (n > 0, f >= n), and x[eos] = -10000 while
//            block_eos is set (beam search's order and values); e[v] = exp(x[v] - max x), Z = sum e.
//   order  words ranked by (x descending, index ascending).  top-k keeps the first k; top-p keeps the shortest prefix whose e
//            sum reaches topp * Z (always at least the first argmax, so topp -> 0 is greedy).  The cut is found as a threshold on
//            an order-preserving 32-bit key (x for top-k, e for top-p) by binary search over the key's bits — no sort — and words
//            tied at the threshold are taken lowest index first, as many as needed.
//   draw   u = Philox(seed; frame f, row) in [0, 1); the chosen word is the first kept word, in index order, whose running e sum
//          exceeds u * (kept e sum).  seq[row, f] = word, score[row, f] = log(e[word] / Z).
// Each thread owns one contiguous chunk of the row in shared memory and every sum is taken in a fixed order (chunk, then a
// fixed shuffle tree), so the result depends on (seed, f, row, logits) only: not on the batch, the grid or the run.
// Finished rows write pad_id and score 0; a row that draws eos_id is marked finished and decrements *live.
using bf16 = __nv_bfloat16;
constexpr int SAMPLE_THREADS = 1024;                               // 32 warps: the block reductions below rely on it
constexpr size_t SAMPLE_SMEM_MAX = 200 * 1024;

__device__ __forceinline__ float head_logit(const bf16* l, const bf16* b, int v) {
  const float x = __bfloat162float(l[v]);
  return b ? __bfloat162float(__float2bfloat16_rn(x + __bfloat162float(b[v]))) : x;
}
__device__ __forceinline__ float head_logit(const float* l, const float* b, int v) { return b ? l[v] + b[v] : l[v]; }

__device__ __forceinline__ unsigned order_key(float x) {           // unsigned order == float order
  const unsigned u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Every thread gets op over the CTA's values; warp shuffle trees in a fixed order.  red: [33] shared.
template <typename T, typename Op>
__device__ __forceinline__ T block_reduce(T v, T* red, Op op) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_down_sync(0xffffffffu, v, o));
  __syncthreads();                                                  // red may still be read by the previous reduction
  if (lane == 0) red[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = red[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_down_sync(0xffffffffu, v, o));
    if (lane == 0) red[32] = v;
  }
  __syncthreads();
  return red[32];
}

// pre[t] = sum of the values of threads < t, pre[SAMPLE_THREADS] = total.  red: [33] shared, pre: [SAMPLE_THREADS + 1] shared.
template <typename T>
__device__ __forceinline__ void block_exclusive_scan(T v, T* red, T* pre) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  T x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  __syncthreads();
  if (lane == 31) red[warp] = x;
  __syncthreads();
  if (warp == 0) {
    T w = red[lane];
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T y = __shfl_up_sync(0xffffffffu, w, o);
      if (lane >= o) w += y;
    }
    const T before = __shfl_up_sync(0xffffffffu, w, 1);
    red[lane] = lane == 0 ? T(0) : before;                         // warps before this one
    if (lane == 31) pre[SAMPLE_THREADS] = w;
  }
  __syncthreads();
  const T in_warp = __shfl_up_sync(0xffffffffu, x, 1);
  pre[threadIdx.x] = red[warp] + (lane == 0 ? T(0) : in_warp);
  __syncthreads();
}

template <typename T>
__global__ void __launch_bounds__(SAMPLE_THREADS) sample_kernel(SampleArgs a) {
  extern __shared__ float sample_smem[];
  __shared__ float redf[33], pref[SAMPLE_THREADS + 1];
  __shared__ int redi[33], prei[SAMPLE_THREADS + 1];
  const int V = a.V, tid = threadIdx.x, row = blockIdx.x;
  const int nwords = (V + 31) >> 5;
  float* val = sample_smem;                                          // [V] x (top-k) or e (top-p)
  unsigned* bits = reinterpret_cast<unsigned*>(val + V);             // [nwords] blocked words
  int* hist = reinterpret_cast<int*>(bits + nwords);                 // [T_cap] history
  long long* out = a.seq + static_cast<size_t>(row) * a.T_cap;
  if (a.finished[row]) {                                             // uniform
    if (tid == 0) {
      out[a.f] = a.pad_id;
      if (a.score) a.score[static_cast<size_t>(row) * a.T_cap + a.f] = 0.f;
    }
    return;
  }

  bool blocked = false;
  if (a.n > 0 && a.f >= a.n) {
    for (int t = tid; t < a.f; t += SAMPLE_THREADS) {
      const long long w = out[t];
      hist[t] = (w >= INT_MIN && w <= INT_MAX) ? static_cast<int>(w) : -1;
    }
    blocked = ngram_candidates(hist, a.f, a.n, V, a.ignore, a.n_ignore, bits);
  }

  // x, coalesced, and its maximum (order-free)
  const T* lrow = static_cast<const T*>(a.logits) + static_cast<size_t>(row) * a.ld;
  const T* bias = static_cast<const T*>(a.bias);
  float mx = -INFINITY;
  for (int v = tid; v < V; v += SAMPLE_THREADS) {
    float x = head_logit(lrow, bias, v);
    if (blocked && ((bits[v >> 5] >> (v & 31)) & 1u)) x += -10000.0f;
    if (a.block_eos && v == a.eos_id) x = -10000.0f;
    val[v] = x;
    mx = fmaxf(mx, x);
  }
  mx = block_reduce(mx, redf, [](float p, float q) { return fmaxf(p, q); });

  // from here on thread t owns words [lo, hi); an odd chunk length keeps the threads' strided reads in distinct banks
  const int C = ((V + SAMPLE_THREADS - 1) / SAMPLE_THREADS) | 1;
  const int lo = min(tid * C, V), hi = min(lo + C, V);
  const bool topp = a.mode == SAMPLE_TOPP;
  float z = 0.f;
  for (int v = lo; v < hi; ++v) {
    const float e = expf(val[v] - mx);
    z += e;
    if (topp) val[v] = e;
  }
  const float Z = block_reduce(z, redf, [](float p, float q) { return p + q; });

  auto key = [&](int v) { return topp ? __float_as_uint(val[v]) : order_key(val[v]); };
  auto weight = [&](int v) { return topp ? val[v] : expf(val[v] - mx); };
  // mass(t): sum of the selection weights (1 for top-k, e for top-p) of the words whose key is >= t.  mass(0) sums in Z's order.
  auto mass = [&](unsigned t) {
    float s = 0.f;
    for (int v = lo; v < hi; ++v) s += key(v) >= t ? (topp ? val[v] : 1.f) : 0.f;
    return block_reduce(s, redf, [](float p, float q) { return p + q; });
  };
  const float target = topp ? a.topp * Z : static_cast<float>(min(a.topk, V));
  // tau = the largest key with mass(tau) >= target; mass(0) >= target always holds
  unsigned klo = 0, khi = topp ? __float_as_uint(1.0f) : order_key(mx);
  if (mass(khi) >= target) {
    klo = khi;
  } else {
    khi -= 1;
    while (klo < khi) {                                              // uniform: every thread sees the same masses
      const unsigned mid = klo + (khi - klo + 1) / 2;
      if (mass(mid) >= target) klo = mid; else khi = mid - 1;
    }
  }
  const unsigned tau = klo;
  const float above = tau == 0xffffffffu ? 0.f : mass(tau + 1);
  int take;                                                           // words tied at tau to keep, lowest index first
  if (!topp) {
    take = static_cast<int>(target - above);
  } else {
    const float w_tie = __uint_as_float(tau);
    take = w_tie > 0.f ? static_cast<int>(fminf(ceilf((target - above) / w_tie), static_cast<float>(V))) : V;
  }
  take = max(take, 1);

  // ties before this chunk, then the kept weight of this chunk
  int ties = 0;
  for (int v = lo; v < hi; ++v) ties += key(v) == tau;
  block_exclusive_scan(ties, redi, prei);
  int rank = prei[tid];
  float kept = 0.f;
  for (int v = lo; v < hi; ++v) {
    const unsigned k = key(v);
    if (k > tau || (k == tau && rank++ < take)) kept += weight(v);
  }
  block_exclusive_scan(kept, redf, pref);

  const uint4 r = Philox::gen(a.seed, static_cast<unsigned long long>(a.f), static_cast<unsigned long long>(row));
  const float u = static_cast<float>(r.x >> 8) * (1.0f / 16777216.0f);
  const float goal = u * pref[SAMPLE_THREADS];
  int found = INT_MAX;
  if (pref[tid] <= goal && goal < pref[tid + 1]) {                  // this chunk holds the draw: walk it
    float acc = pref[tid];
    rank = prei[tid];
    for (int v = lo; v < hi; ++v) {
      const unsigned k = key(v);
      if (!(k > tau || (k == tau && rank++ < take))) continue;
      found = v;                                                     // the last kept word, should rounding leave goal above acc
      acc += weight(v);
      if (goal < acc) break;
    }
  }
  int pick = block_reduce(found, redi, [](int p, int q) { return min(p, q); });
  if (pick == INT_MAX) {                                              // goal fell outside every chunk (rounding): first argmax
    int first = INT_MAX;
    for (int v = lo; v < hi && first == INT_MAX; ++v) if (val[v] == (topp ? 1.0f : mx)) first = v;
    pick = block_reduce(first, redi, [](int p, int q) { return min(p, q); });
  }
  if (tid == 0) {
    out[a.f] = pick;
    if (a.score) a.score[static_cast<size_t>(row) * a.T_cap + a.f] = logf(topp ? val[pick] : expf(val[pick] - mx)) - logf(Z);
    if (pick == a.eos_id) {
      a.finished[row] = 1;
      atomicSub(a.live, 1);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Diverse beam search (Vijayakumar et al., AAAI 2018) of one frame f: K beams per image in G groups of Kg = K / G, with a Hamming
// diversity penalty lambda.  Two launches.
//
// diverse_beam_rows_kernel, one CTA of SAMPLE_THREADS per row (B rows at f = 0, B*K after):
//   history  at f >= 1 with n > 0, hist_out[i] = hist_in[b*K + prev_ptr[i]] ‖ prev_wid[i], exactly as beam_ngram_block_kernel.
//   logp     x[v] = head_logit(row, bias, v); logp[v] = (x[v] - max x) - log(sum exp(x - max x)) in fp32; then -10000 is added at
//            the words the duplicate-n-gram rule blocks (f >= n), and logp[eos] = -10000 while block_eos: beam search's order and
//            values.
//   top K    the K words ranked first by (logp descending, word ascending), found as a threshold on order_key(logp) by binary
//            search over the key's bits plus a scan of the ties in index order (no sort), written in rank order to
//            top_w / top_lp [row, 0:K].
// diverse_beam_merge_kernel, one CTA per image: groups choose in order g = 0 .. G-1.  Group g's candidates are its parents'
//   (beams [g*Kg, (g+1)*Kg); row b at f = 0) row top K with cand = logp + eos_prev * -10000 + score_prev (cand = logp at f = 0);
//   it keeps the Kg with the largest cand - lambda * cnt(w), cnt(w) = beams of groups < g that chose w in this frame, ties to the
//   lower parent then the lower word, in rank order as beams g*Kg ..  The traces get the unpenalised cand.
// Group g penalises at most g*Kg <= K - Kg words, so any (row, word) outside the row's top K has at least Kg unpenalised words of
// the same row ranked strictly ahead of it: the row top K hold every pair a group can keep.  Every sum runs in a fixed order
// (chunk, then a fixed shuffle tree) and the merge only compares, so a frame is bitwise reproducible.
constexpr int MERGE_THREADS = 256;
constexpr int DIVERSE_MAX_CAND = DIVERSE_MAX_BEAMS * DIVERSE_MAX_BEAMS;       // Kg * K <= K * K candidates per group

template <typename T>
__global__ void __launch_bounds__(SAMPLE_THREADS) diverse_beam_rows_kernel(DiverseBeamArgs a) {
  extern __shared__ float rows_smem[];
  __shared__ float redf[33];
  __shared__ int redi[33], prei[SAMPLE_THREADS + 1];
  __shared__ int sel_w[DIVERSE_MAX_BEAMS];
  __shared__ float sel_lp[DIVERSE_MAX_BEAMS];
  const int V = a.V, K = a.K, tid = threadIdx.x, row = blockIdx.x;
  float* val = rows_smem;                                            // [V] logp
  unsigned* bits = reinterpret_cast<unsigned*>(val + V);             // [ceil(V/32)] blocked words
  int* hist = reinterpret_cast<int*>(bits + ((V + 31) >> 5));        // [T_cap] history

  bool blocked = false;
  if (a.n > 0 && a.f >= 1) {                                         // uniform
    const int f = a.f;
    const long long p = f > 1 ? a.prev_ptr[row] : 0;
    const bool parent_ok = p >= 0 && p < K;
    const int* src = a.hist_in + (static_cast<size_t>(row / K) * K + (parent_ok ? p : 0)) * a.T_cap;
    int* dst = a.hist_out + static_cast<size_t>(row) * a.T_cap;
    for (int t = tid; t < f - 1; t += SAMPLE_THREADS) {
      const int w = parent_ok ? src[t] : -1;
      hist[t] = w;
      dst[t] = w;
    }
    if (tid == 0) {
      const long long w64 = a.prev_wid[row];
      const int w = (w64 >= INT_MIN && w64 <= INT_MAX) ? static_cast<int>(w64) : -1;
      hist[f - 1] = w;
      dst[f - 1] = w;
    }
    if (f >= a.n) blocked = ngram_candidates(hist, f, a.n, V, a.ignore, a.n_ignore, bits);
  }

  const T* lrow = static_cast<const T*>(a.logits) + static_cast<size_t>(row) * a.ld;
  const T* bias = static_cast<const T*>(a.bias);
  float mx = -INFINITY;
  for (int v = tid; v < V; v += SAMPLE_THREADS) {
    const float x = head_logit(lrow, bias, v);
    val[v] = x;
    mx = fmaxf(mx, x);
  }
  mx = block_reduce(mx, redf, [](float p, float q) { return fmaxf(p, q); });

  // from here on thread t owns words [lo, hi)
  const int C = ((V + SAMPLE_THREADS - 1) / SAMPLE_THREADS) | 1;
  const int lo = min(tid * C, V), hi = min(lo + C, V);
  float z = 0.f;
  for (int v = lo; v < hi; ++v) z += expf(val[v] - mx);
  const float lse = logf(block_reduce(z, redf, [](float p, float q) { return p + q; }));
  float top = -INFINITY;
  for (int v = lo; v < hi; ++v) {
    float lp = (val[v] - mx) - lse;
    if (blocked && ((bits[v >> 5] >> (v & 31)) & 1u)) lp += -10000.0f;
    if (a.block_eos && v == a.eos_id) lp = -10000.0f;
    val[v] = lp;
    top = fmaxf(top, lp);
  }
  top = block_reduce(top, redf, [](float p, float q) { return fmaxf(p, q); });

  // tau = the largest key with at least K words at or above it
  auto count = [&](unsigned t) {
    int c = 0;
    for (int v = lo; v < hi; ++v) c += order_key(val[v]) >= t;
    return block_reduce(c, redi, [](int p, int q) { return p + q; });
  };
  unsigned klo = 0, khi = order_key(top);
  if (count(khi) >= K) {
    klo = khi;
  } else {
    khi -= 1;
    while (klo < khi) {                                              // uniform: every thread sees the same counts
      const unsigned mid = klo + (khi - klo + 1) / 2;
      if (count(mid) >= K) klo = mid; else khi = mid - 1;
    }
  }
  const unsigned tau = klo;
  const int take = K - (tau == 0xffffffffu ? 0 : count(tau + 1));   // words tied at tau to keep, lowest index first

  int ties = 0;
  for (int v = lo; v < hi; ++v) ties += order_key(val[v]) == tau;
  block_exclusive_scan(ties, redi, prei);
  const int ties_before = prei[tid];
  int rank = ties_before, kept = 0;
  for (int v = lo; v < hi; ++v) {
    const unsigned k = order_key(val[v]);
    kept += k > tau || (k == tau && rank++ < take);
  }
  block_exclusive_scan(kept, redi, prei);                            // the chunk's first slot among the K kept words
  int slot = prei[tid];
  rank = ties_before;
  for (int v = lo; v < hi; ++v) {
    const unsigned k = order_key(val[v]);
    if (k > tau || (k == tau && rank++ < take)) {
      sel_w[slot] = v;
      sel_lp[slot] = val[v];
      ++slot;
    }
  }
  __syncthreads();
  if (tid < K) {                                                     // rank order: (logp descending, word ascending)
    const float lp = sel_lp[tid];
    const unsigned kt = order_key(lp);
    const int w = sel_w[tid];
    int r = 0;
    for (int j = 0; j < K; ++j) {
      const unsigned kj = order_key(sel_lp[j]);
      r += kj > kt || (kj == kt && sel_w[j] < w);
    }
    a.top_w[static_cast<size_t>(row) * K + r] = w;
    a.top_lp[static_cast<size_t>(row) * K + r] = lp;
  }
}

__global__ void __launch_bounds__(MERGE_THREADS) diverse_beam_merge_kernel(DiverseBeamArgs a) {
  __shared__ float pen[DIVERSE_MAX_CAND];
  __shared__ int word[DIVERSE_MAX_CAND];
  __shared__ int chosen[DIVERSE_MAX_BEAMS];                          // words of the beams chosen so far in this frame
  const int b = blockIdx.x, K = a.K, Kg = a.K / a.G, tid = threadIdx.x;
  const bool first = a.f == 0;
  const int nc = first ? K : Kg * K;                                 // one group's candidates: its parents' row top K
  const size_t base = static_cast<size_t>(b) * K;
  // candidate c of group g: parent beam g*Kg + c / K (the image's row at f = 0), the (c % K)-th word of the parent's row top K
  auto parent = [&](int g, int c) { return first ? 0 : g * Kg + c / K; };
  auto slot = [&](int g, int c) { return (first ? static_cast<size_t>(b) : base + parent(g, c)) * K + c % K; };
  auto cand = [&](int g, int c) {
    const float lp = a.top_lp[slot(g, c)];
    const size_t p = base + parent(g, c);
    return first ? lp : lp + a.prev_eos[p] * -10000.0f + a.prev_score[p];
  };
  for (int g = 0; g < a.G; ++g) {
    for (int c = tid; c < nc; c += MERGE_THREADS) {
      const int w = a.top_w[slot(g, c)];
      int cnt = 0;
      for (int q = 0; q < g * Kg; ++q) cnt += chosen[q] == w;
      pen[c] = __fsub_rn(cand(g, c), __fmul_rn(a.lambda, static_cast<float>(cnt)));
      word[c] = w;
    }
    __syncthreads();
    for (int c = tid; c < nc; c += MERGE_THREADS) {
      const float v = pen[c];
      const int w = word[c], pc = c / K;
      int r = 0;                                                     // candidates ranked ahead of c; only r < Kg matters
      for (int d = 0; d < nc && r < Kg; ++d) {
        const float u = pen[d];
        const int pd = d / K;
        r += u > v || (u == v && (pd < pc || (pd == pc && word[d] < w)));
      }
      if (r < Kg) {
        const int k = g * Kg + r;
        chosen[k] = w;
        a.wid[base + k] = w;
        a.ptr[base + k] = parent(g, c);
        a.score[base + k] = cand(g, c);                              // unpenalised
        a.eos[base + k] = w == a.eos_id ? 1.0f : 0.0f;
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Constrained beam search (Anderson et al., EMNLP 2017) of one frame f: K beams in each of S = 2^C constraint states per image, slot
// s*K + k of image b being beam k of state s.  Two launches; vlpk.h states the semantics.
//
// constrained_beam_rows_kernel, one CTA of SAMPLE_THREADS per row (B rows at f = 0, B*S*K after):
//   history  at f >= 1, hist_out[i] = hist_in[b*S*K + prev_ptr[i]] ‖ prev_wid[i], exactly as beam_ngram_block_kernel, always: the
//            constraint match reads it whether or not n-grams are blocked.
//   logp     as diverse_beam_rows_kernel (n-gram and min_len blocks included).
//   complete each of the image's C*A alternatives a of a constraint j not in the row's state s_i is tested by one thread: w = a[-1]
//            completes it when the row's last len(a) - 1 words are a[:-1].  The distinct such words, with dest = s_i ∪ the bits they
//            complete, go to top_w / top_lp / top_dest [row, K + e] (word -1 and dest -1 past the last), and leave the row's word set.
//   top K    of the remaining words (those whose dest is s_i), by the threshold search of diverse_beam_rows_kernel, in rank order to
//            top_w / top_lp [row, 0:K].  A completing word's logp is replaced by a value whose order_key is 0, below every real
//            key; V >= K + C*A keeps at least K words above it.
// constrained_beam_merge_kernel, one CTA per (state s', image b): the candidates of s' are the top K of its own K rows (at f = 0 the
//   image's row, if s' is the root state) and every completing entry of the image's rows with dest == s', with cand = logp +
//   eos_prev * -10000 + score_prev (logp at f = 0); non-finite ones (rows of empty slots) are dropped.  They are staged in dynamic
//   shared memory in any order; every (parent, word) pair is distinct, so the rank by (cand descending, parent ascending, word
//   ascending) does not depend on it.  The K first fill slots s'*K .. in rank order, the rest are left empty.
// Every other word w of a row keeps it in its state, and any such pair outside the row's top K has K pairs of the same row and state
// ranked strictly ahead of it: the rows' top K plus their completing words hold every pair a state can keep.
__device__ __forceinline__ int cbs_root_state(const VlpkConstrainedBeamArgs& a, int b) {
  int s = 0;
  for (int j = 0; j < a.C; ++j) {
    bool empty = true;
    for (int q = 0; q < a.A; ++q) empty &= a.cons[((static_cast<size_t>(b) * a.C + j) * a.A + q) * a.P] == 0;
    s |= empty ? 1 << j : 0;
  }
  return s;
}

template <typename T>
__global__ void __launch_bounds__(SAMPLE_THREADS) constrained_beam_rows_kernel(VlpkConstrainedBeamArgs a) {
  extern __shared__ float cbs_smem[];
  __shared__ float redf[33];
  __shared__ int redi[33], prei[SAMPLE_THREADS + 1];
  __shared__ int sel_w[CBS_MAX_BEAMS];
  __shared__ float sel_lp[CBS_MAX_BEAMS];
  constexpr int MAX_CA = CBS_MAX_CONSTRAINTS * CBS_MAX_ALTS;
  __shared__ int hit[MAX_CA], comp_w[MAX_CA], comp_d[MAX_CA];
  __shared__ int n_comp;
  const int V = a.V, K = a.K, tid = threadIdx.x, row = blockIdx.x, f = a.f;
  const int CA = a.C * a.A, SK = K << a.C, W = K + CA;
  const int b = f == 0 ? row : row / SK;
  const int state = f == 0 ? cbs_root_state(a, b) : (row % SK) / K;
  float* val = cbs_smem;                                             // [V] logp
  unsigned* bits = reinterpret_cast<unsigned*>(val + V);             // [ceil(V/32)] blocked words
  int* hist = reinterpret_cast<int*>(bits + ((V + 31) >> 5));        // [T_cap] history

  if (f >= 1) {                                                      // uniform
    const long long p = f > 1 ? a.prev_ptr[row] : 0;
    const bool parent_ok = p >= 0 && p < SK;
    const int* src = a.hist_in + (static_cast<size_t>(b) * SK + (parent_ok ? p : 0)) * a.T_cap;
    int* dst = a.hist_out + static_cast<size_t>(row) * a.T_cap;
    for (int t = tid; t < f - 1; t += SAMPLE_THREADS) {
      const int w = parent_ok ? src[t] : -1;
      hist[t] = w;
      dst[t] = w;
    }
    if (tid == 0) {
      const long long w64 = a.prev_wid[row];
      const int w = (w64 >= INT_MIN && w64 <= INT_MAX) ? static_cast<int>(w64) : -1;
      hist[f - 1] = w;
      dst[f - 1] = w;
    }
  }
  __syncthreads();
  const bool blocked = a.n > 0 && f >= a.n && ngram_candidates(hist, f, a.n, V, a.ignore, a.n_ignore, bits);

  if (tid < CA) {                                                    // alternative tid: constraint tid / A
    const int64_t* alt = a.cons + (static_cast<size_t>(b) * CA + tid) * a.P;
    int len = 0;
    while (len < a.P && alt[len] != 0) ++len;
    int w = -1;
    if (len > 0 && len - 1 <= f && !((state >> (tid / a.A)) & 1) && alt[len - 1] >= 0 && alt[len - 1] < V) {
      bool match = true;
      for (int t = 0; t < len - 1 && match; ++t) match = hist[f - (len - 1) + t] == alt[t];
      if (match) w = static_cast<int>(alt[len - 1]);
    }
    hit[tid] = w;
  }
  __syncthreads();
  if (tid == 0) {                                                    // distinct completing words in alternative order
    int m = 0;
    for (int q = 0; q < CA; ++q) {
      const int w = hit[q];
      if (w < 0) continue;
      int e = 0;
      while (e < m && comp_w[e] != w) ++e;
      if (e == m) {
        comp_w[m] = w;
        comp_d[m++] = state;
      }
      comp_d[e] |= 1 << (q / a.A);
    }
    n_comp = m;
  }

  const T* lrow = static_cast<const T*>(a.logits) + static_cast<size_t>(row) * a.ld;
  const T* bias = static_cast<const T*>(a.bias);
  float mx = -INFINITY;
  for (int v = tid; v < V; v += SAMPLE_THREADS) {
    const float x = head_logit(lrow, bias, v);
    val[v] = x;
    mx = fmaxf(mx, x);
  }
  mx = block_reduce(mx, redf, [](float p, float q) { return fmaxf(p, q); });

  // from here on thread t owns words [lo, hi)
  const int Cw = ((V + SAMPLE_THREADS - 1) / SAMPLE_THREADS) | 1;
  const int lo = min(tid * Cw, V), hi = min(lo + Cw, V);
  float z = 0.f;
  for (int v = lo; v < hi; ++v) z += expf(val[v] - mx);
  const float lse = logf(block_reduce(z, redf, [](float p, float q) { return p + q; }));
  for (int v = lo; v < hi; ++v) {
    float lp = (val[v] - mx) - lse;
    if (blocked && ((bits[v >> 5] >> (v & 31)) & 1u)) lp += -10000.0f;
    if (a.block_eos && v == a.eos_id) lp = -10000.0f;
    val[v] = lp;
  }
  __syncthreads();
  const size_t out = static_cast<size_t>(row) * W;
  if (tid < CA) {                                                    // completing entries, then out of the top-K search
    const bool used = tid < n_comp;
    const int w = used ? comp_w[tid] : -1;
    a.top_w[out + K + tid] = w;
    a.top_lp[out + K + tid] = used ? val[w] : -INFINITY;
    a.top_dest[static_cast<size_t>(row) * CA + tid] = used ? comp_d[tid] : -1;
    if (used) val[w] = __int_as_float(-1);                         // a NaN whose order_key is 0
  }
  __syncthreads();
  float top = -INFINITY;
  for (int v = lo; v < hi; ++v) top = fmaxf(top, val[v]);            // fmaxf skips the excluded NaNs
  top = block_reduce(top, redf, [](float p, float q) { return fmaxf(p, q); });

  // tau = the largest key with at least K words at or above it
  auto count = [&](unsigned t) {
    int c = 0;
    for (int v = lo; v < hi; ++v) c += order_key(val[v]) >= t;
    return block_reduce(c, redi, [](int p, int q) { return p + q; });
  };
  unsigned klo = 0, khi = order_key(top);
  if (count(khi) >= K) {
    klo = khi;
  } else {
    khi -= 1;
    while (klo < khi) {                                              // uniform: every thread sees the same counts
      const unsigned mid = klo + (khi - klo + 1) / 2;
      if (count(mid) >= K) klo = mid; else khi = mid - 1;
    }
  }
  const unsigned tau = klo;
  const int take = K - (tau == 0xffffffffu ? 0 : count(tau + 1));   // words tied at tau to keep, lowest index first

  int ties = 0;
  for (int v = lo; v < hi; ++v) ties += order_key(val[v]) == tau;
  block_exclusive_scan(ties, redi, prei);
  const int ties_before = prei[tid];
  int rank = ties_before, kept = 0;
  for (int v = lo; v < hi; ++v) {
    const unsigned k = order_key(val[v]);
    kept += k > tau || (k == tau && rank++ < take);
  }
  block_exclusive_scan(kept, redi, prei);                            // the chunk's first slot among the K kept words
  int slot = prei[tid];
  rank = ties_before;
  for (int v = lo; v < hi; ++v) {
    const unsigned k = order_key(val[v]);
    if (k > tau || (k == tau && rank++ < take)) {
      sel_w[slot] = v;
      sel_lp[slot] = val[v];
      ++slot;
    }
  }
  __syncthreads();
  if (tid < K) {                                                     // rank order: (logp descending, word ascending)
    const float lp = sel_lp[tid];
    const unsigned kt = order_key(lp);
    const int w = sel_w[tid];
    int r = 0;
    for (int j = 0; j < K; ++j) {
      const unsigned kj = order_key(sel_lp[j]);
      r += kj > kt || (kj == kt && sel_w[j] < w);
    }
    a.top_w[out + r] = w;
    a.top_lp[out + r] = lp;
  }
}

size_t cbs_merge_smem_bytes(int K, int C, int A) {                   // one state's candidates at most: value, parent, word
  return (static_cast<size_t>(K) * K + (static_cast<size_t>(K) << C) * C * A) * 12;
}

__global__ void __launch_bounds__(MERGE_THREADS) constrained_beam_merge_kernel(VlpkConstrainedBeamArgs a) {
  extern __shared__ float cbs_smem[];
  __shared__ int n_cand;
  const int s = blockIdx.x, b = blockIdx.y, K = a.K, tid = threadIdx.x;
  const int CA = a.C * a.A, SK = K << a.C, W = K + CA;
  const bool first = a.f == 0;
  const int n_stay = first ? (s == cbs_root_state(a, b) ? K : 0) : K * K;     // top-K entries of the state's own rows
  const int n_all = n_stay + (first ? 1 : SK) * CA;                            // ... then every row's completing entries
  float* val = cbs_smem;
  int* par = reinterpret_cast<int*>(val + n_all);
  int* word = par + n_all;
  if (tid == 0) n_cand = 0;
  __syncthreads();
  for (int c = tid; c < n_all; c += MERGE_THREADS) {
    int p, e;                                                        // parent slot, entry of its row
    if (c < n_stay) {
      p = first ? 0 : s * K + c / K;
      e = c % K;
    } else {
      p = first ? 0 : (c - n_stay) / CA;
      e = K + (c - n_stay) % CA;
    }
    const size_t r = first ? static_cast<size_t>(b) : static_cast<size_t>(b) * SK + p;
    if (e >= K && a.top_dest[r * CA + (e - K)] != s) continue;
    const int w = a.top_w[r * W + e];
    if (w < 0) continue;
    const float lp = a.top_lp[r * W + e];
    const float v = first ? lp : lp + a.prev_eos[r] * -10000.0f + a.prev_score[r];
    if (!isfinite(v)) continue;
    const int i = atomicAdd(&n_cand, 1);
    val[i] = v;
    par[i] = p;
    word[i] = w;
  }
  __syncthreads();
  const int n = n_cand;
  const size_t base = static_cast<size_t>(b) * SK + s * K;
  for (int c = tid; c < n; c += MERGE_THREADS) {
    const float v = val[c];
    const int w = word[c], pc = par[c];
    int r = 0;                                                       // candidates ranked ahead of c; only r < K matters
    for (int d = 0; d < n && r < K; ++d) {
      const float u = val[d];
      const int pd = par[d];
      r += u > v || (u == v && (pd < pc || (pd == pc && word[d] < w)));
    }
    if (r < K) {
      a.wid[base + r] = w;
      a.ptr[base + r] = pc;
      a.score[base + r] = v;
      a.eos[base + r] = w == a.eos_id ? 1.0f : 0.0f;
    }
  }
  for (int k = n + tid; k < K; k += MERGE_THREADS) {                 // empty slots
    a.wid[base + k] = 0;
    a.ptr[base + k] = 0;
    a.score[base + k] = -INFINITY;
    a.eos[base + k] = 0.0f;
  }
}

}  // namespace

size_t sample_smem_bytes(int T_cap, int V) {
  return (static_cast<size_t>(V) + (static_cast<size_t>(V) + 31) / 32 + static_cast<size_t>(T_cap)) * 4;
}

int launch_sample(const SampleArgs& a, cudaStream_t s) {
  VLPK_CHECK_ARG(a.rows >= 0 && a.V >= 1 && a.ld >= a.V, "sample: rows=%d V=%d ld=%lld (ld must be >= V >= 1)", a.rows, a.V, a.ld);
  VLPK_CHECK_ARG(a.mode == SAMPLE_TOPK || a.mode == SAMPLE_TOPP, "sample: mode=%d (0 top-k, 1 top-p)", a.mode);
  VLPK_CHECK_ARG(a.mode != SAMPLE_TOPK || (a.topk >= 1 && a.topk <= SAMPLE_MAX_TOPK), "sample: topk=%d outside [1, %d]", a.topk,
                 SAMPLE_MAX_TOPK);
  VLPK_CHECK_ARG(a.mode != SAMPLE_TOPP || (a.topp > 0.f && a.topp <= 1.f), "sample: topp=%g outside (0, 1]", static_cast<double>(a.topp));
  VLPK_CHECK_ARG(a.fp32 == 0 || a.fp32 == 1, "sample: fp32=%d (0 bf16, 1 fp32)", a.fp32);
  VLPK_CHECK_ARG(a.T_cap >= 1 && a.f >= 0 && a.f < a.T_cap, "sample: frame f=%d outside [0, T_cap=%d)", a.f, a.T_cap);
  VLPK_CHECK_ARG(a.n >= 0 && a.n_ignore >= 0 && (a.n_ignore == 0 || a.ignore), "sample: n=%d, ignore set of %d words", a.n, a.n_ignore);
  VLPK_CHECK_ARG(a.logits && a.seq && a.finished && a.live, "sample: null pointer (logits, seq, finished, live)");
  const size_t smem = sample_smem_bytes(a.T_cap, a.V);
  VLPK_CHECK_ARG(smem <= SAMPLE_SMEM_MAX, "sample: T_cap=%d V=%d need %zu bytes of shared memory (at most %zu)", a.T_cap, a.V, smem,
                 SAMPLE_SMEM_MAX);
  if (a.rows == 0) return 0;
  LaunchScope scope(CAT_MISC, (a.fp32 ? 8.0 : 4.0) * a.rows * a.V, s);
  if (a.fp32) {
    static bool attr_set = false;
    if (!attr_set) {
      VLPK_CUDA(cudaFuncSetAttribute(sample_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(SAMPLE_SMEM_MAX)));
      attr_set = true;
    }
    sample_kernel<float><<<a.rows, SAMPLE_THREADS, smem, s>>>(a);
  } else {
    static bool attr_set = false;
    if (!attr_set) {
      VLPK_CUDA(cudaFuncSetAttribute(sample_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(SAMPLE_SMEM_MAX)));
      attr_set = true;
    }
    sample_kernel<bf16><<<a.rows, SAMPLE_THREADS, smem, s>>>(a);
  }
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

int launch_diverse_beam_step(const DiverseBeamArgs& a, cudaStream_t s) {
  VLPK_CHECK_ARG(a.B >= 0 && a.K >= 1 && a.K <= DIVERSE_MAX_BEAMS, "diverse_beam_step: B=%d K=%d (K must lie in [1, %d])", a.B, a.K,
                 DIVERSE_MAX_BEAMS);
  VLPK_CHECK_ARG(a.G >= 1 && a.K % a.G == 0, "diverse_beam_step: G=%d groups do not divide K=%d beams", a.G, a.K);
  VLPK_CHECK_ARG(a.V >= a.K && a.ld >= a.V, "diverse_beam_step: V=%d ld=%lld K=%d (ld >= V >= K needed)", a.V, a.ld, a.K);
  VLPK_CHECK_ARG(a.fp32 == 0 || a.fp32 == 1, "diverse_beam_step: fp32=%d (0 bf16, 1 fp32)", a.fp32);
  VLPK_CHECK_ARG(isfinite(a.lambda) && a.lambda >= 0.f, "diverse_beam_step: diversity penalty %g (finite and >= 0 needed)",
                 static_cast<double>(a.lambda));
  VLPK_CHECK_ARG(a.T_cap >= 1 && a.f >= 0 && a.f < a.T_cap, "diverse_beam_step: frame f=%d outside [0, T_cap=%d)", a.f, a.T_cap);
  VLPK_CHECK_ARG(a.n >= 0 && a.n_ignore >= 0 && (a.n_ignore == 0 || a.ignore), "diverse_beam_step: n=%d, ignore set of %d words", a.n,
                 a.n_ignore);
  VLPK_CHECK_ARG(a.logits && a.top_w && a.top_lp && a.wid && a.ptr && a.score && a.eos,
                 "diverse_beam_step: null pointer (logits, top_w, top_lp, wid, ptr, score, eos)");
  VLPK_CHECK_ARG(a.f == 0 || (a.prev_score && a.prev_eos), "diverse_beam_step: null pointer (prev_score, prev_eos are needed at f=%d)",
                 a.f);
  const bool hist = a.n > 0 && a.f >= 1;
  VLPK_CHECK_ARG(!hist || (a.hist_out && a.prev_wid), "diverse_beam_step: null pointer (hist_out, prev_wid are needed at f=%d)", a.f);
  VLPK_CHECK_ARG(!hist || a.f == 1 || (a.hist_in && a.prev_ptr), "diverse_beam_step: null pointer (hist_in, prev_ptr are needed at f=%d)",
                 a.f);
  VLPK_CHECK_ARG(!hist || a.hist_in != a.hist_out, "diverse_beam_step: hist_in and hist_out must be different buffers");
  const size_t smem = sample_smem_bytes(a.T_cap, a.V);
  VLPK_CHECK_ARG(smem <= SAMPLE_SMEM_MAX, "diverse_beam_step: T_cap=%d V=%d need %zu bytes of shared memory (at most %zu)", a.T_cap, a.V,
                 smem, SAMPLE_SMEM_MAX);
  if (a.B == 0) return 0;
  const int rows = a.f == 0 ? a.B : a.B * a.K;
  {
    LaunchScope scope(CAT_MISC, (a.fp32 ? 8.0 : 4.0) * rows * a.V, s);
    if (a.fp32) {
      static bool attr_set = false;
      if (!attr_set) {
        VLPK_CUDA(cudaFuncSetAttribute(diverse_beam_rows_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(SAMPLE_SMEM_MAX)));
        attr_set = true;
      }
      diverse_beam_rows_kernel<float><<<rows, SAMPLE_THREADS, smem, s>>>(a);
    } else {
      static bool attr_set = false;
      if (!attr_set) {
        VLPK_CUDA(cudaFuncSetAttribute(diverse_beam_rows_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(SAMPLE_SMEM_MAX)));
        attr_set = true;
      }
      diverse_beam_rows_kernel<bf16><<<rows, SAMPLE_THREADS, smem, s>>>(a);
    }
    VLPK_CUDA(cudaGetLastError());
  }
  LaunchScope scope(CAT_MISC, 8.0 * rows * a.K, s);
  diverse_beam_merge_kernel<<<a.B, MERGE_THREADS, 0, s>>>(a);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

int launch_constrained_beam_step(const VlpkConstrainedBeamArgs& a, cudaStream_t s) {
  VLPK_CHECK_ARG(a.C >= 1 && a.C <= CBS_MAX_CONSTRAINTS && a.A >= 1 && a.A <= CBS_MAX_ALTS && a.P >= 1 && a.P <= CBS_MAX_WORDS,
                 "constrained_beam_step: C=%d A=%d P=%d (C in [1, %d], A in [1, %d], P in [1, %d])", a.C, a.A, a.P, CBS_MAX_CONSTRAINTS,
                 CBS_MAX_ALTS, CBS_MAX_WORDS);
  VLPK_CHECK_ARG(a.B >= 0 && a.K >= 1 && a.K <= CBS_MAX_BEAMS && (a.K << a.C) <= CBS_MAX_SLOTS,
                 "constrained_beam_step: B=%d K=%d C=%d (K in [1, %d] and 2^C * K <= %d needed)", a.B, a.K, a.C, CBS_MAX_BEAMS, CBS_MAX_SLOTS);
  VLPK_CHECK_ARG(a.V >= a.K + a.C * a.A && a.ld >= a.V, "constrained_beam_step: V=%d ld=%lld (ld >= V >= K + C*A = %d needed)", a.V,
                 static_cast<long long>(a.ld), a.K + a.C * a.A);
  VLPK_CHECK_ARG(a.fp32 == 0 || a.fp32 == 1, "constrained_beam_step: fp32=%d (0 bf16, 1 fp32)", a.fp32);
  VLPK_CHECK_ARG(a.T_cap >= 1 && a.f >= 0 && a.f < a.T_cap, "constrained_beam_step: frame f=%d outside [0, T_cap=%d)", a.f, a.T_cap);
  VLPK_CHECK_ARG(a.n >= 0 && a.n_ignore >= 0 && (a.n_ignore == 0 || a.ignore), "constrained_beam_step: n=%d, ignore set of %d words", a.n,
                 a.n_ignore);
  VLPK_CHECK_ARG(a.logits && a.cons && a.top_w && a.top_lp && a.top_dest && a.wid && a.ptr && a.score && a.eos,
                 "constrained_beam_step: null pointer (logits, cons, top_w, top_lp, top_dest, wid, ptr, score, eos)");
  VLPK_CHECK_ARG(a.f == 0 || (a.prev_score && a.prev_eos && a.prev_wid && a.hist_out),
                 "constrained_beam_step: null pointer (prev_score, prev_eos, prev_wid, hist_out are needed at f=%d)", a.f);
  VLPK_CHECK_ARG(a.f <= 1 || (a.hist_in && a.prev_ptr), "constrained_beam_step: null pointer (hist_in, prev_ptr are needed at f=%d)", a.f);
  VLPK_CHECK_ARG(a.f == 0 || a.hist_in != a.hist_out, "constrained_beam_step: hist_in and hist_out must be different buffers");
  const size_t smem = sample_smem_bytes(a.T_cap, a.V);
  VLPK_CHECK_ARG(smem <= SAMPLE_SMEM_MAX, "constrained_beam_step: T_cap=%d V=%d need %zu bytes of shared memory (at most %zu)", a.T_cap,
                 a.V, smem, SAMPLE_SMEM_MAX);
  if (a.B == 0) return 0;
  const int SK = a.K << a.C, rows = a.f == 0 ? a.B : a.B * SK;
  {
    LaunchScope scope(CAT_MISC, (a.fp32 ? 8.0 : 4.0) * rows * a.V, s);
    if (a.fp32) {
      static bool attr_set = false;
      if (!attr_set) {
        VLPK_CUDA(cudaFuncSetAttribute(constrained_beam_rows_kernel<float>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(SAMPLE_SMEM_MAX)));
        attr_set = true;
      }
      constrained_beam_rows_kernel<float><<<rows, SAMPLE_THREADS, smem, s>>>(a);
    } else {
      static bool attr_set = false;
      if (!attr_set) {
        VLPK_CUDA(cudaFuncSetAttribute(constrained_beam_rows_kernel<bf16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       static_cast<int>(SAMPLE_SMEM_MAX)));
        attr_set = true;
      }
      constrained_beam_rows_kernel<bf16><<<rows, SAMPLE_THREADS, smem, s>>>(a);
    }
    VLPK_CUDA(cudaGetLastError());
  }
  const size_t merge_smem = cbs_merge_smem_bytes(a.K, a.C, a.A);
  static bool attr_set = false;
  if (!attr_set) {
    VLPK_CUDA(cudaFuncSetAttribute(constrained_beam_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   static_cast<int>(cbs_merge_smem_bytes(CBS_MAX_BEAMS, 2, CBS_MAX_ALTS))));
    attr_set = true;
  }
  LaunchScope scope(CAT_MISC, 8.0 * rows * (a.K + a.C * a.A), s);
  constrained_beam_merge_kernel<<<dim3(1 << a.C, a.B), MERGE_THREADS, merge_smem, s>>>(a);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

size_t ngram_block_smem_bytes(int T_cap, int V) {
  return (static_cast<size_t>(T_cap) + (static_cast<size_t>(V) + 31) / 32) * 4;
}

int launch_beam_ngram_block(const NgramBlockArgs& a, cudaStream_t s) {
  VLPK_CHECK_ARG(a.rows >= 0 && a.K >= 1 && a.rows % a.K == 0, "beam_ngram_block: rows=%d K=%d (rows must be a multiple of K)", a.rows, a.K);
  VLPK_CHECK_ARG(a.n >= 1, "beam_ngram_block: n=%d (n-gram size must be >= 1)", a.n);
  VLPK_CHECK_ARG(a.f >= 1 && a.f <= a.T_cap, "beam_ngram_block: frame f=%d outside [1, T_cap=%d]", a.f, a.T_cap);
  VLPK_CHECK_ARG(a.V >= 1 && a.ld >= a.V, "beam_ngram_block: V=%d ld=%lld (ld must be >= V >= 1)", a.V, a.ld);
  VLPK_CHECK_ARG(a.n_ignore >= 0 && (a.n_ignore == 0 || a.ignore), "beam_ngram_block: ignore set of %d words without a pointer", a.n_ignore);
  VLPK_CHECK_ARG(a.hist_out && a.wid, "beam_ngram_block: null pointer (hist_out, wid)");
  VLPK_CHECK_ARG(a.f == 1 || (a.hist_in && a.ptr), "beam_ngram_block: null pointer (hist_in, ptr are needed at f=%d)", a.f);
  VLPK_CHECK_ARG(a.f < a.n || a.logp, "beam_ngram_block: null pointer (logp is needed at f=%d >= n=%d)", a.f, a.n);
  VLPK_CHECK_ARG(a.hist_in != a.hist_out, "beam_ngram_block: hist_in and hist_out must be different buffers");
  const size_t smem = ngram_block_smem_bytes(a.T_cap, a.V);
  VLPK_CHECK_ARG(smem <= NGRAM_SMEM_MAX, "beam_ngram_block: T_cap=%d V=%d need %zu bytes of shared memory (at most %zu)", a.T_cap, a.V,
                 smem, NGRAM_SMEM_MAX);
  if (a.rows == 0) return 0;
  LaunchScope scope(CAT_MISC, 8.0 * a.rows * a.f, s);
  beam_ngram_block_kernel<<<a.rows, NGRAM_THREADS, smem, s>>>(a);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace vlpk
