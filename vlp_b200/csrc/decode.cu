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

  const int nwords = (a.V + 31) >> 5;
  for (int j = tid; j < nwords; j += blockDim.x) bits[j] = 0u;
  __syncthreads();

  const int m = a.n - 1;                                           // words matched before a candidate
  const int t0 = f - m;                                            // start of the tail
  if (a.n_ignore > 0) {
    int hit = 0;
    for (int t = (m == 0 ? 0 : t0) + tid; t < f; t += blockDim.x) hit |= is_ignored(seq[t], a.ignore, a.n_ignore);
    if (__syncthreads_or(hit)) return;
  }
  int found = 0;
  for (int s = tid; s < t0; s += blockDim.x) {                     // s <= f - n
    bool match = true;
    for (int j = 0; j < m && match; ++j) match = seq[s + j] == seq[t0 + j];
    if (!match) continue;
    const int w = seq[s + m];
    if (w < 0 || w >= a.V) continue;
    if (a.n_ignore > 0 && is_ignored(w, a.ignore, a.n_ignore)) continue;
    atomicOr(bits + (w >> 5), 1u << (w & 31));
    found = 1;
  }
  if (!__syncthreads_or(found)) return;                            // no candidate: the row is not touched

  float* row = a.logp + static_cast<size_t>(i) * a.ld;
  for (int j = tid; j < nwords; j += blockDim.x) {
    unsigned w = bits[j];
    while (w) {
      const int b = __ffs(w) - 1;
      w &= w - 1;
      row[j * 32 + b] += -10000.0f;
    }
  }
}

}  // namespace

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
