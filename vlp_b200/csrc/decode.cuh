// vlp_b200 — beam-search duplicate-n-gram blocking on the device (see decode.cu).
#pragma once
#include "common.cuh"

namespace vlpk {

struct NgramBlockArgs {
  int rows = 0, K = 1;                // hypotheses (B*K) and beam width; row i = b*K + k
  int f = 1;                          // frame: hist_out receives f words, logp is frame f's scores
  int T_cap = 0;                      // words per history row (allocated width of hist_in / hist_out)
  int n = 3;                          // n-gram size
  const int* hist_in = nullptr;       // [rows, T_cap] int32 history of frame f-1 (f-1 words; unused at f = 1)
  int* hist_out = nullptr;            // [rows, T_cap] int32 history of frame f (f words written)
  const long long* ptr = nullptr;     // [rows] back pointers of frame f-1, in [0, K) (unused at f = 1)
  const long long* wid = nullptr;     // [rows] word ids of frame f-1
  const int* ignore = nullptr;        // [n_ignore] word ids exempt from blocking
  int n_ignore = 0;
  float* logp = nullptr;              // [rows, ld] fp32 log-probabilities, += -10000 at blocked words
  long long ld = 0;
  int V = 0;
};

size_t ngram_block_smem_bytes(int T_cap, int V);
int launch_beam_ngram_block(const NgramBlockArgs& a, cudaStream_t s);

}  // namespace vlpk
