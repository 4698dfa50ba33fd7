// vlp_b200 — beam-search duplicate-n-gram blocking on the device (see decode.cu).
#pragma once
#include "../../include/vlpk.h"
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

// Top-k / top-p sampling of one decode frame, one CTA per row (see decode.cu).
enum SampleMode { SAMPLE_TOPK = 0, SAMPLE_TOPP = 1 };
constexpr int SAMPLE_MAX_TOPK = 64;

struct SampleArgs {
  int rows = 0, V = 0;
  const void* logits = nullptr;       // [rows, ld] bf16 or fp32 decoder outputs, without the bias
  long long ld = 0;
  const void* bias = nullptr;         // [V] same dtype, or null
  int fp32 = 0;                       // dtype of logits and bias: 0 bf16, 1 fp32
  int mode = SAMPLE_TOPK;
  int topk = 1;                       // 1 <= topk <= SAMPLE_MAX_TOPK
  float topp = 1.f;                   // 0 < topp <= 1
  unsigned long long seed = 0;
  int f = 0;                          // frame: the token goes to seq[row, f], seq[row, :f] is the row's history
  long long* seq = nullptr;           // [rows, T_cap] int64 word ids
  int T_cap = 0;
  float* score = nullptr;             // [rows, T_cap] log-probability of the chosen token, or null
  int* finished = nullptr;            // [rows] 0 / 1
  int* live = nullptr;                // [1] rows not finished yet
  int eos_id = -1, pad_id = 0;
  int block_eos = 0;                  // 1: frame below min_len, [EOS] is set to -10000
  int n = 0;                          // duplicate-n-gram blocking: n-gram size, 0 = off
  const int* ignore = nullptr;
  int n_ignore = 0;
};

size_t sample_smem_bytes(int T_cap, int V);
int launch_sample(const SampleArgs& a, cudaStream_t s);

// Diverse beam search: one frame's selection, K beams per image in G groups with a Hamming penalty (see decode.cu).
constexpr int DIVERSE_MAX_BEAMS = SAMPLE_MAX_TOPK;

struct DiverseBeamArgs {
  int B = 0, K = 1, G = 1;            // images, beams per image, groups (G divides K; Kg = K / G)
  int f = 0;                          // frame: rows = B at f = 0 (one per image), B*K after (row b*K + k)
  int V = 0;
  const void* logits = nullptr;       // [rows, ld] bf16 or fp32 decoder outputs, without the bias
  long long ld = 0;
  const void* bias = nullptr;         // [V] same dtype, or null
  int fp32 = 0;                       // dtype of logits and bias: 0 bf16, 1 fp32
  float lambda = 0.f;                 // diversity penalty per earlier-group use of a word, >= 0
  int eos_id = -1;
  int block_eos = 0;                  // 1: frame below min_len, logp[eos] = -10000
  int T_cap = 0;                      // words per history row; frames f < T_cap
  int n = 0;                          // duplicate-n-gram blocking: n-gram size, 0 = off
  const int* hist_in = nullptr;       // [B*K, T_cap] int32 history of frame f-1 (read at f >= 2)
  int* hist_out = nullptr;            // [B*K, T_cap] int32 history of frame f (f words; written at f >= 1)
  const int* ignore = nullptr;
  int n_ignore = 0;
  const long long* prev_wid = nullptr;    // [B, K] frame f-1's traces (f >= 1)
  const long long* prev_ptr = nullptr;
  const float* prev_score = nullptr;
  const float* prev_eos = nullptr;
  int* top_w = nullptr;               // [rows, K] scratch: each row's top K words and log-probabilities
  float* top_lp = nullptr;
  long long* wid = nullptr;           // [B, K] frame f's traces
  long long* ptr = nullptr;
  float* score = nullptr;
  float* eos = nullptr;
};

int launch_diverse_beam_step(const DiverseBeamArgs& a, cudaStream_t s);

// Constrained beam search: one frame's selection, K beams in each of the 2^C constraint states (see decode.cu and vlpk.h).
constexpr int CBS_MAX_CONSTRAINTS = 4, CBS_MAX_ALTS = 4, CBS_MAX_WORDS = 8, CBS_MAX_BEAMS = 64, CBS_MAX_SLOTS = 256;

int launch_constrained_beam_step(const VlpkConstrainedBeamArgs& a, cudaStream_t s);

}  // namespace vlpk
