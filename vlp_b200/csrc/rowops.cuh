// vlp_b200 — argument structs for the HBM-bound row kernels (see rowops.cu).
#pragma once
#include "common.cuh"

namespace vlpk {

enum { VLPK_DT_BF16 = 0, VLPK_DT_F32 = 1, VLPK_DT_I64 = 2 };
enum { MASK_ADDITIVE = 0, MASK_ZERO_ONE = 1 };

// y = LayerNorm(dropout(t) + res) * gamma + beta        (eps inside the sqrt; modeling.py:188-192)
struct LnArgs {
  long long M = 0;
  int H = 0;
  float eps = 1e-5f;
  const __nv_bfloat16* t = nullptr;      // [M,H] dense output (bias already added)
  const __nv_bfloat16* res = nullptr;    // [M,H] residual (may be null)
  const __nv_bfloat16* gamma = nullptr;  // [H]
  const __nv_bfloat16* beta = nullptr;   // [H]
  __nv_bfloat16* y = nullptr;            // [M,H]
  float2* stats = nullptr;               // [M] (mean, rstd)
  DropoutCfg drop = {0.f, 1.f, 0u, 0ull, 0ull, nullptr};
  // backward
  const __nv_bfloat16* dy = nullptr;  // [M,H]
  __nv_bfloat16* dz = nullptr;        // [M,H] grad wrt (dropout(t)+res)  == grad wrt res
  __nv_bfloat16* dt = nullptr;        // [M,H] grad wrt t (dropout applied); may be null
  float* dgamma = nullptr;            // [H] fp32 accumulators (atomicAdd)
  float* dbeta = nullptr;
  float* dbias = nullptr;             // [H] column sum of dt = gradient of the dense bias
  float* part = nullptr;              // deterministic mode (set by the launcher): [3][grid][H] per-block dgamma | dbeta | dbias
};

int launch_ln_res_drop_fwd(const LnArgs& a, cudaStream_t s);
int launch_ln_res_drop_bwd(const LnArgs& a, cudaStream_t s);

// y = dropout(LayerNorm(word_or_vis + pos_or_vispe + type))     (modeling.py:217-241)
struct EmbedArgs {
  int B = 0, L = 0, H = 0, R = 0;  // R = len_vis_input
  int vis_input = 1;
  float eps = 1e-5f;
  const long long* ids = nullptr;  // [B,L]
  const long long* tt = nullptr;   // [B,L] (null -> 0)
  const long long* pos = nullptr;  // [B,L] (null -> arange)
  const __nv_bfloat16* word = nullptr;
  const __nv_bfloat16* posw = nullptr;
  const __nv_bfloat16* typew = nullptr;
  const __nv_bfloat16* vis = nullptr;  // [B,R,H] projected region features
  const __nv_bfloat16* vpe = nullptr;  // [B,R,H] projected region positional encodings
  const __nv_bfloat16* gamma = nullptr;
  const __nv_bfloat16* beta = nullptr;
  __nv_bfloat16* y = nullptr;  // [B*L,H]
  float2* stats = nullptr;     // [B*L]
  DropoutCfg drop = {0.f, 1.f, 0u, 0ull, 0ull, nullptr};
  // backward
  const __nv_bfloat16* dy = nullptr;
  __nv_bfloat16* dz = nullptr;  // [B*L,H] grad wrt the pre-LN sum
  float* dgamma = nullptr;
  float* dbeta = nullptr;
  float* part = nullptr;  // deterministic mode (set by the launcher): [2][grid][H] per-block dgamma | dbeta
};

int launch_embed_fwd(const EmbedArgs& a, cudaStream_t s);
int launch_embed_bwd(const EmbedArgs& a, cudaStream_t s);

int launch_mask_pack(const void* mask, int dtype, int mode, int B, int rows, int kv, long long stride_b, long long stride_r,
                     uint32_t* out, cudaStream_t s);
int launch_mask_synth(const int* len_b, const int* mode, int len_a, int B, int L, uint32_t* out, cudaStream_t s);
int launch_mask_synth_grouped(const int* len_b, int G, int len_a, int B, int T, uint32_t* out, cudaStream_t s);
int launch_colsum(const void* x, long long ld, long long M, int N, float* out, cudaStream_t s);
// out[i] += sum_{p < parts} part[p * n + i], in the order p = 0, 1, ... (the same bits on every run)
int launch_sum_parts(const float* part, int parts, long long n, float* out, cudaStream_t s);
int launch_f32_to_bf16(const float* x, void* y, long long n, cudaStream_t s);
int launch_dropout_mask(const DropoutCfg& d, long long n, unsigned char* out, cudaStream_t s);


}  // namespace vlpk
