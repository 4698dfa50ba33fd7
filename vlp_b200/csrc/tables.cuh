// vlp_b200 — gradients of the three embedding tables from the pre-LayerNorm gradient of BertEmbeddings (see tables.cu).
#pragma once
#include "common.cuh"

namespace vlpk {

struct TableGradArgs {
  int B = 0, L = 0, H = 0, R = 0, vis_input = 1;
  int V = 0, P = 0, T = 0;            // rows of the word / position / token-type tables
  const long long* ids = nullptr;     // [B,L]
  const long long* tt = nullptr;      // [B,L] (null -> 0)
  const long long* pos = nullptr;     // [B,L] (null -> arange)
  const __nv_bfloat16* dz = nullptr;  // [B*L,H] gradient wrt the pre-LayerNorm sum (vlpk_embed_bwd)
  __nv_bfloat16* d_word = nullptr;    // [V,H] overwritten (zero except the looked-up rows)
  float* scratch = nullptr;           // [V,H] fp32, uninitialised: only the looked-up rows are touched
  float* d_pos = nullptr;             // [P,H] fp32, zeroed by the caller
  float* d_type = nullptr;            // [T,H] fp32, zeroed by the caller
};

int launch_embed_tables_bwd(const TableGradArgs& a, cudaStream_t s);

}  // namespace vlpk
