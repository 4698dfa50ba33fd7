// vlp_b200 — host-side description of the attention-core launches (see attn.cu).
#pragma once
#include "common.cuh"

namespace vlpk {

struct AttnDesc {
  int B = 0, heads = 0, head_dim = 64;
  int Lq = 0, Lkv = 0;  // query rows / key-value rows per sequence (<= 128)
  // Q: [B, Lq, ld_q] ; K,V: [B, Lkv, ld_kv] ; head h occupies columns [h*64, h*64+64) from each base pointer.
  const void* q = nullptr;
  const void* k = nullptr;
  const void* v = nullptr;
  int64_t ld_q = 0, ld_kv = 0;
  int64_t kv_batch_stride = 0;  // elements between consecutive sequences of K / V (0 = Lkv * ld_kv); a K/V cache has cache_rows * ld_kv
  void* o = nullptr;  // ctx [B, Lq, ld_o]   (bwd: forward output, read for delta)
  int64_t ld_o = 0;
  const uint32_t* mask_bits = nullptr;  // [B, mask_rows, 4] packed by vlpk_mask_pack
  int mask_rows = 0;                    // Lq or 1
  float* lse = nullptr;                 // [B, heads, Lq] (fwd: optional output ; bwd: input)
  DropoutCfg drop = {0.f, 1.f, 0u, 0ull, 0ull, nullptr};   // backward: drop.bits = forward's keep_out (or null: re-evaluate Philox)
  unsigned char* keep_out = nullptr;  // forward, optional: [B*heads*Lq*16] packed keep-decisions of the attention dropout
  // backward only
  const void* d_o = nullptr;  // [B, Lq, ld_o]
  void* dq = nullptr;
  void* dk = nullptr;
  void* dv = nullptr;  // each [B, L, ld_dqkv]
  int64_t ld_dqkv = 0;
  float* dbias = nullptr;  // optional [3 * heads * 64] fp32: += column sums of dQ | dK | dV, summed over sequences in a fixed order
};

int launch_attn_fwd(const AttnDesc& d, cudaStream_t stream);
int launch_attn_bwd(const AttnDesc& d, cudaStream_t stream);

}  // namespace vlpk
