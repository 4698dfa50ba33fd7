// vlp_b200 — host-side description of the attention-core launches (see attn.cu).
#pragma once
#include "common.cuh"

namespace vlpk {

struct AttnDesc {
  int B = 0, heads = 0, head_dim = 64;
  int Lq = 0, Lkv = 0;  // query rows / key-value rows per sequence (<= 128, or <= 512 with kv_slots)
  int kv_slots = 0;     // 0: single-tile layout (Lq, Lkv <= 128); else 128 * ceil(Lkv / 128) key slots per mask / keep-bit row
  // Q: [B, Lq, ld_q] ; K,V: [B, Lkv, ld_kv] ; head h occupies columns [h*64, h*64+64) from each base pointer.
  const void* q = nullptr;
  const void* k = nullptr;
  const void* v = nullptr;
  int64_t ld_q = 0, ld_kv = 0;
  int64_t kv_batch_stride = 0;  // elements between consecutive sequences of K / V (0 = Lkv * ld_kv); a K/V cache has cache_rows * ld_kv
  void* o = nullptr;  // ctx [B, Lq, ld_o]   (bwd: forward output, read for delta)
  int64_t ld_o = 0;
  int64_t q_batch_stride = 0, o_batch_stride = 0;  // forward: as kv_batch_stride for Q and ctx (0 = Lq * ld_q / Lq * ld_o)
  const uint32_t* mask_bits = nullptr;  // [B, mask_rows, S / 32] packed by vlpk_mask_pack, S = kv_slots (128 when 0)
  int mask_rows = 0;                    // Lq or 1
  float* lse = nullptr;                 // [B, heads, Lq] (fwd: optional output ; bwd: input)
  DropoutCfg drop = {0.f, 1.f, 0u, 0ull, 0ull, nullptr};   // backward: drop.bits = forward's keep_out (or null: re-evaluate Philox)
  unsigned char* keep_out = nullptr;  // forward, optional: [B*heads*Lq*S/8] packed keep-decisions of the attention dropout
  // backward only
  const void* d_o = nullptr;  // [B, Lq, ld_o]
  void* dq = nullptr;
  void* dk = nullptr;
  void* dv = nullptr;  // each [B, L, ld_dqkv]
  int64_t ld_dqkv = 0;
  float* dbias = nullptr;  // optional [3 * heads * 64] fp32: += column sums of dQ | dK | dV, summed over sequences in a fixed order
};

// Keys of d.B hypotheses in groups of G per image (vlpk_layer_cached_group_fwd, vlpk_encoder_score_group_fwd): hypothesis b reads
// key r < P from row r of image b / G's prefix [images, prefix_rows, ld_kv], key P + j from text row slots[b * T + j] (j < pos) or
// b * T + j (its own rows) of text [B * T rows, ld_text]; K at column 0, V at column heads * 64 of both.  slots may be NULL when
// pos = 0.  mask_bits has one sequence per image.  Q / ctx take d.q_batch_stride / d.o_batch_stride.
// Forward only, no dropout: d.k / d.v / d.kv_batch_stride unused, d.ld_kv is the row stride of prefix and text.  Needs
// P + pos + Lq == Lkv and pos + Lq <= T; with a self key (AttnSelfKv), P + pos <= Lkv <= P + T instead: key P + j, j < Lkv - P, from
// the hypothesis' text rows, then each query row's own key.
struct AttnGroupKv {
  const void* prefix = nullptr;
  int prefix_rows = 0, P = 0;
  const void* text = nullptr;
  const int32_t* slots = nullptr;
  int T = 0, G = 1, pos = 0;
  int64_t ld_text = 0;  // row stride of text (0: d.ld_kv)
};

// Query row i of sequence b also attends to one extra key, its own (k_self, v_self) row: k_self + b * self_batch_stride + i * ld_self
// (v_self alike), never masked.  Forward only, no dropout; d.mask_rows must be d.Lq.  Lq, Lkv in [1, 512]: the single-tile kernel when
// both are <= 128 (kv_slots 0), else the tiled one (kv_slots = 128 * ceil(Lkv / 128), or 0 for Lkv <= 128: the 128-slot layout).
struct AttnSelfKv {
  const void* k = nullptr;
  const void* v = nullptr;
  int64_t ld = 0, batch_stride = 0;
};

// Keys from d.k / d.v, or from a shared prefix (group non-null); self non-null adds each query row's own key.  Lq, Lkv <= 128: the
// single-tile kernels; longer sequences (or the "attn_tiled" test option): the KV-tiled kernels.
int launch_attn_fwd(const AttnDesc& d, const AttnGroupKv* group, const AttnSelfKv* self, cudaStream_t stream);
int launch_attn_bwd(const AttnDesc& d, cudaStream_t stream);
void set_attn_tiled(bool on);
// Attention probabilities exp(s - lse) of query rows [row0, Lq) into p [B, heads, Lq - row0, ld_p] (sequences p_batch_stride floats
// apart, 0 = heads * (Lq - row0) * ld_p) from d.q / d.k / d.mask_bits / d.lse; q_batch_stride as d.kv_batch_stride for Q.
int launch_attn_probs(const AttnDesc& d, int64_t q_batch_stride, int row0, float* p, int64_t ld_p, int64_t p_batch_stride,
                      cudaStream_t stream);

}  // namespace vlpk
