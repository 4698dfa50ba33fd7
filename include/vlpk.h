/* vlpk.h — C ABI of libvlpk.so, the H100-native (sm_90a) replacement for VLP's data-parallel hot path.
 *
 * The reference (LuoweiZhou/VLP) has no FFI layer: its operator API is the nn.Module surface of
 * pytorch_pretrained_bert/modeling.py.  Each entry point below replaces the eager-PyTorch body of one of
 * those modules (file:line cited per function); vlp_b200/vlp_modules.py keeps the Python surface and
 * binds these symbols with ctypes (see INTEGRATION.md for the reference-side binding).
 *
 * Conventions
 *   - every pointer is a raw CUDA device pointer owned by the caller; the library never allocates or
 *     frees device memory and keeps no references after the call returns;
 *   - activations / parameters are bf16, row-major; Linear weights are [out,in] exactly like nn.Linear;
 *   - gradients of parameters are ACCUMULATED (+=) into caller-provided fp32 buffers (zero them first);
 *   - `stream` is a cudaStream_t; all work is enqueued asynchronously on it, no host synchronisation,
 *     CUDA-graph capturable;
 *   - return value: 0 = OK, < 0 = argument/shape/alignment error (nothing launched),
 *     > 0 = cudaError_t.  vlpk_last_error() returns a thread-local description.
 *   - there is no CPU fallback and no other backend: unsupported configurations are errors.
 */
#ifndef VLPK_H_
#define VLPK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define VLPK_VERSION 102

/* dtype tags for vlpk_mask_pack */
#define VLPK_BF16 0
#define VLPK_F32 1
#define VLPK_I64 2
/* mask interpretation */
#define VLPK_MASK_ADDITIVE 0 /* 0 / -10000 additive mask, modeling.py:832 */
#define VLPK_MASK_ZERO_ONE 1 /* 1 = attend, 0 = masked, seq2seq_loader.py:291-304 */
/* activations for vlpk_linear_* */
#define VLPK_ACT_NONE 0
#define VLPK_ACT_RELU 1

typedef struct VlpkDropout {
  float p;                  /* drop probability; 0 disables */
  uint64_t seed;            /* Philox key */
  const uint64_t* seed_dev; /* optional device counter added to `seed` at run time (CUDA-graph replays) */
} VlpkDropout;

/* Key slots.  Attention over Lkv keys lays its per-row data out in S = 128 * ceil(Lkv / 128) key slots (128, 256, 384 or 512): a
 * packed mask row has S / 32 u32 words, an attention keep-bit row S / 8 bytes, and the attention dropout element of (sequence b, head
 * h, query q, key j) is ((b * heads + h) * Lq + q) * S + j.  For Lkv <= 128 this is the 128-slot layout of earlier versions. */
typedef struct VlpkShape {
  int32_t B;     /* sequences */
  int32_t Lq;    /* query rows per sequence  (<= 128, or <= kv_slots) */
  int32_t Lkv;   /* key/value rows per sequence (<= 128, or <= 512 with kv_slots); == Lq except incremental decode */
  int32_t H;     /* hidden size (multiple of 64) */
  int32_t heads; /* H / 64 */
  int32_t I;     /* intermediate size */
  int32_t kv_slots; /* 0: Lq, Lkv <= 128 and masks / keep-bits in the 128-slot layout; else S = 128 * ceil(Lkv / 128), which every mask
                     * and keep-bit buffer passed with this shape must have.  Added after version 102: a C caller that builds VlpkShape
                     * itself must zero it (e.g. `VlpkShape s = {0}`). */
} VlpkShape;

/* One BertLayer's parameters (modeling.py:244-372), bf16, nn.Linear layout [out,in]. */
typedef struct VlpkLayerWeights {
  const void *wq, *wk, *wv; /* attention.self.{query,key,value}.weight [H,H] */
  const void *bq, *bk, *bv; /* .bias [H] */
  const void *wo, *bo;      /* attention.output.dense [H,H],[H] */
  const void *ln1_g, *ln1_b;/* attention.output.LayerNorm */
  const void *w1, *b1;      /* intermediate.dense [I,H],[I] */
  const void *w2, *b2;      /* output.dense [H,I],[H] */
  const void *ln2_g, *ln2_b;/* output.LayerNorm */
} VlpkLayerWeights;

/* fp32 gradient accumulators for one layer. */
typedef struct VlpkLayerGrads {
  float* wqkv; /* [3H,H] rows = query | key | value */
  float* bqkv; /* [3H] */
  float *wo, *bo, *ln1_g, *ln1_b, *w1, *b1, *w2, *b2, *ln2_g, *ln2_b;
} VlpkLayerGrads;

/* Per-layer activations written by forward and read by backward (all caller-allocated). */
typedef struct VlpkLayerActs {
  void* qkv;     /* [B*Lq, 3H]  (incremental decode: q in [:, :H] of a [B*Lq,H] buffer — see vlpk_mha_fwd) */
  void* ctx;     /* [B*Lq, H]   attention context */
  void* t1;      /* [B*Lq, H]   attention.output.dense result */
  void* y1;      /* [B*Lq, H]   BertAttention output (after LayerNorm) */
  void* u;       /* [B*Lq, I]   gelu'(pre-activation): all that backward needs of it */
  void* hmid;    /* [B*Lq, I]   GELU output */
  void* t2;      /* [B*Lq, H]   output.dense result */
  void* y;       /* [B*Lq, H]   layer output */
  float* lse;    /* [B, heads, Lq] */
  float* stats1; /* [B*Lq, 2]  (mean, rstd) of attention.output.LayerNorm */
  float* stats2; /* [B*Lq, 2] */
  void* kv;      /* incremental decode only: [B*Lkv, 2H] key|value projections; else NULL */
  /* Optional (NULL = attention backward re-evaluates Philox): packed keep-decisions of the attention-probability dropout, 1 bit per
   * element (byte i = elements 8i..8i+7, numbering as in vlpk_debug_dropout_mask; S key slots per query row, S = 128 when
   * kv_slots = 0).  Written by the forward attention kernel, read by the backward one. */
  unsigned char* drop_attn; /* [B*heads*Lq*S/8] */
} VlpkLayerActs;

/* Scratch for backward, shared by all layers (bf16). */
typedef struct VlpkBwdScratch {
  void* dz2;  /* [M,H] */
  void* dt2;  /* [M,H] */
  void* du;   /* [M,I] */
  void* dy1;  /* [M,H] */
  void* dz1;  /* [M,H] */
  void* dt1;  /* [M,H] */
  void* dctx; /* [M,H] */
  void* dqkv; /* [M,3H] */
  void* dx;   /* [M,H] ping-pong buffer for the inter-layer gradient */
} VlpkBwdScratch;

int vlpk_version(void);
const char* vlpk_last_error(void);
/* Leave n SMs out of the persistent GEMM grids (and of the tile cost model) from now on; 0 restores the full machine.  For
 * data-parallel callers while a collective that owns SMs (NCCL all-reduce of the previous gradient arena) runs beside the
 * backward GEMMs: a grid sized for all SMs would have its last CTAs wait behind the collective's. */
void vlpk_set_reserved_sms(int n);
/* Deterministic mode (process-wide, default 0; no launch, cheap enough to call before every library call).  When on, every
 * reduction whose fp32 additions could happen in a run-dependent order (atomics from several blocks, split-K reduce-add, the
 * embedding-table scatter of repeated ids) writes partials that are summed in a fixed order, and the split-K counts no longer
 * depend on vlpk_set_reserved_sms: on one GPU, gradients and BertAdam results are bitwise reproducible.  Slower; the default path
 * is unchanged.  Python selects it with torch.use_deterministic_algorithms(True). */
void vlpk_set_deterministic(int on);
/* host-only: the (tile N, split-K) the cost model picks for a GEMM; out2 = {bn, splits}.  No GPU needed. */
int vlpk_debug_plan_gemm(int M, int N, int K, int a_mn, int b_mn, int nseg, int seg_rows, int epi, int bn, int splits, int* out2);
/* A-B testing only: switch a host-side scheduling choice at run time.  "wgrad_stream" (default 1, env VLPK_WGRAD_STREAM=0 turns it
 * off): the weight-gradient GEMM of each Linear's backward runs on a side stream behind its dgrad.  "attn_tiled" (default 0, test
 * support): the KV-tiled attention kernels, which otherwise run only when Lq or Lkv > 128, run at every length.  < 0: unknown name. */
int vlpk_debug_set_option(const char* name, int value);

/* get_extended_attention_mask (modeling.py:807-833) -> per-row S-bit "attend" bitmask, S = 128 * ceil(kv / 128), kv <= 512.
 * mask: [B, rows, kv] with element strides (stride_b, stride_r, 1); rows may be 1 (2-D mask). out: [B, rows, S / 32] u32 (bits >= kv
 * are 0; for kv <= 128, [B, rows, 4] exactly as in earlier versions). */
int vlpk_mask_pack(const void* mask, int dtype, int mode, int B, int rows, int kv, int64_t stride_b, int64_t stride_r,
                   uint32_t* out, void* stream);

/* Input staging (SURVEY.md §8f-4): the loader's self-attention mask (vlp/seq2seq_loader.py:291-301) synthesised on the device from
 * three integers per sample instead of shipping [B,L,L] int64: len_a region tokens (same for the batch), len_b[b] text tokens,
 * mode[b] (0 = bidirectional, 1 = seq2seq), L <= 512.  Output: [B, L, S / 32] u32, the packed bitmask vlpk_mask_pack would produce
 * from the loader's matrix. */
int vlpk_mask_synth(const int32_t* len_b, const int32_t* mode, int len_a, int B, int L, uint32_t* out, void* stream);

/* y[M,N] = dropout(act(x[M,K] w[N,K]^T + b)) — vis_embed / vis_pe_embed Linears (modeling.py:1003-1018, 1035-1036).
 * K need not be tile aligned but ldx/ldw (elements) must be multiples of 8. */
int vlpk_linear_fwd(int M, int N, int K, const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias, void* y,
                    int64_t ldy, int act, const VlpkDropout* drop, uint64_t site, void* stream);
/* Backward of the above.  dy is the gradient of y; y is the forward output (ReLU/dropout mask is recovered from y>0).
 * dpre: [M,N] bf16 scratch (gradient before activation).  dx may be NULL.  dw [N,ldw_g] / db [N] fp32, accumulated. */
int vlpk_linear_bwd(int M, int N, int K, const void* x, int64_t ldx, const void* w, int64_t ldw, const void* y, int64_t ldy,
                    const void* dy, int64_t lddy, void* dpre, void* dx, int64_t lddx, float* dw, int64_t lddw, float* db,
                    int act, float p_drop, void* stream);

/* BertEmbeddings.forward (modeling.py:217-241): gathers + region splice + LayerNorm(eps 1e-5) + dropout. */
int vlpk_embed_fwd(int B, int L, int H, int R, int vis_input, const int64_t* ids, const int64_t* token_type, const int64_t* pos,
                   const void* word_w, const void* pos_w, const void* type_w, const void* vis, const void* vis_pe,
                   const void* ln_g, const void* ln_b, void* y, float* stats, const VlpkDropout* drop, uint64_t site, void* stream);
/* dz = gradient wrt the pre-LayerNorm sum [B*L,H] (caller scatters it to tables / region projections). */
int vlpk_embed_bwd(int B, int L, int H, int R, int vis_input, const int64_t* ids, const int64_t* token_type, const int64_t* pos,
                   const void* word_w, const void* pos_w, const void* type_w, const void* vis, const void* vis_pe,
                   const void* ln_g, const float* stats, const void* dy, void* dz, float* d_ln_g, float* d_ln_b,
                   const VlpkDropout* drop, uint64_t site, void* stream);

/* Scatter of dz (from vlpk_embed_bwd) into the three embedding tables — autograd backward of the nn.Embedding lookups of
 * BertEmbeddings (modeling.py:217-241).  Rows 1..R of every sample are region rows (vis_input) and do not read the word /
 * position tables; every row reads the token-type table.  d_word [V,H] bf16 is overwritten (zero except looked-up rows; duplicates
 * accumulate in fp32 through word_scratch [V,H] fp32, which may be uninitialised); d_pos [P,H] / d_type [T,H] fp32 are
 * accumulated into (zero them first); T <= 8. */
int vlpk_embed_tables_bwd(int B, int L, int H, int R, int vis_input, const int64_t* ids, const int64_t* token_type, const int64_t* pos,
                          const void* dz, int V, int P, int T, void* d_word, float* word_scratch, float* d_pos, float* d_type,
                          void* stream);

/* y = LayerNorm(dropout(t) + res) (BertSelfOutput / BertOutput tail, modeling.py:315-316, 355-356; eps 1e-5). */
int vlpk_ln_res_drop_fwd(int64_t M, int H, const void* t, const void* res, const void* gamma, const void* beta, void* y,
                         float* stats, const VlpkDropout* drop, uint64_t site, void* stream);
int vlpk_ln_res_drop_bwd(int64_t M, int H, const void* t, const void* res, const void* gamma, const float* stats, const void* dy,
                         void* dz, void* dt, float* dgamma, float* dbeta, float* dbias, const VlpkDropout* drop, uint64_t site,
                         void* stream);

/* softmax(QK^T/8 + mask) V per (sequence, head) — BertSelfAttention core (modeling.py:279-302).  Masks in the 128-slot layout:
 * Lq, Lkv <= 128.  The _wide forms take the key-slot count of the mask (and dropout numbering) as kv_slots, with VlpkShape's meaning:
 * 0 = 128-slot layout with Lq, Lkv <= 128; else 128 * ceil(Lkv / 128) for Lkv <= 512. */
int vlpk_attn_core_fwd(int B, int heads, int Lq, int Lkv, const void* q, int64_t ld_q, const void* k, const void* v, int64_t ld_kv,
                       const uint32_t* mask_bits, int mask_rows, void* ctx, int64_t ld_ctx, float* lse, const VlpkDropout* drop,
                       uint64_t site, void* stream);
int vlpk_attn_core_bwd(int B, int heads, int L, const void* q, const void* k, const void* v, int64_t ld_qkv, const uint32_t* mask_bits,
                       int mask_rows, const void* ctx, const void* dctx, int64_t ld_ctx, const float* lse, void* dq, void* dk,
                       void* dv, int64_t ld_dqkv, const VlpkDropout* drop, uint64_t site, void* stream);
int vlpk_attn_core_fwd_wide(int B, int heads, int Lq, int Lkv, const void* q, int64_t ld_q, const void* k, const void* v, int64_t ld_kv,
                            const uint32_t* mask_bits, int mask_rows, void* ctx, int64_t ld_ctx, float* lse, const VlpkDropout* drop,
                            uint64_t site, int kv_slots, void* stream);
int vlpk_attn_core_bwd_wide(int B, int heads, int L, const void* q, const void* k, const void* v, int64_t ld_qkv,
                            const uint32_t* mask_bits, int mask_rows, const void* ctx, const void* dctx, int64_t ld_ctx, const float* lse,
                            void* dq, void* dk, void* dv, int64_t ld_dqkv, const VlpkDropout* drop, uint64_t site, int kv_slots,
                            void* stream);
/* Attention probabilities of one layer (opt-in: the forward kernels never store them).  Recomputed from the layer's bf16 q, k and the
 * logsumexp its forward attention saved (VlpkLayerActs.lse):
 *   P[b, h, i - row0, j] = exp(s_ij - lse[b, h, i]),  s_ij = q_i . k_j / 8 + (mask bit (i, j) ? 0 : -10000)   (fp32)
 * for query rows i in [row0, Lq) and keys j in [0, Lkv): the reference's attention_probs before dropout (modeling.py:283-295); a
 * fully masked row is the softmax of the unmasked scores (every score is shifted by the same -10000), never zero or NaN.
 *   q: Lq rows per sequence, ld_q elements apart, sequences q_bstride apart (0: Lq * ld_q); head h at columns [64 h, 64 h + 64).
 *      In place in VlpkLayerActs.qkv (ld 3H; decode layouts: ld H).
 *   k: Lkv rows, ld_k apart, sequences k_bstride apart (0: Lkv * ld_k): qkv + H (ld 3H), VlpkLayerActs.kv (ld 2H) or a K/V cache
 *      [B, rows, 2H] (ld 2H, k_bstride = rows * 2H).
 *   mask_bits / mask_rows (1 or Lq) / kv_slots: as for vlpk_attn_core_fwd_wide.  lse: [B, heads, Lq].
 *   p: fp32, [Lq - row0, ld_p] per (sequence, head), heads (Lq - row0) * ld_p floats apart, sequences p_bstride apart (0: heads *
 *      (Lq - row0) * ld_p).  Columns [Lkv, ld_p) are not written.
 * One launch, no allocation, no host synchronisation.  < 0 without launching for: Lq, Lkv or kv_slots outside the attention kernels'
 * range (Lkv <= 512), mask_rows neither 1 nor Lq, row0 outside [0, Lq), ld_p < Lkv, p_bstride below one sequence's block, a NULL
 * pointer, or q / k pointers and strides that are not multiples of 16 bytes (TMA). */
int vlpk_attn_probs(int B, int heads, int Lq, int Lkv, int row0, const void* q, int64_t ld_q, int64_t q_bstride, const void* k, int64_t ld_k,
                    int64_t k_bstride, const uint32_t* mask_bits, int mask_rows, int kv_slots, const float* lse, float* p, int64_t ld_p,
                    int64_t p_bstride, void* stream);

/* Attention core with a per-row self key (forward only, eval: no dropout), for scoring given captions (vlpk_encoder_score_fwd):
 *   ctx_i = softmax([ q_i . k_j / 8 + mask_add(i, j) for j < Lkv ] ++ [ q_i . k_self_i / 8 ]) [ v_0 .. v_{Lkv-1} ; v_self_i ]
 * The self key of query row i is the row k_self + b * q_bstride + i * ld_q (v_self alike: the strides of q), and no mask bit hides
 * it.  lse [B, heads, Lq] is the logsumexp over all Lkv + 1 scores.  q / ctx: Lq rows per sequence, sequences q_bstride / ctx_bstride
 * apart (0: Lq * ld); k / v: Lkv rows, kv_bstride apart (0: Lkv * ld_kv).  mask_bits: [B, Lq, S / 32], one row per query row, with
 * kv_slots as for vlpk_attn_core_fwd_wide, except that Lq need not be <= kv_slots.  Lq, Lkv in [1, 512]; both <= 128: the single-tile
 * kernel, else the KV-tiled one.  < 0 with nothing launched on bad lengths or kv_slots, a NULL pointer, or self rows that are not
 * 16-byte aligned. */
int vlpk_attn_core_self_fwd(int B, int heads, int Lq, int Lkv, const void* q, int64_t ld_q, int64_t q_bstride, const void* k, const void* v,
                            int64_t ld_kv, int64_t kv_bstride, const void* k_self, const void* v_self, const uint32_t* mask_bits, int kv_slots,
                            void* ctx, int64_t ld_ctx, int64_t ctx_bstride, float* lse, void* stream);
/* vlpk_attn_core_self_fwd with the keys of a shared image prefix (the caption matrix, vlpk_encoder_score_group_fwd): B hypotheses in
 * groups of G per image.  Key j < P of hypothesis b is row j of image b / G's prefix [B / G, prefix_rows, ld_prefix] (K at column 0,
 * V at column heads * 64); key P + j, j < Lkv - P, is its text row b * T + j of text [B * T rows, ld_text] (K at column 0, V at column
 * heads * 64; e.g. a pair's word rows in place in a packed qkv: text = qkv + H, ld_text = 3H); then each query row's own key, as for
 * vlpk_attn_core_self_fwd (k_self / v_self with the strides of q).  mask_bits: one sequence per image, [B / G, Lq, S / 32].  The
 * result is bitwise vlpk_attn_core_self_fwd's on each hypothesis' materialised keys [prefix rows | text rows].  < 0 with nothing
 * launched for the refusals of vlpk_attn_core_self_fwd, B % G != 0, P outside [1, prefix_rows], Lkv - P outside [0, T], or text rows
 * that are not 16-byte aligned. */
int vlpk_attn_core_group_self_fwd(int B, int G, int heads, int Lq, int Lkv, int P, const void* q, int64_t ld_q, int64_t q_bstride,
                                  const void* prefix, int prefix_rows, int64_t ld_prefix, const void* text, int T, int64_t ld_text,
                                  const void* k_self, const void* v_self, const uint32_t* mask_bits, int kv_slots, void* ctx, int64_t ld_ctx,
                                  int64_t ctx_bstride, float* lse, void* stream);

/* BertAttention.forward (modeling.py:326-330): QKV projection + attention core + output projection + LN.
 * x_kv == NULL or == x: self-attention over x (training / encoder path).
 * x_kv != x: incremental decode (modeling.py:273-277): keys/values projected from x_kv = cat(history, x), [B*Lkv,H]. */
int vlpk_mha_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const void* x_kv, const uint32_t* mask_bits,
                 int mask_rows, VlpkLayerActs* a, float p_attn, float p_hidden, const VlpkDropout* drop, uint64_t layer_id,
                 void* stream);
/* BertIntermediate + BertOutput (modeling.py:340-343, 353-357): y = LN(dropout(gelu(y1 W1^T+b1) W2^T + b2) + y1). */
int vlpk_ffn_fwd(const VlpkShape* s, const VlpkLayerWeights* w, VlpkLayerActs* a, float p_hidden, const VlpkDropout* drop,
                 uint64_t layer_id, void* stream);
/* BertLayer.forward (modeling.py:367-372) = mha + ffn. */
int vlpk_layer_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const void* x_kv, const uint32_t* mask_bits,
                   int mask_rows, VlpkLayerActs* a, float p_attn, float p_hidden, const VlpkDropout* drop, uint64_t layer_id,
                   void* stream);
/* Backward of BertLayer: dy = gradient of a->y; writes dx (gradient of x); accumulates parameter gradients. */
int vlpk_layer_bwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const uint32_t* mask_bits, int mask_rows,
                   const VlpkLayerActs* a, const void* dy, void* dx, const VlpkLayerGrads* g, const VlpkBwdScratch* ws,
                   float p_attn, float p_hidden, const VlpkDropout* drop, uint64_t layer_id, void* stream);

/* The two halves of vlpk_layer_bwd, for callers that keep BertAttention / BertIntermediate+BertOutput as separate autograd nodes.
 * vlpk_ffn_bwd: dy = gradient of a->y -> dy1 = gradient of a->y1 (may alias dy); accumulates w1,b1,w2,b2,ln2 gradients.
 * vlpk_mha_bwd: dy1 = gradient of a->y1 -> dx = gradient of x (may alias dy1); accumulates wqkv,bqkv,wo,bo,ln1 gradients.
 * vlpk_layer_bwd(dy, dx) == vlpk_ffn_bwd(dy, ws->dy1) followed by vlpk_mha_bwd(ws->dy1, dx). */
int vlpk_ffn_bwd(const VlpkShape* s, const VlpkLayerWeights* w, const VlpkLayerActs* a, const void* dy, void* dy1,
                 const VlpkLayerGrads* g, const VlpkBwdScratch* ws, float p_hidden, const VlpkDropout* drop, uint64_t layer_id,
                 void* stream);
int vlpk_mha_bwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const uint32_t* mask_bits, int mask_rows,
                 const VlpkLayerActs* a, const void* dy1, void* dx, const VlpkLayerGrads* g, const VlpkBwdScratch* ws, float p_attn,
                 float p_hidden, const VlpkDropout* drop, uint64_t layer_id, void* stream);
/* BertAttention.forward with history_states (modeling.py:273-277; BertModelIncr / BertForSeq2SeqDecoder, :856-875, 1189-1253):
 * inference only (no dropout, nothing saved for backward).  x: [B*Lq,H] new rows; x_kv = cat(history, x): [B*Lkv,H]. */
int vlpk_mha_incr_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const void* x_kv, const uint32_t* mask_bits,
                      int mask_rows, VlpkLayerActs* a, uint64_t layer_id, void* stream);
/* BertLayer.forward for incremental decode with a persistent K/V cache (SURVEY.md §8f-2; the reference re-projects K and V of the whole
 * prefix at every step, modeling.py:273-277).  kv_cache [B, cache_rows, 2H] bf16 holds key | value projections of the rows this layer has
 * already seen; `pos` of them are valid.  The Lq new rows x [B*Lq, H] are projected, their K | V appended at rows [pos, pos + Lq), attention
 * runs over rows [0, pos + Lq) (s->Lkv must equal pos + s->Lq), then output projection, LayerNorm and FFN as vlpk_layer_fwd (no dropout).
 * a->qkv receives Q [B*Lq, H]; a->kv [B*Lq, 2H] is scratch for the new rows' K | V.  A later call may overwrite rows (decode keeps only
 * the rows of real tokens: the [MASK] row written at pos + Lq - 1 is overwritten by the next step). */
int vlpk_layer_cached_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, void* kv_cache, int cache_rows, int pos,
                          const uint32_t* mask_bits, int mask_rows, VlpkLayerActs* a, uint64_t layer_id, void* stream);
/* vlpk_layer_cached_fwd for s->B hypotheses in groups of G per image that share one image prefix (several captions per image: beam
 * n-best lists, N samples).  K/V come from two caches instead of one contiguous cache per hypothesis:
 *   prefix [B / G, prefix_rows, 2H] bf16: keys 0 .. P-1 of image b / G (written once, e.g. by vlpk_layer_cached_fwd at B / G rows);
 *   text   [B, T, 2H] bf16: the K | V of the Lq new rows x [B*Lq, H] of hypothesis i go to text[i, pos .. pos + Lq);
 *   slots  [B, T] int32, one table for all layers: key P + j (j < pos) of hypothesis i is the flat text row slots[i * T + j] (a beam
 *          reorder moves table entries, not K/V rows).  Entries outside [0, B * T) are clamped: wrong numbers, never a bad read.
 * Keys P + pos .. P + pos + Lq - 1 are the hypothesis' own new rows; s->Lkv must equal P + pos + Lq (<= 512).  mask_bits: one
 * sequence per image, [B / G, mask_rows, S / 32].  Output, a->qkv / a->kv and the rest as vlpk_layer_cached_fwd: the layer is
 * bitwise what vlpk_layer_cached_fwd computes on each hypothesis' materialised contiguous cache.  < 0 with nothing launched for:
 * B % G != 0, P outside [1, prefix_rows], pos < 0 or pos + Lq > T, Lkv != P + pos + Lq, a bad shape, mask_rows neither 1 nor Lq,
 * a NULL pointer, or x / prefix / text / mask_bits not 16-byte aligned (slots: 4-byte). */
int vlpk_layer_cached_group_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const void* prefix, int prefix_rows, int P,
                                void* text, int T, const int32_t* slots, int G, int pos, const uint32_t* mask_bits, int mask_rows,
                                VlpkLayerActs* a, uint64_t layer_id, void* stream);
/* Host-only: bytes the caller must provide for a shape.  out3 = { all VlpkLayerActs buffers of ONE layer (without the optional
 * drop_attn keep-bytes: B*heads*Lq*S/8),
 * all VlpkBwdScratch buffers (shared by the layers), the fp32 VlpkLayerGrads accumulators of ONE layer }. */
int vlpk_workspace_bytes(const VlpkShape* s, size_t* out3);

/* BertEncoder.forward (modeling.py:382-402): n_layers x BertLayer in one host call.  acts[i].y is layer i's output. */
int vlpk_encoder_fwd(const VlpkShape* s, int n_layers, const VlpkLayerWeights* w, const void* x, const uint32_t* mask_bits,
                     int mask_rows, VlpkLayerActs* acts, float p_attn, float p_hidden, const VlpkDropout* drop, void* stream);
/* Teacher-forced scoring pass of the seq2seq decoder (forward only, eval, no dropout): n_layers x BertLayer over B sequences of
 * S + T rows, x [B, S + T, H].  Rows [0, S) are shared rows ([CLS] regions [SEP] and the caption words but the last); rows [S, S + T)
 * are query rows ([MASK]).  Per layer: QKV projection, output projection, both LayerNorms and the FFN over all S + T rows; attention
 * in two launches: shared rows against the shared rows under shared_bits [B, S, S' / 32], then query rows against the shared rows
 * under query_bits [B, T, S' / 32] plus each query row's own key (vlpk_attn_core_self_fwd); S' = 128 * ceil(S / 128).
 *   s: B, Lq = Lkv = S, H, heads, I, kv_slots (as for an S-row encoder);  T in [1, 512].
 *   acts[i]: layer i's buffers sized for B * (S + T) rows (vlpk_encoder_score_workspace_bytes; kv and drop_attn unused); lse holds
 *   [B, heads, S] of the shared rows, then [B, heads, T] of the query rows.  Layer i reads acts[i - 1].y, so two buffers used in turn
 *   serve any depth.
 * One host call, no allocation, no host synchronisation.  < 0 with nothing launched for: a bad shape, Lq != Lkv, T outside [1, 512],
 * H not a multiple of 128, a NULL pointer, a layer's output aliasing its input, or x / mask bits / qkv / ctx not 16-byte aligned. */
int vlpk_encoder_score_fwd(const VlpkShape* s, int T, int n_layers, const VlpkLayerWeights* w, const void* x, const uint32_t* shared_bits,
                           const uint32_t* query_bits, VlpkLayerActs* acts, void* stream);
/* Host-only: bytes of one layer's VlpkLayerActs buffers for vlpk_encoder_score_fwd (the layout of vlpk_workspace_bytes' out3[0] over
 * B * (S + T) rows, without kv).  A separate entry point because a VlpkShape cannot describe the scoring stack: its rows per sequence
 * (S + T, up to 1023) exceed the 512 vlpk_workspace_bytes' shape check allows, and the attention's key count S differs from them. */
int vlpk_encoder_score_workspace_bytes(const VlpkShape* s, int T, size_t* out1);
/* The caption matrix: the scoring pass of vlpk_encoder_score_fwd for s->B (image, caption) pairs, G captions per image, against
 * per-layer K/V caches of the images' prefixes, so that the P prefix rows run once per image instead of once per pair.  A pair has
 * 2T - 1 rows, x [B, 2T - 1, H]: rows [0, T - 1) are its words c_0 .. c_{T-2}, rows [T - 1, 2T - 1) its T query rows ([MASK]).
 *   s: B pairs (pair i of image i / G), Lq = Lkv = S = P + T - 1 (a pair's keys), H, heads, I, kv_slots (as for an S-row encoder).
 *   prefix[l]: layer l's K | V of the prefix rows, [B / G, prefix_rows, 2H] bf16 (e.g. written by vlpk_layer_cached_fwd at pos 0).
 *   word_bits [B / G, T - 1, S' / 32] (NULL allowed when T = 1) and query_bits [B / G, T, S' / 32]: one sequence per image, shared
 *   by its G pairs; S' = 128 * ceil(S / 128).  Key j < P is prefix row j, key P + j the pair's word j.
 * Per layer: the packed QKV projection over all pair rows; the word rows against [prefix | words] (vlpk_layer_cached_group_fwd's
 * kernel, pos 0); the query rows against [prefix | words] plus each its own key (vlpk_attn_core_group_self_fwd); the output
 * projection, both LayerNorms and the FFN over all rows.  Word K | V are read in place from the layer's qkv, nothing is copied.
 *   acts[i]: layer i's buffers for B * (2T - 1) rows (vlpk_encoder_score_group_workspace_bytes; kv and drop_attn unused); lse holds
 *   [B, heads, T - 1] of the word rows, then [B, heads, T] of the query rows.  Layer i reads acts[i - 1].y: two buffers used in turn
 *   serve any depth.
 * One host call, no allocation, no host synchronisation.  < 0 with nothing launched for: a bad shape, Lq != Lkv, T outside [1, 512],
 * P outside [1, prefix_rows] or P + T - 1 != S, B % G != 0, H not a multiple of 128, a NULL pointer, a layer's output aliasing its
 * input, or x / mask bits / prefix caches / acts misaligned. */
int vlpk_encoder_score_group_fwd(const VlpkShape* s, int T, int G, int P, int n_layers, const VlpkLayerWeights* w, const void* x,
                                 const void* const* prefix, int prefix_rows, const uint32_t* word_bits, const uint32_t* query_bits,
                                 VlpkLayerActs* acts, void* stream);
/* Host-only: bytes of one layer's VlpkLayerActs buffers for vlpk_encoder_score_group_fwd (vlpk_encoder_score_workspace_bytes' layout
 * over B * (2T - 1) rows).  s as for vlpk_encoder_score_group_fwd; T in [1, S]. */
int vlpk_encoder_score_group_workspace_bytes(const VlpkShape* s, int T, size_t* out1);
/* Backward of the stack.  dys[i] (may be NULL) is the gradient flowing into layer i's output from outside the stack
 * (output_all_encoded_layers consumers); dys[n_layers-1] is normally the only non-NULL entry.  dx0 receives d/dx. */
int vlpk_encoder_bwd(const VlpkShape* s, int n_layers, const VlpkLayerWeights* w, const void* x, const uint32_t* mask_bits,
                     int mask_rows, const VlpkLayerActs* acts, const void* const* dys, void* dx0, const VlpkLayerGrads* grads,
                     const VlpkBwdScratch* ws, float p_attn, float p_hidden, const VlpkDropout* drop, void* stream);

/* ---- masked-LM head tail (SURVEY.md §8f-3) -------------------------------------------------------------------------------
 * cls.predictions.decoder (weight tied to the word embeddings [V,H], output-only bias; modeling.py:465-482) + the per-position
 * cross-entropy of crit_mask_lm (modeling.py:1108-1109), without fp32 logits.  Vp = V rounded up to a multiple of 8.
 *   h [R,H] bf16 (output of cls.predictions.transform), w [V,H] bf16 read in place, bias_pad [Vp] bf16 (zero padded),
 *   labels [R] int64 (outside [0,V): ignored position, loss 0 / no gradient, like ignore_index),
 *   logits [R,Vp] bf16 (out), lse [R] fp32 (out), loss [R] fp32 (out). */
int vlpk_decoder_ce_fwd(int R, int V, int H, const void* h, const void* w, const void* bias_pad, const int64_t* labels, void* logits,
                        float* lse, float* loss, void* stream);
/* Backward: dloss [R] fp32 -> dlogits [R,Vp] bf16 (scratch/out), dh [R,H] fp32 (ZEROED by the caller; split-K reduce-add target),
 * dw [V,H] bf16 (overwritten), dbias [Vp] fp32 (ZEROED by the caller). */
int vlpk_decoder_ce_bwd(int R, int V, int H, const void* h, const void* w, const int64_t* labels, const void* logits, const float* lse,
                        const float* dloss, void* dlogits, float* dh, void* dw, float* dbias, void* stream);
/* The same pair with the label-smoothed loss of LabelSmoothingLoss (loss.py:12-48, crit_mask_lm_smoothed, modeling.py:995-999,
 * 1104-1106) in place of the cross-entropy; arguments as above plus eps in (0, 1] (V >= 3, otherwise rc < 0 and nothing runs).
 * Target of a row with label t: q_0 = 0, q_t = 1 - eps, eps / (V - 2) elsewhere.  Label 0 (the reference's ignore index) and labels
 * outside [0,V) are ignored positions: loss 0, dlogits row 0.  loss = KL(q || softmax(logits)), dlogits = (softmax - q) * dloss. */
int vlpk_decoder_ce_ls_fwd(int R, int V, int H, float eps, const void* h, const void* w, const void* bias_pad, const int64_t* labels,
                           void* logits, float* lse, float* loss, void* stream);
int vlpk_decoder_ce_ls_bwd(int R, int V, int H, float eps, const void* h, const void* w, const int64_t* labels, const void* logits,
                           const float* lse, const float* dloss, void* dlogits, float* dh, void* dw, float* dbias, void* stream);

/* ---- optimizer (SURVEY.md §8f-1) ----------------------------------------------------------------------------------------
 * One parameter tensor of a BertAdam step.  64 bytes; the table is read by the kernels from DEVICE memory. */
typedef struct VlpkAdamTensor {
  void* param;         /* model parameter, updated in place; bf16 or fp32 */
  const void* grad;    /* its gradient; bf16 or fp32; NOT modified (the reference's clip rescales p.grad in place) */
  float* master;       /* fp32 master copy, required when param is bf16 (param = bf16(master)); NULL when param is fp32 */
  float* m;            /* fp32 first moment  (state['next_m']) */
  float* v;            /* fp32 second moment (state['next_v']) */
  int64_t n;           /* elements (> 0) */
  float weight_decay;  /* this tensor's group['weight_decay'] (0 for bias / LayerNorm.*, run_img2txt_dist.py:394-401) */
  int32_t param_dtype; /* VLPK_BF16 / VLPK_F32 */
  int32_t grad_dtype;
  int32_t reserved;
} VlpkAdamTensor;

/* Elements of one tensor per work item: chunk_prefix[t+1] - chunk_prefix[t] == ceil(tensors[t].n / vlpk_bertadam_chunk()). */
int vlpk_bertadam_chunk(void);
/* BertAdam.step (pytorch_pretrained_bert/optimization.py:112-182) for n_tensors parameters at once:
 *   per tensor  g *= min(1, max_grad_norm / (||g||_2 + 1e-6))   (clip_grad_norm_ of that single tensor, :145-146; skipped if <= 0)
 *               m = b1 m + (1-b1) g ;  v = b2 v + (1-b2) g g ;  u = m / (sqrt(v) + eps) + weight_decay p ;  p -= lr_scheduled u
 * No bias correction (:176-179).  lr_scheduled = lr * schedule(step / t_total, warmup) is evaluated by the caller (:165-170).
 * tensors_dev / chunk_prefix_dev: device copies of tensors_host / chunk_prefix_host ([n_tensors] / [n_tensors+1] exclusive prefix
 * of chunk counts); the host copies are used for validation only.  sqnorm_dev: [n_tensors] fp32 scratch.  Two launches, no host
 * synchronisation. */
int vlpk_bertadam_step(const VlpkAdamTensor* tensors_host, const VlpkAdamTensor* tensors_dev, const int32_t* chunk_prefix_host,
                       const int32_t* chunk_prefix_dev, int n_tensors, float* sqnorm_dev, double lr_scheduled, double b1, double b2,
                       double eps, double max_grad_norm, void* stream);

/* Launch accounting.  vlpk_launch_count: kernels launched by this library in this process.  With profiling enabled every
 * launch is bracketed by CUDA events on its stream; vlpk_profile_get sums device time (ms), algorithmic work (FLOPs for the
 * tensor-core kernels, HBM bytes for the bandwidth kernels) and launches of one kernel family since the last reset.
 * Families: 0 gemm fwd, 1 gemm dgrad, 2 gemm wgrad, 3 attention fwd, 4 attention bwd, 5 LN fwd, 6 LN bwd, 7 embed, 8 misc. */
void vlpk_profile_enable(int on);
void vlpk_profile_reset(void);
int vlpk_profile_get(int cat, double* ms, double* work, int64_t* launches);
int64_t vlpk_launch_count(void);

/* Beam search: duplicate-n-gram blocking (the reference's forbid_duplicate_ngrams / get_dup_ngram_candidates, modeling.py:1375-1428)
 * for frame f >= 1 of a beam search over rows = B*K hypotheses (row i = b*K + k).  One launch:
 *   hist_out[i, :f-1] = hist_in[b*K + ptr[i], :f-1];  hist_out[i, f-1] = wid[i]
 *     hist_*: int32 [rows, T_cap] (two different buffers, used in turn); ptr / wid: int64 [rows] back pointers and word ids of
 *     frame f-1.  At f = 1 hist_in and ptr are not read (may be NULL).
 *   if f >= n: seq = hist_out[i, :f]; tail = seq[-(n-1):] (all of seq when n = 1); if no tail word is in ignore[0:n_ignore], then
 *     for every s <= f-n with seq[s:s+n-1] == tail the word w = seq[s+n-1] (unless ignored, and only if 0 <= w < V) is blocked:
 *     logp[i*ld + w] += -10000.0f, once per distinct w.  Rows without candidates and columns >= V are not touched.
 *     logp: fp32 [rows, ld], frame f's log-probabilities, before the min_len [EOS] fill.  ignore: int32 device array, NULL if
 *     n_ignore == 0.  Deterministic (no floating-point atomics).
 * Returns < 0 without launching for n < 1, f < 1, f > T_cap, ld < V, hist_in == hist_out, rows not a multiple of K, a NULL
 * pointer that is needed, or (T_cap + V/32) * 4 bytes above 48 KB of shared memory. */
int vlpk_beam_ngram_block(int rows, int K, int f, int T_cap, int n, const int32_t* hist_in, int32_t* hist_out, const int64_t* ptr,
                          const int64_t* wid, const int32_t* ignore, int n_ignore, float* logp, int64_t ld, int V, void* stream);

/* Top-k / top-p sampling of decode frame f (0 <= f < T_cap) over rows sequences, one launch per frame, no host synchronisation:
 *   x[v] = logits[row*ld + v] + bias[v], rounded to the logits' dtype (fp32 = 0: bf16, 1: fp32; bias may be NULL); then, as beam
 *     search does, -10000 is added at the words the duplicate-n-gram rule of vlpk_beam_ngram_block blocks for the row's history
 *     seq[row, :f] (n > 0 and f >= n; ignore / n_ignore as there), and x[eos_id] = -10000 if block_eos (frames below min_len).
 *   Words are ranked by (x descending, index ascending).  mode 0 (top-k, 1 <= topk <= 64) keeps the first topk; mode 1 (top-p,
 *     0 < topp <= 1) keeps the shortest prefix whose probability reaches topp (at least the first argmax).  One draw from the kept
 *     words, renormalised, with a uniform from Philox keyed by (seed; f, row): reproducible for a seed whatever the batch.
 *   seq: int64 [rows, T_cap] receives the word at [row, f]; score: fp32 [rows, T_cap] (or NULL) its log-probability under the
 *     full softmax of x.  finished: int32 [rows]; a finished row writes pad_id (score 0); a row that draws eos_id is marked
 *     finished and decrements live[0] (the host may poll live[0] == 0 to stop a decode early).
 * Returns < 0 without launching for a mode, topk or topp outside its range, ld < V, V < 1, f outside [0, T_cap), a NULL pointer
 * that is needed, or (V + V/32 + T_cap) * 4 bytes above 200 KB of shared memory. */
int vlpk_sample_tokens(int rows, int V, const void* logits, int64_t ld, const void* bias, int fp32, int mode, int topk, float topp,
                       uint64_t seed, int f, int64_t* seq, int T_cap, float* score, int32_t* finished, int32_t* live, int eos_id, int pad_id,
                       int block_eos, int n, const int32_t* ignore, int n_ignore, void* stream);

/* Diverse beam search (Vijayakumar et al., AAAI 2018): the selection of frame f (0 <= f < T_cap) for B images of K beams in G groups
 * of Kg = K / G, with a Hamming penalty, one call per frame (two launches), no host synchronisation.  Rows are b (f = 0) or b*K + k.
 *   logp[i, w]  x = logits[i*ld + w] + bias[w], rounded to the logits' dtype (fp32 = 0: bf16, 1: fp32; bias may be NULL);
 *     logp = x - logsumexp(x) in fp32; then, as beam search does, -10000 is added at the words the duplicate-n-gram rule of
 *     vlpk_beam_ngram_block blocks (n > 0, f >= n; the history carry hist_out[i] = hist_in[b*K + prev_ptr[i]] ‖ prev_wid[i] runs at
 *     every f >= 1 with n > 0), and logp[eos_id] = -10000 if block_eos.
 *   cand(i, w)  logp at f = 0; logp + prev_eos[i] * -10000 + prev_score[i] after (frame f-1's traces, [B, K]).
 *   groups      g = 0 .. G-1 in turn: group g's parents are beams [g*Kg, (g+1)*Kg) (row b at f = 0); it keeps the Kg (parent, word)
 *     pairs with the largest cand - diversity_penalty * cnt(w), cnt(w) = beams of groups < g that chose w in this frame; ties go
 *     to the lower parent, then the lower word.  Its r-th pair becomes beam g*Kg + r.
 *   traces      wid / ptr int64 [B, K] (ptr a beam index in [0, K), 0 at f = 0), score fp32 [B, K] the unpenalised cand, eos fp32
 *     [B, K] (wid == eos_id).  top_w int32 / top_lp fp32 [rows, K] are scratch (each row's top K words).
 * Bitwise reproducible.  Returns < 0 without launching for K outside [1, 64], G not dividing K, V < K, ld < V, a penalty that is
 * negative or not finite, f outside [0, T_cap), fp32 not 0 / 1, a NULL pointer that is needed, hist_in == hist_out, or
 * (V + V/32 + T_cap) * 4 bytes above 200 KB of shared memory. */
int vlpk_diverse_beam_step(int B, int K, int G, int f, int V, const void* logits, int64_t ld, const void* bias, int fp32, float diversity_penalty,
                           int eos_id, int block_eos, int T_cap, int n, const int32_t* hist_in, int32_t* hist_out, const int32_t* ignore,
                           int n_ignore, const int64_t* prev_wid, const int64_t* prev_ptr, const float* prev_score, const float* prev_eos,
                           int32_t* top_w, float* top_lp, int64_t* wid, int64_t* ptr, float* score, float* eos, void* stream);

/* Constrained beam search (Anderson et al., EMNLP 2017): the selection of frame f (0 <= f < T_cap) for B images whose captions must
 * contain C constraints, one call per frame (two launches), no host synchronisation.
 *   constraints  cons int64 [B, C, A, P], 0-padded: constraint j of image b is the disjunction of its alternatives, each a run of
 *     1 .. P word ids (the leading non-zero entries; an alternative whose first entry is 0 is absent).  A constraint with no
 *     alternative is satisfied from the start.
 *   states       a hypothesis' state s is the set of constraints met so far (bit j: an alternative of j occurred as a contiguous run
 *     of its generated words).  S = 2^C states of K beams each: image b's slots are [0, S*K), slot s*K + k is beam k of state s.
 *     Rows are b (f = 0, in the root state: the set of empty constraints) or b*S*K + slot.
 *   logp[i, w]   as vlpk_diverse_beam_step: x = logits + bias rounded to the logits' dtype (fp32 = 0: bf16, 1: fp32), logp = x -
 *     logsumexp(x) in fp32, -10000 added at the words the duplicate-n-gram rule of vlpk_beam_ngram_block blocks (n > 0, f >= n),
 *     logp[eos_id] = -10000 if block_eos.  The history carry hist_out[i] = hist_in[b*S*K + prev_ptr[i]] ‖ prev_wid[i] runs at every
 *     f >= 1, whatever n.
 *   cand(i, w)   logp at f = 0; logp + prev_eos[i] * -10000 + prev_score[i] after (frame f-1's traces, [B, S*K]).
 *   dest(i, w)   s_i ∪ {j : w completes an alternative a of j}: a[-1] == w and the row's last len(a) - 1 words equal a[:-1].
 *   selection    state s' keeps the K (row, word) pairs with dest == s' and the largest finite cand, ties to the lower parent slot, then
 *     the lower word; its r-th pair becomes slot s'*K + r.  Slots it cannot fill are empty: word 0, pointer 0, score -inf, eos 0.
 *   traces       wid / ptr int64 [B, S*K] (ptr a slot in [0, S*K), 0 at f = 0), score fp32 [B, S*K] the cand, eos fp32 [B, S*K]
 *     (wid == eos_id).  top_w int32 / top_lp fp32 [rows, K + C*A] and top_dest int32 [rows, C*A] are scratch: each row's top K
 *     words that keep it in its state, then its completing words and their destinations.
 * Limits: 1 <= C <= 4, 1 <= A <= 4, 1 <= P <= 8, 1 <= K <= 64, S*K <= 256 (so K <= 16 at C = 4 and K <= 64 at C <= 2), V >= K + C*A.
 * Bitwise reproducible.  Returns < 0 without launching for a value outside these limits, ld < V, f outside [0, T_cap), fp32 not 0 / 1,
 * a NULL pointer that is needed, hist_in == hist_out, or (V + V/32 + T_cap) * 4 bytes above 200 KB of shared memory. */
typedef struct VlpkConstrainedBeamArgs {
  int32_t B, K, C, A, P;             /* images, beams per state, constraints, alternatives per constraint, words per alternative */
  int32_t f, V;                      /* frame; vocabulary */
  const void* logits;                /* [rows, ld] bf16 or fp32 decoder outputs, without the bias */
  int64_t ld;
  const void* bias;                  /* [V] same dtype, or NULL */
  int32_t fp32, eos_id, block_eos;
  int32_t T_cap, n;                  /* history width (frames); duplicate-n-gram size, 0 = off */
  const int32_t* hist_in;            /* [B*S*K, T_cap] frame f-1's histories (read at f >= 2) */
  int32_t* hist_out;                 /* [B*S*K, T_cap] frame f's histories (f words, written at f >= 1) */
  const int32_t* ignore;             /* [n_ignore] word ids exempt from n-gram blocking */
  int32_t n_ignore;
  const int64_t* cons;               /* [B, C, A, P] */
  const int64_t* prev_wid;           /* [B, S*K] frame f-1's traces (f >= 1; prev_ptr at f >= 2) */
  const int64_t* prev_ptr;
  const float* prev_score;
  const float* prev_eos;
  int32_t* top_w;                    /* [rows, K + C*A] scratch */
  float* top_lp;                     /* [rows, K + C*A] scratch */
  int32_t* top_dest;                 /* [rows, C*A] scratch */
  int64_t* wid;                      /* [B, S*K] frame f's traces */
  int64_t* ptr;
  float* score;
  float* eos;
} VlpkConstrainedBeamArgs;
int vlpk_constrained_beam_step(const VlpkConstrainedBeamArgs* args, void* stream);

/* utilities */
int vlpk_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream);
int vlpk_colsum(const void* x, int64_t ld, int64_t M, int N, float* out, void* stream);
/* Test support: out[i] = 1 if element i of dropout site `site` is kept under `drop` (p, seed), else 0 — the decision every fused
 * kernel takes through the same counter-based Philox function.  Element numbering per site: LayerNorm / embedding / Linear+ReLU
 * sites: row * width + column; attention site: ((b * heads + h) * Lq + query) * S + key.  Sites: layer * 8 + {0 attention
 * probabilities, 1 attention-output dropout, 2 FFN-output dropout}; 1<<20 embeddings; (1<<21)+{1 vis_embed, 2 vis_pe_embed}.
 * (attention: S key slots per query row, see VlpkShape; 128 for Lkv <= 128.)
 * n must be a multiple of 8. */
int vlpk_debug_dropout_mask(const VlpkDropout* drop, uint64_t site, int64_t n, unsigned char* out, void* stream);
int vlpk_add_bf16(void* dst, const void* a, const void* b, int64_t n, void* stream);

/* Raw GEMM building block (exposed for tests / bring-up).  D[M,N] = sum_k A[m,k] B[n,k].
 * a_mn / b_mn: operand stored with the M (resp. N) index contiguous instead of k.  epi: see csrc/gemm.cuh. */
int vlpk_gemm(int M, int N, int K, int a_mn, const void* A, int64_t lda, int b_mn, const void* B, int64_t ldb, const void* bias,
              void* D0, int64_t ldd0, void* D1, int64_t ldd1, const void* aux, int64_t ld_aux, int epi, int splits, int bn,
              void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VLPK_H_ */
