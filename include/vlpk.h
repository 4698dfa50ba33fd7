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

typedef struct VlpkShape {
  int32_t B;     /* sequences */
  int32_t Lq;    /* query rows per sequence  (<= 128) */
  int32_t Lkv;   /* key/value rows per sequence (<= 128); == Lq except incremental decode */
  int32_t H;     /* hidden size (multiple of 64) */
  int32_t heads; /* H / 64 */
  int32_t I;     /* intermediate size */
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
   * element (byte i = elements 8i..8i+7, numbering as in vlpk_debug_dropout_mask; 128 key slots per query row).  Written by the
   * forward attention kernel, read by the backward one. */
  unsigned char* drop_attn; /* [B*heads*Lq*16] */
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
/* host-only: the (tile N, split-K) the cost model picks for a GEMM; out2 = {bn, splits}.  No GPU needed. */
int vlpk_debug_plan_gemm(int M, int N, int K, int a_mn, int b_mn, int nseg, int seg_rows, int epi, int bn, int splits, int* out2);
/* A-B testing only: switch a host-side scheduling choice at run time.  "wgrad_stream" (default 1, env VLPK_WGRAD_STREAM=0 turns it
 * off): the weight-gradient GEMM of each Linear's backward runs on a side stream behind its dgrad.  < 0: unknown name. */
int vlpk_debug_set_option(const char* name, int value);

/* get_extended_attention_mask (modeling.py:807-833) -> per-row 128-bit "attend" bitmask.
 * mask: [B, rows, kv] with element strides (stride_b, stride_r, 1); rows may be 1 (2-D mask). out: [B, rows, 4] u32. */
int vlpk_mask_pack(const void* mask, int dtype, int mode, int B, int rows, int kv, int64_t stride_b, int64_t stride_r,
                   uint32_t* out, void* stream);

/* Input staging (SURVEY.md §8f-4): the loader's self-attention mask (vlp/seq2seq_loader.py:291-301) synthesised on the device from
 * three integers per sample instead of shipping [B,L,L] int64: len_a region tokens (same for the batch), len_b[b] text tokens,
 * mode[b] (0 = bidirectional, 1 = seq2seq).  Output: the packed bitmask vlpk_mask_pack would produce from the loader's matrix. */
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
/* Data parallelism: add explicit looked-up rows (ids[n], optional pos[n], rows[n,H] bf16 — typically all ranks' rows after an
 * all-gather), scaled by `scale`, INTO an existing bf16 word-table gradient d_word [V,H] and the fp32 position gradient d_pos [P,H]
 * (NULL: skip).  scratch [V,H] fp32 and owner [V] int32 are uninitialised work buffers.  vlpk_embed_tables_bwd with d_word = scratch =
 * d_pos = NULL computes the token-type gradient only. */
int vlpk_table_rows_add(int64_t n, const int64_t* ids, const int64_t* pos, const void* rows, int H, int V, int P, float scale, void* d_word,
                        float* scratch, int32_t* owner, float* d_pos, void* stream);

/* y = LayerNorm(dropout(t) + res) (BertSelfOutput / BertOutput tail, modeling.py:315-316, 355-356; eps 1e-5). */
int vlpk_ln_res_drop_fwd(int64_t M, int H, const void* t, const void* res, const void* gamma, const void* beta, void* y,
                         float* stats, const VlpkDropout* drop, uint64_t site, void* stream);
int vlpk_ln_res_drop_bwd(int64_t M, int H, const void* t, const void* res, const void* gamma, const float* stats, const void* dy,
                         void* dz, void* dt, float* dgamma, float* dbeta, float* dbias, const VlpkDropout* drop, uint64_t site,
                         void* stream);

/* softmax(QK^T/8 + mask) V per (sequence, head) — BertSelfAttention core (modeling.py:279-302). */
int vlpk_attn_core_fwd(int B, int heads, int Lq, int Lkv, const void* q, int64_t ld_q, const void* k, const void* v, int64_t ld_kv,
                       const uint32_t* mask_bits, int mask_rows, void* ctx, int64_t ld_ctx, float* lse, const VlpkDropout* drop,
                       uint64_t site, void* stream);
int vlpk_attn_core_bwd(int B, int heads, int L, const void* q, const void* k, const void* v, int64_t ld_qkv, const uint32_t* mask_bits,
                       int mask_rows, const void* ctx, const void* dctx, int64_t ld_ctx, const float* lse, void* dq, void* dk,
                       void* dv, int64_t ld_dqkv, const VlpkDropout* drop, uint64_t site, void* stream);

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
/* Host-only: bytes the caller must provide for a shape.  out3 = { all VlpkLayerActs buffers of ONE layer (without the optional
 * drop_attn keep-bytes: B*heads*Lq*16),
 * all VlpkBwdScratch buffers (shared by the layers), the fp32 VlpkLayerGrads accumulators of ONE layer }. */
int vlpk_workspace_bytes(const VlpkShape* s, size_t* out3);

/* BertEncoder.forward (modeling.py:382-402): n_layers x BertLayer in one host call.  acts[i].y is layer i's output. */
int vlpk_encoder_fwd(const VlpkShape* s, int n_layers, const VlpkLayerWeights* w, const void* x, const uint32_t* mask_bits,
                     int mask_rows, VlpkLayerActs* acts, float p_attn, float p_hidden, const VlpkDropout* drop, void* stream);
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

/* utilities */
int vlpk_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream);
int vlpk_colsum(const void* x, int64_t ld, int64_t M, int N, float* out, void* stream);
/* Test support: out[i] = 1 if element i of dropout site `site` is kept under `drop` (p, seed), else 0 — the decision every fused
 * kernel takes through the same counter-based Philox function.  Element numbering per site: LayerNorm / embedding / Linear+ReLU
 * sites: row * width + column; attention site: ((b * heads + h) * Lq + query) * 128 + key.  Sites: layer * 8 + {0 attention
 * probabilities, 1 attention-output dropout, 2 FFN-output dropout}; 1<<20 embeddings; (1<<21)+{1 vis_embed, 2 vis_pe_embed}.
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
