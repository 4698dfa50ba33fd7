// vlp_b200 — extern "C" entry points of libvlpk.so (declared in include/vlpk.h).
//
// Host-side orchestration only: every function validates arguments, builds launch descriptors and
// enqueues kernels from gemm.cu / attn.cu / rowops.cu on the caller's stream.  The composite calls
// (mha / ffn / layer / encoder) exist so that one BertEncoder forward or backward is a single
// host call — the reference spends ~60 Python module calls per layer (SURVEY.md §8a a11).
#include "../../include/vlpk.h"

#include <cstdlib>
#include <cstring>

#include "attn.cuh"
#include "decode.cuh"
#include "gemm.cuh"
#include "head.cuh"
#include "host.cuh"
#include "optim.cuh"
#include "rowops.cuh"
#include "tables.cuh"

using namespace vlpk;
typedef __nv_bfloat16 bf16;

namespace {

inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Dropout sites inside one BertLayer.  Distinct (layer, site) pairs give independent Philox streams.
enum { SITE_ATTN = 0, SITE_HID1 = 1, SITE_HID2 = 2 };
inline uint64_t site_of(uint64_t layer_id, int site) { return layer_id * 8 + site; }

inline DropoutCfg mk_drop(const VlpkDropout* d, float p, uint64_t site) {
  if (d == nullptr || p <= 0.f) return make_dropout(0.f, 0, site);
  return make_dropout(p, d->seed, site, reinterpret_cast<const unsigned long long*>(d->seed_dev));
}

int check_shape(const VlpkShape* s) {
  VLPK_CHECK_ARG(s != nullptr, "null shape");
  if (s->kv_slots == 0) {
    VLPK_CHECK_ARG(s->B > 0 && s->Lq > 0 && s->Lkv > 0 && s->Lq <= 128 && s->Lkv <= 128,
                   "shape: B=%d Lq=%d Lkv=%d (sequence length must be in [1,128])", s->B, s->Lq, s->Lkv);
  } else {
    VLPK_CHECK_ARG(s->B > 0 && s->Lq > 0 && s->Lkv > 0 && s->Lkv <= 512 && s->kv_slots == (s->Lkv + 127) / 128 * 128 && s->Lq <= s->kv_slots,
                   "shape: B=%d Lq=%d Lkv=%d kv_slots=%d (sequence length must be in [1,512], kv_slots = 128 * ceil(Lkv / 128) >= Lq)",
                   s->B, s->Lq, s->Lkv, s->kv_slots);
  }
  VLPK_CHECK_ARG(s->H > 0 && s->H % 64 == 0 && s->heads * 64 == s->H, "shape: H=%d heads=%d (head_dim must be 64)", s->H,
                 s->heads);
  VLPK_CHECK_ARG(s->I > 0 && s->I % 64 == 0, "shape: I=%d must be a multiple of 64", s->I);
  return 0;
}

// y[M,N] = x[M,K] w[N,K]^T + b   (single weight)
int fwd_linear(int M, int N, int K, const void* x, int64_t ldx, const void* w, int64_t ldw, const void* b, void* y, int64_t ldy,
               int epi, void* y1, int64_t ldy1, const DropoutCfg& drop, cudaStream_t st) {
  GemmDesc g;
  g.M = M; g.N = N; g.K = K;
  g.A = x; g.lda = ldx;
  g.B[0] = w; g.ldb = ldw; g.nseg = 1;
  g.bias[0] = static_cast<const bf16*>(b);
  g.D0 = y; g.ldd0 = ldy; g.D1 = y1; g.ldd1 = ldy1;
  g.epi = epi;
  g.drop = drop;
  return launch_gemm(g, st);
}

// dx[M,K] = dy[M,N] w[N,K] (+ epilogue with aux)
int dgrad_linear(int M, int N, int K, const void* dy, int64_t lddy, const void* w, int64_t ldw, void* dx, int64_t lddx, int epi,
                 const void* aux, int64_t ld_aux, cudaStream_t st, float* colsum = nullptr) {
  GemmDesc g;
  g.M = M; g.N = K; g.K = N;  // contraction over the Linear's output features
  g.A = dy; g.lda = lddy;
  g.b_mn = true; g.B[0] = w; g.ldb = ldw; g.nseg = 1;
  g.D0 = dx; g.ldd0 = lddx;
  g.epi = epi;
  g.aux = static_cast<const bf16*>(aux); g.ld_aux = ld_aux;
  g.colsum = colsum;
  return launch_gemm(g, st);
}

// dw[N,K] (fp32, +=) = dy[M,N]^T x[M,K]
int wgrad_linear(int M, int N, int K, const void* dy, int64_t lddy, const void* x, int64_t ldx, float* dw, int64_t lddw,
                 cudaStream_t st) {
  GemmDesc g;
  g.M = N; g.N = K; g.K = M;  // contraction over tokens
  g.a_mn = true; g.A = dy; g.lda = lddy;
  g.b_mn = true; g.B[0] = x; g.ldb = ldx; g.nseg = 1;
  g.D0 = dw; g.ldd0 = lddw;
  g.epi = EPI_REDUCE_F32;
  g.splits = 0;  // chosen together with the tile shape by launch_gemm's cost model
  if (deterministic()) return launch_gemm_split_slices(g, SCRATCH_WGRAD, st);
  return launch_gemm(g, st);
}

// ---- side stream ------------------------------------------------------------------------------------------------------------
// One process drives one GPU, so a single side stream per process is enough; fork / join with events (capturable in a CUDA graph).
// Backward: the weight-gradient GEMM of each Linear runs behind its dgrad (VLPK_WGRAD_STREAM=0 / option "wgrad_stream" disables):
// inside one layer the two only share their INPUT; both are persistent one-CTA-per-SM kernels, so the wgrad's CTAs start on the SMs
// the dgrad's partial last wave leaves idle (372 tiles on 132 SMs for the N = 768 shapes) instead of after its last tile.
struct SideStream {
  cudaStream_t stream = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr;
  bool pending = false;
  bool failed = false;
};

int g_wgrad_stream = -1;  // -1: take VLPK_WGRAD_STREAM from the environment on first use, default on

SideStream* side_stream() {
  static SideStream side;
  if (side.stream == nullptr && !side.failed) {
    if (cudaStreamCreateWithFlags(&side.stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&side.fork, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreateWithFlags(&side.join, cudaEventDisableTiming) != cudaSuccess) {
      side.stream = nullptr;
      side.failed = true;
    }
  }
  return side.stream != nullptr ? &side : nullptr;
}

SideStream* wgrad_side() {
  if (g_wgrad_stream < 0) {
    const char* e = getenv("VLPK_WGRAD_STREAM");
    g_wgrad_stream = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  return g_wgrad_stream == 1 ? side_stream() : nullptr;
}

// One Linear's backward: weight gradient + input gradient, which only share their inputs.  Default: wgrad then dgrad on `main`
// With the side stream: dgrad first on `main` (it is on the critical path and takes the
// SMs), then the wgrad on the side stream, whose CTAs fill the SMs the dgrad's partial last wave leaves idle and overlap whatever
// `main` issues next.  wgrad_join(main) must follow before the wgrad's inputs are overwritten.
template <class WgradFn, class DgradFn>
int linear_bwd_pair(cudaStream_t main, WgradFn&& wgrad, DgradFn&& dgrad) {
  SideStream* sd = wgrad_side();
  if (sd == nullptr) {
    VLPK_TRY(wgrad(main));
    return dgrad(main);
  }
  VLPK_CUDA(cudaEventRecord(sd->fork, main));  // everything both kernels read has been issued on `main` by now
  VLPK_CUDA(cudaStreamWaitEvent(sd->stream, sd->fork, 0));
  VLPK_TRY(dgrad(main));
  sd->pending = true;
  return wgrad(sd->stream);
}

int wgrad_join(cudaStream_t main) {
  SideStream* sd = wgrad_side();
  if (sd == nullptr || !sd->pending) return 0;
  VLPK_CUDA(cudaEventRecord(sd->join, sd->stream));
  VLPK_CUDA(cudaStreamWaitEvent(main, sd->join, 0));
  sd->pending = false;
  return 0;
}

struct KvCache {       // incremental decode with a persistent K/V cache (vlpk_layer_cached_fwd, vlpk_layer_cached_group_fwd's text cache)
  void* base = nullptr;  // [B, rows, 2H] bf16: key | value projections of the rows this layer has seen
  int rows = 0;          // allocated rows per sequence
  int pos = 0;           // rows already valid; the call appends the Lq new rows at [pos, pos + Lq)
};

// Packed QKV projection of M rows x [M, H] -> qkv [M, 3H]: the three [H,H] weights read in place as N-segments.
int qkv_fwd(int M, int H, const VlpkLayerWeights* w, const void* x, void* qkv, cudaStream_t st) {
  if (H % 128 != 0) { set_error("mha_fwd: H=%d must be a multiple of 128 for the packed QKV projection", H); return -1; }
  GemmDesc g;
  g.M = M; g.N = 3 * H; g.K = H;
  g.A = x; g.lda = H;
  g.nseg = 3; g.b_seg_rows = H; g.ldb = H;
  g.B[0] = w->wq; g.B[1] = w->wk; g.B[2] = w->wv;
  g.bias[0] = static_cast<const bf16*>(w->bq); g.bias[1] = static_cast<const bf16*>(w->bk); g.bias[2] = static_cast<const bf16*>(w->bv);
  g.D0 = qkv; g.ldd0 = 3 * H;
  g.epi = EPI_STORE;
  g.bn = (H % 256 == 0) ? 0 : 128;
  return launch_gemm(g, st);
}

// K | V projection of M rows x [M, H] -> kv [M, 2H]: the two [H,H] weights read in place as N-segments.
int kv_fwd(int M, int H, const VlpkLayerWeights* w, const void* x, void* kv, cudaStream_t st) {
  GemmDesc g;
  g.M = M; g.N = 2 * H; g.K = H;
  g.A = x; g.lda = H;
  g.nseg = 2; g.b_seg_rows = H; g.ldb = H;
  g.B[0] = w->wk; g.B[1] = w->wv;
  g.bias[0] = static_cast<const bf16*>(w->bk); g.bias[1] = static_cast<const bf16*>(w->bv);
  g.D0 = kv; g.ldd0 = 2 * H;
  g.epi = EPI_STORE;
  g.bn = (H % 256 == 0) ? 0 : 128;
  return launch_gemm(g, st);
}

// BertSelfOutput after the attention core: output projection of a->ctx, residual x, dropout, LayerNorm -> a->y1
int attn_out_ln(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, VlpkLayerActs* a, float p_hidden, const VlpkDropout* drop,
                uint64_t layer_id, cudaStream_t st) {
  const int H = s->H, Mq = s->B * s->Lq;
  const DropoutCfg none = make_dropout(0.f, 0, 0);
  VLPK_TRY(fwd_linear(Mq, H, H, a->ctx, H, w->wo, H, w->bo, a->t1, H, EPI_STORE, nullptr, 0, none, st));
  LnArgs ln;
  ln.M = Mq; ln.H = H;
  ln.t = static_cast<const bf16*>(a->t1); ln.res = static_cast<const bf16*>(x);
  ln.gamma = static_cast<const bf16*>(w->ln1_g); ln.beta = static_cast<const bf16*>(w->ln1_b);
  ln.y = static_cast<bf16*>(a->y1); ln.stats = reinterpret_cast<float2*>(a->stats1);
  ln.drop = mk_drop(drop, p_hidden, site_of(layer_id, SITE_HID1));
  return launch_ln_res_drop_fwd(ln, st);
}

int mha_fwd_impl(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const void* x_kv, const uint32_t* bits, int mask_rows,
                 VlpkLayerActs* a, float p_attn, float p_hidden, const VlpkDropout* drop, uint64_t layer_id, cudaStream_t st,
                 const KvCache* cache = nullptr, const AttnGroupKv* group = nullptr) {
  const int H = s->H, Mq = s->B * s->Lq, Mkv = s->B * s->Lkv;
  const bool incr = (cache == nullptr && x_kv != nullptr && x_kv != x);
  const DropoutCfg none = make_dropout(0.f, 0, 0);
  AttnDesc ad;
  ad.B = s->B; ad.heads = s->heads; ad.Lq = s->Lq; ad.Lkv = s->Lkv; ad.kv_slots = s->kv_slots;
  ad.mask_bits = bits; ad.mask_rows = mask_rows;
  ad.o = a->ctx; ad.ld_o = H; ad.lse = a->lse;
  ad.drop = mk_drop(drop, p_attn, site_of(layer_id, SITE_ATTN));
  ad.keep_out = (ad.drop.p > 0.f) ? a->drop_attn : nullptr;   // forward stores its keep-decisions for backward
  if (cache != nullptr) {
    // Q and K|V of the NEW rows only; K|V are appended to the cache (rows [pos, pos + Lq) of every sequence), attention reads the cache
    // (with a group: the image's prefix cache, then the text cache)
    if (group == nullptr)
      VLPK_CHECK_ARG(a->kv != nullptr && cache->base != nullptr && cache->pos >= 0 && cache->pos + s->Lq == s->Lkv && s->Lkv <= cache->rows,
                     "mha_cached_fwd: pos=%d + Lq=%d must equal Lkv=%d <= cache rows %d", cache->pos, s->Lq, s->Lkv, cache->rows);
    VLPK_TRY(fwd_linear(Mq, H, H, x, H, w->wq, H, w->bq, a->qkv, H, EPI_STORE, nullptr, 0, none, st));
    VLPK_TRY(kv_fwd(Mq, H, w, x, a->kv, st));
    bf16* dst = static_cast<bf16*>(cache->base) + static_cast<size_t>(cache->pos) * 2 * H;
    VLPK_CUDA(cudaMemcpy2DAsync(dst, static_cast<size_t>(cache->rows) * 2 * H * sizeof(bf16), a->kv, static_cast<size_t>(s->Lq) * 2 * H * sizeof(bf16),
                                static_cast<size_t>(s->Lq) * 2 * H * sizeof(bf16), s->B, cudaMemcpyDeviceToDevice, st));
    ad.q = a->qkv; ad.ld_q = H;
    ad.k = cache->base;
    ad.v = static_cast<const bf16*>(cache->base) + H;
    ad.ld_kv = 2 * H;
    ad.kv_batch_stride = static_cast<int64_t>(cache->rows) * 2 * H;
  } else if (!incr) {
    VLPK_CHECK_ARG(s->Lq == s->Lkv, "mha_fwd: Lq != Lkv requires x_kv");
    VLPK_TRY(qkv_fwd(Mq, H, w, x, a->qkv, st));
    ad.q = a->qkv; ad.ld_q = 3 * H;
    ad.k = static_cast<const bf16*>(a->qkv) + H;
    ad.v = static_cast<const bf16*>(a->qkv) + 2 * H;
    ad.ld_kv = 3 * H;
  } else {
    VLPK_CHECK_ARG(a->kv != nullptr, "mha_fwd: incremental decode needs acts.kv");
    VLPK_TRY(fwd_linear(Mq, H, H, x, H, w->wq, H, w->bq, a->qkv, H, EPI_STORE, nullptr, 0, none, st));
    VLPK_TRY(kv_fwd(Mkv, H, w, x_kv, a->kv, st));
    ad.q = a->qkv; ad.ld_q = H;
    ad.k = a->kv;
    ad.v = static_cast<const bf16*>(a->kv) + H;
    ad.ld_kv = 2 * H;
  }
  VLPK_TRY(launch_attn_fwd(ad, group, nullptr, st));
  return attn_out_ln(s, w, x, a, p_hidden, drop, layer_id, st);
}

int ffn_fwd_impl(const VlpkShape* s, const VlpkLayerWeights* w, VlpkLayerActs* a, float p_hidden, const VlpkDropout* drop,
                 uint64_t layer_id, cudaStream_t st) {
  const int H = s->H, I = s->I, M = s->B * s->Lq;
  const DropoutCfg none = make_dropout(0.f, 0, 0);
  VLPK_TRY(fwd_linear(M, I, H, a->y1, H, w->w1, H, w->b1, a->u, I, EPI_GELU, a->hmid, I, none, st));
  VLPK_TRY(fwd_linear(M, H, I, a->hmid, I, w->w2, I, w->b2, a->t2, H, EPI_STORE, nullptr, 0, none, st));
  LnArgs ln;
  ln.M = M; ln.H = H;
  ln.t = static_cast<const bf16*>(a->t2); ln.res = static_cast<const bf16*>(a->y1);
  ln.gamma = static_cast<const bf16*>(w->ln2_g); ln.beta = static_cast<const bf16*>(w->ln2_b);
  ln.y = static_cast<bf16*>(a->y); ln.stats = reinterpret_cast<float2*>(a->stats2);
  ln.drop = mk_drop(drop, p_hidden, site_of(layer_id, SITE_HID2));
  return launch_ln_res_drop_fwd(ln, st);
}

// Backward of BertIntermediate + BertOutput.  dy: gradient of a->y; dy1: receives the gradient of a->y1 (both branches: through
// the two Linears and through LN2's residual input).  dy1 may alias dy (dy is consumed by the first kernel only).
int ffn_bwd_impl(const VlpkShape* s, const VlpkLayerWeights* w, const VlpkLayerActs* a, const void* dy, void* dy1,
                 const VlpkLayerGrads* g, const VlpkBwdScratch* ws, float p_hidden, const VlpkDropout* drop, uint64_t layer_id,
                 cudaStream_t st) {
  VLPK_CHECK_ARG(s->Lq == s->Lkv, "ffn_bwd: training path requires Lq == Lkv");
  const int H = s->H, I = s->I, M = s->B * s->Lq;
  const bool hdrop = (drop != nullptr && p_hidden > 0.f);
  // ---- BertOutput: LN2 backward (also yields d b2 as the column sum of dt2)
  LnArgs l2;
  l2.M = M; l2.H = H;
  l2.t = static_cast<const bf16*>(a->t2); l2.res = static_cast<const bf16*>(a->y1);
  l2.gamma = static_cast<const bf16*>(w->ln2_g); l2.stats = reinterpret_cast<float2*>(a->stats2);
  l2.dy = static_cast<const bf16*>(dy);
  l2.dz = static_cast<bf16*>(ws->dz2);
  l2.dt = hdrop ? static_cast<bf16*>(ws->dt2) : nullptr;
  l2.dgamma = g->ln2_g; l2.dbeta = g->ln2_b; l2.dbias = g->b2;
  l2.drop = mk_drop(drop, p_hidden, site_of(layer_id, SITE_HID2));
  VLPK_TRY(launch_ln_res_drop_bwd(l2, st));
  const void* dt2 = hdrop ? ws->dt2 : ws->dz2;
  // ---- output.dense: dW2 += dt2^T hmid ; dU = (dt2 W2) * gelu'(u)   [gelu'(u) was stored by the forward epilogue in acts.u]
  VLPK_TRY(linear_bwd_pair(
      st, [&](cudaStream_t q) { return wgrad_linear(M, H, I, dt2, H, a->hmid, I, g->w2, I, q); },
      [&](cudaStream_t q) {
        // db1 = column sums of dU: fused into the dgrad's epilogue (atomics), or in deterministic mode a separate ordered column sum
        if (!deterministic()) return dgrad_linear(M, H, I, dt2, H, w->w2, I, ws->du, I, EPI_MUL, a->u, I, q, g->b1);
        VLPK_TRY(dgrad_linear(M, H, I, dt2, H, w->w2, I, ws->du, I, EPI_MUL, a->u, I, q));
        return launch_colsum(ws->du, I, M, I, g->b1, q);
      }));
  // ---- intermediate.dense: dW1 += dU^T y1 ; dy1 = dU W1 + dz2 (residual branch of LN2)
  VLPK_TRY(linear_bwd_pair(
      st, [&](cudaStream_t q) { return wgrad_linear(M, I, H, ws->du, I, a->y1, H, g->w1, H, q); },
      [&](cudaStream_t q) { return dgrad_linear(M, I, H, ws->du, I, w->w1, H, dy1, H, EPI_ADD, ws->dz2, H, q); }));
  return wgrad_join(st);
}

// Backward of BertAttention.  dy1: gradient of a->y1; dx: receives the gradient of the layer input x (attention branch +
// LN1's residual input).  dx may alias dy1.
int mha_bwd_impl(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const uint32_t* bits, int mask_rows,
                 const VlpkLayerActs* a, const void* dy1, void* dx, const VlpkLayerGrads* g, const VlpkBwdScratch* ws, float p_attn,
                 float p_hidden, const VlpkDropout* drop, uint64_t layer_id, cudaStream_t st) {
  VLPK_CHECK_ARG(s->Lq == s->Lkv, "mha_bwd: training path requires Lq == Lkv");
  const int H = s->H, M = s->B * s->Lq;
  const bool hdrop = (drop != nullptr && p_hidden > 0.f);
  // ---- BertSelfOutput: LN1 backward
  LnArgs l1;
  l1.M = M; l1.H = H;
  l1.t = static_cast<const bf16*>(a->t1); l1.res = static_cast<const bf16*>(x);
  l1.gamma = static_cast<const bf16*>(w->ln1_g); l1.stats = reinterpret_cast<float2*>(a->stats1);
  l1.dy = static_cast<const bf16*>(dy1);
  l1.dz = static_cast<bf16*>(ws->dz1);
  l1.dt = hdrop ? static_cast<bf16*>(ws->dt1) : nullptr;
  l1.dgamma = g->ln1_g; l1.dbeta = g->ln1_b; l1.dbias = g->bo;
  l1.drop = mk_drop(drop, p_hidden, site_of(layer_id, SITE_HID1));
  VLPK_TRY(launch_ln_res_drop_bwd(l1, st));
  const void* dt1 = hdrop ? ws->dt1 : ws->dz1;
  // ---- attention.output.dense
  VLPK_TRY(linear_bwd_pair(
      st, [&](cudaStream_t q) { return wgrad_linear(M, H, H, dt1, H, a->ctx, H, g->wo, H, q); },
      [&](cudaStream_t q) { return dgrad_linear(M, H, H, dt1, H, w->wo, H, ws->dctx, H, EPI_STORE, nullptr, 0, q); }));
  // ---- attention core
  AttnDesc ad;
  ad.B = s->B; ad.heads = s->heads; ad.Lq = s->Lq; ad.Lkv = s->Lkv; ad.kv_slots = s->kv_slots;
  ad.q = a->qkv; ad.k = static_cast<const bf16*>(a->qkv) + H; ad.v = static_cast<const bf16*>(a->qkv) + 2 * H;
  ad.ld_q = 3 * H; ad.ld_kv = 3 * H;
  ad.o = a->ctx; ad.ld_o = H; ad.d_o = ws->dctx;
  ad.mask_bits = bits; ad.mask_rows = mask_rows; ad.lse = a->lse;
  ad.dq = ws->dqkv; ad.dk = static_cast<bf16*>(ws->dqkv) + H; ad.dv = static_cast<bf16*>(ws->dqkv) + 2 * H;
  ad.ld_dqkv = 3 * H;
  ad.drop = mk_drop(drop, p_attn, site_of(layer_id, SITE_ATTN));
  if (ad.drop.p > 0.f) ad.drop.bits = a->drop_attn;   // forward's keep-decisions (NULL: re-evaluate Philox)
  ad.dbias = g->bqkv;   // d bqkv = column sums of dQ | dK | dV, folded inside the attention backward kernel
  VLPK_TRY(launch_attn_bwd(ad, st));
  // ---- QKV projection: dWqkv += dqkv^T x ; dx = dqkv Wqkv + dz1 (residual branch of LN1)
  GemmDesc d;
  d.M = M; d.N = H; d.K = 3 * H;
  d.A = ws->dqkv; d.lda = 3 * H;
  d.b_mn = true; d.nseg = 3; d.b_seg_rows = H; d.ldb = H;
  d.B[0] = w->wq; d.B[1] = w->wk; d.B[2] = w->wv;
  d.D0 = dx; d.ldd0 = H;
  d.epi = EPI_ADD;
  d.aux = static_cast<const bf16*>(ws->dz1); d.ld_aux = H;
  VLPK_TRY(linear_bwd_pair(
      st, [&](cudaStream_t q) { return wgrad_linear(M, 3 * H, H, ws->dqkv, 3 * H, x, H, g->wqkv, H, q); },
      [&](cudaStream_t q) { return launch_gemm(d, q); }));
  return wgrad_join(st);
}

int layer_bwd_impl(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const uint32_t* bits, int mask_rows,
                   const VlpkLayerActs* a, const void* dy, void* dx, const VlpkLayerGrads* g, const VlpkBwdScratch* ws, float p_attn,
                   float p_hidden, const VlpkDropout* drop, uint64_t layer_id, cudaStream_t st) {
  VLPK_TRY(ffn_bwd_impl(s, w, a, dy, ws->dy1, g, ws, p_hidden, drop, layer_id, st));
  return mha_bwd_impl(s, w, x, bits, mask_rows, a, ws->dy1, dx, g, ws, p_attn, p_hidden, drop, layer_id, st);
}

__global__ void add_bf16_kernel(bf16* __restrict__ dst, const bf16* __restrict__ a, const bf16* __restrict__ b, long long n) {
  const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i + 8 <= n) {
    const uint4 ua = *reinterpret_cast<const uint4*>(a + i), ub = *reinterpret_cast<const uint4*>(b + i);
    const uint32_t wa[4] = {ua.x, ua.y, ua.z, ua.w}, wb[4] = {ub.x, ub.y, ub.z, ub.w};
    uint32_t o[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 x = unpack_bf16x2(wa[j]), y = unpack_bf16x2(wb[j]);
      o[j] = pack_bf16x2(x.x + y.x, x.y + y.y);
    }
    *reinterpret_cast<uint4*>(dst + i) = make_uint4(o[0], o[1], o[2], o[3]);
  } else {
    for (long long k = i; k < n; ++k) dst[k] = __float2bfloat16_rn(__bfloat162float(a[k]) + __bfloat162float(b[k]));
  }
}

__global__ void relu_bwd_kernel(bf16* __restrict__ dpre, const bf16* __restrict__ dy, const bf16* __restrict__ y, long long M,
                                int N, long long lddy, long long ldy, float scale) {
  const long long i = (static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x) * 8;
  if (i >= M * N) return;
  const long long r = i / N;
  const int c = static_cast<int>(i % N);
  const uint4 ud = *reinterpret_cast<const uint4*>(dy + r * lddy + c), uy = *reinterpret_cast<const uint4*>(y + r * ldy + c);
  const uint32_t wd[4] = {ud.x, ud.y, ud.z, ud.w}, wy[4] = {uy.x, uy.y, uy.z, uy.w};
  uint32_t o[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 d = unpack_bf16x2(wd[j]), v = unpack_bf16x2(wy[j]);
    o[j] = pack_bf16x2(v.x > 0.f ? d.x * scale : 0.f, v.y > 0.f ? d.y * scale : 0.f);
  }
  *reinterpret_cast<uint4*>(dpre + i) = make_uint4(o[0], o[1], o[2], o[3]);
}

// One layer of the scoring stacks over s->B sequences of R rows: the first K = R - T rows attend to the keys through key_bits, then
// the T query rows through query_bits, each also to its own key.
//   group null (vlpk_encoder_score_fwd): R = S + T; the keys are the K = S = s->Lq shared rows themselves.
//   group (vlpk_encoder_score_group_fwd): pairs, G per image, of R = 2T - 1 rows, K = T - 1 of them words (no launch when T = 1).
//   A pair's s->Lkv = P + T - 1 keys are the P rows of its image's prefix cache (group: prefix, prefix_rows, P, G), then its words.
int score_layer_fwd(const VlpkShape* s, int T, const AttnGroupKv* group, const VlpkLayerWeights* w, const void* x, const uint32_t* key_bits,
                    const uint32_t* query_bits, VlpkLayerActs* a, uint64_t layer_id, cudaStream_t st) {
  const int H = s->H, K = group != nullptr ? T - 1 : s->Lq, R = K + T;
  VLPK_TRY(qkv_fwd(s->B * R, H, w, x, a->qkv, st));
  const bf16* qkv = static_cast<const bf16*>(a->qkv);
  AttnGroupKv g;  // keys P + j: word j of the pair, read in place from its rows of the packed qkv
  if (group != nullptr) {
    g = *group;
    g.text = qkv + H; g.ld_text = 3 * H; g.T = R; g.pos = 0;
  }
  AttnDesc ad;
  ad.B = s->B; ad.heads = s->heads; ad.Lkv = s->Lkv; ad.kv_slots = s->kv_slots;
  ad.q = qkv; ad.ld_q = 3 * H; ad.q_batch_stride = static_cast<int64_t>(R) * 3 * H;
  ad.k = qkv + H; ad.v = qkv + 2 * H; ad.kv_batch_stride = static_cast<int64_t>(R) * 3 * H;  // unused with a group
  ad.ld_kv = group != nullptr ? 2 * H : 3 * H;  // the prefix cache's rows, or the packed qkv's
  ad.o = a->ctx; ad.ld_o = H; ad.o_batch_stride = static_cast<int64_t>(R) * H;
  ad.lse = a->lse;
  ad.drop = make_dropout(0.f, 0, 0);
  if (K > 0) {
    AttnDesc kd = ad;
    kd.Lq = K;
    kd.mask_bits = key_bits; kd.mask_rows = K;
    VLPK_TRY(launch_attn_fwd(kd, group != nullptr ? &g : nullptr, nullptr, st));
  }
  AttnDesc qd = ad;
  qd.Lq = T;
  qd.q = qkv + static_cast<size_t>(K) * 3 * H;
  qd.o = static_cast<bf16*>(a->ctx) + static_cast<size_t>(K) * H;
  qd.mask_bits = query_bits; qd.mask_rows = T;
  qd.lse = a->lse + static_cast<size_t>(s->B) * s->heads * K;
  AttnSelfKv sk;
  sk.k = qkv + static_cast<size_t>(K) * 3 * H + H;
  sk.v = qkv + static_cast<size_t>(K) * 3 * H + 2 * H;
  sk.ld = 3 * H; sk.batch_stride = static_cast<int64_t>(R) * 3 * H;
  VLPK_TRY(launch_attn_fwd(qd, group != nullptr ? &g : nullptr, &sk, st));
  VlpkShape rows = *s;  // the row-wise tail (output projection, LayerNorms, FFN) over all B * R rows
  rows.Lq = rows.Lkv = R;
  VLPK_TRY(attn_out_ln(&rows, w, x, a, 0.f, nullptr, layer_id, st));
  return ffn_fwd_impl(&rows, w, a, 0.f, nullptr, layer_id, st);
}

// The layer loop of both scoring stacks; with a group, group->prefix is set to prefix[i] for layer i.
int score_stack_fwd(const VlpkShape* s, int T, int n_layers, const VlpkLayerWeights* w, const void* x, AttnGroupKv* group,
                    const void* const* prefix, const uint32_t* key_bits, const uint32_t* query_bits, VlpkLayerActs* acts, cudaStream_t st) {
  const void* cur = x;
  for (int i = 0; i < n_layers; ++i) {
    if (group != nullptr) group->prefix = prefix[i];
    VLPK_TRY(score_layer_fwd(s, T, group, &w[i], cur, key_bits, query_bits, &acts[i], i, st));
    cur = acts[i].y;
  }
  return 0;
}

// Bytes of one layer's activations over `rows` rows per sequence: eight bf16 buffers (qkv, ctx, t1, y1, u, hmid, t2, y: 8H + 2I per
// row) plus kv_elems bf16 of K | V, then the fp32 logsumexp and the two float2 LayerNorm statistics per row.
size_t act_bytes(const VlpkShape* s, size_t rows, size_t kv_elems) {
  const size_t H = s->H, I = s->I, M = static_cast<size_t>(s->B) * rows;
  const size_t lse = (static_cast<size_t>(s->B) * s->heads * rows + 3) / 4 * 4;  // keeps the float2 statistics behind it aligned
  return 2 * (M * (3 * H + 5 * H + 2 * I) + kv_elems) + 4 * (lse + 4 * M);
}

}  // namespace

#pragma GCC visibility push(default)
extern "C" {

int vlpk_version(void) { return VLPK_VERSION; }
int vlpk_debug_set_option(const char* name, int value) {
  VLPK_CHECK_ARG(name != nullptr, "set_option: null name");
  if (strcmp(name, "wgrad_stream") == 0) { g_wgrad_stream = value ? 1 : 0; return 0; }
  if (strcmp(name, "attn_tiled") == 0) { set_attn_tiled(value != 0); return 0; }
  set_error("set_option: unknown option '%s'", name);
  return -1;
}
int vlpk_debug_plan_gemm(int M, int N, int K, int a_mn, int b_mn, int nseg, int seg_rows, int epi, int bn, int splits, int* out2) {
  GemmDesc g;
  g.M = M; g.N = N; g.K = K;
  g.a_mn = a_mn != 0; g.b_mn = b_mn != 0;
  g.nseg = nseg; g.b_seg_rows = seg_rows;
  g.epi = epi; g.bn = bn; g.splits = splits;
  return plan_gemm(g, &out2[0], &out2[1]);
}
void vlpk_set_reserved_sms(int n) { set_reserved_sms(n); }
void vlpk_set_deterministic(int on) { set_deterministic(on != 0); }
const char* vlpk_last_error(void) { return get_error(); }

int vlpk_mask_pack(const void* mask, int dtype, int mode, int B, int rows, int kv, int64_t stride_b, int64_t stride_r, uint32_t* out,
                   void* stream) {
  VLPK_CHECK_ARG(mask != nullptr && out != nullptr, "mask_pack: null pointer");
  return launch_mask_pack(mask, dtype, mode, B, rows, kv, stride_b, stride_r, out, S(stream));
}

int vlpk_mask_synth(const int32_t* len_b, const int32_t* mode, int len_a, int B, int L, uint32_t* out, void* stream) {
  return launch_mask_synth(len_b, mode, len_a, B, L, out, S(stream));
}

int vlpk_mask_synth_grouped(const int32_t* len_b, int G, int len_a, int B, int T, uint32_t* out, void* stream) {
  return launch_mask_synth_grouped(len_b, G, len_a, B, T, out, S(stream));
}

int vlpk_linear_fwd(int M, int N, int K, const void* x, int64_t ldx, const void* w, int64_t ldw, const void* bias, void* y, int64_t ldy,
                    int act, const VlpkDropout* drop, uint64_t site, void* stream) {
  VLPK_CHECK_ARG(x && w && y, "linear_fwd: null pointer");
  VLPK_CHECK_ARG(act == VLPK_ACT_NONE || act == VLPK_ACT_RELU, "linear_fwd: act %d unsupported", act);
  const DropoutCfg dc = (act == VLPK_ACT_RELU && drop != nullptr) ? mk_drop(drop, drop->p, site) : make_dropout(0.f, 0, site);
  return fwd_linear(M, N, K, x, ldx, w, ldw, bias, y, ldy, act == VLPK_ACT_RELU ? EPI_RELU : EPI_STORE, nullptr, 0, dc, S(stream));
}

int vlpk_linear_bwd(int M, int N, int K, const void* x, int64_t ldx, const void* w, int64_t ldw, const void* y, int64_t ldy,
                    const void* dy, int64_t lddy, void* dpre, void* dx, int64_t lddx, float* dw, int64_t lddw, float* db, int act,
                    float p_drop, void* stream) {
  VLPK_CHECK_ARG(x && w && dy && dw, "linear_bwd: null pointer");
  cudaStream_t st = S(stream);
  const void* g = dy;
  int64_t ldg = lddy;
  if (act == VLPK_ACT_RELU) {
    VLPK_CHECK_ARG(y != nullptr && dpre != nullptr && N % 8 == 0, "linear_bwd: relu needs y, dpre and N %% 8 == 0");
    const long long n = static_cast<long long>(M) * N;
    LaunchScope scope(CAT_MISC, 6.0 * n, st);
    relu_bwd_kernel<<<static_cast<unsigned>((n / 8 + 255) / 256), 256, 0, st>>>(static_cast<bf16*>(dpre), static_cast<const bf16*>(dy),
                                                                             static_cast<const bf16*>(y), M, N, lddy, ldy,
                                                                             p_drop > 0.f ? 1.0f / (1.0f - p_drop) : 1.0f);
    VLPK_CUDA(cudaGetLastError());
    g = dpre;
    ldg = N;
  }
  if (db != nullptr) VLPK_TRY(launch_colsum(g, ldg, M, N, db, st));
  VLPK_TRY(wgrad_linear(M, N, K, g, ldg, x, ldx, dw, lddw, st));
  if (dx != nullptr) VLPK_TRY(dgrad_linear(M, N, K, g, ldg, w, ldw, dx, lddx, EPI_STORE, nullptr, 0, st));
  return 0;
}

static EmbedArgs mk_embed(int B, int L, int H, int R, int vis_input, const int64_t* ids, const int64_t* tt, const int64_t* pos,
                          const void* word_w, const void* pos_w, const void* type_w, const void* vis, const void* vpe,
                          const void* ln_g) {
  EmbedArgs a;
  a.B = B; a.L = L; a.H = H; a.R = R; a.vis_input = vis_input;
  a.ids = reinterpret_cast<const long long*>(ids);
  a.tt = reinterpret_cast<const long long*>(tt);
  a.pos = reinterpret_cast<const long long*>(pos);
  a.word = static_cast<const bf16*>(word_w); a.posw = static_cast<const bf16*>(pos_w); a.typew = static_cast<const bf16*>(type_w);
  a.vis = static_cast<const bf16*>(vis); a.vpe = static_cast<const bf16*>(vpe);
  a.gamma = static_cast<const bf16*>(ln_g);
  return a;
}

int vlpk_embed_fwd(int B, int L, int H, int R, int vis_input, const int64_t* ids, const int64_t* token_type, const int64_t* pos,
                   const void* word_w, const void* pos_w, const void* type_w, const void* vis, const void* vis_pe, const void* ln_g,
                   const void* ln_b, void* y, float* stats, const VlpkDropout* drop, uint64_t site, void* stream) {
  VLPK_CHECK_ARG(ids && word_w && pos_w && type_w && ln_g && ln_b && y, "embed_fwd: null pointer");
  EmbedArgs a = mk_embed(B, L, H, R, vis_input, ids, token_type, pos, word_w, pos_w, type_w, vis, vis_pe, ln_g);
  a.beta = static_cast<const bf16*>(ln_b);
  a.y = static_cast<bf16*>(y);
  a.stats = reinterpret_cast<float2*>(stats);
  a.drop = mk_drop(drop, drop ? drop->p : 0.f, site);
  return launch_embed_fwd(a, S(stream));
}

int vlpk_embed_bwd(int B, int L, int H, int R, int vis_input, const int64_t* ids, const int64_t* token_type, const int64_t* pos,
                   const void* word_w, const void* pos_w, const void* type_w, const void* vis, const void* vis_pe, const void* ln_g,
                   const float* stats, const void* dy, void* dz, float* d_ln_g, float* d_ln_b, const VlpkDropout* drop, uint64_t site,
                   void* stream) {
  VLPK_CHECK_ARG(ids && word_w && pos_w && type_w && ln_g && stats && dy && dz, "embed_bwd: null pointer");
  EmbedArgs a = mk_embed(B, L, H, R, vis_input, ids, token_type, pos, word_w, pos_w, type_w, vis, vis_pe, ln_g);
  a.stats = reinterpret_cast<float2*>(const_cast<float*>(stats));
  a.dy = static_cast<const bf16*>(dy);
  a.dz = static_cast<bf16*>(dz);
  a.dgamma = d_ln_g; a.dbeta = d_ln_b;
  a.drop = mk_drop(drop, drop ? drop->p : 0.f, site);
  return launch_embed_bwd(a, S(stream));
}

int vlpk_embed_tables_bwd(int B, int L, int H, int R, int vis_input, const int64_t* ids, const int64_t* token_type, const int64_t* pos,
                          const void* dz, int V, int P, int T, void* d_word, float* word_scratch, float* d_pos, float* d_type,
                          void* stream) {
  TableGradArgs a;
  a.B = B; a.L = L; a.H = H; a.R = R; a.vis_input = vis_input;
  a.V = V; a.P = P; a.T = T;
  a.ids = reinterpret_cast<const long long*>(ids);
  a.tt = reinterpret_cast<const long long*>(token_type);
  a.pos = reinterpret_cast<const long long*>(pos);
  a.dz = static_cast<const bf16*>(dz);
  a.d_word = static_cast<bf16*>(d_word);
  a.scratch = word_scratch; a.d_pos = d_pos; a.d_type = d_type;
  return launch_embed_tables_bwd(a, S(stream));
}

int vlpk_ln_res_drop_fwd(int64_t M, int H, const void* t, const void* res, const void* gamma, const void* beta, void* y, float* stats,
                         const VlpkDropout* drop, uint64_t site, void* stream) {
  VLPK_CHECK_ARG(t && gamma && beta && y, "ln_res_drop_fwd: null pointer");
  LnArgs a;
  a.M = M; a.H = H;
  a.t = static_cast<const bf16*>(t); a.res = static_cast<const bf16*>(res);
  a.gamma = static_cast<const bf16*>(gamma); a.beta = static_cast<const bf16*>(beta);
  a.y = static_cast<bf16*>(y); a.stats = reinterpret_cast<float2*>(stats);
  a.drop = mk_drop(drop, drop ? drop->p : 0.f, site);
  return launch_ln_res_drop_fwd(a, S(stream));
}

int vlpk_ln_res_drop_bwd(int64_t M, int H, const void* t, const void* res, const void* gamma, const float* stats, const void* dy,
                         void* dz, void* dt, float* dgamma, float* dbeta, float* dbias, const VlpkDropout* drop, uint64_t site,
                         void* stream) {
  VLPK_CHECK_ARG(t && gamma && stats && dy, "ln_res_drop_bwd: null pointer");
  LnArgs a;
  a.M = M; a.H = H;
  a.t = static_cast<const bf16*>(t); a.res = static_cast<const bf16*>(res);
  a.gamma = static_cast<const bf16*>(gamma);
  a.stats = reinterpret_cast<float2*>(const_cast<float*>(stats));
  a.dy = static_cast<const bf16*>(dy);
  a.dz = static_cast<bf16*>(dz); a.dt = static_cast<bf16*>(dt);
  a.dgamma = dgamma; a.dbeta = dbeta; a.dbias = dbias;
  a.drop = mk_drop(drop, drop ? drop->p : 0.f, site);
  return launch_ln_res_drop_bwd(a, S(stream));
}

int vlpk_attn_core_fwd_wide(int B, int heads, int Lq, int Lkv, const void* q, int64_t ld_q, const void* k, const void* v, int64_t ld_kv,
                            const uint32_t* mask_bits, int mask_rows, void* ctx, int64_t ld_ctx, float* lse, const VlpkDropout* drop,
                            uint64_t site, int kv_slots, void* stream) {
  VLPK_CHECK_ARG(q && k && v && ctx, "attn_core_fwd: null pointer");
  AttnDesc d;
  d.B = B; d.heads = heads; d.Lq = Lq; d.Lkv = Lkv; d.kv_slots = kv_slots;
  d.q = q; d.k = k; d.v = v; d.ld_q = ld_q; d.ld_kv = ld_kv;
  d.o = ctx; d.ld_o = ld_ctx;
  d.mask_bits = mask_bits; d.mask_rows = mask_rows; d.lse = lse;
  d.drop = mk_drop(drop, drop ? drop->p : 0.f, site);
  return launch_attn_fwd(d, nullptr, nullptr, S(stream));
}

int vlpk_attn_core_fwd(int B, int heads, int Lq, int Lkv, const void* q, int64_t ld_q, const void* k, const void* v, int64_t ld_kv,
                       const uint32_t* mask_bits, int mask_rows, void* ctx, int64_t ld_ctx, float* lse, const VlpkDropout* drop,
                       uint64_t site, void* stream) {
  return vlpk_attn_core_fwd_wide(B, heads, Lq, Lkv, q, ld_q, k, v, ld_kv, mask_bits, mask_rows, ctx, ld_ctx, lse, drop, site, 0, stream);
}

int vlpk_attn_core_self_fwd(int B, int heads, int Lq, int Lkv, const void* q, int64_t ld_q, int64_t q_bstride, const void* k, const void* v,
                            int64_t ld_kv, int64_t kv_bstride, const void* k_self, const void* v_self, const uint32_t* mask_bits, int kv_slots,
                            void* ctx, int64_t ld_ctx, int64_t ctx_bstride, float* lse, void* stream) {
  AttnDesc d;
  d.B = B; d.heads = heads; d.Lq = Lq; d.Lkv = Lkv; d.kv_slots = kv_slots;
  d.q = q; d.ld_q = ld_q; d.q_batch_stride = q_bstride;
  d.k = k; d.v = v; d.ld_kv = ld_kv; d.kv_batch_stride = kv_bstride;
  d.o = ctx; d.ld_o = ld_ctx; d.o_batch_stride = ctx_bstride;
  d.mask_bits = mask_bits; d.mask_rows = Lq; d.lse = lse;
  AttnSelfKv s;
  s.k = k_self; s.v = v_self; s.ld = ld_q; s.batch_stride = q_bstride;
  return launch_attn_fwd(d, nullptr, &s, S(stream));
}

int vlpk_attn_core_group_self_fwd(int B, int G, int heads, int Lq, int Lkv, int P, const void* q, int64_t ld_q, int64_t q_bstride,
                                  const void* prefix, int prefix_rows, int64_t ld_prefix, const void* text, int T, int64_t ld_text,
                                  const void* k_self, const void* v_self, const uint32_t* mask_bits, int kv_slots, void* ctx, int64_t ld_ctx,
                                  int64_t ctx_bstride, float* lse, void* stream) {
  AttnDesc d;
  d.B = B; d.heads = heads; d.Lq = Lq; d.Lkv = Lkv; d.kv_slots = kv_slots;
  d.q = q; d.ld_q = ld_q; d.q_batch_stride = q_bstride;
  d.ld_kv = ld_prefix;
  d.o = ctx; d.ld_o = ld_ctx; d.o_batch_stride = ctx_bstride;
  d.mask_bits = mask_bits; d.mask_rows = Lq; d.lse = lse;
  AttnGroupKv g;
  g.prefix = prefix; g.prefix_rows = prefix_rows; g.P = P;
  g.text = text; g.T = T; g.G = G; g.pos = 0; g.ld_text = ld_text;
  AttnSelfKv s;
  s.k = k_self; s.v = v_self; s.ld = ld_q; s.batch_stride = q_bstride;
  return launch_attn_fwd(d, &g, &s, S(stream));
}

int vlpk_attn_probs(int B, int heads, int Lq, int Lkv, int row0, const void* q, int64_t ld_q, int64_t q_bstride, const void* k, int64_t ld_k,
                    int64_t k_bstride, const uint32_t* mask_bits, int mask_rows, int kv_slots, const float* lse, float* p, int64_t ld_p,
                    int64_t p_bstride, void* stream) {
  AttnDesc d;
  d.B = B; d.heads = heads; d.Lq = Lq; d.Lkv = Lkv; d.kv_slots = kv_slots;
  d.q = q; d.ld_q = ld_q;
  d.k = k; d.ld_kv = ld_k; d.kv_batch_stride = k_bstride;
  d.mask_bits = mask_bits; d.mask_rows = mask_rows;
  d.lse = const_cast<float*>(lse);
  return launch_attn_probs(d, q_bstride, row0, p, ld_p, p_bstride, S(stream));
}

int vlpk_attn_core_bwd_wide(int B, int heads, int L, const void* q, const void* k, const void* v, int64_t ld_qkv, const uint32_t* mask_bits,
                            int mask_rows, const void* ctx, const void* dctx, int64_t ld_ctx, const float* lse, void* dq, void* dk, void* dv,
                            int64_t ld_dqkv, const VlpkDropout* drop, uint64_t site, int kv_slots, void* stream) {
  VLPK_CHECK_ARG(q && k && v && ctx && dctx && lse && dq && dk && dv, "attn_core_bwd: null pointer");
  AttnDesc d;
  d.B = B; d.heads = heads; d.Lq = L; d.Lkv = L; d.kv_slots = kv_slots;
  d.q = q; d.k = k; d.v = v; d.ld_q = ld_qkv; d.ld_kv = ld_qkv;
  d.o = const_cast<void*>(ctx); d.ld_o = ld_ctx; d.d_o = dctx;
  d.mask_bits = mask_bits; d.mask_rows = mask_rows; d.lse = const_cast<float*>(lse);
  d.dq = dq; d.dk = dk; d.dv = dv; d.ld_dqkv = ld_dqkv;
  d.drop = mk_drop(drop, drop ? drop->p : 0.f, site);
  return launch_attn_bwd(d, S(stream));
}

int vlpk_attn_core_bwd(int B, int heads, int L, const void* q, const void* k, const void* v, int64_t ld_qkv, const uint32_t* mask_bits,
                       int mask_rows, const void* ctx, const void* dctx, int64_t ld_ctx, const float* lse, void* dq, void* dk, void* dv,
                       int64_t ld_dqkv, const VlpkDropout* drop, uint64_t site, void* stream) {
  return vlpk_attn_core_bwd_wide(B, heads, L, q, k, v, ld_qkv, mask_bits, mask_rows, ctx, dctx, ld_ctx, lse, dq, dk, dv, ld_dqkv, drop, site, 0,
                                 stream);
}

int vlpk_mha_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const void* x_kv, const uint32_t* mask_bits, int mask_rows,
                 VlpkLayerActs* a, float p_attn, float p_hidden, const VlpkDropout* drop, uint64_t layer_id, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(w && x && mask_bits && a, "mha_fwd: null pointer");
  return mha_fwd_impl(s, w, x, x_kv, mask_bits, mask_rows, a, p_attn, p_hidden, drop, layer_id, S(stream));
}

int vlpk_ffn_fwd(const VlpkShape* s, const VlpkLayerWeights* w, VlpkLayerActs* a, float p_hidden, const VlpkDropout* drop,
                 uint64_t layer_id, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(w && a, "ffn_fwd: null pointer");
  return ffn_fwd_impl(s, w, a, p_hidden, drop, layer_id, S(stream));
}

int vlpk_layer_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const void* x_kv, const uint32_t* mask_bits,
                   int mask_rows, VlpkLayerActs* a, float p_attn, float p_hidden, const VlpkDropout* drop, uint64_t layer_id,
                   void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(w && x && mask_bits && a, "layer_fwd: null pointer");
  VLPK_TRY(mha_fwd_impl(s, w, x, x_kv, mask_bits, mask_rows, a, p_attn, p_hidden, drop, layer_id, S(stream)));
  return ffn_fwd_impl(s, w, a, p_hidden, drop, layer_id, S(stream));
}

int vlpk_layer_bwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const uint32_t* mask_bits, int mask_rows,
                   const VlpkLayerActs* a, const void* dy, void* dx, const VlpkLayerGrads* g, const VlpkBwdScratch* ws, float p_attn,
                   float p_hidden, const VlpkDropout* drop, uint64_t layer_id, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(w && x && mask_bits && a && dy && dx && g && ws, "layer_bwd: null pointer");
  return layer_bwd_impl(s, w, x, mask_bits, mask_rows, a, dy, dx, g, ws, p_attn, p_hidden, drop, layer_id, S(stream));
}

int vlpk_ffn_bwd(const VlpkShape* s, const VlpkLayerWeights* w, const VlpkLayerActs* a, const void* dy, void* dy1,
                 const VlpkLayerGrads* g, const VlpkBwdScratch* ws, float p_hidden, const VlpkDropout* drop, uint64_t layer_id,
                 void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(w && a && dy && dy1 && g && ws, "ffn_bwd: null pointer");
  return ffn_bwd_impl(s, w, a, dy, dy1, g, ws, p_hidden, drop, layer_id, S(stream));
}

int vlpk_mha_bwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const uint32_t* mask_bits, int mask_rows,
                 const VlpkLayerActs* a, const void* dy1, void* dx, const VlpkLayerGrads* g, const VlpkBwdScratch* ws, float p_attn,
                 float p_hidden, const VlpkDropout* drop, uint64_t layer_id, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(w && x && mask_bits && a && dy1 && dx && g && ws, "mha_bwd: null pointer");
  return mha_bwd_impl(s, w, x, mask_bits, mask_rows, a, dy1, dx, g, ws, p_attn, p_hidden, drop, layer_id, S(stream));
}

int vlpk_mha_incr_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const void* x_kv, const uint32_t* mask_bits,
                      int mask_rows, VlpkLayerActs* a, uint64_t layer_id, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(w && x && x_kv && x_kv != x && mask_bits && a, "mha_incr_fwd: needs x, x_kv (= cat(history, x)), mask and acts");
  return mha_fwd_impl(s, w, x, x_kv, mask_bits, mask_rows, a, 0.f, 0.f, nullptr, layer_id, S(stream));
}

int vlpk_layer_cached_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, void* kv_cache, int cache_rows, int pos,
                          const uint32_t* mask_bits, int mask_rows, VlpkLayerActs* a, uint64_t layer_id, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(w && x && kv_cache && mask_bits && a, "layer_cached_fwd: null pointer");
  KvCache c;
  c.base = kv_cache; c.rows = cache_rows; c.pos = pos;
  VLPK_TRY(mha_fwd_impl(s, w, x, nullptr, mask_bits, mask_rows, a, 0.f, 0.f, nullptr, layer_id, S(stream), &c));
  return ffn_fwd_impl(s, w, a, 0.f, nullptr, layer_id, S(stream));
}

int vlpk_layer_cached_group_fwd(const VlpkShape* s, const VlpkLayerWeights* w, const void* x, const void* prefix, int prefix_rows, int P,
                                void* text, int T, const int32_t* slots, int G, int pos, const uint32_t* mask_bits, int mask_rows,
                                VlpkLayerActs* a, uint64_t layer_id, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(w && x && prefix && text && slots && mask_bits && a && a->qkv && a->kv && a->ctx && a->lse,
                 "layer_cached_group_fwd: null pointer");
  VLPK_CHECK_ARG(G >= 1 && s->B % G == 0, "layer_cached_group_fwd: B=%d hypotheses are not whole groups of G=%d", s->B, G);
  VLPK_CHECK_ARG(P >= 1 && P <= prefix_rows, "layer_cached_group_fwd: P=%d must be in [1, prefix rows %d]", P, prefix_rows);
  VLPK_CHECK_ARG(pos >= 0 && pos + s->Lq <= T, "layer_cached_group_fwd: pos=%d + Lq=%d exceeds the T=%d text rows", pos, s->Lq, T);
  VLPK_CHECK_ARG(P + pos + s->Lq == s->Lkv, "layer_cached_group_fwd: Lkv=%d must equal P=%d + pos=%d + Lq=%d", s->Lkv, P, pos, s->Lq);
  VLPK_CHECK_ARG(mask_rows == 1 || mask_rows == s->Lq, "layer_cached_group_fwd: mask rows %d (1 or Lq=%d)", mask_rows, s->Lq);
  const auto a16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; };
  VLPK_CHECK_ARG(a16(x) && a16(prefix) && a16(text) && a16(mask_bits) && (reinterpret_cast<uintptr_t>(slots) & 3u) == 0,
                 "layer_cached_group_fwd: x, prefix, text and mask_bits must be 16-byte aligned, slots 4-byte aligned");
  AttnGroupKv g;
  g.prefix = prefix; g.prefix_rows = prefix_rows; g.P = P;
  g.text = text; g.slots = slots; g.T = T; g.G = G; g.pos = pos;
  KvCache c;
  c.base = text; c.rows = T; c.pos = pos;
  VLPK_TRY(mha_fwd_impl(s, w, x, nullptr, mask_bits, mask_rows, a, 0.f, 0.f, nullptr, layer_id, S(stream), &c, &g));
  return ffn_fwd_impl(s, w, a, 0.f, nullptr, layer_id, S(stream));
}

int vlpk_workspace_bytes(const VlpkShape* s, size_t* out3) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(out3 != nullptr, "workspace_bytes: null output");
  const size_t H = s->H, I = s->I, Mq = static_cast<size_t>(s->B) * s->Lq, Mkv = static_cast<size_t>(s->B) * s->Lkv;
  out3[0] = act_bytes(s, s->Lq, (s->Lkv != s->Lq) ? Mkv * 2 * H : 0);
  out3[1] = 2 * (Mq * (7 * H + I + 3 * H));
  out3[2] = 4 * (3 * H * H + 3 * H + H * H + H + 2 * H + I * H + I + H * I + H + 2 * H);
  return 0;
}

int vlpk_encoder_fwd(const VlpkShape* s, int n_layers, const VlpkLayerWeights* w, const void* x, const uint32_t* mask_bits, int mask_rows,
                     VlpkLayerActs* acts, float p_attn, float p_hidden, const VlpkDropout* drop, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(n_layers > 0 && w && x && mask_bits && acts, "encoder_fwd: null pointer");
  const void* cur = x;
  for (int i = 0; i < n_layers; ++i) {
    VLPK_TRY(mha_fwd_impl(s, &w[i], cur, nullptr, mask_bits, mask_rows, &acts[i], p_attn, p_hidden, drop, i, S(stream)));
    VLPK_TRY(ffn_fwd_impl(s, &w[i], &acts[i], p_hidden, drop, i, S(stream)));
    cur = acts[i].y;
  }
  return 0;
}

int vlpk_encoder_score_workspace_bytes(const VlpkShape* s, int T, size_t* out1) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(out1 != nullptr, "encoder_score_workspace_bytes: null output");
  VLPK_CHECK_ARG(s->Lq == s->Lkv && T >= 1 && T <= 512, "encoder_score: Lq=%d must equal Lkv=%d (the shared rows S), T=%d in [1,512]", s->Lq,
                 s->Lkv, T);
  out1[0] = act_bytes(s, s->Lq + T, 0);
  return 0;
}

int vlpk_encoder_score_fwd(const VlpkShape* s, int T, int n_layers, const VlpkLayerWeights* w, const void* x, const uint32_t* shared_bits,
                           const uint32_t* query_bits, VlpkLayerActs* acts, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(s->Lq == s->Lkv && T >= 1 && T <= 512, "encoder_score: Lq=%d must equal Lkv=%d (the shared rows S), T=%d in [1,512]", s->Lq,
                 s->Lkv, T);
  VLPK_CHECK_ARG(s->H % 128 == 0, "encoder_score: H=%d must be a multiple of 128 for the packed QKV projection", s->H);
  VLPK_CHECK_ARG(n_layers > 0 && w && x && shared_bits && query_bits && acts, "encoder_score: null pointer");
  const auto al = [](const void* p, uintptr_t n) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; };
  VLPK_CHECK_ARG(al(x, 16) && al(shared_bits, 16) && al(query_bits, 16), "encoder_score: x and the mask bits must be 16-byte aligned");
  for (int i = 0; i < n_layers; ++i) {  // every layer's buffers, so that no check fails after a launch
    const VlpkLayerActs& a = acts[i];
    VLPK_CHECK_ARG(al(a.qkv, 16) && al(a.ctx, 16) && al(a.t1, 16) && al(a.y1, 16) && al(a.u, 16) && al(a.hmid, 16) && al(a.t2, 16) &&
                   al(a.y, 16) && al(a.lse, 4) && al(a.stats1, 8) && al(a.stats2, 8) && (i == 0 || a.y != acts[i - 1].y),
                   "encoder_score: layer %d acts missing or misaligned (16-byte bf16 buffers, 4-byte lse, 8-byte statistics), or its output "
                   "aliases its input", i);
  }
  return score_stack_fwd(s, T, n_layers, w, x, nullptr, nullptr, shared_bits, query_bits, acts, S(stream));
}

int vlpk_encoder_score_group_workspace_bytes(const VlpkShape* s, int T, size_t* out1) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(out1 != nullptr, "encoder_score_group_workspace_bytes: null output");
  VLPK_CHECK_ARG(s->Lq == s->Lkv && T >= 1 && T <= s->Lkv, "encoder_score_group: Lq=%d must equal Lkv=%d (the keys S), T=%d in [1, S]", s->Lq,
                 s->Lkv, T);
  out1[0] = act_bytes(s, 2 * T - 1, 0);
  return 0;
}

int vlpk_encoder_score_group_fwd(const VlpkShape* s, int T, int G, int P, int n_layers, const VlpkLayerWeights* w, const void* x,
                                 const void* const* prefix, int prefix_rows, const uint32_t* word_bits, const uint32_t* query_bits,
                                 VlpkLayerActs* acts, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(s->Lq == s->Lkv && T >= 1 && T <= 512, "encoder_score_group: Lq=%d must equal Lkv=%d (the keys S), T=%d in [1,512]", s->Lq,
                 s->Lkv, T);
  VLPK_CHECK_ARG(P >= 1 && P <= prefix_rows && P + T - 1 == s->Lkv, "encoder_score_group: P=%d must be in [1, prefix rows %d] with P + T - 1 "
                 "= S=%d (T=%d)", P, prefix_rows, s->Lkv, T);
  VLPK_CHECK_ARG(G >= 1 && s->B % G == 0, "encoder_score_group: B=%d pairs are not whole groups of G=%d", s->B, G);
  VLPK_CHECK_ARG(s->H % 128 == 0, "encoder_score_group: H=%d must be a multiple of 128 for the packed QKV projection", s->H);
  VLPK_CHECK_ARG(n_layers > 0 && w && x && prefix && (word_bits || T == 1) && query_bits && acts, "encoder_score_group: null pointer");
  const auto al = [](const void* p, uintptr_t n) { return p != nullptr && (reinterpret_cast<uintptr_t>(p) & (n - 1)) == 0; };
  VLPK_CHECK_ARG(al(x, 16) && (T == 1 || al(word_bits, 16)) && al(query_bits, 16), "encoder_score_group: x and the mask bits must be 16-byte "
                 "aligned");
  for (int i = 0; i < n_layers; ++i) {  // every layer's buffers, so that no check fails after a launch
    const VlpkLayerActs& a = acts[i];
    VLPK_CHECK_ARG(al(prefix[i], 16) && al(a.qkv, 16) && al(a.ctx, 16) && al(a.t1, 16) && al(a.y1, 16) && al(a.u, 16) && al(a.hmid, 16) &&
                   al(a.t2, 16) && al(a.y, 16) && al(a.lse, 4) && al(a.stats1, 8) && al(a.stats2, 8) && a.y != (i == 0 ? x : acts[i - 1].y),
                   "encoder_score_group: layer %d prefix cache or acts missing or misaligned (16-byte bf16 buffers, 4-byte lse, 8-byte "
                   "statistics), or its output aliases its input", i);
  }
  AttnGroupKv g;
  g.prefix_rows = prefix_rows; g.P = P; g.G = G;
  return score_stack_fwd(s, T, n_layers, w, x, &g, prefix, word_bits, query_bits, acts, S(stream));
}

int vlpk_encoder_bwd(const VlpkShape* s, int n_layers, const VlpkLayerWeights* w, const void* x, const uint32_t* mask_bits, int mask_rows,
                     const VlpkLayerActs* acts, const void* const* dys, void* dx0, const VlpkLayerGrads* grads, const VlpkBwdScratch* ws,
                     float p_attn, float p_hidden, const VlpkDropout* drop, void* stream) {
  VLPK_TRY(check_shape(s));
  VLPK_CHECK_ARG(n_layers > 0 && w && x && mask_bits && acts && dys && dx0 && grads && ws, "encoder_bwd: null pointer");
  VLPK_CHECK_ARG(dys[n_layers - 1] != nullptr, "encoder_bwd: gradient of the last layer output is required");
  cudaStream_t st = S(stream);
  const long long n = static_cast<long long>(s->B) * s->Lq * s->H;
  // The inter-layer gradient lives in ws->dx.  layer_bwd may run in place (dx == dy): dy is consumed
  // entirely by its first kernel (LN2 backward) and dx is written only by its last (QKV dgrad).
  const void* cur_dy = dys[n_layers - 1];
  for (int i = n_layers - 1; i >= 0; --i) {
    void* out = (i == 0) ? dx0 : ws->dx;
    const void* xin = (i == 0) ? x : acts[i - 1].y;
    VLPK_TRY(layer_bwd_impl(s, &w[i], xin, mask_bits, mask_rows, &acts[i], cur_dy, out, &grads[i], ws, p_attn, p_hidden, drop, i, st));
    if (i > 0 && dys[i - 1] != nullptr) {
      LaunchScope scope(CAT_MISC, 6.0 * n, st);
      add_bf16_kernel<<<static_cast<unsigned>(((n + 7) / 8 + 255) / 256), 256, 0, st>>>(static_cast<bf16*>(out), static_cast<const bf16*>(out),
                                                                                     static_cast<const bf16*>(dys[i - 1]), n);
      VLPK_CUDA(cudaGetLastError());
    }
    cur_dy = out;
  }
  return 0;
}

int vlpk_decoder_ce_fwd(int R, int V, int H, const void* h, const void* w, const void* bias_pad, const int64_t* labels, void* logits,
                        float* lse, float* loss, void* stream) {
  DecoderCeArgs a;
  a.R = R; a.V = V; a.H = H;
  a.h = h; a.w = w; a.bias_pad = bias_pad;
  a.labels = reinterpret_cast<const long long*>(labels);
  a.logits = logits; a.dlogits = logits;  // (alignment check only)
  a.lse = lse; a.loss = loss;
  return launch_decoder_ce_fwd(a, S(stream));
}

int vlpk_decoder_ce_bwd(int R, int V, int H, const void* h, const void* w, const int64_t* labels, const void* logits, const float* lse,
                        const float* dloss, void* dlogits, float* dh, void* dw, float* dbias, void* stream) {
  DecoderCeArgs a;
  a.R = R; a.V = V; a.H = H;
  a.h = h; a.w = w;
  a.labels = reinterpret_cast<const long long*>(labels);
  a.logits = const_cast<void*>(logits);
  a.lse = const_cast<float*>(lse);
  a.dloss = dloss; a.dlogits = dlogits; a.dh = dh; a.dw = dw; a.dbias = dbias;
  return launch_decoder_ce_bwd(a, S(stream));
}

int vlpk_decoder_ce_ls_fwd(int R, int V, int H, float eps, const void* h, const void* w, const void* bias_pad, const int64_t* labels,
                           void* logits, float* lse, float* loss, void* stream) {
  VLPK_CHECK_ARG(eps > 0.f && eps <= 1.f && V >= 3, "decoder_ce_ls: label smoothing %g with V=%d (needs 0 < eps <= 1, V >= 3)",
                 static_cast<double>(eps), V);
  DecoderCeArgs a;
  a.R = R; a.V = V; a.H = H; a.eps = eps;
  a.h = h; a.w = w; a.bias_pad = bias_pad;
  a.labels = reinterpret_cast<const long long*>(labels);
  a.logits = logits; a.dlogits = logits;  // (alignment check only)
  a.lse = lse; a.loss = loss;
  return launch_decoder_ce_fwd(a, S(stream));
}

int vlpk_decoder_ce_ls_bwd(int R, int V, int H, float eps, const void* h, const void* w, const int64_t* labels, const void* logits,
                           const float* lse, const float* dloss, void* dlogits, float* dh, void* dw, float* dbias, void* stream) {
  VLPK_CHECK_ARG(eps > 0.f && eps <= 1.f && V >= 3, "decoder_ce_ls: label smoothing %g with V=%d (needs 0 < eps <= 1, V >= 3)",
                 static_cast<double>(eps), V);
  DecoderCeArgs a;
  a.R = R; a.V = V; a.H = H; a.eps = eps;
  a.h = h; a.w = w;
  a.labels = reinterpret_cast<const long long*>(labels);
  a.logits = const_cast<void*>(logits);
  a.lse = const_cast<float*>(lse);
  a.dloss = dloss; a.dlogits = dlogits; a.dh = dh; a.dw = dw; a.dbias = dbias;
  return launch_decoder_ce_bwd(a, S(stream));
}

int vlpk_bertadam_chunk(void) { return ADAM_CHUNK; }

int vlpk_bertadam_step(const VlpkAdamTensor* tensors_host, const VlpkAdamTensor* tensors_dev, const int32_t* chunk_prefix_host,
                       const int32_t* chunk_prefix_dev, int n_tensors, float* sqnorm_dev, double lr_scheduled, double b1, double b2,
                       double eps, double max_grad_norm, void* stream) {
  VLPK_CHECK_ARG(b1 >= 0.0 && b1 < 1.0 && b2 >= 0.0 && b2 < 1.0 && eps >= 0.0, "bertadam: b1=%g b2=%g eps=%g out of range", b1, b2, eps);
  AdamHyper h;
  h.lr = static_cast<float>(lr_scheduled);
  h.b1 = static_cast<float>(b1); h.omb1 = static_cast<float>(1.0 - b1);
  h.b2 = static_cast<float>(b2); h.omb2 = static_cast<float>(1.0 - b2);
  h.eps = static_cast<float>(eps);
  h.max_grad_norm = static_cast<float>(max_grad_norm);
  return launch_bertadam(tensors_host, tensors_dev, chunk_prefix_host, chunk_prefix_dev, n_tensors, sqnorm_dev, h, S(stream));
}

void vlpk_profile_enable(int on) { prof_enable(on != 0); }
void vlpk_profile_reset(void) { prof_reset(); }
int vlpk_profile_get(int cat, double* ms, double* work, int64_t* launches) {
  long long n = 0;
  const int rc = prof_get(cat, ms, work, &n);
  *launches = n;
  return rc;
}
int64_t vlpk_launch_count(void) { return launch_count(); }

int vlpk_f32_to_bf16(const float* src, void* dst, int64_t n, void* stream) { return launch_f32_to_bf16(src, dst, n, S(stream)); }

int vlpk_debug_dropout_mask(const VlpkDropout* drop, uint64_t site, int64_t n, unsigned char* out, void* stream) {
  VLPK_CHECK_ARG(drop != nullptr && out != nullptr, "dropout_mask: null pointer");
  return launch_dropout_mask(mk_drop(drop, drop->p, site), n, out, S(stream));
}

int vlpk_beam_ngram_block(int rows, int K, int f, int T_cap, int n, const int32_t* hist_in, int32_t* hist_out, const int64_t* ptr,
                          const int64_t* wid, const int32_t* ignore, int n_ignore, float* logp, int64_t ld, int V, void* stream) {
  NgramBlockArgs a;
  a.rows = rows; a.K = K; a.f = f; a.T_cap = T_cap; a.n = n;
  a.hist_in = hist_in; a.hist_out = hist_out;
  a.ptr = reinterpret_cast<const long long*>(ptr); a.wid = reinterpret_cast<const long long*>(wid);
  a.ignore = ignore; a.n_ignore = n_ignore;
  a.logp = logp; a.ld = ld; a.V = V;
  return launch_beam_ngram_block(a, S(stream));
}

int vlpk_sample_tokens(int rows, int V, const void* logits, int64_t ld, const void* bias, int fp32, int mode, int topk, float topp,
                       uint64_t seed, int f, int64_t* seq, int T_cap, float* score, int32_t* finished, int32_t* live, int eos_id, int pad_id,
                       int block_eos, int n, const int32_t* ignore, int n_ignore, void* stream) {
  SampleArgs a;
  a.rows = rows; a.V = V; a.logits = logits; a.ld = ld; a.bias = bias; a.fp32 = fp32;
  a.mode = mode; a.topk = topk; a.topp = topp; a.seed = seed;
  a.f = f; a.seq = reinterpret_cast<long long*>(seq); a.T_cap = T_cap; a.score = score;
  a.finished = finished; a.live = live; a.eos_id = eos_id; a.pad_id = pad_id; a.block_eos = block_eos;
  a.n = n; a.ignore = ignore; a.n_ignore = n_ignore;
  return launch_sample(a, S(stream));
}

int vlpk_diverse_beam_step(int B, int K, int G, int f, int V, const void* logits, int64_t ld, const void* bias, int fp32, float diversity_penalty,
                           int eos_id, int block_eos, int T_cap, int n, const int32_t* hist_in, int32_t* hist_out, const int32_t* ignore,
                           int n_ignore, const int64_t* prev_wid, const int64_t* prev_ptr, const float* prev_score, const float* prev_eos,
                           int32_t* top_w, float* top_lp, int64_t* wid, int64_t* ptr, float* score, float* eos, void* stream) {
  DiverseBeamArgs a;
  a.B = B; a.K = K; a.G = G; a.f = f; a.V = V;
  a.logits = logits; a.ld = ld; a.bias = bias; a.fp32 = fp32;
  a.lambda = diversity_penalty; a.eos_id = eos_id; a.block_eos = block_eos;
  a.T_cap = T_cap; a.n = n; a.hist_in = hist_in; a.hist_out = hist_out; a.ignore = ignore; a.n_ignore = n_ignore;
  a.prev_wid = reinterpret_cast<const long long*>(prev_wid); a.prev_ptr = reinterpret_cast<const long long*>(prev_ptr);
  a.prev_score = prev_score; a.prev_eos = prev_eos;
  a.top_w = top_w; a.top_lp = top_lp;
  a.wid = reinterpret_cast<long long*>(wid); a.ptr = reinterpret_cast<long long*>(ptr); a.score = score; a.eos = eos;
  return launch_diverse_beam_step(a, S(stream));
}

int vlpk_constrained_beam_step(const VlpkConstrainedBeamArgs* args, void* stream) {
  VLPK_CHECK_ARG(args, "constrained_beam_step: null argument struct");
  return launch_constrained_beam_step(*args, S(stream));
}

static PromptRows prompt_rows(const VlpkPromptRows& p) {
  PromptRows r;
  r.hist_off = p.hist_off;
  r.eos_until = p.eos_until;
  return r;
}

int vlpk_sample_tokens_prompt(int rows, int V, const void* logits, int64_t ld, const void* bias, int fp32, int mode, int topk, float topp,
                              uint64_t seed, int f, int64_t* seq, int T_cap, float* score, int32_t* finished, int32_t* live, int eos_id,
                              int pad_id, int n, const int32_t* ignore, int n_ignore, const VlpkPromptRows* prompt, void* stream) {
  VLPK_CHECK_ARG(prompt, "sample_tokens_prompt: null prompt rows");
  SampleArgs a;
  a.rows = rows; a.V = V; a.logits = logits; a.ld = ld; a.bias = bias; a.fp32 = fp32;
  a.mode = mode; a.topk = topk; a.topp = topp; a.seed = seed;
  a.f = f; a.seq = reinterpret_cast<long long*>(seq); a.T_cap = T_cap; a.score = score;
  a.finished = finished; a.live = live; a.eos_id = eos_id; a.pad_id = pad_id;
  a.n = n; a.ignore = ignore; a.n_ignore = n_ignore;
  const PromptRows p = prompt_rows(*prompt);
  return launch_sample(a, S(stream), &p);
}

int vlpk_diverse_beam_step_prompt(int B, int K, int G, int f, int V, const void* logits, int64_t ld, const void* bias, int fp32,
                                  float diversity_penalty, int eos_id, int T_cap, int n, const int32_t* hist_in, int32_t* hist_out,
                                  const int32_t* ignore, int n_ignore, const int64_t* prev_wid, const int64_t* prev_ptr,
                                  const float* prev_score, const float* prev_eos, int32_t* top_w, float* top_lp, int64_t* wid, int64_t* ptr,
                                  float* score, float* eos, const VlpkPromptRows* prompt, void* stream) {
  VLPK_CHECK_ARG(prompt, "diverse_beam_step_prompt: null prompt rows");
  DiverseBeamArgs a;
  a.B = B; a.K = K; a.G = G; a.f = f; a.V = V;
  a.logits = logits; a.ld = ld; a.bias = bias; a.fp32 = fp32;
  a.lambda = diversity_penalty; a.eos_id = eos_id;
  a.T_cap = T_cap; a.n = n; a.hist_in = hist_in; a.hist_out = hist_out; a.ignore = ignore; a.n_ignore = n_ignore;
  a.prev_wid = reinterpret_cast<const long long*>(prev_wid); a.prev_ptr = reinterpret_cast<const long long*>(prev_ptr);
  a.prev_score = prev_score; a.prev_eos = prev_eos;
  a.top_w = top_w; a.top_lp = top_lp;
  a.wid = reinterpret_cast<long long*>(wid); a.ptr = reinterpret_cast<long long*>(ptr); a.score = score; a.eos = eos;
  const PromptRows p = prompt_rows(*prompt);
  return launch_diverse_beam_step(a, S(stream), &p);
}

int vlpk_constrained_beam_step_prompt(const VlpkConstrainedBeamArgs* args, const VlpkPromptRows* prompt, void* stream) {
  VLPK_CHECK_ARG(args && prompt, "constrained_beam_step_prompt: null argument struct");
  const PromptRows p = prompt_rows(*prompt);
  return launch_constrained_beam_step(*args, S(stream), &p);
}

int vlpk_colsum(const void* x, int64_t ld, int64_t M, int N, float* out, void* stream) {
  VLPK_CHECK_ARG(x && out, "colsum: null pointer");
  return launch_colsum(x, ld, M, N, out, S(stream));
}

int vlpk_add_bf16(void* dst, const void* a, const void* b, int64_t n, void* stream) {
  VLPK_CHECK_ARG(dst && a && b, "add_bf16: null pointer");
  if (n <= 0) return 0;
  LaunchScope scope(CAT_MISC, 6.0 * n, S(stream));
  add_bf16_kernel<<<static_cast<unsigned>(((n + 7) / 8 + 255) / 256), 256, 0, S(stream)>>>(static_cast<bf16*>(dst), static_cast<const bf16*>(a),
                                                                                        static_cast<const bf16*>(b), n);
  VLPK_CUDA(cudaGetLastError());
  return 0;
}

int vlpk_gemm(int M, int N, int K, int a_mn, const void* A, int64_t lda, int b_mn, const void* B, int64_t ldb, const void* bias, void* D0,
              int64_t ldd0, void* D1, int64_t ldd1, const void* aux, int64_t ld_aux, int epi, int splits, int bn, void* stream) {
  VLPK_CHECK_ARG(A && B && D0, "gemm: null pointer");
  GemmDesc g;
  g.M = M; g.N = N; g.K = K;
  g.a_mn = a_mn != 0; g.A = A; g.lda = lda;
  g.b_mn = b_mn != 0; g.B[0] = B; g.ldb = ldb; g.nseg = 1;
  g.bias[0] = static_cast<const bf16*>(bias);
  g.D0 = D0; g.ldd0 = ldd0; g.D1 = D1; g.ldd1 = ldd1;
  g.aux = static_cast<const bf16*>(aux); g.ld_aux = ld_aux;
  g.epi = epi; g.splits = splits; g.bn = bn;
  if (deterministic() && epi == EPI_REDUCE_F32) return launch_gemm_split_slices(g, SCRATCH_SPLITK, S(stream));
  return launch_gemm(g, S(stream));
}

}  // extern "C"
#pragma GCC visibility pop
