// vlp_b200 — host-side description of one wgmma GEMM launch (see gemm.cu).
#pragma once
#include "common.cuh"

namespace vlpk {

// Epilogue variants.  Every Linear on the VLP hot path is D = A * B^T (+bias) followed by a cheap
// pointwise op; fusing it here removes the reference's separate elementwise passes
// (SURVEY.md §6: 66 % of reference self-time is unfused elementwise glue).
enum Epi : int {
  EPI_STORE = 0,       // D0 = acc (+ bias)
  EPI_GELU = 1,        // u = acc + bias ; D0 = gelu'(u) ; D1 = gelu(u)    (modeling.py:340-343, 62-67)
  EPI_RELU = 2,        // D0 = dropout(relu(acc + bias))                   (modeling.py:1003-1018)
  EPI_ADD = 3,         // D0 = acc + aux                                   (dgrad + residual-branch gradient)
  EPI_MUL = 4,         // D0 = acc * aux                                   (dgrad through GELU: aux = saved gelu'(u))
  EPI_DRELU = 5,       // D0 = acc * (aux > 0) * relu_scale                (dgrad through ReLU(+dropout))
  EPI_REDUCE_F32 = 6,  // D0(fp32) += acc   via TMA reduce-add (split-K weight gradients)
};

struct GemmDesc {
  int M = 0, N = 0, K = 0;  // logical problem: D[M,N] = sum_k A[m,k] * B[n,k]
  // A storage.  a_mn=false: row-major [M,K] (K contiguous).  a_mn=true: row-major [K,M] (M contiguous).
  bool a_mn = false;
  const void* A = nullptr;
  int64_t lda = 0;
  // B storage: nseg matrices stacked along B's slow dimension.
  //   b_mn=false: each segment row-major [seg_rows, K]  (segments tile N)
  //   b_mn=true : each segment row-major [seg_rows, N]  (segments tile K)
  bool b_mn = false;
  int nseg = 1;
  const void* B[3] = {nullptr, nullptr, nullptr};
  int64_t ldb = 0;
  int b_seg_rows = 0;
  int b_rows = 0;  // nseg == 1 only: rows that really exist in B's slow dimension (0 = all N resp. K); the rest is zero-filled by TMA
  const __nv_bfloat16* bias[3] = {nullptr, nullptr, nullptr};  // per N-segment (b_mn=false only)
  void* D0 = nullptr;
  int64_t ldd0 = 0;
  void* D1 = nullptr;
  int64_t ldd1 = 0;
  const __nv_bfloat16* aux = nullptr;  // [M,N] row-major side input for ADD / DGELU / DRELU
  int64_t ld_aux = 0;
  int epi = EPI_STORE;
  float relu_scale = 1.0f;  // EPI_DRELU: 1/(1-p) of the forward dropout
  DropoutCfg drop = {0.f, 1.f, 0u, 0ull, 0ull, nullptr};
  float* colsum = nullptr;  // optional [N] fp32: += column sums of the output (bias gradient of a dgrad output)
  int splits = 1;  // split-K (EPI_REDUCE_F32 only); 0 = choose automatically
  // EPI_REDUCE_F32: 0 = every split reduce-adds into D0 (the order of the additions varies from run to run); > 0 = split s adds
  // into its own slice D0 + s * split_stride (zeroed by the caller), which the caller then sums in a fixed order
  int64_t split_stride = 0;
  int bn = 0;      // tile N (0 = auto; 128 is the only width)
};

// Returns 0 on success, <0 on argument error, >0 cudaError_t.  Message via vlpk::set_error.
int launch_gemm(const GemmDesc& g, cudaStream_t stream);
int plan_gemm(const GemmDesc& g, int* bn_out, int* splits_out);
// EPI_REDUCE_F32 with the split count plan_gemm picks, summed in a fixed order: with more than one split, each split reduce-adds
// into its own zeroed slice of scratch slot `slot` and the slices are then added to D0 (fp32, +=, ldd0 == N) in split order.
int launch_gemm_split_slices(GemmDesc g, int slot, cudaStream_t stream);

}  // namespace vlpk
