// vlp_b200 — masked-LM head tail: tied-decoder logits -> per-position cross-entropy, forward and backward (see head.cu).
#pragma once
#include "common.cuh"

namespace vlpk {

struct DecoderCeArgs {
  int R = 0;  // positions (B * max_pred)
  int V = 0;  // vocabulary (decoder rows); logits are stored with leading dimension Vp = round_up(V, 8)
  int H = 0;
  const void* h = nullptr;            // [R,H]  bf16 transformed hidden states
  const void* w = nullptr;            // [V,H]  bf16 tied decoder weight (= word embeddings), read in place
  const void* bias_pad = nullptr;     // [Vp]   bf16 output bias, zero padded
  const long long* labels = nullptr;  // [R]    target ids; outside [0,V) = ignored position (loss 0, no gradient)
  void* logits = nullptr;             // [R,Vp] bf16
  float* lse = nullptr;               // [R]
  float* loss = nullptr;              // [R]
  // backward
  const float* dloss = nullptr;  // [R]
  void* dlogits = nullptr;       // [R,Vp] bf16 (pad columns written as 0)
  float* dh = nullptr;           // [R,H]  fp32, zeroed by the caller (split-K reduce-add target)
  void* dw = nullptr;            // [V,H]  bf16, overwritten
  float* dbias = nullptr;        // [Vp]   fp32, zeroed by the caller
  // label smoothing (LabelSmoothingLoss, ignore index 0): 0 = plain cross-entropy; otherwise eps in (0, 1] and V >= 3, the target
  // is q_0 = 0, q_label = 1 - eps, q_j = eps / (V - 2) elsewhere, and label 0 is an ignored position as well
  float eps = 0.f;
};

int launch_decoder_ce_fwd(const DecoderCeArgs& a, cudaStream_t s);
int launch_decoder_ce_bwd(const DecoderCeArgs& a, cudaStream_t s);

}  // namespace vlpk
