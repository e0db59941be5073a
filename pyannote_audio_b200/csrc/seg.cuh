// Segmentation path (PyanNet: SincNet front-end -> 4x BiLSTM -> Linear x2 -> classifier -> powerset argmax or sigmoid).
#pragma once
#include "../../include/b200diar.h"
#include "common.cuh"

namespace b200 {

// Intermediates copied out after each stage (b200_seg_stages / b200_seg_head_stages); the forward passes null
using SegCapture = b200_seg_capture;
// D2D copy of `bytes` from src into dst when dst is not null
int capture(void* dst, const void* src, size_t bytes, cudaStream_t stream);

// Per-stage lengths of PyanNet on a window of W samples (models/blocks/sincnet.py:163-184): sinc conv (K 251,
// stride 10), MaxPool 3, Conv1d 5, MaxPool 3, Conv1d 5, MaxPool 3.  W = 160000 gives the kSincLen .. kPool2 constants.
constexpr int kSegMinWindow = 1261;  // shortest window with 2 frames (one frame cannot be instance-normalised)
constexpr int kSegTileP = 64;        // pooled outputs per SincNet tile
struct SegGeom {
  int W, sinc_len, pool0, conv1_len, pool1, conv2_len, pool2;
  int tiles0, tiles1, tiles2;        // ceil(pool / 64): tiles (and InstanceNorm partial sums) per stage
};
inline SegGeom seg_geom(int W) {
  SegGeom g;
  g.W = W;
  g.sinc_len = 1 + (W - kSincK) / kSincStride;
  g.pool0 = g.sinc_len / 3;
  g.conv1_len = g.pool0 - 4;
  g.pool1 = g.conv1_len / 3;
  g.conv2_len = g.pool1 - 4;
  g.pool2 = g.conv2_len / 3;
  g.tiles0 = (g.pool0 + kSegTileP - 1) / kSegTileP;
  g.tiles1 = (g.pool1 + kSegTileP - 1) / kSegTileP;
  g.tiles2 = (g.pool2 + kSegTileP - 1) / kSegTileP;
  return g;
}

// SincNet front end (models/blocks/sincnet.py:41-79), shared by PyanNet and XVectorSincNet
struct SincNetWeights {
  float wav_w = 1.f, wav_b = 0.f;   // sincnet.wav_norm1d affine
  __half* sinc_wg_hi = nullptr;     // [80 filters][256 taps] fp16 (hi, lo) for the wgmma sinc layer (taps >= 251 zero)
  __half* sinc_wg_lo = nullptr;
  float* sinc_f = nullptr;          // [126][80]: half filters (k=0..124) + centre tap (k=125); cos ch 0..39, sin 40..79
  float* in_gamma[3] = {nullptr, nullptr, nullptr};   // sincnet.norm1d.{0,1,2}.weight
  float* in_beta[3] = {nullptr, nullptr, nullptr};
  float* conv_w[2] = {nullptr, nullptr};   // [CIN][5][60]
  float* conv_b[2] = {nullptr, nullptr};   // [60]
  __half* conv_wg_hi[2] = {nullptr, nullptr};   // [64 rows = c_out (60 real)][5 taps x Cpad channels] fp16 (hi, lo)
  __half* conv_wg_lo[2] = {nullptr, nullptr};
};

// classifier heads (models/segmentation/PyanNet.py:152-161, core/model.py:271-300): Linear(128, K) then log-softmax
// (mono-label / powerset problems) or sigmoid (binary / multi-label problems)
constexpr int kSegLogSoftmax = 0;
constexpr int kSegSigmoid = 1;
constexpr int kSegMaxClasses = 32;

struct SegWeights {
  bool loaded = false;
  int lstm_layers = 4;
  int num_classes = kClasses;       // K, 1 .. kSegMaxClasses
  int activation = kSegLogSoftmax;
  SincNetWeights sinc;
  // LSTM, per layer: W_ih for both directions [1024][Kpad] with row = dir*512 + unit*4 + gate; bias = b_ih+b_hh
  float* w_ih[8] = {};
  float* b_g[8] = {};
  int k_in[8] = {};                 // padded input size (64, 256, ...)
  float* w_hh[8] = {};              // [2 dir][2 rank][128 k][256]  (smem image of the SIMT recurrent kernel)
  __half* w_hh_hi[8] = {};          // [2 dir][2 rank][256 = 32 jj + 8 gate + u][128 k] fp16 (hi, lo), seg_lstm_wg.cu
  __half* w_hh_lo[8] = {};
  // fp16 (hi, lo) splits of the GEMM weights for the tensor-core path (gemm_tc.cu)
  __half* w_ih_hi[8] = {};
  __half* w_ih_lo[8] = {};
  __half* lin_w_hi[2] = {nullptr, nullptr};
  __half* lin_w_lo[2] = {nullptr, nullptr};
  float* lin_w[2] = {nullptr, nullptr};   // [128][256], [128][128]
  float* lin_b[2] = {nullptr, nullptr};
  float* cls_w = nullptr;           // [K][128]
  float* cls_b = nullptr;           // [K]
};

int sgemm_nt(const float* A, int lda, const float* Bw, int ldb, float* C, int ldc, const float* bias, int M, int N,
             int K, int act, cudaStream_t stream);

// Implicit-GEMM extension of gemm_tc_split (TDNN layers of XVectorSincNet): A is [M][Cpad] with Cpad = K / taps,
// output row r reads A rows r + j * dil for the taps j = 0 .. taps - 1 (K ordered tap-major), and the epilogue
// applies y = act(acc + bias) * scale + shift per column (eval-mode BatchNorm after the activation) when scale != NULL.
struct GemmTaps {
  int taps = 1, dil = 0;
  const float* scale = nullptr;
  const float* shift = nullptr;
};
// split-precision tensor-core GEMM (gemm_tc.cu): C = act(A B^T + bias), A/B as fp16 (hi, lo) pairs
int gemm_tc_split(const __half* A_hi, const __half* A_lo, int lda, const __half* B_hi, const __half* B_lo, int ldb,
                  float* C, int ldc, __half* C_hi, __half* C_lo, int ldc_h, const float* bias, int M, int N, int K,
                  int act, int num_sms, cudaStream_t stream, float* const* C_peers = nullptr, int n_peers = 0,
                  const GemmTaps& taps = GemmTaps());
int split_f16(const float* x, __half* hi, __half* lo, size_t n, cudaStream_t st);
// tensor-core recurrence (seg_lstm_wg.cu): Gx [NB][T][1024] -> layer output as fp16 (hi, lo) [NB][T][256].  impl 1:
// two warpgroups per CTA with Gx software-pipelined into registers; 2: one warpgroup per CTA, bit-identical to 1
int lstm_rec_wg(const float* Gx, const __half* Wh, const __half* Wl, __half* Yh, __half* Yl, int NB, int T, int impl,
                cudaStream_t stream);

// SincNet layers on the tensor cores (seg_conv_wg.cu); same outputs and partial sums as the fp32 twins.  impl 1:
// persistent, weight-resident kernels; 2: one CTA per tile, bit-identical to 1
int sinc_wg_forward(const SegGeom& g, const float* wav, const long long* chunk_off, const int* chunk_valid,
                    const float2* affine, const __half* Wh, const __half* Wl, int NB, float* P0, double2* part,
                    int impl, cudaStream_t stream);
int conv5_wg_forward(const SegGeom& g, int layer, const float* Pin, const float2* affine, const __half* Wh,
                     const __half* Wl, const float* bias, int NB, float* Pout, double2* part, int impl,
                     cudaStream_t stream);

// SincNet front-end on NB windows of g.W samples: wav + per-window (offset, valid) -> X0 [NB][g.pool2][64] fp32
// (60 features + 4 zero pad)
size_t sincnet_workspace_bytes(const SegGeom& g, int NB);
int sincnet_forward(const SincNetWeights& W, const SegGeom& g, const float* wav, const long long* chunk_off,
                    const int* chunk_valid, int NB, void* ws, float* x0, int conv_impl, cudaStream_t stream,
                    const SegCapture* cap = nullptr);

// Outputs of the classifier, written straight to the caller's buffers.  Log-softmax heads: cls [NB][T] u8 (+ optional
// logp [NB][T][K]); sigmoid heads: scores [NB][T][K] and / or max_scores [NB][T] (either may be null).
struct SegHeadOut {
  unsigned char* cls = nullptr;
  float* logp = nullptr;
  float* scores = nullptr;
  float* max_scores = nullptr;
};
// BiLSTM stack + linear layers + classifier on sequences of T frames of k0 = W.k_in[0] features (64: PyanNet's 60
// SincNet features and 4 zero columns; 768: SSeRiouSS)
size_t lstm_workspace_bytes(int NB, int T, int k0);
int lstm_head_forward(const SegWeights& W, const float* x0, int NB, int T, void* ws, const SegHeadOut& out,
                      int num_sms, int gemm_impl, int rec_impl, cudaStream_t stream, const SegCapture* cap = nullptr);

}  // namespace b200
