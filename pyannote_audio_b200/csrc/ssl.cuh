// SSeRiouSS segmentation (models/segmentation/SSeRiouSS.py): the WavLM Base front end (torchaudio's wav2vec2
// components with WavLM attention) -> the PyanNet BiLSTM stack, linear layers and classifier of seg_lstm.cu.
#pragma once
#include "common.cuh"
#include "seg.cuh"

namespace b200 {

constexpr int kSslMinWindow = 400;    // receptive field of one frame: the shortest window
constexpr int kSslLayers = 12;
constexpr int kSslDim = 768;
constexpr int kSslHeads = 12;
constexpr int kSslFfn = 3072;
constexpr int kSslConvDim = 512;
constexpr int kSslPosK = 128;         // positional conv kernel (padding 64, last frame dropped)
constexpr int kSslPosGroups = 16;
constexpr int kSslRelSpan = 1023;     // relative offsets |j - i| above this share the bucket of 1023 (saturated)

// Frame counts of the conv feature extractor on a window of W samples: conv 0 (k 10, s 5), convs 1-4 (k 3, s 2),
// convs 5-6 (k 2, s 2).  Conv l's output of window b lives in rows [b * stride[l], b * stride[l] + len[l]) of its
// buffer; stride[0] is a multiple of 64, so every stride is even and two consecutive frames of a window form one
// contiguous 1024-wide row of the next conv's implicit GEMM.
struct SslGeom {
  int W, len[7], stride[7];
  int T;                              // output frames (len[6])
};
inline SslGeom ssl_geom(int W) {
  SslGeom g;
  g.W = W;
  g.len[0] = 1 + (W - 10) / 5;
  for (int l = 1; l < 7; ++l) g.len[l] = 1 + (g.len[l - 1] - (l <= 4 ? 3 : 2)) / 2;
  g.stride[0] = (g.len[0] + 63) / 64 * 64;
  for (int l = 1; l < 7; ++l) g.stride[l] = g.stride[l - 1] / 2;
  g.T = g.len[6];
  return g;
}

struct SslLayerWeights {
  __half *qkv_hi = nullptr, *qkv_lo = nullptr;   // attention.attention.in_proj_weight [2304][768]
  float* qkv_b = nullptr;
  __half *out_hi = nullptr, *out_lo = nullptr;   // attention.attention.out_proj [768][768]
  float* out_b = nullptr;
  float* gru_w = nullptr;                        // attention.gru_rel_pos_linear.weight [8][64]
  float* gru_b = nullptr;                        // [8]
  float* gru_const = nullptr;                    // attention.gru_rel_pos_const [12]
  float *ln1_w = nullptr, *ln1_b = nullptr;      // layer_norm [768]
  __half *ff1_hi = nullptr, *ff1_lo = nullptr;   // feed_forward.intermediate_dense [3072][768]
  float* ff1_b = nullptr;
  __half *ff2_hi = nullptr, *ff2_lo = nullptr;   // feed_forward.output_dense [768][3072]
  float* ff2_b = nullptr;
  float *ln2_w = nullptr, *ln2_b = nullptr;      // final_layer_norm [768]
};

struct SslWeights {
  bool loaded = false;
  float* conv0_w = nullptr;                      // [512][10]
  float *gn_w = nullptr, *gn_b = nullptr;        // conv_layers.0.layer_norm (GroupNorm(512, 512)) [512]
  __half *conv_hi[6] = {}, *conv_lo[6] = {};     // convs 1-6 as [512][taps x 1024] (see ssl_wavlm.cu)
  float *fp_ln_w = nullptr, *fp_ln_b = nullptr;  // feature_projection.layer_norm [512]
  __half *proj_hi = nullptr, *proj_lo = nullptr; // feature_projection.projection [768][512]
  float* proj_b = nullptr;
  __half *pos_hi = nullptr, *pos_lo = nullptr;   // [16 groups][128 n (48 real)][128 taps x 64 c (48 real)]
  float* pos_b = nullptr;                        // [16][128] (48 real per group)
  float *enc_ln_w = nullptr, *enc_ln_b = nullptr; // encoder.transformer.layer_norm [768]
  float* rel_tab = nullptr;                      // [12 heads][2 * 1023 + 1]: rel_attn_embed of the offset's bucket
  int num_layers = kSslLayers;                   // layers run (12, or wav2vec_layer)
  SslLayerWeights layer[kSslLayers];
  float layer_w[kSslLayers] = {};                // softmax(wav2vec_weights), or 1 for the selected layer
  SegWeights head;                               // BiLSTM (k_in[0] = 768), linear layers, classifier
};

size_t ssl_workspace_bytes(const SslGeom& g, int NB);
// WavLM Base features of NB windows: x0 [NB][T][768] fp32 (the layer average SSeRiouSS feeds its LSTM)
int ssl_frontend_forward(const SslWeights& W, const SslGeom& g, const float* wav, const long long* chunk_off,
                         const int* chunk_valid, int NB, void* ws, float* x0, int num_sms, cudaStream_t stream);

}  // namespace b200
