// extern "C" surface of libb200diar.so (declared in include/b200diar.h): context, weight ingestion
// (BN folding, layout transforms, fp16 conversion on the host), and the forward entry points.
#include "../../include/b200diar.h"
#include "audio.cuh"
#include "cluster.cuh"
#include "common.cuh"
#include "emb.cuh"
#include "post.cuh"
#include "seg.cuh"
#include "ssl.cuh"
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstdlib>

using namespace b200;

// XVectorSincNet (models/embedding/xvector.py:205-349) and XVectorMFCC (xvector.py:42-202): a front end (SincNet or
// MFCC), five TDNN layers (Conv1d -> LeakyReLU -> eval BatchNorm1d) as implicit GEMMs on gemm_tc_split, statistics
// pooling and the embedding Linear
constexpr int kXvecLayers = 5;
constexpr int kXvecMinSamples = 4771;       // 15 SincNet frames: the TDNN stack (receptive field 15) gives one frame
constexpr int kXvecMfccMinSamples = 2800;   // 15 MFCC frames
constexpr int kXvecStatsLd = 3008;          // 2 x 1500 statistics, padded to whole 64-wide k-blocks
struct XvecWeights {
  bool loaded = false;
  SincNetWeights sinc;              // front end of the XVectorSincNet slot
  MfccWeights mfcc;                 // front end of the XVectorMFCC slot
  int taps[kXvecLayers] = {5, 3, 3, 1, 1}, dil[kXvecLayers] = {1, 2, 3, 1, 1};
  int cin_pad[kXvecLayers] = {64, 512, 512, 512, 512}, cout_pad[kXvecLayers] = {512, 512, 512, 512, 1536};
  __half* w_hi[kXvecLayers] = {};   // [cout_pad][taps x cin_pad] fp16 (hi, lo), k = tap * cin_pad + c_in, zero padded
  __half* w_lo[kXvecLayers] = {};
  float* bias[kXvecLayers] = {};    // [cout_pad] conv bias
  float* scale[kXvecLayers] = {};   // [cout_pad] BN gamma / sqrt(var + eps) (0 on padded channels)
  float* shift[kXvecLayers] = {};   // [cout_pad] BN beta - mean * scale
  int dim = 512, dim_pad = 512;     // embedding dimension, rounded up to 128
  __half* emb_hi = nullptr;         // [dim_pad][3008] fp16 (hi, lo) of embedding.weight, zero padded
  __half* emb_lo = nullptr;
  float* emb_b = nullptr;           // [dim_pad]
};

struct b200_ctx {
  int device = 0;
  int num_sms = 132;
  int seg_gemm_impl = 1;   // 1 = split-fp16 wgmma GEMMs for the LSTM input projections / linear layers, 0 = fp32 SIMT
  int seg_rec_impl = 1;    // 1 = LSTM recurrence as split-fp16 wgmma on 2-CTA clusters, two warpgroups per CTA (needs
                           // seg_gemm_impl = 1), 0 = fp32 SIMT, 2 = one warpgroup per CTA (bit-exact reference of 1)
  int seg_conv_impl = 1;   // 1 = SincNet sinc / Conv1d layers as persistent split-fp16 wgmma implicit GEMMs, 0 = fp32
                           // CUDA-core twins, 2 = wgmma with one CTA per tile (bit-exact reference of 1)
  int conv_impl = 1;       // 1 = wgmma implicit-GEMM trunk convs, 0 = fp32 CUDA-core reference conv, 2 = wgmma with
                           // one weight tap per stage for every conv (bit-exact reference of 1)
  // chunks per segmentation sub-batch: 2112 = 33 recurrence tiles of 64 sequences x 2 directions x 2-CTA clusters
  // = 132 CTAs, one per SM of an H100 SXM (seg_lstm.cu launch_rec)
  int seg_max_batch = 2112;
  // chunks per embedding sub-batch: 264 = 2 x 132 SMs, so that the conv tiles of every layer (8 / 4 / 2 / 1 tiles
  // of 128 pixels per image row) split evenly over the machine
  int emb_max_batch = 264;
  // windows of 10 s per SSeRiouSS sub-batch (any window length: at most ssl_max_batch x 160000 samples); ~140 MB of
  // workspace per 10 s, most of it the conv feature extractor's channel-last activations
  int ssl_max_batch = 32;
  int fbank_share = 1;          // 1 = overlapping hop-aligned chunks share their fbank frames (emb.cuh: FbankRun)
  // smallest linkage problem that runs on the whole GPU over packed distances (cluster.cuh); at most the default, so
  // that every problem the dense one-CTA kernel cannot hold goes there
  int linkage_grid_min = kLinkGridMinDefault;
  int64_t launches = 0;
  SegWeights seg;
  EmbWeights emb;
  XvecWeights xvec, xvec_mfcc;
  SslWeights ssl;
  // device allocations holding the weights of each network
  std::vector<void*> owned_seg, owned_emb, owned_xvec, owned_xvec_mfcc, owned_ssl;
  std::vector<void*>* owned = &owned_seg;    // where upload() records allocations (set by the load entry points)
  void* ws = nullptr;
  size_t ws_cap = 0;
  long long* d_off = nullptr;
  int* d_valid = nullptr;
  int* d_frame0 = nullptr;         // first fbank row of every chunk inside its sub-batch
  b200::FbankRun* d_runs = nullptr; // fbank runs of all sub-batches, back to back
  int meta_cap = 0;
  // optional CUDA-event timers around the dominant kernels (bench.py's live roofline measurement)
  int profile = 0;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> trunk_events, seg_events;
  std::vector<cudaEvent_t> event_pool;
  int64_t trunk_segments = 0, seg_chunks = 0;
  // polyphase resampling tables, one per (orig, new) ratio seen (device copies, freed with the ctx)
  struct ResampleTable { int orig, nw, width; float* dev; };
  std::vector<ResampleTable> resample_tables;
};

namespace {

// Scope of an entry point: selects the ctx's device and binds its launch counter, which b200::launch increments, and
// restores both on exit, so that one entry point may call another.
struct CtxScope {
  int prev_device = 0;
  int64_t* prev_counter = g_launch_counter;
  explicit CtxScope(b200_ctx* ctx) {
    cudaGetDevice(&prev_device);
    cudaSetDevice(ctx->device);
    g_launch_counter = &ctx->launches;
  }
  ~CtxScope() {
    cudaSetDevice(prev_device);
    g_launch_counter = prev_counter;
  }
};

template <typename T>
int upload(b200_ctx* ctx, const std::vector<T>& h, T** out) {
  void* p = nullptr;
  B200_CUDA_OK(cudaMalloc(&p, h.size() * sizeof(T) + 16));
  B200_CUDA_OK(cudaMemcpy(p, h.data(), h.size() * sizeof(T), cudaMemcpyHostToDevice));
  ctx->owned->push_back(p);
  *out = reinterpret_cast<T*>(p);
  return B200_OK;
}

// operand of gemm_tc_split and the wgmma kernels: an fp32 array, already in its device layout with zeros in the
// padding, uploaded as fp16 (hi, lo) with hi = fp16(v), lo = fp16(v - hi)
int upload_split(b200_ctx* ctx, const std::vector<float>& h, __half** hi, __half** lo) {
  std::vector<__half> vh(h.size()), vl(h.size());
  for (size_t i = 0; i < h.size(); ++i) {
    vh[i] = __float2half(h[i]);
    vl[i] = __float2half(h[i] - __half2float(vh[i]));
  }
  int rc;
  if ((rc = upload(ctx, vh, hi))) return rc;
  return upload(ctx, vl, lo);
}

cudaEvent_t take_event(b200_ctx* ctx) {
  if (!ctx->event_pool.empty()) {
    cudaEvent_t e = ctx->event_pool.back();
    ctx->event_pool.pop_back();
    return e;
  }
  cudaEvent_t e;
  cudaEventCreate(&e);
  return e;
}

struct ScopedTimer {
  b200_ctx* ctx;
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>>* sink;
  cudaStream_t st;
  cudaEvent_t a = nullptr, b = nullptr;
  // a null sink times nothing
  ScopedTimer(b200_ctx* c, std::vector<std::pair<cudaEvent_t, cudaEvent_t>>* s, cudaStream_t stream)
      : ctx(c), sink(s), st(stream) {
    if (ctx->profile && sink) { a = take_event(ctx); b = take_event(ctx); cudaEventRecord(a, st); }
  }
  ~ScopedTimer() {
    if (ctx->profile && sink) { cudaEventRecord(b, st); sink->push_back({a, b}); }
  }
};

// a reload replaces the previous upload of the same network: free it (after the device drained) instead of leaking
void release_weights(b200_ctx* ctx, std::vector<void*>* list) {
  if (!list->empty()) cudaDeviceSynchronize();
  for (void* p : *list) cudaFree(p);
  list->clear();
  ctx->owned = list;
}

int ensure_ws(b200_ctx* ctx, size_t bytes) {
  if (bytes <= ctx->ws_cap) return B200_OK;
  if (ctx->ws) { cudaDeviceSynchronize(); cudaFree(ctx->ws); ctx->ws = nullptr; ctx->ws_cap = 0; }
  B200_CUDA_OK(cudaMalloc(&ctx->ws, bytes));
  ctx->ws_cap = bytes;
  return B200_OK;
}

int ensure_meta(b200_ctx* ctx, int n) {
  if (n <= ctx->meta_cap) return B200_OK;
  if (ctx->d_off) {
    cudaDeviceSynchronize();
    cudaFree(ctx->d_off); cudaFree(ctx->d_valid); cudaFree(ctx->d_frame0); cudaFree(ctx->d_runs);
  }
  const int cap = n + 1024;
  B200_CUDA_OK(cudaMalloc((void**)&ctx->d_off, sizeof(long long) * cap));
  B200_CUDA_OK(cudaMalloc((void**)&ctx->d_valid, sizeof(int) * cap));
  B200_CUDA_OK(cudaMalloc((void**)&ctx->d_frame0, sizeof(int) * cap));
  B200_CUDA_OK(cudaMalloc((void**)&ctx->d_runs, sizeof(b200::FbankRun) * cap));
  ctx->meta_cap = cap;
  return B200_OK;
}

int push_meta(b200_ctx* ctx, const int64_t* off, const int32_t* valid, int n, cudaStream_t st,
              int max_valid = kChunk) {
  int rc = ensure_meta(ctx, n);
  if (rc) return rc;
  for (int i = 0; i < n; ++i)
    B200_CHECK(valid[i] >= 0 && valid[i] <= max_valid && off[i] >= 0, B200_ERR_INVALID,
               "chunk %d: offset %lld / valid %d out of range", i, (long long)off[i], (int)valid[i]);
  B200_CUDA_OK(cudaMemcpyAsync(ctx->d_off, off, sizeof(long long) * n, cudaMemcpyHostToDevice, st));
  B200_CUDA_OK(cudaMemcpyAsync(ctx->d_valid, valid, sizeof(int) * n, cudaMemcpyHostToDevice, st));
  return B200_OK;
}

// fbank plan of a list of segments of `samples` samples (T0 fbank frames) processed in sub-batches of nbmax (emb.cuh:
// FbankRun): per sub-batch the runs [run_base[s], run_base[s + 1]) and the number of fbank rows; frame0 / runs go to
// the device with the segment table.  share = 0 (and every short or unaligned segment): one private run per segment,
// row0 = b * T0, limit = valid.
struct FbankPlan {
  std::vector<int> run_base, nrows;
};
void plan_fbank(const int64_t* off, const int32_t* valid, int n, int nbmax, bool share, int samples, int T0,
                std::vector<b200::FbankRun>* runs_out, std::vector<int>* frame0_out, FbankPlan* plan) {
  constexpr int kHop = 160;
  std::vector<b200::FbankRun>& runs = *runs_out;
  std::vector<int>& frame0 = *frame0_out;
  runs.clear();
  runs.reserve((size_t)n);
  frame0.assign((size_t)n, 0);
  plan->run_base.clear();
  plan->nrows.clear();
  for (int c0 = 0; c0 < n; c0 += nbmax) {
    const int nb = (n - c0) < nbmax ? (n - c0) : nbmax;
    plan->run_base.push_back((int)runs.size());
    int rows = 0, run_rows = 0;
    bool open = false;                                       // the last run is made of full segments and may be extended
    for (int b = 0; b < nb; ++b) {
      const long long o = off[c0 + b];
      const bool full = share && valid[c0 + b] == samples;
      if (full && open) {
        const long long d = o - runs.back().src;
        if (d >= 0 && d % kHop == 0 && d / kHop <= run_rows) {
          const int f0 = (int)(d / kHop);
          frame0[c0 + b] = runs.back().row0 + f0;
          if (f0 + T0 > run_rows) { rows += f0 + T0 - run_rows; run_rows = f0 + T0; }
          continue;
        }
      }
      runs.push_back(b200::FbankRun{o, rows, full ? INT_MAX : (int)valid[c0 + b]});
      frame0[c0 + b] = rows;
      rows += T0;
      run_rows = T0;
      open = full;
    }
    plan->nrows.push_back(rows);
  }
  plan->run_base.push_back((int)runs.size());
}

int push_fbank_plan(b200_ctx* ctx, const int64_t* off, const int32_t* valid, int n, int nbmax, bool share, int samples,
                    int T0, FbankPlan* plan, cudaStream_t st) {
  std::vector<b200::FbankRun> runs;
  std::vector<int> frame0;
  plan_fbank(off, valid, n, nbmax, share, samples, T0, &runs, &frame0, plan);
  B200_CUDA_OK(cudaMemcpyAsync(ctx->d_frame0, frame0.data(), sizeof(int) * n, cudaMemcpyHostToDevice, st));
  B200_CUDA_OK(cudaMemcpyAsync(ctx->d_runs, runs.data(), sizeof(b200::FbankRun) * runs.size(), cudaMemcpyHostToDevice, st));
  return B200_OK;
}

// ---- kaldi mel bank / window / twiddles (torchaudio.compliance.kaldi.get_mel_banks, _feature_window_function) ----
double mel_scale(double f) { return 1127.0 * std::log(1.0 + f / 700.0); }

int build_fbank_constants(b200_ctx* ctx) {
  EmbWeights& E = ctx->emb;
  std::vector<float> window(400);
  for (int i = 0; i < 400; ++i) window[i] = (float)(0.54 - 0.46 * std::cos(2.0 * M_PI * i / 399.0));
  std::vector<float> tw(512);
  for (int k = 0; k < 256; ++k) {
    tw[2 * k] = (float)std::cos(2.0 * M_PI * k / 512.0);
    tw[2 * k + 1] = (float)(-std::sin(2.0 * M_PI * k / 512.0));
  }
  const int nb = 80, nfft = 256;
  const double low = 20.0, high = 8000.0, bw = 16000.0 / 512.0;
  const double ml = mel_scale(low), mh = mel_scale(high), delta = (mh - ml) / (nb + 1);
  std::vector<float> w;
  std::vector<int> st(nb), ln(nb), off(nb);
  for (int b = 0; b < nb; ++b) {
    const double left = ml + b * delta, center = ml + (b + 1.0) * delta, right = ml + (b + 2.0) * delta;
    int first = -1, last = -1;
    std::vector<float> row(nfft, 0.f);
    for (int k = 0; k < nfft; ++k) {
      const double mel = mel_scale(bw * k);
      const double up = (mel - left) / (center - left), down = (right - mel) / (right - center);
      const double v = std::fmax(0.0, std::fmin(up, down));
      row[k] = (float)v;
      if (v > 0) { if (first < 0) first = k; last = k; }
    }
    if (first < 0) { first = 0; last = -1; }
    st[b] = first; ln[b] = last - first + 1; off[b] = (int)w.size();
    for (int k = first; k <= last; ++k) w.push_back(row[k]);
  }
  int rc;
  if ((rc = upload(ctx, window, &E.window))) return rc;
  if ((rc = upload(ctx, tw, &E.twiddle))) return rc;
  if ((rc = upload(ctx, w, &E.mel_w))) return rc;
  if ((rc = upload(ctx, st, &E.mel_start))) return rc;
  if ((rc = upload(ctx, ln, &E.mel_len))) return rc;
  if ((rc = upload(ctx, off, &E.mel_off))) return rc;
  return B200_OK;
}

// fold eval-mode BatchNorm2d into a conv: w' = w * g/sqrt(v+eps),  b' = beta - mean * g/sqrt(v+eps)
int make_conv(b200_ctx* ctx, const b200_conv_bn& src, int cin, int cout, int k, int stride, ConvLayer* L) {
  B200_CHECK(src.conv_weight && src.bn_weight && src.bn_bias && src.bn_mean && src.bn_var, B200_ERR_INVALID,
             "missing conv/bn tensor (cin=%d cout=%d)", cin, cout);
  L->C_in = cin; L->C_out = cout; L->ksize = k; L->stride = stride;
  std::vector<__half> w((size_t)k * k * cout * cin);
  std::vector<float> bias(cout);
  for (int co = 0; co < cout; ++co) {
    const float s = src.bn_weight[co] / std::sqrt(src.bn_var[co] + 1e-5f);
    bias[co] = src.bn_bias[co] - src.bn_mean[co] * s;
    for (int ci = 0; ci < cin; ++ci)
      for (int t = 0; t < k * k; ++t)
        w[((size_t)t * cout + co) * cin + ci] = __float2half(src.conv_weight[((size_t)co * cin + ci) * k * k + t] * s);
  }
  int rc;
  if ((rc = upload(ctx, w, &L->w))) return rc;
  if ((rc = upload(ctx, bias, &L->bias))) return rc;
  return B200_OK;
}

// the WeSpeaker stem (resnet.conv1 1 -> 32 channels, 3 x 3) with resnet.bn1 folded in, fp32 for conv1_forward
int load_stem(b200_ctx* ctx, const b200_conv_bn& s, EmbWeights* E) {
  B200_CHECK(s.conv_weight && s.bn_weight && s.bn_bias && s.bn_mean && s.bn_var, B200_ERR_INVALID, "stem missing");
  std::vector<float> cw(32 * 9), cb(32);
  for (int c = 0; c < 32; ++c) {
    const float sc = s.bn_weight[c] / std::sqrt(s.bn_var[c] + 1e-5f);
    cb[c] = s.bn_bias[c] - s.bn_mean[c] * sc;
    for (int k = 0; k < 9; ++k) cw[c * 9 + k] = s.conv_weight[c * 9 + k] * sc;
  }
  int rc;
  if ((rc = upload(ctx, cw, &E->conv1_w))) return rc;
  return upload(ctx, cb, &E->conv1_b);
}

// the WeSpeaker resnet.seg_1 Linear (K = 20 C inputs -> 256), fp32 and split for gemm_tc_split
int load_seg1(b200_ctx* ctx, const float* weight, const float* bias, size_t K, EmbWeights* E) {
  std::vector<float> sw(weight, weight + (size_t)kEmbDim * K), sb(bias, bias + kEmbDim);
  int rc;
  if ((rc = upload_split(ctx, sw, &E->seg1_w_hi, &E->seg1_w_lo))) return rc;
  if ((rc = upload(ctx, sw, &E->seg1_w))) return rc;
  return upload(ctx, sb, &E->seg1_b);
}

// the SincNet half of a loader (sincnet.wav_norm1d, the ParamSincFB bank, sincnet.norm1d.*, sincnet.conv1d.{1,2}) in
// the layouts of both implementations; PyanNet and XVectorSincNet share it
int load_sincnet(b200_ctx* ctx, float wav_w, float wav_b, const float* sinc_filters, const float* const norm_weight[3],
                 const float* const norm_bias[3], const float* const conv_weight[2], const float* const conv_bias[2],
                 SincNetWeights* out) {
  SincNetWeights& S = *out;
  S.wav_w = wav_w;
  S.wav_b = wav_b;
  int rc;
  {  // half filter bank [126][80]; the kernel relies on the (anti)symmetry of ParamSincFB filters
    B200_CHECK(sinc_filters, B200_ERR_INVALID, "sinc_filters is NULL");
    std::vector<float> f(126 * 80);
    for (int ch = 0; ch < 80; ++ch) {
      const float* r = sinc_filters + ch * 251;
      const float sign = ch < 40 ? 1.f : -1.f;
      float mx = 0.f, err = 0.f;
      for (int k = 0; k < 125; ++k) {
        mx = std::fmax(mx, std::fabs(r[k]));
        err = std::fmax(err, std::fabs(r[k] - sign * r[250 - k]));
        f[k * 80 + ch] = r[k];
      }
      if (ch >= 40) err = std::fmax(err, std::fabs(r[125]));
      B200_CHECK(err <= 1e-6f * (mx + 1e-30f) + 1e-12f, B200_ERR_INVALID,
                 "sinc filter %d is not (anti)symmetric (err %g): not a ParamSincFB bank", ch, (double)err);
      f[125 * 80 + ch] = ch < 40 ? r[125] : 0.f;
    }
    if ((rc = upload(ctx, f, &S.sinc_f))) return rc;
    std::vector<float> wg((size_t)80 * 256, 0.f);          // wgmma layout: [80][256], taps zero padded
    for (int ch = 0; ch < 80; ++ch)
      for (int k = 0; k < 251; ++k) wg[(size_t)ch * 256 + k] = sinc_filters[ch * 251 + k];
    if ((rc = upload_split(ctx, wg, &S.sinc_wg_hi, &S.sinc_wg_lo))) return rc;
  }
  const int nch[3] = {80, 60, 60};
  for (int i = 0; i < 3; ++i) {
    B200_CHECK(norm_weight[i] && norm_bias[i], B200_ERR_INVALID, "norm1d.%d missing", i);
    std::vector<float> gmm(norm_weight[i], norm_weight[i] + nch[i]), bt(norm_bias[i], norm_bias[i] + nch[i]);
    if ((rc = upload(ctx, gmm, &S.in_gamma[i]))) return rc;
    if ((rc = upload(ctx, bt, &S.in_beta[i]))) return rc;
  }
  const int cin[2] = {80, 60};
  for (int i = 0; i < 2; ++i) {
    B200_CHECK(conv_weight[i] && conv_bias[i], B200_ERR_INVALID, "conv1d.%d missing", i + 1);
    // wgmma layout: [64 rows = c_out][k = tap * Cpad + c_in], Cpad = 80 | 64, padding zero
    const int cpad = i == 0 ? 80 : 64, K = 5 * cpad;
    std::vector<float> wc((size_t)cin[i] * 5 * 60), wg((size_t)64 * K, 0.f), bc(conv_bias[i], conv_bias[i] + 60);
    for (int co = 0; co < 60; ++co)
      for (int ci = 0; ci < cin[i]; ++ci)
        for (int k = 0; k < 5; ++k) {
          const float v = conv_weight[i][((size_t)co * cin[i] + ci) * 5 + k];
          wc[((size_t)ci * 5 + k) * 60 + co] = v;
          wg[(size_t)co * K + k * cpad + ci] = v;
        }
    if ((rc = upload(ctx, wc, &S.conv_w[i]))) return rc;
    if ((rc = upload(ctx, bc, &S.conv_b[i]))) return rc;
    if ((rc = upload_split(ctx, wg, &S.conv_wg_hi[i], &S.conv_wg_lo[i]))) return rc;
  }
  return B200_OK;
}

// The head shape of a PyanNet or SSeRiouSS load, checked before the loader releases the resident weights, so that a
// refused head leaves the loaded model in place
int check_head(int lstm_layers, int num_classes, int activation) {
  B200_CHECK(num_classes >= 1 && num_classes <= kSegMaxClasses, B200_ERR_INVALID,
             "a classifier of %d classes is unsupported (1 .. %d)", num_classes, kSegMaxClasses);
  B200_CHECK(activation == B200_SEG_LOGSOFTMAX || activation == B200_SEG_SIGMOID, B200_ERR_INVALID,
             "unknown classifier activation %d (B200_SEG_LOGSOFTMAX = 0, B200_SEG_SIGMOID = 1)", activation);
  B200_CHECK(lstm_layers >= 1 && lstm_layers <= 4, B200_ERR_INVALID, "lstm_layers=%d unsupported", lstm_layers);
  return B200_OK;
}

// The BiLSTM stack (layer 0: in0 inputs padded to kpad0), linear layers and classifier that PyanNet and SSeRiouSS share
// (b200_seg_weights / b200_ssl_weights fields of the same names), of a head that passed check_head
template <class Wt>
int load_lstm_head(b200_ctx* ctx, const Wt* w, int in0, int kpad0, int num_classes, int activation, SegWeights& S) {
  S.lstm_layers = w->lstm_layers;
  S.num_classes = num_classes;
  S.activation = activation == B200_SEG_SIGMOID ? kSegSigmoid : kSegLogSoftmax;
  int rc;
  for (int l = 0; l < S.lstm_layers; ++l) {
    const int I = l == 0 ? in0 : 256, Kp = l == 0 ? kpad0 : 256;
    S.k_in[l] = Kp;
    std::vector<float> wih((size_t)1024 * Kp, 0.f), bg(1024), whh((size_t)2 * 2 * 128 * 256);
    for (int d = 0; d < 2; ++d) {
      const float *Wi = w->lstm_w_ih[l * 2 + d], *Wh = w->lstm_w_hh[l * 2 + d];
      const float *bi = w->lstm_b_ih[l * 2 + d], *bh = w->lstm_b_hh[l * 2 + d];
      B200_CHECK(Wi && Wh && bi && bh, B200_ERR_INVALID, "lstm layer %d dir %d missing", l, d);
      for (int u = 0; u < 128; ++u)
        for (int gt = 0; gt < 4; ++gt) {
          const int n = d * 512 + u * 4 + gt, src = gt * 128 + u;
          for (int k = 0; k < I; ++k) wih[(size_t)n * Kp + k] = Wi[(size_t)src * I + k];
          bg[n] = bi[src] + bh[src];
        }
      for (int r = 0; r < 2; ++r)
        for (int k = 0; k < 128; ++k)
          for (int p = 0; p < 2; ++p)
            for (int tx = 0; tx < 32; ++tx)
              for (int gt = 0; gt < 4; ++gt) {
                const int unit = 64 * r + 2 * tx + p;
                whh[(((size_t)(d * 2 + r) * 128 + k) * 256) + p * 128 + tx * 4 + gt] = Wh[(size_t)(gt * 128 + unit) * 128 + k];
              }
    }
    if ((rc = upload_split(ctx, wih, &S.w_ih_hi[l], &S.w_ih_lo[l]))) return rc;
    if ((rc = upload(ctx, wih, &S.w_ih[l]))) return rc;
    if ((rc = upload(ctx, bg, &S.b_g[l]))) return rc;
    if ((rc = upload(ctx, whh, &S.w_hh[l]))) return rc;
    // wgmma recurrence: [dir][rank][n = 32 jj + 8 gate + u][k = unit 0..127], local unit 8 jj + u
    std::vector<float> whh_wg((size_t)4 * 256 * 128);
    for (int d = 0; d < 2; ++d)
      for (int r = 0; r < 2; ++r)
        for (int n = 0; n < 256; ++n) {
          const int unit = 64 * r + 8 * (n / 32) + n % 8, gt = (n / 8) % 4;
          for (int k = 0; k < 128; ++k)
            whh_wg[((size_t)(d * 2 + r) * 256 + n) * 128 + k] =
                w->lstm_w_hh[l * 2 + d][(size_t)(gt * 128 + unit) * 128 + k];
        }
    if ((rc = upload_split(ctx, whh_wg, &S.w_hh_hi[l], &S.w_hh_lo[l]))) return rc;
  }
  const int lin_in[2] = {256, 128};
  for (int i = 0; i < 2; ++i) {
    B200_CHECK(w->linear_weight[i] && w->linear_bias[i], B200_ERR_INVALID, "linear.%d missing", i);
    std::vector<float> lw(w->linear_weight[i], w->linear_weight[i] + 128 * lin_in[i]), lb(w->linear_bias[i], w->linear_bias[i] + 128);
    if ((rc = upload_split(ctx, lw, &S.lin_w_hi[i], &S.lin_w_lo[i]))) return rc;
    if ((rc = upload(ctx, lw, &S.lin_w[i]))) return rc;
    if ((rc = upload(ctx, lb, &S.lin_b[i]))) return rc;
  }
  B200_CHECK(w->classifier_weight && w->classifier_bias, B200_ERR_INVALID, "classifier missing");
  std::vector<float> cw(w->classifier_weight, w->classifier_weight + (size_t)num_classes * 128),
      cb(w->classifier_bias, w->classifier_bias + num_classes);
  if ((rc = upload(ctx, cw, &S.cls_w))) return rc;
  if ((rc = upload(ctx, cb, &S.cls_b))) return rc;
  return B200_OK;
}

// The TDNN stack and embedding Linear that both x-vector loaders share (b200_xvec_weights / b200_xvec_mfcc_weights
// fields of the same names), checked before the loader releases the resident weights
template <class Wt>
int check_xvec_tdnn(const Wt* w) {
  B200_CHECK(w->dimension >= 1 && w->dimension <= 65536, B200_ERR_INVALID, "embedding dimension %d unsupported",
             (int)w->dimension);
  for (int l = 0; l < kXvecLayers; ++l)
    B200_CHECK(w->tdnn_weight[l] && w->tdnn_bias[l] && w->bn_weight[l] && w->bn_bias[l] && w->bn_mean[l] && w->bn_var[l],
               B200_ERR_INVALID, "tdnns.%d / tdnns.%d missing", 3 * l, 3 * l + 2);
  B200_CHECK(w->embedding_weight && w->embedding_bias, B200_ERR_INVALID, "embedding missing");
  return B200_OK;
}

// cin0: the front end's features per frame (60 SincNet, 40 MFCC), zero padded to cin_pad[0] = 64
template <class Wt>
int load_xvec_tdnn(b200_ctx* ctx, const Wt* w, int cin0, XvecWeights& X) {
  int rc;
  const int cin[kXvecLayers] = {cin0, 512, 512, 512, 512}, cout[kXvecLayers] = {512, 512, 512, 512, 1500};
  for (int l = 0; l < kXvecLayers; ++l) {
    const int k = X.taps[l], cp = X.cin_pad[l], np = X.cout_pad[l], K = k * cp;
    std::vector<float> wt((size_t)np * K, 0.f), bias(np, 0.f), scale(np, 0.f), shift(np, 0.f);
    for (int co = 0; co < cout[l]; ++co) {
      for (int ci = 0; ci < cin[l]; ++ci)
        for (int j = 0; j < k; ++j)
          wt[(size_t)co * K + j * cp + ci] = w->tdnn_weight[l][((size_t)co * cin[l] + ci) * k + j];
      bias[co] = w->tdnn_bias[l][co];
      scale[co] = w->bn_weight[l][co] / std::sqrt(w->bn_var[l][co] + 1e-5f);
      shift[co] = w->bn_bias[l][co] - w->bn_mean[l][co] * scale[co];
    }
    if ((rc = upload_split(ctx, wt, &X.w_hi[l], &X.w_lo[l]))) return rc;
    if ((rc = upload(ctx, bias, &X.bias[l]))) return rc;
    if ((rc = upload(ctx, scale, &X.scale[l]))) return rc;
    if ((rc = upload(ctx, shift, &X.shift[l]))) return rc;
  }
  X.dim = w->dimension;
  X.dim_pad = (int)ceil_div(X.dim, 128) * 128;
  std::vector<float> ew((size_t)X.dim_pad * kXvecStatsLd, 0.f), b(X.dim_pad, 0.f);
  for (int n = 0; n < X.dim; ++n) {
    for (int kk = 0; kk < 3000; ++kk) ew[(size_t)n * kXvecStatsLd + kk] = w->embedding_weight[(size_t)n * 3000 + kk];
    b[n] = w->embedding_bias[n];
  }
  if ((rc = upload_split(ctx, ew, &X.emb_hi, &X.emb_lo))) return rc;
  return upload(ctx, b, &X.emb_b);
}

// The MFCC buffers in the layouts of xvec_mfcc.cu: the DFT basis with the window folded in (basis values in fp64 from
// the fp32 window, the angle reduced exactly mod 400), every mel filter as its band of bins from the first to the last
// nonzero weight, and dct_mat as is
int load_mfcc(b200_ctx* ctx, const float* window, const float* mel_fb, const float* dct_mat, MfccWeights* out) {
  B200_CHECK(window && mel_fb && dct_mat, B200_ERR_INVALID, "mfcc window / mel_fb / dct_mat missing");
  MfccWeights& M = *out;
  int rc;
  std::vector<float> basis((size_t)kMfccSpecLd * 2 * kMfccRowLd, 0.f);
  for (int k = 0; k < kMfccBins; ++k)
    for (int s = 0; s < kMfccFft; ++s) {
      const int j = s / kMfccHop, col = j * kMfccRowLd + s - j * kMfccHop;
      const double a = 2.0 * M_PI * (double)((k * s) % kMfccFft) / kMfccFft;
      basis[(size_t)k * 2 * kMfccRowLd + col] = (float)((double)window[s] * std::cos(a));
      basis[(size_t)(kMfccSpecLd / 2 + k) * 2 * kMfccRowLd + col] = (float)((double)window[s] * std::sin(a));
    }
  if ((rc = upload_split(ctx, basis, &M.dft_hi, &M.dft_lo))) return rc;
  std::vector<int> start(kMfccMels, 0), len(kMfccMels, 0), off(kMfccMels, 0);
  std::vector<float> band;
  for (int m = 0; m < kMfccMels; ++m) {
    int first = -1, last = -1;
    for (int k = 0; k < kMfccBins; ++k)
      if (mel_fb[(size_t)k * kMfccMels + m] != 0.f) { if (first < 0) first = k; last = k; }
    off[m] = (int)band.size();
    if (first < 0) continue;                               // an all-zero filter: 0 energy, -100 dB
    start[m] = first;
    len[m] = last - first + 1;
    for (int k = first; k <= last; ++k) band.push_back(mel_fb[(size_t)k * kMfccMels + m]);
  }
  band.push_back(0.f);                                     // never empty
  if ((rc = upload(ctx, start, &M.band_start))) return rc;
  if ((rc = upload(ctx, len, &M.band_len))) return rc;
  if ((rc = upload(ctx, off, &M.band_off))) return rc;
  if ((rc = upload(ctx, band, &M.band_w))) return rc;
  std::vector<float> dct(dct_mat, dct_mat + (size_t)kMfccMels * kMfccCoefs);
  return upload(ctx, dct, &M.dct);
}

}  // namespace

extern "C" {

const char* b200_last_error(void) { return b200::last_error(); }
int b200_version(void) { return 100; }

int b200_ctx_create(b200_ctx** out, int device) {
  B200_CHECK(out != nullptr, B200_ERR_INVALID, "ctx pointer is NULL");
  int ndev = 0;
  B200_CUDA_OK(cudaGetDeviceCount(&ndev));
  B200_CHECK(device >= 0 && device < ndev, B200_ERR_INVALID, "device %d not available (%d devices)", device, ndev);
  cudaDeviceProp prop;
  B200_CUDA_OK(cudaGetDeviceProperties(&prop, device));
  B200_CHECK(prop.major == 9 && prop.minor == 0, B200_ERR_STATE,
             "device %d is sm_%d%d; this library is built for sm_90a (H100) only", device, prop.major, prop.minor);
  b200_ctx* c = new b200_ctx();
  c->device = device;
  c->num_sms = prop.multiProcessorCount;
  if (const char* e = std::getenv("B200_CONV_IMPL")) c->conv_impl = std::atoi(e);
  if (const char* e = std::getenv("B200_EMB_MAX_BATCH")) c->emb_max_batch = std::atoi(e) > 0 ? std::atoi(e) : c->emb_max_batch;
  if (const char* e = std::getenv("B200_SEG_MAX_BATCH")) c->seg_max_batch = std::atoi(e) > 0 ? std::atoi(e) : c->seg_max_batch;
  *out = c;
  return B200_OK;
}

int b200_ctx_destroy(b200_ctx* ctx) {
  if (!ctx) return B200_OK;
  CtxScope scope(ctx);
  cudaDeviceSynchronize();
  for (void* p : ctx->owned_seg) cudaFree(p);
  for (void* p : ctx->owned_emb) cudaFree(p);
  for (void* p : ctx->owned_xvec) cudaFree(p);
  for (void* p : ctx->owned_xvec_mfcc) cudaFree(p);
  for (void* p : ctx->owned_ssl) cudaFree(p);
  for (auto& t : ctx->resample_tables) cudaFree(t.dev);
  if (ctx->ws) cudaFree(ctx->ws);
  if (ctx->d_off) cudaFree(ctx->d_off);
  if (ctx->d_valid) cudaFree(ctx->d_valid);
  if (ctx->d_frame0) cudaFree(ctx->d_frame0);
  if (ctx->d_runs) cudaFree(ctx->d_runs);
  delete ctx;
  return B200_OK;
}

int b200_ctx_set_option(b200_ctx* ctx, const char* key, int64_t value) {
  B200_CHECK(ctx && key, B200_ERR_INVALID, "NULL ctx/key");
  std::string k(key);
  if (k == "conv_impl") ctx->conv_impl = (int)value;
  else if (k == "seg_max_batch") ctx->seg_max_batch = (int)value;
  else if (k == "emb_max_batch") ctx->emb_max_batch = (int)value;
  else if (k == "ssl_max_batch") ctx->ssl_max_batch = (int)value;
  else if (k == "profile") ctx->profile = (int)value;
  else if (k == "seg_gemm_impl") ctx->seg_gemm_impl = (int)value;
  else if (k == "seg_conv_impl") ctx->seg_conv_impl = (int)value;
  else if (k == "seg_rec_impl") ctx->seg_rec_impl = (int)value;
  else if (k == "fbank_share") ctx->fbank_share = (int)value;
  else if (k == "linkage_grid_min") {
    B200_CHECK(value >= 2 && value <= kLinkGridMinDefault, B200_ERR_INVALID, "option '%s' value %lld out of range",
               key, (long long)value);
    ctx->linkage_grid_min = (int)value;
  }
  else B200_CHECK(false, B200_ERR_INVALID, "unknown option '%s'", key);
  B200_CHECK(ctx->seg_max_batch >= 1 && ctx->emb_max_batch >= 1 && ctx->ssl_max_batch >= 1 && ctx->conv_impl >= 0 && ctx->conv_impl <= 2 &&
                 ctx->seg_gemm_impl >= 0 && ctx->seg_gemm_impl <= 1 && ctx->seg_conv_impl >= 0 && ctx->seg_conv_impl <= 2 &&
                 ctx->seg_rec_impl >= 0 && ctx->seg_rec_impl <= 2,
             B200_ERR_INVALID, "option '%s' value %lld out of range", key, (long long)value);
  return B200_OK;
}

int64_t b200_ctx_launch_count(const b200_ctx* ctx) { return ctx ? ctx->launches : 0; }

int b200_ctx_timer(b200_ctx* ctx, const char* name, double* total_ms, int64_t* units) {
  B200_CHECK(ctx && name && total_ms && units, B200_ERR_INVALID, "bad arguments");
  CtxScope scope(ctx);
  std::string k(name);
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>>* v = nullptr;
  int64_t* u = nullptr;
  if (k == "trunk") { v = &ctx->trunk_events; u = &ctx->trunk_segments; }
  else if (k == "seg") { v = &ctx->seg_events; u = &ctx->seg_chunks; }
  else B200_CHECK(false, B200_ERR_INVALID, "unknown timer '%s'", name);
  B200_CUDA_OK(cudaDeviceSynchronize());
  double ms = 0.0;
  for (auto& pr : *v) {
    float t = 0.f;
    B200_CUDA_OK(cudaEventElapsedTime(&t, pr.first, pr.second));
    ms += t;
    ctx->event_pool.push_back(pr.first);
    ctx->event_pool.push_back(pr.second);
  }
  v->clear();
  *total_ms = ms;
  *units = *u;
  *u = 0;
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------------
static int64_t gcd64(int64_t a, int64_t b) { while (b) { const int64_t t = a % b; a = b; b = t; } return a; }

int64_t b200_audio_num_frames(int64_t frames_in, int32_t sr_in, int32_t sr_out) {
  if (frames_in <= 0 || sr_in <= 0 || sr_out <= 0) return 0;
  if (sr_in == sr_out) return frames_in;
  const int64_t g = gcd64(sr_in, sr_out), orig = sr_in / g, nw = sr_out / g;
  return (nw * frames_in + orig - 1) / orig;                // ceil(new * length / orig)
}

int b200_audio_ingest(b200_ctx* ctx, const void* pcm, int32_t format, int32_t channels, int64_t frames_in,
                      int32_t sr_in, int32_t sr_out, int32_t channel, float* out, int64_t out_capacity, void* stream) {
  B200_CHECK(ctx && pcm && out && channels >= 1 && frames_in >= 0 && sr_in > 0 && sr_out > 0, B200_ERR_INVALID,
             "bad arguments");
  B200_CHECK(format == B200_PCM_S16_INTERLEAVED || format == B200_PCM_F32_PLANAR, B200_ERR_INVALID,
             "unknown PCM format %d", (int)format);
  B200_CHECK(channel < channels, B200_ERR_INVALID, "channel %d of a %d-channel file", (int)channel, (int)channels);
  const int64_t frames_out = b200_audio_num_frames(frames_in, sr_in, sr_out);
  B200_CHECK(frames_out <= out_capacity, B200_ERR_INVALID, "output holds %lld samples, %lld needed",
             (long long)out_capacity, (long long)frames_out);
  if (frames_out == 0) return B200_OK;
  CtxScope scope(ctx);
  const int64_t gg = gcd64(sr_in, sr_out);
  const int orig = (int)(sr_in / gg), nw = (int)(sr_out / gg);
  const b200_ctx::ResampleTable* tab = nullptr;
  for (auto& t : ctx->resample_tables)
    if (t.orig == orig && t.nw == nw) tab = &t;
  if (!tab) {
    b200_ctx::ResampleTable t{orig, nw, 0, nullptr};
    std::vector<float> host;
    if (orig == nw) { host.assign(1, 1.0f); t.width = 0; }   // same rate: y[i] = 1.0 * x[i] (exact)
    else resample_table(orig, nw, &t.width, &host);
    B200_CUDA_OK(cudaMalloc((void**)&t.dev, host.size() * sizeof(float)));
    B200_CUDA_OK(cudaMemcpy(t.dev, host.data(), host.size() * sizeof(float), cudaMemcpyHostToDevice));
    ctx->resample_tables.push_back(t);
    tab = &ctx->resample_tables.back();
  }
  return audio_ingest(pcm, format, channels, frames_in, channel, tab->dev, tab->orig, tab->nw, tab->width, out,
                      frames_out, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------------
int b200_seg_load_head(b200_ctx* ctx, const b200_seg_weights* w, int32_t num_classes, int32_t activation) {
  B200_CHECK(ctx && w, B200_ERR_INVALID, "NULL ctx/weights");
  int rc;
  if ((rc = check_head(w->lstm_layers, num_classes, activation))) return rc;
  CtxScope scope(ctx);
  SegWeights& S = ctx->seg;
  S.loaded = false;
  release_weights(ctx, &ctx->owned_seg);
  if ((rc = load_sincnet(ctx, w->wav_norm_weight, w->wav_norm_bias, w->sinc_filters, w->norm_weight, w->norm_bias,
                         w->conv_weight, w->conv_bias, &S.sinc)))
    return rc;
  if ((rc = load_lstm_head(ctx, w, 60, 64, num_classes, activation, S))) return rc;
  S.loaded = true;
  return B200_OK;
}

int b200_seg_load(b200_ctx* ctx, const b200_seg_weights* w) {
  return b200_seg_load_head(ctx, w, kClasses, B200_SEG_LOGSOFTMAX);
}

int b200_emb_load(b200_ctx* ctx, const b200_emb_weights* w) {
  B200_CHECK(ctx && w, B200_ERR_INVALID, "NULL ctx/weights");
  CtxScope scope(ctx);
  EmbWeights& E = ctx->emb;
  int rc;
  E.loaded = false;
  release_weights(ctx, &ctx->owned_emb);
  if ((rc = build_fbank_constants(ctx))) return rc;
  if ((rc = load_stem(ctx, w->stem, &E))) return rc;
  E.blocks.clear();
  E.bottlenecks.clear();
  E.C = 256;
  const int planes[4] = {32, 64, 128, 256}, nblk[4] = {3, 4, 6, 3}, strides[4] = {1, 2, 2, 2};
  int in_planes = 32, bi = 0;
  for (int l = 0; l < 4; ++l)
    for (int i = 0; i < nblk[l]; ++i, ++bi) {
      BlockWeights B;
      const int s = i == 0 ? strides[l] : 1;
      if ((rc = make_conv(ctx, w->block_conv1[bi], in_planes, planes[l], 3, s, &B.conv1))) return rc;
      if ((rc = make_conv(ctx, w->block_conv2[bi], planes[l], planes[l], 3, 1, &B.conv2))) return rc;
      B.has_shortcut = (s != 1 || in_planes != planes[l]);
      if (B.has_shortcut)
        if ((rc = make_conv(ctx, w->block_shortcut[bi], in_planes, planes[l], 1, s, &B.shortcut))) return rc;
      in_planes = planes[l];
      E.blocks.push_back(B);
    }
  B200_CHECK(w->seg1_weight && w->seg1_bias, B200_ERR_INVALID, "seg_1 missing");
  if ((rc = load_seg1(ctx, w->seg1_weight, w->seg1_bias, 5120, &E))) return rc;
  E.loaded = true;
  return B200_OK;
}

int b200_emb_load_bottleneck(b200_ctx* ctx, const b200_emb_bottleneck_weights* w) {
  B200_CHECK(ctx && w, B200_ERR_INVALID, "NULL ctx/weights");
  for (int l = 0; l < 4; ++l)
    B200_CHECK(w->num_blocks[l] >= 1 && w->num_blocks[l] <= 1024, B200_ERR_INVALID,
               "layer %d: %d blocks (expected 1 .. 1024)", l + 1, (int)w->num_blocks[l]);
  B200_CHECK(w->block_conv1 && w->block_conv2 && w->block_conv3 && w->block_shortcut, B200_ERR_INVALID,
             "block arrays missing");
  // the shortcut of block i exists exactly where Bottleneck has one (resnet.py:165-176)
  {
    int in_planes = 32, bi = 0;
    for (int l = 0; l < 4; ++l)
      for (int i = 0; i < w->num_blocks[l]; ++i, ++bi) {
        const int p = 32 << l, s = (i == 0 && l > 0) ? 2 : 1;
        const bool need = s != 1 || in_planes != 4 * p;
        B200_CHECK(need == (w->block_shortcut[bi].conv_weight != nullptr), B200_ERR_INVALID,
                   "layer%d.%d: shortcut %s (stride %d, %d -> %d channels)", l + 1, i, need ? "missing" : "unexpected",
                   s, in_planes, 4 * p);
        in_planes = 4 * p;
      }
  }
  B200_CHECK(w->seg1_weight && w->seg1_bias, B200_ERR_INVALID, "seg_1 missing");
  CtxScope scope(ctx);
  EmbWeights& E = ctx->emb;
  int rc;
  E.loaded = false;
  release_weights(ctx, &ctx->owned_emb);
  E.blocks.clear();
  E.bottlenecks.clear();
  E.C = 1024;
  if ((rc = build_fbank_constants(ctx))) return rc;
  if ((rc = load_stem(ctx, w->stem, &E))) return rc;
  int in_planes = 32, bi = 0;
  for (int l = 0; l < 4; ++l)
    for (int i = 0; i < w->num_blocks[l]; ++i, ++bi) {
      BottleneckWeights B;
      const int p = 32 << l, s = (i == 0 && l > 0) ? 2 : 1;
      if ((rc = make_conv(ctx, w->block_conv1[bi], in_planes, p, 1, 1, &B.conv1))) return rc;
      if ((rc = make_conv(ctx, w->block_conv2[bi], p, p, 3, s, &B.conv2))) return rc;
      if ((rc = make_conv(ctx, w->block_conv3[bi], p, 4 * p, 1, 1, &B.conv3))) return rc;
      B.has_shortcut = w->block_shortcut[bi].conv_weight != nullptr;
      if (B.has_shortcut)
        if ((rc = make_conv(ctx, w->block_shortcut[bi], in_planes, 4 * p, 1, s, &B.shortcut))) return rc;
      in_planes = 4 * p;
      E.bottlenecks.push_back(B);
    }
  if ((rc = load_seg1(ctx, w->seg1_weight, w->seg1_bias, (size_t)2 * 10 * E.C, &E))) return rc;
  E.loaded = true;
  return B200_OK;
}

// ------------------------------------------------------------------------------------------------------
// The two front ends of the segmentation head (load_lstm_head, lstm_head_forward): SincNet writes PyanNet's head input
// (60 features and 4 zero columns per frame), WavLM Base that of SSeRiouSS (768 features per frame)
enum class SegFront { kSincNet, kWavLM };

// the head behind a front end, or null while its model is not loaded
static const SegWeights* loaded_head(const b200_ctx* ctx, SegFront front) {
  const bool sinc = front == SegFront::kSincNet;
  if (!ctx || !(sinc ? ctx->seg.loaded : ctx->ssl.loaded)) return nullptr;
  return sinc ? &ctx->seg : &ctx->ssl.head;
}

// A segmentation model on n windows of `window` samples: per sub-batch, the front end writes x0 [nb][T][F] and the
// head classifies it, both phases in the same workspace region.  A sub-batch holds at most max_batch x 160000
// window samples (the workspace of max_batch 10 s windows; option seg_max_batch or ssl_max_batch) and at most 65535
// windows (the y extent of the SincNet grids).  The "seg" timer covers PyanNet's sub-batches.  With front_out, the
// front end writes its head input [n][T][F] there instead of x0 and the head does not run.  With cap (SincNet only),
// the n windows must fit one sub-batch and every stage's result is also copied into cap's buffers.
static int seg_run(b200_ctx* ctx, SegFront front, const float* wav, const int64_t* chunk_off,
                   const int32_t* chunk_valid, int n, int window, const SegHeadOut& out, float* front_out,
                   cudaStream_t st, const SegCapture* cap = nullptr) {
  const bool sinc = front == SegFront::kSincNet;
  const char* model = sinc ? "segmentation" : "SSeRiouSS";
  const SegWeights* head = loaded_head(ctx, front);
  B200_CHECK(head, B200_ERR_STATE, "%s weights not loaded", model);
  B200_CHECK(wav && chunk_off && chunk_valid && n >= 0, B200_ERR_INVALID, "bad arguments");
  const int min_window = sinc ? kSegMinWindow : kSslMinWindow;
  B200_CHECK(window >= min_window, B200_ERR_INVALID,
             "windows of %d samples are too short: %s needs at least %d samples (%s)", window,
             sinc ? "PyanNet" : "SSeRiouSS", min_window, sinc ? "2 output frames" : "one WavLM frame");
  const char* option = sinc ? "seg_max_batch" : "ssl_max_batch";
  const int max_batch = sinc ? ctx->seg_max_batch : ctx->ssl_max_batch;
  const int64_t budget = (int64_t)max_batch * kChunk;
  B200_CHECK(window <= budget, B200_ERR_INVALID,
             "a window of %d samples is longer than the %lld samples of one %s sub-batch (%s %d x 160000): set the "
             "option %s to at least %lld, or segment shorter excerpts",
             window, (long long)budget, model, option, max_batch, option, (long long)((window + kChunk - 1) / kChunk));
  const int64_t sub_batch = std::min<int64_t>(budget / window, 65535);
  B200_CHECK(!cap || n <= sub_batch, B200_ERR_INVALID,
             "%d windows of %d samples are more than one %s sub-batch (%lld: %s %d x 160000 / %d, at most 65535)", n,
             window, model, (long long)sub_batch, option, max_batch, window);
  if (n == 0) return B200_OK;
  CtxScope scope(ctx);
  const int nbmax = (int)std::min<int64_t>(n, sub_batch);
  SegGeom seg_g{};
  SslGeom ssl_g{};
  int T = 0, F = 0;            // frames and features per window
  size_t front_b = 0;
  switch (front) {
    case SegFront::kSincNet:
      seg_g = seg_geom(window);
      T = seg_g.pool2;
      F = 64;
      front_b = sincnet_workspace_bytes(seg_g, nbmax);
      break;
    case SegFront::kWavLM:
      ssl_g = ssl_geom(window);
      T = ssl_g.T;
      F = kSslDim;
      front_b = ssl_workspace_bytes(ssl_g, nbmax);
      break;
  }
  const size_t x0_bytes = align_up((size_t)nbmax * T * F * sizeof(float), 1024);
  int rc = ensure_ws(ctx, x0_bytes + std::max(front_b, lstm_workspace_bytes(nbmax, T, F)) + 4096);
  if (rc) return rc;
  if ((rc = push_meta(ctx, chunk_off, chunk_valid, n, st, window))) return rc;
  float* x0 = reinterpret_cast<float*>(ctx->ws);
  void* region = reinterpret_cast<char*>(ctx->ws) + x0_bytes;
  for (int c0 = 0; c0 < n; c0 += nbmax) {
    const int nb = (n - c0) < nbmax ? (n - c0) : nbmax;
    ScopedTimer timer(ctx, sinc ? &ctx->seg_events : nullptr, st);
    if (ctx->profile && sinc) ctx->seg_chunks += nb;
    float* feat = front_out ? front_out + (size_t)c0 * T * F : x0;
    switch (front) {
      case SegFront::kSincNet:
        rc = sincnet_forward(ctx->seg.sinc, seg_g, wav, ctx->d_off + c0, ctx->d_valid + c0, nb, region, feat,
                             ctx->seg_conv_impl, st, cap);
        break;
      case SegFront::kWavLM:
        rc = ssl_frontend_forward(ctx->ssl, ssl_g, wav, ctx->d_off + c0, ctx->d_valid + c0, nb, region, feat,
                                  ctx->num_sms, st);
        break;
    }
    if (rc) return rc;
    if (front_out) continue;
    const size_t row0 = (size_t)c0 * T, K = head->num_classes;
    SegHeadOut sub;
    sub.cls = out.cls ? out.cls + row0 : nullptr;
    sub.logp = out.logp ? out.logp + row0 * K : nullptr;
    sub.scores = out.scores ? out.scores + row0 * K : nullptr;
    sub.max_scores = out.max_scores ? out.max_scores + row0 : nullptr;
    if ((rc = lstm_head_forward(*head, x0, nb, T, region, sub, ctx->num_sms, ctx->seg_gemm_impl, ctx->seg_rec_impl,
                                st, cap)))
      return rc;
  }
  return B200_OK;
}

// The forward entry points of one activation: kSegLogSoftmax writes out.cls (+ out.logp), kSegSigmoid out.scores and /
// or out.max_scores.  A loaded head of the other activation is refused, naming the entry point to call.
static int seg_forward_head(b200_ctx* ctx, SegFront front, int activation, const float* wav, const int64_t* chunk_off,
                            const int32_t* chunk_valid, int32_t num_chunks, int32_t window, const SegHeadOut& out,
                            void* stream) {
  const bool sinc = front == SegFront::kSincNet, sigmoid = activation == kSegSigmoid;
  const SegWeights* head = loaded_head(ctx, front);
  B200_CHECK(!(head && head->activation != activation), B200_ERR_INVALID,
             "the loaded %s head is a %s head: call b200_%s_forward_%s", sinc ? "segmentation" : "SSeRiouSS",
             sigmoid ? "log-softmax (powerset / mono-label)" : "sigmoid (multi-label / binary)", sinc ? "seg" : "ssl",
             sigmoid ? "window" : "scores");
  if (num_chunks == 0) return B200_OK;
  if (sigmoid) B200_CHECK(out.scores || out.max_scores, B200_ERR_INVALID, "scores and max_scores are both NULL");
  else B200_CHECK(out.cls != nullptr, B200_ERR_INVALID, "classes is NULL");
  return seg_run(ctx, front, wav, chunk_off, chunk_valid, num_chunks, window, out, nullptr, (cudaStream_t)stream);
}

int b200_seg_forward_window(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                            int32_t num_chunks, int32_t window, uint8_t* classes, float* logp, void* stream) {
  return seg_forward_head(ctx, SegFront::kSincNet, kSegLogSoftmax, wav, chunk_off, chunk_valid, num_chunks, window,
                          SegHeadOut{classes, logp}, stream);
}

int b200_seg_forward_scores(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                            int32_t num_chunks, int32_t window, float* scores, float* max_scores, void* stream) {
  return seg_forward_head(ctx, SegFront::kSincNet, kSegSigmoid, wav, chunk_off, chunk_valid, num_chunks, window,
                          SegHeadOut{nullptr, nullptr, scores, max_scores}, stream);
}

int b200_seg_forward(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                     int32_t num_chunks, uint8_t* classes, float* logp, void* stream) {
  return b200_seg_forward_window(ctx, wav, chunk_off, chunk_valid, num_chunks, kChunk, classes, logp, stream);
}

// the classifier outputs of a capture; a log-softmax head writes its classes unconditionally
static int capture_outputs(const SegWeights& head, const SegCapture* cap, SegHeadOut* out) {
  B200_CHECK(head.activation != kSegLogSoftmax || cap->cls, B200_ERR_INVALID,
             "the loaded head is a log-softmax head: cap->cls is required");
  *out = SegHeadOut{cap->cls, cap->logp, cap->scores, cap->max_scores};
  return B200_OK;
}

int b200_seg_stages(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                    int32_t num_chunks, int32_t window, const b200_seg_capture* cap, void* stream) {
  B200_CHECK(cap, B200_ERR_INVALID, "cap is NULL");
  const SegWeights* head = loaded_head(ctx, SegFront::kSincNet);
  B200_CHECK(head, B200_ERR_STATE, "segmentation weights not loaded");
  SegHeadOut out;
  int rc;
  if ((rc = capture_outputs(*head, cap, &out))) return rc;
  return seg_run(ctx, SegFront::kSincNet, wav, chunk_off, chunk_valid, num_chunks, window, out, nullptr,
                 (cudaStream_t)stream, cap);
}

int b200_seg_head_stages(b200_ctx* ctx, int32_t model, const float* x0, int32_t n, int32_t T,
                         const b200_seg_capture* cap, void* stream) {
  B200_CHECK(model == B200_SEG_HEAD_PYANNET || model == B200_SEG_HEAD_SSERIOUSS, B200_ERR_INVALID,
             "unknown model %d (B200_SEG_HEAD_PYANNET = 0, B200_SEG_HEAD_SSERIOUSS = 1)", (int)model);
  const bool sinc = model == B200_SEG_HEAD_PYANNET;
  const SegWeights* head = loaded_head(ctx, sinc ? SegFront::kSincNet : SegFront::kWavLM);
  B200_CHECK(head, B200_ERR_STATE, "%s weights not loaded", sinc ? "segmentation" : "SSeRiouSS");
  B200_CHECK(x0 && cap && n >= 0 && T >= 1, B200_ERR_INVALID, "bad arguments");
  // as in the forward's largest sub-batch, the n * T * 1024 elements of the input projection fit an int
  B200_CHECK((int64_t)n * T * 1024 < INT_MAX, B200_ERR_INVALID, "%d sequences of %d frames are too many", (int)n,
             (int)T);
  SegHeadOut out;
  int rc;
  if ((rc = capture_outputs(*head, cap, &out))) return rc;
  if (n == 0) return B200_OK;
  CtxScope scope(ctx);
  if ((rc = ensure_ws(ctx, lstm_workspace_bytes(n, T, head->k_in[0]) + 4096))) return rc;
  return lstm_head_forward(*head, x0, n, T, ctx->ws, out, ctx->num_sms, ctx->seg_gemm_impl, ctx->seg_rec_impl,
                           (cudaStream_t)stream, cap);
}

// ------------------------------------------------------------------------------------------------------
int b200_ssl_load(b200_ctx* ctx, const b200_ssl_weights* w, int32_t num_classes, int32_t activation) {
  B200_CHECK(ctx && w, B200_ERR_INVALID, "NULL ctx/weights");
  int rc;
  if ((rc = check_head(w->lstm_layers, num_classes, activation))) return rc;
  B200_CHECK(w->num_layers >= 1 && w->num_layers <= kSslLayers, B200_ERR_INVALID, "num_layers=%d unsupported (1 .. 12)",
             (int)w->num_layers);
  B200_CHECK(w->conv0_weight && w->conv0_norm_weight && w->conv0_norm_bias && w->proj_norm_weight &&
                 w->proj_norm_bias && w->proj_weight && w->proj_bias && w->pos_conv_weight && w->pos_conv_bias &&
                 w->encoder_norm_weight && w->encoder_norm_bias &&
                 w->rel_attn_embed && w->rel_bucket,
             B200_ERR_INVALID, "WavLM front-end weights missing");
  for (int l = 0; l < 6; ++l) B200_CHECK(w->conv_weight[l], B200_ERR_INVALID, "conv_layers.%d missing", l + 1);
  for (int l = 0; l < w->num_layers; ++l) {
    const b200_ssl_layer_weights& L = w->layer[l];
    B200_CHECK(L.in_proj_weight && L.in_proj_bias && L.out_proj_weight && L.out_proj_bias && L.gru_weight &&
                   L.gru_bias && L.gru_const && L.layer_norm_weight && L.layer_norm_bias && L.ff1_weight &&
                   L.ff1_bias && L.ff2_weight && L.ff2_bias && L.final_layer_norm_weight && L.final_layer_norm_bias,
               B200_ERR_INVALID, "transformer layer %d missing", l);
  }
  for (int i = 0; i < 2 * kSslRelSpan + 1; ++i)
    B200_CHECK(w->rel_bucket[i] >= 0 && w->rel_bucket[i] < 320, B200_ERR_INVALID, "relative bucket %d out of range",
               (int)w->rel_bucket[i]);
  CtxScope scope(ctx);
  SslWeights& X = ctx->ssl;
  X.loaded = false;
  release_weights(ctx, &ctx->owned_ssl);
  X.head = SegWeights();
  auto up = [&](const float* src, size_t n, float** dst) {
    return upload(ctx, std::vector<float>(src, src + n), dst);
  };
  auto up_split = [&](const float* src, size_t n, __half** hi, __half** lo) {
    return upload_split(ctx, std::vector<float>(src, src + n), hi, lo);
  };
  const int C = kSslConvDim, D = kSslDim;
  if ((rc = up(w->conv0_weight, (size_t)C * 10, &X.conv0_w))) return rc;
  if ((rc = up(w->conv0_norm_weight, C, &X.gn_w))) return rc;
  if ((rc = up(w->conv0_norm_bias, C, &X.gn_b))) return rc;
  // convs 1-6 on pair rows: B[n][tap * 512 + c] = W[n][c][tap], taps padded to an even count with zeros
  for (int l = 0; l < 6; ++l) {
    const int k = l < 4 ? 3 : 2, K = l < 4 ? 2048 : 1024;
    std::vector<float> b((size_t)C * K, 0.f);
    for (int n = 0; n < C; ++n)
      for (int c = 0; c < C; ++c)
        for (int t = 0; t < k; ++t) b[(size_t)n * K + t * C + c] = w->conv_weight[l][((size_t)n * C + c) * k + t];
    if ((rc = upload_split(ctx, b, &X.conv_hi[l], &X.conv_lo[l]))) return rc;
  }
  if ((rc = up(w->proj_norm_weight, C, &X.fp_ln_w))) return rc;
  if ((rc = up(w->proj_norm_bias, C, &X.fp_ln_b))) return rc;
  if ((rc = up_split(w->proj_weight, (size_t)D * C, &X.proj_hi, &X.proj_lo))) return rc;
  if ((rc = up(w->proj_bias, D, &X.proj_b))) return rc;
  {  // positional conv per group: B_g[n][tap * 64 + c] = W[48 g + n][c][tap] (n, c < 48), bias [16][128]
    const int Kp = kSslPosK * 64;
    std::vector<float> b((size_t)kSslPosGroups * 128 * Kp, 0.f), bias((size_t)kSslPosGroups * 128, 0.f);
    for (int gi = 0; gi < kSslPosGroups; ++gi)
      for (int n = 0; n < 48; ++n) {
        bias[gi * 128 + n] = w->pos_conv_bias[gi * 48 + n];
        for (int c = 0; c < 48; ++c)
          for (int t = 0; t < kSslPosK; ++t)
            b[((size_t)gi * 128 + n) * Kp + t * 64 + c] = w->pos_conv_weight[((size_t)(gi * 48 + n) * 48 + c) * kSslPosK + t];
      }
    if ((rc = upload_split(ctx, b, &X.pos_hi, &X.pos_lo))) return rc;
    if ((rc = upload(ctx, bias, &X.pos_b))) return rc;
  }
  if ((rc = up(w->encoder_norm_weight, D, &X.enc_ln_w))) return rc;
  if ((rc = up(w->encoder_norm_bias, D, &X.enc_ln_b))) return rc;
  {
    std::vector<float> tab((size_t)kSslHeads * (2 * kSslRelSpan + 1));
    for (int h = 0; h < kSslHeads; ++h)
      for (int i = 0; i < 2 * kSslRelSpan + 1; ++i)
        tab[(size_t)h * (2 * kSslRelSpan + 1) + i] = w->rel_attn_embed[w->rel_bucket[i] * kSslHeads + h];
    if ((rc = upload(ctx, tab, &X.rel_tab))) return rc;
  }
  X.num_layers = w->num_layers;
  for (int l = 0; l < kSslLayers; ++l) X.layer_w[l] = 0.f;
  for (int l = 0; l < w->num_layers; ++l) {
    const b200_ssl_layer_weights& L = w->layer[l];
    SslLayerWeights& Y = X.layer[l];
    Y = SslLayerWeights();
    X.layer_w[l] = w->layer_weights ? w->layer_weights[l] : (l == w->num_layers - 1 ? 1.f : 0.f);
    if ((rc = up_split(L.in_proj_weight, (size_t)3 * D * D, &Y.qkv_hi, &Y.qkv_lo))) return rc;
    if ((rc = up(L.in_proj_bias, 3 * D, &Y.qkv_b))) return rc;
    if ((rc = up_split(L.out_proj_weight, (size_t)D * D, &Y.out_hi, &Y.out_lo))) return rc;
    if ((rc = up(L.out_proj_bias, D, &Y.out_b))) return rc;
    if ((rc = up(L.gru_weight, 8 * 64, &Y.gru_w))) return rc;
    if ((rc = up(L.gru_bias, 8, &Y.gru_b))) return rc;
    if ((rc = up(L.gru_const, kSslHeads, &Y.gru_const))) return rc;
    if ((rc = up(L.layer_norm_weight, D, &Y.ln1_w))) return rc;
    if ((rc = up(L.layer_norm_bias, D, &Y.ln1_b))) return rc;
    if ((rc = up_split(L.ff1_weight, (size_t)kSslFfn * D, &Y.ff1_hi, &Y.ff1_lo))) return rc;
    if ((rc = up(L.ff1_bias, kSslFfn, &Y.ff1_b))) return rc;
    if ((rc = up_split(L.ff2_weight, (size_t)D * kSslFfn, &Y.ff2_hi, &Y.ff2_lo))) return rc;
    if ((rc = up(L.ff2_bias, D, &Y.ff2_b))) return rc;
    if ((rc = up(L.final_layer_norm_weight, D, &Y.ln2_w))) return rc;
    if ((rc = up(L.final_layer_norm_bias, D, &Y.ln2_b))) return rc;
  }
  if ((rc = load_lstm_head(ctx, w, D, D, num_classes, activation, X.head))) return rc;
  X.loaded = true;
  return B200_OK;
}

int b200_ssl_forward_window(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                            int32_t num_chunks, int32_t window, uint8_t* classes, float* logp, void* stream) {
  return seg_forward_head(ctx, SegFront::kWavLM, kSegLogSoftmax, wav, chunk_off, chunk_valid, num_chunks, window,
                          SegHeadOut{classes, logp}, stream);
}

int b200_ssl_forward_scores(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                            int32_t num_chunks, int32_t window, float* scores, float* max_scores, void* stream) {
  return seg_forward_head(ctx, SegFront::kWavLM, kSegSigmoid, wav, chunk_off, chunk_valid, num_chunks, window,
                          SegHeadOut{nullptr, nullptr, scores, max_scores}, stream);
}

int b200_ssl_features(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                      int32_t num_chunks, int32_t window, float* out, void* stream) {
  B200_CHECK(out != nullptr, B200_ERR_INVALID, "out is NULL");
  return seg_run(ctx, SegFront::kWavLM, wav, chunk_off, chunk_valid, num_chunks, window, SegHeadOut(), out,
                 (cudaStream_t)stream);
}

__global__ void strip_pad_kernel(const float* __restrict__ x64, float* __restrict__ out, size_t rows) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * 60) return;
  out[idx] = x64[(idx / 60) * 64 + idx % 60];
}

int b200_sincnet_forward(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                         int32_t num_chunks, float* out, void* stream) {
  B200_CHECK(out != nullptr, B200_ERR_INVALID, "out is NULL");
  if (num_chunks == 0) return B200_OK;
  CtxScope scope(ctx);
  cudaStream_t st = (cudaStream_t)stream;
  float* tmp = nullptr;
  const size_t rows = (size_t)num_chunks * kFrames;
  B200_CUDA_OK(cudaMalloc((void**)&tmp, rows * 64 * sizeof(float)));
  int rc = seg_run(ctx, SegFront::kSincNet, wav, chunk_off, chunk_valid, num_chunks, kChunk, SegHeadOut(), tmp, st);
  if (rc == B200_OK) {
    rc = launch(strip_pad_kernel, (unsigned)((rows * 60 + 255) / 256), 256, 0, st, tmp, out, rows);
    cudaStreamSynchronize(st);
  }
  cudaFree(tmp);
  return rc;
}

// the map of num_speakers / max_per_frame, checked against the caller's class count
static int powerset_map_for(int32_t num_classes, int32_t num_speakers, int32_t max_per_frame, PowersetMap* map) {
  if (!powerset_map(num_speakers, max_per_frame, map)) return B200_ERR_INVALID;
  B200_CHECK(map->K == num_classes, B200_ERR_INVALID,
             "a powerset of %d speakers with at most %d per frame has %d classes, not %d", (int)num_speakers,
             (int)max_per_frame, map->K, (int)num_classes);
  return B200_OK;
}

int b200_powerset_to_multilabel_generic(b200_ctx* ctx, const uint8_t* classes, int64_t n, int32_t num_classes,
                                        int32_t num_speakers, int32_t max_per_frame, uint8_t* multilabel,
                                        void* stream) {
  B200_CHECK(ctx && classes && multilabel && n >= 0, B200_ERR_INVALID, "bad arguments");
  PowersetMap map;
  int rc;
  if ((rc = powerset_map_for(num_classes, num_speakers, max_per_frame, &map))) return rc;
  if (n == 0) return B200_OK;
  CtxScope scope(ctx);
  return powerset_to_multilabel(classes, n, map, multilabel, (cudaStream_t)stream);
}

int b200_powerset_to_multilabel(b200_ctx* ctx, const uint8_t* classes, int64_t n, uint8_t* multilabel, void* stream) {
  return b200_powerset_to_multilabel_generic(ctx, classes, n, kClasses, kSpeakers, 2, multilabel, stream);
}

// ------------------------------------------------------------------------------------------------------
// fbank frames of `samples` samples (kaldi framing: 400-sample frames every 160, snip_edges)
static int64_t fbank_frames(int64_t samples) { return 1 + (samples - 400) / 160; }

// trunk output width of T0 fbank frames: T0 after layer 1, then (T + 2 - 3) / 2 + 1 after each of layers 2, 3 and 4
// (125 for the 998 frames of 10 s)
static int trunk_width(int T0) {
  int T = T0;
  for (int l = 0; l < 3; ++l) T = (T + 2 - 3) / 2 + 1;
  return T;
}

struct EmbWs {
  float *fbank, *fmean;
  double* part;   // pooling scratch, none when the trunk output has at most kPoolSlice frames
  __half *A, *Bf, *Cf, *D;
};
// Workspace of a sub-batch of NB segments of T0 fbank frames pooled for S speakers.  fbank holds T0 rows per segment,
// the most a plan needs (shared frames need fewer).  ResNet34: A, Bf and Cf hold the largest activation, layer 1's 32
// channels at 80 x T0 per segment.  Bottleneck trunk (every later layer is half the size of layer 1 at the same
// width): A and D the 4p = 128 channels of layer 1, Bf layer 2 block 0's conv1 output (64 channels at layer 1's
// resolution), Cf layer 1's conv2 output (32 channels).
static size_t carve_emb(const EmbWeights& E, int NB, int T0, int S, void* base, EmbWs* w) {
  Workspace ws(base, 1024);
  EmbWs t;
  const size_t act = (size_t)NB * kMel * T0 * 32 * sizeof(__half);   // largest activation (layer1)
  t.fbank = (float*)ws.take((size_t)NB * T0 * kMel * sizeof(float));
  t.fmean = (float*)ws.take((size_t)NB * kMel * sizeof(float));
  t.part = (double*)ws.take(pool_scratch_bytes(NB, S, trunk_width(T0), E.C));
  const bool bn = !E.bottlenecks.empty();
  t.A = (__half*)ws.take(bn ? 4 * act : act);
  t.Bf = (__half*)ws.take(bn ? 2 * act : act);
  t.Cf = (__half*)ws.take(act);
  t.D = bn ? (__half*)ws.take(4 * act) : nullptr;
  if (w) *w = t;
  return ws.bytes();
}

// one BasicBlock on nb segments: A -> (Bf, Cf) -> A, in place on the residual; a block with a fused kernel runs as
// one launch A -> Bf, and A and Bf swap
static int block_run(b200_ctx* ctx, const BlockWeights& B, __half*& A, __half*& Bf, __half* Cf, int nb, int H, int Wd,
                     cudaStream_t st) {
  const int s = B.conv1.stride;
  const int Ho = (H + 2 - 3) / s + 1, Wo = (Wd + 2 - 3) / s + 1;
  int rc;
  if (block_fused(B, ctx->conv_impl)) {
    if ((rc = block_forward(B, A, Bf, nb, H, Wd, ctx->num_sms, st))) return rc;
    std::swap(A, Bf);
    return B200_OK;
  }
  if ((rc = conv_forward(B.conv1, A, nullptr, Bf, nb, H, Wd, 1, ctx->conv_impl, ctx->num_sms, st))) return rc;
  const __half* res = A;
  if (B.has_shortcut) {
    if ((rc = conv_forward(B.shortcut, A, nullptr, Cf, nb, H, Wd, 0, ctx->conv_impl, ctx->num_sms, st))) return rc;
    res = Cf;
  }
  if ((rc = conv_forward(B.conv2, Bf, res, A, nb, Ho, Wo, 1, ctx->conv_impl, ctx->num_sms, st))) return rc;
  return B200_OK;
}

// one Bottleneck on nb segments: conv1 A -> Bf, conv2 Bf -> Cf, shortcut A -> D, conv3 Cf (+ A or D) -> A, in place
// on the residual as block_run
static int bottleneck_run(b200_ctx* ctx, const BottleneckWeights& B, __half* A, __half* Bf, __half* Cf, __half* D,
                          int nb, int H, int Wd, cudaStream_t st) {
  const int s = B.conv2.stride;
  const int Ho = (H + 2 - 3) / s + 1, Wo = (Wd + 2 - 3) / s + 1;
  const int impl = ctx->conv_impl, sms = ctx->num_sms;
  int rc;
  if ((rc = conv_forward(B.conv1, A, nullptr, Bf, nb, H, Wd, 1, impl, sms, st))) return rc;
  if ((rc = conv_forward(B.conv2, Bf, nullptr, Cf, nb, H, Wd, 1, impl, sms, st))) return rc;
  const __half* res = A;
  if (B.has_shortcut) {
    if ((rc = conv_forward(B.shortcut, A, nullptr, D, nb, H, Wd, 0, impl, sms, st))) return rc;
    res = D;
  }
  if ((rc = conv_forward(B.conv3, Cf, res, A, nb, Ho, Wo, 1, impl, sms, st))) return rc;
  return B200_OK;
}

// stages of the loaded trunk: the stem, then its BasicBlocks or its Bottlenecks
static int trunk_stages(const EmbWeights& E) { return 1 + (int)(E.blocks.size() + E.bottlenecks.size()); }

// stride and output channels of trunk stage k (0: the stem)
static void stage_shape(const EmbWeights& E, int k, int* stride, int* C_out) {
  if (k == 0) { *stride = 1; *C_out = 32; return; }
  if (!E.blocks.empty()) { *stride = E.blocks[k - 1].conv1.stride; *C_out = E.blocks[k - 1].conv2.C_out; return; }
  *stride = E.bottlenecks[k - 1].conv2.stride;
  *C_out = E.bottlenecks[k - 1].conv3.C_out;
}

// Stage k of the trunk on nb segments: k = 0 the stem from w.fbank - w.fmean (T0 = Wd frames) into w.A, k >= 1 block
// k - 1 on w.A (H x Wd in, H x Wd updated to its output's).  The result is in w.A: a fused block swaps w.A and w.Bf.
static int trunk_stage(b200_ctx* ctx, int k, EmbWs& w, const int* frame0, int nb, int& H, int& Wd, cudaStream_t st) {
  const EmbWeights& E = ctx->emb;
  if (k == 0) return conv1_forward(w.fbank, w.fmean, frame0, E.conv1_w, E.conv1_b, w.A, nb, Wd, st);
  const int rc = E.blocks.empty() ? bottleneck_run(ctx, E.bottlenecks[k - 1], w.A, w.Bf, w.Cf, w.D, nb, H, Wd, st)
                                  : block_run(ctx, E.blocks[k - 1], w.A, w.Bf, w.Cf, nb, H, Wd, st);
  if (rc) return rc;
  int s, C;
  stage_shape(E, k, &s, &C);
  H = (H + 2 - 3) / s + 1; Wd = (Wd + 2 - 3) / s + 1;
  return B200_OK;
}

// conv1 + the 16 BasicBlocks (or the Bottlenecks) on nb segments of T0 fbank frames; returns the buffer holding the
// result (NHWC fp16 [nb][10][T][C]) and its width T = trunk_width(T0)
static int trunk_run(b200_ctx* ctx, const EmbWs& w, const int* frame0, int nb, int T0, cudaStream_t st,
                     const __half** result, int* T_out) {
  EmbWs cur = w;                // cur.A is the current activation; Bf, Cf and D are scratch
  int rc;
  int H = kMel, Wd = T0;
  for (int k = 0; k < trunk_stages(ctx->emb); ++k)
    if ((rc = trunk_stage(ctx, k, cur, frame0, nb, H, Wd, st))) return rc;
  B200_CHECK(H == 10 && (T0 != kFbankFrames || Wd == kEmbT), B200_ERR_STATE, "unexpected trunk output %dx%d", H, Wd);
  *result = cur.A;
  *T_out = Wd;
  return B200_OK;
}

// the Linear 20 C -> 256 on `rows` pooled statistics rows; with peers its epilogue also pushes every tile to the other
// GPUs (fused all-gather of the embeddings over NVLink)
static int emb_linear(b200_ctx* ctx, const __half* st_hi, const __half* st_lo, int64_t rows, float* emb, cudaStream_t st,
                      float* const* peers = nullptr, int n_peers = 0) {
  const int K = 20 * ctx->emb.C;
  return gemm_tc_split(st_hi, st_lo, K, ctx->emb.seg1_w_hi, ctx->emb.seg1_w_lo, K, emb, kEmbDim, nullptr, nullptr, 0,
                       ctx->emb.seg1_b, (int)rows, kEmbDim, K, 0, ctx->num_sms, st, peers, n_peers);
}

// WeSpeaker embeddings of n segments of `samples` samples: segment i is wav[off[i]] onwards, of which valid[i] samples
// are read (the rest as zero).  Sub-batches of max(1, emb_max_batch * 998 / T0) segments (the workspace of
// emb_max_batch 10 s chunks) run fbank -> trunk -> pooling into the fp16 (hi, lo) statistics rows of every segment;
// one GEMM then runs the Linear on all of them.  share: overlapping full segments read shared fbank frames (FbankRun).
// Pooling weights [n][S][Tw]: u8 masks or fp32 weights (at most one of the two), or neither with S = 1.
static int emb_run(b200_ctx* ctx, const float* wav, const int64_t* off, const int32_t* valid, int n, int samples,
                   bool share, const uint8_t* masks, const float* weights, int S, int Tw, float* emb,
                   float* const* peers, int n_peers, cudaStream_t st) {
  CtxScope scope(ctx);
  const EmbWeights& E = ctx->emb;
  const int T0 = (int)fbank_frames(samples), T = trunk_width(T0);
  const int nbmax = (int)std::min<int64_t>(n, std::max<int64_t>(1, (int64_t)ctx->emb_max_batch * kFbankFrames / T0));
  // pooled statistics of ALL segments as fp16 (hi, lo) pairs -> one tensor-core GEMM for the Linear 20 C -> 256
  // (5120 -> 256 for ResNet34; 20480 -> 256 for a bottleneck trunk, 80 KB of pairs per row)
  const size_t rows = (size_t)n * S;
  const size_t split_bytes = align_up(rows * 2 * 10 * E.C * sizeof(__half), 1024);
  const size_t sub_bytes = carve_emb(E, nbmax, T0, S, nullptr, nullptr);
  int rc = ensure_ws(ctx, sub_bytes + 2 * split_bytes + 4096);
  if (rc) return rc;
  if ((rc = push_meta(ctx, off, valid, n, st, samples))) return rc;
  FbankPlan plan;
  if ((rc = push_fbank_plan(ctx, off, valid, n, nbmax, share, samples, T0, &plan, st))) return rc;
  EmbWs w;
  carve_emb(E, nbmax, T0, S, ctx->ws, &w);
  __half* st_hi = reinterpret_cast<__half*>(reinterpret_cast<char*>(ctx->ws) + sub_bytes);
  __half* st_lo = reinterpret_cast<__half*>(reinterpret_cast<char*>(ctx->ws) + sub_bytes + split_bytes);
  for (int c0 = 0, sb = 0; c0 < n; c0 += nbmax, ++sb) {
    const int nb = std::min(nbmax, n - c0);
    const int* frame0 = ctx->d_frame0 + c0;
    if ((rc = fbank_forward(E, wav, ctx->d_runs + plan.run_base[sb], plan.run_base[sb + 1] - plan.run_base[sb],
                            plan.nrows[sb], frame0, nb, T0, w.fbank, w.fmean, st)))
      return rc;
    const __half* feat = nullptr;
    {
      ScopedTimer timer(ctx, &ctx->trunk_events, st);
      int Tt = 0;
      if ((rc = trunk_run(ctx, w, frame0, nb, T0, st, &feat, &Tt))) return rc;
      B200_CHECK(Tt == T, B200_ERR_STATE, "trunk output width %d, expected %d", Tt, T);
    }
    if (ctx->profile) ctx->trunk_segments += nb;
    const size_t o = (size_t)c0 * S * 2 * 10 * E.C, wo = (size_t)c0 * S * Tw;
    rc = masks ? weighted_pool_forward(feat, nullptr, masks + wo, nb, T, S, Tw, E.C, w.part, st_hi + o, st_lo + o, st)
               : weighted_pool_forward(feat, nullptr, weights ? weights + wo : nullptr, nb, T, S, Tw, E.C, w.part,
                                       st_hi + o, st_lo + o, st);
    if (rc) return rc;
  }
  return emb_linear(ctx, st_hi, st_lo, (int64_t)rows, emb, st, peers, n_peers);
}

int b200_emb_forward(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                     int32_t num_chunks, const uint8_t* masks, float* emb, void* stream) {
  return b200_emb_forward_push(ctx, wav, chunk_off, chunk_valid, num_chunks, masks, emb, nullptr, 0, stream);
}

int b200_emb_forward_push(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                          int32_t num_chunks, const uint8_t* masks, float* emb, float* const* emb_peers,
                          int32_t n_peers, void* stream) {
  B200_CHECK(n_peers >= 0 && n_peers <= 7 && (n_peers == 0 || emb_peers), B200_ERR_INVALID, "bad peer list");
  B200_CHECK(ctx && ctx->emb.loaded, B200_ERR_STATE, "embedding weights not loaded");
  B200_CHECK(wav && chunk_off && chunk_valid && masks && emb && num_chunks >= 0, B200_ERR_INVALID, "bad arguments");
  if (num_chunks == 0) return B200_OK;
  return emb_run(ctx, wav, chunk_off, chunk_valid, num_chunks, kChunk, ctx->fbank_share != 0, masks, nullptr,
                 kSpeakers, kFrames, emb, emb_peers, n_peers, (cudaStream_t)stream);
}

int b200_push(b200_ctx* ctx, const void* src, int64_t bytes, void* const* dsts, int32_t n_dsts, void* stream) {
  B200_CHECK(ctx && src && (n_dsts == 0 || dsts) && bytes >= 0 && n_dsts >= 0, B200_ERR_INVALID, "bad arguments");
  if (bytes == 0 || n_dsts == 0) return B200_OK;
  CtxScope scope(ctx);
  return push_bytes(src, bytes, dsts, n_dsts, (cudaStream_t)stream);
}

int b200_emb_fbank(b200_ctx* ctx, const float* wav, const int64_t* chunk_off, const int32_t* chunk_valid,
                   int32_t num_chunks, float* fbank, void* stream) {
  B200_CHECK(ctx && ctx->emb.loaded, B200_ERR_STATE, "embedding weights not loaded");
  B200_CHECK(wav && chunk_off && chunk_valid && fbank && num_chunks >= 0, B200_ERR_INVALID, "bad arguments");
  if (num_chunks == 0) return B200_OK;
  CtxScope scope(ctx);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ensure_ws(ctx, (size_t)num_chunks * kMel * sizeof(float) + 4096);
  if (rc) return rc;
  if ((rc = push_meta(ctx, chunk_off, chunk_valid, num_chunks, st))) return rc;
  FbankPlan plan;                                            // output layout [B][998][80]: one private run per chunk
  if ((rc = push_fbank_plan(ctx, chunk_off, chunk_valid, num_chunks, num_chunks, false, kChunk, kFbankFrames, &plan,
                            st)))
    return rc;
  float* fmean = reinterpret_cast<float*>(ctx->ws);
  if ((rc = fbank_forward(ctx->emb, wav, ctx->d_runs, num_chunks, plan.nrows[0], ctx->d_frame0, num_chunks, kFbankFrames,
                          fbank, fmean, st)))
    return rc;
  return fbank_center(fbank, fmean, num_chunks, st);
}

int64_t b200_emb_fbank_plan(const int64_t* chunk_off, const int32_t* chunk_valid, int32_t num_chunks, int32_t sub_batch,
                            int32_t share, int32_t* frame0, int32_t* rows_per_sub_batch) {
  if (!chunk_off || !chunk_valid || num_chunks < 0 || sub_batch < 1) return -1;
  for (int i = 0; i < num_chunks; ++i)
    if (chunk_valid[i] < 0 || chunk_valid[i] > kChunk || chunk_off[i] < 0) return -1;
  std::vector<b200::FbankRun> runs;
  std::vector<int> f0;
  FbankPlan plan;
  plan_fbank(chunk_off, chunk_valid, num_chunks, sub_batch, share != 0, kChunk, kFbankFrames, &runs, &f0, &plan);
  if (frame0) std::copy(f0.begin(), f0.end(), frame0);
  if (rows_per_sub_batch) std::copy(plan.nrows.begin(), plan.nrows.end(), rows_per_sub_batch);
  return (int64_t)runs.size();
}

int b200_emb_trunk(b200_ctx* ctx, const float* fbank, int32_t num_chunks, float* frames, void* stream) {
  B200_CHECK(ctx && ctx->emb.loaded, B200_ERR_STATE, "embedding weights not loaded");
  B200_CHECK(fbank && frames && num_chunks >= 0, B200_ERR_INVALID, "bad arguments");
  if (num_chunks == 0) return B200_OK;
  CtxScope scope(ctx);
  cudaStream_t st = (cudaStream_t)stream;
  const int nbmax = num_chunks < ctx->emb_max_batch ? num_chunks : ctx->emb_max_batch;
  int rc = ensure_ws(ctx, carve_emb(ctx->emb, nbmax, kFbankFrames, 1, nullptr, nullptr) + 4096);
  if (rc) return rc;
  EmbWs w;
  carve_emb(ctx->emb, nbmax, kFbankFrames, 1, ctx->ws, &w);
  const int C = ctx->emb.C;
  for (int c0 = 0; c0 < num_chunks; c0 += nbmax) {
    const int nb = (num_chunks - c0) < nbmax ? (num_chunks - c0) : nbmax;
    B200_CUDA_OK(cudaMemcpyAsync(w.fbank, fbank + (size_t)c0 * kFbankFrames * kMel,
                                 (size_t)nb * kFbankFrames * kMel * sizeof(float), cudaMemcpyDeviceToDevice, st));
    B200_CUDA_OK(cudaMemsetAsync(w.fmean, 0, (size_t)nb * kMel * sizeof(float), st));
    const __half* feat = nullptr;
    int T = 0;
    if ((rc = trunk_run(ctx, w, nullptr, nb, kFbankFrames, st, &feat, &T))) return rc;
    if ((rc = frames_to_nchw(feat, frames + (size_t)c0 * C * 10 * kEmbT, nb, T, C, st))) return rc;
  }
  return B200_OK;
}

int b200_emb_trunk_stage(b200_ctx* ctx, int32_t stage, const void* in, const float* fmean, int32_t B, int32_t W,
                         void* out, void* stream) {
  B200_CHECK(ctx && ctx->emb.loaded, B200_ERR_STATE, "embedding weights not loaded");
  const EmbWeights& E = ctx->emb;
  B200_CHECK(in && out && (stage > 0 || fmean) && B >= 0 && W >= 1, B200_ERR_INVALID, "bad arguments");
  B200_CHECK(stage >= 0 && stage < trunk_stages(E), B200_ERR_INVALID, "stage %d: the trunk has stages 0 .. %d",
             (int)stage, trunk_stages(E) - 1);
  // one sub-batch of the embedding paths: the workspace of emb_max_batch 10 s chunks holds every stage at width W
  const int64_t nbmax = std::max<int64_t>(1, (int64_t)ctx->emb_max_batch * kFbankFrames / W);
  B200_CHECK(B <= nbmax, B200_ERR_INVALID,
             "%d segments of width %d are more than one embedding sub-batch (%lld: emb_max_batch %d x 998 / %d)",
             (int)B, (int)W, (long long)nbmax, ctx->emb_max_batch, (int)W);
  if (B == 0) return B200_OK;
  CtxScope scope(ctx);
  cudaStream_t st = (cudaStream_t)stream;
  // the stage's input height and channels: the stem's output shape through the strides of the blocks before it
  int H = kMel, C_in = 32;
  for (int k = 1; k < stage; ++k) {
    int s;
    stage_shape(E, k, &s, &C_in);
    H = (H + 2 - 3) / s + 1;
  }
  int rc = ensure_ws(ctx, carve_emb(E, B, W, 1, nullptr, nullptr) + 4096);
  if (rc) return rc;
  EmbWs w;
  carve_emb(E, B, W, 1, ctx->ws, &w);
  if (stage == 0) {
    w.fbank = (float*)in;
    w.fmean = const_cast<float*>(fmean);
  } else {
    B200_CUDA_OK(cudaMemcpyAsync(w.A, in, (size_t)B * H * W * C_in * sizeof(__half), cudaMemcpyDeviceToDevice, st));
  }
  int Wd = W;
  if ((rc = trunk_stage(ctx, stage, w, nullptr, B, H, Wd, st))) return rc;
  int s, C_out;
  stage_shape(E, stage, &s, &C_out);
  B200_CUDA_OK(cudaMemcpyAsync(out, w.A, (size_t)B * H * Wd * C_out * sizeof(__half), cudaMemcpyDeviceToDevice, st));
  return B200_OK;
}

// ---- embeddings of utterances of any length ------------------------------------------------------------
int b200_emb_forward_utt(b200_ctx* ctx, const float* wav, const int64_t* off, int64_t num_samples, int32_t num_utts,
                         const float* weights, int32_t num_speakers, int32_t num_weights, float* emb, void* stream) {
  B200_CHECK(ctx && ctx->emb.loaded, B200_ERR_STATE, "embedding weights not loaded");
  B200_CHECK(wav && off && emb && num_utts >= 0, B200_ERR_INVALID, "bad arguments");
  B200_CHECK(num_samples >= 400, B200_ERR_INVALID,
             "utterances of %lld samples are shorter than one 400-sample fbank frame", (long long)num_samples);
  B200_CHECK(!weights || (num_speakers >= 1 && num_weights >= 1), B200_ERR_INVALID,
             "weights need num_speakers >= 1 and num_weights >= 1 (got %d, %d)", (int)num_speakers, (int)num_weights);
  if (num_utts == 0) return B200_OK;
  for (int i = 0; i < num_utts; ++i)
    B200_CHECK(off[i] >= 0, B200_ERR_INVALID, "utterance %d: negative offset %lld", i, (long long)off[i]);
  // a sub-batch holds at most emb_max_batch x 998 fbank frames: the workspace of emb_max_batch 10 s chunks
  const int64_t T0 = fbank_frames(num_samples);
  const int64_t budget = (int64_t)ctx->emb_max_batch * kFbankFrames;
  B200_CHECK(T0 <= budget, B200_ERR_INVALID,
             "an utterance of %lld samples has %lld fbank frames, more than the %lld frames of one embedding sub-batch "
             "(emb_max_batch %d x 998): set the option emb_max_batch to at least %lld, or embed shorter excerpts",
             (long long)num_samples, (long long)T0, (long long)budget, ctx->emb_max_batch,
             (long long)((T0 + kFbankFrames - 1) / kFbankFrames));
  const std::vector<int32_t> valid((size_t)num_utts, (int32_t)num_samples);
  return emb_run(ctx, wav, off, valid.data(), num_utts, (int)num_samples, false, nullptr, weights,
                 weights ? num_speakers : 1, num_weights, emb, nullptr, 0, (cudaStream_t)stream);
}

int b200_emb_forward_embedding(b200_ctx* ctx, const float* frames, int32_t B, int32_t T, const float* weights,
                               int32_t num_speakers, int32_t num_weights, float* emb, void* stream) {
  B200_CHECK(ctx && ctx->emb.loaded, B200_ERR_STATE, "embedding weights not loaded");
  B200_CHECK(frames && emb && B >= 0 && T >= 1, B200_ERR_INVALID, "bad arguments");
  B200_CHECK(!weights || (num_speakers >= 1 && num_weights >= 1), B200_ERR_INVALID,
             "weights need num_speakers >= 1 and num_weights >= 1 (got %d, %d)", (int)num_speakers, (int)num_weights);
  if (B == 0) return B200_OK;
  CtxScope scope(ctx);
  cudaStream_t st = (cudaStream_t)stream;
  const int S = weights ? num_speakers : 1;
  const int C = ctx->emb.C;
  const size_t rows = (size_t)B * S;
  const size_t split_bytes = align_up(rows * 2 * 10 * C * sizeof(__half), 1024);
  const size_t part_bytes = align_up(pool_scratch_bytes(B, S, T, C), 1024);
  int rc = ensure_ws(ctx, 2 * split_bytes + part_bytes + 4096);
  if (rc) return rc;
  char* base = reinterpret_cast<char*>(ctx->ws);
  __half* st_hi = reinterpret_cast<__half*>(base);
  __half* st_lo = reinterpret_cast<__half*>(base + split_bytes);
  double* part = part_bytes ? reinterpret_cast<double*>(base + 2 * split_bytes) : nullptr;
  if ((rc = weighted_pool_forward(nullptr, frames, weights, B, T, S, num_weights, C, part, st_hi, st_lo, st))) return rc;
  return emb_linear(ctx, st_hi, st_lo, (int64_t)rows, emb, st);
}

int b200_stats_pool(b200_ctx* ctx, const float* seq, const float* weights, float* out, int32_t B, int32_t F, int32_t T,
                    int32_t S, int32_t Tw, void* stream) {
  B200_CHECK(ctx && seq && out && B >= 0 && F > 0 && T > 0 && S > 0, B200_ERR_INVALID, "bad arguments");
  if (B == 0) return B200_OK;
  CtxScope scope(ctx);
  return stats_pool_generic(seq, weights, out, B, F, T, S, weights ? Tw : T, (cudaStream_t)stream);
}

// ---- XVectorSincNet / XVectorMFCC ---------------------------------------------------------------------------
int b200_xvec_load(b200_ctx* ctx, const b200_xvec_weights* w) {
  B200_CHECK(ctx && w, B200_ERR_INVALID, "NULL ctx/weights");
  int rc;
  if ((rc = check_xvec_tdnn(w))) return rc;
  CtxScope scope(ctx);
  XvecWeights& X = ctx->xvec;
  X.loaded = false;
  release_weights(ctx, &ctx->owned_xvec);
  if ((rc = load_sincnet(ctx, w->wav_norm_weight, w->wav_norm_bias, w->sinc_filters, w->norm_weight, w->norm_bias,
                         w->conv_weight, w->conv_bias, &X.sinc)))
    return rc;
  if ((rc = load_xvec_tdnn(ctx, w, 60, X))) return rc;
  X.loaded = true;
  return B200_OK;
}

int b200_xvec_mfcc_load(b200_ctx* ctx, const b200_xvec_mfcc_weights* w) {
  B200_CHECK(ctx && w, B200_ERR_INVALID, "NULL ctx/weights");
  int rc;
  if ((rc = check_xvec_tdnn(w))) return rc;
  B200_CHECK(w->window && w->mel_fb && w->dct_mat, B200_ERR_INVALID, "mfcc window / mel_fb / dct_mat missing");
  CtxScope scope(ctx);
  XvecWeights& X = ctx->xvec_mfcc;
  X.loaded = false;
  release_weights(ctx, &ctx->owned_xvec_mfcc);
  if ((rc = load_mfcc(ctx, w->window, w->mel_fb, w->dct_mat, &X.mfcc))) return rc;
  if ((rc = load_xvec_tdnn(ctx, w, kMfccCoefs, X))) return rc;
  X.loaded = true;
  return B200_OK;
}

// The two front ends of the x-vector TDNN stack (load_xvec_tdnn): SincNet writes XVectorSincNet's first-layer input
// (60 features and 4 zero columns per frame, through an fp32 copy split afterwards), MFCC that of XVectorMFCC (40
// coefficients and 24 zero columns, split in place)
enum class XvecFront { kSincNet, kMfcc };

// Geometry of one utterance length: F front-end frames, T = F - 14 TDNN frames
struct XvecGeom {
  SegGeom seg{};     // SincNet only
  int F = 0;
};
static XvecGeom xvec_geom(XvecFront front, int num_samples) {
  XvecGeom g;
  switch (front) {
    case XvecFront::kSincNet:
      g.seg = seg_geom(num_samples);
      g.F = g.seg.pool2;
      break;
    case XvecFront::kMfcc:
      g.F = mfcc_num_frames(num_samples);
      break;
  }
  return g;
}

// Workspace of an x-vector sub-batch of nb utterances of L samples (M = nb x F rows): the first layer's input (SincNet:
// X0 fp32 [M][64], then its (hi, lo) split; MFCC: the split only), two ping-pong activations P / Q [M][512] fp16 (hi,
// lo), the last layer's fp32 rows Y [M][1536] (sharing its region with the front end's scratch, which is dead by then)
// and the pooling partials.
struct XvecWs {
  float* x0;
  __half *xh, *xl, *ph, *pl, *qh, *ql;
  float* y;
  void* front;
  double* part;
};
static size_t carve_xvec(XvecFront front, const XvecGeom& g, int L, int nb, int S, void* base, XvecWs* w) {
  Workspace ws(base, 1024);
  const size_t M = (size_t)nb * g.F;
  const bool sinc = front == XvecFront::kSincNet;
  XvecWs t;
  t.x0 = sinc ? (float*)ws.take(M * 64 * sizeof(float)) : nullptr;
  t.xh = (__half*)ws.take(M * 64 * sizeof(__half));
  t.xl = (__half*)ws.take(M * 64 * sizeof(__half));
  t.ph = (__half*)ws.take(M * 512 * sizeof(__half));
  t.pl = (__half*)ws.take(M * 512 * sizeof(__half));
  t.qh = (__half*)ws.take(M * 512 * sizeof(__half));
  t.ql = (__half*)ws.take(M * 512 * sizeof(__half));
  const size_t front_b = sinc ? sincnet_workspace_bytes(g.seg, nb) : mfcc_workspace_bytes(L, nb);
  t.y = (float*)ws.take(std::max(M * kPoolRowsLd * sizeof(float), front_b));
  t.front = t.y;
  t.part = (double*)ws.take(pool_scratch_bytes(nb, S, g.F - 14, kPoolRowsLd, 1));
  if (w) *w = t;
  return ws.bytes();
}

// An x-vector model on num_utts utterances of one length: per sub-batch the front end writes the first layer's input
// rows, the five TDNN layers run on gemm_tc_split and the pooling writes the statistics rows; then one GEMM applies the
// embedding Linear to every row.  A sub-batch holds at most emb_max_batch x 160000 samples (the same budget as the
// WeSpeaker sub-batches).
static int xvec_run(b200_ctx* ctx, XvecFront front, const float* wav, const int64_t* off, int64_t num_samples,
                    int32_t num_utts, const float* weights, int32_t num_speakers, int32_t num_weights, float* emb,
                    void* stream) {
  const bool sinc = front == XvecFront::kSincNet;
  const char* model = sinc ? "XVectorSincNet" : "XVectorMFCC";
  B200_CHECK(ctx && (sinc ? ctx->xvec : ctx->xvec_mfcc).loaded, B200_ERR_STATE, "%s weights not loaded", model);
  B200_CHECK(wav && off && emb && num_utts >= 0, B200_ERR_INVALID, "bad arguments");
  const int min_samples = sinc ? kXvecMinSamples : kXvecMfccMinSamples;
  B200_CHECK(num_samples >= min_samples, B200_ERR_INVALID,
             "utterances of %lld samples are too short: %s needs at least %d samples (15 %s frames for one TDNN output "
             "frame)", (long long)num_samples, model, min_samples, sinc ? "SincNet" : "MFCC");
  B200_CHECK(!weights || (num_speakers >= 1 && num_weights >= 1), B200_ERR_INVALID,
             "weights need num_speakers >= 1 and num_weights >= 1 (got %d, %d)", (int)num_speakers, (int)num_weights);
  const int64_t budget = (int64_t)ctx->emb_max_batch * kChunk;
  B200_CHECK(num_samples <= budget, B200_ERR_INVALID,
             "an utterance of %lld samples is longer than the %lld samples of one embedding sub-batch (emb_max_batch %d "
             "x 160000): set the option emb_max_batch to at least %lld, or embed shorter excerpts",
             (long long)num_samples, (long long)budget, ctx->emb_max_batch,
             (long long)((num_samples + kChunk - 1) / kChunk));
  if (num_utts == 0) return B200_OK;
  for (int i = 0; i < num_utts; ++i)
    B200_CHECK(off[i] >= 0, B200_ERR_INVALID, "utterance %d: negative offset %lld", i, (long long)off[i]);
  CtxScope scope(ctx);
  cudaStream_t st = (cudaStream_t)stream;
  const XvecWeights& X = sinc ? ctx->xvec : ctx->xvec_mfcc;
  const int L = (int)num_samples;
  const XvecGeom geom = xvec_geom(front, L);
  const int F = geom.F, T = F - 14;                         // TDNN output frames (xvector.py:255-275)
  const int S = weights ? num_speakers : 1;
  const int nbmax = (int)std::min<int64_t>(std::min<int64_t>(num_utts, budget / num_samples), 65535);
  const size_t rows = (size_t)num_utts * S;
  const size_t split_bytes = align_up(rows * kXvecStatsLd * sizeof(__half), 1024);
  const size_t out_bytes = X.dim_pad != X.dim ? align_up(rows * X.dim_pad * sizeof(float), 1024) : 0;
  const size_t sub_bytes = carve_xvec(front, geom, L, nbmax, S, nullptr, nullptr);
  int rc = ensure_ws(ctx, sub_bytes + 2 * split_bytes + out_bytes + 4096);
  if (rc) return rc;
  {
    std::vector<int32_t> valid((size_t)num_utts, (int32_t)num_samples);
    if ((rc = push_meta(ctx, off, valid.data(), num_utts, st, (int)num_samples))) return rc;
  }
  XvecWs w;
  carve_xvec(front, geom, L, nbmax, S, ctx->ws, &w);
  char* tail = reinterpret_cast<char*>(ctx->ws) + sub_bytes;
  __half* st_hi = reinterpret_cast<__half*>(tail);
  __half* st_lo = reinterpret_cast<__half*>(tail + split_bytes);
  float* out = out_bytes ? reinterpret_cast<float*>(tail + 2 * split_bytes) : emb;
  B200_CUDA_OK(cudaMemsetAsync(st_hi, 0, 2 * split_bytes, st));   // the 8 padding columns of every statistics row
  for (int u0 = 0; u0 < num_utts; u0 += nbmax) {
    const int nb = std::min(nbmax, num_utts - u0);
    const int M = nb * F;
    switch (front) {
      case XvecFront::kSincNet: {
        // always on the tensor cores; seg_conv_impl = 2 selects the per-tile reference kernels here too
        const int sinc_impl = ctx->seg_conv_impl == 2 ? 2 : 1;
        if ((rc = sincnet_forward(X.sinc, geom.seg, wav, ctx->d_off + u0, ctx->d_valid + u0, nb, w.front, w.x0,
                                  sinc_impl, st)))
          return rc;
        rc = split_f16(w.x0, w.xh, w.xl, (size_t)M * 64, st);
        break;
      }
      case XvecFront::kMfcc:
        rc = mfcc_forward(X.mfcc, wav, ctx->d_off + u0, L, nb, w.front, w.xh, w.xl, nullptr, ctx->num_sms, st);
        break;
    }
    if (rc) return rc;
    // Every window keeps the row stride F through the stack: output row b * F + t of layer l reads input rows
    // b * F + t + j * dil.  Rows t >= F - 4, F - 8, F - 14 (layers 1, 2, 3-5) compute values nothing uses, since a
    // valid row of layer l + 1 reads only valid rows of layer l and the pooling reads the first T = F - 14 rows of
    // every window; taps past the last row of the buffer read zeros (TMA out-of-bounds fill).
    const __half* in_h[kXvecLayers] = {w.xh, w.ph, w.qh, w.ph, w.qh};
    const __half* in_l[kXvecLayers] = {w.xl, w.pl, w.ql, w.pl, w.ql};
    __half* out_h[kXvecLayers - 1] = {w.ph, w.qh, w.ph, w.qh};
    __half* out_l[kXvecLayers - 1] = {w.pl, w.ql, w.pl, w.ql};
    for (int l = 0; l < kXvecLayers; ++l) {
      GemmTaps tp;
      tp.taps = X.taps[l];
      tp.dil = X.dil[l];
      tp.scale = X.scale[l];
      tp.shift = X.shift[l];
      const int K = X.taps[l] * X.cin_pad[l], N = X.cout_pad[l];
      const bool last = l == kXvecLayers - 1;
      rc = gemm_tc_split(in_h[l], in_l[l], X.cin_pad[l], X.w_hi[l], X.w_lo[l], K, last ? w.y : nullptr, N,
                         last ? nullptr : out_h[l], last ? nullptr : out_l[l], N, X.bias[l], M, N, K, 1,
                         ctx->num_sms, st, nullptr, 0, tp);
      if (rc) return rc;
    }
    const size_t o = (size_t)u0 * S * kXvecStatsLd;
    if ((rc = weighted_pool_rows(w.y, F, T, 1500, weights ? weights + (size_t)u0 * S * num_weights : nullptr, nb, S,
                                 num_weights, w.part, st_hi + o, st_lo + o, kXvecStatsLd, st)))
      return rc;
  }
  rc = gemm_tc_split(st_hi, st_lo, kXvecStatsLd, X.emb_hi, X.emb_lo, kXvecStatsLd, out, X.dim_pad, nullptr, nullptr, 0,
                     X.emb_b, (int)rows, X.dim_pad, kXvecStatsLd, 0, ctx->num_sms, st);
  if (rc) return rc;
  if (out != emb)
    B200_CUDA_OK(cudaMemcpy2DAsync(emb, (size_t)X.dim * sizeof(float), out, (size_t)X.dim_pad * sizeof(float),
                                   (size_t)X.dim * sizeof(float), rows, cudaMemcpyDeviceToDevice, st));
  return B200_OK;
}

int b200_xvec_forward(b200_ctx* ctx, const float* wav, const int64_t* off, int64_t num_samples, int32_t num_utts,
                      const float* weights, int32_t num_speakers, int32_t num_weights, float* emb, void* stream) {
  return xvec_run(ctx, XvecFront::kSincNet, wav, off, num_samples, num_utts, weights, num_speakers, num_weights, emb,
                  stream);
}

int b200_xvec_mfcc_forward(b200_ctx* ctx, const float* wav, const int64_t* off, int64_t num_samples, int32_t num_utts,
                           const float* weights, int32_t num_speakers, int32_t num_weights, float* emb, void* stream) {
  return xvec_run(ctx, XvecFront::kMfcc, wav, off, num_samples, num_utts, weights, num_speakers, num_weights, emb,
                  stream);
}

int b200_xvec_mfcc_features(b200_ctx* ctx, const float* wav, const int64_t* off, int64_t num_samples, int32_t num_utts,
                            float* out, void* stream) {
  B200_CHECK(ctx && ctx->xvec_mfcc.loaded, B200_ERR_STATE, "XVectorMFCC weights not loaded");
  B200_CHECK(wav && off && out && num_utts >= 0 && num_utts <= 65535, B200_ERR_INVALID, "bad arguments");
  B200_CHECK(num_samples > kMfccFft / 2 && num_samples <= INT_MAX, B200_ERR_INVALID,
             "utterances of %lld samples: the MFCC front end needs more than %d samples (its reflect padding)",
             (long long)num_samples, kMfccFft / 2);
  if (num_utts == 0) return B200_OK;
  for (int i = 0; i < num_utts; ++i)
    B200_CHECK(off[i] >= 0, B200_ERR_INVALID, "utterance %d: negative offset %lld", i, (long long)off[i]);
  CtxScope scope(ctx);
  cudaStream_t st = (cudaStream_t)stream;
  const int L = (int)num_samples;
  int rc = ensure_ws(ctx, mfcc_workspace_bytes(L, num_utts) + 4096);
  if (rc) return rc;
  {
    std::vector<int32_t> valid((size_t)num_utts, 0);
    if ((rc = push_meta(ctx, off, valid.data(), num_utts, st))) return rc;
  }
  return mfcc_forward(ctx->xvec_mfcc.mfcc, wav, ctx->d_off, L, num_utts, ctx->ws, nullptr, nullptr, out, ctx->num_sms,
                      st);
}

// ------------------------------------------------------------------------------------------------------
int b200_speaker_count(b200_ctx* ctx, const uint8_t* seg, const int32_t* start_frame, int32_t num_chunks,
                       int32_t num_frames, uint8_t* count, void* stream) {
  B200_CHECK(ctx && seg && start_frame && count && num_chunks > 0 && num_frames > 0, B200_ERR_INVALID, "bad arguments");
  CtxScope scope(ctx);
  return speaker_count(seg, start_frame, num_chunks, num_frames, count, (cudaStream_t)stream);
}

int b200_reconstruct(b200_ctx* ctx, const uint8_t* seg, const int8_t* hard_clusters, const int32_t* start_frame,
                     int32_t num_chunks, int32_t num_frames, const uint8_t* count, int32_t num_clusters_out,
                     uint8_t* discrete, void* stream) {
  B200_CHECK(ctx && seg && hard_clusters && start_frame && count && discrete && num_chunks > 0 && num_frames > 0,
             B200_ERR_INVALID, "bad arguments");
  CtxScope scope(ctx);
  return reconstruct(seg, (const signed char*)hard_clusters, start_frame, num_chunks, num_frames, num_clusters_out,
                     count, discrete, (cudaStream_t)stream);
}

int b200_aggregate_window(b200_ctx* ctx, const float* scores, const int32_t* start_frame, int32_t num_chunks,
                          int32_t num_frames, int32_t frames_per_chunk, int32_t num_classes, const double* hamming,
                          const double* warm_up, int32_t skip_average, float missing, float epsilon, float* out,
                          void* stream) {
  B200_CHECK(ctx && scores && start_frame && out && num_chunks > 0 && num_frames > 0 && frames_per_chunk > 0 &&
                 num_classes > 0,
             B200_ERR_INVALID, "bad arguments");
  CtxScope scope(ctx);
  return aggregate_scores(scores, start_frame, num_chunks, num_frames, frames_per_chunk, num_classes, hamming, warm_up,
                          skip_average, missing, epsilon, out, (cudaStream_t)stream);
}

int b200_aggregate(b200_ctx* ctx, const float* scores, const int32_t* start_frame, int32_t num_chunks,
                   int32_t num_frames, int32_t num_classes, const double* hamming, const double* warm_up,
                   int32_t skip_average, float missing, float epsilon, float* out, void* stream) {
  return b200_aggregate_window(ctx, scores, start_frame, num_chunks, num_frames, kFrames, num_classes, hamming,
                               warm_up, skip_average, missing, epsilon, out, stream);
}

int b200_powerset_speech_generic(b200_ctx* ctx, const uint8_t* classes, int64_t n, int32_t num_classes,
                                 int32_t num_speakers, int32_t max_per_frame, float* speech, void* stream) {
  B200_CHECK(ctx && classes && speech && n >= 0, B200_ERR_INVALID, "bad arguments");
  PowersetMap map;
  int rc;
  if ((rc = powerset_map_for(num_classes, num_speakers, max_per_frame, &map))) return rc;
  if (n == 0) return B200_OK;
  CtxScope scope(ctx);
  return powerset_speech(classes, n, map, speech, (cudaStream_t)stream);
}

int b200_powerset_speech(b200_ctx* ctx, const uint8_t* classes, int64_t n, float* speech, void* stream) {
  return b200_powerset_speech_generic(ctx, classes, n, kClasses, kSpeakers, 2, speech, stream);
}

int b200_frame_transitions(b200_ctx* ctx, const uint8_t* discrete, int32_t num_frames, int32_t num_clusters,
                           int32_t cap, int32_t* buf, void* stream) {
  B200_CHECK(ctx && discrete && buf && num_frames > 0 && num_clusters > 0 && cap > 0, B200_ERR_INVALID,
             "bad arguments");
  CtxScope scope(ctx);
  return frame_transitions(discrete, num_frames, num_clusters, cap, buf, (cudaStream_t)stream);
}

int b200_clean_frames(b200_ctx* ctx, const uint8_t* seg, int32_t num_chunks, int32_t* clean, uint8_t* active,
                      void* stream) {
  B200_CHECK(ctx && seg && clean && active && num_chunks >= 0, B200_ERR_INVALID, "bad arguments");
  if (num_chunks == 0) return B200_OK;
  CtxScope scope(ctx);
  return clean_frames(seg, num_chunks, clean, active, (cudaStream_t)stream);
}

// ------------------------------------------------------------------------------------------------------
static int check_linkage_offsets(const int32_t* row_offsets, int32_t num_problems) {
  for (int f = 0; f < num_problems; ++f)
    B200_CHECK(row_offsets[f + 1] >= row_offsets[f] && row_offsets[f + 1] - row_offsets[f] <= kLinkMaxRows,
               B200_ERR_INVALID, "linkage: problem %d has %d observations (row offsets must be non-decreasing, at most "
               "%d per problem)", f, (int)(row_offsets[f + 1] - row_offsets[f]), kLinkMaxRows);
  return B200_OK;
}

int64_t b200_linkage_bytes(const int32_t* row_offsets, int32_t num_problems, int32_t dim) {
  B200_CHECK(row_offsets && num_problems >= 1 && dim >= 1 && row_offsets[0] >= 0, B200_ERR_INVALID, "bad arguments");
  const int rc = check_linkage_offsets(row_offsets, num_problems);
  if (rc) return rc;
  return (int64_t)(linkage_workspace_bytes_batched(row_offsets, num_problems, dim, kLinkGridMinDefault) +
                   linkage_grid_bytes(row_offsets, num_problems, kLinkGridMinDefault));
}

int b200_linkage_centroid_batched(b200_ctx* ctx, const double* x, const int32_t* row_offsets, int32_t num_problems,
                                  int32_t dim, int32_t normalize, double* Z, void* stream) {
  B200_CHECK(ctx && x && row_offsets && Z && num_problems >= 1 && dim >= 1, B200_ERR_INVALID, "bad arguments");
  int rc = check_linkage_offsets(row_offsets, num_problems);
  if (rc) return rc;
  CtxScope scope(ctx);
  rc = ensure_ws(ctx, linkage_workspace_bytes_batched(row_offsets, num_problems, dim, ctx->linkage_grid_min));
  if (rc) return rc;
  return linkage_centroid_batched(x, row_offsets, num_problems, dim, normalize, Z, ctx->ws, (cudaStream_t)stream,
                                  ctx->linkage_grid_min);
}

int b200_linkage_centroid(b200_ctx* ctx, const double* x, int32_t n, int32_t dim, int32_t normalize, double* Z,
                          void* stream) {
  B200_CHECK(n >= 2, B200_ERR_INVALID, "linkage needs at least 2 observations");
  const int32_t offs[2] = {0, n};
  return b200_linkage_centroid_batched(ctx, x, offs, 1, dim, normalize, Z, stream);
}

int b200_fcluster_distance(const double* Z, int32_t n, double t, int32_t* labels) {
  B200_CHECK(Z && labels && n >= 1, B200_ERR_INVALID, "bad arguments");
  return fcluster_distance(Z, n, t, labels);
}

int b200_plda_transform(b200_ctx* ctx, const double* x, int32_t n, int32_t Din, int32_t Dout, int32_t L,
                        const double* mean1, const double* mean2, const double* lda, const double* mu,
                        const double* trT, double* fea, void* stream) {
  B200_CHECK(ctx && x && mean1 && mean2 && lda && mu && trT && fea && n >= 0 && Din >= 1 && Dout >= 1 && L >= 1 &&
                 L <= Dout && Din + Dout <= 4096, B200_ERR_INVALID, "bad arguments");
  if (n == 0) return B200_OK;
  CtxScope scope(ctx);
  return plda_transform(x, n, Din, Dout, L, mean1, mean2, lda, mu, trT, fea, (cudaStream_t)stream);
}

int b200_weighted_centroids(b200_ctx* ctx, const double* q, int32_t n, int32_t S, const int32_t* kept, int32_t K,
                            const double* train, int32_t dim, double* centroids, void* stream) {
  B200_CHECK(ctx && q && train && n >= 1 && S >= 1 && K >= 0 && dim >= 1, B200_ERR_INVALID, "bad arguments");
  if (K == 0) return B200_OK;        // no speaker kept: empty `kept` and `centroids` (null data pointers)
  B200_CHECK(kept && centroids, B200_ERR_INVALID, "bad arguments");
  CtxScope scope(ctx);
  return weighted_centroids(q, n, S, kept, K, train, dim, centroids, (cudaStream_t)stream);
}

int b200_cdist_cosine(b200_ctx* ctx, const double* a, int32_t m, const double* b, int32_t k, int32_t dim, double* d,
                      void* stream) {
  B200_CHECK(ctx && a && b && d && m >= 0 && k >= 1 && dim >= 1, B200_ERR_INVALID, "bad arguments");
  if (m == 0) return B200_OK;
  CtxScope scope(ctx);
  return cdist_cosine(a, m, b, k, dim, d, (cudaStream_t)stream);
}

int b200_vbx_batched(b200_ctx* ctx, const double* fea, const double* phi, const int32_t* n, const int32_t* S,
                     int32_t num_problems, int32_t D, double Fa, double Fb, int32_t max_iters, double epsilon,
                     double* gamma, double* pi, int32_t* iters, void* stream) {
  B200_CHECK(ctx && fea && phi && n && S && gamma && pi && num_problems >= 1 && D >= 1 && max_iters >= 1,
             B200_ERR_INVALID, "bad arguments");
  for (int f = 0; f < num_problems; ++f) B200_CHECK(n[f] >= 0 && S[f] >= 0, B200_ERR_INVALID, "negative problem size");
  CtxScope scope(ctx);
  int rc = ensure_ws(ctx, vbx_workspace_bytes_batched(n, S, num_problems, D));
  if (rc) return rc;
  return vbx_run_batched(fea, phi, n, S, num_problems, D, Fa, Fb, max_iters, epsilon, gamma, pi, iters, ctx->ws,
                         (cudaStream_t)stream);
}

int b200_vbx(b200_ctx* ctx, const double* fea, const double* phi, int32_t n, int32_t D, int32_t S, double Fa,
             double Fb, int32_t max_iters, double epsilon, double* gamma, double* pi, int32_t* iters, void* stream) {
  B200_CHECK(n >= 1 && S >= 1, B200_ERR_INVALID, "bad arguments");
  return b200_vbx_batched(ctx, fea, phi, &n, &S, 1, D, Fa, Fb, max_iters, epsilon, gamma, pi, iters, stream);
}

int b200_assign(b200_ctx* ctx, const double* soft, int32_t num_chunks, int32_t num_clusters, int32_t constrained,
                int8_t* hard, void* stream) {
  B200_CHECK(ctx && soft && hard && num_chunks >= 0 && num_clusters >= 1, B200_ERR_INVALID, "bad arguments");
  B200_CHECK(num_clusters <= 127, B200_ERR_INVALID, "assign: %d clusters, at most 127 fit the int8 cluster ids",
             (int)num_clusters);
  if (num_chunks == 0) return B200_OK;
  CtxScope scope(ctx);
  return assign_clusters(soft, num_chunks, num_clusters, constrained, (signed char*)hard, (cudaStream_t)stream);
}

}  // extern "C"
