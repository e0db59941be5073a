// Embedding path (kaldi fbank -> ResNet34 or bottleneck ResNet trunk -> masked stats pooling -> Linear) declarations.
#pragma once
#include "common.cuh"

namespace b200 {

struct ConvLayer {
  int C_in = 0, C_out = 0, ksize = 3, stride = 1;
  __half* w = nullptr;     // device, [tap][C_out][C_in] fp16, BN scale folded
  float* bias = nullptr;   // device, [C_out] fp32 (folded BN shift)
};

struct ConvParams {
  int B, H_in, W_in, C_in;
  int H_out, W_out, C_out;
  int taps_h, taps_w, stride, pad;
  int Ck, tiles_w, num_tiles, relu;
  int band, bands;         // conv_row_kernel / conv_chunk_row_kernel: output rows per unit, units per column strip
                           // (num_tiles = units)
  const float* bias;
  const __half* residual;
  __half* out;
  // tensor-core plan: a box of a_rows pixels x Ck channels (a_tx bytes, padded to a_bytes); conv_tc_kernel: a stage =
  // a box + the weights of one tap x C_out x Ck (b_bytes); conv_row_kernel takes its plan from RowPlan
  uint32_t a_rows, a_tx, a_bytes, b_bytes, nstages, swizzle;
};

struct BlockWeights {
  ConvLayer conv1, conv2, shortcut;
  bool has_shortcut = false;
};

// Bottleneck (resnet.py:148-212): 1x1 conv1 (in -> p), 3x3 conv2 (p -> p, stride), 1x1 conv3 (p -> 4p)
struct BottleneckWeights {
  ConvLayer conv1, conv2, conv3, shortcut;
  bool has_shortcut = false;
};

struct EmbWeights {
  bool loaded = false;
  int C = 256;                   // trunk output channels: 256 (ResNet34) or 1024 (bottleneck trunks)
  float* conv1_w = nullptr;      // [32][9] folded
  float* conv1_b = nullptr;      // [32]
  std::vector<BlockWeights> blocks;             // ResNet34: 16 BasicBlocks
  std::vector<BottleneckWeights> bottlenecks;   // ResNet152 / 221 / 293: the Bottleneck blocks (blocks is empty)
  float* seg1_w = nullptr;       // [256][20 C] fp32 (PyTorch layout)
  float* seg1_b = nullptr;       // [256]
  __half* seg1_w_hi = nullptr;   // fp16 (hi, lo) split of seg1_w for the tensor-core GEMM
  __half* seg1_w_lo = nullptr;
  // fbank constants
  float* window = nullptr;       // [400] hamming
  float* mel_w = nullptr;        // packed non-zero mel weights
  int* mel_start = nullptr;      // [80] first fft bin
  int* mel_len = nullptr;        // [80] number of bins
  int* mel_off = nullptr;        // [80] offset into mel_w
  float* twiddle = nullptr;      // [256][2] cos/sin(-2 pi k / 512)
};

// impl: 0 = SIMT reference conv, 1 = wgmma tensor-core convs (conv_row_kernel where it applies), 2 = conv_tc_kernel for
// every conv (the bit-exact reference of conv_row_kernel and block_row_kernel)
int conv_forward(const ConvLayer& L, const __half* in, const __half* residual, __half* out, int B, int H_in, int W_in,
                 int relu, int impl, int num_sms, cudaStream_t stream);
// Whether a BasicBlock runs as one block_row_kernel under conv_impl `impl`: impl = 1, stride 1, no shortcut, 32
// channels (ResNet34 layer 1).
bool block_fused(const BlockWeights& B, int impl);
// relu(conv2(relu(conv1(in))) + in) of such a block (BN folded as in ConvLayer), NHWC fp16 [B][H][W][32]; out must not
// alias in.  Bit-identical to conv_forward(conv1) followed by conv_forward(conv2) with `in` as the residual.
int block_forward(const BlockWeights& B, const __half* in, __half* out, int Bn, int H, int W, int num_sms,
                  cudaStream_t stream);
// T0 fbank frames per segment (998 for 10 s); frame0 (device, [B], may be NULL = b * T0): first fbank row of each
// segment, see fbank_forward.  out: NHWC fp16 [B][80][T0][32]
int conv1_forward(const float* fbank, const float* fmean, const int* frame0, const float* w, const float* bias,
                  __half* out, int B, int T0, cudaStream_t stream);

// fbank with SHARED FRAMES.  The sliding chunks of a file overlap by 90 % and a chunk step of 16000 samples is exactly
// 100 frame hops, so frame k of chunk c IS frame k - 100 of chunk c + 1: the same 400 samples through the same
// arithmetic.  The host groups a sub-batch's chunks into runs of hop-aligned, overlapping full chunks; a run's frames
// are computed once into consecutive rows of `fbank` ([nrows][80] fp32) and segment b reads rows
// frame0[b] .. frame0[b] + 997 (conv1_forward, the per-segment mean).  Chunks that are short (valid < 160000: samples
// past `limit` read as zero) or not hop-aligned get a private run, and so does every segment when sharing is off
// (utterances of any length, the public b200_emb_fbank's [B][998][80]): rows b * T0 .. b * T0 + T0 - 1 of a
// sub-batch.  Bit-identical to one private run per chunk; 10x fewer frames on a pipeline batch.
struct FbankRun {
  long long src;   // sample offset of the run's first frame in `wav`
  int row0;        // first row of the run in `fbank`
  int limit;       // valid samples counted from src (INT_MAX for runs of full chunks)
};
// fmean[b] = mean of the T0 rows of segment b (frame0 as in conv1_forward, not NULL)
int fbank_forward(const EmbWeights& W, const float* wav, const FbankRun* runs, int nruns, int nrows,
                  const int* frame0, int B, int T0, float* fbank, float* fmean, cudaStream_t stream);
int fbank_center(float* fbank, const float* fmean, int B, cudaStream_t stream);
// NHWC fp16 [B][10][T][C] -> NCHW fp32 [B][C][10][T]
int frames_to_nchw(const __half* feat, float* out, int B, int T, int C, cudaStream_t stream);

// weighted statistics pooling for any T, S and Tw (pooling.py:30-61, 76-130) -> the fp16 (hi, lo) rows of the Linear:
// feat NHWC fp16 [B][10][T][C] (trunk output) or frames NCHW fp32 [B][C][10][T] (caller frames, exactly one of
// the two), w [B][S][Tw] or NULL (mean and std(correction=1) over the T frames, S = 1): u8 masks (trunk output only)
// or fp32 of any real values.  The weights reach the T frames by torch's CUDA nearest index (upsample_nearest1d).
// Up to kSpeakers speakers of a sequence share one read of its features.  T is split into slices of kPoolSlice
// frames; with several the per-slice fp32 sums are combined in fp64 in slice order (deterministic, no atomics).
// part: fp64 scratch of pool_scratch_bytes(B, S, T, C) bytes (none with one slice).  Rows of stats_hi / stats_lo:
// (b * S + s) * 20 C.  C = 256 or 1024.
constexpr int kPoolSlice = 512;
size_t pool_scratch_bytes(int B, int S, int T, int C, int H = 10);
template <typename W>   // uint8_t or float
int weighted_pool_forward(const __half* feat, const float* frames, const W* w, int B, int T, int S, int Tw, int C,
                          double* part, __half* stats_hi, __half* stats_lo, cudaStream_t stream);
// the same pooling on frame-major fp32 rows x [B][F][kPoolRowsLd] (XVectorSincNet's last TDNN layer): the first T
// frames and the first C channels of every sequence -> stats rows of ld_out fp16 (hi, lo), mean at c and std at C + c
// (StatsPool's [mean, std] concatenation).  part: pool_scratch_bytes(B, S, T, kPoolRowsLd, 1) bytes.
constexpr int kPoolRowsLd = 1536;
int weighted_pool_rows(const float* x, int F, int T, int C, const float* w, int B, int S, int Tw, double* part,
                       __half* stats_hi, __half* stats_lo, int ld_out, cudaStream_t stream);
// generic weighted pooling used by the known-answer tests: seq [B][F][T] fp32, w [B][S][Tw] fp32 -> [B][S][2F]
int stats_pool_generic(const float* seq, const float* w, float* out, int B, int F, int T, int S, int Tw,
                       cudaStream_t stream);

// MFCC front end of XVectorMFCC (xvec_mfcc.cu): torchaudio MFCC with its defaults at 16 kHz
constexpr int kMfccHop = 200, kMfccFft = 400, kMfccBins = 201, kMfccMels = 128, kMfccCoefs = 40;
constexpr int kMfccRowLd = 256;     // one 200-sample row of the padded signal, zero padded to whole 64-wide k-blocks
constexpr int kMfccSpecLd = 512;    // DFT output row: 201 cosine sums at k, 201 sine sums at 256 + k
constexpr int kMfccRowsOut = 64;    // the first TDNN layer's input rows: 40 coefficients, zero padded
inline int mfcc_num_frames(int L) { return 1 + L / kMfccHop; }
struct MfccWeights {
  __half* dft_hi = nullptr;         // [512][2 taps x 256] fp16 (hi, lo) windowed DFT basis (see xvec_mfcc.cu)
  __half* dft_lo = nullptr;
  int* band_start = nullptr;        // [128] first nonzero bin of every mel filter (0 and length 0 for an empty one)
  int* band_len = nullptr;          // [128]
  int* band_off = nullptr;          // [128] offset of the filter's band in band_w
  float* band_w = nullptr;          // the filters' weights over their bands, back to back
  float* dct = nullptr;             // [128][40] dct_mat
};
// workspace of mfcc_forward on nb utterances of L samples
size_t mfcc_workspace_bytes(int L, int nb);
// nb utterances wav[off[b] .. off[b] + L), L > 200 -> F = 1 + L / 200 frames of 40 coefficients per utterance: as
// fp16 (hi, lo) rows [nb * F][64] (x_hi / x_lo, zero columns 40..63) or, with x_hi NULL, fp32 rows [nb * F][40]
int mfcc_forward(const MfccWeights& W, const float* wav, const long long* off, int L, int nb, void* ws, __half* x_hi,
                 __half* x_lo, float* out, int num_sms, cudaStream_t st);

}  // namespace b200
