// The MFCC front end of XVectorMFCC (models/embedding/xvector.py:42-202): torchaudio's
// MFCC(sample_rate=16000, n_mfcc=40, dct_type=2, norm="ortho", log_mels=False), i.e. a centred, reflect-padded STFT
// (Hann window and n_fft 400, hop 200) -> power spectrum (201 bins) -> 128-filter mel bank -> AmplitudeToDB("power",
// top_db=80) -> the 128 x 40 DCT, on nb utterances of L samples (F = 1 + L / 200 frames each).
//
// 1. mfcc_rows_kernel cuts each reflect-padded utterance into R = F + 1 rows of 200 samples (fp16 (hi, lo), 256 wide,
//    zero padded): frame t is rows t and t + 1.
// 2. The windowed DFT is a 2-tap implicit GEMM on gemm_tc_split (taps shift the A row by one): the basis rows hold
//    w[s] cos(2 pi k s / 400) (n = k) and w[s] sin(2 pi k s / 400) (n = 256 + k), so the window is folded in.
// 3. mfcc_mel_db_kernel: |X|^2, the mel projection over each filter's nonzero band, 10 log10(max(., 1e-10)), and the
//    per-utterance maximum of the dB values (AmplitudeToDB's top_db reference is the maximum over the whole utterance,
//    all frames and filters, so no frame can be clamped before every frame of its utterance is done: a second kernel).
// 4. mfcc_dct_kernel: max(dB, max - 80) and the DCT, written as the first TDNN layer's fp16 (hi, lo) input rows
//    [nb * F][64] (40 coefficients, 24 zero columns), or as fp32 [nb * F][40] coefficients.
#include "common.cuh"
#include "emb.cuh"
#include "seg.cuh"

namespace b200 {

namespace {

constexpr int kMelFrames = 8;      // frames per CTA of the mel / dB kernel
constexpr int kDctFrames = 16;     // frames per CTA of the DCT kernel
constexpr float kAmin = 1e-10f;    // AmplitudeToDB's amin
constexpr float kDbFloor = -100.f; // 10 log10(amin) as torch computes it in fp32: the dB value of a zero-energy filter
constexpr float kTopDb = 80.f;

// order-preserving int image of a float, so that atomicMax on ints is a max on floats of any sign
__device__ __forceinline__ int ordered_key(float f) {
  const int i = __float_as_int(f);
  return i >= 0 ? i : i ^ 0x7FFFFFFF;
}
__device__ __forceinline__ float ordered_value(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7FFFFFFF); }

// rows [b * R + r][256] = samples 200 (r - 1) + c, c < 200, of utterance b reflected at both ends (torch.stft's
// center=True padding of n_fft / 2 = 200); columns 200..255 zero.  Also resets the utterance's dB maximum.
__global__ void __launch_bounds__(256) mfcc_rows_kernel(const float* __restrict__ wav, const long long* __restrict__ off,
                                                        int L, int R, __half* __restrict__ hi, __half* __restrict__ lo,
                                                        int* __restrict__ db_max) {
  const int r = blockIdx.x, b = blockIdx.y, c = threadIdx.x;
  if (r == 0 && c == 0) db_max[b] = ordered_key(-INFINITY);
  float v = 0.f;
  if (c < kMfccHop) {
    int i = kMfccHop * (r - 1) + c;
    if (i < 0) i = -i;
    if (i >= L) i = 2 * (L - 1) - i;
    v = wav[off[b] + i];
  }
  const size_t o = ((size_t)b * R + r) * kMfccRowLd + c;
  const __half h = __float2half_rn(v);
  hi[o] = h;
  lo[o] = __float2half_rn(v - __half2float(h));
}

// spec rows [b * R + t][512] (cos part at k, sin part at 256 + k) -> dB [b * F + t][128]; db_max[b] = max over all
__global__ void __launch_bounds__(kMfccMels) mfcc_mel_db_kernel(const float* __restrict__ spec, int F, int R,
                                                               const int* __restrict__ band_start,
                                                               const int* __restrict__ band_len,
                                                               const int* __restrict__ band_off,
                                                               const float* __restrict__ band_w, float* __restrict__ db,
                                                               int* __restrict__ db_max) {
  __shared__ float pw[kMelFrames][kMfccBins];
  __shared__ float wmax[kMfccMels / 32];
  const int b = blockIdx.y, t0 = blockIdx.x * kMelFrames, m = threadIdx.x;
  for (int i = threadIdx.x; i < kMelFrames * kMfccBins; i += blockDim.x) {
    const int f = i / kMfccBins, k = i - f * kMfccBins;
    float p = 0.f;
    if (t0 + f < F) {
      const float* row = spec + ((size_t)b * R + t0 + f) * kMfccSpecLd;
      const float a = hypotf(row[k], row[kMfccSpecLd / 2 + k]);      // spec.abs().pow(2), as torchaudio's Spectrogram
      p = a * a;
    }
    pw[f][k] = p;
  }
  __syncthreads();
  const int s = band_start[m], n = band_len[m], o = band_off[m];
  float mx = -INFINITY;
  for (int f = 0; f < kMelFrames && t0 + f < F; ++f) {
    float acc = 0.f;
    for (int j = 0; j < n; ++j) acc = fmaf(pw[f][s + j], band_w[o + j], acc);
    const float v = acc > kAmin ? 10.f * log10f(acc) : kDbFloor;
    db[((size_t)b * F + t0 + f) * kMfccMels + m] = v;
    mx = fmaxf(mx, v);
  }
  for (int d = 16; d > 0; d >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, d));
  if ((m & 31) == 0) wmax[m >> 5] = mx;
  __syncthreads();
  if (m == 0) {
    for (int w = 1; w < kMfccMels / 32; ++w) mx = fmaxf(mx, wmax[w]);
    atomicMax(db_max + b, ordered_key(mx));
  }
}

// max(dB, max_b - 80) -> DCT: fp16 (hi, lo) rows [b * F + t][64] when hi != NULL, else fp32 out [b * F + t][40]
__global__ void __launch_bounds__(128) mfcc_dct_kernel(const float* __restrict__ db, const int* __restrict__ db_max,
                                                       const float* __restrict__ dct, int F, __half* __restrict__ hi,
                                                       __half* __restrict__ lo, float* __restrict__ out) {
  __shared__ float sd[kMfccMels * kMfccCoefs];
  __shared__ float sx[kDctFrames][kMfccMels];
  const int b = blockIdx.y, t0 = blockIdx.x * kDctFrames;
  const float floor_db = ordered_value(db_max[b]) - kTopDb;
  for (int i = threadIdx.x; i < kMfccMels * kMfccCoefs; i += blockDim.x) sd[i] = dct[i];
  for (int i = threadIdx.x; i < kDctFrames * kMfccMels; i += blockDim.x) {
    const int f = i / kMfccMels, m = i - f * kMfccMels;
    sx[f][m] = t0 + f < F ? fmaxf(db[((size_t)b * F + t0 + f) * kMfccMels + m], floor_db) : 0.f;
  }
  __syncthreads();
  const int c = threadIdx.x & 63;
  for (int f = threadIdx.x >> 6; f < kDctFrames && t0 + f < F; f += 2) {
    float acc = 0.f;
    if (c < kMfccCoefs)
      for (int m = 0; m < kMfccMels; ++m) acc = fmaf(sx[f][m], sd[m * kMfccCoefs + c], acc);
    const size_t row = (size_t)b * F + t0 + f;
    if (hi) {
      const __half h = __float2half_rn(acc);
      hi[row * kMfccRowsOut + c] = h;
      lo[row * kMfccRowsOut + c] = __float2half_rn(acc - __half2float(h));
    } else if (c < kMfccCoefs) {
      out[row * kMfccCoefs + c] = acc;
    }
  }
}

struct MfccWs {
  __half *ah, *al;
  float* spec;
  float* db;
  int* db_max;
};

size_t carve_mfcc(int L, int nb, void* base, MfccWs* w) {
  Workspace ws(base, 1024);
  const size_t F = (size_t)mfcc_num_frames(L), R = F + 1;
  MfccWs t;
  t.ah = (__half*)ws.take((size_t)nb * R * kMfccRowLd * sizeof(__half));
  t.al = (__half*)ws.take((size_t)nb * R * kMfccRowLd * sizeof(__half));
  t.spec = (float*)ws.take((size_t)nb * R * kMfccSpecLd * sizeof(float));
  t.db = (float*)ws.take((size_t)nb * F * kMfccMels * sizeof(float));
  t.db_max = (int*)ws.take((size_t)nb * sizeof(int));
  if (w) *w = t;
  return ws.bytes();
}

}  // namespace

size_t mfcc_workspace_bytes(int L, int nb) { return carve_mfcc(L, nb, nullptr, nullptr); }

int mfcc_forward(const MfccWeights& W, const float* wav, const long long* off, int L, int nb, void* ws, __half* x_hi,
                 __half* x_lo, float* out, int num_sms, cudaStream_t st) {
  B200_CHECK(L > kMfccFft / 2 && nb >= 1 && nb <= 65535, B200_ERR_INVALID, "mfcc_forward: %d x %d samples", nb, L);
  const int F = mfcc_num_frames(L), R = F + 1;
  MfccWs w;
  carve_mfcc(L, nb, ws, &w);
  int rc;
  if ((rc = launch(mfcc_rows_kernel, dim3(R, nb), 256, 0, st, wav, off, L, R, w.ah, w.al, w.db_max))) return rc;
  // output row b * R + t reads rows b * R + t and + 1; the last row of every utterance (t = F) is computed and unused
  GemmTaps taps;
  taps.taps = 2;
  taps.dil = 1;
  if ((rc = gemm_tc_split(w.ah, w.al, kMfccRowLd, W.dft_hi, W.dft_lo, 2 * kMfccRowLd, w.spec, kMfccSpecLd, nullptr,
                          nullptr, 0, nullptr, nb * R, kMfccSpecLd, 2 * kMfccRowLd, 0, num_sms, st, nullptr, 0, taps)))
    return rc;
  if ((rc = launch(mfcc_mel_db_kernel, dim3(ceil_div(F, kMelFrames), nb), kMfccMels, 0, st, w.spec, F, R,
                   W.band_start, W.band_len, W.band_off, W.band_w, w.db, w.db_max)))
    return rc;
  return launch(mfcc_dct_kernel, dim3(ceil_div(F, kDctFrames), nb), 128, 0, st, w.db, w.db_max, W.dct, F, x_hi, x_lo,
                out);
}

}  // namespace b200
