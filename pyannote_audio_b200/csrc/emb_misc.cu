// Embedding path: kaldi-compatible log-mel fbank and masked statistics pooling.
//
// fbank follows torchaudio.compliance.kaldi.fbank as called by the reference
//   (/root/reference/src/pyannote/audio/models/embedding/wespeaker/__init__.py:113-139):
//   x*32768 -> frames of 400 @ hop 160 (snip_edges) -> remove DC -> pre-emphasis 0.97 (replicate pad) ->
//   Hamming -> zero-pad to 512 -> |rFFT|^2 -> 80 triangular mel bins (20 Hz..Nyquist) -> log(max(., eps)).
// The global-mean centring over frames (:137-139) is produced as a separate [B][80] vector that the first
// conv subtracts on load.
//
// stats pooling follows models/blocks/pooling.py:30-61,76-130 via resnet.py:61-66 (TSTP): nearest
// interpolation of the weights (the 589-frame masks of a 10 s chunk) onto the trunk frames, weighted mean and weighted
// unbiased std.
#include "common.cuh"
#include "emb.cuh"
#include <type_traits>

namespace b200 {

constexpr int kFrameLen = 400;
constexpr int kFrameHop = 160;
constexpr int kFft = 512;
constexpr float kEps = 1.1920928955078125e-07f;

__device__ __forceinline__ int bitrev9(int x) { return __brev((unsigned)x) >> 23; }

// smem index with one pad word per 16 elements: the register-blocked FFT passes below read 16 consecutive or
// 16-strided elements per lane, both conflict-free with this padding
__device__ __forceinline__ int fpad(int i) { return i + (i >> 4); }
constexpr int kFftPad = kFft + kFft / 16;   // 544

// 4 radix-2 DIT stages on 16 values held in registers; tw(s, j) returns the twiddle of the butterfly whose upper
// input is local element j in local stage s
template <typename TW>
__device__ __forceinline__ void fft16_stages(float (&xr)[16], float (&xi)[16], TW tw) {
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    const int half = 1 << s;
#pragma unroll
    for (int bf = 0; bf < 8; ++bf) {
      const int pos = bf & (half - 1);
      const int j0 = ((bf >> s) << (s + 1)) + pos, j1 = j0 + half;
      float wr, wi;
      tw(s, pos, wr, wi);
      const float tr = wr * xr[j1] - wi * xi[j1];
      const float ti = wr * xi[j1] + wi * xr[j1];
      const float ur = xr[j0], ui = xi[j0];
      xr[j0] = ur + tr; xi[j0] = ui + ti;
      xr[j1] = ur - tr; xi[j1] = ui - ti;
    }
  }
}

// Round 2: one warp computes TWO frames.  A 512-point real FFT is a 256-point complex FFT of z[n] = x[2n] + i x[2n+1]
// followed by   X[k] = E[k] + W_512^k O[k],  E = (Z[k] + conj Z[256-k]) / 2,  O = (Z[k] - conj Z[256-k]) / 2i,
// and stages 0-7 of the register-blocked 512-point DIT schedule below already ARE two independent 256-point FFTs
// on the two halves of the array (stage 8 was the only one that mixed them): frame A lives in elements [0, 256),
// frame B in [256, 512), half a warp each.  Same arithmetic per butterfly, less than half of it per frame
// (the padded imaginary half of the old complex transform was all zeros).
__global__ void __launch_bounds__(256) fbank_kernel(const float* __restrict__ wav,
                                                    const FbankRun* __restrict__ runs, int nruns, int nrows,
                                                    const float* __restrict__ window,
                                                    const float* __restrict__ twiddle, const float* __restrict__ mel_w,
                                                    const int* __restrict__ mel_start, const int* __restrict__ mel_len,
                                                    const int* __restrict__ mel_off, float* __restrict__ out) {
  __shared__ float s_re[8][kFftPad];
  __shared__ float s_im[8][kFftPad];
  __shared__ float s_tw[256][2];
  __shared__ long long s_src[16];                           // first sample of each of this block's 16 frame rows
  __shared__ int s_lim[16];                                 // samples of the run still valid from there
  for (int i = threadIdx.x; i < 512; i += blockDim.x) (&s_tw[0][0])[i] = twiddle[i];
  if (threadIdx.x < 16) {
    // row -> run: last run whose first row is <= row (runs are sorted by row0, rows of a run are hop-spaced frames)
    int row = blockIdx.x * 16 + threadIdx.x;
    if (row >= nrows) row = nrows - 1;
    int lo = 0, hi = nruns - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (runs[mid].row0 <= row) lo = mid; else hi = mid - 1;
    }
    const FbankRun r = runs[lo];
    const int local = row - r.row0;
    s_src[threadIdx.x] = r.src + (long long)local * kFrameHop;
    const long long left = (long long)r.limit - (long long)local * kFrameHop;
    s_lim[threadIdx.x] = left < 0 ? 0 : (left > kFrameLen ? kFrameLen : (int)left);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int l = lane & 15, f = lane >> 4;                  // half-warp f owns frame row 2 * pair + f
  const int pair = blockIdx.x * 8 + warp;
  if (2 * pair >= nrows) return;                           // warp-uniform
  const int row = 2 * pair + f;                            // row == nrows (odd tail): computed on a clamped source, not stored
  float* re = s_re[warp];
  float* im = s_im[warp];
  const float* xw = wav + s_src[2 * warp + f];
  const int valid = s_lim[2 * warp + f];
  const int h0 = f << 8;                                   // this frame's half of the arrays

  // load + scale, frame mean (sample i = l + 16 j)
  float x[25];
  float sum = 0.f;
#pragma unroll
  for (int j = 0; j < 25; ++j) {
    const int g = l + 16 * j;                              // sample of the frame; xw already points at the frame
    const float v = (g < valid) ? xw[g] * 32768.0f : 0.f;
    x[j] = v;
    sum += v;
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum / (float)kFrameLen;
  // DC removal, pre-emphasis (previous sample from the neighbouring lane; sample 0 replicates itself), window;
  // z[n] = v[2n] + i v[2n+1] scattered to bit-reversed order: even lanes write real parts, odd lanes imaginary parts
  float* dst = (l & 1) ? im : re;
  float carry = 0.f;                                       // lane 15's sample of the previous j (for lane 0)
#pragma unroll
  for (int j = 0; j < 32; ++j) {
    const int i = l + 16 * j;
    float v = 0.f;
    if (j < 25) {
      const float cur = x[j] - mean;
      float prev = __shfl_up_sync(0xffffffffu, cur, 1, 16);
      if (l == 0) prev = (j == 0) ? cur : carry;
      carry = __shfl_sync(0xffffffffu, cur, 15, 16);
      v = (cur - 0.97f * prev) * window[i];
    }
    dst[fpad(h0 + (int)(__brev((unsigned)(i >> 1)) >> 24))] = v;
  }
  __syncwarp();
  // two 256-point radix-2 DIT FFTs (one per half-warp) as 4 + 4 stages: two register-blocked passes of 16 values
  float xr[16], xi[16];
  {  // stages 0-3: lane owns elements 16 lane .. 16 lane + 15 (lanes 16-31: the second frame's half)
#pragma unroll
    for (int j = 0; j < 16; ++j) { xr[j] = re[fpad(16 * lane + j)]; xi[j] = im[fpad(16 * lane + j)]; }
    fft16_stages(xr, xi, [&](int s, int pos, float& wr, float& wi) {
      const int k = pos * (256 >> s);                      // multiples of 32: compile-time after unrolling
      wr = s_tw[k][0];
      wi = s_tw[k][1];
    });
#pragma unroll
    for (int j = 0; j < 16; ++j) { re[fpad(16 * lane + j)] = xr[j]; im[fpad(16 * lane + j)] = xi[j]; }
  }
  __syncwarp();
  {  // stages 4-7: lane owns elements e0 + 16 j of its frame's half
    const int e0 = l + h0;
#pragma unroll
    for (int j = 0; j < 16; ++j) { xr[j] = re[fpad(e0 + 16 * j)]; xi[j] = im[fpad(e0 + 16 * j)]; }
    fft16_stages(xr, xi, [&](int s, int pos, float& wr, float& wi) {
      // global stage 4 + s, position inside the butterfly group = l + 16 pos
      const int k = (l + 16 * pos) * (16 >> s);
      wr = s_tw[k][0];
      wi = s_tw[k][1];
    });
#pragma unroll
    for (int j = 0; j < 16; ++j) { re[fpad(e0 + 16 * j)] = xr[j]; im[fpad(e0 + 16 * j)] = xi[j]; }
  }
  __syncwarp();
  // real-FFT split + power spectrum of bins 0..255 (the Nyquist bin carries zero mel weight: kaldi pads the bank with
  // a zero column); this lane's bins are k = l + 16 j
  float pw[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int k = l + 16 * j, km = (256 - k) & 255;
    const float zr = re[fpad(h0 + k)], zi = im[fpad(h0 + k)];
    const float mr = re[fpad(h0 + km)], mi = im[fpad(h0 + km)];
    const float er = 0.5f * (zr + mr), ei = 0.5f * (zi - mi);
    const float orr = 0.5f * (zi + mi), oi = -0.5f * (zr - mr);
    const float wr = s_tw[k][0], wi = s_tw[k][1];
    const float xr_ = er + (wr * orr - wi * oi), xi_ = ei + (wr * oi + wi * orr);
    const float a = sqrtf(xr_ * xr_ + xi_ * xi_);            // reference: rfft().abs().pow(2)
    pw[j] = a * a;
  }
  __syncwarp();
#pragma unroll
  for (int j = 0; j < 16; ++j) re[h0 + l + 16 * j] = pw[j];
  __syncwarp();
  for (int m = l; m < kMel; m += 16) {
    const int st = mel_start[m], ln = mel_len[m], off = mel_off[m];
    float acc = 0.f;
    for (int i = 0; i < ln; ++i) acc = fmaf(re[h0 + st + i], mel_w[off + i], acc);
    if (row < nrows) out[(size_t)row * kMel + m] = logf(fmaxf(acc, kEps));
  }
}

__global__ void __launch_bounds__(640) fbank_mean_kernel(const float* __restrict__ fb, const int* __restrict__ frame0,
                                                         int T0, float* __restrict__ fmean) {
  // 8 groups of 80 threads each sum an eighth of the T0 frames in fp64, combined in group order
  __shared__ double part[8][kMel];
  const int b = blockIdx.x, m = threadIdx.x % kMel, g = threadIdx.x / kMel;
  const size_t r0 = (size_t)frame0[b];
  double s = 0.0;
#pragma unroll 8
  for (int t = g; t < T0; t += 8) s += (double)fb[(r0 + t) * kMel + m];
  part[g][m] = s;
  __syncthreads();
  if (g == 0) {
    double tot = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) tot += part[k][m];
    fmean[(size_t)b * kMel + m] = (float)(tot / T0);
  }
}

__global__ void fbank_center_kernel(float* __restrict__ fb, const float* __restrict__ fmean, size_t total) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int m = idx % kMel;
  const int b = idx / ((size_t)kMel * kFbankFrames);
  fb[idx] -= fmean[b * kMel + m];
}

int fbank_center(float* fbank, const float* fmean, int B, cudaStream_t stream) {
  const size_t total = (size_t)B * kFbankFrames * kMel;
  return launch(fbank_center_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, fbank, fmean, total);
}

__global__ void frames_to_nchw_kernel(const __half* __restrict__ feat, float* __restrict__ out, int T, int C,
                                      size_t total) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // over NCHW output
  if (idx >= total) return;
  const size_t t = idx % T;
  const size_t h = (idx / T) % 10;
  const size_t c = (idx / ((size_t)T * 10)) % C;
  const size_t b = idx / ((size_t)T * 10 * C);
  out[idx] = __half2float(feat[((b * 10 + h) * T + t) * C + c]);
}

int frames_to_nchw(const __half* feat, float* out, int B, int T, int C, cudaStream_t stream) {
  const size_t total = (size_t)B * C * 10 * T;
  return launch(frames_to_nchw_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, feat, out, T, C, total);
}

int fbank_forward(const EmbWeights& W, const float* wav, const FbankRun* runs, int nruns, int nrows,
                  const int* frame0, int B, int T0, float* fbank, float* fmean, cudaStream_t stream) {
  const unsigned grid = (unsigned)ceil_div(nrows, 16);      // 8 warps x 2 frame rows per block
  const int rc = launch(fbank_kernel, grid, 256, 0, stream, wav, runs, nruns, nrows, W.window, W.twiddle, W.mel_w,
                        W.mel_start, W.mel_len, W.mel_off, fbank);
  if (rc) return rc;
  return launch(fbank_mean_kernel, B, 640, 0, stream, fbank, frame0, T0, fmean);
}

// ------------------------------------------------------------------------------------------------
// weighted statistics pooling for any T, S and Tw (diarization masks, utterances of any length, caller frames, soft
// weights)
// ------------------------------------------------------------------------------------------------
// torch's CUDA nearest index (upsample_nearest1d, the device F.interpolate(mode="nearest") runs on): scale is
// (float)Tw / T, src = min(floor(dst * scale), Tw - 1), with the exact special cases T == Tw and T == 2 Tw.  It differs
// from the integer t * Tw / T on a few frames of long sequences, but not for the 589-frame masks on the 125 trunk
// frames of 10 s: t * 589 / 125 is an integer only at t = 0 and otherwise at least 1/125 away from one, far more than
// the rounding error of t * (589.f / 125.f) for t < 125.
__device__ __forceinline__ int nearest_src(int dst, int T, int Tw, float scale) {
  if (T == Tw) return dst;
  if (T == 2 * Tw) return dst >> 1;
  return min((int)floorf((float)dst * scale), Tw - 1);
}

__device__ __forceinline__ float to_f(__half v) { return __half2float(v); }
__device__ __forceinline__ float to_f(float v) { return v; }

// feature layouts of the pooled sequence: NHWC fp16 [B][10][T][C] (trunk output), NCHW fp32 [B][C][10][T] (caller
// frames), frame-major fp32 rows [B][F][C] of which the first T frames are pooled (TDNN output, one "height")
enum { kPoolNHWC = 0, kPoolNCHW = 1, kPoolRows = 2 };
template <int L> using PoolX = typename std::conditional<L == kPoolNHWC, __half, float>::type;
template <int L> __host__ __device__ constexpr int pool_h() { return L == kPoolRows ? 1 : 10; }

// stats row of Cv channels at H heights: mean at c * H + h, std H * Cv further (the ResNet rows: H = 10, Cv = C)
__device__ __forceinline__ void store_split(__half* hi, __half* lo, size_t row, int c, int h, int H, int Cv, float mean,
                                            float sdv) {
  const __half mh = __float2half_rn(mean), sh = __float2half_rn(sdv);
  hi[row + c * H + h] = mh;
  lo[row + c * H + h] = __float2half_rn(mean - __half2float(mh));
  hi[row + H * Cv + c * H + h] = sh;
  lo[row + H * Cv + c * H + h] = __float2half_rn(sdv - __half2float(sh));
}

struct PoolArgs {
  const void* x;          // NHWC fp16 feat, NCHW fp32 frames or fp32 rows
  const void* w;          // [B][S][Tw] u8 or fp32, or NULL
  int S, T, Tw, nslices;
  float scale;            // (float)Tw / T
  int Cv;                 // channels pooled (C, or fewer than the row width C of kPoolRows)
  int F;                  // kPoolRows: frames per sequence (row stride of a sequence, >= T)
  int ld_out;             // width of an output stats row
  double* part;           // [B * S][H][nslices][4][C]: sum w (sum x), sum w^2, sum w x, sum w (x - mean)^2
  __half *hi, *lo;
};

// x of (b, h, channel c) and the stride between its frames
template <int L, int C>
__device__ __forceinline__ const PoolX<L>* pool_row(const PoolArgs& a, int b, int h, int c, size_t* stride) {
  const PoolX<L>* x = static_cast<const PoolX<L>*>(a.x);
  if constexpr (L == kPoolNHWC) { *stride = C; return x + ((size_t)b * 10 + h) * a.T * C + c; }
  else if constexpr (L == kPoolNCHW) { *stride = 1; return x + (((size_t)b * C + c) * 10 + h) * a.T; }
  else { *stride = C; return x + (size_t)b * a.F * C + c; }
}

// A block pools a group of up to kSpeakers speakers of one sequence, so that it reads x once for all of them; each
// speaker keeps its own sums, in the same order as a group of one.  Unweighted pooling has S = 1.
// PHASE 0: the whole sequence in one slice, finished here; PHASE 1: per-slice fp32 sums; PHASE 2: per-slice sum of
// w (x - mean)^2 around the mean of all slices' sums.  W: weight element type (u8 masks or fp32).
// grid (B * ceil(S / kSpeakers) * H, nslices, C / 256), thread = channel
template <int PHASE, int L, int C, typename W>
__global__ void __launch_bounds__(256) wpool_kernel(PoolArgs a) {
  constexpr int H = pool_h<L>();
  __shared__ float s_w[kSpeakers][kPoolSlice];
  const int groups = (a.S + kSpeakers - 1) / kSpeakers;
  const int grp = blockIdx.x / H, h = blockIdx.x % H;                        // grp = b * groups + g
  const int b = grp / groups, s0 = (grp % groups) * kSpeakers, ns = min(kSpeakers, a.S - s0);
  const int row0 = b * a.S + s0;                                             // row of speaker s0: b * S + s0
  const int c = (C == 256 ? 0 : (int)blockIdx.z * 256) + threadIdx.x;
  const int sl = blockIdx.y;
  const int t0 = sl * kPoolSlice, t1 = min(a.T, t0 + kPoolSlice), n = t1 - t0;
  size_t xs;
  const PoolX<L>* xp = pool_row<L, C>(a, b, h, c, &xs);
  // u8 weights are masks, always given: without the unweighted branch the mask kernel fits in 32 registers
  const bool weighted = std::is_same<W, uint8_t>::value || a.w != nullptr;
  if (weighted) {
    const W* w = static_cast<const W*>(a.w) + (size_t)row0 * a.Tw;
    for (int i = threadIdx.x; i < ns * n; i += blockDim.x) {
      const int s = i / n, t = i % n;
      s_w[s][t] = (float)w[(size_t)s * a.Tw + nearest_src(t0 + t, a.T, a.Tw, a.scale)];
    }
  }
  __syncthreads();
  if (L == kPoolRows && c >= a.Cv) return;                   // padding channels of the rows
  // slot k of slice j of speaker s0 + s: part[s * pstride + (j * 4 + k) * C]
  const size_t pstride = (size_t)H * a.nslices * 4 * C;
  double* part = a.part + (((size_t)row0 * H + h) * a.nslices) * 4 * C + c;
  if (PHASE == 0 || PHASE == 1) {
    float v1[kSpeakers], v2[kSpeakers], sx[kSpeakers];
#pragma unroll
    for (int s = 0; s < kSpeakers; ++s) { v1[s] = 0.f; v2[s] = 0.f; sx[s] = 0.f; }
    if (weighted) {
      for (int t = t0; t < t1; ++t) {
        const float x = to_f(xp[(size_t)t * xs]);
#pragma unroll
        for (int s = 0; s < kSpeakers; ++s) {
          if (s < ns) {
            const float w = s_w[s][t - t0];
            v1[s] += w;
            v2[s] += w * w;
            sx[s] += x * w;
          }
        }
      }
    } else {
      for (int t = t0; t < t1; ++t) sx[0] += to_f(xp[(size_t)t * xs]);
    }
    if (PHASE == 1) {
#pragma unroll
      for (int s = 0; s < kSpeakers; ++s) {
        if (s < ns) {
          part[s * pstride + (sl * 4 + 0) * C] = weighted ? (double)v1[s] : (double)sx[s];
          part[s * pstride + (sl * 4 + 1) * C] = (double)v2[s];
          part[s * pstride + (sl * 4 + 2) * C] = (double)sx[s];
        }
      }
      return;
    }
    if (weighted) {
      float mean[kSpeakers], sd[kSpeakers];
#pragma unroll
      for (int s = 0; s < kSpeakers; ++s) {
        v1[s] += 1e-8f;
        mean[s] = sx[s] / v1[s];
        sd[s] = 0.f;
      }
      for (int t = t0; t < t1; ++t) {
        const float x = to_f(xp[(size_t)t * xs]);
#pragma unroll
        for (int s = 0; s < kSpeakers; ++s) {
          if (s < ns) {
            const float d = x - mean[s];
            sd[s] += d * d * s_w[s][t - t0];
          }
        }
      }
#pragma unroll
      for (int s = 0; s < kSpeakers; ++s) {
        if (s < ns) {
          const float var = sd[s] / (v1[s] - v2[s] / v1[s] + 1e-8f);
          store_split(a.hi, a.lo, (size_t)(row0 + s) * a.ld_out, c, h, H, a.Cv, mean[s], sqrtf(var));
        }
      }
    } else {                                               // torch mean / std(correction=1): T = 1 gives NaN
      const float mean = sx[0] / a.T;
      float acc = 0.f;
      for (int t = t0; t < t1; ++t) {
        const float d = to_f(xp[(size_t)t * xs]) - mean;
        acc += d * d;
      }
      store_split(a.hi, a.lo, (size_t)row0 * a.ld_out, c, h, H, a.Cv, mean, sqrtf(acc / (a.T - 1)));
    }
  } else {
    float mean[kSpeakers], sd[kSpeakers];
#pragma unroll
    for (int s = 0; s < kSpeakers; ++s) {
      double m0 = 0.0, m2 = 0.0;                           // every slice's sums, in slice order
      if (s < ns)
        for (int j = 0; j < a.nslices; ++j) {
          m0 += part[s * pstride + (j * 4 + 0) * C];
          m2 += part[s * pstride + (j * 4 + 2) * C];
        }
      mean[s] = weighted ? (float)(m2 / (m0 + 1e-8)) : (float)(m0 / a.T);
      sd[s] = 0.f;
    }
    for (int t = t0; t < t1; ++t) {
      const float x = to_f(xp[(size_t)t * xs]);
#pragma unroll
      for (int s = 0; s < kSpeakers; ++s) {
        if (s < ns) {
          const float d = x - mean[s];
          sd[s] += weighted ? d * d * s_w[s][t - t0] : d * d;
        }
      }
    }
#pragma unroll
    for (int s = 0; s < kSpeakers; ++s)
      if (s < ns) part[s * pstride + (sl * 4 + 3) * C] = (double)sd[s];
  }
}

// combine the slices in fp64, in slice order; grid (B * S * H, 1, C / 256), thread = channel
template <int L, int C>
__global__ void __launch_bounds__(256) wpool_final_kernel(PoolArgs a) {
  constexpr int H = pool_h<L>();
  const int row = blockIdx.x / H, h = blockIdx.x % H;
  const int c = (C == 256 ? 0 : (int)blockIdx.z * 256) + threadIdx.x;
  if (L == kPoolRows && c >= a.Cv) return;
  const double* part = a.part + (((size_t)row * H + h) * a.nslices) * 4 * C + c;
  double s[4] = {0.0, 0.0, 0.0, 0.0};
  for (int j = 0; j < a.nslices; ++j)
#pragma unroll
    for (int k = 0; k < 4; ++k) s[k] += part[(j * 4 + k) * C];
  float mean;
  double var;
  if (a.w) {
    const double v1 = s[0] + 1e-8;
    mean = (float)(s[2] / v1);
    var = s[3] / (v1 - s[1] / v1 + 1e-8);
  } else {
    mean = (float)(s[0] / a.T);
    var = s[3] / (double)(a.T - 1);
  }
  store_split(a.hi, a.lo, (size_t)row * a.ld_out, c, h, H, a.Cv, mean, (float)sqrt(var));
}

size_t pool_scratch_bytes(int B, int S, int T, int C, int H) {
  const int nslices = ceil_div(T, kPoolSlice);
  return nslices > 1 ? (size_t)B * S * H * nslices * 4 * C * sizeof(double) : 0;
}

template <int L, int C, typename W>
static int wpool_launch(const PoolArgs& a, int B, cudaStream_t stream) {
  const unsigned H = pool_h<L>();
  const dim3 grid((unsigned)B * ceil_div(a.S, kSpeakers) * H, (unsigned)a.nslices, C / 256);
  if (a.nslices == 1) return launch(wpool_kernel<0, L, C, W>, grid, 256, 0, stream, a);
  int rc;
  if ((rc = launch(wpool_kernel<1, L, C, W>, grid, 256, 0, stream, a))) return rc;
  if ((rc = launch(wpool_kernel<2, L, C, W>, grid, 256, 0, stream, a))) return rc;
  return launch(wpool_final_kernel<L, C>, dim3((unsigned)B * a.S * H, 1, C / 256), 256, 0, stream, a);
}

static int pool_args(const void* x, const void* w, int B, int T, int S, int Tw, double* part, __half* stats_hi,
                     __half* stats_lo, PoolArgs* a) {
  B200_CHECK(x != nullptr && T >= 1 && S >= 1 && (w == nullptr ? S == 1 : Tw >= 1), B200_ERR_INVALID,
             "weighted pooling: bad arguments");
  a->x = x;
  a->w = w;
  a->S = S; a->T = T; a->Tw = w ? Tw : T;
  a->nslices = ceil_div(T, kPoolSlice);
  a->scale = (float)a->Tw / (float)T;
  a->part = part;
  a->hi = stats_hi; a->lo = stats_lo;
  B200_CHECK(a->nslices <= 65535 && (size_t)B * S * 10 <= 0x7fffffffu, B200_ERR_INVALID,
             "weighted pooling: %d frames x %lld rows is too large", T, (long long)B * S);
  B200_CHECK(a->nslices == 1 || part != nullptr, B200_ERR_INVALID, "weighted pooling: scratch missing");
  return B200_OK;
}

template <typename W>
int weighted_pool_forward(const __half* feat, const float* frames, const W* w, int B, int T, int S, int Tw, int C,
                          double* part, __half* stats_hi, __half* stats_lo, cudaStream_t stream) {
  constexpr bool fp32_w = std::is_same<W, float>::value;   // u8 masks: always given, on the trunk output only
  B200_CHECK((feat == nullptr) != (frames == nullptr) && (fp32_w || (feat && w)), B200_ERR_INVALID,
             "weighted pooling: bad arguments");
  PoolArgs a;
  int rc;
  if ((rc = pool_args(feat ? (const void*)feat : (const void*)frames, w, B, T, S, Tw, part, stats_hi, stats_lo, &a)))
    return rc;
  a.Cv = C; a.F = T; a.ld_out = 2 * 10 * C;
  B200_CHECK(C == 256 || C == 1024, B200_ERR_STATE, "weighted pooling: %d channels unsupported", C);
  if (feat)
    return C == 256 ? wpool_launch<kPoolNHWC, 256, W>(a, B, stream) : wpool_launch<kPoolNHWC, 1024, W>(a, B, stream);
  if constexpr (fp32_w)
    return C == 256 ? wpool_launch<kPoolNCHW, 256, W>(a, B, stream) : wpool_launch<kPoolNCHW, 1024, W>(a, B, stream);
  return B200_OK;
}
template int weighted_pool_forward(const __half*, const float*, const uint8_t*, int, int, int, int, int, double*,
                                   __half*, __half*, cudaStream_t);
template int weighted_pool_forward(const __half*, const float*, const float*, int, int, int, int, int, double*,
                                   __half*, __half*, cudaStream_t);

int weighted_pool_rows(const float* x, int F, int T, int C, const float* w, int B, int S, int Tw, double* part,
                       __half* stats_hi, __half* stats_lo, int ld_out, cudaStream_t stream) {
  PoolArgs a;
  int rc;
  if ((rc = pool_args(x, w, B, T, S, Tw, part, stats_hi, stats_lo, &a))) return rc;
  B200_CHECK(C >= 1 && C <= kPoolRowsLd && T <= F && ld_out >= 2 * C, B200_ERR_INVALID,
             "weighted pooling: %d channels of %d-wide rows, %d of %d frames", C, kPoolRowsLd, T, F);
  a.Cv = C; a.F = F; a.ld_out = ld_out;
  return wpool_launch<kPoolRows, kPoolRowsLd, float>(a, B, stream);
}

// generic fp32 version (any F, T, S, Tw) used by the known-answer tests of the reference.  It keeps the integer index
// t * Tw / T, which differs from torch's CUDA nearest index (nearest_src above) on a few frames of long sequences;
// moving it to nearest_src is left for later.
__global__ void stats_pool_generic_kernel(const float* __restrict__ seq, const float* __restrict__ w,
                                          float* __restrict__ out, int B, int F, int T, int S, int Tw) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= B * S * F) return;
  const int f = idx % F, s = (idx / F) % S, b = idx / (F * S);
  const float* x = seq + ((size_t)b * F + f) * T;
  float mean, sd;
  if (w == nullptr) {
    float sum = 0.f;
    for (int t = 0; t < T; ++t) sum += x[t];
    mean = sum / T;
    float acc = 0.f;
    for (int t = 0; t < T; ++t) acc += (x[t] - mean) * (x[t] - mean);
    sd = sqrtf(acc / (T - 1));
  } else {
    const float* ww = w + ((size_t)b * S + s) * Tw;
    float v1 = 0.f, v2 = 0.f, sx = 0.f;
    for (int t = 0; t < T; ++t) {
      const float wt = ww[(int)(((long long)t * Tw) / T)];
      v1 += wt; v2 += wt * wt; sx += x[t] * wt;
    }
    v1 += 1e-8f;
    mean = sx / v1;
    float acc = 0.f;
    for (int t = 0; t < T; ++t) {
      const float wt = ww[(int)(((long long)t * Tw) / T)];
      acc += (x[t] - mean) * (x[t] - mean) * wt;
    }
    sd = sqrtf(acc / (v1 - v2 / v1 + 1e-8f));
  }
  float* o = out + ((size_t)b * S + s) * 2 * F;
  o[f] = mean;
  o[F + f] = sd;
}

int stats_pool_generic(const float* seq, const float* w, float* out, int B, int F, int T, int S, int Tw,
                       cudaStream_t stream) {
  const int total = B * S * F;
  return launch(stats_pool_generic_kernel, ceil_div(total, 128), 128, 0, stream, seq, w, out, B, F, T, S, Tw);
}

}  // namespace b200
