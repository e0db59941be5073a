// SincNet front-end kernels (fp32 SIMT; the reference computes this in true fp32, TF32 off).
//
// Reference: /root/reference/src/pyannote/audio/models/blocks/sincnet.py:163-184
//   wav_norm1d (InstanceNorm1d(1, affine), instance stats, biased var, eps 1e-5)
//   -> 80 sinc band-pass FIRs (K=251, stride 10) -> |.| -> MaxPool1d(3,3) -> InstanceNorm1d(80) -> leaky_relu
//   -> Conv1d(80,60,5) -> MaxPool -> InstanceNorm1d(60) -> leaky_relu
//   -> Conv1d(60,60,5) -> MaxPool -> InstanceNorm1d(60) -> leaky_relu            => (B,60,F), F = 589 for 10 s
//
// Kernel plan for windows of any length W (SegGeom).  Each InstanceNorm needs whole-window statistics, so every stage
// ends in per-tile partial sums and the normalisation + leaky_relu is applied by the *consumer* when it loads its
// input tile:
//   wav_stats -> sinc_pool -> in_finalize -> conv5_pool<80> -> in_finalize -> conv5_pool<60> -> in_finalize
//   -> in_apply_transpose (writes the LSTM input [B][F][64], zero-padded 60->64).
// The sinc filters are (anti)symmetric (cos bank even, sin bank odd), which halves the multiplies:
//   cos: sum_k<125 f[k]*(x[a+k]+x[a+250-k]) + f[125]*x[a+125];  sin: sum_k<125 f[k]*(x[a+k]-x[a+250-k]).
#include "common.cuh"
#include "seg.cuh"

namespace b200 {

constexpr int kTileP = kSegTileP;                   // pooled outputs per tile
constexpr int kWavSlice = kChunk;                   // samples per wav_stats block (a 10 s window is one block)
constexpr int kFinGroup = 128;                      // partial sums one thread combines per InstanceNorm level

// ---- per-window waveform statistics -> affine (scale, shift) -------------------------------------
// Every InstanceNorm normalises over the whole padded window: the zero padding counts, so the denominators are W.
__device__ __forceinline__ float2 wav_affine(double S, double SS, int W, float gamma, float beta) {
  const double mean = S / W;                           // zero padding counts (the reference pads, then normalises)
  double var = SS / W - mean * mean;
  if (var < 0) var = 0;
  const float rstd = (float)(1.0 / sqrt(var + 1e-5));
  const float sc = gamma * rstd;
  return make_float2(sc, beta - (float)mean * sc);
}

// grid (ceil(W / kWavSlice), NB): block (slice, b) sums the real samples of one slice.  With one slice the block
// writes the affine itself; otherwise it writes (sum, sum of squares) and wav_finalize_kernel combines the slices
// in slice order, so a window's result does not depend on the other windows of its sub-batch.
__global__ void __launch_bounds__(512) wav_stats_kernel(const float* __restrict__ wav,
                                                        const long long* __restrict__ chunk_off,
                                                        const int* __restrict__ chunk_valid, int W, float gamma,
                                                        float beta, float2* __restrict__ affine,
                                                        double2* __restrict__ part) {
  const int slice = blockIdx.x, b = blockIdx.y, nslices = gridDim.x;
  const float* x = wav + chunk_off[b];
  const int lo = slice * kWavSlice;
  const int hi = (int)min((long long)chunk_valid[b], (long long)lo + kWavSlice);
  double s = 0.0, ss = 0.0;
  for (int i = lo + threadIdx.x; i < hi; i += blockDim.x) {
    const double v = x[i];
    s += v;
    ss += v * v;
  }
  __shared__ double sh[2][16];
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
  }
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = s; sh[1][threadIdx.x >> 5] = ss; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double S = 0, SS = 0;
    for (int i = 0; i < 16; ++i) { S += sh[0][i]; SS += sh[1][i]; }
    if (nslices == 1) affine[b] = wav_affine(S, SS, W, gamma, beta);
    else part[(size_t)b * nslices + slice] = make_double2(S, SS);
  }
}

__global__ void wav_finalize_kernel(const double2* __restrict__ part, int nslices, int W, float gamma, float beta,
                                    float2* __restrict__ affine, int NB) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= NB) return;
  double S = 0, SS = 0;
  for (int t = 0; t < nslices; ++t) {
    const double2 p = part[(size_t)b * nslices + t];
    S += p.x;
    SS += p.y;
  }
  affine[b] = wav_affine(S, SS, W, gamma, beta);
}

// ---- sinc conv + abs + maxpool3 ------------------------------------------------------------------
// block = 128 threads: 64 position-threads (3 consecutive conv outputs = 1 pooled output each) x 2 channel halves
// (20 cos + 20 sin channels each).  smem: normalised samples of the tile + the half filter bank [126][80].
__global__ void __launch_bounds__(128) sinc_pool_kernel(const float* __restrict__ wav,
                                                        const long long* __restrict__ chunk_off,
                                                        const int* __restrict__ chunk_valid,
                                                        const float2* __restrict__ affine,
                                                        const float* __restrict__ filt /*[126][80]*/,
                                                        int W, float* __restrict__ P0 /*[B][80][Lp]*/, int Lp,
                                                        int ntiles, double2* __restrict__ part /*[B][80][ntiles]*/) {
  extern __shared__ float sm[];
  float* xs = sm;                    // 2176
  float* fs = sm + 2176;             // 126*80
  const int tile = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x;
  const int j = tid & 63;            // pooled position inside the tile
  const int half = tid >> 6;         // channel half
  const float2 af = affine[b];
  const float* x = wav + chunk_off[b];
  const int valid = chunk_valid[b];
  const int s0 = tile * kTileP * 30; // first sample of the tile (3 conv outputs x stride 10 per pooled output)
  for (int i = tid; i < 2176; i += 128) {
    const int g = s0 + i;
    const float raw = (g < valid) ? x[g] : 0.f;
    xs[i] = (g < W) ? fmaf(raw, af.x, af.y) : 0.f;
  }
  for (int i = tid; i < 126 * 80 / 4; i += 128)
    reinterpret_cast<float4*>(fs)[i] = reinterpret_cast<const float4*>(filt)[i];
  __syncthreads();

  // accumulators as packed channel pairs (c, c+1)
  f32x2_t ac2[3][10], as2[3][10];
#pragma unroll
  for (int p = 0; p < 3; ++p)
#pragma unroll
    for (int c = 0; c < 10; ++c) { ac2[p][c] = 0ull; as2[p][c] = 0ull; }
  const float* xb = xs + j * 30;
  for (int k = 0; k < 125; ++k) {
    f32x2_t sv[3], dv[3];
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      const float a = xb[p * 10 + k], m = xb[p * 10 + 250 - k];
      sv[p] = pack2(a + m, a + m);
      dv[p] = pack2(a - m, a - m);
    }
    const ulonglong2* fc = reinterpret_cast<const ulonglong2*>(fs + k * 80 + half * 20);
    const ulonglong2* fn = reinterpret_cast<const ulonglong2*>(fs + k * 80 + 40 + half * 20);
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      const ulonglong2 wc = fc[q], wn = fn[q];
#pragma unroll
      for (int p = 0; p < 3; ++p) {
        ffma2(ac2[p][2 * q], sv[p], wc.x);
        ffma2(ac2[p][2 * q + 1], sv[p], wc.y);
        ffma2(as2[p][2 * q], dv[p], wn.x);
        ffma2(as2[p][2 * q + 1], dv[p], wn.y);
      }
    }
  }
  {  // centre tap (cos bank only; the sin bank's centre is exactly 0)
    const ulonglong2* fc = reinterpret_cast<const ulonglong2*>(fs + 125 * 80 + half * 20);
    f32x2_t xc[3];
#pragma unroll
    for (int p = 0; p < 3; ++p) xc[p] = pack2(xb[p * 10 + 125], xb[p * 10 + 125]);
#pragma unroll
    for (int q = 0; q < 5; ++q) {
      const ulonglong2 wc = fc[q];
#pragma unroll
      for (int p = 0; p < 3; ++p) {
        ffma2(ac2[p][2 * q], xc[p], wc.x);
        ffma2(ac2[p][2 * q + 1], xc[p], wc.y);
      }
    }
  }
  float ac[3][20], as[3][20];
#pragma unroll
  for (int p = 0; p < 3; ++p)
#pragma unroll
    for (int c = 0; c < 10; ++c) {
      unpack2(ac2[p][c], ac[p][2 * c], ac[p][2 * c + 1]);
      unpack2(as2[p][c], as[p][2 * c], as[p][2 * c + 1]);
    }
  __syncthreads();                   // everyone done with fs -> reuse as pooled tile [80][65]
  float* pt = fs;
  const int pglob = tile * kTileP + j;
  const bool ok = pglob < Lp;
#pragma unroll
  for (int c = 0; c < 20; ++c) {
    const float vc = fmaxf(fmaxf(fabsf(ac[0][c]), fabsf(ac[1][c])), fabsf(ac[2][c]));
    const float vs = fmaxf(fmaxf(fabsf(as[0][c]), fabsf(as[1][c])), fabsf(as[2][c]));
    const int chc = half * 20 + c, chs = 40 + half * 20 + c;
    pt[chc * 65 + j] = ok ? vc : 0.f;
    pt[chs * 65 + j] = ok ? vs : 0.f;
    if (ok) {
      P0[((size_t)b * 80 + chc) * Lp + pglob] = vc;
      P0[((size_t)b * 80 + chs) * Lp + pglob] = vs;
    }
  }
  __syncthreads();
  if (tid < 80) {
    double s = 0.0, ss = 0.0;
    for (int i = 0; i < kTileP; ++i) {
      const double v = pt[tid * 65 + i];
      s += v;
      ss += v * v;
    }
    part[((size_t)b * 80 + tid) * ntiles + tile] = make_double2(s, ss);
  }
}

// ---- InstanceNorm finalize: partial sums -> per (chunk, channel) affine -------------------------------
__global__ void in_finalize_kernel(const double2* __restrict__ part, int ntiles, int n, int C,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float2* __restrict__ affine, int total) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = idx % C;
  double s = 0, ss = 0;
  for (int t = 0; t < ntiles; ++t) {
    const double2 p = part[(size_t)idx * ntiles + t];
    s += p.x;
    ss += p.y;
  }
  const double mean = s / n;
  double var = ss / n - mean * mean;
  if (var < 0) var = 0;
  const float rstd = (float)(1.0 / sqrt(var + 1e-5));
  const float sc = gamma[c] * rstd;
  affine[idx] = make_float2(sc, beta[c] - (float)mean * sc);
}

// Long windows have thousands of tiles per (window, channel): one level of the reduction combines the partial sums
// of kFinGroup consecutive tiles, in tile order, per thread.
__global__ void part_reduce_kernel(const double2* __restrict__ in, int n_in, double2* __restrict__ out, int n_out,
                                   int rows) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= rows * n_out) return;
  const int row = idx / n_out, g = idx - row * n_out;
  const double2* p = in + (size_t)row * n_in + (size_t)g * kFinGroup;
  const int n = min(kFinGroup, n_in - g * kFinGroup);
  double s = 0, ss = 0;
  for (int t = 0; t < n; ++t) {
    s += p[t].x;
    ss += p[t].y;
  }
  out[idx] = make_double2(s, ss);
}

// partial sums [rows][ntiles] -> affine [rows]; up to kFinGroup tiles (every stage of a 10 s window) take the single
// in_finalize_kernel pass, more are first combined in groups into red0 / red1 (ping-pong)
static int in_stats(const double2* part, int ntiles, double2* red0, double2* red1, int n, int C, const float* gamma,
                    const float* beta, float2* affine, int rows, cudaStream_t stream) {
  const double2* cur = part;
  double2* bufs[2] = {red0, red1};
  int k = 0, rc;
  while (ntiles > kFinGroup) {
    const int n_out = ceil_div(ntiles, kFinGroup);
    if ((rc = launch(part_reduce_kernel, ceil_div(rows * n_out, 256), 256, 0, stream, cur, ntiles, bufs[k], n_out,
                     rows)))
      return rc;
    cur = bufs[k];
    ntiles = n_out;
    k ^= 1;
  }
  return launch(in_finalize_kernel, ceil_div(rows, 128), 128, 0, stream, cur, ntiles, n, C, gamma, beta, affine, rows);
}

// ---- Conv1d(CIN,60,5) + maxpool3 on the normalised, leaky-relu'd input --------------------------------
// block = 192 threads: 64 position-threads (3 conv outputs = 1 pooled) x 3 channel groups of 20.
template <int CIN>
__global__ void __launch_bounds__(192) conv5_pool_kernel(const float* __restrict__ Pin, int Lin,
                                                         const float2* __restrict__ affine /*[B][CIN]*/,
                                                         const float* __restrict__ Wc /*[CIN][5][60]*/,
                                                         const float* __restrict__ bias /*[60]*/,
                                                         float* __restrict__ Pout, int Lp, int ntiles,
                                                         double2* __restrict__ part /*[B][60][ntiles]*/) {
  constexpr int TW = 3 * kTileP + 4;   // 196 input positions per tile
  constexpr int CCH = 20;              // input channels per weight stage
  extern __shared__ float sm[];
  float* xin = sm;                     // [CIN][TW]
  float* ws = sm + CIN * TW;           // [CCH][5][60]
  const int tile = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x;
  const int j = tid & 63, grp = tid >> 6;
  const int t0 = tile * kTileP * 3;
  for (int i = tid; i < CIN * TW; i += 192) {
    const int ci = i / TW, t = i - ci * TW;
    const int g = t0 + t;
    float v = 0.f;
    if (g < Lin) {
      const float2 af = affine[b * CIN + ci];
      v = fmaf(Pin[((size_t)b * CIN + ci) * Lin + g], af.x, af.y);
      v = v > 0.f ? v : 0.01f * v;
    }
    xin[i] = v;
  }
  f32x2_t acc2[3][10];                 // packed channel pairs (c, c+1)
#pragma unroll
  for (int p = 0; p < 3; ++p)
#pragma unroll
    for (int c = 0; c < 10; ++c) acc2[p][c] = 0ull;
  for (int c0 = 0; c0 < CIN; c0 += CCH) {
    __syncthreads();
    for (int i = tid; i < CCH * 5 * 60 / 4; i += 192)
      reinterpret_cast<float4*>(ws)[i] = reinterpret_cast<const float4*>(Wc + (size_t)c0 * 300)[i];
    __syncthreads();
#pragma unroll 2
    for (int cc = 0; cc < CCH; ++cc) {
      const float* xr = xin + (c0 + cc) * TW + j * 3;
      f32x2_t xv[7];
#pragma unroll
      for (int i = 0; i < 7; ++i) xv[i] = pack2(xr[i], xr[i]);
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        const ulonglong2* wp = reinterpret_cast<const ulonglong2*>(ws + (cc * 5 + k) * 60 + grp * 20);
#pragma unroll
        for (int q = 0; q < 5; ++q) {
          const ulonglong2 w4 = wp[q];
#pragma unroll
          for (int p = 0; p < 3; ++p) {
            ffma2(acc2[p][2 * q], xv[p + k], w4.x);
            ffma2(acc2[p][2 * q + 1], xv[p + k], w4.y);
          }
        }
      }
    }
  }
  float acc[3][20];
#pragma unroll
  for (int p = 0; p < 3; ++p)
#pragma unroll
    for (int c = 0; c < 10; ++c) unpack2(acc2[p][c], acc[p][2 * c], acc[p][2 * c + 1]);
  __syncthreads();
  float* pt = ws;                      // pooled tile [60][65] = 3900 floats <= 6000
  const int pglob = tile * kTileP + j;
  const bool ok = pglob < Lp;
#pragma unroll
  for (int c = 0; c < 20; ++c) {
    const int co = grp * 20 + c;
    const float v = fmaxf(fmaxf(acc[0][c], acc[1][c]), acc[2][c]) + bias[co];
    pt[co * 65 + j] = ok ? v : 0.f;
    if (ok) Pout[((size_t)b * 60 + co) * Lp + pglob] = v;
  }
  __syncthreads();
  if (tid < 60) {
    double s = 0.0, ss = 0.0;
    for (int i = 0; i < kTileP; ++i) {
      const double v = pt[tid * 65 + i];
      s += v;
      ss += v * v;
    }
    part[((size_t)b * 60 + tid) * ntiles + tile] = make_double2(s, ss);
  }
}

// ---- final InstanceNorm + leaky_relu + transpose to the LSTM input layout [B][T][64] -----------------
__global__ void in_apply_transpose_kernel(const float* __restrict__ P2, const float2* __restrict__ affine,
                                          float* __restrict__ x0, int NB, int T) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)NB * T * 64;
  if (idx >= total) return;
  const int c = idx & 63;
  const int row = (int)(idx >> 6);
  const int b = row / T, t = row - b * T;
  float v = 0.f;
  if (c < 60) {
    const float2 af = affine[b * 60 + c];
    v = fmaf(P2[((size_t)b * 60 + c) * T + t], af.x, af.y);
    v = v > 0.f ? v : 0.01f * v;
  }
  x0[idx] = v;
}

// ---- host ------------------------------------------------------------------------------------------
struct SincWs {
  float2 *af_wav, *af0, *af1, *af2;
  double2 *wav_part, *part0, *part1, *part2, *red0, *red1;
  float *P0, *P1, *P2;
};

static int wav_slices(const SegGeom& g) { return ceil_div(g.W, kWavSlice); }

static size_t carve(const SegGeom& g, int NB, void* base, SincWs* w) {
  Workspace ws(base, 256);
  SincWs t;
  t.af_wav = (float2*)ws.take(sizeof(float2) * NB);
  t.af0 = (float2*)ws.take(sizeof(float2) * NB * 80);
  t.af1 = (float2*)ws.take(sizeof(float2) * NB * 60);
  t.af2 = (float2*)ws.take(sizeof(float2) * NB * 60);
  t.part0 = (double2*)ws.take(sizeof(double2) * (size_t)NB * 80 * g.tiles0);
  t.part1 = (double2*)ws.take(sizeof(double2) * (size_t)NB * 60 * g.tiles1);
  t.part2 = (double2*)ws.take(sizeof(double2) * (size_t)NB * 60 * g.tiles2);
  t.P0 = (float*)ws.take(sizeof(float) * (size_t)NB * 80 * g.pool0);
  t.P1 = (float*)ws.take(sizeof(float) * (size_t)NB * 60 * g.pool1);
  t.P2 = (float*)ws.take(sizeof(float) * (size_t)NB * 60 * g.pool2);
  t.wav_part = nullptr;
  t.red0 = t.red1 = nullptr;
  if (wav_slices(g) > 1) t.wav_part = (double2*)ws.take(sizeof(double2) * (size_t)NB * wav_slices(g));
  if (g.tiles0 > kFinGroup) {   // the largest stage's first reduction level; later levels are smaller
    const size_t n = (size_t)NB * 80 * ceil_div(g.tiles0, kFinGroup);
    t.red0 = (double2*)ws.take(sizeof(double2) * n);
    t.red1 = (double2*)ws.take(sizeof(double2) * n);
  }
  if (w) *w = t;
  return ws.bytes();
}

size_t sincnet_workspace_bytes(const SegGeom& g, int NB) { return carve(g, NB, nullptr, nullptr); }

int capture(void* dst, const void* src, size_t bytes, cudaStream_t stream) {
  if (dst && bytes) B200_CUDA_OK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, stream));
  return B200_OK;
}

int sincnet_forward(const SincNetWeights& W, const SegGeom& g, const float* wav, const long long* chunk_off,
                    const int* chunk_valid, int NB, void* ws, float* x0, int conv_impl, cudaStream_t stream,
                    const SegCapture* cap) {
  SincWs w;
  carve(g, NB, ws, &w);
  const SegCapture none{};
  const SegCapture& c = cap ? *cap : none;
  const size_t f2 = sizeof(float2) * NB;
  const size_t smem_sinc = (2176 + 126 * 80) * sizeof(float);
  const size_t smem_c80 = (80 * 196 + 20 * 300) * sizeof(float);
  const size_t smem_c60 = (60 * 196 + 20 * 300) * sizeof(float);
  const int nslices = wav_slices(g);
  int rc;
  if ((rc = launch(wav_stats_kernel, dim3(nslices, NB), 512, 0, stream, wav, chunk_off, chunk_valid, g.W, W.wav_w,
                   W.wav_b, w.af_wav, w.wav_part)))
    return rc;
  if (nslices > 1 && (rc = launch(wav_finalize_kernel, ceil_div(NB, 128), 128, 0, stream, w.wav_part, nslices, g.W,
                                  W.wav_w, W.wav_b, w.af_wav, NB)))
    return rc;
  if ((rc = capture(c.af_wav, w.af_wav, f2, stream))) return rc;
  // conv_impl: 1 = persistent split-fp16 wgmma kernels (default), 2 = one wgmma CTA per tile, 0 = the fp32 CUDA-core
  // twins
  if (conv_impl) {
    if ((rc = sinc_wg_forward(g, wav, chunk_off, chunk_valid, w.af_wav, W.sinc_wg_hi, W.sinc_wg_lo, NB, w.P0, w.part0,
                              conv_impl, stream)))
      return rc;
  } else {
    if ((rc = launch(sinc_pool_kernel, dim3(g.tiles0, NB), 128, smem_sinc, stream, wav, chunk_off, chunk_valid,
                     w.af_wav, W.sinc_f, g.W, w.P0, g.pool0, g.tiles0, w.part0)))
      return rc;
  }
  if ((rc = in_stats(w.part0, g.tiles0, w.red0, w.red1, g.pool0, 80, W.in_gamma[0], W.in_beta[0], w.af0, NB * 80,
                     stream)))
    return rc;
  if ((rc = capture(c.P0, w.P0, sizeof(float) * NB * 80 * g.pool0, stream))) return rc;
  if ((rc = capture(c.af0, w.af0, f2 * 80, stream))) return rc;
  if (conv_impl) {
    if ((rc = conv5_wg_forward(g, 0, w.P0, w.af0, W.conv_wg_hi[0], W.conv_wg_lo[0], W.conv_b[0], NB, w.P1, w.part1,
                               conv_impl, stream)))
      return rc;
  } else {
    if ((rc = launch(conv5_pool_kernel<80>, dim3(g.tiles1, NB), 192, smem_c80, stream, w.P0, g.pool0, w.af0,
                     W.conv_w[0], W.conv_b[0], w.P1, g.pool1, g.tiles1, w.part1)))
      return rc;
  }
  if ((rc = in_stats(w.part1, g.tiles1, w.red0, w.red1, g.pool1, 60, W.in_gamma[1], W.in_beta[1], w.af1, NB * 60,
                     stream)))
    return rc;
  if ((rc = capture(c.P1, w.P1, sizeof(float) * NB * 60 * g.pool1, stream))) return rc;
  if ((rc = capture(c.af1, w.af1, f2 * 60, stream))) return rc;
  if (conv_impl) {
    if ((rc = conv5_wg_forward(g, 1, w.P1, w.af1, W.conv_wg_hi[1], W.conv_wg_lo[1], W.conv_b[1], NB, w.P2, w.part2,
                               conv_impl, stream)))
      return rc;
  } else {
    if ((rc = launch(conv5_pool_kernel<60>, dim3(g.tiles2, NB), 192, smem_c60, stream, w.P1, g.pool1, w.af1,
                     W.conv_w[1], W.conv_b[1], w.P2, g.pool2, g.tiles2, w.part2)))
      return rc;
  }
  if ((rc = in_stats(w.part2, g.tiles2, w.red0, w.red1, g.pool2, 60, W.in_gamma[2], W.in_beta[2], w.af2, NB * 60,
                     stream)))
    return rc;
  if ((rc = capture(c.P2, w.P2, sizeof(float) * NB * 60 * g.pool2, stream))) return rc;
  if ((rc = capture(c.af2, w.af2, f2 * 60, stream))) return rc;
  const size_t total = (size_t)NB * g.pool2 * 64;
  if ((rc = launch(in_apply_transpose_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, w.P2, w.af2, x0, NB,
                   g.pool2)))
    return rc;
  return capture(c.x0, x0, sizeof(float) * total, stream);
}

}  // namespace b200
