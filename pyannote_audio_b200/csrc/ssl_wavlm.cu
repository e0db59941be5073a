// WavLM Base front end of SSeRiouSS (torchaudio models/wav2vec2/components.py + wavlm_attention.py, as called by
// SSeRiouSS.forward through Wav2Vec2Model.extract_features):
//
//   conv 0 (1 -> 512, k 10, s 5) -> GroupNorm(512, 512) over the window -> GELU        CUDA cores, fp32
//   convs 1-6 (512 -> 512, k 3 s 2 x4, k 2 s 2 x2) -> GELU                              split-precision wgmma GEMMs
//   LayerNorm(512) -> Linear 512 -> 768                                                 fp32 LN + wgmma GEMM
//   x = LN(x + GELU(grouped positional conv (16 groups, k 128, pad 64, last frame dropped)))
//                                                                                       16 implicit wgmma GEMMs
//   12 post-LN layers: x = LN(x + out(attn(qkv(x)))); x = LN(x + ff2(GELU(ff1(x))))      wgmma GEMMs + fp32 kernels
//   features = sum_l softmax(w)_l * x_l  (or the output of one layer)
//
// The conv activations are channel-last, so two consecutive frames of a window form one 1024-wide row: a stride-2
// conv of kernel 2 is a plain GEMM with K = 1024 and one of kernel 3 an implicit GEMM of 2 taps (GemmTaps, dilation
// 1) with K = 2048 whose second tap has the weights [W2, 0].  The attention is an online-softmax kernel on the CUDA
// cores in fp32: no T x T score matrix exists in memory.  The WavLM relative position bias of head h between query i
// and key j is gate[b][h][i] * rel_tab[h][j - i], with the gate computed from the layer's input.
#include "common.cuh"
#include "ssl.cuh"

namespace b200 {

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.f + erff(x * 0.70710678118654752f)); }

__device__ __forceinline__ void store_split(__half* hi, __half* lo, size_t i, float v) {
  const __half h = __float2half_rn(v);
  hi[i] = h;
  lo[i] = __float2half_rn(v - __half2float(h));
}

// ---- conv 0: raw[b][t][c] = sum_k w[c][k] x[b][5 t + k]  (samples past chunk_valid read as zero) --------------------
constexpr int kConv0T = 32;
__global__ void __launch_bounds__(512) ssl_conv0_kernel(const float* __restrict__ wav, const long long* __restrict__ off,
                                                        const int* __restrict__ valid, const float* __restrict__ w,
                                                        float* __restrict__ raw, int len, int stride) {
  __shared__ float xs[kConv0T * 5 + 10];
  const int b = blockIdx.y, t0 = blockIdx.x * kConv0T, c = threadIdx.x;
  const long long o = off[b];
  const int v = valid[b];
  for (int i = threadIdx.x; i < kConv0T * 5 + 10; i += blockDim.x) {
    const int s = t0 * 5 + i;
    xs[i] = s < v ? wav[o + s] : 0.f;
  }
  float wr[10];
#pragma unroll
  for (int k = 0; k < 10; ++k) wr[k] = w[c * 10 + k];
  __syncthreads();
  for (int t = 0; t < kConv0T && t0 + t < len; ++t) {
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 10; ++k) acc = fmaf(wr[k], xs[t * 5 + k], acc);
    raw[((size_t)b * stride + t0 + t) * kSslConvDim + c] = acc;
  }
}

// GroupNorm(512, 512): per (window, channel) mean and biased variance over the len frames (two passes, fp64 sums)
__global__ void __launch_bounds__(512) ssl_gn_stats_kernel(const float* __restrict__ raw, float2* __restrict__ stats,
                                                           int len, int stride) {
  __shared__ double red[16][33];
  const int b = blockIdx.y, c = blockIdx.x * 32 + threadIdx.x, ty = threadIdx.y;
  const float* col = raw + (size_t)b * stride * kSslConvDim + c;
  double s = 0.0;
  for (int t = ty; t < len; t += 16) s += col[(size_t)t * kSslConvDim];
  red[ty][threadIdx.x] = s;
  __syncthreads();
  if (ty == 0) {
    for (int i = 1; i < 16; ++i) s += red[i][threadIdx.x];
    red[0][threadIdx.x] = s / len;
  }
  __syncthreads();
  const double mean = red[0][threadIdx.x];
  __syncthreads();
  double q = 0.0;
  for (int t = ty; t < len; t += 16) {
    const double d = col[(size_t)t * kSslConvDim] - mean;
    q += d * d;
  }
  red[ty][threadIdx.x] = q;
  __syncthreads();
  if (ty == 0) {
    for (int i = 1; i < 16; ++i) q += red[i][threadIdx.x];
    stats[b * kSslConvDim + c] = make_float2((float)mean, (float)(1.0 / sqrt(q / len + 1e-5)));
  }
}

// normalise + affine + GELU -> fp16 (hi, lo); the padding rows [len, stride) of every window become zero
__global__ void ssl_gn_apply_kernel(const float* __restrict__ raw, const float2* __restrict__ stats,
                                    const float* __restrict__ gamma, const float* __restrict__ beta,
                                    __half* __restrict__ hi, __half* __restrict__ lo, int len, int stride, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % kSslConvDim);
  const size_t row = i / kSslConvDim;
  const int b = (int)(row / stride), t = (int)(row % stride);
  float y = 0.f;
  if (t < len) {
    const float2 st = stats[b * kSslConvDim + c];
    y = gelu_erf((raw[i] - st.x) * st.y * gamma[c] + beta[c]);
  }
  store_split(hi, lo, i, y);
}

// ---- LayerNorm over C channels, one warp per row ------------------------------------------------------------------
// row m = window * T + t reads a[window * a_stride + t] (+ res[m]) and writes y[m] (fp32), (yh, yl)[m] (fp16 pair)
// and avg[m] (+)= avg_w * y: every output optional.
template <int C>
__global__ void __launch_bounds__(256) ssl_ln_kernel(const float* __restrict__ a, const float* __restrict__ res,
                                                     int T, int a_stride, const float* __restrict__ gamma,
                                                     const float* __restrict__ beta, float* __restrict__ y,
                                                     __half* __restrict__ yh, __half* __restrict__ yl,
                                                     float* __restrict__ avg, float avg_w, int avg_assign, int M) {
  constexpr int V = C / 32;
  const int m = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (m >= M) return;
  const float* src = a + ((size_t)(m / T) * a_stride + m % T) * C;
  float v[V];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    v[i] = src[i * 32 + lane];
    if (res) v[i] += res[(size_t)m * C + i * 32 + lane];
    s += v[i];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float d = v[i] - mean;
    q = fmaf(d, d, q);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / C + 1e-5f);
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const int c = i * 32 + lane;
    const size_t idx = (size_t)m * C + c;
    const float r = (v[i] - mean) * rstd * gamma[c] + beta[c];
    if (y) y[idx] = r;
    if (yh) store_split(yh, yl, idx, r);
    if (avg) avg[idx] = avg_assign ? avg_w * r : fmaf(avg_w, r, avg[idx]);
  }
}

// ---- positional conv ------------------------------------------------------------------------------------------------
// x [NB][T][768] -> A [NB][T + 128][16 groups x 64] fp16 (hi, lo): row 64 + t holds frame t, channels 48 g + j at
// column 64 g + j (j < 48); the 64 rows before and after every window and the columns 48..63 of every group are zero.
__global__ void ssl_pos_pack_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo,
                                    int T, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int col = (int)(i % 1024), g = col / 64, j = col % 64;
  const size_t row = i / 1024;
  const int b = (int)(row / (T + kSslPosK)), t = (int)(row % (T + kSslPosK)) - kSslPosK / 2;
  const float v = (j < 48 && t >= 0 && t < T) ? x[((size_t)b * T + t) * kSslDim + g * 48 + j] : 0.f;
  store_split(hi, lo, i, v);
}

// y = x + P (the positional conv after its bias and GELU, [NB][T + 128][16 x 128])
__global__ void ssl_pos_add_kernel(const float* __restrict__ x, const float* __restrict__ P, float* __restrict__ y,
                                   int T, size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % kSslDim);
  const size_t m = i / kSslDim;
  const int b = (int)(m / T), t = (int)(m % T);
  y[i] = x[i] + P[((size_t)b * (T + kSslPosK) + t) * 2048 + (c / 48) * 128 + c % 48];
}

// ---- WavLM gated relative position bias: gate[m][h] from the layer input x (wavlm_attention.py forward) ------------
__global__ void __launch_bounds__(256) ssl_gate_kernel(const float* __restrict__ x, const float* __restrict__ gw,
                                                       const float* __restrict__ gb, const float* __restrict__ gconst,
                                                       float* __restrict__ gate, int M) {
  __shared__ float sw[8 * 64];
  for (int i = threadIdx.x; i < 8 * 64; i += blockDim.x) sw[i] = gw[i];
  __syncthreads();
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= M * kSslHeads) return;
  const int m = idx / kSslHeads, h = idx % kSslHeads;
  const float* xr = x + (size_t)m * kSslDim + h * 64;
  float v[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] = 0.f;
  for (int d = 0; d < 64; ++d) {
    const float xv = xr[d];
#pragma unroll
    for (int k = 0; k < 8; ++k) v[k] = fmaf(sw[k * 64 + d], xv, v[k]);
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) v[k] += gb[k];
  const float ga = 1.f / (1.f + expf(-(((v[0] + v[1]) + v[2]) + v[3])));
  const float gbv = 1.f / (1.f + expf(-(((v[4] + v[5]) + v[6]) + v[7])));
  gate[idx] = ga * (gbv * gconst[h] - 1.f) + 2.f;
}

// ---- attention: softmax(q k^T / 8 + gate_i * rel(j - i)) v per (window, head), online softmax, fp32 ---------------
// CTA = 64 queries of one head of one window, 256 threads: 4 per query, each owning 16 keys of a 64-key tile for the
// scores and 16 of the 64 output dims.
constexpr int kAttTile = 64;
constexpr int kAttLd = 68;                         // padded row (16-byte aligned, conflict-free float4 rows)
constexpr size_t kAttSmem = (size_t)(3 * kAttTile * kAttLd + 128) * sizeof(float);

__global__ void __launch_bounds__(256) ssl_attention_kernel(const float* __restrict__ qkv, const float* __restrict__ gate,
                                                            const float* __restrict__ rel_tab, __half* __restrict__ oh,
                                                            __half* __restrict__ ol, int T) {
  extern __shared__ float4 att_smem4[];
  float* Ks = reinterpret_cast<float*>(att_smem4);
  float* Vs = Ks + kAttTile * kAttLd;
  float* Ps = Vs + kAttTile * kAttLd;
  float* bs = Ps + kAttTile * kAttLd;
  const int h = blockIdx.y, b = blockIdx.z, i0 = blockIdx.x * kAttTile;
  const int qi = threadIdx.x >> 2, part = threadIdx.x & 3;
  const int i = i0 + qi;
  const size_t base = (size_t)b * T;
  float q[64];
  {
    const float* qr = qkv + (base + (i < T ? i : T - 1)) * (3 * kSslDim) + h * 64;
#pragma unroll
    for (int d = 0; d < 64; d += 4) {
      const float4 v = *reinterpret_cast<const float4*>(qr + d);
      q[d] = v.x * 0.125f; q[d + 1] = v.y * 0.125f; q[d + 2] = v.z * 0.125f; q[d + 3] = v.w * 0.125f;
    }
  }
  const float g = gate[(base + (i < T ? i : T - 1)) * kSslHeads + h];
  const float* tab = rel_tab + (size_t)h * (2 * kSslRelSpan + 1) + kSslRelSpan;
  float mrun = -INFINITY, lrun = 0.f, o[16];
#pragma unroll
  for (int d = 0; d < 16; ++d) o[d] = 0.f;

  for (int j0 = 0; j0 < T; j0 += kAttTile) {
    __syncthreads();
    for (int e = threadIdx.x; e < kAttTile * 16; e += blockDim.x) {   // K and V rows, float4 at a time
      const int r = e >> 4, c4 = (e & 15) * 4, j = j0 + r;
      float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
      if (j < T) {
        const float* row = qkv + (base + j) * (3 * kSslDim) + h * 64 + c4;
        kv = *reinterpret_cast<const float4*>(row + kSslDim);
        vv = *reinterpret_cast<const float4*>(row + 2 * kSslDim);
      }
      *reinterpret_cast<float4*>(Ks + r * kAttLd + c4) = kv;
      *reinterpret_cast<float4*>(Vs + r * kAttLd + c4) = vv;
    }
    if (threadIdx.x < 127) {                     // offsets j - i = (j0 - i0) + e - 63 of this tile pair
      int d = j0 - i0 + (int)threadIdx.x - 63;
      d = d < -kSslRelSpan ? -kSslRelSpan : (d > kSslRelSpan ? kSslRelSpan : d);
      bs[threadIdx.x] = tab[d];
    }
    __syncthreads();
    float s[16];
    float tmax = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const int jl = part + 4 * jj;
      const float* kr = Ks + jl * kAttLd;
      float acc = 0.f;
#pragma unroll
      for (int d = 0; d < 64; d += 4) {
        const float4 kv = *reinterpret_cast<const float4*>(kr + d);
        acc = fmaf(q[d], kv.x, acc);
        acc = fmaf(q[d + 1], kv.y, acc);
        acc = fmaf(q[d + 2], kv.z, acc);
        acc = fmaf(q[d + 3], kv.w, acc);
      }
      s[jj] = (j0 + jl < T) ? acc + g * bs[jl - qi + 63] : -INFINITY;
      tmax = fmaxf(tmax, s[jj]);
    }
    tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 1));
    tmax = fmaxf(tmax, __shfl_xor_sync(0xffffffffu, tmax, 2));
    const float mnew = fmaxf(mrun, tmax);
    const float corr = expf(mrun - mnew);
    float psum = 0.f;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const float p = expf(s[jj] - mnew);
      psum += p;
      Ps[qi * kAttLd + part + 4 * jj] = p;
    }
    lrun = lrun * corr + psum;
    mrun = mnew;
#pragma unroll
    for (int d = 0; d < 16; ++d) o[d] *= corr;
    __syncwarp();                                // the 4 threads of a query (one warp) exchange their p
    const float* pr = Ps + qi * kAttLd;
#pragma unroll 4
    for (int j = 0; j < kAttTile; ++j) {
      const float p = pr[j];
      const float* vr = Vs + j * kAttLd + part * 16;
#pragma unroll
      for (int d = 0; d < 16; d += 4) {
        const float4 v = *reinterpret_cast<const float4*>(vr + d);
        o[d] = fmaf(p, v.x, o[d]);
        o[d + 1] = fmaf(p, v.y, o[d + 1]);
        o[d + 2] = fmaf(p, v.z, o[d + 2]);
        o[d + 3] = fmaf(p, v.w, o[d + 3]);
      }
    }
  }
  lrun += __shfl_xor_sync(0xffffffffu, lrun, 1);
  lrun += __shfl_xor_sync(0xffffffffu, lrun, 2);
  if (i >= T) return;
  const float inv = 1.f / lrun;
  const size_t ob = (base + i) * kSslDim + h * 64 + part * 16;
#pragma unroll
  for (int d = 0; d < 16; ++d) store_split(oh, ol, ob + d, o[d] * inv);
}

// ---- host -----------------------------------------------------------------------------------------------------------
struct SslWs {
  float* raw;                 // conv 0 output fp32 [NB][stride0][512]; then the odd convs' fp16 pairs
  __half *ah, *al;            // even convs' fp16 pairs [NB][stride][512]
  __half *bh, *bl;            // = raw reinterpreted
  float *x, *x1, *qkv, *gate, *o, *P;
  __half *xh, *xl, *x1h, *x1l, *atth, *attl, *hh, *hl, *ph, *pl;
};
static size_t carve_ssl(const SslGeom& g, int NB, void* base, SslWs* w) {
  Workspace ws(base, 1024);
  SslWs t;
  const size_t R = (size_t)NB * g.stride[0] * kSslConvDim, M = (size_t)NB * g.T, Mp = (size_t)NB * (g.T + kSslPosK);
  t.raw = (float*)ws.take(R * sizeof(float));
  t.bh = (__half*)t.raw;
  t.bl = t.bh + R / 2;
  t.ah = (__half*)ws.take(R * sizeof(__half));
  t.al = (__half*)ws.take(R * sizeof(__half));
  t.x = (float*)ws.take(M * kSslDim * sizeof(float));
  t.x1 = (float*)ws.take(M * kSslDim * sizeof(float));
  t.o = (float*)ws.take(M * kSslDim * sizeof(float));
  t.qkv = (float*)ws.take(M * 3 * kSslDim * sizeof(float));
  t.gate = (float*)ws.take(M * kSslHeads * sizeof(float));
  t.P = (float*)ws.take(Mp * 2048 * sizeof(float));
  t.xh = (__half*)ws.take(M * kSslDim * sizeof(__half));
  t.xl = (__half*)ws.take(M * kSslDim * sizeof(__half));
  t.x1h = (__half*)ws.take(M * kSslDim * sizeof(__half));
  t.x1l = (__half*)ws.take(M * kSslDim * sizeof(__half));
  t.atth = (__half*)ws.take(M * kSslDim * sizeof(__half));
  t.attl = (__half*)ws.take(M * kSslDim * sizeof(__half));
  t.hh = (__half*)ws.take(M * kSslFfn * sizeof(__half));
  t.hl = (__half*)ws.take(M * kSslFfn * sizeof(__half));
  t.ph = (__half*)ws.take(Mp * 1024 * sizeof(__half));
  t.pl = (__half*)ws.take(Mp * 1024 * sizeof(__half));
  if (w) *w = t;
  return ws.bytes();
}
size_t ssl_workspace_bytes(const SslGeom& g, int NB) { return carve_ssl(g, NB, nullptr, nullptr); }

static unsigned blocks_for(size_t n, int threads) { return (unsigned)((n + threads - 1) / threads); }

int ssl_frontend_forward(const SslWeights& W, const SslGeom& g, const float* wav, const long long* chunk_off,
                         const int* chunk_valid, int NB, void* ws, float* x0, int num_sms, cudaStream_t st) {
  SslWs w;
  carve_ssl(g, NB, ws, &w);
  int rc;
  // feature extractor
  if ((rc = launch(ssl_conv0_kernel, dim3(ceil_div(g.len[0], kConv0T), NB), kSslConvDim, 0, st, wav, chunk_off,
                   chunk_valid, W.conv0_w, w.raw, g.len[0], g.stride[0])))
    return rc;
  float2* stats = reinterpret_cast<float2*>(w.P);          // [NB][512], P is free until the positional conv
  if ((rc = launch(ssl_gn_stats_kernel, dim3(kSslConvDim / 32, NB), dim3(32, 16), 0, st, w.raw, stats, g.len[0],
                   g.stride[0])))
    return rc;
  const size_t R = (size_t)NB * g.stride[0] * kSslConvDim;
  if ((rc = launch(ssl_gn_apply_kernel, blocks_for(R, 256), 256, 0, st, w.raw, stats, W.gn_w, W.gn_b, w.ah, w.al,
                   g.len[0], g.stride[0], R)))
    return rc;
  float* feat = reinterpret_cast<float*>(w.ah);             // conv 6 output fp32 (written into the free even buffer)
  for (int l = 1; l <= 6; ++l) {
    const bool from_a = (l & 1) == 1;
    const __half *inh = from_a ? w.ah : w.bh, *inl = from_a ? w.al : w.bl;
    __half *outh = from_a ? w.bh : w.ah, *outl = from_a ? w.bl : w.al;
    const int M = NB * g.stride[l];                          // pair rows of the input = output rows
    const int K = l <= 4 ? 2048 : 1024;
    GemmTaps taps;
    taps.taps = l <= 4 ? 2 : 1;
    taps.dil = l <= 4 ? 1 : 0;
    if (l < 6)
      rc = gemm_tc_split(inh, inl, 1024, W.conv_hi[l - 1], W.conv_lo[l - 1], K, nullptr, 0, outh, outl, kSslConvDim,
                         nullptr, M, kSslConvDim, K, 2, num_sms, st, nullptr, 0, taps);
    else
      rc = gemm_tc_split(inh, inl, 1024, W.conv_hi[l - 1], W.conv_lo[l - 1], K, feat, kSslConvDim, nullptr, nullptr, 0,
                         nullptr, M, kSslConvDim, K, 2, num_sms, st, nullptr, 0, taps);
    if (rc) return rc;
  }
  // feature projection: LayerNorm(512) of the valid frames (compacted to [NB][T]) -> Linear 512 -> 768
  const int T = g.T, M = NB * T;
  __half *fh = w.xh, *fl = w.x1h;                           // [M][512] pairs in buffers free until layer 0
  if ((rc = launch(ssl_ln_kernel<kSslConvDim>, ceil_div(M, 8), 256, 0, st, feat, nullptr, T, g.stride[6], W.fp_ln_w,
                   W.fp_ln_b, nullptr, fh, fl, nullptr, 0.f, 0, M)))
    return rc;
  if ((rc = gemm_tc_split(fh, fl, kSslConvDim, W.proj_hi, W.proj_lo, kSslConvDim, w.x, kSslDim, nullptr, nullptr, 0,
                          W.proj_b, M, kSslDim, kSslConvDim, 0, num_sms, st)))
    return rc;
  // positional conv: 16 group GEMMs of 128 taps over the zero-padded, group-major copy of x
  const size_t Mp = (size_t)NB * (T + kSslPosK);
  if ((rc = launch(ssl_pos_pack_kernel, blocks_for(Mp * 1024, 256), 256, 0, st, w.x, w.ph, w.pl, T, Mp * 1024)))
    return rc;
  GemmTaps ptaps;
  ptaps.taps = kSslPosK;
  ptaps.dil = 1;
  for (int gi = 0; gi < kSslPosGroups; ++gi) {
    const size_t wo = (size_t)gi * 128 * (kSslPosK * 64);
    if ((rc = gemm_tc_split(w.ph + gi * 64, w.pl + gi * 64, 1024, W.pos_hi + wo, W.pos_lo + wo, kSslPosK * 64,
                            w.P + gi * 128, 2048, nullptr, nullptr, 0, W.pos_b + gi * 128, (int)Mp, 128, kSslPosK * 64,
                            2, num_sms, st, nullptr, 0, ptaps)))
      return rc;
  }
  const size_t MD = (size_t)M * kSslDim;
  if ((rc = launch(ssl_pos_add_kernel, blocks_for(MD, 256), 256, 0, st, w.x, w.P, w.x1, T, MD))) return rc;
  // encoder.transformer.layer_norm: the post-LN encoder's Transformer normalises before its first layer
  if ((rc = launch(ssl_ln_kernel<kSslDim>, ceil_div(M, 8), 256, 0, st, w.x1, nullptr, T, T, W.enc_ln_w, W.enc_ln_b, w.x,
                   w.xh, w.xl, nullptr, 0.f, 0, M)))
    return rc;
  // transformer layers
  bool averaged = false;                                    // x0 holds a first weighted layer output
  for (int l = 0; l < W.num_layers; ++l) {
    const SslLayerWeights& L = W.layer[l];
    if ((rc = launch(ssl_gate_kernel, ceil_div(M * kSslHeads, 256), 256, 0, st, w.x, L.gru_w, L.gru_b, L.gru_const,
                     w.gate, M)))
      return rc;
    if ((rc = gemm_tc_split(w.xh, w.xl, kSslDim, L.qkv_hi, L.qkv_lo, kSslDim, w.qkv, 3 * kSslDim, nullptr, nullptr, 0,
                            L.qkv_b, M, 3 * kSslDim, kSslDim, 0, num_sms, st)))
      return rc;
    if ((rc = launch(ssl_attention_kernel, dim3(ceil_div(T, kAttTile), kSslHeads, NB), 256, kAttSmem, st, w.qkv, w.gate,
                     W.rel_tab, w.atth, w.attl, T)))
      return rc;
    if ((rc = gemm_tc_split(w.atth, w.attl, kSslDim, L.out_hi, L.out_lo, kSslDim, w.o, kSslDim, nullptr, nullptr, 0,
                            L.out_b, M, kSslDim, kSslDim, 0, num_sms, st)))
      return rc;
    if ((rc = launch(ssl_ln_kernel<kSslDim>, ceil_div(M, 8), 256, 0, st, w.o, w.x, T, T, L.ln1_w, L.ln1_b, w.x1, w.x1h,
                     w.x1l, nullptr, 0.f, 0, M)))
      return rc;
    if ((rc = gemm_tc_split(w.x1h, w.x1l, kSslDim, L.ff1_hi, L.ff1_lo, kSslDim, nullptr, 0, w.hh, w.hl, kSslFfn, L.ff1_b,
                            M, kSslFfn, kSslDim, 2, num_sms, st)))
      return rc;
    if ((rc = gemm_tc_split(w.hh, w.hl, kSslFfn, L.ff2_hi, L.ff2_lo, kSslFfn, w.o, kSslDim, nullptr, nullptr, 0, L.ff2_b,
                            M, kSslDim, kSslFfn, 0, num_sms, st)))
      return rc;
    // the layer's output is the next layer's input x; the weighted layer average accumulates into x0
    const float aw = W.layer_w[l];
    if ((rc = launch(ssl_ln_kernel<kSslDim>, ceil_div(M, 8), 256, 0, st, w.o, w.x1, T, T, L.ln2_w, L.ln2_b, w.x, w.xh,
                     w.xl, aw != 0.f ? x0 : nullptr, aw, !averaged, M)))
      return rc;
    averaged = averaged || aw != 0.f;
  }
  return B200_OK;
}

}  // namespace b200
