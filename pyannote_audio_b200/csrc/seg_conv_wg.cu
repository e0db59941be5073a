// SincNet convolutions on the Hopper tensor cores (wgmma), split-precision fp16 with fp32-level accuracy.
//
// Reference: pyannote/audio/models/blocks/sincnet.py:70-90,163-184.  The three layers are one implicit GEMM each,
//     D[t][n] = sum_k X[t * S + k] * W[n][k]          t = conv output position, n = output channel
//   sinc layer:   S = 10 (stride), X = normalised samples,                      K = 256 (251 taps + zeros), N = 80
//   Conv1d(C,60,5): S = Cpad, X = channels-last [position][Cpad] input after InstanceNorm + leaky_relu,
//                 k = tap * Cpad + channel, K = 5 * Cpad,                                      N = 64 (60 real)
// followed by |.| (sinc layer only), MaxPool1d(3, 3), + bias (Conv1d) and fp64 InstanceNorm partial sums per tile.
// A CTA is one warpgroup on one tile of the fp32 twins (sinc_pool_kernel / conv5_pool_kernel): 192 positions = 64
// pooled outputs, three m64 blocks.  The tile's input is staged once as fp16 (hi, lo) pairs; the A fragments of
// every K = 16 step are read from it straight into registers (the im2col rows start 20 bytes apart, which no TMA
// box or shared-memory descriptor expresses).  The weights (hi, lo) arrive by TMA as 128-byte-swizzled K-major tiles.
// Products: A_lo*W_hi + A_hi*W_lo + A_hi*W_hi in fp32 registers, like gemm_tc.cu.
#include "common.cuh"
#include "seg.cuh"
#include "tc_common.cuh"

namespace b200 {

constexpr int kSCThreads = 128;
constexpr int kSCTileP = 64;                 // pooled outputs per tile (= the fp32 twins' tile)
constexpr int kSCPos = 3 * kSCTileP;         // conv output positions per tile
constexpr int kSCPitch = kSCPos + 1;         // epilogue staging [channel][position] pitch (floats)

struct SincConvWgParams {
  // sinc layer input
  const float* wav;
  const long long* chunk_off;
  const int* chunk_valid;
  int W;                       // window samples: staged positions at or past W are zero
  const float2* affine;        // sinc: per-chunk waveform InstanceNorm; Conv1d: per (chunk, input channel)
  // Conv1d input
  const float* Pin;            // [B][CIN][Lin]
  int Lin;
  const float* bias;           // Conv1d: [60]
  float* Pout;                 // [B][NREAL][Lp]
  double2* part;               // [B][NREAL][ntiles]
  int Lp, ntiles;
  int NB;                      // windows (persistent kernels)
  uint32_t xs_bytes, w_off, w_box_bytes, pool_off;
};

// CIN = 0: the sinc layer; else a Conv1d(CIN, 60, 5) with input channels padded to CPAD
template <int CIN, int CPAD, int NW, int NREAL, int KT>
__global__ void __launch_bounds__(kSCThreads)
sinc_conv_wg_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl,
                    SincConvWgParams p) {
  constexpr bool kSinc = CIN == 0;
  constexpr int S = kSinc ? kSincStride : CPAD;
  constexpr int kIn = kSinc ? (kSCPos - 1) * S + KT : (kSCPos + 4) * CPAD;   // staged fp16 values per (hi | lo)
  constexpr int kBoxes = (KT + 63) / 64;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  const uint32_t bar = base;
  __half* xh = reinterpret_cast<__half*>(gbase + 1024);
  __half* xl = xh + kIn;
  const uint32_t w_smem = base + p.w_off;
  const int tile = blockIdx.x, b = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(bar, 2u * kBoxes * p.w_box_bytes);
    for (int i = 0; i < kBoxes; ++i) {
      tma_load_2d(&tmWh, bar, w_smem + i * p.w_box_bytes, 64 * i, 0);
      tma_load_2d(&tmWl, bar, w_smem + (kBoxes + i) * p.w_box_bytes, 64 * i, 0);
    }
  }
  // ---- stage the tile's input as fp16 (hi, lo), same padding rules as the fp32 twins ------------------------------
  if (kSinc) {
    const float2 af = p.affine[b];
    const float* x = p.wav + p.chunk_off[b];
    const int valid = p.chunk_valid[b];
    const int s0 = tile * kSCPos * kSincStride;
    for (int i = tid; i < kIn; i += kSCThreads) {
      const int g = s0 + i;
      const float rv = (g < valid) ? __ldg(x + g) : 0.f;
      const float v = (g < p.W) ? fmaf(rv, af.x, af.y) : 0.f;
      const __half h = __float2half_rn(v);
      xh[i] = h;
      xl[i] = __float2half_rn(v - __half2float(h));
    }
  } else {
    constexpr int TW = kSCPos + 4;
    const int t0 = tile * kSCPos;
    for (int i = tid; i < CPAD * TW; i += kSCThreads) {
      const int c = i / TW, t = i - c * TW, g = t0 + t;
      float v = 0.f;
      if (c < CIN && g < p.Lin) {
        const float2 af = p.affine[b * CIN + c];
        v = fmaf(p.Pin[((size_t)b * CIN + c) * p.Lin + g], af.x, af.y);
        v = v > 0.f ? v : 0.01f * v;
      }
      const __half h = __float2half_rn(v);
      xh[t * CPAD + c] = h;
      xl[t * CPAD + c] = __float2half_rn(v - __half2float(h));
    }
  }
  __syncthreads();
  mbar_wait(bar, 0);

  // ---- three m64 blocks x KT / 16 steps x 3 split products --------------------------------------------------------
  float acc[3][NW / 2];
#pragma unroll
  for (int m = 0; m < 3; ++m)
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[m][i] = 0.f;
  const uint32_t* xh32 = reinterpret_cast<const uint32_t*>(xh);
  const uint32_t* xl32 = reinterpret_cast<const uint32_t*>(xl);
  const int r0 = 16 * warp + (lane >> 2), c0 = 2 * (lane & 3);
  for (int ks = 0; ks < KT / 16; ++ks) {
    uint32_t ah[3][4], al[3][4];
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      const int t = 64 * m + r0;
      const int i0 = (t * S + 16 * ks + c0) >> 1, i1 = ((t + 8) * S + 16 * ks + c0) >> 1;   // even offsets
      ah[m][0] = xh32[i0]; ah[m][1] = xh32[i1]; ah[m][2] = xh32[i0 + 4]; ah[m][3] = xh32[i1 + 4];
      al[m][0] = xl32[i0]; al[m][1] = xl32[i1]; al[m][2] = xl32[i0 + 4]; al[m][3] = xl32[i1 + 4];
    }
    const uint32_t wb = w_smem + (ks >> 2) * p.w_box_bytes + (ks & 3) * 32;
    const uint64_t wh = wg_desc(wb, 128), wl = wg_desc(wb + kBoxes * p.w_box_bytes, 128);
    wg_fence();
#pragma unroll
    for (int m = 0; m < 3; ++m) {
      WgmmaRS<NW>::mma(acc[m], al[m], wh);                 // small cross terms first, hi*hi last
      WgmmaRS<NW>::mma(acc[m], ah[m], wl);
      WgmmaRS<NW>::mma(acc[m], ah[m], wh);
    }
    wg_commit();
    wg_wait<0>();
  }

  // ---- epilogue: stage [channel][position] over the weights, pool, store, partial sums ---------------------------
  __syncthreads();
  float* st = reinterpret_cast<float*>(gbase + p.w_off);
#pragma unroll
  for (int m = 0; m < 3; ++m)
#pragma unroll
    for (int j = 0; j < NW / 8; ++j)
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float v = acc[m][4 * j + 2 * i + e];
          st[(8 * j + c0 + e) * kSCPitch + 64 * m + r0 + 8 * i] = kSinc ? fabsf(v) : v;
        }
  __syncthreads();
  float* pt = reinterpret_cast<float*>(gbase + p.pool_off);   // pooled tile [NREAL][65]
  for (int idx = tid; idx < NREAL * kSCTileP; idx += kSCThreads) {
    const int n = idx / kSCTileP, j = idx - n * kSCTileP;
    const float* r = st + n * kSCPitch + 3 * j;
    float v = fmaxf(fmaxf(r[0], r[1]), r[2]);
    if (!kSinc) v += p.bias[n];
    const int pg = tile * kSCTileP + j;
    const bool ok = pg < p.Lp;
    pt[n * 65 + j] = ok ? v : 0.f;
    if (ok) p.Pout[((size_t)b * NREAL + n) * p.Lp + pg] = v;
  }
  __syncthreads();
  if (tid < NREAL) {
    double s = 0.0, ss = 0.0;
    for (int i = 0; i < kSCTileP; ++i) {
      const double v = pt[tid * 65 + i];
      s += v;
      ss += v * v;
    }
    p.part[((size_t)b * NREAL + tid) * p.ntiles + tile] = make_double2(s, ss);
  }
}

template <int CIN, int CPAD, int NW, int NREAL, int KT>
static int launch_sc(const __half* Wh, const __half* Wl, SincConvWgParams p, int NB, cudaStream_t stream) {
  constexpr int kIn = CIN == 0 ? (kSCPos - 1) * kSincStride + KT : (kSCPos + 4) * CPAD;
  constexpr int kBoxes = (KT + 63) / 64;
  p.xs_bytes = (uint32_t)align_up((size_t)kIn * 2 * sizeof(__half), 1024);
  p.w_off = 1024 + p.xs_bytes;
  p.w_box_bytes = NW * 128;
  uint32_t w_bytes = 2u * kBoxes * p.w_box_bytes;
  const uint32_t st_bytes = (uint32_t)(NW * kSCPitch * sizeof(float));
  if (w_bytes < st_bytes) w_bytes = st_bytes;
  p.pool_off = p.w_off + (uint32_t)align_up(w_bytes, 1024);
  const size_t smem = 1024 + p.pool_off + (size_t)NREAL * 65 * sizeof(float);
  B200_CHECK(smem <= 227 * 1024, B200_ERR_STATE, "sinc/conv wgmma kernel: %zu B of shared memory", smem);
  CUtensorMap th, tl;
  const cuuint64_t dims[2] = {(cuuint64_t)KT, (cuuint64_t)NW}, strides[1] = {(cuuint64_t)KT * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)NW};
  int rc;
  if ((rc = encode_f16_map(&th, 2, Wh, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B, "sinc/conv weights")))
    return rc;
  if ((rc = encode_f16_map(&tl, 2, Wl, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B, "sinc/conv weights")))
    return rc;
  auto kernel = sinc_conv_wg_kernel<CIN, CPAD, NW, NREAL, KT>;
  return launch(kernel, dim3(p.ntiles, NB), kSCThreads, smem, stream, th, tl, p);   // one tile per 64 pooled outputs
}

// ---- persistent, weight-resident kernels (seg_conv_impl = 1) -----------------------------------------------------
// A unit is one tile of sinc_conv_wg_kernel: (window b, 64 pooled outputs), numbered u = b * ntiles + tile.  Each CTA
// loads the (hi, lo) weights once by TMA and keeps them; each of its kWG consumer warpgroups stages, multiplies and
// stores its own units, so one warpgroup's staging and epilogue overlap the other's MMAs.  Accumulator row r of m-block
// m is conv position 3r + m (pool mates): a thread holds the three positions of its pooled outputs in acc[0..2], and
// |.|, the max-pool and the bias happen in registers.  Each output still sums its products in ascending K steps, each
// step lo*hi, hi*lo, hi*hi, so the outputs and the partial sums are bit-identical to sinc_conv_wg_kernel's.
//
// Shared memory: [header: mbarrier | 1 KB] [weights: kBoxes (hi) + kBoxes (lo) 128-byte-swizzled boxes of NW rows]
// then per warpgroup [staged input: fp16 hi then lo, kIn values each] [pooled tile: NREAL x 65 fp32].
template <int CIN, int CPAD, int NW, int NREAL, int KT>
struct PersistPlan {
  static constexpr bool kSinc = CIN == 0;
  // conv1's staged input (196 positions x 88 channels x (hi, lo)) fits once next to its 112 KB of weights, not twice
  static constexpr int kWG = CIN == 80 ? 1 : 2;
  // fp16 between consecutive staged positions: the sinc layer's stride, or the channels padded by 8 so that the eight
  // pool-mate rows a fragment load touches (3 positions apart) fall in distinct banks
  static constexpr int kRow = kSinc ? kSincStride : CPAD + 8;
  static constexpr int kIn = kSinc ? (kSCPos - 1) * kSincStride + KT : (kSCPos + 4) * kRow;
  static constexpr int kBoxes = (KT + 63) / 64;
  static constexpr uint32_t kBoxBytes = NW * 128;
  static constexpr uint32_t kWOff = 1024;
  static constexpr uint32_t kXsBytes = (uint32_t)((2 * kIn * sizeof(__half) + 15) / 16 * 16);
  static constexpr uint32_t kPtBytes = NREAL * 65 * sizeof(float);
  static constexpr uint32_t kWgOff = kWOff + 2 * kBoxes * kBoxBytes;
  static constexpr uint32_t kWgBytes = kXsBytes + kPtBytes;
  static constexpr size_t kSmem = 1024 + kWgOff + kWG * kWgBytes;   // + 1024 to align the base
  static_assert(KT % 16 == 0 && (kSinc || CPAD % 16 == 0), "a K step must not straddle two taps");
  static_assert(kRow % 2 == 0 && (3 * kRow) % 2 == 0, "fragment loads are 4-byte aligned");
  static_assert(kBoxBytes % 1024 == 0, "128-byte-swizzled boxes start 1024-byte aligned");
  static_assert(NREAL <= 128 && NREAL <= NW, "one partial-sum thread per channel");
  static_assert(kSmem <= 227 * 1024, "shared memory per CTA");
};

template <int CIN, int CPAD, int NW, int NREAL, int KT>
__global__ void __launch_bounds__(PersistPlan<CIN, CPAD, NW, NREAL, KT>::kWG * 128, 1)
sinc_conv_persist_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl,
                         SincConvWgParams p) {
  using P = PersistPlan<CIN, CPAD, NW, NREAL, KT>;
  constexpr bool kSinc = P::kSinc;
  constexpr int kSteps = KT / 16;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  uint8_t* gbase = smem_raw + (base - raw);
  const uint32_t bar = base;
  const uint32_t w_smem = base + P::kWOff;
  const int tid = threadIdx.x, wg = tid >> 7, wtid = tid & 127, warp = wtid >> 5, lane = tid & 31;
  __half* xh = reinterpret_cast<__half*>(gbase + P::kWgOff + wg * P::kWgBytes);
  __half* xl = xh + P::kIn;
  float* pt = reinterpret_cast<float*>(gbase + P::kWgOff + wg * P::kWgBytes + P::kXsBytes);

  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(bar, 2u * P::kBoxes * P::kBoxBytes);
    for (int i = 0; i < P::kBoxes; ++i) {
      tma_load_2d(&tmWh, bar, w_smem + i * P::kBoxBytes, 64 * i, 0);
      tma_load_2d(&tmWl, bar, w_smem + (P::kBoxes + i) * P::kBoxBytes, 64 * i, 0);
    }
  }
  bool weights_ready = false;

  const int units = p.NB * p.ntiles, stride = gridDim.x * P::kWG;
  const int r0 = 16 * warp + (lane >> 2), c0 = 2 * (lane & 3);
  for (int u = blockIdx.x * P::kWG + wg; u < units; u += stride) {
    const int b = u / p.ntiles, tile = u - b * p.ntiles;
    // ---- stage the unit's input as fp16 (hi, lo), same values and padding rules as sinc_conv_wg_kernel -----------
    if (kSinc) {
      const float2 af = p.affine[b];
      const float* x = p.wav + p.chunk_off[b];
      const int valid = p.chunk_valid[b];
      const int s0 = tile * kSCPos * kSincStride;
      for (int i = wtid; i < P::kIn; i += 128) {
        const int g = s0 + i;
        const float rv = (g < valid) ? __ldg(x + g) : 0.f;
        const float v = (g < p.W) ? fmaf(rv, af.x, af.y) : 0.f;
        const __half h = __float2half_rn(v);
        xh[i] = h;
        xl[i] = __float2half_rn(v - __half2float(h));
      }
    } else {
      constexpr int TW = kSCPos + 4;
      const int t0 = tile * kSCPos;
      for (int i = wtid; i < CPAD * TW; i += 128) {
        const int c = i / TW, t = i - c * TW, g = t0 + t;
        float v = 0.f;
        if (c < CIN && g < p.Lin) {
          const float2 af = p.affine[b * CIN + c];
          v = fmaf(p.Pin[((size_t)b * CIN + c) * p.Lin + g], af.x, af.y);
          v = v > 0.f ? v : 0.01f * v;
        }
        const __half h = __float2half_rn(v);
        xh[t * P::kRow + c] = h;
        xl[t * P::kRow + c] = __float2half_rn(v - __half2float(h));
      }
    }
    // the next unit's input into L2 while this one multiplies
    if (u + stride < units) {
      const int nb = (u + stride) / p.ntiles, nt = (u + stride) - nb * p.ntiles;
      if (kSinc) {
        const int s0 = nt * kSCPos * kSincStride, n = min(P::kIn, p.chunk_valid[nb] - s0);
        if (32 * wtid < n) asm volatile("prefetch.global.L2 [%0];" ::"l"(p.wav + p.chunk_off[nb] + s0 + 32 * wtid));
      } else {
        constexpr int TW = kSCPos + 4;
        const int t0 = nt * kSCPos, n = min(TW, p.Lin - t0);
        for (int i = wtid; i < CIN * 7; i += 128) {   // 7 x 32 floats cover a channel's 196 positions
          const int c = i / 7, o = 32 * (i - 7 * c);
          if (o < n)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(p.Pin + ((size_t)nb * CIN + c) * p.Lin + t0 + o));
        }
      }
    }
    named_bar_sync(1 + wg);
    if (!weights_ready) {
      mbar_wait(bar, 0);
      weights_ready = true;
    }

    // ---- three m64 blocks x KT / 16 steps x 3 split products, the next step's fragments loaded under the MMAs ----
    float acc[3][NW / 2];
#pragma unroll
    for (int m = 0; m < 3; ++m)
#pragma unroll
      for (int i = 0; i < NW / 2; ++i) acc[m][i] = 0.f;
    const uint32_t* xh32 = reinterpret_cast<const uint32_t*>(xh);
    const uint32_t* xl32 = reinterpret_cast<const uint32_t*>(xl);
    uint32_t fh[2][3][4], fl[2][3][4];
    auto load = [&](int s, int ks) {
      // K step ks: k = 16 ks .. 16 ks + 15; a conv step lies inside one tap (CPAD % 16 == 0)
      const int koff = kSinc ? 16 * ks : (16 * ks / CPAD) * P::kRow + (16 * ks) % CPAD;
#pragma unroll
      for (int m = 0; m < 3; ++m) {
        const int i0 = ((3 * r0 + m) * P::kRow + koff + c0) >> 1;   // rows r0 and r0 + 8: positions 24 apart
        const int i1 = i0 + 12 * P::kRow;
        fh[s][m][0] = xh32[i0]; fh[s][m][1] = xh32[i1]; fh[s][m][2] = xh32[i0 + 4]; fh[s][m][3] = xh32[i1 + 4];
        fl[s][m][0] = xl32[i0]; fl[s][m][1] = xl32[i1]; fl[s][m][2] = xl32[i0 + 4]; fl[s][m][3] = xl32[i1 + 4];
      }
    };
    load(0, 0);
#pragma unroll
    for (int ks = 0; ks < kSteps; ++ks) {
      const int s = ks & 1;
      const uint32_t wb = w_smem + (ks >> 2) * P::kBoxBytes + (ks & 3) * 32;
      const uint64_t wh = wg_desc(wb, 128), wl = wg_desc(wb + P::kBoxes * P::kBoxBytes, 128);
      wg_fence();
#pragma unroll
      for (int m = 0; m < 3; ++m) {
        WgmmaRS<NW>::mma(acc[m], fl[s][m], wh);              // small cross terms first, hi*hi last
        WgmmaRS<NW>::mma(acc[m], fh[s][m], wl);
        WgmmaRS<NW>::mma(acc[m], fh[s][m], wh);
      }
      wg_commit();
      if (ks + 1 < kSteps) {
        wg_wait<1>();                                        // step ks - 1 has read the other fragment set
        load(s ^ 1, ks + 1);
      }
    }
    wg_wait<0>();

    // ---- epilogue: pool the three pool mates in registers, stage the pooled tile, store, partial sums --------------
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int j = r0 + 8 * i;
      const bool ok = tile * kSCTileP + j < p.Lp;
#pragma unroll
      for (int q = 0; q < NW / 8; ++q)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int n = 8 * q + c0 + e, a = 4 * q + 2 * i + e;
          if (n < NREAL) {
            float v = kSinc ? fmaxf(fmaxf(fabsf(acc[0][a]), fabsf(acc[1][a])), fabsf(acc[2][a]))
                            : fmaxf(fmaxf(acc[0][a], acc[1][a]), acc[2][a]);
            if (!kSinc) v += __ldg(p.bias + n);
            pt[n * 65 + j] = ok ? v : 0.f;
          }
        }
    }
    named_bar_sync(1 + wg);
    for (int idx = wtid; idx < NREAL * kSCTileP; idx += 128) {
      const int n = idx / kSCTileP, j = idx - n * kSCTileP;
      const int pg = tile * kSCTileP + j;
      if (pg < p.Lp) p.Pout[((size_t)b * NREAL + n) * p.Lp + pg] = pt[n * 65 + j];
    }
    if (wtid < NREAL) {
      double s = 0.0, ss = 0.0;
      for (int i = 0; i < kSCTileP; ++i) {
        const double v = pt[wtid * 65 + i];
        s += v;
        ss += v * v;
      }
      p.part[((size_t)b * NREAL + wtid) * p.ntiles + tile] = make_double2(s, ss);
    }
    // the next unit's pooled-tile writes come after its staging barrier, by which every thread has left this loop
  }
}

template <int CIN, int CPAD, int NW, int NREAL, int KT>
static int launch_persist(const __half* Wh, const __half* Wl, SincConvWgParams p, int NB, cudaStream_t stream) {
  using P = PersistPlan<CIN, CPAD, NW, NREAL, KT>;
  CUtensorMap th, tl;
  const cuuint64_t dims[2] = {(cuuint64_t)KT, (cuuint64_t)NW}, strides[1] = {(cuuint64_t)KT * 2};
  const cuuint32_t box[2] = {64, (cuuint32_t)NW};
  int rc;
  if ((rc = encode_f16_map(&th, 2, Wh, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B, "sinc/conv weights")))
    return rc;
  if ((rc = encode_f16_map(&tl, 2, Wl, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B, "sinc/conv weights")))
    return rc;
  int dev = 0, sms = 0;
  B200_CUDA_OK(cudaGetDevice(&dev));
  B200_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  p.NB = NB;
  const long long units = (long long)NB * p.ntiles;
  B200_CHECK(units < (1ll << 31), B200_ERR_INVALID, "sinc/conv: %lld tiles in one call", units);
  const int ctas = (int)std::min<long long>((units + P::kWG - 1) / P::kWG, sms);
  auto kernel = sinc_conv_persist_kernel<CIN, CPAD, NW, NREAL, KT>;
  return launch(kernel, ctas, P::kWG * 128, P::kSmem, stream, th, tl, p);
}

// impl 1: the persistent kernels; 2: one CTA per tile (sinc_conv_wg_kernel, the bit-exact reference)
int sinc_wg_forward(const SegGeom& g, const float* wav, const long long* chunk_off, const int* chunk_valid,
                    const float2* affine, const __half* Wh, const __half* Wl, int NB, float* P0, double2* part,
                    int impl, cudaStream_t stream) {
  SincConvWgParams p{};
  p.wav = wav; p.chunk_off = chunk_off; p.chunk_valid = chunk_valid; p.W = g.W; p.affine = affine;
  p.Pout = P0; p.part = part; p.Lp = g.pool0; p.ntiles = g.tiles0;
  if (impl == 1) return launch_persist<0, 1, 80, 80, 256>(Wh, Wl, p, NB, stream);
  return launch_sc<0, 1, 80, 80, 256>(Wh, Wl, p, NB, stream);
}

int conv5_wg_forward(const SegGeom& g, int layer, const float* Pin, const float2* affine, const __half* Wh,
                     const __half* Wl, const float* bias, int NB, float* Pout, double2* part, int impl,
                     cudaStream_t stream) {
  SincConvWgParams p{};
  p.affine = affine; p.bias = bias; p.Pout = Pout; p.part = part; p.Pin = Pin;
  if (layer == 0) {
    p.Lin = g.pool0; p.Lp = g.pool1; p.ntiles = g.tiles1;
    if (impl == 1) return launch_persist<80, 80, 64, 60, 400>(Wh, Wl, p, NB, stream);
    return launch_sc<80, 80, 64, 60, 400>(Wh, Wl, p, NB, stream);
  }
  p.Lin = g.pool1; p.Lp = g.pool2; p.ntiles = g.tiles2;
  if (impl == 1) return launch_persist<60, 64, 64, 60, 320>(Wh, Wl, p, NB, stream);
  return launch_sc<60, 64, 64, 60, 320>(Wh, Wl, p, NB, stream);
}

}  // namespace b200
