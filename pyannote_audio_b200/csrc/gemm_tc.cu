// Split-precision GEMM on the Hopper tensor cores (wgmma) with fp32-level accuracy.
//
//   C[M][N] = act(A[M][K] * B[N][K]^T + bias[N])          (both operands K-contiguous, like sgemm_nt)
//
// The reference computes PyanNet in true fp32 (TF32 disabled, utils/reproducibility.py:68-83) and a 7-way argmax
// decides integer frame boundaries downstream, so single-pass fp16/bf16/tf32 tensor-core math is not acceptable.
// Each fp32 operand is stored as a pair of fp16 values x = hi + lo (hi = fp16(x), lo = fp16(x - hi), 22 significant
// bits) and the product is accumulated in fp32 registers as   A_lo*B_hi + A_hi*B_lo + A_hi*B_hi   (the dropped lo*lo
// term is 2^-22 relative): three wgmma per K=16 step instead of an FFMA loop.
//
// Used for the LSTM input projections (N = 1024, K = 64 | 256; PyanNet.py:98,226-228), the two Linear+LeakyReLU
// layers (N = 128, K = 256 | 128; PyanNet.py:236-238), the embedding Linears (N = 256, K = 5120; N = 512, K = 3008)
// and, as implicit GEMMs, the dilated TDNN layers of XVectorSincNet (xvector.py:205-252, see GemmTaps in seg.cuh).
// One CTA per 128 x 128 output tile: warp 8 is the TMA producer, warpgroups 0 and 1 each own 64 rows of the tile and
// issue their wgmma on the shared A/B stages (ring of mbarrier-guarded stages, 128-byte swizzle).
#include "common.cuh"
#include "seg.cuh"
#include "tc_common.cuh"

namespace b200 {

constexpr int kGemmThreads = 288;
constexpr int kGemmM = 128;
constexpr int kGemmN = 128;
constexpr int kGemmK = 64;       // K per stage: one 128-byte swizzle row of fp16
constexpr int kGemmStages = 3;
constexpr uint32_t kGemmTile = kGemmM * kGemmK * 2;          // 16 KB: one operand half (hi or lo) of A or B
constexpr uint32_t kGemmStageBytes = 4 * kGemmTile;

struct GemmTcParams {
  int M, N, K, kblocks, tiles_n, act;
  const float* bias;
  float* C;            // fp32 output [M][ldc] or nullptr  (act: 0 none, 1 LeakyReLU(0.01), 2 GELU)
  __half* C_hi;        // optional split output [M][ldc_h]
  __half* C_lo;
  int ldc, ldc_h;
  // fused all-gather: the epilogue also stores every fp32 output tile to the same offsets of up to 7 PEER buffers
  // (other GPUs' memory mapped over NVLink: P2P stores), so the exchange of the result overlaps the GEMM tile by tile
  // and no separate collective runs
  float* C_peer[7];
  int n_peer;
  // implicit GEMM over taps: k-block kb belongs to tap kb / tap_kb and reads A rows shifted by tap * dil
  int tap_kb, dil;
  const float* scale;  // post-activation affine (or nullptr)
  const float* shift;
};

// GELU: the exact-GELU epilogue (act 2) is a separate instantiation, so that the other epilogues compile as before
template <bool GELU>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_tc_split_kernel(const __grid_constant__ CUtensorMap tmAh, const __grid_constant__ CUtensorMap tmAl,
                     const __grid_constant__ CUtensorMap tmBh, const __grid_constant__ CUtensorMap tmBl,
                     GemmTcParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t bar_full = base, bar_empty = base + 64;
  const uint32_t stage0 = base + 1024;
  const int warp = threadIdx.x >> 5;
  const int tn = blockIdx.x % p.tiles_n, tm = blockIdx.x / p.tiles_n;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kGemmStages; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if ((threadIdx.x & 31) == 0) {
      uint32_t stage = 0, phase = 0;
      for (int kb = 0; kb < p.kblocks; ++kb) {
        mbar_wait(bar_empty + 8 * stage, phase ^ 1);
        mbar_expect_tx(bar_full + 8 * stage, kGemmStageBytes);
        const uint32_t sa = stage0 + stage * kGemmStageBytes;
        // one tap: tap = 0 and the A box is (kb * 64, tm * 128) as for a plain GEMM
        const int tap = kb / p.tap_kb, ka = (kb - tap * p.tap_kb) * kGemmK, ra = tm * kGemmM + tap * p.dil;
        tma_load_2d(&tmAh, bar_full + 8 * stage, sa, ka, ra);
        tma_load_2d(&tmAl, bar_full + 8 * stage, sa + kGemmTile, ka, ra);
        tma_load_2d(&tmBh, bar_full + 8 * stage, sa + 2 * kGemmTile, kb * kGemmK, tn * kGemmN);
        tma_load_2d(&tmBl, bar_full + 8 * stage, sa + 3 * kGemmTile, kb * kGemmK, tn * kGemmN);
        if (++stage == kGemmStages) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  const int wg = warp >> 2;                                 // rows [64 wg, 64 wg + 64) of the tile
  float acc[kGemmN / 2];
#pragma unroll
  for (int i = 0; i < kGemmN / 2; ++i) acc[i] = 0.f;
  uint32_t stage = 0, phase = 0, prev = 0;
  for (int kb = 0; kb < p.kblocks; ++kb) {
    mbar_wait(bar_full + 8 * stage, phase);
    const uint32_t sa = stage0 + stage * kGemmStageBytes;
    const uint64_t ah = wg_desc(sa + wg * (kGemmTile / 2), 128), al = wg_desc(sa + kGemmTile + wg * (kGemmTile / 2), 128);
    const uint64_t bh = wg_desc(sa + 2 * kGemmTile, 128), bl = wg_desc(sa + 3 * kGemmTile, 128);
    wg_fence();
#pragma unroll
    for (uint32_t k = 0; k < 8; k += 2) {
      // small cross terms first, the dominant hi*hi term last
      Wgmma<kGemmN>::mma(acc, al + k, bh + k);
      Wgmma<kGemmN>::mma(acc, ah + k, bl + k);
      Wgmma<kGemmN>::mma(acc, ah + k, bh + k);
    }
    wg_commit();
    wg_wait<1>();                                           // the previous stage's wgmma have read their operands
    if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_empty + 8 * prev);
    prev = stage;
    if (++stage == kGemmStages) { stage = 0; phase ^= 1; }
  }
  wg_wait<0>();

  const int lane = threadIdx.x & 31, w4 = warp & 3;
  const int col0 = tn * kGemmN + 2 * (lane & 3);
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int m = tm * kGemmM + wg * 64 + w4 * 16 + (lane >> 2) + 8 * i;
    if (m >= p.M) continue;
#pragma unroll
    for (int j = 0; j < kGemmN / 8; ++j) {
      const int col = col0 + 8 * j;
      float a = acc[4 * j + 2 * i], c = acc[4 * j + 2 * i + 1];
      if (p.bias) { a += p.bias[col]; c += p.bias[col + 1]; }
      if (p.act == 1) { a = a > 0.f ? a : 0.01f * a; c = c > 0.f ? c : 0.01f * c; }
      if (GELU) {                                           // exact (erf) GELU, torch.nn.functional.gelu's default
        a = 0.5f * a * (1.f + erff(a * 0.70710678118654752f));
        c = 0.5f * c * (1.f + erff(c * 0.70710678118654752f));
      }
      if (p.scale) { a = a * p.scale[col] + p.shift[col]; c = c * p.scale[col + 1] + p.shift[col + 1]; }
      if (p.C) {
        const float2 v = make_float2(a, c);
        *reinterpret_cast<float2*>(p.C + (size_t)m * p.ldc + col) = v;
        for (int pr = 0; pr < p.n_peer; ++pr)               // push the same values to every peer GPU
          *reinterpret_cast<float2*>(p.C_peer[pr] + (size_t)m * p.ldc + col) = v;
      }
      if (p.C_hi) {
        const __half ah16 = __float2half_rn(a), ch16 = __float2half_rn(c);
        *reinterpret_cast<__half2*>(p.C_hi + (size_t)m * p.ldc_h + col) = __halves2half2(ah16, ch16);
        *reinterpret_cast<__half2*>(p.C_lo + (size_t)m * p.ldc_h + col) =
            __floats2half2_rn(a - __half2float(ah16), c - __half2float(ch16));
      }
    }
  }
}

// fp32 -> (hi, lo) fp16 split, elementwise
__global__ void split_f16_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo,
                                 size_t n) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float v = x[i];
  const __half h = __float2half_rn(v);
  hi[i] = h;
  lo[i] = __float2half_rn(v - __half2float(h));
}

int split_f16(const float* x, __half* hi, __half* lo, size_t n, cudaStream_t st) {
  if (n == 0) return B200_OK;
  return launch(split_f16_kernel, (unsigned)((n + 255) / 256), 256, 0, st, x, hi, lo, n);
}

int gemm_tc_split(const __half* A_hi, const __half* A_lo, int lda, const __half* B_hi, const __half* B_lo, int ldb,
                  float* C, int ldc, __half* C_hi, __half* C_lo, int ldc_h, const float* bias, int M, int N, int K,
                  int act, int num_sms, cudaStream_t stream, float* const* C_peers, int n_peers,
                  const GemmTaps& taps) {
  (void)num_sms;
  B200_CHECK(K % kGemmK == 0 && N % kGemmN == 0 && lda % 8 == 0 && ldb % 8 == 0, B200_ERR_INVALID,
             "gemm_tc_split: unsupported shape M=%d N=%d K=%d", M, N, K);
  B200_CHECK(taps.taps >= 1 && K % (taps.taps * kGemmK) == 0 && taps.dil >= 0 &&
                 (taps.scale == nullptr) == (taps.shift == nullptr),
             B200_ERR_INVALID, "gemm_tc_split: %d taps do not split K=%d into 64-wide k-blocks", taps.taps, K);
  B200_CHECK(n_peers >= 0 && n_peers <= 7 && (n_peers == 0 || (C_peers && C)), B200_ERR_INVALID,
             "gemm_tc_split: at most 7 peer outputs");
  if (M == 0) return B200_OK;
  GemmTcParams p{};
  p.M = M; p.N = N; p.K = K; p.act = act; p.bias = bias; p.C = C; p.C_hi = C_hi; p.C_lo = C_lo; p.ldc = ldc;
  p.ldc_h = ldc_h;
  p.n_peer = n_peers;
  for (int i = 0; i < n_peers; ++i) p.C_peer[i] = C_peers[i];
  p.kblocks = K / kGemmK;
  p.tiles_n = N / kGemmN;
  const int Ka = K / taps.taps;                             // A width: one tap's channels
  p.tap_kb = Ka / kGemmK;
  p.dil = taps.dil;
  p.scale = taps.scale;
  p.shift = taps.shift;
  CUtensorMap tmAh, tmAl, tmBh, tmBl;
  const cuuint64_t a_dims[2] = {(cuuint64_t)Ka, (cuuint64_t)M}, a_str[1] = {(cuuint64_t)lda * 2};
  const cuuint64_t b_dims[2] = {(cuuint64_t)K, (cuuint64_t)N}, b_str[1] = {(cuuint64_t)ldb * 2};
  const cuuint32_t a_box[2] = {kGemmK, kGemmM}, b_box[2] = {kGemmK, kGemmN};
  const CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B;
  int rc;
  // rows of the shifted taps past M read as zero (TMA out-of-bounds fill)
  if ((rc = encode_f16_map(&tmAh, 2, A_hi, a_dims, a_str, a_box, nullptr, swz, "gemm"))) return rc;
  if ((rc = encode_f16_map(&tmAl, 2, A_lo, a_dims, a_str, a_box, nullptr, swz, "gemm"))) return rc;
  if ((rc = encode_f16_map(&tmBh, 2, B_hi, b_dims, b_str, b_box, nullptr, swz, "gemm"))) return rc;
  if ((rc = encode_f16_map(&tmBl, 2, B_lo, b_dims, b_str, b_box, nullptr, swz, "gemm"))) return rc;
  const size_t smem = 1024 + 1024 + (size_t)kGemmStages * kGemmStageBytes;
  const auto kernel = act == 2 ? gemm_tc_split_kernel<true> : gemm_tc_split_kernel<false>;
  const unsigned grid = (unsigned)(ceil_div(M, kGemmM) * p.tiles_n);
  return launch(kernel, grid, kGemmThreads, smem, stream, tmAh, tmAl, tmBh, tmBl, p);
}

}  // namespace b200
