// BiLSTM recurrence on the Hopper tensor cores (wgmma), split-precision fp16 with fp32-level accuracy.
//
// Reference: pyannote/audio/models/segmentation/PyanNet.py:223-228 (nn.LSTM(., 128, bidirectional, batch_first)).
// Per step t:  G[b][(unit, gate)] = Gx[b][t] + h_{t-1}[b] . W_hh^T,  c = f*c + i*g,  h = o * tanh(c).
//
// A 2-CTA cluster runs 64 sequences of one direction; each CTA owns 64 hidden units, i.e. the GEMM
//     D[64 sequences][256 = (unit, gate)] += h[64][128 units] * W[256][128]^T          (m64n256, 8 K=16 steps)
// with its W_hh slice as fp16 (hi, lo) resident in shared memory (TMA once, 128-byte swizzle) and h as the register
// A operand.  The 256 columns are ordered  n = 32 jj + 8 gate + u  (local unit 8 jj + u), so the accumulator
// fragment of a thread holds all four gates of local units 8 jj + 2 (lane % 4) + {0, 1} for its two rows: the gates,
// c (registers) and the new h of those units are computed in place, and the new h pairs are exactly the thread's A
// fragments of the K steps over its own units.  Every thread stores its 16 (hi, lo) pairs into its own CTA's and
// (DSMEM) the peer's h buffer at the same thread index; the next step reads all eight K steps' A fragments from
// there.  One cluster barrier per step.
// Products: h_lo*W_hi + h_hi*W_lo + h_hi*W_hi in fp32, like gemm_tc.cu.
//
// Two kernels: lstm_rec_pipe_kernel (seg_rec_impl = 1) and lstm_rec_wg_kernel (2, the bit-exact reference).  The step
// is a chain of dependent latencies (Gx load, MMAs, gate transcendentals, DSMEM stores, cluster barrier) with only one
// warp per SM sub-partition in the reference; the pipelined kernel splits the 256 columns over two warpgroups (each
// m64n128, the same 24 products per column in the same order) so that every sub-partition interleaves two warps' gate
// math, loads step t+1's Gx into registers behind step t's MMAs and gates, and splits the cluster barrier around the
// Gx -> accumulator copy.
#include "common.cuh"
#include "seg.cuh"
#include "tc_common.cuh"

namespace b200 {

constexpr int kRecThreads = 128;
constexpr int kRecSeqs = 64;
constexpr uint32_t kRecWBox = 256u * 128u;              // one [256 rows][64 k] fp16 box (32 KB)
constexpr uint32_t kRecXOff = 1024u + 4u * kRecWBox;     // h buffers [2 parity][2 source CTA][32 regs][128 threads] u32

__device__ __forceinline__ float rec_sigmoid(float x) { return 1.f / (1.f + expf(-x)); }

__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(kRecThreads, 1)
lstm_rec_wg_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl,
                   const float* __restrict__ Gx /*[NB][T][1024]*/, __half* __restrict__ Yh, __half* __restrict__ Yl,
                   int NB, int T, int ntiles) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t bar = base, w_smem = base + 1024u;
  uint32_t* xbuf = reinterpret_cast<uint32_t*>(smem_raw + (base - raw) + kRecXOff);
  uint32_t rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  const int cid = blockIdx.x >> 1;
  const int dir = cid / ntiles, tile = cid - dir * ntiles;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q = lane & 3;
  uint32_t peer_x;                                       // the peer CTA's h buffers
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer_x) : "r"(base + kRecXOff), "r"(rank ^ 1u));

  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(bar, 4u * kRecWBox);
    const int slice = dir * 2 + (int)rank;
    tma_load_3d(&tmWh, bar, w_smem, 0, 0, slice);
    tma_load_3d(&tmWh, bar, w_smem + kRecWBox, 64, 0, slice);
    tma_load_3d(&tmWl, bar, w_smem + 2 * kRecWBox, 0, 0, slice);
    tma_load_3d(&tmWl, bar, w_smem + 3 * kRecWBox, 64, 0, slice);
  }
  for (int i = threadIdx.x; i < 2 * 32 * kRecThreads; i += kRecThreads) xbuf[i] = 0u;   // h_{-1} = 0 (parity 0)
  // both CTAs of the cluster are running (and zeroed) before anything is stored into the peer
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  mbar_wait(bar, 0);

  int rows[2];
  rows[0] = tile * kRecSeqs + 16 * warp + (lane >> 2);
  rows[1] = rows[0] + 8;
  float c[2][8][2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) c[i][jj][0] = c[i][jj][1] = 0.f;
  const int gcol = dir * 512 + ((int)rank * 64 + 2 * q) * 4;   // + 32 jj: units 8 jj + 2q, +1, four gates each

  float acc[128];
  for (int step = 0; step < T; ++step) {
    const int t = dir ? (T - 1 - step) : step;
    // acc = Gx[b][t] (the input projection with both biases)
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const bool ok = rows[i] < NB;
      const float4* gp = reinterpret_cast<const float4*>(Gx + ((size_t)(ok ? rows[i] : 0) * T + t) * 1024 + gcol);
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        const float4 u0 = ok ? __ldg(gp + 8 * jj) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 u1 = ok ? __ldg(gp + 8 * jj + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float v[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};   // (unit e, gate g) at 4 e + g
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
          for (int e = 0; e < 2; ++e) acc[4 * (4 * jj + g) + 2 * i + e] = v[4 * e + g];
      }
      if (step + 1 < T && ok) {                     // next step's projection into L2
        const int tn = dir ? t - 1 : t + 1;
        const char* np = reinterpret_cast<const char*>(Gx + ((size_t)rows[i] * T + tn) * 1024 + gcol);
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) asm volatile("prefetch.global.L2 [%0];" ::"l"(np + 128 * jj));
      }
    }
    // acc += h_{t-1} W^T over the 8 K steps (K steps 4 r .. 4 r + 3 = the units of CTA r)
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const int s = ks & 3;                               // K step inside one CTA's 64 units: jj = 2s, 2s + 1
      const uint32_t* xb = xbuf + ((step & 1) * 2 + (ks >> 2)) * 32 * kRecThreads;
      uint32_t ah[4], al[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = r & 1, jj = 2 * s + (r >> 1);
        ah[r] = xb[(i * 8 + jj) * kRecThreads + tid];
        al[r] = xb[(16 + i * 8 + jj) * kRecThreads + tid];
      }
      const uint32_t wb = w_smem + (uint32_t)(ks >> 2) * kRecWBox + (uint32_t)(ks & 3) * 32u;
      const uint64_t wh = wg_desc(wb, 128), wl = wg_desc(wb + 2 * kRecWBox, 128);
      WgmmaRS<256>::mma(acc, al, wh);                      // small cross terms first, hi*hi last
      WgmmaRS<256>::mma(acc, ah, wl);
      WgmmaRS<256>::mma(acc, ah, wh);
    }
    wg_commit();
    wg_wait<0>();
    // gates (PyTorch order i, f, g, o), cell update, new h: both CTAs' h buffers, layer output
    const uint32_t hoff = (uint32_t)((((step + 1) & 1) * 2 + (int)rank) * 32 * kRecThreads + tid);
    uint32_t* own = xbuf + hoff;
    const uint32_t px = peer_x + hoff * 4u;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        float hn[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float ig = rec_sigmoid(acc[4 * (4 * jj + 0) + 2 * i + e]);
          const float fg = rec_sigmoid(acc[4 * (4 * jj + 1) + 2 * i + e]);
          const float gg = tanhf(acc[4 * (4 * jj + 2) + 2 * i + e]);
          const float og = rec_sigmoid(acc[4 * (4 * jj + 3) + 2 * i + e]);
          c[i][jj][e] = fmaf(fg, c[i][jj][e], ig * gg);
          hn[e] = og * tanhf(c[i][jj][e]);
        }
        const __half h0 = __float2half_rn(hn[0]), h1 = __float2half_rn(hn[1]);
        const __half2 hi2 = __halves2half2(h0, h1);
        const uint32_t vh = *reinterpret_cast<const uint32_t*>(&hi2);
        const uint32_t vl = pack_h2(hn[0] - __half2float(h0), hn[1] - __half2float(h1));
        own[(i * 8 + jj) * kRecThreads] = vh;
        own[(16 + i * 8 + jj) * kRecThreads] = vl;
        asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(px + (uint32_t)((i * 8 + jj) * kRecThreads) * 4u),
                     "r"(vh) : "memory");
        asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(px + (uint32_t)((16 + i * 8 + jj) * kRecThreads) * 4u),
                     "r"(vl) : "memory");
        if (rows[i] < NB) {
          const size_t o = ((size_t)rows[i] * T + t) * 256 + dir * 128 + rank * 64 + 8 * jj + 2 * q;
          *reinterpret_cast<uint32_t*>(Yh + o) = vh;
          *reinterpret_cast<uint32_t*>(Yl + o) = vl;
        }
      }
    }
    // the peer's h of this step has landed; both CTAs are done reading the buffer the next step overwrites
    asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  }
}

// ---- two consumer warpgroups per CTA, Gx software-pipelined (seg_rec_impl = 1) --------------------------------------
// Warpgroup g owns the CTA's local units 32 g .. 32 g + 31, i.e. columns n = 128 g + 32 j + 8 gate + u (j = 0..3): its
// accumulator is the m64n128 slice of the reference's m64n256 tile that starts at W_hh row 128 g, and each of its
// columns gets the reference's 24 products (K steps 0..7; lo*hi, hi*lo, hi*hi) in the reference's order.  Both
// warpgroups read the same A fragments; thread t of warpgroup g stores its new h at thread index t, at jj = 4 g + j, so
// the h buffers keep the reference's layout.
struct RecPipePlan {
  static constexpr int kWarpgroups = 2;
  static constexpr int kThreads = 128 * kWarpgroups;
  static constexpr int kCols = 256 / kWarpgroups;                  // accumulator columns per warpgroup
  static constexpr uint32_t kBar = 0;                             // weight mbarrier
  static constexpr uint32_t kW = 1024;                            // W_hh (hi, lo) x (k 0..63, 64..127) boxes
  static constexpr uint32_t kWgColBytes = (uint32_t)kCols * 128u;  // one warpgroup's 128 rows of a box
  static constexpr uint32_t kX = kW + 4u * kRecWBox;              // h buffers, as the reference's
  static constexpr uint32_t kXBytes = 2u * 2u * 32u * 128u * 4u;  // [2 parity][2 source CTA][32 regs][128 threads] u32
  static constexpr size_t kSmem = 1024 + kX + kXBytes;            // + alignment slack of the dynamic window
  static_assert(kX == kRecXOff, "same h buffer offset as the reference kernel");
  static_assert(kW % 1024 == 0 && kRecWBox % 1024 == 0 && kWgColBytes % 1024 == 0,
                "128-byte swizzle atoms (8 rows of 128 B) must start 1024-byte aligned");
  static_assert(kCols * kWarpgroups == 256 && kCols == 128, "each warpgroup runs m64n128");
  static_assert(kSmem <= 227u * 1024u, "one CTA per SM");
};

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(RecPipePlan::kThreads, 1)
lstm_rec_pipe_kernel(const __grid_constant__ CUtensorMap tmWh, const __grid_constant__ CUtensorMap tmWl,
                     const float* __restrict__ Gx /*[NB][T][1024]*/, __half* __restrict__ Yh, __half* __restrict__ Yl,
                     int NB, int T, int ntiles) {
  using P = RecPipePlan;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;
  const uint32_t bar = base + P::kBar, w_smem = base + P::kW;
  uint32_t* xbuf = reinterpret_cast<uint32_t*>(smem_raw + (base - raw) + P::kX);
  uint32_t rank;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
  const int cid = blockIdx.x >> 1;
  const int dir = cid / ntiles, tile = cid - dir * ntiles;
  const int tid = threadIdx.x, wg = tid >> 7, t128 = tid & 127, warp = t128 >> 5, lane = tid & 31, q = lane & 3;
  uint32_t peer_x;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(peer_x) : "r"(base + P::kX), "r"(rank ^ 1u));

  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    mbar_expect_tx(bar, 4u * kRecWBox);
    const int slice = dir * 2 + (int)rank;
    tma_load_3d(&tmWh, bar, w_smem, 0, 0, slice);
    tma_load_3d(&tmWh, bar, w_smem + kRecWBox, 64, 0, slice);
    tma_load_3d(&tmWl, bar, w_smem + 2 * kRecWBox, 0, 0, slice);
    tma_load_3d(&tmWl, bar, w_smem + 3 * kRecWBox, 64, 0, slice);
  }
  for (int i = tid; i < 2 * 32 * 128; i += P::kThreads) xbuf[i] = 0u;   // h_{-1} = 0 (parity 0)
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
  mbar_wait(bar, 0);

  int rows[2];
  rows[0] = tile * kRecSeqs + 16 * warp + (lane >> 2);
  rows[1] = rows[0] + 8;
  const bool ok[2] = {rows[0] < NB, rows[1] < NB};
  float c[2][4][2];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) c[i][j][0] = c[i][j][1] = 0.f;
  // + 32 j: units 32 wg + 8 j + 2q, +1, four gates each
  const int gcol = dir * 512 + ((int)rank * 64 + 32 * wg + 2 * q) * 4;

  // gx = Gx[b][t] (the input projection with both biases) in accumulator order: (j, gate, row i, unit e)
  float gx[64];
  auto load_gx = [&](int t) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const float4* gp = reinterpret_cast<const float4*>(Gx + ((size_t)(ok[i] ? rows[i] : 0) * T + t) * 1024 + gcol);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float4 u0 = ok[i] ? __ldg(gp + 8 * j) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float4 u1 = ok[i] ? __ldg(gp + 8 * j + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
        const float v[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};   // (unit e, gate g) at 4 e + g
#pragma unroll
        for (int g = 0; g < 4; ++g)
#pragma unroll
          for (int e = 0; e < 2; ++e) gx[4 * (4 * j + g) + 2 * i + e] = v[4 * e + g];
      }
    }
  };
  load_gx(dir ? T - 1 : 0);
  // h_{-1} is in place: this arrive pairs with the first step's wait
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");

  const uint32_t w_wg = w_smem + (uint32_t)wg * P::kWgColBytes;
  float acc[64];
  for (int step = 0; step < T; ++step) {
    const int t = dir ? (T - 1 - step) : step;
#pragma unroll
    for (int r = 0; r < 64; ++r) acc[r] = gx[r];
    // the peer's h of the previous step has landed; every thread is done reading the buffer this step overwrites
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
    // acc += h_{t-1} W^T over the 8 K steps (K steps 4 r .. 4 r + 3 = the units of CTA r)
    wg_fence();
#pragma unroll
    for (int ks = 0; ks < 8; ++ks) {
      const int s = ks & 3;
      const uint32_t* xb = xbuf + ((step & 1) * 2 + (ks >> 2)) * 32 * 128;
      uint32_t ah[4], al[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int i = r & 1, jj = 2 * s + (r >> 1);
        ah[r] = xb[(i * 8 + jj) * 128 + t128];
        al[r] = xb[(16 + i * 8 + jj) * 128 + t128];
      }
      const uint32_t wb = w_wg + (uint32_t)(ks >> 2) * kRecWBox + (uint32_t)(ks & 3) * 32u;
      const uint64_t wh = wg_desc(wb, 128), wl = wg_desc(wb + 2 * kRecWBox, 128);
      WgmmaRS<P::kCols>::mma(acc, al, wh);                 // small cross terms first, hi*hi last
      WgmmaRS<P::kCols>::mma(acc, ah, wl);
      WgmmaRS<P::kCols>::mma(acc, ah, wh);
    }
    wg_commit();
    if (step + 1 < T) load_gx(dir ? t - 1 : t + 1);      // in flight behind the MMAs and the gate math
    wg_wait<0>();
    // gates (PyTorch order i, f, g, o), cell update, new h: both CTAs' h buffers, layer output
    const uint32_t hoff = (uint32_t)((((step + 1) & 1) * 2 + (int)rank) * 32 * 128 + t128);
    uint32_t* own = xbuf + hoff;
    const uint32_t px = peer_x + hoff * 4u;
    uint32_t yv[2][4][2];                                  // layer output (hi, lo), stored after the arrive
#pragma unroll
    for (int i = 0; i < 2; ++i) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int jj = 4 * wg + j;
        float hn[2];
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const float ig = rec_sigmoid(acc[4 * (4 * j + 0) + 2 * i + e]);
          const float fg = rec_sigmoid(acc[4 * (4 * j + 1) + 2 * i + e]);
          const float gg = tanhf(acc[4 * (4 * j + 2) + 2 * i + e]);
          const float og = rec_sigmoid(acc[4 * (4 * j + 3) + 2 * i + e]);
          c[i][j][e] = fmaf(fg, c[i][j][e], ig * gg);
          hn[e] = og * tanhf(c[i][j][e]);
        }
        const __half h0 = __float2half_rn(hn[0]), h1 = __float2half_rn(hn[1]);
        const __half2 hi2 = __halves2half2(h0, h1);
        const uint32_t vh = *reinterpret_cast<const uint32_t*>(&hi2);
        const uint32_t vl = pack_h2(hn[0] - __half2float(h0), hn[1] - __half2float(h1));
        own[(i * 8 + jj) * 128] = vh;
        own[(16 + i * 8 + jj) * 128] = vl;
        asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(px + (uint32_t)((i * 8 + jj) * 128) * 4u), "r"(vh)
                     : "memory");
        asm volatile("st.shared::cluster.u32 [%0], %1;" ::"r"(px + (uint32_t)((16 + i * 8 + jj) * 128) * 4u), "r"(vl)
                     : "memory");
        yv[i][j][0] = vh;
        yv[i][j][1] = vl;
      }
    }
    // the release fence of the arrive waits for this thread's outstanding stores: the global ones go after it, so
    // that only the next step's arrive (a whole step later) covers them
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (!ok[i]) continue;
      const size_t o = ((size_t)rows[i] * T + t) * 256 + dir * 128 + rank * 64 + 32 * wg + 2 * q;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        *reinterpret_cast<uint32_t*>(Yh + o + 8 * j) = yv[i][j][0];
        *reinterpret_cast<uint32_t*>(Yl + o + 8 * j) = yv[i][j][1];
      }
    }
  }
  // no CTA leaves while its peer may still store into its shared memory
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

int lstm_rec_wg(const float* Gx, const __half* Wh, const __half* Wl, __half* Yh, __half* Yl, int NB, int T, int impl,
                cudaStream_t stream) {
  CUtensorMap tm[2];
  const cuuint64_t dims[3] = {128, 256, 4};                 // [k = unit][n = (unit, gate) column][dir * 2 + rank]
  const cuuint64_t strides[2] = {128 * 2, 256 * 128 * 2};
  const cuuint32_t box[3] = {64, 256, 1};
  int rc;
  for (int h = 0; h < 2; ++h)
    if ((rc = encode_f16_map(&tm[h], 3, h ? Wl : Wh, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_128B,
                             "lstm W_hh")))
      return rc;
  const int ntiles = ceil_div(NB, kRecSeqs);
  if (impl == 1)
    return launch(lstm_rec_pipe_kernel, 2 * 2 * ntiles, RecPipePlan::kThreads, RecPipePlan::kSmem, stream, tm[0], tm[1],
                  Gx, Yh, Yl, NB, T, ntiles);
  const size_t smem = 1024 + kRecXOff + 4u * 32u * kRecThreads * 4u;
  return launch(lstm_rec_wg_kernel, 2 * 2 * ntiles, kRecThreads, smem, stream, tm[0], tm[1], Gx, Yh, Yl, NB, T, ntiles);
}

}  // namespace b200
