// WeSpeaker ResNet34 trunk convolutions for H100 (sm_90a).
//
// Reference semantics: /root/reference/src/pyannote/audio/models/embedding/wespeaker/resnet.py
//   BasicBlock.forward :140-145 (conv3x3-BN-ReLU-conv3x3-BN + shortcut -> ReLU), ResNet.forward :413-419.
// Eval-mode BatchNorm is folded into the conv weights / a per-channel bias on the host (api.cu make_conv).
//
// conv_tc_kernel: implicit-GEMM convolution on the Hopper tensor cores (wgmma), one CTA per output tile.
//   GEMM view  D[M=128 output pixels of one image row][N=C_out] += A[M][K] * B[N][K]^T,  K = taps * C_in walked tap by
//   tap in chunks of Ck channels.  Activations are NHWC fp16 so that one TMA box (Ck channels x consecutive pixels)
//   lands in shared memory as a K-major, hardware-swizzled A tile; convolution padding is TMA out-of-bounds zero fill,
//   stride 2 is the tensor map's element stride.  Weights [tap][C_out][C_in] land the same way as K-major B tiles.
//   A stage of the mbarrier ring, filled by a TMA producer warp (warp 8), holds one 128-pixel box and one weight tap.
//   Warpgroups 0 / 1 = output pixels [0, 64) / [64, 128) of the tile, fp32 accumulators in registers, epilogue
//   (+bias (+residual) -> ReLU -> fp16 NHWC store) straight from the accumulator fragments.
// conv_row_kernel: the stride-1 3x3 convs with one channel chunk and C_in = C_out (32 or 64: ResNet34's 7 stride-1
//   layer-2 convs and the conv2 of the bottleneck trunks' layers 1 and 2), which are bound by HBM rather than by the
//   tensor cores.  Persistent: about num_sms CTAs (two per SM for
//   C_out = 32) walk units of one segment x one 128-pixel column tile x a band of consecutive output rows.
//   - The nine weight taps are loaded once per CTA and stay in shared memory.
//   - Input rows h0 - 1 .. h1 of a band are staged once each, as one box of 128 + 8 pixels, in a ring of row slots;
//     output row h reads slots h - 1, h, h + 1, and tap (kh, kw) reads slot kh from pixel row kw on.  A slot is freed
//     after its three consumer rows are done (rows at the band edges arrive for the missing ones).
//   - Warpgroups 0 / 1 take alternate output rows, each a whole 128-pixel row as two m64 wgmma per K step, so one
//     warpgroup's epilogue runs while the other's MMAs do.
//   - The epilogue goes through a shared-memory tile per warpgroup: the producer stages the row's residual there by
//     TMA while the MMAs run, and the finished row leaves with one TMA store.  The epilogue makes no global loads, so
//     it does not wait on a memory round trip per residual load (the output may alias the residual).
//   The A operand comes straight from shared memory, the descriptor start moved by kw rows of 128 B, except for
//   Ck = 32 (64-B rows: layer 1): those fragments are read with ldmatrix, the 64-B swizzle applied in software, and
//   issued as register-A wgmma.
//   Each output sums its products in the (tap, 16-channel step) order of conv_tc_kernel, and the epilogue is the same,
//   so the two kernels give bit-identical results.
// conv_chunk_row_kernel: the stride-1 3x3 convs with C_in = C_out = 128 or 256 (layers 3 and 4, 16 of the 35, and the
//   conv2 of the bottleneck trunks' layers 3 and 4).  Persistent CTAs, one per SM, walk units of one 128-pixel column
//   tile x two output rows (C_out = 128; warpgroup r computes row h + r) or one (256; warpgroup r computes half r),
//   with conv_tc_kernel's wgmma shapes.  The producer stages each input row of a unit once per 64-channel chunk as a
//   136-pixel box, and tap kw reads it from pixel row kw on, as in conv_row_kernel.  Each weight tile is staged once
//   per unit, so with two rows it feeds four m64 groups instead of two: about half the operand fill from L2 of one
//   row per unit.  The consumers still walk (kh, kw, chunk, 16-channel step), so every chunk box of a kernel row stays
//   resident until its tap kw = 2, and the results are bit-identical to conv_tc_kernel's.  Weight tiles stream through
//   a ring of their own, and the producer stages the next unit while the consumers run the epilogue.
// block_row_kernel: a whole stride-1 BasicBlock with 32 channels (the three blocks of ResNet34 layer 1) in one launch,
//   built on conv_row_kernel's row walk: conv1's output rows go to a ring of intermediate row slots in shared memory
//   and conv2 reads them from there, so a block reads its input and writes its output once instead of making five
//   passes over 80 x T0 x 32 activations.  Bit-identical to the two convs run apart.
#include "common.cuh"
#include "emb.cuh"
#include "tc_common.cuh"

namespace b200 {

constexpr int kWgThreads = 288;
constexpr int kTileM = 128;
constexpr int kRowHalo = 8;                                 // 128 + 2 pixels needed for three taps, 8 keeps 8-row groups
constexpr int kMaxSlots = 16;                               // row slots of conv_row_kernel (barrier area: 1024 B)

// +bias (+residual) -> ReLU -> fp16 of MH = 1 or 2 64 x N accumulator fragments, consecutive at `acc`: fragment m
// holds output pixels [w0 + 64 m, w0 + 64 m + 64) of image row `row` (= b * H_out + h).  A residual aliasing `out` is
// read before it is overwritten, by the same thread.
// WIDE: the fragment is output channels [n0, n0 + N) of C_out (n0 = blockIdx.y * N), pixels C_out channels apart.
template <int N, bool WIDE = false, int MH = 1>
__device__ __forceinline__ void conv_epilogue(const float* acc, const ConvParams& p, size_t row, int w0) {
  const int lane = threadIdx.x & 31;
  const int c0 = 2 * (lane & 3) + (WIDE ? (int)blockIdx.y * N : 0);
#pragma unroll
  for (int m = 0; m < MH; ++m)
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int w = w0 + 64 * m + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2) + 8 * i;
    if (w >= p.W_out) continue;
    const size_t pix = (row * p.W_out + w) * (size_t)(WIDE ? p.C_out : N);
    // up to C_out = 128 all of the pixel's residual loads are issued before its first store: `out` may alias
    // `residual`, so a load after a store cannot be hoisted and each would wait a full memory round trip (at 256 the
    // registers are not there: conv_tc_kernel<256> would spill)
    __half2 res[N / 8];
    if (N <= 128 && p.residual) {
#pragma unroll
      for (int j = 0; j < N / 8; ++j) res[j] = *reinterpret_cast<const __half2*>(p.residual + pix + 8 * j + c0);
    }
#pragma unroll
    for (int j = 0; j < N / 8; ++j) {
      const int c = 8 * j + c0;
      const float2 bb = __ldg(reinterpret_cast<const float2*>(p.bias + c));
      float a = acc[m * (N / 2) + 4 * j + 2 * i] + bb.x, d = acc[m * (N / 2) + 4 * j + 2 * i + 1] + bb.y;
      if (p.residual) {
        const float2 r = __half22float2(N <= 128 ? res[j] : *reinterpret_cast<const __half2*>(p.residual + pix + c));
        a += r.x;
        d += r.y;
      }
      if (p.relu) { a = fmaxf(a, 0.f); d = fmaxf(d, 0.f); }
      *reinterpret_cast<__half2*>(p.out + pix + c) = __floats2half2_rn(a, d);
    }
  }
}

// WIDE: C_out > 256 (the bottleneck trunk's 512 / 1024-channel 1x1 convs), grid.y = the 256-channel column tile
template <int N, int CK, bool WIDE = false>
__global__ void __launch_bounds__(kWgThreads, N == 256 ? 1 : 2)
conv_tc_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, ConvParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw = smem_u32(smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;            // swizzle-128B operands need 1024 B alignment
  const uint32_t bar_full = base, bar_empty = base + 64;    // 8 x 8 B each
  const uint32_t stage0 = base + 1024;
  const uint32_t stage_bytes = p.a_bytes + p.b_bytes;
  const int warp = threadIdx.x >> 5;
  const int wt = blockIdx.x % p.tiles_w;
  const int bh = blockIdx.x / p.tiles_w;                    // = b * H_out + h
  const int cchunks = p.C_in / CK;

  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < p.nstages; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if ((threadIdx.x & 31) == 0) {
      prefetch_tensormap(&tmA);
      prefetch_tensormap(&tmB);
      const int h = bh % p.H_out, b = bh / p.H_out;
      const int w_base = wt * kTileM * p.stride - p.pad, h_base = h * p.stride - p.pad;
      uint32_t stage = 0, phase = 0;
      for (int kh = 0; kh < p.taps_h; ++kh)
        for (int kw = 0; kw < p.taps_w; ++kw)
          for (int cc = 0; cc < cchunks; ++cc) {
            mbar_wait(bar_empty + 8 * stage, phase ^ 1);
            mbar_expect_tx(bar_full + 8 * stage, p.a_tx + p.b_bytes);
            const uint32_t sa = stage0 + stage * stage_bytes;
            tma_load_4d(&tmA, bar_full + 8 * stage, sa, cc * CK, w_base + kw, h_base + kh, b);
            tma_load_3d(&tmB, bar_full + 8 * stage, sa + p.a_bytes, cc * CK, WIDE ? (int)blockIdx.y * N : 0,
                        kh * p.taps_w + kw);
            if (++stage == p.nstages) { stage = 0; phase ^= 1; }
          }
    }
    return;
  }

  const int wg = warp >> 2;
  constexpr uint32_t row_bytes = CK * 2;                   // = the swizzle width (64 or 128 B)
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  const int kblocks = p.taps_h * p.taps_w * cchunks;
  uint32_t stage = 0, phase = 0, prev = 0;
  for (int kb = 0; kb < kblocks; ++kb) {
    mbar_wait(bar_full + 8 * stage, phase);
    const uint32_t st = stage0 + stage * stage_bytes;
    const uint32_t sa = st + (uint32_t)wg * 64u * row_bytes, sb = st + p.a_bytes;
    wg_fence();
    const uint64_t ad = wg_desc(sa, row_bytes), bd = wg_desc(sb, row_bytes);
#pragma unroll
    for (int k = 0; k < CK / 16; ++k) Wgmma<N>::mma(acc, ad + 2 * k, bd + 2 * k);   // +32 B per K=16 step
    wg_commit();
    wg_wait<1>();                                           // the previous stage's wgmma have read their operands
    if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(bar_empty + 8 * prev);
    prev = stage;
    if (++stage == p.nstages) { stage = 0; phase ^= 1; }
  }
  wg_wait<0>();
  conv_epilogue<N, WIDE>(acc, p, (size_t)bh, wt * kTileM + wg * 64);
}

// acc[m] (the 64-pixel halves of a 128-pixel row) += the three kw taps of one kernel row over 32 input channels: the
// row slot at `sa` is read from pixel row kw on, the taps' [N][32] weights lie at wts, wts + N * 64 and wts + N * 128.
// Pixel row r of this warp's 16 (lanes 0-15 / 16-31: K columns 0-7 / 8-15 of each step) at 64-B rows, 16-B chunk c
// stored at chunk c ^ ((row >> 1) & 3) (64-B swizzle; slots are 1024-B aligned).
template <int N>
__device__ __forceinline__ void row_taps_c32(float (&acc)[2][N / 2], uint32_t sa, uint32_t wts) {
  constexpr uint32_t row_bytes = 64;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int kw = 0; kw < 3; ++kw) {
    uint32_t af[2][2][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        const uint32_t row = (uint32_t)(m * 64 + (warp & 3) * 16 + (lane & 15) + kw);
        const uint32_t chunk = (uint32_t)(2 * k + (lane >> 4)) ^ ((row >> 1) & 3u);
        ldsm_x4(af[m][k], sa + row * row_bytes + chunk * 16u);
      }
    wg_fence();
    const uint64_t bd = wg_desc(wts + kw * N * row_bytes, row_bytes);
#pragma unroll
    for (int k = 0; k < 2; ++k)
#pragma unroll
      for (int m = 0; m < 2; ++m) WgmmaRS<N>::mma(acc[m], af[m][k], bd + 2 * k);
    wg_commit();
    wg_wait<0>();                                           // the fragments are rewritten by the next ldmatrix
  }
}

__device__ __forceinline__ void st_shared_u32(uint32_t a, uint32_t v) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_shared_u32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<uint32_t*>(&h); }

// Plan of conv_row_kernel<N> (C_in = C_out = N = the channel chunk): the nine weight taps resident, one epilogue tile
// per warpgroup (its output row: 128 pixels x N channels, the residual's and the output's TMA box) and a ring of input
// row slots (136-pixel boxes, padded to 1024 B).  Two warpgroups on consecutive rows hold four slots, so the rest is
// how many rows the producer stages ahead.
//   N = 64: one CTA per SM, 2 KB of barriers + 72 KB of weights + 2 x 16 KB tiles + 7 slots of 17 KB (225 KB).
//   N = 32: two CTAs per SM at 113 KB, 2 KB + 18 KB + 2 x 8 KB + 8 slots of 9 KB (108 KB).
template <int N>
struct RowPlan {
  static constexpr uint32_t kRowBytes = N * 2;             // one pixel = the swizzle width (64 or 128 B)
  static constexpr uint32_t kTapBytes = N * kRowBytes;
  static constexpr uint32_t kInTx = (kTileM + kRowHalo) * kRowBytes;
  static constexpr uint32_t kSlotBytes = (kInTx + 1023u) & ~1023u;
  static constexpr uint32_t kTileBytes = kTileM * kRowBytes;
  static constexpr uint32_t kSlots = N == 64 ? 7 : 8;
  // the producer stages output row j's residual after input row j + kResLag of the unit (staged rows 0 .. n + 1);
  // the slot of that row is freed by output row j - 2, whose store also frees row j's tile
  static constexpr int kResLag = (int)kSlots - 2;
  static constexpr int kCtasPerSm = N == 32 ? 2 : 1;
  static constexpr size_t kBudget = N == 32 ? 113u * 1024 : 227u * 1024;
  static constexpr size_t kSmem = 2048 + 9 * kTapBytes + 2 * kTileBytes + kSlots * kSlotBytes;
  static_assert(N == 32 || N == 64, "row kernel: 32 or 64 channels");
  static_assert(kSlots >= 6 && kSlots <= kMaxSlots, "row ring: four slots in use and two ahead");
  static_assert(kSmem <= kBudget && kSmem + kSlotBytes > kBudget, "row plan: every slot that fits");
};

// The output row goes through the warpgroup's epilogue tile: the producer stages the residual row there by TMA (zeros
// beyond W_out), each thread replaces its residual values with its results in place, and one TMA store (clipped at
// W_out) writes the row.  The tile is 128 pixels of kRowBytes, 16-B chunk c of pixel px stored at chunk
// c ^ (px & 7) (128-B swizzle) or c ^ ((px >> 1) & 3) (64-B swizzle), as the input boxes.  Barriers: tile "full" (the
// residual's TMA bytes) and "empty" (the warpgroup leader, once the previous store has read the tile).
template <int N, int CK>
__global__ void __launch_bounds__(kWgThreads, N == 32 ? 2 : 1)
conv_row_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                const __grid_constant__ CUtensorMap tmR, const __grid_constant__ CUtensorMap tmO, ConvParams p) {
  using P = RowPlan<N>;
  static_assert(CK == N, "row kernel: one channel chunk");
  constexpr uint32_t row_bytes = P::kRowBytes;
  constexpr uint32_t b_tap_bytes = P::kTapBytes;
  constexpr uint32_t nslots = P::kSlots;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_w = base, bar_full = base + 8, bar_empty = base + 8 + 8 * kMaxSlots;
  const uint32_t tile_full = base + 512, tile_empty = base + 528;   // 2 x 8 B each
  const uint32_t wts = base + 1024;                         // 9 taps x [N][CK]
  const uint32_t tile0 = wts + 9 * b_tap_bytes;             // 18 / 72 KB: tiles and slots stay 1024-B aligned
  const uint32_t slot0 = tile0 + 2 * P::kTileBytes;
  const bool has_res = p.residual != nullptr;
  const int warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    mbar_init(bar_w, 1);
    for (uint32_t s = 0; s < nslots; ++s) { mbar_init(bar_full + 8 * s, 1); mbar_init(bar_empty + 8 * s, 3); }
    for (uint32_t s = 0; s < 2; ++s) { mbar_init(tile_full + 8 * s, 1); mbar_init(tile_empty + 8 * s, 1); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // unit u: column tile u % tiles_w (neighbouring CTAs share the halo pixels in L2), then band, then segment
  if (warp == 8) {
    if ((threadIdx.x & 31) == 0) {
      prefetch_tensormap(&tmA);
      prefetch_tensormap(&tmB);
      if (has_res) prefetch_tensormap(&tmR);
      mbar_expect_tx(bar_w, 9 * b_tap_bytes);
      for (int kh = 0; kh < 3; ++kh) tma_load_3d(&tmB, bar_w, wts + 3 * kh * b_tap_bytes, 0, 0, 3 * kh);
      uint32_t s = 0;                                       // input rows staged so far
      uint32_t k = 0;                                       // residual rows staged so far; row k goes to tile k & 1
      for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
        const int wt = u % p.tiles_w, t = u / p.tiles_w;
        const int h0 = (t % p.bands) * p.band, b = t / p.bands;
        const int n = min(p.band, p.H_out - h0);
        auto stage_residual = [&](int j) {
          const uint32_t tile = k & 1, use = k >> 1;
          mbar_wait(tile_empty + 8 * tile, (use & 1) ^ 1);
          mbar_expect_tx(tile_full + 8 * tile, P::kTileBytes);
          tma_load_4d(&tmR, tile_full + 8 * tile, tile0 + tile * P::kTileBytes, 0, wt * kTileM, h0 + j, b);
          ++k;
        };
        for (int r = 0; r < n + 2; ++r, ++s) {
          const uint32_t slot = s % nslots;
          mbar_wait(bar_empty + 8 * slot, ((s / nslots) & 1) ^ 1);
          mbar_expect_tx(bar_full + 8 * slot, P::kInTx);
          tma_load_4d(&tmA, bar_full + 8 * slot, slot0 + slot * P::kSlotBytes, 0, wt * kTileM - 1, h0 - 1 + r, b);
          if (has_res && r >= P::kResLag) stage_residual(r - P::kResLag);
        }
        if (has_res)
          for (int j = max(0, n + 2 - P::kResLag); j < n; ++j) stage_residual(j);
      }
    }
    return;
  }

  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);  // warp-uniform to the compiler: no wgmma serialisation
  const int lane = threadIdx.x & 31;
  const bool leader = (threadIdx.x & 127) == 0;
  const uint32_t tile = tile0 + wg * P::kTileBytes;
  const int c0 = 2 * (lane & 3);
  float2 bias[N / 8];                                       // channels 8 j + c0, c0 + 1 of this thread's fragments
#pragma unroll
  for (int j = 0; j < N / 8; ++j) bias[j] = __ldg(reinterpret_cast<const float2*>(p.bias + 8 * j + c0));
  if (leader) prefetch_tensormap(&tmO);
  mbar_wait(bar_w, 0);
  uint32_t s = 0;                                           // first input row of the current unit
  int item = 0;                                             // output rows walked so far; row `item` is warpgroup item & 1's
  for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
    const int wt = u % p.tiles_w, t = u / p.tiles_w;
    const int h0 = (t % p.bands) * p.band, b = t / p.bands;
    const int n = min(p.band, p.H_out - h0);
    for (int j = 0; j < n; ++j, ++item) {
      if ((item & 1) != wg) continue;
      float acc[2][N / 2];                                  // output pixels [0, 64) / [64, 128) of the row
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int i = 0; i < N / 2; ++i) {
          acc[m][i] = 0.f;
          asm volatile("" : "+f"(acc[m][i]));               // zeroed before the first wg_fence, not sunk past it
        }
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const uint32_t q = s + j + kh, slot = q % nslots;
        mbar_wait(bar_full + 8 * slot, (q / nslots) & 1);
        const uint32_t sa = slot0 + slot * P::kSlotBytes;
        if constexpr (CK == 32) {
          row_taps_c32<N>(acc, sa, wts + 3 * kh * b_tap_bytes);
        } else {
          wg_fence();
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            const uint64_t bd = wg_desc(wts + (3 * kh + kw) * b_tap_bytes, row_bytes);
#pragma unroll
            for (int m = 0; m < 2; ++m) {
              const uint64_t ad = wg_desc(sa + (uint32_t)(m * 64 + kw) * row_bytes, row_bytes);
#pragma unroll
              for (int k = 0; k < CK / 16; ++k) Wgmma<N>::mma(acc[m], ad + 2 * k, bd + 2 * k);
            }
          }
          wg_commit();
        }
      }
      wg_wait<0>();
      // slot of input row j + kh: one arrival per consumer row, the band's first / last row also for the missing ones
      if (leader)
#pragma unroll
        for (int kh = 0; kh < 3; ++kh)
          mbar_arrive_n(bar_empty + 8 * ((s + j + kh) % nslots), 1 + (j == 0 ? 2 - kh : 0) + (j == n - 1 ? kh : 0));
      // the tile holds this row's residual, or (without one) the previous store has read it
      if (has_res) {
        mbar_wait(tile_full + 8 * wg, (item >> 1) & 1);
      } else {
        if (leader) bulk_wait_read<0>();
        named_bar_sync(1 + wg);
      }
      // conv_epilogue's arithmetic: +bias (+residual) -> ReLU -> fp16, written over the residual it read
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const uint32_t px = m * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
          const uint32_t swz = row_bytes == 128 ? px & 7u : (px >> 1) & 3u;
#pragma unroll
          for (int jj = 0; jj < N / 8; ++jj) {
            const uint32_t ta = tile + px * row_bytes + ((jj ^ swz) << 4) + 2 * c0;
            float a = acc[m][4 * jj + 2 * i] + bias[jj].x, d = acc[m][4 * jj + 2 * i + 1] + bias[jj].y;
            if (has_res) {
              const uint32_t rb = ld_shared_u32(ta);
              const float2 r = __half22float2(*reinterpret_cast<const __half2*>(&rb));
              a += r.x;
              d += r.y;
            }
            if (p.relu) { a = fmaxf(a, 0.f); d = fmaxf(d, 0.f); }
            st_shared_u32(ta, h2_bits(__floats2half2_rn(a, d)));
          }
        }
      fence_proxy_async();                                  // the tile's writes, visible to the TMA store
      named_bar_sync(1 + wg);
      if (leader) {
        tma_store_4d(&tmO, tile, 0, wt * kTileM, h0 + j, b);
        bulk_commit();
        if (has_res) {                                      // the producer stages the next residual once it is read
          bulk_wait_read<0>();
          mbar_arrive(tile_empty + 8 * wg);
        }
      }
    }
    s += n + 2;
  }
  if (leader) bulk_wait<0>();                               // the last stores are done before the CTA exits
}

// Plan of block_row_kernel<32>: both convs' nine taps resident (2 x 18 KB), a ring of input row slots and a ring of
// intermediate row slots (136 pixels of 64 B each, padded to 9 KB), two CTAs per SM (110 KB each).  Four of each:
// conv2 row h holds intermediate rows h - 1 .. h + 1 and input row h (its residual) while conv1 writes intermediate
// row h + 2 from input rows h + 1 .. h + 3, and the fourth input slot lets the producer stage row h + 4 meanwhile.
struct BlockRowPlan {
  static constexpr uint32_t kTapBytes = 32 * 64;
  static constexpr uint32_t kSlotBytes = 9 * 1024;
  static constexpr uint32_t kInTx = (kTileM + kRowHalo) * 64;
  static constexpr uint32_t kInSlots = 4, kMidSlots = 4;
  static constexpr size_t kSmem = 2048 + 2 * 9 * kTapBytes + (kInSlots + kMidSlots) * kSlotBytes;
  static_assert(kInTx <= kSlotBytes && kSmem <= 113 * 1024, "block row plan");
};
constexpr int kStripW = kTileM - 2;                         // output columns per column strip of block_row_kernel

struct BlockParams {
  int H, W, tiles_w, band, bands, num_tiles;
  const float* bias1;
  const float* bias2;
  __half* out;
};


// One stride-1 BasicBlock with 32 channels and an identity shortcut, out = relu(bn2(conv2(relu(bn1(conv1(x))))) + x),
// without the intermediate activation leaving the SM.  Persistent CTAs walk units of one segment x one column strip of
// kStripW output columns [w0, w0 + 126) x a band of output rows [h0, h0 + n), as conv_row_kernel does.
//   - Warp 8 stages input rows h0 - 2 .. h0 + n + 1 once each, as 136-pixel boxes from column w0 - 2.
//   - Warpgroup 0 runs conv1 on intermediate rows h0 - 1 .. h0 + n, 128 pixels each (columns [w0 - 1, w0 + 127)),
//     and its epilogue writes relu(acc + bias) as fp16 into a ring of intermediate row slots, in the 64-B swizzled
//     layout a staged input row has.  Positions outside the image are conv2's zero padding and are written as zero.
//   - Warpgroup 1 runs conv2 on output row h from intermediate rows h - 1 .. h + 1, adds the residual from the staged
//     input row h and stores the first 126 of its 128 pixels.
// The two warpgroups do the same arithmetic per row, so each one's epilogue overlaps the other's MMAs.  Every output
// sums its products in the (tap, 16-channel step) order of conv_tc_kernel, and the intermediate is rounded to fp16 as
// the unfused path stores it, so the result is bit-identical to two conv_forward calls.
// Barriers: input slot "full" (TMA bytes) and "empty" (three conv1 reads + one residual read; conv1 arrives for the
// missing ones at the band's edges, so that no slot waits on a conv2 row that needs a later input row); intermediate slot "full" (128 writer threads) and "empty" (three conv2 reads).
__global__ void __launch_bounds__(kWgThreads, 2)
block_row_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW1,
                 const __grid_constant__ CUtensorMap tmW2, BlockParams p) {
  using P = BlockRowPlan;
  constexpr uint32_t NI = P::kInSlots, NM = P::kMidSlots;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t bar_w = base, in_full = base + 8, in_empty = in_full + 8 * NI;
  const uint32_t mid_full = in_empty + 8 * NI, mid_empty = mid_full + 8 * NM;
  const uint32_t w1 = base + 1024, w2 = w1 + 9 * P::kTapBytes;
  const uint32_t in0 = w2 + 9 * P::kTapBytes, mid0 = in0 + NI * P::kSlotBytes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    mbar_init(bar_w, 1);
    for (uint32_t s = 0; s < NI; ++s) { mbar_init(in_full + 8 * s, 1); mbar_init(in_empty + 8 * s, 4); }
    for (uint32_t s = 0; s < NM; ++s) { mbar_init(mid_full + 8 * s, 128); mbar_init(mid_empty + 8 * s, 3); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == 8) {
    if (lane == 0) {
      prefetch_tensormap(&tmA);
      prefetch_tensormap(&tmW1);
      prefetch_tensormap(&tmW2);
      mbar_expect_tx(bar_w, 18 * P::kTapBytes);
      for (int kh = 0; kh < 3; ++kh) {
        tma_load_3d(&tmW1, bar_w, w1 + 3 * kh * P::kTapBytes, 0, 0, 3 * kh);
        tma_load_3d(&tmW2, bar_w, w2 + 3 * kh * P::kTapBytes, 0, 0, 3 * kh);
      }
      uint32_t s = 0;                                       // input rows staged so far
      for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
        const int wt = u % p.tiles_w, t = u / p.tiles_w;
        const int h0 = (t % p.bands) * p.band, b = t / p.bands;
        const int n = min(p.band, p.H - h0);
        for (int r = 0; r < n + 4; ++r, ++s) {
          const uint32_t slot = s % NI;
          mbar_wait(in_empty + 8 * slot, ((s / NI) & 1) ^ 1);
          mbar_expect_tx(in_full + 8 * slot, P::kInTx);
          tma_load_4d(&tmA, in_full + 8 * slot, in0 + slot * P::kSlotBytes, 0, wt * kStripW - 2, h0 - 2 + r, b);
        }
      }
    }
    return;
  }

  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);  // warp-uniform to the compiler: no wgmma serialisation
  const bool leader = (threadIdx.x & 127) == 0;
  const int c0 = 2 * (lane & 3);
  float2 bias[4];                                           // channels 8 j + c0, c0 + 1 of this thread's fragments
#pragma unroll
  for (int j = 0; j < 4; ++j) bias[j] = __ldg(reinterpret_cast<const float2*>((wg ? p.bias2 : p.bias1) + 8 * j + c0));
  mbar_wait(bar_w, 0);
  uint32_t s = 0, mq = 0;                                   // first input / intermediate row of the current unit
  for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
    const int wt = u % p.tiles_w, t = u / p.tiles_w;
    const int h0 = (t % p.bands) * p.band, b = t / p.bands;
    const int n = min(p.band, p.H - h0);
    const int w0 = wt * kStripW;
    const int rows = wg == 0 ? n + 2 : n;
    for (int j = 0; j < rows; ++j) {
      float acc[2][16];
#pragma unroll
      for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          acc[m][i] = 0.f;
          asm volatile("" : "+f"(acc[m][i]));               // zeroed before the first wg_fence, not sunk past it
        }
      if (wg == 0) {
        // conv1: intermediate row h0 - 1 + j from input rows j .. j + 2 of the unit
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
          const uint32_t q = s + j + kh, slot = q % NI;
          mbar_wait(in_full + 8 * slot, (q / NI) & 1);
          row_taps_c32<32>(acc, in0 + slot * P::kSlotBytes, w1 + 3 * kh * P::kTapBytes);
        }
        // input row k = j + kh: one arrival per conv1 row that reads it (the band's first / last row also for the
        // missing ones), and rows 0, 1, n + 2 and n + 3, which no conv2 row takes as its residual, one more on their
        // last read
        if (leader)
#pragma unroll
          for (int kh = 0; kh < 3; ++kh) {
            const int k = j + kh;
            const bool no_res = (k < 2 || k >= n + 2) && j == min(k, n + 1);
            mbar_arrive_n(in_empty + 8 * ((s + k) % NI),
                          1 + (j == 0 ? 2 - kh : 0) + (j == n + 1 ? kh : 0) + (no_res ? 1 : 0));
          }
        const uint32_t q = mq + j, slot = q % NM, sm = mid0 + slot * P::kSlotBytes;
        mbar_wait(mid_empty + 8 * slot, ((q / NM) & 1) ^ 1);
        const int r = h0 - 1 + j;
        const bool live = r >= 0 && r < p.H;
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int px = m * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i, w = w0 - 1 + px;
            const bool in = live && w >= 0 && w < p.W;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const float a = fmaxf(acc[m][4 * jj + 2 * i] + bias[jj].x, 0.f);
              const float d = fmaxf(acc[m][4 * jj + 2 * i + 1] + bias[jj].y, 0.f);
              const uint32_t v = in ? h2_bits(__floats2half2_rn(a, d)) : 0u;
              st_shared_u32(sm + px * 64u + ((jj ^ ((px >> 1) & 3)) << 4) + 2 * c0, v);
            }
          }
        mbar_arrive(mid_full + 8 * slot);
      } else {
        // conv2: output row h0 + j from intermediate rows j .. j + 2 of the unit, residual = input row j + 2
#pragma unroll
        for (int kh = 0; kh < 3; ++kh) {
          const uint32_t q = mq + j + kh, slot = q % NM;
          mbar_wait(mid_full + 8 * slot, (q / NM) & 1);
          row_taps_c32<32>(acc, mid0 + slot * P::kSlotBytes, w2 + 3 * kh * P::kTapBytes);
        }
        if (leader)
#pragma unroll
          for (int kh = 0; kh < 3; ++kh)
            mbar_arrive_n(mid_empty + 8 * ((mq + j + kh) % NM), 1 + (j == 0 ? 2 - kh : 0) + (j == n - 1 ? kh : 0));
        const uint32_t q = s + j + 2, slot = q % NI, sr = in0 + slot * P::kSlotBytes;
        mbar_wait(in_full + 8 * slot, (q / NI) & 1);
        const size_t row = (size_t)b * p.H + h0 + j;
#pragma unroll
        for (int m = 0; m < 2; ++m)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int px = m * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i, w = w0 + px;
            if (px >= kStripW || w >= p.W) continue;
            const int rp = px + 2;                          // the slot's pixel row of input column w
            __half2* o = reinterpret_cast<__half2*>(p.out + (row * p.W + w) * 32 + c0);
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const uint32_t rb = ld_shared_u32(sr + rp * 64u + ((jj ^ ((rp >> 1) & 3)) << 4) + 2 * c0);
              const float2 rv = __half22float2(*reinterpret_cast<const __half2*>(&rb));
              float a = acc[m][4 * jj + 2 * i] + bias[jj].x, d = acc[m][4 * jj + 2 * i + 1] + bias[jj].y;
              a += rv.x;
              d += rv.y;
              o[4 * jj] = __floats2half2_rn(fmaxf(a, 0.f), fmaxf(d, 0.f));
            }
          }
        asm volatile("bar.sync 1, 128;" ::: "memory");     // every warp has read its residual before the slot is freed
        if (leader) mbar_arrive(in_empty + 8 * slot);
      }
    }
    s += n + 4;
    mq += n + 2;
  }
}

// Plan of conv_chunk_row_kernel<N>: one CTA per SM, a ring of 136-pixel row boxes (one 64-channel chunk each) and a
// ring of (tap, chunk) weight tiles.  A unit is kRows output rows of one 128-pixel column tile.
//   N = 128: two rows, warpgroup r owns row h + r as two m64 halves (128 accumulator registers per thread), so each
//     weight tile feeds four m64n128k16 groups instead of two.  The unit stages four input rows h - 1 .. h + 2 of
//     two chunks; while rows kh and kh + 1 of the unit are read the producer stages row kh + 2, and the next unit's
//     first two rows while the last two are read: 8 box slots and 5 weight slots (218 KB).
//   N = 256 (128 accumulator registers per thread for one m64 half): one row, warpgroup r owns half r; a kernel row
//     keeps all four chunk boxes resident until its last tap, and the box ring holds one more: 5 box slots and 4
//     weight slots (215 KB).
template <int N>
struct ChunkRowPlan {
  static constexpr int kChunks = N / 64;
  static constexpr int kRows = N == 128 ? 2 : 1;
  static constexpr int kHalves = N == 128 ? 2 : 1;         // m64 halves per warpgroup
  static constexpr uint32_t kABytes = (kTileM + kRowHalo) * 128;   // 17 KB, 1024-B multiple
  static constexpr uint32_t kBBytes = N * 128;
  static constexpr uint32_t kASlots = N == 256 ? 5 : 8;
  static constexpr uint32_t kBSlots = N == 256 ? 4 : 5;
  static constexpr size_t kSmem = 2048 + kASlots * kABytes + kBSlots * kBBytes;   // 218 / 215 KB
  // the boxes read at one kh (kRows rows of kChunks) and one more, so that the next kh's first box can be staged
  static_assert(kASlots >= kRows * kChunks + 1 && kASlots <= 8 && kBSlots <= 8, "chunk row ring plan");
  static_assert(kSmem <= 227 * 1024, "chunk row shared memory");
  // ring position of the box of input row r (0 .. kRows + 1 of the unit), chunk cc: the first kRows rows are needed
  // together from kh = 0 on and are staged chunk by chunk, each later row at its kh = r - kRows + 1
  __device__ __forceinline__ static uint32_t box(int r, int cc) {
    return r < kRows ? cc * kRows + r : kRows * kChunks + (r - kRows) * kChunks + cc;
  }
};

template <int N>
__global__ void __launch_bounds__(kWgThreads, 1)
conv_chunk_row_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, ConvParams p) {
  using P = ChunkRowPlan<N>;
  constexpr int CH = P::kChunks, R = P::kRows, KSTEPS = 9 * CH;   // K steps of one unit: (kh, kw, chunk)
  constexpr uint32_t BOXES = (R + 2) * CH;                 // boxes staged per unit
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t full_a = base, empty_a = base + 64, full_b = base + 128, empty_b = base + 192;   // 8 x 8 B each
  const uint32_t ring_a = base + 1024, ring_b = ring_a + P::kASlots * P::kABytes;
  const int warp = threadIdx.x >> 5;

  if (threadIdx.x == 0) {
    for (uint32_t s = 0; s < P::kASlots; ++s) { mbar_init(full_a + 8 * s, 1); mbar_init(empty_a + 8 * s, 2); }
    for (uint32_t s = 0; s < P::kBSlots; ++s) { mbar_init(full_b + 8 * s, 1); mbar_init(empty_b + 8 * s, 2); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // unit u: column tile u % tiles_w (neighbouring CTAs share the halo pixels in L2), then the unit's R output rows,
  // then segment (p.bands units of R rows per column tile; the last one of an odd H_out has one row)
  if (warp == 8) {
    if ((threadIdx.x & 31) == 0) {
      prefetch_tensormap(&tmA);
      prefetch_tensormap(&tmB);
      uint32_t qa = 0, qb = 0;                              // row boxes / weight tiles staged so far
      for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
        const int wt = u % p.tiles_w, t = u / p.tiles_w;
        const int h = (t % p.bands) * R, b = t / p.bands;
        for (int s = 0; s < KSTEPS; ++s) {
          const int cc = s % CH, kw = (s / CH) % 3, kh = s / (3 * CH);
          if (kw == 0)                                      // input rows first read at this kh, chunk cc
            for (int r = kh == 0 ? 0 : kh + R - 1; r < kh + R; ++r) {
              const uint32_t q = qa + P::box(r, cc), slot = q % P::kASlots;
              mbar_wait(empty_a + 8 * slot, ((q / P::kASlots) & 1) ^ 1);
              mbar_expect_tx(full_a + 8 * slot, P::kABytes);
              tma_load_4d(&tmA, full_a + 8 * slot, ring_a + slot * P::kABytes, cc * 64, wt * kTileM - 1, h - 1 + r, b);
            }
          const uint32_t q = qb + s, slot = q % P::kBSlots;
          mbar_wait(empty_b + 8 * slot, ((q / P::kBSlots) & 1) ^ 1);
          mbar_expect_tx(full_b + 8 * slot, P::kBBytes);
          tma_load_3d(&tmB, full_b + 8 * slot, ring_b + slot * P::kBBytes, cc * 64, 0, 3 * kh + kw);
        }
        qa += BOXES;
        qb += KSTEPS;
      }
    }
    return;
  }

  const int wg = __shfl_sync(0xffffffffu, warp >> 2, 0);    // warp-uniform to the compiler: no wgmma serialisation
  const bool leader = (threadIdx.x & 127) == 0;
  const int ro = R == 2 ? wg : 0;                           // this warpgroup's output row of the unit
  // a box holds two arrivals: one per warpgroup for N = 256 (each reads its half), one per reading row for N = 128,
  // whose first and last input rows have one reader, which arrives twice
  uint32_t qa = 0, qb = 0;
  for (int u = blockIdx.x; u < p.num_tiles; u += gridDim.x) {
    const int wt = u % p.tiles_w, t = u / p.tiles_w;
    const int h = (t % p.bands) * R + ro, b = t / p.bands;
    const int w0 = wt * kTileM + (R == 2 ? 0 : wg * 64);    // first output pixel of this warpgroup
    // the epilogue's residual pixels [w0, w0 + 64 kHalves) x N channels (256 lines of 128 B) go to L2 now, so that its
    // loads, issued after the MMAs with no second CTA to hide them, do not wait on HBM
    if (p.residual && h < p.H_out)
#pragma unroll
      for (int l = (threadIdx.x & 127); l < 256; l += 128) {
        const int w = w0 + l / (N / 64);
        if (w < p.W_out)
          asm volatile("prefetch.global.L2 [%0];" ::"l"(p.residual + ((size_t)(b * p.H_out + h) * p.W_out + w) * N +
                                                         (l % (N / 64)) * 64));
      }
    float acc[P::kHalves][N / 2];
#pragma unroll
    for (int m = 0; m < P::kHalves; ++m)
#pragma unroll
      for (int i = 0; i < N / 2; ++i) {
        acc[m][i] = 0.f;
        asm volatile("" : "+f"(acc[m][i]));                 // zeroed before the first wg_fence, not sunk past it
      }
    // the previous K step's slots, released once its wgmma have read them
    uint32_t prev_b = 0, prev_a = 0, prev_frees_a = 0;
    auto release = [&]() {
      if (leader) {
        mbar_arrive(empty_b + 8 * prev_b);
        if (prev_frees_a) mbar_arrive_n(empty_a + 8 * prev_a, prev_frees_a);
      }
    };
    // (kh, kw, chunk, k16): the order of conv_tc_kernel; tap kw reads the row box from pixel row kw on
    for (int s = 0; s < KSTEPS; ++s) {
      const int cc = s % CH, kw = (s / CH) % 3, kh = s / (3 * CH);
      const uint32_t qA = qa + P::box(kh + ro, cc), sa = qA % P::kASlots;
      const uint32_t qB = qb + s, sb = qB % P::kBSlots;
      mbar_wait(full_a + 8 * sa, (qA / P::kASlots) & 1);
      mbar_wait(full_b + 8 * sb, (qB / P::kBSlots) & 1);
      wg_fence();
      const uint64_t bd = wg_desc(ring_b + sb * P::kBBytes, 128);
#pragma unroll
      for (int m = 0; m < P::kHalves; ++m) {
        const uint32_t half = R == 2 ? m : wg;
        const uint64_t ad = wg_desc(ring_a + sa * P::kABytes + (half * 64 + kw) * 128u, 128);
#pragma unroll
        for (int k = 0; k < 4; ++k) Wgmma<N>::mma(acc[m], ad + 2 * k, bd + 2 * k);
      }
      wg_commit();
      wg_wait<1>();
      if (s > 0) release();
      prev_b = sb;
      prev_a = sa;
      // box (kh + ro, cc) is done after tap (kh, 2)
      prev_frees_a = kw == 2 ? (R == 2 && kh == 2 * ro ? 2 : 1) : 0;
    }
    wg_wait<0>();
    release();                                              // the producer stages the next unit during the epilogue
    qa += BOXES;
    qb += KSTEPS;
    if (h < p.H_out) conv_epilogue<N, false, P::kHalves>(acc[0], p, (size_t)b * p.H_out + h, w0);
  }
}

// ------------------------------------------------------------------------------------------------
// SIMT reference conv (same math, CUDA cores) -- A/B check for the tensor-core path
// ------------------------------------------------------------------------------------------------
__global__ void conv_simt_kernel(const __half* __restrict__ in, const __half* __restrict__ wt, ConvParams p) {
  // one thread = one output pixel x 8 output channels
  const int groups = p.C_out / 8;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)p.B * p.H_out * p.W_out * groups;
  if (idx >= total) return;
  const int g = idx % groups;
  size_t pixel = idx / groups;
  const int w = pixel % p.W_out;
  const int h = (pixel / p.W_out) % p.H_out;
  const int b = pixel / ((size_t)p.W_out * p.H_out);
  float acc[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = p.bias[g * 8 + j];
  for (int kh = 0; kh < p.taps_h; ++kh) {
    const int hi = h * p.stride + kh - p.pad;
    if (hi < 0 || hi >= p.H_in) continue;
    for (int kw = 0; kw < p.taps_w; ++kw) {
      const int wi = w * p.stride + kw - p.pad;
      if (wi < 0 || wi >= p.W_in) continue;
      const __half* ip = in + (((size_t)b * p.H_in + hi) * p.W_in + wi) * p.C_in;
      const int tap = kh * p.taps_w + kw;
      for (int ci = 0; ci < p.C_in; ci += 8) {
        uint4 xu = *reinterpret_cast<const uint4*>(ip + ci);
        const __half2* xh = reinterpret_cast<const __half2*>(&xu);
        float x[8];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float2 f = __half22float2(xh[e]);
          x[2 * e] = f.x;
          x[2 * e + 1] = f.y;
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          uint4 wu = *reinterpret_cast<const uint4*>(wt + ((size_t)tap * p.C_out + g * 8 + j) * p.C_in + ci);
          const __half2* wh = reinterpret_cast<const __half2*>(&wu);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            float2 f = __half22float2(wh[e]);
            acc[j] = fmaf(x[2 * e], f.x, acc[j]);
            acc[j] = fmaf(x[2 * e + 1], f.y, acc[j]);
          }
        }
      }
    }
  }
  const size_t o = (((size_t)b * p.H_out + h) * p.W_out + w) * p.C_out + g * 8;
  if (p.residual) {
    uint4 ru = *reinterpret_cast<const uint4*>(p.residual + o);
    const __half2* rh = reinterpret_cast<const __half2*>(&ru);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      float2 f = __half22float2(rh[e]);
      acc[2 * e] += f.x;
      acc[2 * e + 1] += f.y;
    }
  }
  uint4 ou;
  __half2* oh = reinterpret_cast<__half2*>(&ou);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float a = acc[2 * e], c = acc[2 * e + 1];
    if (p.relu) { a = fmaxf(a, 0.f); c = fmaxf(c, 0.f); }
    oh[e] = __floats2half2_rn(a, c);
  }
  *reinterpret_cast<uint4*>(p.out + o) = ou;
}

// ------------------------------------------------------------------------------------------------
// first conv: 1 -> 32 channels on the (mean-centred) fbank, fp32 in, fp16 NHWC out
//   x[b][h=f][w=t] = fbank[b][t][f] - mean[b][f]   (resnet.py:411-413 permute + wespeaker/__init__.py:138)
// ------------------------------------------------------------------------------------------------
// block = (b, tile of 128 of the T0 time frames): the (130 x 80) fbank tile is staged in shared memory with coalesced reads,
// then thread = time frame walks the 80 frequency rows so that every warp store is 32 x 64 B contiguous.
constexpr int kC1Tile = 128;
__global__ void __launch_bounds__(kC1Tile) conv1_kernel(const float* __restrict__ fbank, const float* __restrict__ fmean,
                             const int* __restrict__ frame0, const float* __restrict__ w /*[32][9] folded*/, const float* __restrict__ bias /*[32]*/,
                             __half* __restrict__ out, int T0) {
  __shared__ __align__(16) float sw[9 * 32];               // [tap][channel]: one LDS.128 = 4 channels of a tap
  __shared__ __align__(16) float sb[32];
  __shared__ float sx[(kC1Tile + 2) * (kMel + 1)];        // [t][f], +1 padding against bank conflicts
  const int b = blockIdx.x, t0 = blockIdx.y * kC1Tile;    // segments on x: a sub-batch of 1-frame ones holds 263 472
  const size_t r0 = frame0 ? (size_t)frame0[b] : (size_t)b * T0;             // first fbank row of this segment
  for (int i = threadIdx.x; i < 288; i += blockDim.x) sw[(i % 9) * 32 + i / 9] = w[i];
  if (threadIdx.x < 32) sb[threadIdx.x] = bias[threadIdx.x];
  for (int i = threadIdx.x; i < (kC1Tile + 2) * kMel; i += blockDim.x) {
    const int tt = i / kMel, f = i - tt * kMel;
    const int t = t0 - 1 + tt;
    float v = 0.f;
    if (t >= 0 && t < T0) v = fbank[(r0 + t) * kMel + f] - fmean[(size_t)b * kMel + f];
    sx[tt * (kMel + 1) + f] = v;
  }
  __syncthreads();
  const int t = t0 + threadIdx.x;
  if (t >= T0) return;
  const float* col = sx + threadIdx.x * (kMel + 1);        // rows tt = threadIdx.x + {0,1,2} <-> t-1, t, t+1
  for (int h = 0; h < kMel; ++h) {
    // re-read the weights from shared memory in every row: hoisted out of the loop, 288 weights + 32 biases do not
    // fit in the register file and spill to local memory
    asm volatile("" ::: "memory");
    float x[9];
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int hh = h + kh - 1;
      const bool ok = hh >= 0 && hh < kMel;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) x[kh * 3 + kw] = ok ? col[kw * (kMel + 1) + hh] : 0.f;
    }
    // channel pairs, weights as 16-byte broadcast loads (a scalar version is LDS-bound: one shared-memory load per
    // FMA); the same fma order per channel as a scalar loop, so the result is bit-identical
    f32x2_t acc2[16];
    const ulonglong2* sb2 = reinterpret_cast<const ulonglong2*>(sb);
#pragma unroll
    for (int q = 0; q < 8; ++q) { const ulonglong2 bb = sb2[q]; acc2[2 * q] = bb.x; acc2[2 * q + 1] = bb.y; }
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const f32x2_t xk = pack2(x[k], x[k]);
      const ulonglong2* wk = reinterpret_cast<const ulonglong2*>(sw + k * 32);
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const ulonglong2 w4 = wk[q];
        ffma2(acc2[2 * q], xk, w4.x);
        ffma2(acc2[2 * q + 1], xk, w4.y);
      }
    }
    __half2 o[16];
#pragma unroll
    for (int c = 0; c < 16; ++c) {
      float a0, a1;
      unpack2(acc2[c], a0, a1);
      o[c] = __floats2half2_rn(fmaxf(a0, 0.f), fmaxf(a1, 0.f));
    }
    uint4* op = reinterpret_cast<uint4*>(out + (((size_t)b * kMel + h) * T0 + t) * 32);
    const uint4* src = reinterpret_cast<const uint4*>(o);
#pragma unroll
    for (int i = 0; i < 4; ++i) op[i] = src[i];
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(ptr);
  }
  return fn;
}

int encode_f16_map(CUtensorMap* tm, int rank, const void* ptr, const cuuint64_t* dims, const cuuint64_t* strides,
                   const cuuint32_t* box, const cuuint32_t* estr, CUtensorMapSwizzle swizzle, const char* what) {
  PFN_encodeTiled enc = get_encode();
  B200_CHECK(enc != nullptr, B200_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
  const cuuint32_t ones[5] = {1, 1, 1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(ptr), dims, strides, box,
                   estr ? estr : ones, CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_CHECK(r == CUDA_SUCCESS, B200_ERR_CUDA, "cuTensorMapEncodeTiled(%s) failed: %d", what, (int)r);
  return B200_OK;
}

int conv_forward(const ConvLayer& L, const __half* in, const __half* residual, __half* out, int B, int H_in, int W_in,
                 int relu, int impl, int num_sms, cudaStream_t stream) {
  ConvParams p{};
  p.B = B; p.H_in = H_in; p.W_in = W_in; p.C_in = L.C_in; p.C_out = L.C_out;
  p.taps_h = L.ksize; p.taps_w = L.ksize; p.stride = L.stride; p.pad = L.ksize / 2;
  p.H_out = (H_in + 2 * p.pad - L.ksize) / L.stride + 1;
  p.W_out = (W_in + 2 * p.pad - L.ksize) / L.stride + 1;
  p.relu = relu; p.bias = L.bias; p.residual = residual; p.out = out;
  p.Ck = (L.C_in >= 64) ? 64 : 32;
  p.swizzle = (p.Ck == 64) ? 128 : 64;
  p.tiles_w = ceil_div(p.W_out, kTileM);
  p.num_tiles = B * p.H_out * p.tiles_w;
  // C_out 32 / 64 / 128 with either channel chunk; 256 and, as 256-wide column tiles (grid.y), 512 / 768 / 1024
  // with Ck = 64
  B200_CHECK(L.C_in % p.Ck == 0 && (L.C_out == 32 || L.C_out == 64 || L.C_out == 128 ||
                                    (L.C_out % 256 == 0 && L.C_out <= 1024 && p.Ck == 64)),
             B200_ERR_STATE, "conv %d -> %d channels unsupported", L.C_in, L.C_out);
  const int n_tile = std::min(L.C_out, 256);               // output channels per CTA of conv_tc_kernel
  B200_CHECK(impl >= 0 && impl <= 2, B200_ERR_INVALID,
             "conv_impl %d unknown (0 = CUDA cores, 1 = tensor cores, 2 = tensor cores, one weight tap per stage)", impl);

  if (impl == 0) {
    const size_t total = (size_t)B * p.H_out * p.W_out * (L.C_out / 8);
    return launch(conv_simt_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, in, L.w, p);
  }

  // conv_row_kernel for the stride-1 3x3 convs with one channel chunk and C_in = C_out; impl 2 keeps every conv on
  // conv_tc_kernel, the bit-exact reference of the row kernel
  const bool rows = impl == 1 && L.ksize == 3 && L.stride == 1 && L.C_in == p.Ck && L.C_out == L.C_in;
  // conv_chunk_row_kernel for those with C_in = C_out = 128 or 256 (layers 3 and 4)
  const bool chunk_rows =
      impl == 1 && L.ksize == 3 && L.stride == 1 && L.C_out == L.C_in && (L.C_out == 128 || L.C_out == 256);
  p.a_rows = rows || chunk_rows ? kTileM + kRowHalo : kTileM;
  p.a_tx = p.a_rows * p.Ck * 2;
  p.a_bytes = (p.a_tx + 1023u) & ~1023u;
  size_t smem;
  int ctas = 0;
  if (rows) {
    // RowPlan: resident weights, two epilogue tiles and a ring of row slots; two CTAs per SM for C_out = 32, one for 64
    const int per_sm = L.C_out == 32 ? RowPlan<32>::kCtasPerSm : RowPlan<64>::kCtasPerSm;
    smem = L.C_out == 32 ? RowPlan<32>::kSmem : RowPlan<64>::kSmem;
    // full-height bands while the column strips fill every CTA (a 264-segment sub-batch: 2112 / 1056 strips for
    // layers 1 / 2), else shorter bands so that small batches still reach every SM; each band re-stages two halo rows
    ctas = per_sm * num_sms;
    const int strips = B * p.tiles_w;
    const int nbands = std::min(p.H_out, ceil_div(ctas, strips));
    p.band = ceil_div(p.H_out, nbands);
    p.bands = ceil_div(p.H_out, p.band);
    p.num_tiles = strips * p.bands;
  } else if (chunk_rows) {
    // one persistent CTA per SM over units of ChunkRowPlan::kRows output rows of a column tile
    p.band = L.C_out == 256 ? ChunkRowPlan<256>::kRows : ChunkRowPlan<128>::kRows;
    p.bands = ceil_div(p.H_out, p.band);
    p.num_tiles = B * p.bands * p.tiles_w;
    smem = L.C_out == 256 ? ChunkRowPlan<256>::kSmem : ChunkRowPlan<128>::kSmem;
    ctas = num_sms;
  } else {
    p.b_bytes = (uint32_t)(n_tile * p.Ck * 2);
    // C_out = 256 needs 128 accumulator registers per thread: one CTA per SM with 4 deep stages; the narrower layers
    // run two CTAs per SM (registers allow it) on half the shared memory each
    const uint32_t budget = n_tile == 256 ? 200u * 1024 : 100u * 1024;
    p.nstages = std::min(budget / (p.a_bytes + p.b_bytes), 8u);
    B200_CHECK(p.nstages >= 2, B200_ERR_STATE, "conv %d -> %d: shared memory plan too shallow", L.C_in, L.C_out);
    smem = 1024 + 1024 + (size_t)p.nstages * (p.a_bytes + p.b_bytes);
  }
  const CUtensorMapSwizzle swz = p.swizzle == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
  CUtensorMap tmA, tmB;
  int rc;
  {
    const cuuint64_t dims[4] = {(cuuint64_t)L.C_in, (cuuint64_t)W_in, (cuuint64_t)H_in, (cuuint64_t)B};
    const cuuint64_t strides[3] = {(cuuint64_t)L.C_in * 2, (cuuint64_t)W_in * L.C_in * 2,
                                   (cuuint64_t)H_in * W_in * L.C_in * 2};
    const cuuint32_t box[4] = {(cuuint32_t)p.Ck, (cuuint32_t)(p.a_rows * L.stride), 1, 1};
    const cuuint32_t estr[4] = {1, (cuuint32_t)L.stride, 1, 1};
    if ((rc = encode_f16_map(&tmA, 4, in, dims, strides, box, estr, swz, "A"))) return rc;
  }
  {
    // conv_row_kernel loads the nine taps as three boxes of three
    const cuuint64_t dims[3] = {(cuuint64_t)L.C_in, (cuuint64_t)L.C_out, (cuuint64_t)(L.ksize * L.ksize)};
    const cuuint64_t strides[2] = {(cuuint64_t)L.C_in * 2, (cuuint64_t)L.C_out * L.C_in * 2};
    const cuuint32_t box[3] = {(cuuint32_t)p.Ck, (cuuint32_t)n_tile, rows ? 3u : 1u};
    if ((rc = encode_f16_map(&tmB, 3, L.w, dims, strides, box, nullptr, swz, "B"))) return rc;
  }
  if (rows) {
    // the residual and the output, as 128-pixel boxes of the output's shape: the row kernel's epilogue tiles
    CUtensorMap tmR{}, tmO;
    const cuuint64_t dims[4] = {(cuuint64_t)L.C_out, (cuuint64_t)p.W_out, (cuuint64_t)p.H_out, (cuuint64_t)B};
    const cuuint64_t strides[3] = {(cuuint64_t)L.C_out * 2, (cuuint64_t)p.W_out * L.C_out * 2,
                                   (cuuint64_t)p.H_out * p.W_out * L.C_out * 2};
    const cuuint32_t box[4] = {(cuuint32_t)L.C_out, (cuuint32_t)kTileM, 1, 1};
    if (residual && (rc = encode_f16_map(&tmR, 4, residual, dims, strides, box, nullptr, swz, "residual"))) return rc;
    if ((rc = encode_f16_map(&tmO, 4, out, dims, strides, box, nullptr, swz, "out"))) return rc;
    auto kernel = p.Ck == 32 ? conv_row_kernel<32, 32> : conv_row_kernel<64, 64>;
    return launch(kernel, (unsigned)std::min(p.num_tiles, ctas), kWgThreads, smem, stream, tmA, tmB, tmR, tmO, p);
  }
  const dim3 grid((unsigned)(ctas ? std::min(p.num_tiles, ctas) : p.num_tiles), (unsigned)(L.C_out / n_tile));
  auto run = [&](auto kernel) { return launch(kernel, grid, kWgThreads, smem, stream, tmA, tmB, p); };
  if (chunk_rows) return L.C_out == 256 ? run(conv_chunk_row_kernel<256>) : run(conv_chunk_row_kernel<128>);
  if (p.Ck == 32) {
    switch (L.C_out) {
      case 32: return run(conv_tc_kernel<32, 32>);
      case 64: return run(conv_tc_kernel<64, 32>);
      default: return run(conv_tc_kernel<128, 32>);   // bottleneck layer 1: conv3 / shortcut 32 -> 128
    }
  }
  switch (L.C_out) {
    case 32: return run(conv_tc_kernel<32, 64>);       // bottleneck layer 1: conv1 128 -> 32
    case 64: return run(conv_tc_kernel<64, 64>);
    case 128: return run(conv_tc_kernel<128, 64>);
    case 256: return run(conv_tc_kernel<256, 64>);
    default: return run(conv_tc_kernel<256, 64, true>);
  }
}

bool block_fused(const BlockWeights& Bw, int impl) {
  return impl == 1 && !Bw.has_shortcut && Bw.conv1.stride == 1 && Bw.conv1.ksize == 3 && Bw.conv2.ksize == 3 &&
         Bw.conv1.C_in == 32 && Bw.conv1.C_out == 32 && Bw.conv2.C_in == 32 && Bw.conv2.C_out == 32;
}

int block_forward(const BlockWeights& Bw, const __half* in, __half* out, int B, int H, int W, int num_sms,
                  cudaStream_t stream) {
  B200_CHECK(block_fused(Bw, 1), B200_ERR_STATE, "block %d -> %d (stride %d) has no fused kernel", Bw.conv1.C_in,
             Bw.conv1.C_out, Bw.conv1.stride);
  B200_CHECK(in != out, B200_ERR_INVALID, "fused block: output must not alias the input");
  BlockParams p{};
  p.H = H; p.W = W; p.bias1 = Bw.conv1.bias; p.bias2 = Bw.conv2.bias; p.out = out;
  p.tiles_w = ceil_div(W, kStripW);
  // bands as for conv_row_kernel: full height while the column strips fill every CTA, else shorter ones; each band
  // re-stages four input rows and re-computes two intermediate rows
  const int ctas = 2 * num_sms;
  const int strips = B * p.tiles_w;
  const int nbands = std::min(H, ceil_div(ctas, strips));
  p.band = ceil_div(H, nbands);
  p.bands = ceil_div(H, p.band);
  p.num_tiles = strips * p.bands;
  CUtensorMap tmA, tmW1, tmW2;
  int rc;
  {
    const cuuint64_t dims[4] = {32, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    const cuuint64_t strides[3] = {64, (cuuint64_t)W * 64, (cuuint64_t)H * W * 64};
    const cuuint32_t box[4] = {32, kTileM + kRowHalo, 1, 1};
    if ((rc = encode_f16_map(&tmA, 4, in, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_64B, "block A"))) return rc;
  }
  {
    const cuuint64_t dims[3] = {32, 32, 9};
    const cuuint64_t strides[2] = {64, 32 * 64};
    const cuuint32_t box[3] = {32, 32, 3};
    if ((rc = encode_f16_map(&tmW1, 3, Bw.conv1.w, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_64B, "block W1")))
      return rc;
    if ((rc = encode_f16_map(&tmW2, 3, Bw.conv2.w, dims, strides, box, nullptr, CU_TENSOR_MAP_SWIZZLE_64B, "block W2")))
      return rc;
  }
  const size_t smem = BlockRowPlan::kSmem;
  return launch(block_row_kernel, (unsigned)std::min(p.num_tiles, ctas), kWgThreads, smem, stream, tmA, tmW1, tmW2, p);
}

int conv1_forward(const float* fbank, const float* fmean, const int* frame0, const float* w, const float* bias,
                  __half* out, int B, int T0, cudaStream_t stream) {
  dim3 grid(B, ceil_div(T0, kC1Tile));
  return launch(conv1_kernel, grid, kC1Tile, 0, stream, fbank, fmean, frame0, w, bias, out, T0);
}

}  // namespace b200
