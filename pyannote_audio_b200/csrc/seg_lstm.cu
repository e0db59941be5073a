// BiLSTM stack + linear head + classifier (powerset log-softmax / argmax, or sigmoid) for PyanNet (fp32 SIMT).
//
// Reference: /root/reference/src/pyannote/audio/models/segmentation/PyanNet.py:223-240
//   nn.LSTM(60, 128, num_layers=4, bidirectional, batch_first) -> 2x leaky_relu(Linear) -> Linear(128,7)
//   -> LogSoftmax (core/model.py:284-300) ; Powerset hard decision = argmax (utils/powerset.py:135-140).
//
// Per layer: (1) input projection for both directions as one fp32 GEMM (sgemm.cu) into Gx[b][t][1024] with column
// order (dir, unit, gate) and both biases folded; (2) the recurrence as a persistent kernel on a 2-CTA cluster:
// each CTA keeps the W_hh slice of 64 hidden units (all 4 gates, 128 KB fp32) resident in shared memory for the
// whole T-step window, computes its gates for a tile of NBT sequences, updates c/h in registers and publishes
// its h slice into BOTH CTAs' shared memory (DSMEM), one cluster barrier per step.
#include "common.cuh"
#include "seg.cuh"
#include <cooperative_groups.h>
#include <array>
#include <utility>

namespace cg = cooperative_groups;

namespace b200 {

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// RB = batch rows per thread (8, 4 or 2); tile of NBT = 8*RB sequences per cluster.
// thread (tx = lane = unit pair, ty = warp = row group).  Columns owned by a thread: plane p in {0,1} -> hidden
// unit 64*rank + 2*tx + p, gates i,f,g,o at smem columns p*128 + tx*4 + gate.
template <int RB>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(256, 1)
lstm_rec_kernel(const float* __restrict__ Gx /*[NB][T][1024]*/, const float* __restrict__ Whh /*[2][2][128][256]*/,
                float* __restrict__ Y /*[NB][T][256] or null*/, __half* __restrict__ Yh, __half* __restrict__ Yl,
                int NB, int T, int ntiles) {
  constexpr int NBT = 8 * RB;
  extern __shared__ float sm[];
  float* Ws = sm;                         // [128][256]
  float* hb = sm + 128 * 256;             // [2][128][NBT]
  cg::cluster_group cluster = cg::this_cluster();
  const int rank = (int)cluster.block_rank();
  const int cid = blockIdx.x >> 1;        // cluster id -> (tile, dir)
  const int dir = cid / ntiles;
  const int tile = cid - dir * ntiles;
  const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;
  float* hb_peer = cluster.map_shared_rank(hb, rank ^ 1);

  {
    const float4* src = reinterpret_cast<const float4*>(Whh + ((size_t)(dir * 2 + rank) * 128) * 256);
    float4* dst = reinterpret_cast<float4*>(Ws);
    for (int i = tid; i < 128 * 256 / 4; i += 256) dst[i] = src[i];
    for (int i = tid; i < 2 * 128 * NBT; i += 256) hb[i] = 0.f;
  }
  float c[RB][2];
#pragma unroll
  for (int r = 0; r < RB; ++r) { c[r][0] = 0.f; c[r][1] = 0.f; }

  const int b0 = tile * NBT + ty * RB;
  const int gcol = dir * 512 + rank * 256 + tx * 8;
  float gx[RB][8];
  auto load_gx = [&](int t, float (&dst)[RB][8]) {
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      const int b = b0 + r;
      if (b < NB) {
        const float4* p = reinterpret_cast<const float4*>(Gx + ((size_t)b * T + t) * 1024 + gcol);
        const float4 u = __ldg(p), v = __ldg(p + 1);
        dst[r][0] = u.x; dst[r][1] = u.y; dst[r][2] = u.z; dst[r][3] = u.w;
        dst[r][4] = v.x; dst[r][5] = v.y; dst[r][6] = v.z; dst[r][7] = v.w;
      } else {
#pragma unroll
        for (int j = 0; j < 8; ++j) dst[r][j] = 0.f;
      }
    }
  };
  load_gx(dir ? T - 1 : 0, gx);
  cluster.sync();

  for (int step = 0; step < T; ++step) {
    const int t = dir ? (T - 1 - step) : step;
    const float* hcur = hb + (step & 1) * 128 * NBT;
    float* hnext = hb + ((step + 1) & 1) * 128 * NBT;
    float* hnext_peer = hb_peer + ((step + 1) & 1) * 128 * NBT;
    float acc[RB][8];
#pragma unroll
    for (int r = 0; r < RB; ++r)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[r][j] = gx[r][j];
    if (step + 1 < T) load_gx(dir ? t - 1 : t + 1, gx);      // prefetch next step's input projection

#pragma unroll 4
    for (int k = 0; k < 128; ++k) {
      const float4 w0 = *reinterpret_cast<const float4*>(Ws + k * 256 + tx * 4);
      const float4 w1 = *reinterpret_cast<const float4*>(Ws + k * 256 + 128 + tx * 4);
      float hv[RB];
      if (RB == 8) {
        const float4 h0 = *reinterpret_cast<const float4*>(hcur + k * NBT + ty * RB);
        const float4 h1 = *reinterpret_cast<const float4*>(hcur + k * NBT + ty * RB + 4);
        hv[0] = h0.x; hv[1] = h0.y; hv[2] = h0.z; hv[3] = h0.w;
        hv[4 % RB] = h1.x; hv[5 % RB] = h1.y; hv[6 % RB] = h1.z; hv[7 % RB] = h1.w;
      } else if (RB == 4) {
        const float4 h0 = *reinterpret_cast<const float4*>(hcur + k * NBT + ty * RB);
        hv[0] = h0.x; hv[1] = h0.y; hv[2 % RB] = h0.z; hv[3 % RB] = h0.w;
      } else {
        const float2 h0 = *reinterpret_cast<const float2*>(hcur + k * NBT + ty * RB);
        hv[0] = h0.x; hv[1] = h0.y;
      }
      const float wv[8] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int r = 0; r < RB; ++r)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[r][j] = fmaf(hv[r], wv[j], acc[r][j]);
    }

    // gates (PyTorch order i, f, g, o), cell update, publish h
#pragma unroll
    for (int r = 0; r < RB; ++r) {
      float hn[2];
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const float ig = sigmoidf_(acc[r][p * 4 + 0]);
        const float fg = sigmoidf_(acc[r][p * 4 + 1]);
        const float gg = tanhf(acc[r][p * 4 + 2]);
        const float og = sigmoidf_(acc[r][p * 4 + 3]);
        c[r][p] = fmaf(fg, c[r][p], ig * gg);
        hn[p] = og * tanhf(c[r][p]);
        const int unit = rank * 64 + 2 * tx + p;
        hnext[unit * NBT + ty * RB + r] = hn[p];
        hnext_peer[unit * NBT + ty * RB + r] = hn[p];
      }
      const int b = b0 + r;
      if (b < NB) {
        const size_t o = ((size_t)b * T + t) * 256 + dir * 128 + rank * 64 + 2 * tx;
        if (Y) *reinterpret_cast<float2*>(Y + o) = make_float2(hn[0], hn[1]);
        if (Yh) {   // fp16 (hi, lo) split consumed by the tensor-core GEMM of the next layer
          const __half h0 = __float2half_rn(hn[0]), h1 = __float2half_rn(hn[1]);
          *reinterpret_cast<__half2*>(Yh + o) = __halves2half2(h0, h1);
          *reinterpret_cast<__half2*>(Yl + o) = __floats2half2_rn(hn[0] - __half2float(h0), hn[1] - __half2float(h1));
        }
      }
    }
    cluster.sync();
  }
}

// ---- classifier 128 -> K (one warp per frame) -------------------------------------------------------------
// kSegLogSoftmax: log-softmax + argmax -> cls [M] u8 (+ logp [M][K]); kSegSigmoid: sigmoid -> scores [M][K] and/or
// the per-frame maximum over the K scores [M] (VoiceActivityDetection's pre_aggregation_hook, np.max(axis=-1)).
// K is a template parameter so that the logits stay in registers; K = 7 with log-softmax is the community-1 head.
template <int K, int ACT>
__global__ void __launch_bounds__(256) classifier_kernel(const float* __restrict__ Z /*[M][128]*/,
                                                         const float* __restrict__ Wc /*[K][128]*/,
                                                         const float* __restrict__ bc, unsigned char* __restrict__ cls,
                                                         float* __restrict__ logp, float* __restrict__ scores,
                                                         float* __restrict__ max_scores, int M) {
  __shared__ float sw[K * 128];
  __shared__ float sb[K < 8 ? 8 : K];
  for (int i = threadIdx.x; i < K * 128; i += blockDim.x) sw[i] = Wc[i];
  if (threadIdx.x < K) sb[threadIdx.x] = bc[threadIdx.x];
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int row = blockIdx.x * 8 + warp;
  if (row >= M) return;
  const float4 z = *reinterpret_cast<const float4*>(Z + (size_t)row * 128 + lane * 4);
  float v[K];
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float4 w = *reinterpret_cast<const float4*>(sw + k * 128 + lane * 4);
    float s = z.x * w.x;
    s = fmaf(z.y, w.y, s);
    s = fmaf(z.z, w.z, s);
    s = fmaf(z.w, w.w, s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    v[k] = s + sb[k];
  }
  if (lane != 0) return;
  if (ACT == kSegSigmoid) {
    float mx = 0.f;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const float p = sigmoidf_(v[k]);
      if (scores) scores[(size_t)row * K + k] = p;
      mx = k == 0 ? p : fmaxf(mx, p);
    }
    if (max_scores) max_scores[row] = mx;
    return;
  }
  float mx = v[0];
#pragma unroll
  for (int k = 1; k < K; ++k) mx = fmaxf(mx, v[k]);
  float se = 0.f;
#pragma unroll
  for (int k = 0; k < K; ++k) se += expf(v[k] - mx);
  const float lse = logf(se);
  int best = 0;
  float bv = 0.f;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float lp = (v[k] - mx) - lse;
    if (logp) logp[(size_t)row * K + k] = lp;
    if (k == 0 || lp > bv) { bv = lp; best = k; }     // first maximum wins, like torch.argmax
  }
  cls[row] = (unsigned char)best;
}

typedef void (*ClassifierFn)(const float*, const float*, const float*, unsigned char*, float*, float*, float*, int);
template <int ACT, int... I>
static std::array<ClassifierFn, sizeof...(I)> classifier_table(std::integer_sequence<int, I...>) {
  return {{&classifier_kernel<I + 1, ACT>...}};
}
static const auto kLogSoftmaxHeads = classifier_table<kSegLogSoftmax>(std::make_integer_sequence<int, kSegMaxClasses>());
static const auto kSigmoidHeads = classifier_table<kSegSigmoid>(std::make_integer_sequence<int, kSegMaxClasses>());

// ---- host ------------------------------------------------------------------------------------------
struct LstmWs {
  float *Gx, *Ya, *Yb, *Z1, *Z2;
  __half *Xh, *Xl, *Yah, *Yal, *Ybh, *Ybl, *Z1h, *Z1l;
};
static size_t carve_lstm(int NB, int T, int k0, void* base, LstmWs* w) {
  Workspace ws(base, 256);
  LstmWs t;
  const size_t M = (size_t)NB * T;
  t.Gx = (float*)ws.take(M * 1024 * sizeof(float));
  t.Ya = (float*)ws.take(M * 256 * sizeof(float));
  t.Yb = (float*)ws.take(M * 256 * sizeof(float));
  t.Z1 = (float*)ws.take(M * 128 * sizeof(float));
  t.Z2 = (float*)ws.take(M * 128 * sizeof(float));
  t.Xh = (__half*)ws.take(M * k0 * sizeof(__half));
  t.Xl = (__half*)ws.take(M * k0 * sizeof(__half));
  t.Yah = (__half*)ws.take(M * 256 * sizeof(__half));
  t.Yal = (__half*)ws.take(M * 256 * sizeof(__half));
  t.Ybh = (__half*)ws.take(M * 256 * sizeof(__half));
  t.Ybl = (__half*)ws.take(M * 256 * sizeof(__half));
  t.Z1h = (__half*)ws.take(M * 128 * sizeof(__half));
  t.Z1l = (__half*)ws.take(M * 128 * sizeof(__half));
  if (w) *w = t;
  return ws.bytes();
}
size_t lstm_workspace_bytes(int NB, int T, int k0) { return carve_lstm(NB, T, k0, nullptr, nullptr); }

template <int RB>
static int launch_rec(const float* Gx, const float* Whh, float* Y, __half* Yh, __half* Yl, int NB, int T,
                      cudaStream_t stream) {
  constexpr int NBT = 8 * RB;
  const int ntiles = ceil_div(NB, NBT);
  const size_t smem = (128 * 256 + 2 * 128 * NBT) * sizeof(float);
  return launch(lstm_rec_kernel<RB>, 2 * 2 * ntiles, 256, smem, stream, Gx, Whh, Y, Yh, Yl, NB, T, ntiles);
}

int lstm_head_forward(const SegWeights& W, const float* x0, int NB, int T, void* ws, const SegHeadOut& out,
                      int num_sms, int gemm_impl, int rec_impl, cudaStream_t stream, const SegCapture* cap) {
  LstmWs w;
  carve_lstm(NB, T, W.k_in[0], ws, &w);
  const int M = NB * T;          // rows of every GEMM (< 2^31); element offsets M * 1024 are formed in size_t
  const SegCapture none{};
  const SegCapture& c = cap ? *cap : none;
  const size_t f32 = sizeof(float) * M, f16 = sizeof(__half) * M;
  const int clusters = num_sms / 2;
  const bool tc = gemm_impl != 0;
  int rc;
  const float* in = x0;
  const __half *in_h = w.Xh, *in_l = w.Xl;
  if (tc && (rc = split_f16(x0, w.Xh, w.Xl, (size_t)M * W.k_in[0], stream))) return rc;
  float* outs[2] = {w.Ya, w.Yb};
  __half* outs_h[2] = {w.Yah, w.Ybh};
  __half* outs_l[2] = {w.Yal, w.Ybl};
  for (int l = 0; l < W.lstm_layers; ++l) {
    if (tc)
      rc = gemm_tc_split(in_h, in_l, W.k_in[l], W.w_ih_hi[l], W.w_ih_lo[l], W.k_in[l], w.Gx, 1024, nullptr, nullptr, 0,
                         W.b_g[l], M, 1024, W.k_in[l], 0, num_sms, stream);
    else
      rc = sgemm_nt(in, W.k_in[l], W.w_ih[l], W.k_in[l], w.Gx, 1024, W.b_g[l], M, 1024, W.k_in[l], 0, stream);
    if (rc) return rc;
    if ((rc = capture(c.gx[l], w.Gx, f32 * 1024, stream))) return rc;
    if (tc && rec_impl != 0) {   // tensor-core recurrence (seg_lstm_wg.cu)
      if ((rc = lstm_rec_wg(w.Gx, W.w_hh_hi[l], W.w_hh_lo[l], outs_h[l & 1], outs_l[l & 1], NB, T, rec_impl, stream)))
        return rc;
      in_h = outs_h[l & 1]; in_l = outs_l[l & 1];
      if ((rc = capture(c.y_hi[l], in_h, f16 * 256, stream)) || (rc = capture(c.y_lo[l], in_l, f16 * 256, stream)))
        return rc;
      continue;
    }
    float* y = tc ? nullptr : outs[l & 1];
    __half* yh = tc ? outs_h[l & 1] : nullptr;
    __half* yl = tc ? outs_l[l & 1] : nullptr;
    // largest batch tile that still fills the machine with 2-CTA clusters
    if (2 * ceil_div(NB, 64) >= clusters) rc = launch_rec<8>(w.Gx, W.w_hh[l], y, yh, yl, NB, T, stream);
    else if (2 * ceil_div(NB, 32) >= clusters) rc = launch_rec<4>(w.Gx, W.w_hh[l], y, yh, yl, NB, T, stream);
    else rc = launch_rec<2>(w.Gx, W.w_hh[l], y, yh, yl, NB, T, stream);
    if (rc) return rc;
    in = y; in_h = yh; in_l = yl;
    if (tc && ((rc = capture(c.y_hi[l], yh, f16 * 256, stream)) || (rc = capture(c.y_lo[l], yl, f16 * 256, stream))))
      return rc;
    if (!tc && (rc = capture(c.y[l], y, f32 * 256, stream))) return rc;
  }
  if (tc) {
    rc = gemm_tc_split(in_h, in_l, 256, W.lin_w_hi[0], W.lin_w_lo[0], 256, nullptr, 0, w.Z1h, w.Z1l, 128, W.lin_b[0], M,
                       128, 256, 1, num_sms, stream);
    if (rc) return rc;
    if ((rc = capture(c.z1_hi, w.Z1h, f16 * 128, stream)) || (rc = capture(c.z1_lo, w.Z1l, f16 * 128, stream)))
      return rc;
    rc = gemm_tc_split(w.Z1h, w.Z1l, 128, W.lin_w_hi[1], W.lin_w_lo[1], 128, w.Z2, 128, nullptr, nullptr, 0,
                       W.lin_b[1], M, 128, 128, 1, num_sms, stream);
    if (rc) return rc;
  } else {
    rc = sgemm_nt(in, 256, W.lin_w[0], 256, w.Z1, 128, W.lin_b[0], M, 128, 256, 1, stream);
    if (rc) return rc;
    if ((rc = capture(c.z1, w.Z1, f32 * 128, stream))) return rc;
    rc = sgemm_nt(w.Z1, 128, W.lin_w[1], 128, w.Z2, 128, W.lin_b[1], M, 128, 128, 1, stream);
    if (rc) return rc;
  }
  if ((rc = capture(c.z2, w.Z2, f32 * 128, stream))) return rc;
  const ClassifierFn head = (W.activation == kSegSigmoid ? kSigmoidHeads : kLogSoftmaxHeads)[W.num_classes - 1];
  return launch(head, ceil_div(M, 8), 256, 0, stream, w.Z2, W.cls_w, W.cls_b, out.cls, out.logp, out.scores,
                out.max_scores, M);
}

}  // namespace b200
