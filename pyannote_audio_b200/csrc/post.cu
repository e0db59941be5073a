// Integer post-processing of the segmentation: powerset -> multilabel, speaker counting (overlap-add),
// clustered reconstruction + top-count selection, clean-frame statistics for clustering.
//
// Reference (paths relative to /root/reference/src/pyannote/audio):
//   Powerset.to_multilabel            utils/powerset.py:115-140
//   Inference.aggregate               core/inference.py:498-620   (hamming=False, warm_up=(0,0))
//   speaker_count                     pipelines/utils/diarization.py:150-185   (np.rint of a float32 ratio)
//   reconstruct / to_diarization      pipelines/speaker_diarization.py:480-528, utils/diarization.py:221-268
//   filter_embeddings                 pipelines/clustering.py:77-125
// Everything here is exact small-integer arithmetic; scatter loops of the reference become per-frame gathers
// over the (<= 11) chunks that cover a frame.
#include "common.cuh"
#include "post.cuh"

namespace b200 {

static void powerset_sets(int N, int size, int first, unsigned set, PowersetMap* map) {
  if (size == 0) { map->mask[map->K++] = set; return; }
  for (int j = first; j <= N - size; ++j) powerset_sets(N, size - 1, j + 1, set | (1u << j), map);
}

bool powerset_map(int N, int M, PowersetMap* map) {
  if (N < 1 || N > 32 || M < 1 || M > N) {
    set_error("powerset of %d speakers with at most %d per frame: need 1 <= max_per_frame <= speakers <= 32", N, M);
    return false;
  }
  unsigned long long classes = 0, binom = 1;                 // sum of C(N, k) for k = 0 .. M
  for (int k = 0; k <= M; ++k) {
    classes += binom;
    binom = binom * (N - k) / (k + 1);
  }
  if (classes > (unsigned long long)kPowersetMaxClasses) {
    set_error("powerset of %d speakers with at most %d per frame has %llu classes; at most %d are supported", N, M,
              classes, kPowersetMaxClasses);
    return false;
  }
  *map = PowersetMap();
  map->N = N;
  for (int size = 0; size <= M; ++size) powerset_sets(N, size, 0, 0u, map);
  return true;
}

// Powerset.to_multilabel, hard (utils/powerset.py:115-140), for N speakers and at most M per frame: class c is the
// speaker set mask[c] (bit j = speaker j).  Class ids >= K map to the empty set, as the 7-class kernel always did.
__global__ void powerset_kernel(const unsigned char* __restrict__ cls, long long n, PowersetMap map,
                                unsigned char* __restrict__ ml) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const unsigned m = cls[i] < map.K ? map.mask[cls[i]] : 0u;
  for (int j = 0; j < map.N; ++j) ml[i * map.N + j] = (m >> j) & 1u;
}

int powerset_to_multilabel(const unsigned char* cls, long long n, const PowersetMap& map, unsigned char* ml,
                           cudaStream_t stream) {
  return launch(powerset_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, cls, n, map, ml);
}

// first chunk whose window [start, start+nf) may contain frame f  (start_frame is non-decreasing)
__device__ __forceinline__ int first_chunk(const int* __restrict__ sf, int C, int f, int nf = kFrames) {
  int lo = 0, hi = C;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (sf[mid] + nf <= f) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__global__ void speaker_count_kernel(const unsigned char* __restrict__ seg, const int* __restrict__ sf, int C, int F,
                                     unsigned char* __restrict__ count) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int num = 0, den = 0;
  for (int c = first_chunk(sf, C, f); c < C && sf[c] <= f; ++c) {
    const unsigned char* p = seg + ((size_t)c * kFrames + (f - sf[c])) * 3;
    num += p[0] + p[1] + p[2];
    den += 1;
  }
  float avg = 0.f;                                   // missing = 0.0 where no chunk contributes
  if (den > 0) avg = __fdiv_rn((float)num, (float)den);
  count[f] = (unsigned char)rintf(avg);              // np.rint: round half to even
}

int speaker_count(const unsigned char* seg, const int* sf, int C, int F, unsigned char* count, cudaStream_t stream) {
  return launch(speaker_count_kernel, ceil_div(F, 256), 256, 0, stream, seg, sf, C, F, count);
}

// ---- generic float overlap-add: Inference.aggregate (core/inference.py:498-620) ------------------------------------
// Chunks of any nf frames.  One thread per (frame, class) gathers the chunks covering the frame in ascending chunk
// order, i.e. in the order numpy's per-chunk `+=` scatter visits them, and reproduces numpy's mixed-precision
// arithmetic exactly: the float32 accumulators are updated as float32(float64(acc) + ((float64(score) * mask) * hamming) * warm_up), the
// average is a float32 division by max(count, float32(epsilon)), frames no chunk contributed to get `missing`.
__global__ void __launch_bounds__(256)
aggregate_kernel(const float* __restrict__ scores, const int* __restrict__ sf, int C, int F, int nf, int K,
                 const double* __restrict__ hamming, const double* __restrict__ warm, int skip_average, float missing,
                 float epsilon, float* __restrict__ out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)F * K) return;
  const int f = (int)(idx / K), k = (int)(idx - (long long)f * K);
  float agg = 0.f, cnt = 0.f;
  bool any = false;
  for (int c = first_chunk(sf, C, f, nf); c < C && sf[c] <= f; ++c) {
    const int t = f - sf[c];
    const float s = scores[((size_t)c * nf + t) * K + k];
    const bool valid = !isnan(s);
    const double h = hamming ? hamming[t] : 1.0, w = warm ? warm[t] : 1.0;
    const double m = valid ? 1.0 : 0.0;
    const double sv = valid ? (double)s : 0.0;
    agg = (float)__dadd_rn((double)agg, __dmul_rn(__dmul_rn(__dmul_rn(sv, m), h), w));
    cnt = (float)__dadd_rn((double)cnt, __dmul_rn(__dmul_rn(m, h), w));
    any |= valid;
  }
  float r = skip_average ? agg : __fdiv_rn(agg, fmaxf(cnt, epsilon));
  if (!any) r = missing;
  out[idx] = r;
}

int aggregate_scores(const float* scores, const int* sf, int C, int F, int nf, int K, const double* hamming,
                     const double* warm, int skip_average, float missing, float epsilon, float* out,
                     cudaStream_t stream) {
  const long long n = (long long)F * K;
  return launch(aggregate_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, scores, sf, C, F, nf, K, hamming, warm,
                skip_average, missing, epsilon, out);
}

// speech score of a powerset frame = max over the speakers of its multilabel row = (its speaker set is not empty);
// this is what VoiceActivityDetection's pre_aggregation_hook (np.max(scores, axis=-1, keepdims=True),
// pipelines/voice_activity_detection.py:111-114) makes of the multilabel output
__global__ void powerset_speech_kernel(const unsigned char* __restrict__ cls, long long n, PowersetMap map,
                                       float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (cls[i] < map.K && map.mask[cls[i]] != 0u) ? 1.f : 0.f;
}

int powerset_speech(const unsigned char* cls, long long n, const PowersetMap& map, float* out, cudaStream_t stream) {
  return launch(powerset_speech_kernel, (unsigned)((n + 255) / 256), 256, 0, stream, cls, n, map, out);
}

// push a byte range to the same offsets of up to 7 peer buffers (P2P stores over NVLink, 16 bytes per thread): the
// powerset classes of a rank's chunks next to the embeddings that gemm_tc_split_kernel pushes from its epilogue
struct PushDsts { unsigned char* d[7]; };
__global__ void push_bytes_kernel(const uint4* __restrict__ src, PushDsts dsts, int n, long long n16,
                                  const unsigned char* __restrict__ src_tail, long long tail0, long long bytes) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n16) {
    const uint4 v = src[i];
    for (int p = 0; p < n; ++p) reinterpret_cast<uint4*>(dsts.d[p])[i] = v;
  } else if (i - n16 < bytes - tail0) {
    const long long o = tail0 + (i - n16);
    for (int p = 0; p < n; ++p) dsts.d[p][o] = src_tail[o];
  }
}

int push_bytes(const void* src, long long bytes, void* const* dsts, int n, cudaStream_t stream) {
  if (bytes <= 0 || n <= 0) return B200_OK;
  B200_CHECK(n <= 7, B200_ERR_INVALID, "push: at most 7 peers");
  B200_CHECK((reinterpret_cast<uintptr_t>(src) & 15) == 0, B200_ERR_INVALID, "push: source must be 16-byte aligned");
  PushDsts d{};
  for (int i = 0; i < n; ++i) {
    B200_CHECK((reinterpret_cast<uintptr_t>(dsts[i]) & 15) == 0, B200_ERR_INVALID, "push: destinations must be 16-byte aligned");
    d.d[i] = reinterpret_cast<unsigned char*>(dsts[i]);
  }
  const long long n16 = bytes / 16, tail0 = n16 * 16, total = n16 + (bytes - tail0);
  return launch(push_bytes_kernel, (unsigned)((total + 255) / 256), 256, 0, stream, reinterpret_cast<const uint4*>(src),
                d, n, n16, reinterpret_cast<const unsigned char*>(src), tail0, bytes);
}

constexpr int kMaxK = 32;

// KMAX is a compile-time bound so that the per-frame activation counters stay in registers (static indexing).
template <int KMAX>
__global__ void __launch_bounds__(128) reconstruct_kernel(const unsigned char* __restrict__ seg,
                                                          const signed char* __restrict__ hard,
                                                          const int* __restrict__ sf, int C, int F, int Kout,
                                                          const unsigned char* __restrict__ count,
                                                          unsigned char* __restrict__ out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  int act[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) act[k] = 0;
  for (int c = first_chunk(sf, C, f); c < C && sf[c] <= f; ++c) {
    const unsigned char* p = seg + ((size_t)c * kFrames + (f - sf[c])) * 3;
    const int h0 = hard[c * 3 + 0], h1 = hard[c * 3 + 1], h2 = hard[c * 3 + 2];
    const int p0 = p[0], p1 = p[1], p2 = p[2];
    // per cluster: max over the local speakers mapped to it (0/1 values -> OR), summed over chunks
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
      const int v = ((h0 == k) ? p0 : 0) | ((h1 == k) ? p1 : 0) | ((h2 == k) ? p2 : 0);
      act[k] += v;
    }
  }
  const int cnt = count[f];
  unsigned used = 0, sel = 0;
  for (int i = 0; i < cnt && i < Kout; ++i) {
    int best = 0, bv = -1;
#pragma unroll
    for (int k = 0; k < KMAX; ++k) {
      const bool ok = (k < Kout) && !((used >> k) & 1u) && act[k] > bv;   // ties -> lowest cluster index
      bv = ok ? act[k] : bv;
      best = ok ? k : best;
    }
    used |= 1u << best;
    sel |= 1u << best;
  }
  unsigned char* o = out + (size_t)f * Kout;
  for (int k = 0; k < Kout; ++k) o[k] = (sel >> k) & 1u;
}

// Many-speaker recordings (33..127 clusters; hard clusters are int8 like the reference's constrained_argmax): same
// arithmetic with the per-frame activation counters in (thread-local) memory instead of registers.  A chunk votes
// once for a cluster however many of its local speakers map to it (max over 0/1 values); a selected cluster is
// marked by the sentinel 0xFF (real activations are <= 11 covering chunks).
constexpr int kMaxKGeneric = 127;

__global__ void __launch_bounds__(128) reconstruct_generic_kernel(const unsigned char* __restrict__ seg,
                                                                  const signed char* __restrict__ hard,
                                                                  const int* __restrict__ sf, int C, int F, int Kout,
                                                                  const unsigned char* __restrict__ count,
                                                                  unsigned char* __restrict__ out) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= F) return;
  unsigned char act[kMaxKGeneric + 1];
  for (int k = 0; k < Kout; ++k) act[k] = 0;
  for (int c = first_chunk(sf, C, f); c < C && sf[c] <= f; ++c) {
    const unsigned char* p = seg + ((size_t)c * kFrames + (f - sf[c])) * 3;
    const int h0 = hard[c * 3 + 0], h1 = hard[c * 3 + 1], h2 = hard[c * 3 + 2];
    const bool v0 = p[0] && h0 >= 0 && h0 < Kout;
    const bool v1 = p[1] && h1 >= 0 && h1 < Kout && !(v0 && h1 == h0);
    const bool v2 = p[2] && h2 >= 0 && h2 < Kout && !(v0 && h2 == h0) && !(p[1] && h2 == h1);
    if (v0) act[h0] += 1;
    if (v1) act[h1] += 1;
    if (v2) act[h2] += 1;
  }
  const int cnt = count[f];
  for (int i = 0; i < cnt && i < Kout; ++i) {
    int best = 0, bv = -1;
    for (int k = 0; k < Kout; ++k)
      if (act[k] != 0xFF && (int)act[k] > bv) { bv = act[k]; best = k; }   // ties -> lowest cluster index
    act[best] = 0xFF;
  }
  unsigned char* o = out + (size_t)f * Kout;
  for (int k = 0; k < Kout; ++k) o[k] = act[k] == 0xFF;
}

int reconstruct(const unsigned char* seg, const signed char* hard, const int* sf, int C, int F, int Kout,
                const unsigned char* count, unsigned char* out, cudaStream_t stream) {
  B200_CHECK(Kout >= 1 && Kout <= kMaxKGeneric, B200_ERR_INVALID,
             "reconstruct: %d clusters unsupported (1..%d: hard clusters are int8 as in the reference's "
             "constrained_argmax; cap the speaker count with max_speakers)", Kout, kMaxKGeneric);
  const int grid = ceil_div(F, 128);
  const auto kernel = Kout > kMaxK ? reconstruct_generic_kernel
                      : Kout <= 8  ? reconstruct_kernel<8>
                      : Kout <= 16 ? reconstruct_kernel<16>
                                   : reconstruct_kernel<32>;
  return launch(kernel, grid, 128, 0, stream, seg, hard, sf, C, F, Kout, count, out);
}

// ---- onsets / offsets of the discrete diarization (Binarize with onset = offset = 0.5, utils/signal.py:254-318) ----
// One thread per frame boundary f in [0, F]: speaker k switches on at f when d[f][k] && !d[f-1][k], off when
// d[f-1][k] && !d[f][k] (f = F closes regions still active at the last frame).  Events are appended unordered as
// k * (F + 1) + f; the host sorts the (few hundred) events.  buf = [n_on, n_off, on[cap], off[cap]].
__global__ void __launch_bounds__(256) frame_transitions_kernel(const unsigned char* __restrict__ d, int F, int K,
                                                                int cap, int* __restrict__ buf) {
  const int f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > F) return;
  const unsigned char* cur = d + (size_t)f * K;
  const unsigned char* prev = cur - K;
  for (int k = 0; k < K; ++k) {
    const bool c = f < F && cur[k] != 0, pv = f > 0 && prev[k] != 0;
    if (c == pv) continue;
    const int slot = atomicAdd(buf + (c ? 0 : 1), 1);
    if (slot < cap) buf[2 + (c ? 0 : cap) + slot] = k * (F + 1) + f;
  }
}

int frame_transitions(const unsigned char* discrete, int F, int K, int cap, int* buf, cudaStream_t stream) {
  B200_CUDA_OK(cudaMemsetAsync(buf, 0, 2 * sizeof(int), stream));
  return launch(frame_transitions_kernel, ceil_div(F + 1, 256), 256, 0, stream, discrete, F, K, cap, buf);
}

__global__ void clean_frames_kernel(const unsigned char* __restrict__ seg, int C, int* __restrict__ clean,
                                    unsigned char* __restrict__ active) {
  // one warp per chunk
  const int c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  int cl[3] = {0, 0, 0}, ac[3] = {0, 0, 0};
  for (int t = lane; t < kFrames; t += 32) {
    const unsigned char* p = seg + ((size_t)c * kFrames + t) * 3;
    const int s = p[0] + p[1] + p[2];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      if (s == 1) cl[k] += p[k];
      ac[k] |= p[k];
    }
  }
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    for (int o = 16; o > 0; o >>= 1) {
      cl[k] += __shfl_xor_sync(0xffffffffu, cl[k], o);
      ac[k] |= __shfl_xor_sync(0xffffffffu, ac[k], o);
    }
    if (lane == 0) { clean[c * 3 + k] = cl[k]; active[c * 3 + k] = (unsigned char)ac[k]; }
  }
}

int clean_frames(const unsigned char* seg, int C, int* clean, unsigned char* active, cudaStream_t stream) {
  return launch(clean_frames_kernel, ceil_div(C * 32, 256), 256, 0, stream, seg, C, clean, active);
}

}  // namespace b200
