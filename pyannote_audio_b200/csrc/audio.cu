// Audio ingest on the device: PCM -> float32, downmix, polyphase sinc resampling to the model's sample rate.
//
// Reference (paths relative to /root/reference/src/pyannote/audio):
//   Audio.downmix_and_resample   core/io.py:223-265   (mean over channels, then torchaudio.functional.resample)
//   Audio.__call__ / crop        core/io.py:306-351, 353-484
// torchaudio.functional.resample (installed 2.11; functional.py `_get_sinc_resample_kernel` /
// `_apply_sinc_resample_kernel`, defaults lowpass_filter_width = 6, rolloff = 0.99, sinc_interp_hann):
//   orig, new = sr_in / gcd, sr_out / gcd;  base = min(orig, new) * rolloff;  width = ceil(6 * orig / base)
//   kernel[j][k] = sinc(pi * t) * cos^2(pi * t / 12) * base / orig,  t = clamp((-j / new + (k - width) / orig) * base, -6, 6)
//   y[i * new + j] = sum_k kernel[j][k] * x[i * orig + k - width]   (x = 0 outside), first ceil(new * len / orig) samples
// The reference decodes to float32 on the host and resamples on the CPU; here the raw PCM (int16: half the PCIe
// bytes of float32) crosses PCIe once and one kernel converts, downmixes and resamples: each CTA stages the
// (downmixed) input span of its output tile in shared memory, each thread accumulates one output sample.
#include "common.cuh"
#include "audio.cuh"
#include <cmath>

namespace b200 {

// builds kernel[j][k] (new x klen) exactly like torchaudio does for a float32 waveform: the positions are computed in
// float32 there (dtype = waveform.dtype); we evaluate in double and round once, which agrees to ~1e-7
void resample_table(int orig, int nw, int* width_out, std::vector<float>* table) {
  const double rolloff = 0.99, lpw = 6.0;
  const double base = (orig < nw ? orig : nw) * rolloff;
  const int width = (int)std::ceil(lpw * orig / base);
  const int klen = 2 * width + orig;
  table->assign((size_t)nw * klen, 0.f);
  const double scale = base / orig;
  for (int j = 0; j < nw; ++j)
    for (int k = 0; k < klen; ++k) {
      double t = ((double)(-j) / nw + (double)(k - width) / orig) * base;
      t = t < -lpw ? -lpw : (t > lpw ? lpw : t);
      const double c = std::cos(t * M_PI / lpw / 2.0);
      const double w = c * c;
      const double tp = t * M_PI;
      const double s = tp == 0.0 ? 1.0 : std::sin(tp) / tp;
      (*table)[(size_t)j * klen + k] = (float)(s * w * scale);
    }
  *width_out = width;
}

constexpr int kIngestThreads = 256;
constexpr int kIngestSpan = 8192;          // input samples staged per CTA (32 KB of shared memory)

// FORMAT 0: int16 interleaved [frame][channel];  FORMAT 1: float32 planar [channel][frame]
template <int FORMAT>
__global__ void __launch_bounds__(kIngestThreads)
ingest_kernel(const void* __restrict__ src, int channels, long long frames_in, int channel,
              const float* __restrict__ table, int orig, int nw, int width, int klen, int periods_per_cta,
              float* __restrict__ out, long long frames_out) {
  __shared__ float mono[kIngestSpan];
  const long long i0 = (long long)blockIdx.x * periods_per_cta;            // first input period of this tile
  const long long m0 = i0 * orig - width;                                  // first input sample needed
  const int span = (periods_per_cta - 1) * orig + klen;
  const float inv_c = 1.0f / (float)channels;
  for (int s = threadIdx.x; s < span; s += kIngestThreads) {
    const long long m = m0 + s;
    float v = 0.f;
    if (m >= 0 && m < frames_in) {
      if (FORMAT == 0) {
        const short* p = reinterpret_cast<const short*>(src) + m * channels;
        if (channel >= 0) {
          v = (float)p[channel] / 32768.0f;
        } else {
          float acc = 0.f;
          for (int c = 0; c < channels; ++c) acc += (float)p[c] / 32768.0f;
          v = channels > 1 ? acc / (float)channels : acc;
        }
      } else {
        const float* p = reinterpret_cast<const float*>(src);
        if (channel >= 0) {
          v = p[(long long)channel * frames_in + m];
        } else {
          float acc = 0.f;
          for (int c = 0; c < channels; ++c) acc += p[(long long)c * frames_in + m];
          v = channels > 1 ? acc / (float)channels : acc;                   // torch.mean: sum, then divide
        }
      }
    }
    mono[s] = v;
  }
  (void)inv_c;
  __syncthreads();
  const int outs = periods_per_cta * nw;
  for (int o = threadIdx.x; o < outs; o += kIngestThreads) {
    const int ip = o / nw, j = o - ip * nw;
    const long long og = (i0 + ip) * nw + j;
    if (og >= frames_out) continue;
    const float* kr = table + (size_t)j * klen;
    const float* x = mono + ip * orig;
    float acc = 0.f;
    for (int k = 0; k < klen; ++k) acc = fmaf(kr[k], x[k], acc);
    out[og] = acc;
  }
}

int audio_ingest(const void* src, int format, int channels, long long frames_in, int channel, const float* table,
                 int orig, int nw, int width, float* out, long long frames_out, cudaStream_t stream) {
  const int klen = 2 * width + orig;
  B200_CHECK(klen <= kIngestSpan, B200_ERR_INVALID,
             "resampling ratio %d:%d needs a %d-tap polyphase filter (max %d): reduce the rates by their gcd first",
             orig, nw, klen, kIngestSpan);
  const int periods = (kIngestSpan - klen) / orig + 1;
  const long long total_periods = (frames_out + nw - 1) / nw;
  const long long grid = (total_periods + periods - 1) / periods;
  if (grid == 0) return B200_OK;
  B200_CHECK(grid < (1ll << 31), B200_ERR_INVALID, "audio too long for one launch");
  return launch(format == 0 ? ingest_kernel<0> : ingest_kernel<1>, (unsigned)grid, kIngestThreads, 0, stream, src,
                channels, frames_in, channel, table, orig, nw, width, klen, periods, out, frames_out);
}

}  // namespace b200
