// FP32 SIMT GEMM  C[M][N] = act(A[M][K] * B[N][K]^T + bias[N])   ("NT": both operands K-contiguous, i.e.
// activations row-major and weights in PyTorch's nn.Linear / nn.LSTM [out][in] layout).
// Used for the LSTM input projections (PyanNet.py:98,226-228), the two Linear+LeakyReLU layers (:236-238)
// and the embedding Linear 5120->256 (resnet.py:246,423).  fp32 because the reference runs with TF32
// disabled (utils/reproducibility.py:68-83) and the powerset argmax downstream is integer-exact.
#include "common.cuh"
#include "seg.cuh"

namespace b200 {

constexpr int BM = 128, BN = 128, BK = 16, PADM = 4;

template <int ACT>
__global__ void __launch_bounds__(256) sgemm_nt_kernel(const float* __restrict__ A, int lda,
                                                       const float* __restrict__ Bw, int ldb, float* __restrict__ C,
                                                       int ldc, const float* __restrict__ bias, int M, int N, int K) {
  __shared__ float As[2][BK][BM + PADM];
  __shared__ float Bs[2][BK][BN + PADM];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int lrow = tid >> 2, lkq = tid & 3;       // loader: rows lrow, lrow+64; k quad lkq
  const int ty = tid >> 4, tx = tid & 15;         // compute: rows ty*4 (+64), cols tx*4 (+64)

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 ra[2], rb[2];
  auto gload = [&](int k0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = m0 + lrow + 64 * h;
      ra[h] = (r < M) ? *reinterpret_cast<const float4*>(A + (size_t)r * lda + k0 + lkq * 4)
                      : make_float4(0.f, 0.f, 0.f, 0.f);
      const int c = n0 + lrow + 64 * h;
      rb[h] = (c < N) ? *reinterpret_cast<const float4*>(Bw + (size_t)c * ldb + k0 + lkq * 4)
                      : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = lrow + 64 * h;
      As[buf][lkq * 4 + 0][r] = ra[h].x; As[buf][lkq * 4 + 1][r] = ra[h].y;
      As[buf][lkq * 4 + 2][r] = ra[h].z; As[buf][lkq * 4 + 3][r] = ra[h].w;
      Bs[buf][lkq * 4 + 0][r] = rb[h].x; Bs[buf][lkq * 4 + 1][r] = rb[h].y;
      Bs[buf][lkq * 4 + 2][r] = rb[h].z; Bs[buf][lkq * 4 + 3][r] = rb[h].w;
    }
  };

  gload(0);
  sstore(0);
  __syncthreads();
  const int nk = K / BK;
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) gload((kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int r = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (r >= M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int c = n0 + jh * 64 + tx * 4;
      if (c >= N) continue;
      float4 v;
      float* vp = reinterpret_cast<float*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float x = acc[i][jh * 4 + j] + (bias ? bias[c + j] : 0.f);
        if (ACT == 1) x = x > 0.f ? x : 0.01f * x;
        vp[j] = x;
      }
      *reinterpret_cast<float4*>(C + (size_t)r * ldc + c) = v;
    }
  }
}

int sgemm_nt(const float* A, int lda, const float* Bw, int ldb, float* C, int ldc, const float* bias, int M, int N,
             int K, int act, cudaStream_t stream) {
  B200_CHECK(K % BK == 0 && N % 4 == 0 && lda % 4 == 0 && ldb % 4 == 0 && ldc % 4 == 0, B200_ERR_INVALID,
             "sgemm_nt: unsupported shape M=%d N=%d K=%d", M, N, K);
  dim3 grid(ceil_div(M, BM), ceil_div(N, BN));
  return launch(act == 1 ? sgemm_nt_kernel<1> : sgemm_nt_kernel<0>, grid, 256, 0, stream, A, lda, Bw, ldb, C, ldc, bias,
                M, N, K);
}

}  // namespace b200
