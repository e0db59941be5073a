// Shared helpers for the diarization kernels (H100, sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

namespace b200 {

// ---- error plumbing: no exceptions cross the C ABI; last error message is thread-local ----
void set_error(const char* fmt, ...);
const char* last_error();

#define B200_CUDA_OK(expr)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      b200::set_error("%s:%d CUDA error %d (%s) in `%s`", __FILE__, __LINE__, (int)_e,       \
                      cudaGetErrorString(_e), #expr);                                        \
      return (_e == cudaErrorMemoryAllocation) ? B200_ERR_OOM : B200_ERR_CUDA;               \
    }                                                                                        \
  } while (0)

#define B200_CHECK(cond, code, ...)                                                          \
  do {                                                                                       \
    if (!(cond)) {                                                                           \
      b200::set_error(__VA_ARGS__);                                                          \
      return (code);                                                                         \
    }                                                                                        \
  } while (0)

enum {
  B200_OK = 0,
  B200_ERR_INVALID = -1,
  B200_ERR_CUDA = -2,
  B200_ERR_OOM = -3,
  B200_ERR_STATE = -4,
};

// ---- fixed geometry of the community-1 hot path ----
constexpr int kChunk = 160000;       // samples per 10 s chunk @16 kHz
constexpr int kFrames = 589;         // segmentation frames per chunk
constexpr int kSincK = 251;
constexpr int kSincStride = 10;
constexpr int kSincLen = 15975;      // (160000-251)/10+1
constexpr int kPool0 = 5325;         // after MaxPool1d(3,3)
constexpr int kConv1Len = 5321;
constexpr int kPool1 = 1773;
constexpr int kConv2Len = 1769;
constexpr int kPool2 = 589;
constexpr int kHidden = 128;
constexpr int kClasses = 7;
constexpr int kSpeakers = 3;
constexpr int kFbankFrames = 998;    // 1 + (160000-400)/160
constexpr int kMel = 80;
constexpr int kEmbT = 125;           // ResNet time frames after 3 stride-2 stages
constexpr int kEmbDim = 256;
constexpr int kStatsDim = 2560;      // 256 channels x 10 freq bins

// fp32 pairs packed in one 64-bit register: the FP32 kernels keep channel pairs together.  Hopper has no packed fp32
// FMA, so ffma2 is two IEEE fma.rn (the same rounding as one per lane).
typedef unsigned long long f32x2_t;
#ifdef __CUDACC__
__device__ __forceinline__ f32x2_t pack2(float lo, float hi) {
  f32x2_t r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(lo), "f"(hi));
  return r;
}
__device__ __forceinline__ void unpack2(f32x2_t v, float& lo, float& hi) {
  asm("mov.b64 {%0, %1}, %2;" : "=f"(lo), "=f"(hi) : "l"(v));
}
__device__ __forceinline__ void ffma2(f32x2_t& d, f32x2_t a, f32x2_t b) {   // d = a * b + d (lane-wise)
  float d0, d1, a0, a1, b0, b1;
  unpack2(d, d0, d1);
  unpack2(a, a0, a1);
  unpack2(b, b0, b1);
  d = pack2(__fmaf_rn(a0, b0, d0), __fmaf_rn(a1, b1, d1));
}
#endif

// Launch counter of the ctx whose entry point is running on this thread (api.cu: CtxScope binds it), null outside one.
extern thread_local int64_t* g_launch_counter;

#ifdef __CUDACC__
// Every kernel of the library is launched here.  A kernel that takes dynamic shared memory is first opted into that
// much, also below 48 KB, where its static shared memory may still take it past the default.  The attribute belongs to
// one device's context, so it is set at every launch.  Then the kernel is launched, the
// launch is checked and counted on the bound counter (b200_ctx_launch_count).  Cooperative = true makes a cooperative
// launch, for kernels that synchronise the whole grid.
template <bool Cooperative = false, typename... P, typename... Args>
int launch(void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  B200_CHECK(g_launch_counter, B200_ERR_STATE, "kernel launched outside an entry point's ctx scope");
  if (smem) B200_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if constexpr (Cooperative) {
    auto run = [&](P... a) {   // the arguments converted to the kernel's parameter types, passed by address
      void* argv[] = {&a...};
      return cudaLaunchCooperativeKernel((const void*)kernel, grid, block, argv, smem, st);
    };
    B200_CUDA_OK(run(std::forward<Args>(args)...));
  } else {
    kernel<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
    B200_CUDA_OK(cudaGetLastError());
  }
  ++*g_launch_counter;
  return B200_OK;
}
#endif

inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

// Bump allocator that carves the buffers of one launch sequence out of the ctx's workspace (kernels never
// allocate), each buffer starting on an `align`-byte boundary.  With a null base it only measures: take() returns
// nullptr and bytes() is what the layout needs.
struct Workspace {
  char* base;
  size_t align;
  size_t off = 0;
  Workspace(void* b, size_t a) : base(static_cast<char*>(b)), align(a) {}
  void* take(size_t n) {
    off = align_up(off, align);
    void* p = base ? base + off : nullptr;
    off += n;
    return p;
  }
  size_t bytes() const { return align_up(off, align); }
};

}  // namespace b200
