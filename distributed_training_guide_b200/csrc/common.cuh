// Shared helpers for the sm_90a kernels: error checks, launch accounting, bf16 vector math.
#pragma once
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>

namespace dtg {

constexpr int kMaxRanks = 8;  // one NVSwitch domain

// Every kernel launch of this extension is counted (bench.py reports it as `gpu_launches`).
void note_launch(int n = 1);
unsigned long long launch_count();

inline void check(cudaError_t e, const char* what, const char* file, int line) {
  if (e != cudaSuccess) {
    throw std::runtime_error(std::string(what) + " failed: " + cudaGetErrorString(e) + " at " + file + ":" +
                             std::to_string(line));
  }
}
#define DTG_CUDA_CHECK(x) ::dtg::check((x), #x, __FILE__, __LINE__)
#define DTG_LAUNCH_CHECK() ::dtg::check(cudaGetLastError(), "kernel launch", __FILE__, __LINE__)

inline int sm_count() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 148;
  }
  return n;
}

// CTAs of 256 threads for a grid-strided elementwise kernel over total_threads work items: at most 16 per SM
inline int ew_grid(long long total_threads) {
  long long g = (total_threads + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// A sum of squares of bf16 values at or above kSumSqBig (bf16 reaches 2^128) can overflow fp32.  Such values are
// squared scaled by kSumSqDown, which is exact for every element above 2^-77 (a smaller one is below 2^-94 of the
// largest square and cannot change the sum) and keeps a sum of 2^16 squares of bf16's largest values finite.
constexpr float kSumSqBig = 0x1p56f, kSumSqDown = 0x1p-72f, kSumSqUp = 0x1p72f;

// The one vocabulary rule of every kernel indexed by token id or target (loss, embedding, their TP forms):
//   kIgnoreIndex        a target that is ignored: zero dlogits row, not counted in n_valid;
//   0 <= id < V         valid;
//   anything else       bad: never dereferenced.  A bad target counts in n_valid and gets a NaN row loss and NaN
//                       dlogits row (a NaN loss is what the log shows, without a host synchronise); a bad embedding
//                       id gets a NaN forward row and adds to no row in the backward.
constexpr long long kIgnoreIndex = -100;

// ---- device-side helpers (nvcc only) ----------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ bool in_vocab(long long id, long long V) {
  return (unsigned long long)id < (unsigned long long)V;   // one compare: a negative id wraps past any V
}
__device__ __forceinline__ float nan_f() { return __int_as_float(0x7fffffff); }

struct alignas(16) bf16x8 {
  __nv_bfloat162 v[4];
};

__device__ __forceinline__ void unpack8(const bf16x8& p, float (&f)[8]) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ bf16x8 pack8(const float (&f)[8]) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}
// 16-byte accesses spelled as uint4 so they compile to LDG.128 / STG.128 (a struct of four bfloat162
// is otherwise split into four 32-bit accesses)
__device__ __forceinline__ bf16x8 ld8(const __nv_bfloat16* p) {
  bf16x8 r;
  *reinterpret_cast<uint4*>(&r) = *reinterpret_cast<const uint4*>(p);
  return r;
}
__device__ __forceinline__ void st8(__nv_bfloat16* p, const bf16x8& v) {
  *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&v);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide sum for blockDim.x <= 1024; `red` is a 32-float shared scratch. All threads get the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();  // protect `red` from a previous use
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : 0.f;
  r = warp_sum(r);
  return r;
}
__device__ __forceinline__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : -INFINITY;
  r = warp_max(r);
  return r;
}

// the scale to square values whose largest magnitude is am by, and rsqrt(mean(x^2) + eps) of n values from their sum
// of squares ss taken at that scale (eps is negligible next to a rescued sum)
__device__ __forceinline__ float sumsq_scale(float am) { return am >= kSumSqBig ? kSumSqDown : 1.f; }
__device__ __forceinline__ float sumsq_rstd(float ss, float am, float n, float eps) {
  return am >= kSumSqBig ? rsqrtf(ss / n) * kSumSqDown : rsqrtf(ss / n + eps);
}

#endif  // __CUDACC__

}  // namespace dtg
