// QK-norm + RoPE (Qwen3) in place on the q and k heads of the fused qkv activation [T, nh + 2*nkv, 128]:
//   forward:  y = bf16(bf16(x * rstd) * w),  rstd = rsqrt(mean(x^2) + eps) over the head's 128 elements,
//             w the q gain for heads < nh and the k gain for the others; then the half-rotation RoPE of
//             rope_inplace_kernel on y.  V heads are not touched.
//   backward: inverse rotation of dqkv, then the RMSNorm backward per head, in place on dqkv's q|k heads:
//             dx = rstd * (g - xhat * mean(g * xhat)),  g = dy * w,  xhat = x * rstd;
//             dw_q / dw_k = sum of dy * xhat over all tokens and q (k) heads, as fp32 per-CTA partials reduced
//             by colsum_kernel in a fixed order (no atomics: bit-identical from run to run).
// Eight threads own one head: lane v of the group holds elements [8v, 8v + 8) and [64 + 8v, 64 + 8v + 8), the two
// halves RoPE pairs, as 16-byte vectors.  The head's sum of squares is three shuffles inside the group.  Every
// warp runs its loop uniformly (four heads per trip, groups past the end compute on zeros) so the shuffles always
// see all 32 lanes.  The forward keeps the pre-norm q|k heads (bf16) and rstd (fp32) for the backward: the
// in-place write destroys the input, and dividing the output by the gain cannot recover it where a gain is 0.
#include "api.h"
#include "common.cuh"

namespace dtg {

namespace {

constexpr int kQKD = 128;          // head_dim served by these kernels (every Qwen3 size)
constexpr int kQKThreads = 256;    // 32 heads per CTA
constexpr int kQKWarps = kQKThreads / 32;

__device__ __forceinline__ float group8_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  v += __shfl_xor_sync(0xffffffffu, v, 2);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  return v;
}

__device__ __forceinline__ float group8_max(float v) {
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 1));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 2));
  v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, 4));
  return v;
}

__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

__device__ __forceinline__ void load_table(const float* __restrict__ cs, const float* __restrict__ sn, long long pos,
                                           int v, float (&c)[8], float (&s)[8]) {
  const float4* cp = reinterpret_cast<const float4*>(cs + pos * (kQKD / 2) + v * 8);
  const float4* sp = reinterpret_cast<const float4*>(sn + pos * (kQKD / 2) + v * 8);
  const float4 c0 = cp[0], c1 = cp[1], s0 = sp[0], s1 = sp[1];
  c[0] = c0.x; c[1] = c0.y; c[2] = c0.z; c[3] = c0.w; c[4] = c1.x; c[5] = c1.y; c[6] = c1.z; c[7] = c1.w;
  s[0] = s0.x; s[1] = s0.y; s[2] = s0.z; s[3] = s0.w; s[4] = s1.x; s[5] = s1.y; s[6] = s1.z; s[7] = s1.w;
}

}  // namespace

__global__ void __launch_bounds__(kQKThreads) qk_norm_rope_fwd_kernel(
    __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ qw, const __nv_bfloat16* __restrict__ kw,
    const float* __restrict__ cs, const float* __restrict__ sn, __nv_bfloat16* __restrict__ x_save,
    float* __restrict__ rstd_out, long long T, int S, int n_heads, int nh, int nqk, int per_token, float eps) {
  const int lane = threadIdx.x & 31, v = lane & 7;
  const long long items = T * nqk;
  const long long warps = (long long)gridDim.x * kQKWarps;
  for (long long wi = blockIdx.x * (long long)kQKWarps + (threadIdx.x >> 5); wi * 4 < items; wi += warps) {
    const long long item = wi * 4 + (lane >> 3);
    const bool ok = item < items;
    const long long t = ok ? item / nqk : 0;
    const int head = ok ? (int)(item % nqk) : 0;
    __nv_bfloat16* p = qkv + (t * n_heads + head) * (long long)kQKD + v * 8;
    float a[8], b[8];
    if (ok) {
      const bf16x8 va = ld8(p), vb = ld8(p + kQKD / 2);
      st8(x_save + item * kQKD + v * 8, va);
      st8(x_save + item * kQKD + kQKD / 2 + v * 8, vb);
      unpack8(va, a);
      unpack8(vb, b);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] = b[j] = 0.f;
    }
    // heads with an element at or above 2^56 (bf16 reaches 2^128) would overflow the fp32 sum of squares: they are
    // summed scaled by 2^-64, which is exact, and eps is negligible next to them
    float am = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) am = fmaxf(am, fmaxf(fabsf(a[j]), fabsf(b[j])));
    am = group8_max(am);
    const float pre = am >= 0x1p56f ? 0x1p-64f : 1.f;
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += (a[j] * pre) * (a[j] * pre) + (b[j] * pre) * (b[j] * pre);
    ss = group8_sum(ss);
    const float rstd = am >= 0x1p56f ? rsqrtf(ss / (float)kQKD) * 0x1p-64f : rsqrtf(ss / (float)kQKD + eps);
    if (!ok) continue;
    if (v == 0) rstd_out[item] = rstd;
    const __nv_bfloat16* w = head < nh ? qw : kw;
    float wa[8], wb[8], c[8], s[8];
    unpack8(ld8(w + v * 8), wa);
    unpack8(ld8(w + kQKD / 2 + v * 8), wb);
    load_table(cs, sn, per_token ? t : t % S, v, c, s);
    float o1[8], o2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float ya = round_bf16(round_bf16(a[j] * rstd) * wa[j]);
      const float yb = round_bf16(round_bf16(b[j] * rstd) * wb[j]);
      o1[j] = ya * c[j] - yb * s[j];
      o2[j] = yb * c[j] + ya * s[j];
    }
    st8(p, pack8(o1));
    st8(p + kQKD / 2, pack8(o2));
  }
}

__global__ void __launch_bounds__(kQKThreads) qk_norm_rope_bwd_kernel(
    __nv_bfloat16* __restrict__ dqkv, const __nv_bfloat16* __restrict__ x_save, const float* __restrict__ rstd,
    const __nv_bfloat16* __restrict__ qw, const __nv_bfloat16* __restrict__ kw, const float* __restrict__ cs,
    const float* __restrict__ sn, float* __restrict__ dw_partial, long long T, int S, int n_heads, int nh, int nqk,
    int per_token) {
  __shared__ float red[kQKWarps][2 * kQKD];
  const int lane = threadIdx.x & 31, v = lane & 7, warp = threadIdx.x >> 5;
  // gain-gradient partials of this thread's 16 elements: [0, 8) = first half, [8, 16) = second half
  float accq[16], acck[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) accq[j] = acck[j] = 0.f;
  const long long items = T * nqk;
  const long long warps = (long long)gridDim.x * kQKWarps;
  for (long long wi = blockIdx.x * (long long)kQKWarps + warp; wi * 4 < items; wi += warps) {
    const long long item = wi * 4 + (lane >> 3);
    const bool ok = item < items;
    const long long t = ok ? item / nqk : 0;
    const int head = ok ? (int)(item % nqk) : 0;
    __nv_bfloat16* p = dqkv + (t * n_heads + head) * (long long)kQKD + v * 8;
    float dya[8], dyb[8], xa[8], xb[8], ga[8], gb[8], rs = 0.f, dot = 0.f;
    if (ok) {
      float a[8], b[8], c[8], s[8], wa[8], wb[8];
      unpack8(ld8(p), a);
      unpack8(ld8(p + kQKD / 2), b);
      load_table(cs, sn, per_token ? t : t % S, v, c, s);
      rs = rstd[item];
      unpack8(ld8(x_save + item * kQKD + v * 8), xa);
      unpack8(ld8(x_save + item * kQKD + kQKD / 2 + v * 8), xb);
      const __nv_bfloat16* w = head < nh ? qw : kw;
      unpack8(ld8(w + v * 8), wa);
      unpack8(ld8(w + kQKD / 2 + v * 8), wb);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        dya[j] = a[j] * c[j] + b[j] * s[j];   // inverse rotation
        dyb[j] = b[j] * c[j] - a[j] * s[j];
        xa[j] *= rs;
        xb[j] *= rs;
        ga[j] = dya[j] * wa[j];
        gb[j] = dyb[j] * wb[j];
        dot += ga[j] * xa[j] + gb[j] * xb[j];
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) dya[j] = dyb[j] = xa[j] = xb[j] = ga[j] = gb[j] = 0.f;
    }
    dot = group8_sum(dot) / (float)kQKD;
    if (!ok) continue;
    float o1[8], o2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      o1[j] = rs * (ga[j] - xa[j] * dot);
      o2[j] = rs * (gb[j] - xb[j] * dot);
    }
    st8(p, pack8(o1));
    st8(p + kQKD / 2, pack8(o2));
    if (head < nh) {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        accq[j] += dya[j] * xa[j];
        accq[8 + j] += dyb[j] * xb[j];
      }
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        acck[j] += dya[j] * xa[j];
        acck[8 + j] += dyb[j] * xb[j];
      }
    }
  }
  // the four groups of a warp hold the same elements: fold them, then the warps, in a fixed order
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    accq[j] += __shfl_xor_sync(0xffffffffu, accq[j], 8);
    accq[j] += __shfl_xor_sync(0xffffffffu, accq[j], 16);
    acck[j] += __shfl_xor_sync(0xffffffffu, acck[j], 8);
    acck[j] += __shfl_xor_sync(0xffffffffu, acck[j], 16);
  }
  if (lane < 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      red[warp][v * 8 + j] = accq[j];
      red[warp][kQKD / 2 + v * 8 + j] = accq[8 + j];
      red[warp][kQKD + v * 8 + j] = acck[j];
      red[warp][kQKD + kQKD / 2 + v * 8 + j] = acck[8 + j];
    }
  }
  __syncthreads();
  float sum = 0.f;
#pragma unroll
  for (int w = 0; w < kQKWarps; ++w) sum += red[w][threadIdx.x];
  dw_partial[(size_t)blockIdx.x * (2 * kQKD) + threadIdx.x] = sum;
}
static_assert(kQKThreads == 2 * kQKD, "one thread per column of the [2, 128] gain-gradient partial");

static int qk_items_grid(long long items, int cap) {
  long long g = (items + 4 * kQKWarps - 1) / (4 * kQKWarps);
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

// one wave of resident CTAs (the kernel needs ~106 registers, so 2 per SM): every CTA writes one partial row
int qk_norm_rope_bwd_grid(long long T, int nqk) {
  static int per_sm = 0;
  if (per_sm == 0) {
    DTG_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, qk_norm_rope_bwd_kernel, kQKThreads, 0));
    if (per_sm < 1) per_sm = 1;
  }
  return qk_items_grid(T * nqk, per_sm * sm_count());
}

void qk_norm_rope_fwd(void* qkv, const void* q_w, const void* k_w, const float* cos, const float* sin, void* x_save,
                      float* rstd, long long T, int S, int n_heads, int nh, int nkv, bool per_token, float eps,
                      cudaStream_t s) {
  const int nqk = nh + nkv;
  if (T * nqk == 0) return;
  qk_norm_rope_fwd_kernel<<<qk_items_grid(T * nqk, 16 * sm_count()), kQKThreads, 0, s>>>(
      (__nv_bfloat16*)qkv, (const __nv_bfloat16*)q_w, (const __nv_bfloat16*)k_w, cos, sin, (__nv_bfloat16*)x_save,
      rstd, T, S, n_heads, nh, nqk, per_token ? 1 : 0, eps);
  note_launch();
  DTG_LAUNCH_CHECK();
}

void qk_norm_rope_bwd(void* dqkv, const void* x_save, const float* rstd, const void* q_w, const void* k_w,
                      const float* cos, const float* sin, float* dw_partial, float* dw, long long T, int S, int n_heads,
                      int nh, int nkv, bool per_token, cudaStream_t s) {
  const int nqk = nh + nkv;
  const int grid = qk_norm_rope_bwd_grid(T, nqk);
  if (T * nqk == 0) {
    DTG_CUDA_CHECK(cudaMemsetAsync(dw, 0, 2 * kQKD * sizeof(float), s));
    return;
  }
  qk_norm_rope_bwd_kernel<<<grid, kQKThreads, 0, s>>>(
      (__nv_bfloat16*)dqkv, (const __nv_bfloat16*)x_save, rstd, (const __nv_bfloat16*)q_w,
      (const __nv_bfloat16*)k_w, cos, sin, dw_partial, T, S, n_heads, nh, nqk, per_token ? 1 : 0);
  note_launch();
  DTG_LAUNCH_CHECK();
  colsum(dw_partial, dw, grid, 2 * kQKD, s);
}

}  // namespace dtg
