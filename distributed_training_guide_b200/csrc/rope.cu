// Everything that positions q and k in the fused qkv activation [T, n_heads, d] (bf16), in place:
//   * RoPE (half-rotation layout) on heads [0, n_rot): the pairs (j, j + rot_dim/2), j < rot_dim/2, of each head's
//     first rot_dim elements, rot_dim = d but for GPT-NeoX's partial rotary; elements [rot_dim, d) are never read or
//     written.  The backward is the inverse rotation.
//   * QK-norm + RoPE at head_dim 128: an RMSNorm of the q and k heads, then the same rotation.  Per head (Qwen3) or
//     over each token's whole q region and whole k region (OLMo 2).
// cos/sin: fp32 [S, rot_dim/2] (row t % S) or per-token [T, rot_dim/2].  Each thread works on 2x8 units: elements
// [8v, 8v + 8) and [rot_dim/2 + 8v, rot_dim/2 + 8v + 8) of a head, the two halves of eight RoPE pairs, as 16-byte
// vectors.
#include <type_traits>

#include "api.h"
#include "common.cuh"

namespace dtg {

namespace {

// the cos/sin row of token t: its own row of a per-token table, else its position in the sequence
__device__ __forceinline__ long long rope_row(long long t, int S, int per_token) { return per_token ? t : t % S; }

// the cos and sin of unit v's eight pairs from table row `row` of half_width floats
__device__ __forceinline__ void load_table(const float* __restrict__ cs, const float* __restrict__ sn, long long row,
                                           int half_width, int v, float (&c)[8], float (&s)[8]) {
  const float4* cp = reinterpret_cast<const float4*>(cs + row * half_width + v * 8);
  const float4* sp = reinterpret_cast<const float4*>(sn + row * half_width + v * 8);
  const float4 c0 = cp[0], c1 = cp[1], s0 = sp[0], s1 = sp[1];
  c[0] = c0.x; c[1] = c0.y; c[2] = c0.z; c[3] = c0.w; c[4] = c1.x; c[5] = c1.y; c[6] = c1.z; c[7] = c1.w;
  s[0] = s0.x; s[1] = s0.y; s[2] = s0.z; s[3] = s0.w; s[4] = s1.x; s[5] = s1.y; s[6] = s1.z; s[7] = s1.w;
}

// the rotation of the pairs (a[j], b[j]) by the angles of (c[j], s[j]), and its inverse
__device__ __forceinline__ void rotate(const float (&a)[8], const float (&b)[8], const float (&c)[8],
                                       const float (&s)[8], float (&o1)[8], float (&o2)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o1[j] = a[j] * c[j] - b[j] * s[j];
    o2[j] = b[j] * c[j] + a[j] * s[j];
  }
}
__device__ __forceinline__ void rotate_inv(const float (&a)[8], const float (&b)[8], const float (&c)[8],
                                           const float (&s)[8], float (&o1)[8], float (&o2)[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    o1[j] = a[j] * c[j] + b[j] * s[j];
    o2[j] = b[j] * c[j] - a[j] * s[j];
  }
}

__device__ __forceinline__ float round_bf16(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

}  // namespace

// ------------------------------------------------------------------------------------------
// RoPE: one 2x8 unit per thread, grid-strided; sign -1 rotates backwards
// ------------------------------------------------------------------------------------------
__global__ void rope_inplace_kernel(__nv_bfloat16* __restrict__ qkv, const float* __restrict__ cs,
                                    const float* __restrict__ sn, long long T, int S, int n_heads, int n_rot, int d,
                                    int rot_dim, int per_token, float sign) {
  const int r2 = rot_dim >> 1;
  const int vec_per_head = r2 >> 3;
  const long long total = T * (long long)n_rot * vec_per_head;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % vec_per_head);
    const long long th = idx / vec_per_head;
    const int head = (int)(th % n_rot);
    const long long t = th / n_rot;
    const long long row = rope_row(t, S, per_token);
    __nv_bfloat16* p = qkv + (t * n_heads + head) * (long long)d + v * 8;
    float a[8], b[8], c[8], s[8], o1[8], o2[8];
    unpack8(ld8(p), a);
    unpack8(ld8(p + r2), b);
    load_table(cs, sn, row, r2, v, c, s);
#pragma unroll
    for (int j = 0; j < 8; ++j) s[j] *= sign;
    rotate(a, b, c, s, o1, o2);
    st8(p, pack8(o1));
    st8(p + r2, pack8(o2));
  }
}

void rope_inplace(void* qkv, const float* cos, const float* sin, long long T, int S, int n_heads, int n_rot, int d,
                  int rot_dim, bool per_token, bool inverse, cudaStream_t s) {
  if (d % 16 != 0) throw std::runtime_error("rope: head_dim must be a multiple of 16");
  if (rot_dim % 16 != 0 || rot_dim <= 0 || rot_dim > d)
    throw std::runtime_error("rope: rot_dim must be a positive multiple of 16, <= head_dim");
  rope_inplace_kernel<<<ew_grid(T * (long long)n_rot * (rot_dim / 16)), 256, 0, s>>>(
      (__nv_bfloat16*)qkv, cos, sin, T, S, n_heads, n_rot, d, rot_dim, per_token ? 1 : 0, inverse ? -1.f : 1.f);
  note_launch();
  DTG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// QK-norm + RoPE (Qwen3) on the q and k heads of qkv [T, nh + 2*nkv, 128]:
//   forward:  y = bf16(bf16(x * rstd) * w),  rstd = rsqrt(mean(x^2) + eps) over the head's 128 elements,
//             w the q gain for heads < nh and the k gain for the others; then the rotation of y.  V heads are not
//             touched.
//   backward: inverse rotation of dqkv, then the RMSNorm backward per head, in place on dqkv's q|k heads:
//             dx = rstd * (g - xhat * mean(g * xhat)),  g = dy * w,  xhat = x * rstd;
//             dw_q / dw_k = sum of dy * xhat over all tokens and q (k) heads, as fp32 per-CTA partials reduced
//             by colsum_kernel in a fixed order (no atomics: bit-identical from run to run).
// Eight threads own one head, one unit each.  The head's sum of squares is three shuffles inside the group.  Every
// warp runs its loop uniformly (four heads per trip, groups past the end compute on zeros) so the shuffles always
// see all 32 lanes.  The forward keeps the pre-norm q|k heads (bf16) and rstd (fp32) for the backward: the
// in-place write destroys the input, and dividing the output by the gain cannot recover it where a gain is 0.
// ------------------------------------------------------------------------------------------
namespace {

constexpr int kQKD = 128;          // head_dim served by the QK-norm kernels (every Qwen3 and OLMo 2 size)
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
    float am = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) am = fmaxf(am, fmaxf(fabsf(a[j]), fabsf(b[j])));
    am = group8_max(am);
    const float pre = sumsq_scale(am);
    float ss = 0.f;
#pragma unroll
    for (int j = 0; j < 8; ++j) ss += (a[j] * pre) * (a[j] * pre) + (b[j] * pre) * (b[j] * pre);
    ss = group8_sum(ss);
    const float rstd = sumsq_rstd(ss, am, (float)kQKD, eps);
    if (!ok) continue;
    if (v == 0) rstd_out[item] = rstd;
    const __nv_bfloat16* w = head < nh ? qw : kw;
    float wa[8], wb[8], c[8], s[8], ya[8], yb[8], o1[8], o2[8];
    unpack8(ld8(w + v * 8), wa);
    unpack8(ld8(w + kQKD / 2 + v * 8), wb);
    load_table(cs, sn, rope_row(t, S, per_token), kQKD / 2, v, c, s);
#pragma unroll
    for (int j = 0; j < 8; ++j) {   // two roundings, as HF Qwen3: bf16(bf16(x * rstd) * w)
      ya[j] = round_bf16(round_bf16(a[j] * rstd) * wa[j]);
      yb[j] = round_bf16(round_bf16(b[j] * rstd) * wb[j]);
    }
    rotate(ya, yb, c, s, o1, o2);
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
      load_table(cs, sn, rope_row(t, S, per_token), kQKD / 2, v, c, s);
      rs = rstd[item];
      unpack8(ld8(x_save + item * kQKD + v * 8), xa);
      unpack8(ld8(x_save + item * kQKD + kQKD / 2 + v * 8), xb);
      const __nv_bfloat16* w = head < nh ? qw : kw;
      unpack8(ld8(w + v * 8), wa);
      unpack8(ld8(w + kQKD / 2 + v * 8), wb);
      rotate_inv(a, b, c, s, dya, dyb);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
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

// ------------------------------------------------------------------------------------------
// Full-width QK-norm + RoPE (OLMo 2) on the same layout:
//   forward:  y = bf16(x * rstd_r * w),  rstd_r = rsqrt(mean(x^2) + eps) over the token's whole q region (nh * 128
//             elements) or k region (nkv * 128), w the [nh * 128] q gain or [nkv * 128] k gain, with the one rounding
//             of the RMSNorm forward (norm.cu); then the rotation of y, per head.
//   backward: inverse rotation, then dx = rstd_r * (g - xhat * mean_r(g * xhat)), g = dy * w, per region;
//             dw = sum over tokens of dy * xhat over the (nh + nkv) * 128 gain columns, as fp32 per-CTA partial
//             rows reduced by colsum_kernel in a fixed order (no atomics).
// One CTA per token (forward) or a persistent CTA striding over tokens (backward).  Unit u = head * 8 + v of the
// row is thread u % 256's (u / 256)-th unit.  The two statistics (q and k) are one block reduction of two values.
// The forward keeps the pre-norm q|k row (bf16) and the two rstd (fp32) of each token for the backward.
// ------------------------------------------------------------------------------------------
namespace {

constexpr int kFullThreads = 256;
constexpr int kFullMaxUnits = 3;   // up to 3 * 256 / 8 = 96 q + k heads per token (OLMo-2-13B: 40 + 40)

template <bool MAX>
__device__ __forceinline__ float2 block_reduce2(float a, float b, float (*red)[32]) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ao = __shfl_xor_sync(0xffffffffu, a, o), bo = __shfl_xor_sync(0xffffffffu, b, o);
    a = MAX ? fmaxf(a, ao) : a + ao;
    b = MAX ? fmaxf(b, bo) : b + bo;
  }
  __syncthreads();   // protect `red` from a previous use
  if (lane == 0) {
    red[0][w] = a;
    red[1][w] = b;
  }
  __syncthreads();
  a = lane < kFullThreads / 32 ? red[0][lane] : 0.f;   // 0 is also the identity of a max of |x|
  b = lane < kFullThreads / 32 ? red[1][lane] : 0.f;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ao = __shfl_xor_sync(0xffffffffu, a, o), bo = __shfl_xor_sync(0xffffffffu, b, o);
    a = MAX ? fmaxf(a, ao) : a + ao;
    b = MAX ? fmaxf(b, bo) : b + bo;
  }
  return make_float2(a, b);
}

// f(std::integral_constant<int, NU>()) with NU the units per thread a row of nqk q + k heads needs
template <class F>
void with_units(int nqk, F&& f) {
  const int units = nqk * 8;
  if (units <= kFullThreads) f(std::integral_constant<int, 1>());
  else if (units <= 2 * kFullThreads) f(std::integral_constant<int, 2>());
  else if (units <= kFullMaxUnits * kFullThreads) f(std::integral_constant<int, 3>());
  else throw std::runtime_error("qk_norm_full_rope: more than 96 q + k heads per token unsupported");
}

}  // namespace

template <int NU>
__global__ void __launch_bounds__(kFullThreads) qk_norm_full_rope_fwd_kernel(
    __nv_bfloat16* __restrict__ qkv, const __nv_bfloat16* __restrict__ qw, const __nv_bfloat16* __restrict__ kw,
    const float* __restrict__ cs, const float* __restrict__ sn, __nv_bfloat16* __restrict__ x_save,
    float* __restrict__ rstd_out, int S, int n_heads, int nh, int nkv, int per_token, float eps) {
  __shared__ float red[2][32];
  const long long t = blockIdx.x;
  const int nqk = nh + nkv, units = nqk * 8;
  __nv_bfloat16* row = qkv + t * n_heads * (long long)kQKD;
  __nv_bfloat16* save = x_save + t * nqk * (long long)kQKD;
  bf16x8 ca[NU], cb[NU];
  float amq = 0.f, amk = 0.f;
#pragma unroll
  for (int k = 0; k < NU; ++k) {
    const int u = threadIdx.x + k * kFullThreads;
    if (u < units) {
      const int off = (u >> 3) * kQKD + (u & 7) * 8;
      ca[k] = ld8(row + off);
      cb[k] = ld8(row + off + kQKD / 2);
      st8(save + off, ca[k]);
      st8(save + off + kQKD / 2, cb[k]);
      float a[8], b[8], m = 0.f;
      unpack8(ca[k], a);
      unpack8(cb[k], b);
#pragma unroll
      for (int j = 0; j < 8; ++j) m = fmaxf(m, fmaxf(fabsf(a[j]), fabsf(b[j])));
      if ((u >> 3) < nh) amq = fmaxf(amq, m);
      else amk = fmaxf(amk, m);
    }
  }
  const float2 am = block_reduce2<true>(amq, amk, red);
  const float preq = sumsq_scale(am.x), prek = sumsq_scale(am.y);
  float ssq = 0.f, ssk = 0.f;
#pragma unroll
  for (int k = 0; k < NU; ++k) {
    const int u = threadIdx.x + k * kFullThreads;
    if (u < units) {
      const bool isq = (u >> 3) < nh;
      const float pre = isq ? preq : prek;
      float a[8], b[8], s = 0.f;
      unpack8(ca[k], a);
      unpack8(cb[k], b);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += (a[j] * pre) * (a[j] * pre) + (b[j] * pre) * (b[j] * pre);
      if (isq) ssq += s;
      else ssk += s;
    }
  }
  const float2 ss = block_reduce2<false>(ssq, ssk, red);
  const float rq = sumsq_rstd(ss.x, am.x, (float)(nh * kQKD), eps);
  const float rk = sumsq_rstd(ss.y, am.y, (float)(nkv * kQKD), eps);
  if (threadIdx.x == 0) {
    rstd_out[2 * t] = rq;
    rstd_out[2 * t + 1] = rk;
  }
  const long long pos = rope_row(t, S, per_token);
#pragma unroll
  for (int k = 0; k < NU; ++k) {
    const int u = threadIdx.x + k * kFullThreads;
    if (u < units) {
      const int head = u >> 3, v = u & 7;
      const bool isq = head < nh;
      const float rs = isq ? rq : rk;
      const __nv_bfloat16* w = isq ? qw + head * kQKD : kw + (head - nh) * kQKD;
      float a[8], b[8], wa[8], wb[8], c[8], s[8], ya[8], yb[8], o1[8], o2[8];
      unpack8(ca[k], a);
      unpack8(cb[k], b);
      unpack8(ld8(w + v * 8), wa);
      unpack8(ld8(w + kQKD / 2 + v * 8), wb);
      load_table(cs, sn, pos, kQKD / 2, v, c, s);
#pragma unroll
      for (int j = 0; j < 8; ++j) {   // one rounding, as the RMSNorm forward: bf16(x * rstd * w)
        ya[j] = round_bf16(a[j] * rs * wa[j]);
        yb[j] = round_bf16(b[j] * rs * wb[j]);
      }
      rotate(ya, yb, c, s, o1, o2);
      const int off = head * kQKD + v * 8;
      st8(row + off, pack8(o1));
      st8(row + off + kQKD / 2, pack8(o2));
    }
  }
}

template <int NU>
__global__ void __launch_bounds__(kFullThreads) qk_norm_full_rope_bwd_kernel(
    __nv_bfloat16* __restrict__ dqkv, const __nv_bfloat16* __restrict__ x_save, const float* __restrict__ rstd,
    const __nv_bfloat16* __restrict__ qw, const __nv_bfloat16* __restrict__ kw, const float* __restrict__ cs,
    const float* __restrict__ sn, float* __restrict__ dw_partial, long long T, int S, int n_heads, int nh, int nkv,
    int per_token) {
  __shared__ float red[2][32];
  const int nqk = nh + nkv, units = nqk * 8;
  const float inv_nq = 1.f / (float)(nh * kQKD), inv_nk = 1.f / (float)(nkv * kQKD);
  // gain-gradient partials of this thread's units: [0, 8) first half, [8, 16) second half
  float acc[NU][16];
#pragma unroll
  for (int k = 0; k < NU; ++k)
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[k][j] = 0.f;
  for (long long t = blockIdx.x; t < T; t += gridDim.x) {
    __nv_bfloat16* row = dqkv + t * n_heads * (long long)kQKD;
    const __nv_bfloat16* xrow = x_save + t * nqk * (long long)kQKD;
    const float rq = rstd[2 * t], rk = rstd[2 * t + 1];
    const long long pos = rope_row(t, S, per_token);
    bf16x8 ga8[NU], gb8[NU], xa8[NU], xb8[NU];   // the row's dy and x, re-expanded after the reduction
    float dotq = 0.f, dotk = 0.f;
#pragma unroll
    for (int k = 0; k < NU; ++k) {
      const int u = threadIdx.x + k * kFullThreads;
      if (u < units) {
        const int head = u >> 3, v = u & 7;
        const bool isq = head < nh;
        const int off = head * kQKD + v * 8;
        ga8[k] = ld8(row + off);
        gb8[k] = ld8(row + off + kQKD / 2);
        xa8[k] = ld8(xrow + off);
        xb8[k] = ld8(xrow + off + kQKD / 2);
        const float rs = isq ? rq : rk;
        const __nv_bfloat16* w = isq ? qw + head * kQKD : kw + (head - nh) * kQKD;
        float a[8], b[8], xa[8], xb[8], wa[8], wb[8], c[8], s[8], dya[8], dyb[8], dot = 0.f;
        unpack8(ga8[k], a);
        unpack8(gb8[k], b);
        unpack8(xa8[k], xa);
        unpack8(xb8[k], xb);
        unpack8(ld8(w + v * 8), wa);
        unpack8(ld8(w + kQKD / 2 + v * 8), wb);
        load_table(cs, sn, pos, kQKD / 2, v, c, s);
        rotate_inv(a, b, c, s, dya, dyb);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float ha = xa[j] * rs, hb = xb[j] * rs;
          dot += dya[j] * wa[j] * ha + dyb[j] * wb[j] * hb;
          acc[k][j] += dya[j] * ha;
          acc[k][8 + j] += dyb[j] * hb;
        }
        if (isq) dotq += dot;
        else dotk += dot;
      }
    }
    const float2 dot = block_reduce2<false>(dotq, dotk, red);
    const float mq = dot.x * inv_nq, mk = dot.y * inv_nk;
#pragma unroll
    for (int k = 0; k < NU; ++k) {
      const int u = threadIdx.x + k * kFullThreads;
      if (u < units) {
        const int head = u >> 3, v = u & 7;
        const bool isq = head < nh;
        const float rs = isq ? rq : rk, m = isq ? mq : mk;
        const __nv_bfloat16* w = isq ? qw + head * kQKD : kw + (head - nh) * kQKD;
        float a[8], b[8], xa[8], xb[8], wa[8], wb[8], c[8], s[8], dya[8], dyb[8], o1[8], o2[8];
        unpack8(ga8[k], a);
        unpack8(gb8[k], b);
        unpack8(xa8[k], xa);
        unpack8(xb8[k], xb);
        unpack8(ld8(w + v * 8), wa);
        unpack8(ld8(w + kQKD / 2 + v * 8), wb);
        load_table(cs, sn, pos, kQKD / 2, v, c, s);
        rotate_inv(a, b, c, s, dya, dyb);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          o1[j] = rs * (dya[j] * wa[j] - xa[j] * rs * m);
          o2[j] = rs * (dyb[j] * wb[j] - xb[j] * rs * m);
        }
        const int off = head * kQKD + v * 8;
        st8(row + off, pack8(o1));
        st8(row + off + kQKD / 2, pack8(o2));
      }
    }
  }
  const int W = nqk * kQKD;
#pragma unroll
  for (int k = 0; k < NU; ++k) {
    const int u = threadIdx.x + k * kFullThreads;
    if (u < units) {
      float* dst = dw_partial + (size_t)blockIdx.x * W + (u >> 3) * kQKD + (u & 7) * 8;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float4* d4 = reinterpret_cast<float4*>(dst + h * (kQKD / 2));
        d4[0] = make_float4(acc[k][8 * h + 0], acc[k][8 * h + 1], acc[k][8 * h + 2], acc[k][8 * h + 3]);
        d4[1] = make_float4(acc[k][8 * h + 4], acc[k][8 * h + 5], acc[k][8 * h + 6], acc[k][8 * h + 7]);
      }
    }
  }
}

int qk_norm_full_rope_max_heads() { return kFullMaxUnits * kFullThreads / 8; }

// one wave of resident CTAs: every CTA writes one [(nh + nkv) * 128] partial row, so more CTAs cost partial traffic
int qk_norm_full_rope_bwd_grid(long long T, int nqk) {
  static int per_sm[kFullMaxUnits + 1] = {0, 0, 0, 0};
  int n = 0;
  with_units(nqk, [&](auto nu) {
    constexpr int NU = decltype(nu)::value;
    if (per_sm[NU] == 0)
      DTG_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm[NU], qk_norm_full_rope_bwd_kernel<NU>,
                                                                   kFullThreads, 0));
    n = per_sm[NU];
  });
  long long g = (long long)(n < 1 ? 1 : n) * sm_count();
  if (g > T) g = T;
  return (int)(g < 1 ? 1 : g);
}

void qk_norm_full_rope_fwd(void* qkv, const void* q_w, const void* k_w, const float* cos, const float* sin,
                           void* x_save, float* rstd, long long T, int S, int n_heads, int nh, int nkv, bool per_token,
                           float eps, cudaStream_t s) {
  if (T == 0) return;
  with_units(nh + nkv, [&](auto nu) {
    qk_norm_full_rope_fwd_kernel<decltype(nu)::value><<<(unsigned)T, kFullThreads, 0, s>>>(
        (__nv_bfloat16*)qkv, (const __nv_bfloat16*)q_w, (const __nv_bfloat16*)k_w, cos, sin, (__nv_bfloat16*)x_save,
        rstd, S, n_heads, nh, nkv, per_token ? 1 : 0, eps);
  });
  note_launch();
  DTG_LAUNCH_CHECK();
}

void qk_norm_full_rope_bwd(void* dqkv, const void* x_save, const float* rstd, const void* q_w, const void* k_w,
                           const float* cos, const float* sin, float* dw_partial, float* dw, long long T, int S,
                           int n_heads, int nh, int nkv, bool per_token, cudaStream_t s) {
  const int W = (nh + nkv) * kQKD;
  if (T == 0) {
    DTG_CUDA_CHECK(cudaMemsetAsync(dw, 0, W * sizeof(float), s));
    return;
  }
  const int grid = qk_norm_full_rope_bwd_grid(T, nh + nkv);
  with_units(nh + nkv, [&](auto nu) {
    qk_norm_full_rope_bwd_kernel<decltype(nu)::value><<<grid, kFullThreads, 0, s>>>(
        (__nv_bfloat16*)dqkv, (const __nv_bfloat16*)x_save, rstd, (const __nv_bfloat16*)q_w,
        (const __nv_bfloat16*)k_w, cos, sin, dw_partial, T, S, n_heads, nh, nkv, per_token ? 1 : 0);
  });
  note_launch();
  DTG_LAUNCH_CHECK();
  colsum(dw_partial, dw, grid, W, s);
}

}  // namespace dtg
