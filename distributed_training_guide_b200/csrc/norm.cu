// Row norms of every model family on one forward and one backward kernel template, sm_90a:
//   RMSNorm     y = h * rstd * w,                       rstd = rsqrt(mean(h^2) + eps)
//   LayerNorm   y = bf16((h - mean) * rstd * w + b),    rstd = rsqrt(var(h) + eps)  (StarCoder2)
//   LayerNorm2  two such outputs (w1, b1), (w2, b2) from one statistic (GPT-NeoX's parallel residual)
// with h = x, h = bf16(x + r) stored and normalised (add-before), or, for RMSNorm, h = bf16(r + bf16(y)) stored
// instead of y (add-after, OLMo 2's post-sublayer norms).  The forward runs one CTA per row, the row cached in
// registers as 16-byte vectors between the statistic and the normalisation; the backward strides persistent CTAs
// over rows and writes fp32 gain (and bias) gradient partial rows that colsum adds in a fixed order (no atomics).
// Each variant's per-element expressions are spelled out under `if constexpr` rather than folded into one formula
// with neutral values: x * y + 0 turns -0 into +0 and changes what nvcc contracts into an FFMA, so it changes bits.
#include <type_traits>

#include "api.h"
#include "common.cuh"

namespace dtg {
namespace {

constexpr bool is_ln(NormKind k) { return k != NormKind::kRms; }

// A LayerNorm row whose sums overflow fp32 (elements near the bf16 limit) is redone scaled by kSumSqDown (2^-72,
// common.cuh); mean and rstd are saved in the row's own units.  In the backward h - mean can only overflow when rstd
// is below 2^-121, so rows with rstd < 2^-100 recompute xhat from h and mean scaled likewise.

// ------------------------------------------------------------------------------------------
// Launch table: (NV 16-byte vectors per thread, NT threads per CTA); a hidden size H takes the first row with
// NV * NT * 8 >= H, and a variant's largest H is its last row's.  The forward uses 128 threads up to H 8192, then
// 256 up to 16384 (the dual LayerNorm stops at 8192).  The backward keeps fp32 gradient partials in registers:
// RMSNorm one plane (dw) at the forward's widths; LayerNorm two (dw, db), so above H 4096 the row spreads over
// 256 or 512 threads instead of more registers; the dual LayerNorm four (dw1, db1, dw2, db2), at most 2 vectors a
// thread over up to 512 threads.  No instantiation spills.
// ------------------------------------------------------------------------------------------
struct Width {
  int nv, nt;
};

constexpr Width norm_width(NormKind k, bool bwd, int i) {
  constexpr Width fwd[] = {{1, 128}, {2, 128}, {4, 128}, {8, 128}, {8, 256}};
  constexpr Width ln_bwd[] = {{1, 128}, {2, 128}, {4, 128}, {4, 256}, {4, 512}};
  constexpr Width ln2_bwd[] = {{1, 128}, {2, 128}, {2, 256}, {2, 512}};
  if (k == NormKind::kLn2) return bwd ? (i < 4 ? ln2_bwd[i] : Width{0, 0}) : (i < 4 ? fwd[i] : Width{0, 0});
  if (k == NormKind::kLn && bwd) return i < 5 ? ln_bwd[i] : Width{0, 0};
  return i < 5 ? fwd[i] : Width{0, 0};
}

// Calls f(NV, NT), as std::integral_constants, with the row of the table that fits H.
template <NormKind K, bool BWD, int I = 0, class F>
void with_width(int H, F&& f) {
  constexpr Width w = norm_width(K, BWD, I);
  if constexpr (w.nv == 0) {
    throw std::runtime_error("norm: hidden size " + std::to_string(H) + " is above the launch table");
  } else if (H <= w.nv * w.nt * 8) {
    f(std::integral_constant<int, w.nv>(), std::integral_constant<int, w.nt>());
  } else {
    with_width<K, BWD, I + 1>(H, f);
  }
}

// this thread's sum of h * scale, and of (h * scale - mean)^2, over its cached vectors
template <int NV, int NT>
__device__ __forceinline__ float ln_sum(const bf16x8 (&cache)[NV], int nvec, float scale) {
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (threadIdx.x + k * NT < nvec) {
      float f[8];
      unpack8(cache[k], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) s += f[j] * scale;
    }
  }
  return s;
}
template <int NV, int NT>
__device__ __forceinline__ float ln_sq_dev(const bf16x8 (&cache)[NV], int nvec, float mean, float scale) {
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    if (threadIdx.x + k * NT < nvec) {
      float f[8];
      unpack8(cache[k], f);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float d = f[j] * scale - mean;
        s += d * d;
      }
    }
  }
  return s;
}

// y = bf16((h * scale - mean) * rstd * w + b) for one cached vector
__device__ __forceinline__ void ln_affine(const float (&f)[8], float scale, float mean, float rstd,
                                          const __nv_bfloat16* __restrict__ w, const __nv_bfloat16* __restrict__ b,
                                          __nv_bfloat16* __restrict__ y) {
  float g[8], c[8], o[8];
  unpack8(ld8(w), g);
  unpack8(ld8(b), c);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[j] = (f[j] * scale - mean) * rstd * g[j] + c[j];
  st8(y, pack8(o));
}

__device__ __forceinline__ void st_partial8(float* p, const float (&a)[8]) {
  float4* dst = reinterpret_cast<float4*>(p);
  dst[0] = make_float4(a[0], a[1], a[2], a[3]);
  dst[1] = make_float4(a[4], a[5], a[6], a[7]);
}

// ------------------------------------------------------------------------------------------
// Forward.  Operands a variant does not use are null: b1, w2, b2, y2 and mean for RMSNorm, w2, b2 and y2 for
// LayerNorm, r and h_out without a residual, y1 for add-after.
// ------------------------------------------------------------------------------------------
template <NormKind K, NormRes R, int NV, int NT>
__global__ void __launch_bounds__(NT) norm_fwd_kernel(
    const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ r, const __nv_bfloat16* __restrict__ w1,
    const __nv_bfloat16* __restrict__ b1, const __nv_bfloat16* __restrict__ w2, const __nv_bfloat16* __restrict__ b2,
    __nv_bfloat16* __restrict__ y1, __nv_bfloat16* __restrict__ y2, __nv_bfloat16* __restrict__ h_out,
    float* __restrict__ mean_out, float* __restrict__ rstd_out, int H, float eps) {
  static_assert(K == NormKind::kRms || R != NormRes::kAddAfter, "norm-then-add is an RMSNorm variant");
  __shared__ float red[32];
  const int row = blockIdx.x;
  const int nvec = H >> 3;
  const __nv_bfloat16* xr = x + (size_t)row * H;
  const __nv_bfloat16* rr = R == NormRes::kAddBefore ? r + (size_t)row * H : nullptr;
  bf16x8 cache[NV];
  float s = 0.f;   // sum of h^2 (RMSNorm) or of h (LayerNorm)
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = threadIdx.x + k * NT;
    if (i < nvec) {
      bf16x8 v = ld8(xr + i * 8);
      float f[8];
      unpack8(v, f);
      if constexpr (R == NormRes::kAddBefore) {
        float g[8];
        unpack8(ld8(rr + i * 8), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += g[j];
        v = pack8(f);          // the residual stream is stored (and normalised) in bf16
        unpack8(v, f);
        st8(h_out + (size_t)row * H + i * 8, v);
      }
      cache[k] = v;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if constexpr (is_ln(K)) s += f[j];
        else s += f[j] * f[j];
      }
    }
  }
  float scale = 1.f, mean = 0.f, rstd;
  if constexpr (is_ln(K)) {
    mean = block_sum(s, red) / (float)H;
    float ss = block_sum(ln_sq_dev<NV, NT>(cache, nvec, mean, 1.f), red);
    if (!(isfinite(mean) && isfinite(ss))) {   // uniform over the CTA: block_sum broadcasts
      scale = kSumSqDown;
      mean = block_sum(ln_sum<NV, NT>(cache, nvec, kSumSqDown), red) / (float)H;
      ss = block_sum(ln_sq_dev<NV, NT>(cache, nvec, mean, kSumSqDown), red);
    }
    rstd = rsqrtf(ss / (float)H + eps * scale * scale);
    if (threadIdx.x == 0) {
      mean_out[row] = scale == 1.f ? mean : mean * kSumSqUp;
      rstd_out[row] = scale == 1.f ? rstd : rstd * kSumSqDown;
    }
  } else {
    s = block_sum(s, red);
    rstd = rsqrtf(s / (float)H + eps);
    if (threadIdx.x == 0) rstd_out[row] = rstd;
  }
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = threadIdx.x + k * NT;
    if (i < nvec) {
      float f[8];
      unpack8(cache[k], f);
      if constexpr (is_ln(K)) {
        ln_affine(f, scale, mean, rstd, w1 + i * 8, b1 + i * 8, y1 + (size_t)row * H + i * 8);
        if constexpr (K == NormKind::kLn2) ln_affine(f, scale, mean, rstd, w2 + i * 8, b2 + i * 8, y2 + (size_t)row * H + i * 8);
      } else if constexpr (R == NormRes::kAddAfter) {
        float g[8], fr[8];
        unpack8(ld8(w1 + i * 8), g);
        unpack8(ld8(r + (size_t)row * H + i * 8), fr);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = f[j] * rstd * g[j];
        unpack8(pack8(f), f);   // the normalised branch is rounded to bf16 before the add
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] += fr[j];
        st8(h_out + (size_t)row * H + i * 8, pack8(f));
      } else {
        float g[8];
        unpack8(ld8(w1 + i * 8), g);
#pragma unroll
        for (int j = 0; j < 8; ++j) f[j] = f[j] * rstd * g[j];
        st8(y1 + (size_t)row * H + i * 8, pack8(f));
      }
    }
  }
}

// ------------------------------------------------------------------------------------------
// Backward.  xhat = h * rstd (RMSNorm) or (h - mean) * rstd, g = dy * w, or dy1 * w1 + dy2 * w2 for LayerNorm2:
//   RMSNorm    dx = rstd * (g - xhat * mean(g * xhat)) (+ dres),            dw = sum_rows dy * xhat
//   LayerNorm  dx = rstd * (g - mean(g) - xhat * mean(g * xhat)) (+ dres),  dw_q = sum_rows dy_q * xhat,
//              db_q = sum_rows dy_q
// partial: [norm_grad_planes(K), gridDim.x, H] fp32, one row per CTA and plane.  dy2 and w2 are null but for
// LayerNorm2, mean for RMSNorm.
// ------------------------------------------------------------------------------------------
template <NormKind K, bool HAS_DRES, int NV, int NT>
__global__ void __launch_bounds__(NT) norm_bwd_kernel(
    const __nv_bfloat16* __restrict__ dy1, const __nv_bfloat16* __restrict__ dy2, const __nv_bfloat16* __restrict__ h,
    const __nv_bfloat16* __restrict__ w1, const __nv_bfloat16* __restrict__ w2, const float* __restrict__ mean,
    const float* __restrict__ rstd, const __nv_bfloat16* __restrict__ dres, __nv_bfloat16* __restrict__ dx,
    float* __restrict__ partial, int T, int H) {
  constexpr bool kTwo = K == NormKind::kLn2;
  constexpr int kPlanes = norm_grad_planes(K);
  // The dual LayerNorm reads h again in its second pass: 8 registers fewer, so it does not spill at 512 threads.
  constexpr bool kCacheH = !kTwo;
  __shared__ float red[32];
  const int nvec = H >> 3;
  float* planes[kPlanes];   // taken before the row loop: after it they cost the LayerNorm backward at NV 1 8 registers
#pragma unroll
  for (int q = 0; q < kPlanes; ++q) planes[q] = partial + (size_t)q * gridDim.x * H;
  float acc[kPlanes][NV][8];   // dw; or dw, db; or dw1, db1, dw2, db2
#pragma unroll
  for (int q = 0; q < kPlanes; ++q)
#pragma unroll
    for (int k = 0; k < NV; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[q][k][j] = 0.f;

  for (int row = blockIdx.x; row < T; row += gridDim.x) {
    float rs = rstd[row], mu = 0.f, scale = 1.f;
    if constexpr (is_ln(K)) {
      mu = mean[row];
      if (rs < 0x1p-100f) {
        scale = kSumSqDown;
        mu *= kSumSqDown;
        rs *= kSumSqUp;
      }
    }
    const size_t base = (size_t)row * H;
    float sg = 0.f, sgx = 0.f;   // sums of g and of g * xhat
    bf16x8 c1[NV], c2[kTwo ? NV : 1], cx[kCacheH ? NV : 1];
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int i = threadIdx.x + k * NT;
      if (i < nvec) {
        float fd1[8], fd2[8], fx[8], fw1[8], fw2[8];
        c1[k] = ld8(dy1 + base + i * 8);
        if constexpr (kTwo) {
          c2[k] = ld8(dy2 + base + i * 8);
          unpack8(c1[k], fd1);
          unpack8(c2[k], fd2);
          unpack8(ld8(h + base + i * 8), fx);
          unpack8(ld8(w1 + i * 8), fw1);
          unpack8(ld8(w2 + i * 8), fw2);
        } else {
          cx[k] = ld8(h + base + i * 8);
          unpack8(c1[k], fd1);
          unpack8(cx[k], fx);
          unpack8(ld8(w1 + i * 8), fw1);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if constexpr (!is_ln(K)) {
            const float xhat = fx[j] * rs;
            sgx += fd1[j] * fw1[j] * xhat;
            acc[0][k][j] += fd1[j] * xhat;
          } else {
            const float xhat = (fx[j] * scale - mu) * rs;
            float g;
            if constexpr (kTwo) g = fd1[j] * fw1[j] + fd2[j] * fw2[j];
            else g = fd1[j] * fw1[j];
            sg += g;
            sgx += g * xhat;
            acc[0][k][j] += fd1[j] * xhat;
            acc[1][k][j] += fd1[j];
            if constexpr (kTwo) {
              acc[2][k][j] += fd2[j] * xhat;
              acc[3][k][j] += fd2[j];
            }
          }
        }
      }
    }
    if constexpr (is_ln(K)) sg = block_sum(sg, red) / (float)H;
    sgx = block_sum(sgx, red) / (float)H;
    const float rs_out = scale == 1.f ? rs : rs * kSumSqDown;   // rstd in the row's own units
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int i = threadIdx.x + k * NT;
      if (i < nvec) {
        float fd1[8], fd2[8], fx[8], fw1[8], fw2[8], out[8];
        unpack8(c1[k], fd1);
        if constexpr (kTwo) {
          unpack8(c2[k], fd2);
          unpack8(ld8(h + base + i * 8), fx);
          unpack8(ld8(w1 + i * 8), fw1);
          unpack8(ld8(w2 + i * 8), fw2);
        } else {
          unpack8(cx[k], fx);
          unpack8(ld8(w1 + i * 8), fw1);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if constexpr (!is_ln(K)) {
            out[j] = rs * (fd1[j] * fw1[j] - fx[j] * rs * sgx);
          } else {
            const float xhat = (fx[j] * scale - mu) * rs;
            if constexpr (kTwo) out[j] = rs_out * (fd1[j] * fw1[j] + fd2[j] * fw2[j] - sg - xhat * sgx);
            else out[j] = rs_out * (fd1[j] * fw1[j] - sg - xhat * sgx);
          }
        }
        if constexpr (HAS_DRES) {
          float fr[8];
          unpack8(ld8(dres + base + i * 8), fr);
#pragma unroll
          for (int j = 0; j < 8; ++j) out[j] += fr[j];
        }
        st8(dx + base + i * 8, pack8(out));
      }
    }
  }
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    const int i = threadIdx.x + k * NT;
    if (i < nvec) {
#pragma unroll
      for (int q = 0; q < kPlanes; ++q) st_partial8(planes[q] + (size_t)blockIdx.x * H + i * 8, acc[q][k]);
    }
  }
}

using bf16p = const __nv_bfloat16*;

template <NormKind K, NormRes R>
void launch_fwd(const NormFwdArgs& a, int T, int H, float eps, cudaStream_t s) {
  with_width<K, false>(H, [&](auto nv, auto nt) {
    norm_fwd_kernel<K, R, decltype(nv)::value, decltype(nt)::value><<<T, decltype(nt)::value, 0, s>>>(
        (bf16p)a.x, (bf16p)a.r, (bf16p)a.w[0], (bf16p)a.b[0], (bf16p)a.w[1], (bf16p)a.b[1], (__nv_bfloat16*)a.y[0],
        (__nv_bfloat16*)a.y[1], (__nv_bfloat16*)a.h, a.mean, a.rstd, H, eps);
  });
}

template <NormKind K, bool HAS_DRES>
void launch_bwd(const NormBwdArgs& a, int grid, int T, int H, cudaStream_t s) {
  with_width<K, true>(H, [&](auto nv, auto nt) {
    norm_bwd_kernel<K, HAS_DRES, decltype(nv)::value, decltype(nt)::value><<<grid, decltype(nt)::value, 0, s>>>(
        (bf16p)a.dy[0], (bf16p)a.dy[1], (bf16p)a.h, (bf16p)a.w[0], (bf16p)a.w[1], a.mean, a.rstd, (bf16p)a.dres,
        (__nv_bfloat16*)a.dx, a.partial, T, H);
  });
}

void check_hidden(NormKind k, int H, const char* who) {
  if (H <= 0 || H % 8 != 0 || H > norm_max_hidden(k))
    throw std::runtime_error(std::string(who) + ": hidden size must be a positive multiple of 8 and <= " +
                             std::to_string(norm_max_hidden(k)) + ", got " + std::to_string(H));
}

}  // namespace

int norm_max_hidden(NormKind k) {
  int i = 0;
  while (norm_width(k, false, i + 1).nv != 0) ++i;
  return norm_width(k, false, i).nv * norm_width(k, false, i).nt * 8;
}

// Enough CTAs in flight to cover HBM latency while the [planes, grid, H] fp32 partials stay small: RMSNorm 8 per SM
// (19 MB at H 4096), LayerNorm 1024 threads per SM (the CTA size grows with H; 13 MB at H 6144).  The grid fixes the
// order in which colsum adds the partials, so it fixes the bits of the gradients.
int norm_bwd_grid(NormKind k, int T, int H) {
  check_hidden(k, H, "norm_bwd_grid");
  int g = 8 * sm_count();
  if (is_ln(k)) {
    int i = 0;
    while (norm_width(k, true, i).nv * norm_width(k, true, i).nt * 8 < H) ++i;
    g = sm_count() * (1024 / norm_width(k, true, i).nt);
  }
  return T < g ? T : g;
}

void norm_fwd(NormKind k, NormRes res, const NormFwdArgs& a, int T, int H, float eps, cudaStream_t s) {
  check_hidden(k, H, "norm_fwd");
  if (k == NormKind::kRms) {
    (res == NormRes::kNone       ? launch_fwd<NormKind::kRms, NormRes::kNone>
     : res == NormRes::kAddBefore ? launch_fwd<NormKind::kRms, NormRes::kAddBefore>
                                  : launch_fwd<NormKind::kRms, NormRes::kAddAfter>)(a, T, H, eps, s);
  } else {
    if (res == NormRes::kAddAfter) throw std::runtime_error("norm_fwd: norm-then-add is an RMSNorm variant");
    const bool add = res == NormRes::kAddBefore;
    if (k == NormKind::kLn)
      (add ? launch_fwd<NormKind::kLn, NormRes::kAddBefore> : launch_fwd<NormKind::kLn, NormRes::kNone>)(a, T, H, eps, s);
    else
      (add ? launch_fwd<NormKind::kLn2, NormRes::kAddBefore>
           : launch_fwd<NormKind::kLn2, NormRes::kNone>)(a, T, H, eps, s);
  }
  note_launch();
  DTG_LAUNCH_CHECK();
}

void norm_bwd(NormKind k, const NormBwdArgs& a, int T, int H, cudaStream_t s) {
  const int grid = norm_bwd_grid(k, T, H);
  const bool dres = a.dres != nullptr;
  if (k == NormKind::kRms)
    (dres ? launch_bwd<NormKind::kRms, true> : launch_bwd<NormKind::kRms, false>)(a, grid, T, H, s);
  else if (k == NormKind::kLn)
    (dres ? launch_bwd<NormKind::kLn, true> : launch_bwd<NormKind::kLn, false>)(a, grid, T, H, s);
  else
    (dres ? launch_bwd<NormKind::kLn2, true> : launch_bwd<NormKind::kLn2, false>)(a, grid, T, H, s);
  note_launch();
  DTG_LAUNCH_CHECK();
  for (int q = 0; q < norm_grad_planes(k); ++q)
    colsum(a.partial + (size_t)q * grid * H, a.dparams + (size_t)q * H, grid, H, s);
}

}  // namespace dtg
