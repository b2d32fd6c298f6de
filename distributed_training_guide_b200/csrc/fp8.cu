// FP8 (per-tensor current scaling) casts for the fp8 GEMM of gemm_wgmma.cu:
//
//   amax            max |x| of a bf16 matrix -> one fp32 on the device
//   cast-transpose  bf16 [R, C] -> fp8 [R, C] and / or its transpose fp8 [C, R], scaled by FP8_MAX / amax, plus the
//                   dequantisation scale 1 / scale on the device
//
// The fp8 wgmma reads both operands K-major only, so each GEMM operand that the backward pass multiplies along its
// other dimension is needed in both layouts; one pass over a 128 x 128 tile staged in shared memory writes both with
// coalesced stores.  Recipe (what ops/reference.py computes with torch's float8 casts):
//   scale = amax == 0 ? 1 : FP8_MAX / amax            (correctly rounded fp32 division)
//   scale = scale > FLT_MAX ? FLT_MAX : scale         (a finite amax below FP8_MAX / FLT_MAX overflows the division)
//   q     = cvt.rn.satfinite(x * scale)               (round to nearest even, saturate finite values at +-FP8_MAX)
//   scale_inv = 1 / scale                             (2^-128, a subnormal, for the clamped scale)
// Without the clamp an Inf scale turns every zero into 0 * Inf = NaN.  The clamp is a comparison, not fminf, so a NaN
// scale stays NaN: a non-finite amax gives scale 0 or NaN, so the outputs are not all finite and the NaN / Inf
// reaches the GEMM.
#include <cuda_fp8.h>

#include <cfloat>

#include "api.h"
#include "common.cuh"

namespace dtg {

namespace {

constexpr int kCastTile = 128;
constexpr int kCastThreads = 256;
constexpr int kTilePitch = kCastTile + 4;   // 33 words per row of the staged tile

template <int FMT>
__device__ __forceinline__ uint16_t cvt_fp8x2(float lo, float hi) {
  return (uint16_t)__nv_cvt_float2_to_fp8x2(make_float2(lo, hi), __NV_SATFINITE, FMT == 1 ? __NV_E4M3 : __NV_E5M2);
}

// max over |x| as bf16 bit patterns: for non-negative numbers (sign bit cleared) the integer order is the numeric
// order, NaN patterns sort above Inf, and the fp32 value is the pattern shifted left by 16
__global__ void __launch_bounds__(256) amax_kernel(const __nv_bfloat16* __restrict__ x, long long R, int C, long long ld,
                                                   bool vec, unsigned int* __restrict__ out) {
  const uint16_t* xb = reinterpret_cast<const uint16_t*>(x);
  uint32_t m = 0;
  const long long stride = (long long)gridDim.x * blockDim.x;
  if (vec) {
    const int cv = C / 8;
    const long long total = R * cv;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
      const long long r = i / cv;
      const int c = (int)(i - r * cv) * 8;
      const uint4 v = *reinterpret_cast<const uint4*>(xb + r * ld + c);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) m = max(m, max(w[k] & 0x7FFFu, (w[k] >> 16) & 0x7FFFu));
    }
  } else {
    const long long total = R * C;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride) {
      const long long r = i / C;
      m = max(m, (uint32_t)(xb[r * ld + (i - r * C)] & 0x7FFFu));
    }
  }
  m = __reduce_max_sync(0xffffffffu, m);
  __shared__ uint32_t red[8];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[w] = m;
  __syncthreads();
  if (w == 0) {
    m = lane < (int)(blockDim.x >> 5) ? red[lane] : 0u;
    m = __reduce_max_sync(0xffffffffu, m);
    if (lane == 0 && m) atomicMax(out, m << 16);
  }
}

template <int FMT, bool ROW, bool TRANS>
__global__ void __launch_bounds__(kCastThreads) cast_transpose_kernel(const __nv_bfloat16* __restrict__ x, long long ld,
                                                                      int R, int C, bool vec, const float* __restrict__ amax,
                                                                      uint8_t* __restrict__ out, uint8_t* __restrict__ out_t,
                                                                      float* __restrict__ scale_inv) {
  constexpr float kMax = FMT == 1 ? 448.f : 57344.f;
  const float a = *amax;
  const float s = a == 0.f ? 1.f : __fdiv_rn(kMax, a);
  const float scale = s > FLT_MAX ? FLT_MAX : s;
  if (blockIdx.x == 0 && blockIdx.y == 0 && threadIdx.x == 0) *scale_inv = __fdiv_rn(1.f, scale);
  __shared__ __align__(16) uint8_t tile[kCastTile * kTilePitch];
  const int r0 = blockIdx.y * kCastTile, c0 = blockIdx.x * kCastTile;
  // rows: every thread converts runs of 8 elements of one row
#pragma unroll 2
  for (int i = threadIdx.x; i < kCastTile * kCastTile / 8; i += kCastThreads) {
    const int rr = i >> 4, cc = (i & 15) * 8;
    const int r = r0 + rr, c = c0 + cc;
    const __nv_bfloat16* src = x + (long long)r * ld + c;
    float f[8];
    const bool full = r < R && c + 8 <= C;
    if (full && vec) {
      unpack8(ld8(src), f);
    } else {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = (r < R && c + j < C) ? __bfloat162float(src[j]) : 0.f;
    }
    uint32_t q[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const uint32_t lo = cvt_fp8x2<FMT>(__fmul_rn(f[4 * k], scale), __fmul_rn(f[4 * k + 1], scale));
      const uint32_t hi = cvt_fp8x2<FMT>(__fmul_rn(f[4 * k + 2], scale), __fmul_rn(f[4 * k + 3], scale));
      q[k] = lo | (hi << 16);
    }
    if constexpr (ROW) {
      if (r < R) {
        uint8_t* dst = out + (long long)r * C + c;
        if (full && (C % 8) == 0) {
          *reinterpret_cast<uint2*>(dst) = make_uint2(q[0], q[1]);
        } else {
          for (int j = 0; j < 8 && c + j < C; ++j) dst[j] = (uint8_t)(q[j >> 2] >> (8 * (j & 3)));
        }
      }
    }
    if constexpr (TRANS) {
      uint32_t* t = reinterpret_cast<uint32_t*>(tile + rr * kTilePitch + cc);
      t[0] = q[0];
      t[1] = q[1];
    }
  }
  if constexpr (TRANS) {
    __syncthreads();
    // columns: every thread gathers 8 consecutive rows of one column; 16 threads write 128 contiguous bytes of a row
    // of the transposed output
#pragma unroll 2
    for (int i = threadIdx.x; i < kCastTile * kCastTile / 8; i += kCastThreads) {
      const int cc = i >> 4, rr = (i & 15) * 8;
      const int c = c0 + cc, r = r0 + rr;
      if (c >= C) continue;
      uint32_t q[2] = {0u, 0u};
#pragma unroll
      for (int j = 0; j < 8; ++j) q[j >> 2] |= (uint32_t)tile[(rr + j) * kTilePitch + cc] << (8 * (j & 3));
      uint8_t* dst = out_t + (long long)c * R + r;
      if (r + 8 <= R && (R % 8) == 0) {
        *reinterpret_cast<uint2*>(dst) = make_uint2(q[0], q[1]);
      } else {
        for (int j = 0; j < 8 && r + j < R; ++j) dst[j] = (uint8_t)(q[j >> 2] >> (8 * (j & 3)));
      }
    }
  }
}

template <int FMT>
void launch_cast(const void* x, long long ld, int R, int C, bool vec, const float* amax, void* out, void* out_t,
                 float* scale_inv, cudaStream_t s) {
  const dim3 grid((C + kCastTile - 1) / kCastTile, (R + kCastTile - 1) / kCastTile);
  auto* xp = static_cast<const __nv_bfloat16*>(x);
  auto* o = static_cast<uint8_t*>(out);
  auto* ot = static_cast<uint8_t*>(out_t);
  if (out && out_t) cast_transpose_kernel<FMT, true, true><<<grid, kCastThreads, 0, s>>>(xp, ld, R, C, vec, amax, o, ot, scale_inv);
  else if (out) cast_transpose_kernel<FMT, true, false><<<grid, kCastThreads, 0, s>>>(xp, ld, R, C, vec, amax, o, ot, scale_inv);
  else cast_transpose_kernel<FMT, false, true><<<grid, kCastThreads, 0, s>>>(xp, ld, R, C, vec, amax, o, ot, scale_inv);
}

}  // namespace

void fp8_amax(const void* x, long long R, int C, long long ld, float* amax, cudaStream_t s) {
  DTG_CUDA_CHECK(cudaMemsetAsync(amax, 0, sizeof(float), s));
  if (R <= 0 || C <= 0) return;
  const bool vec = (C % 8) == 0 && (ld % 8) == 0 && (reinterpret_cast<uintptr_t>(x) % 16) == 0;
  const long long work = vec ? R * (C / 8) : R * C;
  long long blocks = (work + 255) / 256;
  const long long cap = 8LL * sm_count();
  if (blocks > cap) blocks = cap;
  amax_kernel<<<(int)blocks, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(x), R, C, ld, vec,
                                          reinterpret_cast<unsigned int*>(amax));
  DTG_LAUNCH_CHECK();
  note_launch();
}

void fp8_cast_transpose(const void* x, long long ld, int R, int C, bool e5m2, const float* amax, void* out, void* out_t,
                        float* scale_inv, cudaStream_t s) {
  if (!out && !out_t) throw std::runtime_error("fp8_cast_transpose: nothing to write");
  if (R <= 0 || C <= 0) throw std::runtime_error("fp8_cast_transpose: empty tensor");
  const bool vec = (ld % 8) == 0 && (reinterpret_cast<uintptr_t>(x) % 16) == 0;
  if (e5m2) launch_cast<2>(x, ld, R, C, vec, amax, out, out_t, scale_inv, s);
  else launch_cast<1>(x, ld, R, C, vec, amax, out, out_t, scale_inv, s);
  DTG_LAUNCH_CHECK();
  note_launch();
}

}  // namespace dtg
