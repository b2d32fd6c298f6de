// Memory-bound ops of the Llama step, hand-written for sm_90a: SwiGLU fwd / bwd, embedding gather / scatter-add,
//   scalar scale, the bias gradient and the fixed-order column sums the norm backwards share, GELU-tanh (StarCoder2)
//   and exact GELU fwd / bwd.  The row norms are in norm.cu, RoPE and QK-norm in rope.cu.
// All are pure-bandwidth kernels: 16-byte vector accesses, fp32 math in registers, one pass
// over the activations.  Replaces the ATen kernels the reference runs in eager chapters, and Inductor's Triton
// fusions in compiled ones (SURVEY.md K4-K6, K9, K10).
#include "api.h"
#include "common.cuh"

namespace dtg {

// out[c] = sum_r partial[r][c]: 32 columns x 8 row lanes per CTA (coalesced 128 B row segments),
// fixed summation order (deterministic)
__global__ void __launch_bounds__(256) colsum_kernel(const float* __restrict__ partial, float* __restrict__ out, int rows,
                                                     int H) {
  __shared__ float sm[8][33];
  const int c = blockIdx.x * 32 + (threadIdx.x & 31);
  const int rg = threadIdx.x >> 5;
  float s = 0.f;
  if (c < H)
    for (int r = rg; r < rows; r += 8) s += partial[(size_t)r * H + c];
  sm[rg][threadIdx.x & 31] = s;
  __syncthreads();
  if (rg == 0 && c < H) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x & 31];
    out[c] = t;
  }
}

void colsum(const float* partial, float* out, int rows, int H, cudaStream_t s) {
  colsum_kernel<<<(H + 31) / 32, 256, 0, s>>>(partial, out, rows, H);
  note_launch();
  DTG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// Bias gradient: db[n] = sum_t dy[t, n].  CTA (x, y) owns 256 columns and the y-th range of rows; its 32 x 8
// threads each sum every 8th row of the range over one 16-byte vector (8 columns) in fp32, the 8 row lanes are
// added in a fixed order through shared memory, and the CTA writes one fp32 partial row.  colsum_kernel adds the
// partial rows, again in a fixed order.  The split depends on T and N only, so every run (and every GPU) sums in
// the same order.
// ------------------------------------------------------------------------------------------
constexpr int kBiasGradCols = 256;       // columns per CTA: 32 vectors of 8
constexpr int kBiasGradMinRows = 64;     // rows per CTA at least (8 per thread)
constexpr int kBiasGradTargetCtas = 1024;

__global__ void __launch_bounds__(256) bias_grad_kernel(const __nv_bfloat16* __restrict__ dy, long long T, int N,
                                                        long long ld, long long rows_per_chunk,
                                                        float* __restrict__ partial) {
  __shared__ float sm[8][kBiasGradCols + 4];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int c0 = blockIdx.x * kBiasGradCols;
  const int col = c0 + 8 * tx;
  const long long r0 = (long long)blockIdx.y * rows_per_chunk;
  const long long r1 = r0 + rows_per_chunk < T ? r0 + rows_per_chunk : T;
  float s[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) s[k] = 0.f;
  if (col < N) {
#pragma unroll 4
    for (long long r = r0 + ty; r < r1; r += 8) {
      const uint4 v = *reinterpret_cast<const uint4*>(dy + r * ld + col);
      const __nv_bfloat162* p = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = __bfloat1622float2(p[k]);
        s[2 * k] += f.x;
        s[2 * k + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) sm[ty][8 * tx + k] = s[k];
  __syncthreads();
  const int c = c0 + (int)threadIdx.x;   // one column per thread for the fixed-order sum of the 8 row lanes
  if (c < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += sm[i][threadIdx.x];
    partial[(size_t)blockIdx.y * N + c] = t;
  }
}

int bias_grad_chunks(long long T, int N) {
  const int col_blocks = (N + kBiasGradCols - 1) / kBiasGradCols;
  long long by_rows = (T + kBiasGradMinRows - 1) / kBiasGradMinRows;
  long long by_ctas = kBiasGradTargetCtas / (col_blocks > 0 ? col_blocks : 1);
  long long c = by_rows < by_ctas ? by_rows : by_ctas;
  return (int)(c < 1 ? 1 : c);
}

void bias_grad(const void* dy, long long T, int N, long long ld, float* partial, float* db, cudaStream_t s) {
  if (N % 8 || ld % 8 || reinterpret_cast<uintptr_t>(dy) % 16)
    throw std::runtime_error("bias_grad: N and the row stride must be multiples of 8, dy 16-byte aligned");
  if (T <= 0 || N <= 0) throw std::runtime_error("bias_grad: dy must have at least one row and one column");
  const int chunks = bias_grad_chunks(T, N);
  const long long rpc = (T + chunks - 1) / chunks;
  bias_grad_kernel<<<dim3((N + kBiasGradCols - 1) / kBiasGradCols, chunks), 256, 0, s>>>(
      (const __nv_bfloat16*)dy, T, N, ld, rpc, partial);
  colsum_kernel<<<(N + 31) / 32, 256, 0, s>>>(partial, db, chunks, N);
  note_launch(2);
  DTG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// GELU, tanh approximation (StarCoder2's gelu_pytorch_tanh), elementwise on the c_fc output:
//   y = 0.5 x (1 + tanh(k (x + 0.044715 x^3))),  k = sqrt(2/pi)
// fp32 math in ATen's operation order with tanhf (not tanh.approx) and one rounding.  The backward is ATen's too,
// except that the sech^2 term is taken as 0 where tanh has saturated, where ATen's 0 * (1 + 3 * 0.044715 * x^2)
// becomes NaN once x^2 overflows.
// ------------------------------------------------------------------------------------------
constexpr float kGeluBeta = 0.7978845608028654f, kGeluKappa = 0.044715f;

__global__ void gelu_tanh_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y,
                                     long long nvec) {
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < nvec;
       idx += (long long)gridDim.x * blockDim.x) {
    float f[8], o[8];
    unpack8(ld8(x + idx * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float cube = f[j] * f[j] * f[j];
      const float inner = kGeluBeta * (f[j] + kGeluKappa * cube);
      o[j] = 0.5f * f[j] * (1.f + tanhf(inner));
    }
    st8(y + idx * 8, pack8(o));
  }
}

__global__ void gelu_tanh_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                     __nv_bfloat16* __restrict__ dx, long long nvec) {
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < nvec;
       idx += (long long)gridDim.x * blockDim.x) {
    float f[8], d[8], o[8];
    unpack8(ld8(x + idx * 8), f);
    unpack8(ld8(dy + idx * 8), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sq = f[j] * f[j];
      const float cube = sq * f[j];
      const float t = tanhf(kGeluBeta * (f[j] + kGeluKappa * cube));
      const float left = 0.5f * f[j];
      const float right = 1.f + t;
      const float sech2 = 1.f - t * t;
      const float right_d = sech2 == 0.f ? 0.f : left * sech2 * kGeluBeta * (1.f + 3.f * kGeluKappa * sq);
      o[j] = d[j] * (0.5f * right + right_d);
    }
    st8(dx + idx * 8, pack8(o));
  }
}

void gelu_tanh_fwd(const void* x, void* y, long long n, cudaStream_t s) {
  if (n % 8 != 0) throw std::runtime_error("gelu_tanh: the element count must be a multiple of 8");
  gelu_tanh_fwd_kernel<<<ew_grid(n / 8), 256, 0, s>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, n / 8);
  note_launch();
  DTG_LAUNCH_CHECK();
}

void gelu_tanh_bwd(const void* dy, const void* x, void* dx, long long n, cudaStream_t s) {
  if (n % 8 != 0) throw std::runtime_error("gelu_tanh: the element count must be a multiple of 8");
  gelu_tanh_bwd_kernel<<<ew_grid(n / 8), 256, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x,
                                                      (__nv_bfloat16*)dx, n / 8);
  note_launch();
  DTG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// GELU, exact (erf) form (GPT-NeoX's hidden_act "gelu"), elementwise on the c_fc output:
//   y = x/2 * (1 + erf(x / sqrt(2)))
// fp32 erff in ATen's operation order, one rounding.  Backward from the saved pre-activation:
//   dx = dy * (Phi(x) + x * phi(x)),  Phi(x) = (1 + erf(x / sqrt(2))) / 2,  phi(x) = exp(-x^2 / 2) / sqrt(2 pi)
// ------------------------------------------------------------------------------------------
constexpr float kSqrtHalf = 0.70710678118654752440f, kInvSqrt2Pi = 0.39894228040143267794f;

__global__ void gelu_fwd_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* __restrict__ y, long long nvec) {
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < nvec;
       idx += (long long)gridDim.x * blockDim.x) {
    float f[8], o[8];
    unpack8(ld8(x + idx * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = f[j] * 0.5f * (1.f + erff(f[j] * kSqrtHalf));
    st8(y + idx * 8, pack8(o));
  }
}

__global__ void gelu_bwd_kernel(const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ x,
                                __nv_bfloat16* __restrict__ dx, long long nvec) {
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < nvec;
       idx += (long long)gridDim.x * blockDim.x) {
    float f[8], d[8], o[8];
    unpack8(ld8(x + idx * 8), f);
    unpack8(ld8(dy + idx * 8), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float cdf = 0.5f * (1.f + erff(f[j] * kSqrtHalf));
      const float pdf = expf(-0.5f * f[j] * f[j]) * kInvSqrt2Pi;
      o[j] = d[j] * (cdf + f[j] * pdf);
    }
    st8(dx + idx * 8, pack8(o));
  }
}

void gelu_fwd(const void* x, void* y, long long n, cudaStream_t s) {
  if (n % 8 != 0) throw std::runtime_error("gelu: the element count must be a multiple of 8");
  gelu_fwd_kernel<<<ew_grid(n / 8), 256, 0, s>>>((const __nv_bfloat16*)x, (__nv_bfloat16*)y, n / 8);
  note_launch();
  DTG_LAUNCH_CHECK();
}

void gelu_bwd(const void* dy, const void* x, void* dx, long long n, cudaStream_t s) {
  if (n % 8 != 0) throw std::runtime_error("gelu: the element count must be a multiple of 8");
  gelu_bwd_kernel<<<ew_grid(n / 8), 256, 0, s>>>((const __nv_bfloat16*)dy, (const __nv_bfloat16*)x,
                                                 (__nv_bfloat16*)dx, n / 8);
  note_launch();
  DTG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// SwiGLU on gu = [gate | up]  ([T, 2I]):  h = silu(g) * u
// ------------------------------------------------------------------------------------------
__global__ void swiglu_fwd_kernel(const __nv_bfloat16* __restrict__ gu, __nv_bfloat16* __restrict__ h, long long T,
                                  int I) {
  const int vpr = I >> 3;
  const long long total = T * vpr;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long t = idx / vpr;
    const int v = (int)(idx % vpr);
    float g[8], u[8], o[8];
    unpack8(ld8(gu + t * 2 * I + v * 8), g);
    unpack8(ld8(gu + t * 2 * I + I + v * 8), u);
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = g[j] / (1.f + __expf(-g[j])) * u[j];
    st8(h + t * I + v * 8, pack8(o));
  }
}

__global__ void swiglu_bwd_kernel(const __nv_bfloat16* __restrict__ dh, const __nv_bfloat16* __restrict__ gu,
                                  __nv_bfloat16* __restrict__ dgu, long long T, int I) {
  const int vpr = I >> 3;
  const long long total = T * vpr;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long t = idx / vpr;
    const int v = (int)(idx % vpr);
    float g[8], u[8], d[8], dg[8], du[8];
    unpack8(ld8(gu + t * 2 * I + v * 8), g);
    unpack8(ld8(gu + t * 2 * I + I + v * 8), u);
    unpack8(ld8(dh + t * I + v * 8), d);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sg = 1.f / (1.f + __expf(-g[j]));
      const float silu = g[j] * sg;
      dg[j] = d[j] * u[j] * (sg + silu * (1.f - sg));
      du[j] = d[j] * silu;
    }
    st8(dgu + t * 2 * I + v * 8, pack8(dg));
    st8(dgu + t * 2 * I + I + v * 8, pack8(du));
  }
}

void swiglu_fwd(const void* gu, void* h, long long T, int I, cudaStream_t s) {
  if (I % 8 != 0) throw std::runtime_error("swiglu: intermediate size must be a multiple of 8");
  swiglu_fwd_kernel<<<ew_grid(T * (I / 8)), 256, 0, s>>>((const __nv_bfloat16*)gu, (__nv_bfloat16*)h, T, I);
  note_launch();
  DTG_LAUNCH_CHECK();
}
void swiglu_bwd(const void* dh, const void* gu, void* dgu, long long T, int I, cudaStream_t s) {
  if (I % 8 != 0) throw std::runtime_error("swiglu: intermediate size must be a multiple of 8");
  swiglu_bwd_kernel<<<ew_grid(T * (I / 8)), 256, 0, s>>>((const __nv_bfloat16*)dh, (const __nv_bfloat16*)gu,
                                                         (__nv_bfloat16*)dgu, T, I);
  note_launch();
  DTG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// Embedding gather and scatter-add
// ------------------------------------------------------------------------------------------
__global__ void embedding_fwd_kernel(const long long* __restrict__ ids, const __nv_bfloat16* __restrict__ w,
                                     __nv_bfloat16* __restrict__ out, long long T, int H) {
  const int vpr = H >> 3;
  const long long total = T * vpr;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long t = idx / vpr;
    const int v = (int)(idx % vpr);
    st8(out + t * H + v * 8, ld8(w + ids[t] * H + v * 8));
  }
}

// Default backward, summed in fp32 with one bf16 rounding per table row (a bf16 atomic per occurrence would round
// once per token, and the most frequent ids of real text occur hundreds of times per batch):
//   1. slot[id] = the first token position that holds id (atomicMin over the tokens; the table starts at ~0u);
//   2. sums[slot[ids[t]]] += dout[t] with fp32 vector atomics, into a zeroed [T, H] fp32 scratch;
//   3. the token at each id's slot writes dw[id] = bf16(sums[slot] (+ dw[id])).
// Every shape is fixed by T, H and V, so nothing waits on the host.
__global__ void embedding_slot_kernel(const long long* __restrict__ ids, unsigned int* __restrict__ slot, long long T) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < T; t += (long long)gridDim.x * blockDim.x)
    atomicMin(slot + ids[t], (unsigned int)t);
}

__global__ void embedding_sum_kernel(const __nv_bfloat16* __restrict__ dout, const long long* __restrict__ ids,
                                     const unsigned int* __restrict__ slot, float* __restrict__ sums, long long T,
                                     int H) {
  const int vpr = H >> 3;
  const long long total = T * vpr;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long t = idx / vpr;
    const int v = (int)(idx % vpr);
    float g[8];
    unpack8(ld8(dout + t * H + v * 8), g);
    float4* dst = reinterpret_cast<float4*>(sums + (long long)slot[ids[t]] * H + v * 8);
    atomicAdd(dst, make_float4(g[0], g[1], g[2], g[3]));
    atomicAdd(dst + 1, make_float4(g[4], g[5], g[6], g[7]));
  }
}

__global__ void embedding_write_kernel(const float* __restrict__ sums, const long long* __restrict__ ids,
                                       const unsigned int* __restrict__ slot, __nv_bfloat16* __restrict__ dw,
                                       long long T, int H, int accumulate) {
  const int vpr = H >> 3;
  const long long total = T * vpr;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long t = idx / vpr;
    const long long id = ids[t];
    if (slot[id] != (unsigned int)t) continue;   // a later occurrence: the first one writes the row
    const int v = (int)(idx % vpr);
    const float4* src = reinterpret_cast<const float4*>(sums + t * H + v * 8);
    const float4 a = src[0], b = src[1];
    float acc[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    if (accumulate) {
      float old[8];
      unpack8(ld8(dw + id * H + v * 8), old);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += old[j];
    }
    st8(dw + id * H + v * 8, pack8(acc));
  }
}

// Deterministic variant (--deterministic): the caller passes the token ids stably sorted with the permutation that
// sorted them; the CTA that starts a run of equal ids sums that run's gradient rows in ascending token order in
// fp32 and writes (or accumulates into) the one table row — no atomics, bit-identical from run to run.
__global__ void embedding_bwd_sorted_kernel(const __nv_bfloat16* __restrict__ dout, const long long* __restrict__ ids_sorted,
                                            const long long* __restrict__ perm, __nv_bfloat16* __restrict__ dw,
                                            long long T, int H, int accumulate) {
  const long long p0 = blockIdx.x;
  const long long id = ids_sorted[p0];
  if (p0 > 0 && ids_sorted[p0 - 1] == id) return;   // not the start of a run
  for (int c = threadIdx.x; c < (H >> 3); c += blockDim.x) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    if (accumulate) unpack8(ld8(dw + id * H + c * 8), acc);
    for (long long p = p0; p < T && ids_sorted[p] == id; ++p) {
      float g[8];
      unpack8(ld8(dout + perm[p] * H + c * 8), g);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += g[j];
    }
    st8(dw + id * H + c * 8, pack8(acc));
  }
}
void embedding_bwd_sorted(const void* dout, const long long* ids_sorted, const long long* perm, void* dw, long long T, int H,
                          bool accumulate, cudaStream_t s) {
  if (H % 8 != 0) throw std::runtime_error("embedding: hidden size must be a multiple of 8");
  if (T <= 0) return;
  embedding_bwd_sorted_kernel<<<(unsigned)T, 128, 0, s>>>((const __nv_bfloat16*)dout, ids_sorted, perm, (__nv_bfloat16*)dw, T, H,
                                                       accumulate ? 1 : 0);
  note_launch();
  DTG_LAUNCH_CHECK();
}

void embedding_fwd(const long long* ids, const void* w, void* out, long long T, int H, cudaStream_t s) {
  if (H % 8 != 0) throw std::runtime_error("embedding: hidden size must be a multiple of 8");
  embedding_fwd_kernel<<<ew_grid(T * (H / 8)), 256, 0, s>>>(ids, (const __nv_bfloat16*)w, (__nv_bfloat16*)out, T, H);
  note_launch();
  DTG_LAUNCH_CHECK();
}
void embedding_bwd(const void* dout, const long long* ids, void* dw, unsigned int* slot, float* sums, long long T,
                   long long V, int H, bool accumulate, cudaStream_t s) {
  if (H % 8 != 0) throw std::runtime_error("embedding: hidden size must be a multiple of 8");
  if (T >= 0xFFFFFFFFLL) throw std::runtime_error("embedding: too many tokens for 32-bit slots");
  if (!accumulate) DTG_CUDA_CHECK(cudaMemsetAsync(dw, 0, (size_t)V * H * sizeof(__nv_bfloat16), s));
  if (T <= 0) return;
  DTG_CUDA_CHECK(cudaMemsetAsync(slot, 0xFF, (size_t)V * sizeof(unsigned int), s));
  DTG_CUDA_CHECK(cudaMemsetAsync(sums, 0, (size_t)T * H * sizeof(float), s));
  embedding_slot_kernel<<<ew_grid(T), 256, 0, s>>>(ids, slot, T);
  embedding_sum_kernel<<<ew_grid(T * (H / 8)), 256, 0, s>>>((const __nv_bfloat16*)dout, ids, slot, sums, T, H);
  embedding_write_kernel<<<ew_grid(T * (H / 8)), 256, 0, s>>>(sums, ids, slot, (__nv_bfloat16*)dw, T, H,
                                                             accumulate ? 1 : 0);
  note_launch(3);
  DTG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// x *= *scale  (device scalar; exits immediately when the scalar is exactly 1)
// ------------------------------------------------------------------------------------------
__global__ void scale_inplace_kernel(__nv_bfloat16* __restrict__ x, const float* __restrict__ scale, long long nvec) {
  const float sc = *scale;
  if (sc == 1.0f) return;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    float f[8];
    unpack8(ld8(x + i * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= sc;
    st8(x + i * 8, pack8(f));
  }
}
void scale_inplace(void* x, const float* scale, long long n, cudaStream_t s) {
  if (n % 8 != 0) throw std::runtime_error("scale_inplace: numel must be a multiple of 8");
  scale_inplace_kernel<<<ew_grid(n / 8), 256, 0, s>>>((__nv_bfloat16*)x, scale, n / 8);
  note_launch();
  DTG_LAUNCH_CHECK();
}

}  // namespace dtg
