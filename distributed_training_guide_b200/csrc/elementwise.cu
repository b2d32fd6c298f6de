// Memory-bound ops of the Llama step, hand-written for sm_90a:
//   fused (residual add +) RMSNorm fwd / bwd, in-place RoPE on the fused qkv activation,
//   SwiGLU fwd / bwd, embedding gather / scatter-add, scalar scale, the bias gradient (column sums).
// All are pure-bandwidth kernels: 16-byte vector accesses, fp32 math in registers, one pass
// over the activations (the row is cached in registers between the statistic and the
// normalisation).  Replaces the ~6 ATen kernels per RMSNorm / ~10 per RoPE the reference runs
// in eager chapters, and Inductor's Triton fusions in compiled ones (SURVEY.md K4-K6, K9, K10).
#include "api.h"
#include "common.cuh"

namespace dtg {

// ------------------------------------------------------------------------------------------
// RMSNorm forward:  h = x (+ r);  y = h * rsqrt(mean(h^2) + eps) * w
// one CTA per row; each thread keeps its slice of the row in registers (<= kMaxVec 16B vectors)
// ------------------------------------------------------------------------------------------
// NV = 16-byte vectors cached per thread, NT = threads per CTA; NV*NT*8 >= H.
template <int kMaxVec, int kNormThreads, bool HAS_RES>
__global__ void __launch_bounds__(kNormThreads) rmsnorm_fwd_kernel(
    const __nv_bfloat16* __restrict__ x, const __nv_bfloat16* __restrict__ r, const __nv_bfloat16* __restrict__ w,
    __nv_bfloat16* __restrict__ y, __nv_bfloat16* __restrict__ h_out, float* __restrict__ rstd_out, int H,
    float eps) {
  __shared__ float red[32];
  const int row = blockIdx.x;
  const int nvec = H >> 3;
  const __nv_bfloat16* xr = x + (size_t)row * H;
  const __nv_bfloat16* rr = HAS_RES ? r + (size_t)row * H : nullptr;
  bf16x8 cache[kMaxVec];
  float ss = 0.f;
#pragma unroll
  for (int k = 0; k < kMaxVec; ++k) {
    const int i = threadIdx.x + k * kNormThreads;
    if (i < nvec) {
      bf16x8 v = ld8(xr + i * 8);
      float f[8];
      unpack8(v, f);
      if (HAS_RES) {
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
      for (int j = 0; j < 8; ++j) ss += f[j] * f[j];
    }
  }
  ss = block_sum(ss, red);
  const float rstd = rsqrtf(ss / (float)H + eps);
  if (threadIdx.x == 0) rstd_out[row] = rstd;
#pragma unroll
  for (int k = 0; k < kMaxVec; ++k) {
    const int i = threadIdx.x + k * kNormThreads;
    if (i < nvec) {
      float f[8], g[8];
      unpack8(cache[k], f);
      unpack8(ld8(w + i * 8), g);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = f[j] * rstd * g[j];
      st8(y + (size_t)row * H + i * 8, pack8(f));
    }
  }
}

// Pick (NV, NT) for a hidden size: 128 threads up to H=8192, 256 threads up to 16384.
#define DTG_NORM_DISPATCH(H, CALL)                                         \
  do {                                                                     \
    const int nvec_ = (H) >> 3;                                            \
    if (nvec_ <= 128) { CALL(1, 128); }                                    \
    else if (nvec_ <= 256) { CALL(2, 128); }                               \
    else if (nvec_ <= 512) { CALL(4, 128); }                               \
    else if (nvec_ <= 1024) { CALL(8, 128); }                              \
    else if (nvec_ <= 2048) { CALL(8, 256); }                              \
    else throw std::runtime_error("rmsnorm: hidden size > 16384 unsupported"); \
  } while (0)

void rmsnorm_fwd(const void* x, const void* res, const void* w, void* y, void* h_out, float* rstd, int T, int H,
                 float eps, cudaStream_t s) {
  if (H % 8 != 0) throw std::runtime_error("rmsnorm: hidden size must be a multiple of 8");
  auto X = (const __nv_bfloat16*)x;
  auto R = (const __nv_bfloat16*)res;
  auto W = (const __nv_bfloat16*)w;
#define CALL_FWD(NV, NT)                                                                                       \
  if (res)                                                                                                     \
    rmsnorm_fwd_kernel<NV, NT, true><<<T, NT, 0, s>>>(X, R, W, (__nv_bfloat16*)y, (__nv_bfloat16*)h_out, rstd, H, eps); \
  else                                                                                                         \
    rmsnorm_fwd_kernel<NV, NT, false><<<T, NT, 0, s>>>(X, R, W, (__nv_bfloat16*)y, nullptr, rstd, H, eps);
  DTG_NORM_DISPATCH(H, CALL_FWD);
#undef CALL_FWD
  note_launch();
  DTG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// RMSNorm backward.  xhat = h*rstd, g = dy*w:
//   dx = rstd * (g - xhat * mean(g*xhat)) (+ dres),   dw = sum_rows dy * xhat
// Persistent CTAs stride over rows and keep their dw partial in registers; partials go to a
// [grid, H] fp32 scratch reduced by a second kernel (deterministic, no atomics).
// ------------------------------------------------------------------------------------------
template <int kMaxVec, int kNormThreads, bool HAS_DRES>
__global__ void __launch_bounds__(kNormThreads) rmsnorm_bwd_kernel(
    const __nv_bfloat16* __restrict__ dy, const __nv_bfloat16* __restrict__ h, const __nv_bfloat16* __restrict__ w,
    const float* __restrict__ rstd, const __nv_bfloat16* __restrict__ dres, __nv_bfloat16* __restrict__ dx,
    float* __restrict__ dw_partial, int T, int H) {
  __shared__ float red[32];
  const int nvec = H >> 3;
  float dw_acc[kMaxVec][8];
#pragma unroll
  for (int k = 0; k < kMaxVec; ++k)
#pragma unroll
    for (int j = 0; j < 8; ++j) dw_acc[k][j] = 0.f;

  for (int row = blockIdx.x; row < T; row += gridDim.x) {
    const float rs = rstd[row];
    const size_t base = (size_t)row * H;
    float dot = 0.f;
    bf16x8 cg[kMaxVec], cx[kMaxVec];  // g = dy*w (as bf16-rounded dy and fp32 recompute) / h
#pragma unroll
    for (int k = 0; k < kMaxVec; ++k) {
      const int i = threadIdx.x + k * kNormThreads;
      if (i < nvec) {
        cg[k] = ld8(dy + base + i * 8);
        cx[k] = ld8(h + base + i * 8);
        float fdy[8], fx[8], fw[8];
        unpack8(cg[k], fdy);
        unpack8(cx[k], fx);
        unpack8(ld8(w + i * 8), fw);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const float xhat = fx[j] * rs;
          dot += fdy[j] * fw[j] * xhat;
          dw_acc[k][j] += fdy[j] * xhat;
        }
      }
    }
    dot = block_sum(dot, red) / (float)H;
#pragma unroll
    for (int k = 0; k < kMaxVec; ++k) {
      const int i = threadIdx.x + k * kNormThreads;
      if (i < nvec) {
        float fdy[8], fx[8], fw[8], out[8];
        unpack8(cg[k], fdy);
        unpack8(cx[k], fx);
        unpack8(ld8(w + i * 8), fw);
#pragma unroll
        for (int j = 0; j < 8; ++j) out[j] = rs * (fdy[j] * fw[j] - fx[j] * rs * dot);
        if (HAS_DRES) {
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
  for (int k = 0; k < kMaxVec; ++k) {
    const int i = threadIdx.x + k * kNormThreads;
    if (i < nvec) {
      float4* dst = reinterpret_cast<float4*>(dw_partial + (size_t)blockIdx.x * H + i * 8);
      dst[0] = make_float4(dw_acc[k][0], dw_acc[k][1], dw_acc[k][2], dw_acc[k][3]);
      dst[1] = make_float4(dw_acc[k][4], dw_acc[k][5], dw_acc[k][6], dw_acc[k][7]);
    }
  }
}

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

// enough CTAs in flight to cover HBM latency (each keeps a dw partial in registers; the partials cost
// grid*H*4 bytes of extra traffic, 19 MB at H=4096)
int rmsnorm_bwd_grid(int T) { return T < 8 * sm_count() ? T : 8 * sm_count(); }

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

void rmsnorm_bwd(const void* dy, const void* h, const void* w, const float* rstd, const void* dres, void* dx,
                 float* dw_partial, float* dw, int T, int H, cudaStream_t s) {
  if (H % 8 != 0) throw std::runtime_error("rmsnorm: hidden size must be a multiple of 8");
  const int grid = rmsnorm_bwd_grid(T);
  auto DY = (const __nv_bfloat16*)dy;
  auto HH = (const __nv_bfloat16*)h;
  auto W = (const __nv_bfloat16*)w;
  auto DR = (const __nv_bfloat16*)dres;
#define CALL_BWD(NV, NT)                                                                                          \
  if (dres)                                                                                                       \
    rmsnorm_bwd_kernel<NV, NT, true><<<grid, NT, 0, s>>>(DY, HH, W, rstd, DR, (__nv_bfloat16*)dx, dw_partial, T, H); \
  else                                                                                                            \
    rmsnorm_bwd_kernel<NV, NT, false><<<grid, NT, 0, s>>>(DY, HH, W, rstd, nullptr, (__nv_bfloat16*)dx, dw_partial, T, H);
  DTG_NORM_DISPATCH(H, CALL_BWD);
#undef CALL_BWD
  colsum_kernel<<<(H + 31) / 32, 256, 0, s>>>(dw_partial, dw, grid, H);
  note_launch(2);
  DTG_LAUNCH_CHECK();
}

// ------------------------------------------------------------------------------------------
// RoPE (half-rotation layout) in place on heads [0, n_rot) of qkv [T, n_heads, d].
// cos/sin: fp32 [S, d/2] (pos = t % S) or per-token [T, d/2].
// ------------------------------------------------------------------------------------------
__global__ void rope_inplace_kernel(__nv_bfloat16* __restrict__ qkv, const float* __restrict__ cs,
                                    const float* __restrict__ sn, long long T, int S, int n_heads, int n_rot, int d,
                                    int per_token, float sign) {
  const int d2 = d >> 1;
  const int vec_per_head = d2 >> 3;  // 8-wide vectors in one half
  const long long total = T * (long long)n_rot * vec_per_head;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const int v = (int)(idx % vec_per_head);
    const long long th = idx / vec_per_head;
    const int head = (int)(th % n_rot);
    const long long t = th / n_rot;
    const long long pos = per_token ? t : (t % S);
    __nv_bfloat16* p = qkv + (t * n_heads + head) * (long long)d + v * 8;
    float a[8], b[8], c[8], s[8];
    unpack8(ld8(p), a);
    unpack8(ld8(p + d2), b);
    const float4* cp = reinterpret_cast<const float4*>(cs + pos * d2 + v * 8);
    const float4* sp = reinterpret_cast<const float4*>(sn + pos * d2 + v * 8);
    float4 c0 = cp[0], c1 = cp[1], s0 = sp[0], s1 = sp[1];
    c[0] = c0.x; c[1] = c0.y; c[2] = c0.z; c[3] = c0.w; c[4] = c1.x; c[5] = c1.y; c[6] = c1.z; c[7] = c1.w;
    s[0] = s0.x; s[1] = s0.y; s[2] = s0.z; s[3] = s0.w; s[4] = s1.x; s[5] = s1.y; s[6] = s1.z; s[7] = s1.w;
    float o1[8], o2[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float sj = s[j] * sign;
      o1[j] = a[j] * c[j] - b[j] * sj;
      o2[j] = b[j] * c[j] + a[j] * sj;
    }
    st8(p, pack8(o1));
    st8(p + d2, pack8(o2));
  }
}

void rope_inplace(void* qkv, const float* cos, const float* sin, long long T, int S, int n_heads, int n_rot, int d,
                  bool per_token, bool inverse, cudaStream_t s) {
  if (d % 16 != 0) throw std::runtime_error("rope: head_dim must be a multiple of 16");
  const long long total = T * (long long)n_rot * (d / 16);
  int grid = (int)((total + 255) / 256);
  const int cap = sm_count() * 16;
  if (grid > cap) grid = cap;
  if (grid < 1) grid = 1;
  rope_inplace_kernel<<<grid, 256, 0, s>>>((__nv_bfloat16*)qkv, cos, sin, T, S, n_heads, n_rot, d, per_token ? 1 : 0,
                                           inverse ? -1.f : 1.f);
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

static int ew_grid(long long total_threads) {
  long long g = (total_threads + 255) / 256;
  const long long cap = (long long)sm_count() * 16;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
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
