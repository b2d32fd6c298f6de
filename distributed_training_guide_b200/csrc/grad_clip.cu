// Global-norm gradient clipping for the data-parallel bucket engine (parallel/ddp.py), with the semantics of
// torch.nn.utils.clip_grad_norm_: norm = ||g||_2 over every parameter element of every bucket, as AdamW consumes
// it; coef = min(1, max_norm / (norm + 1e-6)); every gradient element is multiplied by coef before the update.
//
// The norm needs every bucket, so the update cannot run per bucket inside backward as rs_adamw does.  The step
// is split in three, all on the communication stream and its signal pads, with no host synchronisation:
//
//   reduce_sumsq     in backward, per bucket: reduce my 1/N slice (peer pull or NVLS multimem.ld_reduce), scale,
//                    store the bf16 result (ZeRO-1: into my slice of my own gradient buffer; all-reduce: into every
//                    replica), and square the STORED bf16 values over the parameter ranges only (never the padding
//                    between parameters or at the tail).  One fp64 partial per CTA, no atomics.
//   clip_finalize    in optimizer.step(): sum this rank's partials in a fixed order (fp64), publish the sum in a
//                    symmetric slot, one device barrier, sum every rank's slot in rank order (every rank gets the
//                    same bits), write norm and coef (fp32) to device memory.
//   adamw_clip       per bucket: g *= coef, then the shared adamw_update; push the new parameters to every replica
//                    (peer stores or multimem.st) for ZeRO-1, or update the local replica for plain DDP.
#include "adamw.cuh"
#include "comm.cuh"
#include "comm_device.cuh"
#include "common.cuh"
#include "ptx.cuh"

namespace dtg {
using namespace ptx;

namespace {

// Sum of squares of the 8 values `f` of the vector at bucket element e0, over the elements inside the parameter
// ranges [rb[r], re[r]).  `r` is the first range that ends after the previous vector: vectors of one thread come in
// increasing order, so it only moves forward.
__device__ __forceinline__ float masked_sumsq8(const float (&f)[8], size_t e0, const long long* __restrict__ ranges,
                                               int nranges, int& r) {
  while (r < nranges && (size_t)ranges[2 * r + 1] <= e0) ++r;
  float s = 0.f;
  if (r < nranges && (size_t)ranges[2 * r] <= e0 && (size_t)ranges[2 * r + 1] >= e0 + 8) {
#pragma unroll
    for (int j = 0; j < 8; ++j) s += f[j] * f[j];
    return s;
  }
  // a vector that crosses padding: find which of its elements lie in a range first, so that `f` is only ever
  // indexed with constants (it stays in registers)
  uint32_t mask = 0;
  int q = r;
  for (int j = 0; j < 8; ++j) {
    const size_t e = e0 + j;
    while (q < nranges && (size_t)ranges[2 * q + 1] <= e) ++q;
    if (q < nranges && (size_t)ranges[2 * q] <= e) mask |= 1u << j;
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) s += ((mask >> j) & 1u) ? f[j] * f[j] : 0.f;
  return s;
}

__device__ __forceinline__ void unpack_u4(const uint4& v, float (&f)[8]) {
  const __nv_bfloat162* h = reinterpret_cast<const __nv_bfloat162*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __bfloat1622float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

// The 8-element vector at byte offset `byte_off`, summed over the NR ranks in fp32 (rotated table: ptr[0] is me).
template <int NR>
__device__ __forceinline__ void gather_sum_clip(const SymmPtrs& sp, size_t byte_off, float (&acc)[8]) {
  uint4 v[NR];
#pragma unroll
  for (int k = 0; k < NR; ++k) v[k] = ld_volatile_v4(sp.ptr[k] + byte_off);
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
  for (int k = 0; k < NR; ++k) add8(acc, v[k]);
}

// Block sum in fp64 in a fixed order; thread 0 writes it to *out.
__device__ __forceinline__ void block_partial(float v, double* out) {
  __shared__ double red[kCommThreads / 32];
  double d = (double)v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) red[w] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += red[i];
    *out = s;
  }
}

}  // namespace

// ---- in backward: reduce (+ scale, store) and sum of squares, peer-pointer form -------------------------------
// BCAST=false: reduce-scatter (ZeRO-1, and one rank); the result goes to my slice of my own buffer only.
// BCAST=true:  two-shot all-reduce (plain DDP); the result goes to every replica.
template <int NR, bool BCAST>
// (minimum of one CTA per SM: without it ptxas keeps these kernels at 32 registers and spills in the NR = 2 form)
__global__ void __launch_bounds__(kCommThreads, 1) reduce_sumsq_kernel(SymmPtrs buf, SymmPads pads, size_t elem_off,
                                                                       size_t n, float scale, const long long* ranges,
                                                                       int nranges, double* partials, int rank,
                                                                       uint32_t epoch, int* err) {
  symm_barrier(pads.ptr, rank, NR, blockIdx.x, epoch, err);
  const size_t per = n / NR;
  const size_t base = (elem_off + (size_t)rank * per) * 2;
  const size_t nvec = per / 8;
  float sq = 0.f;
  int r = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float acc[8];
    gather_sum_clip<NR>(buf, base + i * 16, acc);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= scale;
    const uint4 out = pack8_u4(acc);
    if (BCAST) {
#pragma unroll
      for (int k = 0; k < NR; ++k) st_v4(buf.ptr[k] + base + i * 16, out);
    } else {
      st_v4(buf.ptr[0] + base + i * 16, out);
    }
    float stored[8];
    unpack_u4(out, stored);
    sq += masked_sumsq8(stored, (size_t)rank * per + i * 8, ranges, nranges, r);
  }
  block_partial(sq, partials + blockIdx.x);
  symm_barrier(pads.ptr, rank, NR, blockIdx.x, epoch + 1, err);
}

// ---- the same with the in-switch reduction (NVLS) --------------------------------------------------------------
template <bool BCAST>
__global__ void __launch_bounds__(kCommThreads, 1) nvls_reduce_sumsq_kernel(char* mc, char* local, SymmPads pads,
                                                                            size_t elem_off, size_t n, float scale,
                                                                            const long long* ranges, int nranges,
                                                                            double* partials, int rank, int nranks,
                                                                            uint32_t epoch, int* err) {
  symm_barrier(pads.ptr, rank, nranks, blockIdx.x, epoch, err);
  const size_t per = n / nranks;
  const size_t base = (elem_off + (size_t)rank * per) * 2;
  const size_t nvec = per / 8;
  float sq = 0.f;
  int r = 0;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float acc[8];
    unpack_u4(multimem_ld_reduce_bf16x8(mc + base + i * 16), acc);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= scale;
    const uint4 out = pack8_u4(acc);
    if (BCAST) multimem_st_v4(mc + base + i * 16, out);
    else st_v4(local + base + i * 16, out);
    float stored[8];
    unpack_u4(out, stored);
    sq += masked_sumsq8(stored, (size_t)rank * per + i * 8, ranges, nranges, r);
  }
  block_partial(sq, partials + blockIdx.x);
  symm_barrier(pads.ptr, rank, nranks, blockIdx.x, epoch + 1, err);
}

// ---- in optimizer.step(): global norm and clip coefficient --------------------------------------------------
// slots: NOT rotated (ptr[p] = rank p's slot buffer, two doubles: one per step parity, so a rank that runs ahead
// into the next step never overwrites a value a slower peer has still to read).  out[0] = norm, out[1] = coef.
constexpr int kFinalizeThreads = 256;
__global__ void __launch_bounds__(kFinalizeThreads) clip_finalize_kernel(const double* __restrict__ partials,
                                                                         int nparts, SymmPtrs slots, SymmPads pads,
                                                                         int parity, float norm_scale, float max_norm,
                                                                         float* out, int rank, int nranks,
                                                                         uint32_t epoch, int* err) {
  __shared__ double red[kFinalizeThreads];
  double s = 0.0;
  for (int i = threadIdx.x; i < nparts; i += kFinalizeThreads) s += partials[i];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int w = kFinalizeThreads / 2; w > 0; w >>= 1) {
    if ((int)threadIdx.x < w) red[threadIdx.x] += red[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) reinterpret_cast<volatile double*>(slots.ptr[rank])[parity] = red[0];
  symm_barrier(pads.ptr, rank, nranks, 0, epoch, err);  // fences the slot store before signalling the peers
  if (threadIdx.x == 0) {
    double total = 0.0;
    for (int p = 0; p < nranks; ++p) total += reinterpret_cast<volatile const double*>(slots.ptr[p])[parity];
    const float norm = (float)sqrt(total) * norm_scale;
    const float c = max_norm / (norm + 1e-6f);
    out[0] = norm;
    out[1] = (c < 1.f || c != c) ? c : 1.f;  // min(1, c) that keeps a NaN, as torch's clamp does
  }
}

// ---- deferred AdamW with the clip coefficient ----------------------------------------------------------------
// p_src, g, m, v: this rank's range, indexed from 0.  dst.ptr[k]: where the new parameters of the same range go on
// replica k (NR = 1: the local replica, which may be p_src itself).
template <int NR, typename StateT>
__global__ void __launch_bounds__(256) adamw_clip_kernel(SymmPtrs dst, const __nv_bfloat16* p_src,
                                                         const __nv_bfloat16* __restrict__ g, StateT* __restrict__ m,
                                                         StateT* __restrict__ v, long long nvec, AdamWHyper hp,
                                                         const float* __restrict__ coef_ptr) {
  const float coef = *coef_ptr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    float fp[8], fg[8], fm[8], fv[8];
    unpack8(ld8(p_src + i * 8), fp);
    unpack8(ld8(g + i * 8), fg);
    load_state8(m + i * 8, fm);
    load_state8(v + i * 8, fv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      fg[j] *= coef;
      adamw_update(fp[j], fg[j], fm[j], fv[j], hp);
    }
    store_state8(m + i * 8, fm);
    store_state8(v + i * 8, fv);
    const uint4 out = pack8_u4(fp);
#pragma unroll
    for (int k = 0; k < NR; ++k) st_v4(dst.ptr[k] + i * 16, out);
  }
}

// ZeRO-1 with NVLS: one multicast store reaches every replica
template <typename StateT>
__global__ void __launch_bounds__(256) nvls_adamw_clip_kernel(char* dst_mc, const __nv_bfloat16* p_src,
                                                              const __nv_bfloat16* __restrict__ g,
                                                              StateT* __restrict__ m, StateT* __restrict__ v,
                                                              long long nvec, AdamWHyper hp,
                                                              const float* __restrict__ coef_ptr) {
  const float coef = *coef_ptr;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec;
       i += (long long)gridDim.x * blockDim.x) {
    float fp[8], fg[8], fm[8], fv[8];
    unpack8(ld8(p_src + i * 8), fp);
    unpack8(ld8(g + i * 8), fg);
    load_state8(m + i * 8, fm);
    load_state8(v + i * 8, fv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      fg[j] *= coef;
      adamw_update(fp[j], fg[j], fm[j], fv[j], hp);
    }
    store_state8(m + i * 8, fm);
    store_state8(v + i * 8, fv);
    multimem_st_v4(dst_mc + i * 16, pack8_u4(fp));
  }
}

// ---- launchers ----------------------------------------------------------------------------------------------
#define DTG_CLIP_NR_DISPATCH(NRV, ...)                                   \
  switch (NRV) {                                                         \
    case 1: { constexpr int NR = 1; __VA_ARGS__; } break;                \
    case 2: { constexpr int NR = 2; __VA_ARGS__; } break;                \
    case 4: { constexpr int NR = 4; __VA_ARGS__; } break;                \
    case 8: { constexpr int NR = 8; __VA_ARGS__; } break;                \
    default: throw std::runtime_error("symmetric collectives support 1, 2, 4 or 8 ranks"); \
  }

static void check_reduce(size_t n, int nranks, int blocks) {
  if (n % ((size_t)nranks * 8) != 0) throw std::runtime_error("collective size must be a multiple of 8*nranks elements");
  if (blocks < 1 || blocks > kMaxChannels) throw std::runtime_error("comm grid exceeds the signal-pad channels");
}

void comm_reduce_sumsq(const SymmPtrs& buf, const SymmPads& pads, size_t elem_off, size_t n, float scale,
                       bool broadcast, const long long* ranges, int nranges, double* partials, int rank, int nranks,
                       uint32_t epoch, int* err, int blocks, cudaStream_t s) {
  check_reduce(n, nranks, blocks);
  if (broadcast) {
    DTG_CLIP_NR_DISPATCH(nranks, (reduce_sumsq_kernel<NR, true><<<blocks, kCommThreads, 0, s>>>(
                                     buf, pads, elem_off, n, scale, ranges, nranges, partials, rank, epoch, err)));
  } else {
    DTG_CLIP_NR_DISPATCH(nranks, (reduce_sumsq_kernel<NR, false><<<blocks, kCommThreads, 0, s>>>(
                                     buf, pads, elem_off, n, scale, ranges, nranges, partials, rank, epoch, err)));
  }
  note_launch();
  DTG_LAUNCH_CHECK();
}

void comm_nvls_reduce_sumsq(void* mc, void* local, const SymmPads& pads, size_t elem_off, size_t n, float scale,
                            bool broadcast, const long long* ranges, int nranges, double* partials, int rank,
                            int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s) {
  check_reduce(n, nranks, blocks);
  if (mc == nullptr) throw std::runtime_error("NVLS collective called without a multicast address");
  if (broadcast)
    nvls_reduce_sumsq_kernel<true><<<blocks, kCommThreads, 0, s>>>((char*)mc, (char*)local, pads, elem_off, n, scale,
                                                                   ranges, nranges, partials, rank, nranks, epoch, err);
  else
    nvls_reduce_sumsq_kernel<false><<<blocks, kCommThreads, 0, s>>>((char*)mc, (char*)local, pads, elem_off, n, scale,
                                                                    ranges, nranges, partials, rank, nranks, epoch, err);
  note_launch();
  DTG_LAUNCH_CHECK();
}

void comm_clip_finalize(const double* partials, int nparts, const SymmPtrs& slots, const SymmPads& pads, int parity,
                        float norm_scale, float max_norm, float* out, int rank, int nranks, uint32_t epoch, int* err,
                        cudaStream_t s) {
  if (nranks < 1 || nranks > kMaxRanks) throw std::runtime_error("1..8 ranks supported");
  clip_finalize_kernel<<<1, kFinalizeThreads, 0, s>>>(partials, nparts, slots, pads, parity & 1, norm_scale, max_norm,
                                                      out, rank, nranks, epoch, err);
  note_launch();
  DTG_LAUNCH_CHECK();
}

static int adamw_grid(long long nvec) {
  long long grid = (nvec + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  if (grid > cap) grid = cap;
  if (grid < 1) grid = 1;
  return (int)grid;
}

void adamw_clip(const SymmPtrs& dst, void* dst_mc, const void* p_src, const void* g, void* m, void* v, bool state_fp32,
                long long n, const AdamWHyper& hp, const float* coef, int ndst, cudaStream_t s) {
  if (n % 8 != 0) throw std::runtime_error("adamw_clip: range must be a multiple of 8 elements");
  const long long nvec = n / 8;
  const int grid = adamw_grid(nvec);
  const auto* ps = (const __nv_bfloat16*)p_src;
  const auto* gs = (const __nv_bfloat16*)g;
  if (dst_mc != nullptr) {
    if (state_fp32)
      nvls_adamw_clip_kernel<float><<<grid, 256, 0, s>>>((char*)dst_mc, ps, gs, (float*)m, (float*)v, nvec, hp, coef);
    else
      nvls_adamw_clip_kernel<__nv_bfloat16><<<grid, 256, 0, s>>>((char*)dst_mc, ps, gs, (__nv_bfloat16*)m,
                                                                 (__nv_bfloat16*)v, nvec, hp, coef);
  } else if (state_fp32) {
    DTG_CLIP_NR_DISPATCH(ndst, (adamw_clip_kernel<NR, float><<<grid, 256, 0, s>>>(dst, ps, gs, (float*)m, (float*)v,
                                                                                   nvec, hp, coef)));
  } else {
    DTG_CLIP_NR_DISPATCH(ndst, (adamw_clip_kernel<NR, __nv_bfloat16><<<grid, 256, 0, s>>>(
                                   dst, ps, gs, (__nv_bfloat16*)m, (__nv_bfloat16*)v, nvec, hp, coef)));
  }
  note_launch();
  DTG_LAUNCH_CHECK();
}

}  // namespace dtg
