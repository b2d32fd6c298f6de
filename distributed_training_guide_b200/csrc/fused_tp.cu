// Tensor / sequence-parallel support kernels (chapters 06 / 07).  The tensor-core halves of the fused
// paths — all-gather->GEMM, GEMM->reduce-scatter push, wgrad over a sequence-sharded operand — are the
// distributed modes of the wgmma GEMM in gemm_wgmma.cu (operand tiles fetched from / stored to peer
// GPUs over NVLink inside the kernel).  This file holds the pieces around them:
//
//   tp_reduce_parts      out = (residual +) sum of the N partial tiles peers pushed into my staging
//                        buffer: the "reduce" half of GEMM->reduce-scatter, fused with the residual add
//   vocab-parallel CE    lm_head logits stay sharded over the vocabulary: per-row (max, sum-exp, target
//                        logit) go to a symmetric stats buffer, every rank combines the N ranks' stats over
//                        NVLink and writes dlogits for its shard in place.  Replaces the reference's 4 GB
//                        logits all-gather + redundant fp32 CE on every TP rank (SURVEY.md N10 / C19).
//   hidden-parallel embedding   each rank owns H/N columns of the table; the lookup is pushed straight
//                        into the owning rank's sequence shard (the reference's embedding all-to-all, N9),
//                        and the backward pulls its column slice of the peers' gradient shards into a local
//                        staging buffer that the single-GPU embedding backward sums in fp32.
// Token ids and targets follow the vocabulary rule of common.cuh (V = NR * Vl for the loss, w.size(0) for the
// embedding).
#include "api.h"
#include "comm.cuh"
#include "comm_device.cuh"
#include "common.cuh"
#include "ptx.cuh"

namespace dtg {
using namespace ptx;

// ---- out[r, :] = (residual[r, :] +) sum_p parts[p][r, :] --------------------------------------------
__global__ void tp_reduce_parts_kernel(const __nv_bfloat16* __restrict__ parts, const __nv_bfloat16* __restrict__ res,
                                       __nv_bfloat16* __restrict__ out, long long nvec, long long part_stride_vec,
                                       int nparts) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int p = 0; p < nparts; ++p) {
      float f[8];
      unpack8(ld8(parts + (p * part_stride_vec + i) * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
    if (res) {
      float f[8];
      unpack8(ld8(res + i * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
    st8(out + i * 8, pack8(acc));
  }
}

void tp_reduce_parts(const void* parts, const void* residual, void* out, long long n, int nparts, cudaStream_t s) {
  if (n % 8) throw std::runtime_error("tp_reduce_parts: size must be a multiple of 8");
  if (n <= 0) return;
  long long nvec = n / 8;
  long long grid = (nvec + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  if (grid > cap) grid = cap;
  if (grid < 1) grid = 1;
  tp_reduce_parts_kernel<<<(int)grid, 256, 0, s>>>((const __nv_bfloat16*)parts, (const __nv_bfloat16*)residual,
                                                  (__nv_bfloat16*)out, nvec, nvec, nparts);
  note_launch();
  DTG_LAUNCH_CHECK();
}

// ---- GEMM -> reduce-scatter, reduce half on the NVSwitch ------------------------------------------------------
// Every rank's row-parallel GEMM wrote its FULL partial [T, H] into its own copy of a multicast-bound symmetric
// buffer (plain local stores: the GEMM epilogue is the un-distributed one).  This kernel is the whole rest of the
// reduce-scatter: a device-side barrier at entry (every rank's GEMM has completed), then each 16-byte vector of MY
// rows is read once through the multicast address with multimem.ld_reduce — the switch pulls the N copies and
// adds them in fp32 — plus the residual, straight into the sequence-sharded output.  Versus the push variant
// (GEMM pushes row chunks into N staging slots, barrier kernel, N-way sum kernel) that is one launch fewer, no
// N-fold staging write + read in HBM, and 1/N of the NVLink ingress per GPU.
__global__ void __launch_bounds__(kCommThreads) tp_reduce_mc_kernel(const char* __restrict__ part_mc,
                                                                    const __nv_bfloat16* __restrict__ res,
                                                                    __nv_bfloat16* __restrict__ out, long long nvec,
                                                                    SymmPads pads, int rank, int nranks, uint32_t epoch,
                                                                    int* err) {
  symm_barrier(pads.ptr, rank, nranks, blockIdx.x, epoch, err);
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < nvec; i += (long long)gridDim.x * blockDim.x) {
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    add8(acc, multimem_ld_reduce_bf16x8(part_mc + i * 16));
    if (res) {
      float f[8];
      unpack8(ld8(res + i * 8), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] += f[j];
    }
    st8(out + i * 8, pack8(acc));
  }
}

void tp_reduce_mc(const void* part_mc, const void* residual, void* out, long long n, const SymmPads& pads, int rank,
                  int nranks, uint32_t epoch, int* err, cudaStream_t s) {
  if (n % 8) throw std::runtime_error("tp_reduce_mc: size must be a multiple of 8");
  if (part_mc == nullptr) throw std::runtime_error("tp_reduce_mc: no multicast address");
  const long long nvec = n / 8;
  long long grid = (nvec + kCommThreads - 1) / kCommThreads;
  const long long cap = sm_count() < kMaxChannels ? sm_count() : kMaxChannels;   // one barrier channel per CTA
  if (grid > cap) grid = cap;
  if (grid < 1) grid = 1;
  tp_reduce_mc_kernel<<<(int)grid, kCommThreads, 0, s>>>((const char*)part_mc, (const __nv_bfloat16*)residual,
                                                       (__nv_bfloat16*)out, nvec, pads, rank, nranks, epoch, err);
  note_launch();
  DTG_LAUNCH_CHECK();
}

// ---- vocab-parallel cross entropy --------------------------------------------------------------------
constexpr int kVpThreads = 512;

// stats[row] = (local max, local sum exp(x - max), target logit or 0, 1 if the target is in my shard)
__global__ void __launch_bounds__(kVpThreads) vp_ce_stats_kernel(const __nv_bfloat16* __restrict__ logits,
                                                                const long long* __restrict__ targets,
                                                                float4* __restrict__ stats, int Vl, int v0) {
  __shared__ float red[32];
  const int row = blockIdx.x;
  const __nv_bfloat16* lr = logits + (size_t)row * Vl;
  const int nvec = Vl >> 3;
  float mx = -INFINITY, sum = 0.f;
  for (int i = threadIdx.x; i < nvec; i += kVpThreads) {
    float f[8];
    unpack8(ld8(lr + i * 8), f);
    float lm = f[0];
#pragma unroll
    for (int j = 1; j < 8; ++j) lm = fmaxf(lm, f[j]);
    if (lm > mx) {
      sum *= __expf(mx - lm);
      mx = lm;
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) sum += __expf(f[j] - mx);
  }
  const float gmx = block_max(mx, red);
  sum = (mx == -INFINITY) ? 0.f : sum * __expf(mx - gmx);
  sum = block_sum(sum, red);
  if (threadIdx.x == 0) {
    const long long t = targets[row] - v0;   // v0 >= 0, so an ignored or negative target is never mine
    const bool mine = in_vocab(t, Vl);
    stats[row] = make_float4(gmx, sum, mine ? __bfloat162float(lr[t]) : 0.f, mine ? 1.f : 0.f);
  }
}

// combine the N ranks' stats (read over NVLink), write dlogits of my shard in place and the row loss
template <int NR>
__global__ void __launch_bounds__(kVpThreads) vp_ce_grad_kernel(__nv_bfloat16* __restrict__ logits,
                                                               const long long* __restrict__ targets,
                                                               SymmPtrs stats, float* __restrict__ row_loss,
                                                               const float* __restrict__ n_valid, int Vl, int v0) {
  __shared__ float sh[2];
  const int row = blockIdx.x;
  const long long tgt = targets[row];
  const bool valid = in_vocab(tgt, (long long)NR * Vl);
  if (threadIdx.x == 0) {
    float m[NR], s[NR], tl = 0.f;
    float gm = -INFINITY;
#pragma unroll
    for (int k = 0; k < NR; ++k) {
      const uint4 raw = ld_volatile_v4(stats.ptr[k] + (size_t)row * 16);
      m[k] = __uint_as_float(raw.x);
      s[k] = __uint_as_float(raw.y);
      tl += __uint_as_float(raw.w) * __uint_as_float(raw.z);
      gm = fmaxf(gm, m[k]);
    }
    float tot = 0.f;
#pragma unroll
    for (int k = 0; k < NR; ++k) tot += s[k] * __expf(m[k] - gm);
    const float lse = gm + __logf(tot);
    sh[0] = lse;
    row_loss[row] = (tgt == kIgnoreIndex) ? 0.f : valid ? lse - tl : nan_f();
  }
  __syncthreads();
  const float lse = sh[0];
  const float nv = *n_valid;
  const float inv = (tgt == kIgnoreIndex) ? 0.f : valid ? 1.f / nv : nan_f();
  const long long tloc = tgt - v0;
  __nv_bfloat16* lr = logits + (size_t)row * Vl;
  const int nvec = Vl >> 3;
  for (int i = threadIdx.x; i < nvec; i += kVpThreads) {
    float f[8];
    unpack8(ld8(lr + i * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p = __expf(f[j] - lse);
      if ((long long)(i * 8 + j) == tloc) p -= 1.f;
      f[j] = p * inv;
    }
    st8(lr + i * 8, pack8(f));
  }
}

void vp_ce_stats(const void* logits, const long long* targets, void* stats, int T, int Vl, int v0, cudaStream_t s) {
  if (Vl % 8) throw std::runtime_error("vocab shard must be a multiple of 8");
  if (T <= 0) return;
  vp_ce_stats_kernel<<<T, kVpThreads, 0, s>>>((const __nv_bfloat16*)logits, targets, (float4*)stats, Vl, v0);
  note_launch();
  DTG_LAUNCH_CHECK();
}

void vp_ce_grad(void* logits, const long long* targets, const SymmPtrs& stats, float* row_loss, const float* n_valid,
                int T, int Vl, int v0, int nranks, cudaStream_t s) {
  if (T <= 0) return;
#define VP_CASE(NRV)                                                                                         \
  case NRV:                                                                                                  \
    vp_ce_grad_kernel<NRV><<<T, kVpThreads, 0, s>>>((__nv_bfloat16*)logits, targets, stats, row_loss, n_valid, Vl, v0); \
    break;
  switch (nranks) {
    VP_CASE(1) VP_CASE(2) VP_CASE(4) VP_CASE(8)
    default: throw std::runtime_error("vocab-parallel CE supports 1/2/4/8 ranks");
  }
#undef VP_CASE
  note_launch();
  DTG_LAUNCH_CHECK();
}

// ---- hidden-parallel embedding with the all-to-all fused in ------------------------------------------------
// fwd: for every token t of the full batch, my H/N columns of its embedding row are written into the
// sequence shard of the rank that owns token t (dst[owner] + (t % rpp) * H + rank * Hl).
// An id outside [0, V) writes a NaN row, as the single-GPU forward does.
__global__ void tp_embed_fwd_kernel(const long long* __restrict__ ids, const __nv_bfloat16* __restrict__ w,
                                    SymmPtrs dst /*unrotated*/, long long T, long long V, int rpp, int H, int Hl,
                                    int rank) {
  const int vpr = Hl >> 3;
  const long long total = T * vpr;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long t = idx / vpr;
    const int v = (int)(idx % vpr);
    const int owner = (int)(t / rpp);
    __nv_bfloat16* d = reinterpret_cast<__nv_bfloat16*>(dst.ptr[owner]) + (t % rpp) * H + (long long)rank * Hl + v * 8;
    const long long id = ids[t];
    bf16x8 r;
    if (in_vocab(id, V)) {
      r = ld8(w + id * Hl + v * 8);
    } else {
      const float nan8[8] = {nan_f(), nan_f(), nan_f(), nan_f(), nan_f(), nan_f(), nan_f(), nan_f()};
      r = pack8(nan8);
    }
    st8(d, r);
  }
}
// bwd, step 1: staging[t, :] = dx[owner(t)][t % rpp, rank*Hl : (rank+1)*Hl]   (pull from the owner over NVLink).
// Step 2 is embedding_bwd over the staging rows: one fp32 sum and one bf16 rounding per table row.
__global__ void tp_embed_pull_kernel(SymmPtrs dx /*unrotated*/, __nv_bfloat16* __restrict__ staging, long long T,
                                     int rpp, int H, int Hl, int rank) {
  const int vpr = Hl >> 3;
  const long long total = T * vpr;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long t = idx / vpr;
    const int v = (int)(idx % vpr);
    const int owner = (int)(t / rpp);
    const __nv_bfloat16* src =
        reinterpret_cast<const __nv_bfloat16*>(dx.ptr[owner]) + (t % rpp) * H + (long long)rank * Hl + v * 8;
    st8(staging + t * Hl + v * 8, ld8(src));
  }
}

static int ew_grid2(long long total_threads) {
  long long g = (total_threads + 255) / 256;
  const long long cap = (long long)sm_count() * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

void tp_embed_fwd(const long long* ids, const void* w, const SymmPtrs& dst, long long T, long long V, int rpp, int H,
                  int Hl, int rank, cudaStream_t s) {
  if (Hl % 8) throw std::runtime_error("hidden shard must be a multiple of 8");
  if (T <= 0) return;
  tp_embed_fwd_kernel<<<ew_grid2(T * (Hl / 8)), 256, 0, s>>>(ids, (const __nv_bfloat16*)w, dst, T, V, rpp, H, Hl, rank);
  note_launch();
  DTG_LAUNCH_CHECK();
}
void tp_embed_bwd(const long long* ids, const SymmPtrs& dx, void* dw, void* staging, unsigned int* slot, float* sums,
                  long long T, long long V, int rpp, int H, int Hl, int rank, bool accumulate, cudaStream_t s) {
  if (Hl % 8) throw std::runtime_error("hidden shard must be a multiple of 8");
  if (T > 0) {
    tp_embed_pull_kernel<<<ew_grid2(T * (Hl / 8)), 256, 0, s>>>(dx, (__nv_bfloat16*)staging, T, rpp, H, Hl, rank);
    note_launch();
    DTG_LAUNCH_CHECK();
  }
  embedding_bwd(staging, ids, dw, slot, sums, T, V, Hl, accumulate, s);
}

}  // namespace dtg
