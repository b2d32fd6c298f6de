// NVLink / NVSwitch collectives over peer-mapped ("symmetric") memory, fused with the math that
// surrounds them in data-parallel training.  Every kernel takes a device table of the N ranks'
// base pointers to the SAME symmetric buffer plus a table of signal pads, and synchronises
// device-side (st.release.sys / ld.acquire.sys epoch flags, one channel per CTA) — no host
// involvement and no NCCL on these paths.
//
//   allreduce_scale          two-shot all-reduce of a gradient bucket with the 1/N (and loss-scale)
//                            multiply fused in: the DDP bucket kernel (reference: DDP's C++ Reducer
//                            pre-divide + ncclAllReduce, SURVEY.md N2/K11)
//   rs_adamw_ag              ZeRO-1 step for a bucket in ONE kernel: reduce-scatter (pull the N
//                            partial gradients of my slice) -> AdamW on my optimizer shard -> push
//                            the updated bf16 parameters to all N replicas (reference: all-reduce
//                            + local AdamW + 291 per-tensor ncclBroadcast, SURVEY.md N3)
//   rs_adamw                 FSDP: reduce-scatter fused with the partitioned AdamW update
//                            (reference: fp32 reduce_scatter_tensor + foreach casts + fused AdamW, N5/K12)
//   allgather                FSDP unshard: pull every rank's parameter shard into the local full
//                            buffer (reference: copy-in + all_gather_into_tensor + copy-out, N4/K12)
//   barrier                  device-side barrier
//
// With NVLS (multicast pointer bound, `mc` != nullptr) the reduce phase uses
// multimem.ld_reduce (in-switch sum) and the broadcast phase multimem.st.
#include "adamw.cuh"
#include "comm.cuh"
#include "comm_device.cuh"
#include "common.cuh"
#include "ptx.cuh"

namespace dtg {
using namespace ptx;

// Sum the 8-element vector `i` (in units of 16 B from the buffer base + off) over all ranks, fp32.
template <int NR>
__device__ __forceinline__ void gather_sum(const SymmPtrs& sp, size_t byte_off, int rank, float (&acc)[8]) {
  // pointer tables are rotated on the host: ptr[0] is this rank, ptr[k] is rank (rank+k)%NR, so
  // every rank starts on a different peer and the indices are compile-time constants
  uint4 v[NR];
#pragma unroll
  for (int k = 0; k < NR; ++k) v[k] = ld_volatile_v4(sp.ptr[k] + byte_off);
#pragma unroll
  for (int j = 0; j < 8; ++j) acc[j] = 0.f;
#pragma unroll
  for (int k = 0; k < NR; ++k) add8(acc, v[k]);
}

// ---- DDP: all-reduce with fused scale ------------------------------------------------------------
template <int NR>
__global__ void __launch_bounds__(kCommThreads) allreduce_scale_kernel(SymmPtrs buf, SymmPads pads, size_t elem_off,
                                                                       size_t n, float scale, int rank,
                                                                       uint32_t epoch, int* err) {
  symm_barrier(pads.ptr, rank, NR, blockIdx.x, epoch, err);
  const size_t per = n / NR;  // n is a multiple of NR*8
  const size_t base = (elem_off + (size_t)rank * per) * 2;
  const size_t nvec = per / 8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float acc[8];
    gather_sum<NR>(buf, base + i * 16, rank, acc);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= scale;
    const uint4 out = pack8_u4(acc);
#pragma unroll
    for (int k = 0; k < NR; ++k) st_v4(buf.ptr[k] + base + i * 16, out);
  }
  symm_barrier(pads.ptr, rank, NR, blockIdx.x, epoch + 1, err);
}

// ---- ZeRO-1: reduce-scatter -> AdamW(shard) -> all-gather of parameters, one kernel ------------------
// grads / params: symmetric flat buffers of the same geometry; m, v: this rank's optimizer shard
// (local memory, `per` elements).  PUSH_PARAMS=false gives the FSDP variant (parameters stay sharded:
// `param_local` is then this rank's shard buffer, indexed from 0).
template <int NR, typename StateT, bool PUSH_PARAMS>
__global__ void __launch_bounds__(kCommThreads) rs_adamw_kernel(SymmPtrs grads, SymmPtrs params,
                                                                __nv_bfloat16* param_local, StateT* m, StateT* v,
                                                                SymmPads pads, size_t elem_off, size_t n,
                                                                AdamWHyper hp, int rank, uint32_t epoch, int* err) {
  symm_barrier(pads.ptr, rank, NR, blockIdx.x, epoch, err);
  const size_t per = n / NR;
  const size_t base = (elem_off + (size_t)rank * per) * 2;
  const size_t nvec = per / 8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float g[8], p[8], fm[8], fv[8];
    gather_sum<NR>(grads, base + i * 16, rank, g);
    const __nv_bfloat16* psrc =
        PUSH_PARAMS ? reinterpret_cast<const __nv_bfloat16*>(params.ptr[0] + base) + i * 8 : param_local + i * 8;
    unpack8(ld8(psrc), p);
    load_state8(m + i * 8, fm);
    load_state8(v + i * 8, fv);
#pragma unroll
    for (int j = 0; j < 8; ++j) adamw_update(p[j], g[j], fm[j], fv[j], hp);  // hp.grad_scale carries 1/N
    store_state8(m + i * 8, fm);
    store_state8(v + i * 8, fv);
    const uint4 out = pack8_u4(p);
    if (PUSH_PARAMS) {
#pragma unroll
      for (int k = 0; k < NR; ++k) st_v4(params.ptr[k] + base + i * 16, out);
    } else {
      *reinterpret_cast<uint4*>(param_local + i * 8) = out;
    }
  }
  symm_barrier(pads.ptr, rank, NR, blockIdx.x, epoch + 1, err);
}

// ---- FSDP unshard: pull all shards of a group into the local full buffer --------------------------------
// shards: symmetric buffer holding each rank's shard of `per` elements at element offset shard_off;
// full: local destination of NR*per elements.
template <int NR>
__global__ void __launch_bounds__(kCommThreads) allgather_kernel(SymmPtrs shards, __nv_bfloat16* full, SymmPads pads,
                                                                 size_t shard_off, size_t per, int rank,
                                                                 uint32_t epoch, int* err, int do_barrier) {
  if (do_barrier) symm_barrier(pads.ptr, rank, NR, blockIdx.x, epoch, err);
  const size_t nvec = per / 8;
  const size_t total = nvec * NR;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i / nvec);  // dynamic index: the table is copied to local memory once
    const size_t j = i % nvec;
    const int p = (rank + k) % NR;
    const uint4 val = ld_volatile_v4(shards.ptr[k] + (shard_off + j * 8) * 2);
    *reinterpret_cast<uint4*>(full + (size_t)p * per + j * 8) = val;
  }
}

// ---- plain reduce-scatter (mean) into a local shard: used when the optimizer runs elsewhere (CPU offload) ----
template <int NR>
__global__ void __launch_bounds__(kCommThreads) reduce_scatter_kernel(SymmPtrs grads, __nv_bfloat16* out, SymmPads pads,
                                                                      size_t elem_off, size_t n, float scale, int rank,
                                                                      uint32_t epoch, int* err) {
  symm_barrier(pads.ptr, rank, NR, blockIdx.x, epoch, err);
  const size_t per = n / NR;
  const size_t base = (elem_off + (size_t)rank * per) * 2;
  const size_t nvec = per / 8;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    float acc[8];
    gather_sum<NR>(grads, base + i * 16, rank, acc);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] *= scale;
    *reinterpret_cast<uint4*>(out + i * 8) = pack8_u4(acc);
  }
  symm_barrier(pads.ptr, rank, NR, blockIdx.x, epoch + 1, err);
}

__global__ void barrier_kernel(SymmPads pads, int rank, int nranks, uint32_t epoch, int* err) {
  symm_barrier(pads.ptr, rank, nranks, blockIdx.x, epoch, err);
}

// ---- launchers ----------------------------------------------------------------------------------
#define DTG_NR_DISPATCH(NRV, ...)                                        \
  switch (NRV) {                                                         \
    case 1: { constexpr int NR = 1; __VA_ARGS__; } break;                \
    case 2: { constexpr int NR = 2; __VA_ARGS__; } break;                \
    case 4: { constexpr int NR = 4; __VA_ARGS__; } break;                \
    case 8: { constexpr int NR = 8; __VA_ARGS__; } break;                \
    default: throw std::runtime_error("symmetric collectives support 1, 2, 4 or 8 ranks"); \
  }

static void check_geometry(size_t n, int nranks, int blocks) {
  if (n % ((size_t)nranks * 8) != 0) throw std::runtime_error("collective size must be a multiple of 8*nranks elements");
  if (blocks < 1 || blocks > kMaxChannels) throw std::runtime_error("comm grid exceeds the signal-pad channels");
}

void comm_allreduce_scale(const SymmPtrs& buf, const SymmPads& pads, size_t elem_off, size_t n, float scale, int rank,
                          int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s) {
  check_geometry(n, nranks, blocks);
  DTG_NR_DISPATCH(nranks, (allreduce_scale_kernel<NR><<<blocks, kCommThreads, 0, s>>>(buf, pads, elem_off, n, scale,
                                                                                     rank, epoch, err)));
  note_launch();
  DTG_LAUNCH_CHECK();
}

void comm_rs_adamw(const SymmPtrs& grads, const SymmPtrs& params, void* param_local, void* m, void* v, bool state_fp32,
                   bool push_params, const SymmPads& pads, size_t elem_off, size_t n, const AdamWHyper& hp, int rank,
                   int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s) {
  check_geometry(n, nranks, blocks);
#define LAUNCH_RS(ST, PUSH)                                                                                      \
  DTG_NR_DISPATCH(nranks, (rs_adamw_kernel<NR, ST, PUSH><<<blocks, kCommThreads, 0, s>>>(                         \
                              grads, params, (__nv_bfloat16*)param_local, (ST*)m, (ST*)v, pads, elem_off, n, hp, \
                              rank, epoch, err)))
  if (state_fp32) {
    if (push_params) { LAUNCH_RS(float, true); } else { LAUNCH_RS(float, false); }
  } else {
    if (push_params) { LAUNCH_RS(__nv_bfloat16, true); } else { LAUNCH_RS(__nv_bfloat16, false); }
  }
#undef LAUNCH_RS
  note_launch();
  DTG_LAUNCH_CHECK();
}

void comm_allgather(const SymmPtrs& shards, void* full, const SymmPads& pads, size_t shard_off, size_t per, int rank,
                    int nranks, uint32_t epoch, int* err, bool barrier, int blocks, cudaStream_t s) {
  if (per % 8 != 0) throw std::runtime_error("allgather shard must be a multiple of 8 elements");
  if (blocks < 1 || blocks > kMaxChannels) throw std::runtime_error("comm grid exceeds the signal-pad channels");
  DTG_NR_DISPATCH(nranks, (allgather_kernel<NR><<<blocks, kCommThreads, 0, s>>>(shards, (__nv_bfloat16*)full, pads,
                                                                               shard_off, per, rank, epoch, err,
                                                                               barrier ? 1 : 0)));
  note_launch();
  DTG_LAUNCH_CHECK();
}

// All-gather on the copy engines: one device-side barrier (a 1-warp kernel) and then N async peer copies.
// No SM time at all, which matters when the gather is a prefetch running under tensor-core kernels that own
// every SM (FSDP unshard): an SM-driven gather there competes for issue slots and gets stretched.
void comm_allgather_ce(const SymmPtrs& shards, void* full, const SymmPads& pads, size_t shard_off, size_t per, int rank,
                       int nranks, uint32_t epoch, int* err, bool barrier, cudaStream_t s) {
  if (barrier) {
    barrier_kernel<<<1, 32, 0, s>>>(pads, rank, nranks, epoch, err);
    note_launch();
    DTG_LAUNCH_CHECK();
  }
  const size_t bytes = per * sizeof(__nv_bfloat16);
  for (int k = 0; k < nranks; ++k) {
    const int p = (rank + k) % nranks;  // shards.ptr is rotated: entry k belongs to rank (rank + k) % nranks
    DTG_CUDA_CHECK(cudaMemcpyAsync((char*)full + (size_t)p * bytes, shards.ptr[k] + shard_off * sizeof(__nv_bfloat16),
                                   bytes, cudaMemcpyDeviceToDevice, s));
  }
}

void comm_reduce_scatter(const SymmPtrs& grads, void* out, const SymmPads& pads, size_t elem_off, size_t n, float scale,
                         int rank, int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s) {
  check_geometry(n, nranks, blocks);
  DTG_NR_DISPATCH(nranks, (reduce_scatter_kernel<NR><<<blocks, kCommThreads, 0, s>>>(
                              grads, (__nv_bfloat16*)out, pads, elem_off, n, scale, rank, epoch, err)));
  note_launch();
  DTG_LAUNCH_CHECK();
}

void comm_barrier(const SymmPads& pads, int rank, int nranks, uint32_t epoch, int* err, cudaStream_t s) {
  barrier_kernel<<<1, 32, 0, s>>>(pads, rank, nranks, epoch, err);
  note_launch();
  DTG_LAUNCH_CHECK();
}

}  // namespace dtg
