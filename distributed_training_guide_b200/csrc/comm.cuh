// Types and launchers of the NVLink symmetric-memory collectives (comm.cu, fused_tp.cu).
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include <cstdint>

#include "adamw.cuh"

namespace dtg {

constexpr int kMaxChannels = 256;  // one signal-pad channel per CTA of a collective kernel
constexpr int kCommThreads = 512;
constexpr long long kSpinTimeoutCycles = 20LL * 1000 * 1000 * 1000;  // ~10 s at 2 GHz
constexpr size_t kPadBytes = (size_t)kMaxChannels * kMaxRanks * sizeof(uint32_t);

// Base pointers of one symmetric buffer on every rank, ROTATED: ptr[0] = this rank,
// ptr[k] = rank (rank + k) % nranks.
struct SymmPtrs {
  char* ptr[kMaxRanks];
};
// Signal pads (NOT rotated: ptr[p] = rank p's pad): uint32 [kMaxChannels][kMaxRanks]
struct SymmPads {
  uint32_t* ptr[kMaxRanks];
};

void comm_allreduce_scale(const SymmPtrs& buf, const SymmPads& pads, size_t elem_off, size_t n, float scale, int rank,
                          int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s);
void comm_rs_adamw(const SymmPtrs& grads, const SymmPtrs& params, void* param_local, void* m, void* v, bool state_fp32,
                   bool push_params, const SymmPads& pads, size_t elem_off, size_t n, const AdamWHyper& hp, int rank,
                   int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s);
void comm_allgather(const SymmPtrs& shards, void* full, const SymmPads& pads, size_t shard_off, size_t per, int rank,
                    int nranks, uint32_t epoch, int* err, bool barrier, int blocks, cudaStream_t s);
void comm_allgather_ce(const SymmPtrs& shards, void* full, const SymmPads& pads, size_t shard_off, size_t per, int rank,
                       int nranks, uint32_t epoch, int* err, bool barrier, cudaStream_t s);
void comm_reduce_scatter(const SymmPtrs& grads, void* out, const SymmPads& pads, size_t elem_off, size_t n, float scale,
                         int rank, int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s);
void comm_barrier(const SymmPads& pads, int rank, int nranks, uint32_t epoch, int* err, cudaStream_t s);
// NVLS (multicast) variants, comm_nvls.cu: `mc` = the buffer's multicast address
void comm_nvls_allreduce_scale(void* mc, const SymmPads& pads, size_t elem_off, size_t n, float scale, int rank,
                               int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s);
void comm_nvls_rs_adamw(const void* grads_mc, void* params_mc, void* params_local, void* m, void* v, bool state_fp32,
                        bool push_params, const SymmPads& pads, size_t elem_off, size_t n, const AdamWHyper& hp, int rank,
                        int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s);
// Gradient clipping, grad_clip.cu.  `ranges`: device int64 [nranges][2] of [begin, end) parameter element ranges
// of the bucket (sorted, disjoint); `partials`: one fp64 sum of squares per CTA.
void comm_reduce_sumsq(const SymmPtrs& buf, const SymmPads& pads, size_t elem_off, size_t n, float scale,
                       bool broadcast, const long long* ranges, int nranges, double* partials, int rank, int nranks,
                       uint32_t epoch, int* err, int blocks, cudaStream_t s);
void comm_nvls_reduce_sumsq(void* mc, void* local, const SymmPads& pads, size_t elem_off, size_t n, float scale,
                            bool broadcast, const long long* ranges, int nranges, double* partials, int rank,
                            int nranks, uint32_t epoch, int* err, int blocks, cudaStream_t s);
void comm_clip_finalize(const double* partials, int nparts, const SymmPtrs& slots, const SymmPads& pads, int parity,
                        float norm_scale, float max_norm, float* out, int rank, int nranks, uint32_t epoch, int* err,
                        cudaStream_t s);
void adamw_clip(const SymmPtrs& dst, void* dst_mc, const void* p_src, const void* g, void* m, void* v, bool state_fp32,
                long long n, const AdamWHyper& hp, const float* coef, int ndst, cudaStream_t s);


// ---- fused_tp.cu / cross_entropy.cu helpers used by the tensor-parallel path ------------------------
void tp_reduce_parts(const void* parts, const void* residual, void* out, long long n, int nparts, cudaStream_t s);
void tp_reduce_mc(const void* part_mc, const void* residual, void* out, long long n, const SymmPads& pads, int rank,
                  int nranks, uint32_t epoch, int* err, cudaStream_t s);
void vp_ce_stats(const void* logits, const long long* targets, void* stats, int T, int Vl, int v0, cudaStream_t s);
void vp_ce_grad(void* logits, const long long* targets, const SymmPtrs& stats, float* row_loss, const float* n_valid,
                int T, int Vl, int v0, int nranks, cudaStream_t s);
void tp_embed_fwd(const long long* ids, const void* w, const SymmPtrs& dst, long long T, long long V, int rpp, int H,
                  int Hl, int rank, cudaStream_t s);
// dw [V, Hl] = (or +=) the per-id sum of this rank's Hl columns of every token's dx row, pulled from the owning rank
// into staging [T, Hl] bf16 and summed by embedding_bwd (slot [V] and sums [T, Hl] fp32 are its scratch)
void tp_embed_bwd(const long long* ids, const SymmPtrs& dx, void* dw, void* staging, unsigned int* slot, float* sums,
                  long long T, long long V, int rpp, int H, int Hl, int rank, bool accumulate, cudaStream_t s);
void ce_count_valid(const long long* targets, float* n_valid, int T, cudaStream_t s);
void ce_finalize(const float* row_loss, const float* n_valid, float* loss, int T, cudaStream_t s);

}  // namespace dtg
