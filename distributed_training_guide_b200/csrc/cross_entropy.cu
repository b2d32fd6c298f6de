// Softmax cross-entropy over bf16 logits, forward + backward in one sweep:
//   pass 1 (per row): online max / sum-exp -> logsumexp, row loss = lse - logit[target]
//   pass 2 (same CTA, row now in L2): overwrite the logits with (softmax - onehot) / n_valid
// so the loss never materialises an fp32 [T,V] copy nor a separate dlogits tensor (the reference
// path does `.float()` on the logits then log_softmax + nll_loss, SURVEY.md K7).
// Targets follow the vocabulary rule of common.cuh, with V = logits.size(1):
//   -100 (kIgnoreIndex)   zero dlogits row, not counted in n_valid;
//   0 <= t < V            the usual loss and gradient;
//   anything else         counted in n_valid, row loss NaN (so the mean loss is NaN), dlogits row NaN; the logits
//                         are never indexed with it.
#include "api.h"
#include "common.cuh"

namespace dtg {

constexpr int kCEThreads = 512;

__global__ void count_valid_kernel(const long long* __restrict__ targets, float* __restrict__ n_valid, int T) {
  __shared__ float red[32];
  float c = 0.f;
  for (int i = threadIdx.x; i < T; i += blockDim.x) c += (targets[i] != kIgnoreIndex) ? 1.f : 0.f;
  c = block_sum(c, red);
  if (threadIdx.x == 0) *n_valid = c;
}

__global__ void __launch_bounds__(kCEThreads) ce_row_kernel(__nv_bfloat16* __restrict__ logits,
                                                           const long long* __restrict__ targets,
                                                           float* __restrict__ row_loss,
                                                           const float* __restrict__ n_valid, int V) {
  __shared__ float red[32];
  const int row = blockIdx.x;
  __nv_bfloat16* lr = logits + (size_t)row * V;
  const long long tgt = targets[row];
  const bool valid = in_vocab(tgt, V);
  const int nvec = V >> 3;  // V % 8 == 0 enforced by the launcher
  // pass 1: online logsumexp
  float mx = -INFINITY, sum = 0.f;
  for (int i = threadIdx.x; i < nvec; i += kCEThreads) {
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
  const float lse = gmx + __logf(sum);
  const float nv = *n_valid;
  const float inv = (tgt == kIgnoreIndex) ? 0.f : valid ? 1.f / nv : nan_f();
  if (threadIdx.x == 0) {
    float l = 0.f;
    if (tgt != kIgnoreIndex) l = valid ? lse - __bfloat162float(lr[tgt]) : nan_f();
    row_loss[row] = l;
  }
  __syncthreads();  // the target logit is read before anyone overwrites it
  // pass 2: dlogits in place
  for (int i = threadIdx.x; i < nvec; i += kCEThreads) {
    float f[8];
    unpack8(ld8(lr + i * 8), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      float p = __expf(f[j] - lse);
      if ((long long)(i * 8 + j) == tgt) p -= 1.f;
      f[j] = p * inv;
    }
    st8(lr + i * 8, pack8(f));
  }
}

__global__ void ce_finalize_kernel(const float* __restrict__ row_loss, const float* __restrict__ n_valid,
                                   float* __restrict__ loss, int T) {
  __shared__ float red[32];
  float s = 0.f;
  for (int i = threadIdx.x; i < T; i += blockDim.x) s += row_loss[i];
  s = block_sum(s, red);
  if (threadIdx.x == 0) *loss = (*n_valid > 0.f) ? s / *n_valid : 0.f;
}

void ce_count_valid(const long long* targets, float* n_valid, int T, cudaStream_t s) {
  count_valid_kernel<<<1, 1024, 0, s>>>(targets, n_valid, T);
  note_launch();
  DTG_LAUNCH_CHECK();
}
void ce_finalize(const float* row_loss, const float* n_valid, float* loss, int T, cudaStream_t s) {
  ce_finalize_kernel<<<1, 1024, 0, s>>>(row_loss, n_valid, loss, T);
  note_launch();
  DTG_LAUNCH_CHECK();
}

void cross_entropy_fwd_bwd(void* logits, const long long* targets, float* row_loss, float* n_valid, float* loss,
                           int T, int V, cudaStream_t s) {
  if (V % 8 != 0) throw std::runtime_error("cross_entropy: vocab size must be a multiple of 8");
  if (T <= 0) return;
  count_valid_kernel<<<1, 1024, 0, s>>>(targets, n_valid, T);
  ce_row_kernel<<<T, kCEThreads, 0, s>>>((__nv_bfloat16*)logits, targets, row_loss, n_valid, V);
  ce_finalize_kernel<<<1, 1024, 0, s>>>(row_loss, n_valid, loss, T);
  note_launch(3);
  DTG_LAUNCH_CHECK();
}

}  // namespace dtg
