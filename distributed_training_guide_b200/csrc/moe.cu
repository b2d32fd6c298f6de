// Mixture-of-experts routing, token permutation and combine kernels (OLMoE).  The expert GEMMs themselves are the
// grouped mode of the wgmma GEMM (gemm_bf16_grouped, gemm_wgmma.cu); these kernels build its routing tables and move
// rows in and out of the expert-sorted layout.  Nothing here reads a count back to the host: every buffer is sized by
// the upper bound on the permuted rows, and every kernel reads the segment table from device memory.  No kernel uses
// atomics, so the same input gives the same bits on every run.
//
// Layout.  Assignment a = t * k + slot sends token t to expert idx[a].  Expert e owns rows [seg[e], seg[e + 1]) of the
// permuted activations, seg[0] = 0 and every bound a multiple of 128; its count[e] assignments take the first rows of
// the segment, in (t, slot) order (a stable counting sort), and the rest of the segment is padding.  pos[a] is the row
// of assignment a, row_tok[r] the assignment of row r (-1 for a padding row).
//
// Weights.  w[a] is the raw top-k probability, or with NORM (Qwen3-MoE's norm_topk_prob) p_sel / S, S the fp32 sum of
// the token's k selected probabilities added in slot order and the quotient correctly rounded (__fdiv_rn).  Only w
// differs: p, idx and every table are the raw form's bits.  The router backward recomputes S the same way.
//
// Ties.  Experts are ranked by their fp32 probability as moe_topk_kernel computes it, ties to the lower expert.  That
// includes probabilities that underflow to 0 (a row whose logits span more than about 104): they tie, so the lower
// experts win.
//
// Table entries are device data the bindings cannot see, so every kernel that follows one checks it against the
// extent of what it indexes, in the way of common.cuh's vocabulary rule: a bad entry is never dereferenced.
//   row_tok[r]  -1 = padding (a zero row); 0 <= a < T * k valid; anything else (a table built for another T or k) is
//               bad: a NaN row of the permuted output and, in the combine backward, no dw entry (there is none).
//   pos[a]      0 <= pos[a] < rows of yp valid; anything else gives the token a NaN combined row.
#include <cuda_bf16.h>

#include "api.h"
#include "common.cuh"

namespace dtg {

namespace {

constexpr int kMaxE = kMoeMaxExperts;
constexpr int kEPerLane = kMaxE / 32;

// one warp per token: fp32 softmax over the E logits, then k rounds of a warp argmax (ties to the lower expert); NORM
// then divides the token's w row by the sum of its entries (every lane holds the same sum: each round's result is
// known to all lanes), each lane rescaling the slots lane, lane + 32, ...
template <bool NORM>
__global__ void moe_topk_kernel(const __nv_bfloat16* __restrict__ logits, long long ldl, int T, int E, int k,
                                float* __restrict__ p, int* __restrict__ idx, float* __restrict__ w) {
  const int lane = threadIdx.x & 31;
  const long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= T) return;
  float v[kEPerLane];
  float m = -INFINITY;
#pragma unroll
  for (int j = 0; j < kEPerLane; ++j) {
    const int e = lane + 32 * j;
    v[j] = e < E ? __bfloat162float(logits[t * ldl + e]) : -INFINITY;
    m = fmaxf(m, v[j]);
  }
  m = warp_max(m);
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < kEPerLane; ++j) {
    const int e = lane + 32 * j;
    v[j] = e < E ? expf(v[j] - m) : 0.f;
    s += v[j];
  }
  s = warp_sum(s);
  const float inv = 1.f / s;
#pragma unroll
  for (int j = 0; j < kEPerLane; ++j) {
    const int e = lane + 32 * j;
    v[j] = e < E ? v[j] * inv : -1.f;   // taken (-1) or absent experts compare below every probability
    if (e < E) p[t * E + e] = v[j];
  }
  // A NaN probability (a NaN or Inf logit in the row) ranks below every number, so each round still picks a valid
  // expert not taken before: the row's weights are NaN and the NaN reaches the loss, never an index.
#pragma unroll
  for (int j = 0; j < kEPerLane; ++j)
    if (lane + 32 * j < E && v[j] != v[j]) v[j] = -0.5f;
  float sum = 0.f;   // NORM: the selected probabilities in slot order (NaN for a NaN row)
  for (int slot = 0; slot < k; ++slot) {
    float best = -2.f;
    int be = 0x7fffffff;
#pragma unroll
    for (int j = 0; j < kEPerLane; ++j)
      if (v[j] > best) { best = v[j]; be = lane + 32 * j; }   // ascending e: the first maximum is the lowest index
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oe = __shfl_xor_sync(0xffffffffu, be, o);
      if (ob > best || (ob == best && oe < be)) { best = ob; be = oe; }
    }
    if (lane == 0) {
      idx[t * k + slot] = be;
      w[t * k + slot] = best == -0.5f ? nan_f() : best;
    }
    if constexpr (NORM) sum += best == -0.5f ? nan_f() : best;
#pragma unroll
    for (int j = 0; j < kEPerLane; ++j)
      if (lane + 32 * j == be) v[j] = -1.f;
  }
  if constexpr (NORM) {
    __syncwarp();   // lane 0's w stores are visible to the warp
    for (int slot = lane; slot < k; slot += 32) w[t * k + slot] = __fdiv_rn(w[t * k + slot], sum);
  }
}

// one lane per token, one warp per chunk of 32 tokens: for every expert, the chunk's count and each assignment's rank
// among the chunk's earlier assignments to that expert (a token picks an expert at most once, so earlier = earlier
// token).  The rank is kept in pos until moe_pos_kernel adds the bases.
__global__ void moe_rank_kernel(const int* __restrict__ idx, int T, int E, int k, int* __restrict__ chunk_count,
                                int* __restrict__ pos) {
  const int lane = threadIdx.x & 31;
  const int chunk = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int nchunks = (T + 31) / 32;
  if (chunk >= nchunks) return;
  const long long t = (long long)chunk * 32 + lane;
  const bool live = t < T;
  uint32_t sel[kEPerLane];
#pragma unroll
  for (int j = 0; j < kEPerLane; ++j) sel[j] = 0;
  for (int s = 0; s < k && live; ++s) {
    const int e = idx[t * k + s];
    sel[e >> 5] |= 1u << (e & 31);
  }
  const uint32_t lt = (1u << lane) - 1u;
#pragma unroll
  for (int j = 0; j < kEPerLane; ++j) {
    if (32 * j >= E) break;
    for (int b = 0; b < 32 && 32 * j + b < E; ++b) {
      const int e = 32 * j + b;
      const bool mine = (sel[j] >> b) & 1u;
      const uint32_t bal = __ballot_sync(0xffffffffu, mine);
      if (lane == 0) chunk_count[(long long)chunk * E + e] = __popc(bal);
      if (mine)
        for (int s = 0; s < k; ++s)
          if (idx[t * k + s] == e) pos[t * k + s] = __popc(bal & lt);
    }
  }
}

// one CTA: per-expert exclusive scan of the chunk counts (the chunk bases), the counts, the 128-row padded segment
// table, the tile -> expert table for every 128-row tile up to rows_cap, and row_tok = -1 on every padding row
__global__ void moe_scan_kernel(int* __restrict__ chunk_count, int nchunks, int E, int* __restrict__ counts,
                                int* __restrict__ seg, int* __restrict__ tile_expert, int n_tiles,
                                int* __restrict__ row_tok) {
  __shared__ int s_seg[kMaxE + 1];
  __shared__ int s_cnt[kMaxE];
  for (int e = threadIdx.x; e < E; e += blockDim.x) {
    int run = 0;
    for (int c = 0; c < nchunks; ++c) {
      const int n = chunk_count[(long long)c * E + e];
      chunk_count[(long long)c * E + e] = run;   // in place: count -> base
      run += n;
    }
    s_cnt[e] = run;
    counts[e] = run;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int e = 0; e < E; ++e) {
      s_seg[e] = acc;
      acc += (s_cnt[e] + 127) & ~127;
    }
    s_seg[E] = acc;
  }
  __syncthreads();
  for (int e = threadIdx.x; e <= E; e += blockDim.x) seg[e] = s_seg[e];
  for (int i = threadIdx.x; i < n_tiles; i += blockDim.x) {
    const int r = i * 128;
    int e = -1;
    if (r < s_seg[E]) {   // the last expert whose segment starts at or before r
      int lo = 0, hi = E - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (s_seg[mid] <= r) lo = mid; else hi = mid - 1;
      }
      e = lo;
    }
    tile_expert[i] = e;
  }
  for (int i = threadIdx.x; i < E * 128; i += blockDim.x) {
    const int e = i >> 7, r = s_seg[e] + s_cnt[e] + (i & 127);
    if (r < s_seg[e + 1]) row_tok[r] = -1;
  }
}

// one thread per assignment: its row, and the row's assignment
__global__ void moe_pos_kernel(const int* __restrict__ idx, const int* __restrict__ chunk_base,
                               const int* __restrict__ seg, int T, int E, int k, int* __restrict__ pos,
                               int* __restrict__ row_tok) {
  const long long a = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (a >= (long long)T * k) return;
  const long long t = a / k;
  const int e = idx[a];
  const int r = seg[e] + chunk_base[(t >> 5) * E + e] + pos[a];
  pos[a] = r;
  row_tok[r] = (int)a;
}

// rows of the permuted layout, one CTA per row (rows at or past seg[E] are not touched):
//   permute  out[r] = x[t(r)], zero on a padding row
//   dcombine out[r] = bf16(w[a] * dy[t]) and dw[a] = sum_h dy[t, h] * yp[r, h] (fp32, fixed order), zero padding
// n_assign = T * k of src: a row whose assignment is outside [0, n_assign) gets a NaN row and reads nothing
template <bool DCOMBINE>
__global__ void moe_rows_kernel(const __nv_bfloat16* __restrict__ src, const int* __restrict__ row_tok,
                                const int* __restrict__ seg, int E, int k, int H, long long n_assign,
                                const float* __restrict__ w, const __nv_bfloat16* __restrict__ yp,
                                float* __restrict__ dw, __nv_bfloat16* __restrict__ out) {
  __shared__ float red[32];
  const long long r = blockIdx.x;
  if (r >= seg[E]) return;
  const int a = row_tok[r];
  __nv_bfloat16* orow = out + r * H;
  if (a == -1 || (unsigned long long)(long long)a >= (unsigned long long)n_assign) {
    float f[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) f[i] = a == -1 ? 0.f : nan_f();
    const bf16x8 z = pack8(f);
    for (int c = threadIdx.x * 8; c < H; c += blockDim.x * 8) st8(orow + c, z);
    return;
  }
  const __nv_bfloat16* srow = src + (long long)(a / k) * H;
  if constexpr (!DCOMBINE) {
    for (int c = threadIdx.x * 8; c < H; c += blockDim.x * 8) st8(orow + c, ld8(srow + c));
  } else {
    const float wa = w[a];
    float dot = 0.f;
    for (int c = threadIdx.x * 8; c < H; c += blockDim.x * 8) {
      float d[8], y[8], o[8];
      unpack8(ld8(srow + c), d);
      unpack8(ld8(yp + r * H + c), y);
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        o[i] = wa * d[i];
        dot = fmaf(d[i], y[i], dot);
      }
      st8(orow + c, pack8(o));
    }
    dot = block_sum(dot, red);
    if (threadIdx.x == 0) dw[a] = dot;
  }
}

// one CTA per token: out[t] = bf16(sum over slots, in slot order, of w[a] * yp[pos[a]]) in fp32; w null: weight 1.
// A row pos[a] outside [0, yp_rows) is not read: row 0 (yp_rows >= 1, the binding checks) is read in its place with a
// NaN weight, so the token's row is NaN, and the loads stay unconditional.
__global__ void moe_combine_kernel(const __nv_bfloat16* __restrict__ yp, long long yp_rows, const int* __restrict__ pos,
                                   const float* __restrict__ w, int k, int H, __nv_bfloat16* __restrict__ out) {
  const long long t = blockIdx.x;
  for (int c = threadIdx.x * 8; c < H; c += blockDim.x * 8) {
    float acc[8] = {};
    for (int s = 0; s < k; ++s) {
      const long long a = t * k + s;
      const int row = pos[a];
      const bool ok = (unsigned long long)(long long)row < (unsigned long long)yp_rows;
      const float wa = !ok ? nan_f() : (w ? w[a] : 1.f);
      float y[8];
      unpack8(ld8(yp + (ok ? (long long)row : 0ll) * H + c), y);
#pragma unroll
      for (int i = 0; i < 8; ++i) acc[i] = fmaf(wa, y[i], acc[i]);
    }
    st8(out + t * H + c, pack8(acc));
  }
}

// one warp per token: dp = dw at the selected experts (+ dpsum[e] everywhere), dlogits = bf16(p * (dp - sum p dp)).
// NORM (w = p_sel / S): the selected experts' dp is (dw_j - sum_i w_i dw_i) / S instead, with S and w recomputed from
// p and idx as the forward computed them, and the sum over slots in slot order.
template <bool NORM>
__global__ void moe_router_bwd_kernel(const float* __restrict__ p, const int* __restrict__ idx,
                                      const float* __restrict__ dw, const float* __restrict__ dpsum, int T, int E,
                                      int k, __nv_bfloat16* __restrict__ dlogits) {
  const int lane = threadIdx.x & 31;
  const long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= T) return;
  // NORM: S and sum_i w_i dw_i, the same on every lane.  An idx entry outside [0, E) is not followed: its probability
  // reads as NaN, so the token's row of dlogits is NaN.
  float S = 1.f, wdw = 0.f;
  if constexpr (NORM) {
    S = 0.f;
    for (int s = 0; s < k; ++s) {
      const int e = idx[t * k + s];
      S += (unsigned)e < (unsigned)E ? p[t * E + e] : nan_f();
    }
    for (int s = 0; s < k; ++s) {
      const int e = idx[t * k + s];
      const float pe = (unsigned)e < (unsigned)E ? p[t * E + e] : nan_f();
      wdw = fmaf(__fdiv_rn(pe, S), dw[t * k + s], wdw);
    }
  }
  float pv[kEPerLane], dp[kEPerLane];
  float dot = 0.f;
#pragma unroll
  for (int j = 0; j < kEPerLane; ++j) {
    const int e = lane + 32 * j;
    pv[j] = e < E ? p[t * E + e] : 0.f;
    dp[j] = (e < E && dpsum) ? dpsum[e] : 0.f;
    for (int s = 0; s < k; ++s)
      if (idx[t * k + s] == e) {
        if constexpr (NORM) dp[j] += __fdiv_rn(dw[t * k + s] - wdw, S);
        else dp[j] += dw[t * k + s];
      }
    dot = fmaf(pv[j], dp[j], dot);
  }
  dot = warp_sum(dot);
#pragma unroll
  for (int j = 0; j < kEPerLane; ++j) {
    const int e = lane + 32 * j;
    if (e < E) dlogits[t * E + e] = __float2bfloat16(pv[j] * (dp[j] - dot));
  }
}

// whole warps (block_sum shuffles with a full mask), at most 256, one 8-element vector per thread per pass
int row_threads(int H) {
  const int t = (H / 8 + 31) / 32 * 32;
  return t < 256 ? t : 256;
}

}  // namespace

long long moe_rows_cap(long long T, int E, int k) { return ((T * k + (long long)E * 127) + 127) / 128 * 128; }
long long moe_route_scratch(long long T, int E) { return (T + 31) / 32 * E; }

void moe_route(const void* logits, long long ldl, int T, int E, int k, bool norm_topk, float* p, int* idx, float* w,
               int* pos, int* seg, int* tile_expert, int* row_tok, int* counts, int* scratch, cudaStream_t s) {
  const int nchunks = (T + 31) / 32;
  (norm_topk ? moe_topk_kernel<true> : moe_topk_kernel<false>)<<<(T + 7) / 8, 256, 0, s>>>(
      (const __nv_bfloat16*)logits, ldl, T, E, k, p, idx, w);
  DTG_LAUNCH_CHECK();
  moe_rank_kernel<<<(nchunks + 7) / 8, 256, 0, s>>>(idx, T, E, k, scratch, pos);
  DTG_LAUNCH_CHECK();
  const int n_tiles = (int)(moe_rows_cap(T, E, k) / 128);
  moe_scan_kernel<<<1, 1024, 0, s>>>(scratch, nchunks, E, counts, seg, tile_expert, n_tiles, row_tok);
  DTG_LAUNCH_CHECK();
  const long long n = (long long)T * k;
  moe_pos_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(idx, scratch, seg, T, E, k, pos, row_tok);
  DTG_LAUNCH_CHECK();
  note_launch(4);
}

void moe_permute(const void* x, int T, const int* row_tok, const int* seg, int E, int k, int H, long long rows_cap,
                 void* out, cudaStream_t s) {
  if (rows_cap == 0) return;
  moe_rows_kernel<false><<<(unsigned)rows_cap, row_threads(H), 0, s>>>(
      (const __nv_bfloat16*)x, row_tok, seg, E, k, H, (long long)T * k, nullptr, nullptr, nullptr,
      (__nv_bfloat16*)out);
  DTG_LAUNCH_CHECK();
  note_launch();
}

void moe_combine(const void* yp, long long yp_rows, const int* pos, const float* w, int T, int k, int H, void* out,
                 cudaStream_t s) {
  if (T == 0) return;
  moe_combine_kernel<<<T, row_threads(H), 0, s>>>((const __nv_bfloat16*)yp, yp_rows, pos, w, k, H,
                                                  (__nv_bfloat16*)out);
  DTG_LAUNCH_CHECK();
  note_launch();
}

void moe_combine_bwd(const void* dy, int T, const void* yp, const int* row_tok, const int* seg, const float* w, int E,
                     int k, int H, long long rows_cap, void* dyp, float* dw, cudaStream_t s) {
  if (rows_cap == 0) return;
  moe_rows_kernel<true><<<(unsigned)rows_cap, row_threads(H), 0, s>>>(
      (const __nv_bfloat16*)dy, row_tok, seg, E, k, H, (long long)T * k, w, (const __nv_bfloat16*)yp, dw,
      (__nv_bfloat16*)dyp);
  DTG_LAUNCH_CHECK();
  note_launch();
}

void moe_router_bwd(const float* p, const int* idx, const float* dw, const float* dpsum, int T, int E, int k,
                    bool norm_topk, void* dlogits, cudaStream_t s) {
  if (T == 0) return;
  (norm_topk ? moe_router_bwd_kernel<true> : moe_router_bwd_kernel<false>)<<<(T + 7) / 8, 256, 0, s>>>(
      p, idx, dw, dpsum, T, E, k, (__nv_bfloat16*)dlogits);
  DTG_LAUNCH_CHECK();
  note_launch();
}

}  // namespace dtg
