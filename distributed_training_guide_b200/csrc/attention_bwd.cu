// Causal flash-attention backward on wgmma (head_dim D = 64 or 128, GQA).
//
// Two passes of ONE kernel template, each owning a 128-row block R and streaming 64-wide column
// blocks C of the opposite kind (no atomics, deterministic):
//
//   KV pass  R = 128 keys of a kv head, C = 64-query blocks of every q head in its GQA group
//            S^T = K_R Q_C^T,  dP^T = V_R dO_C^T          (wgmma m64n64k16 per warpgroup, fp32 in registers)
//            P^T = exp2(S^T*c - lse_q),  dS^T = P^T o (dP^T - delta_q) * scale
//            dV_R += P^T dO_C,   dK_R += dS^T Q_C         (wgmma m64nDk16, B = the C tile, MN-major)
//   Q pass   R = 128 queries of a q head, C = 64-key blocks
//            S = Q_R K_C^T,  dP = dO_R V_C^T,  dS = P o (dP - delta_q) * scale,   dQ_R += dS K_C
//
// 256 threads = two math warpgroups that own 64 rows of R each and keep their gradient accumulators in
// registers for the whole pass (up to 255 registers a thread: two warps per SM sub-partition); thread 0 also
// issues the TMA loads (resident R tiles once, C tiles into a 3-stage ring two blocks ahead).  delta = rowsum(dO o O) is produced by a small preprocess
// kernel.  DOC (document masking, key k visible to query q iff doc_start[q] <= k <= q): the KV pass stops at the first
// query block whose first query starts its document after the 128 keys, the Q pass starts at the block holding the
// document start of its first query, and the element mask also runs where a document begins inside a block.
// WIN (sliding window W, key k visible to query q only if q - W < k): the KV pass also stops after the query block
// holding R0 + 127 + W - 1 and bounds each key's queries by key + W; the Q pass also starts at the key block holding
// R0 - W + 1 and bounds each row's keys by row - W + 1.  Both bounds are arithmetic: no loads.
// Gradients are written into a dqkv buffer with the same fused layout as qkv, so the
// RoPE-backward kernel and the fused qkv dgrad/wgrad GEMMs consume it directly.
// D: every tile is D / 64 TMA boxes of 128-byte rows; S^T / dP^T take D / 16 k16 steps and each gradient
// accumulator is D / 2 fp32 registers.  Ranges, masks and block skipping do not depend on D.
#include <cuda.h>

#include <cstdlib>

#include "api.h"
#include "attention_common.cuh"
#include "common.cuh"
#include "gemm_common.cuh"
#include "ptx.cuh"

namespace dtg {
using namespace ptx;

namespace bwd {
constexpr int R_HALF = 128 * 128;      // 16 KB: one resident TMA box, [128 rows x 128 B]
constexpr int C_HALF = 64 * 128;       // 8 KB: one streamed TMA box, [64 rows x 128 B]
constexpr int Y_STAGES = 3;                   // TMA ring depth for the streamed tiles
constexpr float LOG2E = 1.4426950408889634f;
constexpr int THREADS = 256;
template <int D>
struct Layout {
  static constexpr int R_TILE = 128 * D * 2;   // resident tile: D / 64 boxes (32 KB at D = 128)
  static constexpr int C_TILE = 64 * D * 2;    // streamed tile: D / 64 boxes (16 KB at D = 128)
  static constexpr int OFF_R1 = 0, OFF_R2 = R_TILE;
  static constexpr int OFF_Y = 2 * R_TILE;                         // [stage][Y1 | Y2]
  static constexpr int OFF_P = OFF_Y + Y_STAGES * 2 * C_TILE;      // 16 KB: [128 rows x 64] bf16, K-major (SS form only)
  static constexpr int OFF_DS = OFF_P + 128 * 128;                 // 16 KB
  static constexpr int OFF_BAR = OFF_DS + 128 * 128;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
};
}  // namespace bwd

// delta[b, h, s] = sum_d dO * O   (one warp per (token, head) row of D elements, D / 32 per lane)
template <int D>
__global__ void attn_bwd_delta_kernel(const __nv_bfloat16* __restrict__ d_o, const __nv_bfloat16* __restrict__ o,
                                      float* __restrict__ delta, long long rows, int S, int nh) {
  const long long row = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const __nv_bfloat162* a = reinterpret_cast<const __nv_bfloat162*>(d_o + row * D) + lane * (D / 64);
  const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(o + row * D) + lane * (D / 64);
  float acc = 0.f;
#pragma unroll
  for (int i = 0; i < D / 64; ++i) {
    const float2 x = __bfloat1622float2(a[i]), y = __bfloat1622float2(b[i]);
    acc += x.x * y.x + x.y * y.y;
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    const long long tok = row / nh;
    const int h = (int)(row % nh);
    const long long bb = tok / S, ss = tok % S;
    delta[(bb * nh + h) * S + ss] = acc;
  }
}

// TS = true: P^T / dS^T (KV pass) and dS (Q pass) never go through shared memory — they are packed to bf16 in the
// registers they were computed in and feed the gradient MMAs as their A operand (RS form).  Per 128x64 block that
// removes 32 KB of shared-memory stores and 32 KB of A-operand reads.  TS = false stages them through
// 128B-swizzled shared memory (SS form).
template <bool KV_MODE, bool TS, bool DOC, bool WIN, int D>
__global__ void __launch_bounds__(bwd::THREADS, 1)
attn_bwd_kernel(const __grid_constant__ CUtensorMap tm_qkv_r, const __grid_constant__ CUtensorMap tm_qkv_c,
                const __grid_constant__ CUtensorMap tm_do_r, const __grid_constant__ CUtensorMap tm_do_c,
                const float* __restrict__ lse, const float* __restrict__ delta, __nv_bfloat16* __restrict__ dqkv,
                int S, int nh, int nkv, float scale, int num_r_blocks, long long* __restrict__ trace,
                const int* __restrict__ doc_start, int window) {
  using namespace bwd;
  using L = Layout<D>;
  constexpr int R_TILE = L::R_TILE, C_TILE = L::C_TILE, OFF_R1 = L::OFF_R1, OFF_R2 = L::OFF_R2, OFF_Y = L::OFF_Y,
                OFF_P = L::OFF_P, OFF_DS = L::OFF_DS, OFF_BAR = L::OFF_BAR;
  // optional in-kernel timeline (attn_bwd(..., trace=int64[1024])): CTA (0,0) records clock64() per column block:
  // [iter][0] scores ready, [1] P / dS computed, [3] gradient MMAs retired (thread 0)
  const bool tracing = trace != nullptr && blockIdx.x == 0 && blockIdx.y == 0;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + OFF_BAR);
  uint64_t* res_full = bars + 0;
  uint64_t* y_full = bars + 1;     // [Y_STAGES]
  uint64_t* y_empty = bars + 5;    // [Y_STAGES]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int group = nh / nkv;
  const int nht = nh + 2 * nkv;
  // KV pass: blockIdx.x = (batch, kv head), early key blocks (most work) first.
  // Q pass:  blockIdx.x = (batch, q head),  late query blocks first.
  const int heads_r = KV_MODE ? nkv : nh;
  const int head_r = blockIdx.x % heads_r;
  const int batch = blockIdx.x / heads_r;
  const int r_block = KV_MODE ? (int)blockIdx.y : num_r_blocks - 1 - (int)blockIdx.y;
  const int R0 = r_block * 128;
  const int kv_head = KV_MODE ? head_r : head_r / group;
  // column-block range
  int c_start = KV_MODE ? R0 / 64 : 0;
  int n_c = KV_MODE ? (S / 64 - c_start) : (R0 + 128) / 64;
  [[maybe_unused]] const int* ds_row = nullptr;   // DOC: this batch row's document starts
  // DOC: where the document mask starts to matter.  KV pass: the first column block holding a query whose document
  // starts after R0; Q pass: the document start of the last query of R.  Kept in a register so that no iteration waits
  // on a load before it can decide whether to mask.
  [[maybe_unused]] int doc_bound = 0;
  if constexpr (DOC) {
    // Every thread derives the same range from the same words (issue_y splits t by n_c), and every index stays
    // inside the plain causal range whatever doc_start holds.
    ds_row = doc_start + (long long)batch * S;
    if (KV_MODE) {
      // last query block whose first query (the smallest start) can see one of the keys R0..R0+127
      int lo = c_start, hi = S / 64 - 1;
      while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (__ldg(ds_row + mid * 64) <= R0 + 127) lo = mid;
        else hi = mid - 1;
      }
      n_c = lo - c_start + 1;
      hi = c_start + n_c;
      lo = c_start;
      while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        if (__ldg(ds_row + mid * 64 + 63) > R0) hi = mid;
        else lo = mid + 1;
      }
      doc_bound = lo;
    } else {
      // first key block: the one holding the document start of the first query
      c_start = min(max(__ldg(ds_row + R0) / 64, 0), n_c - 1);
      n_c -= c_start;
      doc_bound = __ldg(ds_row + R0 + 127);
    }
  }
  if constexpr (WIN) {
    // window >= 1, so both ranges keep at least one block
    if (KV_MODE) {
      // the last query that can see key R0 + 127 is R0 + 127 + W - 1
      n_c = min(n_c, min((R0 + 127 + window - 1) / 64, S / 64 - 1) - c_start + 1);
    } else {
      // the first key that query R0 can see is R0 - W + 1
      const int c_win = max(R0 - window + 1, 0) / 64;
      if (c_win > c_start) {
        n_c -= c_win - c_start;
        c_start = c_win;
      }
    }
  }
  const int n_iter = KV_MODE ? n_c * group : n_c;

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tm_qkv_r);
    prefetch_tensormap(&tm_qkv_c);
    prefetch_tensormap(&tm_do_r);
    prefetch_tensormap(&tm_do_c);
    mbar_init(res_full, 1);
    for (int i = 0; i < Y_STAGES; ++i) {
      mbar_init(&y_full[i], 1);
      mbar_init(&y_empty[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  // TMA issue (thread 0): the resident tiles once, then the streamed tiles Y_STAGES - 1 blocks ahead of the math
  auto issue_y = [&](int t) {
    const int st = t % Y_STAGES;
    const uint32_t ph = (uint32_t)((t / Y_STAGES) & 1);
    const int c = c_start + (KV_MODE ? t % n_c : t);
    const int C0 = c * 64;
    uint8_t* y1 = smem + OFF_Y + st * 2 * C_TILE;
    uint8_t* y2 = y1 + C_TILE;
    mbar_wait_mma(&y_empty[st], ph ^ 1);
    mbar_arrive_expect_tx(&y_full[st], 2 * C_TILE);
    if (KV_MODE) {
      const int qh = kv_head * group + t / n_c;
#pragma unroll
      for (int b = 0; b < D / 64; ++b) tma_load_4d(&tm_qkv_c, &y_full[st], y1 + b * C_HALF, 64 * b, qh, C0, batch);
#pragma unroll
      for (int b = 0; b < D / 64; ++b) tma_load_4d(&tm_do_c, &y_full[st], y2 + b * C_HALF, 64 * b, qh, C0, batch);
    } else {
#pragma unroll
      for (int b = 0; b < D / 64; ++b)
        tma_load_4d(&tm_qkv_c, &y_full[st], y1 + b * C_HALF, 64 * b, nh + kv_head, C0, batch);
#pragma unroll
      for (int b = 0; b < D / 64; ++b)
        tma_load_4d(&tm_qkv_c, &y_full[st], y2 + b * C_HALF, 64 * b, nh + nkv + kv_head, C0, batch);
    }
  };
  if (threadIdx.x == 0) {
    // resident tiles: KV pass -> K_R, V_R ; Q pass -> Q_R, dO_R
    mbar_arrive_expect_tx(res_full, 2 * R_TILE);
    if (KV_MODE) {
#pragma unroll
      for (int b = 0; b < D / 64; ++b)
        tma_load_4d(&tm_qkv_r, res_full, smem + OFF_R1 + b * R_HALF, 64 * b, nh + kv_head, R0, batch);
#pragma unroll
      for (int b = 0; b < D / 64; ++b)
        tma_load_4d(&tm_qkv_r, res_full, smem + OFF_R2 + b * R_HALF, 64 * b, nh + nkv + kv_head, R0, batch);
    } else {
#pragma unroll
      for (int b = 0; b < D / 64; ++b) tma_load_4d(&tm_qkv_r, res_full, smem + OFF_R1 + b * R_HALF, 64 * b, head_r, R0, batch);
#pragma unroll
      for (int b = 0; b < D / 64; ++b) tma_load_4d(&tm_do_r, res_full, smem + OFF_R2 + b * R_HALF, 64 * b, head_r, R0, batch);
    }
    for (int t = 0; t < Y_STAGES - 1 && t < n_iter; ++t) issue_y(t);
  }
  {
    const int half = wg;                               // rows [64*half, 64*half + 64) of R
    const int g = lane >> 2, tq = lane & 3;
    const int rl0 = half * 64 + (warp & 3) * 16 + g;   // my rows of R: rl0 and rl0 + 8
    const bool signal = (threadIdx.x & 127) == 0;
    const bool tr_thread = tracing && threadIdx.x == 0;
    const float sl2 = scale * LOG2E;
    float lse_r[2] = {0.f, 0.f}, delta_r[2] = {0.f, 0.f};
    // DOC, Q pass: my rows' document starts.  KV pass: for each of my two keys, the first query that starts its
    // document after the key (the next document's first token, S if none): with starts non-decreasing along a row,
    // key k is visible to query q >= k iff q < that bound, so the mask needs no per-column load.
    // WIN tightens both: Q pass max(start, row - W + 1), KV pass min(bound, key + W).
    [[maybe_unused]] int ds_r[2] = {0, 0};
    if constexpr (DOC && KV_MODE) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int k = R0 + rl0 + 8 * h;
        int lo = k + 1, hi = S;
        while (lo < hi) {
          const int mid = (lo + hi) >> 1;
          if (__ldg(ds_row + mid) > k) hi = mid;
          else lo = mid + 1;
        }
        ds_r[h] = lo;
      }
    }
    if (!KV_MODE) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const long long idx = ((long long)batch * nh + head_r) * S + R0 + rl0 + 8 * h;
        lse_r[h] = lse[idx] * LOG2E;
        delta_r[h] = delta[idx];
        if constexpr (DOC) ds_r[h] = __ldg(ds_row + R0 + rl0 + 8 * h);
      }
    }
    if constexpr (WIN) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int idx = R0 + rl0 + 8 * h;   // my key (KV pass) or my query (Q pass)
        if constexpr (KV_MODE) ds_r[h] = DOC ? min(ds_r[h], idx + window) : idx + window;
        else ds_r[h] = max(ds_r[h], idx - window + 1);
      }
    }
    [[maybe_unused]] float acc_a[KV_MODE ? D / 2 : 1];   // dV (KV pass)
    float acc_b[D / 2];                                  // dK (KV pass) / dQ (Q pass)
#pragma unroll
    for (int i = 0; i < D / 2; ++i) {
      if constexpr (KV_MODE) acc_a[i] = 0.f;
      acc_b[i] = 0.f;
    }
    const uint32_t r1 = smem_u32(smem + OFF_R1) + (uint32_t)(half * 8192);
    const uint32_t r2 = smem_u32(smem + OFF_R2) + (uint32_t)(half * 8192);
    const uint32_t sp = smem_u32(smem + OFF_P) + (uint32_t)(half * 8192);
    const uint32_t sds = smem_u32(smem + OFF_DS) + (uint32_t)(half * 8192);
    mbar_wait_mma(res_full, 0);
    for (int t = 0; t < n_iter; ++t) {
      // refill the stage block t-1 used (both warpgroups must be done with it; the other one is at most one block
      // behind)
      if (threadIdx.x == 0 && t + Y_STAGES - 1 < n_iter) issue_y(t + Y_STAGES - 1);
      const int ys = t % Y_STAGES;
      const int c = c_start + (KV_MODE ? t % n_c : t);
      const int C0 = c * 64;
      [[maybe_unused]] const float* lq = nullptr;
      [[maybe_unused]] const float* dq = nullptr;
      if (KV_MODE) {  // per-column statistics of the queries of this block
        const int qh = kv_head * group + t / n_c;
        lq = lse + ((long long)batch * nh + qh) * S + C0;
        dq = delta + ((long long)batch * nh + qh) * S + C0;
      }
      mbar_wait_mma(&y_full[ys], (uint32_t)((t / Y_STAGES) & 1));
      const uint32_t y1 = smem_u32(smem + OFF_Y + ys * 2 * C_TILE), y2 = y1 + C_TILE;
      float sc[32], dp[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) sc[i] = dp[i] = 0.f;
      wgmma_fence();
      fence_regs(sc);
      fence_regs(dp);
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t ra = (uint32_t)((kk >> 2) * R_HALF + (kk & 3) * 32);
        const uint32_t cb = (uint32_t)((kk >> 2) * C_HALF + (kk & 3) * 32);
        wgmma_m64n64k16_ss<0, 0>(sc, desc_kmajor_sw128(r1 + ra), desc_kmajor_sw128(y1 + cb), 1u);
      }
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) {
        const uint32_t ra = (uint32_t)((kk >> 2) * R_HALF + (kk & 3) * 32);
        const uint32_t cb = (uint32_t)((kk >> 2) * C_HALF + (kk & 3) * 32);
        wgmma_m64n64k16_ss<0, 0>(dp, desc_kmajor_sw128(r2 + ra), desc_kmajor_sw128(y2 + cb), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(sc);
      fence_regs(dp);
      if (tr_thread && t < 64) trace[t * 8 + 0] = clock64();
      // causal: query index >= key index.  Only blocks that touch the diagonal need the compare.
      bool need_mask = KV_MODE ? (C0 < R0 + 127) : (C0 + 63 > R0);
      // DOC: and key index >= the query's document start, where a document begins inside the block
      if constexpr (DOC) need_mask = need_mask || (KV_MODE ? c >= doc_bound : C0 < doc_bound);
      // WIN: and key index > query index - W, where the window edge of some row of R lies inside the block
      if constexpr (WIN) need_mask = need_mask || (KV_MODE ? C0 + 63 >= R0 + window : C0 < R0 + 128 - window);
#pragma unroll
      for (int i = 0; i < 32; ++i) {
        const int col = 8 * (i >> 2) + 2 * tq + (i & 1);
        const int h = (i >> 1) & 1;
        const int row = rl0 + 8 * h;
        float l2, dl;
        if constexpr (KV_MODE) {
          l2 = __ldg(lq + col) * LOG2E;
          dl = __ldg(dq + col);
        } else {
          l2 = lse_r[h];
          dl = delta_r[h];
        }
        float p = fast_exp2(fmaf(sc[i], sl2, -l2));
        if (need_mask) {
          bool ok = KV_MODE ? (C0 + col >= R0 + row) : (R0 + row >= C0 + col);
          if constexpr (DOC || WIN) ok = ok && (KV_MODE ? C0 + col < ds_r[h] : C0 + col >= ds_r[h]);
          p = ok ? p : 0.f;
        }
        sc[i] = p;
        dp[i] = p * (dp[i] - dl) * scale;
      }
      uint32_t pp[4][4], pd[4][4];   // bf16 A fragments of the four k16 steps of the gradient MMAs
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          pp[kk][r] = pack_bf16x2(sc[8 * kk + 2 * r], sc[8 * kk + 2 * r + 1]);
          pd[kk][r] = pack_bf16x2(dp[8 * kk + 2 * r], dp[8 * kk + 2 * r + 1]);
        }
      if (tr_thread && t < 64) trace[t * 8 + 1] = clock64();
      if constexpr (!TS) {
        // [128 rows x 64 columns] bf16, 128B swizzle (what TMA would have written)
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int row = rl0 + ((r & 1) ? 8 : 0);
            const int col = 16 * kk + ((r & 2) ? 8 : 0) + 2 * tq;
            const int off = row * 128 + (((col >> 3) ^ (row & 7)) << 4) + (col & 7) * 2;
            if (KV_MODE) *reinterpret_cast<uint32_t*>(smem + OFF_P + off) = pp[kk][r];
            *reinterpret_cast<uint32_t*>(smem + OFF_DS + off) = pd[kk][r];
          }
        fence_proxy_async();            // generic-proxy writes -> visible to the async proxy (wgmma)
        named_bar_sync(1 + half, 128);
      }
      wgmma_fence();
      if constexpr (KV_MODE) fence_regs(acc_a);
      fence_regs(acc_b);
      if constexpr (KV_MODE) {
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) {  // dV += P^T dO_C
          const uint64_t db = desc_mnmajor_sw128(y2 + kk * 2048, C_HALF);
          if constexpr (TS) wgmma_bf16_rs<1>(acc_a, pp[kk], db, 1u);
          else wgmma_bf16_ss<0, 1>(acc_a, desc_kmajor_sw128(sp + kk * 32), db, 1u);
        }
      }
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) {    // dK += dS^T Q_C   /   dQ += dS K_C
        const uint64_t db = desc_mnmajor_sw128(y1 + kk * 2048, C_HALF);
        if constexpr (TS) wgmma_bf16_rs<1>(acc_b, pd[kk], db, 1u);
        else wgmma_bf16_ss<0, 1>(acc_b, desc_kmajor_sw128(sds + kk * 32), db, 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      if constexpr (KV_MODE) fence_regs(acc_a);
      fence_regs(acc_b);
      if (signal) mbar_arrive(&y_empty[ys]);
      if constexpr (!TS) named_bar_sync(1 + half, 128);   // every warp's MMAs are done with P / dS
      if (tr_thread && t < 64) trace[t * 8 + 3] = clock64();
    }
    // write the accumulated gradients of my two rows
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const long long tok = (long long)batch * S + R0 + rl0 + 8 * h;
      auto write_row = [&](const float (&acc)[D / 2], int out_head) {
        __nv_bfloat16* dst = dqkv + (tok * nht + out_head) * (long long)D;
#pragma unroll
        for (int nb = 0; nb < D / 8; ++nb)
          *reinterpret_cast<__nv_bfloat162*>(dst + 8 * nb + 2 * tq) =
              __floats2bfloat162_rn(acc[4 * nb + 2 * h], acc[4 * nb + 2 * h + 1]);
      };
      if constexpr (KV_MODE) {
        write_row(acc_a, nh + nkv + kv_head);  // dV
        write_row(acc_b, nh + kv_head);        // dK
      } else {
        write_row(acc_b, head_r);              // dQ
      }
    }
  }
}

template <bool TS, bool DOC, bool WIN, int D>
static void launch_attn_bwd(const CUtensorMap& tq_r, const CUtensorMap& tq_c, const CUtensorMap& td_r,
                            const CUtensorMap& td_c, const float* lse, const float* delta, void* dqkv, int B, int S,
                            int nh, int nkv, float scale, long long* trace, const int* doc_start, int window,
                            cudaStream_t s) {
  constexpr int smem = bwd::Layout<D>::SMEM_BYTES;
  static bool attr = false;
  if (!attr) {
    DTG_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_kernel<true, TS, DOC, WIN, D>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    DTG_CUDA_CHECK(cudaFuncSetAttribute(attn_bwd_kernel<false, TS, DOC, WIN, D>,
                                        cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    attr = true;
  }
  const int nblk = S / 128;
  attn_bwd_kernel<true, TS, DOC, WIN, D><<<dim3(B * nkv, nblk, 1), bwd::THREADS, smem, s>>>(
      tq_r, tq_c, td_r, td_c, lse, delta, (__nv_bfloat16*)dqkv, S, nh, nkv, scale, nblk, trace, doc_start, window);
  attn_bwd_kernel<false, TS, DOC, WIN, D><<<dim3(B * nh, nblk, 1), bwd::THREADS, smem, s>>>(
      tq_r, tq_c, td_r, td_c, lse, delta, (__nv_bfloat16*)dqkv, S, nh, nkv, scale, nblk, trace ? trace + 512 : nullptr,
      doc_start, window);
}

template <bool TS, int D>
static void dispatch_attn_bwd(const CUtensorMap& tq_r, const CUtensorMap& tq_c, const CUtensorMap& td_r,
                              const CUtensorMap& td_c, const float* lse, const float* delta, void* dqkv, int B, int S,
                              int nh, int nkv, float scale, long long* trace, const int* doc_start, int window,
                              cudaStream_t s) {
  // a window that covers the whole sequence masks nothing: run the kernels without it
  if (window > 0 && window < S) {
    if (doc_start) launch_attn_bwd<TS, true, true, D>(tq_r, tq_c, td_r, td_c, lse, delta, dqkv, B, S, nh, nkv, scale, trace, doc_start, window, s);
    else launch_attn_bwd<TS, false, true, D>(tq_r, tq_c, td_r, td_c, lse, delta, dqkv, B, S, nh, nkv, scale, trace, nullptr, window, s);
  } else {
    if (doc_start) launch_attn_bwd<TS, true, false, D>(tq_r, tq_c, td_r, td_c, lse, delta, dqkv, B, S, nh, nkv, scale, trace, doc_start, 0, s);
    else launch_attn_bwd<TS, false, false, D>(tq_r, tq_c, td_r, td_c, lse, delta, dqkv, B, S, nh, nkv, scale, trace, nullptr, 0, s);
  }
}

void attn_bwd(const void* qkv, const void* o, const void* d_o, const float* lse, float* delta, float* trace_buf,
              void* dqkv, int B, int S, int nh, int nkv, float scale, int mode, cudaStream_t s,
              const int* doc_start, int window, int head_dim) {
  long long* trace = reinterpret_cast<long long*>(trace_buf);  // [2][64][8] int64 or nullptr
  if (S % 128 != 0) throw std::runtime_error("attn_bwd: sequence length must be a multiple of 128");
  if (window < 0) throw std::runtime_error("attn_bwd: window must be >= 1 (0 = no window)");
  if (nh < 1 || nkv < 1 || nh % nkv != 0) throw std::runtime_error("attn_bwd: nh must be a positive multiple of nkv");
  if (head_dim != 64 && head_dim != 128) throw std::runtime_error("attn_bwd: head_dim must be 64 or 128");
  // every tensor map is encoded (and can refuse its pointer) before the first launch
  const CUtensorMap tq_r = make_tmap_heads(qkv, B, S, nh + 2 * nkv, 128, head_dim);
  const CUtensorMap tq_c = make_tmap_heads(qkv, B, S, nh + 2 * nkv, 64, head_dim);
  const CUtensorMap td_r = make_tmap_heads(d_o, B, S, nh, 128, head_dim);
  const CUtensorMap td_c = make_tmap_heads(d_o, B, S, nh, 64, head_dim);
  const long long rows = (long long)B * S * nh;
  const unsigned delta_blocks = (unsigned)((rows * 32 + 255) / 256);
  if (head_dim == 128)
    attn_bwd_delta_kernel<128><<<delta_blocks, 256, 0, s>>>((const __nv_bfloat16*)d_o, (const __nv_bfloat16*)o, delta,
                                                            rows, S, nh);
  else
    attn_bwd_delta_kernel<64><<<delta_blocks, 256, 0, s>>>((const __nv_bfloat16*)d_o, (const __nv_bfloat16*)o, delta,
                                                           rows, S, nh);
  static const bool ts_default = []() {   // DTG_ATTN_BWD=rs (default: P / dS stay in registers) | ss
    const char* e = getenv("DTG_ATTN_BWD");
    return e ? e[0] != 's' : true;
  }();
  const bool ts = mode == 0 ? ts_default : mode == 2;   // mode: 0 default, 1 = ss, 2 = rs
  if (head_dim == 128) {
    if (ts) dispatch_attn_bwd<true, 128>(tq_r, tq_c, td_r, td_c, lse, delta, dqkv, B, S, nh, nkv, scale, trace, doc_start, window, s);
    else dispatch_attn_bwd<false, 128>(tq_r, tq_c, td_r, td_c, lse, delta, dqkv, B, S, nh, nkv, scale, trace, doc_start, window, s);
  } else {
    if (ts) dispatch_attn_bwd<true, 64>(tq_r, tq_c, td_r, td_c, lse, delta, dqkv, B, S, nh, nkv, scale, trace, doc_start, window, s);
    else dispatch_attn_bwd<false, 64>(tq_r, tq_c, td_r, td_c, lse, delta, dqkv, B, S, nh, nkv, scale, trace, doc_start, window, s);
  }
  note_launch(3);
  DTG_LAUNCH_CHECK();
}

}  // namespace dtg
