// Causal flash-attention forward on wgmma (head_dim D = 64 or 128, GQA), reading q/k/v straight out of
// the fused qkv activation [B, S, nh + 2*nkv, D] through one strided 4-D TMA descriptor (no
// transposes, no repeat_kv copies).  One CTA = one (batch, q-head, 128-query block), 384 threads:
//
//   warpgroup 0     TMA producer (one elected lane of warp 0): Q once; K_j / V_j into 2-stage rings
//                   (separate barriers so Q K^T can start as soon as K lands)
//   warpgroups 1-2  64 query rows each: S = Q K_j^T (wgmma m64n128k16, fp32 in registers), online
//                   softmax in registers (a row lives in the 4 threads of a quad), O += P_j V_j
//                   (wgmma m64nDk16, V as an MN-major operand), final O / l and the logsumexp written from registers.
//
// D: a 64-wide bf16 row is one 128-byte swizzle span, so every [rows x D] tile is D / 64 TMA boxes of
// [rows x 128 B] ("halves" at D = 128, one box at D = 64); S = Q K^T takes D / 16 k16 steps and the O
// accumulator is D / 2 fp32 registers.  Tiles, threads, masks and block skipping do not depend on D.
//
// P_REGS (version 2): P is packed to bf16 in the registers it was computed in and feeds the PV wgmma as its
// A operand (RS form) — the accumulator fragment of two n8 column blocks is exactly the A fragment of one
// k16 step.  Version 1 stages P through 128B-swizzled shared memory (SS form).
//
// DOC (document masking): doc_start[b, q] is the first token of query q's document and key k is visible to q iff
// doc_start[q] <= k <= q.  The first query of the tile has the smallest start, so the CTA visits key blocks from
// doc_start[q0] / 128 to the diagonal and skips the rest; the element mask runs on the diagonal block and on the
// blocks where some row's document begins.  DOC = false compiles to the plain causal kernel.
//
// WIN (sliding window, runtime `window` = W >= 1): query q sees key k only if k > q - W, a second lower bound that
// also never decreases along a row.  The CTA starts at the key block holding max(doc start, q0 - W + 1) and masks the
// (at most two) blocks that straddle some row's window edge.  WIN = false compiles to the kernel without it.
//
// Replaces torch SDPA / flash-attn-2 (mma.sync) that the reference uses (SURVEY.md K2/K3).
#include <cuda.h>

#include "api.h"
#include "attention_common.cuh"
#include "common.cuh"
#include "gemm_common.cuh"
#include "ptx.cuh"

namespace dtg {
using namespace ptx;

namespace fwd {
constexpr int BM = 128, BN = 128;
constexpr int HALF_BYTES = 128 * 128;      // 16 KB: one TMA box, 64 columns of [128 rows x 128 B]
constexpr int P_BYTES = 128 * 128 * 2;     // 32 KB: P, [128 rows x 128 keys] bf16 (SS form only)
constexpr int THREADS = 384;
template <bool P_REGS, int D>
struct Layout {
  static constexpr int TILE_BYTES = 128 * D * 2;   // one Q / K / V tile: D / 64 boxes
  static constexpr int OFF_Q = 0, OFF_K = TILE_BYTES, OFF_V = 3 * TILE_BYTES, OFF_P = 5 * TILE_BYTES;
  static constexpr int OFF_BAR = P_REGS ? OFF_P : OFF_P + P_BYTES;
  static constexpr int SMEM_BYTES = OFF_BAR + 256 + 1024;
};
}  // namespace fwd

template <bool P_REGS, bool DOC, bool WIN, int D>
__global__ void __launch_bounds__(fwd::THREADS, 1)
attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_qkv, __nv_bfloat16* __restrict__ o, float* __restrict__ lse,
                int S, int nh, int nkv, float scale_log2, int num_m_blocks, const int* __restrict__ doc_start,
                int window) {
  using namespace fwd;
  using L = Layout<P_REGS, D>;
  constexpr int TILE_BYTES = L::TILE_BYTES, OFF_Q = L::OFF_Q, OFF_K = L::OFF_K, OFF_V = L::OFF_V, OFF_P = L::OFF_P;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L::OFF_BAR);
  uint64_t* q_full = bars + 0;
  uint64_t* k_full = bars + 1;    // [2]
  uint64_t* v_full = bars + 3;    // [2]
  uint64_t* k_empty = bars + 5;   // [2]
  uint64_t* v_empty = bars + 7;   // [2]

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  // longest rows first: CTAs are dispatched in blockIdx order, causal work grows with the q block
  // (grid = (B*nh, num_m_blocks): x varies fastest, so every head's longest block goes out first)
  const int m_block = num_m_blocks - 1 - (int)blockIdx.y;
  const int head = blockIdx.x % nh;
  const int batch = blockIdx.x / nh;
  const int kv_head = head / (nh / nkv);
  const int n_blocks = m_block + 1;  // causal, BM == BN
  const int q0 = m_block * BM;
  // first key block: the block holding the start of the tile's first query, clamped into [0, m_block]
  int j_lo = 0;
  if constexpr (DOC) j_lo = min(max(__ldg(doc_start + (long long)batch * S + q0) / BN, 0), m_block);
  // WIN: and the block holding the first query's window start (window >= 1, so never past the diagonal)
  if constexpr (WIN) j_lo = max(j_lo, max(q0 - window + 1, 0) / BN);

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tm_qkv);
    mbar_init(q_full, 1);
    for (int i = 0; i < 2; ++i) {
      mbar_init(&k_full[i], 1);
      mbar_init(&v_full[i], 1);
      mbar_init(&k_empty[i], 2);
      mbar_init(&v_empty[i], 2);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (warp == 0 && elect_one()) {
      // Q tile: D / 64 boxes of 64 columns
      mbar_arrive_expect_tx(q_full, TILE_BYTES);
#pragma unroll
      for (int c = 0; c < D / 64; ++c) tma_load_4d(&tm_qkv, q_full, smem + OFF_Q + c * HALF_BYTES, 64 * c, head, q0, batch);
      const int kh = nh + kv_head, vh = nh + nkv + kv_head;
      for (int j = j_lo; j < n_blocks; ++j) {
        const int st = (j - j_lo) & 1;
        const uint32_t ph = (uint32_t)(((j - j_lo) >> 1) & 1);
        mbar_wait_mma(&k_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&k_full[st], TILE_BYTES);
#pragma unroll
        for (int c = 0; c < D / 64; ++c)
          tma_load_4d(&tm_qkv, &k_full[st], smem + OFF_K + st * TILE_BYTES + c * HALF_BYTES, 64 * c, kh, j * BN, batch);
        mbar_wait_mma(&v_empty[st], ph ^ 1);
        mbar_arrive_expect_tx(&v_full[st], TILE_BYTES);
#pragma unroll
        for (int c = 0; c < D / 64; ++c)
          tma_load_4d(&tm_qkv, &v_full[st], smem + OFF_V + st * TILE_BYTES + c * HALF_BYTES, 64 * c, vh, j * BN, batch);
      }
    }
  } else {
    // ===================== softmax warpgroups =====================
    const int half = wg - 1;                       // query rows [64*half, 64*half + 64) of the tile
    const int g = lane >> 2, tq = lane & 3;
    const int rl0 = half * 64 + (warp & 3) * 16 + g;   // my rows: rl0 and rl0 + 8 (tile-local)
    const bool signal = (threadIdx.x & 127) == 0;
    const uint32_t sq = smem_u32(smem + OFF_Q) + (uint32_t)(half * 8192);
    float acc[D / 2];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) acc[i] = 0.f;
    float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};  // l_run: this thread's partial row sums
    // DOC / WIN: my rows' first visible key, max(document start, row - W + 1)
    [[maybe_unused]] int ds_r[2] = {0, 0};
    if constexpr (DOC && P_REGS) {
      const int* ds = doc_start + (long long)batch * S + q0;
      ds_r[0] = __ldg(ds + rl0);
      ds_r[1] = __ldg(ds + rl0 + 8);
    }
    if constexpr (WIN && P_REGS) {
      ds_r[0] = max(ds_r[0], q0 + rl0 - window + 1);
      ds_r[1] = max(ds_r[1], q0 + rl0 + 8 - window + 1);
    }
    mbar_wait_mma(q_full, 0);
    for (int j = j_lo; j < n_blocks; ++j) {
      const int st = (j - j_lo) & 1;
      const uint32_t ph = (uint32_t)(((j - j_lo) >> 1) & 1);
      float s[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) s[i] = 0.f;
      mbar_wait_mma(&k_full[st], ph);
      {
        const uint32_t sk = smem_u32(smem + OFF_K + st * TILE_BYTES);
        wgmma_fence();
        fence_regs(s);
#pragma unroll
        for (int kk = 0; kk < D / 16; ++kk) {
          const uint32_t off = (uint32_t)((kk >> 2) * HALF_BYTES + (kk & 3) * 32);
          wgmma_m64n128k16_ss<0, 0>(s, desc_kmajor_sw128(sq + off), desc_kmajor_sw128(sk + off), 1u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(s);
      }
      if (signal) mbar_arrive(&k_empty[st]);
      if constexpr (DOC || WIN) {
        // mask keys after the query (diagonal block) and keys before the query's document start or window (blocks
        // where one of my rows' first visible key lies)
        if constexpr (DOC && !P_REGS) {
          // version 1 runs at the 168-register cap: re-read the two starts (L1 hits) rather than keep them live
          const int* ds = doc_start + (long long)batch * S + q0;
          ds_r[0] = __ldg(ds + rl0);
          ds_r[1] = __ldg(ds + rl0 + 8);
        }
        if constexpr (WIN && !P_REGS) {
          ds_r[0] = max(ds_r[0], q0 + rl0 - window + 1);
          ds_r[1] = max(ds_r[1], q0 + rl0 + 8 - window + 1);
        }
        if (j == n_blocks - 1 || j * BN < max(ds_r[0], ds_r[1])) {
#pragma unroll
          for (int i = 0; i < 64; ++i) {
            const int key = j * BN + 8 * (i >> 2) + 2 * tq + (i & 1);
            const int h = (i >> 1) & 1;
            if (key > q0 + rl0 + 8 * h || key < ds_r[h]) s[i] = -INFINITY;
          }
        }
      } else if (j == n_blocks - 1) {   // diagonal block: mask keys after the query
#pragma unroll
        for (int i = 0; i < 64; ++i) {
          const int col = 8 * (i >> 2) + 2 * tq + (i & 1);
          const int row = rl0 + ((i & 2) ? 8 : 0);
          if (col > row) s[i] = -INFINITY;
        }
      }
      float alpha[2], mb[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mx = -INFINITY;
#pragma unroll
        for (int i = 0; i < 32; ++i) mx = fmaxf(mx, s[4 * (i >> 1) + 2 * h + (i & 1)]);
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        mx = fmaxf(m_run[h], mx);
        alpha[h] = fast_exp2((m_run[h] - mx) * scale_log2);  // 0 on the first block (m_run = -inf)
        mb[h] = mx * scale_log2;
        if constexpr (DOC || WIN) {
          // a row whose first visible key comes after every key seen so far: keep it empty (p = 0) instead of
          // exp2(-inf - -inf) = NaN
          if (mx == -INFINITY) {
            alpha[h] = 1.f;
            mb[h] = 0.f;
          }
        }
        m_run[h] = mx;
      }
      float sum[2] = {0.f, 0.f};
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int h = (i >> 1) & 1;
        s[i] = fast_exp2(fmaf(s[i], scale_log2, -mb[h]));
        sum[h] += s[i];
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) l_run[h] = l_run[h] * alpha[h] + sum[h];
#pragma unroll
      for (int i = 0; i < D / 2; ++i) acc[i] *= alpha[(i >> 1) & 1];
      uint32_t pa[8][4];   // P as bf16 A fragments, one per k16 step of the PV MMA
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
#pragma unroll
        for (int r = 0; r < 4; ++r) pa[kk][r] = pack_bf16x2(s[8 * kk + 2 * r], s[8 * kk + 2 * r + 1]);
      uint32_t sp = 0;
      if constexpr (!P_REGS) {
        // P -> [128 rows x 128 keys] bf16, two 64-key halves, 128B swizzle (what TMA would have written)
        uint8_t* pbase = smem + OFF_P;
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
#pragma unroll
          for (int r = 0; r < 4; ++r) {
            const int row = rl0 + ((r & 1) ? 8 : 0);
            const int key = 16 * kk + ((r & 2) ? 8 : 0) + 2 * tq;
            const int chunk = (key & 63) >> 3;
            *reinterpret_cast<uint32_t*>(pbase + (key >> 6) * HALF_BYTES + row * 128 + ((chunk ^ (row & 7)) << 4) +
                                         (key & 7) * 2) = pa[kk][r];
          }
        fence_proxy_async();           // generic-proxy writes of P -> visible to the async proxy (wgmma)
        named_bar_sync(1 + half, 128);
        sp = smem_u32(pbase) + (uint32_t)(half * 8192);
      }
      mbar_wait_mma(&v_full[st], ph);
      {
        const uint32_t sv = smem_u32(smem + OFF_V + st * TILE_BYTES);
        wgmma_fence();
        fence_regs(acc);
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) {
          const uint64_t db = desc_mnmajor_sw128(sv + (uint32_t)(kk * 2048), HALF_BYTES);
          if constexpr (P_REGS) {
            wgmma_bf16_rs<1>(acc, pa[kk], db, 1u);
          } else {
            const uint64_t da = desc_kmajor_sw128(sp + (uint32_t)((kk >> 2) * HALF_BYTES + (kk & 3) * 32));
            wgmma_bf16_ss<0, 1>(acc, da, db, 1u);
          }
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(acc);
      }
      if (signal) mbar_arrive(&v_empty[st]);
      if constexpr (!P_REGS) named_bar_sync(1 + half, 128);   // every warp's PV MMAs are done with P
    }
    // epilogue: O / l -> bf16 -> global ; logsumexp
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float l = l_run[h];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv_l = 1.f / l;
      const int row = rl0 + 8 * h;
      const long long tok = (long long)batch * S + q0 + row;
      __nv_bfloat16* orow = o + (tok * nh + head) * (long long)D;
#pragma unroll
      for (int nb = 0; nb < D / 8; ++nb)
        *reinterpret_cast<__nv_bfloat162*>(orow + 8 * nb + 2 * tq) =
            __floats2bfloat162_rn(acc[4 * nb + 2 * h] * inv_l, acc[4 * nb + 2 * h + 1] * inv_l);
      // natural-log logsumexp of the scaled scores
      if (tq == 0)
        lse[((long long)batch * nh + head) * S + q0 + row] = m_run[h] * scale_log2 * 0.6931471805599453f + __logf(l);
    }
  }
}

CUtensorMap make_tmap_heads(const void* base, int B, int S, int heads, int box_rows, int D) {
  // [B, S, heads, D] bf16 viewed as dims {D, heads, S, B}; box {64, 1, box_rows, 1}, 128B swizzle
  uint64_t dims[4] = {(uint64_t)D, (uint64_t)heads, (uint64_t)S, (uint64_t)B};
  uint64_t strides[3] = {(uint64_t)D * 2, (uint64_t)heads * D * 2, (uint64_t)S * heads * D * 2};
  uint32_t box[4] = {64, 1, (uint32_t)box_rows, 1};
  return make_tmap_bf16(base, 4, dims, strides, box, true);
}

template <bool P_REGS, bool DOC, bool WIN, int D>
static void launch_attn_fwd(const void* qkv, void* o, float* lse, int B, int S, int nh, int nkv, float scale,
                            cudaStream_t s, const int* doc_start, int window) {
  if (S % 128 != 0) throw std::runtime_error("attn_fwd: sequence length must be a multiple of 128");
  if (nh < 1 || nkv < 1 || nh % nkv != 0) throw std::runtime_error("attn_fwd: nh must be a positive multiple of nkv");
  const CUtensorMap tm = make_tmap_heads(qkv, B, S, nh + 2 * nkv, 128, D);
  constexpr int smem = fwd::Layout<P_REGS, D>::SMEM_BYTES;
  static bool attr = false;
  if (!attr) {
    DTG_CUDA_CHECK(cudaFuncSetAttribute(attn_fwd_kernel<P_REGS, DOC, WIN, D>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        smem));
    attr = true;
  }
  const int num_m = S / 128;
  attn_fwd_kernel<P_REGS, DOC, WIN, D><<<dim3(B * nh, num_m, 1), fwd::THREADS, smem, s>>>(
      tm, (__nv_bfloat16*)o, lse, S, nh, nkv, scale * 1.4426950408889634f, num_m, doc_start, window);
  note_launch();
  DTG_LAUNCH_CHECK();
}

template <bool P_REGS, int D>
static void dispatch_attn_fwd(const void* qkv, void* o, float* lse, int B, int S, int nh, int nkv, float scale,
                              cudaStream_t s, const int* doc_start, int window) {
  if (window < 0) throw std::runtime_error("attn_fwd: window must be >= 1 (0 = no window)");
  // a window that covers the whole sequence masks nothing: run the kernel without it
  if (window > 0 && window < S) {
    if (doc_start) launch_attn_fwd<P_REGS, true, true, D>(qkv, o, lse, B, S, nh, nkv, scale, s, doc_start, window);
    else launch_attn_fwd<P_REGS, false, true, D>(qkv, o, lse, B, S, nh, nkv, scale, s, nullptr, window);
  } else {
    if (doc_start) launch_attn_fwd<P_REGS, true, false, D>(qkv, o, lse, B, S, nh, nkv, scale, s, doc_start, 0);
    else launch_attn_fwd<P_REGS, false, false, D>(qkv, o, lse, B, S, nh, nkv, scale, s, nullptr, 0);
  }
}

template <bool P_REGS>
static void dispatch_attn_fwd_d(const void* qkv, void* o, float* lse, int B, int S, int nh, int nkv, float scale,
                                cudaStream_t s, const int* doc_start, int window, int head_dim) {
  if (head_dim == 128) dispatch_attn_fwd<P_REGS, 128>(qkv, o, lse, B, S, nh, nkv, scale, s, doc_start, window);
  else if (head_dim == 64) dispatch_attn_fwd<P_REGS, 64>(qkv, o, lse, B, S, nh, nkv, scale, s, doc_start, window);
  else throw std::runtime_error("attn_fwd: head_dim must be 64 or 128");
}

// version 1: P through shared memory
void attn_fwd(const void* qkv, void* o, float* lse, int B, int S, int nh, int nkv, float scale, cudaStream_t s,
              const int* doc_start, int window, int head_dim) {
  dispatch_attn_fwd_d<false>(qkv, o, lse, B, S, nh, nkv, scale, s, doc_start, window, head_dim);
}
// version 2: P stays in registers (RS-form PV MMA)
void attn_fwd2(const void* qkv, void* o, float* lse, int B, int S, int nh, int nkv, float scale, cudaStream_t s,
               const int* doc_start, int window, int head_dim) {
  dispatch_attn_fwd_d<true>(qkv, o, lse, B, S, nh, nkv, scale, s, doc_start, window, head_dim);
}

}  // namespace dtg
