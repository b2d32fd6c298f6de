// bf16 GEMM on the Hopper tensor cores (wgmma, fp32 accumulators in registers, operands staged by
// TMA into 128B-swizzled shared memory), persistent and warp-specialised, 384 threads:
//
//   warpgroup 0   warp 0  TMA producer     (one elected lane)   smem ring: full/empty mbarriers
//   warpgroups 1-2        consumers        64 rows of the 128 x 256 tile each: wgmma m64n256k16 from shared
//                                          memory, then registers -> bf16 -> shared -> TMA store (optionally
//                                          C += ..., with C TMA-loaded into the same staging area)
//
// CG = 2 runs a cluster of two CTAs on a 256-row tile: each CTA stages its own 128 rows of A and loads half of
// the 256-row B tile, multicast into both CTAs, so every B byte leaves L2 once per pair.
//
// One kernel serves the three training GEMMs by operand majorness (all tensors row-major):
//   fwd   Y[T,N]  = X[T,K]  . W[N,K]^T    A K-major,  B K-major
//   dgrad dX[T,K] = dY[T,N] . W[N,K]      A K-major,  B MN-major
//   wgrad dW[N,K] = dY[T,N]^T . X[T,K]    A MN-major, B MN-major   (accumulate into the flat grad)
// This replaces the cuBLAS calls behind every nn.Linear of the reference (SURVEY.md K1) and its
// mainloop is what the fused all-gather->GEMM / GEMM->reduce-scatter kernels in fused_tp.cu reuse.
#include <cuda.h>
#include <cudaTypedefs.h>

#include <cstdlib>
#include <mutex>
#include <unordered_map>

#include "api.h"
#include "common.cuh"
#include "gemm_common.cuh"
#include "ptx.cuh"

namespace dtg {

using namespace ptx;

// Distributed operand modes (tensor parallelism, fused_tp.cu):
//   A_MODE / B_MODE  0 = one tensor map;  1 = rows (M) of A gathered from the ranks' symmetric buffers
//                    (all-gather -> GEMM);  2 = the reduction dimension K gathered from the ranks (wgrad
//                    over a sequence-sharded activation).  Tiles are fetched from the owning peer by TMA
//                    over NVLink, so the transfer streams under the MMA pipeline.
//   A_MODE           3 = all-gather by COMMUNICATION CTAs of this same kernel: the first `n_comm` CTA pairs
//                    bulk-copy (cp.async.bulk, NVLink -> smem -> local HBM) the peers' row tiles into the
//                    local [M, K] buffer and publish a per-tile flag; the GEMM CTAs start on the local rows and
//                    acquire the flag before their TMA touches a fetched tile.  Each remote byte crosses NVLink
//                    exactly once (peer memory bypasses the local L2, so mode 1 re-fetches it per N tile).
//   C_MODE           0 = local C;  1 = each `rows_per_peer` row chunk of C is stored into its owner's
//                    staging buffer (GEMM -> reduce-scatter push);  2 and 3 = the grouped GEMM (GRP 1 and 2 below).
//
// Epilogue.  A local C (C_MODE 0) leaves through shared memory: each consumer warpgroup converts half of its 64 x 256
// accumulator block at a time into a 32 KB staging area and one thread stores it with two TMA boxes, which clip at M
// and N, so no element needs a bounds test and the writes are whole 128-byte lines.  Accumulate mode TMA-loads the C
// boxes into the same staging area first and adds them there.  C_MODE 1 keeps the register epilogue: its rows go to
// the peers' staging buffers, one base pointer per owner, which one tensor map cannot describe.
template <int C_MODE>
constexpr bool kTmaEpilogue = (C_MODE != 1);

// ET selects the operand element type: 0 = bf16 (every mode above); 1 = fp8, A e4m3 and B e4m3; 2 = fp8, A e5m2 and B
// e4m3.  The fp8 forms take both operands K-major and plain (mode 0): the fp8 wgmma has no transposed operands, so
// the caller passes transposed copies.  A stage then holds a K block of 128 fp8 elements, which is the same 128-byte
// swizzle span, stage size and descriptor stepping as 64 bf16 elements, and the epilogue multiplies the fp32
// accumulators by the two per-tensor dequantisation scales `scale_a[0] * scale_b[0]`, read from device memory.
//
// BIAS adds a bf16 bias [N] to every row of the forward product before the one rounding to bf16: bf16(acc + b), fp8
// bf16(acc * deq + b), with the operation order of the C += path (so the result is bit-identical to accumulating
// over a C prefilled with the broadcast bias).  Every thread holds columns 8j + 2 (lane % 4) + {0, 1} of its
// accumulator fragment, so it reads one bf16 pair per block j of 8 columns, straight from global memory (L1 / L2
// serve the 2 N bytes to all CTAs); N is a multiple of 8, so a block is wholly inside or outside [0, N).  Forward
// layout only (A and B K-major), never together with accumulate.
//
// C_MODE 2 / 3 (GRP 1 / 2) is the grouped GEMM of the mixture-of-experts layers: one launch multiplies every
// expert's rows by that expert's slab of the weights, reading the routing tables (dist.grp_*) from device memory, so
// nothing waits on the host.  Single CTAs only (CG 1): a 128-row tile never straddles two experts, whose segments
// start at multiples of 128.  The C tile leaves through the TMA epilogue of C_MODE 0.
//   GRP 1  fwd / dgrad  C[rows, N] = A[rows, K] . B_e   A K-major; B_e is rows [e * grp_b_rows, (e + 1) * grp_b_rows)
//                       of B as stored, e the expert of the row tile; tiles of no expert (past the last segment) are
//                       skipped.
//   GRP 2  wgrad        C_e[M, N] = A[seg_e, M]^T . B[seg_e, N]   A and B MN-major; the reduction runs over expert
//                       e's rows only, and C_e is rows [e * M, (e + 1) * M) of C.  Tiles run over (expert, m, n).  An
//                       expert without rows writes zeros in overwrite mode and leaves C_e untouched in accumulate mode.
template <bool A_K, bool B_K, int CG, int A_MODE = 0, int B_MODE = 0, int C_MODE = 0, int ET = 0, bool BIAS = false>
__global__ void __launch_bounds__(GemmCfg<CG>::THREADS, 1)
gemm_bf16_kernel(const __grid_constant__ TmapSet<(A_MODE ? kMaxRanks : 1)> tmAs,
                 const __grid_constant__ TmapSet<(B_MODE ? kMaxRanks : 1)> tmBs, const __grid_constant__ GemmDist dist,
                 const __grid_constant__ CUtensorMap tmC, __nv_bfloat16* __restrict__ C, int M, int N, int K,
                 long long ldc, int accumulate, int num_m_tiles, int num_tiles, const float* __restrict__ scale_a,
                 const float* __restrict__ scale_b, const __nv_bfloat16* __restrict__ bias) {
  static_assert(ET == 0 || (A_K && B_K && A_MODE == 0 && B_MODE == 0 && C_MODE == 0),
                "the fp8 GEMM takes K-major operands from one tensor map each");
  static_assert(!BIAS || (A_K && B_K && C_MODE == 0), "the bias epilogue serves the forward layout with a local C");
  constexpr int GRP = C_MODE == 2 ? 1 : (C_MODE == 3 ? 2 : 0);
  static_assert(GRP == 0 || (CG == 1 && A_MODE == 0 && B_MODE == 0 && ET == 0 && !BIAS &&
                             (GRP == 1 ? A_K : (!A_K && !B_K))),
                "the grouped GEMM is a plain bf16 single-CTA GEMM: GRP 1 with A K-major, GRP 2 with both MN-major");
  using Cfg = GemmCfg<CG>;
  constexpr bool TMA_EPI = kTmaEpilogue<C_MODE>;
  constexpr int BK = ET ? 2 * Cfg::BK : Cfg::BK;   // elements of K per stage: one 128-byte span either way
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + Cfg::STAGES * Cfg::STAGE_BYTES);
  uint64_t* full = bars;
  uint64_t* empty = bars + Cfg::STAGES;
  uint64_t* comm_bar = bars + 2 * Cfg::STAGES;  // [COMM_SLOTS] (A_MODE 3)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const uint32_t cta_rank = (CG == 2) ? cluster_ctarank() : 0u;
  const int n_comm = (A_MODE == 3) ? dist.n_comm : 0;
  const bool is_comm = (A_MODE == 3) && (int)(blockIdx.x / CG) < n_comm;
  const int cluster_id = (int)(blockIdx.x / CG) - n_comm;       // index among the GEMM clusters
  const int num_clusters = (int)(gridDim.x / CG) - n_comm;
  const int num_kb = (K + BK - 1) / BK;
  const int local_m_tiles = (A_MODE == 3) ? dist.rows_per_peer / (Cfg::BM * CG) : 0;
  // GRP: tile t -> (m tile, n tile), its expert, the first reduction row (GRP 2) and its K blocks; false: no work
  [[maybe_unused]] auto grp_tile = [&](int t, int& tm, int& tn, int& e, int& k_row0, int& kbs) -> bool {
    if constexpr (GRP == 1) {
      tile_mn(t, num_m_tiles, dist, 0, tm, tn);
      e = dist.grp_tile_expert[tm];
      k_row0 = 0;
      kbs = num_kb;
      return e >= 0;
    } else {
      const int per = num_m_tiles * dist.num_n_tiles;
      e = t / per;
      tile_mn(t - e * per, num_m_tiles, dist, 0, tm, tn);
      k_row0 = dist.grp_seg[e];
      kbs = (dist.grp_seg[e + 1] - k_row0) / BK;
      return kbs > 0 || !accumulate;
    }
  };

  if (threadIdx.x == 0) {
    prefetch_tensormap(&tmAs.m[0]);
    prefetch_tensormap(&tmBs.m[0]);
    if constexpr (TMA_EPI) {
      prefetch_tensormap(&tmC);
      for (int i = 0; i < 2; ++i) mbar_init(&bars[Cfg::EPI_BAR + i], 1);
    }
    for (int i = 0; i < Cfg::STAGES; ++i) {
      mbar_init(&full[i], 1);
      mbar_init(&empty[i], 2 * CG);  // both consumer warpgroups of every CTA that reads the stage's B
    }
    if constexpr (A_MODE == 3)
      for (int i = 0; i < Cfg::COMM_SLOTS; ++i) mbar_init(&comm_bar[i], 1);
    fence_barrier_init();
  }
  if (CG == 2) cluster_sync(); else __syncthreads();

  if (is_comm) {
    // ===================== communication CTA: all-gather the peers' row tiles =====================
    if (warp == 0 && elect_one()) {
      const int cidx = (int)blockIdx.x;  // 0 .. n_comm*CG-1 : also my signal-pad channel
      const int ncta = n_comm * CG;
      const int t_ = dist.nranks, rk = dist.rank;
      // every rank's activation shard is written once its kernel has started (stream order)
      for (int p = 0; p < t_; ++p) st_release_sys(dist.pads[p] + cidx * kMaxRanks + rk, dist.bar_epoch);
      for (int p = 0; p < t_; ++p) {
        const uint32_t* mine = dist.pads[rk] + cidx * kMaxRanks + p;
        const unsigned long long t0 = global_timer_ns();
        while ((int32_t)(ld_acquire_sys(mine) - dist.bar_epoch) < 0)
          if (global_timer_ns() - t0 > kWaitTimeoutNs)  // a peer never launched the matching GEMM: fail loudly
            __trap();  // all-gather GEMM: peer did not arrive at the entry barrier
      }
      constexpr uint32_t PIECE = Cfg::COMM_PIECE;   // ring slots carved out of the (unused) pipeline smem
      constexpr int NB = Cfg::COMM_SLOTS, AHEAD = NB - 2;
      const int lmt = local_m_tiles > 0 ? local_m_tiles : 1;
      const int remote_tiles = (t_ - 1) * lmt;
      const uint32_t pieces_per_tile = (uint32_t)(dist.tile_bytes / PIECE);
      uint32_t issued = 0, stored = 0;  // global piece counters (ring position / barrier parity)
      for (int r = cidx; r < remote_tiles; r += ncta) {
        const int k = 1 + r / lmt, within = r % lmt;
        const int owner = (rk + k) % t_;
        const int m_tile = owner * lmt + within;
        const char* src = dist.ag_src[k] + (long long)m_tile * dist.tile_bytes;
        char* dst = const_cast<char*>(dist.ag_src[0]) + (long long)m_tile * dist.tile_bytes;
        uint32_t li = 0;  // pieces of this tile whose load has been issued
        for (uint32_t si = 0; si < pieces_per_tile; ++si) {
          while (li < pieces_per_tile && li < si + AHEAD) {
            const uint32_t slot = issued % NB;
            // the bulk store that last read this slot was committed >= 2 stores ago
            bulk_wait_group_read<1>();
            mbar_arrive_expect_tx(&comm_bar[slot], PIECE);
            bulk_load_g2s(smem + slot * PIECE, src + (long long)li * PIECE, PIECE, &comm_bar[slot]);
            ++issued;
            ++li;
          }
          const uint32_t slot = stored % NB;
          mbar_wait_mma(&comm_bar[slot], (stored / NB) & 1);
          bulk_store_s2g(dst + (long long)si * PIECE, smem + slot * PIECE, PIECE);
          bulk_commit_group();
          ++stored;
        }
        bulk_wait_group<0>();       // the whole tile is in local memory
        fence_proxy_async_all();
        st_release_gpu(dist.ag_flags + m_tile, dist.ag_epoch);
      }
    }
  } else if (warp == 0) {
    // ===================== TMA producer =====================
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = cluster_id; t < num_tiles; t += num_clusters) {
        int tm_, tn_;
        [[maybe_unused]] int g_e = 0, g_k0 = 0;
        int tile_kb = num_kb;
        if constexpr (GRP != 0) {
          if (!grp_tile(t, tm_, tn_, g_e, g_k0, tile_kb)) continue;
        } else {
          tile_mn(t, num_m_tiles, dist, local_m_tiles, tm_, tn_);
        }
        const int m0 = tm_ * (Cfg::BM * CG) + (int)cta_rank * Cfg::BM;
        // the B rows this CTA loads (for the pair); GRP 1 forward: inside the expert's slab
        const int nb = tn_ * Cfg::BN + (int)cta_rank * Cfg::B_ROWS + ((GRP == 1 && B_K) ? g_e * dist.grp_b_rows : 0);
        const CUtensorMap* tmA_p = &tmAs.m[0];
        int a_m0 = m0;
        if constexpr (A_MODE == 3) {  // fetched tile: wait until the communication CTAs published it
          if (tm_ / (local_m_tiles > 0 ? local_m_tiles : 1) != dist.rank) {
            const unsigned long long t0 = global_timer_ns();
            while ((int32_t)(ld_acquire_gpu(dist.ag_flags + tm_) - dist.ag_epoch) < 0)
              if (global_timer_ns() - t0 > kWaitTimeoutNs)  // never read an unfetched tile
                __trap();  // all-gather GEMM: row tile was never published by the communication CTAs
            fence_proxy_async_all();
          }
        }
        if constexpr (A_MODE == 1) {  // this row block lives on rank m0 / rows_per_peer
          const int peer = m0 / dist.rows_per_peer;
          tmA_p = &tmAs.m[peer];
          a_m0 = m0 - peer * dist.rows_per_peer;
        }
        for (int kbi = 0; kbi < tile_kb; ++kbi) {
          // K-gathered operands start with the local rank's slice of K
          const int kb = (A_MODE == 2 || B_MODE == 2) ? (kbi + dist.k_shift) % num_kb : kbi;
          const int k0 = kb * BK;
          int a_k0 = k0, b_k0 = k0;
          if constexpr (GRP == 2) {   // the expert's rows of both operands
            a_k0 += g_k0;
            b_k0 += g_k0;
          }
          if constexpr (GRP == 1 && !B_K) b_k0 += g_e * dist.grp_b_rows;   // dgrad: the expert's slab of B
          const CUtensorMap* tmB_p = &tmBs.m[0];
          if constexpr (A_MODE == 2) {
            const int peer = k0 / dist.rows_per_peer;
            tmA_p = &tmAs.m[peer];
            a_k0 = k0 - peer * dist.rows_per_peer;
          }
          if constexpr (B_MODE == 2) {
            const int peer = k0 / dist.rows_per_peer;
            tmB_p = &tmBs.m[peer];
            b_k0 = k0 - peer * dist.rows_per_peer;
          }
          const CUtensorMap& tmA = *tmA_p;
          const CUtensorMap& tmB = *tmB_p;
          mbar_wait_mma(&empty[stage], phase ^ 1);   // (CG 2: the peer's consumers released it too)
          uint8_t* sa = smem + stage * Cfg::STAGE_BYTES;
          uint8_t* sb = sa + Cfg::A_BYTES;
          mbar_arrive_expect_tx(&full[stage], Cfg::STAGE_BYTES);
          if constexpr (A_K) {
            tma_load_2d(&tmA, &full[stage], sa, a_k0, a_m0);
          } else {
#pragma unroll
            for (int j = 0; j < Cfg::BM / 64; ++j) tma_load_2d(&tmA, &full[stage], sa + j * 8192, a_m0 + 64 * j, a_k0);
          }
          if constexpr (CG == 1) {
            if constexpr (B_K) {
              tma_load_2d(&tmB, &full[stage], sb, b_k0, nb);
            } else {
#pragma unroll
              for (int j = 0; j < Cfg::B_ROWS / 64; ++j) tma_load_2d(&tmB, &full[stage], sb + j * 8192, nb + 64 * j, b_k0);
            }
          } else {
            // my half of B, into the same offsets of both CTAs of the pair
            if constexpr (B_K) {
              tma_load_2d_mc(&tmB, &full[stage], sb + cta_rank * (Cfg::B_ROWS * 128), b_k0, nb, 0b11);
            } else {
#pragma unroll
              for (int j = 0; j < Cfg::B_ROWS / 64; ++j)
                tma_load_2d_mc(&tmB, &full[stage], sb + (cta_rank * (Cfg::B_ROWS / 64) + j) * 8192, nb + 64 * j, b_k0,
                               0b11);
            }
          }
          if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else if (warp >= 4 && !is_comm) {
    // ===================== consumers: wgmma mainloop + epilogue =====================
    const int half = (warp >> 2) - 1;  // rows [64*half, 64*half + 64) of this CTA's 128
    const int wq = warp & 3;
    const bool signal = (threadIdx.x & 127) == 0;
    const uint32_t peer_empty = (CG == 2) ? mapa(smem_u32(&empty[0]), cta_rank ^ 1u) : 0u;
    auto release = [&](int s) {       // this warpgroup is done reading stage s (here and, CG 2, in the peer)
      if (signal) {
        mbar_arrive(&empty[s]);
        if constexpr (CG == 2) mbar_arrive_cluster(peer_empty + (uint32_t)(s * 8));
      }
    };
    int stage = 0;
    uint32_t phase = 0;
    // TMA epilogue: this warpgroup's staging area (two 64 x 64 boxes), its C-load barrier, and this thread's 4-byte
    // slot for accumulator pair (h = 0, chunk 0) of a box: row 16*wq + lane/4, byte 4*(lane%4) of a 16-byte chunk.
    // 128B swizzle puts chunk c of row r at chunk c ^ (r % 8), and r % 8 = lane / 4 for every row this thread holds.
    [[maybe_unused]] uint8_t* const stg = smem + Cfg::EPI_OFFSET + half * Cfg::EPI_WG_BYTES;
    [[maybe_unused]] uint64_t* const c_bar = bars + Cfg::EPI_BAR + half;
    [[maybe_unused]] uint32_t c_phase = 0;
    [[maybe_unused]] const uint32_t stg_s = smem_u32(stg) + (uint32_t)((wq * 16 + (lane >> 2)) * 128 + 4 * (lane & 3));
    [[maybe_unused]] const int bar_id = 1 + half;   // named barrier of this warpgroup (0 is __syncthreads)
    for (int t = cluster_id; t < num_tiles; t += num_clusters) {
      int tm_, tn_;
      [[maybe_unused]] int g_e = 0, g_k0 = 0;
      int tile_kb = num_kb;
      if constexpr (GRP != 0) {
        if (!grp_tile(t, tm_, tn_, g_e, g_k0, tile_kb)) continue;
      } else {
        tile_mn(t, num_m_tiles, dist, local_m_tiles, tm_, tn_);
      }
      const int m0 = tm_ * (Cfg::BM * CG) + (int)cta_rank * Cfg::BM + half * 64;
      const int n0 = tn_ * Cfg::BN;
      const int cm0 = m0 + (GRP == 2 ? g_e * M : 0);   // row of C (GRP 2: inside the expert's block)
      // accumulate mode: fetch the first 128 columns of C under the mainloop.  The stores of the previous tile must
      // have read the staging area; every thread finished writing it before they were issued.
      // Boxes entirely outside C (rows >= M, columns >= N) are never loaded or stored.
      if constexpr (TMA_EPI) {
        if (accumulate && signal && m0 < M) {
          const int nbox = n0 + 64 < N ? 2 : 1;
          tma_store_wait_read<0>();
          mbar_arrive_expect_tx(c_bar, nbox * Cfg::EPI_BOX_BYTES);
          for (int b = 0; b < nbox; ++b) tma_load_2d(&tmC, c_bar, stg + b * Cfg::EPI_BOX_BYTES, n0 + 64 * b, cm0);
        }
      }
      float acc[128];
#pragma unroll
      for (int i = 0; i < 128; ++i) acc[i] = 0.f;
      int prev = -1;
      for (int kb = 0; kb < tile_kb; ++kb) {
        mbar_wait_mma(&full[stage], phase);
        const uint32_t a_base = smem_u32(smem + stage * Cfg::STAGE_BYTES) + (uint32_t)(half * 8192);
        const uint32_t b_base = smem_u32(smem + stage * Cfg::STAGE_BYTES + Cfg::A_BYTES);
        wgmma_fence();
        fence_regs(acc);
        if constexpr (ET == 0) {
#pragma unroll
          for (int k = 0; k < Cfg::BK / 16; ++k) {
            const uint64_t da = A_K ? desc_kmajor_sw128(a_base + k * 32) : desc_mnmajor_sw128(a_base + k * 2048, 8192);
            const uint64_t db = B_K ? desc_kmajor_sw128(b_base + k * 32) : desc_mnmajor_sw128(b_base + k * 2048, 8192);
            wgmma_m64n256k16_ss<A_K ? 0 : 1, B_K ? 0 : 1>(acc, da, db, 1u);
          }
        } else {
#pragma unroll
          for (int k = 0; k < BK / 32; ++k)
            wgmma_m64n256k32_fp8_ss<ET>(acc, desc_kmajor_sw128(a_base + k * 32), desc_kmajor_sw128(b_base + k * 32), 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();              // the previous stage's MMAs have retired: hand its buffers back
        fence_regs(acc);
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == Cfg::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      fence_regs(acc);
      if (prev >= 0) release(prev);
      // epilogue: accumulator fragment (x dequantisation scale, fp8) -> bf16 pairs -> staging area -> TMA store
      // (C_MODE 1: -> global from registers)
      [[maybe_unused]] float deq = 1.f;
      if constexpr (ET != 0) deq = scale_a[0] * scale_b[0];
      if constexpr (TMA_EPI) {
        if (m0 >= M) continue;
#pragma unroll
        for (int p = 0; p < 2; ++p) {   // columns [n0 + 128p, n0 + 128p + 128): accumulator blocks j = 16p .. 16p+15
          const int c0 = n0 + 128 * p;
          if (c0 >= N) break;
          const int nbox = c0 + 64 < N ? 2 : 1;
          if (accumulate) {
            if (p == 1 && signal) {
              tma_store_wait_read<0>();   // the first half's stores have read the staging area
              mbar_arrive_expect_tx(c_bar, nbox * Cfg::EPI_BOX_BYTES);
              for (int b = 0; b < nbox; ++b) tma_load_2d(&tmC, c_bar, stg + b * Cfg::EPI_BOX_BYTES, c0 + 64 * b, cm0);
            }
            mbar_wait_mma(c_bar, c_phase);
            c_phase ^= 1;
          } else {
            if (signal) tma_store_wait_read<0>();
            named_bar_sync(bar_id, 128);
          }
#pragma unroll
          for (int b = 0; b < 2; ++b) {
#pragma unroll
            for (int jj = 0; jj < 8; ++jj) {
              const int j = 16 * p + 8 * b + jj;
              [[maybe_unused]] float2 bj;
              if constexpr (BIAS) {
                const int col = n0 + 8 * j + 2 * (lane & 3);
                bj = col < N ? __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(bias + col))
                             : make_float2(0.f, 0.f);
              }
#pragma unroll
              for (int h = 0; h < 2; ++h) {   // rows +8h: 8 rows of 128 B further, same swizzle phase
                float x = acc[4 * j + 2 * h], y = acc[4 * j + 2 * h + 1];
                const uint32_t q = stg_s + (uint32_t)(b * Cfg::EPI_BOX_BYTES + h * 1024 + ((jj ^ (lane >> 2)) << 4));
                if constexpr (BIAS) {     // as the C += path below, with the bias in place of C
                  if constexpr (ET != 0) {
                    x = __fmaf_rn(x, deq, bj.x);
                    y = __fmaf_rn(y, deq, bj.y);
                  } else {
                    x += bj.x;
                    y += bj.y;
                  }
                } else if (accumulate) {
                  const uint32_t old = ld_shared_u32(q);
                  const float2 g = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&old));
                  if constexpr (ET != 0) {   // one rounding for the scale and the add: acc * deq + C
                    x = __fmaf_rn(x, deq, g.x);
                    y = __fmaf_rn(y, deq, g.y);
                  } else {
                    x += g.x;
                    y += g.y;
                  }
                } else if constexpr (ET != 0) {
                  x = __fmul_rn(x, deq);
                  y = __fmul_rn(y, deq);
                }
                st_shared_u32(q, pack_bf16x2(x, y));
              }
            }
          }
          fence_proxy_async();            // the generic-proxy writes are visible to the TMA store
          named_bar_sync(bar_id, 128);
          if (signal) {
            for (int b = 0; b < nbox; ++b) tma_store_2d(&tmC, stg + b * Cfg::EPI_BOX_BYTES, c0 + 64 * b, cm0);
            tma_store_commit();
          }
        }
        continue;
      }
      const int r0 = m0 + wq * 16 + (lane >> 2);
      const int c0 = n0 + 2 * (lane & 3);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int row = r0 + 8 * h;
        if (row >= M) continue;
        __nv_bfloat16* crow = C + (size_t)row * ldc;
        if constexpr (C_MODE == 1) {  // push this row into the staging buffer of the rank that owns it
          const int owner = row / dist.rows_per_peer;
          crow = dist.c_ptr[owner < kMaxRanks ? owner : 0] + (size_t)(row - owner * dist.rows_per_peer) * ldc;
        }
#pragma unroll
        for (int j = 0; j < 32; ++j) {
          const int col = c0 + 8 * j;
          if (col < N) {
            float x = acc[4 * j + 2 * h], y = acc[4 * j + 2 * h + 1];
            if constexpr (ET != 0) {
              x *= deq;
              y *= deq;
            }
            __nv_bfloat162* p = reinterpret_cast<__nv_bfloat162*>(crow + col);
            if (accumulate) {
              const float2 g = __bfloat1622float2(*p);
              x += g.x;
              y += g.y;
            }
            *p = __floats2bfloat162_rn(x, y);
          }
        }
      }
    }
    if constexpr (TMA_EPI)
      if (signal) tma_store_wait<0>();   // the staging area must outlive the last stores' reads and writes
  }

  if (CG == 2) cluster_sync();  // no CTA may exit while its peer can still multicast into it or arrive on it
}


// ---------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------
static PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    DTG_CUDA_CHECK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres));
    if (qres != cudaDriverEntryPointSuccess || !p) throw std::runtime_error("cuTensorMapEncodeTiled unavailable");
    fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(p);
  }
  return fn;
}

static CUtensorMap make_tmap_typed(CUtensorMapDataType dtype, const void* base, int rank, const uint64_t* dims,
                                   const uint64_t* strides_bytes, const uint32_t* box, bool swizzle128) {
  // The driver entry point needs a current context; autograd worker threads may reach this before
  // any runtime call has bound the primary context to them.
  static thread_local bool ctx_bound = false;
  if (!ctx_bound) {
    int dev = 0;
    DTG_CUDA_CHECK(cudaGetDevice(&dev));
    DTG_CUDA_CHECK(cudaSetDevice(dev));
    DTG_CUDA_CHECK(cudaFree(nullptr));
    ctx_bound = true;
  }
  CUtensorMap m;
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bdim[i] = box[i];
    estr[i] = 1;
    if (i > 0) gstr[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = get_encode_fn()(&m, dtype, (cuuint32_t)rank, const_cast<void*>(base), gdim,
                               gstr, bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                               swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    throw std::runtime_error("cuTensorMapEncodeTiled failed with code " + std::to_string((int)r) +
                             " (base must be 16B aligned, strides multiples of 16B)");
  }
  return m;
}

CUtensorMap make_tmap_bf16(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                           const uint32_t* box, bool swizzle128) {
  return make_tmap_typed(CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, base, rank, dims, strides_bytes, box, swizzle128);
}

CUtensorMap make_tmap_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes, uint32_t box_inner,
                         uint32_t box_outer) {
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {row_stride_bytes};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap_bf16(base, 2, dims, strides, box, true);
}

// 2-D map of 1-byte elements (fp8 operands), 128B swizzle
static CUtensorMap make_tmap_2d_u8(const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                                   uint32_t box_inner, uint32_t box_outer) {
  uint64_t dims[2] = {inner, outer};
  uint64_t strides[1] = {row_stride_bytes};
  uint32_t box[2] = {box_inner, box_outer};
  return make_tmap_typed(CU_TENSOR_MAP_DATA_TYPE_UINT8, base, 2, dims, strides, box, true);
}

static int g_gemm_variant = 0;  // 0 = env/default
void set_gemm_variant(int v) { g_gemm_variant = v; }
int default_gemm_variant() {
  if (g_gemm_variant) return g_gemm_variant;
  static int env = -1;
  if (env < 0) {
    const char* e = getenv("DTG_GEMM_VARIANT");
    env = e ? atoi(e) : DTG_DEFAULT_GEMM_VARIANT;
  }
  return env;
}

// One launcher for the plain and the tensor-parallel GEMMs.  `a_srcs` / `b_srcs`: base pointer of the
// operand on every rank (only [0] is used in mode 0); `dist.c_ptr` set by the caller for C_MODE 1.
// C_MODE 2 and 3 (grouped): `groups` slabs of B (C_MODE 2) or blocks of C (C_MODE 3) follow one another in memory.
template <bool A_K, bool B_K, int CG, int A_MODE, int B_MODE, int C_MODE, int ET = 0, bool BIAS = false>
static void launch_gemm(const void* const* a_srcs, const void* const* b_srcs, void* C, int M, int N, int K,
                        long long lda, long long ldb, long long ldc, bool accumulate, GemmDist dist, int nranks,
                        cudaStream_t s, const float* scale_a = nullptr, const float* scale_b = nullptr,
                        const void* bias = nullptr, int groups = 1) {
  using Cfg = GemmCfg<CG>;
  constexpr int ESIZE = ET ? 1 : 2;   // bytes per operand element
  constexpr int GRP = C_MODE == 2 ? 1 : (C_MODE == 3 ? 2 : 0);
  TmapSet<(A_MODE ? kMaxRanks : 1)> tmA;
  TmapSet<(B_MODE ? kMaxRanks : 1)> tmB;
  const int rpp = dist.rows_per_peer;
  for (int p = 0; p < ((A_MODE == 1 || A_MODE == 2) ? nranks : 1); ++p) {
    const int rows = (A_MODE == 1) ? rpp : M;   // M extent of this source (mode 3: the local gathered buffer)
    const int ks = (A_MODE == 2) ? rpp : K;     // K extent of this source
    if constexpr (ET != 0) tmA.m[p] = make_tmap_2d_u8(a_srcs[p], ks, rows, lda, 128, Cfg::BM);
    else tmA.m[p] = A_K ? make_tmap_2d(a_srcs[p], ks, rows, lda * 2, 64, Cfg::BM) : make_tmap_2d(a_srcs[p], rows, ks, lda * 2, 64, 64);
  }
  for (int p = 0; p < ((B_MODE == 1 || B_MODE == 2) ? nranks : 1); ++p) {
    const int ks = (B_MODE == 2) ? rpp : K;
    if constexpr (ET != 0) tmB.m[p] = make_tmap_2d_u8(b_srcs[p], ks, N, ldb, 128, Cfg::B_ROWS);
    else if constexpr (GRP == 1)   // every expert's slab: the one stacked extent
      tmB.m[p] = B_K ? make_tmap_2d(b_srcs[p], ks, (uint64_t)N * groups, ldb * 2, 64, Cfg::B_ROWS)
                     : make_tmap_2d(b_srcs[p], N, (uint64_t)ks * groups, ldb * 2, 64, 64);
    else tmB.m[p] = B_K ? make_tmap_2d(b_srcs[p], ks, N, ldb * 2, 64, Cfg::B_ROWS) : make_tmap_2d(b_srcs[p], N, ks, ldb * 2, 64, 64);
  }
  for (int p = ((A_MODE == 1 || A_MODE == 2) ? nranks : 1); p < (A_MODE ? kMaxRanks : 1); ++p) tmA.m[p] = tmA.m[0];
  for (int p = ((B_MODE == 1 || B_MODE == 2) ? nranks : 1); p < (B_MODE ? kMaxRanks : 1); ++p) tmB.m[p] = tmB.m[0];
  const int num_m_tiles = (M + Cfg::BM * CG - 1) / (Cfg::BM * CG);
  const int num_n_tiles = (N + Cfg::BN - 1) / Cfg::BN;
  const int num_tiles = num_m_tiles * num_n_tiles * (GRP == 2 ? groups : 1);
  // C in 64 x 64 boxes (the staging layout of the epilogue); the other modes store from registers
  CUtensorMap tmC{};
  if constexpr (kTmaEpilogue<C_MODE>)
    tmC = make_tmap_2d(C, N, (uint64_t)M * (GRP == 2 ? groups : 1), ldc * 2, 64, 64);
  auto kern = gemm_bf16_kernel<A_K, B_K, CG, A_MODE, B_MODE, C_MODE, ET, BIAS>;
  constexpr int kSmem = kTmaEpilogue<C_MODE> ? Cfg::SMEM_BYTES_EPI : Cfg::SMEM_BYTES;
  static bool attr_set = false;
  if (!attr_set) {
    DTG_CUDA_CHECK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem));
    attr_set = true;
  }
  dist.num_n_tiles = num_n_tiles;
  if constexpr (A_MODE == 0 && B_MODE == 0 && C_MODE != 1) {
    // keep one group's panel of A (group_m x TM x K elements) within ~1/3 of the 50 MB L2; with very long K nothing
    // fits and a squarish block of 8 row tiles by (tiles in flight / 8) column tiles minimises the bytes each
    // wave touches
    static const long long budget = []() {
      const char* e = getenv("DTG_GEMM_L2_BUDGET_MB");
      return (long long)(e ? atoi(e) : 16) << 20;
    }();
    const long long panel = (long long)Cfg::BM * CG * K * ESIZE;
    long long gm = budget / (panel > 0 ? panel : 1);
    if (gm < 8) gm = 8;
    dist.group_m = gm >= num_m_tiles ? 0 : (int)gm;
  }
  int clusters = sm_count() / CG;
  if constexpr (A_MODE == 3) {
    dist.k_shift = num_n_tiles;  // tile_mn() needs the N tile count in this mode
    int gemm_clusters = clusters - dist.n_comm;
    if (gemm_clusters > num_tiles) gemm_clusters = num_tiles;
    clusters = gemm_clusters + dist.n_comm;
  } else if (clusters > num_tiles) {
    clusters = num_tiles;
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(clusters * CG);
  cfg.blockDim = dim3(Cfg::THREADS);
  cfg.dynamicSmemBytes = kSmem;
  cfg.stream = s;
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeClusterDimension;
  attrs[0].val.clusterDim.x = CG;
  attrs[0].val.clusterDim.y = 1;
  attrs[0].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  DTG_CUDA_CHECK(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, dist, tmC, (__nv_bfloat16*)C, M, N, K, ldc,
                                    accumulate ? 1 : 0, num_m_tiles, num_tiles, scale_a, scale_b,
                                    (const __nv_bfloat16*)bias));
  note_launch();
}

// max co-resident clusters of the 2-CTA kernel (diagnostics)
int gemm_max_active_clusters(int cg) {
  cudaLaunchConfig_t cfg{};
  cfg.blockDim = dim3(GemmCfg<1>::THREADS);
  cudaLaunchAttribute attrs[1];
  attrs[0].id = cudaLaunchAttributeClusterDimension;
  attrs[0].val.clusterDim.x = cg;
  attrs[0].val.clusterDim.y = 1;
  attrs[0].val.clusterDim.z = 1;
  cfg.attrs = attrs;
  cfg.numAttrs = 1;
  int n = -1;
  if (cg == 2) {
    auto kern = gemm_bf16_kernel<true, true, 2, 0, 0, 0>;
    cfg.gridDim = dim3(sm_count());
    cfg.dynamicSmemBytes = GemmCfg<2>::SMEM_BYTES_EPI;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<2>::SMEM_BYTES_EPI);
    cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
  } else {
    auto kern = gemm_bf16_kernel<true, true, 1, 0, 0, 0>;
    cfg.gridDim = dim3(sm_count());
    cfg.dynamicSmemBytes = GemmCfg<1>::SMEM_BYTES_EPI;
    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, GemmCfg<1>::SMEM_BYTES_EPI);
    cudaOccupancyMaxActiveClusters(&n, kern, &cfg);
  }
  return n;
}

// TMA operands need 16-byte aligned bases (the tensor-map encoder refuses others); C is stored by TMA too, and with
// ldc % 8 == 0 every row of it starts on a 16-byte boundary as well.
static void check_gemm_bases(const char* who, const void* A, const void* B, const void* C) {
  const struct { const void* p; const char* name; } ops[3] = {{A, "A"}, {B, "B"}, {C, "C"}};
  for (const auto& o : ops)
    if (reinterpret_cast<uintptr_t>(o.p) % 16)
      throw std::runtime_error(std::string(who) + ": " + o.name + " must start at a 16-byte aligned address");
}

// K == 0: the product is zero, so overwrite mode writes zeros over the M x N view and accumulate mode leaves it as is
static void gemm_empty_k(void* C, int M, int N, long long ldc, bool accumulate, cudaStream_t s) {
  if (!accumulate)
    DTG_CUDA_CHECK(cudaMemset2DAsync(C, (size_t)ldc * 2, 0, (size_t)N * 2, (size_t)M, s));
}

// The bias epilogue's preconditions, checked before any launch: forward layout, overwrite mode, K >= 1 (with K = 0 the
// output would be the broadcast bias, which no kernel here writes), and a 16-byte aligned [N] vector.
static void check_bias(const char* who, const void* bias, bool a_kmajor, bool b_kmajor, bool accumulate, int K) {
  if (!bias) return;
  if (!a_kmajor || !b_kmajor)
    throw std::runtime_error(std::string(who) + ": a bias needs the forward layout (A [M,K] and B [N,K], K-major)");
  if (accumulate) throw std::runtime_error(std::string(who) + ": a bias cannot be combined with accumulate");
  if (K <= 0) throw std::runtime_error(std::string(who) + ": a bias needs K >= 1");
  if (reinterpret_cast<uintptr_t>(bias) % 16)
    throw std::runtime_error(std::string(who) + ": bias must start at a 16-byte aligned address");
}

void gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, long long lda, long long ldb, long long ldc,
               bool a_kmajor, bool b_kmajor, bool accumulate, int variant, cudaStream_t s, const void* bias) {
  if (M <= 0 || N <= 0) return;
  if ((N % 8) || (ldc % 8) || (lda % 8) || (ldb % 8))
    throw std::runtime_error("gemm_bf16: N and the leading dimensions must be multiples of 8 elements");
  check_gemm_bases("gemm_bf16", A, B, C);
  check_bias("gemm_bf16", bias, a_kmajor, b_kmajor, accumulate, K);
  if (K <= 0) return gemm_empty_k(C, M, N, ldc, accumulate, s);
  if (variant == 0) variant = default_gemm_variant();
  if (variant == 3) variant = (M > 128) ? 2 : 1;  // auto: the CTA-pair tile is 256 rows tall
  const int cg = (variant == 2) ? 2 : 1;
  const void* as[1] = {A};
  const void* bs[1] = {B};
  GemmDist dist{};
  if (bias) {
    if (cg == 2) launch_gemm<true, true, 2, 0, 0, 0, 0, true>(as, bs, C, M, N, K, lda, ldb, ldc, false, dist, 1, s,
                                                             nullptr, nullptr, bias);
    else launch_gemm<true, true, 1, 0, 0, 0, 0, true>(as, bs, C, M, N, K, lda, ldb, ldc, false, dist, 1, s, nullptr,
                                                      nullptr, bias);
    return;
  }
#define DTG_GEMM_CASE(AK, BK)                                                                                    \
  if (a_kmajor == AK && b_kmajor == BK) {                                                                        \
    if (cg == 2) launch_gemm<AK, BK, 2, 0, 0, 0>(as, bs, C, M, N, K, lda, ldb, ldc, accumulate, dist, 1, s);      \
    else launch_gemm<AK, BK, 1, 0, 0, 0>(as, bs, C, M, N, K, lda, ldb, ldc, accumulate, dist, 1, s);              \
    return;                                                                                                      \
  }
  DTG_GEMM_CASE(true, true)
  DTG_GEMM_CASE(true, false)
  DTG_GEMM_CASE(false, false)
  DTG_GEMM_CASE(false, true)
#undef DTG_GEMM_CASE
}

// C[M,N] (+)= scale_a[0] * scale_b[0] * A8[M,K] . B8[N,K]^T: per-tensor scaled fp8 operands, both stored row-major
// with K contiguous (lda / ldb in elements = bytes), fp32 accumulators, bf16 C with row stride ldc.  A is e4m3, or
// e5m2 when `a_e5m2` (an output gradient); B is e4m3.  The scales are device pointers, so nothing here waits on the
// kernels that computed them.
//
// With deq = fp32(scale_a[0] * scale_b[0]) and acc the accumulator of A8 . B8^T, every element is
//   overwrite   bf16(fp32(acc * deq))
//   accumulate  bf16(fp32(acc * deq + C_old))   one rounding (fmaf)
//   bias        bf16(fp32(acc * deq + bias))    one rounding (fmaf)
// acc is summed in ascending K, one k32 wgmma step at a time, and the fp8 wgmma does not accumulate in full fp32.
// Measured on an H100 over random data at the training shapes:
//   |C - exact| <= 2^-8 |exact| + 0.62 * 2^-13 * deq * sum_t (|S_(t-1)| + sum_(k in t) |a_k b_k|)
// with S_t the exact partial sum of the first 32 t products.  Products of two fp8 values are exact, subnormals
// included (the tensor core does not flush them); a NaN operand makes its row / column of C NaN, an e5m2 +-Inf gives
// +-Inf (NaN against a zero).  Each element's bits depend only on its row of A and column of B, not on the tile, the
// variant or ldc.  When deq falls below fp32's normal range (operands cast from a tiny amax, whose scale_inv is
// 2^-128) the output is finite but deq has lost significant bits, so C is far less precise than the product of the
// dequantised operands; no test holds it to more than being finite.
void gemm_fp8(const void* A, const void* B, void* C, int M, int N, int K, long long lda, long long ldb, long long ldc,
              bool a_e5m2, const float* scale_a, const float* scale_b, bool accumulate, int variant, cudaStream_t s,
              const void* bias) {
  if (M <= 0 || N <= 0) return;
  if ((N % 16) || (lda % 16) || (ldb % 16) || (ldc % 16))
    throw std::runtime_error("gemm_fp8: N and the leading dimensions must be multiples of 16 elements (TMA needs "
                             "16-byte row strides of the fp8 operands)");
  check_gemm_bases("gemm_fp8", A, B, C);
  check_bias("gemm_fp8", bias, true, true, accumulate, K);
  if (bias && a_e5m2) throw std::runtime_error("gemm_fp8: a bias needs an e4m3 A (the forward GEMM)");
  if (K <= 0) return gemm_empty_k(C, M, N, ldc, accumulate, s);
  if (variant == 0) variant = default_gemm_variant();
  if (variant == 3) variant = (M > 128) ? 2 : 1;
  const int cg = (variant == 2) ? 2 : 1;
  const void* as[1] = {A};
  const void* bs[1] = {B};
  GemmDist dist{};
  if (bias) {
    if (cg == 2) launch_gemm<true, true, 2, 0, 0, 0, 1, true>(as, bs, C, M, N, K, lda, ldb, ldc, false, dist, 1, s,
                                                             scale_a, scale_b, bias);
    else launch_gemm<true, true, 1, 0, 0, 0, 1, true>(as, bs, C, M, N, K, lda, ldb, ldc, false, dist, 1, s, scale_a,
                                                      scale_b, bias);
    return;
  }
#define DTG_GEMM_FP8_CASE(ET)                                                                                     \
  if (cg == 2) launch_gemm<true, true, 2, 0, 0, 0, ET>(as, bs, C, M, N, K, lda, ldb, ldc, accumulate, dist, 1, s,  \
                                                       scale_a, scale_b);                                        \
  else launch_gemm<true, true, 1, 0, 0, 0, ET>(as, bs, C, M, N, K, lda, ldb, ldc, accumulate, dist, 1, s, scale_a, \
                                               scale_b);
  if (a_e5m2) {
    DTG_GEMM_FP8_CASE(2)
  } else {
    DTG_GEMM_FP8_CASE(1)
  }
#undef DTG_GEMM_FP8_CASE
}

// Tensor-parallel GEMMs over NVLink symmetric buffers (always the CTA-pair kernel).
//   mode 1  all-gather(M) -> GEMM : A = concat_p a_srcs[p] ([rows_per_peer, K] each, K-major)
//   mode 2  GEMM -> reduce-scatter push : row chunk c of C goes to c_dsts[c] (already offset to my slot)
//   mode 3  wgrad with B gathered along K : B = concat_p b_srcs[p] ([rows_per_peer, N] each), A MN-major local
//   mode 4  wgrad with A gathered along K : A = concat_p a_srcs[p] ([rows_per_peer, M] each), B MN-major local
// Modes 1 and 2 keep the plain GEMM's K order, so their C is bit-identical to gemm_bf16 (variant 2) on the assembled
// operands; modes 3 and 4 start every tile at this rank's K slice (k_shift), which changes the fp32 summation order.
//
// Empty calls, here and in gemm_bf16_ag: with M or N = 0 nothing is launched (and nothing gathered); with K = 0 the
// product is zero, so overwrite mode writes zeros over C (mode 2: over every owner's rows_per_peer rows) and
// accumulate mode leaves C unchanged, as in gemm_bf16.
void gemm_bf16_dist(int mode, const void* const* a_srcs, const void* const* b_srcs, void* const* c_dsts, int M, int N,
                    int K, long long lda, long long ldb, long long ldc, bool b_kmajor, bool accumulate, int nranks,
                    int rank, int rows_per_peer, cudaStream_t s) {
  if (mode < 1 || mode > 4) throw std::runtime_error("gemm_bf16_dist: unknown mode");
  if (nranks < 1 || nranks > kMaxRanks) throw std::runtime_error("gemm_bf16_dist: 1..8 ranks");
  if (rank < 0 || rank >= nranks) throw std::runtime_error("gemm_bf16_dist: rank outside the ranks");
  if (M < 0 || N < 0 || K < 0) throw std::runtime_error("gemm_bf16_dist: negative extent");
  if (mode == 2 && accumulate) throw std::runtime_error("gemm_bf16_dist: mode 2 always overwrites");
  GemmDist dist{};
  dist.rows_per_peer = rows_per_peer;
  constexpr int TM = GemmCfg<2>::BM * 2;
  if (mode == 1 || mode == 2) {
    if (rows_per_peer % TM != 0 || rows_per_peer * nranks != M)
      throw std::runtime_error("gemm_bf16_dist: rows per rank must be a multiple of 256 and sum to M");
    dist.m_tile_shift = (mode == 1) ? rank * (rows_per_peer / TM) : ((rank + 1) % nranks) * (rows_per_peer / TM);
  } else {
    if (rows_per_peer % 64 != 0 || rows_per_peer * nranks != K)
      throw std::runtime_error("gemm_bf16_dist: K rows per rank must be a multiple of 64 and sum to K");
    dist.k_shift = rank * (rows_per_peer / 64);
  }
  if (M == 0 || N == 0) return;
  if ((N % 8) || (ldc % 8) || (lda % 8) || (ldb % 8))
    throw std::runtime_error("gemm_bf16_dist: N and the leading dimensions must be multiples of 8 elements");
  if (K == 0) {
    if (mode == 2)
      for (int p = 0; p < nranks; ++p) gemm_empty_k(c_dsts[p], rows_per_peer, N, ldc, false, s);
    else
      gemm_empty_k(c_dsts[0], M, N, ldc, accumulate, s);
    return;
  }
  for (int p = 0; p < nranks && c_dsts; ++p) dist.c_ptr[p] = (__nv_bfloat16*)c_dsts[p];
  void* C = c_dsts ? c_dsts[0] : nullptr;
  switch (mode) {
    case 1:
      if (b_kmajor) launch_gemm<true, true, 2, 1, 0, 0>(a_srcs, b_srcs, C, M, N, K, lda, ldb, ldc, accumulate, dist, nranks, s);
      else launch_gemm<true, false, 2, 1, 0, 0>(a_srcs, b_srcs, C, M, N, K, lda, ldb, ldc, accumulate, dist, nranks, s);
      break;
    case 2:
      if (b_kmajor) launch_gemm<true, true, 2, 0, 0, 1>(a_srcs, b_srcs, C, M, N, K, lda, ldb, ldc, false, dist, nranks, s);
      else launch_gemm<true, false, 2, 0, 0, 1>(a_srcs, b_srcs, C, M, N, K, lda, ldb, ldc, false, dist, nranks, s);
      break;
    case 3:
      launch_gemm<false, false, 2, 0, 2, 0>(a_srcs, b_srcs, C, M, N, K, lda, ldb, ldc, accumulate, dist, nranks, s);
      break;
    case 4:
      launch_gemm<false, false, 2, 2, 0, 0>(a_srcs, b_srcs, C, M, N, K, lda, ldb, ldc, accumulate, dist, nranks, s);
      break;
    default:
      throw std::runtime_error("gemm_bf16_dist: unknown mode");
  }
}


// all-gather -> GEMM with the gather done by communication CTAs of the same kernel (A_MODE 3).
//   a_bufs[p]: rank p's symmetric [M, K] buffer (its own rows_per_peer rows are valid); a_bufs[rank] is also the
//   destination of the gather.  flags: local uint32 [M / 256].  pads: the group's signal pads.
void gemm_bf16_ag(const void* const* a_bufs, const void* B, void* C, int M, int N, int K, long long ldb, long long ldc,
                  bool b_kmajor, int nranks, int rank, int rows_per_peer, uint32_t* flags, uint32_t ag_epoch,
                  uint32_t* const* pads, uint32_t bar_epoch, int n_comm, cudaStream_t s, const void* bias) {
  constexpr int TM = GemmCfg<2>::BM * 2;
  if (rows_per_peer % TM != 0 || rows_per_peer * nranks != M) throw std::runtime_error("gemm_bf16_ag: bad row split");
  if ((K * 2LL * TM) % GemmCfg<2>::COMM_PIECE != 0) throw std::runtime_error("gemm_bf16_ag: K must be a multiple of 64");
  if (nranks < 1 || nranks > kMaxRanks || rank < 0 || rank >= nranks)
    throw std::runtime_error("gemm_bf16_ag: 1..8 ranks and a rank among them");
  // the first n_comm CTA pairs copy; at least one pair must be left to multiply
  if (n_comm < 1 || n_comm >= sm_count() / 2)
    throw std::runtime_error("gemm_bf16_ag: n_comm must be in [1, " + std::to_string(sm_count() / 2) +
                             ") (at least one CTA pair copies and one multiplies), got " + std::to_string(n_comm));
  check_bias("gemm_bf16_ag", bias, true, b_kmajor, false, K);
  if (M == 0 || N == 0) return;
  if ((N % 8) || (ldc % 8) || (ldb % 8)) throw std::runtime_error("gemm_bf16_ag: N / leading dims must be multiples of 8");
  if (K == 0) return gemm_empty_k(C, M, N, ldc, false, s);
  GemmDist dist{};
  dist.rows_per_peer = rows_per_peer;
  dist.m_tile_shift = rank * (rows_per_peer / TM);
  for (int k = 0; k < nranks; ++k) dist.ag_src[k] = (const char*)a_bufs[(rank + k) % nranks];
  for (int p = 0; p < nranks; ++p) dist.pads[p] = pads[p];
  dist.ag_flags = flags;
  dist.ag_epoch = ag_epoch;
  dist.bar_epoch = bar_epoch;
  dist.n_comm = n_comm;
  dist.rank = rank;
  dist.nranks = nranks;
  dist.tile_bytes = (long long)TM * K * 2;
  const void* as[1] = {a_bufs[rank]};
  const void* bs[1] = {B};
  if (bias) launch_gemm<true, true, 2, 3, 0, 0, 0, true>(as, bs, C, M, N, K, K, ldb, ldc, false, dist, nranks, s,
                                                          nullptr, nullptr, bias);
  else if (b_kmajor) launch_gemm<true, true, 2, 3, 0, 0>(as, bs, C, M, N, K, K, ldb, ldc, false, dist, nranks, s);
  else launch_gemm<true, false, 2, 3, 0, 0>(as, bs, C, M, N, K, K, ldb, ldc, false, dist, nranks, s);
}


// Grouped GEMM of the mixture-of-experts layers (GRP 1 and 2 above), one launch for every expert; the routing tables
// seg [groups + 1] and tile_expert [rows / 128] are device pointers written by moe_route (moe.cu).
//   mode 0  forward  C[R, N] = A[R, K] . B_e[N, K]^T       B = [groups * N, K]   R = rows (a multiple of 128)
//   mode 1  dgrad    C[R, N] = A[R, K] . B_e[K, N]         B = [groups * K, N]   K % 64 == 0
//   mode 2  wgrad    C_e[M, N] (+)= A[seg_e, M]^T . B[seg_e, N]   A [K, M], B [K, N], C = [groups * M, N]; K is the
//                    row count of A and B (a multiple of 128), M % 128 == 0
// Modes 0 and 1 overwrite, and write nothing in row tiles past the last segment.  Every refusal happens before a
// launch.
void gemm_bf16_grouped(int mode, const void* A, const void* B, void* C, int M, int N, int K, long long lda,
                       long long ldb, long long ldc, int groups, const int* seg, const int* tile_expert,
                       bool accumulate, cudaStream_t s) {
  if (mode < 0 || mode > 2) throw std::runtime_error("gemm_bf16_grouped: mode must be 0 (forward), 1 (dgrad) or 2 (wgrad)");
  if (groups < 1) throw std::runtime_error("gemm_bf16_grouped: groups must be >= 1");
  if (M < 0 || N < 0 || K < 1) throw std::runtime_error("gemm_bf16_grouped: M, N >= 0 and K >= 1");
  if ((N % 8) || (ldc % 8) || (lda % 8) || (ldb % 8))
    throw std::runtime_error("gemm_bf16_grouped: N and the leading dimensions must be multiples of 8 elements");
  if (mode != 2 && accumulate) throw std::runtime_error("gemm_bf16_grouped: the forward and dgrad modes overwrite");
  if (mode != 2 && M % 128) throw std::runtime_error("gemm_bf16_grouped: the row count must be a multiple of 128");
  if (mode == 1 && K % 64)
    throw std::runtime_error("gemm_bf16_grouped: dgrad needs K % 64 == 0 (a K block never reaches the next expert)");
  if (mode == 2 && (M % 128 || K % 128))
    throw std::runtime_error("gemm_bf16_grouped: wgrad needs M % 128 == 0 and a row count K that is a multiple of 128");
  if (!seg || (mode != 2 && !tile_expert)) throw std::runtime_error("gemm_bf16_grouped: missing routing table");
  check_gemm_bases("gemm_bf16_grouped", A, B, C);
  if (M == 0 || N == 0) return;
  const void* as[1] = {A};
  const void* bs[1] = {B};
  GemmDist dist{};
  dist.grp_seg = seg;
  dist.grp_tile_expert = tile_expert;
  dist.grp_b_rows = mode == 0 ? N : K;
  if (mode == 0)
    launch_gemm<true, true, 1, 0, 0, 2>(as, bs, C, M, N, K, lda, ldb, ldc, false, dist, 1, s, nullptr,
                                                     nullptr, nullptr, groups);
  else if (mode == 1)
    launch_gemm<true, false, 1, 0, 0, 2>(as, bs, C, M, N, K, lda, ldb, ldc, false, dist, 1, s, nullptr,
                                                      nullptr, nullptr, groups);
  else
    launch_gemm<false, false, 1, 0, 0, 3>(as, bs, C, M, N, K, lda, ldb, ldc, accumulate, dist, 1, s,
                                                       nullptr, nullptr, nullptr, groups);
}

}  // namespace dtg
