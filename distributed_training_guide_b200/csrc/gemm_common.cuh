// Tile configuration shared by the wgmma GEMM and the fused GEMM+collective kernels.
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cstdint>

#include "common.cuh"

#ifndef DTG_DEFAULT_GEMM_VARIANT
#define DTG_DEFAULT_GEMM_VARIANT 3
#endif

namespace dtg {

template <int CG>
struct GemmCfg {
  static constexpr int THREADS = 384;     // producer warpgroup + two consumer warpgroups
  static constexpr int BM = 128;          // C rows per CTA (a CG-CTA cluster covers BM * CG rows)
  static constexpr int BN = 256;          // C columns per tile (wgmma N)
  static constexpr int BK = 64;           // one 128-byte swizzle span of bf16 per stage
  static constexpr int B_ROWS = BN / CG;  // rows of B (N) this CTA loads; CG 2 multicasts them to the pair
  static constexpr int A_BYTES = BM * BK * 2;
  static constexpr int B_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
  static constexpr int STAGES = 4;
  static constexpr int BAR_BYTES = 256;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + BAR_BYTES + 1024;  // +1024: manual alignment slack
  // A_MODE 3 communication CTAs reuse the pipeline smem as a ring of COMM_SLOTS pieces
  static constexpr int COMM_PIECE = 32768;
  static constexpr int COMM_SLOTS = STAGES * STAGE_BYTES / COMM_PIECE;
  // TMA-store epilogue (every mode but C_MODE 1): each consumer warpgroup stages half of its 64 x 256
  // output rows at a time, as two 64 x 64 boxes of 128B-swizzled bf16, behind the barrier area rounded up to 1 KB
  static constexpr int EPI_BOX_BYTES = 64 * 64 * 2;
  static constexpr int EPI_WG_BYTES = 2 * EPI_BOX_BYTES;
  static constexpr int EPI_OFFSET = STAGES * STAGE_BYTES + 1024;
  static constexpr int SMEM_BYTES_EPI = EPI_OFFSET + 2 * EPI_WG_BYTES + 1024;
  static constexpr int EPI_BAR = 2 * STAGES + 8;   // [2]: one C-load barrier per consumer warpgroup (accumulate mode)
  static_assert(2 * STAGES + (COMM_SLOTS > 2 ? COMM_SLOTS : 2) <= EPI_BAR && EPI_BAR + 2 <= BAR_BYTES / 8,
                "barrier area");
  static_assert(SMEM_BYTES_EPI <= 232448, "staging buffer exceeds the 227 KB of shared memory a CTA may have");
};

template <int N>
struct TmapSet {
  CUtensorMap m[N];
};

// Geometry of a tensor-parallel GEMM (all zero / unused for the plain GEMM).  The grouped GEMM of the
// mixture-of-experts layers (C_MODE 2 / 3) shares the storage of fields it never uses for its routing tables, so the
// kernels' parameter layout is the same for every mode.
struct GemmDist {
  union {
    int rows_per_peer;               // rows (M- or K-direction) each rank contributes / owns
    int grp_b_rows;                  // grouped forward / dgrad: rows of one expert's slab of B as stored
  };
  int m_tile_shift;                  // rotate the M tile order so every rank starts on its own rows
  int k_shift;                       // rotate the K block order likewise
  __nv_bfloat16* c_ptr[kMaxRanks];   // C_MODE 1: destination base (already offset to my slot) per owner
  // A_MODE 3 (all-gather by communication CTAs inside the GEMM kernel)
  const char* ag_src[kMaxRanks];     // the symmetric [M, K] buffer on every rank, ROTATED: [0] = mine
  union {
    uint32_t* ag_flags;              // local: one word per 256-row tile, set to ag_epoch once the tile landed
    const int* grp_tile_expert;      // grouped forward / dgrad: int32 [rows / 128], the expert of each row tile, or -1
  };
  uint32_t ag_epoch;
  uint32_t* pads[kMaxRanks];         // signal pads (not rotated) for the start-of-kernel barrier
  uint32_t bar_epoch;
  int n_comm;                        // clusters (CTA pairs) that copy instead of multiplying
  int rank, nranks;
  long long tile_bytes;              // bytes of one 256-row tile of A (contiguous: lda == K)
  const int* grp_seg;                // grouped: int32 [experts + 1], expert e owns rows [seg[e], seg[e + 1])
  // L2-aware rasterisation of the plain GEMM: tiles run M-fastest inside groups of `group_m` row tiles (0 = one
  // group = the whole M extent); `num_n_tiles` is set by the launcher.
  int group_m, num_n_tiles;
};

#ifdef __CUDACC__
__host__ __device__ __forceinline__ int tile_m(int t, int num_m_tiles, const GemmDist& d) {
  int m = t % num_m_tiles + d.m_tile_shift;
  return m >= num_m_tiles ? m - num_m_tiles : m;
}
// Tile order.  Default: M fastest (consecutive CTAs share the B tile) within a group of `group_m` row tiles
// whose slice of A stays L2-resident while B streams past once per group: the ~66 tiles in flight then touch
// group_m row panels of A and 66/group_m column panels of B instead of every row panel of A, which is what keeps
// a tall GEMM (wgrad with M = 22016 or 32000) from re-streaming all of A from HBM for every column of tiles.
// With an in-kernel all-gather
// (`local_m_tiles` > 0): first every tile of my own rows (pure local work while the communication CTAs
// fetch), then the remote row tiles in the order they are being fetched.
__host__ __device__ __forceinline__ void tile_mn(int t, int num_m_tiles, const GemmDist& d, int local_m_tiles, int& m, int& n) {
  if (local_m_tiles <= 0) {
    if (d.group_m > 0 && d.group_m < num_m_tiles) {
      const int per_group = d.group_m * d.num_n_tiles;
      const int g = t / per_group, r = t - g * per_group;
      const int m0 = g * d.group_m;
      const int rest_m = num_m_tiles - m0;
      const int gsz = d.group_m < rest_m ? d.group_m : rest_m;
      m = m0 + r % gsz;
      n = r / gsz;
      return;
    }
    m = tile_m(t, num_m_tiles, d);
    n = t / num_m_tiles;
    return;
  }
  const int num_n = d.k_shift;  // reused field: number of N tiles (K is never gathered in this mode)
  const int phase_a = local_m_tiles * num_n;
  int mm;
  if (t < phase_a) {
    mm = t % local_m_tiles;
    n = t / local_m_tiles;
  } else {
    const int u = t - phase_a, rest = num_m_tiles - local_m_tiles;
    mm = local_m_tiles + u % rest;
    n = u / rest;
  }
  mm += d.m_tile_shift;
  m = mm >= num_m_tiles ? mm - num_m_tiles : mm;
}
#endif

// TMA descriptor builders (gemm_wgmma.cu)
CUtensorMap make_tmap_bf16(const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                           const uint32_t* box, bool swizzle128);
CUtensorMap make_tmap_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes,
                         uint32_t box_inner, uint32_t box_outer);
void set_gemm_variant(int v);
int default_gemm_variant();

}  // namespace dtg
