// Host-side launcher API of the sm_90a kernels (raw pointers + stream; no torch types so the
// .cu files compile in seconds).  bind.cpp adapts torch tensors onto these.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>

namespace dtg {

unsigned long long launch_count();

// ---- norm.cu -------------------------------------------------------------------------------
// Row norms over bf16 [T, H] rows (H % 8 == 0, H <= norm_max_hidden(kind)) with fp32 statistics:
//   kRms  y = bf16(h * rstd * w)
//   kLn   y = bf16((h - mean) * rstd * w + b)                                     (StarCoder2)
//   kLn2  y1, y2 = the kLn output for (w1, b1) and for (w2, b2), one statistic    (GPT-NeoX)
// with h = x (kNone), h = bf16(x + r) written to h and normalised (kAddBefore), or, kRms only, h = bf16(r + y)
// written to h instead of y (kAddAfter, OLMo 2's norm-then-add).  LayerNorm rows whose sums overflow fp32 are
// normalised scaled by 2^-72.
enum class NormKind : int { kRms, kLn, kLn2 };
enum class NormRes : int { kNone, kAddBefore, kAddAfter };
// fp32 [H] gradient planes of a kind: dw; dw, db; dw1, db1, dw2, db2
constexpr int norm_grad_planes(NormKind k) { return k == NormKind::kRms ? 1 : k == NormKind::kLn ? 2 : 4; }
int norm_max_hidden(NormKind k);
// Operands a variant does not use are null.  mean and rstd are fp32 [T]; mean is LayerNorm's only.
struct NormFwdArgs {
  const void* x;
  const void* r;       // kAddBefore / kAddAfter
  const void* w[2];    // [H] gains; w[1] for kLn2
  const void* b[2];    // [H] biases (LayerNorm)
  void* y[2];          // not written by kAddAfter
  void* h;             // kAddBefore / kAddAfter
  float* mean;
  float* rstd;
};
void norm_fwd(NormKind k, NormRes res, const NormFwdArgs& a, int T, int H, float eps, cudaStream_t s);
// Persistent CTAs of the backward (at most T); partial rows per CTA fix the order of the gradient sums.
int norm_bwd_grid(NormKind k, int T, int H);
struct NormBwdArgs {
  const void* dy[2];   // dy[1] for kLn2
  const void* h;       // the normalised rows (x itself without a residual)
  const void* w[2];
  const float* mean;
  const float* rstd;
  const void* dres;    // added to dx when given
  void* dx;
  float* partial;      // fp32 [norm_grad_planes(k), norm_bwd_grid(k, T, H), H] scratch
  float* dparams;      // fp32 [norm_grad_planes(k), H], summed from partial in a fixed order
};
// 1 + norm_grad_planes(k) launches: the norm kernel, then one colsum per gradient plane
void norm_bwd(NormKind k, const NormBwdArgs& a, int T, int H, cudaStream_t s);

// ---- elementwise.cu ------------------------------------------------------------------------
// out[c] = sum over rows r of partial[r][c] (fp32 [rows, H]), in a fixed order
void colsum(const float* partial, float* out, int rows, int H, cudaStream_t s);
// bias gradient: db[n] = sum over t of dy[t, n], dy bf16 [T, N] with row stride ld (elements); N, ld multiples of 8.
// Each CTA sums a fixed range of rows in fp32 into one row of `partial` (fp32 [bias_grad_chunks(T, N), N]), which
// colsum then adds in a fixed order: no atomics, bit-identical from run to run.
int bias_grad_chunks(long long T, int N);
void bias_grad(const void* dy, long long T, int N, long long ld, float* partial, float* db, cudaStream_t s);
// GELU with the tanh approximation on n bf16 elements (n % 8 == 0); the backward from the saved pre-activation x
void gelu_tanh_fwd(const void* x, void* y, long long n, cudaStream_t s);
void gelu_tanh_bwd(const void* dy, const void* x, void* dx, long long n, cudaStream_t s);
// GELU, exact erf form, likewise
void gelu_fwd(const void* x, void* y, long long n, cudaStream_t s);
void gelu_bwd(const void* dy, const void* x, void* dx, long long n, cudaStream_t s);
void swiglu_fwd(const void* gu, void* h, long long T, int I, cudaStream_t s);
void swiglu_bwd(const void* dh, const void* gu, void* dgu, long long T, int I, cudaStream_t s);
// Embedding ids follow the vocabulary rule of common.cuh: an id outside [0, V) gets a NaN row from the forward and adds
// to no row of dw.  out [T,H] = w [V,H] rows.
void embedding_fwd(const long long* ids, const void* w, void* out, long long T, long long V, int H, cudaStream_t s);
// dw [V,H] = (or +=) the per-id sum of dout [T,H], in fp32 with one rounding per row.  Scratch: slot [V] uint32 and
// sums [T,H] fp32, both filled here.  Overwrite mode zeroes the whole table first.
void embedding_bwd(const void* dout, const long long* ids, void* dw, unsigned int* slot, float* sums, long long T,
                   long long V, int H, bool accumulate, cudaStream_t s);
void embedding_bwd_sorted(const void* dout, const long long* ids_sorted, const long long* perm, void* dw, long long T,
                          long long V, int H, bool accumulate, cudaStream_t s);
void scale_inplace(void* x, const float* scale, long long n, cudaStream_t s);

// ---- rope.cu -------------------------------------------------------------------------------
// rotates the first rot_dim elements (rot_dim % 16 == 0, <= d; d for the full head) of heads [0, n_rot); cos/sin
// [S, rot_dim/2] or [T, rot_dim/2]
void rope_inplace(void* qkv, const float* cos, const float* sin, long long T, int S, int n_heads, int n_rot, int d,
                  int rot_dim, bool per_token, bool inverse, cudaStream_t s);
// QK-norm + RoPE (Qwen3) in place on heads [0, nh + nkv) of qkv [T, n_heads, 128] bf16 (n_heads = nh + 2*nkv):
// per head y = bf16(bf16(x * rstd) * w) with w = q_w (heads < nh) or k_w, then the RoPE of rope_inplace.  cos/sin:
// fp32 [S, 64] (pos = t % S) or per-token [T, 64].  Writes x_save [T, nh + nkv, 128] bf16 (the pre-norm q|k heads)
// and rstd [T, nh + nkv] fp32 for the backward.
void qk_norm_rope_fwd(void* qkv, const void* q_w, const void* k_w, const float* cos, const float* sin, void* x_save,
                      float* rstd, long long T, int S, int n_heads, int nh, int nkv, bool per_token, float eps,
                      cudaStream_t s);
int qk_norm_rope_bwd_grid(long long T, int nqk);
// In place on the q|k heads of dqkv: inverse rotation, then the RMSNorm backward.  dw [2, 128] fp32 = the q and
// k gain gradients; dw_partial: [qk_norm_rope_bwd_grid(T, nh + nkv), 256] fp32 scratch.
void qk_norm_rope_bwd(void* dqkv, const void* x_save, const float* rstd, const void* q_w, const void* k_w,
                      const float* cos, const float* sin, float* dw_partial, float* dw, long long T, int S, int n_heads,
                      int nh, int nkv, bool per_token, cudaStream_t s);
// Full-width QK-norm + RoPE (OLMo 2) on the same layout: one RMSNorm over a token's whole q region (nh * 128
// elements, gain q_w [nh * 128]) and one over its k region (k_w [nkv * 128]), y = bf16(x * rstd * w), then the RoPE
// of rope_inplace.  Writes x_save [T, nh + nkv, 128] bf16 and rstd [T, 2] fp32 (q, k).  nh + nkv <=
// qk_norm_full_rope_max_heads().
int qk_norm_full_rope_max_heads();
void qk_norm_full_rope_fwd(void* qkv, const void* q_w, const void* k_w, const float* cos, const float* sin,
                           void* x_save, float* rstd, long long T, int S, int n_heads, int nh, int nkv, bool per_token,
                           float eps, cudaStream_t s);
int qk_norm_full_rope_bwd_grid(long long T, int nqk);
// dw [(nh + nkv) * 128] fp32 = the q gain gradient followed by the k gain gradient; dw_partial:
// [qk_norm_full_rope_bwd_grid(T, nh + nkv), (nh + nkv) * 128] fp32 scratch.
void qk_norm_full_rope_bwd(void* dqkv, const void* x_save, const float* rstd, const void* q_w, const void* k_w,
                           const float* cos, const float* sin, float* dw_partial, float* dw, long long T, int S,
                           int n_heads, int nh, int nkv, bool per_token, cudaStream_t s);

// ---- cross_entropy.cu ----------------------------------------------------------------------
// logits [T,V] bf16 are overwritten with dlogits = (softmax - onehot) / n_valid; loss = mean CE.
void cross_entropy_fwd_bwd(void* logits, const long long* targets, float* row_loss, float* n_valid, float* loss,
                           int T, int V, cudaStream_t s);

// ---- adamw.cu ------------------------------------------------------------------------------
// state_fp32: exp_avg / exp_avg_sq stored as fp32 instead of bf16
void adamw_flat(void* p, const void* g, void* m, void* v, long long n, float lr, float beta1, float beta2, float eps,
                float wd, int step, float grad_scale, bool state_fp32, cudaStream_t s);

// ---- gemm_wgmma.cu -------------------------------------------------------------------------
// out[M,N] (+)= op(A) @ op(B), bf16 in / fp32 register accumulate / bf16 out, row-major storage:
//   a_kmajor: A stored [M,K] (else [K,M]);  b_kmajor: B stored [N,K] (else [K,N]).
// lda/ldb/ldc are row strides in elements.  variant: 0 = auto, 1 = 1-CTA 128x256, 2 = 2-CTA cluster 256x256
// bias: null, or bf16 [N] added to every row before the rounding to bf16 (forward layout, a_kmajor and b_kmajor,
// overwrite mode only; 16-byte aligned).  The same holds for the bias of gemm_fp8 (e4m3 A) and gemm_bf16_ag.
void gemm_bf16(const void* A, const void* B, void* C, int M, int N, int K, long long lda, long long ldb, long long ldc,
               bool a_kmajor, bool b_kmajor, bool accumulate, int variant, cudaStream_t s, const void* bias = nullptr);

// C[M,N] (+)= scale_a[0] * scale_b[0] * A8[M,K] . B8[N,K]^T with fp8 operands (A e4m3, or e5m2 when a_e5m2; B e4m3),
// both K-major; scale_a / scale_b are device pointers.  N, lda, ldb and ldc must be multiples of 16.
void gemm_fp8(const void* A, const void* B, void* C, int M, int N, int K, long long lda, long long ldb, long long ldc,
              bool a_e5m2, const float* scale_a, const float* scale_b, bool accumulate, int variant, cudaStream_t s,
              const void* bias = nullptr);

int gemm_max_active_clusters(int cg);
// tensor-parallel variants over symmetric buffers (see gemm_wgmma.cu)
void gemm_bf16_dist(int mode, const void* const* a_srcs, const void* const* b_srcs, void* const* c_dsts, int M, int N,
                    int K, long long lda, long long ldb, long long ldc, bool b_kmajor, bool accumulate, int nranks,
                    int rank, int rows_per_peer, cudaStream_t s);

void gemm_bf16_ag(const void* const* a_bufs, const void* B, void* C, int M, int N, int K, long long ldb, long long ldc,
                  bool b_kmajor, int nranks, int rank, int rows_per_peer, uint32_t* flags, uint32_t ag_epoch,
                  uint32_t* const* pads, uint32_t bar_epoch, int n_comm, cudaStream_t s, const void* bias = nullptr);

// Grouped GEMM of the mixture-of-experts layers, one launch for every expert (see gemm_wgmma.cu for the modes);
// seg [groups + 1] and tile_expert [rows / 128] are the device tables moe_route writes.
void gemm_bf16_grouped(int mode, const void* A, const void* B, void* C, int M, int N, int K, long long lda,
                       long long ldb, long long ldc, int groups, const int* seg, const int* tile_expert,
                       bool accumulate, cudaStream_t s);

// ---- moe.cu --------------------------------------------------------------------------------
// Routing of T tokens over E <= kMoeMaxExperts experts, top-k (see moe.cu for the layout).  rows_cap = the most
// permuted rows any routing can need, T * k + E * 127 rounded up to 128; scratch: int32 [moe_route_scratch(T, E)].
constexpr int kMoeMaxExperts = 256;
long long moe_rows_cap(long long T, int E, int k);
long long moe_route_scratch(long long T, int E);
// From bf16 router logits [T, E] (row stride ldl): p fp32 [T, E] (softmax), idx int32 [T, k], w fp32 [T, k] (the
// top-k probabilities, ties to the lower expert; norm_topk: divided by their sum), pos int32 [T, k], seg int32
// [E + 1], tile_expert int32 [rows_cap / 128], row_tok int32 [rows_cap] (rows below seg[E]) and counts int32 [E].
void moe_route(const void* logits, long long ldl, int T, int E, int k, bool norm_topk, float* p, int* idx, float* w,
               int* pos, int* seg, int* tile_expert, int* row_tok, int* counts, int* scratch, cudaStream_t s);
// out [rows_cap, H]: row r < seg[E] is x [T, H]'s row of its token, or zeros on a padding row (NaN where row_tok[r]
// is outside [-1, T * k))
void moe_permute(const void* x, int T, const int* row_tok, const int* seg, int E, int k, int H, long long rows_cap,
                 void* out, cudaStream_t s);
// out [T, H] = bf16(sum over slots, in slot order, of w * yp[pos]) in fp32; w null: weights 1 (the input gradient).
// yp has yp_rows >= 1 rows (when T > 0); a token with a pos outside [0, yp_rows) gets a NaN row.
void moe_combine(const void* yp, long long yp_rows, const int* pos, const float* w, int T, int k, int H, void* out,
                 cudaStream_t s);
// The combine's backward: dyp [rows_cap, H] row r < seg[E] = bf16(w[a] * dy[t]) (zeros on padding rows) and dw fp32
// [T, k] = sum_h dy[t, h] * yp[r, h], for a = row_tok[r] and t = a / k (dy [T, H]; a row whose a is outside
// [-1, T * k) gets a NaN dyp row and writes no dw)
void moe_combine_bwd(const void* dy, int T, const void* yp, const int* row_tok, const int* seg, const float* w, int E,
                     int k, int H, long long rows_cap, void* dyp, float* dw, cudaStream_t s);
// dlogits bf16 [T, E] = bf16(p * (dp - sum_e p dp)) with dp = dw at the selected experts, plus dpsum [E] (null: 0);
// norm_topk (w = p_sel / S): dp = (dw - sum_i w_i dw_i) / S at the selected experts, plus dpsum
void moe_router_bwd(const float* p, const int* idx, const float* dw, const float* dpsum, int T, int E, int k,
                    bool norm_topk, void* dlogits, cudaStream_t s);

// ---- fp8.cu --------------------------------------------------------------------------------
// amax[0] = max |x| of a bf16 [R, C] matrix with row stride ld (elements), on the device.
void fp8_amax(const void* x, long long R, int C, long long ld, float* amax, cudaStream_t s);
// q = satfinite(x * scale) in e4m3 (or e5m2), scale = amax == 0 ? 1 : FP8_MAX / amax, written row-major to `out`
// [R, C] and / or transposed to `out_t` [C, R] (either may be null); scale_inv[0] = 1 / scale.
void fp8_cast_transpose(const void* x, long long ld, int R, int C, bool e5m2, const float* amax, void* out, void* out_t,
                        float* scale_inv, cudaStream_t s);

// ---- attention_fwd.cu / attention_bwd.cu ---------------------------------------------------
// qkv: [B,S,nh+2*nkv,D] bf16 (q heads | k heads | v heads); o: [B,S,nh,D]; lse: [B,nh,S] fp32; head_dim D = 64 or 128
// attn_fwd: P through shared memory; attn_fwd2: P kept in registers
// doc_start: null (plain causal) or int32 [B,S], the first token of each token's document (document masking:
// key k is visible to query q iff doc_start[q] <= k <= q)
// window: 0 (none) or W >= 1, sliding-window attention: key k is also visible only if k > q - W.  W >= S masks
// nothing and runs the kernels without a window.
void attn_fwd(const void* qkv, void* o, float* lse, int B, int S, int nh, int nkv, float scale, cudaStream_t s,
              const int* doc_start = nullptr, int window = 0, int head_dim = 128);
void attn_fwd2(const void* qkv, void* o, float* lse, int B, int S, int nh, int nkv, float scale, cudaStream_t s,
               const int* doc_start = nullptr, int window = 0, int head_dim = 128);
void attn_bwd(const void* qkv, const void* o, const void* d_o, const float* lse, float* delta, float* dq_acc,
              void* dqkv, int B, int S, int nh, int nkv, float scale, int mode, cudaStream_t s,
              const int* doc_start = nullptr, int window = 0, int head_dim = 128);

}  // namespace dtg
