/*
 * segtran_b200 — C ABI of the H100-native (sm_90a) Squeeze-and-Expansion hot path.
 *
 * The reference (askerlee/segtran) is pure Python/PyTorch and has no FFI layer: the drop-in
 * boundary is the nn.Module contract of code/networks/segtran_shared.py (SegtranFusionEncoder
 * :819-975 and the modules it owns) and of the Segtran2d/Segtran3d shells.  This header is the
 * C ABI introduced *underneath* that contract (SURVEY.md §8b): every entry point names the
 * reference call sites whose arithmetic it replaces.  Host binding: ctypes (segtran_b200/_lib.py);
 * see INTEGRATION.md for the binding a maintainer of the reference would add.
 *
 * Conventions
 *  - every pointer is a caller-owned DEVICE pointer (tensor.data_ptr()); nothing is retained
 *    after the call returns; scratch is passed in explicitly by the caller;
 *  - `part, part_floats`: scratch for per-CTA partial sums, which a second kernel adds in a fixed order, so results are
 *    bit-identical from run to run; a larger scratch allows more CTAs (up to the machine's width); it must not be in
 *    use by another stream while the call runs;
 *  - every call is asynchronous on the cudaStream_t given (passed as void*);
 *  - return 0 on success, negative on error; sx_last_error() returns a thread-local message;
 *  - no global mutable state apart from one-time function-attribute setup (thread safe: the
 *    autograd engine calls backward entry points from its own worker thread);
 *  - the device is the current CUDA context's device (torch sets it); never assumed to be 0.
 *  - there is NO CPU fallback: a missing GPU / non-sm_90 device is an error.
 */
#ifndef SEGTRAN_B200_H_
#define SEGTRAN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SX_VERSION 1

/* element types */
enum { SX_F32 = 0, SX_BF16 = 1 };
/* GEMM operand arithmetic: TF32 (fp32 storage, 10-bit mantissa in the tensor core) or BF16 */
enum { SX_OP_TF32 = 0, SX_OP_BF16 = 1 };
/* operand majorness: K-major = reduction dim contiguous; MN-major = row/col dim contiguous */
enum { SX_MAJOR_K = 0, SX_MAJOR_MN = 1 };
enum { SX_BIAS_NONE = 0, SX_BIAS_N = 1, SX_BIAS_M = 2 };
enum { SX_ACT_NONE = 0, SX_ACT_GELU = 1,
       SX_ACT_GELU_BWD = 2 /* C = dropmask * (alpha A.B^T) * gelu'(preact): `preact` is an INPUT in C's layout */ };

int sx_version(void);
const char* sx_last_error(void);
/* number of SMs / compute capability of the current device (diagnostics; fails if no GPU) */
int sx_device_info(int* sm_count, int* cc_major, int* cc_minor);

/* ---------------------------------------------------------------------------------------------
 * Batched GEMM on the wgmma tensor cores (TMA-staged operands, fp32 accumulators in registers):
 *     C[z1][z0][m][n] = epilogue( alpha * sum_k A[z1][z0][m][k] * B[z1][z0][n][k] )
 * Replaces every dense contraction on the path: the Q/K/V projections (segtran_shared.py:559-560,
 * :414), Q.K^T (:566), P.V (:447), MMSharedMid's shared Linear (:243), MMPrivateOutput's grouped
 * Conv1d (:267), and all of their backward products.
 * An operand with majorness K stores element (r,k) at ptr[r*ld + k]; majorness MN at ptr[k*ld + r].
 * stride_z0/stride_z1 are in elements; 0 broadcasts the operand over that batch dim.
 * Requirements: ptr 16-byte aligned; ld*elsize and z strides*elsize multiples of 16 bytes.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  const void* ptr;
  int32_t major;
  int32_t _pad;
  int64_t ld;
  int64_t stride_z0;
  int64_t stride_z1;
} sx_operand;

typedef struct {
  int32_t op_dtype;              /* SX_OP_TF32 | SX_OP_BF16 (A and B element type: f32 | bf16) */
  int32_t M, N, K, Z0, Z1;
  sx_operand A, B;
  void* C;
  int32_t c_dtype;               /* SX_F32 | SX_BF16 */
  int32_t round_tf32;            /* round fp32 outputs to TF32 (RN) so a following TF32 GEMM is exact on them */
  int64_t ldc, c_stride_z0, c_stride_z1;
  float alpha;
  int32_t bias_mode;             /* SX_BIAS_* ; bias is fp32 */
  const float* bias;
  int64_t bias_stride_z0, bias_stride_z1;
  int32_t act;                   /* SX_ACT_* */
  int32_t accumulate;            /* 0: store, 1: atomicAdd into fp32 C (needed when split_k > 1) */
  void* preact;                  /* optional: pre-activation (after bias) in C's layout and dtype */
  int32_t split_k;               /* >= 1 */
  int32_t _pad2;
  float* amax;                   /* optional: atomicMax of the stored values (attention-score diagnostics, :569-573) */
  float drop_p;                  /* dropout on the stored value (after act); 0 disables */
  uint32_t _pad3;
  uint64_t drop_seed;            /* counter-based mask: keep(idx) = hash(seed, flat index in C) >= p */
  const uint64_t* drop_seed_dev; /* optional device seed added to drop_seed (CUDA-graph safe) */
  const float* addend;           /* optional fp32 tensor in C's layout: C = epilogue(alpha*A.B^T + addend); used by the
                                    error-compensated 3-pass TF32 mode (A_hi B_hi + A_lo B_hi + A_hi B_lo) */
  float* colsum;                 /* optional [N] fp32: += column sums of the stored values over all rows and batch slices
                                    (a bias gradient that would otherwise need its own pass over the output; float atomics,
                                    so the order of the additions varies: sx_colsum on the output is the ordered form) */
  float* part;                   /* split_k > 1: scratch for the partial tiles (summed in split order); split_k is lowered
                                    to what part_floats holds (128*128 floats per output tile and split), to 1 if NULL */
  int64_t part_floats;
} sx_gemm_args;

int sx_gemm(const sx_gemm_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Sliding-window positional biases (SlidingPosBiases2D/3D, segtran_shared.py:1002-1175), never expanded to [N,N]:
 * the tokens are the cells of a row-major grid grid[0..pd); for a query cell q and a key cell k
 *     bias(q,k) = w * table[(k_0-q_0+R), ..., (k_{pd-1}-q_{pd-1}+R)]   when |k_i - q_i| <= R in every dimension,
 *     bias(q,k) = 0                                                       otherwise;
 * table is [2R+1]^pd fp32 (row-major).  Every entry point that takes an sx_posbias reads it through the one device
 * helper of csrc/sx_posbias.cuh.  table == NULL means no bias.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  const float* table;
  int32_t pd, R;                 /* pd in {2, 3}, R >= 1 */
  int32_t grid[3];
  float w;                       /* pos_code_weight (--posw) */
} sx_posbias;

/* ---------------------------------------------------------------------------------------------
 * Fused attention probabilities of the squeeze-out stage (csrc/sx_attn.cu):
 *     P[b][m] = dropout( softmax_keys( min(alpha * Q[b,:,m] K[b,:,m]^T, clip) ) )
 * One persistent wgmma kernel replaces segtran_shared.py:566-567 (Q.K^T / sqrt(d)), :569-580 (max statistics and
 * conditional clamp), :601 (softmax) and :605 (attention dropout): the scores stay in registers, the softmax runs on
 * the accumulator fragments, only P is written (plus the raw scaled scores S when the backward needs them).  More than
 * 128 keys do not fit one accumulator per row block: the scores are then produced twice (a statistics pass, then a
 * probabilities pass over the key chunks of the same row block) instead of being written and re-read.
 * Q [Bq][U1][M*d] (q_bstride = 0: one query bank shared by the batch), K [B][U2][M*d]; mode m uses columns
 * [m*d, (m+1)*d).  P, S: [B][M][U1][ldp] fp32, ldp % 4 == 0.  lse, rowmax: [B][M][U1] (natural-log units; rowmax is
 * the max of the raw row).  stat: device scratch of three 32-bit words, ZERO-initialised by the caller: [0] the running
 * maximum of the scores under an order-preserving float->uint map (0 = none yet), [1] (float) number of rows whose
 * maximum is below -(clip - 104), [2] (written at the end) the maximum as a plain float — the `amax` of sx_softmax_bwd.  diag (optional, device float[3]): [0] running
 * max, [1] += 1 when the clamp fired (max > clip), [2] += stat[1] in that case (rows where the reference's LOWER
 * clamp could have mattered — the upper clamp is applied exactly; see sx_attn.cu).
 * posbias (table != NULL; self-attention, U1 == U2 == the grid's cell count): the score becomes
 * min(alpha * Q K^T, clip) + bias(q,k) inside the softmax (segtran_shared.py:589-592).  S, rowmax, stat[0] and the clamp
 * decision stay on the raw scores; lse is the log-sum-exp of the biased row; stat[1] counts rows whose raw maximum is
 * below -(clip - 104) + (bmax - bmin), with bmin / bmax the range of {w * table} and 0.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  int32_t B, M, U1, U2, d;
  int32_t round_tf32;
  const float* Q;
  int64_t q_ld, q_bstride;
  const float* K;
  int64_t k_ld, k_bstride;
  float alpha, clip;
  float* P;
  float* S;                      /* optional */
  int64_t ldp;
  float* lse;
  float* rowmax;                 /* optional */
  float* stat;
  float* diag;                   /* optional */
  float drop_p;
  uint32_t _pad;
  uint64_t drop_seed;
  const uint64_t* drop_seed_dev;
  sx_posbias posbias;            /* table == NULL: no positional bias */
} sx_attn_probs_args;
int sx_attn_probs_fwd(const sx_attn_probs_args* args, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Attention-consistency loss of one layer (csrc/sx_consist.cu; train3d.py:426-449 and train2d.py:668-723), without
 * the [B,N,N] affinity matrix X or the [B,N,N] class-consistency matrix ever reaching memory:
 *   c_ij = min(max(sum_k F[b,k,i] F[b,k,j], 0), 1)           F [B][K][N] fp32 (the downsampled mask), K <= 16
 *   SX_CONSIST_BCE    : loss = mean over B*N*N of BCEWithLogits(X, c)       (train3d.py)
 *   SX_CONSIST_MARGIN : mu_b = mean of X_b; element (b,i,j) is inconsistent when (x < mu_b && c != 0) or
 *                       (x > mu_b - 0.1 && c == 0); loss = sum |x - mu_b| over the inconsistent elements of all batches
 *                       divided by their count (NaN when there are none, as in the reference)       (train2d.py)
 * Pair input (X = Xo . Xi, squeezed layers): Xo [B][N][A] and Xt = Xi^T [B][N][A], both K-major (row pitch and batch
 *   stride multiples of 4 floats), TF32 values; A may be the width of K-concatenated hi/lo operand splits
 *   (sx_split_tf32_cat, roles 0 and 1), which makes the product 3-pass.  X is produced tile by tile by a persistent
 *   wgmma kernel and consumed on the accumulator fragments.
 * Dense input (Xo == NULL): X [B][N][N] with row pitch x_ld and batch stride x_bstride.
 * mu (MARGIN only): device [B], the per-batch means of X, computed by the caller.
 * R (optional): the unscaled residual sigmoid(x) - c (BCE) or sign(x - mu)*[inconsistent] (MARGIN), [B][N][ldr],
 *   rounded to TF32 when round_r; the backward products dXo = R Xi^T and dXi = Xo^T R are sx_gemm calls.
 * out (device float [2 + B], written): [0] the layer's loss, [1] d loss / d x per unit residual (1/(B N^2), or 1/count,
 *   0 when count == 0), [2 + b] (MARGIN) the gradient through mu_b per element of batch b and unit residual,
 *   -(sum of sign(x - mu_b) over the inconsistent elements of batch b) / N^2.
 * cap (optional, device float[2]): cap[0] += out[0]; cap[1] = t > 1 ? 1/t : 1 with t = cap_scale * cap[0] — the
 *   factor of train2d.py's `if loss > 1: loss /= loss.item()` after the last layer, without a host read.
 * The per-CTA sums go through `part` and are added in a fixed order: two runs give the same bits.
 * ------------------------------------------------------------------------------------------- */
enum { SX_CONSIST_BCE = 0, SX_CONSIST_MARGIN = 1 };
typedef struct {
  int32_t B, N, A, K;
  int32_t variant;
  int32_t round_r;
  const float* Xo;
  int64_t xo_ld, xo_bstride;
  const float* Xt;
  int64_t xt_ld, xt_bstride;
  const float* X;
  int64_t x_ld, x_bstride;
  const float* F;
  const float* mu;
  float* R;
  int64_t ldr;
  float* out;
  float* cap;
  float cap_scale;
  int32_t _pad;
  float* part;
  int64_t part_floats;
} sx_consist_args;
int sx_attn_consist_fwd(const sx_consist_args* args, void* stream);
/* Gradient of one layer's loss with respect to one input, from the raw backward product G (R Xi^T, Xo^T R, or R itself
 * for a dense input), in place or out of place: for batch b, row r, column c of [B][rows][cols]
 *   dst = s * (G + m_b * v),  s = (*gout) * out[1],  m_b = out[2 + b] (MARGIN; 0 for BCE),
 *   v = vrow[b*rows + r] if vrow, else vcol[b*cols + c] if vcol, else 1
 * (the rank-1 term of the gradient through mu: vrow / vcol are Xo's column sums / Xi's row sums per batch). */
int sx_attn_consist_bwd(const sx_consist_args* args, const float* gout, const float* G, int32_t rows, int32_t cols,
                        int64_t ldg, int64_t g_bstride, const float* vrow, const float* vcol, float* dst, int64_t ldd,
                        int64_t d_bstride, void* stream);

/* The attention scores a layer keeps for the loss above (segtran_shared.py:578-598): the reference keeps them after its
 * conditional clamp.  S [R,L] (row pitch lds), amax = device max of S.
 *   dY == NULL: out = (*amax > clip) ? clamp(S, -clip, clip) : S
 *   otherwise : out = (*amax > clip && |S| > clip) ? 0 : dY       (the clamp's gradient) */
int sx_clamp_if(const float* S, int64_t R, int32_t L, int64_t lds, const float* amax, float clip, const float* dY,
                int64_t ldy, float* out, int64_t ldo, void* stream);

/* Dropout seeds: every dropout-capable entry takes `seed` (by value) and `seed_dev` (device pointer or NULL); the
 * effective seed is seed + *seed_dev, read on the device in stream order, so a captured CUDA graph draws a new mask
 * on every replay.  sx_seed_derive writes out[0] = base[0] + add (the per-call seed an op keeps for its backward);
 * sx_seed_advance bumps the base seed once per training step. */
int sx_seed_derive(const uint64_t* base, uint64_t add, uint64_t* out, void* stream);
int sx_seed_advance(uint64_t* base, uint64_t inc, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Row-wise kernels (HBM-bound).  "act dtype" arguments are SX_F32 | SX_BF16; round_tf32 rounds fp32
 * outputs that feed a TF32 GEMM.  Dropout masks are counter-based: keep(i) = hash(seed, flat index)
 * >= p, so backward regenerates the forward mask from (seed, index) instead of storing it.
 * ------------------------------------------------------------------------------------------- */

/* out[0] = max(x[0..n))                        -- voxels_pos.max(), segtran_shared.py:1231 */
int sx_reduce_max(const float* x, int64_t n, float* out, void* stream);

/* Learnable-sinusoid positional code, LearnedSinuPosEmbedder.forward (segtran_shared.py:989-998) with the
 * pos/pos.max() normalisation of SegtranPosEncoder.forward (:1231).  pos [R,pd], W [C,pd], b [C] -> pe [R,C]. */
int sx_pos_lsinu_fwd(const float* pos, const float* posmax, int64_t R, int32_t pd, const float* W, const float* b,
                     int32_t C, float* pe, void* stream);
/* dpe [R,C] -> dW [C,pd], db [C] accumulated (+=); de_scratch [R,C] is caller-provided scratch. */
int sx_pos_lsinu_bwd(const float* pos, const float* posmax, int64_t R, int32_t pd, const float* W, const float* b,
                     int32_t C, const float* dpe, float* de_scratch, float* dW, float* db, float* part, int64_t part_floats, void* stream);

/* Fused prologue of SegtranFusionEncoder.forward (segtran_shared.py:916, :930-934, :944-946):
 *   h = mask * dropout( LN( LN_{g,b}(x) + posw * pe[..., :C] ) ),  x [B,N,C] fp32, pe rows of length C0,
 *   pe_bstride = 0 when the code is shared by the batch; mask [B*N] fp32 or NULL; stats [B*N,4].
 * pe == NULL (pos_code_type 'bias' / 'none', :940): h = mask * dropout( LN_{g,b}(x) ), no second LayerNorm; C0,
 *   pe_bstride and posw are ignored, stats[r] = {mean, rstd, 0, 1} of x's row, and the backward takes dpe == NULL. */
int sx_prologue_fwd(const float* x, int64_t B, int32_t N, int32_t C, const float* g, const float* b, const float* pe,
                    int32_t C0, int64_t pe_bstride, float posw, const float* mask, float drop_p, uint64_t seed, const uint64_t* seed_dev, void* h,
                    int32_t h_dtype, int32_t round_tf32, float* stats, void* stream);
/* dh fp32 -> dx [B,N,C]; dg, db [C] and dpe (same addressing as pe, may be NULL) are accumulated (+=). */
int sx_prologue_bwd(const float* dh, const float* x, int64_t B, int32_t N, int32_t C, const float* g, const float* b,
                    const float* pe, int32_t C0, int64_t pe_bstride, float posw, const float* mask, float drop_p,
                    uint64_t seed, const uint64_t* seed_dev, const float* stats, float* dx, float* dg, float* db, float* dpe,
                    float* dt_scratch /* [B*N*C] or NULL */, float* part, int64_t part_floats, void* stream);

/* Row softmax with the reference's conditional clamp and attention dropout (segtran_shared.py:578-580, :601-605):
 *   if (*amax > clip) S = clamp(S, -clip, clip);  P = dropout(softmax(S)).  S [R,L] fp32 (row stride lds),
 *   P [R,L] (row stride ldp), lse [R] = log-sum-exp of the (clamped) row, kept for backward.
 *   diag (optional, device float[2]): [0] = running max of *amax, [1] += 1 when the clamp fired — the module's
 *   max_attn / clamp_count counters (:575-587) without the reference's two .item() host syncs per call. */
int sx_softmax_fwd(const float* S, int64_t R, int32_t L, int64_t lds, const float* amax, float clip, float drop_p,
                   uint64_t seed, const uint64_t* seed_dev, void* P, int32_t p_dtype, int64_t ldp, int32_t round_tf32, float* lse, float* diag,
                   void* stream);
int sx_softmax_bwd(const float* dP, int64_t ldd, const float* S, int64_t lds, const float* lse, int64_t R, int32_t L,
                   const float* amax, float clip, float drop_p, uint64_t seed, const uint64_t* seed_dev, int64_t ldp_fwd, void* dS,
                   int32_t ds_dtype, int64_t ldo, int32_t round_tf32, void* stream);
/* The same with a sliding-window positional bias (segtran_shared.py:578-605): row r is query token r % L of a
 * self-attention (L == the grid's cell count, posbias->table != NULL):
 *   S' = clamp_if(S) + bias(q, .);  P = dropout(softmax(S')),  lse = log-sum-exp of S'.
 * Backward: P is recomputed from the raw S, the bias and lse; dS' = P * (g - sum P g) (g = the dropout-masked dP);
 * dS = dS' with the clamp mask, and dtable[o] += w * sum over rows of dS'[row, key(q, o)] — the gradient BEFORE the
 * clamp mask, so clamped elements still feed the table.  dtable [(2R+1)^pd] is accumulated in a fixed order through
 * `part` (no float atomics). */
int sx_softmax_posbias_fwd(const float* S, int64_t R, int32_t L, int64_t lds, const float* amax, float clip, float drop_p,
                           uint64_t seed, const uint64_t* seed_dev, void* P, int32_t p_dtype, int64_t ldp, int32_t round_tf32,
                           float* lse, float* diag, const sx_posbias* posbias, void* stream);
int sx_softmax_posbias_bwd(const float* dP, int64_t ldd, const float* S, int64_t lds, const float* lse, int64_t R, int32_t L,
                           const float* amax, float clip, float drop_p, uint64_t seed, const uint64_t* seed_dev, int64_t ldp_fwd,
                           void* dS, int32_t ds_dtype, int64_t ldo, int32_t round_tf32, const sx_posbias* posbias,
                           float* dtable, float* part, int64_t part_floats, void* stream);

/* LayerNorm with affine over rows, eps 1e-12 (first_norm_layer, segtran_shared.py:456).  stats [R,2]. */
int sx_layernorm_fwd(const float* x, int64_t R, int32_t C, const float* g, const float* b, void* y, int32_t y_dtype,
                     int32_t round_tf32, float* stats, void* stream);
int sx_layernorm_bwd(const float* dy, const float* x, int64_t R, int32_t C, const float* g, const float* stats,
                     void* dx, int32_t dx_dtype, int32_t round_tf32, float* dg, float* db, float* part, int64_t part_floats, void* stream);

/* MMPrivateOutput tail + LearnedSoftAggregate (segtran_shared.py:273-274, :318-325):
 *   Yn = LN_{g,b}(dropout(Y));  w = softmax_modes(Yn.ws + bs);  out = sum_m w_m Yn_m
 *   Y [B,M,N,F] fp32 -> out [B,N,F] fp32; stats [B,M,N,2]; wts [B,M,N]. */
int sx_ln_softaggr_fwd(const float* Y, int32_t B, int32_t M, int32_t N, int32_t F, const float* g, const float* b,
                       const float* ws, const float* bs, float drop_p, uint64_t seed, const uint64_t* seed_dev, float* out, float* stats,
                       float* wts, void* stream);
int sx_ln_softaggr_bwd(const float* dout, const float* Y, int32_t B, int32_t M, int32_t N, int32_t F, const float* g,
                       const float* b, const float* ws, float drop_p, uint64_t seed, const uint64_t* seed_dev, const float* stats,
                       const float* wts, void* dY, int32_t dy_dtype, int32_t round_tf32, float* dg, float* db,
                       float* dws, float* dbs, float* dscore_scratch /* [B*M*N] or NULL */, float* part, int64_t part_floats, void* stream);

/* LearnedSoftAggregate on its own (segtran_shared.py:318-325; the no-FFN branch :453 with M modes — the Polyformer layer):
 *   w = softmax_modes(x_m . ws + bs);  out = sum_m w_m x_m.   x [B,M,N,F] -> out [B,N,F], wts [B,M,N].
 * backward: dx [B,M,N,F] and dscore [B,M,N] (d ws = sum dscore x, d bs = sum dscore are left to the caller). */
int sx_softaggr_fwd(const float* x, int32_t B, int32_t M, int32_t N, int32_t F, const float* ws, const float* bs, float* out,
                    float* wts, void* stream);
int sx_softaggr_bwd(const float* dout, const float* x, int32_t B, int32_t M, int32_t N, int32_t F, const float* ws,
                    const float* wts, float* dx, float* dscore, void* stream);
/* dH = dropout'(dG) * gelu'(H)  (MMSharedMid backward, segtran_shared.py:243-245) */
int sx_gelu_bwd(const float* dG, const void* H, int32_t h_dtype, int64_t n, float drop_p, uint64_t seed, const uint64_t* seed_dev, void* dH,
                int32_t dh_dtype, int32_t round_tf32, void* stream);
/* dtype conversion / TF32 rounding of a flat buffer (weights once per step) */
int sx_convert(const void* x, int32_t x_dtype, int64_t n, void* y, int32_t y_dtype, int32_t round_tf32, void* stream);
/* hi = TF32(x), lo = TF32(x - hi) over a flat fp32 buffer: operand split of the 3-pass error-compensated TF32 products
 * (A_hi B_hi + A_lo B_hi + A_hi B_lo) used by the precision policy for the small / sensitive contractions */
int sx_split_tf32(const float* x, int64_t n, float* hi, float* lo, void* stream);
/* x [Z1][Z0][R][K] with element strides (sz1, sz0, sr, sk) -> out [Z1][Z0][R][3*Kp] contiguous, rows = [lo|hi|hi] (role 0,
 * the "A" operand) or [hi|lo|hi] (role 1, the "B" operand), segments zero-padded to Kp (multiple of 4) columns: ONE
 * sx_gemm launch over K' = 3*Kp on the two outputs is the 3-pass product A_hi B_hi^T + A_lo B_hi^T + A_hi B_lo^T */
int sx_split_tf32_cat(const float* x, int32_t Z1, int32_t Z0, int32_t R, int32_t K, int64_t sz1, int64_t sz0, int64_t sr,
                      int64_t sk, int32_t Kp, int32_t role, float* out, void* stream);
/* out[c] += sum_r X[r,c]   (bias gradients) */
int sx_colsum(const void* X, int32_t x_dtype, int64_t R, int32_t C, int64_t ld, float* out, float* part, int64_t part_floats, void* stream);
/* out[0] += sum_i x[i]*y[i]  and  y = alpha * (*alpha_dev) * x : a linear loss head for benchmarks / checksums */
int sx_dot(const float* x, const float* y, int64_t n, float* out, void* stream);
int sx_scale(const float* x, int64_t n, const float* alpha_dev, float alpha, float* y, void* stream);
/* out[z0][c] += sum_{z1,r} X[z1][z0][r][c]  (per-mode bias gradient of MMPrivateOutput in one launch) */
int sx_colsum_batched(const float* X, int32_t Z1, int64_t stride_z1, int32_t Z0, int64_t stride_z0, int64_t R, int32_t C,
                      int64_t ld, float* out, float* part, int64_t part_floats, void* stream);
/* y = a + b  (residual connection of MMSharedOutput, segtran_shared.py:305) */
int sx_add(const float* a, const float* b, int64_t n, float* y, void* stream);
/* out[r % out_mod] += sum_c X[r,c]  (class-bias gradient of the head: rows = (batch, class)) */
int sx_rowsum(const float* X, int64_t R, int64_t C, int64_t ld, int32_t out_mod, float* out, float* part, int64_t part_floats, void* stream);
/* batched transpose [Z,R,C] -> [Z,C,R] fp32 with output row pitch ldo >= R (floats; columns R..ldo-1 are not written):
   token flatten / scatter (segtran3d.py:328-330, :478-480, ldo = R) and the K-major GEMM operand copies (ldo = R rounded
   up to a multiple of 4, the 16-byte row pitch TMA needs) */
int sx_transpose(const float* in, int64_t Z, int32_t R, int32_t C, int32_t ldo, float* out, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Segmentation head, collapsed form (segtran3d.py:364-367, :381-386, :488-496; segtran2d.py:304-306,
 * :427, :435-436).  curr [B,Cf,V] fp32 channels-first, W [K,Cf], L / dL [B,K,V].
 * ------------------------------------------------------------------------------------------- */
int sx_head_contract_fwd(const float* curr, const float* W, const float* bias, int32_t B, int32_t Cf, int64_t V,
                         int32_t K, float* L, int32_t accumulate, void* stream);
int sx_head_contract_bwd_data(const float* dL, const float* W, int32_t B, int32_t Cf, int64_t V, int32_t K,
                              float* dcurr, void* stream);
int sx_head_contract_bwd_weight(const float* dL, const float* curr, int32_t B, int32_t Cf, int64_t V, int32_t K,
                                float* dW, void* stream);
/* class scores of the fused tokens, exact fp32: out[b,k,n] = sum_f W[k,f] vf[b,n,f]   (Wc . vfeat_fused) */
int sx_token_scores(const float* vf, const float* W, int32_t B, int32_t N, int32_t F, int32_t K, float* out,
                    void* stream);
/* and its data gradient: dvf[b,n,f] = sum_k dt[b,k,n] W[k,f]   (F % 4 == 0) */
int sx_token_scores_bwd(const float* dt, const float* W, int32_t B, int32_t N, int32_t F, int32_t K, float* dvf,
                        void* stream);
/* Out-FPN dropout head (--outdrop; segtran3d.py:372-396, :488-490; segtran2d.py:304-311, :427), which cannot be
 * collapsed: the dropout mask is per channel.  The dropped map X [B,F',D',HW] is never written:
 *   Ls[b,k,d',hw] = bc[k] + sum_f Wc[k,f] keep(b,f,d',hw) X[b,f,d',hw] / (1-p)
 * with X formed on the fly from src [B,Fs,Ds,HW] by the depth map `dmap`:
 *   SX_HEAD_DMAP_NONE   X = src                                    (F' = Fs, D' = Ds; 2-D heads pass Ds = 1)
 *   SX_HEAD_DMAP_INTERP X = linear resize of src along depth to D' = Dk*Ds (F.interpolate, align_corners=False)
 *   SX_HEAD_DMAP_UNFOLD X[b,f,j*Ds+i,hw] = src[b,f*Dk+j,i,hw]      (out_fpn_upsampleD's reshape; F' = Fs/Dk, D' = Dk*Ds)
 * keep(e) = the counter-based dropout hash of the flat index e of the element in [B,F',D',HW] layout with the effective
 * seed seed + *seed_dev (CUDA-graph safe), p in [0, 1).  Wc [K][F'], bc [K] (optional); any K (classes are processed
 * in chunks of 4).  Ls / dLs: [B][K][D'][HW].
 * fwd writes Ls.  bwd writes dsrc [B,Fs,Ds,HW] (or adds to it when accumulate) in gather form and ADDS
 * dWc[k,f] = sum keep dLs X / (1-p) into dWc through ordered per-CTA slots of `part`; the class-bias gradient is the
 * row sum of dLs (sx_rowsum).  No float atomics: two runs give the same bits. */
enum { SX_HEAD_DMAP_NONE = 0, SX_HEAD_DMAP_INTERP = 1, SX_HEAD_DMAP_UNFOLD = 2 };
typedef struct {
  const float* src;
  int32_t B, Fs, Ds;
  int32_t Fo;                    /* F' */
  int64_t HW;
  int32_t Dk;                    /* D_pool_K */
  int32_t dmap;                  /* SX_HEAD_DMAP_* */
  int32_t K;
  int32_t _pad;
  const float* Wc;
  const float* bc;
  float p;
  uint32_t _pad2;
  uint64_t seed;
  const uint64_t* seed_dev;
  float* part;
  int64_t part_floats;
} sx_head_dropout_args;
int sx_head_dropout_fwd(const sx_head_dropout_args* args, float* Ls, void* stream);
int sx_head_dropout_bwd(const sx_head_dropout_args* args, const float* dLs, float* dsrc, int32_t accumulate, float* dWc,
                        void* stream);
/* -------------------------------------------------------------------------------------------
 * FPN pyramid stage (SURVEY.md section 8 row f.1; segtran3d.py:299-313, :347-359, segtran2d.py:244-300):
 *   curr <- GroupNorm_G( conv1x1(curr) + bias + upsample(higher) )
 * conv1x1 + bias + add is ONE sx_gemm launch on the channels-first tensors (A = W [Cout x Cin] broadcast over the batch,
 * B = x[b] read as an MN-major [V x Cin] operand, bias mode SX_BIAS_M, addend = the upsampled level); the upsampling is
 * sx_resize_axis_fwd per axis; GroupNorm is below.  x, y, dy, dx: [B, C, V] fp32.  csum: [B*C*2] double workspace,
 * stats: [B*G*2] (mean, rstd) kept for the backward, coef: [B*G*2] workspace.  dgamma/dbeta are accumulated into.
 * ------------------------------------------------------------------------------------------- */
int sx_groupnorm_fwd(const float* x, int32_t B, int32_t C, int64_t V, int32_t G, const float* gamma, const float* beta,
                     float eps, double* csum, float* stats, float* y, int32_t round_tf32, void* stream);
int sx_groupnorm_bwd(const float* dy, const float* x, int32_t B, int32_t C, int64_t V, int32_t G, const float* gamma,
                     const float* stats, double* csum, float* coef, float* dx, float* dgamma, float* dbeta, void* stream);

/* -------------------------------------------------------------------------------------------
 * Training-step tail (SURVEY.md section 8 row f.2): segmentation loss and BertAdam on flat buckets.
 * Everything the step needs (loss scalars, clip coefficients, scheduled learning rates, the step
 * counter) is produced and consumed on the device, so the step can be captured in a CUDA graph.
 * ------------------------------------------------------------------------------------------- */
/* loss = (1-dice_w) * BCEWithLogits(pos_weight)(logits, mask) + dice_w * sum_{k>=1} class_w[k] * dice_loss_indiv(sigmoid(logits[:,k]), mask[:,k])
 * (train3d.py:731-756, utils/losses.py:47-60).  logits, mask: [B,K,V] fp32 (mask n-hot).  pos_weight, class_w: [K] or NULL (= ones).
 * sums: [B*K*4] double workspace (zeroed here); out3 = {loss, ce, dice}; coef: [B*K*2] Dice gradient coefficients for the backward. */
int sx_seg_loss_fwd(const float* logits, const float* mask, int32_t B, int32_t K, int64_t V, const float* pos_weight,
                    const float* class_w, float dice_w, double* sums, float* out3, float* coef, void* stream);
/* dlogits = (*gout or 1) * d loss / d logits; ce_scale = (1-dice_w) / (B*K*V); coef from sx_seg_loss_fwd */
int sx_seg_loss_bwd(const float* logits, const float* mask, int32_t B, int32_t K, int64_t V, const float* pos_weight,
                    const float* coef, float ce_scale, const float* gout, float* dlogits, void* stream);
/* One optimiser step of the reference's BertAdam (optimization.py:90-164) preceded by the global gradient-norm clip of
 * train3d.py:760-761, on flat fp32 buckets p, g, m, v.  The buckets are cut into segments (<= a few thousand elements of
 * ONE parameter each): seg_param / seg_off / seg_len [nseg].  lr, wd: per-parameter [P].  schedule: SX_SCHED_*; t_total = -1
 * disables the schedule.  step: device counter (read, then incremented).  sumsq [P] double, coef [P], lr_eff [P]: device
 * workspaces.  total_norm: optional device float (the pre-clip global norm).  A parameter whose gradient is exactly zero is
 * left untouched (the reference skips p.grad is None: never-used parameters).  p_tf32 (optional): a second parameter
 * buffer that receives the TF32-rounded new values, so the next forward needs no per-weight rounding pass. */
enum { SX_SCHED_WARMUP_LINEAR = 0, SX_SCHED_WARMUP_CONSTANT = 1 };
int sx_adam_step(float* p, float* p_tf32, const float* g, float* m, float* v, const int32_t* seg_param, const int64_t* seg_off,
                 const int32_t* seg_len, int32_t nseg, int32_t P, const float* lr, const float* wd, double b1, double b2,
                 double eps, float grad_clip, float max_grad_norm, float warmup, int64_t t_total, int32_t schedule,
                 int64_t* step, double* sumsq, float* coef, float* lr_eff, float* total_norm, void* stream);

/* 1-D linear resampling (align_corners=False) of x viewed as [outer, Lin, inner] -> [outer, Lout, inner];
 * F.interpolate(mode='bilinear'|'trilinear') == one pass per axis. */
int sx_resize_axis_fwd(const float* x, int64_t outer, int32_t Lin, int32_t Lout, int64_t inner, float* y,
                       int32_t accumulate, void* stream);
int sx_resize_axis_bwd(const float* dy, int64_t outer, int32_t Lin, int32_t Lout, int64_t inner, float* dx,
                       void* stream);
/* Token-grid resampling of the mince transformer (segtran_shared.py:45-66): linear / bilinear / trilinear interpolation
 * (align_corners=False) of token-major rows on a row-major grid, all axes in one launch.  A 2-D grid passes a leading
 * axis of extent 1 with ratio 1.  ratio[a]: source cells per output cell, as PyTorch computes it: 1/scale_factor when
 * F.interpolate is given a scale factor, Lin/Lout when it is given a size; 1/ratio <= 24.
 * Element (b, g, cell, c) of x / dx is at [b*bs_in + g*gs_in + cell*ld_in + c], of y / dy at
 * [b*bs_out + g*gs_out + cell*ld_out + c]; c < w is the channel window (pass its first column as the pointer).
 * fwd: y = resample(x) for c < w, columns [w, w_pad) of y are written as 0; round_tf32 rounds y for a GEMM consumer.
 * bwd: the adjoint in gather form (every input cell sums, in a fixed order, the output cells that read it; no atomics):
 *   dx = (dx +) resample^T(dy) for c < w; columns [w, w_pad) of dx are written as 0 unless accumulating. */
typedef struct {
  int32_t lin[3];
  int32_t lout[3];
  float ratio[3];
} sx_resample_grid;
int sx_resize_tokens_fwd(const float* x, int64_t bs_in, int64_t gs_in, int64_t ld_in, float* y, int64_t bs_out,
                         int64_t gs_out, int64_t ld_out, int32_t B, int32_t G, int32_t w, int32_t w_pad,
                         const sx_resample_grid* grid, int32_t round_tf32, void* stream);
int sx_resize_tokens_bwd(const float* dy, int64_t bs_out, int64_t gs_out, int64_t ld_out, float* dx, int64_t bs_in,
                         int64_t gs_in, int64_t ld_in, int32_t B, int32_t G, int32_t w, int32_t w_pad,
                         const sx_resample_grid* grid, int32_t accumulate, void* stream);
/* tiny strided fp32 GEMM on CUDA cores (class-dimension products of the collapsed head):
 *   C[z](m,n) (+)= alpha * sum_k A[z](m,k) B[z](k,n), element strides given explicitly */
int sx_sgemm_small(const float* A, const float* B, float* C, int32_t M, int32_t N, int32_t K, int64_t sam, int64_t sak,
                   int64_t sbk, int64_t sbn, int64_t scm, int64_t scn, int32_t Z, int64_t saz, int64_t sbz, int64_t scz,
                   float alpha, int32_t accumulate, void* stream);

/* -------------------------------------------------------------------------------------------
 * Sliding-window inference post-process (SURVEY.md section 8 row f.4; code/test_util3d.py:93-184):
 * sx_sw_accumulate: preds[k][window] += sigmoid(scores[k]), cnt[window] += 1 for one patch ([K][dx][dy][dz] scores, window
 *   origin (x0,y0,z0) in the [K][H][W][D] accumulators)                                              (test_util3d.py:155-159)
 * sx_sw_finalize: preds /= cnt; brats: make_brats_pred_consistent(is_conservative=False) (datasets3d.py:53-59), hard[1:] =
 *   preds >= 0.5, hard[0] = no class fired (hard is [K][V]); otherwise hard[0..V) = argmax_k as a float class index.
 * ------------------------------------------------------------------------------------------- */
int sx_sw_accumulate(const float* scores, int32_t K, int32_t dx, int32_t dy, int32_t dz, float* preds, float* cnt,
                     int32_t H, int32_t W, int32_t D, int32_t x0, int32_t y0, int32_t z0, void* stream);
int sx_sw_finalize(float* preds, const float* cnt, int32_t K, int64_t V, int32_t brats, float* hard, void* stream);

/* -------------------------------------------------------------------------------------------
 * Evaluation metrics of a case (csrc/sx_metrics.cu; code/test_util3d.py:186-215 calculate_metric_percase and medpy 0.4's
 * dc / jc / asd / assd / hd / hd95 with unit voxel spacing and connectivity 1).  The classes of a case are the leading
 * index of [K][n0][n1][n2] uint8 masks (non-zero = foreground, n2 contiguous; a 2-D mask has n0 = 1), so a case costs
 * the same launches for any K.  Distances are exact: every one is sqrt of an integer squared distance d2, and the
 * statistics are read from integer histograms over d2 (bins 0 .. sum (n_i - 1)^2).
 * sx_mask_counts: counts[k*ldc + {0,1,2,3}] = |A|, |B|, |A and B|, |A or B| of class k (int64; written).
 * sx_surface: border = X and not erode(X), the erosion with the 2*ndim axis neighbours and a background outside the volume.
 * sx_edt_sq: dist[k][v] = the squared Euclidean distance from voxel v to the nearest non-zero voxel of border[k] (int32;
 *   2^28 when border[k] is empty).  Extents in [1, 4096] with sum (n_i - 1)^2 < 2^26.
 * sx_surface_hist: hist[k*ldh + d2] = the number of non-zero voxels of src_border[k] with dist d2 (uint32; written).
 * sx_surface_stats: hist[k*ldh + {0, nbins}] are the histograms of the two directions of class k (A's border on B's
 *   transform, then B's on A's); out[k*ldo + 0..7] (fp64) = n of each direction, the mean distance of each (asd, 0 when
 *   empty), the maximum of each, numpy's linear 95th percentile over both directions together (hd95), and n of both.
 *   The mean's fp64 sum has one fixed order: two runs give the same bits.
 * ------------------------------------------------------------------------------------------- */
int sx_mask_counts(const uint8_t* A, const uint8_t* B, int32_t K, int64_t V, int64_t* counts, int64_t ldc, void* stream);
int sx_surface(const uint8_t* X, int32_t K, int32_t ndim, int32_t n0, int32_t n1, int32_t n2, uint8_t* border, void* stream);
int sx_edt_sq(const uint8_t* border, int32_t K, int32_t n0, int32_t n1, int32_t n2, int32_t* dist, void* stream);
int sx_surface_hist(const uint8_t* src_border, const int32_t* dist, int32_t K, int64_t V, int32_t nbins, uint32_t* hist,
                    int64_t ldh, void* stream);
int sx_surface_stats(const uint32_t* hist, int32_t K, int32_t nbins, int64_t ldh, double* out, int64_t ldo, void* stream);

/* debug knobs for bring-up (descriptor field overrides); not part of the stable ABI */
int sx_gemm_debug_set(const char* key, int64_t value);

#ifdef __cplusplus
}
#endif
#endif /* SEGTRAN_B200_H_ */
