/*
 * vilbert_b200.h — C ABI of libvilbert_b200.so: the sm_90a kernels behind the ViLBERT two-stream
 * co-attentional encoder hot path (reference: vilbert/vilbert.py:396-1107 BertLayer / BertImageLayer /
 * BertConnectionLayer / BertEncoder, :320-367 + :1409-1432 embeddings, :1110-1137 poolers,
 * :1140-1258 + :1638-1722 heads).
 *
 * The reference has no FFI of its own (it is pure PyTorch, SURVEY.md §8b); every entry point below
 * cites the reference nn.Module / expression whose arithmetic it replaces. The Python host
 * (vilbert-multi-task_b200/) binds these with ctypes — see INTEGRATION.md.
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless stated otherwise;
 *   - the caller owns every buffer; the library never allocates or frees device memory;
 *   - every launch is asynchronous on the caller-supplied stream (cudaStream_t passed as void*);
 *   - every function returns a vb_status (0 = ok); vb_last_error() gives a message for the calling
 *     thread; no C++ exception crosses the boundary;
 *   - "bf16" buffers are raw uint16 bfloat16; "f32" are IEEE binary32; matrices are row-major with
 *     an explicit leading dimension in ELEMENTS.
 */
#ifndef VILBERT_B200_H_
#define VILBERT_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int vb_status;
enum {
  VB_OK = 0,
  VB_ERR_INVALID = 1,     /* bad shape / alignment / argument                     */
  VB_ERR_UNSUPPORTED = 2, /* device is not sm_90 or an unsupported configuration  */
  VB_ERR_CUDA = 3         /* a CUDA runtime / driver call failed                  */
};

enum { VB_ACT_NONE = 0, VB_ACT_GELU = 1, VB_ACT_RELU = 2, VB_ACT_DGELU = 3 };

/* Dropout descriptor (nn.Dropout at vilbert.py:365,443,472,515,604,631,676,778,800,848-851,1233,1430,1678-1695).
 * Masks are not stored: keep(element) = hash32(index ^ hash32(site + step * 0x9E3779B9)) >= p * 2^32 with
 * hash32 = lowbias32 (x^=x>>16; x*=0x7feb352d; x^=x>>15; x*=0x846ca68b; x^=x>>16), kept values scaled by 1/(1-p).
 * `step` is a device uint32 bumped once per training step; `site` names the dropout layer; `index` is the
 * row-major element index of the tensor the reference applies nn.Dropout to (mod 2^32). step == NULL or p == 0
 * disables dropout (the reference's eval mode). */
typedef struct vb_dropout_site {
  const uint32_t* step;
  uint32_t site;
  float p;
} vb_dropout_site;
/* The descriptor the row-wise kernels take (LayerNorms, residual LayerNorms, small linear heads): a vb_dropout_site with an
 * optional packed-row -> padded-row map (int32 [rows], device; NULL: none). With it, element (r, c) of a row-indexed site
 * [rows, H] draws the mask of element (row_map[r], c) of the padded tensor, so a packed plan (Plan(packed=...)) draws the padded
 * plan's masks. The GEMM epilogue and attention carry a vb_dropout_site: attention indexes its elements at padded coordinates by
 * itself, and no packed plan uses a GEMM-epilogue dropout. */
typedef struct vb_dropout {
  const uint32_t* step;
  uint32_t site;
  float p;
  const int32_t* row_map;
} vb_dropout;

/* ABI version of this header (bumped on incompatible change). v3: vb_gemm_args has no CTA-pair field and no smem descriptor
 * overrides, and vb_gemm_plan returns (block_n, split_k). v4: vb_adamw_group carries one_minus_beta1 / one_minus_beta2. */
int vb_version(void);
/* Message for the last non-OK status returned on this thread ("" if none). */
const char* vb_last_error(void);
/* Number of SMs / compute capability (major*10+minor) of the current device. */
vb_status vb_device_info(int* sm_count, int* cc);

/* ------------------------------------------------------------------------------------------------
 * Dense contraction on the Hopper tensor cores (TMA -> 128B-swizzled smem -> wgmma -> fp32 registers).
 *   D[M,N] = alpha * sum_k A(m,k) * B(n,k)   followed by the fused epilogue
 *   v = D (+ bias[n]); act; (+ residual[m,n]); -> out_f32 / out_bf16
 * Replaces every nn.Linear on the path (vilbert.py:410-412,466,492,509 text; :553-555,625,653,670
 * image; :716-725,830,837,865-869 connection; :1116,1131 poolers; heads :1143,1163,1183,1250,1714-1719)
 * and their autograd (dgrad / wgrad):
 *   forward   y = x W^T + b          A = x  [M,K] k-major,  B = W  [N,K] k-major
 *   dgrad     dx = dy W              A = dy [M,N'] k-major, B = W  [N',K'] stored [red, out] -> b_mn_major
 *   wgrad     dW = dy^T x            A = dy [red, out] -> a_mn_major, B = x [red, in] -> b_mn_major
 * Operand storage:
 *   k-major  : element (row r of the M/N extent, reduction index k) at ptr[r*ld + k]
 *   mn-major : element (r, k) at ptr[k*ld + r]
 * Requirements: ld % 8 == 0, base pointers 16-byte aligned. M, N, K arbitrary (TMA zero-fills the
 * edges, stores are predicated).
 * act: VB_ACT_GELU = erf GELU (vilbert.py:111-117; erf by Abramowitz-Stegun 7.1.26, |err| < 5e-7), out_pre receives
 *      gelu'(pre-activation) as bf16 (what the backward needs); VB_ACT_DGELU multiplies by aux[m,n] (that buffer);
 * atomic_out: accumulate into out_f32 with red.global.add (needed when split_k > 1).
 */
typedef struct vb_gemm_args {
  int32_t M, N, K;
  const void* A;      /* bf16 */
  int64_t lda;
  int32_t a_mn_major;
  const void* B;      /* bf16 */
  int64_t ldb;
  int32_t b_mn_major;
  float alpha;
  const float* bias;     /* [N] or NULL */
  const float* residual; /* f32 [M,N] or NULL; may alias out_f32 */
  int64_t ld_res;
  const void* aux;       /* bf16 [M,N] saved gelu'(pre) for VB_ACT_DGELU, else NULL */
  int64_t ld_aux;
  int32_t act;
  float* out_f32;        /* or NULL */
  int64_t ld_out_f32;
  void* out_bf16;        /* or NULL */
  int64_t ld_out_bf16;
  void* out_pre;         /* bf16 gelu'(pre-activation) (GELU) or NULL */
  int64_t ld_out_pre;
  int32_t atomic_out;    /* 0 store, 1 red.add into out_f32, VB_GEMM_PARTIALS: split s stores into rows [s*M, s*M + M) of out_f32 */
  float* out_colsum;     /* [N] or NULL: += column sums of the epilogue value before the residual add (bias gradients) */
  vb_dropout_site dropout;    /* applied to the epilogue value before the residual add (index m*N + n): LN(dropout(dense(x)) + res) */
  int32_t split_k;       /* >= 1; > 1 requires atomic_out and no act / bf16 outputs */
  int32_t block_n;       /* 0 = auto, else 128 or 256 */
  int32_t max_ctas;      /* 0 = one persistent CTA per SM */
  void* dbg_timeline;    /* NULL, or u64 [grid][10]: per-CTA clock64 / globaltimer stamps (development only) */
  /* ---- ABI v2: 16-bit operand formats and split precision -------------------------------------------------
   * Forward operands (activations, weights) are IEEE fp16 (11 significant bits; the reference's own reduced
   * precision mode is fp16, train_concap.py:504-505), gradient operands are bf16 (range). a_fp16 / b_fp16 / out_fp16:
   * 0 = bf16, 1 = fp16 (out_fp16 is the format of out_bf16 and out_lo). A and B must have the SAME format (wgmma takes
   * one operand type for both), so the backward contractions (dy bf16) read bf16 copies of the forward operands: out_b16 (same ld as out_bf16) is an
   * additional, always-bf16 copy of the 16-bit output, written by the forward GEMM for the weight-gradient GEMM.
   * Split precision ("fp32 parity mode", 1e-3): an operand x is stored as hi = fp16(x), lo = fp16(x - hi); with
   * A_lo and/or B_lo given the contraction is A.B + A_lo.B + A.B_lo (three passes over K into the same register
   * accumulator; the lo.lo term, 2^-22 relative, is dropped). A_lo / B_lo use lda / ldb and the major of A / B.
   * out_lo (same ld as out_bf16) receives the low part of the value written to out_bf16. */
  int32_t a_fp16, b_fp16, out_fp16;
  const void* A_lo;
  const void* B_lo;
  void* out_lo;
  void* out_b16;
} vb_gemm_args;

vb_status vb_gemm_bf16(const vb_gemm_args* args, void* stream);

/* Host-only query: the tile configuration vb_gemm_bf16 would use for `args` (fields block_n / split_k that are non-zero
   in `args` are honoured) on a device with `sm_count` SMs (0 = the current CUDA device). No GPU work, no device
   needed when sm_count > 0; only the shape, layout, epilogue and output fields of `args` are read. */
vb_status vb_gemm_plan(const vb_gemm_args* args, int32_t sm_count, int32_t* block_n, int32_t* split_k);

/* ------------------------------------------------------------------------------------------------
 * Fused attention:  P = softmax(Q K^T * scale + mask[b, key]),  O = P V, heads merged in the output.
 * Replaces BertSelfAttention.forward (vilbert.py:424-460), BertImageSelfAttention.forward (:571-619,
 * dynamic_attention off) and both directions of BertBiAttention.forward (:771-809), including the
 * transpose_for_scores / permute().contiguous() layout ops (:416-422, :447-449).
 *   Q: bf16, element (b, i, h, d) at Q[(b*Nq + i)*ldq + h*D + d]   (read in place from a packed QKV buffer)
 *   K, V: same with Nk / ldk / ldv;  O: bf16 [B*Nq, H*D] with ldo
 *   mask: f32 [B, Nk] additive (0 / -10000, vilbert.py:1350-1362) or NULL
 *   lse:  f32 [B, H, Nq] row log-sum-exp in the log2 domain (saved for backward; may be NULL in fwd)
 * Backward recomputes P from lse: needs dO (bf16), writes dQ/dK/dV (bf16, same indexing as Q/K/V with
 * their own ld) and uses delta [B, H, Nq] f32 as scratch. D in {16, 32, 64, 128}.
 * Sequence limits: the forward streams keys through shared memory in chunks when the K / V panels do not fit. The backward runs
 * one fused kernel for Nq, Nk <= 128 and D >= 32; otherwise two kernels that keep whole panels resident (227 KiB of shared
 * memory): for D = 128 / 64 / 32 / 16 they take Nk <= 320 / 704 / 1344 / 2240 when dQ is requested or dropout is on, and
 * Nq <= 320 / 704 / 1280 / 2176 when dK / dV are requested. Past these vb_attention_bwd returns VB_ERR_UNSUPPORTED and launches
 * nothing.
 * Partial backward: dQ may be NULL (dK / dV only), or dK and dV may both be NULL (dQ only); what is written is bitwise what the
 * full backward writes there. dK without dV (or the reverse) and all three NULL return VB_ERR_INVALID. A bias sum follows its
 * gradient: dbias_q is ignored when dQ is NULL, dbias_k / dbias_v when dK / dV are.
 */
typedef struct vb_attn_args {
  int32_t B, H, Nq, Nk, D;
  const void* Q; int64_t ldq;
  const void* K; int64_t ldk;
  const void* V; int64_t ldv;
  const float* mask;
  float scale;
  void* O; int64_t ldo;
  float* lse;
  const void* dO; int64_t lddo;
  void* dQ; int64_t lddq;
  void* dK; int64_t lddk;
  void* dV; int64_t lddv;
  float* delta;
  /* optional (backward): += column sums of dQ / dK / dV, f32 [H*D] each — the bias gradients of the projections */
  float* dbias_q; float* dbias_k; float* dbias_v;
  vb_dropout_site dropout;   /* on the probabilities; element index ((b*H + h)*Nq + q)*Nk + k */
  /* ---- ABI v2. qkv_fp16: Q, K, V and O are fp16 (forward operands) instead of bf16; dO / dQ / dK / dV are always bf16
   * (the backward converts its Q / K / V panels to bf16 in shared memory). Split precision (forward only): with Q_lo,
   * K_lo, V_lo given (same ld and indexing as Q / K / V) S = Q K^T + Q_lo K^T + Q K_lo^T and O = P V + P_lo V + P V_lo
   * with P split in registers; O_lo (same ld as O) receives the low part of O. */
  int32_t qkv_fp16;
  const void* Q_lo; const void* K_lo; const void* V_lo;
  void* O_lo;
  void* O_b16;   /* forward: optional always-bf16 copy of O (same ldo): the operand of the out-projection's weight gradient.
                    backward: if given, delta = rowsum(dO o O) reads this copy (consistent with the bf16 products of the backward) */
  /* Packed rows (varlen), all four or none (int32 [B] each, device): sample b's queries are rows q_off[b] + i, i < q_len[b], of Q /
   * O / dO / dQ, and its keys rows k_off[b] + j, j < k_len[b], of K / V / dK / dV. Keys past k_len are excluded, so mask must be NULL;
   * every length must be >= 1. Nq / Nk stay the maxima: the grid, lse / delta [B, H, Nq] and the dropout element index
   * ((b*H + h)*Nq + i)*Nk + j remain at padded coordinates, so a packed step draws the padded step's masks. Rows of no sample are not
   * written. NULL: the padded layout (rows b*Nq + i, b*Nk + j). vb_attention_probs refuses packed rows. */
  const int32_t* q_off; const int32_t* q_len; const int32_t* k_off; const int32_t* k_len;
} vb_attn_args;

vb_status vb_attention_fwd(const vb_attn_args* args, void* stream);
vb_status vb_attention_bwd(const vb_attn_args* args, void* stream);
/* Attention-probability export of config.visualization (attn_data["attn"], vilbert.py:451-458, 610-617, 813-821):
 * probs f32 [B, H, Nq, Nk] = softmax(Q K^T * scale + mask) from the Q / K / mask / scale fields of args (eval mode: no dropout). */
vb_status vb_attention_probs(const vb_attn_args* args, float* probs, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Row-wise (HBM-bound) kernels. One warp per row, 128-bit accesses.
 */

/* BertLayerNorm.forward (vilbert.py:304-317): biased variance, eps inside the sqrt, affine after.
 * x f32 [M,H] (ldx); writes y as f32 and/or bf16 (either may be NULL; both use ldy) and the row
 * statistics mean/rstd [M] (may be NULL). H % 4 == 0, H <= 2048. */
vb_status vb_layernorm_fwd(const float* x, int64_t ldx, const float* gamma, const float* beta, float eps,
                           float* y_f32, void* y_bf16, int64_t ldy, float* mean, float* rstd,
                           int32_t M, int32_t H, const vb_dropout* out_dropout /* may be NULL: dropout(LN(x)), embeddings */,
                           int32_t y_fp16 /* format of y_bf16 / y_lo: 0 = bf16, 1 = fp16 */,
                           void* y_lo /* NULL, or the split-precision low part of y_bf16 (same ldy) */,
                           void* y_b16 /* NULL, or an always-bf16 copy of y (same ldy): weight-gradient operand */, void* stream);
/* Autograd of the above. dx as f32 and/or bf16; dgamma/dbeta are ACCUMULATED (atomics) and may be NULL.
 * If gelu_pre (bf16 [M,H], the GELU derivative saved by the forward GEMM) is given, dx_bf16 is multiplied by it — the
 * Linear -> GELU -> LayerNorm head transforms (vilbert.py:1152-1156, 1172-1176, 1714-1718).
 * dbias (may be NULL) += column sums of the dx value written to dx_bf16 (or of dx when dx_bf16 is NULL): the
 * bias gradient of the Linear that produced the LayerNorm input. */
vb_status vb_layernorm_bwd(const float* dy, int64_t lddy, const float* x, int64_t ldx, const float* gamma,
                           const float* mean, const float* rstd, float* dx_f32, void* dx_bf16, int64_t lddx,
                           const void* gelu_pre, int64_t ld_pre, float* dgamma, float* dbeta, float* dbias,
                           int32_t M, int32_t H,
                           const vb_dropout* out_dropout /* NULL or the mask applied to this LN's OUTPUT in forward: dy is masked first */,
                           const vb_dropout* in_dropout  /* NULL or the mask applied to the dense output feeding this LN: dx_bf16 / dbias are masked */,
                           void* stream);

/* The LayerNorm of the residual stream with the residual add fused in: LN(x), x = dropout(d) + residual (BertSelfOutput /
 * BertOutput / BertBiOutput, vilbert.py:470-474, 513-517, 844-855). d f32 [M,H] is the dense output alpha*acc + bias that
 * vb_gemm_bf16 stores without a residual; x is formed exactly as that GEMM's epilogue forms it with `residual` and `dropout`
 * (mask index row*H + col, then one fp32 add), so both paths give the same bits. d and residual share ld (== H when dropout is
 * set). x_out: NULL, or d itself: x is written over d (what vb_add_layernorm_bwd's x then reads). Outputs as vb_layernorm_fwd. */
vb_status vb_add_layernorm_fwd(const float* d, const float* residual, int64_t ld, const vb_dropout* dropout /* may be NULL */,
                               float* x_out, const float* gamma, const float* beta, float eps, float* y_f32, void* y_bf16, int64_t ldy,
                               float* mean, float* rstd, int32_t M, int32_t H, int32_t y_fp16, void* y_lo, void* y_b16, void* stream);
/* vb_layernorm_bwd of dy + dy2 (both f32 [M,H], pitch lddy): the gradient of the LayerNorm output arrives in two parts, the one a
 * dgrad GEMM wrote and the residual-path gradient that GEMM's epilogue would otherwise have added (same fp32 addition). */
vb_status vb_add_layernorm_bwd(const float* dy, const float* dy2, int64_t lddy, const float* x, int64_t ldx, const float* gamma,
                               const float* mean, const float* rstd, float* dx_f32, void* dx_bf16, int64_t lddx,
                               const void* gelu_pre, int64_t ld_pre, float* dgamma, float* dbeta, float* dbias,
                               int32_t M, int32_t H, const vb_dropout* out_dropout, const vb_dropout* in_dropout, void* stream);

/* fp32 -> 16-bit casts: flat (weights shadow, region-feature ingest; bf16 or fp16, optionally hi + lo) and 2-D with independent leading
 * dimensions and a scale (pads operands whose row length is not a multiple of 8). */
vb_status vb_cast_f32_to_bf16(const float* src, void* dst, int64_t n, int32_t fp16 /* 0 = bf16, 1 = fp16 */,
                              void* dst_lo /* NULL or split-precision low part */, void* dst_b16 /* NULL or always-bf16 copy */,
                              void* stream);
vb_status vb_cast2d_f32_to_bf16(const float* src, int64_t lds, void* dst, int64_t ldd, int32_t rows, int32_t cols,
                                float scale, void* stream);

/* BertEmbeddings.forward before its LayerNorm (vilbert.py:346-362): out[b,p,:] = word[ids] + pos[arange] +
 * type[token_type_ids]; if task_ids != NULL the task embedding row is inserted at position 1 (no pos/type
 * term) and the output has Nt+1 rows per sample. ids / token_type_ids [B,Nt] int64, task_ids [B] int64.
 * Backward scatter-adds into the tables (word row 0 = padding_idx gets no gradient, :328-330); any of dword / dpos / dtype /
 * dtask may be NULL (a frozen table: nothing is written to it). */
vb_status vb_embed_text_fwd(const int64_t* ids, const int64_t* token_type_ids, const int64_t* task_ids,
                            const float* word, const float* pos, const float* type, const float* task,
                            float* out, int32_t B, int32_t Nt, int32_t H, void* stream);
vb_status vb_embed_text_bwd(const float* dout, const int64_t* ids, const int64_t* token_type_ids,
                            const int64_t* task_ids, float* dword, float* dpos, float* dtype, float* dtask,
                            int32_t B, int32_t Nt, int32_t H, void* stream);

/* BertImageEmbeddings.image_location_embeddings (vilbert.py:1416,1424): out[m,:] = loc[m,:5] W^T + b,
 * W [H,5]; consumed as the residual of the 2048 -> Hv region-feature GEMM. Backward accumulates dW, db (either may be NULL). */
vb_status vb_loc_proj_fwd(const float* loc, const float* W, const float* b, float* out, int32_t M, int32_t H, void* stream);
vb_status vb_loc_proj_bwd(const float* dy, const float* loc, float* dW, float* db, int32_t M, int32_t H, void* stream);
/* Input gradient of the box projection: dx[m,:5] = dy[m,:] W (written, not accumulated), dy [M,H] fp32, W [H,5]. Fixed-order
 * reductions without atomics: the result does not depend on the launch. */
vb_status vb_loc_proj_dx(const float* dy, const float* W, float* dx, int32_t M, int32_t H, void* stream);

/* Bias gradients: out[n] += sum_m X[m,n]; X is bf16 (is_bf16 != 0) or f32, [M,N] with ld. */
vb_status vb_colsum(const void* X, int32_t is_bf16, int64_t ld, float* out, int32_t M, int32_t N, void* stream);

/* Linears with 1..8 outputs (vil_logit, vil_tri_prediction, vision_logit, linguisic_logit,
 * bi_seq_relationship, the 2-way output of vil_binary_prediction; vilbert.py:1231,1620-1628,1684-1695):
 * y[m,j] = x[m,:] . W[j,:] + b[j] (+ row_addend[m]). Backward: dx (=, or += when accumulate_dx),
 * dW and db ACCUMULATED; each of dx / dW / db may be NULL (not computed). */
vb_status vb_small_linear_fwd(const float* x, int64_t ldx, const float* W, const float* b, const float* row_addend,
                              float* y, int32_t M, int32_t K, int32_t N,
                              const vb_dropout* in_dropout /* NULL or dropout applied to x first (index m*K + k; needs ldx == K) */, void* stream);
vb_status vb_small_linear_bwd(const float* dy, const float* x, int64_t ldx, const float* W, float* dx, int64_t lddx,
                              int32_t accumulate_dx, float* dW, float* db, int32_t M, int32_t K, int32_t N,
                              const vb_dropout* in_dropout, void* stream);

/* pooled_output = pooled_t (*|+) pooled_v (fusion_method, vilbert.py:1677-1682, 1236-1241); backward
 * ACCUMULATES into da / db (either may be NULL). */
vb_status vb_fuse_pooled_fwd(const float* a, const float* b, float* out_f32, void* out_bf16, int64_t n, int32_t mul,
                             const vb_dropout* dropout /* NULL or dropout on the fused vector (index i) */,
                             int32_t out_fp16, void* out_lo /* format / split-precision low part of out_bf16 */,
                             void* out_b16 /* NULL or always-bf16 copy */, void* stream);
vb_status vb_fuse_pooled_bwd(const float* d, const float* a, const float* b, float* da, float* db, int64_t n, int32_t mul,
                             const vb_dropout* dropout, void* stream);
/* ReLU backward of the poolers (vilbert.py:1121,1136): dx = dy * (y > 0). */
vb_status vb_relu_bwd(const float* dy, const float* y, void* dx_bf16, float* dx_f32, int64_t n, void* stream);
/* y += alpha * x (f32): merges gradient contributions. */
vb_status vb_axpy_f32(const float* x, float* y, int64_t n, float alpha, void* stream);

/* VQA objective (task_utils.py:325-327): loss = mean(BCEWithLogits(logits, target)) * cols, written to
 * *loss (device scalar); dlogits = grad_scale * d loss / d logits as f32 and/or bf16 (ld). */
vb_status vb_bce_logits_loss(const float* logits, const float* target, float* loss, float* dlogits_f32, void* dlogits_bf16,
                             int64_t ld_dlogits_bf16, int32_t rows, int32_t cols, float grad_scale, void* stream);

/* Softmax cross-entropy, reduction = mean over the rows whose label != ignore_index (F.cross_entropy / nn.CrossEntropyLoss as
 * used at vilbert.py:1578-1590 for the masked-LM (30522-way, ignore_index -1) and alignment objectives and at
 * task_utils.py:339-343, 366-374 for the VL-logit / binary / tri heads). *loss (device scalar) = the mean (+= when
 * accumulate_loss); dlogits = grad_scale * d loss / d logits as f32 and/or bf16 (the operand of the head's backward GEMMs),
 * zero on ignored rows. No rows to average -> loss = NaN like torch, gradients 0. A label outside [0, cols) other than ignore_index
 * reads nothing: its row's gradient is 0 and the loss is NaN. */
vb_status vb_ce_loss(const float* logits, int64_t ld_logits, const int64_t* labels, int64_t ignore_index, float* loss,
                     float* dlogits_f32, int64_t ld_d32, void* dlogits_bf16, int64_t ld_d16, int32_t rows, int32_t cols,
                     float grad_scale, int32_t accumulate_loss, void* stream);

/* Task objectives and scores of the 12-in-1 task table (task_utils.py:31-376, 618-623), used by the forward-placed objectives of
 * the engine's plans (vilbert_b200.tasks).
 *
 * vb_bce_gather_loss: BCE-with-logits over an optional column gather, V-logit-mc (vision_logit[:, 101:].gather(1, ids), then
 * BCE mean * C, task_utils.py:352-360) and the soft-target binary / tri heads (BCE mean, :362-374):
 *   x[r,c] = logits[r * ld_logits + col_off + (ids ? ids[r*C + c] : c)],  t = target[r*C + c]  (f32 [rows, C])
 *   *loss (+= when accumulate_loss) = loss_mul * mean_{r,c} (max(x,0) - x t + log1p(exp(-|x|)))
 *   dlogits (f32 and/or bf16, `width` columns per row, ld_d32 / ld_d16) = d loss / d logits over the WHOLE row: 0 where nothing
 *   was gathered; a column gathered by several choices gets the sum of their gradients, added in choice order (deterministic).
 * One CTA per row with the row (width floats) and C gradients in shared memory (width*4 + C*8 <= 48 KiB). An id outside
 * [0, width - col_off) reads nothing and makes the loss NaN. row_loss: f32 workspace [rows] (the per-row sums, then added in a
 * fixed order by a second one-CTA launch: no atomics, the loss is bitwise reproducible).
 *
 * vb_task_score: batch score of one task type on the device, *score (+= when accumulate) = sum over rows of
 *   VB_SCORE_SOFT       target[r, a]                    compute_score_with_logits(logits, target).sum()   (:618-623)
 *   VB_SCORE_LABEL      a == labels[r]                  VL-logit: (argmax(vil_logit.view(B, options)) == target).sum()
 *   VB_SCORE_THRESHOLD  target[r, a] > 0.5              V-logit: (target.gather(1, argmax over regions) > 0.5).sum()
 *   VB_SCORE_CHOICE     a == argmax_c target[r, c]      V-logit-mc, a over the gathered logits (ids as above; an id out of
 *                                                       range reads as NaN)
 * where a = argmax_c logits[r * ld_logits + col_off + c] (or of the gathered logits) with torch.max's rules: a NaN is the maximum,
 * the first index wins among equals. target rows have pitch ld_target. preds (int64 [rows], may be NULL) receives a. One CTA. */
enum { VB_SCORE_SOFT = 0, VB_SCORE_LABEL = 1, VB_SCORE_THRESHOLD = 2, VB_SCORE_CHOICE = 3 };
vb_status vb_bce_gather_loss(const float* logits, int64_t ld_logits, int32_t col_off, int32_t width, const int64_t* ids,
                             const float* target, int32_t rows, int32_t C, float loss_mul, float* row_loss, float* loss,
                             int32_t accumulate_loss, float* dlogits_f32, int64_t ld_d32, void* dlogits_bf16, int64_t ld_d16, void* stream);
vb_status vb_task_score(int32_t mode, const float* logits, int64_t ld_logits, int32_t col_off, int32_t cols, const int64_t* ids,
                        int32_t width, const float* target, int64_t ld_target, const int64_t* labels, int32_t rows, float* score,
                        int32_t accumulate, int64_t* preds, void* stream);
/* vb_task_results: the per-row results of one evaluation batch (EvaluatingModel, task_utils.py:777-847), formed on the device so
 * that one device-to-host copy reads them. Rows are addressed as in vb_task_score: x[r, c] = logits[r * ld_logits + col_off + c],
 * or with ids (int64 [rows, cols]) logits[r * ld_logits + col_off + ids[r * cols + c]], an id outside [0, width - col_off)
 * reading as NaN. Always argmax[r] (int64) = a, the argmax of row r with torch.max's rules (a NaN is the maximum, the first
 * index wins among equals); then by mode
 *   VB_RESULT_ARGMAX   nothing else (VL-classifier / GQA answers, V-logit-mc predictions; values may be NULL)
 *   VB_RESULT_SOFTMAX  values[r * ld_values + c] = softmax(x[r, :])_c in fp32 (VL-logit option probabilities); a NaN or +inf in
 *                      the row makes the whole row NaN, as torch.softmax does
 *   VB_RESULT_GATHER   values[r] = target[r * ld_target + a] (V-logit: the IoU of the chosen region)
 * A warp per row, eight rows per CTA, no atomics: every output is written once, results are deterministic. */
enum { VB_RESULT_ARGMAX = 0, VB_RESULT_SOFTMAX = 1, VB_RESULT_GATHER = 2 };
vb_status vb_task_results(int32_t mode, const float* logits, int64_t ld_logits, int32_t col_off, int32_t cols, const int64_t* ids,
                          int32_t width, const float* target, int64_t ld_target, int32_t rows, int64_t* argmax, float* values,
                          int64_t ld_values, void* stream);
/* vb_retrieval_rank: caption-to-image retrieval ranks (eval_retrieval.py:315-337) on the device. Row r of scores (f32 [rows, cols],
 * row pitch ld_scores) is put in the stable descending order: column j comes before column i when s_j > s_i, or s_j == s_i and
 * j < i; -0.0 ties with +0.0 and every NaN comes after every number, NaNs in column order (np.argsort(-s, kind="stable")).
 *   rank_out[r] (int32)     position of column target[r] (int64) in that order, -1 when target[r] is outside [0, cols)
 *   topk_out[r, 0..k) (int32, NULL: none)  the first min(k, cols) columns of that order, -1 after them
 * One CTA per row with the row's keys in dynamic shared memory: one block-wide count for the rank, k block-wide arg-max rounds
 * for the top-k; no atomics, results are deterministic. cols <= 50000, 1 <= k <= 64; otherwise VB_ERR_INVALID. */
vb_status vb_retrieval_rank(const float* scores, int64_t ld_scores, int32_t rows, int32_t cols, const int64_t* target, int32_t k,
                            int32_t* rank_out, int32_t* topk_out, void* stream);
/* vb_retrieval_rank_sets: image-to-text retrieval ranks, where a row has a set of targets (an image and its ground-truth
 * captions). Row r of scores is ordered exactly as vb_retrieval_rank orders it; its targets are the columns
 * set_idx[set_off[r] .. set_off[r+1]) (int64, CSR: set_off has rows + 1 entries).
 *   rank_out[r] (int32)     the smallest position any target of the set takes in that order (its best-placed target); targets
 *                           outside [0, cols) are ignored, and a set with no target inside gives -1
 *   topk_out[r, 0..k) (int32, NULL: none)  as vb_retrieval_rank: the first min(k, cols) columns of the order, -1 after them
 * The best-placed target is the one with the largest key, so the rank is one block-wide count as in vb_retrieval_rank (one
 * kernel serves both). set_off and set_idx are read on the device only and are trusted: the offsets must index set_idx. A row
 * whose offsets are negative or decreasing has an empty set. No atomics, results are deterministic. cols <= 50000,
 * 1 <= k <= 64, set_off and set_idx not NULL; otherwise VB_ERR_INVALID, before any launch. */
vb_status vb_retrieval_rank_sets(const float* scores, int64_t ld_scores, int32_t rows, int32_t cols, const int64_t* set_off,
                                 const int64_t* set_idx, int32_t k, int32_t* rank_out, int32_t* topk_out, void* stream);
/* dst = src * (*scale), f32, scale read on the device: the backward of a forward-placed objective starts from the stored
 * d loss / d head times d(total) / d loss (loss_scale[task] / gradient_accumulation_steps, train_tasks.py:247-251, 545-548)
 * without a host synchronisation. */
vb_status vb_scale_by_device(const float* src, float* dst, int64_t n, const float* scale, void* stream);

/* Masked-region KL objective of BertForMultiModalPreTraining (visual_target == 0, vilbert.py:1506-1525):
 *   loss = sum_{b,r: label[b,r]==1} sum_c t_c (log t_c - log_softmax(scores[b, r+1, :])_c) / max(#(label == 1), 0)
 * scores f32 [B, Nv, C] (region 0 = the global feature is skipped, :1506), target f32 [B, Nv-1, C], label int64 [B, Nv-1].
 * dscores (f32 [B,Nv,C] and/or bf16 with row pitch ld_d16) = grad_scale * d loss / d scores, zero on unmasked rows. */
vb_status vb_kl_masked_loss(const float* scores, const float* target, const int64_t* label, float* loss, float* dscores_f32,
                            void* dscores_bf16, int64_t ld_d16, int32_t B, int32_t Nv, int32_t C, float grad_scale,
                            int32_t accumulate_loss, void* stream);

/* The other two masked-region objectives of BertForMultiModalPreTraining, on scores f32 [B, Nv, D] (region 0 skipped), target f32
 * [B, R, D] and label int64 [B, R], R = Nv - 1; a row is masked where label == 1. One CTA per row of scores writes its loss into
 * row_loss (f32 workspace [B * Nv]), then a one-CTA launch adds them in a fixed order into *loss (+= when accumulate_loss): no
 * atomics, loss and gradient are bitwise reproducible. dscores_f32 (f32 [B, Nv, D], NULL: no gradient) = grad_scale * d loss /
 * d scores, zero on region 0 and on unmasked rows.
 *
 * vb_mse_masked_loss: visual_target == 1 (vilbert.py:1507-1513, MSELoss(reduction="none") over the masked elements)
 *   loss = sum_{masked} sum_d (s - t)^2 / max(n_masked * D, 1)        (no masked row: 0)
 *
 * vb_nce_region_loss: visual_target == 2 (vilbert.py:1523-1575). For a masked (b, r): candidate 0 is target[b, r], candidate
 * k = 1..n_neg is row neg_index[b, r, k-1] (int64 [B, R, n_neg]) of target viewed as [B * R, D]; score_k = <candidate_k,
 * scores[b, r+1]>; loss = mean over the masked rows of CrossEntropy(score, 0) (no masked row: NaN, like torch). The prediction
 * row and the n_neg + 1 scores sit in shared memory ((D + n_neg + 1) * 4 <= 48 KiB); candidates are read with 128-bit loads
 * (D % 4 == 0, 16-byte aligned rows), no [n_masked, n_neg + 1, D] tensor exists. An index outside [0, B * R) is not read and
 * makes the loss NaN. Duplicate indices count once per occurrence. */
vb_status vb_mse_masked_loss(const float* scores, const float* target, const int64_t* label, int32_t B, int32_t Nv, int32_t D,
                             float grad_scale, float* row_loss, float* loss, int32_t accumulate_loss, float* dscores_f32, void* stream);
vb_status vb_nce_region_loss(const float* scores, const float* target, const int64_t* label, const int64_t* neg_index, int32_t B,
                             int32_t Nv, int32_t D, int32_t n_neg, float grad_scale, float* row_loss, float* loss,
                             int32_t accumulate_loss, float* dscores_f32, void* stream);

/* config.dynamic_attention (BertImageSelfAttention, vilbert.py:557-586): the image self-attention's queries and keys are scaled per
 * (sample, channel) by gate = 1 + sigmoid(dyLinear(pool)), pool = mean of the current text states over the unmasked tokens.
 *   vb_masked_mean_fwd  pool[b,:] = sum_n m[b,n] x[b,n,:] / sum_n m[b,n]; x f32 [B,N,H]; add_mask f32 [B,N] is the additive text mask
 *                       ((1-m) * -10000, what vb_mask_to_additive writes); outputs pool f32 [B,H] + its GEMM operand copies
 *                       (pool16 in the forward format, optional low part and bf16 copy)
 *   vb_masked_mean_bwd  dx[b,n,:] (+)= m[b,n] / sum_n m[b,n] * dpool[b,:]
 *   vb_gate_scale_fwd   qk[b*N+n, c] *= 1 + sigmoid(z[b,c]) for c < cols, in place on the Q|K sections of the 16-bit projection
 *                       buffer (row pitch ld elements, hi (+ lo) parts, fp16 or bf16); z f32 [B, cols] = dyLinear_q | dyLinear_k outputs
 *   vb_gate_scale_bwd   dqk (bf16, in place) <- gate * dqk;  dz[b,c] = s(1-s) * sum_n dqk[b,n,c] qk[b,n,c] / gate, s = sigmoid(z);
 *                       qk is the GATED forward buffer; dz f32 [B, cols] and its bf16 operand copy dz16, each may be NULL (both
 *                       NULL: only dqk is scaled, for a frozen gate Linear whose input needs no gradient) */
vb_status vb_masked_mean_fwd(const float* x, const float* add_mask, float* pool, void* pool16, void* pool16_lo, void* pool16_b, int32_t out_fp16,
                             int32_t B, int32_t N, int32_t H, void* stream);
vb_status vb_masked_mean_bwd(const float* dpool, const float* add_mask, float* dx, int32_t accumulate, int32_t B, int32_t N, int32_t H, void* stream);
vb_status vb_gate_scale_fwd(void* qk, void* qk_lo, int64_t ld, const float* z, int32_t B, int32_t N, int32_t cols, int32_t fp16, void* stream);
vb_status vb_gate_scale_bwd(void* dqk, int64_t ldd, const void* qk, const void* qk_lo, int64_t ld, const float* z, float* dz, void* dz16, int32_t B,
                            int32_t N, int32_t cols, int32_t fp16, void* stream);

/* Masked-LM head without materialising the [tokens, 30522] logits when only the loss is wanted: only rows with label != ignore_index
 * enter the cross-entropy (vilbert.py:1578-1583), so the tied decoder GEMM, its CE and its backward run on those rows alone.
 *   vb_compact_rows      idx[r] = r-th row with labels[row] != ignore_index (-1 beyond the count), labels_compact[r] its label
 *                        (ignore_index beyond), *count = number of such rows (compare with cap on the host: rows past cap are dropped)
 *   vb_gather_rows16     dst[r,:] = src[idx[r],:] (zeros where idx[r] < 0), 16-bit rows, optionally a second (src2, dst2) pair
 *   vb_scatter_rows_f32  dst[idx[r],:] = src[r,:] for idx[r] >= 0 (the caller zeroes dst): gradient of the gather. With count and
 *                        poison given, *poison = NaN when *count > cap (rows were dropped: the loss must not look valid) */
vb_status vb_compact_rows(const int64_t* labels, int64_t ignore_index, int32_t rows, int32_t cap, int32_t* idx, int32_t* count,
                          int64_t* labels_compact, void* stream);
/* vb_compact_rows on a packed stream (Plan(packed=...)): row r < rows stands for padded row map[r] and is selected when map[r] >= 0
 * and labels[map[r]] != ignore_index (labels in the padded layout); idx holds packed rows, ascending, so the selected rows come in
 * the order vb_compact_rows gives their padded rows. */
vb_status vb_compact_rows_mapped(const int64_t* labels, int64_t ignore_index, const int32_t* map, int32_t rows, int32_t cap, int32_t* idx,
                                 int32_t* count, int64_t* labels_compact, void* stream);
vb_status vb_gather_rows16(const void* src, void* dst, const void* src2, void* dst2, const int32_t* idx, int32_t cap, int32_t cols, void* stream);
vb_status vb_scatter_rows_f32(const float* src, float* dst, const int32_t* idx, int32_t cap, int32_t cols, const int32_t* count, float* poison,
                              void* stream);

/* Additive attention masks of BertModel.forward (vilbert.py:1341-1362): out[b,j] = (1 - mask[b,j]) * -10000,
 * mask int64 0/1 [B,N]; prepend_one != 0 emits N+1 entries per row with a leading 0 (task-token mask
 * extension, :1331-1334). */
vb_status vb_mask_to_additive(const int64_t* mask, float* out, int32_t B, int32_t N, int32_t prepend_one, void* stream);

/* dst[r] = src for r < repeats (`bytes` each, multiple of 16): BertEncoder's FAST_MODE (vilbert.py:1042-1053) — the text stream
 * of ONE caption, computed at batch 1 up to the first connection layer, broadcast to the image batch (txt_embedding.expand). */
vb_status vb_broadcast_rows(const void* src, void* dst, int64_t bytes, int32_t repeats, void* stream);

/* dst[i * repeats + r] = src[i] for `items` items of `bytes` each (multiple of 16): the batch expansion of the reference's
 * `process: expand / dialog` tasks (task_utils.py:248-274, 198-246): region features / boxes / masks of one image replicated once
 * per answer option, features.unsqueeze(1).expand(B, options, ...).contiguous().view(-1, ...), done in one pass on the device. */
vb_status vb_repeat_rows(const void* src, void* dst, int64_t bytes, int64_t items, int32_t repeats, void* stream);

/* dst[k*n + e] (+)= sum_{r < count_r} src[k*stride_k + r*stride_r + e] for k < count_k, e < n (f32; n and the strides multiples of 4):
 * autograd of BertEncoder's in_batch_pairs expansion (vilbert.py:1008-1040), where every text / image item is expanded to B pairs. */
vb_status vb_sum_strided(const float* src, float* dst, int64_t n, int32_t count_k, int64_t stride_k, int32_t count_r, int64_t stride_r,
                         int32_t accumulate, void* stream);

/* step += 1 on the device (the dropout step counter; one launch per training step, capturable in a CUDA graph). */
vb_status vb_step_counter_bump(uint32_t* step, void* stream);

vb_status vb_memset_zero(void* ptr, int64_t bytes, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Packed task steps (Plan(packed=...)): the valid text tokens and image regions of a batch as contiguous per-sample row ranges.
 * A packed stream has `rows` rows (the valid-row count rounded up to a capacity bucket); sample b owns rows off[b] .. off[b] +
 * len[b] - 1, rows off[B] .. rows - 1 belong to no sample, and map[r] is the padded row (b * N + i) of packed row r (-1: none).
 *   vb_pack_build          off (int32 [B + 1]), len (int32 [B]) and map (int32 [rows]) of both streams from the 0/1 masks, which
 *                          must be prefix-valid; the text length includes the task token's row when has_task (one CTA)
 *   vb_pack_rows_f32       dst[r,:] = src[map[r],:] (zeros where map[r] < 0), f32 rows of cols
 *   vb_pack_regions        the region features of the packed rows cast to a tensor-core operand (hi, optional split-precision lo,
 *                          optional bf16 copy): bitwise vb_cast_f32_to_bf16 of the same elements; cols % 8 == 0
 *   vb_unpack_rows_f32     dst[b*N + i,:] = i < len[b] ? src[off[b] + i,:] : fill (per-region logits back to the padded layout)
 *   vb_scatter_add_rows_f32  dst[idx[r],:] += src[r,:] (distinct idx): the pooled rows' gradient into the packed sequence gradient
 *   vb_zero_tail_rows      rows [*first, rows) of a, b, c (each optional but a; row pitch ld_bytes, row_bytes per row, both multiples
 *                          of 16) set to zero: the rows of no sample that the attention kernels do not write
 *   vb_pack_segments       off, len and map of ONE stream from its 0/1 mask [B, N_in] (vb_pack_build's layout and clamp): the image
 *                          stream of a packed retrieval plan's prefix, and its caption's text stream
 *   vb_broadcast_segment_rows  a one-sample packed stream of L = len[0] valid rows (read on the device) repeated as `repeats`
 *                          contiguous segments: dst row b * L + i (b < repeats) = src row i, every other of the `rows` rows zero;
 *                          row_bytes a multiple of 16 (fp32 rows and each 16-bit operand copy, one launch per tensor) */
vb_status vb_pack_build(const int64_t* text_mask, int32_t Nt_in, int32_t has_task, const int64_t* image_mask, int32_t Nv, int32_t B,
                        int32_t rows_t, int32_t rows_v, int32_t* off_t, int32_t* len_t, int32_t* map_t, int32_t* off_v, int32_t* len_v,
                        int32_t* map_v, void* stream);
vb_status vb_pack_rows_f32(const float* src, float* dst, const int32_t* map, int32_t rows, int32_t cols, void* stream);
vb_status vb_pack_regions(const float* features, const int32_t* map, int32_t rows, int32_t cols, int32_t fp16, void* dst, void* dst_lo,
                          void* dst_b16, void* stream);
vb_status vb_unpack_rows_f32(const float* src, float* dst, const int32_t* off, const int32_t* len, int32_t B, int32_t N, int32_t cols,
                             float fill, void* stream);
vb_status vb_scatter_add_rows_f32(const float* src, float* dst, const int32_t* idx, int32_t rows, int32_t cols, void* stream);
vb_status vb_zero_tail_rows(void* a, void* b, void* c, int64_t ld_bytes, int32_t row_bytes, const int32_t* first, int32_t rows, void* stream);
vb_status vb_pack_segments(const int64_t* mask, int32_t N_in, int32_t has_task, int32_t B, int32_t rows, int32_t* off, int32_t* len,
                           int32_t* map, void* stream);
vb_status vb_broadcast_segment_rows(const void* src, void* dst, int32_t row_bytes, const int32_t* len, int32_t repeats, int32_t rows,
                                    void* stream);

/* Whether a pre-training batch can be packed, from its device-resident masks and labels in one launch (one CTA): text_mask /
 * lm_labels int64 [B, Nt], image_mask int64 [B, Nv], image_label int64 [B, Nv - 1] (regions 1 .. Nv - 1). A NULL mask is all
 * valid; NULL labels count nothing. out (int32 [2B + 5]):
 *   out[b], out[B + b]   valid entries of sample b's text / image mask
 *   out[2B], out[2B + 1] samples whose text / image mask is not prefix-valid or has no valid entry
 *   out[2B + 2]          tokens with lm_labels != -1 where text_mask == 0
 *   out[2B + 3]          regions with image_label == 1 where image_mask == 0
 *   out[2B + 4]          tokens with lm_labels != -1 */
vb_status vb_pack_summary(const int64_t* text_mask, const int64_t* image_mask, int32_t B, int32_t Nt, int32_t Nv, const int64_t* lm_labels,
                          const int64_t* image_label, int32_t* out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Fused multi-tensor AdamW on flat buffers (SURVEY.md §8 f2). Replaces pytorch_transformers==1.0.0 AdamW as the reference
 * builds it (train_tasks.py:401-426: one param group per tensor with its own lr / weight_decay, correct_bias=False),
 * optimizer.step() + model.zero_grad() (train_tasks.py:550-551), and the engine's own weight-shadow cast:
 *   m = b1 m + (1-b1) g;  v = b2 v + (1-b2) g^2;  p -= step_size m / (sqrt(v) + eps);  p -= lr wd p   (decay after, on the new p)
 *   step_size = lr, or lr sqrt(1-b2^t)/(1-b1^t) when correct_bias (t = max(*step, 1), a device int32 the caller advances;
 *   a counter still at 0 steps like t = 1 instead of dividing by 1 - b1^0 = 0), formed in float64 and rounded to fp32 once
 * The (1-b1), (1-b2) factors are the group's one_minus_beta1 / one_minus_beta2: fp32(1 - b) of the host's float64 b, as the
 * reference's fp32 torch ops see `1.0 - beta2`. 1 - fp32(b) would differ: fp32(0.999) rounds 1 - b2 to 0.00099998713.
 * The bias corrections and RAdam's rectification use b = 1 - one_minus_beta in float64 for the same reason.
 * p / g / m / v: flat f32 buffers with one layout. Work list: chunk c covers elements [chunk_start[c], +chunk_count[c]) of one
 * tensor (starts multiples of 4) and uses groups[chunk_group[c]] (a DEVICE array, rewritten by the host when a scheduler
 * changes an lr). g is multiplied by grad_scale on read (gradient accumulation / loss scaling) and zeroed when zero_grad.
 * p16 (may be NULL): the 16-bit operand copy of the updated weights (bf16, or fp16 when p16_fp16), p16_lo its
 * split-precision low part (may be NULL), p16_b an always-bf16 copy for the backward (may be NULL). */
typedef struct vb_adamw_group {
  float lr, beta1, beta2, eps, weight_decay;
  int32_t correct_bias;
  float one_minus_beta1, one_minus_beta2;
} vb_adamw_group;

vb_status vb_adamw_step(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                        const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group, int32_t n_chunks,
                        const vb_adamw_group* groups, const int32_t* step, float grad_scale, int32_t zero_grad, void* stream);

/* Fused multi-tensor RAdam on the same flat buffers, chunk table and group table (correct_bias is ignored): the reference's
 * `--optim RAdam` (vilbert/optimization.py:16-100, built at train_tasks.py:427-428) + model.zero_grad() + the weight-copy cast:
 *   v = b2 v + (1-b2) g^2;  m = b1 m + (1-b1) g;  p -= lr wd p   (own group's betas / lr / wd; decay FIRST, on the old p)
 *   p -= step_size m / (sqrt(v) + eps)  if N_sma >= 5,  else  p -= step_size m
 *   N_sma_max = 2/(1-b2) - 1,  N_sma = N_sma_max - 2t b2^t/(1-b2^t),  t = *step
 *   step_size = lr sqrt((1-b2^t)(N_sma-4)/(N_sma_max-4)(N_sma-2)/N_sma N_sma_max/(N_sma_max-2)) / (1-b1^t)  (N_sma >= 5)
 *             = lr / (1-b1^t)  otherwise
 * N_sma and step_size are computed in float64 from the lr / b1 / b2 of groups[leader_group] and used for every tensor: the
 * reference caches them per step in one buffer shared by all groups, so the first tensor's group supplies them.
 * advance_step != 0: *step += 1 on `stream` first (one call = one capturable step); a call refused for its arguments leaves the
 * counter alone. t = max(*step, 1). Other arguments as vb_adamw_step. */
vb_status vb_radam_step(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                        const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group, int32_t n_chunks,
                        const vb_adamw_group* groups, int32_t leader_group, int32_t* step, int32_t advance_step, float grad_scale,
                        int32_t zero_grad, void* stream);

/* vb_adamw_step_capped / vb_radam_step_capped: vb_adamw_step / vb_radam_step on a grid of at most max_ctas CTAs (0: no cap, the
 * 8 x SMs of the plain calls; < 0 is refused). The same kernels stride over the chunk table, so every element gets bitwise the
 * update, moments and copies of the plain calls. For a step that runs beside the backward's GEMMs (optim.step_in_backward). */
vb_status vb_adamw_step_capped(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                               const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group, int32_t n_chunks,
                               const vb_adamw_group* groups, const int32_t* step, float grad_scale, int32_t zero_grad,
                               int32_t max_ctas, void* stream);
vb_status vb_radam_step_capped(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                               const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group, int32_t n_chunks,
                               const vb_adamw_group* groups, int32_t leader_group, int32_t* step, int32_t advance_step,
                               float grad_scale, int32_t zero_grad, int32_t max_ctas, void* stream);

/* Gradient-norm clipping and non-finite step skipping for the two optimizers above: apex FusedAdam's max_grad_norm (the
 * reference's --fp16 optimizer, train_concap.py:452-457), torch.nn.utils.clip_grad_norm_, and the step skip of
 * torch.amp.GradScaler, decided on the device.
 *
 * vb_grad_norm: sum of g^2 over the chunk table in float64 (one partial per chunk into partials, double [n_chunks], then a
 * one-CTA launch adds them in a fixed order; the result does not depend on the grid, so ranks holding bitwise-equal gradients
 * compute bitwise-equal records), then writes *record:
 *   norm = |grad_scale| sqrt(sum g^2)   in fp32: the norm of the gradient the update uses, before clipping
 *   skip = 1 when the sum is not finite, i.e. some g is NaN or +-inf (a finite fp32 g cannot overflow the float64 sum)
 *   coef = 0 when skip, else min(1, max_norm / (norm + 1e-6)) with torch.nn.utils.clip_grad_norm_'s fp32 arithmetic
 *   skipped += skip;  *step += 1 unless skip (step may be NULL: no counter is advanced)
 * max_norm > 0 (+inf: skip without clipping). n_chunks == 0 writes norm 0 (partials may then be NULL).
 *
 * vb_adamw_step_clipped / vb_radam_step_clipped: vb_adamw_step / vb_radam_step reading *record (written by vb_grad_norm
 * earlier on the stream) after their dependency wait: the update uses g grad_scale coef; when record->skip is set p, m, v and
 * the 16-bit copies are left untouched and g is still zeroed when zero_grad. The plain calls are the record == NULL case of the
 * same kernels. Since vb_grad_norm advances the counter, callers pass advance_step = 0 to vb_radam_step_clipped. */
typedef struct vb_clip_record {
  float norm;
  float coef;
  int32_t skip;
  int32_t skipped;
} vb_clip_record;

vb_status vb_grad_norm(const float* g, const int64_t* chunk_start, const int32_t* chunk_count, int32_t n_chunks, float grad_scale,
                       float max_norm, double* partials, vb_clip_record* record, int32_t* step, void* stream);
vb_status vb_adamw_step_clipped(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group, int32_t n_chunks,
                                const vb_adamw_group* groups, const int32_t* step, float grad_scale, int32_t zero_grad,
                                const vb_clip_record* record, void* stream);
vb_status vb_radam_step_clipped(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                const int64_t* chunk_start, const int32_t* chunk_count, const int32_t* chunk_group, int32_t n_chunks,
                                const vb_adamw_group* groups, int32_t leader_group, int32_t* step, int32_t advance_step,
                                float grad_scale, int32_t zero_grad, const vb_clip_record* record, void* stream);

/* The same steps on one rank's slice of an optimizer state sharded over data-parallel ranks (ZeRO stage 1; optim shard_state=True).
 * vb_adamw_step_sharded / vb_radam_step_sharded: vb_adamw_step / vb_radam_step with the moments compact: m / v of chunk c start
 * at element state_start[c] (int64, multiples of 4) of m / v instead of at chunk_start[c]. p, g and the 16-bit copies keep the
 * flat layout, and every element gets bitwise what the unsharded calls give it (copies written, g zeroed when zero_grad).
 * record: NULL (no clipping) or a record written by vb_clip_finish, as in the _clipped calls; max_ctas as in the _capped calls.
 *
 * vb_grad_norm_partial: *sum = sum of g^2 over the chunk table in float64, in vb_grad_norm's fixed order (partials: double
 * [n_chunks]). The caller adds the ranks' sums (one all-reduce of one double) and passes the result to
 * vb_clip_finish: the record of vb_grad_norm from that sum (norm, coef, skip, skipped; *step += 1 unless skip, step may be NULL).
 * Every rank finishing the same sum writes the same record, so the ranks agree on skip and coefficient. */
vb_status vb_adamw_step_sharded(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                const int64_t* chunk_start, const int64_t* state_start, const int32_t* chunk_count,
                                const int32_t* chunk_group, int32_t n_chunks, const vb_adamw_group* groups, const int32_t* step,
                                float grad_scale, int32_t zero_grad, const vb_clip_record* record, int32_t max_ctas, void* stream);
vb_status vb_radam_step_sharded(float* p, float* g, float* m, float* v, void* p16, void* p16_lo, void* p16_b, int32_t p16_fp16,
                                const int64_t* chunk_start, const int64_t* state_start, const int32_t* chunk_count,
                                const int32_t* chunk_group, int32_t n_chunks, const vb_adamw_group* groups, int32_t leader_group,
                                int32_t* step, int32_t advance_step, float grad_scale, int32_t zero_grad,
                                const vb_clip_record* record, int32_t max_ctas, void* stream);
vb_status vb_grad_norm_partial(const float* g, const int64_t* chunk_start, const int32_t* chunk_count, int32_t n_chunks,
                               double* partials, double* sum, void* stream);
vb_status vb_clip_finish(const double* sum, float grad_scale, float max_norm, vb_clip_record* record, int32_t* step, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Single-stream baseline (BaseBertForVLTasks, vilbert/basebert.py:893-978).
 *
 * vb_concat_embed_ln_fwd: the text rows xt [B*Nt, H] (word + position + type, vb_embed_text_fwd) and the image rows xv [B*Nv, H]
 * (region GEMM + box projection) plus v_type_row (row 1 of the image token-type table) go through their own LayerNorm
 * (gamma_t / beta_t, gamma_v / beta_v) and dropout (index = row within the modality * H + col), written interleaved as the stream
 * [B, Nt+Nv, H]: y_f32 and the operand copies (y16 in the y_fp16 format, y_lo its split-precision low part, y_b16 bf16; each may be
 * NULL), with the row statistics mean / rstd [B*(Nt+Nv)].
 * vb_concat_embed_ln_bwd: dy [B*(Nt+Nv), H] -> dxt [B*Nt, H] (f32), dxv [B*Nv, H] (f32) and dxv_bf16; ACCUMULATES dgamma / dbeta of
 * both LayerNorms and the image column sum of dx into dcol_v and dcol_v2 (the region GEMM's bias and image token-type row 1). Every
 * output may be NULL. H <= 2048. */
vb_status vb_concat_embed_ln_fwd(const float* xt, const float* xv, const float* v_type_row, const float* gamma_t, const float* beta_t,
                                 const float* gamma_v, const float* beta_v, float* y_f32, void* y16, void* y_lo, void* y_b16, int32_t y_fp16,
                                 float* mean, float* rstd, int32_t B, int32_t Nt, int32_t Nv, int32_t H, const vb_dropout* drop_t,
                                 const vb_dropout* drop_v, void* stream);
vb_status vb_concat_embed_ln_bwd(const float* dy, const float* xt, const float* xv, const float* v_type_row, const float* gamma_t,
                                 const float* gamma_v, const float* mean, const float* rstd, float* dxt, float* dxv, void* dxv_bf16,
                                 float* dgamma_t, float* dbeta_t, float* dgamma_v, float* dbeta_v, float* dcol_v, float* dcol_v2,
                                 int32_t B, int32_t Nt, int32_t Nv, int32_t H, const vb_dropout* drop_t, const vb_dropout* drop_v, void* stream);
/* Scatter-add of d(text embeddings) [B*Nt, H] into word / position / token-type tables that all have padding_idx = 0: row 0 of
 * each receives nothing (basebert.py:290-298). Any table may be NULL. */
vb_status vb_embed_text_bwd_padded(const float* dout, const int64_t* ids, const int64_t* token_type_ids, float* dword, float* dpos,
                                   float* dtype, int32_t B, int32_t Nt, int32_t H, void* stream);
/* weight_norm(dim=None) (SimpleClassifier, basebert.py:965-978): w = v * (g / ||v||_F), g a scalar, written as w_f32 and the
 * operand copies (each may be NULL). Backward: dg += <dw, v> / ||v||, dv += (g / ||v||)(dw - (dg / ||v||) v) (either may be NULL).
 * Both reductions are fixed-order (bitwise reproducible). scratch: VB_WEIGHT_NORM_SCRATCH bytes of device memory per launch. */
#define VB_WEIGHT_NORM_SCRATCH 1024
vb_status vb_weight_norm_fwd(const float* v, const float* g, int64_t n, float* w_f32, void* w16, void* w_lo, void* w_b16, int32_t w_fp16,
                             double* scratch, void* stream);
vb_status vb_weight_norm_bwd(const float* dw, const float* v, const float* g, int64_t n, float* dg, float* dv, double* scratch, void* stream);
/* BertPooler's tanh (basebert.py:507-519): y = tanh(x) as y_f32 (may alias x) and operand copies. Backward: dx = dy (1 - y^2) as a
 * bf16 [M, N] operand, dbias[c] += sum over rows of dx (fixed order). */
vb_status vb_tanh_fwd(const float* x, float* y_f32, void* y16, void* y_lo, void* y_b16, int32_t y_fp16, int64_t n, void* stream);
vb_status vb_tanh_bwd(const float* dy, const float* y, void* dx_bf16, float* dbias, int32_t M, int32_t N, void* stream);
/* out [B, Nt+Nv] = cat((1 - mask_t) * -10000, (1 - mask_v) * -10000) (basebert.py:723-750); masks int64 0/1. */
vb_status vb_mask_concat_additive(const int64_t* mask_t, const int64_t* mask_v, float* out, int32_t B, int32_t Nt, int32_t Nv, void* stream);

/* ---- deterministic variants (plans built under torch.use_deterministic_algorithms(True), DESIGN.md §4h)
 * Each replaces the float atomics of its default entry point by per-block partial sums in a caller-owned fp32 workspace `ws`
 * followed by one ordered sum (vb_reduce_slices), with block counts that depend on the shape only: two runs on the same GPU model
 * and build give bitwise identical results. Arguments are those of the default entry point, plus ws.
 *
 * vb_gemm_bf16 with atomic_out = VB_GEMM_PARTIALS (weight gradients): split s of the k dimension stores its fp32 tile into rows
 * [s*M, s*M + M) of out_f32 (pitch ld_out_f32), a workspace of split_k * M rows; split_k must be the value vb_gemm_plan resolves for
 * the same arguments. The caller then adds the slices to the gradient with vb_reduce_slices. */
#define VB_GEMM_PARTIALS 2
#define VB_DET_SLICES 64          /* row blocks of vb_colsum_det / vb_loc_proj_bwd_det, CTAs of vb_small_linear_bwd_det, at most */
#define VB_DET_LN_SLICES 256      /* CTAs of vb_layernorm_bwd_det, at most */
#define VB_DET_LOSS_SLICES 1024   /* CTAs of the _det losses, at most */
/* dst[i] += part[0*stride + i] + part[1*stride + i] + ... + part[(slices-1)*stride + i], summed in slice order, i < n */
vb_status vb_reduce_slices(const float* part, int64_t stride, int32_t slices, int64_t n, float* dst, void* stream);
/* vb_colsum: ws holds VB_DET_SLICES * N floats */
vb_status vb_colsum_det(const void* X, int32_t is_bf16, int64_t ld, float* out, int32_t M, int32_t N, float* ws, void* stream);
/* vb_layernorm_bwd (dy2 == NULL) and vb_add_layernorm_bwd: ws holds 3 * VB_DET_LN_SLICES * H floats (unused when no sum is asked) */
vb_status vb_layernorm_bwd_det(const float* dy, const float* dy2, int64_t lddy, const float* x, int64_t ldx, const float* gamma,
                               const float* mean, const float* rstd, float* dx_f32, void* dx_bf16, int64_t lddx, const void* gelu_pre,
                               int64_t ld_pre, float* dgamma, float* dbeta, float* dbias, int32_t M, int32_t H,
                               const vb_dropout* out_dropout, const vb_dropout* in_dropout, float* ws, void* stream);
/* vb_embed_text_bwd without a workspace: each table row that takes a gradient is summed by one warp over the rows that select it,
 * in row order, and written once (H <= 1024) */
vb_status vb_embed_text_bwd_det(const float* dout, const int64_t* ids, const int64_t* token_type_ids, const int64_t* task_ids,
                                float* dword, float* dpos, float* dtype, float* dtask, int32_t B, int32_t Nt, int32_t H, void* stream);
/* vb_loc_proj_bwd: ws holds VB_DET_SLICES * 6 * H floats */
vb_status vb_loc_proj_bwd_det(const float* dy, const float* loc, float* dW, float* db, int32_t M, int32_t H, float* ws, void* stream);
/* vb_small_linear_bwd: ws holds VB_DET_SLICES * (N * K + N) floats */
vb_status vb_small_linear_bwd_det(const float* dy, const float* x, int64_t ldx, const float* W, float* dx, int64_t lddx,
                                  int32_t accumulate_dx, float* dW, float* db, int32_t M, int32_t K, int32_t N,
                                  const vb_dropout* in_dropout, float* ws, void* stream);
/* the losses: ws holds VB_DET_LOSS_SLICES floats */
vb_status vb_bce_logits_loss_det(const float* logits, const float* target, float* loss, float* dlogits_f32, void* dlogits_bf16,
                                 int64_t ld_dlogits_bf16, int32_t rows, int32_t cols, float grad_scale, float* ws, void* stream);
vb_status vb_ce_loss_det(const float* logits, int64_t ld_logits, const int64_t* labels, int64_t ignore_index, float* loss,
                         float* dlogits_f32, int64_t ld_d32, void* dlogits_bf16, int64_t ld_d16, int32_t rows, int32_t cols,
                         float grad_scale, int32_t accumulate_loss, float* ws, void* stream);
vb_status vb_kl_masked_loss_det(const float* scores, const float* target, const int64_t* label, float* loss, float* dscores_f32,
                                void* dscores_bf16, int64_t ld_d16, int32_t B, int32_t Nv, int32_t C, float grad_scale,
                                int32_t accumulate_loss, float* ws, void* stream);

/* ---- anomaly detection (torch.autograd.set_detect_anomaly(True); plans built with Plan(anomaly=True), DESIGN.md §4i)
 * vb_nan_check scans the regions of a device table on `stream`: region r is rows x cols elements of dtype at ptr, row pitch ld
 * ELEMENTS; only that logical extent is read, never the pitch padding. When a region holds a NaN (an exponent of all ones and a
 * non-zero mantissa, either sign, any payload; an inf is not one) the launch does atomicMin(flag, id). The test is on the bits,
 * so it holds under --use_fast_math. 128-bit loads where a run is 16-byte aligned; every CTA strides over every region, so one
 * launch covers many small regions and a few large ones. reset != 0 (n_regions == 0): *flag = INT32_MAX instead. */
enum { VB_NAN_F32 = 0, VB_NAN_F16 = 1, VB_NAN_BF16 = 2 };
typedef struct vb_nan_region {
  const void* ptr;
  int64_t rows, cols, ld;
  int32_t dtype;   /* VB_NAN_F32 | VB_NAN_F16 | VB_NAN_BF16 */
  int32_t id;
} vb_nan_region;
vb_status vb_nan_check(const vb_nan_region* regions, int32_t n_regions, int32_t* flag, int32_t reset, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VILBERT_B200_H_ */
