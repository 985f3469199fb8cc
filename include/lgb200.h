/* lgb200 -- C ABI of the H100-native LightGlue matcher hot path.
 *
 * The reference (cvg/glue-factory) is pure Python/PyTorch: its "FFI" for this
 * path is the set of PyTorch operator calls inside
 * gluefactory/models/matchers/lightglue.py and gluefactory/models/utils/losses.py.
 * Each entry point below replaces one such group of calls; the citation on each
 * names the reference lines it stands in for.  The host-side plugin
 * (glue-factory_b200/matchers/lightglue.py) binds these with ctypes, see
 * INTEGRATION.md.
 *
 * Conventions
 *  - plain pointers to DEVICE memory + extents + the CUDA stream to launch on;
 *    no torch types.  The caller owns every buffer; kernels keep no state.
 *  - every function returns 0 on success or a negative LGB200_ERR_* code;
 *    lgb200_last_error() returns the message of the last failure on this thread.
 *  - activations are token-major: [batch, tokens, heads, 64] for q/k/v/ctx,
 *    [batch, rows, cols] row-major for similarity/score matrices.
 *  - `dtype` is LGB200_F32 (full-precision parity path, CUDA cores) or
 *    LGB200_BF16 (bf16 operands, fp32 accumulation, Hopper tensor cores).
 *  - head dimension is 64 (descriptor_dim / num_heads of the default
 *    LightGlue configuration, lightglue.py:347); the attention and rotary
 *    entry points with an `_hd` suffix also take 32.
 */
#ifndef LGB200_H_
#define LGB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#ifndef __CUDA_RUNTIME_H__
typedef struct CUstream_st* cudaStream_t;
#endif

#define LGB200_ABI_VERSION 2

#define LGB200_F32 0
#define LGB200_BF16 1

#define LGB200_OK 0
#define LGB200_ERR_INVALID (-1)     /* bad argument (null pointer, empty or misaligned input) */
#define LGB200_ERR_CUDA (-2)        /* a CUDA runtime / driver call failed */
#define LGB200_ERR_UNSUPPORTED (-3) /* shape or device not supported by this build */

int lgb200_abi_version(void);
const char* lgb200_last_error(void);
/* 0 when the current device is sm_90 (H100); LGB200_ERR_UNSUPPORTED otherwise. */
int lgb200_check_device(void);

/* ---- rotary encoding + QKV de-interleave ------------------------------------------------------
 * replaces lightglue.py:157-160 (unflatten(H,-1,3), q/k/v slices, apply_cached_rotary_emb) and
 * lightglue.py:42-49.  qkv [ntok, H*192] with feature = h*192 + d*3 + {q,k,v};
 * theta [ntok, 32] fp32 = posenc.Wr(kpts) (lightglue.py:62); q,k,v [ntok, H*64].
 * Every pointer of both rope entry points must be 16-byte aligned.                          */
int lgb200_rope_split_fwd(const void* qkv, const float* theta, void* q, void* k, void* v, int64_t ntok, int H,
                          int dtype, cudaStream_t stream);
/* dq,dk are gradients w.r.t. the rotated q,k (saved by forward as q,k); writes dqkv [ntok, H*192]
 * and ACCUMULATES dtheta [ntok, 32] (the gradient that reaches posenc.Wr from every layer); dtheta NULL:
 * not computed (a frozen position encoder).                                                  */
int lgb200_rope_split_bwd(const void* dq, const void* dk, const void* dv, const void* q, const void* k,
                          const float* theta, void* dqkv, float* dtheta, int64_t ntok, int H, int dtype,
                          cudaStream_t stream);
/* The same two at head dimension head_dim = 32 or 64: qkv / dqkv [ntok, H*3*head_dim] with feature
 * = h*3*head_dim + d*3 + {q,k,v}, theta / dtheta [ntok, head_dim/2], q,k,v [ntok, H*head_dim]; any other value
 * returns LGB200_ERR_UNSUPPORTED before any CUDA call.  lgb200_rope_split_fwd / _bwd are these with head_dim = 64.
 * Head dimension 32 is LightGlue with descriptor_dim 128 and 4 heads, or 256 and 8 heads.                       */
int lgb200_rope_split_fwd_hd(const void* qkv, const float* theta, void* q, void* k, void* v, int64_t ntok, int H,
                             int dtype, int head_dim, cudaStream_t stream);
int lgb200_rope_split_bwd_hd(const void* dq, const void* dk, const void* dv, const void* q, const void* k,
                             const float* theta, void* dqkv, float* dtheta, int64_t ntok, int H, int dtype,
                             int head_dim, cudaStream_t stream);

/* ---- attention ----------------------------------------------------------------------------------
 * replaces F.scaled_dot_product_attention (lightglue.py:118-121) and the cross-attention einsum/
 * softmax block (lightglue.py:207-216).  out = softmax(scale * q k^T) v per (batch, head).
 * q,out [B,Nq,H,64]; k,v [B,Nk,H,64]; lse [B,H,Nq] fp32.  Keys/values of query batch b are taken
 * from batch (b + kv_shift) % B (kv_shift = B/2 on the [image0; image1] batch = both cross
 * directions in one launch; 0 = self-attention).                                                */
int lgb200_attn_fwd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk, int H,
                    int kv_shift, float scale, int dtype, cudaStream_t stream);
/* dq [B,Nq,H,64]; dk,dv [B,Nk,H,64] (indexed by KEY batch); delta_ws: lgb200_attn_bwd_ws_floats(B,Nq,Nk,H) floats of
 * scratch, 256-byte aligned (the per-query softmax statistics the kernels read: rowsum(dout*out) and, on the bf16
 * path, the base-2 log-sum-exp, padded to whole query tiles).
 * Shared-qk cross-attention (lightglue.py:207-216, one to_qk projection for both directions): when k == q,
 * dk == dq, Nq == Nk and 2 * kv_shift == B, dq receives the total gradient of the shared tensor (dq + dk) from one
 * pass over the shared similarity.  bf16 tensor-core path only; the fp32 path rejects this aliasing.             */
int64_t lgb200_attn_bwd_ws_floats(int B, int Nq, int Nk, int H);
int lgb200_attn_bwd(const void* q, const void* k, const void* v, const void* out, const float* lse, const void* dout,
                    void* dq, void* dk, void* dv, float* delta_ws, int B, int Nq, int Nk, int H, int kv_shift,
                    float scale, int dtype, cudaStream_t stream);
/* The same two at head dimension head_dim = 32 or 64 (every tensor above [.., H, head_dim]); any other value returns
 * LGB200_ERR_UNSUPPORTED.  lgb200_attn_fwd / lgb200_attn_bwd are these with head_dim = 64.  Head dimension 32 is
 * GlueStick with 128-channel descriptors and 4 heads (gluestick.py:524-551).  The workspace does not depend on
 * head_dim; the shared-qk backward is built for head_dim 64 only.                                              */
int lgb200_attn_fwd_hd(const void* q, const void* k, const void* v, void* out, float* lse, int B, int Nq, int Nk,
                       int H, int kv_shift, float scale, int dtype, int head_dim, cudaStream_t stream);
int lgb200_attn_bwd_hd(const void* q, const void* k, const void* v, const void* out, const float* lse,
                       const void* dout, void* dq, void* dk, void* dv, float* delta_ws, int B, int Nq, int Nk, int H,
                       int kv_shift, float scale, int dtype, int head_dim, cudaStream_t stream);
/* Forward only, over packed sequences of different lengths (LightGlue's adaptive depth / width on a batch of pairs):
 * q, out [Tq, H, head_dim]; k, v [Tk, H, head_dim] (token-major, dtype / head_dim as in lgb200_attn_fwd_hd); lse
 * [H, Tq] fp32.  Sequence s < S has the queries q_off[s] .. q_off[s] + q_len[s] - 1 and attends to the keys / values
 * k_off[s] .. k_off[s] + k_len[s] - 1; the four int32 arrays of S entries are device memory and are read by the
 * kernel only (no host copy).  max_q_len bounds every q_len[s] and sizes the grid.  Only the query rows of the
 * sequences are written (rows in no sequence keep their contents); a sequence with q_len or k_len 0 does no work.
 * Key rows past a sequence's end but inside [0, Tk) are read by whole tiles and masked out of the softmax, so they
 * must hold finite values (the tokens of other sequences).  Self-attention: k_off / k_len = q_off / q_len;
 * cross-attention: each sequence's keys are its partner's tokens.                                                  */
int lgb200_attn_fwd_varlen(const void* q, const void* k, const void* v, void* out, float* lse, const int* q_off,
                           const int* q_len, const int* k_off, const int* k_len, int S, int max_q_len, int Tq, int Tk,
                           int H, float scale, int dtype, int head_dim, cudaStream_t stream);

/* ---- FFN LayerNorm + GELU -------------------------------------------------------------------------
 * replaces nn.LayerNorm(2D) + nn.GELU() of the ffn Sequential (lightglue.py:143-148, 178-183).
 * x,y [ntok, W], W in {256,512,1024}; mean,rstd [ntok] saved for backward.
 * x, y, dy, dx, gamma and beta must be 16-byte aligned.                                          */
int lgb200_ln_gelu_fwd(const void* x, const float* gamma, const float* beta, void* y, float* mean, float* rstd,
                       int64_t ntok, int W, float eps, int dtype, cudaStream_t stream);
/* number of partial rows written to dgamma_part / dbeta_part / dxsum_part [parts, W] (caller sums over
 * parts); dxsum = column sums of dx = the bias gradient of the Linear that feeds the LayerNorm.  */
int lgb200_ln_gelu_bwd_parts(int64_t ntok);
int lgb200_ln_gelu_bwd(const void* dy, const void* x, const float* gamma, const float* beta, const float* mean,
                       const float* rstd, void* dx, float* dgamma_part, float* dbeta_part, float* dxsum_part,
                       int64_t ntok, int W, int dtype, cudaStream_t stream);

/* ---- batched bf16 tensor-core GEMM (wgmma, fp32 accumulate) ---------------------------------------
 * replaces torch.einsum("bmd,bnd->bmn") of MatchAssignment (lightglue.py:283) and its two backward
 * contractions.  C[b] (M x N) = opA(A[b]) * opB(B[b]):
 *   a_mn_major = 0: A is [M,K] row-major (lda);  1: A is stored [K,M] row-major (lda)
 *   b_mn_major = 0: B is [N,K] row-major (ldb);  1: B is stored [K,N] row-major (ldb)
 * lda/ldb in elements, multiples of 8; base pointers 16-byte aligned; C row-major with ldc;
 * the result is scaled by alpha in the epilogue (the d^-1/2 of lightglue.py:282).                  */
int lgb200_gemm_bf16(const void* A, const void* B, void* C, int batch, int M, int N, int K, int a_mn_major,
                     int b_mn_major, int64_t lda, int64_t ldb, int64_t ldc, int64_t strideA, int64_t strideB,
                     int64_t strideC, int c_dtype, float alpha, cudaStream_t stream);
/* Split-K form for the weight gradients dW = dy^T a of the Linear layers (torch autograd of F.linear,
 * lightglue.py:139-148 etc.): one fp32 C [M,N] (row pitch ldc) = opA(A) * opB(B) over a very long K (the tokens).
 * The K range is cut into as many pieces as there are idle SMs; the fp32 partial tiles go to ws
 * (gemm_splitk_ws_floats(M,N,K) floats) and are summed in split order (deterministic).                 */
int64_t lgb200_gemm_splitk_ws_floats(int M, int N, int K);
int lgb200_gemm_bf16_splitk(const void* A, const void* B, float* C, int M, int N, int K, int a_mn_major,
                            int b_mn_major, int64_t lda, int64_t ldb, int64_t ldc, float* ws, cudaStream_t stream);
/* One nn.Linear-shaped GEMM on the same persistent wgmma kernel, with the epilogues the layer needs
 * (replaces F.linear / its autograd, lightglue.py:139-148, 156-163, 174-183, 195-221, 280):
 *   C[M,N] (c_dtype, row pitch ldc) = alpha * op(A) op(B)^T + bias[N]          (accumulate == 0)
 *   C[M,N] (fp32)                  += alpha * op(A) op(B)^T + bias[N]          (accumulate != 0; read-modify-write in the epilogue)
 * A: [M,K] row pitch lda (or [K,M] when a_mn_major), B: [N,K] row pitch ldb (or [K,N] when b_mn_major), bf16;
 * bias: fp32 [N] or NULL.  forward: A = x, B = W;  dgrad: A = dy, B = W (b_mn_major);  row pitches let C be a column
 * block of a wider matrix (the [x | msg] FFN input, lightglue.py:162). */
int lgb200_linear(const void* A, const void* B, void* C, const float* bias, int M, int N, int K, int a_mn_major,
                  int b_mn_major, int64_t lda, int64_t ldb, int64_t ldc, int c_dtype, float alpha, int accumulate,
                  cudaStream_t stream);

/* ---- assignment head: sigmoid_log_double_softmax + NLL terms + argmax --------------------------------
 * replaces lightglue.py:256-268 (two log_softmax, transposed copy, slice assignment),
 * losses.py:6-25,62-73 (dense weight matrix and product) and the max() calls of
 * lightglue.py:86-90, 295-296.  sim [B,M,N] fp32.                                                 */
size_t lgb200_assign_ws_bytes(int B, int M, int N);
/* pass 1: lse_row [B,M] = logsumexp_j sim, lse_col [B,N] = logsumexp_i sim                         */
int lgb200_assign_lse(const float* sim, float* lse_row, float* lse_col, void* ws, int B, int M, int N,
                      cudaStream_t stream);
/* pass 2: scores_ij = (sim-lse_row_i) + (sim-lse_col_j) + (ls0_i + ls1_j) for i<M, j<N;
 *   scores [B,M+1,N+1] (optional dense output incl. dustbin column dust0, dustbin row dust1, corner 0)
 *   rowmax/rowarg [B,M]: max_j / argmax_j over j<N (lowest index wins ties); colmax/colarg [B,N] likewise
 *   pos_row_sum [B,M] (optional, needs gt [B,M,N] uint8): sum_j gt_ij (2 sim_ij - lse_row_i - lse_col_j)
 *   row_expsum [B,M] (optional): sum_{j<=N} exp(scores_ij)  (row_norm monitor, lightglue.py:596)     */
int lgb200_assign_scores(const float* sim, const float* lse_row, const float* lse_col, const float* ls0,
                         const float* ls1, const float* dust0, const float* dust1, const uint8_t* gt, float* scores,
                         float* rowmax, int* rowarg, float* colmax, int* colarg, float* pos_row_sum,
                         float* row_expsum, void* ws, int B, int M, int N, cudaStream_t stream);
/* backward of sum_ij gt_ij (2 sim_ij - lse_row_i - lse_col_j) scaled by gcoef[b]
 * (rowcnt_i = sum_j gt_ij, colcnt_j = sum_i gt_ij, as floats):
 *   dsim_ij = gcoef_b (2 gt_ij - exp(sim_ij-lse_row_i) rowcnt_i - exp(sim_ij-lse_col_j) colcnt_j)     */
int lgb200_assign_bwd(const float* sim, const float* lse_row, const float* lse_col, const uint8_t* gt,
                      const float* gcoef, const float* rowcnt, const float* colcnt, void* dsim, int out_dtype, int B,
                      int M, int N, cudaStream_t stream);
/* filter_matches (lightglue.py:293-309): mutual check + threshold; m0,m1 int64, -1 = no match       */
/* ---- assignment head fused with its similarity GEMM (csrc/assign_tc.cu; bf16 mdesc, D % 64 == 0, D <= 256) ----------
 * sim = alpha * mdesc0 . mdesc1^T (lightglue.py:283) is produced tile by tile in tensor memory and consumed there; it
 * is never written to memory.  md0: [B,M,D], md1: [B,N,D] bf16 contiguous.  Same outputs as lgb200_assign_lse /
 * lgb200_assign_scores (without the dense scores) / lgb200_assign_bwd followed by the two d(mdesc) GEMMs. */
int lgb200_assign_fused_lse(const void* md0, const void* md1, float alpha, float* lse_row, float* lse_col, int B, int M,
                            int N, int D, cudaStream_t stream);
/* gt ([B,M,N] bool) and pos_row_sum ([B,M]) are both set or both NULL. */
int lgb200_assign_fused_stats(const void* md0, const void* md1, float alpha, const float* lse_row, const float* lse_col,
                              const float* ls0, const float* ls1, const uint8_t* gt, float* rowmax, int* rowarg,
                              float* colmax, int* colarg, float* pos_row_sum, int B, int M, int N, int D,
                              cudaStream_t stream);
/* dmd0 [B*M, D], dmd1 [B*N, D] bf16 = dsim . md1, dsim^T . md0 with
 * dsim = gcoef[b] (2 gt - softmax_row rowcnt - softmax_col colcnt); gt_t = the [B,N,M] transpose of gt.  gt and gt_t
 * both NULL: dsim without the 2 gt term (labels given as match lists; lgb200_assign_pos_bwd adds it). */
int lgb200_assign_fused_bwd(const void* md0, const void* md1, float alpha, const float* lse_row, const float* lse_col,
                            const uint8_t* gt, const uint8_t* gt_t, const float* gcoef, const float* rowcnt,
                            const float* colcnt, void* dmd0, void* dmd1, int B, int M, int N, int D,
                            cudaStream_t stream);
/* ---- positive term from match lists (one-to-one labels; replaces the mask reads of losses.py:6-25 as used by
 * lightglue.py:578-627).  gt0 [B,M], gt1 [B,N] int64 (gt_matches0/1): row i's only positive is j = gt0[i] >= 0, and the
 * lists must agree, gt1[j] = i <=> gt0[i] = j.  rowcnt = (gt0 >= 0), colcnt = (gt1 >= 0) as floats.
 * pos_fwd: pos_row_sum [B,M] = the dense pos_row_sum of lgb200_assign_scores / _fused_stats: from sim (fp32 [B,M,N],
 * bit-identical to the mask's) or from md0 [B,M,D] / md1 [B,N,D] bf16 (2 alpha md0_i . md1_j - lse_row_i - lse_col_j,
 * fp32 accumulate); exactly one of sim and (md0, md1) is set.  0 without a positive; NaN where gt0[i] >= N or
 * gt1[gt0[i]] != i, so an inconsistent pair's loss is NaN.
 * pos_bwd: dmd0_i += 2 gcoef_b md1_{gt0[i]}, dmd1_j += 2 gcoef_b md0_{gt1[j]} in place (bf16), after
 * lgb200_assign_fused_bwd without masks.
 * bwd_sparse: lgb200_assign_bwd with gt_ij = (gt0[i] == j); bit-identical to it on consistent lists. */
int lgb200_assign_pos_fwd(const void* md0, const void* md1, const float* sim, float alpha, const float* lse_row,
                          const float* lse_col, const int64_t* gt0, const int64_t* gt1, float* pos_row_sum, int B,
                          int M, int N, int D, cudaStream_t stream);
int lgb200_assign_pos_bwd(const void* md0, const void* md1, const float* gcoef, const int64_t* gt0, const int64_t* gt1,
                          void* dmd0, void* dmd1, int B, int M, int N, int D, cudaStream_t stream);
int lgb200_assign_bwd_sparse(const float* sim, const float* lse_row, const float* lse_col, const int64_t* gt0,
                             const float* gcoef, const float* rowcnt, const float* colcnt, void* dsim, int out_dtype,
                             int B, int M, int N, cudaStream_t stream);
int lgb200_filter_matches(const float* rowmax, const int* rowarg, const int* colarg, float th, int64_t* m0,
                          int64_t* m1, float* ms0, float* ms1, int B, int M, int N, cudaStream_t stream);
/* Varlen forms of lgb200_assign_lse / lgb200_assign_scores (evaluation: no gt, no pos_row_sum) / lgb200_filter_matches:
 * one launch each over G pairs of different sizes (the packed evaluation head of LightGlue's adaptive / ragged
 * inference).  pairs [3, G] int32 (device) = (m, n, output batch row) of each pair, 1 <= m <= M, 1 <= n <= N; the
 * operands are padded: sim [G, M, N], ls0 / dust0 [G, M], ls1 / dust1 [G, N], and so are the intermediates lse_row /
 * rowmax / rowarg / row_expsum [G, M] and lse_col / colmax / colarg [G, N]; entries past a pair's extents are never read
 * (they may hold NaN) and, in the intermediates, never written.  ws: lgb200_assign_ws_bytes(G, M, N).  ind0 [G, M] /
 * ind1 [G, N] int32 (device): each row's / column's original keypoint index (< Mo / < No, distinct within a pair).
 * Pair g's scores go to scores [*, Mo + 1, No + 1] at row pairs[2G + g]: (ind0 i, ind1 j) for i < m, j < n, the
 * dustbin column No, the dustbin row Mo and the corner; every other entry keeps its contents.  filter_matches_varlen
 * writes m0 / ms0 [*, Mo] at ind0 and m1 / ms1 [*, No] at ind1 of that row, the matches themselves as original
 * indices.  Per pair the values are bit-identical to a uniform call on [1, m, n] (same kernels, same order).      */
int lgb200_assign_lse_varlen(const float* sim, float* lse_row, float* lse_col, void* ws, const int* pairs, int G, int M,
                             int N, cudaStream_t stream);
int lgb200_assign_scores_varlen(const float* sim, const float* lse_row, const float* lse_col, const float* ls0,
                                const float* ls1, const float* dust0, const float* dust1, float* scores, float* rowmax,
                                int* rowarg, float* colmax, int* colarg, float* row_expsum, void* ws, const int* pairs,
                                const int* ind0, const int* ind1, int G, int M, int N, int Mo, int No,
                                cudaStream_t stream);
int lgb200_filter_matches_varlen(const float* rowmax, const int* rowarg, const int* colarg, float th, int64_t* m0,
                                 int64_t* m1, float* ms0, float* ms1, const int* pairs, const int* ind0,
                                 const int* ind1, int G, int M, int N, int Mo, int No, cudaStream_t stream);

/* O(M+N) terms of one supervised layer (replaces the logsigmoid / weighted-sum / clamp / BCE tensor ops of
 * lightglue.py:264-267, losses.py:13-25, lightglue.py:81-94).  zt [T,2] = per token (matchability logit,
 * token-confidence logit), tokens ordered [image0 (B*M); image1 (B*N)].
 *   head_logsig   : ls = log sigmoid(z), du = log sigmoid(-z)                      [T] each
 *   head_terms_fwd: nll_pos = -(sum pos_row_sum + sum rowcnt ls0 + sum colcnt ls1)/num_pos,
 *                   nll_neg = -(sum neg0 du0 + sum neg1 du1)/num_neg, nll = bal nll_pos + (1-bal) nll_neg,
 *                   conf = token-confidence BCE against [argmax incl. dustbin == fin] (0 when fin* NULL)
 *   head_terms_bwd: d zt for upstream g_nll[B], g_conf[B]                                           */
int lgb200_head_logsig(const float* zt, float* ls, float* du, int64_t T, cudaStream_t stream);
/* The two per-token linear heads in one pass over x [T,D] fp32 (D % 8 == 0, D <= 512):
 *   head_token_fwd: zt[t] = (x[t].wm + bm, x[t].wt + bt)  (wt/bt NULL: column 1 repeats column 0),
 *                   ls/du as head_logsig, x_cast (nullable) = x in `dtype` for final_proj.
 *   head_token_bwd: dx = float(dmdw) + dzt[:,0] wm   (dmdw [T,D] in `dtype` = d md . W_final_proj; the confidence
 *                   head reads a detached x, lightglue.py:82-83), dW2 [2,D] = dzt^T x, db2 [2] = column sums of dzt.
 *                   dmdw and dx both NULL: dx is not computed (x needs no gradient).
 *                   ws: head_token_bwd_ws_floats(D) floats; counter: one uint32, zero before the first call. */
int lgb200_head_token_bwd_ws_floats(int D);
int lgb200_head_token_fwd(const float* x, const float* wm, const float* bm, const float* wt, const float* bt,
                          void* x_cast, float* zt, float* ls, float* du, int64_t ntok, int D, int dtype,
                          cudaStream_t stream);
int lgb200_head_token_bwd(const float* x, const void* dmdw, const float* dzt, const float* wm, float* dx, float* dW2,
                          float* db2, float* ws, unsigned* counter, int64_t ntok, int D, int dtype,
                          cudaStream_t stream);
int lgb200_head_terms_fwd(const float* zt, const float* pos_row_sum, const float* rowcnt, const float* colcnt,
                          const float* neg0, const float* neg1, const float* rowmax, const int* rowarg,
                          const float* colmax, const int* colarg, const int* fin0, const int* fin1,
                          const float* num_pos, const float* num_neg, float bal, float* nll, float* nll_pos,
                          float* nll_neg, float* conf, float* ws /* 4*B*ceil((M+N)/256) floats, 16-byte aligned */,
                          unsigned* counters /* B uint32, zero before the first call, left zero */, int B, int M, int N,
                          cudaStream_t stream);
int lgb200_head_terms_bwd(const float* zt, const float* rowcnt, const float* colcnt, const float* neg0,
                          const float* neg1, const float* rowmax, const int* rowarg, const float* colmax,
                          const int* colarg, const int* fin0, const int* fin1, const float* num_pos,
                          const float* num_neg, float bal, const float* g_nll, const float* g_conf, float* dzt, int B,
                          int M, int N, cudaStream_t stream);

/* ---- adaptive depth / width on a batch of pairs (LightGlue eval, lightglue.py:461-526, 545-576) ------------------
 * One layer's stop / prune step on the packed token state x [T, D] fp32 (D % 4 == 0), theta [T, R] fp32 (rotary
 * angles), ind [T] int32 (each token's keypoint index in its image).  Pair b < B owns segment 2b (image 0) and
 * 2b + 1 (image 1); seg [4][2B] int32 = (offset, length, partner's offset, partner's length), a stopped pair has
 * length 0.  zt [T, 2] = head_token_fwd's (matchability, token-confidence) logits of x; conf_thr: one fp32 threshold
 * of this layer (device).  Per pair with tokens left:
 *   stop   when finish != 0, or when do_stop and 1 - #(sigmoid(zt[:,1]) < thr) / (M + N) > depth_conf: its tokens go
 *          unpruned to rows b (M + N) + i (image 0) / b (M + N) + M + i (image 1) of x_fin [B (M + N), D] and
 *          ind_fin, fin_len[2b], fin_len[2b + 1] = its lengths, stop_layer[b] = layer;
 *   else   a token stays when !do_prune, or sigmoid(zt[t,0]) > width_thr, or do_stop and sigmoid(zt[t,1]) <= thr;
 *          kept tokens are packed pair-major into x_out / theta_out / ind_out (capacity T rows), seg_out gets the new
 *          segments and, with do_prune, prune0 [B, M] / prune1 [B, N] int64 rise by one at the kept keypoints.
 * status [2] int32 = (tokens kept, 1 if a pair that goes on kept no token of one of its views).  zt / conf_thr may be
 * NULL when finish != 0.  ws: lgb200_adaptive_compact_ws_ints(T, B) int32.  Two kernels, no host synchronisation.  */
int64_t lgb200_adaptive_compact_ws_ints(int T, int B);
int lgb200_adaptive_compact(const float* x, const float* theta, const int* ind, const float* zt, const int* seg,
                            float* x_out, float* theta_out, int* ind_out, int* seg_out, float* x_fin, int* ind_fin,
                            int* fin_len, int* stop_layer, int64_t* prune0, int64_t* prune1, int* status, int* ws,
                            const float* conf_thr, float depth_conf, float width_thr, int do_stop, int do_prune,
                            int layer, int finish, int B, int M, int N, int T, int D, int R, cudaStream_t stream);
/* The same step for pairs of different original sizes (LightGlue's ragged batches): pair_pts [B] int32 (device) =
 * each pair's original point count m_b + n_b, which replaces M + N in the stop test; M / N are the padded sizes that
 * lay out x_fin and prune0 / prune1.  pair_pts NULL is lgb200_adaptive_compact.                                    */
int lgb200_adaptive_compact_varlen(const float* x, const float* theta, const int* ind, const float* zt, const int* seg,
                                   float* x_out, float* theta_out, int* ind_out, int* seg_out, float* x_fin,
                                   int* ind_fin, int* fin_len, int* stop_layer, int64_t* prune0, int64_t* prune1,
                                   int* status, int* ws, const float* conf_thr, const int* pair_pts, float depth_conf,
                                   float width_thr, int do_stop, int do_prune, int layer, int finish, int B, int M,
                                   int N, int T, int D, int R, cudaStream_t stream);

/* ---- other assignment heads on the path ----------------------------------------------------------
 * log_double_softmax with a learned bin (gluestick.py:772-783) and log-domain Sinkhorn optimal
 * transport (gluefactory_nonfree/superglue.py:186-214).  scores/out [B,M+1,N+1].
 * ws: lgb200_heads_ws_bytes(B, M, N) bytes of scratch.                                               */
size_t lgb200_heads_ws_bytes(int B, int M, int N);
int lgb200_log_double_softmax(const float* sim, float bin_score, float* scores, void* ws, int B, int M, int N,
                              cudaStream_t stream);
/* the same with the (learnt) bin score read from device memory: no host read-back, capturable into a CUDA graph */
int lgb200_log_double_softmax_dev(const float* sim, const float* bin_score_dev, float* scores, void* ws, int B, int M,
                                  int N, cudaStream_t stream);
/* GlueStick's packed evaluation heads over G pairs of different sizes (eval only, no backward).
 * log_double_softmax_varlen: sim [G, M, N] fp32 padded; pairs [3, G] int32 (device) = (m <= M, n <= N, output batch
 * row) per pair; nothing past a pair's (m, n) is read.  Pair g's scores go to scores [*, Mo + 1, No + 1] at row
 * pairs[2G + g]: (i, j) for i < m, j < n, its dustbin column at No, its dustbin row at Mo and the corner (Mo, No); every
 * other entry keeps its contents.  rowmax / rowarg [G, M] and colarg [G, N] receive the max / argmax of each row and
 * the argmax of each column of the inner block (first index on ties), the input of lgb200_filter_matches_varlen with
 * identity index maps.  ws: lgb200_heads_ws_bytes(G, M, N).  Per pair, the scores are bit-identical to
 * lgb200_log_double_softmax on [1, m, n].
 * line_scores_varlen: raw [G, L0, L1] (i < m, j < n of pairs [2, G]; other entries untouched) from the endpoint
 * similarity sim [G, P0, P1] and the junction indices junc0 [G, 2 L0] / junc1 [G, 2 L1] (< P0 / P1 for the pair's
 * first 2m / 2n entries, not checked here): 0.5 max(s[a0,c0] + s[a1,c1], s[a0,c1] + s[a1,c0]) (gluestick.py:348-361).
 * junction_mean_varlen: x [*, D] fp32 += per target row, the mean of the endpoint updates upd [E, D] fp32 aimed at it;
 * order [E] int32 = the endpoints sorted stably by target row, tgt_sorted [E] = their rows in that order.  Each mean is
 * summed in that order (deterministic).  D % 4 == 0, x and upd 16-byte aligned.                                     */
int lgb200_log_double_softmax_varlen(const float* sim, const float* bin_score_dev, float* scores, float* rowmax,
                                     int* rowarg, int* colarg, void* ws, const int* pairs, int G, int M, int N, int Mo,
                                     int No, cudaStream_t stream);
int lgb200_line_scores_varlen(const float* sim, const int* junc0, const int* junc1, float* raw, const int* pairs, int G,
                              int P0, int P1, int L0, int L1, cudaStream_t stream);
int lgb200_junction_mean_varlen(float* x, const float* upd, const int* order, const int* tgt_sorted, int E, int D,
                                cudaStream_t stream);
/* GlueStick's LineLayer and line heads in training, summed in a fixed order (no atomics: the same bits on every run).
 * line_scores_train: lgb200_line_scores_varlen with torch.maximum's NaN rule (a NaN in either branch gives NaN), and
 * NaN for a line with a junction index outside [0, P0) / [0, P1) (nothing outside the pair's block is read).
 * line_scores_bwd: dsim [G, P0, P1] (every entry written, 0 where no line reads it) from graw = dL/draw [G, L0, L1],
 * the autograd of the torch formula: torch.maximum's backward (the larger branch takes the gradient, each takes half on
 * an exact tie, both take it when either is NaN), the gathers' backward summed per (r, c) over the endpoints at
 * junctions r and c in CSR order.  order0 [G * 2 L0] int32: entries of junc0's flat [G, 2 L0], each pair's endpoints
 * sorted stably by junction index; ptr0 [G, P0 + 1] int32: junction r of pair g has order0[ptr0[g, r] ..
 * ptr0[g, r + 1]); likewise order1 / ptr1.  Lines past a pair's (m, n) of pairs [2+, G] are skipped.
 * junction_sum: x [*, D] fp32 += per target row, the sum over the endpoints e aimed at it (order / tgt_sorted as for
 * junction_mean_varlen) of src[e, 0 .. D-1] + src[e ^ 1, D .. 2D-1], src [E, ld] fp32 with row pitch ld >= 2D: the
 * backward of the LineLayer's gather of [x[tgt[e]] ; x[tgt[e ^ 1]]].  E even, D % 4 == 0, ld % 4 == 0, x and src 16-byte
 * aligned.                                                                                                          */
int lgb200_line_scores_train(const float* sim, const int* junc0, const int* junc1, float* raw, const int* pairs, int G,
                             int P0, int P1, int L0, int L1, cudaStream_t stream);
int lgb200_line_scores_bwd(const float* graw, const float* sim, const int* junc0, const int* junc1, const int* order0,
                           const int* ptr0, const int* order1, const int* ptr1, const int* pairs, float* dsim, int G,
                           int P0, int P1, int L0, int L1, cudaStream_t stream);
int lgb200_junction_sum(float* x, const float* src, const int* order, const int* tgt_sorted, int E, int D, int ld,
                        cudaStream_t stream);
int lgb200_sinkhorn(const float* sim, float alpha, int iters, float* out, void* ws, int B, int M, int N,
                    cudaStream_t stream);
/* The same iterations with their potentials kept (uh [iters,B,M+1], vh [iters,B,N+1], both or neither; out may be
 * NULL), and the reverse sweep that turns grad = dL/dout [B,M+1,N+1] into dsim [B,M,N] plus the gradient entering the
 * dustbin row dzr [B,N+1] and column dzc [B,M] (d alpha = sum of both): the autograd of superglue.py:186-214
 * without its tape.  One persistent cooperative launch each; iters > 0 for the backward.                     */
int lgb200_sinkhorn_fwd(const float* sim, float alpha, int iters, float* out, float* uh, float* vh, void* ws, int B,
                        int M, int N, cudaStream_t stream);
int lgb200_sinkhorn_bwd(const float* sim, float alpha, int iters, const float* grad, const float* uh, const float* vh,
                        float* dsim, float* dzr, float* dzc, void* ws, int B, int M, int N, cudaStream_t stream);
/* The same two with the (learnt) bin score alpha read from device memory at kernel start: no host read-back, so a
 * training step that runs them can be captured into a CUDA graph.  Results equal the host-scalar entry points'.  */
int lgb200_sinkhorn_fwd_dev(const float* sim, const float* alpha_dev, int iters, float* out, float* uh, float* vh,
                            void* ws, int B, int M, int N, cudaStream_t stream);
int lgb200_sinkhorn_bwd_dev(const float* sim, const float* alpha_dev, int iters, const float* grad, const float* uh,
                            const float* vh, float* dsim, float* dzr, float* dzc, void* ws, int B, int M, int N,
                            cudaStream_t stream);
/* SuperGlue's packed evaluation head: the Sinkhorn iterations over G pairs of different sizes in one persistent
 * cooperative launch (eval only, no potentials, no backward).  sim [G, M, N] fp32 padded; pairs [3, G] int32 (device)
 * = (m <= M, n <= N, output batch row) per pair; nothing past a pair's (m, n) is read; alpha_dev the bin score on the
 * device; iters >= 0.  Per pair, superglue.py:186-214 with norm = -log(m + n): out = Z + u + v - norm, pair g's block
 * at row pairs[2G + g] of out [*, Mo + 1, No + 1]: (i, j) for i < m, j < n, its dustbin column at No, its dustbin row
 * at Mo and the corner (Mo, No); every other entry keeps its contents.  A pair's strip geometry and summation orders
 * depend on its (m, n) only, so its result is bit-identical whatever the other pairs of the call; it equals
 * lgb200_sinkhorn_fwd_dev on [1, m, n] up to the order of the column merges.  ws: lgb200_sinkhorn_varlen_ws_bytes. */
size_t lgb200_sinkhorn_varlen_ws_bytes(int G, int M, int N);
int lgb200_sinkhorn_varlen(const float* sim, const float* alpha_dev, int iters, float* out, void* ws, const int* pairs,
                           int G, int M, int N, int Mo, int No, cudaStream_t stream);
/* NLL head on the dense Sinkhorn output Z [B,M+1,N+1] (row pitch N+1; superglue.py:322-352), gt mask u8 [B,M,N],
 * neg0 [B,M] / neg1 [B,N] the 0/1 unmatched indicators (fp32).  Forward, per pair: pos = sum mask * Z[:M,:N],
 * neg = sum neg0 * Z[:M,N] + sum neg1 * Z[M,:N], in a fixed order (two calls are bit-identical); ws: at least
 * 4 * B * ceil(M / 8) bytes (lgb200_heads_ws_bytes suffices).  Backward of nll_pos = -pos / num_pos and
 * nll_neg = -neg / num_neg (num_pos, num_neg [B] the clamped counts) for the incoming gradients gpos, gneg [B], all
 * read on the device: writes every element of dZ [B,M+1,N+1] (0 off the positives and the bins, corner included). */
int lgb200_ot_nll_fwd(const float* Z, const uint8_t* mask, const float* neg0, const float* neg1, float* pos, float* neg,
                      void* ws, int B, int M, int N, cudaStream_t stream);
int lgb200_ot_nll_bwd(const uint8_t* mask, const float* neg0, const float* neg1, const float* num_pos,
                      const float* num_neg, const float* gpos, const float* gneg, float* dZ, int B, int M, int N,
                      cudaStream_t stream);
/* The same with the positives given as match lists (replaces the mask of superglue.py:325-336): gt0 [B,M], gt1 [B,N]
 * int64, one-to-one, positive (i, j) <=> gt0[i] = j >= 0.  pos, neg and dZ are bit-identical to lgb200_ot_nll_fwd /
 * _bwd on the equivalent mask; a row with gt0[i] >= N or gt1[gt0[i]] != i makes its pair's pos NaN. */
int lgb200_ot_nll_fwd_sparse(const float* Z, const int64_t* gt0, const int64_t* gt1, const float* neg0,
                             const float* neg1, float* pos, float* neg, void* ws, int B, int M, int N,
                             cudaStream_t stream);
int lgb200_ot_nll_bwd_sparse(const int64_t* gt0, const float* neg0, const float* neg1, const float* num_pos,
                             const float* num_neg, const float* gpos, const float* gneg, float* dZ, int B, int M, int N,
                             cudaStream_t stream);
/* Row max / argmax and column argmax of the inner block Z[:, :M, :N] (row pitch N+1), first index on ties like
 * torch's CPU max: the inputs of lgb200_filter_matches for SuperGlue's filter (superglue.py:301-311).             */
int lgb200_ot_filter_stats(const float* Z, float* rowmax, int* rowarg, int* colarg, int B, int M, int N,
                           cudaStream_t stream);

/* column sums of a tall [rows, cols] matrix = bias gradient of an nn.Linear (autograd of lightglue.py:156 etc.).
 * ws: lgb200_colsum_slabs(rows, cols) * cols floats of scratch; counters: (cols+63)/64 uint32, zero before the
 * FIRST call (the kernel leaves them zero again); cols % 8 == 0.  One launch, deterministic summation order. */
int lgb200_colsum_slabs(int64_t rows, int cols);
/* rowcnt [B,M] = sum_j mask, colcnt [B,N] = sum_i mask of a 0/1 byte mask [B,M,N] (the `gt.sum(2)` / `gt.sum(1)` of
 * lightglue.py:595-600) in one pass; N % 16 == 0, N <= 4096, mask 16-byte aligned; counts are exact.            */
/* Weight gradient of the position encoder's projection (autograd of lightglue.py:37-44, theta = kp Wr^T):
 * part [lgb200_posenc_wgrad_blocks()][C][KD] per-CTA partials of sum_t g[t][c] kp[t][d]; g [T,C] fp32 with C == 32
 * or 16 (head_dim / 2), kp [T,KD] fp32, KD <= 4.  The caller sums the partials over their first dimension.       */
int lgb200_posenc_wgrad_blocks(void);
int lgb200_posenc_wgrad(const float* g, const float* kp, float* part, int64_t T, int C, int KD, cudaStream_t stream);
int lgb200_mask_counts(const uint8_t* mask, float* rowcnt, float* colcnt, int B, int M, int N, cudaStream_t stream);
int lgb200_colsum(const void* a, float* out, float* ws, unsigned* counters, int64_t rows, int cols, int dtype,
                  cudaStream_t stream);

/* ---- BatchNorm1d + ReLU (GlueStick MLPs, gluestick.py:465-475; nn.SyncBatchNorm under data parallelism) ----------
 * x, y, dy, dx token-major [ntok, C] in `dtype`, C a power of two in [8, 512]; gamma, beta, mean, rstd, running
 * statistics fp32 [C].  The statistics pass and the normalisation pass are separate calls so that the fp64 sum vectors
 * can be summed across ranks in between.  ws: lgb200_colsum_slabs(ntok, C) * 2 * C doubles, counters as for
 * lgb200_colsum (both may be shared with it on one stream).  Deterministic: fixed summation order, no float atomics.
 *   bn_stats          : sums [2C+1] = [sum x | sum x^2 | ntok] (fp64)
 *   bn_relu_fwd       : y = relu((x - mean) rstd gamma + beta) with mean / biased variance from `sums` (training mode;
 *                       the count is sums[2C]) or, when sums is NULL, from running_mean / running_var (eval mode).
 *                       save_mean / save_rstd [C] receive the mean and rstd used.  Training mode also updates
 *                       running_mean / running_var (may be NULL) with `momentum`, the variance unbiased by the count.
 *   bn_relu_bwd_reduce: sums [2C] = [sum dy' | sum dy' xhat], dy' = dy [pre-activation > 0]: dbeta and dgamma.
 *   bn_relu_bwd       : dx = gamma rstd (dy' - sums[0:C] / n - xhat sums[C:2C] / n), n = *count (the forward sums'
 *                       last element); sums = count = NULL (eval mode): dx = gamma rstd dy'.
 * x, y, dy and dx must be 16-byte aligned. */
int lgb200_bn_stats(const void* x, double* sums, double* ws, unsigned* counters, int64_t ntok, int C, int dtype,
                    cudaStream_t stream);
int lgb200_bn_relu_fwd(const void* x, const double* sums, const float* gamma, const float* beta, float* running_mean,
                       float* running_var, float momentum, float eps, void* y, float* save_mean, float* save_rstd,
                       int64_t ntok, int C, int dtype, cudaStream_t stream);
int lgb200_bn_relu_bwd_reduce(const void* dy, const void* x, const float* gamma, const float* beta, const float* mean,
                              const float* rstd, double* sums, double* ws, unsigned* counters, int64_t ntok, int C,
                              int dtype, cudaStream_t stream);
int lgb200_bn_relu_bwd(const void* dy, const void* x, const float* gamma, const float* beta, const float* mean,
                       const float* rstd, const double* sums, const double* count, void* dx, int64_t ntok, int C,
                       int dtype, cudaStream_t stream);
/* The running-statistics update of bn_relu_fwd alone (same formula), from the batch statistics `sums` of an earlier
 * bn_stats call: a second training-mode call of the same BatchNorm on the same batch without redoing the pass over x
 * (SuperGlue's checkpointed GNN recomputes each layer in the backward, updating its BatchNorms again).  One launch. */
int lgb200_bn_running_update(const double* sums, float* running_mean, float* running_var, float momentum, int C,
                             cudaStream_t stream);

/* ---- flat-buffer optimiser (train.py:358-361, 513) and casts --------------------------------------- */
/* Adam over the flat buffers, one launch.  g is multiplied by grad_scale (1/world for the summed all-reduce).
 * step: 1-based step count for the bias correction; the four *_dev pointers (each may be NULL) move the per-step
 * controls into device memory so that ONE captured CUDA graph of the whole training step stays valid while they
 * change:  step_dev (count), lr_dev (scheduler, train.py:347-367), loss_scale_dev (GradScaler scale: gradients are
 * additionally multiplied by 1 / *loss_scale_dev, train.py:490), found_inf_dev (!= 0: the update is skipped --
 * GradScaler.step on overflow and the NaN guard of train.py:477-480, 503-512).
 * lr_scale_per_elem (may be NULL): per-element LR multiplier = the reference's lr_scaling groups (train.py:353-361). */
int lgb200_adam_flat(float* p, const float* g, float* m, float* v, int64_t n, const float* lr_scale_per_elem, float lr,
                     float beta1, float beta2, float eps, float weight_decay, int step, const int* step_dev,
                     float grad_scale, const float* lr_dev, const float* loss_scale_dev, const float* found_inf_dev,
                     cudaStream_t stream);
/* The other rules of train.py:347-361 (train.optimizer) over the same flat buffers, with the same controls as
 * lgb200_adam_flat (grad_scale, lr_scale_per_elem, the *_dev pointers; found_inf_dev set: parameters and state are left
 * untouched), each in the arithmetic and order of operations of torch.optim.<X>'s single-tensor step (no maximize).
 * All buffers 16-byte aligned; one launch each.
 * AdamW: Adam with decoupled decay, p *= 1 - lr * lr_scale * weight_decay, before the update.
 * SGD: momentum_buffer non-NULL exactly when momentum != 0.  The first step (step count 1, read from step_dev when
 * given) sets the buffer to the gradient itself, undampened.  nesterov needs momentum > 0 and dampening 0.
 * RMSprop: momentum_buffer non-NULL exactly when momentum > 0; grad_avg non-NULL selects `centered`.  It keeps no
 * step-dependent term, so it takes no step count.                                                                  */
int lgb200_adamw_flat(float* p, const float* g, float* m, float* v, int64_t n, const float* lr_scale_per_elem,
                      float lr, float beta1, float beta2, float eps, float weight_decay, int step, const int* step_dev,
                      float grad_scale, const float* lr_dev, const float* loss_scale_dev, const float* found_inf_dev,
                      cudaStream_t stream);
int lgb200_sgd_flat(float* p, const float* g, float* momentum_buffer, int64_t n, const float* lr_scale_per_elem,
                    float lr, float momentum, float dampening, int nesterov, float weight_decay, int step,
                    const int* step_dev, float grad_scale, const float* lr_dev, const float* loss_scale_dev,
                    const float* found_inf_dev, cudaStream_t stream);
int lgb200_rmsprop_flat(float* p, const float* g, float* square_avg, float* momentum_buffer, float* grad_avg,
                        int64_t n, const float* lr_scale_per_elem, float lr, float alpha, float eps,
                        float weight_decay, float momentum, float grad_scale, const float* lr_dev,
                        const float* loss_scale_dev, const float* found_inf_dev, cudaStream_t stream);
/* found_inf[0] = 1.0f if any of g[0..n) is non-finite, else 0.0f (GradScaler.unscale_'s check, no host sync). */
int lgb200_flat_grad_check(const float* g, int64_t n, float* found_inf, cudaStream_t stream);
/* Gradient-norm clipping (torch.nn.utils.clip_grad_norm_ with error_if_nonfinite=True after GradScaler.unscale_,
 * train.py:501-512) in place of lgb200_flat_grad_check, without a host sync.  norm_out = ||g[0..n_norm) * grad_scale /
 * s||_2 with s = *loss_scale_dev (1 when NULL), summed in fp64 in a fixed order (bit-identical from call to call) and
 * rounded to fp32.  g[n_norm..n_check) is checked but not normed (the trainer's loss slot); norm_out is NaN when one of
 * those is non-finite.  found_inf = 1.0f when any checked value or the fp32 norm is non-finite, else 0.0f.
 * adam_div_out = s / min(1, max_norm / (norm + 1e-6)) (s when found_inf): passed as lgb200_adam_flat's
 * loss_scale_dev, it makes Adam apply grad_scale * coef / s.  grad_scale > 0, max_norm > 0; g 16-byte aligned.
 * ws: lgb200_flat_grad_norm_ws_bytes(n_norm) bytes of scratch, 16-byte aligned.  Two launches.                      */
size_t lgb200_flat_grad_norm_ws_bytes(int64_t n_norm);
int lgb200_flat_grad_norm(const float* g, int64_t n_norm, int64_t n_check, float grad_scale,
                          const float* loss_scale_dev, float max_norm, float* found_inf, float* norm_out,
                          float* adam_div_out, void* ws, cudaStream_t stream);
/* One step of bookkeeping on the device: ++*step_dev unless *found_inf, and the GradScaler.update rule on
 * *loss_scale / *growth_tracker (both may be NULL): x backoff_factor on overflow, x growth_factor after
 * growth_interval consecutive clean steps. */
int lgb200_amp_update(const float* found_inf, int* step_dev, float* loss_scale, int* growth_tracker,
                      float growth_factor, float backoff_factor, int growth_interval, cudaStream_t stream);
int lgb200_cast_bf16(const float* src, void* dst, int64_t n, cudaStream_t stream);
/* x_out = x + y for two fp32 streams (x_out may alias x) and the compute-dtype copy of the sum: the merge of the two
 * gradients that reach a layer's output (from the next layer and from the layer's supervision head) fused with the cast
 * the layer's backward starts with -- replaces autograd's accumulation kernel + a cast.  n elements, dtype of x_cast. */
int lgb200_add_f32_cast(const float* x, const float* y, float* x_out, void* x_cast, int64_t n, int dtype,
                        cudaStream_t stream);
/* residual update of the fp32 stream fused with the cast for the next GEMM (lightglue.py:163, 219-220):
 * x_out = x + y (y in `dtype`, may be NULL), x_cast = (dtype) x_out; either output may be NULL.   */
int lgb200_residual_add_cast(const float* x, const void* y, float* x_out, void* x_cast, int64_t n, int dtype,
                             cudaStream_t stream);
/* same over [rows, cols] with the cast copy written at row pitch cast_pitch >= cols (elements): the copy lands
 * directly in the left / right half of the [x | msg] operand of ffn.0 (lightglue.py:162, 219), no torch.cat.
 * lgb200_add_f32_cast, lgb200_residual_add_cast and lgb200_residual_add_cast_pitched need 16-byte aligned x, y,
 * x_out and x_cast; lgb200_cast_bf16 needs 16-byte aligned src and dst.                                        */
int lgb200_residual_add_cast_pitched(const float* x, const void* y, float* x_out, void* x_cast, int64_t rows,
                                     int64_t cols, int64_t cast_pitch, int dtype, cudaStream_t stream);

/* ---- ground-truth correspondences from a homography (SURVEY 8f row 1) ---------------------------------
 * replaces the O(M N) part of gt_matches_from_homography (geometry/gt_generation.py:109-161): kp0 [B,M,2],
 * kp1 [B,N,2] pixel coordinates, kp0_1 = warp(kp0, H), kp1_0 = warp(kp1, H^-1) (the O(M+N) warps of
 * homography.py:161-180 are done by the caller).  dist = max(|kp0_1 - kp1|^2, |kp0 - kp1_0|^2); mutual nearest
 * neighbours with dist < pos_th^2 are positives; matches: index, -1 (best one-way error > neg_th^2), -2 (ignored).
 * assignment: [B,M,N] bytes (bool), cleared and filled by the call, or NULL.                              */
size_t lgb200_gt_homography_ws_bytes(int B, int M, int N);
int lgb200_gt_from_homography(const float* kp0, const float* kp1, const float* kp0_1, const float* kp1_0, float pos_th,
                              float neg_th, int64_t* matches0, int64_t* matches1, uint8_t* assignment, void* ws, int B,
                              int M, int N, cudaStream_t stream);
/* Same O(M N) label pass for ANY pair of reprojections (pose + depth ground truth, geometry/gt_generation.py:13-106):
 * vis0 [B,M] / vis1 [B,N] (bool, both or neither): the joint distance of a pair counts only when both points are
 * visible in the other view; valid0 / valid1 (bool, both or neither): "unmatched" (-1) additionally needs a valid depth.
 * assignment_t (may be NULL): the [B,N,M] transpose of `assignment`, written in the same pass (the fused assignment
 * backward walks the mask by columns too).  ws: lgb200_gt_homography_ws_bytes(B, M, N).  With all four masks NULL this is
 * lgb200_gt_from_homography. */
int lgb200_gt_from_reprojection(const float* kp0, const float* kp1, const float* kp0_1, const float* kp1_0,
                                const uint8_t* vis0, const uint8_t* vis1, const uint8_t* valid0, const uint8_t* valid1,
                                float pos_th, float neg_th, int64_t* m0, int64_t* m1, uint8_t* assignment,
                                uint8_t* assignment_t, void* ws, int B, int M, int N, cudaStream_t stream);
/* Extra unmatched labels from epipolar geometry (gt_generation.py:82-90; th_epi of matchers/depth_matcher.py): points
 * without valid depth that are still "ignore" (-2) become -1 when every still-ignored point of the other view is
 * further than th from their epipolar line (symmetric distance of geometry/epipolar.py:59-72, F [B,3,3] row-major).
 * m0 / m1 are updated in place; ws: B * (M + N) bytes. */
int lgb200_gt_epipolar_unmatched(const float* kp0, const float* kp1, const float* F, const uint8_t* valid0,
                                 const uint8_t* valid1, float th, int64_t* m0, int64_t* m1, uint8_t* ws, int B, int M,
                                 int N, cudaStream_t stream);

/* ---- ground-truth line correspondences (gt_line_matches_from_homography / _from_pose_depth,
 * geometry/gt_generation.py:164-558) -------------------------------------------------------------------------
 * lgb200_gt_line_sample: lines [B,L,4] (x0, y0, x1, y1; 16-byte aligned) -> pts [B,L,npts,2], point k =
 * start + ((end - start) / (npts - 1)) * k (sample_pts, :164-170), npts >= 2.                                 */
int lgb200_gt_line_sample(const float* lines, float* pts, int B, int L, int npts, cudaStream_t stream);
/* Exact rectangular linear assignment (minimum cost) of B independent [rows, cols] float64 cost matrices (finite),
 * with the shortest-augmenting-path algorithm and tie rules of scipy.optimize.linear_sum_assignment, so the same
 * optimum is returned.  row2col [B,rows]: assigned column or -1; col2row [B,cols]: assigned row or -1.  One CTA per
 * matrix; shared memory ~33 max(rows,cols) + 13 min(rows,cols) bytes (up to 227 KiB).                           */
int lgb200_lsap(const double* cost, int* row2col, int* col2row, int B, int rows, int cols, cudaStream_t stream);
/* Labels from projected line points.  lines0 [B,L0,4] / lines1 [B,L1,4]: clamped segments (16-byte aligned);
 * pts0_1 [B,L0,npts,2]: the points of lines0 projected into view 1 (w1 x h1), pts1_0 the converse.  visible0/1
 * [B,L*npts] (projected point visible), valid_pts0/1 [B,L*npts] (valid depth at the point): all four NULL for the
 * homography variant, all four given for the depth variant.  valid_lines0/1 [B,L] bytes.  dist_th, overlap_th,
 * min_visibility_th as the reference's arguments.  Writes matches0/1 (int64: partner, -1 unmatched, -2 ignored) and,
 * when assignment is not NULL, the [B,L0,L1] bool positives.  ws: lgb200_gt_lines_ws_bytes(B, L0, L1); on return its
 * first B*L0*L1 float64 hold the cost matrix handed to the assignment (-close0*close1, 1e6 on unmatched / ignored
 * rows and columns).  No host synchronisation.                                                                   */
size_t lgb200_gt_lines_ws_bytes(int B, int L0, int L1);
int lgb200_gt_line_matches(const float* lines0, const float* lines1, const float* pts0_1, const float* pts1_0,
                           const uint8_t* visible0, const uint8_t* visible1, const uint8_t* valid_pts0,
                           const uint8_t* valid_pts1, const uint8_t* valid_lines0, const uint8_t* valid_lines1, int w0,
                           int h0, int w1, int h1, int npts, double dist_th, double overlap_th,
                           double min_visibility_th, int64_t* matches0, int64_t* matches1, uint8_t* assignment,
                           void* ws, int B, int L0, int L1, cudaStream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* LGB200_H_ */
