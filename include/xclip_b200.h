/*
 * xclip_b200.h - C-ABI of the H100-native (sm_90a) CLIP training hot path.
 *
 * This is the drop-in boundary (SURVEY.md 8b): plain `extern "C"` entry points,
 * raw device pointers + explicit shapes, a cudaStream_t, int return codes.  The
 * CALLER (PyTorch, through x_clip_b200/_lib.py) owns every buffer; the library
 * never allocates persistent device memory, never synchronises the host, never
 * throws and never exits.  All pointers are device pointers unless stated.
 *
 * Each entry point names the reference call site it replaces
 * (lucidrains/x-clip v0.14.4, paths relative to /root/reference).
 *
 * Conventions
 *   - "bf16" buffers hold __nv_bfloat16, "f32" buffers hold float.
 *   - Row-major everywhere; `ld*` are leading dimensions in ELEMENTS.
 *   - return 0 on success; otherwise an XCLIP_ERR_* code and xclip_last_error()
 *     returns a thread-local message.
 *   - Work is enqueued on `stream` and is asynchronous w.r.t. the host.
 */
#ifndef XCLIP_B200_H_
#define XCLIP_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define XCLIP_OK 0
#define XCLIP_ERR_INVALID 1      /* bad argument / unsupported shape */
#define XCLIP_ERR_CUDA 2         /* CUDA runtime / driver error */
#define XCLIP_ERR_UNSUPPORTED 3  /* device is not sm_90 */

#define XCLIP_MAJOR_K 0  /* operand stored with the contraction index contiguous */
#define XCLIP_MAJOR_MN 1 /* operand stored transposed (its M / N index contiguous) */

typedef void* xclip_stream_t; /* cudaStream_t */

/* ---- library ---------------------------------------------------------- */
int xclip_abi_version(void);
const char* xclip_last_error(void);
/* Binds to the current CUDA device, checks it is sm_90, resolves the driver
 * entry point used for TMA descriptors.  Idempotent. */
int xclip_init(void);
/* number of kernels this library has launched since the last reset (host counter) */
long long xclip_launch_count(void);
void xclip_launch_count_reset(void);
/* Explicit, process-wide tuning switches for A/B measurements (never read from the environment;
 * results are identical either way).  Returns the previous value, -1 for an unknown knob. */
#define XCLIP_TUNE_LN_FWD_BLOCKS 3 /* LayerNorm forward: cap on resident blocks per SM (0 = built-in 8) */
#define XCLIP_TUNE_LN_BWD_BLOCKS 4 /* LayerNorm backward: blocks per SM (0 = built-in 2) */
#define XCLIP_TUNE_ATTN_STREAM 5   /* attention: != 0 runs the streaming kernels at every n (0 = only n > 320) */
int xclip_tune_set(int knob, int value);

/* ---- dense contraction (wgmma) ------------------------------------------
 * C[M,N] (+)= alpha * A * B^T (+ bias[N]) (+ residual[res_row_idx[row] | row % res_row_mod | row, N])
 * Replaces nn.Linear fwd + its autograd dgrad/wgrad:
 *   x_clip/x_clip.py:191,195 (FeedForward), :209,:210 (Attention to_qkv/to_out),
 *   :358 (patch embedding, with bias), :368 (to_cls_tokens), :556,:570 (latent proj).
 * a_major = K : A is [M,K] (lda >= K).   a_major = MN : A is stored as [K,M] (lda >= M).
 * b_major = K : B is [N,K] (ldb >= K) - the nn.Linear [out,in] layout.
 * b_major = MN: B is stored as [K,N] (ldb >= N).
 * c_dtype 0 = bf16, 1 = f32.  accumulate != 0 (f32 only): C += result (atomic; enables
 * split-K over `K` when the output has too few tiles to fill the GPU - the wgrad case).
 * Requirements: N % 8 == 0, lda/ldb/ldr % 8 == 0, ldc % 8 == 0 (bf16) or % 4 (f32),
 * 16-byte aligned base pointers.  bias is f32, residual is bf16.
 */
int xclip_gemm_bf16(const void* a, int64_t lda, int a_major, const void* b, int64_t ldb,
                    int b_major, void* c, int64_t ldc, int c_dtype, int M, int N, int K,
                    float alpha, const float* bias, const void* residual, int64_t ldr,
                    int res_row_mod, const int32_t* res_row_idx, int accumulate,
                    xclip_stream_t stream);

/* ---- row-wise kernels ---------------------------------------------------
 * Gain-only LayerNorm, biased variance (x_clip/x_clip.py:112-121).  One call can also apply
 * the residual add of the block (:288) and the NEXT pre-norm (:126) so the row is read once:
 *   out  = LN(x) * g (+ res)                      stats  = (mean, rstd) of x        [rows,2] f32
 *   out2 = LN(bf16(out)) * g2   (if g2 != NULL)   stats2 = (mean, rstd) of bf16(out)
 * x/res/out/out2 bf16 [rows, d]; g/g2 f32 [d]; d in 256*{1,2,3,4}.  eps: the reference uses
 * 1e-5 for fp32 activations and 1e-3 otherwise (:118) - the caller chooses. */
int xclip_layernorm_fwd(const void* x, int64_t ldx, const float* g, const void* res,
                        int64_t ldres, void* out, int64_t ldo, float* stats, const float* g2,
                        void* out2, int64_t ldo2, float* stats2, int rows, int d, float eps,
                        xclip_stream_t stream);
/* dx = dLN(dy; x, stats, g) (+ add);  dg += sum_rows dy * xhat   (dg f32 [d], accumulated) */
int xclip_layernorm_bwd(const void* dy, int64_t lddy, const void* x, int64_t ldx,
                        const float* stats, const float* g, const void* add, int64_t ldadd,
                        void* dx, int64_t lddx, float* dg, int rows, int d,
                        xclip_stream_t stream);
/* xclip_layernorm_bwd that also writes xn = bf16(LN(x) * g) (if xn != NULL), the forward's output
 * rebuilt from the saved stats with the forward's fp32 operations (bit for bit xclip_layernorm_fwd's
 * out without res, or its out2 when x is that call's bf16(out)) in the pass that reads x anyway:
 * a backward can take its weight-gradient operand from here instead of keeping it from the forward. */
int xclip_layernorm_bwd_xn(const void* dy, int64_t lddy, const void* x, int64_t ldx,
                           const float* stats, const float* g, const void* add, int64_t ldadd,
                           void* dx, int64_t lddx, float* dg, void* xn, int64_t ldxn, int rows,
                           int d, xclip_stream_t stream);
/* l2norm = F.normalize(dim=-1, eps=1e-12) (x_clip/x_clip.py:54-55, used at :715,:724).
 * p f32 [rows,d] -> z f32 [rows,d], inv = 1/max(|p|,eps), and the split-bf16 operands of the
 * logits contraction: zrow = [hi|lo|hi], zcol = [hi|hi|lo], bf16 [rows,3d], hi = bf16(z),
 * lo = bf16(z - hi).  zrow . zcol^T = hi.hi + lo.hi + hi.lo matches the fp32 dot product to
 * ~2^-17, so the logits keep fp32-level accuracy while running on the bf16 tensor cores. */
int xclip_l2norm_fwd(const float* p, int64_t ldp, float* z, void* zrow, void* zcol, float* inv,
                     int rows, int d, xclip_stream_t stream);
/* dp (bf16) = inv * (dz - z <z,dz>) */
int xclip_l2norm_bwd(const float* dz, const float* z, const float* inv, void* dp, int rows, int d,
                     xclip_stream_t stream);
int xclip_cast_f32_bf16(const float* src, void* dst, int64_t n, xclip_stream_t stream);

/* ---- fused attention ------------------------------------------------------
 * Attention core of x_clip/x_clip.py:217-244 (dim_head = 64, any n).  causal != 0 adds the
 * reference's causal mask (keys j > i get -FLT_MAX, :233-236).
 * n <= 320 runs kernels that hold a head's whole K and V (Q and dO in the backward) in shared
 * memory; n > 320 runs kernels that stream them through shared memory in 64-row blocks (~40-50 KB
 * per CTA for any n).  Both compute the same blocks in the same order: bit-identical results.
 * qkv bf16 [B*n, ld_qkv] holds q | k | v, each heads*64 wide, head-major inside.
 * key_mask uint8 [B, n] (1 = attend; may be NULL).  o bf16 [B*n, ldo] (heads merged).
 * lse f32 [B, heads, n]: base-2 log-sum-exp of scale*log2(e)*scores (saved for backward).
 * A row with no visible key (all its keys masked, or masked and above the causal diagonal) gets, as
 * in the reference, the uniform softmax over all n keys, and lse = -FLT_MAX.  Its backward follows
 * masked_fill: no gradient reaches a masked score, so the row's dq is 0, it adds nothing to dk, and
 * it adds dO / n to the dv of every key.
 * scale must be > 0, ld_* multiples of 8 and at least their operand's width, and qkv, o, d_o and
 * dqkv 16-byte aligned; otherwise both calls return XCLIP_ERR_INVALID without launching. */
int xclip_attn_fwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask, void* o, int64_t ldo,
                   float* lse, int B, int n, int heads, float scale, int causal,
                   xclip_stream_t stream);
/* delta f32 [B, heads, n] is scratch (rowsum(dO*O), written here).  dq_workspace is not used
 * (dQ is accumulated on chip) and may be NULL. */
int xclip_attn_bwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask, const void* o,
                   int64_t ldo, const void* d_o, int64_t lddo, const float* lse, float* delta,
                   void* dqkv, int64_t ld_dqkv, float* dq_workspace, int B, int n, int heads,
                   float scale, int causal, xclip_stream_t stream);
/* The same attention with dropout on the softmax probabilities (x_clip.py:211, :241-243):
 * P' = P M / (1 - p), o = P' v, and lse stays that of the undropped row.  Backward: dv = P'^T dO,
 * dS = P (dO v^T M / (1 - p) - delta), delta = rowsum(dO o) as before.  Element (b, h, i, j) of
 * `layer` is kept iff word j & 3 of Philox4x32-10 with counter (j >> 2, i, b * heads + h, layer) and
 * key *seed (low word first) is below round((1 - p) 2^32).  The mask is a function of the element, so
 * the backward given the same seed and layer sees the forward's mask, on either schedule.  seed is an
 * 8-byte aligned device pointer (read by the kernels, no host sync); p in [0, 1] as fp32 (p = 1 gives
 * o = 0 and zero gradients); layer >= 0.  Other arguments and refusals as xclip_attn_fwd / _bwd. */
int xclip_attn_dropout_fwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask, void* o,
                           int64_t ldo, float* lse, int B, int n, int heads, float scale, int causal,
                           float p, const uint64_t* seed, int layer, xclip_stream_t stream);
int xclip_attn_dropout_bwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask, const void* o,
                           int64_t ldo, const void* d_o, int64_t lddo, const float* lse, float* delta,
                           void* dqkv, int64_t ld_dqkv, int B, int n, int heads, float scale,
                           int causal, float p, const uint64_t* seed, int layer,
                           xclip_stream_t stream);

/* ---- similarity + InfoNCE / DCL (wgmma, logits never materialised in forward) ------------
 * Replaces x_clip/x_clip.py:813-847 for one direction of the loss:
 *   s[r,c] = *temp_exp * <a_r, b_c> (temp_exp: DEVICE scalar exp(temperature), so the host
 *   never synchronises on the parameter),  a bf16 [R,D] = LOCAL unit-norm latents of one modality,
 *   b bf16 [C,D] = ALL latents of the other modality; the positive of row r is column
 *   r + diag_offset.  dcl != 0 removes the positive from the denominator (:834-836).
 * fwd:  lse[r] = log sum_c exp(s[r,c]);  pos[r] = s[r, r+diag_offset];
 *       *loss_accum += loss_scale * sum_r (lse[r] - pos[r])     (loss_accum may be NULL)
 *       part_ws: f32 scratch [2 * xclip_nce_num_col_blocks(C) * R], 8-byte aligned (per block:
 *       max, sum; the log-sum-exp uses an online maximum, so any temperature works).
 *       (the reference's +1e-20 inside its logs, :51-52, is below fp32 resolution here, except
 *       for an empty denominator - dcl with C == 1 - where lse = ln(1e-20) as in the reference)
 * bwd:  g[r,c] = *gscale * (w_row*exp(s - lse_row[r]) + w_col*exp(s - lse_col[c])
 *                           - w_diag*[c == r+diag])     (gscale: DEVICE scalar, upstream grad
 *       / (2*B_global); exp terms skipped on the positive when dcl).  Written as
 *       bf16 temp_exp*g [R, ldg>=roundup8(C)], so the latent gradient is dA = (that) @ b via
 *       xclip_gemm_bf16;  *dtemp += sum g*s (d loss / d temperature) when dtemp != NULL.
 *       lse_col (f32 [C]) is read with 16-byte vector loads: when w_col != 0 it must be 16-byte
 *       aligned, or the call returns XCLIP_ERR_INVALID without launching. */
int xclip_nce_num_col_blocks(int C);
int xclip_nce_fwd(const void* a, const void* b, int R, int C, int D, const float* temp_exp,
                  int diag_offset, int dcl, float* part_ws, float* pos, float* lse,
                  float* loss_accum, float loss_scale, xclip_stream_t stream);
int xclip_nce_bwd(const void* a, const void* b, int R, int C, int D, const float* temp_exp,
                  int diag_offset, int dcl, const float* lse_row, const float* lse_col,
                  float w_row, float w_col, float w_diag, const float* gscale, void* g,
                  int64_t ldg, float* dtemp, xclip_stream_t stream);

/* ---- pairwise sigmoid loss (SigLIP, Zhai et al., ICCV 2023) on the operands of xclip_nce_* -------
 * l[r,c] = *temp_exp * <a_r, b_c> + *logit_bias (both DEVICE scalars), z[r,c] = +1 if c == r +
 * diag_offset else -1.  a, b, R, C, D, diag_offset and alignment as for xclip_nce_fwd / _bwd.
 * fwd:  rowloss[r] = sum_c softplus(-z[r,c] l[r,c]) (f32 [R]);
 *       *loss_accum += loss_scale * sum_r rowloss[r]   (loss_accum may be NULL).
 *       part_ws: f32 scratch [xclip_nce_num_col_blocks(C) * R], 4-byte aligned; its blocks are summed
 *       in a fixed order.  softplus is accurate to fp32 rounding for small terms (log1p, not
 *       log(1 + x)), and a saturated logit gives softplus(x) = max(x, 0) exactly.
 * bwd:  g[r,c] = *gscale * (sigmoid(l[r,c]) - [c == r + diag_offset]) (gscale: DEVICE scalar,
 *       upstream grad / B_global), written as bf16 temp_exp*g [R, ldg >= roundup8(C)], ldg % 8 == 0,
 *       zero in the columns [C, ldg); the latent gradient is then dA = (that) @ b via xclip_gemm_bf16.
 *       *dtemp += sum g * (l - *logit_bias) (d loss / d temperature) and *dbias += sum g
 *       (d loss / d logit_bias), each when non-NULL. */
int xclip_sigmoid_fwd(const void* a, const void* b, int R, int C, int D, const float* temp_exp,
                      const float* logit_bias, int diag_offset, float* part_ws, float* rowloss,
                      float* loss_accum, float loss_scale, xclip_stream_t stream);
int xclip_sigmoid_bwd(const void* a, const void* b, int R, int C, int D, const float* temp_exp,
                      const float* logit_bias, int diag_offset, const float* gscale, void* g,
                      int64_t ldg, float* dtemp, float* dbias, xclip_stream_t stream);

/* ---- vocabulary cross-entropy of the MLM head (x_clip/mlm.py:96-107) on the same kernels ----------
 * l[r,v] = <x_r, w_v> + bias[v] for x bf16 [R,D] (the selected token encodings), w bf16 [V,D] (the
 * bf16 cast of to_logits.weight), bias f32 [V] or NULL; labels int64 [R] hold each row's target in
 * [0, V) (the caller checks the range: a label outside it gives an undefined loss and gradient, never
 * an out-of-bounds access).  Any V >= 1: the columns past V are masked inside the kernel.
 * fwd:  lse[r] = log sum_v exp(l[r,v]), pos[r] = l[r, labels[r]], both f32 [R], with an online
 *       maximum; *loss_accum += loss_scale * sum_r (lse[r] - pos[r]) (loss_accum may be NULL).
 *       part_ws: f32 scratch [2 * xclip_nce_num_col_blocks(V) * R], 8-byte aligned.  The [R, V]
 *       logits are never written.
 * bwd:  g[r,v] = bf16(*gscale * (exp(l[r,v] - lse[r]) - [v == labels[r]])) (gscale: DEVICE scalar),
 *       written as [R, ldg], ldg % 8 == 0, ldg >= roundup8(V), zero in the columns [V, ldg).
 *       dx = g[:, :V] w, dW = g[:, :V]^T x and dbias = column sums then run on xclip_gemm_bf16 and
 *       xclip_colsum_rows; the caller bounds R (a window of rows) to bound g.
 * x, w, g 16-byte aligned, bias 16-byte aligned, labels 8-byte aligned, D % 8 == 0; otherwise
 * both calls return XCLIP_ERR_INVALID without launching. */
int xclip_vocab_ce_fwd(const void* x, const void* w, const float* bias, const int64_t* labels, int R,
                       int V, int D, float* part_ws, float* pos, float* lse, float* loss_accum,
                       float loss_scale, xclip_stream_t stream);
int xclip_vocab_ce_bwd(const void* x, const void* w, const float* bias, const int64_t* labels, int R,
                       int V, int D, const float* lse, const float* gscale, void* g, int64_t ldg,
                       xclip_stream_t stream);

/* ---- similarity regularisation (arXiv 2309.08773; x_clip/x_clip.py:771-784, :870-873) ----------
 * E[r,c] = <t_r, t_c> - <v_r, v_c> for LOCAL rows r and ALL columns c of the global batch, formed in
 * the fp32 accumulator as one contraction a . b^T of the concatenated operands
 *   a = [zrow_t | zrow_v]  bf16 [R, K],   b = [zcol_t | -zcol_v]  bf16 [C, K],   K = 6*D
 * (zrow / zcol: the split-bf16 operands of xclip_l2norm_fwd, each [rows, 3D]).  Row r's own sample is
 * column r + diag_offset; that column and nothing beyond C takes part.  a, b: 16-byte aligned,
 * K % 8 == 0.  diag_offset < 0 or diag_offset + R > C returns XCLIP_ERR_INVALID without a launch.
 * pack : out bf16 [rows, 2k] = [t | v] (negate_v = 0) or [t | -v] (negate_v != 0); t, v bf16 [rows, k]
 *        contiguous, k % 8 == 0, t / v / out 16-byte aligned.  Negation is exact.
 * fwd  : rowsum[r] = sum_{c != r+diag_offset} E[r,c]^2 (f32 [R], may be NULL);
 *        *loss_accum += loss_scale * sum_r rowsum[r]   (loss_accum may be NULL).
 *        part_ws: f32 scratch [xclip_nce_num_col_blocks(C) * R], 4-byte aligned.
 * bwd  : g[r,c] = bf16(*gscale * E[r,c]) (gscale: DEVICE scalar), 0 at c == r+diag_offset and in
 *        the pad columns [C, ldg); g [R, ldg >= roundup8(C)], ldg % 8 == 0, 16-byte aligned.  With
 *        gscale = upstream * 2 w / (B (B-1)) the latent gradients of w * L_sim are dT = g @ T and
 *        dV = -(g @ V) over the columns' latents (xclip_gemm_bf16). */
int xclip_simreg_pack(const void* t, const void* v, int rows, int k, int negate_v, void* out,
                      xclip_stream_t stream);
int xclip_simreg_fwd(const void* a, const void* b, int R, int C, int K, int diag_offset,
                     float* part_ws, float* rowsum, float* loss_accum, float loss_scale,
                     xclip_stream_t stream);
int xclip_simreg_bwd(const void* a, const void* b, int R, int C, int K, int diag_offset,
                     const float* gscale, void* g, int64_t ldg, xclip_stream_t stream);

/* ---- FILIP fine-grained loss (x_clip/x_clip.py:799-811 + :821-847) -----------------------
 * segmax_arg16 : a bf16 [R,D] token latents of one modality, b bf16 [C,D] token latents of the
 *          other, C = n_samples * seg_len (1 <= seg_len <= 65535 tokens per sample).  For every row
 *          r and sample y: seg_max[r,y] = max_i s (f32), seg_arg[r,y] = argmax_i s (16-bit, 2 bytes
 *          per (row, sample): the saved state of a row-chunked FILIP loss) with
 *          s = *temp_exp * <a_r, b_(y,i)> (optionally s*col_mul[c] + col_add[c]: padded text
 *          tokens get col_mul 0 / col_add -FLT_MAX, the reference's masked_fill at :810).
 *          Either output may be null, not both.  Ties go to the lowest index; a segment whose
 *          columns are all masked gives -FLT_MAX at index 0.
 *          keys: caller-owned workspace of 8 * R * (C / seg_len) bytes, 8-byte aligned, no
 *          initialisation needed (the call zeroes it; it holds nothing of use afterwards).  a, b
 *          16-byte aligned; temp_exp, seg_max, col_mul, col_add 4-byte aligned, seg_arg 2-byte
 *          aligned.  Refused without a launch: seg_len < 1 or > 65535, C not a whole number of
 *          segments, both outputs null, null or misaligned pointers, only one of col_mul / col_add.
 * reduce : out[a,b] = sum_k weights[a*len+k] * seg_max[(a*len+k), b]  ([samples, nseg] or
 *          transposed) - the masked mean over text tokens (:807) / mean over image tokens (:811).
 * nce_fwd/bwd : row-wise InfoNCE / DCL on an [R,C] fp32 similarity matrix (R local texts, C all
 *          images, positive of row x at column x + diag_off) (:821-847); bwd writes
 *          g = *gscale * (softmax_row - [positive]).  row_valid (optional, one byte per row): a
 *          row with row_valid[x] == 0 (the image-to-text row of a caption without valid tokens)
 *          adds no loss, gets g = 0 and lse = 0 - as in the reference, where that row is
 *          exp(-inf) = 0 in both the positive and the denominator.
 * expand16 : rows [row0,row0+rows) of the backward operand G[R,C] (bf16): at the argmax column
 *          of each (row, sample) the value *temp_exp * wmat[row/rows_per_sample, sample] *
 *          rowscale[row], zero elsewhere.  seg_arg (from segmax_arg16) holds rows
 *          [row0, row0 + rows) only: row r of G reads seg_arg[(r - row0) * nseg + y], while wmat
 *          and rowscale are indexed by the global row.  d rows = G @ b and d cols += G^T @ a then
 *          run on xclip_gemm_bf16; d loss / d log temperature is sum(d t2i * t2i) +
 *          sum(d i2t * i2t) over the [B,B] matrices.  1 <= seg_len <= 65535; g is [rows, ldg]
 *          with ldg % 8 == 0 and ldg >= nseg * seg_len, 16-byte aligned; seg_arg 2-byte aligned;
 *          row0 >= 0.  Columns [nseg * seg_len, roundup8(nseg * seg_len)) are written as zeros,
 *          the rest of the row is left alone; the gradient GEMMs take G[:, :nseg * seg_len] and
 *          never read past it. */
int xclip_filip_segmax_arg16(const void* a, const void* b, int R, int C, int D,
                             const float* temp_exp, int seg_len, const float* col_mul,
                             const float* col_add, float* seg_max, uint16_t* seg_arg, void* keys,
                             xclip_stream_t stream);
int xclip_filip_reduce(const float* seg_max, const float* weights, int samples, int len, int nseg,
                       float* out, int transpose_out, xclip_stream_t stream);
int xclip_filip_nce_fwd(const float* s, int R, int C, int diag_off, int dcl,
                        const unsigned char* row_valid, float* lse, float* loss_accum,
                        float loss_scale, xclip_stream_t stream);
int xclip_filip_nce_bwd(const float* s, const float* lse, int R, int C, int diag_off, int dcl,
                        const unsigned char* row_valid, const float* gscale, float* g,
                        xclip_stream_t stream);
int xclip_filip_expand16(const uint16_t* seg_arg, const float* wmat, const float* rowscale,
                         const float* temp_exp, int row0, int rows, int rows_per_sample,
                         int seg_len, int nseg, void* g, int64_t ldg, xclip_stream_t stream);

/* ---- FILIP with augmented views (x_clip/x_clip.py:625-650, :797-811, :821-868) ----------------
 * s f32 [m*b, n*B] with row stride lds >= n*B: every (text view i, image view j) block is the [b, B]
 * similarity of this rank's b texts of view i against the B images of view j (all ranks).  Row
 * i*b + x; block j's global sample k lives at column
 *     (k / col_run) * n * col_run + j * col_run + k % col_run
 * with col_run = b (rank-major: the column order of the image-token all-gather, rank r's n views
 * in turn) or col_run = B (view-major); col_run must be b or B.  The positive of row i*b + x in
 * every block is k = x + diag_off (this rank's r*b), 0 <= diag_off <= B - b.
 * blocks_fwd : lse[(i*b + x) * n + j] = log sum_k exp(s) over block (i, j) (the positive left out
 *          when dcl; dcl with B == 1 gives lse = ln(1e-20), the reference's empty denominator);
 *          *loss_accum += sum over rows and blocks of block_w[i*n + j] * (lse - s[positive])
 *          (loss_accum may be NULL).  block_w: DEVICE f32 [m*n], each block's loss weight (scale
 *          included).  row_valid (optional, one byte per row [m*b]): as for nce_fwd, a row with
 *          row_valid 0 adds no loss, has lse 0 in every block.  One launch for the whole matrix.
 * blocks_bwd : g[row, col] = *gscale * block_w[block] * (exp(s - lse) [not on the positive when
 *          dcl] - [positive]) for g f32 [m*b, ldg >= n*B]; rows with row_valid 0 get g = 0.
 * Both refuse without a launch: bad sizes, col_run not b or B, diag_off outside [0, B - b], a
 * matrix of 2^31 or more elements. */
int xclip_filip_nce_blocks_fwd(const float* s, int64_t lds, int m, int n, int b, int B, int col_run,
                               int diag_off, int dcl, const unsigned char* row_valid,
                               const float* block_w, float* lse, float* loss_accum,
                               xclip_stream_t stream);
int xclip_filip_nce_blocks_bwd(const float* s, int64_t lds, const float* lse, int m, int n, int b,
                               int B, int col_run, int diag_off, int dcl,
                               const unsigned char* row_valid, const float* block_w,
                               const float* gscale, float* g, int64_t ldg, xclip_stream_t stream);

/* ---- text embedding (x_clip/x_clip.py:320-332) ---------------------------------------------
 * fwd: out bf16 [B, n+1, d]: out[b,0] = cls, out[b,1+t] = tok[ids[b,t]] + pos[t]  (fp32 tables,
 *      ids int64 [B,n]; an id outside [0, vocab) traps the kernel - the launch
 *      fails like nn.Embedding's device-side assert, nothing is clamped silently).
 * bwd: dx bf16 [B, n+1, d] -> dtok f32 [vocab,d] (+=, vector reductions), dpos f32 [>=n, d] (+=),
 *      dcls f32 [d] (+=).  All three gradients must be zero-initialised by the caller. */
int xclip_text_embed_fwd(const int64_t* ids, const float* tok, const float* pos, const float* cls,
                         void* out, int B, int n, int d, int vocab, xclip_stream_t stream);
int xclip_text_embed_bwd(const int64_t* ids, const void* dx, float* dtok, float* dpos, float* dcls,
                         int B, int n, int d, int vocab, xclip_stream_t stream);

/* ---- fused feed-forward block (x_clip/x_clip.py:180-199) on the wgmma GEMM ----------------------
 * FeedForward = Linear(d, 8d) -> GEGLU -> LayerNorm(4d) -> Linear(4d, d), + residual (:289).
 *   ff_permute_cast : bf16 copy of net.0.weight [8d, d] with rows reordered so that a 128-row tile
 *                     holds 64 value rows and the 64 MATCHING gate rows.
 *   ff_scale_cast   : w2g = bf16(net.4.weight [d, 4d] * net.2.g [4d]) and colvec[j] = sum_k w2g[j,k].
 *   ff_up           : u = [value | gate] bf16 [M, 8d] (reference layout, kept for the backward),
 *                     hp = value * gelu(gate) bf16 [M, 4d], rowsum[r, box] = (sum hp, sum hp^2) of
 *                     every 64-column box (rowsum f32 [M, 4d/64, 2], fully overwritten: no atomics,
 *                     bit-reproducible) - one GEMM, GEGLU in its epilogue.
 *                     u may be NULL (forward-only sweeps: two thirds of the output traffic saved).
 *   ff_down         : (mean_r, rstd_r) from rowsum; out = rstd_r * (hp w2g^T - mean_r * colvec) + residual
 *                     (== LN(hp) g W2^T + x1),
 *                     acc_out = bf16(hp w2g^T), stats[r] = (mean, rstd) - one GEMM.
 *   ff_bwd_prep     : dxs = bf16(dx * rstd_r) [M, d]; vsum[j] += sum_r dxs[r,j] * mean_r; with acc and
 *                     colvec also ab[r] = (mean_k gdh, mean_k gdh*hn) - the two row means of the
 *                     LayerNorm backward, from d-wide data only (gdh = dx w2g is never formed here).
 *   ff_bwd          : du [M, 8d] = backward of LayerNorm(4d) + GEGLU fused into the dgrad GEMM
 *                     gdh = dx w2g (reads u, stats, ab; the [M, 4d] gradient never exists in HBM).
 *   ff_w2_grad_post : in place on raw = dxs^T hp (f32 [d, 4d]): dW2[j,k] = g[k] * (raw[j,k] - vsum[j]);
 *                     with w2/dg also dg[k] += sum_j (raw[j,k] - vsum[j]) * w2[j,k] (gain gradient).
 * d in 256*{1,2,3,4}; all matrices row-major, bf16 unless stated.  Matrices, rowsum and colvec must
 * be 16-byte aligned; stats and ab (read and written as float pairs) 8-byte aligned. */
int xclip_ff_permute_cast(const float* w1, void* out, int d, xclip_stream_t stream);
int xclip_ff_scale_cast(const float* w2, const float* g, void* w2g, float* colvec, int d,
                        xclip_stream_t stream);
int xclip_ff_up(const void* x, int64_t ldx, const void* w1p, void* u, int64_t ldu, void* hp,
                int64_t ldhp, float* rowsum, int M, int d, xclip_stream_t stream);
int xclip_ff_down(const void* hp, int64_t ldhp, const void* w2g, const float* colvec,
                  const float* rowsum, const void* residual, int64_t ldr, void* out, int64_t ldo,
                  void* acc_out, int64_t ldacc, float* stats, float eps, int M, int d,
                  xclip_stream_t stream);
int xclip_ff_bwd_prep(const void* dx, int64_t lddx, const float* stats, const void* acc, int64_t ldacc,
                      const float* colvec, void* dxs, float* vsum, float* ab, int rows, int d,
                      xclip_stream_t stream);
int xclip_ff_bwd(const void* dx, int64_t lddx, const void* w2g, const void* u, int64_t ldu,
                 const float* stats, const float* ab, void* du, int64_t lddu, int M, int d,
                 xclip_stream_t stream);
int xclip_ff_w2_grad_post(float* raw, const float* vsum, const float* g, const float* w2, float* dg,
                          int d, xclip_stream_t stream);

/* ---- fused AdamW (SURVEY 8f: the optimizer step behind the gradient all-reduce; the reference
 * leaves optimisation to the user, README.md:44-58) over one flat f32 buffer; identical update rule to
 * torch.optim.AdamW (decoupled decay, bias correction with `step` >= 1); g is read as g*grad_scale. */
int xclip_adamw_step(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1,
                     float beta2, float eps, float weight_decay, int step, float grad_scale,
                     xclip_stream_t stream);

/* ---- patch-embedding front end (x_clip/x_clip.py:356-359 patchify, :134-151 PatchDropout) -------
 * patchify_gather : img f32 [B,C,H,W] -> bf16 [B*k, patch*patch*C] rows in the reference's
 *                   (p1 p2 c) order for the patches keep[b, j] (int64 [B,k]; NULL = all k = n patches,
 *                   in order): only kept patches are read and embedded.  patch*patch*C %% 8 == 0.
 * patchify_gather_rows: the same for any patch*patch*C, into rows of stride ldo (ldo %% 8 == 0,
 *                   ldo >= patch*patch*C, out 16-byte aligned); columns patch*patch*C .. ldo-1 are
 *                   written as zeros, so the rows are a GEMM operand with K = ldo.  patchify_gather is
 *                   this call with ldo = patch*patch*C.
 * patchify_scatter: the inverse (the image gradient): src f32 [B*k, patch*patch*C] (row stride lds, rows
 *                   in the gather's order, (p1 p2 c) inside a row) -> img_grad f32 [B,C,H,W].  Every
 *                   element is written: pixels of the patch keep[b, j] take row b*k + j, pixels of
 *                   patches absent from keep[b, :] are 0 (allocate img_grad uninitialised).  The indices
 *                   of one sample must be distinct (PatchDropout draws them with topk), so no pixel has
 *                   two sources and no atomics are used; with duplicates the result is unspecified.
 *                   src and img_grad 16-byte aligned, lds %% 4 == 0, patch*patch*C %% 8 == 0,
 *                   0 < k <= n patches; the other refusals are the gather's.
 * patchify_scatter_rows: the same for any patch*patch*C; reads only the first patch*patch*C columns
 *                   of each src row (lds >= patch*patch*C).  patchify_scatter is this call after its
 *                   patch*patch*C %% 8 check.
 * scatter_add_rows: dst f32 [V,d] rows idx[r] (or r %% period) += src bf16 [rows,d]  (gradient of the
 *                   gathered position table);  colsum_rows: dst[d] += column sums (bias gradient). */
int xclip_patchify_gather(const float* img, int B, int C, int H, int W, int patch, const int64_t* keep,
                          int k, void* out, xclip_stream_t stream);
int xclip_patchify_scatter(const float* src, int64_t lds, int B, int C, int H, int W, int patch,
                           const int64_t* keep, int k, float* img_grad, xclip_stream_t stream);
int xclip_patchify_gather_rows(const float* img, int B, int C, int H, int W, int patch,
                               const int64_t* keep, int k, void* out, int64_t ldo, xclip_stream_t stream);
int xclip_patchify_scatter_rows(const float* src, int64_t lds, int B, int C, int H, int W, int patch,
                                const int64_t* keep, int k, float* img_grad, xclip_stream_t stream);
int xclip_scatter_add_rows(const int32_t* idx, int period, const void* src, int64_t lds, float* dst,
                           int64_t rows, int d, int V, xclip_stream_t stream);
int xclip_colsum_rows(const void* src, int64_t lds, float* dst, int64_t rows, int d,
                      xclip_stream_t stream);

/* ---- rotary position embedding (x_clip/x_clip.py:155-176, applied to q, k and v at :221-223) ----
 * In place on the bf16 qkv buffer [rows, ld] (rows = B*n tokens, position = row %% n): in each of
 * the `nslices` consecutive 64-wide head slices the first 32 features are rotated pairwise
 * (j with j+16) by angle[pos, j]; cos_tab / sin_tab f32 [n, 16].  inverse != 0: the transposed
 * rotation (backward, applied to dq | dk | dv). */
int xclip_rotary_inplace(void* qkv, int64_t ld, int64_t rows, int n, int nslices,
                         const float* cos_tab, const float* sin_tab, int inverse,
                         xclip_stream_t stream);

/* ---- SimCLR augmentation of the visual SSL losses (x_clip/visual_ssl.py:24-45) ---------------------
 * One decision per call for the whole batch, applied to x f32 [B, C, H, W] (contiguous) in this order:
 *   colour jitter: ops[k] = 0 brightness, 1 contrast, 2 saturation, 3 hue, -1 none, applied for
 *       k = 0..3 with torchvision's fp32 arithmetic: _blend(img, other, factor[op]) with weights
 *       factor[op] and one_minus[op] (= fp32(1 - factor[op]), rounded from double as torchvision does)
 *       and its clamp to [0, 1]; contrast blends with the per-image grayscale mean of the image as it is
 *       at that point (xclip_augment_mean); hue is _rgb2hsv, (h + factor[3]) % 1, _hsv2rgb;
 *   grayscale != 0: rgb_to_grayscale (0.2989 / 0.587 / 0.114) into all 3 channels;
 *   flip != 0: horizontal flip;
 *   blur != 0: 3x3 cross-correlation with blur_kernel (row-major) and reflect padding at the image
 *       border, so pixels at the crop's edge see their neighbours outside the crop;
 *   crop (top, left, height, width), resized to out_h x out_w by ATen's antialiased bilinear
 *       (align_corners = False); the crop lies inside the image and is no larger than the output;
 *   normalize != 0: (v - mean[c]) / std[c].
 * The colour stages and Normalize need C == 3.  Offsets are 64-bit (any B * C * H * W).
 * mean  : out f32 [B], the grayscale mean per image of the jitter's ops before contrast (C == 3).
 *         Fixed-order reduction: deterministic.
 * apply : out f32 [B, C, out_h, out_w]; mean is read only when ops contain contrast (then required).
 * Both return XCLIP_ERR_INVALID without launching for: a null or misaligned (4-byte) pointer, H or W
 * < 2, a crop outside the image or larger than the output, colour stages at C != 3. */
typedef struct xclip_augment_params {
  int32_t ops[4];
  float factor[4];
  float one_minus[4];
  int32_t grayscale, flip, blur, normalize;
  float blur_kernel[9];
  float mean[3], std[3];
  int32_t top, left, height, width;
  int32_t out_h, out_w;
} xclip_augment_params;
int xclip_augment_mean(const float* x, int B, int C, int H, int W, const xclip_augment_params* params,
                       float* mean, xclip_stream_t stream);
int xclip_augment_apply(const float* x, int B, int C, int H, int W, const xclip_augment_params* params,
                        const float* mean, float* out, xclip_stream_t stream);

#ifdef __cplusplus
}
#endif

#endif /* XCLIP_B200_H_ */
