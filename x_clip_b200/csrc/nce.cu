// All-pairs similarity + InfoNCE / DCL loss (reference x_clip/x_clip.py:813-847) on top of the
// wgmma GEMM mainloop (gemm.cuh) with loss-specific epilogues:
//
//   forward  : s = exp(temperature) * A B^T is produced tile by tile in registers and immediately
//              reduced to per-row, per-column-block (running max, sum of exp(s - max)) pairs;
//              the B_l x B_g logits matrix is never written.  A finalize kernel turns the partials into log-denominators
//              and the loss contribution  scale * sum_r (lse_r - s_rr).
//   backward : the same tiles are recomputed and turned into
//              g = w_row*exp(s - lse_row) + w_col*exp(s - lse_col) - w_diag*[positive]
//              (bf16, the only place a B_l x B_g array exists) which then feeds the plain GEMM
//              dZ = alpha * g @ Y.  sum(g*s) accumulates d loss / d temperature.
//
// Rows are the LOCAL samples of one modality, columns ALL samples of the other one, so under
// data parallelism each rank evaluates only its B_g/W row block (SURVEY.md 8e) instead of the
// reference's redundant full matrix.
//
// The pairwise sigmoid loss (xclip_sigmoid_*) runs on the same operands and row blocks with
// epilogues of its own.  The MLM head's cross-entropy over the vocabulary (xclip_vocab_ce_*, end of
// file) is the same softmax with a bias, a label column as the positive and no temperature.
#include "gemm.cuh"
#include "host.h"

namespace xclip {

constexpr float kLogEmptyDenominator = -46.051701859880914f;   // ln(1e-20)

__global__ void __launch_bounds__(1024)
nce_finalize_kernel(const float* __restrict__ part, int nblk, const float* __restrict__ pos,
                    int rows, const float* __restrict__ alpha_dev, float* __restrict__ lse,
                    float* __restrict__ loss_accum, float scale) {
  __shared__ float red[32];
  float local = 0.f;
  const float2* part2 = reinterpret_cast<const float2*>(part);
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    float m = -INFINITY;
    for (int k = 0; k < nblk; ++k) m = fmaxf(m, part2[(long long)k * rows + r].x);
    float s = 0.f;
    for (int k = 0; k < nblk; ++k) {
      const float2 ps = part2[(long long)k * rows + r];
      if (ps.x > -INFINITY) s += ps.y * exp2f(ps.x - m);
    }
    // Every partial empty: a DCL row whose only column is its own positive (global batch 1).  The
    // reference adds 1e-20 inside the log (x_clip.py:51-52); take its value instead of -inf.
    const float l = m > -INFINITY ? (m + log2f(s)) * 0.6931471805599453f : kLogEmptyDenominator;
    lse[r] = l;
    local += l - pos[r];
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0 && loss_accum != nullptr) atomicAdd(loss_accum, v * scale);
  }
}

template <int BLOCK_N, int EPI>
static int launch_nce(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int grid,
                      cudaStream_t stream) {
  using S = GemmSmem<BLOCK_N>;
  auto kern = gemm_bf16_kernel<BLOCK_N, kMajorK, kMajorK, EPI>;
  {
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), S::kTotal);
    if (rc_attr) return rc_attr;
  }
  kern<<<grid, kGemmThreads, S::kTotal, stream>>>(tmA, tmB, p, CUtensorMap{}, CUtensorMap{});
  XCLIP_LAUNCH_CHECK("gemm_bf16_kernel<nce>");
  return XCLIP_OK;
}

static int nce_common(const void* a, const void* b, int R, int C, int D, GemmParams* p,
                      CUtensorMap* tmA, CUtensorMap* tmB, int* block_n, int* grid) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(a && b, "nce: null latents");
  XCLIP_REQUIRE(R > 0 && C > 0 && D > 0 && D % 8 == 0, "nce: bad sizes R=%d C=%d D=%d", R, C, D);
  XCLIP_REQUIRE(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0,
                "nce: misaligned latents");
  *block_n = C >= 256 ? 256 : 128;
  rc = encode_2d_bf16(tmA, a, (uint64_t)D, (uint64_t)R, (uint64_t)D, 64, kGemmBlockM);
  if (rc) return rc;
  rc = encode_2d_bf16(tmB, b, (uint64_t)D, (uint64_t)C, (uint64_t)D, 64, (uint32_t)*block_n);
  if (rc) return rc;
  GemmParams z = {};
  *p = z;
  p->M = R; p->N = C; p->K = D; p->split_k = 1;
  p->raster_m_fast = 1;   // latents of the local rows stay in L2, all columns stream once
  const long long tiles =
      (long long)((R + kGemmBlockM - 1) / kGemmBlockM) * ((C + *block_n - 1) / *block_n);
  *grid = (int)(tiles < num_sms() ? tiles : num_sms());
  return XCLIP_OK;
}

}  // namespace xclip

using namespace xclip;

extern "C" int xclip_nce_num_col_blocks(int C) { return C >= 256 ? (C + 255) / 256 : (C + 127) / 128; }

extern "C" int xclip_nce_fwd(const void* a, const void* b, int R, int C, int D,
                             const float* temp_exp,
                             int diag_offset, int dcl, float* part_ws, float* pos, float* lse,
                             float* loss_accum, float loss_scale, xclip_stream_t stream) {
  GemmParams p;
  CUtensorMap tmA, tmB;
  int block_n = 0, grid = 0;
  int rc = nce_common(a, b, R, C, D, &p, &tmA, &tmB, &block_n, &grid);
  if (rc) return rc;
  XCLIP_REQUIRE(part_ws && pos && lse && temp_exp, "nce_fwd: null workspace/output");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(part_ws) & 7) == 0,
                "nce_fwd: part_ws must be 8-byte aligned (float2 partials)");
  XCLIP_REQUIRE(diag_offset >= 0 && diag_offset + R <= C, "nce_fwd: positives outside the columns");
  p.alpha_dev = temp_exp; p.diag_offset = diag_offset; p.dcl = dcl;
  p.nce_part = part_ws; p.nce_pos = pos;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  rc = block_n == 256 ? launch_nce<256, EPI_NCE_FWD>(tmA, tmB, p, grid, s)
                      : launch_nce<128, EPI_NCE_FWD>(tmA, tmB, p, grid, s);
  if (rc) return rc;
  const int nblk = xclip_nce_num_col_blocks(C);
  int fgrid = (R + 1023) / 1024;
  if (fgrid > num_sms()) fgrid = num_sms();
  nce_finalize_kernel<<<fgrid, 1024, 0, s>>>(part_ws, nblk, pos, R, temp_exp, lse, loss_accum,
                                             loss_scale);
  XCLIP_LAUNCH_CHECK("nce_finalize_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_nce_bwd(const void* a, const void* b, int R, int C, int D,
                             const float* temp_exp, int diag_offset, int dcl,
                             const float* lse_row, const float* lse_col, float w_row, float w_col,
                             float w_diag, const float* gscale, void* g, int64_t ldg,
                             float* dtemp, xclip_stream_t stream) {
  GemmParams p;
  CUtensorMap tmA, tmB;
  int block_n = 0, grid = 0;
  int rc = nce_common(a, b, R, C, D, &p, &tmA, &tmB, &block_n, &grid);
  if (rc) return rc;
  XCLIP_REQUIRE(g && ldg % 8 == 0 && ldg >= (C + 7) / 8 * 8, "nce_bwd: g needs ld >= roundup8(C)");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "nce_bwd: misaligned g");
  XCLIP_REQUIRE((w_row == 0.f || lse_row) && (w_col == 0.f || lse_col), "nce_bwd: missing lse");
  XCLIP_REQUIRE(w_col == 0.f || (reinterpret_cast<uintptr_t>(lse_col) & 15) == 0,
                "nce_bwd: lse_col must be 16-byte aligned (it is read as float4)");
  XCLIP_REQUIRE(temp_exp && gscale, "nce_bwd: temp_exp / gscale device scalars required");
  p.alpha_dev = temp_exp; p.gscale_dev = gscale; p.diag_offset = diag_offset; p.dcl = dcl;
  p.lse_row = lse_row; p.lse_col = lse_col;
  p.w_row = w_row; p.w_col = w_col; p.w_diag = w_diag;
  p.c = g; p.ldc = ldg; p.dtemp = dtemp;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  return block_n == 256 ? launch_nce<256, EPI_NCE_BWD>(tmA, tmB, p, grid, s)
                        : launch_nce<128, EPI_NCE_BWD>(tmA, tmB, p, grid, s);
}

// ---- pairwise sigmoid loss (SigLIP, Zhai et al. 2023) on the same operands, mainloop and row blocks:
// logit l = exp(temperature) * <a_r, b_c> + logit_bias, label +1 on column r + diag_offset, -1 elsewhere.
// No softmax over the batch: the forward sums softplus(-z l) per row, the backward recomputes the tiles
// into g = gscale * (sigmoid(l) - [positive]).  Nothing R x C is written except the bf16 g.

namespace xclip {

// rowloss[r] = sum of the column-block partials of row r in a fixed order; *loss_accum += scale * sum
__global__ void __launch_bounds__(1024)
sigmoid_finalize_kernel(const float* __restrict__ part, int nblk, int rows, float* __restrict__ rowloss,
                        float* __restrict__ loss_accum, float scale) {
  __shared__ float red[32];
  float local = 0.f;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < nblk; ++k) s += part[(long long)k * rows + r];
    rowloss[r] = s;
    local += s;
  }
  local = warp_sum(local);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local;
  __syncthreads();
  if (threadIdx.x < 32) {
    float v = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    v = warp_sum(v);
    if (threadIdx.x == 0 && loss_accum != nullptr) atomicAdd(loss_accum, v * scale);
  }
}

static int sigmoid_check(int R, int C, const float* temp_exp, const float* logit_bias, int diag_offset,
                         const char* what) {
  XCLIP_REQUIRE(temp_exp && logit_bias, "%s: temp_exp / logit_bias device scalars required", what);
  XCLIP_REQUIRE(diag_offset >= 0 && (long long)diag_offset + R <= C,
                "%s: positives outside the columns (diag_offset=%d R=%d C=%d)", what, diag_offset, R, C);
  return XCLIP_OK;
}

}  // namespace xclip

extern "C" int xclip_sigmoid_fwd(const void* a, const void* b, int R, int C, int D, const float* temp_exp,
                                 const float* logit_bias, int diag_offset, float* part_ws, float* rowloss,
                                 float* loss_accum, float loss_scale, xclip_stream_t stream) {
  GemmParams p;
  CUtensorMap tmA, tmB;
  int block_n = 0, grid = 0;
  int rc = nce_common(a, b, R, C, D, &p, &tmA, &tmB, &block_n, &grid);
  if (rc) return rc;
  rc = sigmoid_check(R, C, temp_exp, logit_bias, diag_offset, "sigmoid_fwd");
  if (rc) return rc;
  XCLIP_REQUIRE(part_ws && rowloss, "sigmoid_fwd: null workspace/output");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(part_ws) & 3) == 0, "sigmoid_fwd: misaligned part_ws");
  p.alpha_dev = temp_exp; p.logit_bias = logit_bias; p.diag_offset = diag_offset;
  p.nce_part = part_ws;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  rc = block_n == 256 ? launch_nce<256, EPI_SIG_FWD>(tmA, tmB, p, grid, s)
                      : launch_nce<128, EPI_SIG_FWD>(tmA, tmB, p, grid, s);
  if (rc) return rc;
  const int nblk = xclip_nce_num_col_blocks(C);
  int fgrid = (R + 1023) / 1024;
  if (fgrid > num_sms()) fgrid = num_sms();
  sigmoid_finalize_kernel<<<fgrid, 1024, 0, s>>>(part_ws, nblk, R, rowloss, loss_accum, loss_scale);
  XCLIP_LAUNCH_CHECK("sigmoid_finalize_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_sigmoid_bwd(const void* a, const void* b, int R, int C, int D, const float* temp_exp,
                                 const float* logit_bias, int diag_offset, const float* gscale, void* g,
                                 int64_t ldg, float* dtemp, float* dbias, xclip_stream_t stream) {
  GemmParams p;
  CUtensorMap tmA, tmB;
  int block_n = 0, grid = 0;
  int rc = nce_common(a, b, R, C, D, &p, &tmA, &tmB, &block_n, &grid);
  if (rc) return rc;
  rc = sigmoid_check(R, C, temp_exp, logit_bias, diag_offset, "sigmoid_bwd");
  if (rc) return rc;
  XCLIP_REQUIRE(g && ldg % 8 == 0 && ldg >= (C + 7) / 8 * 8, "sigmoid_bwd: g needs ld >= roundup8(C)");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "sigmoid_bwd: misaligned g");
  XCLIP_REQUIRE(gscale, "sigmoid_bwd: gscale device scalar required");
  p.alpha_dev = temp_exp; p.logit_bias = logit_bias; p.gscale_dev = gscale; p.diag_offset = diag_offset;
  p.c = g; p.ldc = ldg; p.dtemp = dtemp; p.dbias = dbias;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  return block_n == 256 ? launch_nce<256, EPI_SIG_BWD>(tmA, tmB, p, grid, s)
                        : launch_nce<128, EPI_SIG_BWD>(tmA, tmB, p, grid, s);
}

// ---- vocabulary cross-entropy: the MLM head's F.cross_entropy(x W^T + b, labels) on the same
// mainloop.  Rows are the selected token encodings, columns the V vocabulary rows of W; the
// positive of row r is column labels[r] instead of a diagonal.  The forward reuses the InfoNCE
// partials and finalize, so the [R, V] logits are never written.

static int vce_check(const float* bias, const int64_t* labels, const char* what) {
  XCLIP_REQUIRE(labels, "%s: null labels", what);
  XCLIP_REQUIRE(bias == nullptr || (reinterpret_cast<uintptr_t>(bias) & 15) == 0,
                "%s: bias must be 16-byte aligned (it is read as float4)", what);
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(labels) & 7) == 0, "%s: misaligned labels", what);
  return XCLIP_OK;
}

extern "C" int xclip_vocab_ce_fwd(const void* x, const void* w, const float* bias, const int64_t* labels,
                                  int R, int V, int D, float* part_ws, float* pos, float* lse,
                                  float* loss_accum, float loss_scale, xclip_stream_t stream) {
  GemmParams p;
  CUtensorMap tmA, tmB;
  int block_n = 0, grid = 0;
  int rc = nce_common(x, w, R, V, D, &p, &tmA, &tmB, &block_n, &grid);
  if (rc) return rc;
  rc = vce_check(bias, labels, "vocab_ce_fwd");
  if (rc) return rc;
  XCLIP_REQUIRE(part_ws && pos && lse, "vocab_ce_fwd: null workspace/output");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(part_ws) & 7) == 0,
                "vocab_ce_fwd: part_ws must be 8-byte aligned (float2 partials)");
  p.bias = bias; p.labels = reinterpret_cast<const long long*>(labels);
  p.nce_part = part_ws; p.nce_pos = pos;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  rc = block_n == 256 ? launch_nce<256, EPI_VCE_FWD>(tmA, tmB, p, grid, s)
                      : launch_nce<128, EPI_VCE_FWD>(tmA, tmB, p, grid, s);
  if (rc) return rc;
  const int nblk = xclip_nce_num_col_blocks(V);
  int fgrid = (R + 1023) / 1024;
  if (fgrid > num_sms()) fgrid = num_sms();
  nce_finalize_kernel<<<fgrid, 1024, 0, s>>>(part_ws, nblk, pos, R, nullptr, lse, loss_accum, loss_scale);
  XCLIP_LAUNCH_CHECK("nce_finalize_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_vocab_ce_bwd(const void* x, const void* w, const float* bias, const int64_t* labels,
                                  int R, int V, int D, const float* lse, const float* gscale, void* g,
                                  int64_t ldg, xclip_stream_t stream) {
  GemmParams p;
  CUtensorMap tmA, tmB;
  int block_n = 0, grid = 0;
  int rc = nce_common(x, w, R, V, D, &p, &tmA, &tmB, &block_n, &grid);
  if (rc) return rc;
  rc = vce_check(bias, labels, "vocab_ce_bwd");
  if (rc) return rc;
  XCLIP_REQUIRE(g && ldg % 8 == 0 && ldg >= (V + 7) / 8 * 8, "vocab_ce_bwd: g needs ld >= roundup8(V)");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "vocab_ce_bwd: misaligned g");
  XCLIP_REQUIRE(lse && gscale, "vocab_ce_bwd: lse / gscale required");
  p.bias = bias; p.labels = reinterpret_cast<const long long*>(labels);
  p.lse_row = lse; p.gscale_dev = gscale;
  p.c = g; p.ldc = ldg;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  return block_n == 256 ? launch_nce<256, EPI_VCE_BWD>(tmA, tmB, p, grid, s)
                        : launch_nce<128, EPI_VCE_BWD>(tmA, tmB, p, grid, s);
}
