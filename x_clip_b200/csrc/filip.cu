// FILIP fine-grained contrastive loss (reference x_clip/x_clip.py:799-811 + :821-847).
//
//   sim[x,y,t,i] = exp(temperature) * <zt[x,t], zi[y,i]>
//   t2i[x,y] = masked_mean_t max_i sim          i2t[x,y] = mean_i max_t sim (padded t -> -FLT_MAX)
//   loss     = InfoNCE / DCL over rows x of both [B,B] matrices (the reference keeps the
//              [text,image] orientation for i2t as well)
//
// The 6-D similarity tensor (68.7 G elements at cfg4) is never materialised:
//   xclip_filip_segmax : the wgmma GEMM with the EPI_SEGMAX epilogue produces, per token row and
//                        per sample of the other modality, max + argmax over that sample's tokens
//   xclip_filip_reduce : [tokens, B] maxima -> [B, B] similarity (masked mean / mean)
//   xclip_filip_nce_*  : row-wise InfoNCE / DCL on a [B,B] fp32 matrix (warp-shuffle reductions)
//   xclip_filip_expand : backward: one-hot (at the argmax) weighted bf16 operand G[rows, cols]
//                        for a chunk of rows, which then feeds two plain wgmma GEMMs
//                        (d rows = G @ Zcols, d cols += G^T @ Zrows).
#include "gemm.cuh"
#include "host.h"

namespace xclip {

// out[a, b] = sum_k w[a*len + k] * m[(a*len + k) * nseg + b]      (transpose_out: out[b, a])
__global__ void __launch_bounds__(256)
filip_reduce_kernel(const float* __restrict__ m, const float* __restrict__ w, int samples, int len,
                    int nseg, float* __restrict__ out, int transpose_out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;   // segment (other-modality sample)
  const int a = blockIdx.y;                               // this-modality sample
  if (b >= nseg || a >= samples) return;
  float acc = 0.f;
  for (int k = 0; k < len; ++k) {
    const long long r = (long long)a * len + k;
    const float wk = w[r];
    if (wk != 0.f) acc += wk * m[r * nseg + b];          // skip padded tokens (their max may be -FLT_MAX)
  }
  if (transpose_out) out[(long long)b * samples + a] = acc;
  else out[(long long)a * nseg + b] = acc;
}

// one warp per row of an [R,C] fp32 matrix (R local texts x C global images; the positive of row
// x is column x + diag_off): lse (optionally without the positive), loss partial
__global__ void __launch_bounds__(256)
filip_nce_fwd_kernel(const float* __restrict__ s, int R, int C, int diag_off, int dcl,
                     float* __restrict__ lse, float* __restrict__ loss_accum, float scale) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= R) return;
  const float* r = s + (long long)row * C;
  const int pos = row + diag_off;
  float mx = -INFINITY;
  for (int c = lane; c < C; c += 32)
    if (!(dcl && c == pos)) mx = fmaxf(mx, r[c]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c < C; c += 32)
    if (!(dcl && c == pos)) sum += __expf(r[c] - mx);
  sum = warp_sum(sum);
  if (lane == 0) {
    const float l = mx + logf(sum);
    lse[row] = l;
    if (loss_accum) atomicAdd(loss_accum, (l - r[pos]) * scale);
  }
}

// g[x,y] = gscale * (exp(s - lse_x) [skipped on the positive when dcl] - [y == x + diag_off])
__global__ void __launch_bounds__(256)
filip_nce_bwd_kernel(const float* __restrict__ s, const float* __restrict__ lse, int R, int C,
                     int diag_off, int dcl, const float* __restrict__ gscale,
                     float* __restrict__ g) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)R * C) return;
  const int x = (int)(idx / C), y = (int)(idx % C);
  const bool is_pos = (y == x + diag_off);
  float v = 0.f;
  if (!(dcl && is_pos)) v = __expf(s[idx] - lse[x]);
  if (is_pos) v -= 1.f;
  g[idx] = v * __ldg(gscale);
}

// G[r, c] (bf16) for rows [row0, row0+rows): alpha * wmat[sample(r), seg(c)] * rowscale[r] at the
// argmax column of each segment, zero elsewhere.  dtemp += sum_r,seg w * segmax (w without alpha).
__global__ void __launch_bounds__(256)
filip_expand_kernel(const int* __restrict__ seg_arg, const float* __restrict__ seg_max,
                    const float* __restrict__ wmat, const float* __restrict__ rowscale,
                    const float* __restrict__ alpha_dev, int row0, int rows, int rows_per_sample,
                    int seg_len, int nseg, bf16* __restrict__ g, long long ldg,
                    float* __restrict__ dtemp) {
  const float alpha = __ldg(alpha_dev);
  const int vec_per_row = nseg * seg_len / 8;
  float tsum = 0.f;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x;
       v < (long long)rows * vec_per_row; v += (long long)gridDim.x * blockDim.x) {
    const int lr = (int)(v / vec_per_row);
    const int c0 = (int)(v % vec_per_row) * 8;
    const long long r = row0 + lr;
    const int seg = c0 / seg_len;
    const int in_seg = c0 - seg * seg_len;
    const int a = seg_arg[r * nseg + seg];
    uint4 o = make_uint4(0, 0, 0, 0);
    if (a >= in_seg && a < in_seg + 8) {
      const float w = wmat[(r / rows_per_sample) * nseg + seg] * rowscale[r];
      if (w != 0.f) {
        tsum += w * seg_max[r * nseg + seg];
        bf16 vals[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) vals[k] = __float2bfloat16_rn(0.f);
        vals[a - in_seg] = __float2bfloat16_rn(w * alpha);
        o = *reinterpret_cast<uint4*>(vals);
      }
    }
    *reinterpret_cast<uint4*>(g + lr * ldg + c0) = o;
  }
  if (dtemp != nullptr) {
    tsum = warp_sum(tsum);
    if ((threadIdx.x & 31) == 0 && tsum != 0.f) atomicAdd(dtemp, tsum);
  }
}

}  // namespace xclip

using namespace xclip;

extern "C" int xclip_filip_segmax(const void* a, const void* b, int R, int C, int D,
                                  const float* temp_exp, int seg_len, const float* col_mul,
                                  const float* col_add, float* seg_max, int* seg_arg,
                                  xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(a && b && temp_exp && seg_max && seg_arg, "filip_segmax: null pointer");
  XCLIP_REQUIRE(R > 0 && C > 0 && D > 0 && D % 8 == 0, "filip_segmax: bad sizes");
  XCLIP_REQUIRE(seg_len % 16 == 0 && seg_len <= 256 && C % seg_len == 0,
                "filip_segmax: tokens per sample (%d) must be a multiple of 16, <= 256", seg_len);
  XCLIP_REQUIRE((col_mul == nullptr) == (col_add == nullptr), "filip_segmax: mask tables mismatch");
  XCLIP_REQUIRE(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0,
                "filip_segmax: misaligned latents");
  CUtensorMap tmA, tmB;
  rc = encode_2d_bf16(&tmA, a, (uint64_t)D, (uint64_t)R, (uint64_t)D, 64, kGemmBlockM);
  if (rc) return rc;
  rc = encode_2d_bf16(&tmB, b, (uint64_t)D, (uint64_t)C, (uint64_t)D, 64, 256);
  if (rc) return rc;
  GemmParams p = {};
  p.M = R; p.N = C; p.K = D; p.split_k = 1;
  p.raster_m_fast = (R <= C) ? 1 : 0;
  p.alpha_dev = temp_exp;
  p.seg_len = seg_len;
  p.n_tile_stride = (256 / seg_len) * seg_len;
  p.n_segs = C / seg_len;
  p.col_mul = col_mul; p.col_add = col_add;
  p.seg_max = seg_max; p.seg_arg = seg_arg;
  const long long tiles = (long long)((R + kGemmBlockM - 1) / kGemmBlockM) *
                          ((C + p.n_tile_stride - 1) / p.n_tile_stride);
  const int grid = (int)(tiles < num_sms() ? tiles : num_sms());
  using S = GemmSmem<256>;
  auto kern = gemm_bf16_kernel<256, kMajorK, kMajorK, EPI_SEGMAX>;
  {
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), S::kTotal);
    if (rc_attr) return rc_attr;
  }
  kern<<<grid, kGemmThreads, S::kTotal, reinterpret_cast<cudaStream_t>(stream)>>>(tmA, tmB, p);
  XCLIP_LAUNCH_CHECK("gemm_bf16_kernel<segmax>");
  return XCLIP_OK;
}

extern "C" int xclip_filip_reduce(const float* seg_max, const float* weights, int samples, int len,
                                  int nseg, float* out, int transpose_out, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(seg_max && weights && out && samples > 0 && len > 0 && nseg > 0,
                "filip_reduce: bad arguments");
  dim3 grid((nseg + 255) / 256, samples);
  filip_reduce_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      seg_max, weights, samples, len, nseg, out, transpose_out);
  XCLIP_LAUNCH_CHECK("filip_reduce_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_filip_nce_fwd(const float* s, int R, int C, int diag_off, int dcl, float* lse,
                                   float* loss_accum, float loss_scale, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(s && lse && R > 0 && C > 0 && diag_off >= 0 && diag_off + R <= C,
                "filip_nce_fwd: bad arguments");
  filip_nce_fwd_kernel<<<(R + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      s, R, C, diag_off, dcl, lse, loss_accum, loss_scale);
  XCLIP_LAUNCH_CHECK("filip_nce_fwd_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_filip_nce_bwd(const float* s, const float* lse, int R, int C, int diag_off,
                                   int dcl, const float* gscale, float* g, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(s && lse && gscale && g && R > 0 && C > 0, "filip_nce_bwd: bad arguments");
  const long long n = (long long)R * C;
  filip_nce_bwd_kernel<<<(int)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      s, lse, R, C, diag_off, dcl, gscale, g);
  XCLIP_LAUNCH_CHECK("filip_nce_bwd_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_filip_expand(const int* seg_arg, const float* seg_max, const float* wmat,
                                  const float* rowscale, const float* temp_exp, int row0, int rows,
                                  int rows_per_sample, int seg_len, int nseg, void* g, int64_t ldg,
                                  float* dtemp, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(seg_arg && seg_max && wmat && rowscale && temp_exp && g, "filip_expand: null pointer");
  XCLIP_REQUIRE(rows > 0 && rows_per_sample > 0 && seg_len % 8 == 0 && nseg > 0 &&
                    ldg >= (int64_t)nseg * seg_len && ldg % 8 == 0,
                "filip_expand: bad sizes");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "filip_expand: misaligned g");
  const long long vecs = (long long)rows * nseg * seg_len / 8;
  long long blocks = (vecs + 255) / 256;
  if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
  filip_expand_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      seg_arg, seg_max, wmat, rowscale, temp_exp, row0, rows, rows_per_sample, seg_len, nseg,
      reinterpret_cast<bf16*>(g), ldg, dtemp);
  XCLIP_LAUNCH_CHECK("filip_expand_kernel");
  return XCLIP_OK;
}
