// FILIP fine-grained contrastive loss (reference x_clip/x_clip.py:799-811 + :821-847).
//
//   sim[x,y,t,i] = exp(temperature) * <zt[x,t], zi[y,i]>
//   t2i[x,y] = masked_mean_t max_i sim          i2t[x,y] = mean_i max_t sim (padded t -> -FLT_MAX)
//   loss     = InfoNCE / DCL over rows x of both [B,B] matrices (the reference keeps the
//              [text,image] orientation for i2t as well)
//
// The 6-D similarity tensor (68.7 G elements at cfg4) is never materialised:
//   xclip_filip_segmax_arg16 : the wgmma GEMM with the EPI_SEGMAX epilogue produces, per token row
//                        and per sample of the other modality, max + 16-bit argmax over that
//                        sample's tokens, for any token count up to 65535 (256-column tiles,
//                        samples cut by a tile edge merged through 64-bit keys, then unpacked)
//   xclip_filip_reduce : [tokens, B] maxima -> [B, B] similarity (masked mean / mean)
//   xclip_filip_nce_*  : row-wise InfoNCE / DCL on a [B,B] fp32 matrix (warp-shuffle reductions)
//   xclip_filip_expand16 : backward: one-hot (at the argmax) weighted bf16 operand G[rows, cols]
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
// x is column x + diag_off): lse (optionally without the positive), loss partial.
// row_valid (optional): a row with row_valid[x] == 0 - the image-to-text row of a caption without
// any valid token - has no loss term and no gradient (the reference's row is exp(-inf) = 0 in the
// positive and in the denominator alike); its lse is written as 0.
__global__ void __launch_bounds__(256)
filip_nce_fwd_kernel(const float* __restrict__ s, int R, int C, int diag_off, int dcl,
                     const unsigned char* __restrict__ row_valid, float* __restrict__ lse,
                     float* __restrict__ loss_accum, float scale) {
  const int lane = threadIdx.x & 31;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= R) return;
  if (row_valid != nullptr && !row_valid[row]) {          // warp-uniform
    if (lane == 0) lse[row] = 0.f;
    return;
  }
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

// g[x,y] = gscale * (exp(s - lse_x) [skipped on the positive when dcl] - [y == x + diag_off]);
// rows with row_valid[x] == 0 get g = 0 (see filip_nce_fwd_kernel)
__global__ void __launch_bounds__(256)
filip_nce_bwd_kernel(const float* __restrict__ s, const float* __restrict__ lse, int R, int C,
                     int diag_off, int dcl, const unsigned char* __restrict__ row_valid,
                     const float* __restrict__ gscale, float* __restrict__ g) {
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)R * C) return;
  const int x = (int)(idx / C), y = (int)(idx % C);
  if (row_valid != nullptr && !row_valid[x]) {
    g[idx] = 0.f;
    return;
  }
  const bool is_pos = (y == x + diag_off);
  float v = 0.f;
  if (!(dcl && is_pos)) v = __expf(s[idx] - lse[x]);
  if (is_pos) v -= 1.f;
  g[idx] = v * __ldg(gscale);
}

// Block-structured InfoNCE / DCL for augmented views: s [m*b, n*B] (row stride lds) holds one [b, B]
// block per (text view i, image view j).  Rows i*b + x; block j's global sample k sits at column
// filip_block_col(j, k): runs of col_run consecutive samples, the n views' runs interleaved (col_run = b:
// the rank-major order of the image-token all-gather; col_run = B: view-major).  The positive of row
// i*b + x in every block is k = x + diag_off.  lse is [m*b, n], one entry per (row, block).
__device__ __forceinline__ long long filip_block_col(int j, int k, int n, int col_run) {
  return (long long)(k / col_run) * n * col_run + (long long)j * col_run + k % col_run;
}

// one warp per (row, block); block weights w_blk[i*n + j] carry the loss scale of each block
__global__ void __launch_bounds__(256)
filip_nce_blocks_fwd_kernel(const float* __restrict__ s, long long lds, int m, int n, int b, int B,
                            int col_run, int diag_off, int dcl, const unsigned char* __restrict__ row_valid,
                            const float* __restrict__ w_blk, float* __restrict__ lse,
                            float* __restrict__ loss_accum) {
  const int lane = threadIdx.x & 31;
  const long long wid = blockIdx.x * (long long)(blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= (long long)m * b * n) return;
  const int row = (int)(wid / n), j = (int)(wid % n);
  if (row_valid != nullptr && !row_valid[row]) {          // warp-uniform
    if (lane == 0) lse[wid] = 0.f;
    return;
  }
  const float* r = s + (long long)row * lds;
  const int pos = row % b + diag_off;
  float mx = -INFINITY;
  for (int k = lane; k < B; k += 32)
    if (!(dcl && k == pos)) mx = fmaxf(mx, r[filip_block_col(j, k, n, col_run)]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int k = lane; k < B; k += 32)
    if (!(dcl && k == pos)) sum += __expf(r[filip_block_col(j, k, n, col_run)] - mx);
  sum = warp_sum(sum);
  if (lane == 0) {
    // DCL over a global batch of 1 leaves the denominator empty: the reference's log(0 + 1e-20)
    const float l = (dcl && B == 1) ? logf(1e-20f) : mx + logf(sum);
    lse[wid] = l;
    if (loss_accum) {
      const float w = w_blk[(row / b) * n + j];
      atomicAdd(loss_accum, (l - r[filip_block_col(j, pos, n, col_run)]) * w);
    }
  }
}

// g[row, col] = *gscale * w_blk[block] * (exp(s - lse[row, j]) [skipped on the positive when dcl]
// - [positive]); rows with row_valid[row] == 0 get g = 0.  g is [m*b, ldg].
__global__ void __launch_bounds__(256)
filip_nce_blocks_bwd_kernel(const float* __restrict__ s, long long lds, const float* __restrict__ lse,
                            int m, int n, int b, int B, int col_run, int diag_off, int dcl,
                            const unsigned char* __restrict__ row_valid, const float* __restrict__ w_blk,
                            const float* __restrict__ gscale, float* __restrict__ g, long long ldg) {
  const int C = n * B;
  const long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (idx >= (long long)m * b * C) return;
  const int row = (int)(idx / C), col = (int)(idx % C);
  float* out = g + (long long)row * ldg + col;
  if (row_valid != nullptr && !row_valid[row]) {
    *out = 0.f;
    return;
  }
  const int run = n * col_run;
  const int j = (col % run) / col_run;
  const int k = (col / run) * col_run + col % col_run;
  const bool is_pos = (k == row % b + diag_off);
  float v = 0.f;
  if (!(dcl && is_pos)) v = __expf(s[(long long)row * lds + col] - lse[(long long)row * n + j]);
  if (is_pos) v -= 1.f;
  *out = v * (__ldg(gscale) * w_blk[(row / b) * n + j]);
}

// G[r, c] (bf16) for rows [row0, row0+rows): alpha * wmat[sample(r), seg(c)] * rowscale[r] at the
// argmax column of each segment, zero elsewhere.  seg_arg holds rows [row0, row0 + rows) only.
__global__ void __launch_bounds__(256)
filip_expand_kernel(const unsigned short* __restrict__ seg_arg, const float* __restrict__ wmat,
                    const float* __restrict__ rowscale, const float* __restrict__ alpha_dev, int row0,
                    int rows, int rows_per_sample, int seg_len, int nseg, bf16* __restrict__ g,
                    long long ldg) {
  const float alpha = __ldg(alpha_dev);
  const int vec_per_row = nseg * seg_len / 8;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x;
       v < (long long)rows * vec_per_row; v += (long long)gridDim.x * blockDim.x) {
    const int lr = (int)(v / vec_per_row);
    const int c0 = (int)(v % vec_per_row) * 8;
    const long long r = row0 + lr;
    const int seg = c0 / seg_len;
    const int in_seg = c0 - seg * seg_len;
    const int a = seg_arg[(long long)lr * nseg + seg];
    uint4 o = make_uint4(0, 0, 0, 0);
    if (a >= in_seg && a < in_seg + 8) {
      const float w = wmat[(r / rows_per_sample) * nseg + seg] * rowscale[r];
      if (w != 0.f) {
        bf16 vals[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) vals[k] = __float2bfloat16_rn(0.f);
        vals[a - in_seg] = __float2bfloat16_rn(w * alpha);
        o = *reinterpret_cast<uint4*>(vals);
      }
    }
    *reinterpret_cast<uint4*>(g + lr * ldg + c0) = o;
  }
}

// filip_expand_kernel for seg_len % 8 != 0: an 8-column vector may hold the end of one segment and
// the start of the next (several when seg_len < 8), so every column steps its own (segment,
// position).  Columns [nseg * seg_len, roundup8) of the last vector are written as zeros.
__global__ void __launch_bounds__(256)
filip_expand_any_kernel(const unsigned short* __restrict__ seg_arg, const float* __restrict__ wmat,
                        const float* __restrict__ rowscale, const float* __restrict__ alpha_dev,
                        int row0, int rows, int rows_per_sample, int seg_len, int nseg,
                        bf16* __restrict__ g, long long ldg) {
  const float alpha = __ldg(alpha_dev);
  const int C = nseg * seg_len;
  const int vec_per_row = (C + 7) / 8;
  for (long long v = blockIdx.x * (long long)blockDim.x + threadIdx.x;
       v < (long long)rows * vec_per_row; v += (long long)gridDim.x * blockDim.x) {
    const int lr = (int)(v / vec_per_row);
    const int c0 = (int)(v % vec_per_row) * 8;
    const long long r = row0 + lr;
    const unsigned short* arg_row = seg_arg + (long long)lr * nseg;
    const float* w_row = wmat + (r / rows_per_sample) * nseg;
    int seg = c0 / seg_len;
    int pos = c0 - seg * seg_len;
    int a = arg_row[seg];
    bf16 vals[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      vals[k] = __float2bfloat16_rn(0.f);
      if (c0 + k < C) {
        if (pos == a) {
          const float w = w_row[seg] * rowscale[r];
          if (w != 0.f) vals[k] = __float2bfloat16_rn(w * alpha);
        }
        if (++pos == seg_len) {
          pos = 0;
          if (++seg < nseg) a = arg_row[seg];
        }
      }
    }
    *reinterpret_cast<uint4*>(g + lr * ldg + c0) = *reinterpret_cast<const uint4*>(vals);
  }
}

// keys of EPI_SEGMAX -> seg_max (f32, optional) and a 16-bit seg_arg (optional): the compact
// argmax a saved chunk keeps for its backward (seg_len <= 65535)
__global__ void __launch_bounds__(256)
filip_unpack_keys16_kernel(const unsigned long long* __restrict__ keys, long long n,
                           float* __restrict__ seg_max, unsigned short* __restrict__ seg_arg) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n;
       i += (long long)gridDim.x * blockDim.x) {
    const unsigned long long k = keys[i];
    if (seg_max != nullptr) seg_max[i] = segmax_key_value(k);
    if (seg_arg != nullptr) seg_arg[i] = (unsigned short)segmax_key_index(k);
  }
}

}  // namespace xclip

using namespace xclip;

// The segment-max GEMM: checks its arguments, zeroes the keys and launches EPI_SEGMAX.  Returns
// non-zero (nothing launched) when an argument is refused.
static int filip_segmax_keys(const char* who, const void* a, const void* b, int R, int C, int D,
                             const float* temp_exp, int seg_len, const float* col_mul,
                             const float* col_add, void* keys, cudaStream_t st) {
  XCLIP_REQUIRE(a && b && temp_exp && keys, "%s: null pointer", who);
  XCLIP_REQUIRE(R > 0 && C > 0 && D > 0 && D % 8 == 0, "%s: bad sizes", who);
  XCLIP_REQUIRE(seg_len >= 1 && C % seg_len == 0,
                "%s: C (%d) must be a whole number of segments of seg_len (%d) >= 1 tokens", who,
                C, seg_len);
  XCLIP_REQUIRE((col_mul == nullptr) == (col_add == nullptr), "%s: mask tables mismatch", who);
  XCLIP_REQUIRE(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0,
                "%s: misaligned latents", who);
  XCLIP_REQUIRE(((reinterpret_cast<uintptr_t>(temp_exp) | reinterpret_cast<uintptr_t>(col_mul) |
                  reinterpret_cast<uintptr_t>(col_add)) & 3) == 0,
                "%s: misaligned fp32 pointer", who);
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(keys) & 7) == 0, "%s: misaligned keys", who);
  const int nseg = C / seg_len;
  const long long nkeys = (long long)R * nseg;
  CUtensorMap tmA, tmB;
  int rc = encode_2d_bf16(&tmA, a, (uint64_t)D, (uint64_t)R, (uint64_t)D, 64, kGemmBlockM);
  if (rc) return rc;
  rc = encode_2d_bf16(&tmB, b, (uint64_t)D, (uint64_t)C, (uint64_t)D, 64, 256);
  if (rc) return rc;
  GemmParams p = {};
  p.M = R; p.N = C; p.K = D; p.split_k = 1;
  p.raster_m_fast = (R <= C) ? 1 : 0;
  p.alpha_dev = temp_exp;
  p.seg_len = seg_len;
  p.n_segs = nseg;
  p.col_mul = col_mul; p.col_add = col_add;
  p.seg_keys = reinterpret_cast<unsigned long long*>(keys);
  const long long tiles = (long long)((R + kGemmBlockM - 1) / kGemmBlockM) * ((C + 255) / 256);
  const int grid = (int)(tiles < num_sms() ? tiles : num_sms());
  using S = GemmSmem<256>;
  auto kern = gemm_bf16_kernel<256, kMajorK, kMajorK, EPI_SEGMAX>;
  {
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), S::kTotal);
    if (rc_attr) return rc_attr;
  }
  XCLIP_CUDA(cudaMemsetAsync(keys, 0, (size_t)nkeys * 8, st));
  kern<<<grid, kGemmThreads, S::kTotal, st>>>(tmA, tmB, p, CUtensorMap{}, CUtensorMap{});
  XCLIP_LAUNCH_CHECK("gemm_bf16_kernel<segmax>");
  return XCLIP_OK;
}

static int unpack_blocks(long long nkeys) {
  long long blocks = (nkeys + 255) / 256;
  if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
  return (int)blocks;
}

extern "C" int xclip_filip_segmax_arg16(const void* a, const void* b, int R, int C, int D,
                                        const float* temp_exp, int seg_len, const float* col_mul,
                                        const float* col_add, float* seg_max, uint16_t* seg_arg,
                                        void* keys, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(seg_max || seg_arg, "filip_segmax_arg16: neither seg_max nor seg_arg requested");
  XCLIP_REQUIRE(seg_len <= 65535, "filip_segmax_arg16: seg_len %d does not fit a 16-bit argmax (<= 65535)",
                seg_len);
  XCLIP_REQUIRE(((reinterpret_cast<uintptr_t>(seg_max) & 3) | (reinterpret_cast<uintptr_t>(seg_arg) & 1)) == 0,
                "filip_segmax_arg16: misaligned seg_max / seg_arg");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rc = filip_segmax_keys("filip_segmax_arg16", a, b, R, C, D, temp_exp, seg_len, col_mul, col_add, keys, st);
  if (rc) return rc;
  const long long nkeys = (long long)R * (C / seg_len);
  filip_unpack_keys16_kernel<<<unpack_blocks(nkeys), 256, 0, st>>>(
      reinterpret_cast<const unsigned long long*>(keys), nkeys, seg_max,
      reinterpret_cast<unsigned short*>(seg_arg));
  XCLIP_LAUNCH_CHECK("filip_unpack_keys16_kernel");
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

extern "C" int xclip_filip_nce_fwd(const float* s, int R, int C, int diag_off, int dcl,
                                   const unsigned char* row_valid, float* lse, float* loss_accum,
                                   float loss_scale, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(s && lse && R > 0 && C > 0 && diag_off >= 0 && diag_off + R <= C,
                "filip_nce_fwd: bad arguments");
  filip_nce_fwd_kernel<<<(R + 7) / 8, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      s, R, C, diag_off, dcl, row_valid, lse, loss_accum, loss_scale);
  XCLIP_LAUNCH_CHECK("filip_nce_fwd_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_filip_nce_bwd(const float* s, const float* lse, int R, int C, int diag_off,
                                   int dcl, const unsigned char* row_valid, const float* gscale,
                                   float* g, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(s && lse && gscale && g && R > 0 && C > 0, "filip_nce_bwd: bad arguments");
  const long long n = (long long)R * C;
  filip_nce_bwd_kernel<<<(int)((n + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      s, lse, R, C, diag_off, dcl, row_valid, gscale, g);
  XCLIP_LAUNCH_CHECK("filip_nce_bwd_kernel");
  return XCLIP_OK;
}

static int filip_nce_blocks_check(const char* who, const float* s, int64_t lds, int m, int n, int b,
                                  int B, int col_run, int diag_off) {
  XCLIP_REQUIRE(s != nullptr, "%s: null s", who);
  XCLIP_REQUIRE(m > 0 && n > 0 && b > 0 && B >= b && col_run > 0 && B % col_run == 0 &&
                    (col_run == B || col_run == b) && lds >= (int64_t)n * B,
                "%s: bad sizes (m %d n %d b %d B %d col_run %d lds %lld)", who, m, n, b, B, col_run,
                (long long)lds);
  XCLIP_REQUIRE(diag_off >= 0 && diag_off + b <= B, "%s: diag_off %d outside [0, B - b]", who, diag_off);
  XCLIP_REQUIRE((long long)m * b * n * B < (1LL << 31), "%s: matrix too large", who);
  return XCLIP_OK;
}

extern "C" int xclip_filip_nce_blocks_fwd(const float* s, int64_t lds, int m, int n, int b, int B,
                                          int col_run, int diag_off, int dcl,
                                          const unsigned char* row_valid, const float* block_w,
                                          float* lse, float* loss_accum, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  rc = filip_nce_blocks_check("filip_nce_blocks_fwd", s, lds, m, n, b, B, col_run, diag_off);
  if (rc) return rc;
  XCLIP_REQUIRE(lse && block_w, "filip_nce_blocks_fwd: null lse / block_w");
  const long long warps = (long long)m * b * n;
  filip_nce_blocks_fwd_kernel<<<(int)((warps + 7) / 8), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      s, lds, m, n, b, B, col_run, diag_off, dcl, row_valid, block_w, lse, loss_accum);
  XCLIP_LAUNCH_CHECK("filip_nce_blocks_fwd_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_filip_nce_blocks_bwd(const float* s, int64_t lds, const float* lse, int m, int n,
                                          int b, int B, int col_run, int diag_off, int dcl,
                                          const unsigned char* row_valid, const float* block_w,
                                          const float* gscale, float* g, int64_t ldg,
                                          xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  rc = filip_nce_blocks_check("filip_nce_blocks_bwd", s, lds, m, n, b, B, col_run, diag_off);
  if (rc) return rc;
  XCLIP_REQUIRE(lse && block_w && gscale && g && ldg >= (int64_t)n * B, "filip_nce_blocks_bwd: bad arguments");
  const long long elems = (long long)m * b * n * B;
  filip_nce_blocks_bwd_kernel<<<(int)((elems + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      s, lds, lse, m, n, b, B, col_run, diag_off, dcl, row_valid, block_w, gscale, g, ldg);
  XCLIP_LAUNCH_CHECK("filip_nce_blocks_bwd_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_filip_expand16(const uint16_t* seg_arg, const float* wmat, const float* rowscale,
                                    const float* temp_exp, int row0, int rows, int rows_per_sample,
                                    int seg_len, int nseg, void* g, int64_t ldg, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(seg_arg && wmat && rowscale && temp_exp && g, "filip_expand16: null pointer");
  XCLIP_REQUIRE(row0 >= 0 && rows > 0 && rows_per_sample > 0 && seg_len >= 1 && seg_len <= 65535 &&
                    nseg > 0 && ldg >= (int64_t)nseg * seg_len && ldg % 8 == 0,
                "filip_expand16: bad sizes");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "filip_expand16: misaligned g");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(seg_arg) & 1) == 0, "filip_expand16: misaligned seg_arg");
  const long long vecs = (long long)rows * ((nseg * seg_len + 7) / 8);
  long long blocks = (vecs + 255) / 256;
  if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
  const unsigned short* arg = reinterpret_cast<const unsigned short*>(seg_arg);
  if (seg_len % 8 == 0) {
    filip_expand_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        arg, wmat, rowscale, temp_exp, row0, rows, rows_per_sample, seg_len, nseg,
        reinterpret_cast<bf16*>(g), ldg);
    XCLIP_LAUNCH_CHECK("filip_expand_kernel");
  } else {
    filip_expand_any_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        arg, wmat, rowscale, temp_exp, row0, rows, rows_per_sample, seg_len, nseg,
        reinterpret_cast<bf16*>(g), ldg);
    XCLIP_LAUNCH_CHECK("filip_expand_any_kernel");
  }
  return XCLIP_OK;
}
