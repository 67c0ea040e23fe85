// The SimCLR augmentation of the visual SSL losses (reference x_clip/visual_ssl.py:24-45) as two
// memory-bound kernels.  The pipeline draws one decision per call for the whole batch, so every
// stage is a per-pixel map, a 3x3 stencil or a resampling with a handful of scalars:
//
//   colour jitter (brightness / contrast / saturation / hue in the drawn order) -> grayscale ->
//   horizontal flip -> 3x3 Gaussian blur (reflect padding at the image border) -> crop + bilinear
//   antialiased resize to out_h x out_w -> Normalize
//
//   mean  : per-image grayscale mean of the image as it is just before contrast (only needed when the
//           jitter applies); one CTA per image, fixed-order reduction in double.
//   apply : one CTA per 32 x 32 output tile, all channels.  It loads the input window the tile needs
//           (the crop window mapped through the flip, the bilinear footprint and the one-pixel blur
//           halo), applies the colour stages once per pixel into shared memory, blurs the crop region
//           it needs into a second buffer, then resamples, normalises and writes each output once.
//
// The colour stages and Normalize repeat torchvision's fp32 op-by-op rounding (every intermediate
// torch materialises is rounded here too: __fmul_rn / __fadd_rn, true division), so they match
// torchvision on CUDA bit for bit; only the blur and resample sums run in a different order.
#include "common.cuh"
#include "host.h"

namespace xclip {

constexpr int kAugTile = 32;      // output tile edge
constexpr int kAugThreads = 256;
// crop rows / cols a 32-wide output tile reads when the crop is no larger than the output (support
// 1): xmin moves by at most 31 over the tile and the last pixel reads at most 2, so at most 33; one
// more on each side for the blur halo
constexpr int kAugBlurSpan = 33;
constexpr int kAugWin = kAugBlurSpan + 2;
constexpr int kAugMeanThreads = 512;

__device__ __forceinline__ float aug_gray(float r, float g, float b) {
  // rgb_to_grayscale: (0.2989 * r + 0.587 * g + 0.114 * b), each product and sum rounded
  return __fadd_rn(__fadd_rn(__fmul_rn((float)0.2989, r), __fmul_rn((float)0.587, g)),
                   __fmul_rn((float)0.114, b));
}

// _blend(img1, img2, ratio): (ratio * img1 + (1 - ratio) * img2).clamp(0, 1)
__device__ __forceinline__ float aug_blend(float x, float y, float w, float wc) {
  const float v = __fadd_rn(__fmul_rn(w, x), __fmul_rn(wc, y));
  return fminf(fmaxf(v, 0.f), 1.f);
}

__device__ __forceinline__ float aug_clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

// adjust_hue: _rgb2hsv, (h + hue) % 1, _hsv2rgb, with torch's CUDA arithmetic (h / 6.0 by a CPU
// scalar is a multiplication by its fp32 reciprocal there)
__device__ __forceinline__ void aug_hue(float& r, float& g, float& b, float hue) {
  const float maxc = fmaxf(fmaxf(r, g), b);
  const float minc = fminf(fminf(r, g), b);
  const bool eqc = maxc == minc;
  const float cr = __fsub_rn(maxc, minc);
  const float s = __fdiv_rn(cr, eqc ? 1.f : maxc);
  const float crd = eqc ? 1.f : cr;
  const float rc = __fdiv_rn(__fsub_rn(maxc, r), crd);
  const float gc = __fdiv_rn(__fsub_rn(maxc, g), crd);
  const float bc = __fdiv_rn(__fsub_rn(maxc, b), crd);
  const float hr = __fmul_rn(maxc == r ? 1.f : 0.f, __fsub_rn(bc, gc));
  const float hg = __fmul_rn((maxc == g && maxc != r) ? 1.f : 0.f, __fsub_rn(__fadd_rn(2.f, rc), bc));
  const float hb = __fmul_rn((maxc != g && maxc != r) ? 1.f : 0.f, __fsub_rn(__fadd_rn(4.f, gc), rc));
  float h = __fadd_rn(__fadd_rn(hr, hg), hb);
  h = fmodf(__fadd_rn(__fmul_rn(h, 1.f / 6.f), 1.f), 1.f);
  h = fmodf(__fadd_rn(h, hue), 1.f);                      // torch.remainder(x, 1.0)
  if (h != 0.f && h < 0.f) h = __fadd_rn(h, 1.f);
  const float h6 = __fmul_rn(h, 6.f);
  const float fl = floorf(h6);
  const float f = __fsub_rn(h6, fl);
  int i = (int)fl % 6;
  if (i < 0) i += 6;
  const float v = maxc;
  const float p = aug_clamp01(__fmul_rn(v, __fsub_rn(1.f, s)));
  const float q = aug_clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, f))));
  const float t = aug_clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, __fsub_rn(1.f, f)))));
  switch (i) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// the jitter ops in the drawn order; stop_at_contrast: the prefix before contrast (the mean pass)
__device__ __forceinline__ void aug_jitter(float& r, float& g, float& b, const xclip_augment_params& a,
                                           float mean, bool stop_at_contrast) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int op = a.ops[k];
    if (op == 0) {
      const float w = a.factor[0], wc = a.one_minus[0];
      r = aug_blend(r, 0.f, w, wc); g = aug_blend(g, 0.f, w, wc); b = aug_blend(b, 0.f, w, wc);
    } else if (op == 1) {
      if (stop_at_contrast) return;
      const float w = a.factor[1], wc = a.one_minus[1];
      r = aug_blend(r, mean, w, wc); g = aug_blend(g, mean, w, wc); b = aug_blend(b, mean, w, wc);
    } else if (op == 2) {
      const float w = a.factor[2], wc = a.one_minus[2];
      const float y = aug_gray(r, g, b);
      r = aug_blend(r, y, w, wc); g = aug_blend(g, y, w, wc); b = aug_blend(b, y, w, wc);
    } else if (op == 3) {
      aug_hue(r, g, b, a.factor[3]);
    }
  }
}

__global__ void __launch_bounds__(kAugMeanThreads)
augment_mean_kernel(const float* __restrict__ x, long long hw, xclip_augment_params a,
                    float* __restrict__ mean) {
  __shared__ double red[kAugMeanThreads / 32];
  const float* img = x + (long long)blockIdx.x * 3 * hw;
  double acc = 0.0;
  for (long long i = threadIdx.x; i < hw; i += kAugMeanThreads) {
    float r = img[i], g = img[hw + i], b = img[2 * hw + i];
    aug_jitter(r, g, b, a, 0.f, true);
    acc += (double)aug_gray(r, g, b);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    double v = threadIdx.x < kAugMeanThreads / 32 ? red[threadIdx.x] : 0.0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (threadIdx.x == 0) mean[blockIdx.x] = (float)(v / (double)hw);
  }
}

// ATen's antialiased bilinear span and weights (_compute_weights_span / _compute_weights with the
// triangle filter) for output index i; support 1, invscale 1 (the crop is never larger than the output)
// (at support 1 a span has at most 2 taps)
__device__ __forceinline__ int aug_span(int i, float scale, int in_size, int& xmin, float (&w)[2]) {
  const float center = scale * (i + 0.5f);
  xmin = max(static_cast<int>(center - 1.f + 0.5f), 0);
  const int xsize = min(min(static_cast<int>(center + 1.f + 0.5f), in_size) - xmin, 2);
  const float xmin_m_center = xmin - center;
  float total = 0.f;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    float t = fabsf(j + xmin_m_center + 0.5f);
    t = (j < xsize && t < 1.f) ? 1.f - t : 0.f;
    w[j] = t;
    total += t;
  }
  if (total != 0.f) {
#pragma unroll
    for (int j = 0; j < 2; ++j) w[j] /= total;
  }
  return xsize;
}

__device__ __forceinline__ int aug_reflect(int v, int n) { return v < 0 ? -v : (v >= n ? 2 * n - 2 - v : v); }

// NC = 3: the colour stages run on the pixel's three channels; NC = 1: one channel at a time
template <int NC>
__global__ void __launch_bounds__(kAugThreads)
augment_apply_kernel(const float* __restrict__ x, int C, int H, int W, int tiles_x, int tiles,
                     xclip_augment_params a, const float* __restrict__ mean, float* __restrict__ out) {
  __shared__ float win[NC][kAugWin][kAugWin + 1];
  __shared__ float blr[NC][kAugBlurSpan][kAugBlurSpan + 1];
  const long long b = blockIdx.x / tiles;
  const int tile = blockIdx.x % tiles;
  const int OH = a.out_h, OW = a.out_w;
  const int oy0 = (tile / tiles_x) * kAugTile, ox0 = (tile % tiles_x) * kAugTile;
  const int oy1 = min(oy0 + kAugTile, OH) - 1, ox1 = min(ox0 + kAugTile, OW) - 1;
  const float sy = (float)a.height / (float)OH, sx = (float)a.width / (float)OW;

  // crop-relative rows / cols the tile reads, then the image window with the blur halo
  float wtmp[2];
  int cy0, cx0, cy1, cx1, t0;
  aug_span(oy0, sy, a.height, cy0, wtmp);
  cy1 = aug_span(oy1, sy, a.height, t0, wtmp) + t0 - 1;
  aug_span(ox0, sx, a.width, cx0, wtmp);
  cx1 = aug_span(ox1, sx, a.width, t0, wtmp) + t0 - 1;
  const int halo = a.blur ? 1 : 0;
  const int wy0 = max(a.top + cy0 - halo, 0), wy1 = min(a.top + cy1 + halo, H - 1);
  const int wx0 = max(a.left + cx0 - halo, 0), wx1 = min(a.left + cx1 + halo, W - 1);
  const int wh = wy1 - wy0 + 1, ww = wx1 - wx0 + 1;
  const int bh = cy1 - cy0 + 1, bw = cx1 - cx0 + 1;
  const long long plane = (long long)H * W;
  const float img_mean = (NC == 3 && mean != nullptr) ? mean[b] : 0.f;

  // per-thread output columns (fixed for the tile) and their x weights
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int ox = ox0 + lane;
  int xmin;
  float wx[2];
  const int xsize = aug_span(ox < OW ? ox : OW - 1, sx, a.width, xmin, wx);

  for (int c0 = 0; c0 < C; c0 += NC) {
    const float* src = x + (b * C + c0) * plane;
    for (int idx = threadIdx.x; idx < wh * ww; idx += kAugThreads) {
      const int ry = idx / ww, rx = idx - ry * ww;
      const int y = wy0 + ry, xf = wx0 + rx;
      const long long off = (long long)y * W + (a.flip ? W - 1 - xf : xf);
      if (NC == 3) {
        float r = src[off], g = src[plane + off], bb = src[2 * plane + off];
        aug_jitter(r, g, bb, a, img_mean, false);
        if (a.grayscale) r = g = bb = aug_gray(r, g, bb);
        win[0][ry][rx] = r;
        win[NC > 1 ? 1 : 0][ry][rx] = g;
        win[NC > 2 ? 2 : 0][ry][rx] = bb;
      } else {
        win[0][ry][rx] = src[off];
      }
    }
    __syncthreads();
    // the crop region's blurred values (reflect indexing at the image border), or the window itself
    const float* base[NC];
    int ld;
    if (a.blur) {
      for (int idx = threadIdx.x; idx < bh * bw; idx += kAugThreads) {
        const int ry = idx / bw, rx = idx - ry * bw;
        const int y = a.top + cy0 + ry, xi = a.left + cx0 + rx;
        int ys[3], xs[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
          ys[d] = aug_reflect(y + d - 1, H) - wy0;
          xs[d] = aug_reflect(xi + d - 1, W) - wx0;
        }
#pragma unroll
        for (int k = 0; k < NC; ++k) {
          float s = 0.f;
#pragma unroll
          for (int i = 0; i < 3; ++i)
#pragma unroll
            for (int j = 0; j < 3; ++j) s = fmaf(a.blur_kernel[3 * i + j], win[k][ys[i]][xs[j]], s);
          blr[k][ry][rx] = s;
        }
      }
      __syncthreads();
#pragma unroll
      for (int k = 0; k < NC; ++k) base[k] = &blr[k][0][0];
      ld = kAugBlurSpan + 1;
    } else {
#pragma unroll
      for (int k = 0; k < NC; ++k) base[k] = &win[k][a.top + cy0 - wy0][a.left + cx0 - wx0];
      ld = kAugWin + 1;
    }
    // resample (rows of horizontal sums, then the vertical sum, as ATen), Normalize, one write
    if (ox <= ox1) {
      for (int oy = oy0 + warp; oy <= oy1; oy += kAugThreads / 32) {
        int ymin;
        float wy[2];
        const int ysize = aug_span(oy, sy, a.height, ymin, wy);
#pragma unroll
        for (int k = 0; k < NC; ++k) {
          float v = 0.f;
          for (int i = 0; i < ysize; ++i) {
            const float* row = base[k] + (ymin - cy0 + i) * ld + (xmin - cx0);
            float t = row[0] * wx[0];
            for (int j = 1; j < xsize; ++j) t += row[j] * wx[j];
            v = i == 0 ? t * wy[0] : v + t * wy[i];
          }
          const int c = c0 + k;
          if (a.normalize) v = __fdiv_rn(__fsub_rn(v, a.mean[c]), a.std[c]);
          out[((b * C + c) * OH + oy) * (long long)OW + ox] = v;
        }
      }
    }
    __syncthreads();
  }
}

static int augment_check(const float* x, int B, int C, int H, int W, const xclip_augment_params* p,
                         const char* what) {
  XCLIP_REQUIRE(x && p, "%s: null pointer", what);
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(x) & 3) == 0, "%s: misaligned input", what);
  XCLIP_REQUIRE(B > 0 && C > 0 && H >= 2 && W >= 2, "%s: bad shape B=%d C=%d H=%d W=%d (H, W >= 2)",
                what, B, C, H, W);
  XCLIP_REQUIRE(p->out_h > 0 && p->out_w > 0, "%s: bad output size %dx%d", what, p->out_h, p->out_w);
  XCLIP_REQUIRE(p->height > 0 && p->width > 0 && p->top >= 0 && p->left >= 0 &&
                    (long long)p->top + p->height <= H && (long long)p->left + p->width <= W,
                "%s: crop (%d, %d, %d, %d) outside the %dx%d image", what, p->top, p->left, p->height,
                p->width, H, W);
  XCLIP_REQUIRE(p->height <= p->out_h && p->width <= p->out_w,
                "%s: crop %dx%d larger than the %dx%d output (only upsampling is supported)", what,
                p->height, p->width, p->out_h, p->out_w);
  bool colour = p->grayscale != 0 || p->normalize != 0;
  for (int k = 0; k < 4; ++k) {
    XCLIP_REQUIRE(p->ops[k] >= -1 && p->ops[k] <= 3, "%s: bad jitter op %d", what, p->ops[k]);
    colour = colour || p->ops[k] >= 0;
  }
  XCLIP_REQUIRE(!colour || C == 3, "%s: the colour stages need 3 channels, got %d", what, C);
  return XCLIP_OK;
}

static bool has_contrast(const xclip_augment_params* p) {
  for (int k = 0; k < 4; ++k)
    if (p->ops[k] == 1) return true;
  return false;
}

}  // namespace xclip

using namespace xclip;

extern "C" int xclip_augment_mean(const float* x, int B, int C, int H, int W,
                                  const xclip_augment_params* params, float* mean,
                                  xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  rc = augment_check(x, B, C, H, W, params, "augment_mean");
  if (rc) return rc;
  XCLIP_REQUIRE(C == 3, "augment_mean: needs 3 channels, got %d", C);
  XCLIP_REQUIRE(mean && (reinterpret_cast<uintptr_t>(mean) & 3) == 0, "augment_mean: null or misaligned mean");
  augment_mean_kernel<<<B, kAugMeanThreads, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      x, (long long)H * W, *params, mean);
  XCLIP_LAUNCH_CHECK("augment_mean_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_augment_apply(const float* x, int B, int C, int H, int W,
                                   const xclip_augment_params* params, const float* mean, float* out,
                                   xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  rc = augment_check(x, B, C, H, W, params, "augment_apply");
  if (rc) return rc;
  XCLIP_REQUIRE(out && (reinterpret_cast<uintptr_t>(out) & 3) == 0, "augment_apply: null or misaligned out");
  XCLIP_REQUIRE(!has_contrast(params) || (mean && (reinterpret_cast<uintptr_t>(mean) & 3) == 0),
                "augment_apply: contrast needs the per-image mean (xclip_augment_mean)");
  const int tiles_x = (params->out_w + kAugTile - 1) / kAugTile;
  const int tiles = tiles_x * ((params->out_h + kAugTile - 1) / kAugTile);
  const long long grid = (long long)B * tiles;
  XCLIP_REQUIRE(grid < (1LL << 31), "augment_apply: %lld tiles exceed one launch", grid);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (C == 3)
    augment_apply_kernel<3><<<(unsigned)grid, kAugThreads, 0, s>>>(x, C, H, W, tiles_x, tiles, *params,
                                                                   has_contrast(params) ? mean : nullptr, out);
  else
    augment_apply_kernel<1><<<(unsigned)grid, kAugThreads, 0, s>>>(x, C, H, W, tiles_x, tiles, *params,
                                                                   nullptr, out);
  XCLIP_LAUNCH_CHECK("augment_apply_kernel");
  return XCLIP_OK;
}
