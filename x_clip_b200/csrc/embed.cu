// Text token embedding + absolute position + CLS prepend (reference TextTransformer.forward,
// x_clip/x_clip.py:320-332) fused into one HBM pass, and its backward.
//   fwd : out[b,0,:] = cls ; out[b,1+t,:] = tok[ids[b,t],:] + pos[t,:]      fp32 tables -> bf16
//   bwd : dtok[ids[b,t],:] += dx[b,1+t,:]   (vector fp32 reductions into the table gradient)
//         dpos[t,:] = sum_b dx[b,1+t,:] ; dcls = sum_b dx[b,0,:]            (column sums, no atomics)
#include <climits>

#include "common.cuh"
#include "host.h"

namespace xclip {

__global__ void __launch_bounds__(256)
text_embed_fwd_kernel(const long long* __restrict__ ids, const float* __restrict__ tok,
                      const float* __restrict__ pos, const float* __restrict__ cls,
                      bf16* __restrict__ out, int B, int n, int d, int vocab) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long rows = (long long)B * (n + 1);
  for (long long r = warp; r < rows; r += nwarps) {
    const int j = (int)(r % (n + 1));
    const long long b = r / (n + 1);
    const float* src = cls;
    const float* add = nullptr;
    if (j > 0) {
      const long long id = ids[b * n + (j - 1)];
      if (id < 0 || id >= vocab) {   // nn.Embedding raises a device-side assert here (x_clip.py:320)
        if (lane == 0)
          printf("xclip text_embed: token id %lld at [%lld,%d] outside the vocabulary [0,%d)\n", id,
                 b, j - 1, vocab);
        __trap();
      }
      src = tok + id * d;
      add = pos + (long long)(j - 1) * d;
    }
    for (int c = lane * 8; c < d; c += 256) {
      float4 a0 = *reinterpret_cast<const float4*>(src + c);
      float4 a1 = *reinterpret_cast<const float4*>(src + c + 4);
      if (add != nullptr) {
        const float4 p0 = *reinterpret_cast<const float4*>(add + c);
        const float4 p1 = *reinterpret_cast<const float4*>(add + c + 4);
        a0.x += p0.x; a0.y += p0.y; a0.z += p0.z; a0.w += p0.w;
        a1.x += p1.x; a1.y += p1.y; a1.z += p1.z; a1.w += p1.w;
      }
      uint4 o;
      o.x = pack_bf16x2(a0.x, a0.y); o.y = pack_bf16x2(a0.z, a0.w);
      o.z = pack_bf16x2(a1.x, a1.y); o.w = pack_bf16x2(a1.z, a1.w);
      *reinterpret_cast<uint4*>(out + r * d + c) = o;
    }
  }
}

__global__ void __launch_bounds__(256)
text_embed_scatter_kernel(const long long* __restrict__ ids, const bf16* __restrict__ dx,
                          float* __restrict__ dtok, int B, int n, int d, int vocab) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long rows = (long long)B * n;
  for (long long r = warp; r < rows; r += nwarps) {
    const long long b = r / n;
    const int t = (int)(r % n);
    const long long id = ids[r];
    if (id < 0 || id >= vocab) __trap();   // (the forward already reported it)
    const bf16* src = dx + (b * (n + 1) + 1 + t) * d;
    float* dst = dtok + id * d;
    for (int c = lane * 8; c < d; c += 256) {
      const uint4 u = *reinterpret_cast<const uint4*>(src + c);
      const float2 a = unpack_bf16x2(u.x), bb = unpack_bf16x2(u.y), cc = unpack_bf16x2(u.z),
                   dd = unpack_bf16x2(u.w);
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + c), "f"(a.x),
                   "f"(a.y), "f"(bb.x), "f"(bb.y)
                   : "memory");
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(dst + c + 4), "f"(cc.x),
                   "f"(cc.y), "f"(dd.x), "f"(dd.y)
                   : "memory");
    }
  }
}

// block (j, chunk): sums dx[b, j, chunk*512 .. +512) over a slice of b; 256 threads x 2 columns
__global__ void __launch_bounds__(256)
text_embed_colsum_kernel(const bf16* __restrict__ dx, float* __restrict__ dpos,
                         float* __restrict__ dcls, int B, int n, int d, int bsplit) {
  const int j = blockIdx.x;                 // 0..n
  const int c = blockIdx.y * 512 + threadIdx.x * 2;
  const int part = blockIdx.z;
  if (c >= d) return;
  float s0 = 0.f, s1 = 0.f;
  for (int b = part; b < B; b += bsplit) {
    const uint32_t u = *reinterpret_cast<const uint32_t*>(dx + ((long long)b * (n + 1) + j) * d + c);
    const float2 v = unpack_bf16x2(u);
    s0 += v.x;
    s1 += v.y;
  }
  float* dst = (j == 0) ? dcls + c : dpos + (long long)(j - 1) * d + c;
  atomicAdd(dst, s0);
  atomicAdd(dst + 1, s1);
}

}  // namespace xclip

using namespace xclip;

extern "C" int xclip_text_embed_fwd(const int64_t* ids, const float* tok, const float* pos,
                                    const float* cls, void* out, int B, int n, int d, int vocab,
                                    xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(ids && tok && pos && cls && out, "text_embed_fwd: null pointer");
  XCLIP_REQUIRE(B > 0 && n > 0 && d % 8 == 0 && vocab > 0, "text_embed_fwd: bad sizes");
  const long long rows = (long long)B * (n + 1);
  long long blocks = (rows + 7) / 8;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  text_embed_fwd_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const long long*>(ids), tok, pos, cls, reinterpret_cast<bf16*>(out), B, n, d,
      vocab);
  XCLIP_LAUNCH_CHECK("text_embed_fwd_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_text_embed_bwd(const int64_t* ids, const void* dx, float* dtok, float* dpos,
                                    float* dcls, int B, int n, int d, int vocab,
                                    xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(ids && dx && dtok && dpos && dcls, "text_embed_bwd: null pointer");
  XCLIP_REQUIRE(B > 0 && n > 0 && d % 8 == 0 && vocab > 0, "text_embed_bwd: bad sizes");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long rows = (long long)B * n;
  long long blocks = (rows + 7) / 8;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  text_embed_scatter_kernel<<<(int)blocks, 256, 0, s>>>(reinterpret_cast<const long long*>(ids),
                                                        reinterpret_cast<const bf16*>(dx), dtok, B,
                                                        n, d, vocab);
  XCLIP_LAUNCH_CHECK("text_embed_scatter_kernel");
  int bsplit = (num_sms() * 4) / ((n + 1) * ((d + 511) / 512));
  if (bsplit < 1) bsplit = 1;
  if (bsplit > B) bsplit = B;
  dim3 grid(n + 1, (d + 511) / 512, bsplit);
  text_embed_colsum_kernel<<<grid, 256, 0, s>>>(reinterpret_cast<const bf16*>(dx), dpos, dcls, B, n,
                                                d, bsplit);
  XCLIP_LAUNCH_CHECK("text_embed_colsum_kernel");
  return XCLIP_OK;
}

// ---------------------------------------------------------------------------------------------
// Rotary position embedding of the text tower (x_clip/x_clip.py:155-176, applied to q, k AND v at
// :221-223), in place on the bf16 qkv buffer right after the QKV projection.  The first 32
// features of every 64-wide head slice are rotated pairwise (feature j with j+16) by the angle
// pos * inv_freq[j]; cos/sin tables [n, 16] come from the caller (the module's inv_freq buffer).
// inverse != 0 applies the transposed rotation: the backward of the same op on dq | dk | dv.
namespace xclip {
__global__ void __launch_bounds__(256)
rotary_inplace_kernel(bf16* __restrict__ qkv, long long ld, long long rows, int n, int nslices,
                      const float* __restrict__ cos_tab, const float* __restrict__ sin_tab,
                      int inverse) {
  const long long total = rows * nslices;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / nslices;
    const int slice = (int)(idx - row * nslices);
    const int pos = (int)(row % n);
    bf16* ptr = qkv + row * ld + (long long)slice * 64;
    uint4 raw[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) raw[i] = reinterpret_cast<const uint4*>(ptr)[i];
    float t[32];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const uint32_t w[4] = {raw[i].x, raw[i].y, raw[i].z, raw[i].w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const float2 f = unpack_bf16x2(w[k]);
        t[i * 8 + k * 2] = f.x;
        t[i * 8 + k * 2 + 1] = f.y;
      }
    }
    float o[32];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float c = __ldg(cos_tab + pos * 16 + j);
      const float s0 = __ldg(sin_tab + pos * 16 + j);
      const float s = inverse ? -s0 : s0;
      o[j] = t[j] * c - t[j + 16] * s;
      o[j + 16] = t[j + 16] * c + t[j] * s;
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      uint4 w;
      w.x = pack_bf16x2(o[i * 8 + 0], o[i * 8 + 1]);
      w.y = pack_bf16x2(o[i * 8 + 2], o[i * 8 + 3]);
      w.z = pack_bf16x2(o[i * 8 + 4], o[i * 8 + 5]);
      w.w = pack_bf16x2(o[i * 8 + 6], o[i * 8 + 7]);
      reinterpret_cast<uint4*>(ptr)[i] = w;
    }
  }
}
}  // namespace xclip

extern "C" int xclip_rotary_inplace(void* qkv, int64_t ld, int64_t rows, int n, int nslices,
                                    const float* cos_tab, const float* sin_tab, int inverse,
                                    xclip_stream_t stream) {
  using namespace xclip;
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(qkv && cos_tab && sin_tab, "rotary: null pointer");
  XCLIP_REQUIRE(rows > 0 && n > 0 && nslices > 0 && rows % n == 0, "rotary: bad sizes");
  XCLIP_REQUIRE(ld % 8 == 0 && ld >= (int64_t)nslices * 64 &&
                    (reinterpret_cast<uintptr_t>(qkv) & 15) == 0,
                "rotary: qkv must be 16-byte aligned with ld %% 8 == 0");
  const long long total = (long long)rows * nslices;
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
  rotary_inplace_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<bf16*>(qkv), ld, rows, n, nslices, cos_tab, sin_tab, inverse);
  XCLIP_LAUNCH_CHECK("rotary_inplace_kernel");
  return XCLIP_OK;
}

// ---------------------------------------------------------------------------------------------
// Patch embedding front end (x_clip/x_clip.py:356-359 'b c (h p1) (w p2) -> b (h w) (p1 p2 c)' and
// PatchDropout :134-151): one pass from the fp32 image to the bf16 A operand of the patch-embedding
// GEMM, reading ONLY the kept patches (keep[b, j] = patch index, or all patches in order when NULL).
// Mathematically the reference embeds every patch and drops half afterwards; embedding only the
// kept ones gives the same tokens (the position-table row is selected by the same index).
// ---------------------------------------------------------------------------------------------
namespace xclip {
// Rows have stride ldo (a multiple of 8): columns patch_dim .. ldo-1 are written as exact zeros, so a
// row of any patch_dim is a whole number of 16-byte stores and a GEMM A operand with K = ldo.
__global__ void __launch_bounds__(256)
patchify_gather_kernel(const float* __restrict__ img, int B, int C, int H, int W, int P,
                       const long long* __restrict__ keep, int k, int n_patches,
                       bf16* __restrict__ out, int ldo) {
  const int gw_n = W / P;
  const int patch_dim = P * P * C;
  const int vec_per_row = ldo / 8;
  const long long total = (long long)B * k * vec_per_row;
  for (long long idx = blockIdx.x * (long long)blockDim.x + threadIdx.x; idx < total;
       idx += (long long)gridDim.x * blockDim.x) {
    const long long row = idx / vec_per_row;
    const int e0 = (int)(idx - row * vec_per_row) * 8;
    const long long b = row / k;
    long long pidx = keep ? keep[row] : (row - b * k);
    if (pidx < 0 || pidx >= n_patches) __trap();
    const int gh = (int)(pidx / gw_n), gw = (int)(pidx - (long long)gh * gw_n);
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int el = e0 + e;
      const int q = el / C, c = el - q * C;
      const int p1 = q / P, p2 = q - p1 * P;
      f[e] = el < patch_dim
                 ? __ldg(img + ((b * C + c) * H + gh * P + p1) * (long long)W + gw * P + p2)
                 : 0.f;
    }
    uint4 o;
    o.x = pack_bf16x2(f[0], f[1]); o.y = pack_bf16x2(f[2], f[3]);
    o.z = pack_bf16x2(f[4], f[5]); o.w = pack_bf16x2(f[6], f[7]);
    *reinterpret_cast<uint4*>(out + row * ldo + e0) = o;
  }
}

// Inverse of the gather (the image gradient): block (b, chunk) owns patches [lo, lo + ppc) of sample b
// and writes every pixel of them, the src row of a kept patch or 0 for a dropped one.  The row of each
// owned patch comes from an inverse map of keep[b, :] built in shared memory (indices of one sample are
// distinct, so each slot has at most one writer).
//   CT > 0 (C == CT): a thread owns V horizontally adjacent pixels of one patch row (V = 4 when
//          patch % 4 == 0, V = 2 when patch % 4 == 2): CT V-wide vector loads of the (p1 p2 c) row
//          (V pixels x CT channels, contiguous), transposed in registers, CT V-wide stores, one per
//          channel plane.  Consecutive threads walk along p2, so loads are contiguous across a warp
//          and stores fill whole 32-byte sectors of an image row.  Vector alignment: lds % 4 == 0 and
//          16-byte aligned src / img; (p1 * P + p2) * C and every image offset are multiples of V.
//   CT == 0 (V == 1): any C / patch, one pixel x C channels per thread with scalar accesses.
// With V < 4 a patch row is not a whole number of 32-byte sectors (14 pixels: 56 bytes), so the work
// items run along image rows across the block's patches rather than patch by patch: consecutive
// threads then store consecutive pixels of an image row whichever patch they fall in.
// Only the first patch_dim columns of a src row are read.
constexpr int kScatterMaxPatchesPerBlock = 1024;

template <int CT, int V>
__global__ void __launch_bounds__(256)
patchify_scatter_kernel(const float* __restrict__ src, long long lds, int B, int C, int H, int W, int P,
                        const long long* __restrict__ keep, int k, int n_patches, int ppc,
                        float* __restrict__ img) {
  __shared__ int inv[kScatterMaxPatchesPerBlock];
  const long long b = blockIdx.x;
  const int lo = blockIdx.y * ppc;
  const int cnt = min(ppc, n_patches - lo);
  if (cnt <= 0) return;
  if (keep != nullptr) {
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) inv[i] = -1;
    __syncthreads();
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
      const long long p = keep[b * k + j];
      if (p < 0 || p >= n_patches) __trap();
      if (p >= lo && p < lo + cnt) inv[p - lo] = j;
    }
    __syncthreads();
  }
  const int gw_n = W / P;
  const int per_row = P / V;               // work items per patch row
  const int per_patch = P * per_row;
  const int items = cnt * per_patch;       // < 2^31 for patch sizes up to 2048
  for (int it = threadIdx.x; it < items; it += blockDim.x) {
    int pl, p1, p2;
    if constexpr (V == 4) {                // patch by patch: a warp's loads are one contiguous run
      pl = it / per_patch;
      const int w = it - pl * per_patch;
      p1 = w / per_row;
      p2 = (w - p1 * per_row) * V;
    } else {                               // pixel row p1 of every owned patch in turn: a warp's
      const int per_line = cnt * per_row;  // stores run along an image row across patches
      p1 = it / per_line;
      const int r = it - p1 * per_line;
      pl = r / per_row;
      p2 = (r - pl * per_row) * V;
    }
    const int pidx = lo + pl;
    const int j = keep != nullptr ? inv[pl] : pidx;
    const int gh = pidx / gw_n, gw = pidx - gh * gw_n;
    const long long plane = (long long)H * W;
    float* dst = img + (b * C) * plane + (long long)(gh * P + p1) * W + gw * P + p2;
    const float* s = j >= 0 ? src + (b * k + j) * lds + (long long)(p1 * P + p2) * C : nullptr;
    if constexpr (CT > 0) {
      float v[V * CT];
      if (j >= 0) {
#pragma unroll
        for (int i = 0; i < CT; ++i) {
          if constexpr (V == 4) {
            const float4 t = *reinterpret_cast<const float4*>(s + 4 * i);
            v[4 * i] = t.x; v[4 * i + 1] = t.y; v[4 * i + 2] = t.z; v[4 * i + 3] = t.w;
          } else {
            const float2 t = *reinterpret_cast<const float2*>(s + 2 * i);
            v[2 * i] = t.x; v[2 * i + 1] = t.y;
          }
        }
      } else {
#pragma unroll
        for (int i = 0; i < V * CT; ++i) v[i] = 0.f;
      }
#pragma unroll
      for (int c = 0; c < CT; ++c) {
        if constexpr (V == 4)
          *reinterpret_cast<float4*>(dst + c * plane) =
              make_float4(v[c], v[CT + c], v[2 * CT + c], v[3 * CT + c]);
        else
          *reinterpret_cast<float2*>(dst + c * plane) = make_float2(v[c], v[CT + c]);
      }
    } else {
      for (int c = 0; c < C; ++c) dst[c * plane] = j >= 0 ? s[c] : 0.f;
    }
  }
}

// dst[idx[r] or r %% period, :] += src[r, :]  (f32 += bf16): gradient of a gathered / periodic table
__global__ void __launch_bounds__(256)
scatter_add_rows_kernel(const int* __restrict__ idx, int period, const bf16* __restrict__ src,
                        long long lds, float* __restrict__ dst, long long rows, int d, int V) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  for (long long r = warp; r < rows; r += nwarps) {
    const long long t = idx ? idx[r] : (r % period);
    if (t < 0 || t >= V) __trap();
    const bf16* s = src + r * lds;
    float* o = dst + t * d;
    for (int c = lane * 8; c < d; c += 256) {
      const uint4 u = *reinterpret_cast<const uint4*>(s + c);
      const float2 a = unpack_bf16x2(u.x), bb = unpack_bf16x2(u.y), cc = unpack_bf16x2(u.z),
                   dd = unpack_bf16x2(u.w);
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o + c), "f"(a.x), "f"(a.y),
                   "f"(bb.x), "f"(bb.y) : "memory");
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(o + c + 4), "f"(cc.x), "f"(cc.y),
                   "f"(dd.x), "f"(dd.y) : "memory");
    }
  }
}

// dst[c] += sum_r src[r, c]   (bias gradient): block (column chunk, row slice)
__global__ void __launch_bounds__(256)
colsum_rows_kernel(const bf16* __restrict__ src, long long lds, float* __restrict__ dst, long long rows,
                   int d, int slices) {
  const int c = blockIdx.x * 512 + threadIdx.x * 2;
  if (c >= d) return;
  float s0 = 0.f, s1 = 0.f;
  for (long long r = blockIdx.y; r < rows; r += slices) {
    const float2 v = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(src + r * lds + c));
    s0 += v.x;
    s1 += v.y;
  }
  atomicAdd(dst + c, s0);
  atomicAdd(dst + c + 1, s1);
}
}  // namespace xclip

extern "C" int xclip_patchify_gather_rows(const float* img, int B, int C, int H, int W, int patch,
                                          const int64_t* keep, int k, void* out, int64_t ldo,
                                          xclip_stream_t stream) {
  using namespace xclip;
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(img && out && B > 0 && C > 0 && patch > 0 && H % patch == 0 && W % patch == 0,
                "patchify: bad arguments");
  const int n_patches = (H / patch) * (W / patch);
  const long long patch_dim = (long long)patch * patch * C;
  XCLIP_REQUIRE(ldo % 8 == 0 && ldo >= patch_dim && ldo <= INT_MAX,
                "patchify: ldo=%lld must be a multiple of 8 and >= patch_dim=%lld", (long long)ldo,
                patch_dim);
  XCLIP_REQUIRE(k > 0 && (keep != nullptr || k == n_patches), "patchify: k=%d", k);
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(out) & 15) == 0, "patchify: misaligned output");
  const long long total = (long long)B * k * (ldo / 8);
  long long blocks = (total + 255) / 256;
  if (blocks > (long long)num_sms() * 16) blocks = (long long)num_sms() * 16;
  patchify_gather_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      img, B, C, H, W, patch, reinterpret_cast<const long long*>(keep), k, n_patches,
      reinterpret_cast<bf16*>(out), (int)ldo);
  XCLIP_LAUNCH_CHECK("patchify_gather_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_patchify_gather(const float* img, int B, int C, int H, int W, int patch,
                                     const int64_t* keep, int k, void* out, xclip_stream_t stream) {
  using namespace xclip;
  XCLIP_REQUIRE(((long long)patch * patch * C) % 8 == 0,
                "patchify: channels*patch^2 must be a multiple of 8");
  return xclip_patchify_gather_rows(img, B, C, H, W, patch, keep, k, out,
                                    (int64_t)patch * patch * C, stream);
}

namespace xclip {
template <int V>
static void launch_scatter_vec(int C, dim3 grid, cudaStream_t s, const float* src, long long lds, int B,
                               int H, int W, int P, const long long* keep, int k, int n_patches,
                               int ppc, float* img) {
  switch (C) {
    case 1: patchify_scatter_kernel<1, V><<<grid, 256, 0, s>>>(src, lds, B, C, H, W, P, keep, k, n_patches, ppc, img); break;
    case 2: patchify_scatter_kernel<2, V><<<grid, 256, 0, s>>>(src, lds, B, C, H, W, P, keep, k, n_patches, ppc, img); break;
    case 3: patchify_scatter_kernel<3, V><<<grid, 256, 0, s>>>(src, lds, B, C, H, W, P, keep, k, n_patches, ppc, img); break;
    default: patchify_scatter_kernel<4, V><<<grid, 256, 0, s>>>(src, lds, B, C, H, W, P, keep, k, n_patches, ppc, img); break;
  }
}
}  // namespace xclip

extern "C" int xclip_patchify_scatter_rows(const float* src, int64_t lds, int B, int C, int H, int W,
                                           int patch, const int64_t* keep, int k, float* img_grad,
                                           xclip_stream_t stream) {
  using namespace xclip;
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(src && img_grad && B > 0 && C > 0 && patch > 0 && H % patch == 0 && W % patch == 0,
                "patchify_scatter: bad arguments");
  const int n_patches = (H / patch) * (W / patch);
  const long long patch_dim = (long long)patch * patch * C;
  XCLIP_REQUIRE(k > 0 && k <= n_patches && (keep != nullptr || k == n_patches), "patchify_scatter: k=%d", k);
  XCLIP_REQUIRE(lds >= patch_dim && lds % 4 == 0 && (reinterpret_cast<uintptr_t>(src) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(img_grad) & 15) == 0,
                "patchify_scatter: src and img_grad must be 16-byte aligned with lds %% 4 == 0");
  // about 8 blocks per SM in all, at most kScatterMaxPatchesPerBlock patches per block
  const long long target = (long long)num_sms() * 8;
  long long chunks = (target + B - 1) / B;
  if (chunks > n_patches) chunks = n_patches;
  int ppc = (int)((n_patches + chunks - 1) / chunks);
  if (ppc > kScatterMaxPatchesPerBlock) ppc = kScatterMaxPatchesPerBlock;
  chunks = (n_patches + ppc - 1) / ppc;
  XCLIP_REQUIRE(chunks <= 65535, "patchify_scatter: %d patches per image", n_patches);
  dim3 grid((unsigned)B, (unsigned)chunks);
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const long long* kp = reinterpret_cast<const long long*>(keep);
  if (patch % 4 == 0 && C <= 4) {
    launch_scatter_vec<4>(C, grid, s, src, lds, B, H, W, patch, kp, k, n_patches, ppc, img_grad);
  } else if (patch % 2 == 0 && C <= 4) {
    launch_scatter_vec<2>(C, grid, s, src, lds, B, H, W, patch, kp, k, n_patches, ppc, img_grad);
  } else {
    patchify_scatter_kernel<0, 1><<<grid, 256, 0, s>>>(src, lds, B, C, H, W, patch, kp, k, n_patches, ppc, img_grad);
  }
  XCLIP_LAUNCH_CHECK("patchify_scatter_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_patchify_scatter(const float* src, int64_t lds, int B, int C, int H, int W, int patch,
                                      const int64_t* keep, int k, float* img_grad, xclip_stream_t stream) {
  using namespace xclip;
  XCLIP_REQUIRE(((long long)patch * patch * C) % 8 == 0,
                "patchify_scatter: channels*patch^2 must be a multiple of 8");
  return xclip_patchify_scatter_rows(src, lds, B, C, H, W, patch, keep, k, img_grad, stream);
}

extern "C" int xclip_scatter_add_rows(const int32_t* idx, int period, const void* src, int64_t lds,
                                      float* dst, int64_t rows, int d, int V, xclip_stream_t stream) {
  using namespace xclip;
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(src && dst && rows > 0 && d % 8 == 0 && V > 0 && (idx != nullptr || period > 0),
                "scatter_add_rows: bad arguments");
  XCLIP_REQUIRE(lds % 8 == 0 && lds >= d && (reinterpret_cast<uintptr_t>(src) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(dst) & 15) == 0,
                "scatter_add_rows: misaligned");
  long long blocks = (rows + 7) / 8;
  if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
  scatter_add_rows_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      idx, period, reinterpret_cast<const bf16*>(src), lds, dst, rows, d, V);
  XCLIP_LAUNCH_CHECK("scatter_add_rows_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_colsum_rows(const void* src, int64_t lds, float* dst, int64_t rows, int d,
                                 xclip_stream_t stream) {
  using namespace xclip;
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(src && dst && rows > 0 && d % 2 == 0, "colsum_rows: bad arguments");
  int slices = (int)(rows < 256 ? rows : 256);
  dim3 grid((d + 511) / 512, slices);
  colsum_rows_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const bf16*>(src), lds, dst, rows, d, slices);
  XCLIP_LAUNCH_CHECK("colsum_rows_kernel");
  return XCLIP_OK;
}
