// Fused attention core of x_clip/x_clip.py:217-244 for dim_head = 64 and n <= 320 (sm_90a).
//
// One CTA = 4 warps = 64 rows of one (batch, head) (1-D grid: row block fastest, then head, then
// batch); every warp owns 16 rows and runs bf16
// m16n8k16 tensor-core MMAs on fragments loaded from XOR-swizzled shared memory with ldmatrix.
// A whole head's keys and values (<= 320 x 64 bf16 each) fit in shared memory, so each CTA loads
// its operands once and loops over 64-wide blocks in shared memory.
//   forward : O = softmax(scale q k^T) v with an online softmax; lse = base-2 log-sum-exp.
//   backward: delta = rowsum(dO * O); one kernel per 64-key block accumulates dK, dV over all
//             queries, one per 64-query block accumulates dQ over all keys (P and dP recomputed),
//             so every gradient is written exactly once, without atomics.
// Masking follows the reference: a masked key (key_mask = 0, or j > i under the causal mask of
// :233-236) gets the score -FLT_MAX after scaling; keys beyond n do not exist (-inf).
#include "common.cuh"
#include "host.h"

namespace xclip {

constexpr int kAttnDh = 64;
constexpr int kAttnRows = 64;       // rows (queries or keys) per CTA
constexpr int kAttnThreads = 128;
constexpr float kLog2e = 1.4426950408889634f;

// byte offset of 16-byte chunk `chunk` of row `row` in a [rows x 64] bf16 tile (128 B rows)
__device__ __forceinline__ uint32_t attn_swz(int row, int chunk) {
  return (uint32_t)(row * 128 + ((chunk ^ (row & 7)) << 4));
}

// rows [row0, row0 + rows) of a 64-wide bf16 slice (row stride ld) -> swizzled smem; rows >= n are zero
__device__ __forceinline__ void attn_load_rows(uint8_t* dst, const bf16* src, long long ld, int row0,
                                               int rows, int n) {
  const uint32_t base = smem_u32(dst);
  for (int idx = threadIdx.x; idx < rows * 8; idx += kAttnThreads) {
    const int r = idx >> 3, c = idx & 7;
    const int gr = row0 + r;
    const bf16* g = src + (long long)(gr < n ? gr : 0) * ld + c * 8;
    const uint32_t bytes = gr < n ? 16u : 0u;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(base + attn_swz(r, c)), "l"(g),
                 "r"(bytes)
                 : "memory");
  }
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr));
}
// c[16 x 8] += a[16 x 16] * b[16 x 8]  (bf16 in, fp32 accumulate)
__device__ __forceinline__ void mma_bf16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}

// A fragments (16 rows x 64) of this warp's rows [r0, r0 + 16) of a swizzled tile
__device__ __forceinline__ void load_a_frags(const uint8_t* tile, int r0, uint32_t (&f)[4][4]) {
  const int lane = threadIdx.x & 31;
  const int r = r0 + (lane & 15);
#pragma unroll
  for (int ks = 0; ks < 4; ++ks) ldsm_x4(smem_u32(tile) + attn_swz(r, ks * 2 + (lane >> 4)), f[ks]);
}

// acc[16 x 64] += A[16 x 64 (k)] * T[c0 .. c0 + 64, :]^T : T rows are the output columns, the
// contraction runs over the 64 features of T (q k^T, dO v^T)
__device__ __forceinline__ void mma_abt(float (&acc)[8][4], const uint32_t (&a)[4][4], const uint8_t* t, int c0) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int ks = 0; ks < 4; ++ks)
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b[4];
      ldsm_x4(smem_u32(t) + attn_swz(c0 + np * 16 + (lane >> 4) * 8 + (lane & 7), ks * 2 + ((lane >> 3) & 1)), b);
      mma_bf16(acc[2 * np], a[ks], b[0], b[1]);
      mma_bf16(acc[2 * np + 1], a[ks], b[2], b[3]);
    }
}

// acc[16 x 64] += P[16 x 64 (k)] * T[k0 .. k0 + 64, :] : the contraction runs over T's rows (p v, ds k)
__device__ __forceinline__ void mma_ab(float (&acc)[8][4], const uint32_t (&p)[4][4], const uint8_t* t, int k0) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk)
#pragma unroll
    for (int dp = 0; dp < 4; ++dp) {
      uint32_t b[4];
      ldsm_x4_t(smem_u32(t) + attn_swz(k0 + kk * 16 + (lane & 7) + ((lane >> 3) & 1) * 8, dp * 2 + (lane >> 4)), b);
      mma_bf16(acc[2 * dp], p[kk], b[0], b[1]);
      mma_bf16(acc[2 * dp + 1], p[kk], b[2], b[3]);
    }
}

// accumulator fragments of a 16 x 64 block -> bf16 A fragments (the C and A layouts line up)
__device__ __forceinline__ void acc_to_a(const float (&s)[8][4], uint32_t (&p)[4][4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    p[kk][0] = pack_bf16x2(s[2 * kk][0], s[2 * kk][1]);
    p[kk][1] = pack_bf16x2(s[2 * kk][2], s[2 * kk][3]);
    p[kk][2] = pack_bf16x2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
    p[kk][3] = pack_bf16x2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
  }
}

__device__ __forceinline__ void zero_acc(float (&a)[8][4]) {
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int e = 0; e < 4; ++e) a[i][e] = 0.f;
}

// key flags: 0 = attend, 1 = masked (score -FLT_MAX), 2 = no such key (j >= n)
__device__ __forceinline__ void load_key_flags(uint8_t* flags, const uint8_t* mask, int b, int n, int j0, int cnt) {
  for (int j = threadIdx.x; j < cnt; j += kAttnThreads) {
    const int gj = j0 + j;
    flags[j] = gj >= n ? 2 : ((mask != nullptr && !mask[(long long)b * n + gj]) ? 1 : 0);
  }
}

// scaled, masked score in the base-2 domain
__device__ __forceinline__ float attn_t(float s, float scale_log2, int flag, bool causal_masked) {
  if (flag == 2) return -INFINITY;
  if (flag == 1 || causal_masked) return -FLT_MAX;
  return s * scale_log2;
}

// writes a 16 x 64 fp32 fragment block (rows r0.., scaled) as bf16 into rows of `dst` (< n only)
__device__ __forceinline__ void store_rows(bf16* dst, long long ld, int r0, int n, const float (&a)[8][4], float mul) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int r = r0 + (lane >> 2) + 8 * half;
    if (r >= n) continue;
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const int c = nt * 8 + 2 * (lane & 3);
      *reinterpret_cast<uint32_t*>(dst + (long long)r * ld + c) =
          pack_bf16x2(a[nt][2 * half] * mul, a[nt][2 * half + 1] * mul);
    }
  }
}

template <bool kCausal>
__global__ void __launch_bounds__(kAttnThreads)
attn_fwd_kernel(const bf16* __restrict__ qkv, long long ld, const uint8_t* __restrict__ mask,
                bf16* __restrict__ o, long long ldo, float* __restrict__ lse, int n, int H, float scale_log2) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int NP = (n + 63) & ~63;
  uint8_t* sQ = sm;
  uint8_t* sK = sQ + kAttnRows * 128;
  uint8_t* sV = sK + NP * 128;
  uint8_t* sFlag = sV + NP * 128;
  const int nblk = NP / kAttnRows, bh_ = blockIdx.x / nblk;
  const int b = bh_ / H, h = bh_ % H;
  const int q0 = (blockIdx.x % nblk) * kAttnRows;
  const bf16* base = qkv + (long long)b * n * ld;
  attn_load_rows(sQ, base + h * kAttnDh, ld, q0, kAttnRows, n);
  attn_load_rows(sK, base + (H + h) * kAttnDh, ld, 0, NP, n);
  attn_load_rows(sV, base + (2 * H + h) * kAttnDh, ld, 0, NP, n);
  load_key_flags(sFlag, mask, b, n, 0, NP);
  cp_async_wait_all();
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = warp * 16;
  uint32_t qf[4][4];
  load_a_frags(sQ, r0, qf);
  const int row[2] = {q0 + r0 + (lane >> 2), q0 + r0 + (lane >> 2) + 8};
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float oacc[8][4];
  zero_acc(oacc);

  for (int kb = 0; kb < NP; kb += 64) {
    float s[8][4];
    zero_acc(s);
    mma_abt(s, qf, sK, kb);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = kb + nt * 8 + 2 * (lane & 3) + (e & 1);
        const float t = attn_t(s[nt][e], scale_log2, sFlag[col], kCausal && col > row[e >> 1]);
        s[nt][e] = t;
        mx[e >> 1] = fmaxf(mx[e >> 1], t);
      }
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 1));
      mx[hh] = fmaxf(mx[hh], __shfl_xor_sync(0xffffffffu, mx[hh], 2));
      const float mn = fmaxf(m[hh], mx[hh]);
      const float corr = exp2f(m[hh] - mn);
      m[hh] = mn;
      l[hh] *= corr;
#pragma unroll
      for (int nt = 0; nt < 8; ++nt) {
        oacc[nt][2 * hh] *= corr;
        oacc[nt][2 * hh + 1] *= corr;
      }
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = exp2f(s[nt][e] - m[e >> 1]);
        s[nt][e] = pv;
        l[e >> 1] += pv;
      }
    uint32_t pf[4][4];
    acc_to_a(s, pf);
    mma_ab(oacc, pf, sV, kb);
  }
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 1);
    l[hh] += __shfl_xor_sync(0xffffffffu, l[hh], 2);
  }
  const float inv[2] = {1.f / l[0], 1.f / l[1]};
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) oacc[nt][e] *= inv[e >> 1];
  store_rows(o + (long long)b * n * ldo + h * kAttnDh, ldo, q0 + r0, n, oacc, 1.f);
  if ((lane & 3) == 0) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      if (row[hh] < n) lse[((long long)b * H + h) * n + row[hh]] = m[hh] + log2f(l[hh]);
  }
}

// delta[b,h,i] = sum_d dO[b,i,h,d] * O[b,i,h,d]; one warp per (token, 4 heads at a time)
__global__ void __launch_bounds__(256)
attn_delta_kernel(const bf16* __restrict__ o, long long ldo, const bf16* __restrict__ d_o,
                  long long lddo, float* __restrict__ delta, int B, int n, int H) {
  const int lane = threadIdx.x & 31;
  const long long warp = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5;
  const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
  const long long tokens = (long long)B * n;
  const int groups = (H + 3) / 4;  // 4 heads (256 elements) per warp pass, 8 lanes per head
  for (long long w = warp; w < tokens * groups; w += nwarps) {
    const long long tok = w / groups;
    const int hg = (int)(w % groups);
    const int h = hg * 4 + (lane >> 3);
    float s = 0.f;
    if (h < H) {
      const int col = h * kAttnDh + (lane & 7) * 8;
      const uint4 a = *reinterpret_cast<const uint4*>(o + tok * ldo + col);
      const uint4 c = *reinterpret_cast<const uint4*>(d_o + tok * lddo + col);
      const uint32_t aa[4] = {a.x, a.y, a.z, a.w}, cc[4] = {c.x, c.y, c.z, c.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float2 x = unpack_bf16x2(aa[i]), y = unpack_bf16x2(cc[i]);
        s += x.x * y.x + x.y * y.y;
      }
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    s += __shfl_xor_sync(0xffffffffu, s, 2);
    s += __shfl_xor_sync(0xffffffffu, s, 4);
    if (h < H && (lane & 7) == 0) {
      const long long b = tok / n, i = tok % n;
      delta[(b * H + h) * n + i] = s;
    }
  }
}

// dK, dV of the 64 keys [k0, k0 + 64) of one (batch, head): loops over all queries.
// The warp's accumulators are S^T / dP^T (keys x queries), so P^T and dS^T feed the next MMAs
// straight from registers.
template <bool kCausal>
__global__ void __launch_bounds__(kAttnThreads)
attn_bwd_dkdv_kernel(const bf16* __restrict__ qkv, long long ld, const uint8_t* __restrict__ mask,
                     const bf16* __restrict__ d_o, long long lddo, const float* __restrict__ lse,
                     const float* __restrict__ delta, bf16* __restrict__ dqkv, long long ldd, int n, int H,
                     float scale, float scale_log2) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int NP = (n + 63) & ~63;
  uint8_t* sK = sm;
  uint8_t* sV = sK + kAttnRows * 128;
  uint8_t* sQ = sV + kAttnRows * 128;
  uint8_t* sdO = sQ + NP * 128;
  float* sLse = reinterpret_cast<float*>(sdO + NP * 128);
  float* sDelta = sLse + NP;
  uint8_t* sFlag = reinterpret_cast<uint8_t*>(sDelta + NP);
  const int nblk = NP / kAttnRows, bh_ = blockIdx.x / nblk;
  const int b = bh_ / H, h = bh_ % H;
  const int k0 = (blockIdx.x % nblk) * kAttnRows;
  const bf16* base = qkv + (long long)b * n * ld;
  attn_load_rows(sK, base + (H + h) * kAttnDh, ld, k0, kAttnRows, n);
  attn_load_rows(sV, base + (2 * H + h) * kAttnDh, ld, k0, kAttnRows, n);
  attn_load_rows(sQ, base + h * kAttnDh, ld, 0, NP, n);
  attn_load_rows(sdO, d_o + (long long)b * n * lddo + h * kAttnDh, lddo, 0, NP, n);
  const long long bh = (long long)b * H + h;
  for (int i = threadIdx.x; i < NP; i += kAttnThreads) {
    sLse[i] = i < n ? lse[bh * n + i] : 0.f;
    sDelta[i] = i < n ? delta[bh * n + i] : 0.f;
  }
  load_key_flags(sFlag, mask, b, n, k0, kAttnRows);
  cp_async_wait_all();
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = warp * 16;
  uint32_t kf[4][4], vf[4][4];
  load_a_frags(sK, r0, kf);
  load_a_frags(sV, r0, vf);
  const int kr[2] = {r0 + (lane >> 2), r0 + (lane >> 2) + 8};   // key rows inside the block
  const int flag[2] = {sFlag[kr[0]], sFlag[kr[1]]};
  float dk[8][4], dv[8][4];
  zero_acc(dk);
  zero_acc(dv);

  for (int qb = 0; qb < NP; qb += 64) {
    float st[8][4], dpt[8][4];
    zero_acc(st);
    zero_acc(dpt);
    mma_abt(st, kf, sQ, qb);
    mma_abt(dpt, vf, sdO, qb);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int q = qb + nt * 8 + 2 * (lane & 3) + (e & 1);
        const int key = k0 + kr[e >> 1];
        const float t = q < n ? attn_t(st[nt][e], scale_log2, flag[e >> 1], kCausal && key > q) : -INFINITY;
        const float pv = exp2f(t - sLse[q]);
        st[nt][e] = pv;
        dpt[nt][e] = pv * (dpt[nt][e] - sDelta[q]);
      }
    uint32_t pf[4][4], df[4][4];
    acc_to_a(st, pf);
    acc_to_a(dpt, df);
    mma_ab(dv, pf, sdO, qb);
    mma_ab(dk, df, sQ, qb);
  }
  bf16* out = dqkv + (long long)b * n * ldd;
  store_rows(out + (H + h) * kAttnDh, ldd, k0 + r0, n, dk, scale);
  store_rows(out + (2 * H + h) * kAttnDh, ldd, k0 + r0, n, dv, 1.f);
}

// dQ of the 64 queries [q0, q0 + 64) of one (batch, head): loops over all keys.
template <bool kCausal>
__global__ void __launch_bounds__(kAttnThreads)
attn_bwd_dq_kernel(const bf16* __restrict__ qkv, long long ld, const uint8_t* __restrict__ mask,
                   const bf16* __restrict__ d_o, long long lddo, const float* __restrict__ lse,
                   const float* __restrict__ delta, bf16* __restrict__ dqkv, long long ldd, int n, int H,
                   float scale, float scale_log2) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int NP = (n + 63) & ~63;
  uint8_t* sQ = sm;
  uint8_t* sdO = sQ + kAttnRows * 128;
  uint8_t* sK = sdO + kAttnRows * 128;
  uint8_t* sV = sK + NP * 128;
  uint8_t* sFlag = sV + NP * 128;
  const int nblk = NP / kAttnRows, bh_ = blockIdx.x / nblk;
  const int b = bh_ / H, h = bh_ % H;
  const int q0 = (blockIdx.x % nblk) * kAttnRows;
  const bf16* base = qkv + (long long)b * n * ld;
  attn_load_rows(sQ, base + h * kAttnDh, ld, q0, kAttnRows, n);
  attn_load_rows(sdO, d_o + (long long)b * n * lddo + h * kAttnDh, lddo, q0, kAttnRows, n);
  attn_load_rows(sK, base + (H + h) * kAttnDh, ld, 0, NP, n);
  attn_load_rows(sV, base + (2 * H + h) * kAttnDh, ld, 0, NP, n);
  load_key_flags(sFlag, mask, b, n, 0, NP);
  cp_async_wait_all();
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = warp * 16;
  uint32_t qf[4][4], of[4][4];
  load_a_frags(sQ, r0, qf);
  load_a_frags(sdO, r0, of);
  const long long bh = (long long)b * H + h;
  const int row[2] = {q0 + r0 + (lane >> 2), q0 + r0 + (lane >> 2) + 8};
  float lr[2], dr[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    lr[hh] = row[hh] < n ? lse[bh * n + row[hh]] : 0.f;
    dr[hh] = row[hh] < n ? delta[bh * n + row[hh]] : 0.f;
  }
  float dq[8][4];
  zero_acc(dq);
  for (int kb = 0; kb < NP; kb += 64) {
    float s[8][4], dp[8][4];
    zero_acc(s);
    zero_acc(dp);
    mma_abt(s, qf, sK, kb);
    mma_abt(dp, of, sV, kb);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = kb + nt * 8 + 2 * (lane & 3) + (e & 1);
        const float t = attn_t(s[nt][e], scale_log2, sFlag[col], kCausal && col > row[e >> 1]);
        const float pv = row[e >> 1] < n ? exp2f(t - lr[e >> 1]) : 0.f;
        s[nt][e] = pv * (dp[nt][e] - dr[e >> 1]);
      }
    uint32_t df[4][4];
    acc_to_a(s, df);
    mma_ab(dq, df, sK, kb);
  }
  store_rows(dqkv + (long long)b * n * ldd + h * kAttnDh, ldd, q0 + r0, n, dq, scale);
}

}  // namespace xclip

using namespace xclip;

extern "C" int xclip_attn_fwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask, void* o,
                              int64_t ldo, float* lse, int B, int n, int heads, float scale,
                              int causal, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(qkv && o && lse, "attn_fwd: null pointer");
  XCLIP_REQUIRE(B > 0 && heads > 0 && n > 0, "attn_fwd: bad sizes B=%d n=%d heads=%d", B, n, heads);
  XCLIP_REQUIRE(n <= 320, "attn_fwd: sequence length %d > 320 is not supported by this kernel", n);
  XCLIP_REQUIRE(scale > 0.f, "attn_fwd: scale must be positive");
  XCLIP_REQUIRE(ld_qkv % 8 == 0 && ld_qkv >= 3 * heads * kAttnDh, "attn_fwd: bad ld_qkv");
  XCLIP_REQUIRE(ldo % 8 == 0 && ldo >= heads * kAttnDh, "attn_fwd: bad ldo");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(o) & 15) == 0,
                "attn_fwd: misaligned pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int NP = (n + 63) & ~63;
  const int smem = kAttnRows * 128 + 2 * NP * 128 + NP;
  const long long blocks = (long long)(NP / kAttnRows) * B * heads;
  XCLIP_REQUIRE(blocks <= 0x7fffffffLL, "attn: B=%d x heads=%d is too large", B, heads);
  const dim3 grid((unsigned)blocks);
  auto kern = causal ? attn_fwd_kernel<true> : attn_fwd_kernel<false>;
  rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), smem);
  if (rc) return rc;
  kern<<<grid, kAttnThreads, smem, s>>>(reinterpret_cast<const bf16*>(qkv), ld_qkv, key_mask,
                                        reinterpret_cast<bf16*>(o), ldo, lse, n, heads,
                                        scale * kLog2e);
  XCLIP_LAUNCH_CHECK("attn_fwd_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_attn_bwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask,
                              const void* o, int64_t ldo, const void* d_o, int64_t lddo,
                              const float* lse, float* delta, void* dqkv, int64_t ld_dqkv,
                              float* dq_workspace, int B, int n, int heads, float scale,
                              int causal, xclip_stream_t stream) {
  (void)dq_workspace;
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(qkv && o && d_o && lse && delta && dqkv, "attn_bwd: null pointer");
  XCLIP_REQUIRE(B > 0 && heads > 0 && n > 0 && n <= 320, "attn_bwd: bad sizes B=%d n=%d heads=%d",
                B, n, heads);
  XCLIP_REQUIRE(ld_qkv % 8 == 0 && ld_qkv >= 3 * heads * kAttnDh && ld_dqkv % 8 == 0 &&
                    ld_dqkv >= 3 * heads * kAttnDh && ldo % 8 == 0 && lddo % 8 == 0 &&
                    ldo >= heads * kAttnDh && lddo >= heads * kAttnDh,
                "attn_bwd: bad leading dimensions");
  XCLIP_REQUIRE(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(o) |
                  reinterpret_cast<uintptr_t>(d_o) | reinterpret_cast<uintptr_t>(dqkv)) & 15) == 0,
                "attn_bwd: misaligned pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  {
    const long long warps = (long long)B * n * ((heads + 3) / 4);
    long long blocks = (warps + 7) / 8;
    if (blocks > (long long)num_sms() * 8) blocks = (long long)num_sms() * 8;
    attn_delta_kernel<<<(int)blocks, 256, 0, s>>>((const bf16*)o, ldo, (const bf16*)d_o, lddo,
                                                  delta, B, n, heads);
    XCLIP_LAUNCH_CHECK("attn_delta_kernel");
  }
  const int NP = (n + 63) & ~63;
  const long long blocks = (long long)(NP / kAttnRows) * B * heads;
  XCLIP_REQUIRE(blocks <= 0x7fffffffLL, "attn: B=%d x heads=%d is too large", B, heads);
  const dim3 grid((unsigned)blocks);
  const bf16* q = reinterpret_cast<const bf16*>(qkv);
  const bf16* g = reinterpret_cast<const bf16*>(d_o);
  bf16* d = reinterpret_cast<bf16*>(dqkv);
  const float sl2 = scale * kLog2e;
  {
    const int smem = 2 * kAttnRows * 128 + 2 * NP * 128 + 2 * NP * 4 + kAttnRows;
    auto kern = causal ? attn_bwd_dkdv_kernel<true> : attn_bwd_dkdv_kernel<false>;
    rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), smem);
    if (rc) return rc;
    kern<<<grid, kAttnThreads, smem, s>>>(q, ld_qkv, key_mask, g, lddo, lse, delta, d, ld_dqkv, n, heads,
                                          scale, sl2);
    XCLIP_LAUNCH_CHECK("attn_bwd_dkdv_kernel");
  }
  {
    const int smem = 2 * kAttnRows * 128 + 2 * NP * 128 + NP;
    auto kern = causal ? attn_bwd_dq_kernel<true> : attn_bwd_dq_kernel<false>;
    rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), smem);
    if (rc) return rc;
    kern<<<grid, kAttnThreads, smem, s>>>(q, ld_qkv, key_mask, g, lddo, lse, delta, d, ld_dqkv, n, heads,
                                          scale, sl2);
    XCLIP_LAUNCH_CHECK("attn_bwd_dq_kernel");
  }
  return XCLIP_OK;
}
