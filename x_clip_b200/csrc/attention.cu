// Fused attention core of x_clip/x_clip.py:217-244 for dim_head = 64 and any sequence length (sm_90a).
//
// One CTA = 4 warps = 64 rows of one (batch, head) (1-D grid: row block fastest, then head, then
// batch); every warp owns 16 rows and runs bf16
// m16n8k16 tensor-core MMAs on fragments loaded from XOR-swizzled shared memory with ldmatrix.
//   forward : O = softmax(scale q k^T) v with an online softmax; lse = base-2 log-sum-exp.
//   backward: delta = rowsum(dO * O); one kernel per 64-key block accumulates dK, dV over all
//             queries, one per 64-query block accumulates dQ over all keys (P and dP recomputed),
//             so every gradient is written exactly once, without atomics.
// Two schedules run the same per-block bodies (attn_*_block) in the same block order, so they give
// bit-identical results:
//   resident  (n <= 320): a whole head's other operand (<= 320 x 64 bf16 per tensor) is loaded into
//             shared memory once and the CTA loops over its 64-row blocks there (up to ~100 KB).
//   streaming (n > 320) : only the CTA's own 64-row block stays on chip; the other operand passes
//             through a 2-stage cp.async ring of 64-row blocks (with their key flags or lse / delta
//             values), ~40-50 KB per CTA whatever n is.  XCLIP_TUNE_ATTN_STREAM forces it for any n.
// Masking follows the reference: a masked key (key_mask = 0, or j > i under the causal mask of
// :233-236) gets the score -FLT_MAX after scaling; keys beyond n do not exist (-inf).  Causal blocks
// wholly above the diagonal are not skipped: a row whose visible keys are all key-masked gets the
// reference's uniform softmax over all n keys, and lse = -FLT_MAX (-FLT_MAX + log2(n) rounds to
// -FLT_MAX; no row with a visible key can have that lse).  Its backward follows masked_fill, which
// passes no gradient to a masked score: dq = 0, nothing into dk, and dO / n into the dv of every key.
// The backward kernels read such a row's lse as +inf, so the block bodies give it p = 0 everywhere
// (on every other row a hidden score already has p = 0 exactly, hence ds = 0), and the dK / dV
// kernels add its dO / n to dv after the key loop (attn_dv_empty_rows).
// Every kernel is also instantiated with kDropout (xclip_attn_dropout_*): the block bodies then drop
// probabilities with a Philox mask that is a function of the element alone (see AttnDrop); the
// kDropout = false instantiations are the plain kernels.
#include "common.cuh"
#include "host.h"
#include "philox.cuh"

namespace xclip {

constexpr int kAttnDh = 64;
constexpr int kAttnRows = 64;       // rows (queries or keys) per CTA
constexpr int kAttnThreads = 128;
constexpr int kAttnTile = kAttnRows * 128;  // bytes of one swizzled 64 x 64 bf16 tile
constexpr int kAttnResidentMaxN = 320;      // longest sequence the resident kernels take
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
__device__ __forceinline__ uint8_t key_flag(const uint8_t* mask, int b, int n, int gj) {
  return gj >= n ? 2 : ((mask != nullptr && !mask[(long long)b * n + gj]) ? 1 : 0);
}
__device__ __forceinline__ void load_key_flags(uint8_t* flags, const uint8_t* mask, int b, int n, int j0, int cnt) {
  for (int j = threadIdx.x; j < cnt; j += kAttnThreads) flags[j] = key_flag(mask, b, n, j0 + j);
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

// lse as the backward reads it: +inf for a row with no visible key (-FLT_MAX), so that the block
// bodies give it p = exp2(t - lse) = 0 on every key, hence ds = 0 and nothing into dq, dk or dv
__device__ __forceinline__ float attn_bwd_lse(float lse) { return lse == -FLT_MAX ? INFINITY : lse; }

// dv += (sum of dO_i over the head's rows i with no visible key) / n: the reference's uniform p = 1/n
// of those rows, the same for every key.  Called by all threads after the key loop when such a row
// exists; `scratch` is 128 floats of shared memory that the key loop does not read.
__device__ __forceinline__ void attn_dv_empty_rows(float (&dv)[8][4], const bf16* dO, long long lddo,
                                                   const float* lse_bh, int n, float* scratch) {
  const int lane = threadIdx.x & 31, d = threadIdx.x & 63;
  float sum = 0.f;
  for (int i = threadIdx.x >> 6; i < n; i += 2)
    if (lse_bh[i] == -FLT_MAX) sum += __bfloat162float(dO[(long long)i * lddo + d]);
  __syncthreads();   // no warp still loads its fragments from the scratch tile
  scratch[threadIdx.x] = sum;
  __syncthreads();
  const float inv_n = 1.f / (float)n;
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int c = nt * 8 + 2 * (lane & 3) + (e & 1);
      dv[nt][e] += (scratch[c] + scratch[kAttnRows + c]) * inv_n;
    }
}

// ---- attention dropout (DESIGN.md, Dropout) ------------------------------------------------------
// Element (b, h, i, j) of layer L is kept iff word j & 3 of philox4x32_10((j >> 2, i, b H + h, L), seed)
// is <= keep_le, so the mask is a function of the element alone: every schedule and block order
// draws the same one.  A kept p is scaled by inv_keep = 1 / (1 - p) before it meets V or dP.
struct AttnDrop {
  const uint64_t* seed;   // the 64-bit Philox key, read on the device (low word first)
  uint32_t keep_le;       // round((1 - p) 2^32) - 1, saturated at 2^32 - 1
  float inv_keep;         // 1 / (1 - p); 0 at p = 1, which drops every element
  uint32_t layer;
};

// what a thread of a dropout kernel needs: the kernel's AttnDrop (read from the parameter bank where
// used, so that it holds no registers through the block loops), the counter's b H + h word and the
// warp's 32-word staging area for one block's mask bits
struct DropCtx {
  const AttnDrop& d;
  uint32_t bh;
  uint32_t* bits;
};

template <bool kDropout>
__device__ __forceinline__ DropCtx drop_ctx(const AttnDrop& d, long long bh) {
  if constexpr (kDropout) {
    __shared__ uint32_t bits[kAttnThreads];   // 512 B, in the dropout kernels only
    return DropCtx{d, (uint32_t)bh, bits + (threadIdx.x & ~31)};
  } else {
    return DropCtx{d, 0u, nullptr};
  }
}

// the Philox key: the seed, re-read (an L1 hit) by every block instead of held in registers
__device__ __forceinline__ uint2 drop_key(const DropCtx& dc) {
  const unsigned long long s = __ldg(reinterpret_cast<const unsigned long long*>(dc.d.seed));
  return make_uint2((uint32_t)s, (uint32_t)(s >> 32));
}

__device__ __forceinline__ uint32_t drop_keep4(uint4 w, uint32_t le) {
  return (uint32_t)(w.x <= le) | ((uint32_t)(w.y <= le) << 1) | ((uint32_t)(w.z <= le) << 2) |
         ((uint32_t)(w.w <= le) << 3);
}

// Mask bits of the warp's 16 rows [i0, i0 + 16) x 64 keys [j0, j0 + 64) (forward and dQ blocks):
// word 2 r + h holds keys j0 + 32 h + [0, 32) of row i0 + r.  8 Philox calls per lane, none wasted.
__device__ __forceinline__ void drop_bits_rows(const DropCtx& dc, int i0, int j0) {
  const int lane = threadIdx.x & 31;
  const uint32_t jg = (uint32_t)(j0 + (lane & 1) * 32) >> 2, i = (uint32_t)(i0 + (lane >> 1));
  const uint2 key = drop_key(dc);
  uint32_t w = 0;
#pragma unroll
  for (int g = 0; g < 8; ++g)
    w |= drop_keep4(philox4x32_10(make_uint4(jg + g, i, dc.bh, dc.d.layer), key), dc.d.keep_le) << (4 * g);
  __syncwarp();   // every lane has read the previous block's bits
  dc.bits[lane] = w;
  __syncwarp();
}
// row hh (0: lane / 4, 1: lane / 4 + 8) of the warp's 16, key nt * 8 + 2 (lane & 3) + e1 of the block
__device__ __forceinline__ float drop_mul_rows(const DropCtx& dc, int hh, int nt, int e1) {
  const int lane = threadIdx.x & 31;
  const uint32_t w = dc.bits[((lane >> 2) + 8 * hh) * 2 + (nt >> 2)];
  return (w >> ((nt & 3) * 8 + 2 * (lane & 3) + e1)) & 1u ? dc.d.inv_keep : 0.f;
}

// Mask bits of the warp's 16 keys [j0, j0 + 16) x 64 rows [i0, i0 + 64) (dK / dV blocks): word m holds
// row i0 + 2 m in bits 0..15 and row i0 + 2 m + 1 in bits 16..31, bit = key - j0.
__device__ __forceinline__ void drop_bits_keys(const DropCtx& dc, int j0, int i0) {
  const int lane = threadIdx.x & 31;
  const uint32_t jg = (uint32_t)j0 >> 2;
  const uint2 key = drop_key(dc);
  uint32_t w = 0;
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int g = 0; g < 4; ++g)
      w |= drop_keep4(philox4x32_10(make_uint4(jg + g, (uint32_t)(i0 + 2 * lane + r), dc.bh, dc.d.layer), key),
                      dc.d.keep_le) << (16 * r + 4 * g);
  __syncwarp();
  dc.bits[lane] = w;
  __syncwarp();
}
// row nt * 8 + 2 (lane & 3) + e1 of the block, key hh (0: lane / 4, 1: lane / 4 + 8) of the warp's 16
__device__ __forceinline__ float drop_mul_keys(const DropCtx& dc, int hh, int nt, int e1) {
  const int lane = threadIdx.x & 31;
  const uint32_t w = dc.bits[nt * 4 + (lane & 3)];
  return (w >> (16 * e1 + (lane >> 2) + 8 * hh)) & 1u ? dc.d.inv_keep : 0.f;
}

// attn_dv_empty_rows under dropout: the uniform p = 1/n of a row with no visible key is dropped per
// key like any other p, so row i adds M_ij inv_keep dO_i / n to the dv of key j (one Philox call per
// row and key; such rows are the rare left padding of a causal caption or a wholly masked item).
__device__ __forceinline__ void attn_dv_empty_rows_drop(float (&dv)[8][4], const bf16* dO, long long lddo,
                                                        const float* lse_bh, int n, const int (&key)[2],
                                                        const DropCtx& dc) {
  const int lane = threadIdx.x & 31;
  const float w = dc.d.inv_keep / (float)n;
  const uint2 k = drop_key(dc);
  for (int i = 0; i < n; ++i) {
    if (lse_bh[i] != -FLT_MAX) continue;
    float mk[2];
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) {
      const uint4 r = philox4x32_10(make_uint4((uint32_t)key[hh] >> 2, (uint32_t)i, dc.bh, dc.d.layer), k);
      const int c = key[hh] & 3;
      const uint32_t word = c == 0 ? r.x : c == 1 ? r.y : c == 2 ? r.z : r.w;
      mk[hh] = word <= dc.d.keep_le ? w : 0.f;
    }
    const bf16* g = dO + (long long)i * lddo + 2 * (lane & 3);
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      const float2 x = unpack_bf16x2(*reinterpret_cast<const uint32_t*>(g + nt * 8));
      dv[nt][0] += mk[0] * x.x;
      dv[nt][1] += mk[0] * x.y;
      dv[nt][2] += mk[1] * x.x;
      dv[nt][3] += mk[1] * x.y;
    }
  }
}

// ---- per-block bodies, shared by the resident and the streaming kernels ---------------------------
// Each processes one 64-row block of the streamed operand for the warp's 16 rows.  The block's tiles
// sit at rows [c0, c0 + 64) of tK / tV (tQ / tdO); kb (qb) is the block's first global row and
// flags[j] (lse_b[j], delta_b[j]) belong to global row kb + j (qb + j).

// forward: s = q k^T, online-softmax update of (m, l, oacc), oacc += p v.  Under dropout l sums the
// undropped p (the lse is that of the whole row) and oacc takes p M / (1 - p).
template <bool kCausal, bool kDropout>
__device__ __forceinline__ void attn_fwd_block(const uint32_t (&qf)[4][4], const uint8_t* tK, const uint8_t* tV,
                                               int c0, const uint8_t* flags, int kb, const int (&row)[2],
                                               float scale_log2, float (&m)[2], float (&l)[2],
                                               float (&oacc)[8][4], const DropCtx& dc) {
  const int lane = threadIdx.x & 31;
  if constexpr (kDropout) drop_bits_rows(dc, row[0] - (lane >> 2), kb);
  float s[8][4];
  zero_acc(s);
  mma_abt(s, qf, tK, c0);
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = nt * 8 + 2 * (lane & 3) + (e & 1);
      const float t = attn_t(s[nt][e], scale_log2, flags[j], kCausal && kb + j > row[e >> 1]);
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
      if constexpr (kDropout) {
        s[nt][e] = pv * drop_mul_rows(dc, e >> 1, nt, e & 1);
      } else {
        s[nt][e] = pv;
      }
      l[e >> 1] += pv;
    }
  uint32_t pf[4][4];
  acc_to_a(s, pf);
  mma_ab(oacc, pf, tV, c0);
}

// forward epilogue: o = oacc / l for rows [rr0, rr0 + 16) (o and lse_bh point at this (batch, head))
__device__ __forceinline__ void attn_fwd_finish(float (&oacc)[8][4], const float (&m)[2], float (&l)[2],
                                                const int (&row)[2], bf16* o, long long ldo, int rr0,
                                                float* lse_bh, int n) {
  const int lane = threadIdx.x & 31;
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
  store_rows(o, ldo, rr0, n, oacc, 1.f);
  if ((lane & 3) == 0) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh)
      if (row[hh] < n) lse_bh[row[hh]] = m[hh] + log2f(l[hh]);
  }
}

// dK / dV: the warp's accumulators are S^T / dP^T (keys x queries), so P^T and dS^T feed the next
// MMAs straight from registers.  key[] are the thread's two global key rows, flag[] their flags.
// Under dropout dv takes (P M / (1 - p))^T dO and ds = p (dp M / (1 - p) - delta).
template <bool kCausal, bool kDropout>
__device__ __forceinline__ void attn_dkdv_block(const uint32_t (&kf)[4][4], const uint32_t (&vf)[4][4],
                                                const uint8_t* tQ, const uint8_t* tdO, int c0,
                                                const float* lse_b, const float* delta_b, int qb,
                                                const int (&key)[2], const int (&flag)[2], int n,
                                                float scale_log2, float (&dk)[8][4], float (&dv)[8][4],
                                                const DropCtx& dc) {
  const int lane = threadIdx.x & 31;
  if constexpr (kDropout) drop_bits_keys(dc, key[0] - (lane >> 2), qb);
  float st[8][4], dpt[8][4];
  zero_acc(st);
  zero_acc(dpt);
  mma_abt(st, kf, tQ, c0);
  mma_abt(dpt, vf, tdO, c0);
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = nt * 8 + 2 * (lane & 3) + (e & 1);
      const int q = qb + j;
      const float t = q < n ? attn_t(st[nt][e], scale_log2, flag[e >> 1], kCausal && key[e >> 1] > q) : -INFINITY;
      const float pv = exp2f(t - lse_b[j]);
      if constexpr (kDropout) {
        const float mul = drop_mul_keys(dc, e >> 1, nt, e & 1);
        st[nt][e] = pv * mul;
        dpt[nt][e] = pv * (dpt[nt][e] * mul - delta_b[j]);
      } else {
        st[nt][e] = pv;
        dpt[nt][e] = pv * (dpt[nt][e] - delta_b[j]);
      }
    }
  uint32_t pf[4][4], df[4][4];
  acc_to_a(st, pf);
  acc_to_a(dpt, df);
  mma_ab(dv, pf, tdO, c0);
  mma_ab(dk, df, tQ, c0);
}

// dQ: ds = p (dp - delta) over one block of keys, dq += ds k (a hidden score has p = 0, so ds = 0);
// under dropout dp is scaled by M / (1 - p) first
template <bool kCausal, bool kDropout>
__device__ __forceinline__ void attn_dq_block(const uint32_t (&qf)[4][4], const uint32_t (&of)[4][4],
                                              const uint8_t* tK, const uint8_t* tV, int c0,
                                              const uint8_t* flags, int kb, const int (&row)[2], int n,
                                              const float (&lr)[2], const float (&dr)[2], float scale_log2,
                                              float (&dq)[8][4], const DropCtx& dc) {
  const int lane = threadIdx.x & 31;
  if constexpr (kDropout) drop_bits_rows(dc, row[0] - (lane >> 2), kb);
  float s[8][4], dp[8][4];
  zero_acc(s);
  zero_acc(dp);
  mma_abt(s, qf, tK, c0);
  mma_abt(dp, of, tV, c0);
#pragma unroll
  for (int nt = 0; nt < 8; ++nt)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int j = nt * 8 + 2 * (lane & 3) + (e & 1);
      const float t = attn_t(s[nt][e], scale_log2, flags[j], kCausal && kb + j > row[e >> 1]);
      const float pv = row[e >> 1] < n ? exp2f(t - lr[e >> 1]) : 0.f;
      if constexpr (kDropout) {
        s[nt][e] = pv * (dp[nt][e] * drop_mul_rows(dc, e >> 1, nt, e & 1) - dr[e >> 1]);
      } else {
        s[nt][e] = pv * (dp[nt][e] - dr[e >> 1]);
      }
    }
  uint32_t df[4][4];
  acc_to_a(s, df);
  mma_ab(dq, df, tK, c0);
}

// ---- forward ------------------------------------------------------------------------------------
// resident: the head's whole K, V and key flags in shared memory
template <bool kCausal, bool kDropout>
__global__ void __launch_bounds__(kAttnThreads)
attn_fwd_kernel(const bf16* __restrict__ qkv, long long ld, const uint8_t* __restrict__ mask,
                bf16* __restrict__ o, long long ldo, float* __restrict__ lse, int n, int H, float scale_log2, AttnDrop drop) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int NP = (n + 63) & ~63;
  uint8_t* sQ = sm;
  uint8_t* sK = sQ + kAttnTile;
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
  const DropCtx dc = drop_ctx<kDropout>(drop, (long long)b * H + h);
  uint32_t qf[4][4];
  load_a_frags(sQ, r0, qf);
  const int row[2] = {q0 + r0 + (lane >> 2), q0 + r0 + (lane >> 2) + 8};
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float oacc[8][4];
  zero_acc(oacc);
  for (int kb = 0; kb < NP; kb += 64)
    attn_fwd_block<kCausal, kDropout>(qf, sK, sV, kb, sFlag + kb, kb, row, scale_log2, m, l, oacc, dc);
  attn_fwd_finish(oacc, m, l, row, o + (long long)b * n * ldo + h * kAttnDh, ldo, q0 + r0,
                  lse + ((long long)b * H + h) * n, n);
}

// streaming: the CTA's Q block stays; K, V and key flags of 64-key block i + 1 are fetched into the
// other ring stage while block i is computed (flags through a register, K and V by cp.async)
template <bool kCausal, bool kDropout>
__global__ void __launch_bounds__(kAttnThreads)
attn_fwd_stream_kernel(const bf16* __restrict__ qkv, long long ld, const uint8_t* __restrict__ mask,
                       bf16* __restrict__ o, long long ldo, float* __restrict__ lse, int n, int H,
                       float scale_log2, AttnDrop drop) {
  extern __shared__ __align__(128) uint8_t sm[];
  uint8_t* sQ = sm;
  uint8_t* ring = sQ + kAttnTile;            // stage s: K tile at ring + 2 s kAttnTile, V tile after it
  uint8_t* sFlag = ring + 4 * kAttnTile;     // stage s: 64 key flags at sFlag + 64 s
  const int nblk = (n + 63) / kAttnRows, bh_ = blockIdx.x / nblk;
  const int b = bh_ / H, h = bh_ % H;
  const int q0 = (blockIdx.x % nblk) * kAttnRows;
  const bf16* base = qkv + (long long)b * n * ld;
  const bf16* gK = base + (H + h) * kAttnDh;
  const bf16* gV = base + (2 * H + h) * kAttnDh;
  attn_load_rows(sQ, base + h * kAttnDh, ld, q0, kAttnRows, n);
  attn_load_rows(ring, gK, ld, 0, kAttnRows, n);
  attn_load_rows(ring + kAttnTile, gV, ld, 0, kAttnRows, n);
  load_key_flags(sFlag, mask, b, n, 0, kAttnRows);
  cp_async_wait_all();
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = warp * 16;
  const DropCtx dc = drop_ctx<kDropout>(drop, (long long)b * H + h);
  uint32_t qf[4][4];
  load_a_frags(sQ, r0, qf);
  const int row[2] = {q0 + r0 + (lane >> 2), q0 + r0 + (lane >> 2) + 8};
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
  float oacc[8][4];
  zero_acc(oacc);
  for (int i = 0; i < nblk; ++i) {
    const int kb = i * kAttnRows, nxt = (i + 1) & 1;
    const bool more = i + 1 < nblk;
    uint8_t next_flag = 0;
    if (more) {
      attn_load_rows(ring + nxt * 2 * kAttnTile, gK, ld, kb + kAttnRows, kAttnRows, n);
      attn_load_rows(ring + nxt * 2 * kAttnTile + kAttnTile, gV, ld, kb + kAttnRows, kAttnRows, n);
      if (threadIdx.x < kAttnRows) next_flag = key_flag(mask, b, n, kb + kAttnRows + threadIdx.x);
    }
    const uint8_t* cur = ring + (i & 1) * 2 * kAttnTile;
    attn_fwd_block<kCausal, kDropout>(qf, cur, cur + kAttnTile, 0, sFlag + (i & 1) * kAttnRows, kb, row, scale_log2,
                            m, l, oacc, dc);
    if (more && threadIdx.x < kAttnRows) sFlag[nxt * kAttnRows + threadIdx.x] = next_flag;
    cp_async_wait_all();   // block i + 1 landed, and no thread reads stage i & 1 any more
    __syncthreads();
  }
  attn_fwd_finish(oacc, m, l, row, o + (long long)b * n * ldo + h * kAttnDh, ldo, q0 + r0,
                  lse + ((long long)b * H + h) * n, n);
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

// ---- backward -----------------------------------------------------------------------------------
// dK, dV of the 64 keys [k0, k0 + 64) of one (batch, head): loops over all queries.
// resident: the head's whole Q, dO, lse and delta in shared memory
template <bool kCausal, bool kDropout>
__global__ void __launch_bounds__(kAttnThreads)
attn_bwd_dkdv_kernel(const bf16* __restrict__ qkv, long long ld, const uint8_t* __restrict__ mask,
                     const bf16* __restrict__ d_o, long long lddo, const float* __restrict__ lse,
                     const float* __restrict__ delta, bf16* __restrict__ dqkv, long long ldd, int n, int H,
                     float scale, float scale_log2, AttnDrop drop) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int NP = (n + 63) & ~63;
  uint8_t* sK = sm;
  uint8_t* sV = sK + kAttnTile;
  uint8_t* sQ = sV + kAttnTile;
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
  bool empty = false;   // some row of the head has no visible key
  for (int i = threadIdx.x; i < NP; i += kAttnThreads) {
    const float l = i < n ? lse[bh * n + i] : 0.f;
    empty |= l == -FLT_MAX;
    sLse[i] = attn_bwd_lse(l);
    sDelta[i] = i < n ? delta[bh * n + i] : 0.f;
  }
  load_key_flags(sFlag, mask, b, n, k0, kAttnRows);
  cp_async_wait_all();
  const bool any_empty = __syncthreads_or(empty);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = warp * 16;
  const DropCtx dc = drop_ctx<kDropout>(drop, (long long)b * H + h);
  uint32_t kf[4][4], vf[4][4];
  load_a_frags(sK, r0, kf);
  load_a_frags(sV, r0, vf);
  const int kr[2] = {r0 + (lane >> 2), r0 + (lane >> 2) + 8};   // key rows inside the block
  const int key[2] = {k0 + kr[0], k0 + kr[1]};
  const int flag[2] = {sFlag[kr[0]], sFlag[kr[1]]};
  float dk[8][4], dv[8][4];
  zero_acc(dk);
  zero_acc(dv);
  for (int qb = 0; qb < NP; qb += 64)
    attn_dkdv_block<kCausal, kDropout>(kf, vf, sQ, sdO, qb, sLse + qb, sDelta + qb, qb, key, flag, n, scale_log2, dk, dv, dc);
  if (any_empty) {
    if constexpr (kDropout)
      attn_dv_empty_rows_drop(dv, d_o + (long long)b * n * lddo + h * kAttnDh, lddo, lse + bh * n, n, key, dc);
    else
      attn_dv_empty_rows(dv, d_o + (long long)b * n * lddo + h * kAttnDh, lddo, lse + bh * n, n,
                         reinterpret_cast<float*>(sK));
  }
  bf16* out = dqkv + (long long)b * n * ldd;
  store_rows(out + (H + h) * kAttnDh, ldd, k0 + r0, n, dk, scale);
  store_rows(out + (2 * H + h) * kAttnDh, ldd, k0 + r0, n, dv, 1.f);
}

// streaming: the CTA's K, V block stays; Q, dO (cp.async) and the 64 lse / delta values (through a
// register) of query block i + 1 are fetched into the other ring stage while block i is computed
template <bool kCausal, bool kDropout>
__global__ void __launch_bounds__(kAttnThreads)
attn_bwd_dkdv_stream_kernel(const bf16* __restrict__ qkv, long long ld, const uint8_t* __restrict__ mask,
                            const bf16* __restrict__ d_o, long long lddo, const float* __restrict__ lse,
                            const float* __restrict__ delta, bf16* __restrict__ dqkv, long long ldd, int n,
                            int H, float scale, float scale_log2, AttnDrop drop) {
  extern __shared__ __align__(128) uint8_t sm[];
  uint8_t* sK = sm;
  uint8_t* sV = sK + kAttnTile;
  uint8_t* ring = sV + kAttnTile;                            // stage s: Q tile, dO tile at ring + 2 s kAttnTile
  float* sStat = reinterpret_cast<float*>(ring + 4 * kAttnTile);   // stage s: 64 lse, 64 delta at sStat + 128 s
  uint8_t* sFlag = reinterpret_cast<uint8_t*>(sStat + 4 * kAttnRows);
  const int nblk = (n + 63) / kAttnRows, bh_ = blockIdx.x / nblk;
  const int b = bh_ / H, h = bh_ % H;
  const int k0 = (blockIdx.x % nblk) * kAttnRows;
  const bf16* base = qkv + (long long)b * n * ld;
  const bf16* gQ = base + h * kAttnDh;
  const bf16* gdO = d_o + (long long)b * n * lddo + h * kAttnDh;
  const long long bh = (long long)b * H + h;
  // thread t < 64 carries lse of query qb + t, thread 64 + t delta of query qb + t
  const float* gStat = (threadIdx.x < kAttnRows ? lse : delta) + bh * n;
  const int srow = threadIdx.x & (kAttnRows - 1);
  attn_load_rows(sK, base + (H + h) * kAttnDh, ld, k0, kAttnRows, n);
  attn_load_rows(sV, base + (2 * H + h) * kAttnDh, ld, k0, kAttnRows, n);
  attn_load_rows(ring, gQ, ld, 0, kAttnRows, n);
  attn_load_rows(ring + kAttnTile, gdO, lddo, 0, kAttnRows, n);
  const bool is_lse = threadIdx.x < kAttnRows;
  float stat0 = srow < n ? gStat[srow] : 0.f;
  bool empty = is_lse && stat0 == -FLT_MAX;   // some row of the head has no visible key
  sStat[threadIdx.x] = is_lse ? attn_bwd_lse(stat0) : stat0;
  load_key_flags(sFlag, mask, b, n, k0, kAttnRows);
  cp_async_wait_all();
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = warp * 16;
  const DropCtx dc = drop_ctx<kDropout>(drop, (long long)b * H + h);
  uint32_t kf[4][4], vf[4][4];
  load_a_frags(sK, r0, kf);
  load_a_frags(sV, r0, vf);
  const int kr[2] = {r0 + (lane >> 2), r0 + (lane >> 2) + 8};
  const int key[2] = {k0 + kr[0], k0 + kr[1]};
  const int flag[2] = {sFlag[kr[0]], sFlag[kr[1]]};
  float dk[8][4], dv[8][4];
  zero_acc(dk);
  zero_acc(dv);
  for (int i = 0; i < nblk; ++i) {
    const int qb = i * kAttnRows, nxt = (i + 1) & 1;
    const bool more = i + 1 < nblk;
    float next_stat = 0.f;
    if (more) {
      attn_load_rows(ring + nxt * 2 * kAttnTile, gQ, ld, qb + kAttnRows, kAttnRows, n);
      attn_load_rows(ring + nxt * 2 * kAttnTile + kAttnTile, gdO, lddo, qb + kAttnRows, kAttnRows, n);
      const int q = qb + kAttnRows + srow;
      if (q < n) next_stat = gStat[q];
      if (is_lse) {
        empty |= next_stat == -FLT_MAX;
        next_stat = attn_bwd_lse(next_stat);
      }
    }
    const uint8_t* cur = ring + (i & 1) * 2 * kAttnTile;
    const float* st = sStat + (i & 1) * 2 * kAttnRows;
    attn_dkdv_block<kCausal, kDropout>(kf, vf, cur, cur + kAttnTile, 0, st, st + kAttnRows, qb, key, flag, n, scale_log2,
                             dk, dv, dc);
    if (more) sStat[nxt * 2 * kAttnRows + threadIdx.x] = next_stat;
    cp_async_wait_all();   // block i + 1 landed, and no thread reads stage i & 1 any more
    __syncthreads();
  }
  if (__syncthreads_or(empty)) {
    if constexpr (kDropout)
      attn_dv_empty_rows_drop(dv, gdO, lddo, lse + bh * n, n, key, dc);
    else
      attn_dv_empty_rows(dv, gdO, lddo, lse + bh * n, n, reinterpret_cast<float*>(sK));
  }
  bf16* out = dqkv + (long long)b * n * ldd;
  store_rows(out + (H + h) * kAttnDh, ldd, k0 + r0, n, dk, scale);
  store_rows(out + (2 * H + h) * kAttnDh, ldd, k0 + r0, n, dv, 1.f);
}

// dQ of the 64 queries [q0, q0 + 64) of one (batch, head): loops over all keys.
// resident: the head's whole K, V and key flags in shared memory
template <bool kCausal, bool kDropout>
__global__ void __launch_bounds__(kAttnThreads)
attn_bwd_dq_kernel(const bf16* __restrict__ qkv, long long ld, const uint8_t* __restrict__ mask,
                   const bf16* __restrict__ d_o, long long lddo, const float* __restrict__ lse,
                   const float* __restrict__ delta, bf16* __restrict__ dqkv, long long ldd, int n, int H,
                   float scale, float scale_log2, AttnDrop drop) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int NP = (n + 63) & ~63;
  uint8_t* sQ = sm;
  uint8_t* sdO = sQ + kAttnTile;
  uint8_t* sK = sdO + kAttnTile;
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
  const DropCtx dc = drop_ctx<kDropout>(drop, (long long)b * H + h);
  uint32_t qf[4][4], of[4][4];
  load_a_frags(sQ, r0, qf);
  load_a_frags(sdO, r0, of);
  const long long bh = (long long)b * H + h;
  const int row[2] = {q0 + r0 + (lane >> 2), q0 + r0 + (lane >> 2) + 8};
  float lr[2], dr[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    lr[hh] = row[hh] < n ? attn_bwd_lse(lse[bh * n + row[hh]]) : 0.f;
    dr[hh] = row[hh] < n ? delta[bh * n + row[hh]] : 0.f;
  }
  float dq[8][4];
  zero_acc(dq);
  for (int kb = 0; kb < NP; kb += 64)
    attn_dq_block<kCausal, kDropout>(qf, of, sK, sV, kb, sFlag + kb, kb, row, n, lr, dr, scale_log2, dq, dc);
  store_rows(dqkv + (long long)b * n * ldd + h * kAttnDh, ldd, q0 + r0, n, dq, scale);
}

// streaming: the CTA's Q, dO block stays; K, V and key flags of 64-key block i + 1 are fetched into
// the other ring stage while block i is computed
template <bool kCausal, bool kDropout>
__global__ void __launch_bounds__(kAttnThreads)
attn_bwd_dq_stream_kernel(const bf16* __restrict__ qkv, long long ld, const uint8_t* __restrict__ mask,
                          const bf16* __restrict__ d_o, long long lddo, const float* __restrict__ lse,
                          const float* __restrict__ delta, bf16* __restrict__ dqkv, long long ldd, int n,
                          int H, float scale, float scale_log2, AttnDrop drop) {
  extern __shared__ __align__(128) uint8_t sm[];
  uint8_t* sQ = sm;
  uint8_t* sdO = sQ + kAttnTile;
  uint8_t* ring = sdO + kAttnTile;           // stage s: K tile at ring + 2 s kAttnTile, V tile after it
  uint8_t* sFlag = ring + 4 * kAttnTile;     // stage s: 64 key flags at sFlag + 64 s
  const int nblk = (n + 63) / kAttnRows, bh_ = blockIdx.x / nblk;
  const int b = bh_ / H, h = bh_ % H;
  const int q0 = (blockIdx.x % nblk) * kAttnRows;
  const bf16* base = qkv + (long long)b * n * ld;
  const bf16* gK = base + (H + h) * kAttnDh;
  const bf16* gV = base + (2 * H + h) * kAttnDh;
  attn_load_rows(sQ, base + h * kAttnDh, ld, q0, kAttnRows, n);
  attn_load_rows(sdO, d_o + (long long)b * n * lddo + h * kAttnDh, lddo, q0, kAttnRows, n);
  attn_load_rows(ring, gK, ld, 0, kAttnRows, n);
  attn_load_rows(ring + kAttnTile, gV, ld, 0, kAttnRows, n);
  load_key_flags(sFlag, mask, b, n, 0, kAttnRows);
  cp_async_wait_all();
  __syncthreads();

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int r0 = warp * 16;
  const DropCtx dc = drop_ctx<kDropout>(drop, (long long)b * H + h);
  uint32_t qf[4][4], of[4][4];
  load_a_frags(sQ, r0, qf);
  load_a_frags(sdO, r0, of);
  const long long bh = (long long)b * H + h;
  const int row[2] = {q0 + r0 + (lane >> 2), q0 + r0 + (lane >> 2) + 8};
  float lr[2], dr[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    lr[hh] = row[hh] < n ? attn_bwd_lse(lse[bh * n + row[hh]]) : 0.f;
    dr[hh] = row[hh] < n ? delta[bh * n + row[hh]] : 0.f;
  }
  float dq[8][4];
  zero_acc(dq);
  for (int i = 0; i < nblk; ++i) {
    const int kb = i * kAttnRows, nxt = (i + 1) & 1;
    const bool more = i + 1 < nblk;
    uint8_t next_flag = 0;
    if (more) {
      attn_load_rows(ring + nxt * 2 * kAttnTile, gK, ld, kb + kAttnRows, kAttnRows, n);
      attn_load_rows(ring + nxt * 2 * kAttnTile + kAttnTile, gV, ld, kb + kAttnRows, kAttnRows, n);
      if (threadIdx.x < kAttnRows) next_flag = key_flag(mask, b, n, kb + kAttnRows + threadIdx.x);
    }
    const uint8_t* cur = ring + (i & 1) * 2 * kAttnTile;
    attn_dq_block<kCausal, kDropout>(qf, of, cur, cur + kAttnTile, 0, sFlag + (i & 1) * kAttnRows, kb, row, n, lr, dr,
                           scale_log2, dq, dc);
    if (more && threadIdx.x < kAttnRows) sFlag[nxt * kAttnRows + threadIdx.x] = next_flag;
    cp_async_wait_all();   // block i + 1 landed, and no thread reads stage i & 1 any more
    __syncthreads();
  }
  store_rows(dqkv + (long long)b * n * ldd + h * kAttnDh, ldd, q0 + r0, n, dq, scale);
}

}  // namespace xclip

using namespace xclip;

namespace {

// launches of the plain (kDropout = false) and the dropout kernels; the callers have checked `drop`
template <bool kDropout>
int attn_fwd_run(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask, void* o, int64_t ldo, float* lse,
                 int B, int n, int heads, float scale, int causal, AttnDrop drop, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(qkv && o && lse, "attn_fwd: null pointer");
  XCLIP_REQUIRE(B > 0 && heads > 0 && n > 0, "attn_fwd: bad sizes B=%d n=%d heads=%d", B, n, heads);
  XCLIP_REQUIRE(scale > 0.f, "attn_fwd: scale must be positive");
  XCLIP_REQUIRE(ld_qkv % 8 == 0 && ld_qkv >= 3 * heads * kAttnDh, "attn_fwd: bad ld_qkv");
  XCLIP_REQUIRE(ldo % 8 == 0 && ldo >= heads * kAttnDh, "attn_fwd: bad ldo");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(o) & 15) == 0,
                "attn_fwd: misaligned pointer");
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  const int NP = (n + 63) & ~63;
  const bool streaming = n > kAttnResidentMaxN || tune(XCLIP_TUNE_ATTN_STREAM) != 0;
  // resident: Q block + the head's K, V and flags; streaming: Q block + 2 stages of (K, V, 64 flags)
  const int smem = streaming ? 5 * kAttnTile + 2 * kAttnRows : kAttnTile + 2 * NP * 128 + NP;
  const long long blocks = (long long)(NP / kAttnRows) * B * heads;
  XCLIP_REQUIRE(blocks <= 0x7fffffffLL, "attn: B=%d x heads=%d is too large", B, heads);
  const dim3 grid((unsigned)blocks);
  auto kern = streaming ? (causal ? attn_fwd_stream_kernel<true, kDropout> : attn_fwd_stream_kernel<false, kDropout>)
                        : (causal ? attn_fwd_kernel<true, kDropout> : attn_fwd_kernel<false, kDropout>);
  rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), smem);
  if (rc) return rc;
  kern<<<grid, kAttnThreads, smem, s>>>(reinterpret_cast<const bf16*>(qkv), ld_qkv, key_mask,
                                        reinterpret_cast<bf16*>(o), ldo, lse, n, heads,
                                        scale * kLog2e, drop);
  XCLIP_LAUNCH_CHECK(streaming ? "attn_fwd_stream_kernel" : "attn_fwd_kernel");
  return XCLIP_OK;
}

template <bool kDropout>
int attn_bwd_run(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask, const void* o, int64_t ldo,
                 const void* d_o, int64_t lddo, const float* lse, float* delta, void* dqkv, int64_t ld_dqkv, int B,
                 int n, int heads, float scale, int causal, AttnDrop drop, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(qkv && o && d_o && lse && delta && dqkv, "attn_bwd: null pointer");
  XCLIP_REQUIRE(B > 0 && heads > 0 && n > 0, "attn_bwd: bad sizes B=%d n=%d heads=%d", B, n, heads);
  XCLIP_REQUIRE(scale > 0.f, "attn_bwd: scale must be positive");
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
  const bool streaming = n > kAttnResidentMaxN || tune(XCLIP_TUNE_ATTN_STREAM) != 0;
  {
    // resident: K, V block + the head's Q, dO, lse, delta; streaming: K, V block + 2 stages of
    // (Q, dO, 64 lse, 64 delta); both + the block's 64 key flags
    const int smem = streaming ? 6 * kAttnTile + 4 * kAttnRows * 4 + kAttnRows
                               : 2 * kAttnTile + 2 * NP * 128 + 2 * NP * 4 + kAttnRows;
    auto kern = streaming ? (causal ? attn_bwd_dkdv_stream_kernel<true, kDropout>
                                    : attn_bwd_dkdv_stream_kernel<false, kDropout>)
                          : (causal ? attn_bwd_dkdv_kernel<true, kDropout> : attn_bwd_dkdv_kernel<false, kDropout>);
    rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), smem);
    if (rc) return rc;
    kern<<<grid, kAttnThreads, smem, s>>>(q, ld_qkv, key_mask, g, lddo, lse, delta, d, ld_dqkv, n, heads,
                                          scale, sl2, drop);
    XCLIP_LAUNCH_CHECK(streaming ? "attn_bwd_dkdv_stream_kernel" : "attn_bwd_dkdv_kernel");
  }
  {
    // resident: Q, dO block + the head's K, V and flags; streaming: Q, dO block + 2 stages of (K, V, 64 flags)
    const int smem = streaming ? 6 * kAttnTile + 2 * kAttnRows : 2 * kAttnTile + 2 * NP * 128 + NP;
    auto kern = streaming ? (causal ? attn_bwd_dq_stream_kernel<true, kDropout>
                                    : attn_bwd_dq_stream_kernel<false, kDropout>)
                          : (causal ? attn_bwd_dq_kernel<true, kDropout> : attn_bwd_dq_kernel<false, kDropout>);
    rc = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), smem);
    if (rc) return rc;
    kern<<<grid, kAttnThreads, smem, s>>>(q, ld_qkv, key_mask, g, lddo, lse, delta, d, ld_dqkv, n, heads,
                                          scale, sl2, drop);
    XCLIP_LAUNCH_CHECK(streaming ? "attn_bwd_dq_stream_kernel" : "attn_bwd_dq_kernel");
  }
  return XCLIP_OK;
}

// p in [0, 1] -> the kernels' keep threshold and scale; refuses a bad p, seed or layer
int attn_drop_args(const char* what, float p, const uint64_t* seed, int layer, AttnDrop* d) {
  XCLIP_REQUIRE(p >= 0.f && p <= 1.f, "%s: dropout p=%g must lie in [0, 1]", what, (double)p);
  XCLIP_REQUIRE(seed != nullptr && (reinterpret_cast<uintptr_t>(seed) & 7) == 0, "%s: seed must be an aligned "
                "device pointer", what);
  XCLIP_REQUIRE(layer >= 0, "%s: layer must be >= 0", what);
  // keep iff the Philox word < round((1 - p) 2^32); p below 2^-33 keeps every element
  const double thr = nearbyint((1.0 - (double)p) * 4294967296.0);
  d->seed = seed;
  d->keep_le = thr >= 4294967296.0 ? 0xffffffffu : thr >= 1.0 ? (uint32_t)(thr - 1.0) : 0u;
  d->inv_keep = p == 1.f ? 0.f : 1.f / (1.f - p);
  d->layer = (uint32_t)layer;
  return XCLIP_OK;
}

}  // namespace

extern "C" int xclip_attn_fwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask, void* o,
                              int64_t ldo, float* lse, int B, int n, int heads, float scale,
                              int causal, xclip_stream_t stream) {
  return attn_fwd_run<false>(qkv, ld_qkv, key_mask, o, ldo, lse, B, n, heads, scale, causal, AttnDrop{}, stream);
}

extern "C" int xclip_attn_bwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask,
                              const void* o, int64_t ldo, const void* d_o, int64_t lddo,
                              const float* lse, float* delta, void* dqkv, int64_t ld_dqkv,
                              float* dq_workspace, int B, int n, int heads, float scale,
                              int causal, xclip_stream_t stream) {
  (void)dq_workspace;
  return attn_bwd_run<false>(qkv, ld_qkv, key_mask, o, ldo, d_o, lddo, lse, delta, dqkv, ld_dqkv, B, n, heads,
                             scale, causal, AttnDrop{}, stream);
}

extern "C" int xclip_attn_dropout_fwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask, void* o,
                                      int64_t ldo, float* lse, int B, int n, int heads, float scale, int causal,
                                      float p, const uint64_t* seed, int layer, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  AttnDrop d;
  rc = attn_drop_args("attn_dropout_fwd", p, seed, layer, &d);
  if (rc) return rc;
  return attn_fwd_run<true>(qkv, ld_qkv, key_mask, o, ldo, lse, B, n, heads, scale, causal, d, stream);
}

extern "C" int xclip_attn_dropout_bwd(const void* qkv, int64_t ld_qkv, const uint8_t* key_mask,
                                      const void* o, int64_t ldo, const void* d_o, int64_t lddo,
                                      const float* lse, float* delta, void* dqkv, int64_t ld_dqkv, int B, int n,
                                      int heads, float scale, int causal, float p, const uint64_t* seed,
                                      int layer, xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  AttnDrop d;
  rc = attn_drop_args("attn_dropout_bwd", p, seed, layer, &d);
  if (rc) return rc;
  return attn_bwd_run<true>(qkv, ld_qkv, key_mask, o, ldo, d_o, lddo, lse, delta, dqkv, ld_dqkv, B, n, heads,
                            scale, causal, d, stream);
}
