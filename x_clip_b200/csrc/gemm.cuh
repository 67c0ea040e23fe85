// Persistent, warp-specialised wgmma GEMM for sm_90a.
//
//   C[M,N] = alpha * A * B^T (+ bias[N]) (+ residual[M,N])        bf16 x bf16 -> fp32 accum
//
// Operand storage (both cases are fed straight from global memory by TMA, no transposes):
//   a_major = K  : A is [M,K] row-major (K contiguous)          - activations in fwd / dgrad
//   a_major = MN : A is given as At[K,M] row-major (M contiguous)- dY^T in wgrad
//   b_major = K  : B is [N,K] row-major                          - nn.Linear weight [out,in] in fwd
//   b_major = MN : B is given as Bt[K,N] row-major (N contiguous)- weight in dgrad, X in wgrad
//
// This one kernel covers the reference's nn.Linear call sites on the hot path
// (x_clip/x_clip.py:191,195,209,210,358,368,556,570) and their autograd backward, the logits of the
// contrastive loss (NCE / FILIP epilogues), the similarity regularisation (SIMREG epilogues, see
// simreg.cu) and the fused feed-forward (FF epilogues, see ff.cu).
//
// Structure (one CTA per SM, 384 threads), output tile 128 x BLOCK_N:
//   warps 0-3  : consumer warpgroup 0
//   warps 4-7  : consumer warpgroup 1
//   warps 8-11 : producer warpgroup; one elected lane of warp 8 issues the TMA loads.  It drops to
//                40 registers (setmaxnreg) so that the consumers can run with 232: the 128 fp32
//                accumulators of a warpgroup plus the epilogue fit without spilling.
// Pipeline: shared-memory ring full/empty (TMA <-> wgmma), static persistent tile scheduler with
// optional split-K; the producer fills the ring in tile order.  After its k-loop a warpgroup parks
// its accumulator (fp32 registers) in a 128 x 128 staging tile in shared memory; the epilogue then
// gives every thread one row (thread t = row t) and walks the columns, so row reductions (softmax
// partials, segment maxima, LayerNorm sums) stay in registers.  The feed-forward's elementwise UP and
// BWD epilogues skip the staging tile: they work on the accumulator fragments and move their bf16
// activations through a per-warpgroup shared-memory buffer by TMA.  Each warpgroup always computes a
// 128 x 128 block (two m64n128k16 per k16 step); BLOCK_N picks the schedule at compile time:
//   BLOCK_N = 128, ping-pong : each warpgroup owns whole tiles (the k-th tile of the CTA goes to
//       warpgroup k & 1), has its own staging tile and runs its own epilogue, so one warpgroup's
//       epilogue runs while the other's wgmma keeps the tensor cores busy.  A ring stage is read and
//       released by one warpgroup.  The two k-loops take turns through an order barrier.
//   BLOCK_N = 256, cooperative : warpgroup w computes columns [128 w, 128 w + 128) of every tile;
//       both read every ring stage.  Warpgroup 0 runs the epilogue over the whole tile row, the two
//       halves passing through one staging tile one after the other while warpgroup 1 already runs
//       the next tile's k-loop.  Used where an epilogue needs a row's 256 columns in one thread
//       (NCE / SIMREG column blocks, FILIP segments) and by the plain GEMM where it measures faster.
//
// The kernel contains no function call (barrier waits trap without printf): a call anywhere in it
// makes ptxas serialise the wgmma pipeline.
#pragma once

#include "common.cuh"

namespace xclip {

struct GemmParams {
  int M, N, K;
  void* c;
  long long ldc;
  int c_is_f32;        // 0: bf16 out, 1: fp32 out
  int atomic_add;      // fp32 out only: red.add into C (required when split_k > 1)
  int split_k;
  float alpha;
  const float* bias;   // [N] or null
  const bf16* residual;  // bf16 [*, N] or null
  long long ldr;
  int res_row_mod;     // residual row = row % res_row_mod when > 0 (positional tables)
  const int* res_row_idx;  // or residual row = res_row_idx[row] (gathered positional rows), else row
  int raster_m_fast;   // tile order: 0 = N fastest (big A streamed once, B tile L2 resident),
                       //             1 = M fastest (small A resident, big B streamed once)
  // ---- InfoNCE / DCL epilogues (EPI_NCE_FWD, EPI_NCE_BWD); logits s = alpha * acc, alpha = exp(temperature)
  int diag_offset;       // positive of local row r sits in column r + diag_offset
  int dcl;               // decoupled contrastive learning: drop the positive from the denominators
  float* nce_part;       // FWD: [num_n_blocks, M, 2] per block (max of x, sum of 2^(x - max)), x = s*log2(e)
  float* nce_pos;        // FWD: [M] positive logits
  const float* lse_row;  // BWD: [M]  log-denominator of each row (this direction)
  const float* lse_col;  // BWD: [N]  log-denominator of each column (other direction)
  float w_row, w_col, w_diag;
  float* dtemp;          // BWD: scalar accumulator of sum(g * s) or null
  const float* alpha_dev;  // NCE: exp(temperature) read from device memory (no host sync)
  const float* gscale_dev; // BWD: upstream scalar gradient / (2*B_global), multiplies the weights
  const long long* labels; // EPI_VCE_*: [M] column of each row's target (the positive)
  // ---- FILIP segment-max epilogue (EPI_SEGMAX): columns are grouped in segments of seg_len
  // tokens (one segment = one sample of the other modality); the result goes to one packed key
  // per (row, segment) (segmax_key), zeroed before the launch
  int seg_len, n_segs;
  const float* col_mul;    // [N] or null: per-column multiplier (0 for masked text tokens)
  const float* col_add;    // [N] or null: per-column addend (-FLT_MAX for masked text tokens)
  unsigned long long* seg_keys;  // [M, n_segs]
  // ---- fused feed-forward epilogues (EPI_FF_*)
  float* ff_rowsum;        // [M, 4d/64, 2] per-box (sum, sum of squares) of the GEGLU output rows: UP writes, DOWN sums
  const float* ff_colvec;  // DOWN: c[N] = row sums of the gain-scaled down-projection weight
  float* ff_stats;         // DOWN: [M,2] (mean, rstd) of the GEGLU output rows, written for the backward
  float ff_eps;            // LayerNorm epsilon
  float ff_inv_hidden;     // DOWN: 1 / ff_hidden, divided on the host (a device division is a call)
  int ff_hidden;           // 4*dim: LayerNorm width; column offset of the gate half inside u
  int ff_skip_u;           // UP: do not write u = [value | gate] (inference / no-grad sweeps need only hp)
  bf16* ff_out2;           // DOWN: bf16(acc) [M, d]
  long long ff_ld2;
  const float* ff_ab;      // BWD: [M,2] per-row (mean_k(gdh), mean_k(gdh * hn)) from xclip_ff_bwd_prep
};

constexpr int EPI_STORE = 0;    // C = alpha*acc (+bias) (+residual)
constexpr int EPI_NCE_FWD = 1;  // row partial sums of exp(s - alpha) and the positives
constexpr int EPI_NCE_BWD = 2;  // C = g = w_row*exp(s-lse_row) + w_col*exp(s-lse_col) - w_diag*[diag]
// FILIP: per row and column segment of seg_len >= 1 columns, max and argmax of alpha*acc
// (BLOCK_N = 256).  A segment may start or end anywhere in a tile, and may span several tiles.
// Each (row, segment) result is one 64-bit key (segmax_key); a segment wholly inside the tile
// stores it, a piece cut by a tile edge merges it with atom.max.  filip.cu unpacks the keys.
constexpr int EPI_SEGMAX = 3;
// Fused feed-forward (x_clip/x_clip.py:180-199), BLOCK_N = 128:
//   EPI_FF_UP   B is the up-projection weight with its rows permuted so that a tile holds the value
//               columns [64 t, 64 t + 64) and the MATCHING gate columns; writes u = [value | gate]
//               (reference layout, needed by the backward), hp = value * gelu(gate) (bf16) and the
//               per-row (sum, sum^2) of bf16(hp) over the tile's 64 hidden units.
//   EPI_FF_DOWN down-projection with the LayerNorm folded in (:193-195):
//               x2 = LN(hp) g W2^T + x1 = rstd_r (acc_rj - mean_r c_j) + x1_rj  with
//               acc = hp (W2 . g)^T and c_j = sum_k (W2 . g)_jk; also writes bf16(acc) and
//               (mean, rstd) for the backward.
//   EPI_FF_BWD  backward of LayerNorm(4d) + GEGLU fused into the down-projection's dgrad GEMM
//               gdh = dx (W2 . g): per element
//                 hn = (value*gelu(gate) - mean) rstd;  dhp = rstd (gdh - a_r - hn b_r)
//                 d value = dhp gelu(gate);  d gate = dhp value gelu'(gate)
//               with the two row means a_r = mean_k gdh, b_r = mean_k gdh*hn supplied by
//               xclip_ff_bwd_prep.  Reads u = [value | gate], writes du.
// UP and BWD work on the accumulator fragments in registers and move their bf16 activations
// through a per-warpgroup activation buffer in place of the fp32 staging tile (see GemmSmem).
constexpr int EPI_FF_UP = 4;
constexpr int EPI_FF_DOWN = 5;
constexpr int EPI_FF_BWD = 6;
// Similarity regularisation (simreg.cu): acc = E = T T^T - V V^T, formed inside the accumulator by
// contracting [T | V] against [T | -V] (K = 2 x the split-bf16 width).  The positive column
// r + diag_offset and the columns >= N are excluded.
//   EPI_SIMREG_FWD  nce_part[n_blk * M + row] = sum over the tile's columns of E^2
//   EPI_SIMREG_BWD  C = bf16(*gscale_dev * E), zero on the excluded columns up to ldc
constexpr int EPI_SIMREG_FWD = 7;
constexpr int EPI_SIMREG_BWD = 8;
// Vocabulary cross-entropy (nce.cu): logits l = acc + bias[c] over the N = V columns, the target
// of row r is column labels[r]; columns >= N are masked here, so any V >= 1 works.
//   EPI_VCE_FWD  nce_part[n_blk * M + row] = (max, sum of 2^(x - max)) over the block, x = l log2(e);
//                nce_pos[row] = l[row, labels[row]]
//   EPI_VCE_BWD  C = bf16(*gscale_dev * (exp(l - lse_row[row]) - [c == labels[row]])), zero in [N, ldc)
constexpr int EPI_VCE_FWD = 9;
constexpr int EPI_VCE_BWD = 10;

constexpr int kGemmBlockM = 128;
constexpr int kGemmBlockK = 64;
constexpr int kGemmConsumerThreads = 256;
constexpr int kGemmThreads = kGemmConsumerThreads + 128;
// 128 * (40 + 2 * 232) = 64,512 of the 65,536 registers of an SM
constexpr int kGemmProducerRegs = 40;
constexpr int kGemmConsumerRegs = 232;
// named barriers: 2 = staging tile (cooperative), 2 + wg = staging tile of warpgroup wg and
// 4 + wg = "warpgroup wg may start its k-loop" (ping-pong)
constexpr int kBarStage = 2;
constexpr int kBarOrder = 4;

// Layout: ring stages | staging tiles | mbarriers.  For EPI_FF_UP / EPI_FF_BWD each warpgroup's
// staging tile is instead a bf16 activation buffer of the same 64 KiB: four 128-row x 64-column
// boxes in the 128-byte swizzle of their TMA maps (BWD: u value [128 n, +128), u gate, rewritten in
// place as du; UP: u value, u gate, hp).  Their mbarriers act_full / act_empty[wg] follow the ring's;
// only BWD, whose producer fills the buffer, waits on them (UP's store issuer waits for its own bulk
// stores to have read the buffer before the warpgroup rewrites it).
template <int BLOCK_N, int EPI = EPI_STORE>
struct GemmSmem {
  static constexpr bool kPingPong = BLOCK_N == 128;
  static constexpr bool kActTile = EPI == EPI_FF_UP || EPI == EPI_FF_BWD;
  static constexpr int kABytes = kGemmBlockM * kGemmBlockK * 2;  // 16 KiB
  static constexpr int kBBytes = BLOCK_N * kGemmBlockK * 2;      // 16/32 KiB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = 3;
  static constexpr int kAccBytes = kGemmBlockM * 128 * 4;        // fp32 staging tile, 128 columns
  static constexpr int kActBoxBytes = kGemmBlockM * 64 * 2;      // one 128 x 64 bf16 box
  static_assert(4 * kActBoxBytes == kAccBytes, "an activation buffer replaces a staging tile");
  static_assert(!kActTile || kPingPong, "activation buffers are per ping-pong warpgroup");
  static constexpr int kAccTiles = kPingPong ? 2 : 1;            // one per warpgroup in ping-pong
  static constexpr int kBarrierBytes = 256;
  static constexpr int kTotal = kStages * kStageBytes + kAccTiles * kAccBytes + kBarrierBytes;
  static_assert(kTotal <= 232448, "over the 227 KiB of shared memory a CTA can opt in to");
};

__device__ __forceinline__ float nce_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// Staging tile: 128 rows of 128 fp32, unpadded.  The 16-byte chunk q of row r is stored at chunk
// q ^ acc_swz(r).  The epilogue's row reads (a quarter-warp reads one chunk of 8 consecutive rows)
// and the accumulator fragment writes (a half-warp writes two adjacent chunks of 4 consecutive rows)
// both hit 8 distinct 16-byte bank groups.
__device__ __forceinline__ int acc_swz(int r) { return ((r & 3) << 1) | ((r >> 2) & 1); }

// 32 consecutive fp32 accumulator columns [col, col + 32) of this thread's row from the staging
// tile; `sw` = acc_swz(row)
__device__ __forceinline__ void acc_ld32(const float* row, int sw, int col, float (&f)[32]) {
  const float4* src = reinterpret_cast<const float4*>(row);
  const int q0 = (col & 127) >> 2;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = src[(q0 + i) ^ sw];
    f[4 * i] = v.x; f[4 * i + 1] = v.y; f[4 * i + 2] = v.z; f[4 * i + 3] = v.w;
  }
}
__device__ __forceinline__ void acc_ld16(const float* row, int sw, int col, float (&f)[16]) {
  const float4* src = reinterpret_cast<const float4*>(row);
  const int q0 = (col & 127) >> 2;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 v = src[(q0 + i) ^ sw];
    f[4 * i] = v.x; f[4 * i + 1] = v.y; f[4 * i + 2] = v.z; f[4 * i + 3] = v.w;
  }
}

__device__ __forceinline__ void st_bf16x8(bf16* dst, const float* f) {
  uint4 o;
  o.x = pack_bf16x2(f[0], f[1]);
  o.y = pack_bf16x2(f[2], f[3]);
  o.z = pack_bf16x2(f[4], f[5]);
  o.w = pack_bf16x2(f[6], f[7]);
  *reinterpret_cast<uint4*>(dst) = o;
}
__device__ __forceinline__ float bf16_rn(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

// (value, index) of a segment maximum as one unsigned 64-bit key whose integer order is the order
// of the results: high word = the order-preserving image of the fp32 value (negative values
// bit-inverted, positive ones with the sign bit set), low word = 0xFFFFFFFF - index, so that on
// equal values the lower index is the larger key.  Every key, -FLT_MAX and -inf included, is > 0.
__device__ __forceinline__ unsigned long long segmax_key(float v, int idx) {
  const uint32_t b = __float_as_uint(v);
  const uint32_t o = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  return (static_cast<unsigned long long>(o) << 32) | (0xFFFFFFFFu - static_cast<uint32_t>(idx));
}
__device__ __forceinline__ float segmax_key_value(unsigned long long k) {
  const uint32_t o = static_cast<uint32_t>(k >> 32);
  return __uint_as_float((o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o);
}
__device__ __forceinline__ int segmax_key_index(unsigned long long k) {
  return static_cast<int>(0xFFFFFFFFu - static_cast<uint32_t>(k));
}

// EPI_VCE_*: v[i] += bias[col0 + i] over the columns < N (bias 16-byte aligned, or null)
__device__ __forceinline__ void vce_add_bias(const GemmParams& p, int col0, float (&v)[32]) {
  if (p.bias == nullptr) return;
  if (col0 + 32 <= p.N) {
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      const float4 b4 = __ldg(reinterpret_cast<const float4*>(p.bias + col0 + i));
      v[i] += b4.x; v[i + 1] += b4.y; v[i + 2] += b4.z; v[i + 3] += b4.w;
    }
  } else {
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (col0 + i < p.N) v[i] += __ldg(p.bias + col0 + i);
  }
}

// Epilogue of one 128 x BLOCK_N tile for EPI_STORE; `stage(c)` makes column c of the tile readable.
template <int BLOCK_N, class Stage>
__device__ __forceinline__ void gemm_epilogue_store(const GemmParams& p, const float* acc_row, int acc_sw,
                                                    int row, int n_blk, int split, Stage&& stage) {
  const bool row_ok = row < p.M;
  const bf16* res_row = nullptr;
  if (p.residual != nullptr && row_ok && split == 0) {
    const long long rr = p.res_row_idx ? p.res_row_idx[row] : (p.res_row_mod > 0 ? (row % p.res_row_mod) : row);
    res_row = p.residual + rr * p.ldr;
  }
  // the residual of chunk c + 1 is loaded before chunk c is processed: one DRAM round trip in
  // flight behind the math instead of one per chunk
  uint4 res_next[4] = {};
  auto load_res = [&](int c) {
    const int col0 = n_blk * BLOCK_N + c * 32;
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (col0 + 8 * i < p.N) res_next[i] = *reinterpret_cast<const uint4*>(res_row + col0 + 8 * i);
  };
  if (res_row != nullptr) load_res(0);
#pragma unroll 1
  for (int c = 0; c < BLOCK_N / 32; ++c) {
    stage(c * 32);
    const int col0 = n_blk * BLOCK_N + c * 32;
    if (!row_ok || col0 >= p.N) continue;
    uint4 res_cur[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) res_cur[i] = res_next[i];
    if (res_row != nullptr && c + 1 < BLOCK_N / 32 && col0 + 32 < p.N) load_res(c + 1);
    float f[32];
    acc_ld32(acc_row, acc_sw, c * 32, f);
#pragma unroll
    for (int i = 0; i < 32; ++i) f[i] *= p.alpha;
    if (p.bias != nullptr && split == 0) {
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        if (col0 + i < p.N) {
          const float4 b4 = *reinterpret_cast<const float4*>(p.bias + col0 + i);
          f[i] += b4.x; f[i + 1] += b4.y; f[i + 2] += b4.z; f[i + 3] += b4.w;
        }
      }
    }
    if (res_row != nullptr) {
#pragma unroll
      for (int i = 0; i < 32; i += 8) {
        if (col0 + i < p.N) {
          const uint4 r4 = res_cur[i / 8];
          float2 a = unpack_bf16x2(r4.x), b = unpack_bf16x2(r4.y);
          float2 cc = unpack_bf16x2(r4.z), d = unpack_bf16x2(r4.w);
          f[i] += a.x; f[i + 1] += a.y; f[i + 2] += b.x; f[i + 3] += b.y;
          f[i + 4] += cc.x; f[i + 5] += cc.y; f[i + 6] += d.x; f[i + 7] += d.y;
        }
      }
    }
    if (p.c_is_f32) {
      float* crow = reinterpret_cast<float*>(p.c) + static_cast<long long>(row) * p.ldc + col0;
      if (p.atomic_add) {
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          if (col0 + i < p.N) {
            asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(crow + i),
                         "f"(f[i]), "f"(f[i + 1]), "f"(f[i + 2]), "f"(f[i + 3])
                         : "memory");
          }
        }
      } else {
#pragma unroll
        for (int i = 0; i < 32; i += 4) {
          if (col0 + i < p.N)
            *reinterpret_cast<float4*>(crow + i) = make_float4(f[i], f[i + 1], f[i + 2], f[i + 3]);
        }
      }
    } else {
      bf16* crow = reinterpret_cast<bf16*>(p.c) + static_cast<long long>(row) * p.ldc + col0;
#pragma unroll
      for (int i = 0; i < 32; i += 8) {
        if (col0 + i < p.N) st_bf16x8(crow + i, f + i);
      }
    }
  }
}

// ---- fused feed-forward epilogues on the accumulator fragments (ping-pong, one warpgroup) ----
// Thread wt = 32 w + l of the warpgroup holds acc[h][j] at row 64 h + 16 w + l / 4 + 8 ((j / 2) % 2),
// column 8 (j / 4) + 2 (l % 4) + j % 2.  A column pair is one 32-bit word of a 128 x 64 bf16
// activation box; every fragment row of the thread has swizzle phase l / 4, so a warp's word
// accesses hit 32 distinct banks.  ff_frag_off(h, j) = byte offset of acc[h][j]'s pair in its box
// (column j / 4 mod 8 chunk); `frag` = (16 w + l / 4) * 128 + (l % 4) * 4, `sw` = l / 4.
__device__ __forceinline__ uint32_t ff_frag_off(uint32_t frag, uint32_t sw, int h, int j) {
  return frag + (h * 64 + 8 * ((j >> 1) & 1)) * 128 + ((((j >> 2) & 7) ^ sw) << 4);
}

// EPI_FF_UP.  Tile columns [0, 64) are the value and [64, 128) the gate columns of hidden units
// [64 n_blk, +64): value column c and gate column 64 + c sit in the same thread (acc[h][j] and
// acc[h][j + 32]).  Boxes: 0 = u value, 1 = u gate, 2 = hp; stored by TMA, rows >= M clipped.
// `issuer` is the warpgroup's one thread that issues (and later waits on) the bulk stores.
__device__ __forceinline__ void ff_up_epilogue(const GemmParams& p, const CUtensorMap* tm_u, const CUtensorMap* tm_out,
                                               const float (&acc)[2][64], uint8_t* act, int wg, int wt, int m_blk,
                                               int n_blk, bool issuer) {
  constexpr int kBox = kGemmBlockM * 64 * 2;
  const int lane = wt & 31;
  const uint32_t frag = (uint32_t)((wt >> 5) * 16 + (lane >> 2)) * 128u + (lane & 3) * 4u;
  const uint32_t sw = lane >> 2;
  uint8_t* box_v = act;
  uint8_t* box_g = act + kBox;
  uint8_t* box_h = act + 2 * kBox;
  // the previous tile's stores have read the buffer, and its rowsum reads are done
  if (issuer) bulk_wait_group_read<0>();
  named_bar_sync(kBarStage + wg, 128);
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int j = 0; j < 32; j += 2) {
      const uint32_t off = ff_frag_off(frag, sw, h, j);
      const float v0 = acc[h][j], v1 = acc[h][j + 1], g0 = acc[h][j + 32], g1 = acc[h][j + 33];
      const GeluParts2 gp = gelu_parts2(g0, g1);
      const f32x2 ge = f2_mul(f2_pack(g0, g1), gp.cdf);                                     // gelu(gate)
      *reinterpret_cast<uint32_t*>(box_h + off) = f2_to_bf16x2(f2_mul(f2_pack(v0, v1), ge));  // hp
      if (!p.ff_skip_u) {
        *reinterpret_cast<uint32_t*>(box_v + off) = pack_bf16x2(v0, v1);
        *reinterpret_cast<uint32_t*>(box_g + off) = pack_bf16x2(g0, g1);
      }
    }
  fence_proxy_async_smem();
  named_bar_sync(kBarStage + wg, 128);
  const int m0 = m_blk * kGemmBlockM, hcol = n_blk * 64;
  if (issuer) {
    if (!p.ff_skip_u) {
      tma_store_2d(tm_u, box_v, hcol, m0);
      tma_store_2d(tm_u, box_g, p.ff_hidden + hcol, m0);
    }
    tma_store_2d(tm_out, box_h, hcol, m0);
    bulk_commit_group();
  }
  // Per-row (sum, sum^2) of the bf16 hp the next GEMM reads: thread wt re-reads row wt and sums it in
  // column order in two lanes (even / odd columns).  One slot per row and 64-column box, summed in a
  // fixed order by the down-projection: the statistics (and the loss) are bit-reproducible.
  f32x2 s1p = f2_splat(0.f), s2p = f2_splat(0.f);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const uint4 w4 = *reinterpret_cast<const uint4*>(box_h + swz128(wt, q));
    const uint32_t w[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const f32x2 hr = f2_from_bf16x2(w[k]);
      s1p = f2_add(s1p, hr);
      s2p = f2_fma(hr, hr, s2p);
    }
  }
  const int row = m0 + wt;
  if (row < p.M) {
    const int nparts = p.ff_hidden >> 6;                     // 4d / 64 boxes per row
    *reinterpret_cast<float2*>(p.ff_rowsum + 2ll * ((long long)row * nparts + n_blk)) =
        make_float2(s1p.x + s1p.y, s2p.x + s2p.y);
  }
}

// EPI_FF_BWD: (mean, rstd, a, b) of row r, zeros past M
__device__ __forceinline__ float4 ff_row_stats(const GemmParams& p, int r) {
  float2 st = make_float2(0.f, 0.f), ab = make_float2(0.f, 0.f);
  if (r < p.M) {
    st = *reinterpret_cast<const float2*>(p.ff_stats + 2ll * r);
    ab = *reinterpret_cast<const float2*>(p.ff_ab + 2ll * r);
  }
  return make_float4(st.x, st.y, ab.x, ab.y);
}

// EPI_FF_BWD.  Tile columns = hidden units [128 n_blk, +128).  The producer has loaded u into boxes
// 0, 1 (value) and 2, 3 (gate) and signalled act_full; du overwrites them in place and leaves by
// TMA; act_empty hands the buffer back once the stores have read it.  The thread's four fragment
// rows row0 + 64 h + 8 i (global row indices) are done one after the other, so that only one row's
// statistics are in use and one more in flight: the 128 accumulators leave no room for more.
// `rs` = ff_row_stats of row0, loaded by the caller.
__device__ __forceinline__ void ff_bwd_epilogue(const GemmParams& p, const CUtensorMap* tm_out, const float (&acc)[2][64],
                                                float4 rs, int row0, uint8_t* act, uint64_t* act_empty, int wg,
                                                int wt, int m_blk, int n_blk, bool issuer) {
  constexpr int kBox = kGemmBlockM * 64 * 2;
  const int lane = wt & 31;
  const uint32_t frag = (uint32_t)((wt >> 5) * 16 + (lane >> 2)) * 128u + (lane & 3) * 4u;
  const uint32_t sw = lane >> 2;
  float4 st = rs;
#pragma unroll
  for (int hi = 0; hi < 4; ++hi) {                          // row 64 h + 8 i of the fragment, hi = 2 h + i
    const int h = hi >> 1;
    float4 st_next = st;
    if (hi < 3) st_next = ff_row_stats(p, row0 + 64 * ((hi + 1) >> 1) + 8 * ((hi + 1) & 1));
#pragma unroll
    for (int q = 0; q < 16; ++q) {                          // columns 8 q + 2 (l % 4) + {0, 1}
      const int j = 4 * q + 2 * (hi & 1);
      const f32x2 rstd2 = f2_splat(st.y), nmr = f2_splat(-st.x * st.y), namr = f2_splat(-st.z * st.y),
                  nbmr = f2_splat(-st.w * st.y);
      uint32_t* pv = reinterpret_cast<uint32_t*>(act + (j >> 5) * kBox + ff_frag_off(frag, sw, h, j));
      uint32_t* pg = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(pv) + 2 * kBox);
      const uint32_t wv = *pv, wgt = *pg;
      const float g0 = __uint_as_float(wgt << 16), g1 = __uint_as_float(wgt & 0xffff0000u);
      const f32x2 gate = f2_pack(g0, g1), val = f2_from_bf16x2(wv);
      const GeluParts2 gp = gelu_parts2(g0, g1);
      const f32x2 ge = f2_mul(gate, gp.cdf);                // gelu(gate)
      const f32x2 gd = f2_fma(gate, gp.pdf, gp.cdf);        // gelu'(gate)
      const f32x2 hn = f2_fma(f2_mul(val, ge), rstd2, nmr); // (val*ge - mean) rstd
      f32x2 dhp = f2_fma(f2_pack(acc[h][j], acc[h][j + 1]), rstd2, namr);   // rstd (gdh - a)
      dhp = f2_fma(hn, nbmr, dhp);                          //   - rstd b hn
      *pv = f2_to_bf16x2(f2_mul(dhp, ge));
      *pg = f2_to_bf16x2(f2_mul(f2_mul(dhp, val), gd));
    }
    st = st_next;
  }
  fence_proxy_async_smem();
  named_bar_sync(kBarStage + wg, 128);
  if (issuer) {
    const int m0 = m_blk * kGemmBlockM, col = n_blk * 128;
#pragma unroll
    for (int b = 0; b < 4; ++b)
      tma_store_2d(tm_out, act + b * kBox, (b >> 1) * p.ff_hidden + col + (b & 1) * 64, m0);
    bulk_commit_group();
    bulk_wait_group_read<0>();
    mbar_arrive(act_empty);
  }
}

// tmU / tmOut: 128-row x 64-column box maps of EPI_FF_UP (u [M, 8d] unless ff_skip_u, hp [M, 4d];
// stores) and EPI_FF_BWD (u [M, 8d] loaded, du [M, 8d] stored).  Every other epilogue ignores them
// (launch with empty maps); they follow p so that its parameter offsets do not depend on them.
template <int BLOCK_N, int A_MAJOR, int B_MAJOR, int EPI = EPI_STORE>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p, const __grid_constant__ CUtensorMap tmU,
                 const __grid_constant__ CUtensorMap tmOut) {
  using S = GemmSmem<BLOCK_N, EPI>;
  constexpr int kStages = S::kStages;
  constexpr bool kPingPong = S::kPingPong;
  constexpr int kPasses = kPingPong ? 1 : 2;   // trips of a tile through its 128-column staging tile
  static_assert(BLOCK_N == 128 || BLOCK_N == 256, "BLOCK_N must be 128 or 256");

  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * S::kABytes;
  float* acc_smem = reinterpret_cast<float*>(smem + kStages * S::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * S::kStageBytes + S::kAccTiles * S::kAccBytes);
  uint64_t* full_bar = bars;                    // [kStages]
  uint64_t* empty_bar = bars + kStages;         // [kStages]
  uint64_t* act_full = bars + 2 * kStages;      // [2] activation buffers (S::kActTile)
  uint64_t* act_empty = act_full + 2;           // [2]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int num_m = (p.M + kGemmBlockM - 1) / kGemmBlockM;
  const int num_n = (p.N + BLOCK_N - 1) / BLOCK_N;
  const int num_kb = (p.K + kGemmBlockK - 1) / kGemmBlockK;
  const int splits = p.split_k > 0 ? p.split_k : 1;
  const int kb_per_split = (num_kb + splits - 1) / splits;
  const int num_tiles = num_m * num_n * splits;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();   // the 128-byte swizzle needs 1024-byte aligned tiles
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      // released by every warp that reads the stage: one warpgroup (ping-pong) or both
      mbar_init(&empty_bar[i], (kPingPong ? 128 : kGemmConsumerThreads) / 32);
    }
    if constexpr (S::kActTile) {
      for (int i = 0; i < 2; ++i) {
        mbar_init(&act_full[i], 1);    // the producer's expect_tx
        mbar_init(&act_empty[i], 1);   // the warpgroup's store issuer
      }
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= kGemmConsumerThreads / 32) {
    // ===================== TMA producer =====================
    setmaxnreg_dec<kGemmProducerRegs>();
    if (warp == kGemmConsumerThreads / 32 && XCLIP_ONE_LANE(lane)) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      int stage = 0;
      uint32_t phase = 0;
      int it = 0;                              // index of the tile among this CTA's tiles
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++it) {
        const int tmn = t % (num_n * num_m);
        const int n_blk = p.raster_m_fast ? tmn / num_m : tmn % num_n;
        const int m_blk = p.raster_m_fast ? tmn % num_m : tmn / num_n;
        const int split = t / (num_n * num_m);
        const int kb0 = split * kb_per_split;
        const int kb1 = min(kb0 + kb_per_split, num_kb);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait_nocall(&empty_bar[stage], phase ^ 1);
          mbar_arrive_expect_tx(&full_bar[stage], S::kStageBytes);
          uint8_t* sa = smem_a + stage * S::kABytes;
          uint8_t* sb = smem_b + stage * S::kBBytes;
          if (A_MAJOR == kMajorK) {
            tma_load_2d(sa, &tmA, &full_bar[stage], kb * kGemmBlockK, m_blk * kGemmBlockM);
          } else {
#pragma unroll
            for (int g = 0; g < kGemmBlockM / 64; ++g)
              tma_load_2d(sa + g * (kGemmBlockK * 128), &tmA, &full_bar[stage],
                          m_blk * kGemmBlockM + g * 64, kb * kGemmBlockK);
          }
          if (B_MAJOR == kMajorK) {
            tma_load_2d(sb, &tmB, &full_bar[stage], kb * kGemmBlockK, n_blk * BLOCK_N);
          } else {
#pragma unroll
            for (int g = 0; g < BLOCK_N / 64; ++g)
              tma_load_2d(sb + g * (kGemmBlockK * 128), &tmB, &full_bar[stage],
                          n_blk * BLOCK_N + g * 64, kb * kGemmBlockK);
          }
          if constexpr (EPI == EPI_FF_BWD) {
            // the tile's u (value and gate columns of hidden units [128 n_blk, +128)) lands in its
            // warpgroup's activation buffer during the k-loop, once the buffer's last stores have read it
            if (kb == kb0) {
              const int w = it & 1;
              mbar_wait_nocall(&act_empty[w], ((it >> 1) & 1) ^ 1);
              mbar_arrive_expect_tx(&act_full[w], S::kAccBytes);
              uint8_t* act = smem + kStages * S::kStageBytes + w * S::kAccBytes;
#pragma unroll
              for (int b = 0; b < 4; ++b)
                tma_load_2d(act + b * S::kActBoxBytes, &tmU, &act_full[w],
                            (b >> 1) * p.ff_hidden + n_blk * BLOCK_N + (b & 1) * 64, m_blk * kGemmBlockM);
            }
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers (warpgroups 0 and 1) =====================
  setmaxnreg_inc<kGemmConsumerRegs>();
  const int wg = threadIdx.x >> 7;
  const int wt = threadIdx.x & 127;            // thread inside the warpgroup
  // K-major: SBO = 1024 (8 rows x 128 B), LBO unused.  MN-major: SBO = 1024 between 8-row K groups,
  // LBO = BLOCK_K*128 between 64-wide M/N groups (one TMA box each).
  constexpr uint32_t kLboMN = kGemmBlockK * 128;
  constexpr uint32_t kAStep = (A_MAJOR == kMajorK) ? 32u : 2048u;  // bytes per k16
  constexpr uint32_t kBStep = (B_MAJOR == kMajorK) ? 32u : 2048u;
  // the warpgroup's 128 columns of the B tile (cooperative: half wg) and the second m64 half of A
  const uint32_t b_off = kPingPong ? 0u : (B_MAJOR == kMajorK) ? wg * 128 * 128 : wg * 2 * kLboMN;
  constexpr uint32_t kAHalf = (A_MAJOR == kMajorK) ? 64 * 128 : kLboMN;
  float* acc_tile = acc_smem + (kPingPong ? wg * (S::kAccBytes / 4) : 0);
  const float* acc_row = acc_tile + wt * 128;  // epilogue: this thread's row of the staging tile
  const int acc_sw = acc_swz(wt);
  const int frag_sw = acc_swz(lane >> 2);      // every fragment row of this thread is lane / 4 mod 8

  int stage = 0;
  uint32_t phase = 0;
  int it = 0;                                  // index of the tile among this CTA's tiles
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x, ++it) {
    const int tmn = t % (num_n * num_m);
    const int n_blk = p.raster_m_fast ? tmn / num_m : tmn % num_n;
    const int m_blk = p.raster_m_fast ? tmn % num_m : tmn / num_n;
    const int split = t / (num_n * num_m);
    const int kb0 = split * kb_per_split;
    const int kb1 = min(kb0 + kb_per_split, num_kb);
    if (kPingPong && (it & 1) != wg) {         // the other warpgroup's tile: skip its ring slots
      stage += kb1 - kb0;
      phase ^= (stage / kStages) & 1;
      stage %= kStages;
      continue;
    }
    // Ping-pong: start the k-loop only once the other warpgroup has issued its previous tile's.
    // Besides keeping the MMAs of the two warpgroups from interleaving, this is what keeps the
    // parity waits sound: every slot before this tile's has then been filled, so no full barrier
    // is two phases behind the one waited for (a parity wait cannot tell those apart).
    if (kPingPong && it > 0) named_bar_sync(kBarOrder + wg, kGemmConsumerThreads);
    int prev_stage = -1;               // stage read by the wgmma group still in flight

    float acc[2][64];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < 64; ++j) acc[h][j] = 0.f;

    for (int kb = kb0; kb < kb1; ++kb) {
      mbar_wait_nocall(&full_bar[stage], phase);
      const uint64_t adesc = make_smem_desc(smem_u32(smem_a + stage * S::kABytes),
                                            A_MAJOR == kMajorK ? 0u : kLboMN, 1024u);
      const uint64_t bdesc = make_smem_desc(smem_u32(smem_b + stage * S::kBBytes) + b_off,
                                            B_MAJOR == kMajorK ? 0u : kLboMN, 1024u);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kGemmBlockK / 16; ++k) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const uint64_t da = desc_advance(adesc, h * kAHalf + k * kAStep);
          const uint64_t db = desc_advance(bdesc, k * kBStep);
          wgmma_m64n128k16<A_MAJOR, B_MAJOR>(acc[h], da, db);
        }
      }
      wgmma_commit();
      // keep this k-block's MMAs in flight while the next one is issued: only the previous group must
      // have retired before its stage goes back to the producer
      wgmma_wait<1>();
      __syncwarp();
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
      prev_stage = stage;
      if (++stage == kStages) { stage = 0; phase ^= 1; }
    }
    // EPI_FF_BWD: (mean, rstd, a, b) of the thread's first fragment row, loaded while the last wgmma
    // group runs
    const int ff_row0 = m_blk * kGemmBlockM + (wt >> 5) * 16 + (lane >> 2);
    float4 ff_rs;
    if constexpr (EPI == EPI_FF_BWD) ff_rs = ff_row_stats(p, ff_row0);
    if (kPingPong && t + (int)gridDim.x < num_tiles)
      named_bar_arrive(kBarOrder + (wg ^ 1), kGemmConsumerThreads);
    wgmma_wait<0>();
    __syncwarp();
    if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

    if constexpr (S::kActTile) {
      uint8_t* act = smem + kStages * S::kStageBytes + wg * S::kAccBytes;
      const bool issuer = wt < 32 && XCLIP_ONE_LANE(lane);
      if constexpr (EPI == EPI_FF_UP) {
        ff_up_epilogue(p, &tmU, &tmOut, acc, act, wg, wt, m_blk, n_blk, issuer);
      } else {
        mbar_wait_nocall(&act_full[wg], (it >> 1) & 1);
        ff_bwd_epilogue(p, &tmOut, acc, ff_rs, ff_row0, act, &act_empty[wg], wg, wt, m_blk, n_blk, issuer);
      }
      continue;
    }

    // ---- accumulator -> staging tile (the warpgroup's 128 columns).  Ping-pong: one pass into the
    // warpgroup's own tile.  Cooperative: pass q holds tile columns [128 q, 128 q + 128), written by
    // warpgroup q.
    auto write_acc = [&]() {
      const int w = wt >> 5;
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int j = 0; j < 64; j += 2) {
          const int r = h * 64 + w * 16 + (lane >> 2) + 8 * ((j >> 1) & 1);
          const int q = (j >> 2) * 2 + ((lane & 3) >> 1);        // 16-byte chunk of column 8 (j/4) + 2 (lane%4)
          *reinterpret_cast<float2*>(acc_tile + r * 128 + ((q ^ frag_sw) << 2) + (lane & 1) * 2) =
              make_float2(acc[h][j], acc[h][j + 1]);
        }
    };
    int staged = 0;
    auto stage_pass = [&](bool write) {
      named_bar_sync(kBarStage, kGemmConsumerThreads);    // the previous pass has been read
      if (write) write_acc();
      named_bar_sync(kBarStage, kGemmConsumerThreads);    // the pass is complete
      ++staged;
    };
    if constexpr (kPingPong) {
      named_bar_sync(kBarStage + wg, 128);                // this warpgroup's last epilogue is done
      write_acc();
      named_bar_sync(kBarStage + wg, 128);
      staged = 1;
    } else if (wg == 1) {                                 // warpgroup 1 only feeds the staging tile
      stage_pass(false);
      stage_pass(true);
      continue;
    } else {
      stage_pass(true);     // up front, so that the accumulator registers are free for the epilogue
    }
    // column c of the tile is readable once the pass that holds it has been staged
    auto need = [&](int col) {
      if constexpr (!kPingPong) {
        while (staged <= (col >> 7) && staged < kPasses) stage_pass(false);
      }
    };

    const int row = m_blk * kGemmBlockM + wt;
    const bool row_ok = row < p.M;
    if constexpr (EPI == EPI_STORE) {
      gemm_epilogue_store<BLOCK_N>(p, acc_row, acc_sw, row, n_blk, split, need);
    } else if constexpr (EPI == EPI_NCE_FWD) {
      // Per row and column block: running maximum m and sum of 2^(x - m), x = s*log2(e), with an
      // online rescale per 32-column chunk (no fixed shift: a fixed exp(s - alpha) underflows
      // to sum = 0 once exp(temperature) reaches CLIP's usual logit scales of 50-100).
      const float alpha = __ldg(p.alpha_dev);
      const float a2 = alpha * 1.4426950408889634f;
      const int diag_col = row + p.diag_offset;
      float run_m = -INFINITY, run_s = 0.f;
#pragma unroll 1
      for (int c = 0; c < BLOCK_N / 32; ++c) {
        need(c * 32);
        const int col0 = n_blk * BLOCK_N + c * 32;
        if (col0 >= p.N) continue;
        float v[32];
        acc_ld32(acc_row, acc_sw, c * 32, v);
        const bool interior = col0 + 32 <= p.N && (diag_col < col0 || diag_col >= col0 + 32);
        float cm = -INFINITY;
        if (interior) {
#pragma unroll
          for (int i = 0; i < 32; ++i) cm = fmaxf(cm, v[i]);
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int col = col0 + i;
            const bool is_diag = (col == diag_col);
            if (is_diag && row_ok) p.nce_pos[row] = v[i] * alpha;
            if (col >= p.N || (p.dcl && is_diag)) v[i] = -INFINITY;   // not in the sum
            cm = fmaxf(cm, v[i]);
          }
        }
        cm *= a2;                                   // a2 > 0: max commutes with the scaling
        if (cm > run_m) { run_s *= exp2f(run_m - cm); run_m = cm; }
        if (run_m > -INFINITY) {
#pragma unroll
          for (int i = 0; i < 32; ++i) run_s += exp2f(fmaf(v[i], a2, -run_m));
        }
      }
      if (row_ok) {
        float2* dst = reinterpret_cast<float2*>(p.nce_part) + ((long long)n_blk * p.M + row);
        *dst = make_float2(run_m, run_s);
      }
    } else if constexpr (EPI == EPI_SEGMAX) {
      // (segment, position) of the tile's first column from one division, then stepped per column;
      // the column walk is the same for every thread of the CTA, so its branches do not diverge.
      // A strict '>' scan: ties go to the lowest index.
      const float alpha = __ldg(p.alpha_dev);
      const int L = p.seg_len;
      const int col_base = n_blk * BLOCK_N;
      const int valid = min(BLOCK_N, p.N - col_base);
      int seg = col_base / L;
      int pos = col_base - seg * L;
      bool whole = pos == 0;                       // the current segment starts inside this tile
      float best = -INFINITY;
      int best_i = 0;
      unsigned long long* keys = p.seg_keys + (long long)(row_ok ? row : 0) * p.n_segs;
      auto close_segment = [&]() {                 // the current segment ends at this column
        if (row_ok) {
          const unsigned long long k = segmax_key(best, best_i);
          if (whole) keys[seg] = k;
          else atomicMax(keys + seg, k);
        }
        ++seg; pos = 0; whole = true; best = -INFINITY; best_i = 0;
      };
#pragma unroll 1
      for (int c0 = 0; c0 < valid; c0 += 16) {
        need(c0);
        float v[16];
        acc_ld16(acc_row, acc_sw, c0, v);
        const int col0 = col_base + c0;
        if (c0 + 16 <= valid && pos + 16 <= L) {  // the whole chunk lies inside one segment
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            float sv = v[i] * alpha;
            if (p.col_mul != nullptr) sv = fmaf(v[i] * alpha, p.col_mul[col0 + i], p.col_add[col0 + i]);
            if (sv > best) { best = sv; best_i = pos + i; }
          }
          pos += 16;
          if (pos == L) close_segment();
        } else {                                   // segment boundaries inside the chunk, or C ends
#pragma unroll
          for (int i = 0; i < 16; ++i) {
            if (c0 + i < valid) {
              float sv = v[i] * alpha;
              if (p.col_mul != nullptr) sv = fmaf(v[i] * alpha, p.col_mul[col0 + i], p.col_add[col0 + i]);
              if (sv > best) { best = sv; best_i = pos; }
              if (++pos == L) close_segment();
            }
          }
        }
      }
      // a segment that goes on in the next tile: merge this piece (C is a whole number of
      // segments, so this happens only on a full tile)
      if (pos != 0 && row_ok) atomicMax(keys + seg, segmax_key(best, best_i));
    } else if constexpr (EPI == EPI_NCE_BWD) {
      const float alpha = __ldg(p.alpha_dev);
      const float gs = __ldg(p.gscale_dev);
      const float w_row = p.w_row * gs, w_col = p.w_col * gs, w_diag = p.w_diag * gs;
      const float a2 = alpha * 1.4426950408889634f;
      const int diag_col = row + p.diag_offset;
      const float lr2 = (row_ok && p.lse_row) ? p.lse_row[row] * 1.4426950408889634f : 0.f;
      float tsum = 0.f;
#pragma unroll 1
      for (int c = 0; c < BLOCK_N / 32; ++c) {
        need(c * 32);
        const int col0 = n_blk * BLOCK_N + c * 32;
        if (!row_ok || col0 >= (int)p.ldc) continue;   // pad columns [N, ldc) get zeros
        float v[32];
        acc_ld32(acc_row, acc_sw, c * 32, v);
        float gq[32];
        // interior chunk (all 32 columns exist, the positive is elsewhere): two ex2.approx per
        // element; the general path keeps the per-element predicates
        const bool interior = col0 + 32 <= p.N && (diag_col < col0 || diag_col >= col0 + 32);
        if (interior) {
          float part = 0.f;
          if (p.w_col != 0.f) {
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
              const float4 lc = __ldg(reinterpret_cast<const float4*>(p.lse_col + col0 + i));
              const float l4[4] = {lc.x, lc.y, lc.z, lc.w};
#pragma unroll
              for (int e = 0; e < 4; ++e) {
                const float acc_v = v[i + e];
                const float x = acc_v * a2;
                float gv = w_col * nce_ex2(fmaf(l4[e], -1.4426950408889634f, x));
                if (p.w_row != 0.f) gv = fmaf(w_row, nce_ex2(x - lr2), gv);
                part = fmaf(gv, acc_v, part);
                gq[i + e] = gv * alpha;
              }
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) {
              const float acc_v = v[i];
              const float gv = w_row * nce_ex2(fmaf(acc_v, a2, -lr2));
              part = fmaf(gv, acc_v, part);
              gq[i] = gv * alpha;
            }
          }
          tsum = fmaf(part, alpha, tsum);
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int col = col0 + i;
            const float acc_v = v[i];
            const bool is_diag = (col == diag_col);
            float gv = 0.f;
            if (col < p.N) {
              if (!(p.dcl && is_diag)) {
                if (p.w_row != 0.f) gv += w_row * nce_ex2(acc_v * a2 - lr2);
                if (p.w_col != 0.f)
                  gv += w_col * nce_ex2(acc_v * a2 - __ldg(p.lse_col + col) * 1.4426950408889634f);
              }
              if (is_diag) gv -= w_diag;
              tsum += gv * acc_v * alpha;
            }
            gq[i] = gv * alpha;   // temperature folded in: d rows = gq @ cols; 0 beyond N
          }
        }
        bf16* grow = reinterpret_cast<bf16*>(p.c) + (long long)row * p.ldc + col0;
#pragma unroll
        for (int i = 0; i < 32; i += 8)
          if (col0 + i < (int)p.ldc) st_bf16x8(grow + i, gq + i);
      }
      if (p.dtemp != nullptr) {
        tsum = warp_sum(tsum);
        if (lane == 0) atomicAdd(p.dtemp, tsum);
      }
    } else if constexpr (EPI == EPI_SIMREG_FWD) {
      const int diag_col = row + p.diag_offset;
      float s4[4] = {0.f, 0.f, 0.f, 0.f};          // four chains: the fma latency is not serialised
#pragma unroll 1
      for (int c = 0; c < BLOCK_N / 32; ++c) {
        need(c * 32);
        const int col0 = n_blk * BLOCK_N + c * 32;
        if (col0 >= p.N) continue;
        float v[32];
        acc_ld32(acc_row, acc_sw, c * 32, v);
        if (!(col0 + 32 <= p.N && (diag_col < col0 || diag_col >= col0 + 32))) {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            const int col = col0 + i;
            if (col >= p.N || col == diag_col) v[i] = 0.f;
          }
        }
#pragma unroll
        for (int i = 0; i < 32; ++i) s4[i & 3] = fmaf(v[i], v[i], s4[i & 3]);
      }
      if (row_ok) p.nce_part[(long long)n_blk * p.M + row] = (s4[0] + s4[1]) + (s4[2] + s4[3]);
    } else if constexpr (EPI == EPI_VCE_FWD) {
      // EPI_NCE_FWD's online (max, sum) per 32-column chunk, on l = acc + bias
      constexpr float kLog2e = 1.4426950408889634f;
      const long long label = row_ok ? p.labels[row] : -1;
      float run_m = -INFINITY, run_s = 0.f;
#pragma unroll 1
      for (int c = 0; c < BLOCK_N / 32; ++c) {
        need(c * 32);
        const int col0 = n_blk * BLOCK_N + c * 32;
        if (col0 >= p.N) continue;
        float v[32];
        acc_ld32(acc_row, acc_sw, c * 32, v);
        vce_add_bias(p, col0, v);
        if (label >= col0 && label < col0 + 32) {
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (col0 + i == label) p.nce_pos[row] = v[i];
        }
        float cm = -INFINITY;
        if (col0 + 32 <= p.N) {
#pragma unroll
          for (int i = 0; i < 32; ++i) cm = fmaxf(cm, v[i]);
        } else {
#pragma unroll
          for (int i = 0; i < 32; ++i) {
            if (col0 + i >= p.N) v[i] = -INFINITY;        // not in the sum
            cm = fmaxf(cm, v[i]);
          }
        }
        cm *= kLog2e;
        if (cm > run_m) { run_s *= exp2f(run_m - cm); run_m = cm; }
#pragma unroll
        for (int i = 0; i < 32; ++i) run_s += exp2f(fmaf(v[i], kLog2e, -run_m));
      }
      if (row_ok) {
        float2* dst = reinterpret_cast<float2*>(p.nce_part) + ((long long)n_blk * p.M + row);
        *dst = make_float2(run_m, run_s);
      }
    } else if constexpr (EPI == EPI_VCE_BWD) {
      constexpr float kLog2e = 1.4426950408889634f;
      const float gs = __ldg(p.gscale_dev);
      const long long label = row_ok ? p.labels[row] : -1;
      const float lr2 = row_ok ? p.lse_row[row] * kLog2e : 0.f;
#pragma unroll 1
      for (int c = 0; c < BLOCK_N / 32; ++c) {
        need(c * 32);
        const int col0 = n_blk * BLOCK_N + c * 32;
        if (!row_ok || col0 >= (int)p.ldc) continue;   // pad columns [N, ldc) get zeros
        float v[32];
        acc_ld32(acc_row, acc_sw, c * 32, v);
        vce_add_bias(p, col0, v);
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = gs * nce_ex2(fmaf(v[i], kLog2e, -lr2));
        if (col0 + 32 > p.N) {
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (col0 + i >= p.N) v[i] = 0.f;
        }
        if (label >= col0 && label < col0 + 32) {
#pragma unroll
          for (int i = 0; i < 32; ++i)
            if (col0 + i == label) v[i] -= gs;
        }
        bf16* grow = reinterpret_cast<bf16*>(p.c) + (long long)row * p.ldc + col0;
#pragma unroll
        for (int i = 0; i < 32; i += 8)
          if (col0 + i < (int)p.ldc) st_bf16x8(grow + i, v + i);
      }
    } else if constexpr (EPI == EPI_SIMREG_BWD) {
      const float gs = __ldg(p.gscale_dev);
      const int diag_col = row + p.diag_offset;
#pragma unroll 1
      for (int c = 0; c < BLOCK_N / 32; ++c) {
        need(c * 32);
        const int col0 = n_blk * BLOCK_N + c * 32;
        if (!row_ok || col0 >= (int)p.ldc) continue;   // pad columns [N, ldc) get zeros
        float v[32];
        acc_ld32(acc_row, acc_sw, c * 32, v);
#pragma unroll
        for (int i = 0; i < 32; ++i) {
          const int col = col0 + i;
          v[i] = (col < p.N && col != diag_col) ? gs * v[i] : 0.f;
        }
        bf16* grow = reinterpret_cast<bf16*>(p.c) + (long long)row * p.ldc + col0;
#pragma unroll
        for (int i = 0; i < 32; i += 8)
          if (col0 + i < (int)p.ldc) st_bf16x8(grow + i, v + i);
      }
    } else if constexpr (EPI == EPI_FF_DOWN) {
      static_assert(BLOCK_N == 128, "the feed-forward epilogues use 128-column tiles");
      need(0);
      const float invD = p.ff_inv_hidden;
      float mean = 0.f, rstd = 0.f;
      if (row_ok) {
        const int nparts = p.ff_hidden >> 6;
        const float4* parts = reinterpret_cast<const float4*>(p.ff_rowsum + 2ll * (long long)row * nparts);
        float sx = 0.f, sy = 0.f;
        for (int k = 0; k < nparts / 2; ++k) {                   // fixed order
          const float4 v = __ldg(parts + k);
          sx += v.x; sy += v.y; sx += v.z; sy += v.w;
        }
        mean = sx * invD;
        rstd = rsqrtf(fmaxf(sy * invD - mean * mean, 0.f) + p.ff_eps);
        if (n_blk == 0) *reinterpret_cast<float2*>(p.ff_stats + 2ll * row) = make_float2(mean, rstd);
      }
      const bf16* res_row = (p.residual != nullptr && row_ok) ? p.residual + (long long)row * p.ldr : nullptr;
#pragma unroll 1
      for (int c = 0; c < BLOCK_N; c += 32) {
        const int col0 = n_blk * BLOCK_N + c;
        if (!row_ok || col0 >= p.N) continue;
        float v[32];
        acc_ld32(acc_row, acc_sw, c, v);
#pragma unroll
        for (int i = 0; i < 32; i += 8) {
          float o8[8];
          float r8[8] = {0, 0, 0, 0, 0, 0, 0, 0};
          if (res_row != nullptr) {
            const uint4 r4 = *reinterpret_cast<const uint4*>(res_row + col0 + i);
            float2 x0 = unpack_bf16x2(r4.x), x1 = unpack_bf16x2(r4.y);
            float2 x2 = unpack_bf16x2(r4.z), x3 = unpack_bf16x2(r4.w);
            r8[0] = x0.x; r8[1] = x0.y; r8[2] = x1.x; r8[3] = x1.y;
            r8[4] = x2.x; r8[5] = x2.y; r8[6] = x3.x; r8[7] = x3.y;
          }
          const float4 c0 = *reinterpret_cast<const float4*>(p.ff_colvec + col0 + i);
          const float4 c1 = *reinterpret_cast<const float4*>(p.ff_colvec + col0 + i + 4);
          const float c8[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
#pragma unroll
          for (int e = 0; e < 8; ++e) o8[e] = fmaf(rstd, v[i + e] - mean * c8[e], r8[e]);
          st_bf16x8(reinterpret_cast<bf16*>(p.c) + (long long)row * p.ldc + col0 + i, o8);
          st_bf16x8(p.ff_out2 + (long long)row * p.ff_ld2 + col0 + i, v + i);
        }
      }
    }
    if constexpr (!kPingPong)
      while (staged < kPasses) stage_pass(false);      // keep the staging handshake in lock-step
  }
  if constexpr (S::kActTile) {
    if (wt < 32 && XCLIP_ONE_LANE(lane)) bulk_wait_group<0>();   // the last tile's stores
  }
}

}  // namespace xclip
