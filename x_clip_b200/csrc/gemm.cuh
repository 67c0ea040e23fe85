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
// contrastive loss (NCE / FILIP epilogues) and the fused feed-forward (FF epilogues, see ff.cu).
//
// Structure (one CTA per SM, 288 threads), output tile 128 x BLOCK_N:
//   warps 0-3 : consumer warpgroup 0 - wgmma on columns [0, BLOCK_N/2) of the tile, then the epilogue
//   warps 4-7 : consumer warpgroup 1 - wgmma on columns [BLOCK_N/2, BLOCK_N)
//   warp  8   : TMA producer (one elected lane)
// Pipeline: shared-memory ring full/empty (TMA <-> wgmma), static persistent tile scheduler with
// optional split-K.  After its k-loop each warpgroup parks its accumulator (fp32 registers) in a
// 128 x 128 staging tile in shared memory; the epilogue then gives every thread of warpgroup 0 one
// row (thread t = row t) and walks the columns, so row reductions (softmax partials, segment maxima,
// LayerNorm sums) stay in registers.  With BLOCK_N = 256 the two halves pass through the staging tile
// one after the other while warpgroup 1 already runs the next tile's k-loop.
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
  // ---- FILIP segment-max epilogue (EPI_SEGMAX): columns are grouped in segments of seg_len
  // tokens (one segment = one sample of the other modality); n_tile_stride = columns a tile
  // advances by (a whole number of segments, <= BLOCK_N)
  int seg_len, n_tile_stride, n_segs;
  const float* col_mul;    // [N] or null: per-column multiplier (0 for masked text tokens)
  const float* col_add;    // [N] or null: per-column addend (-FLT_MAX for masked text tokens)
  float* seg_max;          // [M, n_segs]  max_i s
  int* seg_arg;            // [M, n_segs]  argmax (index inside the segment)
  // ---- fused feed-forward epilogues (EPI_FF_*)
  float* ff_rowsum;        // [M, 4d/64, 2] per-box (sum, sum of squares) of the GEGLU output rows: UP writes, DOWN sums
  const float* ff_colvec;  // DOWN: c[N] = row sums of the gain-scaled down-projection weight
  float* ff_stats;         // DOWN: [M,2] (mean, rstd) of the GEGLU output rows, written for the backward
  float ff_eps;            // LayerNorm epsilon
  int ff_hidden;           // 4*dim: LayerNorm width; column offset of the gate half inside u
  int ff_skip_u;           // UP: do not write u = [value | gate] (inference / no-grad sweeps need only hp)
  bf16* ff_u;              // UP: [value | gate] output [M, 8d];  BWD: saved [value | gate] activations
  long long ff_ldu;
  bf16* ff_out2;           // UP: hp [M, 4d];  DOWN: bf16(acc) [M, d]
  long long ff_ld2;
  const float* ff_ab;      // BWD: [M,2] per-row (mean_k(gdh), mean_k(gdh * hn)) from xclip_ff_bwd_prep
};

constexpr int EPI_STORE = 0;    // C = alpha*acc (+bias) (+residual)
constexpr int EPI_NCE_FWD = 1;  // row partial sums of exp(s - alpha) and the positives
constexpr int EPI_NCE_BWD = 2;  // C = g = w_row*exp(s-lse_row) + w_col*exp(s-lse_col) - w_diag*[diag]
constexpr int EPI_SEGMAX = 3;   // per row and column segment: max and argmax of alpha*acc (FILIP)
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
constexpr int EPI_FF_UP = 4;
constexpr int EPI_FF_DOWN = 5;
constexpr int EPI_FF_BWD = 6;

constexpr int kGemmBlockM = 128;
constexpr int kGemmBlockK = 64;
constexpr int kGemmConsumerThreads = 256;
constexpr int kGemmThreads = kGemmConsumerThreads + 32;
constexpr int kAccLd = 128 + 4;   // staging row stride (floats): conflict-free 16-byte row reads

template <int BLOCK_N>
struct GemmSmem {
  static constexpr int kABytes = kGemmBlockM * kGemmBlockK * 2;  // 16 KiB
  static constexpr int kBBytes = BLOCK_N * kGemmBlockK * 2;      // 16/32 KiB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kStages = (BLOCK_N == 256) ? 3 : 4;
  static constexpr int kAccBytes = kGemmBlockM * kAccLd * 4;     // fp32 staging tile, 128 columns
  static constexpr int kBarrierBytes = 256;
  static constexpr int kTotal = kStages * kStageBytes + kAccBytes + kBarrierBytes;
};

__device__ __forceinline__ float nce_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// 32 consecutive fp32 accumulator columns [col, col + 32) of this thread's row from the staging tile
__device__ __forceinline__ void acc_ld32(const float* row, int col, float (&f)[32]) {
  const float4* src = reinterpret_cast<const float4*>(row + (col & 127));
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const float4 v = src[i];
    f[4 * i] = v.x; f[4 * i + 1] = v.y; f[4 * i + 2] = v.z; f[4 * i + 3] = v.w;
  }
}
__device__ __forceinline__ void acc_ld16(const float* row, int col, float (&f)[16]) {
  const float4* src = reinterpret_cast<const float4*>(row + (col & 127));
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float4 v = src[i];
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

// Epilogue of one 128 x BLOCK_N tile for EPI_STORE; `stage(c)` makes column c of the tile readable.
template <int BLOCK_N, class Stage>
__device__ __forceinline__ void gemm_epilogue_store(const GemmParams& p, const float* acc_row, int row,
                                                    int n_blk, int split, Stage&& stage) {
  const bool row_ok = row < p.M;
  const bf16* res_row = nullptr;
  if (p.residual != nullptr && row_ok) {
    const long long rr = p.res_row_idx ? p.res_row_idx[row] : (p.res_row_mod > 0 ? (row % p.res_row_mod) : row);
    res_row = p.residual + rr * p.ldr;
  }
#pragma unroll 1
  for (int c = 0; c < BLOCK_N / 32; ++c) {
    stage(c * 32);
    const int col0 = n_blk * BLOCK_N + c * 32;
    if (!row_ok || col0 >= p.N) continue;
    float f[32];
    acc_ld32(acc_row, c * 32, f);
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
    if (res_row != nullptr && split == 0) {
#pragma unroll
      for (int i = 0; i < 32; i += 8) {
        if (col0 + i < p.N) {
          const uint4 r4 = *reinterpret_cast<const uint4*>(res_row + col0 + i);
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

template <int BLOCK_N, int A_MAJOR, int B_MAJOR, int EPI = EPI_STORE>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_bf16_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const GemmParams p) {
  using S = GemmSmem<BLOCK_N>;
  constexpr int kStages = S::kStages;
  constexpr int kHalfN = BLOCK_N / 2;          // columns of one consumer warpgroup
  constexpr int kFrag = kHalfN / 2;            // fp32 accumulator registers per m64 half
  constexpr int kPasses = BLOCK_N / 128;       // trips through the 128-column staging tile
  static_assert(BLOCK_N == 128 || BLOCK_N == 256, "BLOCK_N must be 128 or 256");

  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* smem_a = smem;
  uint8_t* smem_b = smem + kStages * S::kABytes;
  float* acc_smem = reinterpret_cast<float*>(smem + kStages * S::kStageBytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kStages * S::kStageBytes + S::kAccBytes);
  uint64_t* full_bar = bars;                    // [kStages]
  uint64_t* empty_bar = bars + kStages;         // [kStages]

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  const int num_m = (p.M + kGemmBlockM - 1) / kGemmBlockM;
  const int n_stride = (EPI == EPI_SEGMAX) ? p.n_tile_stride : BLOCK_N;
  const int num_n = (p.N + n_stride - 1) / n_stride;
  const int num_kb = (p.K + kGemmBlockK - 1) / kGemmBlockK;
  const int splits = p.split_k > 0 ? p.split_k : 1;
  const int kb_per_split = (num_kb + splits - 1) / splits;
  const int num_tiles = num_m * num_n * splits;

  if (threadIdx.x == 0) {
    if ((smem_u32(smem) & 1023u) != 0) __trap();   // the 128-byte swizzle needs 1024-byte aligned tiles
    for (int i = 0; i < kStages; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], kGemmConsumerThreads / 32);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == kGemmConsumerThreads / 32) {
    // ===================== TMA producer =====================
    if (XCLIP_ONE_LANE(lane)) {
      tma_prefetch_desc(&tmA);
      tma_prefetch_desc(&tmB);
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
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
            tma_load_2d(sb, &tmB, &full_bar[stage], kb * kGemmBlockK, n_blk * n_stride);
          } else {
#pragma unroll
            for (int g = 0; g < BLOCK_N / 64; ++g)
              tma_load_2d(sb + g * (kGemmBlockK * 128), &tmB, &full_bar[stage],
                          n_blk * n_stride + g * 64, kb * kGemmBlockK);
          }
          if (++stage == kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers (warpgroups 0 and 1) =====================
  const int wg = threadIdx.x >> 7;
  const int wt = threadIdx.x & 127;            // thread inside the warpgroup
  // K-major: SBO = 1024 (8 rows x 128 B), LBO unused.  MN-major: SBO = 1024 between 8-row K groups,
  // LBO = BLOCK_K*128 between 64-wide M/N groups (one TMA box each).
  constexpr uint32_t kLboMN = kGemmBlockK * 128;
  constexpr uint32_t kAStep = (A_MAJOR == kMajorK) ? 32u : 2048u;  // bytes per k16
  constexpr uint32_t kBStep = (B_MAJOR == kMajorK) ? 32u : 2048u;
  // this warpgroup's half of the B tile and the second m64 half of the A tile
  const uint32_t b_off = (B_MAJOR == kMajorK) ? wg * kHalfN * 128 : wg * (kHalfN / 64) * kLboMN;
  constexpr uint32_t kAHalf = (A_MAJOR == kMajorK) ? 64 * 128 : kLboMN;
  const float* acc_row = acc_smem + wt * kAccLd;   // epilogue: this thread's row of the staging tile

  int stage = 0;
  uint32_t phase = 0;
  for (int t = blockIdx.x; t < num_tiles; t += gridDim.x) {
    const int tmn = t % (num_n * num_m);
    const int n_blk = p.raster_m_fast ? tmn / num_m : tmn % num_n;
    const int m_blk = p.raster_m_fast ? tmn % num_m : tmn / num_n;
    const int split = t / (num_n * num_m);
    const int kb0 = split * kb_per_split;
    const int kb1 = min(kb0 + kb_per_split, num_kb);
    int prev_stage = -1;               // stage read by the wgmma group still in flight

    float acc[2][kFrag];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int j = 0; j < kFrag; ++j) acc[h][j] = 0.f;

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
          if constexpr (kHalfN == 128) wgmma_m64n128k16<A_MAJOR, B_MAJOR>(acc[h], da, db);
          else wgmma_m64n64k16<A_MAJOR, B_MAJOR>(acc[h], da, db);
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
    wgmma_wait<0>();
    __syncwarp();
    if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);

    // ---- accumulator -> staging tile.  Pass q holds tile columns [128 q, 128 q + 128): with
    // BLOCK_N = 128 both warpgroups write their 64 columns in pass 0, with 256 warpgroup q writes pass q.
    int staged = 0;
    auto stage_pass = [&]() {
      named_bar_sync(2, kGemmConsumerThreads);            // the previous pass has been read
      if (kPasses == 1 || wg == staged) {
        const int w = wt >> 5;
        const int cbase = (kPasses == 1) ? wg * kHalfN : 0;
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < kFrag; j += 2) {
            const int r = h * 64 + w * 16 + (lane >> 2) + 8 * ((j >> 1) & 1);
            const int c = cbase + (j >> 2) * 8 + (lane & 3) * 2;
            *reinterpret_cast<float2*>(acc_smem + r * kAccLd + c) = make_float2(acc[h][j], acc[h][j + 1]);
          }
      }
      named_bar_sync(2, kGemmConsumerThreads);            // the pass is complete
      ++staged;
    };
    if (wg == 1) {                                       // warpgroup 1 only feeds the staging tile
      while (staged < kPasses) stage_pass();
      continue;
    }
    // column c of the tile is readable once the pass that holds it has been staged
    auto need = [&](int col) {
      while (staged <= (col >> 7) && staged < kPasses) stage_pass();
    };

    const int row = m_blk * kGemmBlockM + wt;
    const bool row_ok = row < p.M;
    if constexpr (EPI == EPI_STORE) {
      gemm_epilogue_store<BLOCK_N>(p, acc_row, row, n_blk, split, need);
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
        acc_ld32(acc_row, c * 32, v);
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
      const float alpha = __ldg(p.alpha_dev);
      const int col_base = n_blk * n_stride;
      const int valid = min(n_stride, p.N - col_base);        // multiple of seg_len (and of 16)
      float best = -INFINITY;
      int best_i = 0;
#pragma unroll 1
      for (int c0 = 0; c0 < valid; c0 += 16) {
        need(c0);
        float v[16];
        acc_ld16(acc_row, c0, v);
        const int in_seg = c0 % p.seg_len;
        if (in_seg == 0) { best = -INFINITY; best_i = 0; }
#pragma unroll
        for (int i = 0; i < 16; ++i) {
          float sv = v[i] * alpha;
          if (p.col_mul != nullptr)
            sv = fmaf(v[i] * alpha, p.col_mul[col_base + c0 + i], p.col_add[col_base + c0 + i]);
          if (sv > best) { best = sv; best_i = in_seg + i; }
        }
        if (in_seg + 16 == p.seg_len && row_ok) {
          const long long o = (long long)row * p.n_segs + (col_base + c0) / p.seg_len;
          p.seg_max[o] = best;
          p.seg_arg[o] = best_i;
        }
      }
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
        acc_ld32(acc_row, c * 32, v);
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
    } else if constexpr (EPI == EPI_FF_UP) {
      // tile columns [0,64) = value, [64,128) = gate of hidden units [64 n_blk, +64)
      static_assert(BLOCK_N == 128, "the feed-forward epilogues use 128-column tiles");
      need(0);
      const int hcol = n_blk * 64;
      f32x2 s1p = f2_splat(0.f), s2p = f2_splat(0.f);
#pragma unroll 1
      for (int c = 0; c < 64; c += 16) {
        float vv[16], gg[16];
        acc_ld16(acc_row, c, vv);
        acc_ld16(acc_row, 64 + c, gg);
        float hv[16];
#pragma unroll
        for (int i = 0; i < 16; i += 2) {
          const GeluParts2 gp = gelu_parts2(gg[i], gg[i + 1]);
          const f32x2 ge = f2_mul(f2_pack(gg[i], gg[i + 1]), gp.cdf);               // gelu(gate)
          const uint32_t hw = f2_to_bf16x2(f2_mul(f2_pack(vv[i], vv[i + 1]), ge));   // hp, rounded to bf16
          const f32x2 hr = f2_from_bf16x2(hw);           // statistics of what the next GEMM reads
          s1p = f2_add(s1p, hr);
          s2p = f2_fma(hr, hr, s2p);
          hv[i] = hr.x; hv[i + 1] = hr.y;
        }
        if (row_ok) {
          if (!p.ff_skip_u) {
            bf16* urow = p.ff_u + (long long)row * p.ff_ldu + hcol + c;
            st_bf16x8(urow, vv); st_bf16x8(urow + 8, vv + 8);
            st_bf16x8(urow + p.ff_hidden, gg); st_bf16x8(urow + p.ff_hidden + 8, gg + 8);
          }
          bf16* hrow = p.ff_out2 + (long long)row * p.ff_ld2 + hcol + c;
          st_bf16x8(hrow, hv); st_bf16x8(hrow + 8, hv + 8);
        }
      }
      // one (sum, sum^2) slot per row and 64-column box: plain stores, summed in a fixed order by
      // the down-projection -> the statistics (and the loss) are bit-reproducible run to run
      if (row_ok) {
        const int nparts = p.ff_hidden >> 6;                     // 4d / 64 boxes per row
        *reinterpret_cast<float2*>(p.ff_rowsum + 2ll * ((long long)row * nparts + n_blk)) =
            make_float2(s1p.x + s1p.y, s2p.x + s2p.y);
      }
    } else if constexpr (EPI == EPI_FF_DOWN) {
      static_assert(BLOCK_N == 128, "the feed-forward epilogues use 128-column tiles");
      need(0);
      const float invD = 1.f / (float)p.ff_hidden;
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
        acc_ld32(acc_row, c, v);
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
    } else {   // EPI_FF_BWD: tile columns = hidden units [128 n_blk, +128)
      static_assert(BLOCK_N == 128, "the feed-forward epilogues use 128-column tiles");
      need(0);
      float mean = 0.f, rstd = 0.f, am = 0.f, bm = 0.f;
      if (row_ok) {
        const float2 st = *reinterpret_cast<const float2*>(p.ff_stats + 2ll * row);
        const float2 ab = *reinterpret_cast<const float2*>(p.ff_ab + 2ll * row);
        mean = st.x; rstd = st.y; am = ab.x; bm = ab.y;
      }
      const f32x2 rstd2 = f2_splat(rstd), nmr = f2_splat(-mean * rstd), namr = f2_splat(-am * rstd),
                  nbmr = f2_splat(-bm * rstd);
      const bf16* urow = p.ff_u + (long long)(row_ok ? row : 0) * p.ff_ldu;
      bf16* drow = reinterpret_cast<bf16*>(p.c) + (long long)(row_ok ? row : 0) * p.ldc;
#pragma unroll 1
      for (int c = 0; c < BLOCK_N; c += 16) {
        if (!row_ok) break;
        const int kq = n_blk * BLOCK_N + c;
        float v[16];
        acc_ld16(acc_row, c, v);
#pragma unroll
        for (int i = 0; i < 16; i += 8) {
          const uint4 wv4 = *reinterpret_cast<const uint4*>(urow + kq + i);
          const uint4 wg4 = *reinterpret_cast<const uint4*>(urow + p.ff_hidden + kq + i);
          const uint32_t wv[4] = {wv4.x, wv4.y, wv4.z, wv4.w}, wgt[4] = {wg4.x, wg4.y, wg4.z, wg4.w};
          uint32_t dvw[4], dgw[4];
#pragma unroll
          for (int k = 0; k < 4; ++k) {                           // two columns per step
            const float g0 = __uint_as_float(wgt[k] << 16), g1 = __uint_as_float(wgt[k] & 0xffff0000u);
            const f32x2 gate = f2_pack(g0, g1), val = f2_from_bf16x2(wv[k]);
            const GeluParts2 gp = gelu_parts2(g0, g1);
            const f32x2 ge = f2_mul(gate, gp.cdf);                // gelu(gate)
            const f32x2 gd = f2_fma(gate, gp.pdf, gp.cdf);        // gelu'(gate)
            const f32x2 hn = f2_fma(f2_mul(val, ge), rstd2, nmr); // (val*ge - mean) rstd
            f32x2 dhp = f2_fma(f2_pack(v[i + 2 * k], v[i + 2 * k + 1]), rstd2, namr);   // rstd (gdh - a)
            dhp = f2_fma(hn, nbmr, dhp);                          //   - rstd b hn
            dvw[k] = f2_to_bf16x2(f2_mul(dhp, ge));
            dgw[k] = f2_to_bf16x2(f2_mul(f2_mul(dhp, val), gd));
          }
          *reinterpret_cast<uint4*>(drow + kq + i) = make_uint4(dvw[0], dvw[1], dvw[2], dvw[3]);
          *reinterpret_cast<uint4*>(drow + p.ff_hidden + kq + i) = make_uint4(dgw[0], dgw[1], dgw[2], dgw[3]);
        }
      }
    }
    while (staged < kPasses) stage_pass();             // keep the staging handshake in lock-step
  }
}

}  // namespace xclip
