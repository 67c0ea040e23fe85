// Similarity regularisation (arXiv 2309.08773; reference x_clip/x_clip.py:771-784, :870-873) on top of
// the wgmma GEMM mainloop (gemm.cuh):
//
//   L_sim = mean_{i != j} (T T^T - V V^T)_ij^2     per latent pair (T texts, V images, unit rows)
//
// The difference E = T T^T - V V^T is formed inside the fp32 accumulator by one contraction of the
// concatenated operands  [T | V] . [T | -V]^T  (K = 2 x the split-bf16 width of xclip_l2norm_fwd), so
// E keeps fp32-level accuracy even when the two similarity matrices agree to 1e-3 - subtracting two
// separately rounded matrices would lose those digits.  Negating a bf16 operand is exact.
//
//   pack     : out = [t | v] (row operand) or [t | -v] (column operand), bf16
//   forward  : per row and column block the sum of E^2 over the columns, the diagonal excluded;
//              a finalize kernel sums the blocks per row and adds scale * sum to *loss_accum.
//              The B_l x B_g matrix is never written.
//   backward : the same tiles are recomputed into g = bf16(gscale * E) (zero on the diagonal),
//              which feeds two plain GEMMs: dT = g @ T_cols, dV = -g @ V_cols.
//
// Rows are the LOCAL samples, columns ALL samples of the global batch, exactly as in nce.cu.
#include "gemm.cuh"
#include "host.h"

namespace xclip {

// one row per block iteration, 8 bf16 per thread and step; sign = 0x80008000 flips both halves' signs
__global__ void simreg_pack_kernel(const uint4* __restrict__ t, const uint4* __restrict__ v, int rows,
                                   int k8, uint32_t sign, uint4* __restrict__ out) {
  for (int r = blockIdx.x; r < rows; r += gridDim.x) {
    const uint4* tr = t + (long long)r * k8;
    const uint4* vr = v + (long long)r * k8;
    uint4* o = out + (long long)r * 2 * k8;
    for (int c = threadIdx.x; c < k8; c += blockDim.x) {
      o[c] = tr[c];
      uint4 x = vr[c];
      x.x ^= sign; x.y ^= sign; x.z ^= sign; x.w ^= sign;
      o[k8 + c] = x;
    }
  }
}

__global__ void __launch_bounds__(1024)
simreg_finalize_kernel(const float* __restrict__ part, int nblk, int rows, float* __restrict__ rowsum,
                       float* __restrict__ loss_accum, float scale) {
  __shared__ float red[32];
  float local = 0.f;
  for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < rows; r += gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < nblk; ++k) s += part[(long long)k * rows + r];   // fixed order
    if (rowsum != nullptr) rowsum[r] = s;
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

template <int BLOCK_N, int EPI>
static int launch_simreg(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int grid,
                         cudaStream_t stream) {
  using S = GemmSmem<BLOCK_N>;
  auto kern = gemm_bf16_kernel<BLOCK_N, kMajorK, kMajorK, EPI>;
  {
    const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), S::kTotal);
    if (rc_attr) return rc_attr;
  }
  kern<<<grid, kGemmThreads, S::kTotal, stream>>>(tmA, tmB, p, CUtensorMap{}, CUtensorMap{});
  XCLIP_LAUNCH_CHECK("gemm_bf16_kernel<simreg>");
  return XCLIP_OK;
}

static int simreg_common(const void* a, const void* b, int R, int C, int K, int diag_offset,
                         GemmParams* p, CUtensorMap* tmA, CUtensorMap* tmB, int* block_n, int* grid) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(a && b, "simreg: null operands");
  XCLIP_REQUIRE(R > 0 && C > 0 && K > 0 && K % 8 == 0, "simreg: bad sizes R=%d C=%d K=%d", R, C, K);
  XCLIP_REQUIRE(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15) == 0,
                "simreg: misaligned operands");
  XCLIP_REQUIRE(diag_offset >= 0 && (long long)diag_offset + R <= C,
                "simreg: diagonal outside the columns (diag_offset=%d R=%d C=%d)", diag_offset, R, C);
  *block_n = C >= 256 ? 256 : 128;
  rc = encode_2d_bf16(tmA, a, (uint64_t)K, (uint64_t)R, (uint64_t)K, 64, kGemmBlockM);
  if (rc) return rc;
  rc = encode_2d_bf16(tmB, b, (uint64_t)K, (uint64_t)C, (uint64_t)K, 64, (uint32_t)*block_n);
  if (rc) return rc;
  GemmParams z = {};
  *p = z;
  p->M = R; p->N = C; p->K = K; p->split_k = 1;
  p->raster_m_fast = 1;   // the local rows stay in L2, all columns stream once
  p->diag_offset = diag_offset;
  const long long tiles =
      (long long)((R + kGemmBlockM - 1) / kGemmBlockM) * ((C + *block_n - 1) / *block_n);
  *grid = (int)(tiles < num_sms() ? tiles : num_sms());
  return XCLIP_OK;
}

}  // namespace xclip

using namespace xclip;

extern "C" int xclip_simreg_pack(const void* t, const void* v, int rows, int k, int negate_v, void* out,
                                 xclip_stream_t stream) {
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(t && v && out, "simreg_pack: null pointer");
  XCLIP_REQUIRE(rows > 0 && k > 0 && k % 8 == 0, "simreg_pack: bad sizes rows=%d k=%d", rows, k);
  XCLIP_REQUIRE(((reinterpret_cast<uintptr_t>(t) | reinterpret_cast<uintptr_t>(v) |
                  reinterpret_cast<uintptr_t>(out)) & 15) == 0,
                "simreg_pack: t, v and out must be 16-byte aligned");
  const int k8 = k / 8;
  const int grid = rows < 16 * num_sms() ? rows : 16 * num_sms();
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  simreg_pack_kernel<<<grid, 128, 0, s>>>(reinterpret_cast<const uint4*>(t),
                                                reinterpret_cast<const uint4*>(v), rows, k8,
                                                negate_v ? 0x80008000u : 0u, reinterpret_cast<uint4*>(out));
  XCLIP_LAUNCH_CHECK("simreg_pack_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_simreg_fwd(const void* a, const void* b, int R, int C, int K, int diag_offset,
                                float* part_ws, float* rowsum, float* loss_accum, float loss_scale,
                                xclip_stream_t stream) {
  GemmParams p;
  CUtensorMap tmA, tmB;
  int block_n = 0, grid = 0;
  int rc = simreg_common(a, b, R, C, K, diag_offset, &p, &tmA, &tmB, &block_n, &grid);
  if (rc) return rc;
  XCLIP_REQUIRE(part_ws, "simreg_fwd: null workspace");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(part_ws) & 3) == 0, "simreg_fwd: misaligned part_ws");
  p.nce_part = part_ws;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  rc = block_n == 256 ? launch_simreg<256, EPI_SIMREG_FWD>(tmA, tmB, p, grid, s)
                      : launch_simreg<128, EPI_SIMREG_FWD>(tmA, tmB, p, grid, s);
  if (rc) return rc;
  const int nblk = xclip_nce_num_col_blocks(C);
  int fgrid = (R + 1023) / 1024;
  if (fgrid > num_sms()) fgrid = num_sms();
  simreg_finalize_kernel<<<fgrid, 1024, 0, s>>>(part_ws, nblk, R, rowsum, loss_accum, loss_scale);
  XCLIP_LAUNCH_CHECK("simreg_finalize_kernel");
  return XCLIP_OK;
}

extern "C" int xclip_simreg_bwd(const void* a, const void* b, int R, int C, int K, int diag_offset,
                                const float* gscale, void* g, int64_t ldg, xclip_stream_t stream) {
  GemmParams p;
  CUtensorMap tmA, tmB;
  int block_n = 0, grid = 0;
  int rc = simreg_common(a, b, R, C, K, diag_offset, &p, &tmA, &tmB, &block_n, &grid);
  if (rc) return rc;
  XCLIP_REQUIRE(g && ldg % 8 == 0 && ldg >= (C + 7) / 8 * 8, "simreg_bwd: g needs ld >= roundup8(C)");
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(g) & 15) == 0, "simreg_bwd: misaligned g");
  XCLIP_REQUIRE(gscale, "simreg_bwd: gscale device scalar required");
  p.gscale_dev = gscale;
  p.c = g; p.ldc = ldg;
  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  return block_n == 256 ? launch_simreg<256, EPI_SIMREG_BWD>(tmA, tmB, p, grid, s)
                        : launch_simreg<128, EPI_SIMREG_BWD>(tmA, tmB, p, grid, s);
}
