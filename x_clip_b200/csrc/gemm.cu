// C-ABI launcher for the wgmma GEMM (see gemm.cuh and include/xclip_b200.h).
#include "gemm.cuh"
#include "host.h"

namespace xclip {

template <int BLOCK_N, int A_MAJOR, int B_MAJOR>
static int launch_gemm(const CUtensorMap& tmA, const CUtensorMap& tmB, const GemmParams& p, int grid,
                       cudaStream_t stream) {
  using S = GemmSmem<BLOCK_N>;
  auto kern = gemm_bf16_kernel<BLOCK_N, A_MAJOR, B_MAJOR>;
  const int rc_attr = ensure_dynamic_smem(reinterpret_cast<const void*>(kern), S::kTotal);
  if (rc_attr) return rc_attr;
  kern<<<grid, kGemmThreads, S::kTotal, stream>>>(tmA, tmB, p);
  XCLIP_LAUNCH_CHECK("gemm_bf16_kernel");
  return XCLIP_OK;
}

template <int BLOCK_N>
static int dispatch_major(int a_major, int b_major, const CUtensorMap& tmA, const CUtensorMap& tmB,
                          const GemmParams& p, int grid, cudaStream_t stream) {
  if (a_major == kMajorK && b_major == kMajorK)
    return launch_gemm<BLOCK_N, kMajorK, kMajorK>(tmA, tmB, p, grid, stream);
  if (a_major == kMajorK && b_major == kMajorMN)
    return launch_gemm<BLOCK_N, kMajorK, kMajorMN>(tmA, tmB, p, grid, stream);
  if (a_major == kMajorMN && b_major == kMajorK)
    return launch_gemm<BLOCK_N, kMajorMN, kMajorK>(tmA, tmB, p, grid, stream);
  return launch_gemm<BLOCK_N, kMajorMN, kMajorMN>(tmA, tmB, p, grid, stream);
}

}  // namespace xclip

extern "C" int xclip_gemm_bf16(const void* a, int64_t lda, int a_major, const void* b, int64_t ldb,
                               int b_major, void* c, int64_t ldc, int c_dtype, int M, int N, int K,
                               float alpha, const float* bias, const void* residual, int64_t ldr,
                               int res_row_mod, const int32_t* res_row_idx, int accumulate,
                               xclip_stream_t stream) {
  using namespace xclip;
  int rc = xclip_init();
  if (rc) return rc;
  XCLIP_REQUIRE(a && b && c, "gemm: null pointer");
  XCLIP_REQUIRE(M > 0 && N > 0 && K > 0, "gemm: empty problem M=%d N=%d K=%d", M, N, K);
  XCLIP_REQUIRE(N % 8 == 0, "gemm: N=%d must be a multiple of 8", N);
  XCLIP_REQUIRE(a_major == 0 || a_major == 1, "gemm: bad a_major %d", a_major);
  XCLIP_REQUIRE(b_major == 0 || b_major == 1, "gemm: bad b_major %d", b_major);
  XCLIP_REQUIRE(c_dtype == 0 || c_dtype == 1, "gemm: bad c_dtype %d", c_dtype);
  XCLIP_REQUIRE(lda % 8 == 0 && ldb % 8 == 0, "gemm: lda=%lld ldb=%lld must be multiples of 8",
                (long long)lda, (long long)ldb);
  XCLIP_REQUIRE(ldc % (c_dtype ? 4 : 8) == 0, "gemm: ldc=%lld misaligned", (long long)ldc);
  XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(a) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(b) & 15) == 0 &&
                    (reinterpret_cast<uintptr_t>(c) & 15) == 0,
                "gemm: base pointers must be 16-byte aligned");
  XCLIP_REQUIRE(!accumulate || c_dtype == 1, "gemm: accumulate needs f32 output");
  XCLIP_REQUIRE(lda >= (a_major == 0 ? K : M), "gemm: lda too small");
  XCLIP_REQUIRE(ldb >= (b_major == 0 ? K : N), "gemm: ldb too small");
  XCLIP_REQUIRE(ldc >= N, "gemm: ldc too small");
  if (residual) {
    XCLIP_REQUIRE(ldr % 8 == 0 && ldr >= N, "gemm: bad ldr");
    XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(residual) & 15) == 0, "gemm: residual misaligned");
  }
  if (bias) XCLIP_REQUIRE((reinterpret_cast<uintptr_t>(bias) & 15) == 0, "gemm: bias misaligned");

  const int block_n = (N % 256 == 0 || N > 1024) ? 256 : 128;

  CUtensorMap tmA, tmB;
  if (a_major == 0) {
    rc = encode_2d_bf16(&tmA, a, (uint64_t)K, (uint64_t)M, (uint64_t)lda, 64, kGemmBlockM);
  } else {
    rc = encode_2d_bf16(&tmA, a, (uint64_t)M, (uint64_t)K, (uint64_t)lda, 64, kGemmBlockK);
  }
  if (rc) return rc;
  if (b_major == 0) {
    rc = encode_2d_bf16(&tmB, b, (uint64_t)K, (uint64_t)N, (uint64_t)ldb, 64, (uint32_t)block_n);
  } else {
    rc = encode_2d_bf16(&tmB, b, (uint64_t)N, (uint64_t)K, (uint64_t)ldb, 64, kGemmBlockK);
  }
  if (rc) return rc;

  const int units = num_sms();      // CTAs that run concurrently (one per SM)
  const int num_m = (M + kGemmBlockM - 1) / kGemmBlockM;
  const int num_n = (N + block_n - 1) / block_n;
  const int num_kb = (K + kGemmBlockK - 1) / kGemmBlockK;
  const long long tiles_mn = (long long)num_m * num_n;
  int splits = 1;
  if (accumulate && tiles_mn < units) {
    // wgrad-shaped problem: few output tiles, very long K.  Split K so that the CTAs form whole
    // waves over the SMs: among split counts that give between ~2 and ~8 waves (and keep >= 8
    // k-blocks per split to amortise the fp32 reduction) take the one with the best last-wave
    // fill; e.g. 64 output tiles: 5 splits = 2.16 waves (72 % fill) vs 9 splits = 3.89 (97 %).
    const long long sms = units;
    const long long lo = (2 * sms + tiles_mn - 1) / tiles_mn;
    long long hi = (8 * sms) / tiles_mn;
    const long long max_by_k = num_kb / 8 > 0 ? num_kb / 8 : 1;
    if (hi > max_by_k) hi = max_by_k;
    long long best = lo < max_by_k ? lo : max_by_k;
    if (best < 1) best = 1;
    double best_fill = 0.0;
    for (long long sp = best; sp <= hi; ++sp) {
      const long long t = tiles_mn * sp;
      const double fill = (double)t / (double)(((t + sms - 1) / sms) * sms);
      if (fill > best_fill + 0.02) { best_fill = fill; best = sp; }
    }
    splits = (int)best;
    const int kb_per = (num_kb + splits - 1) / splits;
    splits = (num_kb + kb_per - 1) / kb_per;  // no empty splits
  }
  const long long total_tiles = tiles_mn * splits;
  int grid = (int)(total_tiles < units ? total_tiles : units);

  GemmParams p = {};
  p.M = M; p.N = N; p.K = K;
  p.c = c; p.ldc = ldc; p.c_is_f32 = c_dtype; p.atomic_add = accumulate ? 1 : 0;
  p.split_k = splits; p.alpha = alpha; p.bias = bias;
  p.residual = reinterpret_cast<const bf16*>(residual); p.ldr = ldr; p.res_row_mod = res_row_mod;
  p.res_row_idx = res_row_idx;

  cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  if (block_n == 256) return dispatch_major<256>(a_major, b_major, tmA, tmB, p, grid, s);
  return dispatch_major<128>(a_major, b_major, tmA, tmB, p, grid, s);
}
