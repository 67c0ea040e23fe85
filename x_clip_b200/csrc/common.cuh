// Device-side primitives for the sm_90a kernels of x_clip_b200: mbarrier, TMA
// (cp.async.bulk.tensor), wgmma (warpgroup MMA from shared-memory descriptors) and the descriptor
// builder.
//
// Everything here is inline PTX; nothing depends on CUTLASS/CuTe.  The shared-memory matrix
// descriptor follows the PTX ISA "wgmma" chapter (the fields CuTe names in
// cute/arch/mma_sm90_desc.hpp: start_address[0,14) LBO[16,30) SBO[32,46) base_offset[49,52)
// layout_type[62,64), 1 = SWIZZLE_128B).
#pragma once

#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <float.h>
#include <stdio.h>

namespace xclip {

typedef __nv_bfloat16 bf16;

constexpr int kMajorK = 0;   // operand stored with the contraction index contiguous
constexpr int kMajorMN = 1;  // operand stored with its M (or N) index contiguous

// ---------------------------------------------------------------------------
// small helpers
// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint32_t lane_id() { return threadIdx.x & 31; }

// Single-thread regions that issue TMA instructions are entered through elect.sync: with
// `lane == 0` ptxas cannot prove that one thread is active and wraps every issue in a loop.
#define XCLIP_ONE_LANE(lane) (::xclip::elect_one())

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

__device__ __forceinline__ float2 unpack_bf16x2(uint32_t u) {
  __nv_bfloat162 v = *reinterpret_cast<__nv_bfloat162*>(&u);
  return __bfloat1622float2(v);
}

// ---------------------------------------------------------------------------
// mbarrier
// ---------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)
               : "memory");
}

__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}

// make generic-proxy writes to shared memory visible to the async proxy (TMA, wgmma)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}

__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(done)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return done != 0;
}

// Bounded wait: a protocol bug turns into a trap (launch failure the host reports)
// instead of a hung GPU.  ~4 s at 2 GHz.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000ll) {
      printf("xclip: mbarrier timeout block=(%d,%d) thread=%d bar=%u parity=%u\n", blockIdx.x,
             blockIdx.y, threadIdx.x, smem_u32(bar), parity);
      __trap();
    }
  }
}

// The same bound without the diagnostic printf, for kernels that issue wgmma: a function call
// (printf) anywhere in such a kernel makes ptxas serialise the wgmma pipeline.
__device__ __forceinline__ void mbar_wait_nocall(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > 8000000000ll) __trap();
  }
}

// ---------------------------------------------------------------------------
// TMA
// ---------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// pull a tensor box towards L2 (no shared memory, no barrier): the later tma_load of the same box
// then sees L2 instead of HBM latency
__device__ __forceinline__ void tma_prefetch_l2_3d(const CUtensorMap* m, int32_t c0, int32_t c1, int32_t c2) {
  asm volatile("cp.async.bulk.prefetch.tensor.3d.L2.global [%0, {%1, %2, %3}];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}

__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int32_t c0, int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// ---------------------------------------------------------------------------
// descriptors
// ---------------------------------------------------------------------------
// Shared-memory matrix descriptor (wgmma) for a SWIZZLE_128B tile whose base is 1024 B aligned.
//   K-major  : rows (M/N index) of 128 B (64 bf16 along K); 8-row groups SBO apart
//              (1024 B when the tile is dense); LBO unused.
//   MN-major : rows (K index) of 128 B (64 bf16 along M/N); 8-row K-groups SBO apart
//              (1024 B); 64-element M/N groups LBO apart.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr, uint32_t lbo_bytes,
                                                   uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;  // SWIZZLE_128B
  return d;
}

// advance a descriptor's start address by `bytes` (must keep the 1024 B swizzle phase)
__device__ __forceinline__ uint64_t desc_advance(uint64_t desc, uint32_t bytes) {
  return desc + static_cast<uint64_t>(bytes >> 4);
}

// ---------------------------------------------------------------------------
// wgmma: D[64 x N] (fp32, registers of one warpgroup) += A[smem] * B[smem], bf16 inputs.
// kTransA / kTransB = 1 when the operand is MN-major.  Fragment layout of D (thread t of the
// warpgroup, w = t / 32, l = t % 32): d[j] sits at row 16 w + l / 4 + 8 ((j / 2) % 2),
// column 8 (j / 4) + 2 (l % 4) + (j % 2).
// ---------------------------------------------------------------------------
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

template <int kTransA, int kTransB>
__device__ __forceinline__ void wgmma_m64n64k16(float (&d)[32], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %34, %35;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "n"(kTransA), "n"(kTransB));
}

template <int kTransA, int kTransB>
__device__ __forceinline__ void wgmma_m64n128k16(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %66, %67;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "n"(kTransA), "n"(kTransB));
}

__device__ __forceinline__ void named_bar_sync(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// byte offset of 16 B chunk `c16` of 128 B row `row` inside a SWIZZLE_128B tile
// (Swizzle<3,4,3>: chunk index XOR row%8); tile base must be 1024 B aligned.
__device__ __forceinline__ uint32_t swz128(uint32_t row, uint32_t c16) {
  return row * 128u + ((c16 ^ (row & 7u)) << 4);
}

// ---------------------------------------------------------------------------
// GELU (erf form, x_clip/x_clip.py:183 F.gelu) shared by the row-wise kernels and the fused
// feed-forward GEMM epilogues
// ---------------------------------------------------------------------------
// erf by Abramowitz & Stegun 7.1.26 (|error| <= 1.5e-7, far below bf16 output resolution):
// one MUFU.RCP + one MUFU.EX2 + 6 FMA instead of libdevice erff's ~25 instructions.  The GEGLU
// kernels would otherwise be instruction-bound, not HBM-bound.  exp(-x^2/2) is shared with the
// Gaussian density that gelu'(x) needs.
struct GeluParts {
  float cdf;   // Phi(x) = 0.5 * (1 + erf(x / sqrt(2)))
  float pdf;   // phi(x) = exp(-x^2/2) / sqrt(2 pi)
};
__device__ __forceinline__ GeluParts gelu_parts(float x) {
  const float z = fabsf(x) * 0.70710678118654752f;            // |x| / sqrt(2)
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.f)));
  float poly = fmaf(1.061405429f, t, -1.453152027f);
  poly = fmaf(poly, t, 1.421413741f);
  poly = fmaf(poly, t, -0.284496736f);
  poly = fmaf(poly, t, 0.254829592f);
  poly *= t;
  float e_half;                                                // exp(-x^2/2) == exp(-z^2)
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e_half) : "f"(-0.72134752044448170f * x * x));
  const float erfc_z = poly * e_half;
  const float half_erfc = 0.5f * erfc_z;
  GeluParts g;
  g.cdf = x >= 0.f ? 1.f - half_erfc : half_erfc;
  g.pdf = 0.3989422804014327f * e_half;
  return g;
}
__device__ __forceinline__ float gelu_erf(float x) { return x * gelu_parts(x).cdf; }

// ---------------------------------------------------------------------------
// fp32 pairs: the GELU epilogues of the fused feed-forward handle two adjacent columns at a time
// (two independent dependency chains per thread).
// ---------------------------------------------------------------------------
struct f32x2 {
  float x, y;
};
__device__ __forceinline__ f32x2 f2_pack(float lo, float hi) { return f32x2{lo, hi}; }
__device__ __forceinline__ f32x2 f2_splat(float v) { return f32x2{v, v}; }
__device__ __forceinline__ void f2_unpack(f32x2 v, float& lo, float& hi) { lo = v.x; hi = v.y; }
__device__ __forceinline__ f32x2 f2_fma(f32x2 a, f32x2 b, f32x2 c) {
  return f32x2{fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)};
}
__device__ __forceinline__ f32x2 f2_mul(f32x2 a, f32x2 b) { return f32x2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ f32x2 f2_add(f32x2 a, f32x2 b) { return f32x2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
// two consecutive bf16 of one 32-bit word -> fp32 pair (element 0 in the low half)
__device__ __forceinline__ f32x2 f2_from_bf16x2(uint32_t w) {
  return f2_pack(__uint_as_float(w << 16), __uint_as_float(w & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_to_bf16x2(f32x2 v) { return pack_bf16x2(v.x, v.y); }

// gelu_parts for two elements at once: cdf = Phi(x), pdf = phi(x) (same A&S 7.1.26 polynomial).
struct GeluParts2 {
  f32x2 cdf, pdf;
};
__device__ __forceinline__ GeluParts2 gelu_parts2(float x0, float x1) {
  const f32x2 x = f2_pack(x0, x1);
  const f32x2 z = f2_mul(f2_pack(fabsf(x0), fabsf(x1)), f2_splat(0.70710678118654752f));
  float d0, d1, t0, t1;
  f2_unpack(f2_fma(f2_splat(0.3275911f), z, f2_splat(1.f)), d0, d1);
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t0) : "f"(d0));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t1) : "f"(d1));
  const f32x2 t = f2_pack(t0, t1);
  f32x2 poly = f2_fma(f2_splat(1.061405429f), t, f2_splat(-1.453152027f));
  poly = f2_fma(poly, t, f2_splat(1.421413741f));
  poly = f2_fma(poly, t, f2_splat(-0.284496736f));
  poly = f2_fma(poly, t, f2_splat(0.254829592f));
  poly = f2_mul(poly, t);
  float a0, a1, e0, e1;
  f2_unpack(f2_mul(f2_mul(x, f2_splat(-0.72134752044448170f)), x), a0, a1);     // -x^2/2 * log2(e)
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e0) : "f"(a0));
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e1) : "f"(a1));
  const f32x2 e_half = f2_pack(e0, e1);
  // q = 0.5 - 0.5 erfc(|x|/sqrt2) >= 0;  Phi(x) = 0.5 + sign(x) q
  float q0, q1;
  f2_unpack(f2_fma(f2_mul(poly, e_half), f2_splat(-0.5f), f2_splat(0.5f)), q0, q1);
  q0 = __uint_as_float(__float_as_uint(q0) | (__float_as_uint(x0) & 0x80000000u));
  q1 = __uint_as_float(__float_as_uint(q1) | (__float_as_uint(x1) & 0x80000000u));
  GeluParts2 g;
  g.cdf = f2_add(f2_pack(q0, q1), f2_splat(0.5f));
  g.pdf = f2_mul(e_half, f2_splat(0.3989422804014327f));
  return g;
}


}  // namespace xclip
