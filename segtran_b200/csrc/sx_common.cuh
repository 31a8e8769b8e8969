// Shared device/host helpers: error plumbing, sm_90a PTX wrappers (mbarrier, TMA, wgmma).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/segtran_b200.h"

// ------------------------------------------------------------------------------------------------
// host-side error plumbing
// ------------------------------------------------------------------------------------------------
void sx_set_error(const char* fmt, ...);

#define SX_CHECK_CUDA(expr)                                                                     \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) {                                                                    \
      sx_set_error("%s:%d CUDA error %s: %s", __FILE__, __LINE__, cudaGetErrorName(_e),         \
                   cudaGetErrorString(_e));                                                     \
      return -2;                                                                                \
    }                                                                                           \
  } while (0)

#define SX_REQUIRE(cond, ...)                                                                   \
  do {                                                                                          \
    if (!(cond)) {                                                                              \
      sx_set_error(__VA_ARGS__);                                                                \
      return -1;                                                                                \
    }                                                                                           \
  } while (0)

// floor of a window weight (MONAI's): keeps cnt > 0 at window corners that only one window covers
constexpr float kSwMinWeight = 1e-3f;

static inline int sx_ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }

// SM count of the CURRENT device (cached per device ordinal: a process may drive several GPUs)
static inline int sm_count_cached() {
  static int n[64] = {0};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 0;
  if (n[dev] == 0) {
    int v = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    n[dev] = v;
  }
  return n[dev];
}


// ------------------------------------------------------------------------------------------------
// device helpers
// ------------------------------------------------------------------------------------------------
namespace sx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t.reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.b32 %0, 1, 0, P;\n\t}\n"
      : "=r"(pred));
  return pred != 0;
}

// ---- mbarrier ----
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a protocol bug must surface as a trap (error at the next sync), never as a hung GPU.
#ifndef SX_MBAR_TIMEOUT_NS
#define SX_MBAR_TIMEOUT_NS 4000000000ull
#endif
__device__ __forceinline__ uint64_t globaltimer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok = 0;
  const uint32_t addr = smem_u32(bar);
  uint64_t t0 = 0;
  while (true) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.b32 %0, 1, 0, p;\n\t}\n"
        : "=r"(ok)
        : "r"(addr), "r"(parity)
        : "memory");
    if (ok) break;
    const uint64_t now = globaltimer_ns();
    if (t0 == 0) t0 = now;
    if (now - t0 > SX_MBAR_TIMEOUT_NS) __trap();      // (no printf: a call here would serialise the wgmma pipeline)
  }
}

// ---- TMA (cp.async.bulk.tensor) ----
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// L2 eviction-priority policies for TMA loads (same encodings CUTLASS uses for TMA::CacheHintSm90)
constexpr uint64_t kEvictNormal = 0x1000000000000000ull;
constexpr uint64_t kEvictFirst = 0x12F0000000000000ull;
constexpr uint64_t kEvictLast = 0x14F0000000000000ull;
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1,
                                            int c2, int c3, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint "
      "[%0], [%1, {%3, %4, %5, %6}], [%2], %7;" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "l"(policy)
      : "memory");
}

// ---- wgmma (sm_90a warpgroup MMA: 4 warps, accumulators in registers) ----
// Shared-memory matrix descriptor: start[0,14) lbo[16,30) sbo[32,46) (all >> 4), layout_type[62,64) (1 = SWIZZLE_128B).
//   K-major SWIZZLE_128B : rows of 128 B of K, 8-row groups SBO = 1024 B apart (LBO unused);
//   MN-major SWIZZLE_128B: 128-byte spans of MN, LBO = bytes between consecutive spans, SBO = bytes between 8-row K groups.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int N>
__device__ __forceinline__ void acc_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x 128] (+)= A[64 x 8] . B[128 x 8]^T, tf32 operands (both K-major in shared memory), fp32 accumulators.
// Fragment of thread t of warp w: d[4j + 2h + e] = D[16w + 8h + t/4][8j + 2(t%4) + e].
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate));
}
// D[64 x 256] (+)= A[64 x 8] . B[256 x 8]^T: the same operand layout (B is 256 K-major rows, one contiguous SW128 operand)
// and the same fragment rule, d[4j + 2h + e] = D[16w + 8h + t/4][8j + 2(t%4) + e], with j up to 31.
__device__ __forceinline__ void wgmma_tf32_n256(float (&d)[128], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
      "%128, %129, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(accumulate));
}
// same for bf16 operands (K = 16); TA / TB = 1: that operand is MN-major in shared memory
template <int TA, int TB>
__device__ __forceinline__ void wgmma_bf16(float (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, %67, %68;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(accumulate), "n"(TA), "n"(TB));
}
// ---- numerics ----
__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// erf by Abramowitz & Stegun 7.1.26 (|abs error| <= 1.5e-7, one MUFU.RCP + one MUFU.EX2 + 7 FMA) — used in the GEMM
// epilogue where the libdevice erff (~30 instructions) made the 4/8 epilogue warps the bottleneck.
// Branch-free erf: erf(|x|) = 1 - 2^(-t q(t)), t = min(|x|, 3.93), q a degree-7 polynomial fitted (weighted minimax) to
// -log2(erfc(t))/t.  Max abs error 1.2e-7 + the ex2.approx error (<= 2 ulp of a value <= 1), i.e. <= 2.5e-7 absolute —
// three orders below the TF32 operand rounding that follows; 13 instructions, no divergence (libdevice erff takes two
// branches inside most warps).  Checked against fp64 erf in tests/test_gpu_ops.py and in tf32x3 mode end to end.
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float erf_fast(float x) {
  const float t = fminf(fabsf(x), 3.93f);
  float r = 4.5856195356464013e-05f;
  r = fmaf(r, t, -4.4942606473341584e-04f);
  r = fmaf(r, t, 1.5015227254480124e-03f);
  r = fmaf(r, t, 7.559903897345066e-04f);
  r = fmaf(r, t, -2.8238432481884956e-02f);
  r = fmaf(r, t, 1.4847517013549805e-01f);
  r = fmaf(r, t, 9.184176325798035e-01f);
  r = fmaf(r, t, 1.62790846824646f);
  const float y = 1.0f - ex2_approx(-r * t);
  return copysignf(y, x);
}
__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erf_fast(x * 0.70710678118654752f)); }
// d/dx of 0.5 x (1 + erf(x/sqrt2))
__device__ __forceinline__ float gelu_erf_grad(float x) {
  return 0.5f * (1.0f + erf_fast(x * 0.70710678118654752f)) + x * 0.3989422804014327f * __expf(-0.5f * x * x);
}
// Counter-based dropout bits: every group of 4 consecutive elements (index >> 2) owns two independent 32-bit hash words
// (word 0: elements 0,1; word 1: elements 2,3; 16 bits per element); keep(idx) <=> field(idx & 3) >= p16 with
// p16 = round(p * 65536).  Each word is one lowbias32 avalanche of the group index keyed by its own multiplier and
// seed half, so a thread that holds only two elements of a group computes only the word it needs; ~5 integer ops per
// element, cheap enough to regenerate the mask in backward instead of storing it.
__device__ __forceinline__ uint32_t drop_p16(float p) {
  const float v = p * 65536.f + 0.5f;
  return v >= 65535.f ? 65535u : (uint32_t)v;
}
__device__ __forceinline__ uint32_t drop_mul(int w) { return w ? 0x85EBCA77u : 0x9E3779B1u; }
// word key: a splitmix64 finalisation of the whole 64-bit seed offset by a per-word constant — both words depend on all
// seed bits (two seeds that differ in one 32-bit half only must not share a word's mask).  Loop-invariant in every kernel.
__device__ __forceinline__ uint32_t drop_key(unsigned long long seed, int w) {
  unsigned long long z = seed + (w ? 0x68E31DA4A0761D65ull : 0x9E3779B97F4A7C15ull);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (uint32_t)z ^ (uint32_t)(z >> 32);
}
__device__ __forceinline__ uint32_t drop_word_k(uint32_t mul, uint32_t key, unsigned long long idx4) {
  uint32_t a = ((uint32_t)idx4 * mul) ^ key;
  a ^= (uint32_t)(idx4 >> 32) * 0xC2B2AE3Du;
  a ^= a >> 16; a *= 0x7FEB352Du; a ^= a >> 15; a *= 0x846CA68Bu; a ^= a >> 16;
  return a;
}
__device__ __forceinline__ uint2 drop_hash(unsigned long long seed, unsigned long long idx4) {
  return make_uint2(drop_word_k(drop_mul(0), drop_key(seed, 0), idx4), drop_word_k(drop_mul(1), drop_key(seed, 1), idx4));
}
__device__ __forceinline__ bool drop_keep(uint2 h, int j, uint32_t p16) {
  const uint32_t w = (j & 2) ? h.y : h.x;
  return ((w >> ((j & 1) * 16)) & 0xFFFFu) >= p16;
}
// scalar form (any alignment)
__device__ __forceinline__ bool drop_keep1(unsigned long long seed, unsigned long long idx, uint32_t p16) {
  const int j = (int)(idx & 3);
  const uint32_t w = drop_word_k(drop_mul(j >> 1), drop_key(seed, j >> 1), idx >> 2);
  return ((w >> ((j & 1) * 16)) & 0xFFFFu) >= p16;
}
__device__ __forceinline__ void atomic_max_float(float* addr, float v) {
  // valid for any sign mix: order-preserving int compare
  if (v >= 0.f)
    atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
  else
    atomicMin(reinterpret_cast<unsigned int*>(addr), __float_as_uint(v));
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

}  // namespace sx
