// Shared pieces of the wgmma / TMA kernels (sx_gemm.cu, sx_attn.cu): tile constants, tensor-map construction,
// per-device caches.
#pragma once
#include <mutex>

#include "sx_common.cuh"

namespace sxtc {

constexpr int BM = 128;          // tile rows   (two consumer warpgroups x wgmma M = 64)
constexpr int BN = 128;          // tile cols   (wgmma N)
constexpr int BKB = 128;         // bytes of K per stage row (one 128B swizzle span)
constexpr int A_STAGE_BYTES = BM * BKB;       // 16 KB
constexpr int B_STAGE_BYTES = BN * BKB;       // 16 KB


typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* f = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &f, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(f);
  });
  return fn;
}


static int make_map(CUtensorMap* tm, const sx_operand& op, int es, int rows, int K, int Z0, int Z1, int box_rows,
             const char* name) {
  PFN_encodeTiled enc = get_encode();
  SX_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled not available (no CUDA driver?)");
  SX_REQUIRE((reinterpret_cast<uintptr_t>(op.ptr) & 15) == 0, "sx_gemm: operand %s not 16-byte aligned", name);
  SX_REQUIRE((op.ld * es) % 16 == 0, "sx_gemm: operand %s ld*elsize (%lld) not a multiple of 16", name,
             (long long)op.ld * es);
  const int z0 = op.stride_z0 ? Z0 : 1, z1 = op.stride_z1 ? Z1 : 1;
  SX_REQUIRE((op.stride_z0 * es) % 16 == 0 && (op.stride_z1 * es) % 16 == 0,
             "sx_gemm: operand %s batch strides not multiples of 16 bytes", name);
  const int inner = BKB / es;      // elements in a 128-byte span
  cuuint64_t gdim[4];
  cuuint64_t gstr[3];
  cuuint32_t box[4];
  cuuint32_t estr[4] = {1, 1, 1, 1};
  if (op.major == SX_MAJOR_K) {
    gdim[0] = (cuuint64_t)K; gdim[1] = (cuuint64_t)rows;
    box[0] = inner; box[1] = box_rows;
  } else {
    gdim[0] = (cuuint64_t)rows; gdim[1] = (cuuint64_t)K;
    box[0] = inner; box[1] = inner;            // BK rows of k, each 128 B of mn
  }
  gdim[2] = z0; gdim[3] = z1;
  box[2] = 1; box[3] = 1;
  gstr[0] = (cuuint64_t)op.ld * es;
  const cuuint64_t dflt = gstr[0] * gdim[1];
  gstr[1] = op.stride_z0 ? (cuuint64_t)op.stride_z0 * es : dflt;
  gstr[2] = op.stride_z1 ? (cuuint64_t)op.stride_z1 * es : (gstr[1] * gdim[2]);
  CUtensorMapDataType dt = (es == 4) ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16;
  const CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B;
  CUresult r = enc(tm, dt, 4, const_cast<void*>(op.ptr), gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SX_REQUIRE(r == CUDA_SUCCESS,
             "cuTensorMapEncodeTiled(%s) failed: %d (gdim %llu,%llu,%llu,%llu gstr %llu,%llu,%llu box %u,%u)", name,
             (int)r, (unsigned long long)gdim[0], (unsigned long long)gdim[1], (unsigned long long)gdim[2],
             (unsigned long long)gdim[3], (unsigned long long)gstr[0], (unsigned long long)gstr[1],
             (unsigned long long)gstr[2], box[0], box[1]);
  return 0;
}

// cudaFuncSetAttribute(MaxDynamicSharedMemorySize) is a per-(kernel, device) setting: done once for each pair (the
// kernels are template instantiations that share one function-pointer TYPE, so the cache is keyed by pointer VALUE)
template <typename K>
static cudaError_t set_max_smem_once(K kern, int bytes) {
  static std::mutex mu;
  static const void* seen[64 * 32];
  static int nseen = 0;
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  const void* key = reinterpret_cast<const void*>(reinterpret_cast<uintptr_t>(kern) * 64u + (uintptr_t)(dev & 63));
  std::lock_guard<std::mutex> lk(mu);
  for (int i = 0; i < nseen; ++i)
    if (seen[i] == key) return cudaSuccess;
  e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  if (e != cudaSuccess) return e;
  if (nseen < 64 * 32) seen[nseen++] = key;
  return cudaSuccess;
}

}  // namespace sxtc
