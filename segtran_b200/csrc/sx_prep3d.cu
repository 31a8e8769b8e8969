// Batch preparation of the 3-D training loop (reference train3d.py:711-715, dataloaders/datasets3d.py):
//
//   brats_map_label   out[b,k,v] = class k of label[b,v] in the BraTS n-hot map (datasets3d.py:16-40): one pass, the
//                     label read once and the K class planes written once.
//   draw_resized_crop one thread draws the RandomResizedCrop record (s_h, s_w, s_d, h_start, w_start, d_start) from a
//                     64-bit seed (datasets3d.py:611-657's torch.rand / torch.randint, same distributions).
//   resized_crop      y[b,c,o] = the crop at the record's starts of F.pad(F.interpolate(x, (int(H s_h), int(W s_w),
//                     int(D s_d)), trilinear, align_corners=False)): every output voxel gathers its 8 taps per channel
//                     straight from x (sx::src_index, the rule pinned to F.interpolate), 0 where the padding lies; the
//                     resized and padded intermediate is never stored.  The taps are computed once per voxel and shared
//                     by every channel of both operands (volume and n-hot mask).
#include <algorithm>

#include "sx_common.cuh"
#include "sx_resample.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxLen = 1 << 30;             // bound on a record's intermediate length and starts (keeps int32 math exact)

template <typename T>
__global__ void __launch_bounds__(kThreads)
brats_map_label_kernel(const T* __restrict__ label, long long V, long long n, int binarize, float* __restrict__ out) {
  const int K = binarize ? 2 : 4;
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < n; i += (long long)gridDim.x * kThreads) {
    const T v = label[i];
    const long long b = i / V, p = i - b * V;
    float* o = out + b * K * V + p;
    // the reference's comparisons in the label's own type: NaN and negative values belong to no class
    o[0] = v == T(0) ? 1.f : 0.f;
    if (binarize) {
      o[V] = v > T(0) ? 1.f : 0.f;
    } else {
      const bool et = v == T(3), ncr = v == T(1), ed = v == T(2);
      o[V] = et ? 1.f : 0.f;                              // ET = 3
      o[2 * V] = (et || ncr || ed) ? 1.f : 0.f;           // WT = 1, 2, 3
      o[3 * V] = (et || ncr) ? 1.f : 0.f;                 // TC = 1, 3
    }
  }
}

// splitmix64 of the seed and a draw index: independent 64-bit words per (seed, k)
__device__ __forceinline__ unsigned long long draw_word(unsigned long long seed, int k) {
  unsigned long long z = seed + (unsigned long long)(k + 1) * 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// the intermediate length int(L * s) in float32, as the reference computes it; NaN or s <= 0 give 0 (an empty axis)
__device__ __forceinline__ int resized_len(int L, float s) {
  const float v = __fmul_rn((float)L, s);
  if (!(v >= 1.f)) return 0;
  return v >= (float)kMaxLen ? kMaxLen : __float2int_rz(v);
}

__device__ __forceinline__ int record_start(float v) {
  return __float2int_rz(fminf(fmaxf(v, -(float)kMaxLen), (float)kMaxLen));   // NaN -> 0
}

__global__ void draw_resized_crop_kernel(const unsigned long long* seed_dev, unsigned long long seed, int3 in, int3 out,
                                         float smin, float smax, int isotropic, float* rec) {
  const unsigned long long sd = seed_dev ? seed_dev[0] : seed;
  float s[3];
  for (int a = 0; a < 3; ++a) {
    if (a > 0 && isotropic) {
      s[a] = s[0];
      continue;
    }
    // u uniform on [0, 1) in steps of 2^-24 (torch.rand's float32 resolution); s = u (max - min) + min, kept below max
    const float u = (float)(draw_word(sd, a) >> 40) * 5.9604644775390625e-8f;
    float v = __fadd_rn(__fmul_rn(u, __fsub_rn(smax, smin)), smin);
    if (v >= smax && smax > smin) v = nextafterf(smax, smin);
    s[a] = v;
  }
  const int L[3] = {in.x, in.y, in.z}, O[3] = {out.x, out.y, out.z};
  for (int a = 0; a < 3; ++a) {
    const int padded = max(resized_len(L[a], s[a]), O[a]);
    // start uniform on [0, padded - out]: the high half of a 64-bit word scaled to the count of starts
    const unsigned long long cnt = (unsigned long long)(padded - O[a] + 1);
    const unsigned long long w = draw_word(sd, 3 + a) >> 32;
    rec[a] = s[a];
    rec[3 + a] = (float)((w * cnt) >> 32);
  }
}

// one axis of an output voxel: the taps into x, or false where the cell lies in the padding / outside the intermediate
__device__ __forceinline__ bool axis_taps(int o, int L, float s, float start, int O, int& i0, int& i1, float& w1) {
  const int R = resized_len(L, s);
  const int r = o + record_start(start) - max(O - R, 0) / 2;       // cell of the resized (unpadded) intermediate
  if (r < 0 || r >= R) return false;
  sx::src_index(r, __fdiv_rn((float)L, (float)R), L, i0, i1, w1);  // F.interpolate's scale: (float)in / out
  return true;
}

// one operand's channels at one output voxel: the taps were computed once for both operands
__device__ __forceinline__ void crop_channels(const sx_crop_operand& p, int b, long long V, long long o, bool inside,
                                              int h0, int h1, float wh, int w0, int w1, float ww, int d0, int d1,
                                              float wd) {
  float* y = p.y + (long long)b * p.C * V + o;
  if (!inside) {
    for (int c = 0; c < p.C; ++c) y[c * V] = 0.f;
    return;
  }
  const long long sh = p.stride[2], sw = p.stride[3], sd = p.stride[4];
  const long long e00 = h0 * sh + w0 * sw, e01 = h0 * sh + w1 * sw, e10 = h1 * sh + w0 * sw, e11 = h1 * sh + w1 * sw;
  const long long f0 = d0 * sd, f1 = d1 * sd;
  const float* x = p.x + (long long)b * p.stride[0];
  for (int c = 0; c < p.C; ++c, x += p.stride[1]) {
    // PyTorch's nesting (upsample_trilinear3d): h0 * (w0 (d0 x000 + d1 x001) + w1 (...)) + h1 * (...)
    const float p00 = (1.f - wd) * __ldg(x + e00 + f0) + wd * __ldg(x + e00 + f1);
    const float p01 = (1.f - wd) * __ldg(x + e01 + f0) + wd * __ldg(x + e01 + f1);
    const float p10 = (1.f - wd) * __ldg(x + e10 + f0) + wd * __ldg(x + e10 + f1);
    const float p11 = (1.f - wd) * __ldg(x + e11 + f0) + wd * __ldg(x + e11 + f1);
    y[c * V] = (1.f - wh) * ((1.f - ww) * p00 + ww * p01) + wh * ((1.f - ww) * p10 + ww * p11);
  }
}

__global__ void __launch_bounds__(kThreads)
resized_crop_kernel(const sx_crop_operand a, const sx_crop_operand b2, int nops, int3 in, int3 out,
                    const float* __restrict__ rec, int n) {
  const int idx = blockIdx.x * kThreads + threadIdx.x;
  if (idx >= n) return;
  const int od = idx % out.z;
  int t = idx / out.z;
  const int ow = t % out.y;
  t /= out.y;
  const int oh = t % out.x;
  const int b = t / out.x;
  int h0 = 0, h1 = 0, w0 = 0, w1 = 0, d0 = 0, d1 = 0;
  float wh = 0.f, ww = 0.f, wd = 0.f;
  const bool inside = axis_taps(oh, in.x, __ldg(rec + 0), __ldg(rec + 3), out.x, h0, h1, wh) &&
                      axis_taps(ow, in.y, __ldg(rec + 1), __ldg(rec + 4), out.y, w0, w1, ww) &&
                      axis_taps(od, in.z, __ldg(rec + 2), __ldg(rec + 5), out.z, d0, d1, wd);
  const long long V = (long long)out.x * out.y * out.z, o = ((long long)oh * out.y + ow) * out.z + od;
  crop_channels(a, b, V, o, inside, h0, h1, wh, w0, w1, ww, d0, d1, wd);
  if (nops > 1) crop_channels(b2, b, V, o, inside, h0, h1, wh, w0, w1, ww, d0, d1, wd);
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int sx_brats_map_label(const void* label, int32_t dtype, int32_t B, int64_t V, int32_t binarize, float* out,
                                  void* stream) {
  SX_REQUIRE(B >= 1 && V >= 1, "sx_brats_map_label: empty label map (B=%d V=%lld)", B, (long long)V);
  const long long n = (long long)B * V;
  const int grid = (int)std::max<long long>(
      1, std::min<long long>((n + kThreads - 1) / kThreads, (long long)sm_count_cached() * 16));
  const int bin = binarize ? 1 : 0;
  switch (dtype) {
    case SX_LABEL_U8: brats_map_label_kernel<<<grid, kThreads, 0, ST(stream)>>>((const uint8_t*)label, V, n, bin, out); break;
    case SX_LABEL_I16: brats_map_label_kernel<<<grid, kThreads, 0, ST(stream)>>>((const int16_t*)label, V, n, bin, out); break;
    case SX_LABEL_I32: brats_map_label_kernel<<<grid, kThreads, 0, ST(stream)>>>((const int32_t*)label, V, n, bin, out); break;
    case SX_LABEL_I64: brats_map_label_kernel<<<grid, kThreads, 0, ST(stream)>>>((const int64_t*)label, V, n, bin, out); break;
    case SX_LABEL_F32: brats_map_label_kernel<<<grid, kThreads, 0, ST(stream)>>>((const float*)label, V, n, bin, out); break;
    default: SX_REQUIRE(false, "sx_brats_map_label: unknown label type %d", dtype);
  }
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_draw_resized_crop(const uint64_t* seed_dev, uint64_t seed, int32_t H, int32_t W, int32_t D, int32_t oh,
                                    int32_t ow, int32_t od, float min_scale, float max_scale, int32_t isotropic, float* rec,
                                    void* stream) {
  SX_REQUIRE(H >= 1 && W >= 1 && D >= 1 && oh >= 1 && ow >= 1 && od >= 1 && H < kMaxLen && W < kMaxLen && D < kMaxLen &&
                 oh < kMaxLen && ow < kMaxLen && od < kMaxLen,
             "sx_draw_resized_crop: bad sizes (%d,%d,%d) -> (%d,%d,%d)", H, W, D, oh, ow, od);
  SX_REQUIRE(min_scale > 0.f && max_scale >= min_scale && max_scale <= 3.0e38f,
             "sx_draw_resized_crop: bad scale range [%g, %g)", (double)min_scale, (double)max_scale);
  draw_resized_crop_kernel<<<1, 1, 0, ST(stream)>>>((const unsigned long long*)seed_dev, seed, make_int3(H, W, D),
                                                     make_int3(oh, ow, od), min_scale, max_scale, isotropic, rec);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static int check_operand(const sx_crop_operand* p, const char* what) {
  SX_REQUIRE(p->x != nullptr && p->y != nullptr && p->C >= 1, "sx_resized_crop: %s operand is empty", what);
  return 0;
}

extern "C" int sx_resized_crop(const sx_crop_operand* a, const sx_crop_operand* b, int32_t B, int32_t H, int32_t W,
                               int32_t D, int32_t oh, int32_t ow, int32_t od, const float* rec, void* stream) {
  SX_REQUIRE(a != nullptr && rec != nullptr, "sx_resized_crop: NULL operand or record");
  if (int rc = check_operand(a, "first")) return rc;
  if (b)
    if (int rc = check_operand(b, "second")) return rc;
  SX_REQUIRE(B >= 1 && H >= 1 && W >= 1 && D >= 1 && oh >= 1 && ow >= 1 && od >= 1,
             "sx_resized_crop: bad sizes B=%d (%d,%d,%d) -> (%d,%d,%d)", B, H, W, D, oh, ow, od);
  SX_REQUIRE(H < kMaxLen && W < kMaxLen && D < kMaxLen, "sx_resized_crop: input too large");
  const long long n = (long long)B * oh * ow * od;
  SX_REQUIRE(n < (1ll << 31), "sx_resized_crop: %lld output voxels", n);
  resized_crop_kernel<<<(unsigned)((n + kThreads - 1) / kThreads), kThreads, 0, ST(stream)>>>(
      *a, b ? *b : *a, b ? 2 : 1, make_int3(H, W, D), make_int3(oh, ow, od), rec, (int)n);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
