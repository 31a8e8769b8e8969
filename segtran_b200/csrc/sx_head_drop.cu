// Out-FPN dropout head (--outdrop, segtran3d.py:392-396, :488-490; segtran2d.py:308-311, :427): the class scores of
// the dropped, depth-upsampled feature map without that map ever reaching memory.
//
//   Ls[b,k,v'] = bc[k] + sum_f Wc[k,f] keep(b,f,v') X[b,f,v'] / (1-p)          v' = (d', hw) on [D', H1*W1]
//
// X [B,F',D',HW] is formed on the fly from the source map Y (element (b, fs, i, hw)) by the depth map:
//   SX_HEAD_DMAP_NONE   X = Y                                   (F' = Fs, D' = Ds; the 2-D head passes Ds = 1)
//   SX_HEAD_DMAP_INTERP X = linear(Y) along depth, D' = Dk Ds  (F.interpolate, align_corners=False: sx::src_index)
//   SX_HEAD_DMAP_UNFOLD X[f, j Ds + i] = Y[f Dk + j, i]        (the reshape after out_fpn_upsampleD, F' = Fs / Dk)
//   SX_HEAD_DMAP_UNFOLD_INTERLEAVED X[f, i Dk + j] = Y[f Dk + j, i]   (the 2.5-D model's reshape, segtran25d.py:357-362)
// Y is depth-major [B,Fs,Ds,HW] (3-D and 2-D heads) or slice-major [B,Ds,Fs,HW] (the 2.5-D head, whose maps are
// [B*Ds, Fs, H1, W1]); the layout is the template parameter SLICE, so the depth-major instantiations keep their
// addressing: a source channel's base is src_chan() and its depth slices are `sD` floats apart.
// keep() is sx::drop_keep1 at the flat index of the element in [B,F',D',HW], so the mask is the one a dropout over the
// materialised map with the same counter-based hash would draw.
//
// Backward (gather form, no float atomics): one thread per (b, source depth slice i, hw) walks the source channels; for
// each it sums the d' its slice feeds with their interpolation weights, keep(.) (sum_k Wc[k,f] dLs[k,d']) / (1-p).
// dWc[k,f] = sum keep dLs X / (1-p) is counted by the source slice that is the d' element's first tap; per-warp sums per
// (k, f) live in shared memory, each CTA writes its slot of `part`, and a second kernel adds the slots in slot order.
#include <algorithm>

#include "sx_common.cuh"
#include "sx_part.cuh"
#include "sx_resample.cuh"

namespace {

constexpr int KC = 4;             // classes per launch (the entry points loop over class chunks)
constexpr int THREADS = 128;
constexpr int WARPS = THREADS / 32;

struct DropGeom {
  const float* src;
  int Fs, Ds, Fo, Do, Dk, dmap;
  long long HW;
  float p, scale;
  uint32_t p16;
  unsigned long long seed;
  const unsigned long long* seed_dev;
};

// offset of element (b, fs, 0, 0) of the source, and the distance between its depth slices
template <int SLICE>
__device__ __forceinline__ long long src_chan(const DropGeom& g, int b, int fs) {
  if constexpr (SLICE) return ((long long)b * g.Ds * g.Fs + fs) * g.HW;
  return ((long long)b * g.Fs + fs) * g.Ds * g.HW;
}
template <int SLICE>
__device__ __forceinline__ long long src_dstride(const DropGeom& g) {
  if constexpr (SLICE) return (long long)g.Fs * g.HW;
  return g.HW;
}

__device__ __forceinline__ bool is_unfold(int dmap) {
  return dmap == SX_HEAD_DMAP_UNFOLD || dmap == SX_HEAD_DMAP_UNFOLD_INTERLEAVED;
}

// one thread: VEC consecutive hw of one output depth plane; all classes of the chunk
template <int VEC, int SLICE>
__global__ void __launch_bounds__(THREADS)
head_dropout_fwd_kernel(DropGeom g, const float* __restrict__ Wc, const float* __restrict__ bc, int kc,
                        float* __restrict__ Ls, long long ls_bstride) {
  extern __shared__ float sW[];                       // [kc][Fo]
  for (int i = threadIdx.x; i < kc * g.Fo; i += blockDim.x) sW[i] = Wc[i];
  __syncthreads();
  const unsigned long long seed = g.seed + (g.seed_dev ? *g.seed_dev : 0ull);
  const int b = blockIdx.y;
  const long long Vo = (long long)g.Do * g.HW;
  const long long v0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * VEC;
  if (v0 >= Vo) return;
  const int d = (int)(v0 / g.HW);
  const long long hw = v0 - (long long)d * g.HW;
  float acc[KC][VEC];
#pragma unroll
  for (int k = 0; k < KC; ++k)
#pragma unroll
    for (int v = 0; v < VEC; ++v) acc[k][v] = 0.f;
  // source addressing of this depth plane: two taps (interp), one slice (none / unfold)
  int i0 = d, i1 = d, jj = 0;
  float w1 = 0.f;
  if (g.dmap == SX_HEAD_DMAP_INTERP) sx::src_index(d, (float)g.Ds / (float)g.Do, g.Ds, i0, i1, w1);
  if (g.dmap == SX_HEAD_DMAP_UNFOLD) { jj = d / g.Ds; i0 = i1 = d - jj * g.Ds; }
  if (g.dmap == SX_HEAD_DMAP_UNFOLD_INTERLEAVED) { i0 = i1 = d / g.Dk; jj = d - i0 * g.Dk; }
  const bool unfold = is_unfold(g.dmap);
  const long long sD = src_dstride<SLICE>(g);
  const float w0 = 1.f - w1;
  for (int f = 0; f < g.Fo; ++f) {
    const int fs = unfold ? f * g.Dk + jj : f;
    const float* s = g.src + src_chan<SLICE>(g, b, fs) + hw;
    float x[VEC];
    if constexpr (VEC == 4) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(s + (long long)i0 * sD));
      x[0] = a.x; x[1] = a.y; x[2] = a.z; x[3] = a.w;
      if (g.dmap == SX_HEAD_DMAP_INTERP) {
        const float4 c = __ldg(reinterpret_cast<const float4*>(s + (long long)i1 * sD));
        x[0] = w0 * a.x + w1 * c.x; x[1] = w0 * a.y + w1 * c.y; x[2] = w0 * a.z + w1 * c.z; x[3] = w0 * a.w + w1 * c.w;
      }
    } else {
      x[0] = __ldg(s + (long long)i0 * sD);
      if (g.dmap == SX_HEAD_DMAP_INTERP) x[0] = w0 * x[0] + w1 * __ldg(s + (long long)i1 * sD);
    }
    const unsigned long long base = (((unsigned long long)b * g.Fo + f) * g.Do + d) * (unsigned long long)g.HW + hw;
#pragma unroll
    for (int v = 0; v < VEC; ++v) x[v] = sx::drop_keep1(seed, base + v, g.p16) ? x[v] * g.scale : 0.f;
#pragma unroll
    for (int k = 0; k < KC; ++k)
      if (k < kc) {
        const float w = sW[k * g.Fo + f];
#pragma unroll
        for (int v = 0; v < VEC; ++v) acc[k][v] = fmaf(w, x[v], acc[k][v]);
      }
  }
#pragma unroll
  for (int k = 0; k < KC; ++k)
    if (k < kc) {
      float* dst = Ls + (long long)b * ls_bstride + (long long)k * Vo + v0;
      const float bk = bc ? bc[k] : 0.f;
#pragma unroll
      for (int v = 0; v < VEC; ++v) dst[v] = acc[k][v] + bk;
    }
}

// one thread: VEC consecutive hw of one source depth slice i of batch b; walks every source channel.
// Candidates t: the output planes d'_t that read slice i (interp: nonzero tap weight; unfold: d' = t Ds + i, interleaved
// unfold: d' = i Dk + t, only the candidate t = fs % Dk is live for source channel fs; none: d' = i).
template <int VEC, int TMAX, int SLICE>
__global__ void __launch_bounds__(THREADS)
head_dropout_bwd_kernel(DropGeom g, const float* __restrict__ Wc, int kc, const float* __restrict__ dLs,
                        long long dl_bstride, float* __restrict__ dsrc, int accumulate, float* __restrict__ part,
                        long long tiles_per_slice, long long tiles) {
  extern __shared__ float smem[];
  float* sW = smem;                                   // [kc][Fo]
  float* sP = smem + kc * g.Fo;                       // [WARPS][kc][Fo]: this warp's dWc partial sums
  for (int i = threadIdx.x; i < kc * g.Fo; i += blockDim.x) sW[i] = Wc[i];
  for (int i = threadIdx.x; i < WARPS * kc * g.Fo; i += blockDim.x) sP[i] = 0.f;
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* myP = sP + warp * kc * g.Fo;
  const unsigned long long seed = g.seed + (g.seed_dev ? *g.seed_dev : 0ull);
  const long long Vo = (long long)g.Do * g.HW;
  const float ratio = (float)g.Ds / (float)g.Do;

  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const long long bi = tile / tiles_per_slice;      // (b, i)
    const int b = (int)(bi / g.Ds), i = (int)(bi - (long long)b * g.Ds);
    const long long hw = ((tile - bi * tiles_per_slice) * THREADS + threadIdx.x) * VEC;
    const bool live = hw < g.HW;
    // candidate planes
    int dc[TMAX], own[TMAX], oth[TMAX];
    float wt[TMAX], wo0[TMAX], wo1[TMAX];
#pragma unroll
    for (int t = 0; t < TMAX; ++t) { dc[t] = i; own[t] = 0; oth[t] = i; wt[t] = 0.f; wo0[t] = 1.f; wo1[t] = 0.f; }
    int nt = 0;
    if (g.dmap == SX_HEAD_DMAP_INTERP) {
      int jlo, jhi;
      sx::src_readers(i, (float)g.Do / (float)g.Ds, g.Ds, g.Do, jlo, jhi);
      for (int j = jlo; j <= jhi; ++j) {
        int a0, a1;
        float w1;
        sx::src_index(j, ratio, g.Ds, a0, a1, w1);
        float w = 0.f;
        if (a0 == i) w += 1.f - w1;
        if (a1 == i) w += w1;
        if (w != 0.f || a0 == i) {
#pragma unroll
          for (int t = 0; t < TMAX; ++t)
            if (t == nt) { dc[t] = j; wt[t] = w; own[t] = (a0 == i); oth[t] = a1; wo0[t] = 1.f - w1; wo1[t] = w1; }
          ++nt;
        }
      }
    } else {
      nt = is_unfold(g.dmap) ? g.Dk : 1;
#pragma unroll
      for (int t = 0; t < TMAX; ++t) {
        dc[t] = g.dmap == SX_HEAD_DMAP_UNFOLD ? t * g.Ds + i : (g.dmap == SX_HEAD_DMAP_UNFOLD_INTERLEAVED ? i * g.Dk + t : i);
        wt[t] = 1.f; own[t] = 1; oth[t] = i; wo0[t] = 1.f; wo1[t] = 0.f;
      }
    }
    float gv[TMAX][KC][VEC];
#pragma unroll
    for (int t = 0; t < TMAX; ++t)
#pragma unroll
      for (int k = 0; k < KC; ++k)
#pragma unroll
        for (int v = 0; v < VEC; ++v)
          gv[t][k][v] = (live && t < nt && k < kc)
                            ? __ldg(dLs + (long long)b * dl_bstride + (long long)k * Vo + (long long)dc[t] * g.HW + hw + v)
                            : 0.f;

    const bool unfold = is_unfold(g.dmap);
    const long long sD = src_dstride<SLICE>(g);
    for (int fs = 0; fs < g.Fs; ++fs) {
      const int f = unfold ? fs / g.Dk : fs;
      const int tsel = unfold ? fs - f * g.Dk : -1;
      const long long chan = src_chan<SLICE>(g, b, fs);
      const float* s = g.src + chan + hw;
      float y[VEC], dy[VEC], cw[KC];
#pragma unroll
      for (int v = 0; v < VEC; ++v) {
        y[v] = live ? __ldg(s + (long long)i * sD + v) : 0.f;
        dy[v] = 0.f;
      }
#pragma unroll
      for (int k = 0; k < KC; ++k) cw[k] = 0.f;
#pragma unroll
      for (int t = 0; t < TMAX; ++t) {
        if (t >= nt || (tsel >= 0 && t != tsel)) continue;
        const unsigned long long base = (((unsigned long long)b * g.Fo + f) * g.Do + dc[t]) * (unsigned long long)g.HW + hw;
        float xo[VEC];
#pragma unroll
        for (int v = 0; v < VEC; ++v) xo[v] = y[v];
        if (own[t] && g.dmap == SX_HEAD_DMAP_INTERP) {
#pragma unroll
          for (int v = 0; v < VEC; ++v)
            xo[v] = wo0[t] * y[v] + wo1[t] * (live ? __ldg(s + (long long)oth[t] * sD + v) : 0.f);
        }
#pragma unroll
        for (int v = 0; v < VEC; ++v) {
          const float m = (live && sx::drop_keep1(seed, base + v, g.p16)) ? g.scale : 0.f;
          float sk = 0.f;
#pragma unroll
          for (int k = 0; k < KC; ++k)
            if (k < kc) sk = fmaf(sW[k * g.Fo + f], gv[t][k][v], sk);
          dy[v] = fmaf(wt[t] * m, sk, dy[v]);
          if (own[t]) {
            const float mx = m * xo[v];
#pragma unroll
            for (int k = 0; k < KC; ++k) cw[k] = fmaf(gv[t][k][v], mx, cw[k]);
          }
        }
      }
      if (live) {
        float* d = dsrc + chan + (long long)i * sD + hw;
#pragma unroll
        for (int v = 0; v < VEC; ++v) d[v] = accumulate ? d[v] + dy[v] : dy[v];
      }
#pragma unroll
      for (int k = 0; k < KC; ++k)
        if (k < kc) {
          const float sum = sx::warp_sum(cw[k]);
          if (lane == 0) myP[k * g.Fo + f] += sum;
        }
    }
  }
  __syncthreads();
  float* slot = part + (long long)blockIdx.x * kc * g.Fo;
  for (int e = threadIdx.x; e < kc * g.Fo; e += blockDim.x) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < WARPS; ++w) s += sP[w * kc * g.Fo + e];
    slot[e] = s;
  }
}

int check_args(const sx_head_dropout_args* a, const char* who) {
  SX_REQUIRE(a != nullptr && a->src && a->Wc, "%s: null pointer", who);
  SX_REQUIRE(a->B >= 1 && a->B <= 65535 && a->Fs >= 1 && a->Ds >= 1 && a->HW >= 1 && a->K >= 1 && a->Dk >= 1,
             "%s: bad shape", who);
  SX_REQUIRE(a->dmap == SX_HEAD_DMAP_NONE || a->dmap == SX_HEAD_DMAP_INTERP || a->dmap == SX_HEAD_DMAP_UNFOLD ||
                 a->dmap == SX_HEAD_DMAP_UNFOLD_INTERLEAVED,
             "%s: unknown depth map %d", who, a->dmap);
  SX_REQUIRE(a->src_layout == SX_HEAD_SRC_DEPTH_MAJOR || a->src_layout == SX_HEAD_SRC_SLICE_MAJOR,
             "%s: unknown source layout %d", who, a->src_layout);
  const bool unfold = a->dmap == SX_HEAD_DMAP_UNFOLD || a->dmap == SX_HEAD_DMAP_UNFOLD_INTERLEAVED;
  SX_REQUIRE(!unfold || (a->Fs % a->Dk == 0 && a->Fo == a->Fs / a->Dk), "%s: unfold needs Fs = F' * D_pool_K", who);
  SX_REQUIRE(unfold || a->Fo == a->Fs, "%s: F' must equal the source channels", who);
  SX_REQUIRE(!unfold || a->Dk <= 8, "%s: unfold supports D_pool_K <= 8", who);
  SX_REQUIRE(a->dmap != SX_HEAD_DMAP_INTERP || a->Dk <= 4, "%s: interp supports D_pool_K <= 4", who);
  SX_REQUIRE(a->p >= 0.f && a->p < 1.f, "%s: dropout probability %g not in [0, 1)", who, (double)a->p);
  SX_REQUIRE((size_t)5 * KC * a->Fo * 4 <= 200 * 1024, "%s: F'=%d too large", who, a->Fo);
  return 0;
}

DropGeom make_geom(const sx_head_dropout_args* a) {
  DropGeom g{};
  g.src = a->src; g.Fs = a->Fs; g.Ds = a->Ds; g.Fo = a->Fo; g.Dk = a->Dk; g.dmap = a->dmap; g.HW = a->HW;
  g.Do = a->dmap == SX_HEAD_DMAP_NONE ? a->Ds : a->Ds * a->Dk;
  g.p = a->p;
  g.scale = 1.f / (1.f - a->p);
  const float v = a->p * 65536.f + 0.5f;                     // sx::drop_p16 on the host
  g.p16 = v >= 65535.f ? 65535u : (uint32_t)v;
  g.seed = a->seed;
  g.seed_dev = reinterpret_cast<const unsigned long long*>(a->seed_dev);
  return g;
}

template <typename Kern>
cudaError_t allow_smem(Kern k, size_t bytes) {
  if (bytes <= 48 * 1024) return cudaSuccess;
  return cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)

template <int VEC, int SLICE>
static int launch_fwd(const DropGeom& g, const float* W, const float* bc, int kc, float* out, int K, int B, size_t smem,
                      cudaStream_t st) {
  const long long Vo = (long long)g.Do * g.HW;
  SX_CHECK_CUDA(allow_smem(head_dropout_fwd_kernel<VEC, SLICE>, smem));
  dim3 grid(sx_ceil_div(Vo, THREADS * VEC), B);
  head_dropout_fwd_kernel<VEC, SLICE><<<grid, THREADS, smem, st>>>(g, W, bc, kc, out, (long long)K * Vo);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_head_dropout_fwd(const sx_head_dropout_args* a, float* Ls, void* stream) {
  if (int rc = check_args(a, "sx_head_dropout_fwd")) return rc;
  SX_REQUIRE(Ls, "sx_head_dropout_fwd: null output");
  const DropGeom g = make_geom(a);
  const long long Vo = (long long)g.Do * g.HW;
  const bool vec4 = g.HW % 4 == 0 && ((reinterpret_cast<uintptr_t>(a->src) | reinterpret_cast<uintptr_t>(Ls)) & 15) == 0;
  for (int c0 = 0; c0 < a->K; c0 += KC) {
    const int kc = std::min(KC, a->K - c0);
    const size_t smem = (size_t)kc * g.Fo * 4;
    const float* W = a->Wc + (long long)c0 * g.Fo;
    const float* bc = a->bc ? a->bc + c0 : nullptr;
    float* out = Ls + (long long)c0 * Vo;
    const bool slice = a->src_layout == SX_HEAD_SRC_SLICE_MAJOR;
    if (int rc = vec4 ? (slice ? launch_fwd<4, 1>(g, W, bc, kc, out, a->K, a->B, smem, ST(stream))
                               : launch_fwd<4, 0>(g, W, bc, kc, out, a->K, a->B, smem, ST(stream)))
                      : (slice ? launch_fwd<1, 1>(g, W, bc, kc, out, a->K, a->B, smem, ST(stream))
                               : launch_fwd<1, 0>(g, W, bc, kc, out, a->K, a->B, smem, ST(stream))))
      return rc;
  }
  return 0;
}

template <int VEC, int TMAX, int SLICE>
static int launch_bwd(const DropGeom& g, const sx_head_dropout_args* a, const float* dLs, float* dsrc, int accumulate,
                      float* dWc, cudaStream_t st) {
  const long long Vo = (long long)g.Do * g.HW;
  const long long tps = (g.HW + (long long)THREADS * VEC - 1) / ((long long)THREADS * VEC);
  const long long tiles = (long long)a->B * g.Ds * tps;
  const int sms = sm_count_cached();
  SX_REQUIRE(sms > 0, "sx_head_dropout_bwd: no CUDA device (this library has no CPU fallback)");
  for (int c0 = 0; c0 < a->K; c0 += KC) {
    const int kc = std::min(KC, a->K - c0);
    const size_t smem = (size_t)(1 + WARPS) * kc * g.Fo * 4;
    const long long slots = a->part_floats / ((long long)kc * g.Fo);
    const int grid = (int)std::min<long long>({tiles, (long long)sms * 4, slots});
    SX_REQUIRE(grid >= 1, "sx_head_dropout_bwd: needs at least %d floats of scratch", kc * g.Fo);
    SX_CHECK_CUDA(allow_smem(head_dropout_bwd_kernel<VEC, TMAX, SLICE>, smem));
    head_dropout_bwd_kernel<VEC, TMAX, SLICE><<<grid, THREADS, smem, st>>>(
        g, a->Wc + (long long)c0 * g.Fo, kc, dLs + (long long)c0 * Vo, (long long)a->K * Vo, dsrc,
        (accumulate || c0 > 0) ? 1 : 0, a->part, tps, tiles);
    SX_CHECK_CUDA(cudaGetLastError());
    if (int rc = part_reduce(a->part, grid, kc * g.Fo,
                             PartDst{{dWc + (long long)c0 * g.Fo, nullptr, nullptr, nullptr}, {kc * g.Fo, 0, 0, 0}}, st))
      return rc;
  }
  return 0;
}

template <int SLICE>
static int dispatch_bwd(const DropGeom& g, const sx_head_dropout_args* a, const float* dLs, float* dsrc, int accumulate,
                        float* dWc, int need, bool vec2, cudaStream_t st) {
  if (need <= 1) return vec2 ? launch_bwd<2, 1, SLICE>(g, a, dLs, dsrc, accumulate, dWc, st)
                             : launch_bwd<1, 1, SLICE>(g, a, dLs, dsrc, accumulate, dWc, st);
  if (need <= 6) return vec2 ? launch_bwd<2, 6, SLICE>(g, a, dLs, dsrc, accumulate, dWc, st)
                             : launch_bwd<1, 6, SLICE>(g, a, dLs, dsrc, accumulate, dWc, st);
  return vec2 ? launch_bwd<2, 10, SLICE>(g, a, dLs, dsrc, accumulate, dWc, st)
              : launch_bwd<1, 10, SLICE>(g, a, dLs, dsrc, accumulate, dWc, st);
}

extern "C" int sx_head_dropout_bwd(const sx_head_dropout_args* a, const float* dLs, float* dsrc, int32_t accumulate,
                                   float* dWc, void* stream) {
  if (int rc = check_args(a, "sx_head_dropout_bwd")) return rc;
  SX_REQUIRE(dLs && dsrc && dWc && a->part, "sx_head_dropout_bwd: null pointer");
  const DropGeom g = make_geom(a);
  const bool vec2 = g.HW % 2 == 0 && ((reinterpret_cast<uintptr_t>(a->src) | reinterpret_cast<uintptr_t>(dLs) |
                                       reinterpret_cast<uintptr_t>(dsrc)) & 7) == 0;
  // live candidate planes per source slice: 1 (none), D_pool_K (unfold), up to 2 D_pool_K + 1 (interp, first taps too)
  const int need = a->dmap == SX_HEAD_DMAP_NONE
                       ? 1
                       : ((a->dmap == SX_HEAD_DMAP_UNFOLD || a->dmap == SX_HEAD_DMAP_UNFOLD_INTERLEAVED) ? a->Dk
                                                                                                       : 2 * a->Dk + 2);
  cudaStream_t st = ST(stream);
  if (a->src_layout == SX_HEAD_SRC_SLICE_MAJOR) return dispatch_bwd<1>(g, a, dLs, dsrc, accumulate, dWc, need, vec2, st);
  return dispatch_bwd<0>(g, a, dLs, dsrc, accumulate, dWc, need, vec2, st);
}
