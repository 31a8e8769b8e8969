// Voxel-wise segmentation head in collapsed form (SURVEY.md §7) and its building blocks.
//
// Reference (segtran3d.py:364-367, 381-386, 488-496; segtran2d.py:304-306, 427, 435-436):
//   logits = interp_out( conv_cls( interp_D( conv_bridge(curr) + interp(vfeat_fused) ) ) )
// Every stage is linear and interpolation weights sum to one, so
//   logits = interp_out( interp_D( (Wc Wb) curr + interp(Wc vfeat) + Wc bb + bc ) )
// which turns a Cf->F conv over every voxel plus three F-channel full-resolution tensors into ONE pass over
// `curr` producing `num_classes` channels (HBM-bound: curr is read exactly once, forward and backward).
//
//   head_contract_fwd        L[b,k,v]   = sum_c W[k,c] curr[b,c,v] + bias[k]          (reads curr)
//   head_contract_bwd_data   dcurr[b,c,v] = sum_k W[k,c] dL[b,k,v]                    (writes dcurr)
//   head_contract_bwd_weight dW[k,c]   += sum_{b,v} dL[b,k,v] curr[b,c,v]             (reads curr; V % 4 != 0)
//   resize_axis_fwd / _bwd   1-D linear resampling along one axis (align_corners=False), PyTorch semantics;
//                            tri/bi-linear interpolation is applied as a sequence of axis passes.
//   sgemm_small              strided fp32 GEMM on CUDA cores for the tiny class-dimension products.
#include <cstdlib>

#include "sx_common.cuh"
#include "sx_part.cuh"
#include "sx_resample.cuh"

namespace {

constexpr int MAXK = 8;          // max classes handled per pass

// ---- forward contraction: block = 128 threads x float4 = 512 voxels, loop over channels ----
template <int VEC, int KMAX, int UNR = 8, int MINB = 12>
__global__ void __launch_bounds__(128, (KMAX <= 4 && VEC == 4) ? MINB : 1)
head_contract_fwd_kernel(const float* __restrict__ curr, const float* __restrict__ W, const float* __restrict__ bias,
                         int Cf, long long V, int K, float* __restrict__ L, int accumulate) {
  extern __shared__ float sW[];             // [K][Cf]
  for (int i = threadIdx.x; i < K * Cf; i += blockDim.x) sW[i] = W[i];
  __syncthreads();
  const int b = blockIdx.y;
  const long long v0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * VEC;
  if (v0 >= V) return;
  const float* src = curr + (long long)b * Cf * V + v0;
  float acc[KMAX][VEC];
#pragma unroll
  for (int k = 0; k < KMAX; ++k)
#pragma unroll
    for (int j = 0; j < VEC; ++j) acc[k][j] = 0.f;
#pragma unroll UNR
  for (int c = 0; c < Cf; ++c) {
    float x[VEC];
    if constexpr (VEC == 4) {
      const float4 t = __ldcs(reinterpret_cast<const float4*>(src + (long long)c * V));     // streamed once: evict-first
      x[0] = t.x; x[1] = t.y; x[2] = t.z; x[3] = t.w;
    } else {
      x[0] = __ldg(src + (long long)c * V);
    }
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
      if (k < K) {
        const float w = sW[k * Cf + c];
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[k][j] = fmaf(w, x[j], acc[k][j]);
      }
  }
#pragma unroll
  for (int k = 0; k < KMAX; ++k)
    if (k < K) {
      float* dst = L + ((long long)b * K + k) * V + v0;
      const float bk = bias ? bias[k] : 0.f;
#pragma unroll
      for (int j = 0; j < VEC; ++j) {
        const float r = acc[k][j] + bk;
        dst[j] = accumulate ? dst[j] + r : r;
      }
    }
}

template <int VEC>
__global__ void __launch_bounds__(128)
head_contract_bwd_data_kernel(const float* __restrict__ dL, const float* __restrict__ W, int Cf, long long V, int K,
                              float* __restrict__ dcurr) {
  extern __shared__ float sW[];
  for (int i = threadIdx.x; i < K * Cf; i += blockDim.x) sW[i] = W[i];
  __syncthreads();
  const int b = blockIdx.y;
  const long long v0 = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * VEC;
  if (v0 >= V) return;
  float g[MAXK][VEC];
#pragma unroll
  for (int k = 0; k < MAXK; ++k)
#pragma unroll
    for (int j = 0; j < VEC; ++j) g[k][j] = (k < K) ? dL[((long long)b * K + k) * V + v0 + j] : 0.f;
  float* dst = dcurr + (long long)b * Cf * V + v0;
#pragma unroll 4
  for (int c = 0; c < Cf; ++c) {
    float o[VEC];
#pragma unroll
    for (int j = 0; j < VEC; ++j) o[j] = 0.f;
#pragma unroll
    for (int k = 0; k < MAXK; ++k)
      if (k < K) {
        const float w = sW[k * Cf + c];
#pragma unroll
        for (int j = 0; j < VEC; ++j) o[j] = fmaf(w, g[k][j], o[j]);
      }
    if constexpr (VEC == 4)
      *reinterpret_cast<float4*>(dst + (long long)c * V) = make_float4(o[0], o[1], o[2], o[3]);
    else
      dst[(long long)c * V] = o[0];
  }
}

// one warp per channel; lanes stride over a voxel chunk; the (chunk, batch) CTA's sums dW[k,c] = sum_v dL[k,v] curr[c,v]
// go to its slot (blockIdx.z * gridDim.y + blockIdx.y, [K * Cf]) of `part`
__global__ void __launch_bounds__(256)
head_contract_bwd_weight_kernel(const float* __restrict__ dL, const float* __restrict__ curr, int Cf, long long V,
                                int K, long long chunk, float* __restrict__ part) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c = blockIdx.x * 8 + warp;
  const int b = blockIdx.z;
  const long long v_begin = (long long)blockIdx.y * chunk;
  long long v_end = v_begin + chunk;
  if (v_end > V) v_end = V;
  if (c >= Cf) return;
  const float* x = curr + ((long long)b * Cf + c) * V;
  const float* g = dL + (long long)b * K * V;
  float acc[MAXK];
#pragma unroll
  for (int k = 0; k < MAXK; ++k) acc[k] = 0.f;
  for (long long v = v_begin + lane; v < v_end; v += 32) {
    const float xv = __ldg(x + v);
#pragma unroll
    for (int k = 0; k < MAXK; ++k)
      if (k < K) acc[k] = fmaf(xv, g[(long long)k * V + v], acc[k]);
  }
#pragma unroll
  for (int k = 0; k < MAXK; ++k)
    if (k < K) {
      const float s = sx::warp_sum(acc[k]);
      if (lane == 0) part[((long long)blockIdx.z * gridDim.y + blockIdx.y) * K * Cf + k * Cf + c] = s;
    }
}

// ---- 1-D linear resize along one axis of x viewed as [outer, Lin, inner] -> [outer, Lout, inner] ----
// (ratio Lin/Lout: F.interpolate with a target size; sx::src_index is in sx_resample.cuh)

template <typename I>
__global__ void resize_axis_fwd_kernel(const float* __restrict__ x, long long outer_, int Lin, int Lout, long long inner_,
                                       float* __restrict__ y, int accumulate) {
  const float scale = (float)Lin / (float)Lout;
  const I inner = (I)inner_;
  const I total = (I)(outer_ * Lout * inner_);
  for (I idx = (I)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (I)gridDim.x * blockDim.x) {
    const I in = idx % inner;
    const I t = idx / inner;
    const int j = (int)(t % (I)Lout);
    const I o = t / (I)Lout;
    int i0, i1;
    float w1;
    sx::src_index(j, scale, Lin, i0, i1, w1);
    const float* base = x + o * Lin * inner + in;
    const float v = (1.f - w1) * base[(long long)i0 * inner] + w1 * base[(long long)i1 * inner];
    y[idx] = accumulate ? y[idx] + v : v;
  }
}

// adjoint (gather form): dx[o,i,in] = sum_j w(j->i) dy[o,j,in]
template <typename I>
__global__ void resize_axis_bwd_kernel(const float* __restrict__ dy, long long outer_, int Lin, int Lout,
                                       long long inner_, float* __restrict__ dx) {
  const float scale = (float)Lin / (float)Lout;
  const float inv = (float)Lout / (float)Lin;
  const I inner = (I)inner_;
  const I total = (I)(outer_ * Lin * inner_);
  for (I idx = (I)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (I)gridDim.x * blockDim.x) {
    const I in = idx % inner;
    const I t = idx / inner;
    const int i = (int)(t % (I)Lin);
    const I o = t / (I)Lin;
    int jlo = (int)floorf(((float)i - 1.f + 0.5f) * inv - 0.5f) - 1;
    int jhi = (int)ceilf(((float)i + 1.f + 0.5f) * inv - 0.5f) + 1;
    if (i == 0) jlo = 0;                       // clamped sources (s < 0) map to i = 0
    if (i == Lin - 1) jhi = Lout - 1;
    if (jlo < 0) jlo = 0;
    if (jhi > Lout - 1) jhi = Lout - 1;
    const float* base = dy + o * Lout * inner + in;
    float acc = 0.f;
    for (int j = jlo; j <= jhi; ++j) {
      int i0, i1;
      float w1;
      sx::src_index(j, scale, Lin, i0, i1, w1);
      float w = 0.f;
      if (i0 == i) w += 1.f - w1;
      if (i1 == i) w += w1;
      if (w != 0.f) acc = fmaf(w, base[(long long)j * inner], acc);
    }
    dx[idx] = acc;
  }
}

// float4 flavours: `inner` is a multiple of 4 (all but the innermost axis): one index computation per 4 elements
__global__ void resize_axis_fwd_v4_kernel(const float4* __restrict__ x, unsigned outer, int Lin, int Lout,
                                          unsigned inner4, float4* __restrict__ y, int accumulate) {
  const float scale = (float)Lin / (float)Lout;
  const unsigned total = outer * (unsigned)Lout * inner4;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned in = idx % inner4, t = idx / inner4;
    const int j = (int)(t % (unsigned)Lout);
    const unsigned o = t / (unsigned)Lout;
    int i0, i1;
    float w1;
    sx::src_index(j, scale, Lin, i0, i1, w1);
    const float4* base = x + (size_t)o * Lin * inner4 + in;
    const float4 a = __ldg(base + (size_t)i0 * inner4), b = __ldg(base + (size_t)i1 * inner4);
    const float w0 = 1.f - w1;
    float4 v = make_float4(w0 * a.x + w1 * b.x, w0 * a.y + w1 * b.y, w0 * a.z + w1 * b.z, w0 * a.w + w1 * b.w);
    if (accumulate) { const float4 c = y[idx]; v.x += c.x; v.y += c.y; v.z += c.z; v.w += c.w; }
    y[idx] = v;
  }
}

__global__ void resize_axis_bwd_v4_kernel(const float4* __restrict__ dy, unsigned outer, int Lin, int Lout,
                                          unsigned inner4, float4* __restrict__ dx) {
  const float scale = (float)Lin / (float)Lout, inv = (float)Lout / (float)Lin;
  const unsigned total = outer * (unsigned)Lin * inner4;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned in = idx % inner4, t = idx / inner4;
    const int i = (int)(t % (unsigned)Lin);
    const unsigned o = t / (unsigned)Lin;
    int jlo = (int)floorf(((float)i - 0.5f) * inv - 0.5f) - 1;
    int jhi = (int)ceilf(((float)i + 1.5f) * inv - 0.5f) + 1;
    if (i == 0) jlo = 0;
    if (i == Lin - 1) jhi = Lout - 1;
    if (jlo < 0) jlo = 0;
    if (jhi > Lout - 1) jhi = Lout - 1;
    const float4* base = dy + (size_t)o * Lout * inner4 + in;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int j = jlo; j <= jhi; ++j) {
      int i0, i1;
      float w1;
      sx::src_index(j, scale, Lin, i0, i1, w1);
      float w = 0.f;
      if (i0 == i) w += 1.f - w1;
      if (i1 == i) w += w1;
      if (w != 0.f) {
        const float4 g = __ldg(base + (size_t)j * inner4);
        acc.x = fmaf(w, g.x, acc.x); acc.y = fmaf(w, g.y, acc.y); acc.z = fmaf(w, g.z, acc.z); acc.w = fmaf(w, g.w, acc.w);
      }
    }
    dx[idx] = acc;
  }
}

// innermost axis (inner == 1): each thread produces 4 consecutive outputs (Lout % 4 == 0) / inputs (Lin % 4 == 0)
__global__ void resize_last_fwd_kernel(const float* __restrict__ x, unsigned rows, int Lin, int Lout,
                                       float* __restrict__ y, int accumulate) {
  const float scale = (float)Lin / (float)Lout;
  const unsigned q = (unsigned)Lout / 4, total = rows * q;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned r = idx / q;
    const int j0 = (int)(idx % q) * 4;
    const float* base = x + (size_t)r * Lin;
    float o[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      int i0, i1;
      float w1;
      sx::src_index(j0 + u, scale, Lin, i0, i1, w1);
      o[u] = (1.f - w1) * __ldg(base + i0) + w1 * __ldg(base + i1);
    }
    float4* dst = reinterpret_cast<float4*>(y + (size_t)r * Lout + j0);
    float4 v = make_float4(o[0], o[1], o[2], o[3]);
    if (accumulate) { const float4 c = *dst; v.x += c.x; v.y += c.y; v.z += c.z; v.w += c.w; }
    *dst = v;
  }
}

__global__ void resize_last_bwd_kernel(const float* __restrict__ dy, unsigned rows, int Lin, int Lout,
                                       float* __restrict__ dx) {
  const float scale = (float)Lin / (float)Lout, inv = (float)Lout / (float)Lin;
  const unsigned q = (unsigned)Lin / 4, total = rows * q;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned r = idx / q;
    const int i00 = (int)(idx % q) * 4;
    const float* base = dy + (size_t)r * Lout;
    float o[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int i = i00 + u;
      int jlo = (int)floorf(((float)i - 0.5f) * inv - 0.5f) - 1;
      int jhi = (int)ceilf(((float)i + 1.5f) * inv - 0.5f) + 1;
      if (i == 0) jlo = 0;
      if (i == Lin - 1) jhi = Lout - 1;
      if (jlo < 0) jlo = 0;
      if (jhi > Lout - 1) jhi = Lout - 1;
      float acc = 0.f;
      for (int j = jlo; j <= jhi; ++j) {
        int i0, i1;
        float w1;
        sx::src_index(j, scale, Lin, i0, i1, w1);
        float w = 0.f;
        if (i0 == i) w += 1.f - w1;
        if (i1 == i) w += w1;
        if (w != 0.f) acc = fmaf(w, __ldg(base + j), acc);
      }
      o[u] = acc;
    }
    *reinterpret_cast<float4*>(dx + (size_t)r * Lin + i00) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// ---- exact x2 up-sampling along the innermost axis (Lout == 2*Lin, align_corners=False): closed-form weights
//      y[2i] = .25 x[i-1] + .75 x[i] ; y[2i+1] = .75 x[i] + .25 x[i+1]   (edges clamp)     [the W axis of every final
//      tri/bi-linear pass: 45 MB -> 90 MB at cfg 4] ; each thread handles 4 inputs <-> 8 outputs with float4 accesses
__global__ void resize_last_x2_fwd_kernel(const float* __restrict__ x, unsigned rows, int Lin, float* __restrict__ y,
                                          int accumulate) {
  const unsigned q = (unsigned)Lin / 4, total = rows * q;
  const int Lout = 2 * Lin;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned r = idx / q;
    const int i0 = (int)(idx % q) * 4;
    const float* base = x + (size_t)r * Lin;
    const float4 c = __ldg(reinterpret_cast<const float4*>(base + i0));
    const float l = i0 > 0 ? __ldg(base + i0 - 1) : c.x;
    const float rr = i0 + 4 < Lin ? __ldg(base + i0 + 4) : c.w;
    float4 o0, o1;
    o0.x = 0.25f * l + 0.75f * c.x;   o0.y = 0.75f * c.x + 0.25f * c.y;
    o0.z = 0.25f * c.x + 0.75f * c.y; o0.w = 0.75f * c.y + 0.25f * c.z;
    o1.x = 0.25f * c.y + 0.75f * c.z; o1.y = 0.75f * c.z + 0.25f * c.w;
    o1.z = 0.25f * c.z + 0.75f * c.w; o1.w = 0.75f * c.w + 0.25f * rr;
    float4* dst = reinterpret_cast<float4*>(y + (size_t)r * Lout + 2 * i0);
    if (accumulate) {
      const float4 a = dst[0], b = dst[1];
      o0.x += a.x; o0.y += a.y; o0.z += a.z; o0.w += a.w; o1.x += b.x; o1.y += b.y; o1.z += b.z; o1.w += b.w;
    }
    dst[0] = o0; dst[1] = o1;
  }
}

// adjoint: dx[i] = .75 (dy[2i] + dy[2i+1]) + .25 (dy[2i-1] + dy[2i+2]); the clamped edges fold their .25 back in
__global__ void resize_last_x2_bwd_kernel(const float* __restrict__ dy, unsigned rows, int Lin, float* __restrict__ dx) {
  const unsigned q = (unsigned)Lin / 4, total = rows * q;
  const int Lout = 2 * Lin;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const unsigned r = idx / q;
    const int i0 = (int)(idx % q) * 4;
    const float* base = dy + (size_t)r * Lout + 2 * i0;
    const float4 a = __ldg(reinterpret_cast<const float4*>(base)), b = __ldg(reinterpret_cast<const float4*>(base + 4));
    const float g[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    const float gl = i0 > 0 ? __ldg(base - 1) : 0.f;                 // dy[2*i0 - 1]
    const float gr = i0 + 4 < Lin ? __ldg(base + 8) : 0.f;           // dy[2*(i0+4)]
    float o[4];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const float left = u > 0 ? g[2 * u - 1] : gl, right = u < 3 ? g[2 * u + 2] : gr;
      o[u] = 0.75f * (g[2 * u] + g[2 * u + 1]) + 0.25f * (left + right);
    }
    if (i0 == 0) o[0] += 0.25f * g[0];                               // y[0] = x[0] exactly (clamped source)
    if (i0 + 4 == Lin) o[3] += 0.25f * g[7];                         // y[Lout-1] = x[Lin-1]
    *reinterpret_cast<float4*>(dx + (size_t)r * Lin + i0) = make_float4(o[0], o[1], o[2], o[3]);
  }
}

// ---- class scores of the fused tokens, exact fp32: out[b,k,n] = sum_f W[k,f] vf[b,n,f]; one warp per token ----
// KMAX: rows handled per pass (8 for the class rows of the collapsed head; 16 / 32 for the 4 sub-pixel rows per class
// of the direct head), so a token row is read once for all of them
template <bool V4, int KMAX>
__global__ void token_scores_kernel(const float* __restrict__ vf, const float* __restrict__ W, long long T, int N,
                                    int F, int K, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long t = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (t >= T) return;
  const float* x = vf + t * F;
  float acc[KMAX];
#pragma unroll
  for (int k = 0; k < KMAX; ++k) acc[k] = 0.f;
  if (V4) {                                 // F % 4 == 0, 16-byte aligned rows: 4 x 512 B of the token row in flight
#pragma unroll 4
    for (int f = lane * 4; f < F; f += 128) {
      const float4 xv = *reinterpret_cast<const float4*>(x + f);
#pragma unroll
      for (int k = 0; k < KMAX; ++k)
        if (k < K) {
          const float4 w = __ldg(reinterpret_cast<const float4*>(W + (long long)k * F + f));
          acc[k] = fmaf(xv.x, w.x, fmaf(xv.y, w.y, fmaf(xv.z, w.z, fmaf(xv.w, w.w, acc[k]))));
        }
    }
  } else {
    for (int f = lane; f < F; f += 32) {
      const float xv = x[f];
#pragma unroll
      for (int k = 0; k < KMAX; ++k)
        if (k < K) acc[k] = fmaf(xv, __ldg(W + (long long)k * F + f), acc[k]);
    }
  }
  const long long b = t / N, n = t % N;
#pragma unroll
  for (int k = 0; k < KMAX; ++k)
    if (k < K) {
      const float s = sx::warp_sum(acc[k]);
      if (lane == 0) out[(b * K + k) * N + n] = s;
    }
}

// ---- its data gradient: dvf[b,n,f] = sum_k dt[b,k,n] W[k,f]; one thread per 4 channels, writes coalesced ----
template <int KMAX>
__global__ void token_scores_bwd_kernel(const float* __restrict__ dt, const float* __restrict__ W, long long T, int N,
                                        int F, int K, float* __restrict__ dvf) {
  const int F4 = F >> 2;
  const long long total = T * F4;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long t = i / F4;
    const int f = (int)(i - t * F4) * 4;
    const long long b = t / N, n = t - b * N;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int k = 0; k < KMAX; ++k)
      if (k < K) {
        const float d = __ldg(dt + (b * K + k) * N + n);
        const float4 w = __ldg(reinterpret_cast<const float4*>(W + (long long)k * F + f));
        acc.x = fmaf(d, w.x, acc.x); acc.y = fmaf(d, w.y, acc.y); acc.z = fmaf(d, w.z, acc.z); acc.w = fmaf(d, w.w, acc.w);
      }
    *reinterpret_cast<float4*>(dvf + t * F + f) = acc;
  }
}

// ---- tiny strided fp32 GEMM: C[z][m][n] (+)= alpha * sum_k A[z](m,k) B[z](k,n) ----
__global__ void sgemm_small_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C,
                                   int M, int N, int K, long long sam, long long sak, long long sbk, long long sbn,
                                   long long scm, long long scn, long long saz, long long sbz, long long scz, float alpha,
                                   int accumulate) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  const int m = blockIdx.y * blockDim.y + threadIdx.y;
  const long long z = blockIdx.z;
  if (m >= M || n >= N) return;
  const float* a = A + z * saz + (long long)m * sam;
  const float* b = B + z * sbz + (long long)n * sbn;
  float acc = 0.f;
  int k = 0;
  for (; k + 8 <= K; k += 8) {             // 16 independent loads in flight per thread (latency-bound otherwise)
    float av[8], bv[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      av[u] = a[(long long)(k + u) * sak];
      bv[u] = b[(long long)(k + u) * sbk];
    }
#pragma unroll
    for (int u = 0; u < 8; ++u) acc = fmaf(av[u], bv[u], acc);
  }
  for (; k < K; ++k) acc = fmaf(a[(long long)k * sak], b[(long long)k * sbk], acc);
  float* c = C + z * scz + (long long)m * scm + (long long)n * scn;
  *c = accumulate ? *c + alpha * acc : alpha * acc;
}

// same product, one WARP per output element, lanes stride over k (few outputs, long reductions)
__global__ void sgemm_small_warp_kernel(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C,
                                        int M, int N, int K, long long sam, long long sak, long long sbk, long long sbn,
                                        long long scm, long long scn, long long saz, long long sbz, long long scz,
                                        float alpha, int accumulate) {
  const int lane = threadIdx.x & 31;
  const long long o = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (o >= (long long)M * N) return;
  const int m = (int)(o / N), n = (int)(o % N);
  const long long z = blockIdx.z;
  const float* a = A + z * saz + (long long)m * sam;
  const float* b = B + z * sbz + (long long)n * sbn;
  float acc = 0.f;
#pragma unroll 8
  for (int k = lane; k < K; k += 32) acc = fmaf(a[(long long)k * sak], b[(long long)k * sbk], acc);   // 16 loads in flight
  acc = sx::warp_sum(acc);
  if (lane == 0) {
    float* c = C + z * scz + (long long)m * scm + (long long)n * scn;
    *c = accumulate ? *c + alpha * acc : alpha * acc;
  }
}

// ---- direct class head (out_fpn_layers == in_fpn_layers): sub-pixel scores -> logits in their final layout ----
// S [B][4K][N], row 4k + 2a + c = sub-pixel (a, c) of class k's 2x2 transposed-conv output, token n = d*H2*W2 + y*W2 + x.
// The virtual grid V[b,k] (2H2, 2W2, D2) holds V[i,j,d] = S[b, 4k + 2(i%2) + j%2, d*H2*W2 + (i/2)*W2 + j/2]; the logits
// [B][K][H][W][D] are its trilinear resampling to (H, W, D) (2-D: D2 = D = 1), plus bias[k].
__device__ __forceinline__ long long subpixel_src(int i, int j, int d, int H2, int W2, long long N) {
  return (long long)(((i & 1) << 1) | (j & 1)) * N + (long long)d * H2 * W2 + (long long)(i >> 1) * W2 + (j >> 1);
}

// one thread per logit; blockIdx.y = b*K + k; the innermost output axis is the fastest (coalesced writes)
__global__ void subpixel_resize_fwd_kernel(const float* __restrict__ S, const float* __restrict__ bias, int K, int D2,
                                           int H2, int W2, int H, int W, int D, float* __restrict__ out) {
  const int bk = blockIdx.y, k = bk % K;
  const long long N = (long long)D2 * H2 * W2;
  const float* s = S + (long long)bk * 4 * N;
  float* o = out + (long long)bk * H * W * D;
  const float rh = (float)(2 * H2) / (float)H, rw = (float)(2 * W2) / (float)W, rd = (float)D2 / (float)D;
  const float bv = bias ? bias[k] : 0.f;
  const unsigned total = (unsigned)H * W * D;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int dd = (int)(idx % (unsigned)D);
    const unsigned t = idx / (unsigned)D;
    const int w = (int)(t % (unsigned)W), h = (int)(t / (unsigned)W);
    int i0, i1, j0, j1, d0, d1;
    float ti, tj, td;
    sx::src_index(h, rh, 2 * H2, i0, i1, ti);
    sx::src_index(w, rw, 2 * W2, j0, j1, tj);
    sx::src_index(dd, rd, D2, d0, d1, td);
    auto g = [&](int i, int j) {
      return (1.f - td) * __ldg(s + subpixel_src(i, j, d0, H2, W2, N)) + td * __ldg(s + subpixel_src(i, j, d1, H2, W2, N));
    };
    const float v = (1.f - ti) * ((1.f - tj) * g(i0, j0) + tj * g(i0, j1)) + ti * ((1.f - tj) * g(i1, j0) + tj * g(i1, j1));
    o[idx] = v + bv;
  }
}

// weight of input cell i in output cell j of a 1-D linear resampling (both taps may be i at a clamped edge)
__device__ __forceinline__ float tap_weight(int j, float ratio, int Lin, int i) {
  int i0, i1;
  float w1;
  sx::src_index(j, ratio, Lin, i0, i1, w1);
  return (i0 == i ? 1.f - w1 : 0.f) + (i1 == i ? w1 : 0.f);
}

// adjoint in gather form: one thread per virtual cell (i, j, d), d fastest; dS[b, 4k + s, n] = sum over the logits that
// read the cell of weight * dout, in a fixed order (no atomics)
__global__ void subpixel_resize_bwd_kernel(const float* __restrict__ dout, int D2, int H2, int W2, int H, int W, int D,
                                           float* __restrict__ dS) {
  const int bk = blockIdx.y;
  const long long N = (long long)D2 * H2 * W2;
  const float* g = dout + (long long)bk * H * W * D;
  float* ds = dS + (long long)bk * 4 * N;
  const int Li = 2 * H2, Lj = 2 * W2;
  const float rh = (float)Li / (float)H, rw = (float)Lj / (float)W, rd = (float)D2 / (float)D;
  const unsigned total = (unsigned)Li * Lj * D2;
  for (unsigned idx = blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += gridDim.x * blockDim.x) {
    const int d = (int)(idx % (unsigned)D2);
    const unsigned t = idx / (unsigned)D2;
    const int j = (int)(t % (unsigned)Lj), i = (int)(t / (unsigned)Lj);
    int hlo, hhi, wlo, whi, dlo, dhi;
    sx::src_readers(i, (float)H / (float)Li, Li, H, hlo, hhi);
    sx::src_readers(j, (float)W / (float)Lj, Lj, W, wlo, whi);
    sx::src_readers(d, (float)D / (float)D2, D2, D, dlo, dhi);
    float acc = 0.f;
    for (int h = hlo; h <= hhi; ++h) {
      const float wh = tap_weight(h, rh, Li, i);
      if (wh == 0.f) continue;
      float acc_h = 0.f;
      for (int w = wlo; w <= whi; ++w) {
        const float ww = tap_weight(w, rw, Lj, j);
        if (ww == 0.f) continue;
        const float* row = g + ((long long)h * W + w) * D;
        float acc_w = 0.f;
        for (int dd = dlo; dd <= dhi; ++dd) {
          const float wd = tap_weight(dd, rd, D2, d);
          if (wd != 0.f) acc_w = fmaf(wd, __ldg(row + dd), acc_w);
        }
        acc_h = fmaf(ww, acc_w, acc_h);
      }
      acc = fmaf(wh, acc_h, acc);
    }
    ds[subpixel_src(i, j, d, H2, W2, N)] = acc;
  }
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int sx_head_contract_fwd(const float* curr, const float* W, const float* bias, int32_t B, int32_t Cf,
                                    int64_t V, int32_t K, float* L, int32_t accumulate, void* stream) {
  SX_REQUIRE(K >= 1 && K <= MAXK, "sx_head_contract_fwd: num_classes %d not in 1..%d", K, MAXK);
  const size_t smem = (size_t)K * Cf * 4;
  SX_REQUIRE(smem <= 48 * 1024, "sx_head_contract_fwd: K*Cf=%d too large", K * Cf);
  const bool vec4 = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(curr) & 15) == 0);
  if (vec4) {
    dim3 grid(sx_ceil_div(V, 128 * 4), B);
    if (K <= 4)        // 16 channel rows (8 KB per warp) in flight, 6 blocks / SM: 6.4 TB/s at cfg 4 (8-deep at 12 blocks: 5.1)
      head_contract_fwd_kernel<4, 4, 16, 6><<<grid, 128, smem, ST(stream)>>>(curr, W, bias, Cf, V, K, L, accumulate);
    else
      head_contract_fwd_kernel<4, MAXK><<<grid, 128, smem, ST(stream)>>>(curr, W, bias, Cf, V, K, L, accumulate);
  } else {
    dim3 grid(sx_ceil_div(V, 128), B);
    head_contract_fwd_kernel<1, MAXK><<<grid, 128, smem, ST(stream)>>>(curr, W, bias, Cf, V, K, L, accumulate);
  }
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_head_contract_bwd_data(const float* dL, const float* W, int32_t B, int32_t Cf, int64_t V, int32_t K,
                                         float* dcurr, void* stream) {
  SX_REQUIRE(K >= 1 && K <= MAXK, "sx_head_contract_bwd_data: num_classes %d not in 1..%d", K, MAXK);
  const size_t smem = (size_t)K * Cf * 4;
  SX_REQUIRE(smem <= 48 * 1024, "sx_head_contract_bwd_data: K*Cf=%d too large", K * Cf);
  const bool vec4 = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(dcurr) & 15) == 0);
  if (vec4) {
    dim3 grid(sx_ceil_div(V, 128 * 4), B);
    head_contract_bwd_data_kernel<4><<<grid, 128, smem, ST(stream)>>>(dL, W, Cf, V, K, dcurr);
  } else {
    dim3 grid(sx_ceil_div(V, 128), B);
    head_contract_bwd_data_kernel<1><<<grid, 128, smem, ST(stream)>>>(dL, W, Cf, V, K, dcurr);
  }
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_head_contract_bwd_weight(const float* dL, const float* curr, int32_t B, int32_t Cf, int64_t V,
                                           int32_t K, float* dW, float* part, int64_t part_floats, void* stream) {
  SX_REQUIRE(K >= 1 && K <= MAXK, "sx_head_contract_bwd_weight: num_classes %d not in 1..%d", K, MAXK);
  // one slot per (chunk, batch) CTA: chunks of 8192 voxels, fewer and longer when the scratch or the grid runs short
  const int max_chunks = std::min(part_slots(part_floats, (long long)K * Cf) / B, 65535);
  SX_REQUIRE(part && max_chunks >= 1, "sx_head_contract_bwd_weight: needs at least %lld floats of scratch",
             (long long)B * K * Cf);
  long long chunk = 8192;
  int chunks = sx_ceil_div(V, chunk);
  if (chunks > max_chunks) { chunk = sx_ceil_div(V, max_chunks); chunks = sx_ceil_div(V, chunk); }
  dim3 grid(sx_ceil_div(Cf, 8), chunks, B);
  head_contract_bwd_weight_kernel<<<grid, 256, 0, ST(stream)>>>(dL, curr, Cf, V, K, chunk, part);
  SX_CHECK_CUDA(cudaGetLastError());
  return part_reduce(part, chunks * B, K * Cf, PartDst{{dW, nullptr, nullptr, nullptr}, {K * Cf, 0, 0, 0}}, ST(stream));
}

static int ew_grid(long long total) {
  long long g = (total + 255) / 256;
  if (g > sm_count_cached() * 16ll) g = sm_count_cached() * 16ll;
  if (g < 1) g = 1;
  return (int)g;
}

extern "C" int sx_resize_axis_fwd(const float* x, int64_t outer, int32_t Lin, int32_t Lout, int64_t inner, float* y,
                                  int32_t accumulate, void* stream) {
  const long long big = outer * (Lin > Lout ? Lin : Lout) * inner;
  const bool a16 = ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15) == 0;
  if (big < (1ll << 31) && a16 && inner % 4 == 0) {
    resize_axis_fwd_v4_kernel<<<ew_grid(outer * Lout * inner / 4), 256, 0, ST(stream)>>>(
        (const float4*)x, (unsigned)outer, Lin, Lout, (unsigned)(inner / 4), (float4*)y, accumulate);
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (big < (1ll << 31) && a16 && inner == 1 && Lout == 2 * Lin && Lin % 4 == 0) {
    resize_last_x2_fwd_kernel<<<ew_grid(outer * Lin / 4), 256, 0, ST(stream)>>>(x, (unsigned)outer, Lin, y, accumulate);
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (big < (1ll << 31) && a16 && inner == 1 && Lout % 4 == 0) {
    resize_last_fwd_kernel<<<ew_grid(outer * Lout / 4), 256, 0, ST(stream)>>>(x, (unsigned)outer, Lin, Lout, y,
                                                                             accumulate);
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (big < (1ll << 31))
    resize_axis_fwd_kernel<unsigned int><<<ew_grid(outer * Lout * inner), 256, 0, ST(stream)>>>(x, outer, Lin, Lout,
                                                                                                 inner, y, accumulate);
  else
    resize_axis_fwd_kernel<long long><<<ew_grid(outer * Lout * inner), 256, 0, ST(stream)>>>(x, outer, Lin, Lout, inner,
                                                                                              y, accumulate);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_resize_axis_bwd(const float* dy, int64_t outer, int32_t Lin, int32_t Lout, int64_t inner, float* dx,
                                  void* stream) {
  const long long big = outer * (Lin > Lout ? Lin : Lout) * inner;
  const bool a16 = ((reinterpret_cast<uintptr_t>(dy) | reinterpret_cast<uintptr_t>(dx)) & 15) == 0;
  if (big < (1ll << 31) && a16 && inner % 4 == 0) {
    resize_axis_bwd_v4_kernel<<<ew_grid(outer * Lin * inner / 4), 256, 0, ST(stream)>>>(
        (const float4*)dy, (unsigned)outer, Lin, Lout, (unsigned)(inner / 4), (float4*)dx);
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (big < (1ll << 31) && a16 && inner == 1 && Lout == 2 * Lin && Lin % 4 == 0) {
    resize_last_x2_bwd_kernel<<<ew_grid(outer * Lin / 4), 256, 0, ST(stream)>>>(dy, (unsigned)outer, Lin, dx);
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (big < (1ll << 31) && a16 && inner == 1 && Lin % 4 == 0) {
    resize_last_bwd_kernel<<<ew_grid(outer * Lin / 4), 256, 0, ST(stream)>>>(dy, (unsigned)outer, Lin, Lout, dx);
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (big < (1ll << 31))
    resize_axis_bwd_kernel<unsigned int><<<ew_grid(outer * Lin * inner), 256, 0, ST(stream)>>>(dy, outer, Lin, Lout,
                                                                                                inner, dx);
  else
    resize_axis_bwd_kernel<long long><<<ew_grid(outer * Lin * inner), 256, 0, ST(stream)>>>(dy, outer, Lin, Lout, inner,
                                                                                             dx);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_sgemm_small(const float* A, const float* B, float* C, int32_t M, int32_t N, int32_t K, int64_t sam,
                              int64_t sak, int64_t sbk, int64_t sbn, int64_t scm, int64_t scn, int32_t Z, int64_t saz,
                              int64_t sbz, int64_t scz, float alpha, int32_t accumulate, void* stream) {
  SX_REQUIRE(Z >= 1 && Z <= 65535, "sx_sgemm_small: batch %d out of range", Z);
  if ((long long)M * N <= 16384 && K >= 64) {
    dim3 grid(sx_ceil_div((long long)M * N, 8), 1, Z);
    sgemm_small_warp_kernel<<<grid, 256, 0, ST(stream)>>>(A, B, C, M, N, K, sam, sak, sbk, sbn, scm, scn, saz, sbz, scz,
                                                         alpha, accumulate);
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  dim3 blk(32, 8), grid(sx_ceil_div(N, 32), sx_ceil_div(M, 8), Z);
  sgemm_small_kernel<<<grid, blk, 0, ST(stream)>>>(A, B, C, M, N, K, sam, sak, sbk, sbn, scm, scn, saz, sbz, scz, alpha,
                                                   accumulate);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// rows per pass of the token-score kernels: the collapsed head's class rows (<= 8, unchanged), or the direct head's
// 4 sub-pixel rows per class (<= 32)
constexpr int MAXROWS = 32;

template <int KMAX>
static void token_scores_launch(const float* vf, const float* W, long long T, int N, int F, int K, float* out,
                                cudaStream_t st) {
  if (F % 4 == 0 && (reinterpret_cast<uintptr_t>(vf) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0)
    token_scores_kernel<true, KMAX><<<sx_ceil_div(T, 8), 256, 0, st>>>(vf, W, T, N, F, K, out);
  else
    token_scores_kernel<false, KMAX><<<sx_ceil_div(T, 8), 256, 0, st>>>(vf, W, T, N, F, K, out);
}

extern "C" int sx_token_scores(const float* vf, const float* W, int32_t B, int32_t N, int32_t F, int32_t K, float* out,
                               void* stream) {
  SX_REQUIRE(K >= 1 && K <= MAXROWS, "sx_token_scores: rows %d not in 1..%d", K, MAXROWS);
  const long long T = (long long)B * N;
  if (K <= MAXK)
    token_scores_launch<MAXK>(vf, W, T, N, F, K, out, ST(stream));
  else if (K <= 16)
    token_scores_launch<16>(vf, W, T, N, F, K, out, ST(stream));
  else
    token_scores_launch<MAXROWS>(vf, W, T, N, F, K, out, ST(stream));
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_token_scores_bwd(const float* dt, const float* W, int32_t B, int32_t N, int32_t F, int32_t K, float* dvf,
                                   void* stream) {
  SX_REQUIRE(dt && W && dvf && B >= 1 && N >= 1 && F >= 1, "sx_token_scores_bwd: bad arguments");
  SX_REQUIRE(K >= 1 && K <= MAXROWS, "sx_token_scores_bwd: rows %d not in 1..%d", K, MAXROWS);
  SX_REQUIRE(F % 4 == 0 && (reinterpret_cast<uintptr_t>(dvf) & 15) == 0 && (reinterpret_cast<uintptr_t>(W) & 15) == 0,
             "sx_token_scores_bwd: F must be a multiple of 4 and W/dvf 16-byte aligned");
  const long long T = (long long)B * N, total = T * (F / 4);
  const int grid = (int)std::min<long long>(sx_ceil_div(total, 256), sm_count_cached() * 16ll);
  if (K <= MAXK)
    token_scores_bwd_kernel<MAXK><<<grid, 256, 0, ST(stream)>>>(dt, W, T, N, F, K, dvf);
  else if (K <= 16)
    token_scores_bwd_kernel<16><<<grid, 256, 0, ST(stream)>>>(dt, W, T, N, F, K, dvf);
  else
    token_scores_bwd_kernel<MAXROWS><<<grid, 256, 0, ST(stream)>>>(dt, W, T, N, F, K, dvf);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

static bool subpixel_shape_ok(int32_t B, int32_t K, int32_t D2, int32_t H2, int32_t W2, int32_t H, int32_t W, int32_t D) {
  return B >= 1 && K >= 1 && (long long)B * K <= 65535 && D2 >= 1 && H2 >= 1 && W2 >= 1 && H >= 1 && W >= 1 && D >= 1 &&
         (long long)H * W * D < (1ll << 31) && 4ll * H2 * W2 * D2 < (1ll << 31);
}

extern "C" int sx_subpixel_resize_fwd(const float* S, const float* bias, int32_t B, int32_t K, int32_t D2, int32_t H2,
                                      int32_t W2, int32_t H, int32_t W, int32_t D, float* out, void* stream) {
  SX_REQUIRE(S && out && subpixel_shape_ok(B, K, D2, H2, W2, H, W, D), "sx_subpixel_resize_fwd: bad arguments");
  const long long per = (long long)H * W * D;
  const int gx = (int)std::max<long long>(1, std::min<long long>(sx_ceil_div(per, 256),
                                                                 sm_count_cached() * 16ll / (B * K) + 1));
  subpixel_resize_fwd_kernel<<<dim3(gx, B * K), 256, 0, ST(stream)>>>(S, bias, K, D2, H2, W2, H, W, D, out);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_subpixel_resize_bwd(const float* dout, int32_t B, int32_t K, int32_t D2, int32_t H2, int32_t W2,
                                      int32_t H, int32_t W, int32_t D, float* dS, void* stream) {
  SX_REQUIRE(dout && dS && subpixel_shape_ok(B, K, D2, H2, W2, H, W, D), "sx_subpixel_resize_bwd: bad arguments");
  const long long cells = 4ll * H2 * W2 * D2;
  subpixel_resize_bwd_kernel<<<dim3(sx_ceil_div(cells, 128), B * K), 128, 0, ST(stream)>>>(dout, D2, H2, W2, H, W, D, dS);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
