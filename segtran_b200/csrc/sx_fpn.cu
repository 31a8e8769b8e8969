// FPN pyramid pieces either side of the hot path (SURVEY.md §8 f.1; segtran3d.py:299-313, :347-359, segtran2d.py:244-300):
// GroupNorm on channels-first tensors.  The 1x1 convolution + bias + "add the upsampled coarser level" of a pyramid stage is
// one sx_gemm launch (W [Cout x Cin] times the channels-first activation read as an MN-major operand, bias per output
// row, addend = the upsampled level); GroupNorm(G) then needs one reduction pass and one apply pass.
//
// x: [B, C, V] fp32, V = prod(spatial).  A group = C/G consecutive channels = one contiguous block of (C/G) V floats.
//   forward : per-(b,c) sum / sum of squares (fp64 atomics) -> per-(b,g) mean / rstd -> y = (x - mean) rstd gamma_c + beta_c
//   backward: per-(b,c) S1 = sum dy, S2 = sum dy xhat -> per-(b,g) c1 = sum_c gamma_c S1 / m, c2 = sum_c gamma_c S2 / m
//             dx = rstd (gamma_c dy - c1 - xhat c2);   dgamma_c += sum_b S2, dbeta_c += sum_b S1      (m = (C/G) V)
#include <algorithm>

#include "../../include/segtran_b200.h"
#include "sx_common.cuh"

namespace {

__device__ __forceinline__ float block_sum256(float v, float* red) {
  v = sx::warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  v = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
  if (w == 0) v = sx::warp_sum(v);
  return v;
}

// grid (chunks, B*C): csum[(b*C+c)*2 + {0,1}] += {sum x, sum x^2} of this chunk of the channel row
__global__ void __launch_bounds__(256)
gn_channel_sums_kernel(const float* __restrict__ x, long long V, double* __restrict__ csum, int vec4) {
  __shared__ float red[32];
  const float* xr = x + (long long)blockIdx.y * V;
  float s = 0.f, q = 0.f;
  if (vec4) {
    const long long V4 = V >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V4; i += (long long)gridDim.x * blockDim.x) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(xr) + i);
      s += (a.x + a.y) + (a.z + a.w);
      q += (a.x * a.x + a.y * a.y) + (a.z * a.z + a.w * a.w);
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (long long)gridDim.x * blockDim.x) {
      const float a = xr[i];
      s += a;
      q = fmaf(a, a, q);
    }
  }
  s = block_sum256(s, red);
  q = block_sum256(q, red);
  if (threadIdx.x == 0) {
    atomicAdd(&csum[blockIdx.y * 2 + 0], (double)s);
    atomicAdd(&csum[blockIdx.y * 2 + 1], (double)q);
  }
}

__global__ void gn_finalize_kernel(const double* __restrict__ csum, int B, int C, int G, long long V, float eps,
                                   float* __restrict__ stats) {
  const int Cg = C / G;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < B * G; i += gridDim.x * blockDim.x) {
    const int b = i / G, g = i % G;
    double s = 0.0, q = 0.0;
    for (int c = g * Cg; c < (g + 1) * Cg; ++c) {
      s += csum[((long long)b * C + c) * 2];
      q += csum[((long long)b * C + c) * 2 + 1];
    }
    const double m = (double)Cg * (double)V;
    const double mean = s / m;
    double var = q / m - mean * mean;                          // biased variance, like nn.GroupNorm
    if (var < 0.0) var = 0.0;
    stats[i * 2] = (float)mean;
    stats[i * 2 + 1] = (float)(1.0 / sqrt(var + (double)eps));
  }
}

__global__ void __launch_bounds__(256)
gn_apply_kernel(const float* __restrict__ x, int C, int G, long long V, const float* __restrict__ gamma,
                const float* __restrict__ beta, const float* __restrict__ stats, float* __restrict__ y, int rnd, int vec4) {
  const int bc = blockIdx.y, c = bc % C, b = bc / C;
  const int g = c / (C / G);
  const float mean = stats[(b * G + g) * 2], rstd = stats[(b * G + g) * 2 + 1];
  const float sc = rstd * (gamma ? gamma[c] : 1.f), sh = (beta ? beta[c] : 0.f) - mean * sc;
  const float* xr = x + (long long)bc * V;
  float* yr = y + (long long)bc * V;
  if (vec4) {
    const long long V4 = V >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V4; i += (long long)gridDim.x * blockDim.x) {
      const float4 a = __ldcs(reinterpret_cast<const float4*>(xr) + i);
      float4 o = make_float4(fmaf(a.x, sc, sh), fmaf(a.y, sc, sh), fmaf(a.z, sc, sh), fmaf(a.w, sc, sh));
      if (rnd) { o.x = sx::round_tf32(o.x); o.y = sx::round_tf32(o.y); o.z = sx::round_tf32(o.z); o.w = sx::round_tf32(o.w); }
      reinterpret_cast<float4*>(yr)[i] = o;
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (long long)gridDim.x * blockDim.x) {
      const float o = fmaf(xr[i], sc, sh);
      yr[i] = rnd ? sx::round_tf32(o) : o;
    }
  }
}

// grid (chunks, B*C): csum[(b*C+c)*2 + {0,1}] += {sum dy, sum dy xhat}
__global__ void __launch_bounds__(256)
gn_bwd_channel_sums_kernel(const float* __restrict__ dy, const float* __restrict__ x, int C, int G, long long V,
                           const float* __restrict__ stats, double* __restrict__ csum, int vec4) {
  __shared__ float red[32];
  const int bc = blockIdx.y, c = bc % C, b = bc / C;
  const int g = c / (C / G);
  const float mean = stats[(b * G + g) * 2], rstd = stats[(b * G + g) * 2 + 1];
  const float* xr = x + (long long)bc * V;
  const float* dr = dy + (long long)bc * V;
  float s1 = 0.f, s2 = 0.f;
  if (vec4) {
    const long long V4 = V >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V4; i += (long long)gridDim.x * blockDim.x) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(xr) + i);
      const float4 d = __ldg(reinterpret_cast<const float4*>(dr) + i);
      s1 += (d.x + d.y) + (d.z + d.w);
      s2 += (d.x * (a.x - mean) + d.y * (a.y - mean)) + (d.z * (a.z - mean) + d.w * (a.w - mean));
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (long long)gridDim.x * blockDim.x) {
      s1 += dr[i];
      s2 = fmaf(dr[i], xr[i] - mean, s2);
    }
  }
  s1 = block_sum256(s1, red);
  s2 = block_sum256(s2, red) * rstd;
  if (threadIdx.x == 0) {
    atomicAdd(&csum[bc * 2 + 0], (double)s1);
    atomicAdd(&csum[bc * 2 + 1], (double)s2);
  }
}

__global__ void gn_bwd_finalize_kernel(const double* __restrict__ csum, int B, int C, int G, long long V,
                                       const float* __restrict__ gamma, float* __restrict__ coef,
                                       float* __restrict__ dgamma, float* __restrict__ dbeta) {
  const int Cg = C / G;
  const int tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
  for (int i = tid; i < B * G; i += nth) {
    const int b = i / G, g = i % G;
    double a = 0.0, q = 0.0;
    for (int c = g * Cg; c < (g + 1) * Cg; ++c) {
      const double gm = gamma ? (double)gamma[c] : 1.0;
      a += gm * csum[((long long)b * C + c) * 2];
      q += gm * csum[((long long)b * C + c) * 2 + 1];
    }
    const double m = (double)Cg * (double)V;
    coef[i * 2] = (float)(a / m);
    coef[i * 2 + 1] = (float)(q / m);
  }
  for (int c = tid; c < C; c += nth) {
    double s1 = 0.0, s2 = 0.0;
    for (int b = 0; b < B; ++b) {
      s1 += csum[((long long)b * C + c) * 2];
      s2 += csum[((long long)b * C + c) * 2 + 1];
    }
    if (dbeta) dbeta[c] += (float)s1;
    if (dgamma) dgamma[c] += (float)s2;
  }
}

__global__ void __launch_bounds__(256)
gn_bwd_apply_kernel(const float* __restrict__ dy, const float* __restrict__ x, int C, int G, long long V,
                    const float* __restrict__ gamma, const float* __restrict__ stats, const float* __restrict__ coef,
                    float* __restrict__ dx, int vec4) {
  const int bc = blockIdx.y, c = bc % C, b = bc / C;
  const int g = c / (C / G);
  const float mean = stats[(b * G + g) * 2], rstd = stats[(b * G + g) * 2 + 1];
  const float c1 = coef[(b * G + g) * 2], c2 = coef[(b * G + g) * 2 + 1];
  const float gm = gamma ? gamma[c] : 1.f;
  // dx = rstd (gm dy - c1 - xhat c2) = (rstd gm) dy - (rstd^2 c2) x + rstd (mean rstd c2 - c1)
  const float k_dy = rstd * gm, k_x = -rstd * rstd * c2, k_0 = rstd * (mean * rstd * c2 - c1);
  const float* xr = x + (long long)bc * V;
  const float* dr = dy + (long long)bc * V;
  float* o = dx + (long long)bc * V;
  if (vec4) {
    const long long V4 = V >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V4; i += (long long)gridDim.x * blockDim.x) {
      const float4 a = __ldcs(reinterpret_cast<const float4*>(xr) + i);
      const float4 d = __ldcs(reinterpret_cast<const float4*>(dr) + i);
      reinterpret_cast<float4*>(o)[i] = make_float4(fmaf(k_dy, d.x, fmaf(k_x, a.x, k_0)), fmaf(k_dy, d.y, fmaf(k_x, a.y, k_0)),
                                                    fmaf(k_dy, d.z, fmaf(k_x, a.z, k_0)), fmaf(k_dy, d.w, fmaf(k_x, a.w, k_0)));
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (long long)gridDim.x * blockDim.x)
      o[i] = fmaf(k_dy, dr[i], fmaf(k_x, xr[i], k_0));
  }
}

int chunks_for(long long work, int rows) {
  const long long want = std::max<long long>(1, (sm_count_cached() * 16ll) / std::max(rows, 1));
  return (int)std::max<long long>(1, std::min<long long>(sx_ceil_div(work, 256 * 4), want));
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int sx_groupnorm_fwd(const float* x, int32_t B, int32_t C, int64_t V, int32_t G, const float* gamma,
                                const float* beta, float eps, double* csum, float* stats, float* y, int32_t round_tf32,
                                void* stream) {
  SX_REQUIRE(x && csum && stats && y && B >= 1 && C >= 1 && V >= 1 && G >= 1 && C % G == 0,
             "sx_groupnorm_fwd: bad arguments (C=%d must be a multiple of G=%d)", C, G);
  SX_CHECK_CUDA(cudaMemsetAsync(csum, 0, sizeof(double) * 2 * B * C, ST(stream)));
  const int vec4 = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && ((reinterpret_cast<uintptr_t>(y) & 15) == 0);
  dim3 grid(chunks_for(vec4 ? V / 4 : V, B * C), B * C);
  gn_channel_sums_kernel<<<grid, 256, 0, ST(stream)>>>(x, V, csum, vec4);
  SX_CHECK_CUDA(cudaGetLastError());
  gn_finalize_kernel<<<sx_ceil_div(B * G, 128), 128, 0, ST(stream)>>>(csum, B, C, G, V, eps, stats);
  SX_CHECK_CUDA(cudaGetLastError());
  gn_apply_kernel<<<grid, 256, 0, ST(stream)>>>(x, C, G, V, gamma, beta, stats, y, round_tf32, vec4);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_groupnorm_bwd(const float* dy, const float* x, int32_t B, int32_t C, int64_t V, int32_t G,
                                const float* gamma, const float* stats, double* csum, float* coef, float* dx,
                                float* dgamma, float* dbeta, void* stream) {
  SX_REQUIRE(dy && x && stats && csum && coef && dx && B >= 1 && C >= 1 && V >= 1 && G >= 1 && C % G == 0,
             "sx_groupnorm_bwd: bad arguments");
  SX_CHECK_CUDA(cudaMemsetAsync(csum, 0, sizeof(double) * 2 * B * C, ST(stream)));
  const int vec4 = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(dy) & 15) == 0) && ((reinterpret_cast<uintptr_t>(dx) & 15) == 0);
  dim3 grid(chunks_for(vec4 ? V / 4 : V, B * C), B * C);
  gn_bwd_channel_sums_kernel<<<grid, 256, 0, ST(stream)>>>(dy, x, C, G, V, stats, csum, vec4);
  SX_CHECK_CUDA(cudaGetLastError());
  gn_bwd_finalize_kernel<<<sx_ceil_div(std::max(B * G, C), 128), 128, 0, ST(stream)>>>(csum, B, C, G, V, gamma, coef, dgamma,
                                                                                        dbeta);
  SX_CHECK_CUDA(cudaGetLastError());
  gn_bwd_apply_kernel<<<grid, 256, 0, ST(stream)>>>(dy, x, C, G, V, gamma, stats, coef, dx, vec4);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
