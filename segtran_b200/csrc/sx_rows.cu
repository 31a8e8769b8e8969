// Row-wise (HBM-bound) kernels of the hot path: positional code, fused prologue, softmax, LayerNorm,
// LayerNorm + learned soft-aggregation over modes, GELU backward, casts and column reductions.
// One warp owns one row; rows are staged once in shared memory and re-read from there, so every
// tensor is read from HBM exactly once and written once.  All statistics are fp32.
#include <algorithm>

#include "sx_common.cuh"
#include "sx_part.cuh"
#include "sx_posbias.cuh"

namespace {

constexpr int ROW_WARPS = 8;
constexpr float LN_EPS = 1e-12f;     // every LayerNorm on the path (segtran_shared.py:263, :371, :885, :888, :984)

__device__ __forceinline__ float rnd1(float v, int rnd) { return rnd ? sx::round_tf32(v) : v; }

// Adds the warps' accumulator rows (row pitch `pitch` floats, the first n of each) in warp order and stores the CTA's
// sums in its slot (blockIdx.x, pitch n) of `part`: the fixed-order column sums of the warp-per-row backward kernels.
__device__ __forceinline__ void warps_to_slot(const float* sm, int warps, long long pitch, int n, float* __restrict__ part) {
  __syncthreads();
  for (int c = threadIdx.x; c < n; c += blockDim.x) {
    float v = 0.f;
    for (int w = 0; w < warps; ++w) v += sm[w * pitch + c];
    part[(long long)blockIdx.x * n + c] = v;
  }
}

__device__ __forceinline__ void warp_mean_rstd(const float* row, int C, int lane, float& mean, float& rstd) {
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s += row[c];
  mean = sx::warp_sum(s) / C;
  float v = 0.f;
  for (int c = lane; c < C; c += 32) { const float d = row[c] - mean; v += d * d; }
  rstd = rsqrtf(sx::warp_sum(v) / C + LN_EPS);
}

// ------------------------------------------------------------------------------------------------
// max over a small tensor (voxels_pos.max(), segtran_shared.py:1231)
// ------------------------------------------------------------------------------------------------
__global__ void reduce_max_kernel(const float* x, long long n, float* out) {
  float m = -3.0e38f;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, x[i]);
  m = sx::warp_max(m);
  __shared__ float s[32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? s[threadIdx.x] : -3.0e38f;
    m = sx::warp_max(m);
    if (threadIdx.x == 0) *out = m;
  }
}

// ------------------------------------------------------------------------------------------------
// learnable-sinusoid positional code (segtran_shared.py:989-998): rows = positions
//   e = (pos/posmax) W^T + b ; even cols sin, odd cols cos ; LayerNorm without affine
// ------------------------------------------------------------------------------------------------
__global__ void pos_lsinu_fwd_kernel(const float* __restrict__ pos, const float* __restrict__ posmax, int R, int pd,
                                     const float* __restrict__ W, const float* __restrict__ b, int C,
                                     float* __restrict__ pe) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* row = sm + warp * C;
  const float inv = 1.f / *posmax;
  for (int r = blockIdx.x * ROW_WARPS + warp; r < R; r += gridDim.x * ROW_WARPS) {
    float pn[3] = {0.f, 0.f, 0.f};
    for (int j = 0; j < pd; ++j) pn[j] = pos[(long long)r * pd + j] * inv;
    for (int c = lane; c < C; c += 32) {
      float e = b[c];
      for (int j = 0; j < pd; ++j) e += pn[j] * W[c * pd + j];
      row[c] = (c & 1) ? cosf(e) : sinf(e);
    }
    __syncwarp();
    float mean, rstd;
    warp_mean_rstd(row, C, lane, mean, rstd);
    for (int c = lane; c < C; c += 32) pe[(long long)r * C + c] = (row[c] - mean) * rstd;
    __syncwarp();
  }
}

// backward: dpe [R,C] -> de [R,C] (gradient w.r.t. the pre-activation e); column reductions follow.
__global__ void pos_lsinu_bwd_kernel(const float* __restrict__ pos, const float* __restrict__ posmax, int R, int pd,
                                     const float* __restrict__ W, const float* __restrict__ b, int C,
                                     const float* __restrict__ dpe, float* __restrict__ de) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* row = sm + warp * 2 * C;      // [C] activations, [C] d/de of activation
  float* dact = row + C;
  const float inv = 1.f / *posmax;
  for (int r = blockIdx.x * ROW_WARPS + warp; r < R; r += gridDim.x * ROW_WARPS) {
    float pn[3] = {0.f, 0.f, 0.f};
    for (int j = 0; j < pd; ++j) pn[j] = pos[(long long)r * pd + j] * inv;
    for (int c = lane; c < C; c += 32) {
      float e = b[c];
      for (int j = 0; j < pd; ++j) e += pn[j] * W[c * pd + j];
      float s, co;
      sincosf(e, &s, &co);
      row[c] = (c & 1) ? co : s;
      dact[c] = (c & 1) ? -s : co;
    }
    __syncwarp();
    float mean, rstd;
    warp_mean_rstd(row, C, lane, mean, rstd);
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float g = dpe[(long long)r * C + c], yh = (row[c] - mean) * rstd;
      s1 += g; s2 += g * yh;
    }
    s1 = sx::warp_sum(s1) / C; s2 = sx::warp_sum(s2) / C;
    for (int c = lane; c < C; c += 32) {
      const float g = dpe[(long long)r * C + c], yh = (row[c] - mean) * rstd;
      de[(long long)r * C + c] = rstd * (g - s1 - yh * s2) * dact[c];
    }
    __syncwarp();
  }
}

// dW[c*pd + j] += sum_r de[r,c] * pos[r,j]/posmax   (j < pd) ; db[c] += sum_r de[r,c]  (slot blockIdx.y of `part`)
__global__ void pos_param_grad_kernel(const float* __restrict__ de, const float* __restrict__ pos,
                                      const float* __restrict__ posmax, int R, int pd, int C, float* __restrict__ part) {
  const int c = blockIdx.x * 32 + threadIdx.x;      // blockDim = (32, 8)
  const float inv = 1.f / *posmax;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  if (c < C)
    for (int r = blockIdx.y * blockDim.y + threadIdx.y; r < R; r += gridDim.y * blockDim.y) {
      const float g = de[(long long)r * C + c];
      acc[3] += g;
      for (int j = 0; j < pd; ++j) acc[j] += g * pos[(long long)r * pd + j] * inv;
    }
  __shared__ float s[8][4][33];
  for (int j = 0; j < 4; ++j) s[threadIdx.y][j][threadIdx.x] = acc[j];
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {                // slot blockIdx.y: [dW (C*pd) | db (C)]
    float* slot = part + (long long)blockIdx.y * (C * pd + C);
    for (int j = 0; j < 4; ++j) {
      float t = 0.f;
      for (int y = 0; y < 8; ++y) t += s[y][j][threadIdx.x];
      if (j == 3) slot[C * pd + c] = t;
      else if (j < pd) slot[c * pd + j] = t;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// fused prologue (segtran_shared.py:916, :930-934, :944-946):
//   h = mask * dropout( LN( LN_{g,b}(x) + posw * pe[:, :C] ) )
// ------------------------------------------------------------------------------------------------
__global__ void prologue_fwd_kernel(const float* __restrict__ x, long long R, int N, int C, const float* __restrict__ g,
                                    const float* __restrict__ b, const float* __restrict__ pe, int C0,
                                    long long pe_bstride, float posw, const float* __restrict__ mask, float drop_p,
                                    unsigned long long seed, const unsigned long long* __restrict__ seed_dev, float* __restrict__ h, float* __restrict__ stats, int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* row = sm + warp * C;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = (long long)blockIdx.x * ROW_WARPS + warp; r < R; r += (long long)gridDim.x * ROW_WARPS) {
    const float* xr = x + r * C;
    for (int c = lane; c < C; c += 32) row[c] = xr[c];
    __syncwarp();
    float m1, r1;
    warp_mean_rstd(row, C, lane, m1, r1);
    const long long bi = r / N, ni = r % N;
    const float* per = pe + bi * pe_bstride + ni * C0;
    for (int c = lane; c < C; c += 32) row[c] = (row[c] - m1) * r1 * g[c] + b[c] + posw * per[c];
    __syncwarp();
    float m2, r2;
    warp_mean_rstd(row, C, lane, m2, r2);
    const float mk = mask ? mask[r] : 1.f;
    float* hr = h + r * C;
    for (int c = lane; c < C; c += 32) {
      float v = (row[c] - m2) * r2 * mk;
      if (drop_p > 0.f) v = sx::drop_keep1(seed, (unsigned long long)(r * C + c), sx::drop_p16(drop_p)) ? v * keep_scale : 0.f;
      hr[c] = rnd1(v, rnd);
    }
    if (lane == 0) {
      stats[r * 4 + 0] = m1; stats[r * 4 + 1] = r1; stats[r * 4 + 2] = m2; stats[r * 4 + 3] = r2;
    }
    __syncwarp();
  }
}

// backward of the fused prologue for the widths and views prologue_bwd_cta rejects.  dh fp32 [R,C] -> dx [R,C], and
// dt [R,C] = the gradient at the inner LayerNorm's input, which pos_grad_from_dt reduces into dpe (dt_out may be NULL
// when no dpe is wanted).  dg / db: one accumulator row per warp (a lane owns the columns c = lane mod 32), the warps
// added in order into the CTA's slot of `part`, as in prologue_nopos_bwd_kernel.
__global__ void prologue_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ x, long long R, int N,
                                    int C, const float* __restrict__ g, const float* __restrict__ b,
                                    const float* __restrict__ pe, int C0, long long pe_bstride, float posw,
                                    const float* __restrict__ mask, float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                                    const float* __restrict__ stats, float* __restrict__ dx, float* __restrict__ dt_out,
                                    float* __restrict__ part) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  extern __shared__ float sm[];
  const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* acc = sm + (long long)warp * 5 * C;  // per warp: dg [C], db [C], yhat1 [C], yhat2 [C], d [C]
  float* y1 = acc + 2 * C;
  float* y2 = y1 + C;
  float* dd = y2 + C;
  for (int c = lane; c < 2 * C; c += 32) acc[c] = 0.f;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = (long long)blockIdx.x * warps + warp; r < R; r += (long long)gridDim.x * warps) {
    const float m1 = stats[r * 4 + 0], r1 = stats[r * 4 + 1], m2 = stats[r * 4 + 2], r2 = stats[r * 4 + 3];
    const long long bi = r / N, ni = r % N;
    const float* per = pe + bi * pe_bstride + ni * C0;
    const float mk = mask ? mask[r] : 1.f;
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float a = (x[r * C + c] - m1) * r1;
      const float t = a * g[c] + b[c] + posw * per[c];
      const float yh = (t - m2) * r2;
      float d = dh[r * C + c] * mk;
      if (drop_p > 0.f) d = sx::drop_keep1(seed, (unsigned long long)(r * C + c), sx::drop_p16(drop_p)) ? d * keep_scale : 0.f;
      y1[c] = a; y2[c] = yh; dd[c] = d;
      s1 += d; s2 += d * yh;
    }
    s1 = sx::warp_sum(s1) / C; s2 = sx::warp_sum(s2) / C;
    float s3 = 0.f, s4 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float dt = r2 * (dd[c] - s1 - y2[c] * s2);
      acc[c] += dt * y1[c];
      acc[C + c] += dt;
      if (dt_out) dt_out[r * C + c] = dt;
      const float da = dt * g[c];
      dd[c] = da;
      s3 += da; s4 += da * y1[c];
    }
    s3 = sx::warp_sum(s3) / C; s4 = sx::warp_sum(s4) / C;
    for (int c = lane; c < C; c += 32) dx[r * C + c] = r1 * (dd[c] - s3 - y1[c] * s4);
    __syncwarp();
  }
  warps_to_slot(sm, warps, 5ll * C, 2 * C, part);
}

// ------------------------------------------------------------------------------------------------
// softmax over rows with the reference's conditional clamp (segtran_shared.py:578-580, :601-605)
//   if (*amax > clip) S = clamp(S, -clip, clip);  P = softmax(S);  Pd = dropout(P)
// ------------------------------------------------------------------------------------------------
__global__ void softmax_fwd_kernel(const float* __restrict__ S, long long R, int L, long long lds,
                                   const float* __restrict__ amax, float clip, float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                                   float* __restrict__ P, long long ldp, float* __restrict__ lse, int rnd,
                                   float* __restrict__ diag) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  extern __shared__ float sm[];
  const int warps = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* row = sm + (long long)warp * L;
  const bool do_clip = amax && (*amax > clip);
  if (diag && amax && blockIdx.x == 0 && threadIdx.x == 0) {
    diag[0] = fmaxf(diag[0], *amax);
    if (do_clip) diag[1] += 1.f;
  }
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = (long long)blockIdx.x * warps + warp; r < R; r += (long long)gridDim.x * warps) {
    const float* sr = S + r * lds;
    float m = -3.0e38f;
    for (int c = lane; c < L; c += 32) {
      float v = sr[c];
      if (do_clip) v = fminf(fmaxf(v, -clip), clip);
      row[c] = v;
      m = fmaxf(m, v);
    }
    m = sx::warp_max(m);
    float s = 0.f;
    for (int c = lane; c < L; c += 32) { const float e = __expf(row[c] - m); row[c] = e; s += e; }
    s = sx::warp_sum(s);
    const float inv = 1.f / s;
    float* pr = P + r * ldp;
    for (int c = lane; c < L; c += 32) {
      float v = row[c] * inv;
      if (drop_p > 0.f) v = sx::drop_keep1(seed, (unsigned long long)(r * ldp + c), sx::drop_p16(drop_p)) ? v * keep_scale : 0.f;
      pr[c] = rnd1(v, rnd);
    }
    if (lane == 0 && lse) lse[r] = m + __logf(s);
    __syncwarp();
  }
}

// dS = P * (g - sum_j P_j g_j) with g = dPd * keep/(1-p); zero where the clamp was active.
__global__ void softmax_bwd_kernel(const float* __restrict__ dP, long long ldd, const float* __restrict__ S,
                                   long long lds, const float* __restrict__ lse, long long R, int L,
                                   const float* __restrict__ amax, float clip, float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                                   long long ldp_fwd, float* __restrict__ dS, long long ldo, int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  extern __shared__ float sm[];
  const int warps = blockDim.x >> 5;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* prow = sm + (long long)warp * 2 * L;
  float* grow = prow + L;
  const bool do_clip = amax && (*amax > clip);
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = (long long)blockIdx.x * warps + warp; r < R; r += (long long)gridDim.x * warps) {
    const float l = lse[r];
    float dot = 0.f;
    for (int c = lane; c < L; c += 32) {
      float v = S[r * lds + c];
      if (do_clip) v = fminf(fmaxf(v, -clip), clip);
      const float pv = __expf(v - l);
      float gv = dP[r * ldd + c];
      if (drop_p > 0.f)
        gv = sx::drop_keep1(seed, (unsigned long long)(r * ldp_fwd + c), sx::drop_p16(drop_p)) ? gv * keep_scale : 0.f;
      prow[c] = pv; grow[c] = gv;
      dot += pv * gv;
    }
    dot = sx::warp_sum(dot);
    for (int c = lane; c < L; c += 32) {
      float d = prow[c] * (grow[c] - dot);
      if (do_clip) { const float v = S[r * lds + c]; if (v < -clip || v > clip) d = 0.f; }
      dS[r * ldo + c] = rnd1(d, rnd);
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// prologue without a positional code (pos_code_type 'bias' / 'none', segtran_shared.py:916, :940, :944-946):
//   h = mask * dropout( LN_{g,b}(x) ),  stats[r] = {mean, rstd, 0, 1}
// One warp per row.  The backward keeps one dg / db accumulator row per warp (a lane owns the columns c = lane mod 32,
// so there are no atomics), adds the warps in order and stores the CTA's sums in its slot of `part`.
// ------------------------------------------------------------------------------------------------
constexpr int NOPOS_WARPS = 4;

__global__ void __launch_bounds__(NOPOS_WARPS * 32)
prologue_nopos_fwd_kernel(const float* __restrict__ x, long long R, int C, const float* __restrict__ g,
                          const float* __restrict__ b, const float* __restrict__ mask, float drop_p, unsigned long long seed,
                          const unsigned long long* __restrict__ seed_dev, float* __restrict__ h, float* __restrict__ stats, int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = (long long)blockIdx.x * NOPOS_WARPS + warp; r < R; r += (long long)gridDim.x * NOPOS_WARPS) {
    const float* xr = x + r * C;
    float m1, r1;
    warp_mean_rstd(xr, C, lane, m1, r1);
    const float mk = mask ? mask[r] : 1.f;
    float* hr = h + r * C;
    for (int c = lane; c < C; c += 32) {
      float v = ((xr[c] - m1) * r1 * g[c] + b[c]) * mk;
      if (drop_p > 0.f) v = sx::drop_keep1(seed, (unsigned long long)(r * C + c), sx::drop_p16(drop_p)) ? v * keep_scale : 0.f;
      hr[c] = rnd1(v, rnd);
    }
    if (lane == 0) {
      stats[r * 4 + 0] = m1; stats[r * 4 + 1] = r1; stats[r * 4 + 2] = 0.f; stats[r * 4 + 3] = 1.f;
    }
  }
}

__global__ void __launch_bounds__(NOPOS_WARPS * 32)
prologue_nopos_bwd_kernel(const float* __restrict__ dh, const float* __restrict__ x, long long R, int C,
                          const float* __restrict__ g, const float* __restrict__ mask, float drop_p, unsigned long long seed,
                          const unsigned long long* __restrict__ seed_dev, const float* __restrict__ stats,
                          float* __restrict__ dx, float* __restrict__ part) {
  seed += seed_dev ? *seed_dev : 0ull;
  extern __shared__ float sm[];                     // [NOPOS_WARPS][2C]: dg | db per warp
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* acc = sm + (long long)warp * 2 * C;
  for (int c = lane; c < 2 * C; c += 32) acc[c] = 0.f;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = (long long)blockIdx.x * NOPOS_WARPS + warp; r < R; r += (long long)gridDim.x * NOPOS_WARPS) {
    const float m1 = stats[r * 4 + 0], r1 = stats[r * 4 + 1];
    const float mk = mask ? mask[r] : 1.f;
    const float* xr = x + r * C;
    const float* dr = dh + r * C;
    auto dy_at = [&](int c) {
      float d = dr[c] * mk;
      if (drop_p > 0.f) d = sx::drop_keep1(seed, (unsigned long long)(r * C + c), sx::drop_p16(drop_p)) ? d * keep_scale : 0.f;
      return d;
    };
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float xh = (xr[c] - m1) * r1, dy = dy_at(c);
      acc[c] += dy * xh;
      acc[C + c] += dy;
      const float da = dy * g[c];
      s1 += da; s2 += da * xh;
    }
    s1 = sx::warp_sum(s1) / C; s2 = sx::warp_sum(s2) / C;
    for (int c = lane; c < C; c += 32) {
      const float xh = (xr[c] - m1) * r1;
      dx[r * C + c] = r1 * (dy_at(c) * g[c] - s1 - xh * s2);
    }
  }
  warps_to_slot(sm, NOPOS_WARPS, 2ll * C, 2 * C, part);
}

// ------------------------------------------------------------------------------------------------
// softmax with a sliding-window positional bias (segtran_shared.py:578-605): one CTA per row, the row staged in shared
// memory.  The bias is applied by walking the (2R+1)^pd window offsets of the row's query (each offset addresses at
// most one key), and the backward gathers the row's dS' into the CTA's table accumulator the same way — one row at a
// time, so the sums need no atomics; the CTA's table then goes to its slot of `part`.
// ------------------------------------------------------------------------------------------------
constexpr int PB_THREADS = 256;

__device__ __forceinline__ float block_max(float v, float* red) {
  v = sx::warp_max(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float m = red[0];
  for (int w = 1; w < PB_THREADS / 32; ++w) m = fmaxf(m, red[w]);
  __syncthreads();
  return m;
}
__device__ __forceinline__ float block_sum(float v, float* red) {
  v = sx::warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  for (int w = 0; w < PB_THREADS / 32; ++w) s += red[w];
  __syncthreads();
  return s;
}

// row <- clamp_if(S row) + w * bias(q, .)
__device__ __forceinline__ void posbias_stage_row(const float* __restrict__ sr, int L, bool do_clip, float clip,
                                                  const float* __restrict__ table, const sxpb::Geom& G, int q, float* row) {
  for (int c = threadIdx.x; c < L; c += PB_THREADS) {
    float v = sr[c];
    if (do_clip) v = fminf(fmaxf(v, -clip), clip);
    row[c] = v;
  }
  __syncthreads();
  int qc[3];
  sxpb::coords(G, q, qc);
  for (int o = threadIdx.x; o < G.T; o += PB_THREADS) {
    const int k = sxpb::key_of(G, qc, o);
    if (k >= 0) row[k] += G.w * table[o];
  }
  __syncthreads();
}

__global__ void __launch_bounds__(PB_THREADS)
softmax_posbias_fwd_kernel(const float* __restrict__ S, long long R, int L, long long lds, const float* __restrict__ amax,
                           float clip, float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                           float* __restrict__ P, long long ldp, float* __restrict__ lse, int rnd, float* __restrict__ diag,
                           const float* __restrict__ table, const sxpb::Geom G) {
  seed += seed_dev ? *seed_dev : 0ull;
  extern __shared__ float sm[];
  float* red = sm;                                  // [32]
  float* row = sm + 32;                             // [L]
  const bool do_clip = amax && (*amax > clip);
  if (diag && amax && blockIdx.x == 0 && threadIdx.x == 0) {
    diag[0] = fmaxf(diag[0], *amax);
    if (do_clip) diag[1] += 1.f;
  }
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = blockIdx.x; r < R; r += gridDim.x) {
    posbias_stage_row(S + r * lds, L, do_clip, clip, table, G, (int)(r % L), row);
    float m = -3.0e38f;
    for (int c = threadIdx.x; c < L; c += PB_THREADS) m = fmaxf(m, row[c]);
    m = block_max(m, red);
    float s = 0.f;
    for (int c = threadIdx.x; c < L; c += PB_THREADS) { const float e = __expf(row[c] - m); row[c] = e; s += e; }
    s = block_sum(s, red);
    const float inv = 1.f / s;
    float* pr = P + r * ldp;
    for (int c = threadIdx.x; c < L; c += PB_THREADS) {
      float v = row[c] * inv;
      if (drop_p > 0.f) v = sx::drop_keep1(seed, (unsigned long long)(r * ldp + c), sx::drop_p16(drop_p)) ? v * keep_scale : 0.f;
      pr[c] = rnd1(v, rnd);
    }
    if (threadIdx.x == 0 && lse) lse[r] = m + __logf(s);
    __syncthreads();
  }
}

__global__ void __launch_bounds__(PB_THREADS)
softmax_posbias_bwd_kernel(const float* __restrict__ dP, long long ldd, const float* __restrict__ S, long long lds,
                           const float* __restrict__ lse, long long R, int L, const float* __restrict__ amax, float clip,
                           float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                           long long ldp_fwd, float* __restrict__ dS, long long ldo, int rnd, const float* __restrict__ table,
                           const sxpb::Geom G, float* __restrict__ part) {
  seed += seed_dev ? *seed_dev : 0ull;
  extern __shared__ float sm[];
  float* red = sm;                                  // [32]
  float* tab = sm + 32;                             // [T] this CTA's table gradient
  float* prow = tab + G.T;                          // [L] P, recomputed
  float* grow = prow + L;                           // [L] masked dP, then dS'
  for (int o = threadIdx.x; o < G.T; o += PB_THREADS) tab[o] = 0.f;
  const bool do_clip = amax && (*amax > clip);
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = blockIdx.x; r < R; r += gridDim.x) {
    const int q = (int)(r % L);
    posbias_stage_row(S + r * lds, L, do_clip, clip, table, G, q, prow);
    const float l = lse[r];
    float dot = 0.f;
    for (int c = threadIdx.x; c < L; c += PB_THREADS) {
      const float pv = __expf(prow[c] - l);
      float gv = dP[r * ldd + c];
      if (drop_p > 0.f)
        gv = sx::drop_keep1(seed, (unsigned long long)(r * ldp_fwd + c), sx::drop_p16(drop_p)) ? gv * keep_scale : 0.f;
      prow[c] = pv; grow[c] = gv;
      dot += pv * gv;
    }
    dot = block_sum(dot, red);
    for (int c = threadIdx.x; c < L; c += PB_THREADS) {
      const float d = prow[c] * (grow[c] - dot);
      grow[c] = d;
      float o = d;
      if (do_clip) { const float v = S[r * lds + c]; if (v < -clip || v > clip) o = 0.f; }
      dS[r * ldo + c] = rnd1(o, rnd);
    }
    __syncthreads();
    int qc[3];
    sxpb::coords(G, q, qc);
    for (int o = threadIdx.x; o < G.T; o += PB_THREADS) {
      const int k = sxpb::key_of(G, qc, o);
      if (k >= 0) tab[o] += grow[k];
    }
    __syncthreads();
  }
  for (int o = threadIdx.x; o < G.T; o += PB_THREADS) part[(long long)blockIdx.x * G.T + o] = G.w * tab[o];
}

// ------------------------------------------------------------------------------------------------
// LayerNorm with affine over rows (first_norm_layer, segtran_shared.py:456)
// ------------------------------------------------------------------------------------------------
__global__ void layernorm_fwd_kernel(const float* __restrict__ x, long long R, int C, const float* __restrict__ g,
                                     const float* __restrict__ b, float* __restrict__ y, float* __restrict__ stats,
                                     int rnd) {
  extern __shared__ float sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* row = sm + warp * C;
  for (long long r = (long long)blockIdx.x * ROW_WARPS + warp; r < R; r += (long long)gridDim.x * ROW_WARPS) {
    for (int c = lane; c < C; c += 32) row[c] = x[r * C + c];
    __syncwarp();
    float m, rs;
    warp_mean_rstd(row, C, lane, m, rs);
    for (int c = lane; c < C; c += 32) y[r * C + c] = rnd1((row[c] - m) * rs * g[c] + b[c], rnd);
    if (lane == 0) { stats[r * 2] = m; stats[r * 2 + 1] = rs; }
    __syncwarp();
  }
}

// backward for the widths and views layernorm_bwd_rows_fast rejects: per-warp dg | db rows, added in warp order into
// the CTA's slot of `part`
__global__ void layernorm_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, long long R, int C,
                                     const float* __restrict__ g, const float* __restrict__ stats, float* __restrict__ dx,
                                     float* __restrict__ part, int rnd) {
  extern __shared__ float sm[];
  const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* acc = sm + (long long)warp * 4 * C;  // per warp: dg [C], db [C], yhat [C], d [C]
  float* yh = acc + 2 * C;
  float* dd = yh + C;
  for (int c = lane; c < 2 * C; c += 32) acc[c] = 0.f;
  for (long long r = (long long)blockIdx.x * warps + warp; r < R; r += (long long)gridDim.x * warps) {
    const float m = stats[r * 2], rs = stats[r * 2 + 1];
    float s1 = 0.f, s2 = 0.f;
    for (int c = lane; c < C; c += 32) {
      const float a = (x[r * C + c] - m) * rs, d0 = dy[r * C + c];
      acc[c] += d0 * a;
      acc[C + c] += d0;
      const float d = d0 * g[c];
      yh[c] = a; dd[c] = d;
      s1 += d; s2 += d * a;
    }
    s1 = sx::warp_sum(s1) / C; s2 = sx::warp_sum(s2) / C;
    for (int c = lane; c < C; c += 32) dx[r * C + c] = rnd1(rs * (dd[c] - s1 - yh[c] * s2), rnd);
    __syncwarp();
  }
  warps_to_slot(sm, warps, 4ll * C, 2 * C, part);
}

// ------------------------------------------------------------------------------------------------
// MMPrivateOutput tail + LearnedSoftAggregate (segtran_shared.py:273-274, :318-325):
//   Yn_m = LN_{g,b}(dropout(Y_m)) ; w = softmax_m(Yn_m . ws + bs) ; out = sum_m w_m Yn_m
// Y [B,M,N,F] fp32, one warp per token (all M modes), out [B,N,F] fp32.
// ------------------------------------------------------------------------------------------------
constexpr int MAX_MODES = 8;

__global__ void ln_softaggr_fwd_kernel(const float* __restrict__ Y, int B, int M, int N, int F,
                                       const float* __restrict__ g, const float* __restrict__ b,
                                       const float* __restrict__ ws, const float* __restrict__ bs, float drop_p,
                                       unsigned long long seed, const unsigned long long* __restrict__ seed_dev, float* __restrict__ out, float* __restrict__ stats,
                                       float* __restrict__ wts) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  extern __shared__ float sm[];
  const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* rows = sm + (long long)warp * M * F;       // normalised rows of the M modes
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const long long T_ = (long long)B * N;
  for (long long t = (long long)blockIdx.x * warps + warp; t < T_; t += (long long)gridDim.x * warps) {
    const long long bi = t / N, ni = t % N;
    float sc[MAX_MODES];
    for (int m = 0; m < M; ++m) {
      const long long ro = ((bi * M + m) * N + ni);
      const float* yr = Y + ro * F;
      float* row = rows + m * F;
      for (int c = lane; c < F; c += 32) {
        float v = yr[c];
        if (drop_p > 0.f)
          v = sx::drop_keep1(seed, (unsigned long long)(ro * F + c), sx::drop_p16(drop_p)) ? v * keep_scale : 0.f;
        row[c] = v;
      }
      __syncwarp();
      float mean, rstd;
      warp_mean_rstd(row, F, lane, mean, rstd);
      float dot = 0.f;
      for (int c = lane; c < F; c += 32) {
        const float v = (row[c] - mean) * rstd * g[c] + b[c];
        row[c] = v;
        dot += v * ws[c];
      }
      sc[m] = sx::warp_sum(dot) + bs[0];
      if (lane == 0) { stats[ro * 2] = mean; stats[ro * 2 + 1] = rstd; }
    }
    float mx = -3.0e38f;
    for (int m = 0; m < M; ++m) mx = fmaxf(mx, sc[m]);
    float den = 0.f;
    for (int m = 0; m < M; ++m) { sc[m] = __expf(sc[m] - mx); den += sc[m]; }
    for (int m = 0; m < M; ++m) sc[m] /= den;
    if (lane == 0)
      for (int m = 0; m < M; ++m) wts[(bi * M + m) * N + ni] = sc[m];
    __syncwarp();
    for (int c = lane; c < F; c += 32) {
      float o = 0.f;
      for (int m = 0; m < M; ++m) o += sc[m] * rows[m * F + c];
      out[t * F + c] = o;
    }
    __syncwarp();
  }
}

// backward: dout [B,N,F] -> dY [B,M,N,F], plus dg, db, dws [F] and dbs [1]: per-warp rows [dg | db | dws | dbs], added
// in warp order into the CTA's slot of `part`
__global__ void ln_softaggr_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ Y, int B, int M,
                                       int N, int F, const float* __restrict__ g, const float* __restrict__ b,
                                       const float* __restrict__ ws, float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                                       const float* __restrict__ stats, const float* __restrict__ wts,
                                       float* __restrict__ dY, float* __restrict__ part, int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  extern __shared__ float sm[];
  const int warps = blockDim.x >> 5, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* acc = sm + (long long)warp * (5 * F + 1);  // per warp: dg [F], db [F], dws [F], dbs [1], yhat [F], d [F]
  float* sdb = acc + F;
  float* sdw = sdb + F;
  float* yh = sdw + F + 1;
  float* dd = yh + F;
  for (int c = lane; c < 3 * F + 1; c += 32) acc[c] = 0.f;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const long long T_ = (long long)B * N;
  float dbs_acc = 0.f;
  for (long long t = (long long)blockIdx.x * warps + warp; t < T_; t += (long long)gridDim.x * warps) {
    const long long bi = t / N, ni = t % N;
    const float* go = dout + t * F;
    // pass 1: dw_m = <dout, Yn_m>
    float dwm[MAX_MODES], w[MAX_MODES];
    for (int m = 0; m < M; ++m) {
      const long long ro = ((bi * M + m) * N + ni);
      const float mean = stats[ro * 2], rstd = stats[ro * 2 + 1];
      float dot = 0.f;
      for (int c = lane; c < F; c += 32) {
        float v = Y[ro * F + c];
        if (drop_p > 0.f)
          v = sx::drop_keep1(seed, (unsigned long long)(ro * F + c), sx::drop_p16(drop_p)) ? v * keep_scale : 0.f;
        dot += go[c] * ((v - mean) * rstd * g[c] + b[c]);
      }
      dwm[m] = sx::warp_sum(dot);
      w[m] = wts[(bi * M + m) * N + ni];
    }
    float wd = 0.f;
    for (int m = 0; m < M; ++m) wd += w[m] * dwm[m];
    for (int m = 0; m < M; ++m) {
      const float dscore = w[m] * (dwm[m] - wd);        // softmax backward over modes
      dbs_acc += dscore;
      const long long ro = ((bi * M + m) * N + ni);
      const float mean = stats[ro * 2], rstd = stats[ro * 2 + 1];
      float s1 = 0.f, s2 = 0.f;
      for (int c = lane; c < F; c += 32) {
        float v = Y[ro * F + c];
        if (drop_p > 0.f)
          v = sx::drop_keep1(seed, (unsigned long long)(ro * F + c), sx::drop_p16(drop_p)) ? v * keep_scale : 0.f;
        const float a = (v - mean) * rstd;
        const float yn = a * g[c] + b[c];
        const float dyn = w[m] * go[c] + dscore * ws[c];
        sdw[c] += dscore * yn;
        acc[c] += dyn * a;
        sdb[c] += dyn;
        const float d = dyn * g[c];
        yh[c] = a; dd[c] = d;
        s1 += d; s2 += d * a;
      }
      s1 = sx::warp_sum(s1) / F; s2 = sx::warp_sum(s2) / F;
      for (int c = lane; c < F; c += 32) {
        float d = rstd * (dd[c] - s1 - yh[c] * s2);
        if (drop_p > 0.f)
          d = sx::drop_keep1(seed, (unsigned long long)(ro * F + c), sx::drop_p16(drop_p)) ? d * keep_scale : 0.f;
        dY[ro * F + c] = rnd1(d, rnd);
      }
      __syncwarp();
    }
  }
  if (lane == 0) sdw[F] = dbs_acc;            // identical in all lanes of the warp
  warps_to_slot(sm, warps, 5ll * F + 1, 3 * F + 1, part);
}

#include "sx_rows_fast.cuh"
#include "sx_rows_cta.cuh"

// ------------------------------------------------------------------------------------------------
// elementwise helpers
// ------------------------------------------------------------------------------------------------
// dH = dGd * keep/(1-p) * gelu'(H)   (MMSharedMid backward, segtran_shared.py:243-245); GELU = false: dH = dGd * keep/(1-p),
// the backward of a dropout epilogue without an activation (the output Linear of MultiHeadFeatTrans, segtran_ablation.py:137-143)
template <bool GELU>
__global__ void gelu_bwd_kernel(const float* __restrict__ dG, const float* __restrict__ H, long long n, float drop_p,
                                unsigned long long seed, const unsigned long long* __restrict__ seed_dev, float* __restrict__ dH, int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    float d = dG[i];
    if (drop_p > 0.f) d = sx::drop_keep1(seed, (unsigned long long)i, sx::drop_p16(drop_p)) ? d * keep_scale : 0.f;
    if constexpr (GELU) d *= sx::gelu_erf_grad(H[i]);
    dH[i] = rnd1(d, rnd);
  }
}

// fp32 float4 version (n % 4 == 0, 16-byte aligned)
template <bool GELU>
__global__ void gelu_bwd_f4_kernel(const float4* __restrict__ dG, const float4* __restrict__ H, long long n4, float drop_p,
                                   unsigned long long seed, const unsigned long long* __restrict__ seed_dev, float4* __restrict__ dH, int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 d = dG[i];
    if (drop_p > 0.f) d = drop4(d, drop_p, keep_scale, seed, (unsigned long long)(i * 4));
    if constexpr (GELU) {
      const float4 h = H[i];
      d.x *= sx::gelu_erf_grad(h.x); d.y *= sx::gelu_erf_grad(h.y); d.z *= sx::gelu_erf_grad(h.z); d.w *= sx::gelu_erf_grad(h.w);
    }
    dH[i] = rnd4(d, rnd);
  }
}

__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__nv_bfloat16 v) { return __bfloat162float(v); }
__device__ __forceinline__ void store_cvt(float* p, float v, int rnd) { *p = rnd1(v, rnd); }
__device__ __forceinline__ void store_cvt(__nv_bfloat16* p, float v, int) { *p = __float2bfloat16_rn(v); }

template <typename TI, typename TO>
__global__ void convert_kernel(const TI* __restrict__ x, long long n, TO* __restrict__ y, int rnd) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    store_cvt(y + i, to_f32(x[i]), rnd);
}

// ------------------------------------------------------------------------------------------------
// LearnedSoftAggregate on its own (segtran_shared.py:318-325; the no-FFN branch of ExpandedFeatTrans, :453, used by the
// Polyformer layer with M modes):  w = softmax_m(x_m . ws + bs);  out = sum_m w_m x_m.   x [B,M,N,F] -> out [B,N,F].
// One warp per token; rows are streamed (no shared memory), M <= MAX_MODES.
// ------------------------------------------------------------------------------------------------
__global__ void softaggr_fwd_kernel(const float* __restrict__ x, int B, int M, int N, int F, const float* __restrict__ ws,
                                    const float* __restrict__ bs, float* __restrict__ out, float* __restrict__ wts) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  for (long long t = (long long)blockIdx.x * warps + warp; t < (long long)B * N; t += (long long)gridDim.x * warps) {
    const int b = (int)(t / N), n = (int)(t % N);
    float sc[MAX_MODES];
    float mx = -3.0e38f;
    for (int m = 0; m < M; ++m) {
      const float* xr = x + (((long long)b * M + m) * N + n) * F;
      float a = 0.f;
      for (int c = lane; c < F; c += 32) a += xr[c] * ws[c];
      a = sx::warp_sum(a) + bs[0];
      sc[m] = a;
      mx = fmaxf(mx, a);
    }
    float den = 0.f;
    for (int m = 0; m < M; ++m) { sc[m] = __expf(sc[m] - mx); den += sc[m]; }
    const float inv = 1.f / den;
    for (int m = 0; m < M; ++m) {
      sc[m] *= inv;
      if (lane == 0) wts[((long long)b * M + m) * N + n] = sc[m];
    }
    float* o = out + ((long long)b * N + n) * F;
    for (int c = lane; c < F; c += 32) {
      float a = 0.f;
      for (int m = 0; m < M; ++m) a += sc[m] * x[(((long long)b * M + m) * N + n) * F + c];
      o[c] = a;
    }
  }
}

// dx_m = w_m dout + dscore_m ws,  dscore_m = w_m (<dout, x_m> - sum_k w_k <dout, x_k>);  dscore [B,M,N] is also written
// out (the caller reduces d ws = sum dscore x and d bs = sum dscore with the library's small-GEMM / row-sum kernels)
__global__ void softaggr_bwd_kernel(const float* __restrict__ dout, const float* __restrict__ x, int B, int M, int N, int F,
                                    const float* __restrict__ ws, const float* __restrict__ wts, float* __restrict__ dx,
                                    float* __restrict__ dscore) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  for (long long t = (long long)blockIdx.x * warps + warp; t < (long long)B * N; t += (long long)gridDim.x * warps) {
    const int b = (int)(t / N), n = (int)(t % N);
    const float* dr = dout + ((long long)b * N + n) * F;
    float w[MAX_MODES], dw[MAX_MODES];
    float wd = 0.f;
    for (int m = 0; m < M; ++m) {
      const float* xr = x + (((long long)b * M + m) * N + n) * F;
      float a = 0.f;
      for (int c = lane; c < F; c += 32) a += dr[c] * xr[c];
      dw[m] = sx::warp_sum(a);
      w[m] = wts[((long long)b * M + m) * N + n];
      wd += w[m] * dw[m];
    }
    for (int m = 0; m < M; ++m) {
      const float ds = w[m] * (dw[m] - wd);
      if (lane == 0) dscore[((long long)b * M + m) * N + n] = ds;
      float* o = dx + (((long long)b * M + m) * N + n) * F;
      for (int c = lane; c < F; c += 32) o[c] = w[m] * dr[c] + ds * ws[c];
    }
  }
}

// hi = TF32(x), lo = TF32(x - hi): the operand split of the error-compensated 3-pass TF32 products
__global__ void split_tf32_kernel(const float* __restrict__ x, long long n, float* __restrict__ hi, float* __restrict__ lo) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float v = x[i];
    const float h = sx::round_tf32(v);
    hi[i] = h;
    lo[i] = sx::round_tf32(v - h);
  }
}

// x[z1][z0][r][k] (arbitrary element strides) -> out[z1][z0][r][3*Kp] = [lo | hi | hi] (role 0) or [hi | lo | hi] (role 1),
// hi = TF32(x), lo = TF32(x - hi), each segment zero-padded to Kp columns: the K-concatenated operands of a ONE-launch
// error-compensated product  A'.B'^T = A_lo B_hi^T + A_hi B_lo^T + A_hi B_hi^T
__global__ void split_cat_kernel(const float* __restrict__ x, int Z0, int R, int K, long long sz1, long long sz0,
                                 long long sr, long long sk, int Kp, int role, float* __restrict__ out) {
  const long long row = blockIdx.x;                      // (z1, z0, r) flattened
  const int r = (int)(row % R);
  const long long z = row / R;
  const int z0 = (int)(z % Z0);
  const long long z1 = z / Z0;
  const float* xr = x + z1 * sz1 + z0 * sz0 + (long long)r * sr;
  float* o = out + row * 3ll * Kp;
  for (int k = threadIdx.x; k < Kp; k += blockDim.x) {
    float h = 0.f, l = 0.f;
    if (k < K) {
      const float v = xr[(long long)k * sk];
      h = sx::round_tf32(v);
      l = sx::round_tf32(v - h);
    }
    // the two small cross products come FIRST in the reduction order: the tensor core's fp32 accumulator is still small
    // while they are added, so they are not swallowed by the rounding of the large hi.hi partial sum
    o[k] = role == 0 ? l : h;
    o[Kp + k] = role == 0 ? h : l;
    o[2 * Kp + k] = h;
  }
}

// out[z0*C + c] += sum_{z1,r} X[z1*sz1 + z0*sz0 + r*ld + c]   (bias gradients, per mode in one launch).  blockDim
// (32, 8), grid (C/32, row blocks, Z0); the partial sums of row block y go to slot y of `part` ([Z0 * C])
__global__ void colsum_kernel(const float* __restrict__ X, int Z1, long long sz1, long long sz0, long long R, int C,
                              long long ld, float* __restrict__ part) {
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int z0 = blockIdx.z;
  float acc = 0.f;
  if (c < C)
    for (int z1 = 0; z1 < Z1; ++z1) {
      const float* base = X + z1 * sz1 + z0 * sz0;
      for (long long r = (long long)blockIdx.y * blockDim.y + threadIdx.y; r < R; r += (long long)gridDim.y * blockDim.y)
        acc += base[r * ld + c];
    }
  __shared__ float s[8][33];
  s[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t = 0.f;
    for (int y = 0; y < 8; ++y) t += s[y][threadIdx.x];
    part[((long long)blockIdx.y * gridDim.z + z0) * C + c] = t;
  }
}

// float4 flavour of colsum_kernel: lane = 4 consecutive columns (512 B per warp and row), 4 rows in flight per thread.
// out[z0*C + c] += sum_{z1,r} X[z1*sz1 + z0*sz0 + r*ld + c];  blockDim (32, 8), grid (C/128, row blocks, Z0); the partial
// sums of row block y go to slot y of `part` ([Z0 * C]) and part_reduce adds them into out
__global__ void __launch_bounds__(256)
colsum_v4_kernel(const float* __restrict__ X, int Z1, long long sz1, long long sz0, long long R, int C, long long ld,
                 float* __restrict__ part) {
  const int c = (blockIdx.x * 32 + threadIdx.x) * 4;
  const int z0 = blockIdx.z;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  if (c < C) {
    const long long step = (long long)gridDim.y * blockDim.y;
    for (int z1 = 0; z1 < Z1; ++z1) {
      const float* base = X + z1 * sz1 + z0 * sz0 + c;
      long long r = (long long)blockIdx.y * blockDim.y + threadIdx.y;
      for (; r + 3 * step < R; r += 4 * step) {
        const float4 a0 = __ldg(reinterpret_cast<const float4*>(base + r * ld));
        const float4 a1 = __ldg(reinterpret_cast<const float4*>(base + (r + step) * ld));
        const float4 a2 = __ldg(reinterpret_cast<const float4*>(base + (r + 2 * step) * ld));
        const float4 a3 = __ldg(reinterpret_cast<const float4*>(base + (r + 3 * step) * ld));
        acc.x += (a0.x + a1.x) + (a2.x + a3.x); acc.y += (a0.y + a1.y) + (a2.y + a3.y);
        acc.z += (a0.z + a1.z) + (a2.z + a3.z); acc.w += (a0.w + a1.w) + (a2.w + a3.w);
      }
      for (; r < R; r += step) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(base + r * ld));
        acc.x += a.x; acc.y += a.y; acc.z += a.z; acc.w += a.w;
      }
    }
  }
  __shared__ float4 s4[8][32];
  s4[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int y = 0; y < 8; ++y) {
      const float4 u = s4[y][threadIdx.x];
      t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
    }
    // slot blockIdx.y: [Z0 * C]
    *reinterpret_cast<float4*>(part + (long long)blockIdx.y * gridDim.z * C + (long long)z0 * C + c) = t;
  }
}

// batched 2-D transpose: in [Z, R, C] -> out [Z, C, R] with row pitch ldo   (flatten / scatter, segtran3d.py:328-330,
// :478-480; K-major GEMM operand copies)
__global__ void transpose_kernel(const float* __restrict__ in, int R, int C, int ldo, float* __restrict__ out) {
  __shared__ float tile[32][33];
  const long long z = blockIdx.z;
  const float* src = in + z * (long long)R * C;
  float* dst = out + z * (long long)C * ldo;
  const int c0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int r = r0 + j, c = c0 + threadIdx.x;
    if (r < R && c < C) tile[j][threadIdx.x] = src[(long long)r * C + c];
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j, r = r0 + threadIdx.x;
    if (r < R && c < C) dst[(long long)c * ldo + r] = tile[threadIdx.x][j];
  }
}

// sum_i x[i] * y[i] (linear synthetic loss / checksums): block b's sum goes to slot b of `part`
__global__ void dot_kernel(const float* __restrict__ x, const float* __restrict__ y, long long n, float* __restrict__ part) {
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc = fmaf(x[i], y[i], acc);
  acc = sx::warp_sum(acc);
  __shared__ float s[32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    acc = threadIdx.x < (blockDim.x >> 5) ? s[threadIdx.x] : 0.f;
    acc = sx::warp_sum(acc);
    if (threadIdx.x == 0) part[blockIdx.x] = acc;
  }
}

// out[j] += sum_{r = j mod out_mod} sum_c X[r, c]: block (j, y) sums column chunk y of those rows in a fixed order into
// slot y of `part` ([out_mod]); part_reduce adds the slots
__global__ void rowsum_kernel(const float* __restrict__ X, long long R, long long C, long long ld, int out_mod,
                              float* __restrict__ part) {
  const long long cs = (C + gridDim.y - 1) / gridDim.y, c0 = blockIdx.y * cs, c1 = c0 + cs < C ? c0 + cs : C;
  float acc = 0.f;
  for (long long r = blockIdx.x; r < R; r += out_mod) {
    const float* x = X + r * ld;
    for (long long c = c0 + threadIdx.x; c < c1; c += blockDim.x) acc += x[c];
  }
  acc = sx::warp_sum(acc);
  __shared__ float s[32];
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 32) {
    acc = threadIdx.x < (blockDim.x >> 5) ? s[threadIdx.x] : 0.f;
    acc = sx::warp_sum(acc);
    if (threadIdx.x == 0) part[(long long)blockIdx.y * out_mod + blockIdx.x] = acc;
  }
}

// y = a + b (residual of MMSharedOutput, segtran_shared.py:305), float4 when possible
__global__ void add_kernel(const float* __restrict__ a, const float* __restrict__ b, long long n, float* __restrict__ y) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = a[i] + b[i];
}

// y[i] = alpha * x[i]
__global__ void scale_kernel(const float* __restrict__ x, long long n, const float* __restrict__ alpha_dev, float alpha,
                             float* __restrict__ y) {
  const float a = alpha_dev ? alpha * (*alpha_dev) : alpha;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    y[i] = a * x[i];
}

int grid_for_rows(long long rows, int per_block, int sms) {
  long long g = (rows + per_block - 1) / per_block;
  long long cap = (long long)sms * 8;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  return (int)g;
}

int sms_cached() {
  const int n = sm_count_cached();
  return n > 0 ? n : 1;
}

template <typename K>
int set_smem(K kern, size_t bytes) {
  if (bytes > 48 * 1024) SX_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  return 0;
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int sx_reduce_max(const float* x, int64_t n, float* out, void* stream) {
  reduce_max_kernel<<<1, 256, 0, ST(stream)>>>(x, n, out);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_pos_lsinu_fwd(const float* pos, const float* posmax, int64_t R, int32_t pd, const float* W,
                                const float* b, int32_t C, float* pe, void* stream) {
  SX_REQUIRE(pd >= 1 && pd <= 3, "sx_pos_lsinu_fwd: pos_dim %d not in 1..3", pd);
  const size_t smem = (size_t)ROW_WARPS * C * 4;
  SX_REQUIRE(smem <= 200 * 1024, "sx_pos_lsinu_fwd: C=%d too large", C);
  if (set_smem(pos_lsinu_fwd_kernel, smem)) return -2;
  pos_lsinu_fwd_kernel<<<grid_for_rows(R, ROW_WARPS, sms_cached()), ROW_WARPS * 32, smem, ST(stream)>>>(
      pos, posmax, (int)R, pd, W, b, C, pe);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_pos_lsinu_bwd(const float* pos, const float* posmax, int64_t R, int32_t pd, const float* W,
                                const float* b, int32_t C, const float* dpe, float* de_scratch, float* dW, float* db,
                                float* part, int64_t part_floats, void* stream) {
  SX_REQUIRE(pd >= 1 && pd <= 3, "sx_pos_lsinu_bwd: pos_dim %d not in 1..3", pd);
  const size_t smem = (size_t)ROW_WARPS * 2 * C * 4;
  SX_REQUIRE(smem <= 200 * 1024, "sx_pos_lsinu_bwd: C=%d too large", C);
  if (set_smem(pos_lsinu_bwd_kernel, smem)) return -2;
  pos_lsinu_bwd_kernel<<<grid_for_rows(R, ROW_WARPS, sms_cached()), ROW_WARPS * 32, smem, ST(stream)>>>(
      pos, posmax, (int)R, pd, W, b, C, dpe, de_scratch);
  SX_CHECK_CUDA(cudaGetLastError());
  dim3 grid(sx_ceil_div(C, 32), 16), blk(32, 8);
  SX_REQUIRE(part && part_floats >= 16ll * (C * pd + C), "sx_pos_lsinu_bwd: needs %lld floats of scratch",
             16ll * (C * pd + C));
  pos_param_grad_kernel<<<grid, blk, 0, ST(stream)>>>(de_scratch, pos, posmax, (int)R, pd, C, part);
  SX_CHECK_CUDA(cudaGetLastError());
  return part_reduce(part, 16, C * pd + C, PartDst{{dW, db, nullptr, nullptr}, {C * pd, C, 0, 0}}, ST(stream));
}

// warps per CTA of a warp-per-row kernel that stages `floats_per_warp` floats in shared memory: at most 8, and 0 when
// one warp's share does not fit
static int smem_warps(long long floats_per_warp) {
  return (int)std::min<long long>(ROW_WARPS, (200 * 1024) / (floats_per_warp * 4));
}

extern "C" int sx_prologue_fwd(const float* x, int64_t B, int32_t N, int32_t C, const float* g, const float* b,
                               const float* pe, int32_t C0, int64_t pe_bstride, float posw, const float* mask,
                               float drop_p, uint64_t seed, const uint64_t* seed_dev, float* h, int32_t round_tf32, float* stats,
                               void* stream) {
  if (!pe) {                                        // no positional code: h = mask * dropout(LN_{g,b}(x))
    const long long R = (long long)B * N;
    const int grid = grid_for_rows(R, NOPOS_WARPS, sms_cached());
    prologue_nopos_fwd_kernel<<<grid, NOPOS_WARPS * 32, 0, ST(stream)>>>(
        x, R, C, g, b, mask, drop_p, seed, (const unsigned long long*)seed_dev, h, stats, round_tf32);
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (C % 4 == 0 && C <= 2048 && C0 % 4 == 0 && pe_bstride % 4 == 0 && al16(x) && al16(h) && al16(pe) &&
      al16(g) && al16(b)) {
    // CTA-per-row kernel: the row in registers, 16-byte accesses at every width
    const long long R = (long long)B * N;
#define SX_LAUNCH(NV_, TT_)                                                                                             \
  prologue_fwd_cta<NV_, TT_><<<(int)std::min<long long>(R, (long long)sms_cached() * (1024 / TT_)), TT_, 0, ST(stream)>>>( \
      x, R, N, C, g, b, pe, C0, pe_bstride, posw, mask, drop_p, seed, (const unsigned long long*)seed_dev, h, stats, \
      round_tf32)
    if (C <= 512) SX_LAUNCH(1, 128); else if (C <= 1024) SX_LAUNCH(2, 128); else SX_LAUNCH(2, 256);
#undef SX_LAUNCH
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  const size_t smem = (size_t)ROW_WARPS * C * 4;
  SX_REQUIRE(smem <= 200 * 1024, "sx_prologue_fwd: C=%d too large", C);
  const long long R = (long long)B * N;
  const int grid = grid_for_rows(R, ROW_WARPS, sms_cached());
  if (set_smem(prologue_fwd_kernel, smem)) return -2;
  prologue_fwd_kernel<<<grid, ROW_WARPS * 32, smem, ST(stream)>>>(
      x, R, N, C, g, b, pe, C0, pe_bstride, posw, mask, drop_p, seed, (const unsigned long long*)seed_dev, h, stats, round_tf32);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_prologue_bwd(const float* dh, const float* x, int64_t B, int32_t N, int32_t C, const float* g,
                               const float* b, const float* pe, int32_t C0, int64_t pe_bstride, float posw,
                               const float* mask, float drop_p, uint64_t seed, const uint64_t* seed_dev, const float* stats, float* dx, float* dg,
                               float* db, float* dpe, float* dt_scratch, float* part, int64_t part_floats, void* stream) {
  const long long R = (long long)B * N;
  SX_REQUIRE(part && part_floats >= 2ll * C, "sx_prologue_bwd: needs at least %lld floats of scratch", 2ll * C);
  const PartDst dgb{{dg, db, nullptr, nullptr}, {C, C, 0, 0}};
  if (!pe) {
    SX_REQUIRE(!dpe, "sx_prologue_bwd: dpe must be NULL without a positional code");
    const int grid = std::min(grid_for_rows(R, NOPOS_WARPS, sms_cached()), part_slots(part_floats, 2ll * C));
    const size_t smem = (size_t)NOPOS_WARPS * 2 * C * 4;
    SX_REQUIRE(smem <= 200 * 1024, "sx_prologue_bwd: C=%d too large", C);
    if (set_smem(prologue_nopos_bwd_kernel, smem)) return -2;
    prologue_nopos_bwd_kernel<<<grid, NOPOS_WARPS * 32, smem, ST(stream)>>>(
        dh, x, R, C, g, mask, drop_p, seed, (const unsigned long long*)seed_dev, stats, dx, part);
    SX_CHECK_CUDA(cudaGetLastError());
    return part_reduce(part, grid, 2 * C, dgb, ST(stream));
  }
  SX_REQUIRE(!dpe || dt_scratch, "sx_prologue_bwd: dpe needs dt_scratch");
  float* dt = dpe ? dt_scratch : nullptr;
  const bool vec = C % 4 == 0 && C0 % 4 == 0 && pe_bstride % 4 == 0 && (!dpe || (al16(dt_scratch) && al16(dpe)));
  if (vec && C <= 2048 && al16(dh) && al16(x) && al16(dx) && al16(pe) && al16(g) && al16(b)) {
    // CTA-per-row kernel: x / dh read once, dx (and dt, when the positional-code gradient needs it) written once, dg / db
    // accumulated in registers
    auto pgrid = [&](int tt) {
      return (int)std::min<long long>(std::min<long long>(R, (long long)sms_cached() * (768 / tt)), part_slots(part_floats, 2 * C));
    };
#define SX_LAUNCH(NV_, TT_)                                                                                             \
  prologue_bwd_cta<NV_, TT_><<<pgrid(TT_), TT_, 0, ST(stream)>>>(                                                    \
      dh, x, R, N, C, g, b, pe, C0, pe_bstride, posw, mask, drop_p, seed, (const unsigned long long*)seed_dev, stats, dx, dt, \
      part)
    if (C <= 512) SX_LAUNCH(1, 128); else if (C <= 1024) SX_LAUNCH(2, 128); else SX_LAUNCH(2, 256);
#undef SX_LAUNCH
    SX_CHECK_CUDA(cudaGetLastError());
    if (part_reduce(part, pgrid(C <= 1024 ? 128 : 256), 2 * C, dgb, ST(stream))) return -2;
  } else {
    const int warps = smem_warps(5ll * C);
    SX_REQUIRE(warps >= 1, "sx_prologue_bwd: C=%d too large", C);
    const size_t smem = (size_t)warps * 5 * C * 4;
    const int grid = std::min(grid_for_rows(R, warps * 4, sms_cached()), part_slots(part_floats, 2ll * C));
    if (set_smem(prologue_bwd_kernel, smem)) return -2;
    prologue_bwd_kernel<<<grid, warps * 32, smem, ST(stream)>>>(
        dh, x, R, N, C, g, b, pe, C0, pe_bstride, posw, mask, drop_p, seed, (const unsigned long long*)seed_dev, stats, dx, dt, part);
    SX_CHECK_CUDA(cudaGetLastError());
    if (part_reduce(part, grid, 2 * C, dgb, ST(stream))) return -2;
  }
  if (dpe) {
    if (vec)
      pos_grad_from_dt<4><<<grid_for_rows((long long)N * (C / 4), 256, sms_cached()), 256, 0, ST(stream)>>>(
          dt, (int)B, N, C, C0, pe_bstride, posw, dpe);
    else
      pos_grad_from_dt<1><<<grid_for_rows((long long)N * C, 256, sms_cached()), 256, 0, ST(stream)>>>(
          dt, (int)B, N, C, C0, pe_bstride, posw, dpe);
    SX_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

extern "C" int sx_softmax_fwd(const float* S, int64_t R, int32_t L, int64_t lds, const float* amax, float clip,
                              float drop_p, uint64_t seed, const uint64_t* seed_dev, float* P, int64_t ldp, int32_t round_tf32,
                              float* lse, float* diag, void* stream) {
  if (L % 4 == 0 && lds % 4 == 0 && ldp % 4 == 0 && al16(S) && al16(P) && nv_for(L)) {
    const int grid = grid_for_rows(R, FAST_WARPS, sms_cached() * 2);
#define SX_LAUNCH(NV_)                                                                                          \
  softmax_fwd_fast<NV_><<<grid, FAST_WARPS * 32, 0, ST(stream)>>>(S, R, L, lds, amax, clip, drop_p, seed, (const unsigned long long*)seed_dev, P, \
                                                                  ldp, lse, round_tf32, diag)
    switch (nv_for(L)) { case 2: SX_LAUNCH(2); break; case 4: SX_LAUNCH(4); break; case 8: SX_LAUNCH(8); break;
                         default: SX_LAUNCH(16); }
#undef SX_LAUNCH
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (L % 4 == 0 && lds % 4 == 0 && ldp % 4 == 0 && al16(S) && al16(P) && L <= 8192) {
    const int grid = (int)(R < (long long)sms_cached() * 16 ? R : (long long)sms_cached() * 16);
#define SX_LAUNCH(E_)                                                                                          \
  softmax_fwd_block<E_><<<grid, 256, 0, ST(stream)>>>(S, R, L, lds, amax, clip, drop_p, seed,                     \
                                                      (const unsigned long long*)seed_dev, P, ldp, lse,          \
                                                      round_tf32, diag)
    if (L <= 3072) SX_LAUNCH(3); else if (L <= 6144) SX_LAUNCH(6); else SX_LAUNCH(8);
#undef SX_LAUNCH
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  const int w = smem_warps(L);
  SX_REQUIRE(w >= 1, "sx_softmax_fwd: row length %d too large", L);
  const size_t smem = (size_t)w * L * 4;
  const int grid = grid_for_rows(R, w, sms_cached());
  if (set_smem(softmax_fwd_kernel, smem)) return -2;
  softmax_fwd_kernel<<<grid, w * 32, smem, ST(stream)>>>(S, R, L, lds, amax, clip, drop_p, seed, (const unsigned long long*)seed_dev, P, ldp,
                                                         lse, round_tf32, diag);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_softmax_bwd(const float* dP, int64_t ldd, const float* S, int64_t lds, const float* lse, int64_t R,
                              int32_t L, const float* amax, float clip, float drop_p, uint64_t seed, const uint64_t* seed_dev, int64_t ldp_fwd,
                              float* dS, int64_t ldo, int32_t round_tf32, void* stream) {
  if (L % 4 == 0 && lds % 4 == 0 && ldd % 4 == 0 && ldo % 4 == 0 && al16(S) && al16(dP) && al16(dS) && nv_for(L)) {
    const int grid = grid_for_rows(R, FAST_WARPS, sms_cached() * 2);
#define SX_LAUNCH(NV_)                                                                                             \
  softmax_bwd_fast<NV_><<<grid, FAST_WARPS * 32, 0, ST(stream)>>>(dP, ldd, S, lds, lse, R, L, amax, clip, drop_p, seed, (const unsigned long long*)seed_dev, \
                                                                  ldp_fwd, dS, ldo, round_tf32)
    switch (nv_for(L)) { case 2: SX_LAUNCH(2); break; case 4: SX_LAUNCH(4); break; case 8: SX_LAUNCH(8); break;
                         default: SX_LAUNCH(16); }
#undef SX_LAUNCH
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  if (L % 4 == 0 && lds % 4 == 0 && ldd % 4 == 0 && ldo % 4 == 0 && al16(S) && al16(dP) && al16(dS) && L <= 8192) {
    const int grid = (int)(R < (long long)sms_cached() * 16 ? R : (long long)sms_cached() * 16);
#define SX_LAUNCH(E_)                                                                                            \
  softmax_bwd_block<E_><<<grid, 256, 0, ST(stream)>>>(dP, ldd, S, lds, lse, R, L, amax, clip, drop_p, seed,         \
                                                      (const unsigned long long*)seed_dev, ldp_fwd, dS, ldo,       \
                                                      round_tf32)
    if (L <= 3072) SX_LAUNCH(3); else if (L <= 6144) SX_LAUNCH(6); else SX_LAUNCH(8);
#undef SX_LAUNCH
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  const int w = smem_warps(2ll * L);
  SX_REQUIRE(w >= 1, "sx_softmax_bwd: row length %d too large", L);
  const size_t smem = (size_t)w * 2 * L * 4;
  const int grid = grid_for_rows(R, w, sms_cached());
  if (set_smem(softmax_bwd_kernel, smem)) return -2;
  softmax_bwd_kernel<<<grid, w * 32, smem, ST(stream)>>>(dP, ldd, S, lds, lse, R, L, amax, clip, drop_p, seed, (const unsigned long long*)seed_dev,
                                                         ldp_fwd, dS, ldo, round_tf32);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_layernorm_fwd(const float* x, int64_t R, int32_t C, const float* g, const float* b, float* y,
                                int32_t round_tf32, float* stats, void* stream) {
  const size_t smem = (size_t)ROW_WARPS * C * 4;
  SX_REQUIRE(smem <= 200 * 1024, "sx_layernorm_fwd: C=%d too large", C);
  const int grid = grid_for_rows(R, ROW_WARPS, sms_cached());
  if (set_smem(layernorm_fwd_kernel, smem)) return -2;
  layernorm_fwd_kernel<<<grid, ROW_WARPS * 32, smem, ST(stream)>>>(x, R, C, g, b, y, stats, round_tf32);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_layernorm_bwd(const float* dy, const float* x, int64_t R, int32_t C, const float* g,
                                const float* stats, float* dx, int32_t round_tf32, float* dg, float* db,
                                float* part, int64_t part_floats, void* stream) {
  SX_REQUIRE(part && part_floats >= 2ll * C, "sx_layernorm_bwd: needs at least %lld floats of scratch", 2ll * C);
  const PartDst dgb{{dg, db, nullptr, nullptr}, {C, C, 0, 0}};
  if (C % 4 == 0 && nv_for(C) && al16(dy) && al16(x) && al16(dx) && al16(g)) {
    const int grid = grid_for_rows(R, FAST_WARPS, sms_cached() * 2);
#define SX_LAUNCH(NV_)                                                                                         \
  layernorm_bwd_rows_fast<NV_><<<grid, FAST_WARPS * 32, 0, ST(stream)>>>(dy, x, R, C, g, stats, dx, round_tf32)
    switch (nv_for(C)) { case 2: SX_LAUNCH(2); break; case 4: SX_LAUNCH(4); break; case 8: SX_LAUNCH(8); break;
                         default: SX_LAUNCH(16); }
#undef SX_LAUNCH
    SX_CHECK_CUDA(cudaGetLastError());
    int gy = (int)((R + 8 * 64 - 1) / (8 * 64));
    const int cap = sx_ceil_div(sms_cached() * 8, sx_ceil_div(C, 128));
    if (gy > cap) gy = cap;
    gy = std::min(gy, part_slots(part_floats, 2 * C));
    if (gy < 1) gy = 1;
    dim3 grid2(sx_ceil_div(C, 128), gy), blk(32, 8);
    ln_param_grad_cols_fast<<<grid2, blk, 0, ST(stream)>>>(dy, x, R, C, stats, 2, part);
    SX_CHECK_CUDA(cudaGetLastError());
    return part_reduce(part, gy, 2 * C, dgb, ST(stream));
  }
  const int warps = smem_warps(4ll * C);
  SX_REQUIRE(warps >= 1, "sx_layernorm_bwd: C=%d too large", C);
  const size_t smem = (size_t)warps * 4 * C * 4;
  const int grid = std::min(grid_for_rows(R, warps * 4, sms_cached()), part_slots(part_floats, 2ll * C));
  if (set_smem(layernorm_bwd_kernel, smem)) return -2;
  layernorm_bwd_kernel<<<grid, warps * 32, smem, ST(stream)>>>(dy, x, R, C, g, stats, dx, part, round_tf32);
  SX_CHECK_CUDA(cudaGetLastError());
  return part_reduce(part, grid, 2 * C, dgb, ST(stream));
}

extern "C" int sx_ln_softaggr_fwd(const float* Y, int32_t B, int32_t M, int32_t N, int32_t F, const float* g,
                                  const float* b, const float* ws, const float* bs, float drop_p, uint64_t seed, const uint64_t* seed_dev,
                                  float* out, float* stats, float* wts, void* stream) {
  SX_REQUIRE(M >= 1 && M <= MAX_MODES, "sx_ln_softaggr_fwd: num_modes %d not in 1..%d", M, MAX_MODES);
  if (F % 4 == 0 && F <= 2048 && (M == 1 || M == 2 || M == 4) && al16(Y) && al16(out) && al16(g) && al16(b) && al16(ws)) {
    // CTA-per-token kernel: every mode row of a token in registers, Y read once
    const long long T = (long long)B * N;
    const int grid = (int)std::min<long long>(T, (long long)sms_cached() * (F <= 1024 ? 4 : 2));
#define SX_LAUNCH(NV_, MM_, TT_)                                                                                        \
  ln_softaggr_fwd_cta<NV_, MM_, TT_><<<grid, TT_, 0, ST(stream)>>>(Y, B, N, F, g, b, ws, bs, drop_p, seed,              \
                                                                    (const unsigned long long*)seed_dev, out, stats, wts)
#define SX_MODES(NV_, TT_) do { if (M == 4) SX_LAUNCH(NV_, 4, TT_); else if (M == 2) SX_LAUNCH(NV_, 2, TT_); else SX_LAUNCH(NV_, 1, TT_); } while (0)
    if (F <= 512) SX_MODES(1, 128); else if (F <= 1024) SX_MODES(2, 128); else SX_MODES(2, 256);
#undef SX_MODES
#undef SX_LAUNCH
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  const int warps = smem_warps((long long)M * F);
  SX_REQUIRE(warps >= 1, "sx_ln_softaggr_fwd: M*F=%d too large", M * F);
  const size_t smem = (size_t)warps * M * F * 4;
  if (set_smem(ln_softaggr_fwd_kernel, smem)) return -2;
  ln_softaggr_fwd_kernel<<<grid_for_rows((long long)B * N, warps, sms_cached()), warps * 32, smem, ST(stream)>>>(
      Y, B, M, N, F, g, b, ws, bs, drop_p, seed, (const unsigned long long*)seed_dev, out, stats, wts);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_ln_softaggr_bwd(const float* dout, const float* Y, int32_t B, int32_t M, int32_t N, int32_t F,
                                  const float* g, const float* b, const float* ws, float drop_p, uint64_t seed, const uint64_t* seed_dev,
                                  const float* stats, const float* wts, float* dY, int32_t round_tf32,
                                  float* dg, float* db, float* dws, float* dbs, float* part, int64_t part_floats, void* stream) {
  SX_REQUIRE(M >= 1 && M <= MAX_MODES, "sx_ln_softaggr_bwd: num_modes %d not in 1..%d", M, MAX_MODES);
  const long long T = (long long)B * N;
  if (F % 4 == 0 && F <= 2048 && (M == 1 || M == 2 || M == 4) && al16(Y) && al16(dout) && al16(dY) &&
      al16(g) && al16(b) && al16(ws)) {
    // CTA-per-token kernel: Y and dout read once, dY written once, column gradients accumulated in registers
    const int grid = (int)std::min<long long>(std::min<long long>(T, (long long)sms_cached() * (F <= 1024 ? 3 : 2)),
                                              part_slots(part_floats, 3 * F + 4));
    SX_REQUIRE(part && grid >= 1, "sx_ln_softaggr_bwd: needs at least %lld floats of scratch", 3ll * F + 4);
#define SX_LAUNCH(NV_, MM_, TT_)                                                                                        \
  ln_softaggr_bwd_cta<NV_, MM_, TT_><<<grid, TT_, 0, ST(stream)>>>(dout, Y, B, N, F, g, b, ws, drop_p, seed,            \
                                                                    (const unsigned long long*)seed_dev, stats, wts,    \
                                                                    dY, round_tf32, part)
#define SX_MODES(NV_, TT_) do { if (M == 4) SX_LAUNCH(NV_, 4, TT_); else if (M == 2) SX_LAUNCH(NV_, 2, TT_); else SX_LAUNCH(NV_, 1, TT_); } while (0)
    if (F <= 512) SX_MODES(1, 128); else if (F <= 1024) SX_MODES(2, 128); else SX_MODES(2, 256);
#undef SX_MODES
#undef SX_LAUNCH
    SX_CHECK_CUDA(cudaGetLastError());
    return part_reduce(part, grid, 3 * F + 4, PartDst{{dg, db, dws, dbs}, {F, F, F, 1}}, ST(stream));
  }
  const int warps = smem_warps(5ll * F + 1);
  SX_REQUIRE(warps >= 1, "sx_ln_softaggr_bwd: F=%d too large", F);
  const size_t smem = (size_t)warps * (5 * F + 1) * 4;
  const int grid = std::min(grid_for_rows(T, warps * 4, sms_cached()), part_slots(part_floats, 3ll * F + 1));
  SX_REQUIRE(part && grid >= 1, "sx_ln_softaggr_bwd: needs at least %lld floats of scratch", 3ll * F + 1);
  if (set_smem(ln_softaggr_bwd_kernel, smem)) return -2;
  ln_softaggr_bwd_kernel<<<grid, warps * 32, smem, ST(stream)>>>(
      dout, Y, B, M, N, F, g, b, ws, drop_p, seed, (const unsigned long long*)seed_dev, stats, wts, dY, part, round_tf32);
  SX_CHECK_CUDA(cudaGetLastError());
  return part_reduce(part, grid, 3 * F + 1, PartDst{{dg, db, dws, dbs}, {F, F, F, 1}}, ST(stream));
}

extern "C" int sx_gelu_bwd(const float* dG, const float* H, int64_t n, float drop_p, uint64_t seed, const uint64_t* seed_dev,
                           float* dH, int32_t round_tf32, void* stream) {
  const auto* sd = (const unsigned long long*)seed_dev;
  if (n % 4 == 0 && al16(dG) && al16(H) && al16(dH)) {
    const int grid = grid_for_rows(n / 4, 256 * 4, sms_cached());
    if (H) gelu_bwd_f4_kernel<true><<<grid, 256, 0, ST(stream)>>>((const float4*)dG, (const float4*)H, n / 4, drop_p, seed, sd, (float4*)dH, round_tf32);
    else gelu_bwd_f4_kernel<false><<<grid, 256, 0, ST(stream)>>>((const float4*)dG, nullptr, n / 4, drop_p, seed, sd, (float4*)dH, round_tf32);
  } else {
    const int grid = grid_for_rows(n, 256 * 8, sms_cached());
    if (H) gelu_bwd_kernel<true><<<grid, 256, 0, ST(stream)>>>(dG, H, n, drop_p, seed, sd, dH, round_tf32);
    else gelu_bwd_kernel<false><<<grid, 256, 0, ST(stream)>>>(dG, nullptr, n, drop_p, seed, sd, dH, round_tf32);
  }
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_convert(const void* x, int32_t x_dtype, int64_t n, void* y, int32_t y_dtype, int32_t round_tf32,
                          void* stream) {
  const int grid = grid_for_rows(n, 256 * 8, sms_cached());
  if (x_dtype == SX_F32 && y_dtype == SX_F32)
    convert_kernel<float, float><<<grid, 256, 0, ST(stream)>>>((const float*)x, n, (float*)y, round_tf32);
  else if (x_dtype == SX_F32 && y_dtype == SX_BF16)
    convert_kernel<float, __nv_bfloat16><<<grid, 256, 0, ST(stream)>>>((const float*)x, n, (__nv_bfloat16*)y, 0);
  else if (x_dtype == SX_BF16 && y_dtype == SX_F32)
    convert_kernel<__nv_bfloat16, float><<<grid, 256, 0, ST(stream)>>>((const __nv_bfloat16*)x, n, (float*)y, 0);
  else
    SX_REQUIRE(false, "sx_convert: unsupported dtype pair %d -> %d", x_dtype, y_dtype);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_softaggr_fwd(const float* x, int32_t B, int32_t M, int32_t N, int32_t F, const float* ws, const float* bs,
                               float* out, float* wts, void* stream) {
  SX_REQUIRE(M >= 1 && M <= MAX_MODES && B > 0 && N > 0 && F > 0, "sx_softaggr_fwd: bad shape (modes %d)", M);
  softaggr_fwd_kernel<<<grid_for_rows((long long)B * N, ROW_WARPS, sms_cached() * 4), ROW_WARPS * 32, 0, ST(stream)>>>(
      x, B, M, N, F, ws, bs, out, wts);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_softaggr_bwd(const float* dout, const float* x, int32_t B, int32_t M, int32_t N, int32_t F, const float* ws,
                               const float* wts, float* dx, float* dscore, void* stream) {
  SX_REQUIRE(M >= 1 && M <= MAX_MODES && B > 0 && N > 0 && F > 0, "sx_softaggr_bwd: bad shape (modes %d)", M);
  softaggr_bwd_kernel<<<grid_for_rows((long long)B * N, ROW_WARPS, sms_cached() * 4), ROW_WARPS * 32, 0, ST(stream)>>>(
      dout, x, B, M, N, F, ws, wts, dx, dscore);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_split_tf32(const float* x, int64_t n, float* hi, float* lo, void* stream) {
  if (n <= 0) return 0;
  long long blocks = (n + 255) / 256;
  if (blocks > sms_cached() * 16) blocks = sms_cached() * 16;
  split_tf32_kernel<<<(int)blocks, 256, 0, ST(stream)>>>(x, n, hi, lo);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_split_tf32_cat(const float* x, int32_t Z1, int32_t Z0, int32_t R, int32_t K, int64_t sz1, int64_t sz0,
                                 int64_t sr, int64_t sk, int32_t Kp, int32_t role, float* out, void* stream) {
  SX_REQUIRE(Z1 > 0 && Z0 > 0 && R > 0 && K > 0 && Kp >= K && Kp % 4 == 0, "sx_split_tf32_cat: bad shape");
  const long long rows = (long long)Z1 * Z0 * R;
  SX_REQUIRE(rows < (1ll << 31), "sx_split_tf32_cat: too many rows");
  split_cat_kernel<<<(unsigned)rows, Kp >= 256 ? 256 : 64, 0, ST(stream)>>>(x, Z0, R, K, sz1, sz0, sr, sk, Kp, role, out);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_transpose(const float* in, int64_t Z, int32_t R, int32_t C, int32_t ldo, float* out, void* stream) {
  SX_REQUIRE(Z <= 65535, "sx_transpose: batch %lld too large", (long long)Z);
  SX_REQUIRE(R > 0 && C > 0 && ldo >= R, "sx_transpose: bad shape R=%d C=%d ldo=%d", R, C, ldo);
  if (R % 4 == 0 && C % 4 == 0 && ldo % 4 == 0 && al16(in) && al16(out)) {
    dim3 gridv(sx_ceil_div(C, 128), sx_ceil_div(R, 32), (unsigned)Z);
    transpose_v4_kernel<<<gridv, 256, 0, ST(stream)>>>(in, R, C, ldo, out);
    SX_CHECK_CUDA(cudaGetLastError());
    return 0;
  }
  dim3 grid(sx_ceil_div(C, 32), sx_ceil_div(R, 32), (unsigned)Z), blk(32, 8);
  transpose_kernel<<<grid, blk, 0, ST(stream)>>>(in, R, C, ldo, out);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_dot(const float* x, const float* y, int64_t n, float* out, float* part, int64_t part_floats, void* stream) {
  SX_REQUIRE(part && part_floats >= 1, "sx_dot: needs scratch");
  const int grid = std::min(grid_for_rows(n, 256 * 8, sms_cached()), part_slots(part_floats, 1));
  dot_kernel<<<grid, 256, 0, ST(stream)>>>(x, y, n, part);
  SX_CHECK_CUDA(cudaGetLastError());
  return part_reduce(part, grid, 1, PartDst{{out, nullptr, nullptr, nullptr}, {1, 0, 0, 0}}, ST(stream));
}

extern "C" int sx_scale(const float* x, int64_t n, const float* alpha_dev, float alpha, float* y, void* stream) {
  scale_kernel<<<grid_for_rows(n, 256 * 8, sms_cached()), 256, 0, ST(stream)>>>(x, n, alpha_dev, alpha, y);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_rowsum(const float* X, int64_t R, int64_t C, int64_t ld, int32_t out_mod, float* out, float* part, int64_t part_floats, void* stream) {
  SX_REQUIRE(R >= 1 && R <= 2147483647ll && out_mod >= 1, "sx_rowsum: bad shape");
  SX_REQUIRE(part && part_floats >= out_mod, "sx_rowsum: needs at least %d floats of scratch", out_mod);
  // column chunks: enough blocks for the machine, at least 512 columns each, as many slots as the scratch holds
  long long chunks = sx_ceil_div((long long)sms_cached() * 8, out_mod);
  chunks = std::min<long long>(chunks, sx_ceil_div(C, 512));
  chunks = std::max<long long>(1, std::min<long long>({chunks, 65535ll, (long long)part_slots(part_floats, out_mod)}));
  rowsum_kernel<<<dim3((unsigned)out_mod, (unsigned)chunks), 512, 0, ST(stream)>>>(X, R, C, ld, out_mod, part);
  SX_CHECK_CUDA(cudaGetLastError());
  return part_reduce(part, (int)chunks, out_mod, PartDst{{out, nullptr, nullptr, nullptr}, {out_mod, 0, 0, 0}}, ST(stream));
}

extern "C" int sx_colsum_batched(const float* X, int32_t Z1, int64_t stride_z1, int32_t Z0, int64_t stride_z0, int64_t R,
                                 int32_t C, int64_t ld, float* out, float* part, int64_t part_floats, void* stream) {
  SX_REQUIRE(Z0 >= 1 && Z0 <= 65535 && Z1 >= 1, "sx_colsum_batched: bad batch dims");
  const int slots = part_slots(part_floats, (long long)Z0 * C);
  SX_REQUIRE(part && slots >= 1, "sx_colsum_batched: needs at least %lld floats of scratch", (long long)Z0 * C);
  dim3 blk(32, 8);
  int gy;
  if (C % 4 == 0 && ld % 4 == 0 && stride_z0 % 4 == 0 && stride_z1 % 4 == 0 && al16(X)) {
    gy = (int)((R + 127) / 128);
    const int cap = sx_ceil_div(sms_cached() * 8, sx_ceil_div(C, 128) * Z0);
    if (gy > cap) gy = cap;
    gy = std::min(gy, slots);
    colsum_v4_kernel<<<dim3(sx_ceil_div(C, 128), gy, Z0), blk, 0, ST(stream)>>>(X, Z1, stride_z1, stride_z0, R, C, ld, part);
  } else {
    gy = std::max(1, std::min({(int)std::min<long long>((R + 255) / 256, 32), slots}));
    colsum_kernel<<<dim3(sx_ceil_div(C, 32), gy, Z0), blk, 0, ST(stream)>>>(X, Z1, stride_z1, stride_z0, R, C, ld, part);
  }
  SX_CHECK_CUDA(cudaGetLastError());
  return part_reduce(part, gy, Z0 * C, PartDst{{out, nullptr, nullptr, nullptr}, {Z0 * C, 0, 0, 0}}, ST(stream));
}

namespace {
__global__ void seed_derive_kernel(const unsigned long long* base, unsigned long long add, unsigned long long* out) {
  out[0] = (base ? base[0] : 0ull) + add;
}
__global__ void seed_advance_kernel(unsigned long long* base, unsigned long long inc) { base[0] += inc; }
}  // namespace

extern "C" int sx_seed_derive(const uint64_t* base, uint64_t add, uint64_t* out, void* stream) {
  seed_derive_kernel<<<1, 1, 0, ST(stream)>>>((const unsigned long long*)base, add, (unsigned long long*)out);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_seed_advance(uint64_t* base, uint64_t inc, void* stream) {
  seed_advance_kernel<<<1, 1, 0, ST(stream)>>>((unsigned long long*)base, inc);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_add(const float* a, const float* b, int64_t n, float* y, void* stream) {
  add_kernel<<<grid_for_rows(n, 256 * 4, sms_cached()), 256, 0, ST(stream)>>>(a, b, n, y);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_softmax_posbias_fwd(const float* S, int64_t R, int32_t L, int64_t lds, const float* amax, float clip,
                                      float drop_p, uint64_t seed, const uint64_t* seed_dev, float* P, int64_t ldp, int32_t round_tf32, float* lse, float* diag, const sx_posbias* posbias,
                                      void* stream) {
  const char* err = sxpb::check(posbias, L);
  SX_REQUIRE(err == nullptr, "sx_softmax_posbias_fwd: %s", err);
  SX_REQUIRE(R % L == 0, "sx_softmax_posbias_fwd: rows must be whole [L x L] blocks");
  const sxpb::Geom G = sxpb::make_geom(*posbias);
  const size_t smem = (size_t)(32 + L) * 4;
  SX_REQUIRE(smem <= 200 * 1024, "sx_softmax_posbias_fwd: L=%d too large", L);
  const int grid = (int)std::min<long long>(R, (long long)sms_cached() * 8);
  if (set_smem(softmax_posbias_fwd_kernel, smem)) return -2;
  softmax_posbias_fwd_kernel<<<grid, PB_THREADS, smem, ST(stream)>>>(
      S, R, L, lds, amax, clip, drop_p, seed, (const unsigned long long*)seed_dev, P, ldp, lse, round_tf32, diag,
      posbias->table, G);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_softmax_posbias_bwd(const float* dP, int64_t ldd, const float* S, int64_t lds, const float* lse, int64_t R,
                                      int32_t L, const float* amax, float clip, float drop_p, uint64_t seed,
                                      const uint64_t* seed_dev, int64_t ldp_fwd, float* dS, int64_t ldo,
                                      int32_t round_tf32, const sx_posbias* posbias, float* dtable, float* part,
                                      int64_t part_floats, void* stream) {
  const char* err = sxpb::check(posbias, L);
  SX_REQUIRE(err == nullptr, "sx_softmax_posbias_bwd: %s", err);
  SX_REQUIRE(R % L == 0, "sx_softmax_posbias_bwd: rows must be whole [L x L] blocks");
  SX_REQUIRE(dtable != nullptr, "sx_softmax_posbias_bwd: null dtable");
  const sxpb::Geom G = sxpb::make_geom(*posbias);
  SX_REQUIRE(part && part_floats >= G.T, "sx_softmax_posbias_bwd: needs at least %d floats of scratch", G.T);
  const size_t smem = (size_t)(32 + G.T + 2 * (size_t)L) * 4;
  SX_REQUIRE(smem <= 200 * 1024, "sx_softmax_posbias_bwd: L=%d too large", L);
  const int grid = (int)std::min<long long>(std::min<long long>(R, (long long)sms_cached() * 4), part_slots(part_floats, G.T));
  if (set_smem(softmax_posbias_bwd_kernel, smem)) return -2;
  softmax_posbias_bwd_kernel<<<grid, PB_THREADS, smem, ST(stream)>>>(
      dP, ldd, S, lds, lse, R, L, amax, clip, drop_p, seed, (const unsigned long long*)seed_dev, ldp_fwd, dS, ldo,
      round_tf32, posbias->table, G, part);
  SX_CHECK_CUDA(cudaGetLastError());
  return part_reduce(part, grid, G.T, PartDst{{dtable, nullptr, nullptr, nullptr}, {G.T, 0, 0, 0}}, ST(stream));
}
