// Register-resident fast paths of the row kernels (fp32 I/O, row length a multiple of 4, <= 128*NV floats).
// A row lives in NV float4 registers per lane (lane l holds columns 4l+128i .. +3), so there is no shared-memory
// staging, occupancy is register-limited only (32+ warps/SM) and every global access is a 16-byte vector access.
// Parameter gradients that are column sums over all rows are produced by separate column-parallel reductions.
// Included by sx_rows.cu inside its anonymous namespace.
#pragma once

template <int NV>
__device__ __forceinline__ void row_load(float4 (&v)[NV], const float* __restrict__ p, int C, int lane) {
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 4 * lane + 128 * i;
    v[i] = (c < C) ? *reinterpret_cast<const float4*>(p + c) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}
template <int NV>
__device__ __forceinline__ void row_store(const float4 (&v)[NV], float* __restrict__ p, int C, int lane) {
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 4 * lane + 128 * i;
    if (c < C) *reinterpret_cast<float4*>(p + c) = v[i];
  }
}
template <int NV>
__device__ __forceinline__ void row_mean_rstd(const float4 (&v)[NV], int C, int lane, float& mean, float& rstd) {
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);     // out-of-range entries are zero
  mean = sx::warp_sum(s) / C;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < NV; ++i)
    if (4 * lane + 128 * i < C) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += (a * a + b * b) + (c * c + d * d);
    }
  rstd = rsqrtf(sx::warp_sum(q) / C + LN_EPS);
}
// idx must be a multiple of 4 (start of a float4 group)
__device__ __forceinline__ float4 drop4(float4 v, float p, float scale, unsigned long long seed, unsigned long long idx) {
  const uint2 h = sx::drop_hash(seed, idx >> 2);
  const uint32_t p16 = sx::drop_p16(p);
  v.x = sx::drop_keep(h, 0, p16) ? v.x * scale : 0.f;
  v.y = sx::drop_keep(h, 1, p16) ? v.y * scale : 0.f;
  v.z = sx::drop_keep(h, 2, p16) ? v.z * scale : 0.f;
  v.w = sx::drop_keep(h, 3, p16) ? v.w * scale : 0.f;
  return v;
}
// keep bits of one float4 group (bit j = element j is kept) and their application: the two-pass row kernels hash each
// group once and park the bits in shared memory instead of re-hashing in every pass
__device__ __forceinline__ uint32_t keep4(unsigned long long seed, unsigned long long idx, uint32_t p16) {
  const uint2 h = sx::drop_hash(seed, idx >> 2);
  return (sx::drop_keep(h, 0, p16) ? 1u : 0u) | (sx::drop_keep(h, 1, p16) ? 2u : 0u) |
         (sx::drop_keep(h, 2, p16) ? 4u : 0u) | (sx::drop_keep(h, 3, p16) ? 8u : 0u);
}
__device__ __forceinline__ float4 mask4(float4 v, uint32_t bits, float scale) {
  v.x = (bits & 1u) ? v.x * scale : 0.f;
  v.y = (bits & 2u) ? v.y * scale : 0.f;
  v.z = (bits & 4u) ? v.z * scale : 0.f;
  v.w = (bits & 8u) ? v.w * scale : 0.f;
  return v;
}
__device__ __forceinline__ float4 rnd4(float4 v, int rnd) {
  if (rnd) { v.x = sx::round_tf32(v.x); v.y = sx::round_tf32(v.y); v.z = sx::round_tf32(v.z); v.w = sx::round_tf32(v.w); }
  return v;
}
__device__ __forceinline__ float4 ld4(const float* __restrict__ p) { return __ldg(reinterpret_cast<const float4*>(p)); }

constexpr int FAST_WARPS = 8;

// ------------------------------------------------------------------------------------------------
// softmax forward / backward with the row in registers (L <= 128*NV)
// ------------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(FAST_WARPS * 32)
softmax_fwd_fast(const float* __restrict__ S, long long R, int L, long long lds, const float* __restrict__ amax,
                 float clip, float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev, float* __restrict__ P, long long ldp,
                 float* __restrict__ lse, int rnd, float* __restrict__ diag) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool do_clip = amax && (*amax > clip);
  if (diag && amax && blockIdx.x == 0 && threadIdx.x == 0) {
    diag[0] = fmaxf(diag[0], *amax);
    if (do_clip) diag[1] += 1.f;
  }
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = (long long)blockIdx.x * FAST_WARPS + warp; r < R; r += (long long)gridDim.x * FAST_WARPS) {
    float4 v[NV];
    row_load<NV>(v, S + r * lds, L, lane);
    float m = -3.0e38f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (4 * lane + 128 * i < L) {
        if (do_clip) {
          v[i].x = fminf(fmaxf(v[i].x, -clip), clip); v[i].y = fminf(fmaxf(v[i].y, -clip), clip);
          v[i].z = fminf(fmaxf(v[i].z, -clip), clip); v[i].w = fminf(fmaxf(v[i].w, -clip), clip);
        }
        m = fmaxf(m, fmaxf(fmaxf(v[i].x, v[i].y), fmaxf(v[i].z, v[i].w)));
      }
    m = sx::warp_max(m);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (4 * lane + 128 * i < L) {
        v[i].x = __expf(v[i].x - m); v[i].y = __expf(v[i].y - m); v[i].z = __expf(v[i].z - m); v[i].w = __expf(v[i].w - m);
        s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
      }
    s = sx::warp_sum(s);
    const float inv = 1.f / s;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      if (c < L) {
        float4 p = make_float4(v[i].x * inv, v[i].y * inv, v[i].z * inv, v[i].w * inv);
        if (drop_p > 0.f) p = drop4(p, drop_p, keep_scale, seed, (unsigned long long)(r * ldp + c));
        *reinterpret_cast<float4*>(P + r * ldp + c) = rnd4(p, rnd);
      }
    }
    if (lane == 0 && lse) lse[r] = m + __logf(s);
  }
}

template <int NV>
__global__ void __launch_bounds__(FAST_WARPS * 32)
softmax_bwd_fast(const float* __restrict__ dP, long long ldd, const float* __restrict__ S, long long lds,
                 const float* __restrict__ lse, long long R, int L, const float* __restrict__ amax, float clip,
                 float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev, long long ldp_fwd, float* __restrict__ dS, long long ldo,
                 int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool do_clip = amax && (*amax > clip);
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = (long long)blockIdx.x * FAST_WARPS + warp; r < R; r += (long long)gridDim.x * FAST_WARPS) {
    const float l = lse[r];
    float4 p[NV], gv[NV];
    row_load<NV>(p, S + r * lds, L, lane);
    row_load<NV>(gv, dP + r * ldd, L, lane);
    float dot = 0.f;
    unsigned inside = 0;                        // bit i*4+j: element was inside the clamp range
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      if (c < L) {
        float x[4] = {p[i].x, p[i].y, p[i].z, p[i].w};
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          bool in = true;
          if (do_clip) { in = (x[j] >= -clip && x[j] <= clip); x[j] = fminf(fmaxf(x[j], -clip), clip); }
          if (in && NV <= 8) inside |= 1u << (i * 4 + j);
          x[j] = __expf(x[j] - l);
        }
        p[i] = make_float4(x[0], x[1], x[2], x[3]);
        if (drop_p > 0.f) gv[i] = drop4(gv[i], drop_p, keep_scale, seed, (unsigned long long)(r * ldp_fwd + c));
        dot += (p[i].x * gv[i].x + p[i].y * gv[i].y) + (p[i].z * gv[i].z + p[i].w * gv[i].w);
      } else {
        p[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    dot = sx::warp_sum(dot);
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      if (c < L) {
        float4 d = make_float4(p[i].x * (gv[i].x - dot), p[i].y * (gv[i].y - dot), p[i].z * (gv[i].z - dot),
                               p[i].w * (gv[i].w - dot));
        if (do_clip) {
          if (NV <= 8) {
            if (!(inside >> (i * 4 + 0) & 1u)) d.x = 0.f;
            if (!(inside >> (i * 4 + 1) & 1u)) d.y = 0.f;
            if (!(inside >> (i * 4 + 2) & 1u)) d.z = 0.f;
            if (!(inside >> (i * 4 + 3) & 1u)) d.w = 0.f;
          } else {
            const float4 raw = ld4(S + r * lds + c);
            if (raw.x < -clip || raw.x > clip) d.x = 0.f;
            if (raw.y < -clip || raw.y > clip) d.y = 0.f;
            if (raw.z < -clip || raw.z > clip) d.z = 0.f;
            if (raw.w < -clip || raw.w > clip) d.w = 0.f;
          }
        }
        *reinterpret_cast<float4*>(dS + r * ldo + c) = rnd4(d, rnd);
      }
    }
  }
}

// column part of a LayerNorm-type backward:  dg[c] += sum_r dy[r,c] * (x[r,c]-mean_r)*rstd_r ; db[c] += sum_r dy[r,c]
// (per row-block partials into slot blockIdx.y of `part`, [dg | db]; part_reduce adds them)
// stats rows have `sstride` floats with mean/rstd at offsets 0/1.  block (32 lanes x 8 row slots), lane owns 4 columns.
__global__ void __launch_bounds__(256)
ln_param_grad_cols_fast(const float* __restrict__ dy, const float* __restrict__ x, long long R, int C,
                        const float* __restrict__ stats, int sstride, float* __restrict__ part) {
  const int c = (blockIdx.x * 32 + threadIdx.x) * 4;
  float4 ag = make_float4(0.f, 0.f, 0.f, 0.f), ab = ag;
  if (c < C)
  {
    const long long step = (long long)gridDim.y * 8;
    for (long long r0 = (long long)blockIdx.y * 8 + threadIdx.y; r0 < R; r0 += 4 * step) {
      float4 v[4], d[4];
      float mean[4], rstd[4];
      bool ok[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long r = r0 + u * step;
        ok[u] = r < R;
        if (ok[u]) {
          mean[u] = stats[r * sstride]; rstd[u] = stats[r * sstride + 1];
          v[u] = ld4(x + r * C + c); d[u] = ld4(dy + r * C + c);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (ok[u]) {
          ag.x += d[u].x * (v[u].x - mean[u]) * rstd[u]; ag.y += d[u].y * (v[u].y - mean[u]) * rstd[u];
          ag.z += d[u].z * (v[u].z - mean[u]) * rstd[u]; ag.w += d[u].w * (v[u].w - mean[u]) * rstd[u];
          ab.x += d[u].x; ab.y += d[u].y; ab.z += d[u].z; ab.w += d[u].w;
        }
    }
  }
  __shared__ float4 s[2][8][32];
  s[0][threadIdx.y][threadIdx.x] = ag; s[1][threadIdx.y][threadIdx.x] = ab;
  __syncthreads();
  if (threadIdx.y < 2 && c < C) {
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int y = 0; y < 8; ++y) {
      const float4 u = s[threadIdx.y][y][threadIdx.x];
      t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
    }
    // slot blockIdx.y: [dg (C) | db (C)], added by part_reduce
    *reinterpret_cast<float4*>(part + (long long)blockIdx.y * (2 * C) + threadIdx.y * C + c) = t;
  }
}

// VEC consecutive floats (VEC = 4: one 16-byte access), through the read-only path when RO
template <int VEC, bool RO = false>
__device__ __forceinline__ void ldv(float (&v)[VEC], const float* p) {
  if constexpr (VEC == 4) {
    const float4 t = RO ? ld4(p) : *reinterpret_cast<const float4*>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
  } else {
    v[0] = RO ? __ldg(p) : *p;
  }
}
template <int VEC>
__device__ __forceinline__ void stv(float* p, const float (&v)[VEC]) {
  if constexpr (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(v[0], v[1], v[2], v[3]);
  else *p = v[0];
}
// dpe[(b*bstride) + n*C0 + c] += posw * sum over the batch (shared code) or the sample itself (per-sample code) of dt,
// the batch added in order.  VEC = 4: float4 accesses (C, C0 and pe_bstride multiples of 4, 16-byte aligned); VEC = 1:
// any width.
template <int VEC>
__global__ void pos_grad_from_dt(const float* __restrict__ dt, int B, int N, int C, int C0, long long pe_bstride,
                                 float posw, float* __restrict__ dpe) {
  const int CV = C / VEC;
  const long long total = (long long)N * CV;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / CV;
    const int c = (int)(i % CV) * VEC;
    float v[VEC], cur[VEC];
    if (pe_bstride == 0) {
      float acc[VEC];
#pragma unroll
      for (int j = 0; j < VEC; ++j) acc[j] = 0.f;
      for (int bi = 0; bi < B; ++bi) {
        ldv<VEC, true>(v, dt + ((long long)bi * N + n) * C + c);
#pragma unroll
        for (int j = 0; j < VEC; ++j) acc[j] += v[j];
      }
      float* o = dpe + n * C0 + c;
      ldv<VEC>(cur, o);
#pragma unroll
      for (int j = 0; j < VEC; ++j) cur[j] += posw * acc[j];
      stv<VEC>(o, cur);
    } else {
      for (int bi = 0; bi < B; ++bi) {
        ldv<VEC, true>(v, dt + ((long long)bi * N + n) * C + c);
        float* o = dpe + bi * pe_bstride + n * C0 + c;
        ldv<VEC>(cur, o);
#pragma unroll
        for (int j = 0; j < VEC; ++j) cur[j] += posw * v[j];
        stv<VEC>(o, cur);
      }
    }
  }
}

// LayerNorm (affine) backward, row part: dx only
template <int NV>
__global__ void __launch_bounds__(FAST_WARPS * 32)
layernorm_bwd_rows_fast(const float* __restrict__ dy, const float* __restrict__ x, long long R, int C,
                        const float* __restrict__ g, const float* __restrict__ stats, float* __restrict__ dx, int rnd) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long long r = (long long)blockIdx.x * FAST_WARPS + warp; r < R; r += (long long)gridDim.x * FAST_WARPS) {
    const float m = stats[r * 2], rs = stats[r * 2 + 1];
    float4 a[NV], d[NV];
    row_load<NV>(a, x + r * C, C, lane);
    row_load<NV>(d, dy + r * C, C, lane);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      if (c < C) {
        const float4 gg = ld4(g + c);
        a[i].x = (a[i].x - m) * rs; a[i].y = (a[i].y - m) * rs; a[i].z = (a[i].z - m) * rs; a[i].w = (a[i].w - m) * rs;
        d[i].x *= gg.x; d[i].y *= gg.y; d[i].z *= gg.z; d[i].w *= gg.w;
        s1 += (d[i].x + d[i].y) + (d[i].z + d[i].w);
        s2 += (d[i].x * a[i].x + d[i].y * a[i].y) + (d[i].z * a[i].z + d[i].w * a[i].w);
      }
    }
    s1 = sx::warp_sum(s1) / C; s2 = sx::warp_sum(s2) / C;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      if (c < C) {
        float4 o;
        o.x = rs * (d[i].x - s1 - a[i].x * s2); o.y = rs * (d[i].y - s1 - a[i].y * s2);
        o.z = rs * (d[i].z - s1 - a[i].z * s2); o.w = rs * (d[i].w - s1 - a[i].w * s2);
        *reinterpret_cast<float4*>(dx + r * C + c) = rnd4(o, rnd);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// softmax over LONG rows (L up to 1024*EPT): one 256-thread block per row, the row lives in registers
// (thread t holds float4 columns 4t + 1024 i), block-wide max / sum through warp shuffles + shared memory.
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float block_reduce(float v, bool is_max, float* sbuf) {
  v = is_max ? sx::warp_max(v) : sx::warp_sum(v);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();                                  // sbuf reuse
  if (lane == 0) sbuf[warp] = v;
  __syncthreads();
  float r = (lane < (blockDim.x >> 5)) ? sbuf[lane] : (is_max ? -3.0e38f : 0.f);
  r = is_max ? sx::warp_max(r) : sx::warp_sum(r);
  return r;
}

template <int EPT>
__global__ void __launch_bounds__(256)
softmax_fwd_block(const float* __restrict__ S, long long R, int L, long long lds, const float* __restrict__ amax,
                  float clip, float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                  float* __restrict__ P, long long ldp, float* __restrict__ lse, int rnd, float* __restrict__ diag) {
  seed += seed_dev ? *seed_dev : 0ull;
  __shared__ float sbuf[8];
  const bool do_clip = amax && (*amax > clip);
  if (diag && amax && blockIdx.x == 0 && threadIdx.x == 0) {
    diag[0] = fmaxf(diag[0], *amax);
    if (do_clip) diag[1] += 1.f;
  }
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = blockIdx.x; r < R; r += gridDim.x) {
    float4 v[EPT];
    float m = -3.0e38f;
#pragma unroll
    for (int i = 0; i < EPT; ++i) {
      const int c = 4 * threadIdx.x + 1024 * i;
      if (c < L) {
        v[i] = ld4(S + r * lds + c);
        if (do_clip) {
          v[i].x = fminf(fmaxf(v[i].x, -clip), clip); v[i].y = fminf(fmaxf(v[i].y, -clip), clip);
          v[i].z = fminf(fmaxf(v[i].z, -clip), clip); v[i].w = fminf(fmaxf(v[i].w, -clip), clip);
        }
        m = fmaxf(m, fmaxf(fmaxf(v[i].x, v[i].y), fmaxf(v[i].z, v[i].w)));
      }
    }
    m = block_reduce(m, true, sbuf);
    float sum = 0.f;
#pragma unroll
    for (int i = 0; i < EPT; ++i)
      if (4 * threadIdx.x + 1024 * i < L) {
        v[i].x = __expf(v[i].x - m); v[i].y = __expf(v[i].y - m); v[i].z = __expf(v[i].z - m); v[i].w = __expf(v[i].w - m);
        sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
      }
    sum = block_reduce(sum, false, sbuf);
    const float inv = 1.f / sum;
#pragma unroll
    for (int i = 0; i < EPT; ++i) {
      const int c = 4 * threadIdx.x + 1024 * i;
      if (c < L) {
        float4 p = make_float4(v[i].x * inv, v[i].y * inv, v[i].z * inv, v[i].w * inv);
        if (drop_p > 0.f) p = drop4(p, drop_p, keep_scale, seed, (unsigned long long)(r * ldp + c));
        *reinterpret_cast<float4*>(P + r * ldp + c) = rnd4(p, rnd);
      }
    }
    if (threadIdx.x == 0 && lse) lse[r] = m + __logf(sum);
  }
}

template <int EPT>
__global__ void __launch_bounds__(256)
softmax_bwd_block(const float* __restrict__ dP, long long ldd, const float* __restrict__ S, long long lds,
                  const float* __restrict__ lse, long long R, int L, const float* __restrict__ amax, float clip,
                  float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                  long long ldp_fwd, float* __restrict__ dS, long long ldo, int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;
  __shared__ float sbuf[8];
  const bool do_clip = amax && (*amax > clip);
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = blockIdx.x; r < R; r += gridDim.x) {
    const float l = lse[r];
    float4 p[EPT], gv[EPT];
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < EPT; ++i) {
      const int c = 4 * threadIdx.x + 1024 * i;
      if (c < L) {
        float4 x = ld4(S + r * lds + c);
        if (do_clip) {
          x.x = fminf(fmaxf(x.x, -clip), clip); x.y = fminf(fmaxf(x.y, -clip), clip);
          x.z = fminf(fmaxf(x.z, -clip), clip); x.w = fminf(fmaxf(x.w, -clip), clip);
        }
        p[i] = make_float4(__expf(x.x - l), __expf(x.y - l), __expf(x.z - l), __expf(x.w - l));
        gv[i] = ld4(dP + r * ldd + c);
        if (drop_p > 0.f) gv[i] = drop4(gv[i], drop_p, keep_scale, seed, (unsigned long long)(r * ldp_fwd + c));
        dot += (p[i].x * gv[i].x + p[i].y * gv[i].y) + (p[i].z * gv[i].z + p[i].w * gv[i].w);
      }
    }
    dot = block_reduce(dot, false, sbuf);
#pragma unroll
    for (int i = 0; i < EPT; ++i) {
      const int c = 4 * threadIdx.x + 1024 * i;
      if (c < L) {
        float4 d = make_float4(p[i].x * (gv[i].x - dot), p[i].y * (gv[i].y - dot), p[i].z * (gv[i].z - dot),
                               p[i].w * (gv[i].w - dot));
        if (do_clip) {
          const float4 raw = ld4(S + r * lds + c);
          if (raw.x < -clip || raw.x > clip) d.x = 0.f;
          if (raw.y < -clip || raw.y > clip) d.y = 0.f;
          if (raw.z < -clip || raw.z > clip) d.z = 0.f;
          if (raw.w < -clip || raw.w > clip) d.w = 0.f;
        }
        *reinterpret_cast<float4*>(dS + r * ldo + c) = rnd4(d, rnd);
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------
// batched transpose [Z,R,C] -> [Z,C,R] with output row pitch ldo, 32 x 128 tiles, float4 global accesses on both sides
// (R%4==0, C%4==0, ldo%4==0)
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
transpose_v4_kernel(const float* __restrict__ in, int R, int C, int ldo, float* __restrict__ out) {
  __shared__ float tile[32][129];
  const long long z = blockIdx.z;
  const float* src = in + z * (long long)R * C;
  float* dst = out + z * (long long)C * ldo;
  const int c0 = blockIdx.x * 128, r0 = blockIdx.y * 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;          // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int r = r0 + j, c = c0 + tx * 4;
    if (r < R && c < C) {
      const float4 v = ld4(src + (long long)r * C + c);
      tile[j][tx * 4 + 0] = v.x; tile[j][tx * 4 + 1] = v.y; tile[j][tx * 4 + 2] = v.z; tile[j][tx * 4 + 3] = v.w;
    }
  }
  __syncthreads();
  const int r4 = (threadIdx.x & 7) * 4;                            // 8 threads cover one 32-float output row segment
  for (int pass = 0; pass < 4; ++pass) {
    const int cl = pass * 32 + (threadIdx.x >> 3);
    const int c = c0 + cl, r = r0 + r4;
    if (c < C && r < R) {
      const float4 v = make_float4(tile[r4][cl], tile[r4 + 1][cl], tile[r4 + 2][cl], tile[r4 + 3][cl]);
      *reinterpret_cast<float4*>(dst + (long long)c * ldo + r) = v;
    }
  }
}

// launch helpers ---------------------------------------------------------------------------------
inline int nv_for(int C) { return C <= 256 ? 2 : (C <= 512 ? 4 : (C <= 1024 ? 8 : (C <= 2048 ? 16 : 0))); }
inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
