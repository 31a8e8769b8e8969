// Register-resident fast paths of the row kernels (fp32 I/O, row length a multiple of 4, <= 128*NV floats).
// A row lives in NV float4 registers per lane (lane l holds columns 4l+128i .. +3), so there is no shared-memory
// staging, occupancy is register-limited only (32+ warps/SM) and every global access is a 16-byte vector access.
// Parameter gradients that are column sums over all rows are produced by separate column-parallel reductions
// instead of shared-memory atomics.  Included by sx_rows.cu inside its anonymous namespace.
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
// LN + soft aggregate, forward.  Pass 1 per mode: stats + score; pass 2 re-reads the (L2-resident) rows.
// ------------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(FAST_WARPS * 32, NV <= 8 ? 2 : 1)
ln_softaggr_fwd_fast(const float* __restrict__ Y, int B, int M, int N, int F, const float* __restrict__ g,
                     const float* __restrict__ b, const float* __restrict__ ws, const float* __restrict__ bs,
                     float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                     float* __restrict__ out, float* __restrict__ stats, float* __restrict__ wts) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  __shared__ float s_sc[FAST_WARPS][MAX_MODES], s_mu[FAST_WARPS][MAX_MODES], s_rs[FAST_WARPS][MAX_MODES];
  __shared__ uint32_t s_keep[FAST_WARPS][MAX_MODES][(NV + 7) / 8][32];      // dropout keep bits of pass 1, reused in pass 2
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const uint32_t p16 = sx::drop_p16(drop_p);
  const long long T_ = (long long)B * N;
  for (long long t = (long long)blockIdx.x * FAST_WARPS + warp; t < T_; t += (long long)gridDim.x * FAST_WARPS) {
    const long long bi = t / N, ni = t % N;
    // pass 1 (mode loop deliberately not unrolled: one row of registers at a time keeps occupancy high)
#pragma unroll 1
    for (int m = 0; m < M; ++m) {
      const long long ro = (bi * M + m) * N + ni;
      float4 v[NV];
      row_load<NV>(v, Y + ro * F, F, lane);
      if (drop_p > 0.f) {
        uint32_t kb[(NV + 7) / 8];
#pragma unroll
        for (int w = 0; w < (NV + 7) / 8; ++w) kb[w] = 0u;
#pragma unroll
        for (int i = 0; i < NV; ++i)
          if (4 * lane + 128 * i < F) {
            const uint32_t bits = keep4(seed, (unsigned long long)(ro * F + 4 * lane + 128 * i), p16);
            kb[i >> 3] |= bits << (4 * (i & 7));
            v[i] = mask4(v[i], bits, keep_scale);
          }
#pragma unroll
        for (int w = 0; w < (NV + 7) / 8; ++w) s_keep[warp][m][w][lane] = kb[w];
      }
      float mean, rstd;
      row_mean_rstd<NV>(v, F, lane, mean, rstd);
      float dot = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
        if (c < F) {
          const float4 gg = ld4(g + c), bb = ld4(b + c), ww = ld4(ws + c);
          dot += ((v[i].x - mean) * rstd * gg.x + bb.x) * ww.x + ((v[i].y - mean) * rstd * gg.y + bb.y) * ww.y +
                 ((v[i].z - mean) * rstd * gg.z + bb.z) * ww.z + ((v[i].w - mean) * rstd * gg.w + bb.w) * ww.w;
        }
      }
      dot = sx::warp_sum(dot) + bs[0];
      if (lane == 0) {
        s_sc[warp][m] = dot; s_mu[warp][m] = mean; s_rs[warp][m] = rstd;
        stats[ro * 2] = mean; stats[ro * 2 + 1] = rstd;
      }
    }
    __syncwarp();
    float mx = -3.0e38f, den = 0.f;
    for (int m = 0; m < M; ++m) mx = fmaxf(mx, s_sc[warp][m]);
    for (int m = 0; m < M; ++m) den += __expf(s_sc[warp][m] - mx);
    __syncwarp();
    if (lane < M) {
      const float w = __expf(s_sc[warp][lane] - mx) / den;
      s_sc[warp][lane] = w;
      wts[(bi * M + lane) * N + ni] = w;
    }
    __syncwarp();
    float4 o[NV];
#pragma unroll
    for (int i = 0; i < NV; ++i) o[i] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 1
    for (int m = 0; m < M; ++m) {
      const long long ro = (bi * M + m) * N + ni;
      const float w = s_sc[warp][m], mean = s_mu[warp][m], rstd = s_rs[warp][m];
      float4 v[NV];
      row_load<NV>(v, Y + ro * F, F, lane);
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
        if (c < F) {
          if (drop_p > 0.f) v[i] = mask4(v[i], s_keep[warp][m][i >> 3][lane] >> (4 * (i & 7)), keep_scale);
          const float4 gg = ld4(g + c), bb = ld4(b + c);
          o[i].x += w * ((v[i].x - mean) * rstd * gg.x + bb.x);
          o[i].y += w * ((v[i].y - mean) * rstd * gg.y + bb.y);
          o[i].z += w * ((v[i].z - mean) * rstd * gg.z + bb.z);
          o[i].w += w * ((v[i].w - mean) * rstd * gg.w + bb.w);
        }
      }
    }
    row_store<NV>(o, out + t * F, F, lane);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// LN + soft aggregate, backward, row part: dY and the per-(mode,token) score gradient (kept for the column pass)
// ------------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(FAST_WARPS * 32, NV <= 8 ? 2 : 1)
ln_softaggr_bwd_rows_fast(const float* __restrict__ dout, const float* __restrict__ Y, int B, int M, int N, int F,
                          const float* __restrict__ g, const float* __restrict__ b, const float* __restrict__ ws,
                          float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev,
                          const float* __restrict__ stats, const float* __restrict__ wts, float* __restrict__ dY,
                          float* __restrict__ dscore_out, float* __restrict__ dbs, int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  __shared__ float s_dw[FAST_WARPS][MAX_MODES], s_w[FAST_WARPS][MAX_MODES];
  __shared__ uint32_t s_keep[FAST_WARPS][MAX_MODES][(NV + 7) / 8][32];      // dropout keep bits: hashed once, used 3 times
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const uint32_t p16 = sx::drop_p16(drop_p);
  const long long T_ = (long long)B * N;
  float dbs_acc = 0.f;
  for (long long t = (long long)blockIdx.x * FAST_WARPS + warp; t < T_; t += (long long)gridDim.x * FAST_WARPS) {
    const long long bi = t / N, ni = t % N;
    float4 go[NV];
    row_load<NV>(go, dout + t * F, F, lane);
#pragma unroll 1
    for (int m = 0; m < M; ++m) {                       // pass 1: dw_m = <dout, Yn_m>
      const long long ro = (bi * M + m) * N + ni;
      const float mean = stats[ro * 2], rstd = stats[ro * 2 + 1];
      float4 v[NV];
      row_load<NV>(v, Y + ro * F, F, lane);
      float dot = 0.f;
      uint32_t kb[(NV + 7) / 8];
#pragma unroll
      for (int w = 0; w < (NV + 7) / 8; ++w) kb[w] = 0u;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
        if (c < F) {
          if (drop_p > 0.f) {
            const uint32_t bits = keep4(seed, (unsigned long long)(ro * F + c), p16);
            kb[i >> 3] |= bits << (4 * (i & 7));
            v[i] = mask4(v[i], bits, keep_scale);
          }
          const float4 gg = ld4(g + c), bb = ld4(b + c);
          dot += go[i].x * ((v[i].x - mean) * rstd * gg.x + bb.x) + go[i].y * ((v[i].y - mean) * rstd * gg.y + bb.y) +
                 go[i].z * ((v[i].z - mean) * rstd * gg.z + bb.z) + go[i].w * ((v[i].w - mean) * rstd * gg.w + bb.w);
        }
      }
      dot = sx::warp_sum(dot);
      if (drop_p > 0.f) {
#pragma unroll
        for (int w = 0; w < (NV + 7) / 8; ++w) s_keep[warp][m][w][lane] = kb[w];
      }
      if (lane == 0) { s_dw[warp][m] = dot; s_w[warp][m] = wts[(bi * M + m) * N + ni]; }
    }
    __syncwarp();
    float wd = 0.f;
    for (int m = 0; m < M; ++m) wd += s_w[warp][m] * s_dw[warp][m];
#pragma unroll 1
    for (int m = 0; m < M; ++m) {                       // pass 2: dY_m
      const float wm = s_w[warp][m];
      const float dscore = wm * (s_dw[warp][m] - wd);   // softmax backward over modes
      dbs_acc += dscore;
      const long long ro = (bi * M + m) * N + ni;
      if (lane == 0) dscore_out[ro] = dscore;
      const float mean = stats[ro * 2], rstd = stats[ro * 2 + 1];
      float4 v[NV];
      row_load<NV>(v, Y + ro * F, F, lane);
      float s1 = 0.f, s2 = 0.f;
      // v <- normalised row a (dropout applied), go-derived d kept implicitly: d = (wm*go + dscore*ws) * g
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
        if (c < F) {
          if (drop_p > 0.f) v[i] = mask4(v[i], s_keep[warp][m][i >> 3][lane] >> (4 * (i & 7)), keep_scale);
          const float4 gg = ld4(g + c), ww = ld4(ws + c);
          v[i].x = (v[i].x - mean) * rstd; v[i].y = (v[i].y - mean) * rstd;
          v[i].z = (v[i].z - mean) * rstd; v[i].w = (v[i].w - mean) * rstd;
          const float d0 = (wm * go[i].x + dscore * ww.x) * gg.x, d1 = (wm * go[i].y + dscore * ww.y) * gg.y;
          const float d2 = (wm * go[i].z + dscore * ww.z) * gg.z, d3 = (wm * go[i].w + dscore * ww.w) * gg.w;
          s1 += (d0 + d1) + (d2 + d3);
          s2 += (d0 * v[i].x + d1 * v[i].y) + (d2 * v[i].z + d3 * v[i].w);
        }
      }
      s1 = sx::warp_sum(s1) / F; s2 = sx::warp_sum(s2) / F;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * lane + 128 * i;
        if (c < F) {
          const float4 gg = ld4(g + c), ww = ld4(ws + c);
          float4 r;
          r.x = rstd * ((wm * go[i].x + dscore * ww.x) * gg.x - s1 - v[i].x * s2);
          r.y = rstd * ((wm * go[i].y + dscore * ww.y) * gg.y - s1 - v[i].y * s2);
          r.z = rstd * ((wm * go[i].z + dscore * ww.z) * gg.z - s1 - v[i].z * s2);
          r.w = rstd * ((wm * go[i].w + dscore * ww.w) * gg.w - s1 - v[i].w * s2);
          if (drop_p > 0.f) r = mask4(r, s_keep[warp][m][i >> 3][lane] >> (4 * (i & 7)), keep_scale);
          *reinterpret_cast<float4*>(dY + ro * F + c) = rnd4(r, rnd);
        }
      }
    }
    __syncwarp();
  }
  if (lane == 0 && dbs_acc != 0.f) atomicAdd(dbs, dbs_acc);
}

// column part: dg[c] += sum_r dyn a ; db[c] += sum_r dyn ; dws[c] += sum_r dscore yn   (r over all (b,m,n) rows)
// block (32 lanes x 8 row-slots); lane owns 4 consecutive columns.
__global__ void __launch_bounds__(256)
ln_softaggr_bwd_cols_fast(const float* __restrict__ dout, const float* __restrict__ Y, int B, int M, int N, int F,
                          const float* __restrict__ g, const float* __restrict__ b, const float* __restrict__ ws,
                          float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev, const float* __restrict__ stats,
                          const float* __restrict__ wts, const float* __restrict__ dscore_in, float* __restrict__ dg,
                          float* __restrict__ db, float* __restrict__ dws) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  const int c = (blockIdx.x * 32 + threadIdx.x) * 4;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  float4 ag = make_float4(0.f, 0.f, 0.f, 0.f), ab = ag, aw = ag;
  const long long R = (long long)B * M * N;
  if (c < F) {
    const float4 gg = ld4(g + c), bb = ld4(b + c), ww = ld4(ws + c);
    const long long step = (long long)gridDim.y * 8;
    for (long long r0 = (long long)blockIdx.y * 8 + threadIdx.y; r0 < R; r0 += 4 * step) {
      // 4 independent rows per iteration: 8 float4 loads in flight per thread
      float4 v[4], go[4];
      float mean[4], rstd[4], w[4], ds[4];
      bool ok[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const long long r = r0 + u * step;
        ok[u] = r < R;
        if (ok[u]) {
          const long long bm = r / N, ni = r % N, bi = bm / M;
          mean[u] = stats[r * 2]; rstd[u] = stats[r * 2 + 1]; w[u] = wts[r]; ds[u] = dscore_in[r];
          v[u] = ld4(Y + r * F + c);
          go[u] = ld4(dout + (bi * N + ni) * F + c);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (ok[u]) {
          const long long r = r0 + u * step;
          float4 x = v[u];
          if (drop_p > 0.f) x = drop4(x, drop_p, keep_scale, seed, (unsigned long long)(r * F + c));
          const float a0 = (x.x - mean[u]) * rstd[u], a1 = (x.y - mean[u]) * rstd[u], a2 = (x.z - mean[u]) * rstd[u],
                      a3 = (x.w - mean[u]) * rstd[u];
          const float d0 = w[u] * go[u].x + ds[u] * ww.x, d1 = w[u] * go[u].y + ds[u] * ww.y,
                      d2 = w[u] * go[u].z + ds[u] * ww.z, d3 = w[u] * go[u].w + ds[u] * ww.w;
          ag.x += d0 * a0; ag.y += d1 * a1; ag.z += d2 * a2; ag.w += d3 * a3;
          ab.x += d0; ab.y += d1; ab.z += d2; ab.w += d3;
          aw.x += ds[u] * (a0 * gg.x + bb.x); aw.y += ds[u] * (a1 * gg.y + bb.y);
          aw.z += ds[u] * (a2 * gg.z + bb.z); aw.w += ds[u] * (a3 * gg.w + bb.w);
        }
    }
  }
  __shared__ float4 s[3][8][32];
  s[0][threadIdx.y][threadIdx.x] = ag; s[1][threadIdx.y][threadIdx.x] = ab; s[2][threadIdx.y][threadIdx.x] = aw;
  __syncthreads();
  if (threadIdx.y < 3 && c < F) {
    float4 t = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int y = 0; y < 8; ++y) {
      const float4 u = s[threadIdx.y][y][threadIdx.x];
      t.x += u.x; t.y += u.y; t.z += u.z; t.w += u.w;
    }
    float* dst = threadIdx.y == 0 ? dg : (threadIdx.y == 1 ? db : dws);
    atomicAdd(dst + c, t.x); atomicAdd(dst + c + 1, t.y); atomicAdd(dst + c + 2, t.z); atomicAdd(dst + c + 3, t.w);
  }
}

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

// ------------------------------------------------------------------------------------------------
// prologue backward: row part (dx, and dt = gradient at the inner LayerNorm's input, kept for the column pass)
// ------------------------------------------------------------------------------------------------
template <int NV>
__global__ void __launch_bounds__(FAST_WARPS * 32)
prologue_bwd_rows_fast(const float* __restrict__ dh, const float* __restrict__ x, long long R, int N, int C,
                       const float* __restrict__ g, const float* __restrict__ b, const float* __restrict__ pe, int C0,
                       long long pe_bstride, float posw, const float* __restrict__ mask, float drop_p,
                       unsigned long long seed, const unsigned long long* __restrict__ seed_dev, const float* __restrict__ stats, float* __restrict__ dx,
                       float* __restrict__ dt_out) {
  seed += seed_dev ? *seed_dev : 0ull;      // per-call device seed (CUDA-graph safe)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  for (long long r = (long long)blockIdx.x * FAST_WARPS + warp; r < R; r += (long long)gridDim.x * FAST_WARPS) {
    const float m1 = stats[r * 4 + 0], r1 = stats[r * 4 + 1], m2 = stats[r * 4 + 2], r2 = stats[r * 4 + 3];
    const long long bi = r / N, ni = r % N;
    const float* per = pe + bi * pe_bstride + ni * C0;
    const float mk = mask ? mask[r] : 1.f;
    float4 a[NV], yh[NV], d[NV];
    row_load<NV>(a, x + r * C, C, lane);
    row_load<NV>(d, dh + r * C, C, lane);
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      yh[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < C) {
        const float4 gg = ld4(g + c), bb = ld4(b + c), pp = ld4(per + c);
        a[i].x = (a[i].x - m1) * r1; a[i].y = (a[i].y - m1) * r1; a[i].z = (a[i].z - m1) * r1; a[i].w = (a[i].w - m1) * r1;
        yh[i].x = (a[i].x * gg.x + bb.x + posw * pp.x - m2) * r2; yh[i].y = (a[i].y * gg.y + bb.y + posw * pp.y - m2) * r2;
        yh[i].z = (a[i].z * gg.z + bb.z + posw * pp.z - m2) * r2; yh[i].w = (a[i].w * gg.w + bb.w + posw * pp.w - m2) * r2;
        d[i].x *= mk; d[i].y *= mk; d[i].z *= mk; d[i].w *= mk;
        if (drop_p > 0.f) d[i] = drop4(d[i], drop_p, keep_scale, seed, (unsigned long long)(r * C + c));
        s1 += (d[i].x + d[i].y) + (d[i].z + d[i].w);
        s2 += (d[i].x * yh[i].x + d[i].y * yh[i].y) + (d[i].z * yh[i].z + d[i].w * yh[i].w);
      }
    }
    s1 = sx::warp_sum(s1) / C; s2 = sx::warp_sum(s2) / C;
    float s3 = 0.f, s4 = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      if (c < C) {
        const float4 gg = ld4(g + c);
        float4 dt;
        dt.x = r2 * (d[i].x - s1 - yh[i].x * s2); dt.y = r2 * (d[i].y - s1 - yh[i].y * s2);
        dt.z = r2 * (d[i].z - s1 - yh[i].z * s2); dt.w = r2 * (d[i].w - s1 - yh[i].w * s2);
        *reinterpret_cast<float4*>(dt_out + r * C + c) = dt;
        d[i] = make_float4(dt.x * gg.x, dt.y * gg.y, dt.z * gg.z, dt.w * gg.w);
        s3 += (d[i].x + d[i].y) + (d[i].z + d[i].w);
        s4 += (d[i].x * a[i].x + d[i].y * a[i].y) + (d[i].z * a[i].z + d[i].w * a[i].w);
      }
    }
    s3 = sx::warp_sum(s3) / C; s4 = sx::warp_sum(s4) / C;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * lane + 128 * i;
      if (c < C) {
        float4 o;
        o.x = r1 * (d[i].x - s3 - a[i].x * s4); o.y = r1 * (d[i].y - s3 - a[i].y * s4);
        o.z = r1 * (d[i].z - s3 - a[i].z * s4); o.w = r1 * (d[i].w - s3 - a[i].w * s4);
        *reinterpret_cast<float4*>(dx + r * C + c) = o;
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

// dpe[(b*bstride) + n*C0 + c] += posw * sum over the batch (shared code) or the sample itself (per-sample code) of dt
__global__ void pos_grad_from_dt_fast(const float* __restrict__ dt, int B, int N, int C, int C0, long long pe_bstride,
                                      float posw, float* __restrict__ dpe) {
  const long long total = (long long)N * (C / 4);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long n = i / (C / 4);
    const int c = (int)(i % (C / 4)) * 4;
    if (pe_bstride == 0) {
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int bi = 0; bi < B; ++bi) {
        const float4 v = ld4(dt + ((long long)bi * N + n) * C + c);
        acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
      }
      float4* o = reinterpret_cast<float4*>(dpe + n * C0 + c);
      float4 cur = *o;
      cur.x += posw * acc.x; cur.y += posw * acc.y; cur.z += posw * acc.z; cur.w += posw * acc.w;
      *o = cur;
    } else {
      for (int bi = 0; bi < B; ++bi) {
        const float4 v = ld4(dt + ((long long)bi * N + n) * C + c);
        float4* o = reinterpret_cast<float4*>(dpe + bi * pe_bstride + n * C0 + c);
        float4 cur = *o;
        cur.x += posw * v.x; cur.y += posw * v.y; cur.z += posw * v.z; cur.w += posw * v.w;
        *o = cur;
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
