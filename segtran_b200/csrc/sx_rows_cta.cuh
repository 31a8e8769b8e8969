// CTA-per-token forms of the LayerNorm + soft-aggregate kernels (MMPrivateOutput tail + LearnedSoftAggregate,
// segtran_shared.py:273-274, :318-325).  One 128- or 256-thread CTA owns one token: thread t holds columns 4t + 4 TT i (i < NV)
// of ALL MM mode rows in registers, so every row of Y is read from HBM exactly once (the warp-per-token kernels re-read
// each row two to three times and, at the 2-D widths F = 1792 / 2048, keep 64+ row registers per lane and drop to 8 warps
// per SM), statistics are block reductions batched over the modes (one barrier per batch), and the backward accumulates
// the LayerNorm / score-weight column gradients in registers across the tokens a CTA visits (stored once per CTA in its
// slot of the caller's partial-sum scratch and summed in slot order by part_reduce) instead of a second column-parallel kernel that reads Y again.
// Included by sx_rows.cu inside its anonymous namespace (after sx_rows_fast.cuh).
#pragma once

// TT = threads per token (128, or 256 for rows of more than 1024 floats: the register footprint per thread stays that of
// the 1024-wide case)

// sum of K per-thread values over the CTA, all results to all threads; `red` holds 2 * CTA_W * K floats (double buffered by
// `par` so that one barrier per call suffices)
template <int K, int TT>
__device__ __forceinline__ void cta_sum(float (&v)[K], float* red, int& par) {
  constexpr int CTA_W = TT / 32;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* buf = red + par * (CTA_W * K);
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float s = sx::warp_sum(v[k]);
    if (lane == 0) buf[warp * K + k] = s;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < CTA_W; ++w) s += buf[w * K + k];
    v[k] = s;
  }
  par ^= 1;
}

template <int NV, int MM, int TT>
__global__ void __launch_bounds__(TT, TT == 256 ? 2 : 4)
ln_softaggr_fwd_cta(const float* __restrict__ Y, int B, int N, int F, const float* __restrict__ g, const float* __restrict__ b,
                    const float* __restrict__ ws, const float* __restrict__ bs, float drop_p, unsigned long long seed,
                    const unsigned long long* __restrict__ seed_dev, float* __restrict__ out, float* __restrict__ stats,
                    float* __restrict__ wts) {
  seed += seed_dev ? *seed_dev : 0ull;
  __shared__ float red[2 * (TT / 32) * MM];
  int par = 0;
  const int tid = threadIdx.x;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const uint32_t p16 = sx::drop_p16(drop_p);
  float4 gg[NV], bb[NV], ww[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 4 * tid + 4 * TT * i;
    if (c < F) {
      gg[i] = ld4(g + c); bb[i] = ld4(b + c); ww[i] = ld4(ws + c);
    } else {
      gg[i] = bb[i] = ww[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  const float bs0 = bs[0];
  const long long T_ = (long long)B * N;
  for (long long t = blockIdx.x; t < T_; t += gridDim.x) {
    const long long bi = t / N, ni = t % N;
    float4 v[MM][NV];
#pragma unroll
    for (int m = 0; m < MM; ++m) {
      const long long ro = (bi * MM + m) * N + ni;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * tid + 4 * TT * i;
        v[m][i] = c < F ? *reinterpret_cast<const float4*>(Y + ro * F + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    if (drop_p > 0.f) {
#pragma unroll
      for (int m = 0; m < MM; ++m) {
        const long long ro = (bi * MM + m) * N + ni;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          const int c = 4 * tid + 4 * TT * i;
          if (c < F) v[m][i] = mask4(v[m][i], keep4(seed, (unsigned long long)(ro * F + c), p16), keep_scale);
        }
      }
    }
    float mean[MM], rstd[MM], sc[MM];
#pragma unroll
    for (int m = 0; m < MM; ++m) {
      float s = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) s += (v[m][i].x + v[m][i].y) + (v[m][i].z + v[m][i].w);
      mean[m] = s;
    }
    cta_sum<MM, TT>(mean, red, par);
#pragma unroll
    for (int m = 0; m < MM; ++m) {
      mean[m] /= F;
      float q = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i)
        if (4 * tid + 4 * TT * i < F) {
          const float a0 = v[m][i].x - mean[m], a1 = v[m][i].y - mean[m], a2 = v[m][i].z - mean[m], a3 = v[m][i].w - mean[m];
          v[m][i] = make_float4(a0, a1, a2, a3);                    // keep the centred values
          q += (a0 * a0 + a1 * a1) + (a2 * a2 + a3 * a3);
        }
      rstd[m] = q;
    }
    cta_sum<MM, TT>(rstd, red, par);
#pragma unroll
    for (int m = 0; m < MM; ++m) {
      rstd[m] = rsqrtf(rstd[m] / F + LN_EPS);
      float d = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        v[m][i].x = v[m][i].x * rstd[m] * gg[i].x + bb[i].x; v[m][i].y = v[m][i].y * rstd[m] * gg[i].y + bb[i].y;
        v[m][i].z = v[m][i].z * rstd[m] * gg[i].z + bb[i].z; v[m][i].w = v[m][i].w * rstd[m] * gg[i].w + bb[i].w;
        d += (v[m][i].x * ww[i].x + v[m][i].y * ww[i].y) + (v[m][i].z * ww[i].z + v[m][i].w * ww[i].w);
      }
      sc[m] = d;                                                     // (out-of-range columns: g = b = ws = 0 -> contribute 0)
    }
    cta_sum<MM, TT>(sc, red, par);
    float mx = -3.0e38f, den = 0.f;
#pragma unroll
    for (int m = 0; m < MM; ++m) { sc[m] += bs0; mx = fmaxf(mx, sc[m]); }
#pragma unroll
    for (int m = 0; m < MM; ++m) { sc[m] = __expf(sc[m] - mx); den += sc[m]; }
    const float inv = 1.f / den;
    if (tid == 0) {
#pragma unroll
      for (int m = 0; m < MM; ++m) {
        const long long ro = (bi * MM + m) * N + ni;
        stats[ro * 2] = mean[m]; stats[ro * 2 + 1] = rstd[m];
        wts[ro] = sc[m] * inv;
      }
    }
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * tid + 4 * TT * i;
      if (c < F) {
        float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int m = 0; m < MM; ++m) {
          const float w = sc[m] * inv;
          o.x += w * v[m][i].x; o.y += w * v[m][i].y; o.z += w * v[m][i].z; o.w += w * v[m][i].w;
        }
        *reinterpret_cast<float4*>(out + t * F + c) = o;
      }
    }
  }
}

template <int NV, int MM, int TT>
__global__ void __launch_bounds__(TT, TT == 256 ? 2 : 3)
ln_softaggr_bwd_cta(const float* __restrict__ dout, const float* __restrict__ Y, int B, int N, int F, const float* __restrict__ g,
                    const float* __restrict__ b, const float* __restrict__ ws, float drop_p, unsigned long long seed,
                    const unsigned long long* __restrict__ seed_dev, const float* __restrict__ stats,
                    const float* __restrict__ wts, float* __restrict__ dY, int rnd, float* __restrict__ part) {
  seed += seed_dev ? *seed_dev : 0ull;
  __shared__ float red[2 * (TT / 32) * 2 * MM];
  int par = 0;
  const int tid = threadIdx.x;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const uint32_t p16 = sx::drop_p16(drop_p);
  float4 gg[NV], bb[NV], ww[NV], ag[NV], ab[NV], aw[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 4 * tid + 4 * TT * i;
    if (c < F) { gg[i] = ld4(g + c); bb[i] = ld4(b + c); ww[i] = ld4(ws + c); }
    else gg[i] = bb[i] = ww[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    ag[i] = ab[i] = aw[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float dbs_acc = 0.f;
  const long long T_ = (long long)B * N;
  for (long long t = blockIdx.x; t < T_; t += gridDim.x) {
    const long long bi = t / N, ni = t % N;
    float4 v[MM][NV], go[NV];
    unsigned long long keep = ~0ull;                      // 4 bits per (mode, i) float4 group
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * tid + 4 * TT * i;
      go[i] = c < F ? *reinterpret_cast<const float4*>(dout + t * F + c) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
    float mean[MM], rstd[MM], w[MM];
#pragma unroll
    for (int m = 0; m < MM; ++m) {
      const long long ro = (bi * MM + m) * N + ni;
      mean[m] = stats[ro * 2]; rstd[m] = stats[ro * 2 + 1]; w[m] = wts[ro];
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * tid + 4 * TT * i;
        v[m][i] = c < F ? *reinterpret_cast<const float4*>(Y + ro * F + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    if (drop_p > 0.f) {
      keep = 0ull;
#pragma unroll
      for (int m = 0; m < MM; ++m) {
        const long long ro = (bi * MM + m) * N + ni;
#pragma unroll
        for (int i = 0; i < NV; ++i) {
          const int c = 4 * tid + 4 * TT * i;
          if (c < F) {
            const uint32_t bits = keep4(seed, (unsigned long long)(ro * F + c), p16);
            keep |= (unsigned long long)bits << (4 * (m * NV + i));
            v[m][i] = mask4(v[m][i], bits, keep_scale);
          }
        }
      }
    }
    // x-hat (normalised rows) in place, and dw_m = <dout, Yn_m>
    float dw[MM];
#pragma unroll
    for (int m = 0; m < MM; ++m) {
      float d = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        v[m][i].x = (v[m][i].x - mean[m]) * rstd[m]; v[m][i].y = (v[m][i].y - mean[m]) * rstd[m];
        v[m][i].z = (v[m][i].z - mean[m]) * rstd[m]; v[m][i].w = (v[m][i].w - mean[m]) * rstd[m];
        d += go[i].x * (v[m][i].x * gg[i].x + bb[i].x) + go[i].y * (v[m][i].y * gg[i].y + bb[i].y) +
             go[i].z * (v[m][i].z * gg[i].z + bb[i].z) + go[i].w * (v[m][i].w * gg[i].w + bb[i].w);
      }
      dw[m] = d;                                          // (columns >= F: go = 0)
    }
    cta_sum<MM, TT>(dw, red, par);
    float wd = 0.f;
#pragma unroll
    for (int m = 0; m < MM; ++m) wd += w[m] * dw[m];
    float ds[MM], s12[2 * MM];
#pragma unroll
    for (int m = 0; m < MM; ++m) {
      ds[m] = w[m] * (dw[m] - wd);                         // softmax backward over the modes
      float s1 = 0.f, s2 = 0.f;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const float d0 = (w[m] * go[i].x + ds[m] * ww[i].x), d1 = (w[m] * go[i].y + ds[m] * ww[i].y);
        const float d2 = (w[m] * go[i].z + ds[m] * ww[i].z), d3 = (w[m] * go[i].w + ds[m] * ww[i].w);
        // parameter-gradient column partials (d = gradient w.r.t. the normalised-affine row Yn_m)
        ag[i].x += d0 * v[m][i].x; ag[i].y += d1 * v[m][i].y; ag[i].z += d2 * v[m][i].z; ag[i].w += d3 * v[m][i].w;
        ab[i].x += d0; ab[i].y += d1; ab[i].z += d2; ab[i].w += d3;
        aw[i].x += ds[m] * (v[m][i].x * gg[i].x + bb[i].x); aw[i].y += ds[m] * (v[m][i].y * gg[i].y + bb[i].y);
        aw[i].z += ds[m] * (v[m][i].z * gg[i].z + bb[i].z); aw[i].w += ds[m] * (v[m][i].w * gg[i].w + bb[i].w);
        const float e0 = d0 * gg[i].x, e1 = d1 * gg[i].y, e2 = d2 * gg[i].z, e3 = d3 * gg[i].w;
        s1 += (e0 + e1) + (e2 + e3);
        s2 += (e0 * v[m][i].x + e1 * v[m][i].y) + (e2 * v[m][i].z + e3 * v[m][i].w);
      }
      s12[2 * m] = s1; s12[2 * m + 1] = s2;
    }
    cta_sum<2 * MM, TT>(s12, red, par);
    if (tid == 0) {
#pragma unroll
      for (int m = 0; m < MM; ++m) dbs_acc += ds[m];
    }
#pragma unroll
    for (int m = 0; m < MM; ++m) {
      const long long ro = (bi * MM + m) * N + ni;
      const float s1 = s12[2 * m] / F, s2 = s12[2 * m + 1] / F;
#pragma unroll
      for (int i = 0; i < NV; ++i) {
        const int c = 4 * tid + 4 * TT * i;
        if (c < F) {
          float4 r;
          r.x = rstd[m] * ((w[m] * go[i].x + ds[m] * ww[i].x) * gg[i].x - s1 - v[m][i].x * s2);
          r.y = rstd[m] * ((w[m] * go[i].y + ds[m] * ww[i].y) * gg[i].y - s1 - v[m][i].y * s2);
          r.z = rstd[m] * ((w[m] * go[i].z + ds[m] * ww[i].z) * gg[i].z - s1 - v[m][i].z * s2);
          r.w = rstd[m] * ((w[m] * go[i].w + ds[m] * ww[i].w) * gg[i].w - s1 - v[m][i].w * s2);
          if (drop_p > 0.f) r = mask4(r, (uint32_t)(keep >> (4 * (m * NV + i))) & 15u, keep_scale);
          *reinterpret_cast<float4*>(dY + ro * F + c) = rnd4(r, rnd);
        }
      }
    }
  }
  // column gradients: this CTA's partial sums -> its slot [dg (F) | db (F) | dws (F) | dbs (1)], added by part_reduce
  float* slot = part + (long long)blockIdx.x * (3 * F + 4);      // (slot rows stay 16-byte aligned)
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 4 * tid + 4 * TT * i;
    if (c < F) {
      *reinterpret_cast<float4*>(slot + c) = ag[i];
      *reinterpret_cast<float4*>(slot + F + c) = ab[i];
      *reinterpret_cast<float4*>(slot + 2 * F + c) = aw[i];
    }
  }
  if (tid == 0) slot[3 * F] = dbs_acc;
}

// ------------------------------------------------------------------------------------------------
// Fused prologue, CTA-per-row forms (segtran_shared.py:916, :930-934, :944-946):
//   h = mask * dropout( LN( LN_{g,b}(x) + posw * pe[..., :C] ) )
// One CTA per token row, the row in NV float4 registers per thread: x is read once and h written once with 16-byte
// accesses at any width (the warp-per-row forward staged rows in shared memory with 4-byte accesses; the backward kept
// 64 row registers per lane at the 2-D widths), and the backward accumulates dg / db in registers across the rows a CTA
// visits instead of a column-parallel kernel that re-reads x and dt.
// ------------------------------------------------------------------------------------------------
template <int NV, int TT>
__global__ void __launch_bounds__(TT, 1024 / TT)
prologue_fwd_cta(const float* __restrict__ x, long long R, int N, int C, const float* __restrict__ g, const float* __restrict__ b,
                 const float* __restrict__ pe, int C0, long long pe_bstride, float posw, const float* __restrict__ mask,
                 float drop_p, unsigned long long seed, const unsigned long long* __restrict__ seed_dev, float* __restrict__ h,
                 float* __restrict__ stats, int rnd) {
  seed += seed_dev ? *seed_dev : 0ull;
  __shared__ float red[2 * (TT / 32)];
  int par = 0;
  const int tid = threadIdx.x;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const uint32_t p16 = sx::drop_p16(drop_p);
  for (long long r = blockIdx.x; r < R; r += gridDim.x) {
    const long long bi = r / N, ni = r % N;
    const float* per = pe + bi * pe_bstride + ni * C0;
    float4 v[NV];
    float s[1] = {0.f};
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * tid + 4 * TT * i;
      v[i] = c < C ? *reinterpret_cast<const float4*>(x + r * C + c) : make_float4(0.f, 0.f, 0.f, 0.f);
      s[0] += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
    cta_sum<1, TT>(s, red, par);
    const float m1 = s[0] / C;
    s[0] = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (4 * tid + 4 * TT * i < C) {
        v[i].x -= m1; v[i].y -= m1; v[i].z -= m1; v[i].w -= m1;
        s[0] += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
      }
    cta_sum<1, TT>(s, red, par);
    const float r1 = rsqrtf(s[0] / C + LN_EPS);
    s[0] = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * tid + 4 * TT * i;
      if (c < C) {
        const float4 gg = ld4(g + c), bb = ld4(b + c), pp = ld4(per + c);
        v[i].x = v[i].x * r1 * gg.x + bb.x + posw * pp.x; v[i].y = v[i].y * r1 * gg.y + bb.y + posw * pp.y;
        v[i].z = v[i].z * r1 * gg.z + bb.z + posw * pp.z; v[i].w = v[i].w * r1 * gg.w + bb.w + posw * pp.w;
        s[0] += (v[i].x + v[i].y) + (v[i].z + v[i].w);
      }
    }
    cta_sum<1, TT>(s, red, par);
    const float m2 = s[0] / C;
    s[0] = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i)
      if (4 * tid + 4 * TT * i < C) {
        v[i].x -= m2; v[i].y -= m2; v[i].z -= m2; v[i].w -= m2;
        s[0] += (v[i].x * v[i].x + v[i].y * v[i].y) + (v[i].z * v[i].z + v[i].w * v[i].w);
      }
    cta_sum<1, TT>(s, red, par);
    const float r2 = rsqrtf(s[0] / C + LN_EPS);
    const float mk = (mask ? mask[r] : 1.f) * r2;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * tid + 4 * TT * i;
      if (c < C) {
        float4 o = make_float4(v[i].x * mk, v[i].y * mk, v[i].z * mk, v[i].w * mk);
        if (drop_p > 0.f) o = mask4(o, keep4(seed, (unsigned long long)(r * C + c), p16), keep_scale);
        *reinterpret_cast<float4*>(h + r * C + c) = rnd4(o, rnd);
      }
    }
    if (tid == 0) { stats[r * 4 + 0] = m1; stats[r * 4 + 1] = r1; stats[r * 4 + 2] = m2; stats[r * 4 + 3] = r2; }
  }
}

// dx from dh; dt (the gradient at the inner LayerNorm's input, needed by the positional-code gradient) is written to
// dt_out; dg[c] += sum_r dt * xhat1, db[c] += sum_r dt accumulated in registers, stored once per CTA in its scratch slot
template <int NV, int TT>
__global__ void __launch_bounds__(TT, 768 / TT)
prologue_bwd_cta(const float* __restrict__ dh, const float* __restrict__ x, long long R, int N, int C, const float* __restrict__ g,
                 const float* __restrict__ b, const float* __restrict__ pe, int C0, long long pe_bstride, float posw,
                 const float* __restrict__ mask, float drop_p, unsigned long long seed,
                 const unsigned long long* __restrict__ seed_dev, const float* __restrict__ stats, float* __restrict__ dx,
                 float* __restrict__ dt_out, float* __restrict__ part) {
  seed += seed_dev ? *seed_dev : 0ull;
  __shared__ float red[2 * (TT / 32) * 2];
  int par = 0;
  const int tid = threadIdx.x;
  const float keep_scale = drop_p > 0.f ? 1.f / (1.f - drop_p) : 1.f;
  const uint32_t p16 = sx::drop_p16(drop_p);
  float4 ag[NV], ab[NV];
#pragma unroll
  for (int i = 0; i < NV; ++i) ag[i] = ab[i] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (long long r = blockIdx.x; r < R; r += gridDim.x) {
    const float m1 = stats[r * 4 + 0], r1 = stats[r * 4 + 1], m2 = stats[r * 4 + 2], r2 = stats[r * 4 + 3];
    const long long bi = r / N, ni = r % N;
    const float* per = pe + bi * pe_bstride + ni * C0;
    const float mk = mask ? mask[r] : 1.f;
    float4 a[NV], yh[NV], d[NV];
    float s[2] = {0.f, 0.f};
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * tid + 4 * TT * i;
      yh[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < C) {
        a[i] = *reinterpret_cast<const float4*>(x + r * C + c);
        d[i] = *reinterpret_cast<const float4*>(dh + r * C + c);
        const float4 gg = ld4(g + c), bb = ld4(b + c), pp = ld4(per + c);
        a[i].x = (a[i].x - m1) * r1; a[i].y = (a[i].y - m1) * r1; a[i].z = (a[i].z - m1) * r1; a[i].w = (a[i].w - m1) * r1;
        yh[i].x = (a[i].x * gg.x + bb.x + posw * pp.x - m2) * r2; yh[i].y = (a[i].y * gg.y + bb.y + posw * pp.y - m2) * r2;
        yh[i].z = (a[i].z * gg.z + bb.z + posw * pp.z - m2) * r2; yh[i].w = (a[i].w * gg.w + bb.w + posw * pp.w - m2) * r2;
        d[i].x *= mk; d[i].y *= mk; d[i].z *= mk; d[i].w *= mk;
        if (drop_p > 0.f) d[i] = mask4(d[i], keep4(seed, (unsigned long long)(r * C + c), p16), keep_scale);
        s[0] += (d[i].x + d[i].y) + (d[i].z + d[i].w);
        s[1] += (d[i].x * yh[i].x + d[i].y * yh[i].y) + (d[i].z * yh[i].z + d[i].w * yh[i].w);
      } else {
        a[i] = d[i] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    cta_sum<2, TT>(s, red, par);
    const float s1 = s[0] / C, s2 = s[1] / C;
    s[0] = s[1] = 0.f;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * tid + 4 * TT * i;
      if (c < C) {
        const float4 gg = ld4(g + c);
        float4 dt;
        dt.x = r2 * (d[i].x - s1 - yh[i].x * s2); dt.y = r2 * (d[i].y - s1 - yh[i].y * s2);
        dt.z = r2 * (d[i].z - s1 - yh[i].z * s2); dt.w = r2 * (d[i].w - s1 - yh[i].w * s2);
        if (dt_out) *reinterpret_cast<float4*>(dt_out + r * C + c) = dt;
        ag[i].x += dt.x * a[i].x; ag[i].y += dt.y * a[i].y; ag[i].z += dt.z * a[i].z; ag[i].w += dt.w * a[i].w;
        ab[i].x += dt.x; ab[i].y += dt.y; ab[i].z += dt.z; ab[i].w += dt.w;
        d[i] = make_float4(dt.x * gg.x, dt.y * gg.y, dt.z * gg.z, dt.w * gg.w);
        s[0] += (d[i].x + d[i].y) + (d[i].z + d[i].w);
        s[1] += (d[i].x * a[i].x + d[i].y * a[i].y) + (d[i].z * a[i].z + d[i].w * a[i].w);
      }
    }
    cta_sum<2, TT>(s, red, par);
    const float s3 = s[0] / C, s4 = s[1] / C;
#pragma unroll
    for (int i = 0; i < NV; ++i) {
      const int c = 4 * tid + 4 * TT * i;
      if (c < C) {
        float4 o;
        o.x = r1 * (d[i].x - s3 - a[i].x * s4); o.y = r1 * (d[i].y - s3 - a[i].y * s4);
        o.z = r1 * (d[i].z - s3 - a[i].z * s4); o.w = r1 * (d[i].w - s3 - a[i].w * s4);
        *reinterpret_cast<float4*>(dx + r * C + c) = o;
      }
    }
  }
  // this CTA's partial sums -> its slot [dg (C) | db (C)], added by part_reduce
  float* slot = part + (long long)blockIdx.x * (2 * C);
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const int c = 4 * tid + 4 * TT * i;
    if (c < C) {
      *reinterpret_cast<float4*>(slot + c) = ag[i];
      *reinterpret_cast<float4*>(slot + C + c) = ab[i];
    }
  }
}
