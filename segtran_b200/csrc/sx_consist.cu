// Attention-consistency loss of one layer (train3d.py:426-449, train2d.py:668-723) without the N x N matrices.
//
// Pair input (squeezed layers, X_b = Xo_b . Xi_b): a persistent wgmma kernel, a sibling of sx_attn_probs_kernel.  A work
// item is 128 rows i of one batch; the CTA walks the 128-column chunks j, each chunk's X tile is one accumulator per
// consumer warpgroup (64 rows each), and the loss term, its per-thread sums and the optional residual are computed on
// the fragments.  The K x 128 column slice of the mask F a chunk needs is staged in shared memory (double-buffered per
// warpgroup, one named barrier per chunk); the warpgroup's 64-row slice once per item.
//
// Dense input (--nosqueeze layers, X given as [B,N,N]): a row kernel with the same per-element code (sx_consist.cuh).
//
// Sums: every thread keeps (sum, sign sum, count) for the item / batch it is on; at the end of an item (pair) or of a
// batch's rows (dense) the CTA reduces them in a fixed order and adds them to its own slot of `part` ([B][3]); one
// thread then adds the slots in slot order (consist_finalize_kernel).  Counts travel as integers.  No float atomics.
#include <algorithm>

#include "sx_common.cuh"
#include "sx_consist.cuh"
#include "sx_tc.cuh"

namespace {
using namespace sxtc;

constexpr int NUM_THREADS = 384;          // warpgroup 0: TMA producer; warpgroups 1-2: MMA + loss terms, 64 rows each
constexpr int STAGES = 4;
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int F_ROW_FLOATS = sxcs::MAX_K * 64;                 // per consumer warpgroup: [K][64] row slice
constexpr int F_COL_FLOATS = sxcs::MAX_K * BN;                 //                         [K][128] column slice, x2
constexpr int F_WG_FLOATS = F_ROW_FLOATS + 2 * F_COL_FLOATS;
constexpr int F_OFFSET = STAGES * STAGE_BYTES + 256;
constexpr int RED_OFFSET = F_OFFSET + 2 * F_WG_FLOATS * 4;     // [2 parities][8 consumer warps][3]
constexpr int SMEM_BYTES = RED_OFFSET + 2 * 8 * 3 * 4 + 1024 /*align*/;
constexpr int DENSE_THREADS = 256;

struct CsParams {
  int B, N, K, variant, tiles, num_kb, items, round_r;
  const float* F;
  const float* mu;
  float* R;
  long long ldr;
  float* part;                    // this launch's slots: [gridDim.x][B][3]
};

__device__ __forceinline__ void named_bar(int id, int n) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n) : "memory"); }

// residual pair -> R (TF32-rounded when it feeds the backward GEMMs)
__device__ __forceinline__ void store_r(float* row, int col, int N, float r0, float r1, int rnd) {
  if (rnd) { r0 = sx::round_tf32(r0); r1 = sx::round_tf32(r1); }
  if (col + 1 < N) *reinterpret_cast<float2*>(row + col) = make_float2(r0, r1);
  else row[col] = r0;
}

// a warp's (sum, sgn, cnt) -> red[3w..3w+2] (butterfly order), then one thread adds the warps in order to slot[0..2]
__device__ __forceinline__ void warp_partial(const sxcs::Acc& a, float* red, int w, int lane) {
  float s = a.sum, g = a.sgn;
  int c = a.cnt;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    g += __shfl_xor_sync(0xffffffffu, g, o);
    c += __shfl_xor_sync(0xffffffffu, c, o);
  }
  if (lane == 0) { red[3 * w] = s; red[3 * w + 1] = g; red[3 * w + 2] = __int_as_float(c); }
}
__device__ __forceinline__ void slot_add(const float* red, int nwarps, float* slot) {
  float s = 0.f, g = 0.f;
  int c = 0;
  for (int w = 0; w < nwarps; ++w) { s += red[3 * w]; g += red[3 * w + 1]; c += __float_as_int(red[3 * w + 2]); }
  slot[0] += s;
  slot[1] += g;
  slot[2] = __int_as_float(__float_as_int(slot[2]) + c);
}

__global__ void __launch_bounds__(NUM_THREADS, 1)
consist_pair_kernel(const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmT, const CsParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* empty_bar = full_bar + STAGES;
  float* red = reinterpret_cast<float*>(smem + RED_OFFSET);
  float* slot = p.part + (long long)blockIdx.x * p.B * 3;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    sx::tma_prefetch_desc(&tmO);
    sx::tma_prefetch_desc(&tmT);
    for (int s = 0; s < STAGES; ++s) {
      sx::mbar_init(&full_bar[s], 1);
      sx::mbar_init(&empty_bar[s], 2);
    }
    sx::fence_barrier_init();
  }
  for (int i = threadIdx.x; i < p.B * 3; i += NUM_THREADS) slot[i] = 0.f;      // (0 is also integer 0)
  __syncthreads();

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (warp == 0 && sx::elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
        const int mb = it % p.tiles, b = it / p.tiles;
        for (int nb = 0; nb < p.tiles; ++nb)
          for (int kb = 0; kb < p.num_kb; ++kb) {
            sx::mbar_wait(&empty_bar[stage], phase ^ 1);
            sx::mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
            uint8_t* sa = smem + stage * STAGE_BYTES;
            sx::tma_load_4d(sa, &tmO, &full_bar[stage], kb * 32, mb * BM, 0, b, sx::kEvictLast);
            sx::tma_load_4d(sa + A_STAGE_BYTES, &tmT, &full_bar[stage], kb * 32, nb * BN, 0, b, sx::kEvictLast);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  // thread: rows 8h + lane/4 (h = 0, 1) of its warp's 16; columns 8j + 2(lane%4) + e of each 128-column chunk
  const int cw = wg - 1;
  const int wtid = threadIdx.x & 127;
  const int wq = warp & 3;
  const int tr = lane >> 2;
  const int tc = (lane & 3) * 2;
  float* frow = reinterpret_cast<float*>(smem + F_OFFSET) + cw * F_WG_FLOATS;   // [K][64]
  float* fcol = frow + F_ROW_FLOATS;                                            // [2][K][128]
  const int N = p.N, K = p.K;
  int stage = 0;
  uint32_t phase = 0, par = 0, ipar = 0;
  float acc[64];

  for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
    const int mb = it % p.tiles, b = it / p.tiles;
    const float* Fb = p.F + (long long)b * K * N;
    const int row0 = mb * BM + cw * 64;
    for (int i = wtid; i < K * 64; i += 128) {
      const int k = i >> 6, r = row0 + (i & 63);
      frow[i] = r < N ? Fb[(long long)k * N + r] : 0.f;
    }
    const float mu = p.variant == SX_CONSIST_MARGIN ? p.mu[b] : 0.f;
    sxcs::Acc a;
    for (int nb = 0; nb < p.tiles; ++nb) {
      float* fc = fcol + par * F_COL_FLOATS;
      for (int i = wtid; i < K * BN; i += 128) {
        const int k = i >> 7, c = nb * BN + (i & 127);
        fc[i] = c < N ? Fb[(long long)k * N + c] : 0.f;
      }
      named_bar(2 + cw, 128);
      for (int kb = 0; kb < p.num_kb; ++kb) {
        sx::mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = sx::smem_u32(smem + stage * STAGE_BYTES);
        const uint32_t oa = sa + (uint32_t)(cw * 64 * BKB), ta = sa + A_STAGE_BYTES;
        sx::acc_fence(acc);
        sx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          sx::wgmma_tf32(acc, sx::gmma_desc(oa + kk * 32, 16, 1024), sx::gmma_desc(ta + kk * 32, 16, 1024),
                         (kb > 0 || kk > 0) ? 1u : 0u);
        sx::wgmma_commit();
        sx::wgmma_wait<0>();
        sx::acc_fence(acc);
        if (wtid == 0) sx::mbar_arrive(&empty_bar[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int lr = wq * 16 + 8 * h + tr, row = row0 + lr;
        if (row >= N) continue;
        float* rrow = p.R ? p.R + ((long long)b * N + row) * p.ldr : nullptr;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int cl = 8 * j + tc, col = nb * BN + cl;
          if (col >= N) continue;
          const float c0 = sxcs::target(frow + lr, 64, fc + cl, BN, K);
          const float r0 = sxcs::term(p.variant, acc[4 * j + 2 * h], c0, mu, a);
          float r1 = 0.f;
          if (col + 1 < N) {
            const float c1 = sxcs::target(frow + lr, 64, fc + cl + 1, BN, K);
            r1 = sxcs::term(p.variant, acc[4 * j + 2 * h + 1], c1, mu, a);
          }
          if (rrow) store_r(rrow, col, N, r0, r1, p.round_r);
        }
      }
      par ^= 1;
    }
    // the item's sums -> this CTA's slot of batch b (both warpgroups, fixed order)
    float* rd = red + ipar * 24;
    warp_partial(a, rd, warp - 4, lane);
    named_bar(1, 256);
    if (threadIdx.x == 128) slot_add(rd, 8, slot + 3 * b);
    ipar ^= 1;
  }
}

__global__ void __launch_bounds__(DENSE_THREADS)
consist_dense_kernel(const float* __restrict__ X, long long x_ld, long long x_bstride, const CsParams p) {
  __shared__ float red[8 * 3];
  float* slot = p.part + (long long)blockIdx.x * p.B * 3;
  for (int i = threadIdx.x; i < p.B * 3; i += DENSE_THREADS) slot[i] = 0.f;
  __syncthreads();
  const int N = p.N, K = p.K;
  const long long rows = (long long)p.B * N;
  sxcs::Acc a;
  for (long long rr = blockIdx.x; rr < rows; rr += gridDim.x) {
    const int b = (int)(rr / N), i = (int)(rr % N);
    const float* Fb = p.F + (long long)b * K * N;
    const float* x = X + b * x_bstride + (long long)i * x_ld;
    const float mu = p.variant == SX_CONSIST_MARGIN ? p.mu[b] : 0.f;
    float* rrow = p.R ? p.R + rr * p.ldr : nullptr;
    for (int j = threadIdx.x; j < N; j += DENSE_THREADS) {
      const float c = sxcs::target(Fb + i, N, Fb + j, N, K);
      const float r = sxcs::term(p.variant, x[j], c, mu, a);
      if (rrow) rrow[j] = p.round_r ? sx::round_tf32(r) : r;
    }
    const long long nx = rr + gridDim.x;
    if (nx >= rows || (int)(nx / N) != b) {         // this block's last row of batch b: flush (uniform over the block)
      warp_partial(a, red, threadIdx.x >> 5, threadIdx.x & 31);
      __syncthreads();
      if (threadIdx.x == 0) slot_add(red, DENSE_THREADS / 32, slot + 3 * b);
      __syncthreads();
      a = sxcs::Acc();
    }
  }
}

// slots -> the layer's loss, residual scale and mu terms (+ the running cap of train2d.py); one thread, slot order
__global__ void consist_finalize_kernel(const float* __restrict__ part, int slots, int B, int N, int variant,
                                        float* out, float* cap, float cap_scale) {
  const double nn = (double)N * N;
  double tot = 0.0;
  long long cnt = 0;
  for (int b = 0; b < B; ++b)
    for (int s = 0; s < slots; ++s) {
      tot += part[((long long)s * B + b) * 3];
      cnt += __float_as_int(part[((long long)s * B + b) * 3 + 2]);
    }
  float loss, coef;
  if (variant == SX_CONSIST_BCE) {
    loss = (float)(tot / (B * nn));
    coef = (float)(1.0 / (B * nn));
  } else {
    loss = cnt > 0 ? (float)(tot / (double)cnt) : __int_as_float(0x7fffffff);
    coef = cnt > 0 ? (float)(1.0 / (double)cnt) : 0.f;
    for (int b = 0; b < B; ++b) {
      double sg = 0.0;
      for (int s = 0; s < slots; ++s) sg += part[((long long)s * B + b) * 3 + 1];
      out[2 + b] = cnt > 0 ? (float)(-sg / nn) : 0.f;      // (times out[1] = 1/count in the backward)
    }
  }
  out[0] = loss;
  out[1] = coef;
  if (cap) {
    cap[0] += loss;
    const float t = cap_scale * cap[0];
    cap[1] = t > 1.f ? 1.f / t : 1.f;
  }
}

// dst = s * (G + m_b * v)
__global__ void consist_bwd_kernel(const float* __restrict__ out, const float* __restrict__ gout, int variant, int B,
                                   int rows, int cols, const float* G, long long ldg, long long gbs,
                                   const float* __restrict__ vrow, const float* __restrict__ vcol, float* dst,
                                   long long ldd, long long dbs) {
  const float s = (gout ? *gout : 1.f) * out[1];
  for (long long rr = blockIdx.x; rr < (long long)B * rows; rr += gridDim.x) {
    const int b = (int)(rr / rows), r = (int)(rr % rows);
    const float* g = G + b * gbs + (long long)r * ldg;
    float* d = dst + b * dbs + (long long)r * ldd;
    if (variant == SX_CONSIST_BCE) {
      for (int c = threadIdx.x; c < cols; c += blockDim.x) d[c] = s * g[c];
    } else {
      const float m = out[2 + b];
      const float vr = vrow ? vrow[(long long)b * rows + r] : 1.f;
      for (int c = threadIdx.x; c < cols; c += blockDim.x)
        d[c] = s * fmaf(m, vcol ? vcol[(long long)b * cols + c] : vr, g[c]);
    }
  }
}

// forward (dY == NULL): out = (*amax > clip) ? clamp(S, -clip, clip) : S;
// backward: out = dY where the forward passed S through (clamp gradient, bounds included), 0 where it clamped
__global__ void clamp_if_kernel(const float* __restrict__ S, long long R, int L, long long lds,
                                const float* __restrict__ amax, float clip, const float* __restrict__ dY, long long ldy,
                                float* __restrict__ out, long long ldo) {
  const bool on = *amax > clip;
  for (long long r = blockIdx.x; r < R; r += gridDim.x) {
    const float* s = S + r * lds;
    float* o = out + r * ldo;
    if (dY) {
      const float* g = dY + r * ldy;
      for (int c = threadIdx.x; c < L; c += blockDim.x) o[c] = (on && fabsf(s[c]) > clip) ? 0.f : g[c];
    } else {
      for (int c = threadIdx.x; c < L; c += blockDim.x) o[c] = on ? fminf(fmaxf(s[c], -clip), clip) : s[c];
    }
  }
}

}  // namespace

extern "C" int sx_clamp_if(const float* S, int64_t R, int32_t L, int64_t lds, const float* amax, float clip,
                           const float* dY, int64_t ldy, float* out, int64_t ldo, void* stream) {
  SX_REQUIRE(S && amax && out && R > 0 && L > 0 && lds >= L && ldo >= L && (!dY || ldy >= L),
             "sx_clamp_if: bad arguments");
  const int sms = sm_count_cached();
  SX_REQUIRE(sms > 0, "sx_clamp_if: no CUDA device (this library has no CPU fallback)");
  const int grid = (int)std::min<long long>(R, (long long)sms * 16);
  clamp_if_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(S, R, L, lds, amax, clip, dY, ldy, out, ldo);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_attn_consist_fwd(const sx_consist_args* a, void* stream) {
  SX_REQUIRE(a != nullptr, "sx_attn_consist_fwd: null args");
  SX_REQUIRE(a->B > 0 && a->N > 0, "sx_attn_consist_fwd: bad shape");
  SX_REQUIRE(a->K >= 1 && a->K <= sxcs::MAX_K, "sx_attn_consist_fwd: %d mask channels (1..%d supported)", a->K,
             sxcs::MAX_K);
  SX_REQUIRE(a->variant == SX_CONSIST_BCE || a->variant == SX_CONSIST_MARGIN, "sx_attn_consist_fwd: bad variant");
  SX_REQUIRE(a->F && a->out && a->part, "sx_attn_consist_fwd: null pointer");
  SX_REQUIRE(a->variant == SX_CONSIST_BCE || a->mu, "sx_attn_consist_fwd: the margin variant needs mu");
  SX_REQUIRE(!a->R || (a->ldr >= a->N && a->ldr % 4 == 0 && (reinterpret_cast<uintptr_t>(a->R) & 15) == 0),
             "sx_attn_consist_fwd: R needs a row pitch >= N, multiple of 4, and 16-byte alignment");
  const int sms = sm_count_cached();
  SX_REQUIRE(sms > 0, "sx_attn_consist_fwd: no CUDA device (this library has no CPU fallback)");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);

  CsParams p{};
  p.B = a->B; p.N = a->N; p.K = a->K; p.variant = a->variant; p.round_r = a->round_r;
  p.F = a->F; p.mu = a->mu; p.R = a->R; p.ldr = a->ldr; p.part = a->part;
  const long long max_slots = a->part_floats / (3ll * a->B);
  int grid;
  if (a->Xo) {
    SX_REQUIRE(a->Xt && a->A > 0, "sx_attn_consist_fwd: pair input needs Xo, Xt and A");
    p.tiles = sx_ceil_div(a->N, BM);
    p.num_kb = sx_ceil_div(a->A, 32);
    const long long items = (long long)a->B * p.tiles;
    SX_REQUIRE(items < (1ll << 30), "sx_attn_consist_fwd: too many row blocks");
    p.items = (int)items;
    grid = (int)std::min<long long>({(long long)sms, items, max_slots});
    SX_REQUIRE(grid >= 1, "sx_attn_consist_fwd: needs at least %d floats of scratch", 3 * a->B);
    sx_operand oo{}, ot{};
    oo.ptr = a->Xo; oo.major = SX_MAJOR_K; oo.ld = a->xo_ld; oo.stride_z1 = a->B > 1 ? a->xo_bstride : 0;
    ot.ptr = a->Xt; ot.major = SX_MAJOR_K; ot.ld = a->xt_ld; ot.stride_z1 = a->B > 1 ? a->xt_bstride : 0;
    CUtensorMap to, tt;
    int rc = make_map(&to, oo, 4, a->N, a->A, 1, a->B, BM, "Xo");
    if (rc) return rc;
    rc = make_map(&tt, ot, 4, a->N, a->A, 1, a->B, BN, "Xt");
    if (rc) return rc;
    SX_CHECK_CUDA(set_max_smem_once(consist_pair_kernel, SMEM_BYTES));
    consist_pair_kernel<<<grid, NUM_THREADS, SMEM_BYTES, st>>>(to, tt, p);
  } else {
    SX_REQUIRE(a->X && a->x_ld >= a->N, "sx_attn_consist_fwd: dense input needs X with a row pitch >= N");
    grid = (int)std::min<long long>({(long long)sms * 4, (long long)a->B * a->N, max_slots});
    SX_REQUIRE(grid >= 1, "sx_attn_consist_fwd: needs at least %d floats of scratch", 3 * a->B);
    consist_dense_kernel<<<grid, DENSE_THREADS, 0, st>>>(a->X, a->x_ld, a->x_bstride, p);
  }
  SX_CHECK_CUDA(cudaGetLastError());
  consist_finalize_kernel<<<1, 1, 0, st>>>(a->part, grid, a->B, a->N, a->variant, a->out, a->cap, a->cap_scale);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_attn_consist_bwd(const sx_consist_args* a, const float* gout, const float* G, int32_t rows,
                                   int32_t cols, int64_t ldg, int64_t g_bstride, const float* vrow, const float* vcol,
                                   float* dst, int64_t ldd, int64_t d_bstride, void* stream) {
  SX_REQUIRE(a != nullptr && a->out && G && dst, "sx_attn_consist_bwd: null pointer");
  SX_REQUIRE(a->B > 0 && rows > 0 && cols > 0 && ldg >= cols && ldd >= cols, "sx_attn_consist_bwd: bad shape");
  const int sms = sm_count_cached();
  SX_REQUIRE(sms > 0, "sx_attn_consist_bwd: no CUDA device (this library has no CPU fallback)");
  const long long R = (long long)a->B * rows;
  const int grid = (int)std::min<long long>(R, (long long)sms * 16);
  consist_bwd_kernel<<<grid, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      a->out, gout, a->variant, a->B, rows, cols, G, ldg, g_bstride, vrow, vcol, dst, ldd, d_bstride);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
