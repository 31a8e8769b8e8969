// Batched GEMM on the sm_90a warpgroup tensor cores (wgmma).
//
//   C[z][m][n] = epilogue(alpha * sum_k A[z][m][k] * B[z][n][k])
//
// Persistent, warp-specialised kernel, one CTA per SM, 128 x 128 output tiles:
//   warpgroup 0    : TMA producer (one elected thread: cp.async.bulk.tensor 4-D boxes, 128-byte swizzle, 4-stage
//                    mbarrier ring)
//   warpgroups 1-2 : consumers, 64 tile rows each: wgmma.mma_async with the fp32 accumulators in registers, then the
//                    epilogue (bias / GELU / dropout / TF32 rounding) straight from the accumulator fragments to global
// Operands may be K-major or MN-major, so forward (x W^T), data-gradient (dy W) and weight-gradient (dy^T x) products
// all run without transposes in global memory.  bf16 operands reach wgmma in either majorness (its transpose bits);
// tf32 wgmma reads K-major operands only, so an MN-major tf32 tile is transposed in shared memory by the consumers
// (conflict-free 16-byte stores into the K-major swizzled layout) before its MMAs.
// Operand arithmetic: tf32 on fp32 storage (parity-grade) or bf16 storage (fast).
//
// Replaces in the reference: nn.Linear / torch.matmul / grouped Conv1d call sites on the hot path,
// code/networks/segtran_shared.py:243, :267, :414, :447, :559-560, :566 (and their autograd backward).
#include <algorithm>
#include <string>

#include "sx_common.cuh"
#include "sx_tc.cuh"

namespace {
using namespace sxtc;

constexpr int NUM_THREADS = 384;          // warpgroup 0: TMA producer; warpgroups 1-2: MMA + epilogue
constexpr int STAGES = 4;
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;     // 32 KB

template <int ES, bool A_MN, bool B_MN>
constexpr int smem_bytes() {
  // MN-major tf32 operands: two K-major copies of a stage (double buffered between the consumer warpgroups)
  return STAGES * STAGE_BYTES + ((ES == 4 && (A_MN || B_MN)) ? 2 * STAGE_BYTES : 0) + 1024 /*align*/ + 256 /*barriers*/;
}

struct GemmParams {
  int M, N, K, Z0, Z1;
  int tiles_m, tiles_n, split_k, kb_per_split, num_kb, total_tiles;
  int z1_loop;           // > 1: the z1 slices are reduced into one output inside the k loop of each tile (no atomics)
  float* part;           // split_k > 1: [output tile][ks][BM x BN] partial tiles, summed in ks order by split_reduce_kernel
  int a_uses_z0, a_uses_z1, b_uses_z0, b_uses_z1;
  void* C;
  int c_bf16;
  int round_tf32;
  int c_vec_ok;
  long long ldc, c_sz0, c_sz1;
  float alpha;
  int bias_mode;
  const float* bias;
  long long bias_sz0, bias_sz1;
  int act;
  int accumulate;
  void* preact;
  float* amax;
  float drop_p;
  unsigned long long drop_seed;
  const unsigned long long* drop_seed_dev;
  const float* addend;   // optional fp32 tensor in C's layout added to alpha*acc before bias/activation (tf32x3 passes)
  float* colsum;         // optional [N]: += column sums of the stored values over all rows and batch slices (bias gradients)
  int stream_out;        // output larger than half the L2: store with evict-first (st.global.cs), keep operands (evict-last)
};

// MN-major tf32 rows [r0, r0 + nrows) of a tile as TMA left them (boxes of 32 rows x 32 k, SWIZZLE_128B) -> the K-major
// SWIZZLE_128B layout wgmma reads (row r: 128 bytes of k, 16-byte chunk c at (c ^ (r & 7))).  Consecutive threads take
// consecutive rows: the reads of a warp cover one 128-byte span, the 16-byte stores of each quarter-warp 8 distinct chunks.
__device__ __forceinline__ void xpose_tf32(const uint8_t* src, uint8_t* dst, int r0, int nrows, int tid, int nthr) {
  for (int i = tid; i < nrows * 8; i += nthr) {
    const int r = r0 + i % nrows, kc = i / nrows;
    const uint8_t* s = src + (r >> 5) * 4096 + (r & 3) * 4;
    float v[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = 4 * kc + e;
      v[e] = *reinterpret_cast<const float*>(s + k * 128 + ((((r & 31) >> 2) ^ (k & 7)) << 4));
    }
    *reinterpret_cast<float4*>(dst + r * 128 + ((kc ^ (r & 7)) << 4)) = make_float4(v[0], v[1], v[2], v[3]);
  }
}

template <int ES, bool A_MN, bool B_MN>
__global__ void __launch_bounds__(NUM_THREADS, 1)
sx_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  constexpr bool kTF32 = (ES == 4);
  constexpr bool XA = kTF32 && A_MN, XB = kTF32 && B_MN;   // tiles transposed in shared memory before the MMAs
  constexpr int BK = BKB / ES;                 // elements of K per stage: 64 (bf16) / 32 (tf32)
  constexpr int MN_BOX = BKB / ES;             // contiguous MN elements per MN-major box: 64 / 32
  constexpr int MN_BOX_BYTES = BK * BKB;       // bytes of one MN-major box (BK rows of 128 B)
  constexpr int KSTEPS = 4;                    // wgmma per stage, 32 bytes of K each (k8 tf32 / k16 bf16)

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* xbuf = smem + STAGES * STAGE_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(xbuf + ((XA || XB) ? 2 * STAGE_BYTES : 0));
  uint64_t* full_bar = bars;                   // [STAGES]  TMA -> consumers
  uint64_t* empty_bar = bars + STAGES;         // [STAGES]  consumers -> TMA (one arrival per consumer warpgroup)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    sx::tma_prefetch_desc(&tmA);
    sx::tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      sx::mbar_init(&full_bar[s], 1);
      sx::mbar_init(&empty_bar[s], 2);
    }
    sx::fence_barrier_init();
  }
  __syncthreads();

  auto decode = [&](int t, int& z0, int& z1, int& mb, int& nb, int& ks) {
    nb = t % p.tiles_n; t /= p.tiles_n;
    mb = t % p.tiles_m; t /= p.tiles_m;
    ks = t % p.split_k; t /= p.split_k;
    z0 = t % p.Z0;
    z1 = t / p.Z0;
  };

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");   // the producer hands its registers over
    // ===================== TMA producer =====================
    if (warp == 0 && sx::elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      // operand tiles are re-read by every CTA of the same tile row / column: keep them in L2 while a large
      // output streams through
      const uint64_t pol = p.stream_out ? sx::kEvictLast : sx::kEvictNormal;
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
        int z0, z1, mb, nb, ks;
        decode(t, z0, z1, mb, nb, ks);
        const int kb0 = ks * p.kb_per_split;
        const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);
        const int az0 = p.a_uses_z0 ? z0 : 0, bz0 = p.b_uses_z0 ? z0 : 0;
        const int m0 = mb * BM, n0 = nb * BN;
        const int nkb = kb1 - kb0;
        for (int q = 0; q < p.z1_loop * nkb; ++q) {
          const int kb = kb0 + q % nkb, zc = p.z1_loop > 1 ? q / nkb : z1;
          const int az1 = p.a_uses_z1 ? zc : 0, bz1 = p.b_uses_z1 ? zc : 0;
          sx::mbar_wait(&empty_bar[stage], phase ^ 1);
          sx::mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
          uint8_t* sa = smem + stage * STAGE_BYTES;
          uint8_t* sb = sa + A_STAGE_BYTES;
          const int k0 = kb * BK;
          if constexpr (!A_MN) {
            sx::tma_load_4d(sa, &tmA, &full_bar[stage], k0, m0, az0, az1, pol);
          } else {
#pragma unroll
            for (int j = 0; j < BM / MN_BOX; ++j)
              sx::tma_load_4d(sa + j * MN_BOX_BYTES, &tmA, &full_bar[stage], m0 + j * MN_BOX, k0, az0, az1, pol);
          }
          if constexpr (!B_MN) {
            sx::tma_load_4d(sb, &tmB, &full_bar[stage], k0, n0, bz0, bz1, pol);
          } else {
#pragma unroll
            for (int j = 0; j < BN / MN_BOX; ++j)
              sx::tma_load_4d(sb + j * MN_BOX_BYTES, &tmB, &full_bar[stage], n0 + j * MN_BOX, k0, bz0, bz1, pol);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  // ===================== consumers: MMA + epilogue =====================
  const int cw = wg - 1;                        // tile rows 64 cw .. 64 cw + 63
  const int wtid = threadIdx.x & 127;           // thread within the warpgroup
  const int wq = warp & 3;                      // warp within the warpgroup: rows 16 wq .. 16 wq + 15 of those
  const int tr = lane >> 2;                     // row within an 8-row group
  const int tc = (lane & 3) * 2;                // first column of this thread's pair within an 8-column group
  float tmax = -3.0e38f;
  int stage = 0;
  uint32_t phase = 0;
  int xi = 0;

  // descriptors of this warpgroup's A rows and of the B tile for k-step kk (operand bases are 1 KB aligned)
  auto desc_a = [&](const uint8_t* base, int kk, bool mn) -> uint64_t {
    const uint32_t a = sx::smem_u32(base) + (uint32_t)(cw * 64 * BKB);        // 64 rows (K-major) = one MN box (bf16)
    return mn ? sx::gmma_desc(a + kk * 16 * BKB, MN_BOX_BYTES, 1024) : sx::gmma_desc(a + kk * 32, 16, 1024);
  };
  auto desc_b = [&](const uint8_t* base, int kk, bool mn) -> uint64_t {
    const uint32_t b = sx::smem_u32(base);
    return mn ? sx::gmma_desc(b + kk * 16 * BKB, MN_BOX_BYTES, 1024) : sx::gmma_desc(b + kk * 32, 16, 1024);
  };

  // f index: [j][h][e] -> 4*j + 2*h + e ; row = row0 + 8h + tr ; col = col0 + 8j + tc + e
  auto store_frag = [&](void* base, const float (&f)[16], long long zoff, int row0, int col0, bool atomic_add) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int grow = row0 + 8 * h + tr;
      if (grow < p.M) {
        const long long roff_ = zoff + (long long)grow * p.ldc;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = col0 + 8 * j + tc;
          const float a = f[4 * j + 2 * h], b = f[4 * j + 2 * h + 1];
          if (col + 1 < p.N) {
            if (p.c_bf16) {
              __nv_bfloat162 hb = __floats2bfloat162_rn(a, b);
              __nv_bfloat16* o = reinterpret_cast<__nv_bfloat16*>(base) + roff_ + col;
              if (p.c_vec_ok) *reinterpret_cast<__nv_bfloat162*>(o) = hb;
              else { o[0] = hb.x; o[1] = hb.y; }
            } else {
              float* o = reinterpret_cast<float*>(base) + roff_ + col;
              if (atomic_add) { atomicAdd(o, a); atomicAdd(o + 1, b); }
              else if (p.c_vec_ok) {
                if (p.stream_out) __stcs(reinterpret_cast<float2*>(o), make_float2(a, b));
                else *reinterpret_cast<float2*>(o) = make_float2(a, b);
              }
              else { o[0] = a; o[1] = b; }
            }
          } else if (col < p.N) {
            if (p.c_bf16) reinterpret_cast<__nv_bfloat16*>(base)[roff_ + col] = __float2bfloat16_rn(a);
            else if (atomic_add) atomicAdd(reinterpret_cast<float*>(base) + roff_ + col, a);
            else reinterpret_cast<float*>(base)[roff_ + col] = a;
          }
        }
      }
    }
  };

  // fp32 tensor in C's layout -> the same fragment distribution (out-of-range elements read as 0)
  auto load_frag = [&](const float* base, float (&g)[16], long long zoff, int row0, int col0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int grow = row0 + 8 * h + tr;
      const float* ar = base + zoff + (long long)(grow < p.M ? grow : 0) * p.ldc;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int col = col0 + 8 * j + tc;
        const int i0 = 4 * j + 2 * h;
        if (grow < p.M && col + 1 < p.N && p.c_vec_ok) {
          const float2 v = *reinterpret_cast<const float2*>(ar + col);
          g[i0] = v.x; g[i0 + 1] = v.y;
        } else {
          g[i0] = (grow < p.M && col < p.N) ? ar[col] : 0.f;
          g[i0 + 1] = (grow < p.M && col + 1 < p.N) ? ar[col + 1] : 0.f;
        }
      }
    }
  };

  // dropout constants of this thread (the word key is a 64-bit mix of the seed: computed once, not per chunk)
  const float drop_scale = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
  const uint32_t drop_p16v = sx::drop_p16(p.drop_p);
  const unsigned long long drop_seed = p.drop_p > 0.f ? p.drop_seed + (p.drop_seed_dev ? *p.drop_seed_dev : 0ull) : 0ull;
  const uint32_t drop_mul_t = sx::drop_mul((tc >> 1) & 1), drop_key_t = sx::drop_key(drop_seed, (tc >> 1) & 1);

  float acc[64];
  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
    int z0, z1, mb, nb, ks;
    decode(t, z0, z1, mb, nb, ks);
    const int kb0 = ks * p.kb_per_split;
    const int kb1 = min(p.num_kb, kb0 + p.kb_per_split);

    // ---------------- main loop ----------------
    int prev = -1;                              // stage whose MMAs may still be in flight (no-transpose path)
    for (int q = 0; q < p.z1_loop * (kb1 - kb0); ++q) {
      sx::mbar_wait(&full_bar[stage], phase);
      const uint8_t* sa = smem + stage * STAGE_BYTES;
      const uint8_t* sb = sa + A_STAGE_BYTES;
      if constexpr (XA || XB) {
        uint8_t* xa = xbuf + xi * STAGE_BYTES;
        uint8_t* xb = xa + A_STAGE_BYTES;
        // a K-major copy of the MN-major tile(s); the buffer xi was last read by MMAs that both warpgroups completed
        // before the previous named barrier
        if constexpr (XA) xpose_tf32(sa, xa, cw * 64, 64, wtid, 128);
        if constexpr (XB) xpose_tf32(sb, xb, cw * 64, 64, wtid, 128);
        sx::fence_proxy_async_smem();
        if constexpr (XB) asm volatile("bar.sync 1, 256;" ::: "memory");
        else asm volatile("bar.sync %0, 128;" ::"r"(2 + cw) : "memory");
        if constexpr (XA) sa = xa;
        if constexpr (XB) sb = xb;
      }
      sx::acc_fence(acc);
      sx::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
        const uint64_t da = desc_a(sa, kk, A_MN && !kTF32), db = desc_b(sb, kk, B_MN && !kTF32);
        const uint32_t accum = (q > 0 || kk > 0) ? 1u : 0u;
        if constexpr (kTF32) sx::wgmma_tf32(acc, da, db, accum);
        else sx::wgmma_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, accum);
      }
      sx::wgmma_commit();
      sx::acc_fence(acc);
      if constexpr (XA || XB) {
        sx::wgmma_wait<0>();
        if (wtid == 0) sx::mbar_arrive(&empty_bar[stage]);
        xi ^= 1;
      } else {
        sx::wgmma_wait<1>();                    // the previous stage's MMAs are done: release it
        if (prev >= 0 && wtid == 0) sx::mbar_arrive(&empty_bar[prev]);
        prev = stage;
      }
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    if constexpr (!(XA || XB)) {
      sx::wgmma_wait<0>();
      sx::acc_fence(acc);
      if (prev >= 0 && wtid == 0) sx::mbar_arrive(&empty_bar[prev]);
    }

    // ---------------- epilogue: accumulator fragments -> bias / GELU / dropout / rounding -> global ----------------
    const int row0 = mb * BM + cw * 64 + wq * 16;
    const long long zoff = (long long)z1 * p.c_sz1 + (long long)z0 * p.c_sz0;
    const float* bias = p.bias ? p.bias + (long long)z1 * p.bias_sz1 + (long long)z0 * p.bias_sz0 : nullptr;
    const bool add_bias = (bias != nullptr) && (ks == 0);
    float bias_m[2] = {0.f, 0.f};                         // [h]
    if (add_bias && p.bias_mode == SX_BIAS_M) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = row0 + 8 * h + tr;
        bias_m[h] = r < p.M ? bias[r] : 0.f;
      }
    }
#pragma unroll
    for (int c = 0; c < BN / 32; ++c) {
      const int col0 = nb * BN + c * 32;
      if (col0 >= p.N) break;                   // warp-uniform
      float f[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) f[i] = acc[16 * c + i] * p.alpha + bias_m[(i >> 1) & 1];
      if (p.addend) {
        float g[16];
        load_frag(p.addend, g, zoff, row0, col0);
#pragma unroll
        for (int i = 0; i < 16; ++i) f[i] += g[i];
      }
      if (add_bias && p.bias_mode == SX_BIAS_N) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int col = col0 + 8 * j + tc;
          const float b0 = col < p.N ? bias[col] : 0.f, b1 = col + 1 < p.N ? bias[col + 1] : 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            f[4 * j + 2 * h] += b0;
            f[4 * j + 2 * h + 1] += b1;
          }
        }
      }
      auto apply_dropout = [&]() {
        if (p.drop_p > 0.f) {
          if (((p.ldc | zoff) & 3) == 0) {
            // rows start on a 4-element hash group: this thread's pair is always elements (tc&2, tc&2 + 1) of its
            // group, i.e. one 32-bit word per pair with a per-thread constant multiplier / key
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const unsigned long long g0 =
                  (unsigned long long)((zoff + (long long)(row0 + 8 * h + tr) * p.ldc + col0 + tc) >> 2);
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const uint32_t bits = sx::drop_word_k(drop_mul_t, drop_key_t, g0 + 2 * j);
                const int i0 = 4 * j + 2 * h;
                f[i0] = (bits & 0xFFFFu) >= drop_p16v ? f[i0] * drop_scale : 0.f;
                f[i0 + 1] = (bits >> 16) >= drop_p16v ? f[i0 + 1] * drop_scale : 0.f;
              }
            }
          } else {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const long long rbase = zoff + (long long)(row0 + 8 * h + tr) * p.ldc;
#pragma unroll
              for (int j = 0; j < 4; ++j) {
                const unsigned long long e0 = (unsigned long long)(rbase + col0 + 8 * j + tc);
                const int i0 = 4 * j + 2 * h;
                f[i0] = sx::drop_keep1(drop_seed, e0, drop_p16v) ? f[i0] * drop_scale : 0.f;
                f[i0 + 1] = sx::drop_keep1(drop_seed, e0 + 1, drop_p16v) ? f[i0 + 1] * drop_scale : 0.f;
              }
            }
          }
        }
      };
      if (p.act == SX_ACT_GELU_BWD) {           // C = mask * acc * gelu'(h), h = the forward pre-activation (read-only)
        apply_dropout();                        // (commutes with the gelu' factor)
        float g[16];
        load_frag(reinterpret_cast<const float*>(p.preact), g, zoff, row0, col0);
#pragma unroll
        for (int i = 0; i < 16; ++i) f[i] *= sx::gelu_erf_grad(g[i]);
      } else {
        if (p.preact) store_frag(p.preact, f, zoff, row0, col0, false);
        if (p.act == SX_ACT_GELU) {
#pragma unroll
          for (int i = 0; i < 16; ++i) f[i] = sx::gelu_erf(f[i]);
        }
        apply_dropout();
      }
      if (p.round_tf32 && !p.c_bf16) {
#pragma unroll
        for (int i = 0; i < 16; ++i) f[i] = sx::round_tf32(f[i]);
      }
      if (p.colsum) {
        // this thread's 8 columns (j, e), summed over its 2 rows, then over the 8 lanes that share the columns
        float cs[8];
#pragma unroll
        for (int j = 0; j < 4; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            float a = 0.f;
#pragma unroll
            for (int h = 0; h < 2; ++h)
              if (row0 + 8 * h + tr < p.M) a += f[4 * j + 2 * h + e];
            a += __shfl_xor_sync(0xffffffffu, a, 4);
            a += __shfl_xor_sync(0xffffffffu, a, 8);
            a += __shfl_xor_sync(0xffffffffu, a, 16);
            cs[2 * j + e] = a;
          }
        if (tr == 0) {
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int col = col0 + 8 * j + tc + e;
              if (col < p.N) atomicAdd(p.colsum + col, cs[2 * j + e]);
            }
        }
      }
      if (p.amax) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (row0 + 8 * h + tr < p.M) {
#pragma unroll
            for (int j = 0; j < 4; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (col0 + 8 * j + tc + e < p.N) tmax = fmaxf(tmax, f[4 * j + 2 * h + e]);
          }
      }
      if (p.split_k > 1) {
        // this split's partial tile (local row-major 128 x 128), summed over the splits in order by split_reduce_kernel
        float* pt = p.part + ((((long long)z1 * p.Z0 + z0) * p.tiles_m + mb) * p.tiles_n + nb) * p.split_k * (BM * BN) +
                    (long long)ks * (BM * BN);
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
          for (int j = 0; j < 4; ++j)
            *reinterpret_cast<float2*>(pt + (row0 - mb * BM + 8 * h + tr) * BN + (col0 - nb * BN) + 8 * j + tc) =
                make_float2(f[4 * j + 2 * h], f[4 * j + 2 * h + 1]);
      } else {
        store_frag(p.C, f, zoff, row0, col0, p.accumulate != 0);
      }
    }
  }
  if (p.amax) {
    tmax = sx::warp_max(tmax);
    if (lane == 0 && tmax > -3.0e38f) sx::atomic_max_float(p.amax, tmax);
  }
}

// C[tile] += sum over ks (in order) of the split partials of the tile: one thread per output element
__global__ void split_reduce_kernel(const GemmParams p) {
  const long long total = (long long)p.total_tiles / p.split_k * (BM * BN);
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int e = (int)(i % (BM * BN));
    long long t = i / (BM * BN);
    const int nb = (int)(t % p.tiles_n); t /= p.tiles_n;
    const int mb = (int)(t % p.tiles_m); t /= p.tiles_m;
    const int z0 = (int)(t % p.Z0), z1 = (int)(t / p.Z0);
    const int row = mb * BM + e / BN, col = nb * BN + e % BN;
    if (row >= p.M || col >= p.N) continue;
    const float* pt = p.part + (i / (BM * BN)) * p.split_k * (BM * BN) + e;
    float s = 0.f;
    for (int ks = 0; ks < p.split_k; ++ks) s += pt[(long long)ks * (BM * BN)];
    reinterpret_cast<float*>(p.C)[(long long)z1 * p.c_sz1 + (long long)z0 * p.c_sz0 + (long long)row * p.ldc + col] += s;
  }
}

// ------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------
long long g_max_ctas = -1;         // cap on the persistent grid (tests drive the multi-tile-per-CTA schedule with it)

template <int ES, bool A_MN, bool B_MN>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int grid, cudaStream_t st) {
  auto kern = sx_gemm_kernel<ES, A_MN, B_MN>;
  constexpr int bytes = smem_bytes<ES, A_MN, B_MN>();
  SX_CHECK_CUDA(set_max_smem_once(kern, bytes));         // per device (a process may drive several GPUs)
  kern<<<grid, NUM_THREADS, bytes, st>>>(ta, tb, p);
  SX_CHECK_CUDA(cudaGetLastError());
  if (p.split_k > 1) {
    const long long n = (long long)p.total_tiles / p.split_k * (BM * BN);
    split_reduce_kernel<<<(int)std::min<long long>(sx_ceil_div(n, 256), 65535), 256, 0, st>>>(p);
    SX_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}

}  // namespace

extern "C" int sx_gemm_debug_set(const char* key, int64_t value) {
  std::string k(key);
  if (k == "max_ctas") g_max_ctas = value;
  else {
    sx_set_error("sx_gemm_debug_set: unknown key %s", key);
    return -1;
  }
  return 0;
}

extern "C" int sx_gemm(const sx_gemm_args* a, void* stream) {
  SX_REQUIRE(a != nullptr, "sx_gemm: null args");
  SX_REQUIRE(a->M > 0 && a->N > 0 && a->K > 0 && a->Z0 > 0 && a->Z1 > 0, "sx_gemm: bad shape M=%d N=%d K=%d Z=%dx%d",
             a->M, a->N, a->K, a->Z0, a->Z1);
  SX_REQUIRE(a->op_dtype == SX_OP_TF32 || a->op_dtype == SX_OP_BF16, "sx_gemm: bad op_dtype %d", a->op_dtype);
  SX_REQUIRE(a->C != nullptr && a->A.ptr != nullptr && a->B.ptr != nullptr, "sx_gemm: null pointer");
  const int es = a->op_dtype == SX_OP_TF32 ? 4 : 2;
  const int bk = BKB / es;
  const int sms = sm_count_cached();
  SX_REQUIRE(sms > 0, "sx_gemm: no CUDA device (this library has no CPU fallback)");

  GemmParams p{};
  p.M = a->M; p.N = a->N; p.K = a->K; p.Z0 = a->Z0; p.Z1 = a->Z1;
  p.tiles_m = sx_ceil_div(a->M, BM);
  p.tiles_n = sx_ceil_div(a->N, BN);
  p.num_kb = sx_ceil_div(a->K, bk);
  // all z1 slices add into one output (c_stride_z1 == 0): each output tile runs the z1 slices as extra k-blocks, so
  // every output element has one writer and the sum has a fixed order
  const bool fold_z1 = a->Z1 > 1 && a->c_stride_z1 == 0;
  SX_REQUIRE(!fold_z1 || (a->accumulate && !a->bias && !a->addend && a->act == SX_ACT_NONE && !a->preact && a->drop_p == 0.f),
             "sx_gemm: a z1-reduced output needs accumulate=1 and a linear epilogue without bias");
  p.z1_loop = fold_z1 ? a->Z1 : 1;
  p.Z1 = fold_z1 ? 1 : a->Z1;
  int split = a->split_k < 1 ? 1 : a->split_k;
  if (split > p.num_kb) split = p.num_kb;
  {
    // split partial tiles must fit the caller's scratch (fewer splits otherwise; 1 needs none)
    const long long out_tiles = (long long)p.tiles_m * p.tiles_n * a->Z0 * p.Z1;
    const long long fit = a->part ? a->part_floats / ((long long)BM * BN * out_tiles) : 0;
    if (split > fit) split = fit < 2 ? 1 : (int)fit;
  }
  p.kb_per_split = sx_ceil_div(p.num_kb, split);
  p.split_k = sx_ceil_div(p.num_kb, p.kb_per_split);      // no empty splits
  SX_REQUIRE(p.split_k == 1 || (a->accumulate && a->c_dtype == SX_F32 && a->act == SX_ACT_NONE && !a->preact &&
                                a->drop_p == 0.f && !a->amax),
             "sx_gemm: split_k > 1 needs accumulate=1 into fp32 C and a linear epilogue");
  SX_REQUIRE(!a->accumulate || a->c_dtype == SX_F32, "sx_gemm: accumulate needs fp32 C");
  SX_REQUIRE(!a->round_tf32 || (!a->accumulate && p.split_k == 1),
             "sx_gemm: round_tf32 cannot be combined with accumulate / split_k > 1 (a sum of rounded partials is not a TF32 "
             "value): round the finished output instead");
  SX_REQUIRE(p.split_k == 1 || !a->colsum, "sx_gemm: colsum needs split_k=1");
  const long long tt = (long long)p.tiles_m * p.tiles_n * p.split_k * a->Z0 * p.Z1;
  SX_REQUIRE(tt < (1ll << 30), "sx_gemm: too many tiles");
  p.total_tiles = (int)tt;
  p.a_uses_z0 = a->A.stride_z0 != 0; p.a_uses_z1 = a->A.stride_z1 != 0;
  p.b_uses_z0 = a->B.stride_z0 != 0; p.b_uses_z1 = a->B.stride_z1 != 0;
  p.C = a->C; p.c_bf16 = a->c_dtype == SX_BF16; p.round_tf32 = a->round_tf32;
  p.ldc = a->ldc; p.c_sz0 = a->c_stride_z0; p.c_sz1 = a->c_stride_z1;
  // the epilogue stores column pairs (8 bytes fp32 / 4 bytes bf16): pairs must stay naturally aligned
  p.c_vec_ok = ((reinterpret_cast<uintptr_t>(a->C) & 7) == 0) && (a->ldc % 2 == 0) && (a->c_stride_z0 % 2 == 0) &&
               (a->c_stride_z1 % 2 == 0) && (!a->preact || (reinterpret_cast<uintptr_t>(a->preact) & 7) == 0) &&
               (!a->addend || (reinterpret_cast<uintptr_t>(a->addend) & 7) == 0);
  p.alpha = a->alpha; p.bias_mode = a->bias ? a->bias_mode : SX_BIAS_NONE; p.bias = a->bias;
  p.bias_sz0 = a->bias_stride_z0; p.bias_sz1 = a->bias_stride_z1;
  p.act = a->act; p.accumulate = a->accumulate; p.preact = a->preact; p.amax = a->amax;
  p.addend = a->addend;
  p.colsum = a->colsum;
  SX_REQUIRE(a->act != SX_ACT_GELU_BWD || (a->preact && a->c_dtype == SX_F32 && p.split_k == 1 && !a->accumulate),
             "sx_gemm: SX_ACT_GELU_BWD needs the fp32 pre-activation in `preact`, fp32 C, split_k=1, accumulate=0");
  SX_REQUIRE(!a->addend || (p.split_k == 1 && !a->accumulate && a->c_dtype == SX_F32), "sx_gemm: addend needs split_k=1, accumulate=0, fp32 C");
  p.drop_p = a->drop_p; p.drop_seed = a->drop_seed;
  p.drop_seed_dev = reinterpret_cast<const unsigned long long*>(a->drop_seed_dev);
  {
    // H100: 50 MB of L2
    const double out_bytes = (double)a->M * a->N * a->Z0 * a->Z1 * (p.c_bf16 ? 2 : 4) * (a->preact ? 2 : 1);
    p.stream_out = out_bytes > 25.0 * 1024 * 1024;
  }

  CUtensorMap ta, tb;
  int rc = make_map(&ta, a->A, es, a->M, a->K, a->Z0, a->Z1, BM, "A");
  if (rc) return rc;
  rc = make_map(&tb, a->B, es, a->N, a->K, a->Z0, a->Z1, BN, "B");
  if (rc) return rc;

  int grid = p.total_tiles < sms ? p.total_tiles : sms;
  if (g_max_ctas > 0 && grid > g_max_ctas) grid = (int)g_max_ctas;
  p.part = a->part;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const bool amn = a->A.major == SX_MAJOR_MN, bmn = a->B.major == SX_MAJOR_MN;
  if (es == 4) {
    if (!amn && !bmn) return launch<4, false, false>(ta, tb, p, grid, st);
    if (!amn && bmn) return launch<4, false, true>(ta, tb, p, grid, st);
    if (amn && !bmn) return launch<4, true, false>(ta, tb, p, grid, st);
    return launch<4, true, true>(ta, tb, p, grid, st);
  }
  if (!amn && !bmn) return launch<2, false, false>(ta, tb, p, grid, st);
  if (!amn && bmn) return launch<2, false, true>(ta, tb, p, grid, st);
  if (amn && !bmn) return launch<2, true, false>(ta, tb, p, grid, st);
  return launch<2, true, true>(ta, tb, p, grid, st);
}
