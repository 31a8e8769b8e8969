// Batched GEMM on the sm_90a warpgroup tensor cores (wgmma).
//
//   C[z][m][n] = epilogue(alpha * sum_k A[z][m][k] * B[z][n][k])
//
// Persistent, warp-specialised kernel, one CTA per SM, 128 x 128 output tiles, or 128 x 256 for large TF32 products with
// both operands K-major (see sx_gemm() for the rule):
//   warpgroup 0    : warp 0: TMA producer (one elected thread: cp.async.bulk.tensor 4-D boxes, 128-byte swizzle);
//                    warps 1-3: transposers (tf32 MN-major operands only, see below)
//   warpgroups 1-2 : consumers, 64 tile rows each: wgmma.mma_async with the fp32 accumulators in registers, then the
//                    epilogue (bias / GELU / dropout / TF32 rounding) straight from the accumulator fragments to global
// Operands may be K-major or MN-major, so forward (x W^T), data-gradient (dy W) and weight-gradient (dy^T x) products
// all run without transposes in global memory.  bf16 operands reach wgmma in either majorness (its transpose bits);
// tf32 wgmma reads K-major operands only, so TMA lands an MN-major tf32 tile in a raw ring and the transposer warps
// rewrite it into the K-major stage the consumers read.  The consumers run the same loop for every majorness.
// Operand arithmetic: tf32 on fp32 storage (parity-grade) or bf16 storage (fast).
// A 128 x 256 tile (each consumer issues m64n256k8 into 128 accumulators) moves 25 % fewer operand bytes from L2 into
// shared memory per FLOP than a 128 x 128 tile.  Every output element still sees the same k-blocks in the same order and
// the same k8 steps, so both tile widths give bit-identical results.
// K-major tf32 launches may also write the final values transposed (`ct`), staged through shared memory so the stores
// stay coalesced: a product that later contracts over C's rows then reads that copy K-major.
//
// Replaces in the reference: nn.Linear / torch.matmul / grouped Conv1d call sites on the hot path,
// code/networks/segtran_shared.py:243, :267, :414, :447, :559-560, :566 (and their autograd backward).
#include <algorithm>
#include <string>

#include "sx_common.cuh"
#include "sx_tc.cuh"

namespace {
using namespace sxtc;

constexpr int NUM_THREADS = 384;          // warpgroup 0: TMA + transposers; warpgroups 1-2: MMA + epilogue
constexpr int STAGES = 4;                 // K-major operand ring (what wgmma reads)
constexpr int XPOSE_WARPS = 3;            // warps 1-3 of warpgroup 0
constexpr int BN_WIDE = 256;              // tile cols of the wide instantiation (tf32, both operands K-major)
// transposed second output (ct): each consumer warpgroup stages one 64-row x 32-column chunk column-major, 68 floats per
// column: a warp's fragment stores (8 rows x 4 column pairs) then hit 32 distinct banks, and a column is 16-byte aligned
constexpr int CT_LD = 68;
constexpr int CT_WG_FLOATS = 32 * CT_LD;  // 8.5 KB per warpgroup

// Shared-memory plan of one instantiation.  A tf32 MN-major operand goes through a raw ring (as TMA lands it) before
// the transposers write its K-major copy into the stage; everything else lands in the stage directly.  BN_T = 256 (the
// wide tile) has K-major tf32 operands only: 16 KB of A + 32 KB of B per stage, no raw ring.  The K-major tf32
// instantiations also hold the two warpgroups' ct staging chunks.
template <int ES, bool A_MN, bool B_MN, int BN_T>
struct Plan {
  static_assert(BN_T == BN || (BN_T == BN_WIDE && ES == 4 && !A_MN && !B_MN),
                "sx_gemm: the 256-column tile is instantiated for K-major tf32 operands only");
  static constexpr int B_BYTES = BN_T * BKB;                          // B operand tile per stage: 16 / 32 KB
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_BYTES;         // 32 / 48 KB
  static constexpr bool XA = ES == 4 && A_MN, XB = ES == 4 && B_MN;
  static constexpr bool XPOSE = XA || XB;
  static constexpr int RAW_BYTES = (XA ? A_STAGE_BYTES : 0) + (XB ? B_STAGE_BYTES : 0);      // per raw slot
  static constexpr int RAW_SLOTS = !XPOSE ? 0 : (XA && XB ? 3 : 4);
  static constexpr int DIRECT_BYTES = STAGE_BYTES - RAW_BYTES;   // per stage, loaded by TMA straight into the stage
  static constexpr bool CT = ES == 4 && !A_MN && !B_MN;
  static constexpr int CT_BYTES = CT ? 2 * CT_WG_FLOATS * 4 : 0;
  static constexpr int SMEM = STAGES * STAGE_BYTES + RAW_SLOTS * RAW_BYTES + 1024 /*align*/ + 256 /*barriers*/ + CT_BYTES;
  static_assert(SMEM <= 227 * 1024, "sx_gemm: shared memory plan exceeds 227 KB");   // wide: 4 x 48 KB + 18.25 KB
  // the transposers address B at A's offset + A_STAGE_BYTES in both the raw slot and the stage, and move 256 4 x 4
  // blocks (4 boxes of 32 x 32) per operand: both hold only for 128 x 128 tf32 operand tiles
  static_assert(!XPOSE || (A_STAGE_BYTES == 16384 && B_STAGE_BYTES == 16384 && BM == 128 && BN == 128),
                "sx_gemm: the transposer assumes 128-row, 16 KB tf32 operand tiles");
};

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
  int stream_out;        // output larger than half the L2: store with evict-first (st.global.cs), keep operands (evict-last)
  float* ct;             // optional transposed copy of the final C values: ct[z][n][m] (K-major tf32 instantiations)
  long long ldct, ct_sz0, ct_sz1;
};

// MN-major tf32 operand tile as TMA left it (4 boxes of 32 k rows x 128 B of MN, SWIZZLE_128B: 16-byte chunk c of k row
// k at (c ^ (k & 7))) -> the K-major SWIZZLE_128B tile wgmma reads (MN row r: 128 B of k, chunk kc at (kc ^ (r & 7))).
// Block b moves MN 4c..4c+3 x k 4kc..4kc+3 of box b >> 6 with four 16-byte loads (one per k row) and four 16-byte
// stores (one per MN row).  c = b & 7 and kc = c ^ ((b >> 3) & 7): within each quarter-warp (fixed b >> 3) both the
// loaded chunks c ^ (k & 7) and the stored chunks kc ^ (r & 7) are 8 distinct 16-byte bank groups.
__device__ __forceinline__ void xpose_load(uint32_t src, int b, float4 (&v)[4]) {
  const int c = b & 7, kc = c ^ ((b >> 3) & 7);
  const uint32_t s = src + (b >> 6) * 4096;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int k = 4 * kc + e;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v[e].x), "=f"(v[e].y), "=f"(v[e].z), "=f"(v[e].w)
                 : "r"(s + k * 128 + ((c ^ (k & 7)) << 4)) : "memory");
  }
}
__device__ __forceinline__ void xpose_store(uint32_t dst, int b, const float4 (&v)[4]) {
  const int c = b & 7, kc = c ^ ((b >> 3) & 7);
  const int r0 = (b >> 6) * 32 + 4 * c;
  auto st = [&](int i, float x, float y, float z, float w) {
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};"
                 ::"r"(dst + (r0 + i) * 128 + ((kc ^ ((r0 + i) & 7)) << 4)), "f"(x), "f"(y), "f"(z), "f"(w) : "memory");
  };
  st(0, v[0].x, v[1].x, v[2].x, v[3].x);
  st(1, v[0].y, v[1].y, v[2].y, v[3].y);
  st(2, v[0].z, v[1].z, v[2].z, v[3].z);
  st(3, v[0].w, v[1].w, v[2].w, v[3].w);
}

// barrier of one consumer warpgroup (ids 1, 2; id 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id) { asm volatile("bar.sync %0, 128;" ::"r"(id) : "memory"); }

template <int ES, bool A_MN, bool B_MN, int BN_T>
__global__ void __launch_bounds__(NUM_THREADS, 1)
sx_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GemmParams p) {
  using PL = Plan<ES, A_MN, B_MN, BN_T>;
  constexpr bool kTF32 = (ES == 4);
  constexpr bool WIDE = BN_T == BN_WIDE;
  constexpr int STAGE_BYTES = PL::STAGE_BYTES;
  constexpr bool XA = PL::XA, XB = PL::XB;
  constexpr int BK = BKB / ES;                 // elements of K per stage: 64 (bf16) / 32 (tf32)
  constexpr int MN_BOX = BKB / ES;             // contiguous MN elements per MN-major box: 64 / 32
  constexpr int MN_BOX_BYTES = BK * BKB;       // bytes of one MN-major box (BK rows of 128 B)
  constexpr int KSTEPS = 4;                    // wgmma per stage, 32 bytes of K each (k8 tf32 / k16 bf16)

  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* raw = smem + STAGES * STAGE_BYTES;  // [RAW_SLOTS][A (XA) | B (XB)] MN-major tf32 tiles as TMA lands them
  uint64_t* bars = reinterpret_cast<uint64_t*>(raw + PL::RAW_SLOTS * PL::RAW_BYTES);
  uint64_t* full_bar = bars;                   // [STAGES]  TMA bytes + transposer arrivals -> consumers
  uint64_t* empty_bar = bars + STAGES;         // [STAGES]  consumers -> TMA / transposers (one arrival per warpgroup)
  uint64_t* raw_full = bars + 2 * STAGES;      // [RAW_SLOTS]  TMA -> transposers
  uint64_t* raw_empty = raw_full + PL::RAW_SLOTS;   // [RAW_SLOTS]  transposers -> TMA
  float* ct_stage = reinterpret_cast<float*>(reinterpret_cast<uint8_t*>(bars) + 256);   // [2][32][CT_LD] (PL::CT)

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    sx::tma_prefetch_desc(&tmA);
    sx::tma_prefetch_desc(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      sx::mbar_init(&full_bar[s], (PL::DIRECT_BYTES ? 1 : 0) + (PL::XPOSE ? XPOSE_WARPS : 0));
      sx::mbar_init(&empty_bar[s], 2);
    }
    for (int s = 0; s < PL::RAW_SLOTS; ++s) {
      sx::mbar_init(&raw_full[s], 1);
      sx::mbar_init(&raw_empty[s], XPOSE_WARPS);
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
  // k-blocks of split ks (the last split may be shorter)
  auto split_kbs = [&](int ks) { return min(p.num_kb, (ks + 1) * p.kb_per_split) - ks * p.kb_per_split; };

  if (wg == 0) {
    // the producers hand their registers over (the wide tile has no transposers: its producer keeps only 40)
    if constexpr (WIDE) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    else asm volatile("setmaxnreg.dec.sync.aligned.u32 56;" ::: "memory");
    if (warp == 0) {
      // ===================== TMA producer =====================
      if (sx::elect_one()) {
        int stage = 0, rs = 0;
        uint32_t phase = 0, rphase = 0;
        // operand tiles are re-read by every CTA of the same tile row / column: keep them in L2 while a large
        // output streams through
        const uint64_t pol = p.stream_out ? sx::kEvictLast : sx::kEvictNormal;
        for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
          int z0, z1, mb, nb, ks;
          decode(t, z0, z1, mb, nb, ks);
          const int kb0 = ks * p.kb_per_split;
          const int az0 = p.a_uses_z0 ? z0 : 0, bz0 = p.b_uses_z0 ? z0 : 0;
          const int m0 = mb * BM, n0 = nb * BN_T;
          const int nkb = split_kbs(ks);
          for (int q = 0; q < p.z1_loop * nkb; ++q) {
            const int kb = kb0 + q % nkb, zc = p.z1_loop > 1 ? q / nkb : z1;
            const int az1 = p.a_uses_z1 ? zc : 0, bz1 = p.b_uses_z1 ? zc : 0;
            const int k0 = kb * BK;
            if constexpr (PL::XPOSE) {
              sx::mbar_wait(&raw_empty[rs], rphase ^ 1);
              sx::mbar_expect_tx(&raw_full[rs], PL::RAW_BYTES);
              uint8_t* ra = raw + rs * PL::RAW_BYTES;
              uint8_t* rb = ra + (XA ? A_STAGE_BYTES : 0);
              if constexpr (XA) {
#pragma unroll
                for (int j = 0; j < BM / MN_BOX; ++j)
                  sx::tma_load_4d(ra + j * MN_BOX_BYTES, &tmA, &raw_full[rs], m0 + j * MN_BOX, k0, az0, az1, pol);
              }
              if constexpr (XB) {
#pragma unroll
                for (int j = 0; j < BN_T / MN_BOX; ++j)
                  sx::tma_load_4d(rb + j * MN_BOX_BYTES, &tmB, &raw_full[rs], n0 + j * MN_BOX, k0, bz0, bz1, pol);
              }
              if (++rs == PL::RAW_SLOTS) { rs = 0; rphase ^= 1; }
            }
            if constexpr (PL::DIRECT_BYTES > 0) {
              sx::mbar_wait(&empty_bar[stage], phase ^ 1);
              sx::mbar_expect_tx(&full_bar[stage], PL::DIRECT_BYTES);
              uint8_t* sa = smem + stage * STAGE_BYTES;
              uint8_t* sb = sa + A_STAGE_BYTES;
              if constexpr (!XA) {
                if constexpr (!A_MN) {
                  sx::tma_load_4d(sa, &tmA, &full_bar[stage], k0, m0, az0, az1, pol);
                } else {
#pragma unroll
                  for (int j = 0; j < BM / MN_BOX; ++j)
                    sx::tma_load_4d(sa + j * MN_BOX_BYTES, &tmA, &full_bar[stage], m0 + j * MN_BOX, k0, az0, az1, pol);
                }
              }
              if constexpr (!XB) {
                if constexpr (!B_MN) {
                  sx::tma_load_4d(sb, &tmB, &full_bar[stage], k0, n0, bz0, bz1, pol);
                } else {
#pragma unroll
                  for (int j = 0; j < BN_T / MN_BOX; ++j)
                    sx::tma_load_4d(sb + j * MN_BOX_BYTES, &tmB, &full_bar[stage], n0 + j * MN_BOX, k0, bz0, bz1, pol);
                }
              }
            }
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    } else if constexpr (PL::XPOSE) {
      // ===================== transposers: raw MN-major slot -> K-major stage =====================
      constexpr int NT = XPOSE_WARPS * 32;
      constexpr int NBLK = (XA && XB ? 2 : 1) * 256;     // 4 x 4 blocks per stage (256 per operand)
      const int xt = threadIdx.x - 32;
      int stage = 0, rs = 0;
      uint32_t phase = 0, rphase = 0;
      for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
        int z0, z1, mb, nb, ks;
        decode(t, z0, z1, mb, nb, ks);
        const int nq = p.z1_loop * split_kbs(ks);
        for (int q = 0; q < nq; ++q) {
          sx::mbar_wait(&raw_full[rs], rphase);
          sx::mbar_wait(&empty_bar[stage], phase ^ 1);
          const uint32_t src = sx::smem_u32(raw + rs * PL::RAW_BYTES);
          const uint32_t dst = sx::smem_u32(smem + stage * STAGE_BYTES + (XA ? 0 : A_STAGE_BYTES));
          for (int b = xt; b < NBLK; b += NT) {
            float4 v[4];
            xpose_load(src + (b >> 8) * A_STAGE_BYTES, b & 255, v);
            xpose_store(dst + (b >> 8) * A_STAGE_BYTES, b & 255, v);
          }
          sx::fence_proxy_async_smem();        // this thread's stores -> visible to wgmma (async proxy)
          __syncwarp();
          if (lane == 0) {
            sx::mbar_arrive(&full_bar[stage]);
            sx::mbar_arrive(&raw_empty[rs]);
          }
          if (++rs == PL::RAW_SLOTS) { rs = 0; rphase ^= 1; }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  if constexpr (WIDE) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");    // 128 x 40 + 256 x 232
  else asm volatile("setmaxnreg.inc.sync.aligned.u32 224;" ::: "memory");
  // ===================== consumers: MMA + epilogue =====================
  const int cw = wg - 1;                        // tile rows 64 cw .. 64 cw + 63
  const int wtid = threadIdx.x & 127;           // thread within the warpgroup
  const int wq = warp & 3;                      // warp within the warpgroup: rows 16 wq .. 16 wq + 15 of those
  const int tr = lane >> 2;                     // row within an 8-row group
  const int tc = (lane & 3) * 2;                // first column of this thread's pair within an 8-column group
  int stage = 0;
  uint32_t phase = 0;

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

  float acc[BN_T / 2];                          // 64 rows x BN_T cols over 128 threads
  for (int t = blockIdx.x; t < p.total_tiles; t += gridDim.x) {
    int z0, z1, mb, nb, ks;
    decode(t, z0, z1, mb, nb, ks);
    const int nq = p.z1_loop * split_kbs(ks);

    // ---------------- main loop ----------------
    int prev = -1;                              // stage whose MMAs may still be in flight
    for (int q = 0; q < nq; ++q) {
      sx::mbar_wait(&full_bar[stage], phase);
      const uint8_t* sa = smem + stage * STAGE_BYTES;
      const uint8_t* sb = sa + A_STAGE_BYTES;
      sx::acc_fence(acc);
      sx::wgmma_fence();
#pragma unroll
      for (int kk = 0; kk < KSTEPS; ++kk) {
        const uint64_t da = desc_a(sa, kk, A_MN && !kTF32), db = desc_b(sb, kk, B_MN && !kTF32);
        const uint32_t accum = (q > 0 || kk > 0) ? 1u : 0u;
        if constexpr (WIDE) sx::wgmma_tf32_n256(acc, da, db, accum);
        else if constexpr (kTF32) sx::wgmma_tf32(acc, da, db, accum);
        else sx::wgmma_bf16<A_MN ? 1 : 0, B_MN ? 1 : 0>(acc, da, db, accum);
      }
      sx::wgmma_commit();
      sx::acc_fence(acc);
      sx::wgmma_wait<1>();                      // the previous stage's MMAs are done: release it
      if (prev >= 0 && wtid == 0) sx::mbar_arrive(&empty_bar[prev]);
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    }
    sx::wgmma_wait<0>();
    sx::acc_fence(acc);
    if (prev >= 0 && wtid == 0) sx::mbar_arrive(&empty_bar[prev]);

    // ---------------- epilogue: accumulator fragments -> bias / GELU / dropout / rounding -> global ----------------
    const long long zoff = (long long)z1 * p.c_sz1 + (long long)z0 * p.c_sz0;
    const float* bias = p.bias ? p.bias + (long long)z1 * p.bias_sz1 + (long long)z0 * p.bias_sz0 : nullptr;
    const bool add_bias = (bias != nullptr) && (ks == 0);
    const int row0 = mb * BM + cw * 64 + wq * 16;
    float tmax = -3.0e38f;                                // running max of this tile's outputs (p.amax)
    float bias_m[2] = {0.f, 0.f};                         // [h]
    if (add_bias && p.bias_mode == SX_BIAS_M) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int r = row0 + 8 * h + tr;
        bias_m[h] = r < p.M ? bias[r] : 0.f;
      }
    }
    // the wide tile runs its 8 column chunks as a rolled loop (unrolled, the 128 accumulators plus the interleaved
    // epilogues of several chunks exceed the consumer's registers): it always takes acc[0..15], then moves the
    // remaining chunks forward
    constexpr int EPI_UNROLL = WIDE ? 1 : BN_T / 32;
#pragma unroll EPI_UNROLL
    for (int c = 0; c < BN_T / 32; ++c) {
      const int col0 = nb * BN_T + c * 32;
      if (col0 >= p.N) break;                   // warp-uniform
      float f[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) f[i] = acc[(WIDE ? 0 : 16 * c) + i] * p.alpha + bias_m[(i >> 1) & 1];
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
      if (!WIDE && p.split_k > 1) {           // (the wide tile never splits)
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
      if constexpr (PL::CT) {
        if (p.ct) {                             // the same values, transposed: staged so each ct row segment is 256 B
          float* cs = ct_stage + cw * CT_WG_FLOATS;
          named_bar_sync(1 + cw);               // the previous chunk's reads of cs are done
#pragma unroll
          for (int j = 0; j < 4; ++j)
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
              for (int e = 0; e < 2; ++e) cs[(8 * j + tc + e) * CT_LD + wq * 16 + 8 * h + tr] = f[4 * j + 2 * h + e];
          named_bar_sync(1 + cw);
          const int m0 = mb * BM + cw * 64;
          const long long ctz = (long long)z1 * p.ct_sz1 + (long long)z0 * p.ct_sz0;
#pragma unroll
          for (int i = 0; i < 4; ++i) {         // 32 columns x 16 float4 over the 128 threads
            const int v = wtid + 128 * i, n = v >> 4, r = (v & 15) * 4;
            const int gn = col0 + n, gm = m0 + r;
            if (gn < p.N && gm < p.M) {
              const float4 x = *reinterpret_cast<const float4*>(cs + n * CT_LD + r);
              float* o = p.ct + ctz + (long long)gn * p.ldct + gm;
              if (gm + 3 < p.M) {
                if (p.stream_out) __stcs(reinterpret_cast<float4*>(o), x);
                else *reinterpret_cast<float4*>(o) = x;
              } else {
                o[0] = x.x;
                if (gm + 1 < p.M) o[1] = x.y;
                if (gm + 2 < p.M) o[2] = x.z;
              }
            }
          }
        }
      }
      if constexpr (WIDE) {
#pragma unroll
        for (int i = 0; i < BN_T / 2 - 16; ++i) acc[i] = acc[i + 16];
      }
    }
    // reduced per tile: a running max held across the whole persistent loop keeps ptxas from giving the consumers
    // setmaxnreg's registers (the wide tile's 128 accumulators then spill)
    if (p.amax) {
      tmax = sx::warp_max(tmax);
      if (lane == 0 && tmax > -3.0e38f) sx::atomic_max_float(p.amax, tmax);
    }
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
int g_wide_tiles = -1;             // 128 x 256 tiles: -1 by shape, 0 never, 1 wherever legal (tests compare the two widths)

template <int ES, bool A_MN, bool B_MN, int BN_T = BN>
int launch(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, int grid, cudaStream_t st) {
  auto kern = sx_gemm_kernel<ES, A_MN, B_MN, BN_T>;
  constexpr int bytes = Plan<ES, A_MN, B_MN, BN_T>::SMEM;
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
  else if (k == "wide_tiles") g_wide_tiles = value < 0 ? -1 : (value ? 1 : 0);
  else {
    sx_set_error("sx_gemm_debug_set: unknown key %s", key);
    return -1;
  }
  return 0;
}

// t: the transposed second output, or null
extern "C" int sx_gemm(const sx_gemm_args* a, const sx_gemm_tout* t, void* stream) {
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
  // 128 x 256 tiles (fewer operand bytes per FLOP) for tf32 products with both operands K-major and no split, when N
  // spans more than one narrow tile and the narrow tiles would take more than one wave.  (H100 SXM at 700 W, plain
  // products: 2744x1024x1024 z16 1.27x faster at 1408 wide tiles, 4096x1024x1024 1.42x at 128; 2744x512x1024 z4,
  // 176 wide tiles = 1.3 waves, 1.01x.)
  const bool amn = a->A.major == SX_MAJOR_MN, bmn = a->B.major == SX_MAJOR_MN;
  const bool wide_legal = es == 4 && !amn && !bmn && p.split_k == 1;
  const long long wide_tt = (long long)p.tiles_m * sx_ceil_div(a->N, BN_WIDE) * a->Z0 * p.Z1;
  const bool wide = wide_legal && (g_wide_tiles == 1 || (g_wide_tiles < 0 && a->N > BN && 2 * wide_tt > sms));
  if (wide) p.tiles_n = sx_ceil_div(a->N, BN_WIDE);
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
  SX_REQUIRE(a->act != SX_ACT_GELU_BWD || (a->preact && a->c_dtype == SX_F32 && p.split_k == 1 && !a->accumulate),
             "sx_gemm: SX_ACT_GELU_BWD needs the fp32 pre-activation in `preact`, fp32 C, split_k=1, accumulate=0");
  SX_REQUIRE(!a->addend || (p.split_k == 1 && !a->accumulate && a->c_dtype == SX_F32), "sx_gemm: addend needs split_k=1, accumulate=0, fp32 C");
  p.drop_p = a->drop_p; p.drop_seed = a->drop_seed;
  p.drop_seed_dev = reinterpret_cast<const unsigned long long*>(a->drop_seed_dev);
  if (t) {
    SX_REQUIRE(t->ct != nullptr, "sx_gemm: null ct");
    SX_REQUIRE(es == 4 && !amn && !bmn, "sx_gemm: ct needs tf32 operands, both K-major");
    SX_REQUIRE(p.split_k == 1 && !a->accumulate && a->c_dtype == SX_F32,
               "sx_gemm: ct needs split_k=1, accumulate=0, fp32 C");
    SX_REQUIRE((reinterpret_cast<uintptr_t>(t->ct) & 15) == 0 && t->ldct % 4 == 0 && t->ct_stride_z0 % 4 == 0 &&
                   t->ct_stride_z1 % 4 == 0 && t->ldct >= a->M,
               "sx_gemm: ct must be 16-byte aligned with ldct >= M and ldct, z strides multiples of 4");
    p.ct = t->ct; p.ldct = t->ldct; p.ct_sz0 = t->ct_stride_z0; p.ct_sz1 = t->ct_stride_z1;
  }
  {
    // H100: 50 MB of L2
    const double out_bytes =
        (double)a->M * a->N * a->Z0 * a->Z1 * (p.c_bf16 ? 2 : 4) * (1 + (a->preact ? 1 : 0) + (t ? 1 : 0));
    p.stream_out = out_bytes > 25.0 * 1024 * 1024;
  }

  CUtensorMap ta, tb;
  int rc = make_map(&ta, a->A, es, a->M, a->K, a->Z0, a->Z1, BM, "A");
  if (rc) return rc;
  rc = make_map(&tb, a->B, es, a->N, a->K, a->Z0, a->Z1, wide ? BN_WIDE : BN, "B");
  if (rc) return rc;

  int grid = p.total_tiles < sms ? p.total_tiles : sms;
  if (g_max_ctas > 0 && grid > g_max_ctas) grid = (int)g_max_ctas;
  p.part = a->part;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (wide) return launch<4, false, false, BN_WIDE>(ta, tb, p, grid, st);
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
