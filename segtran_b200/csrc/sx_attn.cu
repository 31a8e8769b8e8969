// Fused attention-probability kernel of the squeeze-out stage:
//
//   P[b][m] = dropout( softmax_rows( min( alpha * Q[b,:,m] K[b,:,m]^T , clip ) ) )
//
// i.e. reference segtran_shared.py:566-567 (Q.K^T / sqrt(d)), :569-580 (max statistics, conditional clamp), :601
// (softmax over the keys) and :605 (attention dropout) in ONE persistent wgmma kernel: the scores never leave the SM —
// they are accumulated in registers (wgmma fragments: a query row is spread over the four threads of a quad), and the
// row max / sum / exp / dropout / TF32 rounding run on those fragments.  Only P (and, for training, the raw scores the
// backward recomputes P from) is written.
//
// Work decomposition: an item is (batch b, mode m, block of 128 query rows); the CTA owns the item's complete rows
// (two consumer warpgroups of 64 rows), so the softmax statistics need only quad shuffles:
//   keys <= 128 : the scores of the row block are one accumulator: statistics and probabilities come from the same
//                 registers (single pass);
//   keys  > 128 : the scores are produced twice: pass 0 keeps only the running (max, sum) of each row over the 128-key
//                 chunks, pass 1 recomputes each chunk and emits exp2(s - max) / sum.  The recomputation costs d/F of the
//                 P.V contraction that follows and replaces the S write + S read + P write of an unfused path by one
//                 P write.
//
// Clamp (segtran_shared.py:578-580: `if scores.max() > clip: scores = clamp(scores, -clip, clip)`): the upper clamp
// is applied unconditionally — an element above clip implies the global maximum is above clip, so this is exactly the
// reference.  The lower clamp can only change a row whose own maximum is below -(clip - 104) while another row of the
// same call exceeds +clip (fp32 exp underflow makes it a no-op everywhere else); such rows are counted in
// stat[1] and surfaced by sx_attn_diag as diag[2] so that the host can assert it never happened.
#include "sx_common.cuh"
#include "sx_tc.cuh"

namespace {
using namespace sxtc;

constexpr int NUM_THREADS = 384;          // warpgroup 0: TMA producer; warpgroups 1-2: MMA + softmax, 64 rows each
constexpr int STAGES = 4;                 // 4 x (16 KB of Q rows + 16 KB of keys), 32 elements of d each
constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align*/ + 256;
constexpr float LOG2E = 1.4426950408889634f, LN2 = 0.6931471805599453f;

// order-preserving float -> uint map with key(x) > 0 for every finite x, so a ZERO-initialised word is the identity of
// atomicMax (the statistics buffer comes out of the step's zero arena: no fill launch)
__device__ __forceinline__ unsigned int ordered_key(float v) {
  const unsigned int b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ordered_val(unsigned int k) {
  return k == 0u ? -3.0e38f : __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

struct AttnParams {
  int B, M, U1, U2, d;
  int tiles_m, tiles_n, num_kb, items, nsub;
  int q_bcast;                    // Q has batch 1 (shared by the batch)
  float alpha2, clip2;            // alpha * log2(e), clip * log2(e)
  float alpha, clip;
  float* P;
  float* S;                       // raw scaled scores (may be null)
  float* lse;                     // [B][M][U1]  natural-log LSE of the clamped row
  float* rowmax;                  // [B][M][U1]  max of the raw scaled row (may be null)
  float* stat;                    // zero-initialised; [0] ordered_key(max raw scaled score), [1] += rows whose max < -(clip - 104)
  long long ldp;                  // row pitch of P (and S) in elements, multiple of 4
  float drop_p;
  unsigned long long drop_seed;
  const unsigned long long* drop_seed_dev;
  int round_tf32;
};

__global__ void __launch_bounds__(NUM_THREADS, 1)
sx_attn_probs_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const AttnParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = threadIdx.x >> 7;

  if (threadIdx.x == 0) {
    sx::tma_prefetch_desc(&tmQ);
    sx::tma_prefetch_desc(&tmK);
    for (int s = 0; s < STAGES; ++s) {
      sx::mbar_init(&full_bar[s], 1);
      sx::mbar_init(&empty_bar[s], 2);
    }
    sx::fence_barrier_init();
  }
  __syncthreads();

  auto decode = [&](int it, int& b, int& m, int& mb) {
    mb = it % p.tiles_m; it /= p.tiles_m;
    m = it % p.M;
    b = it / p.M;
  };

  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");   // the producer hands its registers over
    // ===================== TMA producer: per chunk and k-block, 128 query rows + 128 keys =====================
    if (warp == 0 && sx::elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
        int b, m, mb;
        decode(it, b, m, mb);
        const int qb = p.q_bcast ? 0 : b;
        for (int sub = 0; sub < p.nsub; ++sub) {
          const int nb = sub % p.tiles_n;
          for (int kb = 0; kb < p.num_kb; ++kb) {
            sx::mbar_wait(&empty_bar[stage], phase ^ 1);
            sx::mbar_expect_tx(&full_bar[stage], STAGE_BYTES);
            uint8_t* sa = smem + stage * STAGE_BYTES;
            sx::tma_load_4d(sa, &tmQ, &full_bar[stage], kb * 32, mb * BM, m, qb, sx::kEvictLast);
            sx::tma_load_4d(sa + A_STAGE_BYTES, &tmK, &full_bar[stage], kb * 32, nb * BN, m, b, sx::kEvictLast);
            if (++stage == STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
    return;
  }

  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
  // ===================== consumers: scores (wgmma) -> softmax on the fragments =====================
  // thread: rows 8h + lane/4 (h = 0, 1) of its warp's 16; columns 8j + 2(lane%4) + e of each 128-key chunk
  const int cw = wg - 1;
  const int wtid = threadIdx.x & 127;
  const int wq = warp & 3;
  const int tr = lane >> 2;
  const int tc = (lane & 3) * 2;
  int stage = 0;
  uint32_t phase = 0;
  float gmax = -3.0e38f;
  int lowrows = 0;
  const uint32_t p16 = sx::drop_p16(p.drop_p);
  const float keep_scale = p.drop_p > 0.f ? 1.f / (1.f - p.drop_p) : 1.f;
  const unsigned long long dseed = p.drop_seed + (p.drop_seed_dev ? *p.drop_seed_dev : 0ull);
  // this thread's column pair is elements (tc & 2, tc & 2 + 1) of a 4-element hash group: one word per pair
  const uint32_t dmul = sx::drop_mul((tc >> 1) & 1), dkey = sx::drop_key(dseed, (tc >> 1) & 1);
  float acc[64];

  for (int it = blockIdx.x; it < p.items; it += gridDim.x) {
    int b, m, mb;
    decode(it, b, m, mb);
    int grow[2];
    long long rowflat[2];
    float rm[2], rl[2], rraw[2], rcp[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      grow[h] = mb * BM + cw * 64 + wq * 16 + 8 * h + tr;
      rowflat[h] = ((long long)b * p.M + m) * p.U1 + grow[h];
      rm[h] = -3.0e38f; rl[h] = 0.f; rraw[h] = -3.0e38f; rcp[h] = 0.f;
    }

    // running statistics of the row over one chunk (log2 units; quad-uniform after the shuffles)
    auto chunk_stats = [&](int nb) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float cm = -3.0e38f;
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (nb * BN + 8 * j + tc + e < p.U2) cm = fmaxf(cm, acc[4 * j + 2 * h + e]);
        cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 1));
        cm = fmaxf(cm, __shfl_xor_sync(0xffffffffu, cm, 2));
        cm *= p.alpha2;                                       // alpha2 > 0: the max commutes with the scaling
        rraw[h] = fmaxf(rraw[h], cm);
        const float mn = fmaxf(rm[h], fminf(cm, p.clip2));
        float s = 0.f;
#pragma unroll
        for (int j = 0; j < 16; ++j)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (nb * BN + 8 * j + tc + e < p.U2) s += sx::ex2_approx(fminf(acc[4 * j + 2 * h + e] * p.alpha2, p.clip2) - mn);
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        s += __shfl_xor_sync(0xffffffffu, s, 2);
        rl[h] = rl[h] * sx::ex2_approx(rm[h] - mn) + s;
        rm[h] = mn;
      }
    };
    // final (max, sum, raw max) of the rows -> 1/sum; lse / rowmax / global statistics
    auto publish = [&]() {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        rcp[h] = 1.f / rl[h];
        if (grow[h] < p.U1) {
          gmax = fmaxf(gmax, rraw[h]);
          if ((lane & 3) == 0) {
            p.lse[rowflat[h]] = (rm[h] + __log2f(rl[h])) * LN2;
            if (p.rowmax) p.rowmax[rowflat[h]] = rraw[h] * LN2;
            if (rraw[h] * LN2 < -(p.clip - 104.f)) ++lowrows;
          }
        }
      }
    };
    // probabilities of one chunk -> P (and the raw scores -> S)
    auto chunk_probs = [&](int nb) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (grow[h] >= p.U1) continue;
        const long long roff = rowflat[h] * p.ldp;
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int col = nb * BN + 8 * j + tc;
          if (col >= p.U2) continue;
          const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
          if (p.S) {
            if (col + 1 < p.U2) *reinterpret_cast<float2*>(p.S + roff + col) = make_float2(v0 * p.alpha, v1 * p.alpha);
            else p.S[roff + col] = v0 * p.alpha;
          }
          float f0 = sx::ex2_approx(fminf(v0 * p.alpha2, p.clip2) - rm[h]) * rcp[h];
          float f1 = sx::ex2_approx(fminf(v1 * p.alpha2, p.clip2) - rm[h]) * rcp[h];
          if (p.drop_p > 0.f) {
            const uint32_t w = sx::drop_word_k(dmul, dkey, (unsigned long long)((roff + col) >> 2));
            f0 = (w & 0xFFFFu) >= p16 ? f0 * keep_scale : 0.f;
            f1 = (w >> 16) >= p16 ? f1 * keep_scale : 0.f;
          }
          if (p.round_tf32) {
            f0 = sx::round_tf32(f0);
            f1 = sx::round_tf32(f1);
          }
          if (col + 1 < p.U2) *reinterpret_cast<float2*>(p.P + roff + col) = make_float2(f0, f1);
          else p.P[roff + col] = f0;
        }
      }
    };

    for (int sub = 0; sub < p.nsub; ++sub) {
      const int nb = sub % p.tiles_n;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        sx::mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = sx::smem_u32(smem + stage * STAGE_BYTES);
        const uint32_t qa = sa + (uint32_t)(cw * 64 * BKB), ka = sa + A_STAGE_BYTES;
        sx::acc_fence(acc);
        sx::wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
          sx::wgmma_tf32(acc, sx::gmma_desc(qa + kk * 32, 16, 1024), sx::gmma_desc(ka + kk * 32, 16, 1024),
                         (kb > 0 || kk > 0) ? 1u : 0u);
        sx::wgmma_commit();
        sx::wgmma_wait<0>();
        sx::acc_fence(acc);
        if (wtid == 0) sx::mbar_arrive(&empty_bar[stage]);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      if (p.nsub == 1) {                        // the whole row block is resident: statistics, then probabilities
        chunk_stats(nb);
        publish();
        chunk_probs(nb);
      } else if (sub < p.tiles_n) {             // pass 0 keeps the running statistics ...
        chunk_stats(nb);
        if (sub == p.tiles_n - 1) publish();
      } else {                                  // ... pass 1 recomputes each chunk and emits the probabilities
        chunk_probs(nb);
      }
    }
  }
  gmax = sx::warp_max(gmax);
  if (lane == 0 && gmax > -3.0e38f) atomicMax(reinterpret_cast<unsigned int*>(&p.stat[0]), ordered_key(gmax * LN2));
  int lr = lowrows;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lr += __shfl_xor_sync(0xffffffffu, lr, o);
  if (lane == 0 && lr > 0) atomicAdd(&p.stat[1], (float)lr);
}

// diag[0] = running max of the scores, diag[1] += 1 when the clamp fired, diag[2] += rows the lower clamp could have
// touched in a clamped call (see the header comment)  — the module's max_attn / clamp_count counters
// (segtran_shared.py:575-587) without host synchronisation
__global__ void attn_diag_kernel(float* stat, float clip, float* diag) {
  const float mx = ordered_val(__float_as_uint(stat[0]));
  stat[2] = mx;                                  // the plain float maximum (what sx_softmax_bwd's `amax` expects)
  if (diag) {
    diag[0] = fmaxf(diag[0], mx);
    if (mx > clip) {
      diag[1] += 1.f;
      diag[2] += stat[1];
    }
  }
}

}  // namespace

extern "C" int sx_attn_probs_fwd(const sx_attn_probs_args* a, void* stream) {
  SX_REQUIRE(a != nullptr, "sx_attn_probs_fwd: null args");
  SX_REQUIRE(a->B > 0 && a->M > 0 && a->U1 > 0 && a->U2 > 0 && a->d > 0, "sx_attn_probs_fwd: bad shape");
  SX_REQUIRE(a->Q && a->K && a->P && a->lse && a->stat, "sx_attn_probs_fwd: null pointer");
  SX_REQUIRE(a->d % 4 == 0 && a->ldp % 4 == 0 && a->ldp >= a->U2, "sx_attn_probs_fwd: d and ldp must be multiples of 4");
  SX_REQUIRE((reinterpret_cast<uintptr_t>(a->P) & 15) == 0 && (!a->S || (reinterpret_cast<uintptr_t>(a->S) & 15) == 0),
             "sx_attn_probs_fwd: outputs must be 16-byte aligned");
  const int sms = sm_count_cached();
  SX_REQUIRE(sms > 0, "sx_attn_probs_fwd: no CUDA device (this library has no CPU fallback)");

  AttnParams p{};
  p.B = a->B; p.M = a->M; p.U1 = a->U1; p.U2 = a->U2; p.d = a->d;
  p.tiles_m = sx_ceil_div(a->U1, BM);
  p.tiles_n = sx_ceil_div(a->U2, BN);
  p.num_kb = sx_ceil_div(a->d, 32);
  p.nsub = p.tiles_n == 1 ? 1 : 2 * p.tiles_n;
  const long long items = (long long)a->B * a->M * p.tiles_m;
  SX_REQUIRE(items < (1ll << 30), "sx_attn_probs_fwd: too many row blocks");
  p.items = (int)items;
  p.q_bcast = a->q_bstride == 0 && a->B > 1;
  p.alpha = a->alpha; p.clip = a->clip;
  p.alpha2 = a->alpha * LOG2E; p.clip2 = a->clip * LOG2E;
  p.P = reinterpret_cast<float*>(a->P); p.S = reinterpret_cast<float*>(a->S);
  p.lse = a->lse; p.rowmax = a->rowmax; p.stat = a->stat;
  p.ldp = a->ldp;
  p.drop_p = a->drop_p; p.drop_seed = a->drop_seed;
  p.drop_seed_dev = reinterpret_cast<const unsigned long long*>(a->drop_seed_dev);
  p.round_tf32 = a->round_tf32;

  // Q [Bq][U1][M*d] and K [B][U2][M*d] as (k, row, mode, batch) tensor maps: the per-mode slices are strided views
  sx_operand oq{}, ok{};
  oq.ptr = a->Q; oq.major = SX_MAJOR_K; oq.ld = a->q_ld; oq.stride_z0 = a->d; oq.stride_z1 = p.q_bcast ? 0 : a->q_bstride;
  ok.ptr = a->K; ok.major = SX_MAJOR_K; ok.ld = a->k_ld; ok.stride_z0 = a->d; ok.stride_z1 = a->k_bstride;
  if (a->M == 1) { oq.stride_z0 = 0; ok.stride_z0 = 0; }
  if (a->B == 1) { oq.stride_z1 = 0; ok.stride_z1 = 0; }
  CUtensorMap tq, tk;
  int rc = make_map(&tq, oq, 4, a->U1, a->d, a->M, a->B, BM, "Q");
  if (rc) return rc;
  rc = make_map(&tk, ok, 4, a->U2, a->d, a->M, a->B, BN, "K");
  if (rc) return rc;

  SX_CHECK_CUDA(set_max_smem_once(sx_attn_probs_kernel, SMEM_BYTES));
  const int grid = p.items < sms ? p.items : sms;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  sx_attn_probs_kernel<<<grid, NUM_THREADS, SMEM_BYTES, st>>>(tq, tk, p);
  SX_CHECK_CUDA(cudaGetLastError());
  attn_diag_kernel<<<1, 1, 0, st>>>(a->stat, a->clip, a->diag);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
