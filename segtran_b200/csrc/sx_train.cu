// Training-step tail of the hot path (SURVEY.md §8 f.2): the segmentation loss on the logits and the BertAdam update of
// the flat parameter / gradient buckets.  All HBM-bound streaming kernels; every scalar the step needs (loss, clip
// coefficients, scheduled learning rates, the step counter) stays on the device so the whole step is CUDA-graph safe.
//
//   loss  (train3d.py:731-756, utils/losses.py:47-60):
//     ce    = mean_{b,k,v} [ pw_k y softplus(-x) + (1-y) softplus(x) ]                 BCEWithLogits(pos_weight)
//     dice  = sum_{k>=1} cw_k mean_b [ 1 - (2 I + eps) / (Z + Y + eps) ],  I = sum s y, Z = sum s^2, Y = sum y^2, s = sigmoid(x)
//     loss  = (1-W) ce + W dice
//   optimiser (optimization.py:90-164 + train3d.py:760-761): global norm clip, per-parameter norm clip, Adam moments
//     without bias correction, decoupled weight decay, warm-up schedule; parameters whose gradient is exactly zero are
//     skipped like the reference skips `p.grad is None` (never-used parameters).
#include <algorithm>

#include "../../include/segtran_b200.h"
#include "sx_common.cuh"

namespace {

constexpr float DICE_EPS = 1e-5f;

__device__ __forceinline__ float block_sum(float v, float* red) {      // red: 32 floats of shared memory
  v = sx::warp_sum(v);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  v = (threadIdx.x < (blockDim.x >> 5)) ? red[threadIdx.x] : 0.f;
  if (w == 0) v = sx::warp_sum(v);
  return v;                                                             // valid in thread 0
}

struct LossTerms { float bce, inter, z, y; };

__device__ __forceinline__ void loss_terms(float x, float y, float pw, LossTerms& t) {
  // e in (0,1]: the fast exp / log / divide are each within ~2 ulp, i.e. <= 2e-7 absolute per voxel on terms of
  // magnitude <= |x| + 0.7 — far inside the 1e-5 loss parity (tests/test_gpu_train.py) and 5x fewer instructions
  const float e = __expf(-fabsf(x));
  const float l1p = __logf(1.f + e);
  const float sp_pos = fmaxf(x, 0.f) + l1p;                             // softplus(x)  = -log(1 - sigmoid(x))
  const float sp_neg = sp_pos - x;                                      // softplus(-x) = -log(sigmoid(x))
  const float s = __fdividef(x >= 0.f ? 1.f : e, 1.f + e);
  t.bce += pw * y * sp_neg + (1.f - y) * sp_pos;
  t.inter += s * y;
  t.z += s * s;
  t.y += y * y;
}

// grid (chunks, B*K); sums[(b*K+k)*4 + {bce, I, Z, Y}] (double, zeroed by the caller)
__global__ void __launch_bounds__(256)
seg_loss_fwd_kernel(const float* __restrict__ x, const float* __restrict__ y, long long V, int K,
                    const float* __restrict__ pw, double* __restrict__ sums, int vec4) {
  __shared__ float red[32];
  const int bk = blockIdx.y;
  const float p = pw ? pw[bk % K] : 1.f;
  const float* xr = x + (long long)bk * V;
  const float* yr = y + (long long)bk * V;
  LossTerms t = {0.f, 0.f, 0.f, 0.f};
  if (vec4) {
    const long long V4 = V >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V4; i += (long long)gridDim.x * blockDim.x) {
      const float4 a = __ldcs(reinterpret_cast<const float4*>(xr) + i);
      const float4 b = __ldcs(reinterpret_cast<const float4*>(yr) + i);
      loss_terms(a.x, b.x, p, t); loss_terms(a.y, b.y, p, t); loss_terms(a.z, b.z, p, t); loss_terms(a.w, b.w, p, t);
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (long long)gridDim.x * blockDim.x)
      loss_terms(xr[i], yr[i], p, t);
  }
  const float s0 = block_sum(t.bce, red), s1 = block_sum(t.inter, red), s2 = block_sum(t.z, red), s3 = block_sum(t.y, red);
  if (threadIdx.x == 0) {
    atomicAdd(&sums[bk * 4 + 0], (double)s0);
    atomicAdd(&sums[bk * 4 + 1], (double)s1);
    atomicAdd(&sums[bk * 4 + 2], (double)s2);
    atomicAdd(&sums[bk * 4 + 3], (double)s3);
  }
}

// one block: loss scalars + the per-(b,k) Dice gradient coefficients used by the backward pass
__global__ void seg_loss_finalize_kernel(const double* __restrict__ sums, int B, int K, long long V,
                                         const float* __restrict__ cw, float dice_w, float* __restrict__ out3,
                                         float* __restrict__ coef) {
  __shared__ double sh_ce[256], sh_dice[256];
  double ce = 0.0, dice = 0.0;
  for (int i = threadIdx.x; i < B * K; i += blockDim.x) {
    const int k = i % K;
    const double I = sums[i * 4 + 1], Z = sums[i * 4 + 2], Y = sums[i * 4 + 3];
    ce += sums[i * 4 + 0];
    const double w = (k >= 1 && cw) ? (double)cw[k] : (k >= 1 ? 1.0 : 0.0);
    const double D = Z + Y + (double)DICE_EPS, num = 2.0 * I + (double)DICE_EPS;
    dice += w * (1.0 - num / D) / B;
    // d loss / d s = dice_w * w * (-1/B) * ( 2 y / D - 2 s num / D^2 )  =  a y + c s
    coef[i * 2 + 0] = (float)(-(double)dice_w * w * 2.0 / (D * B));
    coef[i * 2 + 1] = (float)((double)dice_w * w * 2.0 * num / (D * D * B));
  }
  sh_ce[threadIdx.x] = ce; sh_dice[threadIdx.x] = dice;
  __syncthreads();
  if (threadIdx.x == 0) {
    double c = 0.0, d = 0.0;
    for (int i = 0; i < blockDim.x; ++i) { c += sh_ce[i]; d += sh_dice[i]; }
    c /= (double)B * K * (double)V;
    out3[0] = (float)((1.0 - (double)dice_w) * c + (double)dice_w * d);
    out3[1] = (float)c;
    out3[2] = (float)d;
  }
}

__device__ __forceinline__ float loss_grad(float x, float y, float pw, float ce_scale, float a, float c, float g) {
  const float e = __expf(-fabsf(x));
  const float s = __fdividef(x >= 0.f ? 1.f : e, 1.f + e);
  const float dce = s * (1.f - y) - pw * y * (1.f - s);
  return g * (ce_scale * dce + (a * y + c * s) * s * (1.f - s));
}

__global__ void __launch_bounds__(256)
seg_loss_bwd_kernel(const float* __restrict__ x, const float* __restrict__ y, long long V, int K,
                    const float* __restrict__ pw, const float* __restrict__ coef, float ce_scale,
                    const float* __restrict__ gout, float* __restrict__ dx, int vec4) {
  const int bk = blockIdx.y;
  const float p = pw ? pw[bk % K] : 1.f;
  const float a = coef[bk * 2 + 0], c = coef[bk * 2 + 1];
  const float g = gout ? *gout : 1.f;
  const float* xr = x + (long long)bk * V;
  const float* yr = y + (long long)bk * V;
  float* dr = dx + (long long)bk * V;
  if (vec4) {
    const long long V4 = V >> 2;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V4; i += (long long)gridDim.x * blockDim.x) {
      const float4 xv = __ldcs(reinterpret_cast<const float4*>(xr) + i);
      const float4 yv = __ldcs(reinterpret_cast<const float4*>(yr) + i);
      float4 o;
      o.x = loss_grad(xv.x, yv.x, p, ce_scale, a, c, g); o.y = loss_grad(xv.y, yv.y, p, ce_scale, a, c, g);
      o.z = loss_grad(xv.z, yv.z, p, ce_scale, a, c, g); o.w = loss_grad(xv.w, yv.w, p, ce_scale, a, c, g);
      reinterpret_cast<float4*>(dr)[i] = o;
    }
  } else {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (long long)gridDim.x * blockDim.x)
      dr[i] = loss_grad(xr[i], yr[i], p, ce_scale, a, c, g);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// BertAdam on flat buckets.  A segment = <= SEG elements of ONE parameter: (param index, offset in the bucket, length).
// ------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
adam_sumsq_kernel(const float* __restrict__ g, const int* __restrict__ seg_param, const long long* __restrict__ seg_off,
                  const int* __restrict__ seg_len, double* __restrict__ sumsq) {
  __shared__ float red[32];
  const int s = blockIdx.x;
  const float* gp = g + seg_off[s];
  const int n = seg_len[s];
  float acc = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float v = gp[i];
    acc = fmaf(v, v, acc);
  }
  acc = block_sum(acc, red);
  if (threadIdx.x == 0 && acc != 0.f) atomicAdd(&sumsq[seg_param[s]], (double)acc);
}

// one block: clip coefficients, scheduled learning rates, step counter
__global__ void adam_finalize_kernel(const double* __restrict__ sumsq, int P, float grad_clip, float max_grad_norm,
                                     const float* __restrict__ lr, float warmup, long long t_total, int schedule,
                                     long long* __restrict__ step, float* __restrict__ coef, float* __restrict__ lr_eff,
                                     float* __restrict__ total_norm) {
  __shared__ double sh[256];
  double t = 0.0;
  for (int i = threadIdx.x; i < P; i += blockDim.x) t += sumsq[i];
  sh[threadIdx.x] = t;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0.0;
    for (int i = 0; i < blockDim.x; ++i) a += sh[i];
    sh[0] = sqrt(a);
  }
  __syncthreads();
  const double total = sh[0];
  const double cg = grad_clip > 0.f ? fmin((double)grad_clip / (total + 1e-6), 1.0) : 1.0;      // clip_grad_norm_
  double sched = 1.0;
  if (t_total != -1) {
    const double x = (double)(*step) / (double)t_total;
    if (x < (double)warmup) sched = x / (double)warmup;
    else if (schedule == SX_SCHED_WARMUP_LINEAR) sched = fmax((x - 1.0) / ((double)warmup - 1.0), 0.0);
    else sched = 1.0;                                                                           // warmup_constant
  }
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    const double n2 = sumsq[i];
    if (n2 == 0.0) {
      coef[i] = -1.f;                                                 // gradient exactly zero: parameter not used, skip it
    } else {
      const double np = cg * sqrt(n2);                                // its norm after the global clip
      const double cp = max_grad_norm > 0.f ? fmin((double)max_grad_norm / (np + 1e-6), 1.0) : 1.0;
      coef[i] = (float)(cg * cp);
    }
    lr_eff[i] = (float)((double)lr[i] * sched);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    if (total_norm) *total_norm = (float)total;
    *step += 1;
  }
}

__global__ void __launch_bounds__(256)
adam_update_kernel(float* __restrict__ p, float* __restrict__ p_tf32, const float* __restrict__ g, float* __restrict__ m,
                   float* __restrict__ v,
                   const int* __restrict__ seg_param, const long long* __restrict__ seg_off,
                   const int* __restrict__ seg_len, const float* __restrict__ coef, const float* __restrict__ lr_eff,
                   const float* __restrict__ wd, float b1, float omb1, float b2, float omb2, float eps) {
  const int s = blockIdx.x;
  const int pi = seg_param[s];
  const float cf = coef[pi];
  if (cf < 0.f) return;                                               // block-uniform
  const float lr = lr_eff[pi], decay = wd[pi];
  const long long off = seg_off[s];
  const int n = seg_len[s];
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const float gg = g[off + i] * cf;
    const float pp = p[off + i];
    const float mm = b1 * m[off + i] + omb1 * gg;            // omb = 1 - beta rounded from double, like the reference's
    const float vv = b2 * v[off + i] + omb2 * gg * gg;       // python-float alpha / value arguments
    float upd = mm / (sqrtf(vv) + eps);
    if (decay > 0.f) upd += decay * pp;
    m[off + i] = mm;
    v[off + i] = vv;
    const float pn = pp - lr * upd;
    p[off + i] = pn;
    if (p_tf32) p_tf32[off + i] = sx::round_tf32(pn);       // TF32 twin the next forward feeds to the tensor cores
  }
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)

extern "C" int sx_seg_loss_fwd(const float* logits, const float* mask, int32_t B, int32_t K, int64_t V,
                               const float* pos_weight, const float* class_w, float dice_w, double* sums, float* out3,
                               float* coef, void* stream) {
  SX_REQUIRE(logits && mask && sums && out3 && coef && B >= 1 && K >= 1 && V >= 1, "sx_seg_loss_fwd: bad arguments");
  SX_CHECK_CUDA(cudaMemsetAsync(sums, 0, sizeof(double) * 4 * B * K, ST(stream)));
  const int vec4 = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(mask) & 15) == 0);
  const long long work = vec4 ? V / 4 : V;
  const int chunks = (int)std::max<long long>(1, std::min<long long>(sx_ceil_div(work, 256 * 4), (sm_count_cached() * 8ll) / (B * K) + 1));
  dim3 grid(chunks, B * K);
  seg_loss_fwd_kernel<<<grid, 256, 0, ST(stream)>>>(logits, mask, V, K, pos_weight, sums, vec4);
  SX_CHECK_CUDA(cudaGetLastError());
  seg_loss_finalize_kernel<<<1, 256, 0, ST(stream)>>>(sums, B, K, V, class_w, dice_w, out3, coef);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_seg_loss_bwd(const float* logits, const float* mask, int32_t B, int32_t K, int64_t V,
                               const float* pos_weight, const float* coef, float ce_scale, const float* gout,
                               float* dlogits, void* stream) {
  SX_REQUIRE(logits && mask && coef && dlogits && B >= 1 && K >= 1 && V >= 1, "sx_seg_loss_bwd: bad arguments");
  const int vec4 = (V % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) &&
                   ((reinterpret_cast<uintptr_t>(mask) & 15) == 0) && ((reinterpret_cast<uintptr_t>(dlogits) & 15) == 0);
  const long long work = vec4 ? V / 4 : V;
  const int chunks = (int)std::max<long long>(1, std::min<long long>(sx_ceil_div(work, 256 * 4), (sm_count_cached() * 8ll) / (B * K) + 1));
  dim3 grid(chunks, B * K);
  seg_loss_bwd_kernel<<<grid, 256, 0, ST(stream)>>>(logits, mask, V, K, pos_weight, coef, ce_scale, gout, dlogits, vec4);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_adam_step(float* p, float* p_tf32, const float* g, float* m, float* v, const int32_t* seg_param,
                            const int64_t* seg_off, const int32_t* seg_len, int32_t nseg, int32_t P, const float* lr,
                            const float* wd, double b1, double b2, double eps, float grad_clip, float max_grad_norm,
                            float warmup, int64_t t_total, int32_t schedule, int64_t* step, double* sumsq, float* coef,
                            float* lr_eff, float* total_norm, void* stream) {
  SX_REQUIRE(p && g && m && v && seg_param && seg_off && seg_len && lr && wd && step && sumsq && coef && lr_eff,
             "sx_adam_step: null argument");
  SX_REQUIRE(nseg >= 1 && P >= 1, "sx_adam_step: empty parameter set");
  SX_REQUIRE(schedule == SX_SCHED_WARMUP_LINEAR || schedule == SX_SCHED_WARMUP_CONSTANT, "sx_adam_step: bad schedule %d",
             schedule);
  SX_REQUIRE(t_total == -1 || (warmup > 0.f && warmup < 1.f), "sx_adam_step: warmup must be in (0,1) when t_total is set");
  SX_CHECK_CUDA(cudaMemsetAsync(sumsq, 0, sizeof(double) * P, ST(stream)));
  adam_sumsq_kernel<<<nseg, 256, 0, ST(stream)>>>(g, seg_param, reinterpret_cast<const long long*>(seg_off), seg_len, sumsq);
  SX_CHECK_CUDA(cudaGetLastError());
  adam_finalize_kernel<<<1, 256, 0, ST(stream)>>>(sumsq, P, grad_clip, max_grad_norm, lr, warmup, t_total, schedule,
                                                 reinterpret_cast<long long*>(step), coef, lr_eff, total_norm);
  SX_CHECK_CUDA(cudaGetLastError());
  adam_update_kernel<<<nseg, 256, 0, ST(stream)>>>(p, p_tf32, g, m, v, seg_param, reinterpret_cast<const long long*>(seg_off),
                                                   seg_len, coef, lr_eff, wd, (float)b1, (float)(1.0 - b1), (float)b2, (float)(1.0 - b2),
                                                   (float)eps);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
