// 2-D sliding-window inference post-process and per-image evaluation (reference code/test_util2d.py:169-265
// test_single_batch / calc_dice / calc_batch_metric, dataloaders/datasets2d.py:178-196 harden_segmap2d and
// utils/losses.py:76-127 calc_vcdr without a batch dimension).
//
// The reference upsamples each window's logits to the window size, writes them, writes their sigmoid, then adds it into
// the accumulator; for the metrics it resizes every soft prediction to its ground truth's size, hardens it and reduces
// each class with a host sync.  Here the bilinear resize (align_corners=False, the tap rule of sx_resample.cuh) is
// evaluated on the fly where its value is consumed, so neither the resized logits, the probabilities nor the resized
// prediction are ever written.  All three kernels are bandwidth-bound.
//
// Determinism: windows are accumulated by sequential launches (overlapping windows never race, and each pixel's sum is
// added in the reference's window order); the metric kernel only produces integer counts and row extrema with integer
// atomics, which give the same result in any order.
#include "sx_common.cuh"
#include "sx_resample.cuh"

namespace {

constexpr float kThreshold = 0.5f;     // harden_segmap2d's T and calc_vcdr's thres
constexpr int kMaxClasses = 8;
constexpr int kRowSlots = 8;           // {pred, gt} x {disc (class 1), cup (class 2)} x {max, min}

// bilinear value of one [h][w] plane at the taps (y0, y1, wy) x (x0, x1, wx), in PyTorch's upsample_bilinear2d order
__device__ __forceinline__ float bilerp(const float* __restrict__ p, int w, int y0, int y1, float wy, int x0, int x1, float wx) {
  const float hy = 1.f - wy, hx = 1.f - wx;
  return hy * (hx * __ldg(p + (long long)y0 * w + x0) + wx * __ldg(p + (long long)y0 * w + x1)) +
         wy * (hx * __ldg(p + (long long)y1 * w + x0) + wx * __ldg(p + (long long)y1 * w + x1));
}

// preds[b][k][xs+i][ys+j] += sigmoid(upsample(flip_m(scores[b][k]))[i][j]);  cnt[xs+i][ys+j] += 1   (test_util2d.py:209-214)
// mirror bit 0 reverses the h axis, bit 1 the w axis: the flip is applied to the source taps, before the upsample.
// kWeighted: both terms are scaled by g = max(tx[i] * ty[j], 1e-3), the window weight at the upsampled position (i, j);
// the weight tables are the trailing arguments, which the unweighted instantiation never reads.
template <bool kWeighted>
__global__ void sw2d_accumulate_kernel(const float* __restrict__ scores, int B, int K, int h, int w, int dx, int dy,
                                       float* __restrict__ preds, float* __restrict__ cnt, int H2, int W2, int xs, int ys,
                                       int mirror, const float* __restrict__ tx, const float* __restrict__ ty) {
  const long long pw = (long long)dx * dy;
  const long long total = (long long)B * pw;
  const float ry = (float)h / (float)dx, rx = (float)w / (float)dy;
  const long long plane_in = (long long)h * w, plane_out = (long long)H2 * W2;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(t / pw);
    const int r = (int)(t - (long long)b * pw);
    const int i = r / dy, j = r - (r / dy) * dy;
    int y0, y1, x0, x1;
    float wy, wx;
    sx::src_index(i, ry, h, y0, y1, wy);
    sx::src_index(j, rx, w, x0, x1, wx);
    if (mirror & 1) { y0 = h - 1 - y0; y1 = h - 1 - y1; }
    if (mirror & 2) { x0 = w - 1 - x0; x1 = w - 1 - x1; }
    const long long o = (long long)(xs + i) * W2 + (ys + j);
    if constexpr (kWeighted) {
      const float g = fmaxf(__ldg(tx + i) * __ldg(ty + j), kSwMinWeight);
      for (int k = 0; k < K; ++k) {
        const long long bk = (long long)b * K + k;
        const float s = bilerp(scores + bk * plane_in, w, y0, y1, wy, x0, x1, wx);
        preds[bk * plane_out + o] += __fmul_rn(g, 1.f / (1.f + expf(-s)));   // rounded product, then the add
      }
      if (b == 0) cnt[o] += g;
    } else {
      for (int k = 0; k < K; ++k) {
        const long long bk = (long long)b * K + k;
        const float s = bilerp(scores + bk * plane_in, w, y0, y1, wy, x0, x1, wx);
        preds[bk * plane_out + o] += 1.f / (1.f + expf(-s));     // torch.sigmoid
      }
      if (b == 0) cnt[o] += 1.f;                                   // one count map: every image sees the same windows
    }
  }
}

// soft[b][k][y][x] = preds[b][k][hl+y][wl+x] / cnt[hl+y][wl+x]; hard[k>=1] = soft >= T, hard[0] = no class >= 1 fired
__global__ void sw2d_finalize_kernel(const float* __restrict__ preds, const float* __restrict__ cnt, int B, int K, int H2,
                                     int W2, int hl, int wl, int H, int W, float* __restrict__ soft, int* __restrict__ hard) {
  const long long pw = (long long)H * W;
  const long long total = (long long)B * pw;
  const long long plane_in = (long long)H2 * W2;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long b = t / pw;
    const long long r = t - b * pw;
    const int y = (int)(r / W), x = (int)(r - (r / W) * W);
    const long long o = (long long)(hl + y) * W2 + (wl + x);
    const float c = cnt[o];
    int fired = 0;
    for (int k = 0; k < K; ++k) {
      const long long bk = b * K + k;
      const float v = preds[bk * plane_in + o] / c;
      soft[bk * pw + r] = v;
      if (k > 0) {
        const int hk = v >= kThreshold ? 1 : 0;
        hard[bk * pw + r] = hk;
        fired |= hk;
      }
    }
    hard[b * K * pw + r] = fired ? 0 : 1;
  }
}

// Per-image counts of one [K][Hg][Wg] ground truth against the [K][h][w] soft prediction resized to Hg x Wg and hardened.
// counts[b] (int32, zeroed by the host): for each class c = 1..K-1, |P and G|, |P|, |G| at 3(c-1) + {0,1,2}; then the row
// slots at 3(K-1) + {0..7}: for the prediction then the ground truth, for class 1 then class 2, (last row + 1) and
// (Hg - first row) of the rows the class occupies (both 0 when it occupies none, so a zeroed slot means "empty" and every
// slot is an atomicMax); then the number of ground-truth values of classes >= 1 that are neither 0 nor 1.  P is
// soft >= T, G is gt >= T.  pred == nullptr skips the prediction (its counts and slots stay 0).
__global__ void __launch_bounds__(256) eval2d_counts_kernel(const float* __restrict__ pred, int K, int h, int w,
                                                            const float* __restrict__ gt, int Hg, int Wg,
                                                            int* __restrict__ counts) {
  constexpr int kMaxSlots = 3 * (kMaxClasses - 1) + kRowSlots + 1;
  __shared__ int acc[kMaxSlots];
  const int b = blockIdx.y;
  const int nc = K - 1;
  const int nslots = 3 * nc + kRowSlots + 1;
  for (int s = threadIdx.x; s < nslots; s += blockDim.x) acc[s] = 0;
  __syncthreads();

  const long long pw = (long long)Hg * Wg;
  const float* pb = pred ? pred + (long long)b * K * h * w : nullptr;
  const float* gb = gt + (long long)b * K * pw;
  const float ry = pred ? (float)h / (float)Hg : 0.f, rx = pred ? (float)w / (float)Wg : 0.f;
  int n[3 * (kMaxClasses - 1)];
  int rows[kRowSlots];
  int nonbin = 0;
#pragma unroll
  for (int s = 0; s < 3 * (kMaxClasses - 1); ++s) n[s] = 0;
#pragma unroll
  for (int s = 0; s < kRowSlots; ++s) rows[s] = 0;

  for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; p < pw; p += (long long)gridDim.x * blockDim.x) {
    const int y = (int)(p / Wg), x = (int)(p - (long long)y * Wg);
    int y0 = 0, y1 = 0, x0 = 0, x1 = 0;
    float wy = 0.f, wx = 0.f;
    if (pb) {
      sx::src_index(y, ry, h, y0, y1, wy);
      sx::src_index(x, rx, w, x0, x1, wx);
    }
#pragma unroll
    for (int c = 1; c < kMaxClasses; ++c) {
      if (c < K) {
        const float g = __ldg(gb + (long long)c * pw + p);
        const int gh = g >= kThreshold ? 1 : 0;
        nonbin += (g != 0.f && g != 1.f) ? 1 : 0;
        int ph = 0;
        if (pb) ph = bilerp(pb + (long long)c * h * w, w, y0, y1, wy, x0, x1, wx) >= kThreshold ? 1 : 0;
        n[3 * (c - 1) + 0] += ph & gh;
        n[3 * (c - 1) + 1] += ph;
        n[3 * (c - 1) + 2] += gh;
        if (c <= 2) {
          if (ph) {
            rows[2 * (c - 1) + 0] = max(rows[2 * (c - 1) + 0], y + 1);
            rows[2 * (c - 1) + 1] = max(rows[2 * (c - 1) + 1], Hg - y);
          }
          if (gh) {
            rows[4 + 2 * (c - 1) + 0] = max(rows[4 + 2 * (c - 1) + 0], y + 1);
            rows[4 + 2 * (c - 1) + 1] = max(rows[4 + 2 * (c - 1) + 1], Hg - y);
          }
        }
      }
    }
  }

  // warp, then CTA, then one global atomic per slot and CTA
#pragma unroll
  for (int c = 1; c < kMaxClasses; ++c) {
    if (c < K) {
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const unsigned v = __reduce_add_sync(0xffffffffu, (unsigned)n[3 * (c - 1) + q]);
        if ((threadIdx.x & 31) == 0 && v) atomicAdd(&acc[3 * (c - 1) + q], (int)v);
      }
    }
  }
#pragma unroll
  for (int s = 0; s < kRowSlots; ++s) {
    const int v = __reduce_max_sync(0xffffffffu, rows[s]);
    if ((threadIdx.x & 31) == 0 && v) atomicMax(&acc[3 * nc + s], v);
  }
  const unsigned nb = __reduce_add_sync(0xffffffffu, (unsigned)nonbin);
  if ((threadIdx.x & 31) == 0 && nb) atomicAdd(&acc[3 * nc + kRowSlots], (int)nb);
  __syncthreads();

  int* out = counts + (long long)b * nslots;
  for (int s = threadIdx.x; s < nslots; s += blockDim.x) {
    const int v = acc[s];
    if (!v) continue;
    if (s >= 3 * nc && s < 3 * nc + kRowSlots) atomicMax(out + s, v);
    else atomicAdd(out + s, v);
  }
}

int grid_for(long long work, int per_launch_cap) {
  long long blocks = (work + 255) / 256;
  if (blocks > per_launch_cap) blocks = per_launch_cap;
  return (int)(blocks < 1 ? 1 : blocks);
}

}  // namespace

extern "C" int sx_sw2d_accumulate(const float* scores, int32_t B, int32_t K, int32_t h, int32_t w, int32_t dx, int32_t dy,
                                  float* preds, float* cnt, int32_t H2, int32_t W2, int32_t xs, int32_t ys, int32_t mirror,
                                  const sx_sw_weights* wt, void* stream) {
  SX_REQUIRE(B > 0 && K > 0 && h > 0 && w > 0 && dx > 0 && dy > 0 && xs >= 0 && ys >= 0 && xs + dx <= H2 && ys + dy <= W2,
             "sx_sw2d_accumulate: window [%d+%d, %d+%d] outside the %dx%d image, or empty scores (%dx%d)", xs, dx, ys, dy, H2, W2,
             h, w);
  SX_REQUIRE(mirror >= 0 && mirror <= 3, "sx_sw2d_accumulate: mirror mask %d is not a subset of {H, W} (0..3)", mirror);
  SX_REQUIRE(!wt || (wt->wx && wt->wy && wt->nx > 0 && wt->ny > 0 && wt->nz > 0),
             "sx_sw2d_accumulate: empty or missing table (wx=%p nx=%d, wy=%p ny=%d, nz=%d)", (const void*)wt->wx, wt->nx,
             (const void*)wt->wy, wt->ny, wt->nz);
  SX_REQUIRE(!wt || (wt->nx == dx && wt->ny == dy && wt->nz == 1),
             "sx_sw2d_accumulate: window weight tables of %dx%dx%d for a %dx%d window", wt->nx, wt->ny, wt->nz, dx, dy);
  const int blocks = grid_for((long long)B * dx * dy, sm_count_cached() * 8);
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (wt)
    sw2d_accumulate_kernel<true><<<blocks, 256, 0, st>>>(scores, B, K, h, w, dx, dy, preds, cnt, H2, W2, xs, ys, mirror, wt->wx,
                                                         wt->wy);
  else
    sw2d_accumulate_kernel<false><<<blocks, 256, 0, st>>>(scores, B, K, h, w, dx, dy, preds, cnt, H2, W2, xs, ys, mirror,
                                                          nullptr, nullptr);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_sw2d_finalize(const float* preds, const float* cnt, int32_t B, int32_t K, int32_t H2, int32_t W2, int32_t hl,
                                int32_t wl, int32_t H, int32_t W, float* soft, int32_t* hard, void* stream) {
  SX_REQUIRE(B > 0 && K > 0 && H > 0 && W > 0 && hl >= 0 && wl >= 0 && hl + H <= H2 && wl + W <= W2,
             "sx_sw2d_finalize: crop [%d+%d, %d+%d] outside the %dx%d accumulator", hl, H, wl, W, H2, W2);
  const int blocks = grid_for((long long)B * H * W, sm_count_cached() * 8);
  sw2d_finalize_kernel<<<blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(preds, cnt, B, K, H2, W2, hl, wl, H, W,
                                                                                   soft, hard);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_eval2d_counts(const float* pred, int32_t B, int32_t K, int32_t h, int32_t w, const float* gt, int32_t Hg,
                                int32_t Wg, int32_t* counts, void* stream) {
  SX_REQUIRE(B > 0 && B <= 65535 && K >= 2 && K <= kMaxClasses && Hg > 0 && Wg > 0 && (!pred || (h > 0 && w > 0)),
             "sx_eval2d_counts: need 1..65535 images of 2..%d classes and non-empty maps (got B=%d K=%d, %dx%d pred, %dx%d gt)",
             kMaxClasses, B, K, h, w, Hg, Wg);
  const int cap = sm_count_cached() * 8 / B;
  const int blocks = grid_for((long long)Hg * Wg, cap < 1 ? 1 : cap);
  eval2d_counts_kernel<<<dim3(blocks, B), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(pred, K, h, w, gt, Hg, Wg, counts);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
