// Sliding-window inference post-process (SURVEY.md §8 f.4; reference code/test_util3d.py:93-184 test_single_case and
// code/dataloaders/datasets3d.py:43-61 make_brats_pred_consistent): the per-patch "sigmoid -> accumulate -> count" update
// and the final "average -> BraTS consistency -> threshold / arg-max" as two HBM-bound kernels on the class-score volumes.
// Mirror test-time augmentation: a window-gather kernel writes a batch of mirrored windows straight from the padded image,
// and the accumulate kernel reads a variant's scores through reversed indices, so no flipped map is ever written.
// Mirror masks: bit 0 reverses H (dx), bit 1 W (dy), bit 2 D (dz).
// Window weighting (Gaussian blending): an accumulate given per-axis weight tables (sx_sw_weights) adds w * sigmoid and w
// instead of sigmoid and 1; the 2-D accumulate of sx_eval2d.cu takes the same tables.
#include "sx_common.cuh"

namespace {

constexpr int kGatherWindows = 64;     // window origins passed by value per gather launch

struct WindowOrigins {
  int o[kGatherWindows][3];
};

// preds[k][x0+i][y0+j][z0+l] += sigmoid(flip_m(scores)[k][i][j][l]);  cnt[x0+i][y0+j][z0+l] += 1   (test_util3d.py:155-159)
// kWeighted: both terms are scaled by w = max(wx[i] * wy[j] * wz[l], 1e-3), the window weight at the accumulator position
// (i, j, l); the weight tables are the trailing arguments, which the unweighted instantiation never reads.
template <bool kWeighted>
__global__ void sw_accumulate_kernel(const float* __restrict__ scores, int K, int dx, int dy, int dz, float* __restrict__ preds,
                                     float* __restrict__ cnt, int H, int W, int D, int x0, int y0, int z0, int mirror,
                                     const float* __restrict__ wx, const float* __restrict__ wy, const float* __restrict__ wz) {
  const long long pv = (long long)dx * dy * dz;
  const long long V = (long long)H * W * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pv; i += (long long)gridDim.x * blockDim.x) {
    const int l = (int)(i % dz);
    const int j = (int)((i / dz) % dy);
    const int ii = (int)(i / ((long long)dz * dy));
    const long long o = ((long long)(x0 + ii) * W + (y0 + j)) * D + (z0 + l);
    const long long si = mirror == 0 ? i
                                     : ((long long)((mirror & 1) ? dx - 1 - ii : ii) * dy + ((mirror & 2) ? dy - 1 - j : j)) * dz +
                                           ((mirror & 4) ? dz - 1 - l : l);
    if constexpr (kWeighted) {
      const float w = fmaxf(__ldg(wx + ii) * __ldg(wy + j) * __ldg(wz + l), kSwMinWeight);
      for (int k = 0; k < K; ++k) {
        const float s = scores[k * pv + si];
        preds[k * V + o] += __fmul_rn(w, 1.f / (1.f + expf(-s)));   // rounded product, then the add: no FMA contraction
      }
      cnt[o] += w;
    } else {
      for (int k = 0; k < K; ++k) {
        const float s = scores[k * pv + si];
        preds[k * V + o] += 1.f / (1.f + expf(-s));          // torch.sigmoid
      }
      cnt[o] += 1.f;
    }
  }
}

// preds /= cnt; mode 1 (BraTS): WT = max(ET, WT, TC), TC = max(ET, TC) (classes 1: ET, 2: WT, 3: TC; not conservative),
// hard[k>=1] = preds >= 0.5, hard[0] = no class fired; mode 0: hard[0] = argmax_k preds (written as float class index)
__global__ void sw_finalize_kernel(float* __restrict__ preds, const float* __restrict__ cnt, int K, long long V, int mode,
                                   float* __restrict__ hard) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (long long)gridDim.x * blockDim.x) {
    const float c = cnt[i];
    if (mode == 1) {
      float pr[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) pr[k] = preds[k * V + i] / c;
      const float wt = fmaxf(pr[1], fmaxf(pr[2], pr[3]));     // preds_soft2[2] = max(preds_soft[1:])
      const float tc = fmaxf(pr[1], pr[3]);                   // preds_soft2[3] = max(preds_soft[[1,3]])
      pr[2] = wt;
      pr[3] = tc;
      float any = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) preds[k * V + i] = pr[k];
#pragma unroll
      for (int k = 1; k < 4; ++k) {
        const float hk = pr[k] >= 0.5f ? 1.f : 0.f;
        hard[k * V + i] = hk;
        any += hk;
      }
      hard[i] = any == 0.f ? 1.f : 0.f;
    } else {
      float best = -3.0e38f;
      int arg = 0;
      for (int k = 0; k < K; ++k) {
        const float v = preds[k * V + i] / c;
        preds[k * V + i] = v;
        if (v > best) { best = v; arg = k; }                  // first maximum, like torch.argmax
      }
      hard[i] = (float)arg;
    }
  }
}

// out[w][b][c][i][j][l] = img[b][c][x0_w + i'][y0_w + j'][z0_w + l'], with i' = dx-1-i where bit 0 of mirror is set (j', l'
// likewise for bits 1 and 2): window w of image b, mirrored, in the layout torch.flip(torch.stack(windows)) would have.
__global__ void sw_gather_kernel(const float* __restrict__ img, int B, int C, int H, int W, int D, WindowOrigins org, int n,
                                 int dx, int dy, int dz, int mirror, float* __restrict__ out) {
  const long long pv = (long long)dx * dy * dz;
  const long long total = (long long)n * B * C * pv;
  const long long bc_n = (long long)B * C;
  for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const long long q = t / pv;
    const long long r = t - q * pv;
    const int l = (int)(r % dz);
    const int j = (int)((r / dz) % dy);
    const int ii = (int)(r / ((long long)dz * dy));
    const int w = (int)(q / bc_n);
    const long long bc = q - (long long)w * bc_n;
    const int si = org.o[w][0] + ((mirror & 1) ? dx - 1 - ii : ii);
    const int sj = org.o[w][1] + ((mirror & 2) ? dy - 1 - j : j);
    const int sl = org.o[w][2] + ((mirror & 4) ? dz - 1 - l : l);
    out[t] = __ldg(img + ((bc * H + si) * W + sj) * D + sl);
  }
}

}  // namespace

extern "C" int sx_sw_accumulate(const float* scores, int32_t K, int32_t dx, int32_t dy, int32_t dz, float* preds, float* cnt,
                                int32_t H, int32_t W, int32_t D, int32_t x0, int32_t y0, int32_t z0, int32_t mirror,
                                const sx_sw_weights* wt, void* stream) {
  SX_REQUIRE(K > 0 && dx > 0 && dy > 0 && dz > 0 && x0 >= 0 && y0 >= 0 && z0 >= 0 && x0 + dx <= H && y0 + dy <= W && z0 + dz <= D,
             "sx_sw_accumulate: window [%d+%d, %d+%d, %d+%d] outside the %dx%dx%d volume", x0, dx, y0, dy, z0, dz, H, W, D);
  SX_REQUIRE(mirror >= 0 && mirror <= 7, "sx_sw_accumulate: mirror mask %d is not a subset of {H, W, D} (0..7)", mirror);
  SX_REQUIRE(!wt || (wt->wx && wt->wy && wt->nx > 0 && wt->ny > 0 && wt->nz > 0),
             "sx_sw_accumulate: empty or missing table (wx=%p nx=%d, wy=%p ny=%d, wz=%p nz=%d)", (const void*)wt->wx,
             wt->nx, (const void*)wt->wy, wt->ny, (const void*)wt->wz, wt->nz);
  SX_REQUIRE(!wt || (wt->wz && wt->nx == dx && wt->ny == dy && wt->nz == dz),
             "sx_sw_accumulate: window weight tables of %dx%dx%d (z table %s) for a %dx%dx%d window", wt->nx, wt->ny,
             wt->nz, wt->wz ? "given" : "missing", dx, dy, dz);
  const long long pv = (long long)dx * dy * dz;
  long long blocks = (pv + 255) / 256;
  if (blocks > sm_count_cached() * 8) blocks = sm_count_cached() * 8;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (wt)
    sw_accumulate_kernel<true><<<(int)blocks, 256, 0, st>>>(scores, K, dx, dy, dz, preds, cnt, H, W, D, x0, y0, z0, mirror,
                                                            wt->wx, wt->wy, wt->wz);
  else
    sw_accumulate_kernel<false><<<(int)blocks, 256, 0, st>>>(scores, K, dx, dy, dz, preds, cnt, H, W, D, x0, y0, z0, mirror,
                                                             nullptr, nullptr, nullptr);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_sw_finalize(float* preds, const float* cnt, int32_t K, int64_t V, int32_t brats, float* hard, void* stream) {
  SX_REQUIRE(K > 0 && V > 0 && (!brats || K == 4), "sx_sw_finalize: the BraTS consistency rule needs 4 classes (got %d)", K);
  long long blocks = (V + 255) / 256;
  if (blocks > sm_count_cached() * 8) blocks = sm_count_cached() * 8;
  sw_finalize_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(preds, cnt, K, V, brats ? 1 : 0, hard);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_sw_gather(const float* img, int32_t B, int32_t C, int32_t H, int32_t W, int32_t D, const int32_t* origins,
                            int32_t n, int32_t dx, int32_t dy, int32_t dz, int32_t mirror, float* out, void* stream) {
  SX_REQUIRE(B > 0 && C > 0 && H > 0 && W > 0 && D > 0 && n > 0 && origins && dx > 0 && dy > 0 && dz > 0,
             "sx_sw_gather: empty image (%dx%dx%dx%dx%d), window (%dx%dx%d) or window list (%d)", B, C, H, W, D, dx, dy, dz, n);
  SX_REQUIRE(mirror >= 0 && mirror <= 7, "sx_sw_gather: mirror mask %d is not a subset of {H, W, D} (0..7)", mirror);
  for (int w = 0; w < n; ++w) {
    const int x0 = origins[3 * w], y0 = origins[3 * w + 1], z0 = origins[3 * w + 2];
    SX_REQUIRE(x0 >= 0 && y0 >= 0 && z0 >= 0 && x0 + dx <= H && y0 + dy <= W && z0 + dz <= D,
               "sx_sw_gather: window %d [%d+%d, %d+%d, %d+%d] outside the %dx%dx%d image", w, x0, dx, y0, dy, z0, dz, H, W, D);
  }
  const long long per_window = (long long)B * C * dx * dy * dz;
  for (int w0 = 0; w0 < n; w0 += kGatherWindows) {       // origins go by value, kGatherWindows per launch
    const int m = n - w0 < kGatherWindows ? n - w0 : kGatherWindows;
    WindowOrigins org{};
    for (int w = 0; w < m; ++w)
      for (int a = 0; a < 3; ++a) org.o[w][a] = origins[3 * (w0 + w) + a];
    long long blocks = (m * per_window + 255) / 256;
    if (blocks > sm_count_cached() * 8) blocks = sm_count_cached() * 8;
    sw_gather_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(img, B, C, H, W, D, org, m, dx, dy, dz,
                                                                                       mirror, out + w0 * per_window);
    SX_CHECK_CUDA(cudaGetLastError());
  }
  return 0;
}
