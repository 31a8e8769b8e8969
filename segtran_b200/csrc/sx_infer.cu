// Sliding-window inference post-process (SURVEY.md §8 f.4; reference code/test_util3d.py:93-184 test_single_case and
// code/dataloaders/datasets3d.py:43-61 make_brats_pred_consistent): the per-patch "sigmoid -> accumulate -> count" update
// and the final "average -> BraTS consistency -> threshold / arg-max" as two HBM-bound kernels on the class-score volumes.
#include "sx_common.cuh"

namespace {

// preds[k][x0+i][y0+j][z0+l] += sigmoid(scores[k][i][j][l]);  cnt[x0+i][y0+j][z0+l] += 1      (test_util3d.py:155-159)
__global__ void sw_accumulate_kernel(const float* __restrict__ scores, int K, int dx, int dy, int dz, float* __restrict__ preds,
                                     float* __restrict__ cnt, int H, int W, int D, int x0, int y0, int z0) {
  const long long pv = (long long)dx * dy * dz;
  const long long V = (long long)H * W * D;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < pv; i += (long long)gridDim.x * blockDim.x) {
    const int l = (int)(i % dz);
    const int j = (int)((i / dz) % dy);
    const int ii = (int)(i / ((long long)dz * dy));
    const long long o = ((long long)(x0 + ii) * W + (y0 + j)) * D + (z0 + l);
    for (int k = 0; k < K; ++k) {
      const float s = scores[k * pv + i];
      preds[k * V + o] += 1.f / (1.f + expf(-s));          // torch.sigmoid
    }
    cnt[o] += 1.f;
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

}  // namespace

extern "C" int sx_sw_accumulate(const float* scores, int32_t K, int32_t dx, int32_t dy, int32_t dz, float* preds, float* cnt,
                                int32_t H, int32_t W, int32_t D, int32_t x0, int32_t y0, int32_t z0, void* stream) {
  SX_REQUIRE(K > 0 && dx > 0 && dy > 0 && dz > 0 && x0 >= 0 && y0 >= 0 && z0 >= 0 && x0 + dx <= H && y0 + dy <= W && z0 + dz <= D,
             "sx_sw_accumulate: window [%d+%d, %d+%d, %d+%d] outside the %dx%dx%d volume", x0, dx, y0, dy, z0, dz, H, W, D);
  const long long pv = (long long)dx * dy * dz;
  long long blocks = (pv + 255) / 256;
  if (blocks > sm_count_cached() * 8) blocks = sm_count_cached() * 8;
  sw_accumulate_kernel<<<(int)blocks, 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(scores, K, dx, dy, dz, preds, cnt, H, W, D,
                                                                                         x0, y0, z0);
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
