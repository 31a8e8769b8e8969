// Token-grid resampling of the mince transformer (reference segtran_shared.py:45-66, resize_flat_features):
// linear / bilinear / trilinear interpolation with align_corners=False of token-major rows on a row-major 2-D or 3-D
// grid, over G groups (modes) of a channel window, all axes in one pass.
//
//   resize_tokens_fwd  y[b,g,o,c] = sum of the 2^3 trilinear taps of x[b,g,.,c]   (c < w; columns [w, w_pad) = 0)
//   resize_tokens_bwd  dx[b,g,i,c] = sum over the output cells o that read i of weight(o->i) dy[b,g,o,c]
//                      (gather form: fixed summation order, no atomics)
// A 2-D grid is a 3-D grid with a leading unit axis (ratio 1: the identity along it).
#include "sx_common.cuh"
#include "sx_resample.cuh"

namespace {

constexpr int WARPS = 8;         // one warp per row (b, g, cell); lanes stride over the channel window
constexpr int MAXJ = 64;         // output cells that read one input cell, per axis (the host bounds 1/ratio by 24)

struct Strides {
  long long bs, gs, ld;          // batch, group, row strides (elements)
};

__global__ void __launch_bounds__(WARPS * 32)
resize_tokens_fwd_kernel(const float* __restrict__ x, Strides si, float* __restrict__ y, Strides so, int G, int w,
                         int w_pad, sx_resample_grid g, long long rows, int rnd) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nout = g.lout[0] * g.lout[1] * g.lout[2];
  const unsigned t = (unsigned)row / (unsigned)nout, b = t / (unsigned)G, grp = t - b * (unsigned)G;   // 32-bit: host-checked
  const int cell = (int)((unsigned)row - t * (unsigned)nout);
  const long long ib = (long long)b * si.bs + (long long)grp * si.gs;
  const long long ob = (long long)b * so.bs + (long long)grp * so.gs;
  const int o2 = cell % g.lout[2], o1 = (cell / g.lout[2]) % g.lout[1], o0 = cell / (g.lout[2] * g.lout[1]);
  int a0, a1, b0, b1, c0, c1;
  float wa, wb, wc;
  sx::src_index(o0, g.ratio[0], g.lin[0], a0, a1, wa);
  sx::src_index(o1, g.ratio[1], g.lin[1], b0, b1, wb);
  sx::src_index(o2, g.ratio[2], g.lin[2], c0, c1, wc);
  const long long L1 = g.lin[1], L2 = g.lin[2];
  const float* x00 = x + ib + ((a0 * L1 + b0) * L2) * si.ld;
  const float* x01 = x + ib + ((a0 * L1 + b1) * L2) * si.ld;
  const float* x10 = x + ib + ((a1 * L1 + b0) * L2) * si.ld;
  const float* x11 = x + ib + ((a1 * L1 + b1) * L2) * si.ld;
  const long long e0 = c0 * si.ld, e1 = c1 * si.ld;
  float* yr = y + ob + (long long)cell * so.ld;
  for (int c = lane; c < w_pad; c += 32) {
    float v = 0.f;
    if (c < w) {
      // PyTorch's nesting: t0 * (h0 * (w0 x000 + w1 x001) + h1 * (...)) + t1 * (...)
      const float p00 = (1.f - wc) * __ldg(x00 + e0 + c) + wc * __ldg(x00 + e1 + c);
      const float p01 = (1.f - wc) * __ldg(x01 + e0 + c) + wc * __ldg(x01 + e1 + c);
      const float p10 = (1.f - wc) * __ldg(x10 + e0 + c) + wc * __ldg(x10 + e1 + c);
      const float p11 = (1.f - wc) * __ldg(x11 + e0 + c) + wc * __ldg(x11 + e1 + c);
      v = (1.f - wa) * ((1.f - wb) * p00 + wb * p01) + wa * ((1.f - wb) * p10 + wb * p11);
      if (rnd) v = sx::round_tf32(v);
    }
    yr[c] = v;
  }
}

// the output cells j of one axis that read input cell i with a nonzero weight, in ascending j: element offset j*step into
// so, weight into sw; -> count
__device__ __forceinline__ int axis_readers(int i, float ratio, int Lin, int Lout, int step, int lane, int* so, float* sw) {
  int jlo, jhi;
  sx::src_readers(i, __fdividef(1.f, ratio), Lin, Lout, jlo, jhi);    // approximate: the range has a one-cell margin
  int n = 0;
  for (int base = jlo; base <= jhi; base += 32) {
    const int j = base + lane;
    float wt = 0.f;
    if (j <= jhi) {
      int i0, i1;
      float w1;
      sx::src_index(j, ratio, Lin, i0, i1, w1);
      if (i0 == i) wt += 1.f - w1;
      if (i1 == i) wt += w1;
    }
    const unsigned nz = __ballot_sync(0xffffffffu, wt != 0.f);
    if (wt != 0.f) {
      const int k = n + __popc(nz & ((1u << lane) - 1u));
      if (k < MAXJ) { so[k] = j * step; sw[k] = wt; }
    }
    n += __popc(nz);
  }
  return n < MAXJ ? n : MAXJ;
}

__global__ void __launch_bounds__(WARPS * 32)
resize_tokens_bwd_kernel(const float* __restrict__ dy, Strides so, float* __restrict__ dx, Strides si, int G, int w,
                         int w_pad, sx_resample_grid g, long long rows, int accumulate) {
  __shared__ int sj[WARPS][3][MAXJ];           // element offsets into dy of the reading output cells, per axis
  __shared__ float sw[WARPS][3][MAXJ];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const long long row = (long long)blockIdx.x * WARPS + warp;
  if (row >= rows) return;                    // warp-uniform
  const int nin = g.lin[0] * g.lin[1] * g.lin[2];
  const unsigned t = (unsigned)row / (unsigned)nin, b = t / (unsigned)G, grp = t - b * (unsigned)G;   // 32-bit: host-checked
  const int cell = (int)((unsigned)row - t * (unsigned)nin);
  const long long ib = (long long)b * si.bs + (long long)grp * si.gs;
  const long long ob = (long long)b * so.bs + (long long)grp * so.gs;
  const int i2 = cell % g.lin[2], i1 = (cell / g.lin[2]) % g.lin[1], i0 = cell / (g.lin[2] * g.lin[1]);
  const int ld = (int)so.ld;                  // the host checks that every output offset fits in 32 bits
  const int n0 = axis_readers(i0, g.ratio[0], g.lin[0], g.lout[0], g.lout[1] * g.lout[2] * ld, lane, sj[warp][0], sw[warp][0]);
  const int n1 = axis_readers(i1, g.ratio[1], g.lin[1], g.lout[1], g.lout[2] * ld, lane, sj[warp][1], sw[warp][1]);
  const int n2 = axis_readers(i2, g.ratio[2], g.lin[2], g.lout[2], ld, lane, sj[warp][2], sw[warp][2]);
  __syncwarp();
  const float* dyb = dy + ob;
  float* dxr = dx + ib + (long long)cell * si.ld;
  for (int c = lane; c < w_pad; c += 32) {
    if (c >= w) {                             // padding columns: zero in write mode, untouched when accumulating
      if (!accumulate) dxr[c] = 0.f;
      continue;
    }
    float acc = 0.f;
    for (int ka = 0; ka < n0; ++ka) {
      const float wa = sw[warp][0][ka];
      for (int kb = 0; kb < n1; ++kb) {
        const float wab = wa * sw[warp][1][kb];
        const float* r = dyb + (sj[warp][0][ka] + sj[warp][1][kb] + c);
        for (int kc = 0; kc < n2; ++kc) acc = fmaf(wab * sw[warp][2][kc], __ldg(r + sj[warp][2][kc]), acc);
      }
    }
    dxr[c] = accumulate ? dxr[c] + acc : acc;
  }
}

}  // namespace

#define ST(s) reinterpret_cast<cudaStream_t>(s)

static int check_grid(const sx_resample_grid* g, const char* what) {
  SX_REQUIRE(g != nullptr, "%s: grid is NULL", what);
  for (int a = 0; a < 3; ++a) {
    SX_REQUIRE(g->lin[a] >= 1 && g->lout[a] >= 1, "%s: empty axis %d (%d -> %d)", what, a, g->lin[a], g->lout[a]);
    // every input cell is read by at most 2.5/ratio + 2 output cells per axis: keep that within MAXJ
    SX_REQUIRE(g->ratio[a] > 0.f && 1.f / g->ratio[a] <= 24.f, "%s: ratio %g of axis %d out of range (>= 1/24)", what,
               (double)g->ratio[a], a);
  }
  SX_REQUIRE((long long)g->lin[0] * g->lin[1] * g->lin[2] < (1ll << 31) &&
             (long long)g->lout[0] * g->lout[1] * g->lout[2] < (1ll << 31), "%s: grid too large", what);
  return 0;
}

extern "C" int sx_resize_tokens_fwd(const float* x, int64_t bs_in, int64_t gs_in, int64_t ld_in, float* y, int64_t bs_out,
                                    int64_t gs_out, int64_t ld_out, int32_t B, int32_t G, int32_t w, int32_t w_pad,
                                    const sx_resample_grid* grid, int32_t round_tf32, void* stream) {
  if (int rc = check_grid(grid, "sx_resize_tokens_fwd")) return rc;
  SX_REQUIRE(B >= 1 && G >= 1 && w >= 1 && w_pad >= w, "sx_resize_tokens_fwd: bad sizes B=%d G=%d w=%d w_pad=%d", B, G, w,
             w_pad);
  const long long rows = (long long)B * G * grid->lout[0] * grid->lout[1] * grid->lout[2];
  SX_REQUIRE(rows < (1ll << 31), "sx_resize_tokens_fwd: %lld rows", rows);
  resize_tokens_fwd_kernel<<<(unsigned)((rows + WARPS - 1) / WARPS), WARPS * 32, 0, ST(stream)>>>(
      x, Strides{bs_in, gs_in, ld_in}, y, Strides{bs_out, gs_out, ld_out}, G, w, w_pad, *grid, rows, round_tf32);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_resize_tokens_bwd(const float* dy, int64_t bs_out, int64_t gs_out, int64_t ld_out, float* dx,
                                    int64_t bs_in, int64_t gs_in, int64_t ld_in, int32_t B, int32_t G, int32_t w,
                                    int32_t w_pad, const sx_resample_grid* grid, int32_t accumulate, void* stream) {
  if (int rc = check_grid(grid, "sx_resize_tokens_bwd")) return rc;
  SX_REQUIRE(B >= 1 && G >= 1 && w >= 1 && w_pad >= w, "sx_resize_tokens_bwd: bad sizes B=%d G=%d w=%d w_pad=%d", B, G, w,
             w_pad);
  const long long rows = (long long)B * G * grid->lin[0] * grid->lin[1] * grid->lin[2];
  SX_REQUIRE(rows < (1ll << 31), "sx_resize_tokens_bwd: %lld rows", rows);
  SX_REQUIRE((long long)grid->lout[0] * grid->lout[1] * grid->lout[2] * ld_out < (1ll << 31),
             "sx_resize_tokens_bwd: dy group too large for 32-bit offsets");
  resize_tokens_bwd_kernel<<<(unsigned)((rows + WARPS - 1) / WARPS), WARPS * 32, 0, ST(stream)>>>(
      dy, Strides{bs_out, gs_out, ld_out}, dx, Strides{bs_in, gs_in, ld_in}, G, w, w_pad, *grid, rows, accumulate);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
