// Per-element term of the attention-consistency loss, shared by the pair (wgmma) and the dense (row) kernels of
// sx_consist.cu, so both compute every element with the same arithmetic.
//
//   c    = min(max(sum_k F[k,i] F[k,j], 0), 1)        the class-consistency target of tokens i and j
//   BCE    (train3d.py:426-449): loss term max(x,0) - x c + log1p(exp(-|x|)),  residual sigmoid(x) - c
//   MARGIN (train2d.py:668-723): x is inconsistent when (x < mu && c != 0) || (x > mu - 0.1 && c == 0); over those
//            elements the loss term is |x - mu|, the residual sign(x - mu); every other element contributes nothing.
#pragma once
#include "sx_common.cuh"

namespace sxcs {

constexpr int MAX_K = 16;

struct Acc {            // one thread's partial sums over the elements it visited (of one batch)
  float sum = 0.f;      // BCE: sum of the loss terms; MARGIN: sum of |x - mu| over the inconsistent elements
  float sgn = 0.f;      // MARGIN: sum of sign(x - mu) over the inconsistent elements
  int cnt = 0;          // MARGIN: number of inconsistent elements
};

// c from the K mask channels of token i (fi, stride si) and token j (fj, stride sj), summed in k order
__device__ __forceinline__ float target(const float* fi, int si, const float* fj, int sj, int K) {
  float c = 0.f;
  for (int k = 0; k < K; ++k) c = fmaf(fi[k * si], fj[k * sj], c);
  return fminf(fmaxf(c, 0.f), 1.f);
}

// adds the element's loss term to `a` and returns its (unscaled) residual
__device__ __forceinline__ float term(int variant, float x, float c, float mu, Acc& a) {
  if (variant == SX_CONSIST_BCE) {
    const float e = expf(-fabsf(x));
    a.sum += fmaxf(x, 0.f) - x * c + log1pf(e);
    return (x >= 0.f ? 1.f : e) / (1.f + e) - c;            // sigmoid(x) from the same exponential

  }
  const bool inc = c != 0.f ? (x < mu) : (x > mu - 0.1f);
  if (!inc) return 0.f;
  const float d = x - mu;
  const float s = d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f);
  a.sum += fabsf(d);
  a.sgn += s;
  a.cnt += 1;
  return s;
}

}  // namespace sxcs
