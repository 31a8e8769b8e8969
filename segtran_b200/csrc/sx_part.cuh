// Deterministic cross-CTA sums.  A kernel whose CTAs each hold partial sums stores them in its slot (= CTA index along
// the reduced dimension) of the caller's scratch `part`, laid out [slot][stride]; part_reduce then adds the slots in slot
// order into the destinations.  Float atomics would add them in whatever order the CTAs finish, and the last-bit
// differences grow through TF32 rounding and the optimiser: two runs of the same step on the same inputs would not
// agree.  The number of slots adapts to the scratch size (part_floats / stride).
#pragma once
#include <algorithm>

#include "sx_common.cuh"

namespace {

struct PartDst {                                                 // slot row = concatenation of up to 4 destination arrays
  float* p[4];
  int n[4];
};

__global__ void part_reduce_kernel(const float* __restrict__ part, int slots, int stride, int total, PartDst d) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    int a = 0, c = i;
    while (c >= d.n[a]) { c -= d.n[a]; ++a; }
    float s = 0.f;
    for (int g = 0; g < slots; ++g) s += part[(long long)g * stride + i];
    if (d.p[a]) d.p[a][c] += s;
  }
}

// dst arrays += the sum of `slots` slot rows of part (row pitch `stride` >= the summed array lengths), in slot order
inline int part_reduce(const float* part, int slots, int stride, PartDst d, cudaStream_t st) {
  const int total = d.n[0] + d.n[1] + d.n[2] + d.n[3];
  part_reduce_kernel<<<sx_ceil_div(total, 256), 256, 0, st>>>(part, slots, stride, total, d);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

// most slots of pitch `stride` that fit a scratch of part_floats floats
inline int part_slots(int64_t part_floats, long long stride) { return (int)std::min<long long>(part_floats / stride, 1 << 30); }

}  // namespace
