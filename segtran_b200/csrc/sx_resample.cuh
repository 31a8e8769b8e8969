// Source-index rule of PyTorch's linear interpolation with align_corners=False (area_pixel_compute_source_index),
// shared by the per-axis resize kernels (sx_head.cu) and the token-grid resampling (sx_resample.cu).
//   ratio: source cells per output cell.  F.interpolate uses Lin/Lout when a size is given and 1/scale_factor when a
//   scale factor is given (so a 7-cell axis downsampled by scale_factor=1/2 reads 3 cells at stride 2.0, not 2.33).
#pragma once

namespace sx {

// output cell j reads input cells i0 and i1 with weights 1-w1 and w1
__device__ __forceinline__ void src_index(int j, float ratio, int Lin, int& i0, int& i1, float& w1) {
  float s = ((float)j + 0.5f) * ratio - 0.5f;
  if (s < 0.f) s = 0.f;
  i0 = (int)s;
  if (i0 > Lin - 1) i0 = Lin - 1;
  i1 = i0 + ((i0 < Lin - 1) ? 1 : 0);
  w1 = s - (float)i0;
}

// a range [jlo, jhi] of output cells that contains every output cell reading input cell i (inv = 1/ratio)
__device__ __forceinline__ void src_readers(int i, float inv, int Lin, int Lout, int& jlo, int& jhi) {
  jlo = (int)floorf(((float)i - 0.5f) * inv - 0.5f) - 1;
  jhi = (int)ceilf(((float)i + 1.5f) * inv - 0.5f) + 1;
  if (i == 0) jlo = 0;                       // clamped sources (s < 0) map to i = 0
  if (i == Lin - 1) jhi = Lout - 1;
  if (jlo < 0) jlo = 0;
  if (jhi > Lout - 1) jhi = Lout - 1;
}

}  // namespace sx
