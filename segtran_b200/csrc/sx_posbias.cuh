// Sliding-window positional biases (SlidingPosBiases2D/3D, segtran_shared.py:1002-1175): the one place where device
// code turns an sx_posbias descriptor into bias(q,k).  Tokens are the cells of a row-major grid; a 2-D grid is handled
// as a 3-D grid with a leading extent of 1 and a zero table stride along it, so every kernel runs one 3-D code path.
#pragma once
#include "sx_common.cuh"

namespace sxpb {

struct Geom {
  int g[3];        // grid extents (leading 1 for pd == 2)
  int ts[3];       // table strides ((2R+1)^2, 2R+1, 1), ts[0] = 0 for pd == 2
  int R, T;        // radius, table size (2R+1)^pd
  float w;
};

inline Geom make_geom(const sx_posbias& pb) {
  Geom G{};
  const int W = 2 * pb.R + 1;
  if (pb.pd == 2) {
    G.g[0] = 1; G.g[1] = pb.grid[0]; G.g[2] = pb.grid[1];
    G.ts[0] = 0; G.ts[1] = W; G.ts[2] = 1;
    G.T = W * W;
  } else {
    G.g[0] = pb.grid[0]; G.g[1] = pb.grid[1]; G.g[2] = pb.grid[2];
    G.ts[0] = W * W; G.ts[1] = W; G.ts[2] = 1;
    G.T = W * W * W;
  }
  G.R = pb.R;
  G.w = pb.w;
  return G;
}

// host-side validation shared by the entry points; returns an error message or nullptr
inline const char* check(const sx_posbias* pb, long long ntok) {
  if (!pb || !pb->table) return "posbias: null table";
  if (pb->pd != 2 && pb->pd != 3) return "posbias: pd must be 2 or 3";
  if (pb->R < 1 || pb->R > 16) return "posbias: R must be in 1..16";
  long long n = 1;
  for (int i = 0; i < pb->pd; ++i) {
    if (pb->grid[i] < 1) return "posbias: bad grid";
    n *= pb->grid[i];
  }
  if (n != ntok) return "posbias: the grid's cell count differs from the number of tokens";
  return nullptr;
}

// row-major cell index -> coordinates
__device__ __forceinline__ void coords(const Geom& G, int t, int (&c)[3]) {
  c[2] = t % G.g[2]; t /= G.g[2];
  c[1] = t % G.g[1];
  c[0] = t / G.g[1];
}

// advance coordinates by d >= 0 cells in row-major order (no division: d is small next to a row of the grid)
__device__ __forceinline__ void step(const Geom& G, int (&c)[3], int d) {
  c[2] += d;
  while (c[2] >= G.g[2]) {
    c[2] -= G.g[2];
    if (++c[1] >= G.g[1]) { c[1] = 0; ++c[0]; }
  }
}

// bias(q,k) as a table offset: -1 when k lies outside q's window
__device__ __forceinline__ int offset(const Geom& G, const int (&q)[3], const int (&k)[3]) {
  int o = 0;
  bool in = true;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int r = k[i] - q[i] + G.R;
    in = in && (unsigned)r <= (unsigned)(2 * G.R);
    o += r * G.ts[i];
  }
  return in ? o : -1;
}

// the inverse map: the key cell that table offset o addresses for query q, or -1 when it falls off the grid
__device__ __forceinline__ int key_of(const Geom& G, const int (&q)[3], int o) {
  const int W = 2 * G.R + 1;
  int r[3];
  r[2] = o % W; o /= W;
  r[1] = o % W;
  r[0] = o / W;                                    // 0 for pd == 2
  int k = 0;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const int c = q[i] + r[i] - (G.ts[i] ? G.R : 0);
    if ((unsigned)c >= (unsigned)G.g[i]) return -1;
    k = k * G.g[i] + c;
  }
  return k;
}

}  // namespace sxpb
