// Evaluation metrics of a segmented case (reference code/test_util3d.py:186-215 calculate_metric_percase and the medpy
// 0.4 functions it calls: dc, jc, asd, and hd / hd95): overlap counts, surface maps, an exact integer squared Euclidean
// distance transform, a histogram of the squared surface distances and the statistics read from it.
//
// Every distance with unit spacing is the square root of an integer squared distance d2 <= sum_i (n_i - 1)^2, so a
// histogram over d2 holds everything the metrics need, exactly: the maximum is the largest non-empty bin, a percentile is
// two order statistics found by a prefix scan over the bins, the mean is sum_k count_k sqrt(k) / n.  Nothing is sorted,
// and the only atomics are integer ones (order-free, so every run gives the same bits).
//
// Layout: the classes of a case go through every launch together, as the leading index of [K][n0][n1][n2] uint8 masks
// (n2 contiguous).  A 2-D mask passes n0 = 1 and ndim = 2, which only changes the erosion footprint (sx_surface): the
// distance transform does not care, an axis of extent 1 adds nothing to a distance.
#include <climits>

#include "sx_common.cuh"

namespace {

constexpr int kEdtInf = 1 << 28;             // "no border voxel": with d2 <= 3 * 4095^2 < 2^26, kEdtInf + q^2 and the
                                             // differences of two such terms stay far inside int32
constexpr int kMaxExtent = 4096;
constexpr long long kMaxD2 = 1ll << 26;

// |A|, |B|, |A and B|, |A or B| of each class (operands non-zero = true); counts [K] rows of pitch ldc, zeroed by the host
__global__ void mask_counts_kernel(const uint8_t* __restrict__ A, const uint8_t* __restrict__ B, long long V,
                                   unsigned long long* __restrict__ counts, long long ldc) {
  const int k = blockIdx.y;
  const uint8_t* a = A + (long long)k * V;
  const uint8_t* b = B + (long long)k * V;
  uint32_t na = 0, nb = 0, ni = 0, nu = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (long long)gridDim.x * blockDim.x) {
    const uint32_t x = a[i] != 0, y = b[i] != 0;
    na += x;
    nb += y;
    ni += x & y;
    nu += x | y;
  }
  na = __reduce_add_sync(0xffffffffu, na);
  nb = __reduce_add_sync(0xffffffffu, nb);
  ni = __reduce_add_sync(0xffffffffu, ni);
  nu = __reduce_add_sync(0xffffffffu, nu);
  if ((threadIdx.x & 31) == 0) {
    unsigned long long* c = counts + k * ldc;
    if (na) atomicAdd(c + 0, (unsigned long long)na);
    if (nb) atomicAdd(c + 1, (unsigned long long)nb);
    if (ni) atomicAdd(c + 2, (unsigned long long)ni);
    if (nu) atomicAdd(c + 3, (unsigned long long)nu);
  }
}

// border = X and not erode(X): a foreground voxel is a border voxel when one of its 2*ndim axis neighbours is background
// or lies outside the volume (scipy.ndimage.binary_erosion with the connectivity-1 cross and border_value = 0)
__global__ void surface_kernel(const uint8_t* __restrict__ X, long long total, int ndim, int n0, int n1, int n2,
                               uint8_t* __restrict__ border) {
  const long long s1 = n2, s0 = (long long)n1 * n2;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    uint8_t out = 0;
    if (X[i] != 0) {
      const int i2 = (int)(i % n2);
      const int i1 = (int)((i / n2) % n1);
      bool edge = i2 == 0 || i2 == n2 - 1 || X[i - 1] == 0 || X[i + 1] == 0 ||
                  i1 == 0 || i1 == n1 - 1 || X[i - s1] == 0 || X[i + s1] == 0;
      if (!edge && ndim == 3) {
        const int i0 = (int)((i / s0) % n0);
        edge = i0 == 0 || i0 == n0 - 1 || X[i - s0] == 0 || X[i + s0] == 0;
      }
      out = edge ? 1 : 0;
    }
    border[i] = out;
  }
}

// First axis: per line, the two-sweep 1-D distance to the nearest border voxel, squared (kEdtInf when the line has none).
// Line l starts at (l / inner) * n * inner + l % inner and has stride inner: neighbouring threads read neighbouring bytes.
__global__ void edt_sweep_kernel(const uint8_t* __restrict__ border, int* __restrict__ dist, long long lines, int n,
                                 long long inner) {
  const long long l = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= lines) return;
  const long long base = (l / inner) * n * inner + l % inner;
  int g = n + 1;                                          // n + 1: "none seen yet", any real distance is < n
  for (int i = 0; i < n; ++i) {
    const long long o = base + i * inner;
    g = border[o] ? 0 : min(g + 1, n + 1);
    dist[o] = g;
  }
  g = n + 1;
  for (int i = n - 1; i >= 0; --i) {
    const long long o = base + i * inner;
    g = border[o] ? 0 : min(g + 1, n + 1);
    const int d = min(dist[o], g);
    dist[o] = d > n ? kEdtInf : d * d;
  }
}

__device__ __forceinline__ int floor_div(int a, int b) {   // b > 0
  const int q = a / b;
  return (a % b != 0 && a < 0) ? q - 1 : q;
}

// Every further axis: d[p] = min_q f[q] + (p - q)^2 by the lower envelope of the parabolas (Felzenszwalb &
// Huttenlocher), in integers: parabola q beats parabola p < q exactly at the integers x > floor(sep(p, q)).  A block
// takes T consecutive lines; their values are staged in shared memory as [n][T + 1] (the pad spreads the column walk of
// the tile load over the banks), the envelope's vertex list too; the intersections are recomputed from them instead of
// being stored.  CONTIG (the contiguous axis): T lines are one contiguous run of memory, loaded and stored through the
// tile; otherwise each thread's line has stride inner and the threads of a warp read and write neighbouring words.
template <bool CONTIG>
__global__ void edt_envelope_kernel(int* __restrict__ dist, long long lines, int n, long long inner) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int T = blockDim.x, P = T + 1, t = threadIdx.x;
  int* f = reinterpret_cast<int*>(smem);
  int* o = f + (long long)n * P;                                     // CONTIG only
  uint16_t* v = reinterpret_cast<uint16_t*>(f + (long long)n * P * (CONTIG ? 2 : 1));
  const long long l0 = (long long)blockIdx.x * T;
  const int nl = (int)min((long long)T, lines - l0);
  const long long base = CONTIG ? l0 * n : ((l0 + t) / inner) * n * inner + (l0 + t) % inner;
  if (CONTIG) {
    for (int j = t; j < nl * n; j += T) f[(j % n) * P + j / n] = dist[base + j];
    __syncthreads();
  } else if (t < nl) {
    for (int i = 0; i < n; ++i) f[i * P + t] = dist[base + i * inner];
  }
  if (t < nl) {
    auto F = [&](int i) { return f[i * P + t]; };
    auto sep = [&](int p, int q) { return floor_div((F(q) + q * q) - (F(p) + p * p), 2 * (q - p)); };
    int k = 0, ztop = INT_MIN;                                       // ztop: left end of the top parabola's range
    v[t] = 0;
    for (int q = 1; q < n; ++q) {
      int s = sep(v[k * P + t], q);
      while (k > 0 && s <= ztop) {
        --k;
        ztop = k > 0 ? sep(v[(k - 1) * P + t], v[k * P + t]) : INT_MIN;
        s = sep(v[k * P + t], q);
      }
      ++k;
      v[k * P + t] = (uint16_t)q;
      ztop = s;
    }
    const int m = k;
    k = 0;
    int vk = v[t];
    int znext = m > 0 ? sep(vk, v[P + t]) : INT_MAX;
    for (int p = 0; p < n; ++p) {
      while (znext < p) {
        ++k;
        vk = v[k * P + t];
        znext = k < m ? sep(vk, v[(k + 1) * P + t]) : INT_MAX;
      }
      const int d = min((p - vk) * (p - vk) + F(vk), kEdtInf);
      if (CONTIG)
        o[p * P + t] = d;
      else
        dist[base + p * inner] = d;
    }
  }
  if (CONTIG) {
    __syncthreads();
    for (int j = t; j < nl * n; j += T) dist[base + j] = o[(j % n) * P + j / n];
  }
}

// hist[k][d2] += 1 at every border voxel of the source mask (hist rows of pitch ldh, zeroed by the host); values outside
// the bin range (the sentinel of a class whose other mask has no border) are skipped
__global__ void surface_hist_kernel(const uint8_t* __restrict__ src, const int* __restrict__ dist, long long V,
                                    long long total, int nbins, uint32_t* __restrict__ hist, long long ldh) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    if (src[i]) {
      const int d = dist[i];
      if ((unsigned)d < (unsigned)nbins) atomicAdd(hist + (i / V) * ldh + d, 1u);
    }
  }
}

// One CTA per class.  Thread t owns bins [t*chunk, (t+1)*chunk) of both directions' histograms; its partial sums are
// added by a fixed tree, so the fp64 sum has one order.  out[k*ldo + ...]:
//   0, 1: n of direction 0 / 1        2, 3: mean distance (asd) of direction 0 / 1 (0 when n = 0)
//   4, 5: max distance of direction 0 / 1        6: numpy's linear 95th percentile over both directions together
//   7: n of both directions
constexpr int kStatsThreads = 512;
__global__ void __launch_bounds__(kStatsThreads) surface_stats_kernel(const uint32_t* __restrict__ hist, int nbins,
                                                                      long long ldh, double* __restrict__ out, long long ldo) {
  __shared__ unsigned long long sn[2][kStatsThreads], scan[kStatsThreads];
  __shared__ double ss[2][kStatsThreads];
  __shared__ int sm[2][kStatsThreads];
  __shared__ double sval[2];
  const int k = blockIdx.x, t = threadIdx.x;
  const uint32_t* h[2] = {hist + k * ldh, hist + k * ldh + nbins};
  const int chunk = (nbins + kStatsThreads - 1) / kStatsThreads;
  const int lo = min(t * chunk, nbins), hi = min(lo + chunk, nbins);
  for (int d = 0; d < 2; ++d) {
    unsigned long long n = 0;
    double s = 0.0;
    int mx = -1;
    for (int b = lo; b < hi; ++b) {
      const uint32_t c = h[d][b];
      if (c) {
        n += c;
        s = __dadd_rn(s, __dmul_rn((double)c, sqrt((double)b)));
        mx = b;
      }
    }
    sn[d][t] = n;
    ss[d][t] = s;
    sm[d][t] = mx;
  }
  scan[t] = sn[0][t] + sn[1][t];
  __syncthreads();
  // inclusive scan of the per-thread counts (Hillis-Steele), then the tree sums
  for (int off = 1; off < kStatsThreads; off <<= 1) {
    const unsigned long long add = t >= off ? scan[t - off] : 0ull;
    __syncthreads();
    scan[t] += add;
    __syncthreads();
  }
  for (int half = kStatsThreads / 2; half > 0; half >>= 1) {
    if (t < half) {
      for (int d = 0; d < 2; ++d) {
        sn[d][t] += sn[d][t + half];
        ss[d][t] = __dadd_rn(ss[d][t], ss[d][t + half]);
        sm[d][t] = max(sm[d][t], sm[d][t + half]);
      }
    }
    __syncthreads();
  }
  const unsigned long long N = sn[0][0] + sn[1][0];
  // np.percentile(..., 95), method 'linear': vi = (N-1)*0.95, a = s[floor(vi)], b = s[min(floor(vi)+1, N-1)]
  double g = 0.0;
  if (N > 0) {
    const double vi = __dmul_rn((double)(N - 1), 0.95);
    const unsigned long long r0 = (unsigned long long)floor(vi);
    g = __dsub_rn(vi, (double)r0);
    const unsigned long long r[2] = {r0, min(r0 + 1, N - 1)};
    const unsigned long long incl = scan[t], excl = t ? scan[t - 1] : 0ull;
    for (int j = 0; j < 2; ++j) {
      if (r[j] >= excl && r[j] < incl) {
        unsigned long long c = excl;
        for (int b = lo; b < hi; ++b) {
          c += (unsigned long long)h[0][b] + h[1][b];
          if (c > r[j]) {
            sval[j] = sqrt((double)b);
            break;
          }
        }
      }
    }
  }
  __syncthreads();
  if (t == 0) {
    double* o = out + k * ldo;
    for (int d = 0; d < 2; ++d) {
      o[d] = (double)sn[d][0];
      o[2 + d] = sn[d][0] ? ss[d][0] / (double)sn[d][0] : 0.0;
      o[4 + d] = sm[d][0] >= 0 ? sqrt((double)sm[d][0]) : 0.0;
    }
    double p = 0.0;
    if (N > 0) {
      const double a = sval[0], b = sval[1], diff = __dsub_rn(b, a);
      p = g >= 0.5 ? __dsub_rn(b, __dmul_rn(diff, __dsub_rn(1.0, g))) : __dadd_rn(a, __dmul_rn(diff, g));
    }
    o[6] = p;
    o[7] = (double)N;
  }
}

int grid_for(long long n) {
  long long blocks = (n + 255) / 256;
  const long long cap = (long long)sm_count_cached() * 8;
  return (int)(blocks < cap ? (blocks > 0 ? blocks : 1) : cap);
}

cudaStream_t ST(void* s) { return reinterpret_cast<cudaStream_t>(s); }

template <bool CONTIG>
int launch_envelope(int* dist, long long lines, int n, long long inner, cudaStream_t st) {
  const int bpe = CONTIG ? 10 : 6;                         // f (+ staged output) int32, vertex list uint16
  int T = 32;
  while (T > 1 && (long long)n * (T + 1) * bpe > 200 * 1024) T >>= 1;
  const size_t smem = (size_t)n * (T + 1) * bpe + 16;
  SX_CHECK_CUDA(cudaFuncSetAttribute(edt_envelope_kernel<CONTIG>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  edt_envelope_kernel<CONTIG><<<(unsigned)((lines + T - 1) / T), T, smem, st>>>(dist, lines, n, inner);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" int sx_mask_counts(const uint8_t* A, const uint8_t* B, int32_t K, int64_t V, int64_t* counts, int64_t ldc,
                              void* stream) {
  SX_REQUIRE(K > 0 && V > 0 && ldc >= 4, "sx_mask_counts: bad sizes K=%d V=%lld ldc=%lld", K, (long long)V, (long long)ldc);
  SX_REQUIRE(K <= 65535, "sx_mask_counts: at most 65535 classes (got %d)", K);
  SX_CHECK_CUDA(cudaMemset2DAsync(counts, ldc * sizeof(int64_t), 0, 4 * sizeof(int64_t), K, ST(stream)));
  long long bx = (V + 255) / 256;
  const long long cap = (long long)sm_count_cached() * 8 / K + 1;
  if (bx > cap) bx = cap;
  mask_counts_kernel<<<dim3((unsigned)bx, K), 256, 0, ST(stream)>>>(A, B, V, reinterpret_cast<unsigned long long*>(counts), ldc);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_surface(const uint8_t* X, int32_t K, int32_t ndim, int32_t n0, int32_t n1, int32_t n2, uint8_t* border,
                          void* stream) {
  SX_REQUIRE(ndim == 2 || ndim == 3, "sx_surface: ndim must be 2 or 3 (got %d)", ndim);
  SX_REQUIRE(K > 0 && n0 > 0 && n1 > 0 && n2 > 0 && (ndim == 3 || n0 == 1),
             "sx_surface: bad extents K=%d [%d,%d,%d] for ndim %d (a 2-D mask passes n0 = 1)", K, n0, n1, n2, ndim);
  const long long total = (long long)K * n0 * n1 * n2;
  surface_kernel<<<grid_for(total), 256, 0, ST(stream)>>>(X, total, ndim, n0, n1, n2, border);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_edt_sq(const uint8_t* border, int32_t K, int32_t n0, int32_t n1, int32_t n2, int32_t* dist, void* stream) {
  SX_REQUIRE(K > 0 && n0 > 0 && n1 > 0 && n2 > 0 && n0 <= kMaxExtent && n1 <= kMaxExtent && n2 <= kMaxExtent,
             "sx_edt_sq: extents [%d,%d,%d] must lie in [1, %d]", n0, n1, n2, kMaxExtent);
  const long long d2 = (long long)(n0 - 1) * (n0 - 1) + (long long)(n1 - 1) * (n1 - 1) + (long long)(n2 - 1) * (n2 - 1);
  SX_REQUIRE(d2 < kMaxD2, "sx_edt_sq: the squared diagonal %lld of [%d,%d,%d] exceeds the bin range %lld", d2, n0, n1, n2,
             kMaxD2);
  const long long V = (long long)n0 * n1 * n2;
  const long long lines0 = (long long)K * n1 * n2;
  edt_sweep_kernel<<<(unsigned)((lines0 + 127) / 128), 128, 0, ST(stream)>>>(border, dist, lines0, n0, (long long)n1 * n2);
  SX_CHECK_CUDA(cudaGetLastError());
  if (n1 > 1 && launch_envelope<false>(dist, K * V / n1, n1, n2, ST(stream))) return -2;
  if (n2 > 1 && launch_envelope<true>(dist, K * V / n2, n2, 1, ST(stream))) return -2;
  return 0;
}

extern "C" int sx_surface_hist(const uint8_t* src_border, const int32_t* dist, int32_t K, int64_t V, int32_t nbins,
                               uint32_t* hist, int64_t ldh, void* stream) {
  SX_REQUIRE(K > 0 && V > 0 && nbins > 0 && ldh >= nbins, "sx_surface_hist: bad sizes K=%d V=%lld nbins=%d ldh=%lld", K,
             (long long)V, nbins, (long long)ldh);
  SX_CHECK_CUDA(cudaMemset2DAsync(hist, ldh * sizeof(uint32_t), 0, (size_t)nbins * sizeof(uint32_t), K, ST(stream)));
  surface_hist_kernel<<<grid_for(K * V), 256, 0, ST(stream)>>>(src_border, dist, V, K * V, nbins, hist, ldh);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}

extern "C" int sx_surface_stats(const uint32_t* hist, int32_t K, int32_t nbins, int64_t ldh, double* out, int64_t ldo,
                                void* stream) {
  SX_REQUIRE(K > 0 && nbins > 0 && ldh >= 2 * (int64_t)nbins && ldo >= 8,
             "sx_surface_stats: bad sizes K=%d nbins=%d ldh=%lld ldo=%lld", K, nbins, (long long)ldh, (long long)ldo);
  surface_stats_kernel<<<K, kStatsThreads, 0, ST(stream)>>>(hist, nbins, ldh, out, ldo);
  SX_CHECK_CUDA(cudaGetLastError());
  return 0;
}
