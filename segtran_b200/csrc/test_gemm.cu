// Stand-alone bring-up / regression driver for sx_gemm (no Python, no torch).
//   ./test_gemm [key=value ...]     keys: the sx_gemm_debug_set knobs, plus perf=1 only=<substr>
// Every case is checked against a double-precision host product of the (pre-rounded) operands.
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "sx_common.cuh"

static float bf16_round(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }
static float tf32_round(float x) {
  uint32_t u;
  memcpy(&u, &x, 4);
  u += 0x00000FFFu + ((u >> 13) & 1u);      // round-to-nearest-even on the low 13 bits
  u &= 0xFFFFE000u;
  float r;
  memcpy(&r, &u, 4);
  return r;
}
static float frand() { return (float)rand() / RAND_MAX * 2.f - 1.f; }

struct Case {
  const char* name;
  int op;          // SX_OP_*
  int amaj, bmaj;
  int M, N, K, Z0, Z1;
  int b_bcast_z0;  // B broadcast over z0
  int split_k;
  int bias_mode, act, c_bf16, round_tf32, preact, amax;
  float alpha;
};

static double gelu_d(double x) { return 0.5 * x * (1.0 + erf(x / sqrt(2.0))); }

static int run_case(const Case& c, bool verbose) {
  const int es = c.op == SX_OP_TF32 ? 4 : 2;
  const int al = 16 / es;                                  // elements per 16 bytes
  auto pad = [&](int x) { return (x + al - 1) / al * al; };
  const int Z = c.Z0 * c.Z1;
  // logical A[z][m][k], B[z][n][k]
  const long long lda = c.amaj == SX_MAJOR_K ? pad(c.K) + al : pad(c.M) + al;   // padded leading dims
  const long long ldb = c.bmaj == SX_MAJOR_K ? pad(c.K) + al : pad(c.N) + al;
  const long long a_rows = c.amaj == SX_MAJOR_K ? c.M : c.K;
  const long long b_rows = c.bmaj == SX_MAJOR_K ? c.N : c.K;
  const long long a_z = a_rows * lda, b_z = b_rows * ldb;
  const int BZ = c.b_bcast_z0 ? c.Z1 : Z;
  std::vector<float> hA((size_t)a_z * Z), hB((size_t)b_z * BZ);
  for (auto& v : hA) v = c.op == SX_OP_TF32 ? tf32_round(frand()) : bf16_round(frand());
  for (auto& v : hB) v = c.op == SX_OP_TF32 ? tf32_round(frand()) : bf16_round(frand());
  const long long ldc = pad(c.N) + 8;
  const long long c_z = (long long)c.M * ldc;
  std::vector<float> hbias(c.bias_mode == SX_BIAS_M ? (size_t)c.M * Z : (size_t)c.N * Z);
  for (auto& v : hbias) v = frand();

  void *dA, *dB, *dC, *dP = nullptr;
  float *dbias, *damax = nullptr;
  cudaMalloc(&dA, hA.size() * es);
  cudaMalloc(&dB, hB.size() * es);
  const int ces = c.c_bf16 ? 2 : 4;
  cudaMalloc(&dC, (size_t)c_z * Z * ces);
  cudaMemset(dC, 0, (size_t)c_z * Z * ces);
  if (c.preact) { cudaMalloc(&dP, (size_t)c_z * Z * ces); cudaMemset(dP, 0, (size_t)c_z * Z * ces); }
  cudaMalloc(&dbias, hbias.size() * 4);
  cudaMemcpy(dbias, hbias.data(), hbias.size() * 4, cudaMemcpyHostToDevice);
  if (c.amax) { cudaMalloc(&damax, 4); float ninf = -3.0e38f; cudaMemcpy(damax, &ninf, 4, cudaMemcpyHostToDevice); }
  if (es == 4) {
    cudaMemcpy(dA, hA.data(), hA.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dB, hB.data(), hB.size() * 4, cudaMemcpyHostToDevice);
  } else {
    std::vector<__nv_bfloat16> t(hA.size());
    for (size_t i = 0; i < hA.size(); ++i) t[i] = __float2bfloat16_rn(hA[i]);
    cudaMemcpy(dA, t.data(), t.size() * 2, cudaMemcpyHostToDevice);
    t.resize(hB.size());
    for (size_t i = 0; i < hB.size(); ++i) t[i] = __float2bfloat16_rn(hB[i]);
    cudaMemcpy(dB, t.data(), t.size() * 2, cudaMemcpyHostToDevice);
  }

  sx_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.op_dtype = c.op;
  g.M = c.M; g.N = c.N; g.K = c.K; g.Z0 = c.Z0; g.Z1 = c.Z1;
  g.A.ptr = dA; g.A.major = c.amaj; g.A.ld = lda; g.A.stride_z0 = a_z; g.A.stride_z1 = a_z * c.Z0;
  g.B.ptr = dB; g.B.major = c.bmaj; g.B.ld = ldb;
  if (c.b_bcast_z0) { g.B.stride_z0 = 0; g.B.stride_z1 = b_z; } else { g.B.stride_z0 = b_z; g.B.stride_z1 = b_z * c.Z0; }
  if (Z == 1) { g.A.stride_z0 = g.A.stride_z1 = g.B.stride_z0 = g.B.stride_z1 = 0; }
  g.C = dC; g.c_dtype = c.c_bf16 ? SX_BF16 : SX_F32; g.round_tf32 = c.round_tf32;
  g.ldc = ldc; g.c_stride_z0 = c_z; g.c_stride_z1 = c_z * c.Z0;
  g.alpha = c.alpha;
  g.bias_mode = c.bias_mode; g.bias = c.bias_mode ? dbias : nullptr;
  g.bias_stride_z0 = c.bias_mode == SX_BIAS_M ? c.M : c.N;
  g.bias_stride_z1 = g.bias_stride_z0 * c.Z0;
  g.act = c.act; g.accumulate = c.split_k > 1; g.preact = dP; g.split_k = c.split_k; g.amax = damax;
  int rc = sx_gemm(&g, nullptr);
  cudaError_t e = cudaDeviceSynchronize();
  if (rc != 0 || e != cudaSuccess) {
    printf("CASE %-28s LAUNCH-FAIL rc=%d err=%s cuda=%s\n", c.name, rc, sx_last_error(), cudaGetErrorString(e));
    return 2;
  }
  std::vector<float> hC((size_t)c_z * Z), hP;
  auto fetch = [&](void* d, std::vector<float>& h) {
    h.resize((size_t)c_z * Z);
    if (c.c_bf16) {
      std::vector<__nv_bfloat16> t(h.size());
      cudaMemcpy(t.data(), d, t.size() * 2, cudaMemcpyDeviceToHost);
      for (size_t i = 0; i < h.size(); ++i) h[i] = __bfloat162float(t[i]);
    } else {
      cudaMemcpy(h.data(), d, h.size() * 4, cudaMemcpyDeviceToHost);
    }
  };
  fetch(dC, hC);
  if (c.preact) fetch(dP, hP);
  float gmax = 0;
  if (c.amax) cudaMemcpy(&gmax, damax, 4, cudaMemcpyDeviceToHost);

  double maxerr = 0, maxref = 0, maxerr_p = 0, refmax_val = -1e300;
  long long bad_pad = 0;
  for (int z1 = 0; z1 < c.Z1; ++z1)
    for (int z0 = 0; z0 < c.Z0; ++z0) {
      const int z = z1 * c.Z0 + z0;
      const float* A = hA.data() + (size_t)z * a_z;
      const float* B = hB.data() + (size_t)(c.b_bcast_z0 ? z1 : z) * b_z;
      for (int m = 0; m < c.M; ++m)
        for (int n = 0; n < c.N; ++n) {
          double s = 0;
          for (int k = 0; k < c.K; ++k) {
            const float a = c.amaj == SX_MAJOR_K ? A[(size_t)m * lda + k] : A[(size_t)k * lda + m];
            const float b = c.bmaj == SX_MAJOR_K ? B[(size_t)n * ldb + k] : B[(size_t)k * ldb + n];
            s += (double)a * b;
          }
          s *= c.alpha;
          if (c.bias_mode == SX_BIAS_N) s += hbias[(size_t)z * c.N + n];
          if (c.bias_mode == SX_BIAS_M) s += hbias[(size_t)z * c.M + m];
          const double pre = s;
          if (c.act == SX_ACT_GELU) s = gelu_d(s);
          const size_t idx = (size_t)z * c_z + (size_t)m * ldc + n;
          maxerr = fmax(maxerr, fabs(hC[idx] - s));
          maxref = fmax(maxref, fabs(s));
          refmax_val = fmax(refmax_val, s);
          if (c.preact) maxerr_p = fmax(maxerr_p, fabs(hP[idx] - pre));
        }
      // padding columns of C must stay untouched (zero)
      for (int m = 0; m < c.M; ++m)
        for (long long n = c.N; n < ldc; ++n)
          if (hC[(size_t)z * c_z + (size_t)m * ldc + n] != 0.f) ++bad_pad;
    }
  double tol = (c.c_bf16 ? 6e-3 : (c.round_tf32 ? 8e-4 : 1e-4)) * fmax(maxref, 1e-6) * (c.split_k > 1 ? 2 : 1);
  bool ok = maxerr <= tol && maxerr_p <= tol && bad_pad == 0;
  if (c.amax) ok = ok && fabs(gmax - refmax_val) <= tol;
  printf("CASE %-28s %s  maxerr %.3e (tol %.1e) maxref %.3e preact_err %.2e pad_violations %lld amax %.4f/%.4f\n",
         c.name, ok ? "PASS" : "FAIL", maxerr, tol, maxref, maxerr_p, bad_pad, gmax, c.amax ? refmax_val : 0.0);
  if (!ok && verbose) {
    printf("   C[0..3][0..7] got/ref:\n");
    for (int m = 0; m < 4 && m < c.M; ++m) {
      printf("   ");
      for (int n = 0; n < 8 && n < c.N; ++n) printf("%9.4f ", hC[(size_t)m * ldc + n]);
      printf("\n");
    }
  }
  cudaFree(dA); cudaFree(dB); cudaFree(dC); cudaFree(dbias);
  if (dP) cudaFree(dP);
  if (damax) cudaFree(damax);
  return ok ? 0 : 1;
}

static void perf(int op, int amaj, int bmaj, int M, int N, int K, int Z) {
  const int es = op == SX_OP_TF32 ? 4 : 2;
  void *dA, *dB, *dC;
  cudaMalloc(&dA, (size_t)M * K * Z * es);
  cudaMalloc(&dB, (size_t)N * K * Z * es);
  cudaMalloc(&dC, (size_t)M * N * Z * 4);
  cudaMemset(dA, 0, (size_t)M * K * Z * es);
  cudaMemset(dB, 0, (size_t)N * K * Z * es);
  sx_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.op_dtype = op; g.M = M; g.N = N; g.K = K; g.Z0 = Z; g.Z1 = 1;
  g.A.ptr = dA; g.A.major = amaj; g.A.ld = amaj == SX_MAJOR_K ? K : M; g.A.stride_z0 = Z > 1 ? (long long)M * K : 0;
  g.B.ptr = dB; g.B.major = bmaj; g.B.ld = bmaj == SX_MAJOR_K ? K : N; g.B.stride_z0 = Z > 1 ? (long long)N * K : 0;
  g.C = dC; g.c_dtype = SX_F32; g.ldc = N; g.c_stride_z0 = (long long)M * N; g.alpha = 1.f; g.split_k = 1;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 3; ++i) sx_gemm(&g, nullptr);
  cudaDeviceSynchronize();
  const int iters = 10;
  cudaEventRecord(e0);
  for (int i = 0; i < iters; ++i) sx_gemm(&g, nullptr);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  ms /= iters;
  const double tf = 2.0 * M * N * K * Z / (ms * 1e-3) / 1e12;
  printf("PERF %s A%s B%s M=%d N=%d K=%d Z=%d : %.3f ms  %.1f TFLOP/s  (%s)\n", op == SX_OP_TF32 ? "tf32" : "bf16",
         amaj ? "mn" : "k", bmaj ? "mn" : "k", M, N, K, Z, ms, tf, cudaGetErrorString(cudaGetLastError()));
  cudaFree(dA); cudaFree(dB); cudaFree(dC);
}

__global__ void fill_rand_kernel(float* p, size_t n, unsigned seed, float scale) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    unsigned h = (unsigned)i * 2654435761u + seed;
    h ^= h >> 15; h *= 0x2c1b3c6du; h ^= h >> 12; h *= 0x297a2d39u; h ^= h >> 15;
    p[i] = ((int)(h >> 8) - (1 << 23)) * (scale / (1 << 23));
  }
}

// epilogue cost decomposition on the fused P.V' shape of the cfg-4 step: 16 x (2744 x 1024 x 1024), A K-major, B MN-major
static void perf_epi(const char* name, int bias, int pre, int gelu, float drop, int rnd) {
  const int M = 2744, N = 1024, K = 1024, Z = 16;
  float *dA, *dB, *dC, *dP = nullptr, *dbias;
  cudaMalloc(&dA, (size_t)M * K * Z * 4); cudaMalloc(&dB, (size_t)N * K * Z * 4); cudaMalloc(&dC, (size_t)M * N * Z * 4);
  cudaMalloc(&dbias, N * 4);
  if (pre) cudaMalloc(&dP, (size_t)M * N * Z * 4);
  fill_rand_kernel<<<1024, 256>>>(dA, (size_t)M * K * Z, 1u, 1.0f / 32);        // softmax-like magnitudes
  fill_rand_kernel<<<1024, 256>>>(dB, (size_t)N * K * Z, 2u, 2.0f);
  fill_rand_kernel<<<4, 256>>>(dbias, N, 3u, 0.1f);
  sx_gemm_args g;
  memset(&g, 0, sizeof(g));
  g.op_dtype = SX_OP_TF32; g.M = M; g.N = N; g.K = K; g.Z0 = Z; g.Z1 = 1;
  g.A.ptr = dA; g.A.major = SX_MAJOR_K; g.A.ld = K; g.A.stride_z0 = (long long)M * K;
  g.B.ptr = dB; g.B.major = SX_MAJOR_MN; g.B.ld = N; g.B.stride_z0 = (long long)N * K;
  g.C = dC; g.c_dtype = SX_F32; g.ldc = N; g.c_stride_z0 = (long long)M * N; g.alpha = 1.f; g.split_k = 1;
  if (bias) { g.bias = dbias; g.bias_mode = SX_BIAS_N; }
  g.preact = dP; g.act = gelu ? SX_ACT_GELU : SX_ACT_NONE; g.drop_p = drop; g.drop_seed = 77; g.round_tf32 = rnd;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 3; ++i) sx_gemm(&g, nullptr);
  cudaDeviceSynchronize();
  const int iters = 20;
  cudaEventRecord(e0);
  for (int i = 0; i < iters; ++i) sx_gemm(&g, nullptr);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms = 0;
  cudaEventElapsedTime(&ms, e0, e1);
  ms /= iters;
  printf("EPI %-28s : %.1f us  %.1f TFLOP/s  (%s)\n", name, ms * 1e3, 2.0 * M * N * K * Z / (ms * 1e-3) / 1e12,
         cudaGetErrorString(cudaGetLastError()));
  cudaFree(dA); cudaFree(dB); cudaFree(dC); cudaFree(dbias);
  if (dP) cudaFree(dP);
}

int main(int argc, char** argv) {
  bool do_perf = false, ksweep = false, episweep = false;
  std::string only;
  for (int i = 1; i < argc; ++i) {
    char* eq = strchr(argv[i], '=');
    if (!eq) continue;
    std::string k(argv[i], eq - argv[i]);
    if (k == "perf") { do_perf = atoi(eq + 1) != 0; continue; }
    if (k == "ksweep") { ksweep = atoi(eq + 1) != 0; continue; }
    if (k == "episweep") { episweep = atoi(eq + 1) != 0; continue; }
    if (k == "only") { only = eq + 1; continue; }
    if (sx_gemm_debug_set(k.c_str(), atoll(eq + 1)) != 0) { printf("bad knob %s\n", k.c_str()); return 3; }
    printf("knob %s=%lld\n", k.c_str(), atoll(eq + 1));
  }
  int sms, ma, mi;
  if (sx_device_info(&sms, &ma, &mi) != 0) { printf("device: %s\n", sx_last_error()); return 4; }
  printf("device sm_%d%d, %d SMs\n", ma, mi, sms);
  srand(1234);
  const int K_ = SX_MAJOR_K, MN = SX_MAJOR_MN, T = SX_OP_TF32, H = SX_OP_BF16;
  std::vector<Case> cases = {
      // name                      op amaj bmaj   M    N    K  Z0 Z1 bb sk bias act bf16 rnd pre amax alpha
      {"bf16_kk_exact",            H, K_, K_, 128, 256,  64, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"bf16_kk_k256",             H, K_, K_, 128, 256, 256, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_kk_exact",            T, K_, K_, 128, 256,  32, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_kk_k256",             T, K_, K_, 128, 256, 256, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"bf16_kmn_exact",           H, K_, MN, 128, 256,  64, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"bf16_mnk_exact",           H, MN, K_, 128, 256,  64, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"bf16_mnmn_k256",           H, MN, MN, 128, 256, 256, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_kmn_exact",           T, K_, MN, 128, 256,  32, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_mnk_exact",           T, MN, K_, 128, 256,  32, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_mnmn_k256",           T, MN, MN, 128, 256, 256, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"bf16_kk_ragged",           H, K_, K_, 300, 520, 200, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_kk_ragged",           T, K_, K_, 300, 520, 200, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_kmn_ragged",          T, K_, MN, 300, 520, 200, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_mnk_ragged",          T, MN, K_, 300, 520, 200, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_mnmn_ragged",         T, MN, MN, 300, 520, 200, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"bf16_mnmn_ragged",         H, MN, MN, 300, 520, 200, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_small",               T, K_, K_,  40,  24,  12, 1, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_batched",             T, K_, K_, 150, 260, 100, 3, 2, 0, 1, 0, 0, 0, 0, 0, 0, 0.5f},
      {"tf32_batched_bcastB",      T, K_, MN, 150, 260, 100, 3, 2, 1, 1, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_splitk3",             T, MN, MN, 200, 300, 1000, 1, 1, 0, 3, 0, 0, 0, 0, 0, 0, 1.f},
      {"bf16_splitk4_batched",     H, MN, MN, 200, 300, 1000, 2, 1, 0, 4, 0, 0, 0, 0, 0, 0, 1.f},
      {"tf32_bias_n_gelu_pre",     T, K_, K_, 300, 520, 200, 2, 1, 0, 1, 1, 1, 0, 0, 1, 0, 1.f},
      {"tf32_bias_m",              T, K_, K_, 300, 520, 200, 1, 1, 0, 1, 2, 0, 0, 0, 0, 0, 1.f},
      {"tf32_round_amax",          T, K_, K_, 300, 520, 200, 1, 1, 0, 1, 1, 0, 0, 1, 0, 1, 0.25f},
      {"bf16_out_bf16_gelu",       H, K_, K_, 300, 520, 200, 1, 1, 0, 1, 1, 1, 1, 0, 1, 0, 1.f},
      {"tf32_many_tiles",          T, K_, K_, 1300, 2100, 96, 2, 1, 0, 1, 0, 0, 0, 0, 0, 0, 1.f},
  };
  int fails = 0, ran = 0;
  for (auto& c : cases) {
    if (!only.empty() && std::string(c.name).find(only) == std::string::npos) continue;
    int r = run_case(c, true);
    ++ran;
    if (r) ++fails;
    if (r == 2) { printf("aborting after launch failure (context likely poisoned)\n"); break; }
  }
  printf("SUMMARY %d/%d cases passed\n", ran - fails, ran);
  if (episweep) {
    perf_epi("plain", 0, 0, 0, 0.f, 0);
    perf_epi("round", 0, 0, 0, 0.f, 1);
    perf_epi("bias+round", 1, 0, 0, 0.f, 1);
    perf_epi("bias+round+preact", 1, 1, 0, 0.f, 1);
    perf_epi("bias+round+gelu", 1, 0, 1, 0.f, 1);
    perf_epi("bias+round+dropout", 1, 0, 0, 0.2f, 1);
    perf_epi("bias+round+gelu+dropout", 1, 0, 1, 0.2f, 1);
    perf_epi("all (preact+gelu+dropout)", 1, 1, 1, 0.2f, 1);
    return 0;
  }
  if (ksweep) {
    const int Ks[] = {128, 256, 512, 1024, 2048, 4096};
    for (int kk : Ks) perf(T, K_, K_, 128 * 66, 128 * 20, kk, 1);      // 1320 tiles = exactly 10 waves of 132
    for (int kk : Ks) perf(H, K_, K_, 128 * 66, 128 * 20, kk, 1);
    return 0;
  }
  if (do_perf) {
    perf(H, K_, K_, 8192, 8192, 8192, 1);
    perf(T, K_, K_, 8192, 8192, 8192, 1);
    perf(H, K_, MN, 8192, 8192, 8192, 1);
    perf(H, MN, MN, 8192, 8192, 8192, 1);
    perf(T, MN, MN, 8192, 8192, 8192, 1);
    perf(T, K_, K_, 2744, 1024, 1024, 16);
    perf(H, K_, K_, 2744, 1024, 1024, 16);
    perf(T, K_, K_, 2744, 1024, 256, 16);
  }
  return fails ? 1 : 0;
}
