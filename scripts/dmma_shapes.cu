// Developer micro-benchmark (GPU box): the fp64 tensor-core shapes of mma.sync on Hopper -- m8n8k4, m16n8k4, m16n8k8, m16n8k16 --
// checked against a host product with the fragment layouts of csrc/kernels.cuh, then timed:
//   throughput  one CTA per SM, WARPS warps, CHAINS independent accumulators per warp  -> MAC / clk / SM
//   latency     one warp, one accumulator, every step depends on the previous one      -> cycles per dependent step
// Cycles are clock64 deltas inside the kernel; CUDA events time the throughput launch for an fp64 TFLOP/s figure.  The card's name,
// power limit and SM clocks are printed by the same run.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -o /tmp/dmma_shapes scripts/dmma_shapes.cu && /tmp/dmma_shapes
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

// lane = 4 grp + tig.  m8n8k4: A[grp][tig], B[tig][grp], C[grp][2 tig + h].  m16n8kK (K = 4 j): A[grp + 8 (i & 1)][tig + 4 (i >> 1)] (a_i),
// B[tig + 4 i][grp] (b_i), C[grp + 8 (i >> 1)][2 tig + (i & 1)] (c_i).
template <int SHAPE> struct Shape;
template <> struct Shape<0> {
  static constexpr int M = 8, K = 4, NA = 1, NB = 1, NCF = 2; static constexpr const char* name = "m8n8k4";
  __device__ static void mma(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c[0]), "+d"(c[1]) : "d"(a[0]), "d"(b[0]));
  }
  static int arow(int l, int) { return l >> 2; }
  static int acol(int l, int) { return l & 3; }
  static int crow(int l, int) { return l >> 2; }
};
template <> struct Shape<1> {
  static constexpr int M = 16, K = 4, NA = 2, NB = 1, NCF = 4; static constexpr const char* name = "m16n8k4";
  __device__ static void mma(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(b[0]));
  }
  static int arow(int l, int i) { return (l >> 2) + 8 * (i & 1); }
  static int acol(int l, int i) { return (l & 3) + 4 * (i >> 1); }
  static int crow(int l, int i) { return (l >> 2) + 8 * (i >> 1); }
};
template <> struct Shape<2> {
  static constexpr int M = 16, K = 8, NA = 4, NB = 2, NCF = 4; static constexpr const char* name = "m16n8k8";
  __device__ static void mma(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(b[0]), "d"(b[1]));
  }
  static int arow(int l, int i) { return Shape<1>::arow(l, i); }
  static int acol(int l, int i) { return Shape<1>::acol(l, i); }
  static int crow(int l, int i) { return Shape<1>::crow(l, i); }
};
template <> struct Shape<3> {
  static constexpr int M = 16, K = 16, NA = 8, NB = 4, NCF = 4; static constexpr const char* name = "m16n8k16";
  __device__ static void mma(double* c, const double* a, const double* b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a[0]), "d"(a[1]), "d"(a[2]), "d"(a[3]), "d"(a[4]), "d"(a[5]), "d"(a[6]), "d"(a[7]), "d"(b[0]), "d"(b[1]), "d"(b[2]), "d"(b[3]));
  }
  static int arow(int l, int i) { return Shape<1>::arow(l, i); }
  static int acol(int l, int i) { return Shape<1>::acol(l, i); }
  static int crow(int l, int i) { return Shape<1>::crow(l, i); }
};

// one product C = A B of A [M][K], B [K][8] with the fragments loaded by the layouts above
template <int SHAPE>
__global__ void k_check(const double* A, const double* B, double* C) {
  using S = Shape<SHAPE>;
  const int l = threadIdx.x, grp = l >> 2, tig = l & 3;
  double a[S::NA], b[S::NB], c[S::NCF];
  for (int i = 0; i < S::NA; i++) a[i] = SHAPE == 0 ? A[grp * S::K + tig] : A[((grp + 8 * (i & 1)) * S::K) + tig + 4 * (i >> 1)];
  for (int i = 0; i < S::NB; i++) b[i] = B[(tig + 4 * i) * 8 + grp];
  for (int i = 0; i < S::NCF; i++) c[i] = 0.0;
  S::mma(c, a, b);
  for (int i = 0; i < S::NCF; i++) C[(grp + 8 * (i >> 1)) * 8 + 2 * tig + (i & 1)] = c[i];
}

template <int SHAPE, int CHAINS>
__global__ void k_rate(int iters, double seed, double* sink, long long* cyc) {
  using S = Shape<SHAPE>;
  double a[S::NA], b[S::NB], c[CHAINS][S::NCF];
  for (int i = 0; i < S::NA; i++) a[i] = seed * (threadIdx.x + i);
  for (int i = 0; i < S::NB; i++) b[i] = seed * (threadIdx.x - i);
#pragma unroll
  for (int q = 0; q < CHAINS; q++)
#pragma unroll
    for (int i = 0; i < S::NCF; i++) c[q][i] = 0.0;
  __syncthreads();
  const long long t0 = clock64();
  for (int it = 0; it < iters; it++) {
#pragma unroll
    for (int q = 0; q < CHAINS; q++) S::mma(c[q], a, b);
  }
  __syncthreads();
  const long long t1 = clock64();
  double s = 0.0;
#pragma unroll
  for (int q = 0; q < CHAINS; q++)
#pragma unroll
    for (int i = 0; i < S::NCF; i++) s += c[q][i];
  if (s == 1234.5) sink[0] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

static void card() {
  FILE* f = popen("nvidia-smi --query-gpu=name,power.limit,clocks.sm,clocks.max.sm --format=csv,noheader", "r");
  char line[256];
  if (f && fgets(line, sizeof line, f)) printf("card: %s", line);
  if (f) pclose(f);
}

template <int SHAPE>
static bool check() {
  using S = Shape<SHAPE>;
  std::vector<double> A(S::M * S::K), B(S::K * 8), C(S::M * 8), R(S::M * 8, 0.0);
  for (size_t i = 0; i < A.size(); i++) A[i] = std::ldexp(1.0, (int)(i % 7)) + 0.25 * (double)i;
  for (size_t i = 0; i < B.size(); i++) B[i] = 1.0 - 0.125 * (double)i;
  for (int i = 0; i < S::M; i++)
    for (int j = 0; j < 8; j++)
      for (int k = 0; k < S::K; k++) R[i * 8 + j] += A[i * S::K + k] * B[k * 8 + j];
  double *dA, *dB, *dC;
  CK(cudaMalloc(&dA, A.size() * 8)); CK(cudaMalloc(&dB, B.size() * 8)); CK(cudaMalloc(&dC, C.size() * 8));
  CK(cudaMemcpy(dA, A.data(), A.size() * 8, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dB, B.data(), B.size() * 8, cudaMemcpyHostToDevice));
  k_check<SHAPE><<<1, 32>>>(dA, dB, dC);
  CK(cudaMemcpy(C.data(), dC, C.size() * 8, cudaMemcpyDeviceToHost));
  double err = 0.0;
  for (size_t i = 0; i < C.size(); i++) err = std::fmax(err, std::fabs(C[i] - R[i]) / (1.0 + std::fabs(R[i])));
  printf("%-9s layout check: max rel err %.1e  %s\n", S::name, err, err < 1e-14 ? "ok" : "MISMATCH");
  cudaFree(dA); cudaFree(dB); cudaFree(dC);
  return err < 1e-14;
}

template <int SHAPE>
static void measure(int sms, double* sink, long long* dcyc) {
  using S = Shape<SHAPE>;
  constexpr int CHAINS = 8, WARPS = 8;
  const double mac = S::M * 8.0 * S::K;
  const int iters = 4096;
  std::vector<long long> cyc(sms);
  cudaEvent_t e0, e1;
  CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  k_rate<SHAPE, CHAINS><<<sms, 32 * WARPS>>>(iters, 1e-3, sink, dcyc);       // warm-up
  CK(cudaEventRecord(e0));
  k_rate<SHAPE, CHAINS><<<sms, 32 * WARPS>>>(iters, 1e-3, sink, dcyc);
  CK(cudaEventRecord(e1));
  CK(cudaEventSynchronize(e1));
  float ms = 0.f;
  CK(cudaEventElapsedTime(&ms, e0, e1));
  CK(cudaMemcpy(cyc.data(), dcyc, sms * sizeof(long long), cudaMemcpyDeviceToHost));
  long long cmax = 0;
  for (long long v : cyc) cmax = v > cmax ? v : cmax;
  const double per_sm = mac * CHAINS * WARPS * iters;
  const double tflops = 2.0 * per_sm * sms / (ms * 1e-3) / 1e12;
  // latency: one warp, one chain
  const int liters = 8192;
  k_rate<SHAPE, 1><<<1, 32>>>(liters, 1e-3, sink, dcyc);
  k_rate<SHAPE, 1><<<1, 32>>>(liters, 1e-3, sink, dcyc);
  long long lc = 0;
  CK(cudaMemcpy(&lc, dcyc, sizeof(long long), cudaMemcpyDeviceToHost));
  CK(cudaGetLastError());
  printf("%-9s %5.0f MAC/instr  throughput %7.1f MAC/clk/SM  %6.2f instr/clk/SM  %5.1f TFLOP/s fp64 (%.3f ms)   dependent step %6.1f clk  (%5.2f MAC/clk on one chain)\n",
         S::name, mac, per_sm / cmax, per_sm / cmax / mac, tflops, ms, (double)lc / liters, mac * liters / lc);
  cudaEventDestroy(e0); cudaEventDestroy(e1);
}

int main() {
  card();
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  bool ok = check<0>() & check<1>() & check<2>() & check<3>();
  double* sink; long long* dcyc;
  CK(cudaMalloc(&sink, 8)); CK(cudaMalloc(&dcyc, sms * sizeof(long long)));
  printf("throughput: %d CTAs (one per SM) x 8 warps x 8 independent chains; latency: 1 warp, 1 chain\n", sms);
  measure<0>(sms, sink, dcyc);
  measure<1>(sms, sink, dcyc);
  measure<2>(sms, sink, dcyc);
  measure<3>(sms, sink, dcyc);
  card();
  cudaFree(sink); cudaFree(dcyc);
  return ok ? 0 : 1;
}
