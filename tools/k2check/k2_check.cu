// Stand-alone check of k2_dots<E> / k2_update<E> against naive kernels: which tiles / elements differ?
// build: nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -I../../bifurcationkit.jl_b200/csrc k2_check.cu -o k2_check
#include <cstdio>
#include <cstdlib>
#include <cmath>
#include <vector>
#include <algorithm>
#include "bk_krylov_tma.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e_), __LINE__); exit(1); } } while (0)

__global__ void k_fill(double* p, long long n, unsigned long long seed) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    unsigned long long z = (i + 1) * 0x9E3779B97F4A7C15ull + seed;
    z ^= z >> 30; z *= 0xBF58476D1CE4E5B9ull; z ^= z >> 27; z *= 0x94D049BB133111EBull; z ^= z >> 31;
    p[i] = (double)(z >> 11) * (1.0 / 9007199254740992.0) - 0.5;
  }
}
__global__ void k_ref_update(const double* w, long long n, const double* V, long long ld, int j, const double* g, double* out) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    double v = w[i];
    for (int k = j - 1; k >= 0; --k) v = fma(-g[k], V[(long long)k * ld + i], v);  // k2_update walks the basis backwards (round 2)
    out[i] = v;
  }
}
__global__ void k_cmp(const double* a, const double* b, long long n, int tile, unsigned int* bad_per_tile, long long* first_bad) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    if (a[i] != b[i]) {
      atomicAdd(&bad_per_tile[i / tile], 1u);
      atomicMin((unsigned long long*)first_bad + i / tile, (unsigned long long)(i % tile));
    }
  }
}
// per-tile reference dots: out[t*j + k] = sum over tile t of V_k * w
__global__ void k_ref_tiledots(const double* w, long long n, const double* V, long long ld, int j, int tile, double* out) {
  const long long base = (long long)blockIdx.x * tile;
  __shared__ double s[256];
  for (int k = 0; k < j; ++k) {
    double a = 0;
    for (int q = threadIdx.x; q < tile; q += blockDim.x) if (base + q < n) a = fma(V[(long long)k * ld + base + q], w[base + q], a);
    s[threadIdx.x] = a; __syncthreads();
    for (int o = 128; o > 0; o >>= 1) { if (threadIdx.x < o) s[threadIdx.x] += s[threadIdx.x + o]; __syncthreads(); }
    if (threadIdx.x == 0) out[(long long)blockIdx.x * j + k] = s[0];
    __syncthreads();
  }
}

template <int E>
static void run(long long n, int j, int NS, int reps, int pdl) {
  const long long ld = (n + 2 + 31) / 32 * 32;
  const int tile = E * BK2_ROW;
  const int G = (int)((n + tile - 1) / tile);
  double *V, *w, *g, *out, *ref, *partials, *hout, *scales, *hcol, *gcoef, *refd;
  unsigned int *counter, *bad; long long* first;
  CK(cudaMalloc(&V, 8 * ld * (size_t)j)); CK(cudaMalloc(&w, 8 * ld)); CK(cudaMalloc(&out, 8 * ld)); CK(cudaMalloc(&ref, 8 * ld));
  CK(cudaMalloc(&g, 8 * 64)); CK(cudaMalloc(&scales, 8 * 64)); CK(cudaMalloc(&hcol, 8 * 64)); CK(cudaMalloc(&gcoef, 8 * 64));
  CK(cudaMalloc(&partials, 8 * (size_t)(j + 4) * G)); CK(cudaMalloc(&hout, 16)); CK(cudaMalloc(&counter, 64)); CK(cudaMemset(counter, 0, 64));
  CK(cudaMalloc(&bad, 4 * (size_t)G)); CK(cudaMalloc(&first, 8 * (size_t)G)); CK(cudaMalloc(&refd, 8 * (size_t)G * j));
  k_fill<<<2048, 256>>>(V, ld * j, 1); k_fill<<<2048, 256>>>(w, ld, 2); k_fill<<<1, 64>>>(g, 64, 3);
  std::vector<double> ones(64, 1.0); CK(cudaMemcpy(scales, ones.data(), 8 * 64, cudaMemcpyHostToDevice));
  k_ref_update<<<2048, 256>>>(w, n, V, ld, j, g, ref);
  k_ref_tiledots<<<G, 256>>>(w, n, V, ld, j, tile, refd);
  CK(cudaDeviceSynchronize());
  const size_t sred = 8 * 8 * (size_t)(j + 2), ring = (size_t)NS * tile * 8, smem = ring + sred;
  CK(cudaFuncSetAttribute(k2_update<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CK(cudaFuncSetAttribute(k2_dots<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  CK(cudaFuncSetAttribute(k2_update<E>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  CK(cudaFuncSetAttribute(k2_dots<E>, cudaFuncAttributePreferredSharedMemoryCarveout, 100));
  int occ_u = 0, occ_d = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_u, k2_update<E>, BK2_THREADS, smem);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_d, k2_dots<E>, BK2_THREADS, smem);
  printf("E=%d n=%lld G=%d NS=%d smem=%zu occupancy update=%d dots=%d pdl=%d\n", E, n, G, NS, smem, occ_u, occ_d, pdl);
  if (pdl) setenv("BK_NO_PDL", "1", 0);
  for (int rep = 0; rep < reps; ++rep) {
    CK(cudaMemset(out, 0, 8 * ld)); CK(cudaMemset(bad, 0, 4 * (size_t)G)); CK(cudaMemset(first, 0x7f, 8 * (size_t)G));
    CK(bk_launch_pdl(k2_update<E>, dim3(G), dim3(BK2_THREADS), smem, 0, true, (const double*)w, n, (const double*)V, ld, j, (const double*)g, out, partials, counter, hout, hout + 1, 0, NS));
    CK(cudaDeviceSynchronize());
    k_cmp<<<2048, 256>>>(out, ref, n, tile, bad, first);
    CK(cudaDeviceSynchronize());
    std::vector<unsigned int> hb(G); std::vector<long long> hf(G);
    CK(cudaMemcpy(hb.data(), bad, 4 * (size_t)G, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(hf.data(), first, 8 * (size_t)G, cudaMemcpyDeviceToHost));
    int nbad = 0; long long tot = 0;
    for (int t = 0; t < G; ++t) if (hb[t]) { ++nbad; tot += hb[t]; }
    printf("  update rep %d: bad tiles %d / %d, bad elements %lld;", rep, nbad, G, tot);
    int shown = 0;
    for (int t = 0; t < G && shown < 12; ++t) if (hb[t]) { printf(" [cta %d n=%u first=%lld]", t, hb[t], hf[t]); ++shown; }
    printf("\n");
    // dots: compare per-CTA partials with per-tile reference
    CK(bk_launch_pdl(k2_dots<E>, dim3(G), dim3(BK2_THREADS), smem, 0, true, (const double*)w, n, (const double*)V, ld, j, (const double*)scales, partials, counter + 1, hcol, gcoef, 0, NS, (int)(ring / 8)));
    CK(cudaDeviceSynchronize());
    std::vector<double> hp((size_t)j * G), hr((size_t)G * j);
    CK(cudaMemcpy(hp.data(), partials, 8 * (size_t)j * G, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(hr.data(), refd, 8 * (size_t)G * j, cudaMemcpyDeviceToHost));
    int dbad = 0; shown = 0;
    for (int t = 0; t < G; ++t) {
      bool b = false;
      for (int k = 0; k < j; ++k) if (fabs(hp[(size_t)k * G + t] - hr[(size_t)t * j + k]) > 1e-9 * (1 + fabs(hr[(size_t)t * j + k]))) b = true;
      if (b) { ++dbad; if (shown++ < 8) { printf("   dots bad cta %d:", t); for (int k = 0; k < j; ++k) printf(" %d:%+.3e/%+.3e", k, hp[(size_t)k * G + t], hr[(size_t)t * j + k]); printf("\n"); } }
    }
    printf("  dots rep %d: bad tiles %d / %d\n", rep, dbad, G);
  }
  {  // timing (kernel pairs back to back, after the checks)
    cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
    const int T = 20;
    cudaEventRecord(e0);
    for (int r = 0; r < T; ++r)
      bk_launch_pdl(k2_update<E>, dim3(G), dim3(BK2_THREADS), smem, 0, true, (const double*)w, n, (const double*)V, ld, j, (const double*)g, out, partials, counter, hout, hout + 1, 0, NS);
    cudaEventRecord(e1); CK(cudaDeviceSynchronize());
    float mu = 0; cudaEventElapsedTime(&mu, e0, e1);
    cudaEventRecord(e0);
    for (int r = 0; r < T; ++r)
      bk_launch_pdl(k2_dots<E>, dim3(G), dim3(BK2_THREADS), smem, 0, true, (const double*)w, n, (const double*)V, ld, j, (const double*)scales, partials, counter + 1, hcol, gcoef, 0, NS, (int)(ring / 8));
    cudaEventRecord(e1); CK(cudaDeviceSynchronize());
    float md = 0; cudaEventElapsedTime(&md, e0, e1);
    const double bu = 8.0 * n * (j + 2), bd = 8.0 * n * (j + 1);
    printf("  time: update %.1f us (%.0f GB/s)  dots %.1f us (%.0f GB/s)\n", 1e3 * mu / T, bu / (1e6 * mu / T), 1e3 * md / T, bd / (1e6 * md / T));
  }
  cudaFree(V); cudaFree(w); cudaFree(out); cudaFree(ref); cudaFree(partials); cudaFree(bad); cudaFree(first); cudaFree(refd);
}

int main(int argc, char** argv) {
  long long n = argc > 1 ? atoll(argv[1]) : 3932161;
  int E = argc > 2 ? atoi(argv[2]) : 8, j = argc > 3 ? atoi(argv[3]) : 6, NS = argc > 4 ? atoi(argv[4]) : 3, reps = argc > 5 ? atoi(argv[5]) : 2;
  int nopdl = argc > 6 ? atoi(argv[6]) : 0;
  switch (E) {
    case 6: run<6>(n, j, NS, reps, nopdl); break;
    case 7: run<7>(n, j, NS, reps, nopdl); break;
    default: run<8>(n, j, NS, reps, nopdl); break;
  }
  return 0;
}
