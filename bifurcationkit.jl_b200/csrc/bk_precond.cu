// bk_precond.cu -- K6: preconditioners honouring the reference's Pl/Pr contract
// (ldiv!(y, P, x), src/Preconditioner.jl:11-37).
//
// BK_PC_SH_DCT: the examples precondition Swift-Hohenberg with a sparse factorisation of L1 + I
//   (examples/SH2d-fronts.jl:120-122  Pl = lu(par.L1 + I); examples/SH3d.jl:88 cholesky(L1)).  The
//   Neumann-closure Laplacian (SH2d-fronts.jl:13-29) is diagonalised by the DCT-II, so
//   (L1 + shift I)^-1 r = IDCT( DCT(r) / ((1 + lx_i + ly_j [+ lz_k])^2 + shift) )  exactly
//   (identity pinned in tests/test_oracle_palc.py::test_dct_symbol_diagonalises_L1).
//   Power-of-two line lengths 64..2048 run the register-resident FFT kernels of bk_fft_fast.cuh (two lines per complex
//   FFT, the last dimension fused: forward + symbol + inverse, so an application is 3 kernels in 2-D and 5 in 3-D);
//   every other length runs the mixed-radix kernel of bk_fft_gen.cuh.  No library on this path.
// BK_PC_SH_FFT: (L1 + shift I)^-1 on the periodic grid of BK_SH2D_PERIODIC (examples/SH2d-fronts-cuda.jl:55-64), the real 2-D FFT
//   pipeline of bk_periodic_setup / periodic_pipeline below, which also applies that kind's residual and JVP.
// BK_PC_CHAN_TRIDIAG: lu(P) of examples/chan.jl:108-111 (Thomas algorithm, one thread: n = 1e3 plumbing).
// BK_PC_CGL_DST: per-component (a0 I + a1 Lap_dirichlet)^-1 by DST-I (stand-in for the ILU of
//   examples/cGL2d.jl:209-213); for potrap contexts it is applied slice by slice (block Jacobi, cf.
//   jacobian_block_diag, src/periodicorbit/PeriodicOrbitTrapeze.jl:619-643).
// BK_PC_POTRAP_CIRC: block-circulant-in-time linearisation of the Trapeze functional at the trivial state, inverted
//   exactly: DST-I in space, u1 +- i u2, DFT over the M-1 cyclic slices, scalar symbol.  While J' is selected
//   (bk_jac_set_transpose) it applies the exact transpose P'^-1, so that the J' solves are preconditioned with P'.
#include <cmath>
#include <cstdlib>
#include <vector>
#include "bk_common.cuh"

#include "bk_fft_fast.cuh"
#include "bk_fft_gen.cuh"

// divide by the symbol
static __global__ void __launch_bounds__(256) k_sh_symbol_div(double* __restrict__ a, int nx, int ny, int nz,
                                                              const double* __restrict__ lx, const double* __restrict__ ly,
                                                              const double* __restrict__ lz, double shift, double scale) {
  const long long total = (long long)nx * ny * nz;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    int i = (int)(q % nx), j = (int)((q / nx) % ny), k = (int)(q / ((long long)nx * ny));
    double t = 1.0 + lx[i] + ly[j] + (lz ? lz[k] : 0.0);
    a[q] = a[q] * scale / (t * t + shift);
  }
}
static __global__ void __launch_bounds__(256) k_helmholtz_symbol_div(double* __restrict__ a, int nx, int ny, long long nblocks,
                                                                     const double* __restrict__ lx,
                                                                     const double* __restrict__ ly, double a0, double a1) {
  const long long n = (long long)nx * ny, total = n * nblocks;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    long long g = q % n;
    int i = (int)(g % nx), j = (int)(g / nx);
    a[q] = a[q] / (a0 + a1 * (lx[i] + ly[j]));
  }
}
// BK_PC_RD: field f of the transformed blocks divided by a0 + a1 D_f (lx + ly) (times scale: 1 / prod 2 n_d for the DCT-II)
struct RdDiff {
  double d[BK_RD_MAX_FIELDS];
};
static __global__ void __launch_bounds__(256) k_rd_symbol_div(double* __restrict__ a, int nx, int ny, int fields,
                                                              const double* __restrict__ lx, const double* __restrict__ ly,
                                                              double a0, double a1, RdDiff D, double scale) {
  const long long n = (long long)nx * ny, total = n * fields;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    const long long g = q % n;
    const int f = (int)(q / n), i = (int)(g % nx), j = (int)(g / nx);
    const double df = f == 0 ? D.d[0] : f == 1 ? D.d[1] : f == 2 ? D.d[2] : D.d[3];
    a[q] = a[q] * scale / (a0 + a1 * df * (lx[i] + (ly ? ly[j] : 0.0)));
  }
}

// ---- potrap circulant preconditioner: time direction -------------------------------------------------------------------
// B holds the DST-I coefficients of all 2M slice components (field f = 2*slice + comp, n values each).  One thread per
// spatial mode: w+- = u1 +- i u2 over the K = M-1 cyclic slices, DFT in time, divide by
//   s+-_k = (1 - g_k) - h/2 (1 + g_k)(lambda + r +- i nu),   g_k = exp(-2 pi i k/K),
// inverse DFT, back to (u1, u2).  In place.
// TR: the same solve with the transposed block circulant (P'^-1 while J' is selected).  Its time blocks are x_k - x_{k+1} (the
// shift the other way: g_k -> conj g_k) and its reaction block is [[a, nu], [-nu, a]] (nu -> -nu on w+-), so its symbol is
// conj(s+-_k).  The closure slice M-1 is added to slice 0 first: the transpose of x_M = r_M + x_1.
#define BK_PO_KMAX 64
template <bool TR>
static __global__ void __launch_bounds__(128) k_potrap_time(double* __restrict__ B, long long n, int nx, int K,
                                                            const double* __restrict__ lamx, const double* __restrict__ lamy,
                                                            double h, double r, double nu, const double2* __restrict__ tw) {
  const long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= n) return;
  const double lam = lamx[g % nx] + lamy[g / nx];
  double2 wp[BK_PO_KMAX], wm[BK_PO_KMAX];
  for (int i = 0; i < K; ++i) {
    double a = B[(long long)(2 * i) * n + g], b = B[(long long)(2 * i + 1) * n + g];
    if constexpr (TR) {
      if (i == 0) {  // + the closure slice M-1 (field pair 2K, 2K+1, transformed with the rest)
        a += B[(long long)(2 * K) * n + g];
        b += B[(long long)(2 * K + 1) * n + g];
      }
    }
    wp[i] = make_double2(a, b);
    wm[i] = make_double2(a, -b);
  }
  double2 yp[BK_PO_KMAX], ym[BK_PO_KMAX];
  const double invK = 1.0 / K;
  for (int k = 0; k < K; ++k) {
    double2 ap = make_double2(0, 0), am = make_double2(0, 0);
    int idx = 0;
    for (int i = 0; i < K; ++i) {
      const double2 t = tw[idx];  // exp(-2 pi i k i / K)
      ap.x += wp[i].x * t.x - wp[i].y * t.y;
      ap.y += wp[i].x * t.y + wp[i].y * t.x;
      am.x += wm[i].x * t.x - wm[i].y * t.y;
      am.y += wm[i].x * t.y + wm[i].y * t.x;
      idx += k;
      if (idx >= K) idx -= K;
    }
    const double2 gk = tw[k];
    // s = (1 - g) - h/2 (1 + g) (lam + r +- i nu)
    const double2 omg = make_double2(1.0 - gk.x, -gk.y), opg = make_double2(1.0 + gk.x, gk.y);
    const double cr = lam + r;
    double2 sp = make_double2(omg.x - 0.5 * h * (opg.x * cr - opg.y * nu), omg.y - 0.5 * h * (opg.x * nu + opg.y * cr));
    double2 sm = make_double2(omg.x - 0.5 * h * (opg.x * cr + opg.y * nu), omg.y - 0.5 * h * (-opg.x * nu + opg.y * cr));
    if constexpr (TR) {  // the transposed symbols conj(s+-_k)
      sp.y = -sp.y;
      sm.y = -sm.y;
    }
    const double dp = 1.0 / (sp.x * sp.x + sp.y * sp.y), dm = 1.0 / (sm.x * sm.x + sm.y * sm.y);
    yp[k] = make_double2((ap.x * sp.x + ap.y * sp.y) * dp * invK, (ap.y * sp.x - ap.x * sp.y) * dp * invK);
    ym[k] = make_double2((am.x * sm.x + am.y * sm.y) * dm * invK, (am.y * sm.x - am.x * sm.y) * dm * invK);
  }
  for (int i = 0; i < K; ++i) {
    double2 ap = make_double2(0, 0), am = make_double2(0, 0);
    int idx = 0;
    for (int k = 0; k < K; ++k) {
      const double2 t = tw[idx];  // conj -> exp(+2 pi i k i / K)
      ap.x += yp[k].x * t.x + yp[k].y * t.y;
      ap.y += yp[k].y * t.x - yp[k].x * t.y;
      am.x += ym[k].x * t.x + ym[k].y * t.y;
      am.y += ym[k].y * t.x - ym[k].x * t.y;
      idx += i;
      if (idx >= K) idx -= K;
    }
    B[(long long)(2 * i) * n + g] = 0.5 * (ap.x + am.x);      // Re((yp + ym)/2)
    B[(long long)(2 * i + 1) * n + g] = 0.5 * (ap.y - am.y);  // Re((yp - ym)/(2i)) = Im(yp - ym)/2
  }
}
// closure row of the preconditioner: x_M = r_M + x_1; the period entry passes through
static __global__ void __launch_bounds__(256) k_potrap_close(const double* __restrict__ in, double* __restrict__ out,
                                                             long long Ns, int M) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < Ns) out[(long long)(M - 1) * Ns + i] = in[(long long)(M - 1) * Ns + i] + out[i];
  if (i == 0) out[(long long)M * Ns] = in[(long long)M * Ns];
}

// Thomas solve with precomputed factors: tri = [cprime (n) | denom_inv (n) | lower (n)]
static __global__ void k_thomas(const double* __restrict__ tri, const double* __restrict__ in, double* __restrict__ out, int n) {
  if (blockIdx.x != 0 || threadIdx.x != 0) return;
  const double* cp = tri;
  const double* di = tri + n;
  const double* lo = tri + 2 * n;
  double prev = in[0] * di[0];
  out[0] = prev;
  for (int i = 1; i < n; ++i) {
    prev = (in[i] - lo[i] * prev) * di[i];
    out[i] = prev;
  }
  for (int i = n - 2; i >= 0; --i) out[i] -= cp[i] * out[i + 1];
}

// ------------------------------------------------------------------------------------------------ host
static int upload(bk_ctx* c, void** dst, const void* src, size_t bytes) {
  if (*dst) cudaFree(*dst);
  *dst = nullptr;
  BK_CUDA(c, cudaMalloc(dst, bytes));
  BK_CUDA(c, cudaMemcpy(*dst, src, bytes, cudaMemcpyHostToDevice));
  return BK_OK;
}

// ---- fast path: one instantiation per (values per thread, line length) -----------------------------------------------------
// Values per thread E = 2^loge of the fast kernels for a line of length n: E = 8 for n >= 1024, E = 4 below, chosen for the
// GMRES loop, where more warps per SM hide the latencies that the neighbouring kernels' PDL overlap does not (an isolated
// kernel can favour a larger E).  BK_FFT_LOGE overrides (2..5).
static int fast_loge(long long n) {
  static const int e = [] {  // read once; thread-safe initialisation
    const char* a = getenv("BK_FFT_LOGE");
    const int v = a ? atoi(a) : 0;
    return v < 2 || v > 5 ? 0 : v;
  }();
  if (e) return e;
  return n >= 1024 ? 3 : 2;
}
static int fast_logn(long long n) {
  static const int off = getenv("BK_FFT_NO_FAST") ? 1 : 0;  // diagnostics: force the general kernel everywhere; read once
  if (off) return 0;
  for (int l = fast_loge(n) + 1; l <= 11; ++l)
    if (l >= 6 && n == (1LL << l)) return l;
  return 0;
}
#define BKF_DISPATCH_N(LE, LOGN, ...)                                                   \
  switch (LOGN) {                                                                      \
    case 6: { using FC = bkf::Cfg<6, LE>; __VA_ARGS__; } break;                        \
    case 7: { using FC = bkf::Cfg<7, LE>; __VA_ARGS__; } break;                        \
    case 8: { using FC = bkf::Cfg<8, LE>; __VA_ARGS__; } break;                        \
    case 9: { using FC = bkf::Cfg<9, LE>; __VA_ARGS__; } break;                        \
    case 10: { using FC = bkf::Cfg<10, LE>; __VA_ARGS__; } break;                      \
    default: { using FC = bkf::Cfg<11, LE>; __VA_ARGS__; } break;                      \
  }
#define BKF_DISPATCH(LOGN, ...)                                                        \
  switch (fast_loge(1LL << (LOGN))) {                                                               \
    case 2: BKF_DISPATCH_N(2, LOGN, __VA_ARGS__) break;                                \
    case 3: BKF_DISPATCH_N(3, LOGN, __VA_ARGS__) break;                                \
    case 4: BKF_DISPATCH_N(4, LOGN, __VA_ARGS__) break;                                \
    default: BKF_DISPATCH_N(5, LOGN, __VA_ARGS__) break;                               \
  }

// strided: mode 0 forward (2 C), 1 inverse (n x), 2 fused forward + symbol + inverse, 3 periodic fused y pass;
// contiguous: mode 0 forward, 1 inverse, 2 periodic r2c, 3 periodic c2r (prologue / epilogue pw)
static int fast_launch(bk_ctx* c, const Line& ln, bool strided, int mode, const double* in, double* out, const bkf::Geom& g,
                       const bkf::Symbol* sy, const PerPw* pw = nullptr) {
  bkf::Tables tb{ln.ftw, ln.fom, ln.flam2};
  bkf::Symbol s0{};
  if (sy) s0 = *sy;
  PerPw p0{};
  if (pw) p0 = *pw;
  int st;
  BKF_DISPATCH(ln.fast, {
    if (strided) {
      static decltype(&bkf::k_strided<FC, 0>) const kern[4] = {bkf::k_strided<FC, 0>, bkf::k_strided<FC, 1>, bkf::k_strided<FC, 2>,
                                                               bkf::k_strided<FC, 3>};
      const dim3 grid((g.nb + 2 * FC::PP - 1) / (2 * FC::PP), g.nouter);
      st = bk_launch(c, kern[mode], grid, dim3(FC::THREADS), mode >= 2 ? FC::SMEM_FUSED : FC::SMEM, in, out, g, tb, s0);
    } else {
      static decltype(&bkf::k_contig<FC, 0>) const kern[4] = {bkf::k_contig<FC, 0>, bkf::k_contig<FC, 1>, bkf::k_contig<FC, 2>,
                                                              bkf::k_contig<FC, 3>};
      const dim3 grid((unsigned)((g.nb + 2 * FC::PP - 1) / (2 * FC::PP)));
      st = bk_launch(c, kern[mode], grid, dim3(FC::THREADS), FC::SMEM, in, out, g, tb, p0);
    }
  });
  return st;
}

// ---- general path ----------------------------------------------------------------------------------------------------------
static void factorize(int L, bkg::Plan& pl) {
  pl.npass = 0;
  while (L % 4 == 0 && pl.npass < BKG_MAXPASS) {
    pl.radix[pl.npass++] = 4;
    L /= 4;
  }
  for (int p = 2; L > 1 && pl.npass < BKG_MAXPASS; ++p)
    while (L % p == 0 && pl.npass < BKG_MAXPASS) {
      pl.radix[pl.npass++] = p;
      L /= p;
    }
}
#define BKG_THREADS 512
#define BKG_SMEM_BUDGET (100 * 1024)   // two CTAs per SM
#define BKG_SMEM_MAX (200 * 1024)
static int gen_ppg(int L) {
  long long per = 32LL * L;  // two buffers of L complex values per pair
  int p = (int)(BKG_SMEM_BUDGET / per);
  if (p < 1) p = 1;
  if (p > 8) p = 8;
  return p;
}

static int gen_setup(bk_ctx* c, Line& ln) {
  bkg::Plan& pl = ln.plan;
  const int n = ln.n;
  pl.n = n;
  pl.L = ln.type == 0 ? 2 * n : 2 * n + 2;
  BK_CHECK(c, 32LL * pl.L <= BKG_SMEM_MAX, "line too long for the general transform kernel (n <= 3199)");
  factorize(pl.L, pl);
  const long double PI = 3.14159265358979323846264338327950288L;
  std::vector<double> wl(2 * (size_t)pl.L), ph(2 * (size_t)n);
  for (int t = 0; t < pl.L; ++t) {
    wl[2 * t] = (double)cosl(-2.0L * PI * t / pl.L);
    wl[2 * t + 1] = (double)sinl(-2.0L * PI * t / pl.L);
  }
  for (int k = 0; k < n; ++k) {
    ph[2 * k] = (double)cosl(-PI * k / (2.0L * n));
    ph[2 * k + 1] = (double)sinl(-PI * k / (2.0L * n));
  }
  BK_TRY(upload(c, (void**)&ln.gwl, wl.data(), 8 * wl.size()));
  BK_TRY(upload(c, (void**)&ln.gph, ph.data(), 8 * ph.size()));
  pl.wl = ln.gwl;
  pl.ph = ln.gph;
  pl.dst_scale = 0.5 * sqrt(2.0 / (n + 1.0));
  return BK_OK;
}

// mode 0 DCT forward (2 C), 1 DCT inverse (n x), 2 DST-I (orthonormal)
static int gen_launch(bk_ctx* c, const Line& ln, bool strided, int mode, const double* in, double* out, const bkf::Geom& g) {
  const bkg::Plan& pl = ln.plan;
  const int ppg = gen_ppg(pl.L);
  const size_t sm = 32 * (size_t)pl.L * ppg;
  const long long npairs = ((long long)g.nb + 1) / 2;
  dim3 grid((unsigned)((npairs + ppg - 1) / ppg), strided ? g.nouter : 1);
  static decltype(&bkg::k_gen<false, 0>) const kern[2][3] = {{bkg::k_gen<false, 0>, bkg::k_gen<false, 1>, bkg::k_gen<false, 2>},
                                                              {bkg::k_gen<true, 0>, bkg::k_gen<true, 1>, bkg::k_gen<true, 2>}};
  return bk_launch(c, kern[strided][mode], grid, dim3(BKG_THREADS), sm, in, out, g, pl, ppg);
}

// The transform of one dimension: its eigenvalues lam (n = lam.size()) and the tables of the kernels that may run it.  The
// fast kernels take DCT-II lines of a power-of-two length whose grid rows hold an even number of values (16-byte accesses);
// with `general` the line also gets the general plan, which unaligned vectors fall back to.  Without it (the periodic
// pipeline, which has no general kernel) the line is a power of two and always runs on the fast kernels.
static int line_setup(bk_ctx* c, Line& ln, int type, const std::vector<double>& lam, bool general) {
  const long long n = (long long)lam.size();
  ln.n = (int)n;
  ln.type = type;
  BK_TRY(upload(c, (void**)&ln.lam, lam.data(), 8 * n));
  if (general) {
    ln.fast = (type == 0 && c->dims[0] % 2 == 0) ? fast_logn(n) : 0;
  } else {
    ln.fast = 0;
    while ((1LL << ln.fast) < n) ++ln.fast;
  }
  if (ln.fast) {
    std::vector<double> tw, om, lam2;
    BKF_DISPATCH(ln.fast, bkf::build_tables<FC>(tw, om, lam2, lam.data()));
    if (tw.empty()) tw.assign(2, 0.0);
    BK_TRY(upload(c, (void**)&ln.ftw, tw.data(), 8 * tw.size()));
    BK_TRY(upload(c, (void**)&ln.fom, om.data(), 8 * om.size()));
    BK_TRY(upload(c, (void**)&ln.flam2, lam2.data(), 8 * lam2.size()));
  }
  return general ? gen_setup(c, ln) : BK_OK;
}

void line_free(Line& ln) {
  void* tabs[] = {ln.lam, ln.ftw, ln.fom, ln.flam2, ln.gwl, ln.gph};
  for (void* t : tabs)
    if (t) cudaFree(t);
}

// the eigenvalues of dimension d of a grid Laplacian. type 0: DCT-II (Neumann), 1: DST-I (Dirichlet)
static std::vector<double> dim_eigenvalues(const bk_ctx* c, int d, int type) {
  const long long n = c->dims[d];
  const double inv_h2 = bk_inv_h2(c, d);
  std::vector<double> lam(n);
  const long double PI = 3.14159265358979323846264338327950288L;
  for (long long k = 0; k < n; ++k)
    lam[k] = (type == 0) ? (double)((2.0L * cosl(PI * k / n) - 2.0L)) * inv_h2
                         : (double)(-(2.0L - 2.0L * cosl(PI * (k + 1) / (n + 1)))) * inv_h2;
  return lam;
}
// the transform of dimension d of a grid Laplacian
static int setup_dim(bk_ctx* c, int d, int type) { return line_setup(c, c->pc.line[d], type, dim_eigenvalues(c, d, type), true); }

// ---- BK_SH2D_PERIODIC: real 2-D FFT pipeline -------------------------------------------------------------------------------
// Tables for both dimensions are built once at bk_ctx_create: every operator application (residual, JVP, preconditioner, the
// one-transform preconditioned operator) is  x r2c (k_contig MODE 2) -> y forward * symbol * inverse (k_strided MODE 3) ->
// x c2r (k_contig MODE 3), through the two work buffers.  Periodic eigenvalues of the Laplacian: lambda[k] = -(pi k / l)^2 with
// the signed frequency k (examples/SH2d-fronts-cuda.jl:48-50).
int bk_periodic_setup(bk_ctx* c) {
  Precond& pc = c->pc;
  const long double PI = 3.14159265358979323846264338327950288L;
  for (int d = 0; d < 2; ++d) {
    const long long n = c->dims[d];
    std::vector<double> lam(n);
    for (long long k = 0; k < n; ++k) {
      const long double ks = (long double)(k <= n / 2 ? k : k - n), w = PI * ks / (long double)c->lengths[d];
      lam[k] = (double)(-w * w);
    }
    BK_TRY(line_setup(c, pc.line[d], 0, lam, false));
  }
  if (!pc.work) BK_CUDA(c, cudaMalloc(&pc.work, 8 * (size_t)c->ld));
  if (!pc.work2) BK_CUDA(c, cudaMalloc(&pc.work2, 8 * (size_t)c->ld));
  return BK_OK;
}

// out = epilogue(F^-1 sigma F prologue(in)), sigma = gain / (Nx Ny) * (neg ? -L1 : 1 / (L1 + shift)); 3 kernels, 64N bytes at most.
// The y pass also copies the border entries of `tail` (border_tail).
static int periodic_pipeline(bk_ctx* c, const double* in, double* out, const PerPw& pw, bool neg, double gain, double shift,
                             const bkf::Symbol& tail = {}) {
  Precond& pc = c->pc;
  const int nx = (int)c->dims[0], ny = (int)c->dims[1];
  const bkf::Geom gx{1, nx, ny, 1}, gy{nx, (long long)nx * ny, nx, 1};
  const bkf::Symbol sy{pc.line[0].lam, nullptr, shift, gain / ((double)nx * (double)ny), tail.tail_src, tail.tail_dst, tail.tail_n,
                       neg ? 1 : 0};
  BK_TRY(fast_launch(c, pc.line[0], false, 2, in, pc.work, gx, nullptr, &pw));
  BK_TRY(fast_launch(c, pc.line[1], true, 3, pc.work, pc.work2, gy, &sy));
  return fast_launch(c, pc.line[0], false, 3, pc.work2, out, gx, nullptr, &pw);
}

int bk_periodic_residual(bk_ctx* c, const OpDesc& op, const double* u, double* out) {
  const PerPw pw{0, PW_RESID, u, nullptr, nullptr, 0.0, 0.0, op.par[0], op.par[1], 0.0};
  return periodic_pipeline(c, u, out, pw, true, 1.0, 0.0);
}
int bk_periodic_jvp(bk_ctx* c, const OpDesc& op, const double* in, const double* sp, double* out) {
  const PerPw pw{0, PW_JVP, in, op.u, sp, op.a0, op.a1, op.par[0], op.par[1], 0.0};
  return periodic_pipeline(c, in, out, pw, true, op.a1, 0.0);
}
int bk_periodic_fused(bk_ctx* c, const OpDesc& op, const double* in, const double* sp, double* out, bool left) {
  BK_CHECK(c, c->pc.kind == BK_PC_SH_FFT && !op.bordered && !op.cplx, "internal: one-transform operator needs BK_PC_SH_FFT, unbordered, real");
  const PerPw pw{left ? PW_D : 0, left ? PW_FLEFT : PW_FRIGHT, in, op.u, sp, op.a0, op.a1, op.par[0], op.par[1], c->pc.a0};
  return periodic_pipeline(c, in, out, pw, false, 1.0, c->pc.a0);
}

extern "C" int32_t bk_precond_setup(bk_ctx* c, int32_t kind, double a0, double a1) {
  BK_ENTER(c);
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  Precond& pc = c->pc;
  if (kind == BK_PC_NONE) {
    pc.kind = BK_PC_NONE;
    return BK_OK;
  }
  if (!pc.work) BK_CUDA(c, cudaMalloc(&pc.work, 8 * (size_t)c->ld));
  if (!pc.work2) BK_CUDA(c, cudaMalloc(&pc.work2, 8 * (size_t)c->ld));
  if (kind == BK_PC_SH_DCT) {
    BK_CHECK(c, c->kind == BK_SH2D || c->kind == BK_SH3D, "BK_PC_SH_DCT needs a Swift-Hohenberg context");
    for (int d = 0; d < bk_traits(c)->ndims; ++d) BK_TRY(setup_dim(c, d, 0));
  } else if (kind == BK_PC_SH_FFT) {
    BK_CHECK(c, c->kind == BK_SH2D_PERIODIC, "BK_PC_SH_FFT needs a BK_SH2D_PERIODIC context");
    BK_CHECK(c, a0 > 0, "BK_PC_SH_FFT: a0 must be > 0 (the symbol of L1 vanishes at |k| = 1)");
    // tables and work buffers are the context's own (bk_periodic_setup)
  } else if (kind == BK_PC_CGL_DST) {
    BK_CHECK(c, c->kind == BK_CGL2D || c->kind == BK_POTRAP_CGL2D, "BK_PC_CGL_DST needs a cGL context");
    for (int d = 0; d < 2; ++d) BK_TRY(setup_dim(c, d, 1));
  } else if (kind == BK_PC_POTRAP_CIRC) {
    BK_CHECK(c, c->kind == BK_POTRAP_CGL2D, "BK_PC_POTRAP_CIRC needs a Trapeze (potrap) context");
    const int K = (int)c->dims[2] - 1;
    BK_CHECK(c, K >= 1 && K <= BK_PO_KMAX, "BK_PC_POTRAP_CIRC supports 2 <= M <= 65 time slices");
    BK_CHECK(c, a0 > 0, "BK_PC_POTRAP_CIRC: a0 must be the period T > 0");
    for (int d = 0; d < 2; ++d) BK_TRY(setup_dim(c, d, 1));
    std::vector<double2> tw(K);
    const long double PI = 3.14159265358979323846264338327950288L;
    for (int j = 0; j < K; ++j) tw[j] = make_double2((double)cosl(-2.0L * PI * j / K), (double)sinl(-2.0L * PI * j / K));
    BK_TRY(upload(c, (void**)&pc.tdft, tw.data(), 16 * (size_t)K));
    pc.po_T = a0;
    pc.po_r = c->par[0];   // (r, mu, nu, c3, c5)
    pc.po_nu = c->par[2];
  } else if (kind == BK_PC_RD) {
    BK_CHECK(c, c->kind == BK_RD, "BK_PC_RD needs a BK_RD context");
    const int nd = bk_traits(c)->ndims, type = c->rd_model.bc == BK_BC_DIRICHLET ? 1 : 0;
    std::vector<double> lam[2] = {dim_eigenvalues(c, 0, type), nd == 2 ? dim_eigenvalues(c, 1, type) : std::vector<double>(1, 0.0)};
    // a vanishing symbol a0 + a1 D_f lambda has no inverse; one that cancels to rounding level is treated as vanishing.  Every
    // field is checked before anything of the context's preconditioner changes, so a refused set-up leaves the previous one intact
    for (int f = 0; f < bk_traits(c)->fields; ++f) {
      const double df = c->rd_par.diff[f];
      for (double ly : lam[1])
        for (double lx : lam[0]) {
          const double t = a1 * df * (lx + ly);
          BK_CHECK(c, std::isfinite(a0 + t) && fabs(a0 + t) > 1e-13 * (fabs(a0) + fabs(t)),
                   "BK_PC_RD: the symbol a0 + a1 D_i lambda vanishes for a mode of the grid (no inverse)");
        }
    }
    for (int d = 0; d < nd; ++d) BK_TRY(setup_dim(c, d, type));
    for (int f = 0; f < bk_traits(c)->fields; ++f) pc.rd_diff[f] = c->rd_par.diff[f];
  } else if (kind == BK_PC_CHAN_TRIDIAG) {
    BK_CHECK(c, c->kind == BK_CHAN, "BK_PC_CHAN_TRIDIAG needs a chan context");
    long long n = c->N0;
    double s = (double)(n - 1) * (double)(n - 1);
    std::vector<double> lo(n, s), di(n, -2 * s), up(n, s), tri(3 * n);
    di[0] = 1;
    up[0] = 0;
    lo[n - 1] = 0;
    di[n - 1] = 1;  // P[1,1:2] = [1,0]; P[end,end-1:end] = [0,1]  (chan.jl:109)
    lo[0] = 0;
    up[n - 1] = 0;
    // forward elimination factors
    double denom = di[0];
    tri[n + 0] = 1.0 / denom;
    tri[0] = up[0] / denom;
    for (long long i = 1; i < n; ++i) {
      denom = di[i] - lo[i] * tri[i - 1];
      tri[n + i] = 1.0 / denom;
      tri[i] = up[i] / denom;
      tri[2 * n + i] = lo[i];
    }
    BK_TRY(upload(c, (void**)&pc.tri, tri.data(), 8 * 3 * n));
  } else {
    return bk_fail(c, BK_ERR_ARG, "unknown preconditioner kind", __FILE__, __LINE__);
  }
  pc.kind = kind;
  pc.a0 = a0;
  pc.a1 = a1;
  return BK_OK;
}

// one 1-D transform pass of line ln along dimension d over fields of nx * ny * nz values.
// mode 0: forward, 1: inverse; fused != NULL (fast path): forward + symbol + inverse in one kernel.  The fast kernels run when the
// line has them and in / out are 16-byte aligned, the general kernel otherwise.
// Conventions: DCT forward returns 2 C, DCT inverse returns n x (the caller's symbol carries 1 / prod(2 n_d)); DST-I is orthonormal.
static int transform_pass(bk_ctx* c, const Line& ln, int d, int mode, const double* in, double* out, int nx, int ny, int nz,
                          bool aligned, const bkf::Symbol* fused = nullptr) {
  bkf::Geom g;
  bool strided = d != 0;
  if (d == 0) {
    g.es = 1;
    g.os = nx;
    g.nb = ny * nz;  // number of lines
    g.nouter = 1;
  } else if (d == 1) {
    g.es = nx;
    g.nb = nx;
    g.os = (long long)nx * ny;
    g.nouter = nz;
  } else {
    g.es = (long long)nx * ny;
    g.nb = nx;
    g.os = nx;
    g.nouter = ny;
  }
  if (ln.fast && aligned) return fast_launch(c, ln, strided, fused ? 2 : mode, in, out, g, fused);
  BK_CHECK(c, !fused, "internal: fused transform on the general path");
  return gen_launch(c, ln, strided, ln.type == 1 ? 2 : mode, in, out, g);
}

static inline bool aligned16(const void* a, const void* b) { return ((((uintptr_t)a) | ((uintptr_t)b)) & 15) == 0; }

// Border entries behind the N grid values of an n-vector ride along with a transform kernel that can carry them (up to 32, in
// its symbol sy); returns whether they do.  Otherwise precond_apply_one copies them.
static bool border_tail(bkf::Symbol& sy, const double* in, double* out, long long n, long long N) {
  if (n <= N || n - N > 32) return false;
  sy.tail_src = in + N;
  sy.tail_dst = out + N;
  sy.tail_n = (int)(n - N);
  return true;
}

// A spectral solve along the first nd dimensions of fields of nx * ny * nz values, in to out: forward passes d = 0 .. nd-1, the
// middle step in the transformed basis, inverse passes d = nd-1 .. 0, each pass from one work buffer to the other.  Only the
// first and the last pass touch in / out, so only they take the caller's alignment al.  A middle step the fast kernels can fuse
// comes as its symbol sy (SH_DCT): it is fused into the last forward pass when that pass is on the fast path and al holds, and
// the border entries of the n-vector then ride along (sy->tail_n > 0).  Otherwise mid(buffer) applies it in place.
template <class Mid>
static int spectral_solve(bk_ctx* c, int nd, int nx, int ny, int nz, const double* in, double* out, long long n, bool al,
                          bkf::Symbol* sy, Mid mid) {
  const Line* ln = c->pc.line;
  double* buf[2] = {c->pc.work, c->pc.work2};
  const bool fuse = sy && ln[nd - 1].fast && al;
  if (fuse) border_tail(*sy, in, out, n, c->N0);
  const int npass = fuse ? 2 * nd - 1 : 2 * nd;
  int p = 0;
  auto pass = [&](int d, int mode, const bkf::Symbol* fused) {
    const bool edge = p == 0 || p == npass - 1;
    const double* src = p == 0 ? in : buf[(p - 1) & 1];
    double* dst = p == npass - 1 ? out : buf[p & 1];
    ++p;
    return transform_pass(c, ln[d], d, mode, src, dst, nx, ny, nz, edge ? al : true, fused);
  };
  for (int d = 0; d < nd; ++d) BK_TRY(pass(d, 0, fuse && d == nd - 1 ? sy : nullptr));
  if (!fuse) BK_TRY(mid(buf[(nd - 1) & 1]));
  for (int d = fuse ? nd - 2 : nd - 1; d >= 0; --d) BK_TRY(pass(d, 1, nullptr));
  return BK_OK;
}

static int precond_apply_one(bk_ctx* c, const double* in, double* out, long long n);

int bk_precond_apply_dev(bk_ctx* c, const double* in, double* out, long long n) {
  BK_CHECK(c, c->pc.kind != BK_PC_NONE, "no preconditioner set up (bk_precond_setup)");
  BK_CHECK(c, in != out, "preconditioner: in-place application is not supported");
  if (!c->cplx) return precond_apply_one(c, in, out, n);
  // split complex vector: the real preconditioner on both halves (border entries, if any, follow the second half)
  BK_CHECK(c, n >= c->N, "preconditioner: vector shorter than the complexified problem");
  BK_TRY(precond_apply_one(c, in, out, c->N0));
  return precond_apply_one(c, in + c->N0, out + c->N0, n - c->N0);
}

static int precond_apply_one(bk_ctx* c, const double* in, double* out, long long n) {
  Precond& pc = c->pc;
  const Line* ln = pc.line;
  const long long N = c->N0;
  bool tail_done = false;
  const bool timed = c->timing_now;  // per-application device time for bench.py's breakdown
  if (timed) c->pc_timer.begin(c->stream);
  const bool al = aligned16(in, out);
  if (pc.kind == BK_PC_SH_DCT) {
    const int nd = bk_traits(c)->ndims;
    const int nx = (int)c->dims[0], ny = (int)c->dims[1], nz = nd == 3 ? (int)c->dims[2] : 1;
    double scale = 1.0;
    for (int d = 0; d < nd; ++d) scale /= 2.0 * (double)c->dims[d];
    bkf::Symbol sy{ln[0].lam, nd == 3 ? ln[1].lam : nullptr, pc.a0, scale, nullptr, nullptr, 0};
    BK_TRY(spectral_solve(c, nd, nx, ny, nz, in, out, n, al, &sy, [&](double* v) {
      return bk_launch_ordered(c, k_sh_symbol_div, bk_lin_grid(c, N), 256, 0, v, nx, ny, nz, ln[0].lam, ln[1].lam,
                               nd == 3 ? ln[2].lam : nullptr, pc.a0, scale);
    }));
    tail_done = sy.tail_n > 0;
  } else if (pc.kind == BK_PC_SH_FFT) {
    bkf::Symbol tail{};
    tail_done = border_tail(tail, in, out, n, N);
    const PerPw pw{0, PW_NONE, in, nullptr, nullptr, 0.0, 0.0, 0.0, 0.0, 0.0};
    BK_TRY(periodic_pipeline(c, in, out, pw, false, 1.0, pc.a0, tail));
  } else if (pc.kind == BK_PC_CGL_DST) {
    const int nx = (int)c->dims[0], ny = (int)c->dims[1];
    const long long nblk = (c->kind == BK_POTRAP_CGL2D) ? 2 * c->dims[2] : 2;  // components x slices
    BK_TRY(spectral_solve(c, 2, nx, ny, (int)nblk, in, out, n, al, nullptr, [&](double* v) {
      return bk_launch_ordered(c, k_helmholtz_symbol_div, bk_lin_grid(c, (long long)nx * ny * nblk), 256, 0, v, nx, ny, nblk,
                               ln[0].lam, ln[1].lam, pc.a0, pc.a1);
    }));
    if (c->kind == BK_POTRAP_CGL2D) BK_CUDA(c, cudaMemcpyAsync(out + N - 1, in + N - 1, 8, cudaMemcpyDeviceToDevice, c->stream));
  } else if (pc.kind == BK_PC_POTRAP_CIRC) {
    const int nx = (int)c->dims[0], ny = (int)c->dims[1], M = (int)c->dims[2];
    const long long nn = (long long)nx * ny, Ns = 2 * nn;
    // DST-I in space over all 2M slice components (mixed-radix FFT of the odd extension, bk_fft_gen.cuh), the circulant
    // solve in time per spatial mode, DST-I back.  While J' is selected (bk_jac_set_transpose) this is P'^-1: the transposed
    // time solve, then x_M = r_M and the period entry pass through (one copy: they are the last Ns + 1 entries).
    BK_TRY(spectral_solve(c, 2, nx, ny, 2 * M, in, out, n, al, nullptr, [&](double* v) {
      return bk_launch_ordered(c, c->transpose ? k_potrap_time<true> : k_potrap_time<false>, (unsigned)((nn + 127) / 128), 128, 0,
                               v, nn, nx, M - 1, ln[0].lam, ln[1].lam, pc.po_T / M, pc.po_r, pc.po_nu, pc.tdft);
    }));
    if (c->transpose)
      BK_CUDA(c, cudaMemcpyAsync(out + (M - 1) * Ns, in + (M - 1) * Ns, 8 * (size_t)(Ns + 1), cudaMemcpyDeviceToDevice, c->stream));
    else
      BK_TRY(bk_launch_ordered(c, k_potrap_close, (unsigned)((Ns + 255) / 256), 256, 0, in, out, Ns, M));
  } else if (pc.kind == BK_PC_RD) {
    const int nd = bk_traits(c)->ndims, nx = (int)c->dims[0], ny = (int)c->dims[1], F = bk_traits(c)->fields;
    double scale = 1.0;
    if (c->rd_model.bc == BK_BC_NEUMANN)
      for (int d = 0; d < nd; ++d) scale /= 2.0 * (double)c->dims[d];
    RdDiff D;
    for (int f = 0; f < BK_RD_MAX_FIELDS; ++f) D.d[f] = pc.rd_diff[f];
    BK_TRY(spectral_solve(c, nd, nx, ny, F, in, out, n, al, nullptr, [&](double* v) {
      return bk_launch_ordered(c, k_rd_symbol_div, bk_lin_grid(c, N), 256, 0, v, nx, ny, F, ln[0].lam, nd == 2 ? ln[1].lam : nullptr,
                               pc.a0, pc.a1, D, scale);
    }));
  } else if (pc.kind == BK_PC_CHAN_TRIDIAG) {
    BK_TRY(bk_launch_ordered(c, k_thomas, 1, 32, 0, pc.tri, in, out, (int)N));
  }
  if (n > N && !tail_done)
    BK_CUDA(c, cudaMemcpyAsync(out + N, in + N, 8 * (size_t)(n - N), cudaMemcpyDeviceToDevice, c->stream));
  if (timed) c->pc_timer.end(c->stream);
  return BK_OK;
}

extern "C" int32_t bk_precond_apply(bk_ctx* c, const double* in, double* out) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_precond_apply");
  double *din, *dout;
  BK_TRY(bk_stage_in(c, in, c->N, 10, true, &din));
  BK_TRY(bk_stage_in(c, out, c->N, 11, false, &dout));
  BK_TRY(bk_precond_apply_dev(c, din, dout, c->N));
  return bk_stage_out(c, out, c->N, dout);
}
