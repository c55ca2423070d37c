// bk_problems.cu -- K1/K2: residual F(u;p) and Jacobian-vector product a0 v + a1 J(u) v of the
// named PDE stencils as stand-alone kernels, the MatrixFreeBLS bordered map (K2') and the
// trapezoid periodic-orbit functional (K7).  Reference definitions:
//   P1 examples/chan.jl:5-19,85-95        P2 examples/SH2d-fronts.jl:13-34,124-127
//   P3 examples/SH3d.jl:16-53             P4 examples/cGL2d.jl:6-22,262-318
//   P5 src/periodicorbit/PeriodicOrbitTrapeze.jl:209-330,362-386
//   bordered map src/LinearBorderSolver.jl:299-335
// Also the jets d2F / d3F (k_jet) and their contractions (k_jet_moments), which share one per-point form per kind (jet_form),
// and the deflation moments.  Every cGL2d point, stand-alone or a Trapeze slice, is cgl_point on the one Dirichlet stencil
// (lap_dirichlet); the Trapeze kernels split their flat index with trap_point, and k_potrap_section writes both the section
// and the F-cache.  bk_jet_moments and bk_deflation_moments share their host plumbing: staging (stage_rows), the work buffer
// (moment_work) and the read-back through a pinned buffer (moment_results).
#include <algorithm>
#include <cstring>

#include "bk_common.cuh"
#include "bk_stencil.cuh"
#include "bk_krylov_tma.cuh"

// ------------------------------------------------------------------------------------------ SH
template <int DIM, int MODE>
static __global__ void __launch_bounds__(BK_THREADS) k_sh_apply(OpDesc op, const double* __restrict__ in,
                                                                const double* __restrict__ in_scale_ptr,
                                                                double* __restrict__ out) {
  extern __shared__ double smem[];
  double val[BK_EPT];
  long long off[BK_EPT];
  double s = in_scale_ptr ? __ldg(in_scale_ptr) : 1.0;
  sh_tile_eval<DIM, MODE>(op, in, s, smem, val, off);
#pragma unroll
  for (int e = 0; e < BK_EPT; ++e)
    if (off[e] >= 0) out[off[e]] = val[e];
}

// ------------------------------------------------------------------------------------------ chan
__device__ __forceinline__ double chan_Nl(double x, double b) { return 1.0 + (x + 0.5 * x * x) / (1.0 + b * x * x); }
__device__ __forceinline__ double chan_dNl(double x, double b) {
  double d = 1.0 + b * x * x;
  return (1.0 - b * x * x + 2.0 * 0.5 * x) / (d * d);
}
// MODE 0 JVP, 1 residual
template <int MODE>
static __global__ void __launch_bounds__(256) k_chan_apply(OpDesc op, const double* __restrict__ in,
                                                           const double* __restrict__ in_scale_ptr,
                                                           double* __restrict__ out) {
  const int n = op.nx;
  const double alpha = op.par[0], beta = op.par[1];
  const double s = in_scale_ptr ? __ldg(in_scale_ptr) : 1.0;
  const double h2 = (double)(n - 1) * (double)(n - 1);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    double v = s * in[i];
    double r;
    if (i == 0 || i == n - 1) {
      r = (MODE == 0) ? v : v - beta;
    } else {
      double lap = (s * in[i - 1] - 2.0 * v + s * in[i + 1]) * h2;
      r = (MODE == 0) ? lap + alpha * chan_dNl(op.u[i], beta) * v : lap + alpha * chan_Nl(v, beta);
    }
    out[i] = (MODE == 0) ? op.a0 * v + op.a1 * r : r;
  }
}

// ------------------------------------------------------------------------------------------ cGL
struct CglPar {
  double r, mu, nu, c3, c5;
};
__device__ __forceinline__ void cgl_nl(const CglPar& p, double u1, double u2, double& f1, double& f2) {
  double ua = u1 * u1 + u2 * u2;
  f1 = p.r * u1 - p.nu * u2 - ua * (p.c3 * u1 - p.mu * u2) - p.c5 * ua * ua * u1;
  f2 = p.r * u2 + p.nu * u1 - ua * (p.c3 * u2 + p.mu * u1) - p.c5 * ua * ua * u2;
}
template <bool TR = false>
__device__ __forceinline__ void cgl_dnl(const CglPar& p, double u1, double u2, double d1, double d2, double& f1,
                                        double& f2) {
  double u12 = u1 * u1, u22 = u2 * u2;
  double a11 = -5 * p.c5 * u12 * u12 + (-6 * p.c5 * u22 - 3 * p.c3) * u12 + 2 * p.mu * u1 * u2 - p.c5 * u22 * u22 -
               p.c3 * u22 + p.r;
  double a12 = -4 * p.c5 * u2 * u12 * u1 + p.mu * u12 + (-4 * p.c5 * u22 * u2 - 2 * p.c3 * u2) * u1 + 3 * u22 * p.mu - p.nu;
  double a21 = -4 * p.c5 * u2 * u12 * u1 - 3 * p.mu * u12 + (-4 * p.c5 * u22 * u2 - 2 * p.c3 * u2) * u1 - u22 * p.mu + p.nu;
  double a22 = -p.c5 * u12 * u12 + (-6 * p.c5 * u22 - p.c3) * u12 - 2 * p.mu * u1 * u2 - 5 * p.c5 * u22 * u22 -
               3 * p.c3 * u22 + p.r;
  f1 = a11 * d1 + (TR ? a21 : a12) * d2;  // TR: J' (the Laplacian is symmetric, only this 2 x 2 block changes)
  f2 = (TR ? a12 : a21) * d1 + a22 * d2;
}
// Dirichlet 5-point Laplacian (zero ghost cells; diagonal -2/h^2 everywhere, examples/cGL2d.jl:12-16) of the field whose value
// at point g is at(g): one field, or the sum of two (one stencil evaluation for the two slices of a J' row)
template <typename At>
__device__ __forceinline__ double lap_dirichlet(At at, int i, int j, int nx, int ny, double cx, double cy, double s) {
  const long long g = i + (long long)j * nx;
  const double c = at(g);
  const double xm = i > 0 ? at(g - 1) : 0.0, xp = i < nx - 1 ? at(g + 1) : 0.0;
  const double ym = j > 0 ? at(g - nx) : 0.0, yp = j < ny - 1 ? at(g + nx) : 0.0;
  return s * (cx * (xm - 2.0 * c + xp) + cy * (ym - 2.0 * c + yp));
}
struct Field {
  const double* __restrict__ a;
  __device__ __forceinline__ double operator()(long long g) const { return a[g]; }
};
struct FieldSum {
  const double* __restrict__ a;
  const double* __restrict__ b;
  __device__ __forceinline__ double operator()(long long g) const { return a[g] + b[g]; }
};
// Vector field / JVP at one grid point of one slice: base pointers to the slice's [u1;u2].
template <int MODE, bool TR = false>
__device__ __forceinline__ void cgl_point(const CglPar& p, const double* __restrict__ u, const double* __restrict__ v,
                                          double s, int i, int j, int nx, int ny, double cx, double cy, double& o1,
                                          double& o2) {
  const long long n = (long long)nx * ny, g = i + (long long)j * nx;
  if (MODE == 1) cgl_nl(p, s * v[g], s * v[g + n], o1, o2);
  else cgl_dnl<TR>(p, u[g], u[g + n], s * v[g], s * v[g + n], o1, o2);
  o1 += lap_dirichlet(Field{v}, i, j, nx, ny, cx, cy, s);
  o2 += lap_dirichlet(Field{v + n}, i, j, nx, ny, cx, cy, s);
}
__device__ __forceinline__ CglPar cgl_par(const OpDesc& op) {
  CglPar p;
  p.r = op.par[0];
  p.mu = op.par[1];
  p.nu = op.par[2];
  p.c3 = op.par[3];
  p.c5 = op.par[4];
  return p;
}
// Point q < n M of a Trapeze orbit (n = nx ny points, M slices of Ns = 2 n values): grid point g = i + j nx of slice sl, whose
// first field is at o = sl Ns + g.  i and j are formed where they are used (k_potrap_apply_tr spills if they live longer).
struct TrapPoint {
  long long g, o;
  int sl;
  __device__ __forceinline__ int i(int nx) const { return (int)(g % nx); }
  __device__ __forceinline__ int j(int nx) const { return (int)(g / nx); }
};
__device__ __forceinline__ TrapPoint trap_point(long long q, long long n) {
  TrapPoint t;
  t.g = q % n;
  t.sl = (int)(q / n);
  t.o = (long long)t.sl * (2 * n) + t.g;
  return t;
}

template <int MODE>
static __global__ void __launch_bounds__(256) k_cgl_apply(OpDesc op, const double* __restrict__ in,
                                                          const double* __restrict__ in_scale_ptr,
                                                          double* __restrict__ out) {
  const int nx = op.nx, ny = op.ny;
  const long long n = (long long)nx * ny;
  const double s = in_scale_ptr ? __ldg(in_scale_ptr) : 1.0;
  const CglPar p = cgl_par(op);
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += (long long)gridDim.x * blockDim.x) {
    int i = (int)(g % nx), j = (int)(g / nx);
    double o1, o2;
    if (MODE == 0 && op.transpose) cgl_point<MODE, true>(p, op.u, in, s, i, j, nx, ny, op.cx, op.cy, o1, o2);
    else cgl_point<MODE>(p, op.u, in, s, i, j, nx, ny, op.cx, op.cy, o1, o2);
    if (MODE == 0) {
      out[g] = op.a0 * s * in[g] + op.a1 * o1;
      out[g + n] = op.a0 * s * in[g + n] + op.a1 * o2;
    } else {
      out[g] = o1;
      out[g + n] = o2;
    }
  }
}

// ------------------------------------------------------------------------------------------ potrap over cGL
// x = [x_1 .. x_M ; T], slice length Ns = 2 nx ny.  Rows i = 1..M-1: (x_i - x_{i-1}) - h/2 (F(x_i) + F(x_{i-1})),
// x_0 == x_{M-1}; row M: x_M - x_1; last: <x - xpi, phi>  (phase condition written by a second kernel).
// MODE 1: residual.  MODE 0: JVP with F(x_i) read from the cache filled at bk_jac_set_state
// (the reference recomputes it on every po_jvp!, PeriodicOrbitTrapeze.jl:310-317; results identical).
template <int MODE>
static __global__ void __launch_bounds__(256) k_potrap_apply(OpDesc op, const double* __restrict__ in,
                                                             const double* __restrict__ in_scale_ptr,
                                                             double* __restrict__ out) {
  const int nx = op.nx, ny = op.ny, M = op.nz;
  const long long n = (long long)nx * ny, Ns = 2 * n;
  const double s = in_scale_ptr ? __ldg(in_scale_ptr) : 1.0;
  const CglPar p = cgl_par(op);
  const double T = (MODE == 1) ? s * in[Ns * M] : op.u[Ns * M];
  const double dT = (MODE == 0) ? s * in[Ns * M] : 0.0;
  const double h2 = 0.5 * T / M, dh2 = 0.5 * dT / M;
  const long long total = n * M;
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    const TrapPoint t = trap_point(q, n);
    const long long g = t.g, o = t.o;
    const int sl = t.sl, i = t.i(nx), j = t.j(nx);
    if (sl == M - 1) {
      double c1 = s * (in[o] - in[g]), c2 = s * (in[o + n] - in[g + n]);
      out[o] = (MODE == 0) ? op.a0 * s * in[o] + op.a1 * c1 : c1;
      out[o + n] = (MODE == 0) ? op.a0 * s * in[o + n] + op.a1 * c2 : c2;
      continue;
    }
    int sp = sl > 0 ? sl - 1 : M - 2;
    const double* vi = in + (long long)sl * Ns;
    const double* vp = in + (long long)sp * Ns;
    double a1, a2, b1, b2;
    if (MODE == 1) {
      cgl_point<1>(p, nullptr, vi, s, i, j, nx, ny, op.cx, op.cy, a1, a2);
      cgl_point<1>(p, nullptr, vp, s, i, j, nx, ny, op.cx, op.cy, b1, b2);
      out[o] = s * (vi[g] - vp[g]) - h2 * (a1 + b1);
      out[o + n] = s * (vi[g + n] - vp[g + n]) - h2 * (a2 + b2);
    } else {
      const double* ui = op.u + (long long)sl * Ns;
      const double* up = op.u + (long long)sp * Ns;
      cgl_point<0>(p, ui, vi, s, i, j, nx, ny, op.cx, op.cy, a1, a2);
      cgl_point<0>(p, up, vp, s, i, j, nx, ny, op.cx, op.cy, b1, b2);
      const double* fi = op.fcache + (long long)sl * Ns;
      const double* fp = op.fcache + (long long)sp * Ns;
      double r1 = s * (vi[g] - vp[g]) - h2 * (a1 + b1) - dh2 * (fi[g] + fp[g]);
      double r2 = s * (vi[g + n] - vp[g + n]) - h2 * (a2 + b2) - dh2 * (fi[g + n] + fp[g + n]);
      out[o] = op.a0 * s * vi[g] + op.a1 * r1;
      out[o + n] = op.a0 * s * vi[g + n] + op.a1 * r2;
    }
  }
}
// phi_i = scale F(x_i) for every slice and, unless xpi is null, xpi = x without the period, in one pass over x: the section of
// the phase condition from an orbit x (updatesection!, PeriodicOrbitTrapeze.jl:665-679: scale = 1/M; re_make :1077-1080:
// scale = 1), or the F-cache at the Jacobian's state (scale = 1, no xpi)
static __global__ void __launch_bounds__(256) k_potrap_section(OpDesc op, const double* __restrict__ x, double scale,
                                                               double* __restrict__ phi, double* __restrict__ xpi) {
  bk_pdl_sync();
  const int nx = op.nx, ny = op.ny, M = op.nz;
  const long long n = (long long)nx * ny, total = n * M;
  const CglPar p = cgl_par(op);
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    const TrapPoint t = trap_point(q, n);
    double a1, a2;
    cgl_point<1>(p, nullptr, x + (t.o - t.g), 1.0, t.i(nx), t.j(nx), nx, ny, op.cx, op.cy, a1, a2);
    phi[t.o] = scale * a1;
    phi[t.o + n] = scale * a2;
    if (xpi) {
      xpi[t.o] = x[t.o];
      xpi[t.o + n] = x[t.o + n];
    }
  }
}

// ------------------------------------------------------------------------------------------ jets d2F / d3F
// Second and third differentials of F in u (src/Problems.jl:107-110,165-183).  The linear parts of F (Laplacians, L1, the
// spectral symbol) drop out, so both are pointwise; the boundary rows of chan are linear too.  ORDER 2: out = d2F(u)[a, b],
// ORDER 3: out = d3F(u)[a, b, c].  One thread per grid point; cGL2d points carry the pair (u1, u2) = Re, Im of A.
// chan_Nl = 1 + g / h with g = x + x^2 / 2, h = 1 + b x^2 (examples/chan.jl:5-7, b = beta as chan_F):
//   Nl'' = (1 - 6 b x - 3 b x^2 + 2 b^2 x^3) / h^3,   Nl''' = (-6 b - 12 b x + 36 b^2 x^2 + 12 b^2 x^3 - 6 b^3 x^4) / h^4
__device__ __forceinline__ double chan_d2Nl(double x, double b) {
  const double h = 1.0 + b * x * x;
  return (1.0 - 6.0 * b * x - 3.0 * b * x * x + 2.0 * b * b * x * x * x) / (h * h * h);
}
__device__ __forceinline__ double chan_d3Nl(double x, double b) {
  const double h = 1.0 + b * x * x, x2 = x * x;
  return (-6.0 * b - 12.0 * b * x + 36.0 * b * b * x2 + 12.0 * b * b * x2 * x - 6.0 * b * b * b * x2 * x2) / (h * h * h * h);
}
// cGL2d: NL(A) = (r + i nu) A - (c3 + i mu) |A|^2 A - c5 |A|^4 A (examples/cGL2d.jl:262-279).  With s = |A|^2 and
// s_xy = 2 Re(x conj y), the forms are real-multilinear (s is not holomorphic):
//   d2(s A)[a,b]     = s_ab A + s_A(a) b + s_A(b) a,                   s_A(x) = 2 Re(A conj x)
//   d2(s^2 A)[a,b]   = 2 (s_A(a) s_A(b) + s s_ab) A + 2 s (s_A(a) b + s_A(b) a)
//   d3(s A)[a,b,c]   = s_ab c + s_ac b + s_bc a
//   d3(s^2 A)[a,b,c] = 2 (s_ab s_A(c) + s_ac s_A(b) + s_bc s_A(a)) A + 2 (s_A(a) s_A(b) + s s_ab) c
//                      + 2 (s_A(a) s_A(c) + s s_ac) b + 2 (s_A(b) s_A(c) + s s_bc) a
template <int ORDER>
__device__ __forceinline__ void cgl_jet(const CglPar& p, double2 A, double2 a, double2 b, double2 c, double& o1, double& o2) {
  auto sdot = [](double2 x, double2 y) { return 2.0 * (x.x * y.x + x.y * y.y); };
  double2 t3, t5;  // the jets of |A|^2 A and |A|^4 A
  const double sab = sdot(a, b);
  if (ORDER == 2) {
    const double s = sdot(A, A) * 0.5, sa = sdot(A, a), sb = sdot(A, b);
    t3.x = sab * A.x + sa * b.x + sb * a.x;
    t3.y = sab * A.y + sa * b.y + sb * a.y;
    const double k = 2.0 * (sa * sb + s * sab);
    t5.x = k * A.x + 2.0 * s * (sa * b.x + sb * a.x);
    t5.y = k * A.y + 2.0 * s * (sa * b.y + sb * a.y);
  } else {
    const double s = sdot(A, A) * 0.5, sa = sdot(A, a), sb = sdot(A, b), sc = sdot(A, c);
    const double sac = sdot(a, c), sbc = sdot(b, c);
    t3.x = sab * c.x + sac * b.x + sbc * a.x;
    t3.y = sab * c.y + sac * b.y + sbc * a.y;
    const double k = 2.0 * (sab * sc + sac * sb + sbc * sa);
    const double kc = 2.0 * (sa * sb + s * sab), kb = 2.0 * (sa * sc + s * sac), ka = 2.0 * (sb * sc + s * sbc);
    t5.x = k * A.x + kc * c.x + kb * b.x + ka * a.x;
    t5.y = k * A.y + kc * c.y + kb * b.y + ka * a.y;
  }
  o1 = -(p.c3 * t3.x - p.mu * t3.y) - p.c5 * t5.x;
  o2 = -(p.c3 * t3.y + p.mu * t3.x) - p.c5 * t5.y;
}
// The jet of kind KIND at grid point g of pts, from the values there of u, a, b and c (c is read for ORDER 3 only): d2F(u)[a, b]
// (ORDER 2) or d3F(u)[a, b, c].  KIND is BK_CHAN, BK_CGL2D (double2 values: the pair (u1, u2)) or BK_SH2D for the three SH kinds.
template <int KIND, int ORDER, typename V>
__device__ __forceinline__ V jet_form(const OpDesc& op, V u, V a, V b, V c, long long g, long long pts) {
  if constexpr (KIND == BK_CGL2D) {
    V o;
    cgl_jet<ORDER>(cgl_par(op), u, a, b, c, o.x, o.y);
    return o;
  } else if constexpr (KIND == BK_CHAN) {  // alpha = par[0], beta = par[1]; the boundary rows are linear
    const double ab = a * b;
    const double r = ORDER == 2 ? op.par[0] * chan_d2Nl(u, op.par[1]) * ab : op.par[0] * chan_d3Nl(u, op.par[1]) * ab * c;
    return g > 0 && g < pts - 1 ? r : 0.0;
  } else {  // F = -L1 u + l u + nu u^2 - u^3
    const double ab = a * b;
    return ORDER == 2 ? (2.0 * op.par[1] - 6.0 * u) * ab : -6.0 * ab * c;
  }
}
// the pair (v[p], v[p + ld]) of a cGL2d point
__device__ __forceinline__ double2 cgl_pair(const double* v, long long p, long long ld) { return make_double2(v[p], v[p + ld]); }
template <int ORDER>
static __global__ void __launch_bounds__(256) k_jet(OpDesc op, const double* u, const double* a, const double* b,
                                                    const double* c, double* out, long long n) {
  bk_pdl_sync();
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += (long long)gridDim.x * blockDim.x) {
    if (op.kind == BK_CGL2D) {
      const double2 o = jet_form<BK_CGL2D, ORDER>(op, cgl_pair(u, g, n), cgl_pair(a, g, n), cgl_pair(b, g, n),
                                                  ORDER == 3 ? cgl_pair(c, g, n) : make_double2(0.0, 0.0), g, n);
      out[g] = o.x;
      out[g + n] = o.y;
    } else if (op.kind == BK_CHAN) {
      out[g] = jet_form<BK_CHAN, ORDER>(op, u[g], a[g], b[g], ORDER == 3 ? c[g] : 0.0, g, n);
    } else {
      const double ag = a[g], bg = b[g];  // before u[g]: this load order keeps the loop's unrolling and registers
      out[g] = jet_form<BK_SH2D, ORDER>(op, u[g], ag, bg, ORDER == 3 ? c[g] : 0.0, g, n);
    }
  }
}

// ------------------------------------------------------------------------------------------ jet moments
// out[t] = <v_i, d2F(u)[v_j, v_k]> (tuple t < n2) or <v_i, d3F(u)[v_j, v_k, v_l]> (t >= n2) for a list of tuples over nvec
// vectors, in one pass over the vectors: the per-point forms are those of k_jet, and the inner products are pointwise sums.
// Each CTA stages a tile of BK_MOM_TP grid points of every vector (and of u) in shared memory, one row per (vector, field),
// padded by one double so that the threads of a warp, each on its own tuple, read distinct rows from distinct banks.  Thread
// t of the CTA owns the tuples t, t + 256, ..; it sums a tuple over the tile's points in order and adds the tile's sum to the
// tuple's accumulator in shared memory.  The CTA's accumulators go to partials[blockIdx.x * ntup + t], which
// k_jet_moments_fold sums over the CTAs in order: the summation order depends on the grid and the tuple list only.
#define BK_MOM_TP 32
struct MomVecs {
  const double* v[BK_JET_MOMENTS_MAX_VEC + 1];  // the nvec vectors, then u
};
// KIND: BK_CHAN, BK_CGL2D, or BK_SH2D for the three SH kinds
template <int KIND, int ORDER>
__device__ __forceinline__ double moment_tile(const OpDesc& op, const double* __restrict__ s_v, int4 q, int urow, int np,
                                              long long base, long long pts) {
  constexpr int F = KIND == BK_CGL2D ? 2 : 1, LD = BK_MOM_TP + 1;
  const double* vi = s_v + q.x * F * LD;
  const double* va = s_v + q.y * F * LD;
  const double* vb = s_v + q.z * F * LD;
  const double* vc = s_v + (ORDER == 3 ? q.w : q.z) * F * LD;
  const double* uu = s_v + urow * LD;
  double s = 0.0;
  for (int p = 0; p < np; ++p) {
    if constexpr (KIND == BK_CGL2D) {
      const double2 o = jet_form<KIND, ORDER>(op, cgl_pair(uu, p, LD), cgl_pair(va, p, LD), cgl_pair(vb, p, LD),
                                              ORDER == 3 ? cgl_pair(vc, p, LD) : make_double2(0.0, 0.0), base + p, pts);
      s = fma(vi[p], o.x, s);
      s = fma(vi[p + LD], o.y, s);
    } else {
      s = fma(vi[p], jet_form<KIND, ORDER>(op, uu[p], va[p], vb[p], vc[p], base + p, pts), s);
    }
  }
  return s;
}
// The pass of a moment kernel over the tiles, for F fields per point: tile2 / tile3 (s_v, q, urow, np, base) return the sum of an
// order-2 / order-3 tuple q over the np points of the tile that starts at point base
template <int F, class Tile2, class Tile3>
__device__ __forceinline__ void jet_moments_pass(const MomVecs& vs, int nvec, const int4* __restrict__ tup, int ntup, int n2,
                                                 long long pts, double* __restrict__ partials, Tile2 tile2, Tile3 tile3) {
  constexpr int LD = BK_MOM_TP + 1;
  extern __shared__ double smem[];
  const int rows = (nvec + 1) * F;
  double* s_v = smem;                // rows x LD: row (vector, field), u last
  double* s_acc = smem + rows * LD;  // ntup accumulators
  for (int t = threadIdx.x; t < ntup; t += blockDim.x) s_acc[t] = 0.0;
  const long long ntiles = (pts + BK_MOM_TP - 1) / BK_MOM_TP;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const long long base = tile * BK_MOM_TP;
    const int np = (int)(pts - base < BK_MOM_TP ? pts - base : BK_MOM_TP);
    __syncthreads();  // the previous tile has been read
    for (int e = threadIdx.x; e < rows * BK_MOM_TP; e += blockDim.x) {
      const int r = e / BK_MOM_TP, p = e % BK_MOM_TP;
      s_v[r * LD + p] = p < np ? vs.v[r / F][base + p + (r % F) * pts] : 0.0;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < ntup; t += blockDim.x) {
      const int4 q = tup[t];
      s_acc[t] += t < n2 ? tile2(s_v, q, nvec * F, np, base) : tile3(s_v, q, nvec * F, np, base);
    }
  }
  for (int t = threadIdx.x; t < ntup; t += blockDim.x) partials[(size_t)blockIdx.x * ntup + t] = s_acc[t];
}
template <int KIND>
static __global__ void __launch_bounds__(256) k_jet_moments(OpDesc op, MomVecs vs, int nvec, const int4* __restrict__ tup,
                                                            int ntup, int n2, long long pts, double* __restrict__ partials) {
  bk_pdl_sync();
  constexpr int F = KIND == BK_CGL2D ? 2 : 1;
  jet_moments_pass<F>(
      vs, nvec, tup, ntup, n2, pts, partials,
      [&](const double* s_v, int4 q, int urow, int np, long long base) { return moment_tile<KIND, 2>(op, s_v, q, urow, np, base, pts); },
      [&](const double* s_v, int4 q, int urow, int np, long long base) { return moment_tile<KIND, 3>(op, s_v, q, urow, np, base, pts); });
}
// out[t] = the sum of the G partials of tuple t, in CTA order
static __global__ void __launch_bounds__(256) k_jet_moments_fold(const double* __restrict__ partials, int ntup, int G,
                                                                 double* __restrict__ out) {
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < ntup; t += gridDim.x * blockDim.x) {
    double s = 0.0;
    for (int b = 0; b < G; ++b) s += partials[(size_t)b * ntup + t];
    out[t] = s;
  }
}

// ------------------------------------------------------------------------------------------ reaction-diffusion (BK_RD)
// F_i(u) = D_i Lap u_i + R_i(u), R_i = sum of the terms c_t prod_j u_j^a_tj with eq_t = i (bk200.h), over the table of effective
// coefficients of bk_set_params (RdTable, by value: each context launches with its own).  One thread per grid point evaluates
// every field there: the 2 ND stencil neighbours per field, then the terms in table order.  Exponents are run-time values, so
// powers are bounded unrolled multiplications and a term reaches its equation by a select over the F fields: nothing indexes a
// per-thread array at run time, and the values of a point stay in registers.
__device__ __forceinline__ int rd_exp(int alpha, int j) { return (alpha >> (3 * j)) & 7; }
// x^e for a run-time e <= BK_RD_MAX_DEGREE; 1 for e <= 0
__device__ __forceinline__ double rd_pow(double x, int e) {
  double r = 1.0;
#pragma unroll
  for (int k = 0; k < BK_RD_MAX_DEGREE; ++k) r = k < e ? r * x : r;
  return r;
}
// acc[e] += x for the run-time field index e < F
template <int F>
__device__ __forceinline__ void rd_add(double (&acc)[F], int e, double x) {
#pragma unroll
  for (int f = 0; f < F; ++f)
    if (e == f) acc[f] += x;
}
// the gradient of the monomial alpha at u: g_k = a_k u_k^(a_k - 1) prod_{j != k} u_j^a_j
template <int F>
__device__ __forceinline__ void rd_grad(int alpha, const double (&u)[F], double (&g)[F]) {
  double pw[F], pd[F];
#pragma unroll
  for (int j = 0; j < F; ++j) {
    const int a = rd_exp(alpha, j);
    const double p = rd_pow(u[j], a - 1);
    pd[j] = a * p;
    pw[j] = a > 0 ? p * u[j] : 1.0;
  }
#pragma unroll
  for (int k = 0; k < F; ++k) {
    double t = pd[k];
#pragma unroll
    for (int j = 0; j < F; ++j)
      if (j != k) t *= pw[j];
    g[k] = t;
  }
}
// The Laplacian of the field at v (unscaled) at point g = i + j nx: Neumann = clamp-to-edge ghost cells, Dirichlet = zero ghosts
template <int ND>
__device__ __forceinline__ double rd_lap(const double* __restrict__ v, long long g, int i, int j, int nx, int ny, double cx,
                                         double cy, bool dirichlet) {
  const double c = v[g], ghost = dirichlet ? 0.0 : c;
  const double xm = i > 0 ? v[g - 1] : ghost, xp = i < nx - 1 ? v[g + 1] : ghost;
  if constexpr (ND == 2) {
    const double ym = j > 0 ? v[g - nx] : ghost, yp = j < ny - 1 ? v[g + nx] : ghost;
    return cx * (xm - 2.0 * c + xp) + cy * (ym - 2.0 * c + yp);
  }
  return cx * (xm - 2.0 * c + xp);
}
// MODE 1: out = F(s v).  MODE 0: out = a0 s v + a1 J s v.  MODE 2: out = a0 s v + a1 J' s v (J' = the symmetric Laplacian plus
// the transposed F x F reaction block).  s = *sp (1 when sp is NULL).
template <int F, int ND, int MODE>
static __global__ void __launch_bounds__(256) k_rd_apply(OpDesc op, const __grid_constant__ RdTable tb, const double* __restrict__ in,
                                                         const double* __restrict__ sp, double* __restrict__ out) {
  const int nx = op.nx, ny = ND == 2 ? op.ny : 1;
  const long long n = (long long)nx * ny;
  const double s = sp ? __ldg(sp) : 1.0;
  const bool dir = tb.bc == BK_BC_DIRICHLET;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += (long long)gridDim.x * blockDim.x) {
    const int i = ND == 2 ? (int)(g % nx) : (int)g, j = ND == 2 ? (int)(g / nx) : 0;
    double v[F], u[F], r[F];
#pragma unroll
    for (int f = 0; f < F; ++f) {
      v[f] = s * in[g + f * n];
      r[f] = tb.diff[f] * (s * rd_lap<ND>(in + f * n, g, i, j, nx, ny, op.cx, op.cy, dir));
      if (MODE != 1) u[f] = op.u[g + f * n];
    }
    for (int t = 0; t < tb.nterms; ++t) {
      const int alpha = tb.alpha[t], e = tb.eq[t];
      const double c = tb.coef[t];
      if constexpr (MODE == 1) {
        double m = c;
#pragma unroll
        for (int k = 0; k < F; ++k) m *= rd_pow(v[k], rd_exp(alpha, k));
        rd_add(r, e, m);
      } else {
        double gr[F];
        rd_grad(alpha, u, gr);
        if constexpr (MODE == 0) {
          double d = 0.0;
#pragma unroll
          for (int k = 0; k < F; ++k) d = fma(gr[k], v[k], d);
          rd_add(r, e, c * d);
        } else {
          double we = 0.0;
#pragma unroll
          for (int f = 0; f < F; ++f) we = e == f ? v[f] : we;
#pragma unroll
          for (int k = 0; k < F; ++k) r[k] += c * gr[k] * we;
        }
      }
    }
#pragma unroll
    for (int f = 0; f < F; ++f) out[g + f * n] = MODE == 1 ? r[f] : op.a0 * v[f] + op.a1 * r[f];
  }
}
// The RD point form of the jets: o = d2F(u)[a, b] (ORDER 2) or d3F(u)[a, b, c] (ORDER 3) at one point; the Laplacian drops out.
// Each monomial is expanded as a product of its factors (u_j + s a_j + t b_j + r c_j)^a_j, truncated to the multilinear terms in
// the ORDER directions: component S (a subset of the directions, as a bit mask) of a factor is a_j^(|S|) u_j^(a_j - |S|) times
// the product of the directions in S (x^(k) the falling factorial), and the full component of the product is the jet.
template <int F, int ORDER>
__device__ __forceinline__ void rd_jet(const RdTable& tb, const double (&u)[F], const double (&a)[F], const double (&b)[F],
                                       const double (&c)[F], double (&o)[F]) {
  constexpr int NS = 1 << ORDER;
#pragma unroll
  for (int f = 0; f < F; ++f) o[f] = 0.0;
  for (int t = 0; t < tb.nterms; ++t) {
    const int alpha = tb.alpha[t];
    double m[NS];
#pragma unroll
    for (int S = 0; S < NS; ++S) m[S] = S == 0 ? 1.0 : 0.0;
#pragma unroll
    for (int j = 0; j < F; ++j) {
      const int ae = rd_exp(alpha, j);
      double pk[ORDER + 1];  // a^(k) u^(a - k)
#pragma unroll
      for (int k = 0; k <= ORDER; ++k) {
        double ff = 1.0;
#pragma unroll
        for (int q = 0; q < k; ++q) ff *= (double)(ae - q);
        pk[k] = ff * rd_pow(u[j], ae - k);
      }
      double fac[NS];
#pragma unroll
      for (int S = 0; S < NS; ++S) {
        double x = pk[__builtin_popcount(S)];
        if (S & 1) x *= a[j];
        if (S & 2) x *= b[j];
        if (S & 4) x *= c[j];
        fac[S] = x;
      }
      double p[NS];
#pragma unroll
      for (int S = 0; S < NS; ++S) {
        double acc = 0.0;
#pragma unroll
        for (int T = 0; T < NS; ++T)
          if ((T & S) == T) acc = fma(m[T], fac[S & ~T], acc);
        p[S] = acc;
      }
#pragma unroll
      for (int S = 0; S < NS; ++S) m[S] = p[S];
    }
    rd_add(o, tb.eq[t], tb.coef[t] * m[NS - 1]);
  }
}
template <int F, int ORDER>
static __global__ void __launch_bounds__(256) k_rd_jet(const __grid_constant__ RdTable tb, const double* u, const double* a,
                                                       const double* b, const double* c, double* out, long long n) {
  bk_pdl_sync();
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < n; g += (long long)gridDim.x * blockDim.x) {
    double uu[F], aa[F], bb[F], cc[F], o[F];
#pragma unroll
    for (int f = 0; f < F; ++f) {
      uu[f] = u[g + f * n];
      aa[f] = a[g + f * n];
      bb[f] = b[g + f * n];
      cc[f] = ORDER == 3 ? c[g + f * n] : 0.0;
    }
    rd_jet<F, ORDER>(tb, uu, aa, bb, cc, o);
#pragma unroll
    for (int f = 0; f < F; ++f) out[g + f * n] = o[f];
  }
}
// k_jet_moments for BK_RD: the same pass and fold, with rd_jet as the point form
template <int F, int ORDER>
__device__ __forceinline__ double rd_moment_tile(const RdTable& tb, const double* __restrict__ s_v, int4 q, int urow, int np) {
  constexpr int LD = BK_MOM_TP + 1;
  const double* vi = s_v + q.x * F * LD;
  const double* va = s_v + q.y * F * LD;
  const double* vb = s_v + q.z * F * LD;
  const double* vc = s_v + (ORDER == 3 ? q.w : q.z) * F * LD;
  const double* uu = s_v + urow * LD;
  double s = 0.0;
  for (int p = 0; p < np; ++p) {
    double u[F], a[F], b[F], c[F], o[F];
#pragma unroll
    for (int f = 0; f < F; ++f) {
      u[f] = uu[p + f * LD];
      a[f] = va[p + f * LD];
      b[f] = vb[p + f * LD];
      c[f] = vc[p + f * LD];
    }
    rd_jet<F, ORDER>(tb, u, a, b, c, o);
#pragma unroll
    for (int f = 0; f < F; ++f) s = fma(vi[p + f * LD], o[f], s);
  }
  return s;
}
template <int F>
static __global__ void __launch_bounds__(256) k_rd_jet_moments(const __grid_constant__ RdTable tb, MomVecs vs, int nvec,
                                                               const int4* __restrict__ tup, int ntup, int n2, long long pts,
                                                               double* __restrict__ partials) {
  bk_pdl_sync();
  jet_moments_pass<F>(
      vs, nvec, tup, ntup, n2, pts, partials,
      [&](const double* s_v, int4 q, int urow, int np, long long) { return rd_moment_tile<F, 2>(tb, s_v, q, urow, np); },
      [&](const double* s_v, int4 q, int urow, int np, long long) { return rd_moment_tile<F, 3>(tb, s_v, q, urow, np); });
}

// ------------------------------------------------------------------------------------------ deflation moments
// Per root r_i: s_i = <d, d>, m_i = max |d|, t_{i,a} = <d, h_a> with d = u - r_i, and q_ab = <h_a, h_b>, in one pass (bk200.h).
// A tile is 256 x BK_DEFL_PPT points, thread t owning points t, t + 256, ..; the CTAs of the grid (bk_reduce_grid of the tiles'
// thread count) take the tiles in a grid-stride loop.  Per tile a thread keeps its points of u and of the directions in
// registers and takes the roots in batches of BK_DEFL_RB: all the batch's loads are issued before the sums.  Each value is
// folded over the warp (xor-shuffle tree) and added, in tile order, to that warp's own accumulator in shared memory, so the tile
// loop has no barrier; after it, the 8 warps' accumulators are folded in warp order into partials[k * G + blockIdx.x], and
// k_deflation_moments_fold folds those in CTA order.  A root's arithmetic is the same whichever batch slot it has, so its
// outputs depend on n only.
#define BK_DEFL_PPT 4
#define BK_DEFL_RB 4
struct DeflVecs {
  const double* r[BK_DEFLATION_MAX_ROOTS];
  const double* h[2];
  const double* u;
};
// acc[k] += (or max=, for the m columns: k % W == 1 with W > 0) the warp total of v[k], for k < live (uniform over the warp)
template <int K, int W>
__device__ __forceinline__ void defl_warp_add(const double (&v)[K], int live, double* acc) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    if (k < live) {
      const bool mx = W > 0 && k % W == 1;
      const double t = mx ? bk_warp_max(v[k]) : bk_warp_sum(v[k]);
      if (lane == 0) acc[k] = mx ? bk_nanmax(acc[k], t) : acc[k] + t;
    }
  }
}
template <int NDIR>
static __global__ void __launch_bounds__(256) k_deflation_moments(DeflVecs vs, int nroots, long long n,
                                                                  double* __restrict__ partials) {
  bk_pdl_sync();
  constexpr int W = 2 + NDIR, NQ = NDIR * (NDIR + 1) / 2, TP = 256 * BK_DEFL_PPT, LDA = BK_DEFLATION_MAX_ROOTS * W + 3;
  __shared__ double s_acc[8 * LDA];  // one row of accumulators per warp
  const int ncol = nroots * W + NQ;
  for (int k = threadIdx.x; k < 8 * LDA; k += blockDim.x) s_acc[k] = 0.0;
  __syncthreads();
  double* acc = s_acc + (threadIdx.x >> 5) * LDA;
  const long long ntiles = (n + TP - 1) / TP;
  for (long long tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    long long idx[BK_DEFL_PPT];
    double u[BK_DEFL_PPT], h[2][BK_DEFL_PPT];
#pragma unroll
    for (int p = 0; p < BK_DEFL_PPT; ++p) {
      idx[p] = tile * TP + threadIdx.x + 256 * p;
      const bool in = idx[p] < n;
      u[p] = in ? vs.u[idx[p]] : 0.0;
#pragma unroll
      for (int a = 0; a < 2; ++a) h[a][p] = in && a < NDIR ? vs.h[a][idx[p]] : 0.0;
    }
    if constexpr (NQ > 0) {
      double q[3] = {0.0, 0.0, 0.0};
#pragma unroll
      for (int p = 0; p < BK_DEFL_PPT; ++p) {
        q[0] = fma(h[0][p], h[0][p], q[0]);
        q[1] = fma(h[0][p], h[1][p], q[1]);
        q[2] = fma(h[1][p], h[1][p], q[2]);
      }
      defl_warp_add<3, 0>(q, NQ, acc + nroots * W);
    }
    for (int r0 = 0; r0 < nroots; r0 += BK_DEFL_RB) {
      const int live = nroots - r0 < BK_DEFL_RB ? nroots - r0 : BK_DEFL_RB;
      double x[BK_DEFL_RB][BK_DEFL_PPT];
#pragma unroll
      for (int j = 0; j < BK_DEFL_RB; ++j)
#pragma unroll
        for (int p = 0; p < BK_DEFL_PPT; ++p) x[j][p] = j < live && idx[p] < n ? vs.r[r0 + j][idx[p]] : u[p];
      double v[BK_DEFL_RB * W];
#pragma unroll
      for (int j = 0; j < BK_DEFL_RB; ++j) {
        double s = 0.0, m = 0.0, t[2] = {0.0, 0.0};
#pragma unroll
        for (int p = 0; p < BK_DEFL_PPT; ++p) {
          const double d = u[p] - x[j][p];
          s = fma(d, d, s);
          m = bk_nanmax(m, fabs(d));
#pragma unroll
          for (int a = 0; a < NDIR; ++a) t[a] = fma(d, h[a][p], t[a]);
        }
        v[j * W] = s;
        v[j * W + 1] = m;
#pragma unroll
        for (int a = 0; a < NDIR; ++a) v[j * W + 2 + a] = t[a];
      }
      defl_warp_add<BK_DEFL_RB * W, W>(v, live * W, acc + r0 * W);
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < ncol; k += blockDim.x) {
    const bool mx = k < nroots * W && k % W == 1;
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t = mx ? bk_nanmax(t, s_acc[w * LDA + k]) : t + s_acc[w * LDA + k];
    partials[(size_t)k * gridDim.x + blockIdx.x] = t;
  }
}
// out[k] = the fold of the G partials of column k in a fixed order: one warp per column, lane l taking the CTAs l, l + 32, ..
// in order, then the xor-shuffle tree; max for the m columns (k < nmom, k % W == 1), sums otherwise
static __global__ void __launch_bounds__(256) k_deflation_moments_fold(const double* __restrict__ partials, int ncol, int nmom,
                                                                       int W, int G, double* __restrict__ out) {
  const int k = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (k >= ncol) return;  // uniform over the warp
  const bool mx = k < nmom && k % W == 1;
  double s = 0.0;
  for (int b = lane; b < G; b += 32) {
    const double x = partials[(size_t)k * G + b];
    s = mx ? bk_nanmax(s, x) : s + x;
  }
  s = mx ? bk_warp_max(s) : bk_warp_sum(s);
  if (lane == 0) out[k] = s;
}

// ------------------------------------------------------------------------------------------ tail reductions
// Bordered map with NB = 1 or 2 borders (MatrixFreeBLSmap, src/LinearBorderSolver.jl:299-335; tuple form :338-389), one pass
// after the operator has written out.u = Op(s x.u):   xp = s x.p,
//   out.u[i] += xp0 a[i] (+ xp1 a2[i]) + bshift s x.u[i];   out.p = s bscale [<b, x.u>; <b2, x.u>] + [bc bc01; bc10 bc11] xp
template <int NB>
static __global__ void __launch_bounds__(256) k_tail(OpDesc op, const double* __restrict__ in,
                                                     const double* __restrict__ in_scale_ptr, double* __restrict__ out,
                                                     long long n, double* __restrict__ partials, unsigned int* counter) {
  const double s = in_scale_ptr ? __ldg(in_scale_ptr) : 1.0;
  const double xp0 = s * in[n], xp1 = NB == 2 ? s * in[n + 1] : 0.0;
  double acc[NB] = {};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double v = in[i];
    acc[0] = fma(v, op.bb[i], acc[0]);
    if constexpr (NB == 2) {
      acc[1] = fma(v, op.bb2[i], acc[1]);
      out[i] += xp0 * op.ba[i] + xp1 * op.ba2[i] + op.bshift * s * v;
    } else {
      out[i] += xp0 * op.ba[i] + op.bshift * s * v;
    }
  }
  if (!bk_grid_reduce<NB>(acc, partials, counter)) return;
  if constexpr (NB == 2) {
    out[n] = s * op.bscale * acc[0] + op.bc * xp0 + op.bc01 * xp1;
    out[n + 1] = s * op.bscale * acc[1] + op.bc10 * xp0 + op.bc11 * xp1;
  } else {
    out[n] = s * op.bscale * acc[0] + op.bc * xp0;
  }
}

// potrap phase condition, the last row: out[n] = s <in, phi> - beta0 (residual, beta0 = <xpi, phi>), or a0 s in[n] + a1 s
// <in, phi> (JVP)
static __global__ void __launch_bounds__(256) k_potrap_phase(OpDesc op, const double* __restrict__ in,
                                                             const double* __restrict__ in_scale_ptr, double* __restrict__ out,
                                                             long long n, double beta0, int jvp_mode,
                                                             double* __restrict__ partials, unsigned int* counter) {
  const double s = in_scale_ptr ? __ldg(in_scale_ptr) : 1.0;
  double acc[1] = {0.0};
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    acc[0] = fma(in[i], op.phi[i], acc[0]);
  if (!bk_grid_reduce<1>(acc, partials, counter)) return;
  const double ph = s * acc[0] - beta0;
  out[n] = jvp_mode ? op.a0 * s * in[n] + op.a1 * ph : ph;
}

// J' of the Trapeze functional: the transpose of k_potrap_apply<0> with its phase row, in one pass.  With h/2 = T / (2M),
// A_k = J_F(x_k), f_k = F(x_k) (fcache) and next(k) = k + 1, next(M - 2) = 0 (the inverse of the row map sl -> sp):
//   (J'w)_k     = (w_k - w_next(k)) - h/2 A_k' (w_k + w_next(k)) + phi_k w_T   (k <= M - 2; slice 0 also - w_{M-1})
//   (J'w)_{M-1} = w_{M-1} + phi_{M-1} w_T
//   (J'w)_T     = -1/(2M) sum_{k <= M-2} <f_k, w_k + w_next(k)>
// A_k' is the Dirichlet Laplacian (symmetric) plus the transposed 2 x 2 reaction block, so each point needs one stencil
// evaluation, on w_k + w_next(k).  out = a0 s w + a1 s J'w (s = *in_scale_ptr); the period entry is the fixed-order grid
// reduction of k_tail, written by the last CTA.
static __global__ void __launch_bounds__(256, 3) k_potrap_apply_tr(OpDesc op, const double* __restrict__ in,
                                                                const double* __restrict__ in_scale_ptr, double* __restrict__ out,
                                                                double* __restrict__ partials, unsigned int* counter) {
  const int nx = op.nx, ny = op.ny, M = op.nz;
  const long long n = (long long)nx * ny, Ns = 2 * n, total = n * M;
  const double s = in_scale_ptr ? __ldg(in_scale_ptr) : 1.0;
  const CglPar p = cgl_par(op);
  const double h2 = 0.5 * op.u[Ns * M] / M;
  const double wT = s * in[Ns * M];
  const double* wl = in + (long long)(M - 1) * Ns;
  double acc[1] = {0.0};
  for (long long q = (long long)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (long long)gridDim.x * blockDim.x) {
    const TrapPoint t = trap_point(q, n);
    const long long g = t.g, o = t.o;
    const int sl = t.sl;
    double r1 = op.phi[o] * wT, r2 = op.phi[o + n] * wT;
    if (sl == M - 1) {
      r1 += s * in[o];
      r2 += s * in[o + n];
    } else {
      const int nk = sl < M - 2 ? sl + 1 : 0;
      const double* wk = in + (long long)sl * Ns;
      const double* wn = in + (long long)nk * Ns;
      const double* uk = op.u + (long long)sl * Ns;
      const double* fk = op.fcache + (long long)sl * Ns;
      const double d1 = wk[g] + wn[g], d2 = wk[g + n] + wn[g + n];
      double a1, a2;
      cgl_dnl<true>(p, uk[g], uk[g + n], s * d1, s * d2, a1, a2);
      const int i = t.i(nx), j = t.j(nx);
      a1 += lap_dirichlet(FieldSum{wk, wn}, i, j, nx, ny, op.cx, op.cy, s);
      a2 += lap_dirichlet(FieldSum{wk + n, wn + n}, i, j, nx, ny, op.cx, op.cy, s);
      r1 += s * (wk[g] - wn[g]) - h2 * a1;
      r2 += s * (wk[g + n] - wn[g + n]) - h2 * a2;
      if (sl == 0) {
        r1 -= s * wl[g];
        r2 -= s * wl[g + n];
      }
      acc[0] = fma(fk[g], d1, acc[0]);
      acc[0] = fma(fk[g + n], d2, acc[0]);
    }
    out[o] = op.a0 * s * in[o] + op.a1 * r1;
    out[o + n] = op.a0 * s * in[o + n] + op.a1 * r2;
  }
  if (!bk_grid_reduce<1>(acc, partials, counter)) return;
  out[Ns * M] = op.a0 * wT + op.a1 * (-0.5 / M) * s * acc[0];
}

// ------------------------------------------------------------------------------------------ host side
static void fill_grid(bk_ctx* c, OpDesc& op) {
  op.kind = c->kind;
  op.nx = (int)c->dims[0];
  op.ny = (int)c->dims[1];
  op.nz = (int)c->dims[2];
  op.cx = bk_inv_h2(c, 0);
  op.cy = bk_inv_h2(c, 1);
  op.cz = (c->kind == BK_SH3D) ? bk_inv_h2(c, 2) : 0.0;
  op.N = c->N;
  op.bordered = 0;
  op.ba = op.bb = nullptr;
  op.bc = op.bshift = 0.0;
  op.bscale = 1.0;
  op.ba2 = op.bb2 = nullptr;
  op.bc01 = op.bc10 = op.bc11 = 0.0;
  op.phi = c->phi;
  op.fcache = c->fcache;
  op.cplx = c->cplx ? 1 : 0;
  op.a0i = c->shift_imag;
  op.transpose = c->transpose ? 1 : 0;
}

OpDesc bk_make_op(bk_ctx* c, double a0, double a1) {
  OpDesc op;
  fill_grid(c, op);
  for (int i = 0; i < BK_MAX_PAR; ++i) op.par[i] = c->jpar[i];
  op.u = c->u_state;
  op.a0 = a0;
  op.a1 = a1;
  return op;
}
OpDesc bk_make_residual_op(bk_ctx* c) {
  OpDesc op;
  fill_grid(c, op);
  for (int i = 0; i < BK_MAX_PAR; ++i) op.par[i] = c->par[i];
  op.u = nullptr;
  op.a0 = 0;
  op.a1 = 1;
  op.N = c->N0;  // F acts on the real state also in a BK_COMPLEX context
  op.cplx = 0;
  op.transpose = 0;
  return op;
}

// SH2d on the TMA-staged tile (bk_krylov_tma.cuh): the tallest of the tiles E = 8, 4, 2, 1 that still gives every SM about
// two CTAs
template <int E, int MODE>
static int launch_k2_apply(bk_ctx* c, const OpDesc& op, const double* in, const double* sp, double* out) {
  const int grid = ((op.nx + BK2_ROW - 1) / BK2_ROW) * ((op.ny + E - 1) / E);
  if constexpr (E > 1)
    if (grid < 2LL * c->nsm) return launch_k2_apply<E / 2, MODE>(c, op, in, sp, out);
  return bk_launch_ordered(c, k2_apply<E, MODE>, grid, BK2_THREADS, Sh2Scratch<E>::BYTES, op, in, sp, out);
}

// The RD kernel of the context's fields and dimensions, as a function pointer out of a table
#define BK_RD_BY_FIELDS(K, ...) {K<1, __VA_ARGS__>, K<2, __VA_ARGS__>, K<3, __VA_ARGS__>, K<4, __VA_ARGS__>}
template <int MODE>
static int launch_rd(bk_ctx* c, const OpDesc& op, const double* in, const double* sp, double* out) {
  // residual at the context's params, JVP / J' at the Jacobian's (bk_jac_set_state)
  const int mode = MODE == 1 ? 1 : op.transpose ? 2 : 0;
  static decltype(&k_rd_apply<1, 1, 0>) const kern[2][3][4] = {
      {BK_RD_BY_FIELDS(k_rd_apply, 1, 0), BK_RD_BY_FIELDS(k_rd_apply, 1, 1), BK_RD_BY_FIELDS(k_rd_apply, 1, 2)},
      {BK_RD_BY_FIELDS(k_rd_apply, 2, 0), BK_RD_BY_FIELDS(k_rd_apply, 2, 1), BK_RD_BY_FIELDS(k_rd_apply, 2, 2)}};
  const BkKindTraits* kt = bk_traits(c);
  return bk_launch_ordered(c, kern[kt->ndims - 1][mode][kt->fields - 1], bk_lin_grid(c, (long long)op.nx * op.ny), 256, 0, op,
                           MODE == 1 ? c->rd_par : c->rd_jpar, in, sp, out);
}

template <int MODE>
static int launch_kind(bk_ctx* c, const OpDesc& op, const double* in, const double* sp, double* out) {
  switch (op.kind) {
    case BK_RD: return launch_rd<MODE>(c, op, in, sp, out);
    case BK_SH2D:
      if ((op.nx % 2 == 0) && ((((uintptr_t)in) & 15) == 0)) return launch_k2_apply<BK2_EMAX, MODE>(c, op, in, sp, out);
      return bk_launch_ordered(c, k_sh_apply<2, MODE>, sh_num_tiles<2>(op.nx, op.ny, 1), BK_THREADS, ShSmem<2>::BYTES, op, in,
                               sp, out);
    case BK_SH3D:
      return bk_launch_ordered(c, k_sh_apply<3, MODE>, sh_num_tiles<3>(op.nx, op.ny, op.nz), BK_THREADS, ShSmem<3>::BYTES, op,
                               in, sp, out);
    case BK_SH2D_PERIODIC:  // spectral: three transform kernels (bk_precond.cu)
      return MODE == 1 ? bk_periodic_residual(c, op, in, out) : bk_periodic_jvp(c, op, in, sp, out);
    case BK_CHAN: return bk_launch_ordered(c, k_chan_apply<MODE>, bk_lin_grid(c, op.nx), 256, 0, op, in, sp, out);
    case BK_CGL2D:
      return bk_launch_ordered(c, k_cgl_apply<MODE>, bk_lin_grid(c, (long long)op.nx * op.ny), 256, 0, op, in, sp, out);
    case BK_POTRAP_CGL2D:
      if (MODE == 0 && op.transpose)  // J': one kernel for the slices and the period entry
        return bk_launch_ordered(c, k_potrap_apply_tr, bk_reduce_grid(c, (long long)op.nx * op.ny * op.nz), 256, 0, op, in, sp, out,
                                 c->partials, c->counters + 9);
      BK_TRY(bk_launch_ordered(c, k_potrap_apply<MODE>, bk_lin_grid(c, (long long)op.nx * op.ny * op.nz), 256, 0, op, in, sp,
                               out));
      return bk_launch_ordered(c, k_potrap_phase, bk_reduce_grid(c, op.N - 1), 256, 0, op, in, sp, out, op.N - 1,
                               (MODE == 1) ? c->phi_dot_xpi : 0.0, MODE == 0 ? 1 : 0, c->partials, c->counters + 9);
    default: return bk_fail(c, BK_ERR_ARG, "unknown kind", __FILE__, __LINE__);
  }
}

int bk_launch_residual(bk_ctx* c, const double* u, double* out) {
  OpDesc op = bk_make_residual_op(c);
  return launch_kind<1>(c, op, u, nullptr, out);
}

// imaginary part of the shift on a split complex vector: out_re -= a0i s in_im, out_im += a0i s in_re
static __global__ void __launch_bounds__(256) k_cshift(double* __restrict__ out, const double* __restrict__ in,
                                                       const double* __restrict__ in_scale_ptr, double a0i, long long n0) {
  const double s = (in_scale_ptr ? __ldg(in_scale_ptr) : 1.0) * a0i;
  for (long long g = (long long)blockIdx.x * blockDim.x + threadIdx.x; g < n0; g += (long long)gridDim.x * blockDim.x) {
    const double xr = in[g], xi = in[g + n0];
    out[g] -= s * xi;
    out[g + n0] += s * xr;
  }
}

int bk_launch_apply(bk_ctx* c, const OpDesc& op, const double* in, const double* sp, double* out) {
  if (op.transpose) BK_CHECK(c, bk_traits(c)->has_jt, "J' is not available for this problem kind");
  if (op.cplx) {
    // ((a0 + i a0i) I + a1 J)(x + i y): the real operator on both halves, then the cross terms of the imaginary shift
    OpDesc half = op;
    half.cplx = 0;
    half.N = op.N / 2;
    half.bordered = 0;
    BK_TRY(launch_kind<0>(c, half, in, sp, out));
    BK_TRY(launch_kind<0>(c, half, in + half.N, sp, out + half.N));
    if (op.a0i != 0.0) BK_TRY(bk_launch_ordered(c, k_cshift, bk_lin_grid(c, half.N), 256, 0, out, in, sp, op.a0i, half.N));
  } else {
    BK_TRY(launch_kind<0>(c, op, in, sp, out));
  }
  if (!op.bordered) return BK_OK;
  return bk_launch_ordered(c, op.bordered == 2 ? k_tail<2> : k_tail<1>, bk_reduce_grid(c, op.N), 256, 0, op, in, sp, out, op.N,
                           c->partials, c->counters + 9);
}

int bk_potrap_refresh_cache(bk_ctx* c) {
  if (c->kind != BK_POTRAP_CGL2D) return BK_OK;
  const OpDesc op = bk_make_op(c, 0, 1);
  return bk_launch(c, k_potrap_section, bk_lin_grid(c, (long long)op.nx * op.ny * op.nz), 256, 0, op, c->u_state, 1.0, c->fcache,
                   (double*)nullptr);
}

// ------------------------------------------------------------------------------------------ C ABI
extern "C" int32_t bk_residual(bk_ctx* c, const double* u, double* out) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_residual");
  double *du, *dout;
  BK_TRY(bk_stage_in(c, u, c->N0, 0, true, &du));
  BK_TRY(bk_stage_in(c, out, c->N0, 1, false, &dout));
  BK_TRY(bk_launch_residual(c, du, dout));
  return bk_stage_out(c, out, c->N0, dout);
}

extern "C" int32_t bk_jac_set_state(bk_ctx* c, const double* u) {
  BK_ENTER(c);
  BK_CHECK(c, u != nullptr, "null state");
  cudaMemcpyKind kind = bk_is_device_ptr(u) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  BK_CUDA(c, cudaMemcpyAsync(c->u_state, u, 8 * (size_t)c->N0, kind, c->stream));
  if (kind == cudaMemcpyHostToDevice) c->stats.h2d_bytes += 8 * c->N0;
  for (int i = 0; i < BK_MAX_PAR; ++i) c->jpar[i] = c->par[i];
  c->rd_jpar = c->rd_par;
  c->have_state = true;
  return bk_potrap_refresh_cache(c);
}

extern "C" int32_t bk_jac_set_shift_imag(bk_ctx* c, double a0_imag) {
  BK_ENTER(c);
  BK_CHECK(c, c->cplx || a0_imag == 0.0, "an imaginary shift needs a BK_COMPLEX context");
  c->shift_imag = a0_imag;
  return BK_OK;
}

extern "C" int32_t bk_jac_set_transpose(bk_ctx* c, int32_t on) {
  BK_ENTER(c);
  BK_CHECK(c, !on || bk_traits(c)->has_jt, "J' is not available for this problem kind");
  c->transpose = on != 0;
  return BK_OK;
}

extern "C" int32_t bk_jvp(bk_ctx* c, const double* v, double* out, double a0, double a1) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_jvp");
  BK_CHECK(c, c->have_state, "bk_jac_set_state must be called before bk_jvp");
  double *dv, *dout;
  BK_TRY(bk_stage_in(c, v, c->N, 0, true, &dv));
  BK_TRY(bk_stage_in(c, out, c->N, 1, false, &dout));
  BK_CHECK(c, dv != dout, "bk_jvp: in-place application is not supported");
  OpDesc op = bk_make_op(c, a0, a1);
  BK_TRY(bk_launch_apply(c, op, dv, nullptr, dout));
  return bk_stage_out(c, out, c->N, dout);
}

// The checks bk_d2f, bk_d3f and bk_jet_moments share, then the jet form (jet_form) of the context's kind in *kind: BK_CHAN,
// BK_CGL2D, BK_SH2D for the three SH kinds, or BK_RD (rd_jet)
static int jet_kind(bk_ctx* c, int* kind) {
  BK_CHECK(c, bk_traits(c)->has_jets, "d2F / d3F are not available for this problem kind");
  BK_CHECK(c, !c->cplx, "d2F / d3F act on real states: not available in a BK_COMPLEX context");
  *kind = c->kind == BK_CHAN || c->kind == BK_CGL2D || c->kind == BK_RD ? c->kind : BK_SH2D;
  return BK_OK;
}

// d2F (dx3 == nullptr) or d3F at the context's current params; every vector N0 doubles, host or device
static int jet(bk_ctx* c, const double* u, const double* dx1, const double* dx2, const double* dx3, double* out) {
  int kind;
  BK_TRY(jet_kind(c, &kind));
  const long long n = c->N0;
  double *du, *d1, *d2, *d3 = nullptr, *dout;
  BK_TRY(bk_stage_in(c, u, n, 0, true, &du));
  BK_TRY(bk_stage_in(c, dx1, n, 2, true, &d1));
  BK_TRY(bk_stage_in(c, dx2, n, 3, true, &d2));
  if (dx3) BK_TRY(bk_stage_in(c, dx3, n, 4, true, &d3));
  BK_TRY(bk_stage_in(c, out, n, 1, false, &dout));
  OpDesc op = bk_make_residual_op(c);
  op.kind = kind;  // k_jet branches on the jet form
  const int fields = bk_traits(c)->fields;
  const long long pts = n / fields;
  if (kind == BK_RD) {
    static decltype(&k_rd_jet<1, 2>) const kern[2][4] = {BK_RD_BY_FIELDS(k_rd_jet, 2), BK_RD_BY_FIELDS(k_rd_jet, 3)};
    BK_TRY(bk_launch(c, kern[dx3 ? 1 : 0][fields - 1], bk_lin_grid(c, pts), 256, 0, c->rd_par, du, d1, d2, d3, dout, pts));
    return bk_stage_out(c, out, n, dout);
  }
  if (dx3) BK_TRY(bk_launch(c, k_jet<3>, bk_lin_grid(c, pts), 256, 0, op, du, d1, d2, d3, dout, pts));
  else BK_TRY(bk_launch(c, k_jet<2>, bk_lin_grid(c, pts), 256, 0, op, du, d1, d2, d3, dout, pts));
  return bk_stage_out(c, out, n, dout);
}

extern "C" int32_t bk_d2f(bk_ctx* c, const double* u, const double* dx1, const double* dx2, double* out) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_d2f");
  return jet(c, u, dx1, dx2, nullptr, out);
}

extern "C" int32_t bk_d3f(bk_ctx* c, const double* u, const double* dx1, const double* dx2, const double* dx3, double* out) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_d3f");
  BK_CHECK(c, dx3 != nullptr, "null vector argument");
  return jet(c, u, dx1, dx2, dx3, out);
}

// grow a lazily allocated per-context buffer to at least `bytes` (its contents are not kept)
static int grow(bk_ctx* c, void** buf, size_t* cap, size_t bytes) {
  if (bytes <= *cap) return BK_OK;
  if (*buf) {
    BK_CUDA(c, cudaStreamSynchronize(c->stream));
    BK_CUDA(c, cudaFree(*buf));
    *buf = nullptr;
    *cap = 0;
  }
  BK_CUDA(c, cudaMalloc(buf, bytes));
  *cap = bytes;
  return BK_OK;
}

// The device pointers of the k vectors v[0 .. k-1] of n doubles in d: a host vector is copied into row i of mom_stage (k rows),
// a device pointer passes through
static int stage_rows(bk_ctx* c, const double* const* v, int k, long long n, const double** d) {
  for (int i = 0; i < k; ++i) {
    d[i] = v[i];
    if (bk_is_device_ptr(v[i])) continue;
    BK_TRY(grow(c, (void**)&c->mom_stage, &c->mom_stage_cap, 8 * (size_t)n * k));
    double* row = c->mom_stage + (size_t)n * i;
    BK_CUDA(c, cudaMemcpyAsync(row, v[i], 8 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    c->stats.h2d_bytes += 8 * n;
    d[i] = row;
  }
  return BK_OK;
}

// The work buffer of a moment pass, mom_work: `head` bytes from its start (the tuples), then the nres results at *res and the
// G x nres partials at *part, each 256-byte aligned
static int moment_work(bk_ctx* c, size_t head, int nres, int G, double** res, double** part) {
  const size_t res_off = (head + 255) / 256 * 256, part_off = res_off + (8 * (size_t)nres + 255) / 256 * 256;
  BK_TRY(grow(c, &c->mom_work, &c->mom_work_cap, part_off + 8 * (size_t)nres * G));
  *res = (double*)((char*)c->mom_work + res_off);
  *part = (double*)((char*)c->mom_work + part_off);
  return BK_OK;
}

// The nres results of a moment pass to the host array out, through the pinned buffer mom_pinned
static int moment_results(bk_ctx* c, const double* res, int nres, double* out) {
  static_assert(BK_DEFLATION_MAX_ROOTS * 4 + 3 <= BK_JET_MOMENTS_MAX_TUPLES, "mom_pinned holds any result list");
  if (!c->mom_pinned) BK_CUDA(c, cudaMallocHost((void**)&c->mom_pinned, 8 * (size_t)BK_JET_MOMENTS_MAX_TUPLES));
  BK_CUDA(c, cudaMemcpyAsync(c->mom_pinned, res, 8 * (size_t)nres, cudaMemcpyDeviceToHost, c->stream));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  memcpy(out, c->mom_pinned, 8 * (size_t)nres);
  c->stats.d2h_bytes += 8 * nres;
  return BK_OK;
}

extern "C" int32_t bk_jet_moments(bk_ctx* c, const double* u, int32_t nvec, const double* const* vecs, int32_t n2,
                                  const int32_t* idx2, int32_t n3, const int32_t* idx3, double* out) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_jet_moments");
  int kind;
  BK_TRY(jet_kind(c, &kind));
  BK_CHECK(c, nvec >= 1 && nvec <= BK_JET_MOMENTS_MAX_VEC, "bk_jet_moments: nvec out of range");
  BK_CHECK(c, n2 >= 0 && n3 >= 0 && (long long)n2 + n3 <= BK_JET_MOMENTS_MAX_TUPLES, "bk_jet_moments: too many tuples");
  BK_CHECK(c, u && vecs && out && (n2 == 0 || idx2) && (n3 == 0 || idx3), "null argument");
  for (int i = 0; i < nvec; ++i) BK_CHECK(c, vecs[i] != nullptr, "null vector argument");
  const int ntup = n2 + n3;
  std::vector<int4> tup(ntup);
  for (int t = 0; t < ntup; ++t) {
    const int32_t* q = t < n2 ? idx2 + 3 * t : idx3 + 4 * (t - n2);
    const int k = t < n2 ? 3 : 4;
    for (int e = 0; e < k; ++e) BK_CHECK(c, q[e] >= 0 && q[e] < nvec, "bk_jet_moments: vector index out of range");
    tup[t] = make_int4(q[0], q[1], q[2], k == 4 ? q[3] : 0);
  }
  if (ntup == 0) return BK_OK;
  const long long n = c->N0, fields = bk_traits(c)->fields, pts = n / fields;
  MomVecs vs = {};  // the nvec vectors, then u
  const double* src[BK_JET_MOMENTS_MAX_VEC + 1];
  std::copy(vecs, vecs + nvec, src);
  src[nvec] = u;
  BK_TRY(stage_rows(c, src, nvec + 1, n, vs.v));
  const int G = bk_reduce_grid(c, pts);
  const size_t tup_bytes = 16 * (size_t)ntup;
  double *dres, *dpart;
  BK_TRY(moment_work(c, tup_bytes, ntup, G, &dres, &dpart));
  BK_CUDA(c, cudaMemcpyAsync(c->mom_work, tup.data(), tup_bytes, cudaMemcpyHostToDevice, c->stream));
  c->stats.h2d_bytes += tup_bytes;
  const OpDesc op = bk_make_residual_op(c);
  const size_t smem = 8 * ((size_t)(nvec + 1) * fields * (BK_MOM_TP + 1) + ntup);
  if (kind == BK_RD) {
    static decltype(&k_rd_jet_moments<1>) const kern[4] = {k_rd_jet_moments<1>, k_rd_jet_moments<2>, k_rd_jet_moments<3>,
                                                               k_rd_jet_moments<4>};
    BK_TRY(bk_launch(c, kern[fields - 1], G, 256, smem, c->rd_par, vs, (int)nvec, (const int4*)c->mom_work, ntup, (int)n2, pts,
                     dpart));
  } else {
    const auto kern = kind == BK_CGL2D ? k_jet_moments<BK_CGL2D> : kind == BK_CHAN ? k_jet_moments<BK_CHAN> : k_jet_moments<BK_SH2D>;
    BK_TRY(bk_launch(c, kern, G, 256, smem, op, vs, (int)nvec, (const int4*)c->mom_work, ntup, (int)n2, pts, dpart));
  }
  BK_TRY(bk_launch_ordered(c, k_jet_moments_fold, (ntup + 255) / 256, 256, 0, (const double*)dpart, ntup, G, dres));
  return moment_results(c, dres, ntup, out);
}

extern "C" int32_t bk_deflation_moments(bk_ctx* c, const double* u, int32_t nroots, const double* const* roots, int32_t ndir,
                                        const double* const* dirs, int64_t n, double* out) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_deflation_moments");
  BK_CHECK(c, !c->cplx, "bk_deflation_moments: not available in a BK_COMPLEX context");
  BK_CHECK(c, nroots >= 1 && nroots <= BK_DEFLATION_MAX_ROOTS, "bk_deflation_moments: nroots out of range");
  BK_CHECK(c, ndir >= 0 && ndir <= 2, "bk_deflation_moments: ndir out of range");
  BK_CHECK(c, n >= 1 && n <= c->N0, "bk_deflation_moments: n out of range");
  BK_CHECK(c, u && roots && out && (ndir == 0 || dirs), "null argument");
  for (int i = 0; i < nroots; ++i) BK_CHECK(c, roots[i] != nullptr, "null root");
  for (int a = 0; a < ndir; ++a) BK_CHECK(c, dirs[a] != nullptr, "null direction");
  const double* src[BK_DEFLATION_MAX_ROOTS + 3];  // the roots, the directions, u
  const double* dev[BK_DEFLATION_MAX_ROOTS + 3];
  std::copy(roots, roots + nroots, src);
  std::copy(dirs, dirs + ndir, src + nroots);
  src[nroots + ndir] = u;
  BK_TRY(stage_rows(c, src, nroots + ndir + 1, n, dev));
  DeflVecs vs = {};
  std::copy(dev, dev + nroots, vs.r);
  std::copy(dev + nroots, dev + nroots + ndir, vs.h);
  vs.u = dev[nroots + ndir];
  const int W = 2 + ndir, ncol = nroots * W + ndir * (ndir + 1) / 2;
  const int G = bk_reduce_grid(c, (n + BK_DEFL_PPT - 1) / BK_DEFL_PPT);
  double *dres, *dpart;
  BK_TRY(moment_work(c, 0, ncol, G, &dres, &dpart));
  const auto kern = ndir == 0 ? k_deflation_moments<0> : ndir == 1 ? k_deflation_moments<1> : k_deflation_moments<2>;
  BK_TRY(bk_launch(c, kern, G, 256, 0, vs, (int)nroots, (long long)n, dpart));
  BK_TRY(bk_launch_ordered(c, k_deflation_moments_fold, (32 * ncol + 255) / 256, 256, 0, (const double*)dpart, ncol, nroots * W, W,
                           G, dres));
  return moment_results(c, dres, ncol, out);
}

extern "C" int32_t bk_potrap_set_section(bk_ctx* c, const double* phi, const double* xpi) {
  BK_ENTER(c);
  BK_CHECK(c, c->kind == BK_POTRAP_CGL2D, "not a potrap context");
  long long n = c->N - 1;
  cudaMemcpyKind k1 = bk_is_device_ptr(phi) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
  BK_CUDA(c, cudaMemcpyAsync(c->phi, phi, 8 * (size_t)n, k1, c->stream));
  if (xpi) {
    cudaMemcpyKind k2 = bk_is_device_ptr(xpi) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    BK_CUDA(c, cudaMemcpyAsync(c->xpi, xpi, 8 * (size_t)n, k2, c->stream));
  } else {
    BK_CUDA(c, cudaMemsetAsync(c->xpi, 0, 8 * (size_t)n, c->stream));
  }
  return bk_dev_dot(c, c->xpi, c->phi, n, &c->phi_dot_xpi);
}

extern "C" int32_t bk_potrap_update_section(bk_ctx* c, const double* x, double scale) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_potrap_update_section");
  BK_CHECK(c, c->kind == BK_POTRAP_CGL2D, "not a potrap context");
  BK_CHECK(c, x != nullptr, "null orbit");
  const long long n = c->N - 1;
  double* dx;
  BK_TRY(bk_stage_in(c, x, n, 0, true, &dx));
  const OpDesc op = bk_make_residual_op(c);  // F at the context's current params, as the residual
  BK_TRY(bk_launch(c, k_potrap_section, bk_lin_grid(c, (long long)op.nx * op.ny * op.nz), 256, 0, op, dx, scale, c->phi, c->xpi));
  return bk_dev_dot(c, c->xpi, c->phi, n, &c->phi_dot_xpi);
}
