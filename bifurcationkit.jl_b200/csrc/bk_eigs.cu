// bk_eigs.cu -- S10 / K5: shift-invert Arnoldi eigensolver for stability detection.
//
// Replaces (eig_si::ShiftInvert)(J, nev) (src/EigSolver.jl:257-266) together with the Krylov package
// behind it (ArnoldiMethod.partialschur / KrylovKit.eigsolve, src/EigSolver.jl:157-160,204-225; the
// hand-rolled equivalent examples/SH3d.jl:103-113 uses krylovdim = max(30, nev+30)):
//   Jmap(rhs) = ls(J, rhs; a0 = -sigma, a1 = 1)[1]   -> one bk_gmres_dev solve per Arnoldi vector,
//   i.e. the same fused JVP+Arnoldi kernels as the corrector;
//   eigenvalues theta of (J - sigma)^-1 of largest magnitude, lambda = sigma + 1/theta, sorted by
//   decreasing real part (src/EigSolver.jl:16-19).
// Outer iteration: Arnoldi with two classical Gram-Schmidt passes (CGS2) on the device (same k2_dots /
// k2_update kernels as GMRES), restarted by thick_restart for kinds with a symmetric Jacobian (Jacobi on
// the projected matrix) and by explicit_restart for the others (the small Hessenberg eigenproblem by
// complex shifted QR + inverse iteration on the host, like the Givens rotations of GMRES).  Both fill one
// Ritz result and share one convergence test; eig_work grows the workspace only after every argument check.
#include <algorithm>
#include <cmath>
#include <complex>
#include <vector>
#include "bk_common.cuh"

typedef std::complex<double> cplx;

// Eigenvalues of a real upper-Hessenberg matrix (n x n, column-major H[i + j*ldh]) by the complex
// single-shift QR algorithm with Wilkinson shifts and deflation.
static bool hess_eigvals(const std::vector<double>& Hr, int n, int ldh, std::vector<cplx>& ev) {
  std::vector<cplx> A((size_t)n * n);
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < n; ++i) A[i + (size_t)j * n] = (i <= j + 1) ? cplx(Hr[i + (size_t)j * ldh], 0.0) : cplx(0, 0);
  ev.assign(n, cplx(0, 0));
  int hi = n - 1, iter = 0;
  const double eps = 2.2e-16;
  std::vector<cplx> cs(n), sn(n);
  while (hi >= 0) {
    if (hi == 0) {
      ev[0] = A[0];
      break;
    }
    int l = hi;
    while (l > 0) {
      double s = std::abs(A[(l - 1) + (size_t)(l - 1) * n]) + std::abs(A[l + (size_t)l * n]);
      if (s == 0.0) s = 1.0;
      if (std::abs(A[l + (size_t)(l - 1) * n]) < eps * s) {
        A[l + (size_t)(l - 1) * n] = 0.0;
        break;
      }
      --l;
    }
    if (l == hi) {
      ev[hi] = A[hi + (size_t)hi * n];
      --hi;
      iter = 0;
      continue;
    }
    if (++iter > 60 * n) return false;
    // Wilkinson shift from the trailing 2x2 block
    cplx a = A[(hi - 1) + (size_t)(hi - 1) * n], b = A[(hi - 1) + (size_t)hi * n], c = A[hi + (size_t)(hi - 1) * n],
         d = A[hi + (size_t)hi * n];
    cplx tr = a + d, det = a * d - b * c;
    cplx disc = std::sqrt(tr * tr - 4.0 * det);
    cplx m1 = 0.5 * (tr + disc), m2 = 0.5 * (tr - disc);
    cplx mu = (std::abs(m1 - d) < std::abs(m2 - d)) ? m1 : m2;
    if (iter % 11 == 10) mu += cplx(std::abs(c), 0.37 * std::abs(c));  // exceptional shift
    // QR step on the active block l..hi
    for (int i = l; i <= hi; ++i) A[i + (size_t)i * n] -= mu;
    for (int k = l; k < hi; ++k) {
      cplx x = A[k + (size_t)k * n], y = A[(k + 1) + (size_t)k * n];
      double r = std::sqrt(std::norm(x) + std::norm(y));
      cplx c_, s_;
      if (r == 0.0) {
        c_ = 1.0;
        s_ = 0.0;
      } else {
        c_ = x / r;
        s_ = y / r;
      }
      cs[k] = c_;
      sn[k] = s_;
      // rows k, k+1:  [ conj(c) conj(s); -s c ]
      for (int j = k; j < n; ++j) {
        cplx t1 = A[k + (size_t)j * n], t2 = A[(k + 1) + (size_t)j * n];
        A[k + (size_t)j * n] = std::conj(c_) * t1 + std::conj(s_) * t2;
        A[(k + 1) + (size_t)j * n] = -s_ * t1 + c_ * t2;
      }
    }
    for (int k = l; k < hi; ++k) {
      cplx c_ = cs[k], s_ = sn[k];
      int top = std::min(hi, k + 2);
      for (int i = 0; i <= top; ++i) {
        cplx t1 = A[i + (size_t)k * n], t2 = A[i + (size_t)(k + 1) * n];
        A[i + (size_t)k * n] = t1 * c_ + t2 * s_;
        A[i + (size_t)(k + 1) * n] = -t1 * std::conj(s_) + t2 * std::conj(c_);
      }
    }
    for (int i = l; i <= hi; ++i) A[i + (size_t)i * n] += mu;
  }
  return true;
}

// Eigenvector of the real Hessenberg matrix for eigenvalue theta by inverse iteration (complex LU with
// partial pivoting).  Returns the unit-norm vector y.
static void hess_eigvec(const std::vector<double>& Hr, int n, int ldh, cplx theta, std::vector<cplx>& y) {
  double hn = 0;
  for (int j = 0; j < n; ++j)
    for (int i = 0; i <= std::min(n - 1, j + 1); ++i) hn = std::max(hn, std::fabs(Hr[i + (size_t)j * ldh]));
  if (hn == 0) hn = 1;
  cplx th = theta + cplx(1e-10 * hn, 1e-11 * hn);  // perturb so that the matrix is invertible
  std::vector<cplx> A((size_t)n * n);
  for (int j = 0; j < n; ++j)
    for (int i = 0; i < n; ++i) {
      cplx v = (i <= j + 1) ? cplx(Hr[i + (size_t)j * ldh], 0.0) : cplx(0, 0);
      if (i == j) v -= th;
      A[i + (size_t)j * n] = v;
    }
  std::vector<int> piv(n);
  for (int k = 0; k < n; ++k) {
    int p = k;
    double best = std::abs(A[k + (size_t)k * n]);
    for (int i = k + 1; i < n; ++i)
      if (std::abs(A[i + (size_t)k * n]) > best) {
        best = std::abs(A[i + (size_t)k * n]);
        p = i;
      }
    piv[k] = p;
    if (p != k)
      for (int j = 0; j < n; ++j) std::swap(A[k + (size_t)j * n], A[p + (size_t)j * n]);
    if (std::abs(A[k + (size_t)k * n]) < 1e-300) A[k + (size_t)k * n] = 1e-300;
    for (int i = k + 1; i < n; ++i) {
      cplx f = A[i + (size_t)k * n] / A[k + (size_t)k * n];
      A[i + (size_t)k * n] = f;
      if (f != cplx(0, 0))
        for (int j = k + 1; j < n; ++j) A[i + (size_t)j * n] -= f * A[k + (size_t)j * n];
    }
  }
  y.assign(n, cplx(1.0, 0.0));
  for (int i = 0; i < n; ++i) y[i] = cplx(1.0 / (1.0 + i), 0.3 / (2.0 + i));
  for (int it = 0; it < 3; ++it) {
    for (int k = 0; k < n; ++k)
      if (piv[k] != k) std::swap(y[k], y[piv[k]]);  // whole rows were swapped (getrf style): permute first
    for (int k = 0; k < n; ++k)
      for (int i = k + 1; i < n; ++i) y[i] -= A[i + (size_t)k * n] * y[k];
    for (int k = n - 1; k >= 0; --k) {
      for (int j = k + 1; j < n; ++j) y[k] -= A[k + (size_t)j * n] * y[j];
      y[k] /= A[k + (size_t)k * n];
    }
    double nr = 0;
    for (auto& v : y) nr += std::norm(v);
    nr = std::sqrt(nr);
    for (auto& v : y) v /= nr;
  }
  // fix the phase: largest component real positive
  int im = 0;
  for (int i = 1; i < n; ++i)
    if (std::abs(y[i]) > std::abs(y[im])) im = i;
  cplx ph = std::conj(y[im]) / std::abs(y[im]);
  for (auto& v : y) v *= ph;
}

// Host-only utility (no GPU needed): eigen-decomposition of a real upper-Hessenberg matrix, the small dense
// problem the Arnoldi eigensolver hands to the host.  Exposed so that it can be validated on CPU against
// the reference's golden spectrum (test/linear_solvers/test_linear.jl:595-614).
extern "C" int32_t bk_hessenberg_eig(const double* H, int32_t n, int32_t ldh, double* wr, double* wi, double* vec_re,
                                     double* vec_im) {
  if (!H || n < 1 || ldh < n || !wr || !wi) return BK_ERR_ARG;
  std::vector<double> Hc((size_t)ldh * n);
  for (size_t i = 0; i < Hc.size(); ++i) Hc[i] = H[i];
  std::vector<cplx> ev;
  if (!hess_eigvals(Hc, n, ldh, ev)) return BK_NOT_CONVERGED;
  std::vector<cplx> y;
  for (int q = 0; q < n; ++q) {
    wr[q] = ev[q].real();
    wi[q] = ev[q].imag();
    if (vec_re && vec_im) {
      hess_eigvec(Hc, n, ldh, ev[q], y);
      for (int i = 0; i < n; ++i) {
        vec_re[i + (size_t)q * n] = y[i].real();
        vec_im[i + (size_t)q * n] = y[i].imag();
      }
    }
  }
  return BK_OK;
}

// Symmetric eigen-decomposition by cyclic Jacobi rotations: A (n x n, column-major, overwritten) = S diag(w) S^T.
static void jacobi_eig(std::vector<double>& A, int n, std::vector<double>& w, std::vector<double>& S) {
  S.assign((size_t)n * n, 0.0);
  for (int i = 0; i < n; ++i) S[i + (size_t)i * n] = 1.0;
  for (int sweep = 0; sweep < 60; ++sweep) {
    double off = 0, dg = 0;
    for (int j = 0; j < n; ++j)
      for (int i = 0; i < n; ++i) (i == j ? dg : off) += A[i + (size_t)j * n] * A[i + (size_t)j * n];
    if (off <= 1e-32 * (dg + 1e-300)) break;
    for (int p = 0; p < n - 1; ++p)
      for (int q = p + 1; q < n; ++q) {
        double apq = A[p + (size_t)q * n];
        if (apq == 0.0) continue;
        double app = A[p + (size_t)p * n], aqq = A[q + (size_t)q * n];
        double th = (aqq - app) / (2.0 * apq);
        double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
        double cs = 1.0 / sqrt(t * t + 1.0), sn = t * cs;
        for (int k = 0; k < n; ++k) {  // columns p, q
          double akp = A[k + (size_t)p * n], akq = A[k + (size_t)q * n];
          A[k + (size_t)p * n] = cs * akp - sn * akq;
          A[k + (size_t)q * n] = sn * akp + cs * akq;
        }
        for (int k = 0; k < n; ++k) {  // rows p, q
          double apk = A[p + (size_t)k * n], aqk = A[q + (size_t)k * n];
          A[p + (size_t)k * n] = cs * apk - sn * aqk;
          A[q + (size_t)k * n] = sn * apk + cs * aqk;
        }
        for (int k = 0; k < n; ++k) {
          double skp = S[k + (size_t)p * n], skq = S[k + (size_t)q * n];
          S[k + (size_t)p * n] = cs * skp - sn * skq;
          S[k + (size_t)q * n] = sn * skp + cs * skq;
        }
      }
  }
  w.resize(n);
  for (int i = 0; i < n; ++i) w[i] = A[i + (size_t)i * n];
}

static __global__ void k_fill_ones(double* p, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 1.0;
}
// deterministic start vector (the reference uses rand(); any generic vector works)
static __global__ void k_start_vector(double* v, long long n) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    unsigned long long z = (unsigned long long)i * 0x9E3779B97F4A7C15ULL + 0x1234567ULL;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ULL;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBULL;
    z ^= z >> 31;
    v[i] = (double)(z >> 11) * (1.0 / 9007199254740992.0) + 0.05;
  }
}

// Arnoldi workspace of the eigensolver: slots of S = m + 4 doubles in c->eig_dev and the pinned host mirror c->eig_pinned
struct EigWork {
  int S;
  double* ones;  // all ones: the basis Q is stored normalised
  double* hA;    // H column of the first Gram-Schmidt pass, followed by hB
  double* hB;    // second-pass corrections
  double* gco;   // dot-product coefficients handed from k2_dots to k2_update
  double* coef;  // 2 S: lincomb coefficients
  double* hp;    // pinned host copy of hA | hB; also the staged coefficients of q_lincomb
};

// The workspace for Krylov dimension m: grows Q, eig_dev and eig_pinned together (and Q2 for the thick restart of sym kinds)
static int eig_work(bk_ctx* c, int m, bool sym, EigWork* ws) {
  if (c->qcap < m) {
    BK_CUDA(c, cudaStreamSynchronize(c->stream));
    if (c->Q) cudaFree(c->Q);
    if (c->eig_dev) cudaFree(c->eig_dev);
    if (c->eig_pinned) cudaFreeHost(c->eig_pinned);
    c->Q = c->eig_dev = c->eig_pinned = nullptr;
    BK_CUDA(c, cudaMalloc(&c->Q, 8 * (size_t)c->ld * (m + 1)));
    BK_CUDA(c, cudaMalloc(&c->eig_dev, 8 * (size_t)(m + 4) * 6));
    BK_CUDA(c, cudaMallocHost(&c->eig_pinned, 8 * (size_t)(m + 4) * 6));
    c->qcap = m;
    BK_TRY(bk_launch_ordered(c, k_fill_ones, (m + 4 + 255) / 256, 256, 0, c->eig_dev, m + 4));
  }
  if (sym && (!c->Q2 || c->q2cap < m)) {
    BK_CUDA(c, cudaStreamSynchronize(c->stream));
    if (c->Q2) cudaFree(c->Q2);
    BK_CUDA(c, cudaMalloc(&c->Q2, 8 * (size_t)c->ld * (m + 1)));
    c->q2cap = m;
  }
  const int S = m + 4;
  *ws = EigWork{S, c->eig_dev, c->eig_dev + S, c->eig_dev + 2 * S, c->eig_dev + 3 * S, c->eig_dev + 4 * S, c->eig_pinned};
  return BK_OK;
}

// dst = sum_i coef[i] Q_i over the first k columns (coef on the host), copied on to host memory `host` when given.  The
// coefficients travel through the pinned ws.hp, so the call ends with a stream synchronise before ws.hp can be written again.
static int q_lincomb(bk_ctx* c, const EigWork& ws, const double* coef, int k, long long n, double* dst, double* host = nullptr) {
  std::copy(coef, coef + k, ws.hp);
  BK_CUDA(c, cudaMemcpyAsync(ws.coef, ws.hp, 8 * (size_t)k, cudaMemcpyHostToDevice, c->stream));
  BK_TRY(bk_launch_lincomb(c, c->Q, nullptr, dst, 0.0, n, k, ws.coef));
  if (host) {
    BK_CUDA(c, cudaMemcpyAsync(host, dst, 8 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
    c->stats.d2h_bytes += 8 * n;
  }
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  return BK_OK;
}

// Q_0 = x / ||x||
static int arnoldi_start(bk_ctx* c, const EigWork& ws, const double* x, long long n) {
  BK_TRY(bk_launch_update(c, c->Q, ws.gco, x, n, 0, c->Q, ws.hA, ws.hB));
  BK_CUDA(c, cudaMemcpyAsync(ws.hp, ws.hA, 8, cudaMemcpyDeviceToHost, c->stream));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  BK_CHECK(c, ws.hp[0] > 0, "zero start vector");
  BK_TRY(bk_dev_scale(c, c->Q, 1.0 / ws.hp[0], n));
  return BK_OK;
}

// Arnoldi expansion of columns kstart..m-1 of H ((m + 1) x m, column-major): Q_{k+1} from one inner solve x = (J - sigma)^-1 Q_k
// and two classical Gram-Schmidt passes.  Stops early at an invariant subspace; *keff is the number of columns of H filled.
// Adds the inner solves to *nops.
static int arnoldi_expand(bk_ctx* c, const EigWork& ws, const OpDesc& op, const bk_gmres_opts* inner, double* x, long long n,
                          int m, int kstart, std::vector<double>& H, int* keff, int* nops) {
  const int S = ws.S;
  *keff = m;
  for (int k = kstart; k < m; ++k) {
    const int j = k + 1;
    int cv = 0, it = 0;
    int st = bk_gmres_dev(c, op, c->Q + (size_t)k * c->ld, x, inner, &cv, &it, nullptr);
    if (st < 0) return st;
    ++*nops;
    double* qn = c->Q + (size_t)(k + 1) * c->ld;
    BK_TRY(bk_launch_dots(c, c->Q, ws.ones, x, n, j, ws.hA, ws.gco));
    BK_TRY(bk_launch_update(c, c->Q, ws.gco, x, n, j, qn, ws.hA + j, ws.hB + S - 1));
    BK_TRY(bk_launch_dots(c, c->Q, ws.ones, qn, n, j, ws.hB, ws.gco));
    BK_TRY(bk_launch_update(c, c->Q, ws.gco, qn, n, j, qn, ws.hA + j, ws.hB + S - 1));
    BK_CUDA(c, cudaMemcpyAsync(ws.hp, ws.hA, 8 * (size_t)(2 * S), cudaMemcpyDeviceToHost, c->stream));
    BK_CUDA(c, cudaStreamSynchronize(c->stream));
    const double* hp = ws.hp;
    double cn = 0;
    for (int i = 0; i < j; ++i) {
      H[i + (size_t)k * (m + 1)] = hp[i] + hp[S + i];
      cn = fmax(cn, fabs(H[i + (size_t)k * (m + 1)]));
    }
    double hk1 = hp[j];
    H[j + (size_t)k * (m + 1)] = hk1;
    if (!(hk1 > 1e-14 * fmax(cn, 1e-300))) {  // invariant subspace found
      *keff = k + 1;
      return BK_OK;
    }
    BK_TRY(bk_dev_scale(c, qn, 1.0 / hk1, n));
  }
  return BK_OK;
}

namespace {
// What a restart strategy hands back: the min(nev, keff) wanted Ritz values theta of (J - sigma)^-1, their vectors y in the
// basis Q_0..Q_{keff-1}, whether they converged, and the inner solves spent
struct Ritz {
  std::vector<cplx> theta;
  std::vector<std::vector<cplx>> Y;
  int keff;
  bool converged = false;
  int nops = 0;
};
}  // namespace

// The Ritz test shared by both restarts on the pairs (theta_q, y_q), q < min(nev, keff), of one Arnoldi factorisation: the
// residual |h_{m+1,m}| |y_q[keff-1]| of every pair is within tol |theta_q|, or the Krylov space is invariant (keff < m).  The
// thick restart's pairs are real: std::abs(cplx(x, 0)) is hypot(x, 0) = |x| exactly.
static void ritz_test(Ritz& r, int nev, int m, const std::vector<double>& H, double tol) {
  const int nv = std::min(nev, r.keff);
  const double hlast = (r.keff == m) ? H[m + (size_t)(m - 1) * (m + 1)] : 0.0;
  bool all = true;
  for (int q = 0; q < nv; ++q)
    if (fabs(hlast) * std::abs(r.Y[q][r.keff - 1]) > tol * fmax(std::abs(r.theta[q]), 1e-300)) all = false;
  r.converged = all || r.keff < m;
}

// Symmetric operators (Swift-Hohenberg): thick restart (Krylov-Schur with Ritz vectors).  Each restart keeps the pkeep
// wanted Ritz vectors and the residual direction, and expands from there.
static int thick_restart(bk_ctx* c, const EigWork& ws, const OpDesc& op, const bk_gmres_opts* inner, double* x, long long n,
                         int m, int nev, double tol, int maxrestart, Ritz& r) {
  std::vector<double> H((size_t)(m + 1) * m), S, w;
  std::vector<int> order;
  BK_TRY(arnoldi_start(c, ws, x, n));
  int kstart = 0;
  for (int rs = 0; rs < maxrestart && !r.converged; ++rs) {
    BK_TRY(arnoldi_expand(c, ws, op, inner, x, n, m, kstart, H, &r.keff, &r.nops));
    const int keff = r.keff;
    // symmetrised projected matrix (exactly symmetric in exact arithmetic), mirrored from the upper triangle of H.  After a
    // restart the retained Ritz values sit on the diagonal of columns 0..kstart-1, and the arrow <Q_q, Op q_kstart> that couples
    // them to the residual direction is column kstart's Gram-Schmidt coefficients, so the lower triangle is never needed.
    std::vector<double> A((size_t)keff * keff);
    for (int jj = 0; jj < keff; ++jj)
      for (int i = 0; i < keff; ++i) A[i + (size_t)jj * keff] = H[std::min(i, jj) + (size_t)std::max(i, jj) * (m + 1)];
    jacobi_eig(A, keff, w, S);
    order.resize(keff);
    for (int i = 0; i < keff; ++i) order[i] = i;
    std::sort(order.begin(), order.end(), [&](int a, int b) { return fabs(w[a]) > fabs(w[b]); });
    for (int q = 0; q < std::min(nev, keff); ++q) {
      r.theta[q] = cplx(w[order[q]], 0.0);
      r.Y[q].assign(S.begin() + (size_t)order[q] * keff, S.begin() + (size_t)(order[q] + 1) * keff);  // column order[q] of S
    }
    ritz_test(r, nev, m, H, tol);
    if (!r.converged && rs + 1 < maxrestart) {
      int pkeep = std::min(keff - 2, nev + std::max(8, (m - nev) / 3));
      if (pkeep < 1) pkeep = 1;
      for (int q = 0; q < pkeep; ++q)  // Q2_q = Q S[:, order[q]]
        BK_TRY(q_lincomb(c, ws, S.data() + (size_t)order[q] * keff, keff, n, c->Q2 + (size_t)q * c->ld));
      BK_TRY(bk_dev_copy(c, c->Q2 + (size_t)pkeep * c->ld, c->Q + (size_t)keff * c->ld, n));  // residual direction q_{m+1}
      BK_CUDA(c, cudaMemcpyAsync(c->Q, c->Q2, 8 * (size_t)c->ld * (pkeep + 1), cudaMemcpyDeviceToDevice, c->stream));
      std::fill(H.begin(), H.end(), 0.0);
      for (int q = 0; q < pkeep; ++q) H[q + (size_t)q * (m + 1)] = w[order[q]];
      kstart = pkeep;
    }
  }
  return BK_OK;
}

// The other operators: explicit restart from the sum of the real parts of the wanted Ritz vectors.
static int explicit_restart(bk_ctx* c, const EigWork& ws, const OpDesc& op, const bk_gmres_opts* inner, double* x, long long n,
                            int m, int nev, double tol, int maxrestart, Ritz& r) {
  std::vector<double> H((size_t)(m + 1) * m);
  std::vector<cplx> ev;
  for (int rs = 0; rs < maxrestart && !r.converged; ++rs) {
    std::fill(H.begin(), H.end(), 0.0);
    BK_TRY(arnoldi_start(c, ws, x, n));
    BK_TRY(arnoldi_expand(c, ws, op, inner, x, n, m, 0, H, &r.keff, &r.nops));
    const int keff = r.keff;
    BK_CHECK(c, hess_eigvals(H, keff, m + 1, ev), "QR iteration on the Hessenberg matrix did not converge");
    // the complex QR returns the members of a conjugate pair with moduli that differ in the last bits: make them exact
    // conjugates, so that the tie rule below, and not rounding, decides which member an nev cutting the pair keeps
    for (int i = 0; i < keff; ++i) {
      if (!(ev[i].imag() > 0)) continue;
      int jb = -1;
      for (int j = 0; j < keff; ++j)
        if (ev[j].imag() < 0 && (jb < 0 || std::abs(ev[j] - std::conj(ev[i])) < std::abs(ev[jb] - std::conj(ev[i])))) jb = j;
      if (jb < 0) continue;
      const double d = std::abs(ev[jb] - std::conj(ev[i]));
      if (d <= 1e-8 * std::abs(ev[i]) && d < ev[i].imag()) ev[jb] = std::conj(ev[i]);
    }
    std::sort(ev.begin(), ev.end(), [](const cplx& a, const cplx& b) {
      double da = std::abs(a), db = std::abs(b);
      if (da != db) return da > db;
      return a.imag() > b.imag();
    });
    const int nv = std::min(nev, keff);
    for (int q = 0; q < nv; ++q) {
      r.theta[q] = ev[q];
      hess_eigvec(H, keff, m + 1, ev[q], r.Y[q]);
    }
    ritz_test(r, nev, m, H, tol);
    if (!r.converged && rs + 1 < maxrestart) {
      std::vector<double> v(keff, 0.0);  // restart vector = sum of the real parts of the wanted Ritz vectors
      for (int q = 0; q < nv; ++q)
        for (int i = 0; i < keff; ++i) v[i] += r.Y[q][i].real();
      BK_TRY(q_lincomb(c, ws, v.data(), keff, n, x));
    }
  }
  return BK_OK;
}

extern "C" int32_t bk_eigs_shift_invert(bk_ctx* c, double sigma, int32_t nev, int32_t krylovdim, double tol,
                                        int32_t maxrestart, const bk_gmres_opts* inner, const double* v0, double* vals_re,
                                        double* vals_im, double* vecs, int32_t* nconv, int32_t* nops) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_eigs_shift_invert");
  // the operator of a complex context is the real-equivalent form of ((-sigma + i a0_imag) I + J): neither symmetric for the
  // thick restart nor mapped back by lambda = sigma + 1/theta, and every eigenvalue of J would come out twice
  BK_CHECK(c, !c->cplx, "bk_eigs_shift_invert: not available in a BK_COMPLEX context");
  BK_CHECK(c, c->have_state, "bk_jac_set_state must be called first");
  BK_CHECK(c, inner != nullptr && vals_re && vals_im, "null argument");
  const long long n = c->N;
  int m = krylovdim;
  if ((long long)m > n) m = (int)n;
  BK_CHECK(c, nev >= 1 && nev <= m, "need 1 <= nev <= krylovdim <= N");
  // partial-sum buffer must hold m rows
  BK_CHECK(c, m <= c->m, "krylovdim exceeds the context's krylov_m (partial-sum workspace)");
  if (maxrestart < 1) maxrestart = 1;
  const bool sym = bk_traits(c)->jac_sym;
  EigWork ws;
  BK_TRY(eig_work(c, m, sym, &ws));
  double* x;
  BK_TRY(bk_tmp(c, 3, &x));
  OpDesc op = bk_make_op(c, -sigma, 1.0);  // (a0 I + a1 J) with a0 = -sigma (src/EigSolver.jl:260)
  if (v0) {
    cudaMemcpyKind kd = bk_is_device_ptr(v0) ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice;
    BK_CUDA(c, cudaMemcpyAsync(x, v0, 8 * (size_t)n, kd, c->stream));
  } else {
    BK_TRY(bk_launch_ordered(c, k_start_vector, c->nsm * 4, 256, 0, x, n));
  }
  Ritz r{std::vector<cplx>(nev), std::vector<std::vector<cplx>>(nev), m};
  BK_TRY((sym ? thick_restart : explicit_restart)(c, ws, op, inner, x, n, m, nev, tol, maxrestart, r));
  // map back, sort by decreasing real part (ties: decreasing imaginary part)
  const int nv = std::min<int>(nev, r.keff);
  std::vector<int> idx(nv);
  std::vector<cplx> lam(nv);
  for (int q = 0; q < nv; ++q) {
    idx[q] = q;
    lam[q] = sigma + 1.0 / r.theta[q];
  }
  std::sort(idx.begin(), idx.end(), [&](int a, int b) {
    if (lam[a].real() != lam[b].real()) return lam[a].real() > lam[b].real();
    return lam[a].imag() > lam[b].imag();
  });
  for (int q = 0; q < nev; ++q) {
    vals_re[q] = q < nv ? lam[idx[q]].real() : NAN;
    vals_im[q] = q < nv ? lam[idx[q]].imag() : NAN;
  }
  if (vecs) {
    // column q = Re(Q y_q) for real eigenvalues and for the member of a pair with Im >= 0; Im(Q y_q) for Im < 0
    double* tmpv;
    BK_TRY(bk_tmp(c, 4, &tmpv));
    const bool dev_out = bk_is_device_ptr(vecs);
    std::vector<double> yq(r.keff);
    for (int q = 0; q < nv; ++q) {
      const std::vector<cplx>& y = r.Y[idx[q]];
      const bool use_im = lam[idx[q]].imag() < 0;
      for (int i = 0; i < r.keff; ++i) yq[i] = use_im ? y[i].imag() : y[i].real();
      double* col = vecs + (size_t)q * n;
      BK_TRY(q_lincomb(c, ws, yq.data(), r.keff, n, dev_out ? col : tmpv, dev_out ? nullptr : col));
    }
  }
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  if (nconv) *nconv = r.converged ? nv : 0;
  if (nops) *nops = r.nops;
  return r.converged ? BK_OK : BK_NOT_CONVERGED;
}
