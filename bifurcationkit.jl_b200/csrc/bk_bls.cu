// bk_bls.cu -- S3/S4: bordered linear solvers of src/LinearBorderSolver.jl on device vectors.
//   BorderingBLS  (:88-123) = BEC (:125-144) [+ residualBEC (:146-166) refinement rounds]
//   MatrixFreeBLS (:404-437) = one GMRES on the (N+1)-system through MatrixFreeBLSmap (:299-335),
//                              rhs = vcat(R, n) (use_bordered_array = false, :414,:434)
// dotp(x, y) = dotscale * <x, y>  (PALC passes 1/N: src/continuation/Palc.jl:4, LinearBorderSolver.jl:22).
#include <cmath>
#include "bk_common.cuh"

// BEC: x1, dx = (shift I + J)^-1 R, (shift I + J)^-1 dR ; dl = (n - xiu dotp(dzu,x1)) / (xip dzp - xiu dotp(dzu,dx));
// dX = x1 - dl dx.   All pointers device.  dX receives the result; tmp_dx is scratch.
static int bec(bk_ctx* c, const double* dR, const double* dzu, double dzp, const double* R, double n, double xiu, double xip,
               double a0, double dotscale, const bk_gmres_opts* o, double* dX, double* tmp_dx, double* dl, int* cv,
               int iters[2]) {
  const long long N = c->N;
  OpDesc op = bk_make_op(c, a0, 1.0);
  int c1 = 0, c2 = 0, i1 = 0, i2 = 0;
  int st = bk_gmres_dev(c, op, R, dX, o, &c1, &i1, nullptr);
  if (st < 0) return st;
  st = bk_gmres_dev(c, op, dR, tmp_dx, o, &c2, &i2, nullptr);
  if (st < 0) return st;
  double d1 = 0, d2 = 0;
  BK_TRY(bk_dev_dot(c, dzu, dX, N, &d1));
  BK_TRY(bk_dev_dot(c, dzu, tmp_dx, N, &d2));
  double l = (n - dotscale * d1 * xiu) / (dzp * xip - dotscale * d2 * xiu);
  BK_TRY(bk_dev_axpby(c, dX, -l, tmp_dx, 1.0, N));  // dX = x1 - dl dx
  *dl = l;
  *cv = c1 & c2;
  iters[0] = i1;
  iters[1] = i2;
  return BK_OK;
}

extern "C" int32_t bk_bls_bordering(bk_ctx* c, const double* dR, const double* dzu, double dzp, const double* R, double n,
                                    double xiu, double xip, int32_t has_shift, double shift, double dotscale,
                                    const bk_gmres_opts* opts, int32_t check_precision, int32_t kmax, double tol, double* dX,
                                    double* dl, int32_t* converged, int32_t iters[2]) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_bls_bordering");
  BK_CHECK(c, c->have_state, "bk_jac_set_state must be called first");
  BK_CHECK(c, opts != nullptr, "opts required");
  const long long N = c->N;
  double *d_dR, *d_dzu, *d_R, *d_dX;
  BK_TRY(bk_stage_in(c, dR, N, 6, true, &d_dR));
  BK_TRY(bk_stage_in(c, dzu, N, 7, true, &d_dzu));
  BK_TRY(bk_stage_in(c, R, N, 8, true, &d_R));
  BK_TRY(bk_stage_in(c, dX, N, 9, false, &d_dX));
  double *t_dx, *t_res, *t_dX1;
  BK_TRY(bk_tmp(c, 0, &t_dx));
  const double a0 = has_shift ? shift : 0.0;
  double l = 0;
  int cv = 0, it[2] = {0, 0};
  BK_TRY(bec(c, d_dR, d_dzu, dzp, d_R, n, xiu, xip, a0, dotscale, opts, d_dX, t_dx, &l, &cv, it));
  int k = 0;
  bool fail = true;
  while (check_precision && k < kmax && fail) {
    // residualBEC: dXr = R - (shift I + J) dX - dl dR ; dlr = n - xip dzp dl - xiu dotp(dzu, dX)
    BK_TRY(bk_tmp(c, 1, &t_res));
    BK_TRY(bk_tmp(c, 2, &t_dX1));
    OpDesc op = bk_make_op(c, a0, 1.0);
    BK_TRY(bk_launch_apply(c, op, d_dX, nullptr, t_res));
    BK_TRY(bk_dev_axpby(c, t_res, l, d_dR, 1.0, N));
    BK_TRY(bk_dev_axpby(c, t_res, 1.0, d_R, -1.0, N));
    double dd = 0, nr = 0;
    BK_TRY(bk_dev_dot(c, d_dzu, d_dX, N, &dd));
    double rl = n - xip * dzp * l - xiu * dotscale * dd;
    BK_TRY(bk_dev_dot(c, t_res, t_res, N, &nr));
    fail = sqrt(nr) > tol || fabs(rl) > tol;
    if (fail) {
      double l1 = 0;
      BK_TRY(bec(c, d_dR, d_dzu, dzp, t_res, rl, xiu, xip, a0, dotscale, opts, t_dX1, t_dx, &l1, &cv, it));
      BK_TRY(bk_dev_axpby(c, d_dX, 1.0, t_dX1, 1.0, N));
      l += l1;
      ++k;
    }
  }
  if (dl) *dl = l;
  if (converged) *converged = cv;
  if (iters) {
    iters[0] = it[0];
    iters[1] = it[1];
  }
  BK_TRY(bk_stage_out(c, dX, N, d_dX));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  return cv ? BK_OK : BK_NOT_CONVERGED;
}

// ------------------------------------------------------------------------------------------------ block / tuple borders
// solve_bls_block (src/LinearBorderSolver.jl:168-206 BorderingBLS, :440-450 MatrixFreeBLS over the tuple form of
// MatrixFreeBLSmap :338-389):   [ shift I + J   a_1 .. a_m ] [u]   [rhst]
//                               [ dotp(b_i, .)      c      ] [p] = [rhsb]       m = 1 or 2 (the Hopf / codim-2 systems)
// cmat is m x m, column-major (Julia layout).  One border (MatrixFreeBLS :404-437, MatrixFreeBLSmap :299-335) is m = 1.
static int stage_borders(bk_ctx* c, int m, const double* const* a, const double* const* b, double* da[2], double* db[2]) {
  static const int slot_a[2] = {6, 12}, slot_b[2] = {7, 13};
  for (int i = 0; i < m; ++i) {
    BK_TRY(bk_stage_in(c, a[i], c->N, slot_a[i], true, &da[i]));
    BK_TRY(bk_stage_in(c, b[i], c->N, slot_b[i], true, &db[i]));
  }
  return BK_OK;
}
static void set_block_borders(OpDesc& op, int m, double* const da[2], double* const db[2], const double* cmat, int has_shift,
                              double shift, double dotscale) {
  op.bordered = m;
  op.ba = da[0];
  op.bb = db[0];
  op.bc = cmat[0];
  if (m == 2) {
    op.ba2 = da[1];
    op.bb2 = db[1];
    op.bc10 = cmat[1];  // c[2,1]
    op.bc01 = cmat[2];  // c[1,2]
    op.bc11 = cmat[3];
  }
  op.bshift = has_shift ? shift : 0.0;
  op.bscale = dotscale;
}

static int block_map(bk_ctx* c, int m, const double* const* a, const double* const* b, const double* cmat, int has_shift,
                     double shift, double dotscale, const double* x, double* out) {
  double *da[2], *db[2], *dx, *dout;
  BK_TRY(stage_borders(c, m, a, b, da, db));
  BK_TRY(bk_stage_in(c, x, c->N + m, 0, true, &dx));
  BK_TRY(bk_stage_in(c, out, c->N + m, 1, false, &dout));
  OpDesc op = bk_make_op(c, 0.0, 1.0);
  set_block_borders(op, m, da, db, cmat, has_shift, shift, dotscale);
  BK_TRY(bk_launch_apply(c, op, dx, nullptr, dout));
  return bk_stage_out(c, out, c->N + m, dout);
}

extern "C" int32_t bk_bls_map(bk_ctx* c, const double* a, const double* b, double bc, int32_t has_shift, double shift,
                              double dotscale, const double* x, double* out) {
  BK_ENTER(c);
  BK_CHECK(c, c->have_state, "bk_jac_set_state must be called first");
  return block_map(c, 1, &a, &b, &bc, has_shift, shift, dotscale, x, out);
}

extern "C" int32_t bk_bls_block_map(bk_ctx* c, int32_t m, const double* const* a, const double* const* b, const double* cmat,
                                    int32_t has_shift, double shift, double dotscale, const double* x, double* out) {
  BK_ENTER(c);
  BK_CHECK(c, c->have_state, "bk_jac_set_state must be called first");
  BK_CHECK(c, m == 1 || m == 2, "block borders: m must be 1 or 2");
  BK_CHECK(c, a && b && cmat, "null border");
  return block_map(c, m, a, b, cmat, has_shift, shift, dotscale, x, out);
}

// the border entries of the right-hand side: v[0] = p0 (, v[1] = p1)
static __global__ void k_set_tail(double* v, int m, double p0, double p1) {
  v[0] = p0;
  if (m == 2) v[1] = p1;
}

// rhs = vcat(rhst, rhsb) (use_bordered_array = false, :414,:434), one GMRES on the (N + m)-system; rhsb and solp on the host
static int block_matrixfree(bk_ctx* c, int m, const double* const* a, const double* const* b, const double* cmat,
                            const double* rhst, const double* rhsb, int has_shift, double shift, double dotscale,
                            const bk_gmres_opts* opts, double* solu, double* solp, int32_t* converged, int32_t* iters) {
  const long long N = c->N;
  double *da[2], *db[2], *d_R;
  BK_TRY(stage_borders(c, m, a, b, da, db));
  BK_TRY(bk_stage_in(c, rhst, N, 8, true, &d_R));
  double *rhs, *sol;
  BK_TRY(bk_tmp(c, 0, &rhs));
  BK_TRY(bk_tmp(c, 1, &sol));
  BK_TRY(bk_dev_copy(c, rhs, d_R, N));
  BK_TRY(bk_launch_ordered(c, k_set_tail, 1, 1, 0, rhs + N, m, rhsb[0], m == 2 ? rhsb[1] : 0.0));
  OpDesc op = bk_make_op(c, 0.0, 1.0);
  set_block_borders(op, m, da, db, cmat, has_shift, shift, dotscale);
  int cv = 0, it = 0;
  int st = bk_gmres_dev(c, op, rhs, sol, opts, &cv, &it, nullptr);
  if (st < 0) return st;
  BK_CUDA(c, cudaMemcpyAsync(c->red_pinned + 1, sol + N, 8 * (size_t)m, cudaMemcpyDeviceToHost, c->stream));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  for (int i = 0; i < m; ++i) solp[i] = c->red_pinned[1 + i];
  if (converged) *converged = cv;
  if (iters) *iters = it;
  if (bk_is_device_ptr(solu)) {
    BK_TRY(bk_dev_copy(c, solu, sol, N));
    BK_CUDA(c, cudaStreamSynchronize(c->stream));
  } else {
    BK_TRY(bk_stage_out(c, solu, N, sol));
  }
  return cv ? BK_OK : BK_NOT_CONVERGED;
}

extern "C" int32_t bk_bls_matrixfree(bk_ctx* c, const double* dR, const double* dzu, double dzp, const double* R, double n,
                                     double xiu, double xip, int32_t has_shift, double shift, double dotscale,
                                     const bk_gmres_opts* opts, double* dX, double* dl, int32_t* converged, int32_t* iters) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_bls_matrixfree");
  BK_CHECK(c, c->have_state, "bk_jac_set_state must be called first");
  BK_CHECK(c, opts != nullptr, "opts required");
  // linearmap = MatrixFreeBLSmap(J, dR, xiu*dzu, dzp*xip, shift, dotp)  (:433)
  const double cm = dzp * xip;
  double p = 0;
  const int st = block_matrixfree(c, 1, &dR, &dzu, &cm, R, &n, has_shift, shift, dotscale * xiu, opts, dX, &p, converged, iters);
  if (st >= 0 && dl) *dl = p;
  return st;
}

extern "C" int32_t bk_bls_block_matrixfree(bk_ctx* c, int32_t m, const double* const* a, const double* const* b,
                                           const double* cmat, const double* rhst, const double* rhsb, int32_t has_shift,
                                           double shift, double dotscale, const bk_gmres_opts* opts, double* solu, double* solp,
                                           int32_t* converged, int32_t* iters) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_bls_block_matrixfree");
  BK_CHECK(c, c->have_state, "bk_jac_set_state must be called first");
  BK_CHECK(c, opts != nullptr, "opts required");
  BK_CHECK(c, m == 1 || m == 2, "block borders: m must be 1 or 2");
  BK_CHECK(c, a && b && cmat && rhsb && solp, "null border");
  return block_matrixfree(c, m, a, b, cmat, rhst, rhsb, has_shift, shift, dotscale, opts, solu, solp, converged, iters);
}

extern "C" int32_t bk_bls_block_bordering(bk_ctx* c, int32_t m, const double* const* a, const double* const* b,
                                          const double* cmat, const double* rhst, const double* rhsb, int32_t has_shift,
                                          double shift, const bk_gmres_opts* opts, double* solu, double* solp,
                                          int32_t* converged, int32_t iters[3]) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_bls_block_bordering");
  BK_CHECK(c, c->have_state, "bk_jac_set_state must be called first");
  BK_CHECK(c, opts != nullptr, "opts required");
  BK_CHECK(c, m == 1 || m == 2, "block borders: m must be 1 or 2");
  BK_CHECK(c, a && b && cmat && rhsb && solp, "null border");
  const long long N = c->N;
  double *da[2], *db[2], *d_R, *d_u;
  BK_TRY(stage_borders(c, m, a, b, da, db));
  BK_TRY(bk_stage_in(c, rhst, N, 8, true, &d_R));
  BK_TRY(bk_stage_in(c, solu, N, 9, false, &d_u));
  // x1 = A^-1 rhst, x2_j = A^-1 a_j;  S = c - [<b_i, x2_j>],  h = rhsb - [<b_i, x1>],  p = S \ h,  u = x1 - sum p_j x2_j
  OpDesc op = bk_make_op(c, has_shift ? shift : 0.0, 1.0);
  int cv = 1, ci = 0, it = 0;
  int st = bk_gmres_dev(c, op, d_R, d_u, opts, &ci, &it, nullptr);
  if (st < 0) return st;
  cv &= ci;
  if (iters) iters[0] = it;
  double* x2[2] = {nullptr, nullptr};
  for (int j = 0; j < m; ++j) {
    BK_TRY(bk_tmp(c, j, &x2[j]));
    st = bk_gmres_dev(c, op, da[j], x2[j], opts, &ci, &it, nullptr);
    if (st < 0) return st;
    cv &= ci;
    if (iters) iters[1 + j] = it;
  }
  double S[4] = {0, 0, 0, 0}, h[2] = {0, 0};
  for (int i = 0; i < m; ++i) {
    double d = 0;
    BK_TRY(bk_dev_dot(c, db[i], d_u, N, &d));
    h[i] = rhsb[i] - d;
    for (int j = 0; j < m; ++j) {
      BK_TRY(bk_dev_dot(c, db[i], x2[j], N, &d));
      S[i + 2 * j] = cmat[i + m * j] - d;
    }
  }
  double p[2] = {0, 0};
  if (m == 1) {
    p[0] = h[0] / S[0];
  } else {
    const double det = S[0] * S[3] - S[2] * S[1];
    p[0] = (h[0] * S[3] - S[2] * h[1]) / det;
    p[1] = (S[0] * h[1] - S[1] * h[0]) / det;
  }
  for (int j = 0; j < m; ++j) {
    BK_TRY(bk_dev_axpby(c, d_u, -p[j], x2[j], 1.0, N));
    solp[j] = p[j];
  }
  if (converged) *converged = cv;
  BK_TRY(bk_stage_out(c, solu, N, d_u));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  return cv ? BK_OK : BK_NOT_CONVERGED;
}
