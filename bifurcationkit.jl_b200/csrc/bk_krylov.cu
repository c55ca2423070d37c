// bk_krylov.cu -- K3: the GMRES(m) Arnoldi step on device and the GMRES driver (S1/S2).
//
// Replaces IterativeSolvers.gmres as called by (l::GMRESIterativeSolvers)(J, rhs; a0, a1)
// (src/LinearSolver.jl:186-206): left/right preconditioning, tolerance max(reltol*||Pl\r0||, abstol)
// on the preconditioned residual, `iters` = total inner iterations capped by maxiter, x updated at
// restart and at the end.  Orthogonalisation is single-pass classical Gram-Schmidt in two sweeps
// over the basis (the reference's backend uses modified GS => tolerance parity, not bit parity).
// The basis streams through a TMA ring in every sweep (bk_krylov_tma.cuh):
//
//   pass 1  k2_fused<E,B>     : w = a0 v_j + a1 J(u) v_j evaluated as the SH2d stencil from a TMA-staged tile
//                               and, in the same kernel, h_i = <v_i, w> for i <= j (per-CTA partials ->
//                               deterministic last-block sum).  Algorithmic traffic 8N(j+2) bytes: read u,
//                               V_1..V_j, write w.  Only real SH2d with an even nx, at most one border and no
//                               left preconditioner (Solve::fuses_jvp); every other operator runs its stand-alone
//                               apply and then
//           k2_dots<E>        : h_i = <v_i, w> over w already in memory, 8N(j+1).
//   pass 2  k2_update<E>      : v'_{j+1} = w - sum_i h_i v_i, ||v'_{j+1}||^2 reduced the same way.
//                               Algorithmic traffic 8N(j+2): read w, V_1..V_j, write v'_{j+1}.
//   k_lincomb                 : x = beta x + sum_i y_i s_i v'_i at restart and at the end.
//
// Periodic SH2d (BK_SH2D_PERIODIC) with BK_PC_SH_FFT on either side and fused set (Solve::fuses_pc): the preconditioned operator
// of a step is ONE spectral pipeline (bk_periodic_fused: 3 transform kernels, 64N) in place of apply + preconditioner, then
// k2_dots.
//
// The basis is stored UN-normalised (v'_i) with the scalars s_i = 1/||v'_i|| kept on device, so
// normalisation costs no memory pass ("deferred as a scalar") and the host never has to be in the
// loop to launch the next step: Givens rotations run on the host one iteration behind the GPU.
//
// Host: plan_solve checks the arguments and makes every per-solve decision once (a Solve); bk_gmres_dev runs the restart
// loop with the true-residual check; each restart runs one cycle (Arnoldi steps launched ahead, the Givens rotations one
// column behind) and then update_solution (back substitution, then x += M V' y).
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <vector>
#include "bk_common.cuh"
#include "bk_stencil.cuh"
#include "bk_krylov_tma.cuh"

// ---- x = beta x + sum_i coef_i * scales_i * V'_i -----------------------------------------------------------
static __global__ void __launch_bounds__(BK_THREADS) k_lincomb(double* __restrict__ x, double beta, long long n,
                                                               const double* __restrict__ V, long long ld, int k,
                                                               const double* __restrict__ coef,
                                                               const double* __restrict__ scales) {
  const long long base = (long long)blockIdx.x * BK_TILE;
  double val[BK_EPT];
  int off[BK_EPT];
  bool ok[BK_EPT];
#pragma unroll
  for (int e = 0; e < BK_EPT; ++e) {
    long long g = base + threadIdx.x + e * BK_THREADS;
    ok[e] = g < n;
    off[e] = ok[e] ? (int)g : 0;
    val[e] = (ok[e] && beta != 0.0) ? beta * x[g] : 0.0;
  }
  for (int i = 0; i < k; ++i) {
    const double ci = coef[i] * (scales ? scales[i] : 1.0);
    const double* Vi = V + (long long)i * ld;
#pragma unroll
    for (int e = 0; e < BK_EPT; ++e) val[e] = fma(ci, __ldg(Vi + off[e]), val[e]);
  }
#pragma unroll
  for (int e = 0; e < BK_EPT; ++e)
    if (ok[e]) x[off[e]] = val[e];
}


// ------------------------------------------------------------------------------------------------ v2 (TMA ring) planning
#define BK2_BLOCKS_PER_SM 4
struct Plan2 {
  int E, grid, NS, sred_off, keep;
  size_t smem;
};
// per-CTA dynamic shared memory budget that still lets BK2_BLOCKS_PER_SM CTAs share one SM (228 KB, 1 KB reserved per CTA)
static inline size_t bk2_budget() { return (size_t)(233472 / BK2_BLOCKS_PER_SM) - 1024 - 512; }

static Plan2 plan2(bk_ctx* c, long long units_of_256, size_t scratch_bytes_per_E(int), int force_E = 0) {
  Plan2 p;
  const long long slots = (long long)c->nsm * BK2_BLOCKS_PER_SM;
  // Tile height: a taller tile amortises the per-vector cost of a CTA (barrier wait + warp reduction).  Single wave: the
  // tallest tile that still gives every SM about two CTAs.  Several waves: the height in 5..8 that fills the waves most evenly.
  long long E = BK2_EMAX;
  while (E > 1 && (units_of_256 + E - 1) / E < (17 * (long long)c->nsm) / 10) --E;
  if ((units_of_256 + E - 1) / E > slots) {
    double best = -1.0;
    for (long long cand = BK2_EMAX; cand >= 5; --cand) {
      long long g = (units_of_256 + cand - 1) / cand, w = (g + slots - 1) / slots;
      double eff = (double)g / (double)(w * slots);
      if (eff > best + 1e-9) {
        best = eff;
        E = cand;
      }
    }
  }
  if (force_E) E = force_E;
  {
    static const int env_e = [] {  // read once; thread-safe initialisation
      const char* a = getenv("BK2_E");
      return a ? atoi(a) : 0;
    }();
    if (env_e >= 1 && env_e <= BK2_EMAX) E = env_e;  // tuning override
  }
  p.E = (int)E;
  p.grid = (int)((units_of_256 + E - 1) / E);
  const size_t sred = sizeof(double) * 8 * (size_t)(c->m + 2);
  const size_t stage = sizeof(double) * (size_t)E * BK2_ROW;
  size_t budget = bk2_budget();
  long long ns = budget > sred ? (long long)((budget - sred) / stage) : 2;
  if (ns > BK2_MAXSTAGES) ns = BK2_MAXSTAGES;
  if (ns < 2) ns = 2;
  p.NS = (int)ns;
  size_t ring = stage * (size_t)p.NS;
  size_t scratch = scratch_bytes_per_E ? scratch_bytes_per_E(p.E) : 0;
  size_t lo = ring > scratch ? ring : scratch;
  lo = (lo + 127) / 128 * 128;
  p.sred_off = (int)(lo / sizeof(double));
  p.smem = lo + sred;
  // basis vectors at the end of a ring pass that stay in L2 (evict_last) for the next pass, which starts with them: half of
  // the L2; the other half holds w, the pass's output vector and the kernels in between (the preconditioner's transforms)
  p.keep = (int)(c->l2_bytes / 2 / (units_of_256 * BK2_ROW * (long long)sizeof(double)));
  return p;
}
static size_t sh2_scratch_bytes(int E) { return sizeof(double) * (size_t)((BK2_ROW + 4) * (E + 4) + (BK2_ROW + 2) * (E + 2)); }

#define BK2_DISPATCH(E, ...) \
  switch (E) {                \
    case 1: { constexpr int EE = 1; __VA_ARGS__; } break; \
    case 2: { constexpr int EE = 2; __VA_ARGS__; } break; \
    case 3: { constexpr int EE = 3; __VA_ARGS__; } break; \
    case 4: { constexpr int EE = 4; __VA_ARGS__; } break; \
    case 5: { constexpr int EE = 5; __VA_ARGS__; } break; \
    case 6: { constexpr int EE = 6; __VA_ARGS__; } break; \
    case 7: { constexpr int EE = 7; __VA_ARGS__; } break; \
    default: { constexpr int EE = 8; __VA_ARGS__; } break; \
  }

namespace {
// One GMRES solve: its operator and size, the restart length clamped to the workspace and to n, and the decisions that hold for
// the whole solve.  orth is the only field that changes: a failed true-residual check switches a CGS solve to CGS2.
struct Solve {
  OpDesc op;
  long long n;
  int restart, maxiter;
  bool left, right;     // a preconditioner is set up and applied on that side
  bool fuses_jvp, fuses_pc;
  int orth;
  std::vector<double> H, g, cs, sn;  // Hessenberg columns after the Givens rotations, rotated rhs, rotations
};
}  // namespace

static int launch_fused(bk_ctx* c, const OpDesc& op, const double* in, const double* sp, double* w, int j, double* hcol) {
  const int tiles_x = (op.nx + BK2_ROW - 1) / BK2_ROW;
  Plan2 p = plan2(c, (long long)tiles_x * op.ny, sh2_scratch_bytes);
  p.grid = tiles_x * ((op.ny + p.E - 1) / p.E);
  BK_CHECK(c, p.grid <= c->gmax, "partial-sum workspace too small for the fused grid");  // dots_finish indexes partials by CTA
  BK2_DISPATCH(p.E, {
    auto kern = op.bordered ? k2_fused<EE, true> : k2_fused<EE, false>;
    return bk_launch(c, kern, dim3(p.grid), dim3(BK2_THREADS), p.smem, op, in, sp, w, c->V, c->ld, j, c->scales, c->partials,
                     c->counters + 0, hcol, c->gcoef, p.keep, p.NS, p.sred_off);
  });
}

// ------------------------------------------------------------------------------------------------ host
static inline int chunk_grid(long long n) { return (int)((n + BK_TILE - 1) / BK_TILE); }

int bk_launch_dots(bk_ctx* c, const double* basis, const double* scales, const double* w, long long n, int j, double* hcol,
                   double* gcoef) {
  Plan2 p = plan2(c, (n + BK2_ROW - 1) / BK2_ROW, nullptr);
  BK_CHECK(c, p.grid <= c->gmax, "partial-sum workspace too small");
  BK2_DISPATCH(p.E, return bk_launch(c, k2_dots<EE>, dim3(p.grid), dim3(BK2_THREADS), p.smem, w, n, basis, c->ld, j, scales,
                                     c->partials, c->counters + 1, hcol, gcoef, p.keep, p.NS, p.sred_off));
}

int bk_launch_update(bk_ctx* c, const double* basis, const double* gcoef, const double* w, long long n, int j, double* vout,
                     double* h_out, double* scale_out) {
  Plan2 p = plan2(c, (n + BK2_ROW - 1) / BK2_ROW, nullptr);
  BK_CHECK(c, p.grid <= c->gmax, "partial-sum workspace too small");
  BK2_DISPATCH(p.E, return bk_launch(c, k2_update<EE>, dim3(p.grid), dim3(BK2_THREADS), p.smem, w, n, basis, c->ld, j, gcoef, vout,
                                     c->partials, c->counters + 2, h_out, scale_out, p.keep, p.NS));
}

int bk_launch_lincomb(bk_ctx* c, const double* basis, const double* scales, double* x, double beta, long long n, int k,
                      const double* coef_dev) {
  return bk_launch_ordered(c, k_lincomb, chunk_grid(n), BK_THREADS, 0, x, beta, n, basis, c->ld, k, coef_dev, scales);
}

static int plan_solve(bk_ctx* c, const OpDesc& op, const bk_gmres_opts* o, Solve* s) {
  s->op = op;
  const long long n = s->n = op.N + op.bordered;
  BK_CHECK(c, n <= c->ld, "system larger than the context");
  // the TMA rows of k2_dots / k2_update are read in pairs: an odd length needs one zero pad element behind it
  BK_CHECK(c, (n % 2 == 0) || n + 1 <= c->ld, "no pad element left for an odd-sized bordered system");
  int& restart = s->restart = o->restart;
  if (restart > c->m) restart = c->m;
  if ((long long)restart > n) restart = (int)n;
  BK_CHECK(c, restart >= 1, "restart must be >= 1");
  BK_CHECK(c, o->pc_side == BK_SIDE_NONE || c->pc.kind != BK_PC_NONE, "pc_side set but no preconditioner was set up");
  s->maxiter = o->maxiter;
  s->left = o->pc_side == BK_SIDE_LEFT && c->pc.kind != BK_PC_NONE;
  s->right = o->pc_side == BK_SIDE_RIGHT && c->pc.kind != BK_PC_NONE;
  // Whether the Arnoldi steps run k2_fused (JVP + dots in one kernel) or the stand-alone apply + k2_dots.  k2_fused tiles one
  // real SH2d grid in TMA rows of an even length and carries at most one border; the operator output must feed the dots
  // directly, so no left preconditioner.  3-D always runs unfused: a ring kernel would gain < 5 % (DESIGN.md §4.4).
  s->fuses_jvp = o->fused && op.kind == BK_SH2D && op.nx % 2 == 0 && !op.cplx && op.bordered <= 1 && !s->left;
  // Whether the Arnoldi steps apply the preconditioned operator of BK_SH2D_PERIODIC in ONE spectral pipeline (bk_periodic_fused:
  // P (a0 I + a1 J) = P d - a1 I, (a0 I + a1 J) P = d P - a1 I) instead of precond + apply or apply + precond.
  s->fuses_pc = o->fused && op.kind == BK_SH2D_PERIODIC && c->pc.kind == BK_PC_SH_FFT && (s->left || s->right) &&
                op.bordered == 0 && !op.cplx;
  s->orth = o->orth;
  s->H.resize((size_t)(restart + 1) * restart);
  s->g.resize(restart + 1);
  s->cs = s->sn = std::vector<double>(restart);
  return BK_OK;
}

// One Arnoldi step k (0-based): basis v'_0..v'_k -> v'_{k+1}, H column k on device (+ async copy to pinned host).
static int arnoldi_step(bk_ctx* c, const Solve& s, int k) {
  const int j = k + 1;
  const int mh = c->m + 4;
  // The H column is written by the kernels' last CTA straight into pinned, device-mapped host memory (UVA): no
  // D2H memcpy on the copy engine sits between two Arnoldi steps of the same stream any more.
  double* hcol = c->h_pinned + (size_t)k * mh;
  double* hcol2 = c->h_pinned + (size_t)(c->m + 1) * mh + (size_t)k * mh;
  const double* in = c->V + (size_t)k * c->ld;
  const double* sp = c->scales + k;
  if (s.right && !s.fuses_pc) {
    BK_TRY(bk_precond_apply_dev(c, in, c->z, s.n));
    in = c->z;
  }
  const bool timed = c->timing_now;
  const double* wfin = c->w;
  if (s.fuses_pc) {
    BK_TRY(bk_periodic_fused(c, s.op, in, sp, c->w, s.left));
  } else if (!s.fuses_jvp) {
    BK_TRY(bk_launch_apply(c, s.op, in, sp, c->w));
    if (s.left) {
      BK_TRY(bk_precond_apply_dev(c, c->w, c->r, s.n));
      wfin = c->r;
    }
  }
  if (timed) c->fused_timer.begin(c->stream);
  BK_TRY(s.fuses_jvp ? launch_fused(c, s.op, in, sp, c->w, j, hcol)
                     : bk_launch_dots(c, c->V, c->scales, wfin, s.n, j, hcol, c->gcoef));
  if (timed) c->fused_timer.end(c->stream);
  double* vnext = c->V + (size_t)(k + 1) * c->ld;
  if (timed) c->fused_timer.begin(c->stream);
  BK_TRY(bk_launch_update(c, c->V, c->gcoef, wfin, s.n, j, vnext, hcol + j, c->scales + k + 1));
  if (timed) c->fused_timer.end(c->stream);
  if (s.orth == BK_ORTH_CGS2) {
    BK_TRY(bk_launch_dots(c, c->V, c->scales, vnext, s.n, j, hcol2, c->gcoef));
    BK_TRY(bk_launch_update(c, c->V, c->gcoef, vnext, s.n, j, vnext, hcol + j, c->scales + k + 1));
  }
  BK_CUDA(c, cudaEventRecord(c->events[k], c->stream));
  // algorithmic bytes of the step (SURVEY 8d): B(j) = 8N(2j+4); the bordered map reads a and b as well (+16N, "40N" K2')
  const long long step_bytes = 8LL * s.n * (2LL * j + 4) + (s.op.bordered ? 16LL * s.n : 0LL);
  c->stats.last_fused_bytes += step_bytes;
  c->stats.last_fused_launches += 2;
  if (s.fuses_jvp && (c->timing_now || !c->timing)) {  // with sampled timing the totals cover the timed solves only (bytes and ms must match)
    c->stats.total_fused_bytes += step_bytes;
    c->stats.total_fused_launches += 2;
  }
  return BK_OK;
}

// initial (preconditioned) residual -> v'_0, returns beta on the host
static int init_residual(bk_ctx* c, const Solve& s, const double* rhs, const double* x, bool x_zero, double* beta) {
  const double* r = rhs;
  if (!x_zero) {
    BK_TRY(bk_launch_apply(c, s.op, x, nullptr, c->w));
    BK_TRY(bk_dev_axpby(c, c->w, 1.0, rhs, -1.0, s.n));  // w = rhs - A x
    r = c->w;
  }
  if (s.left) {
    BK_TRY(bk_precond_apply_dev(c, r, c->r, s.n));
    r = c->r;
  }
  BK_TRY(bk_launch_update(c, c->V, c->gcoef, r, s.n, 0, c->V, c->red_out, c->scales));
  BK_CUDA(c, cudaMemcpyAsync(c->red_pinned, c->red_out, 8, cudaMemcpyDeviceToHost, c->stream));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  *beta = c->red_pinned[0];
  return BK_OK;
}

// One restart cycle from v'_0 with norm beta: the device runs at most two Arnoldi steps ahead of the host, which applies the
// Givens rotations of each column once its event has fired.  *k is the number of columns kept, *res the residual estimate after
// the last of them (unchanged when k = 0); *total counts the columns of every cycle.  Speculative steps may still be in flight
// on return: they only touch gcoef, not coef_pinned.
static int cycle(bk_ctx* c, Solve& s, double beta, double tol, int* total, int* k, double* res) {
  const int mh = c->m + 4;
  std::fill(s.g.begin(), s.g.end(), 0.0);
  s.g[0] = beta;
  int kl = 0, kd = 0;
  while (true) {
    if (kl < s.restart && *total + (kl - kd) < s.maxiter && kl - kd < 2) {
      BK_TRY(arnoldi_step(c, s, kl++));
      continue;
    }
    if (kd == kl) break;
    BK_CUDA(c, cudaEventSynchronize(c->events[kd]));
    // ---- Givens update of column kd on the host (one step behind the device) ----
    const double* hc = c->h_pinned + (size_t)kd * mh;
    const double* hc2 = c->h_pinned + (size_t)(c->m + 1) * mh + (size_t)kd * mh;
    double* Hk = s.H.data() + (size_t)kd * (s.restart + 1);
    for (int i = 0; i <= kd; ++i) Hk[i] = hc[i] + (s.orth == BK_ORTH_CGS2 ? hc2[i] : 0.0);
    const double hk1 = hc[kd + 1];
    for (int i = 0; i < kd; ++i) {
      double t = s.cs[i] * Hk[i] + s.sn[i] * Hk[i + 1];
      Hk[i + 1] = -s.sn[i] * Hk[i] + s.cs[i] * Hk[i + 1];
      Hk[i] = t;
    }
    double d = hypot(Hk[kd], hk1);
    if (!(d > 0.0) || !std::isfinite(d)) break;  // unusable column (exact breakdown): stop with the columns gathered so far
    s.cs[kd] = Hk[kd] / d;
    s.sn[kd] = hk1 / d;
    Hk[kd] = d;
    s.g[kd + 1] = -s.sn[kd] * s.g[kd];
    s.g[kd] = s.cs[kd] * s.g[kd];
    *res = fabs(s.g[kd + 1]);
    ++kd;
    ++*total;
    if (*res <= tol || *total >= s.maxiter || hk1 == 0.0) break;
  }
  *k = kd;
  return BK_OK;
}

// x += M V' diag(s) y with R y = g over the first k columns, M the right preconditioner or I (x_zero: x is still all zeros)
static int update_solution(bk_ctx* c, const Solve& s, int k, double* x, bool x_zero) {
  double* y = c->coef_pinned;  // in-flight speculative steps only touch gcoef, never coef_pinned
  for (int i = k - 1; i >= 0; --i) {  // back substitution R y = g
    double t = s.g[i];
    for (int q = i + 1; q < k; ++q) t -= s.H[(size_t)q * (s.restart + 1) + i] * y[q];
    y[i] = t / s.H[(size_t)i * (s.restart + 1) + i];
  }
  double* coef_dev = c->hcols2 + (size_t)c->m * (c->m + 4);  // last row of hcols2 is free scratch
  BK_CUDA(c, cudaMemcpyAsync(coef_dev, c->coef_pinned, 8 * (size_t)k, cudaMemcpyHostToDevice, c->stream));
  if (s.right) {
    BK_TRY(bk_launch_lincomb(c, c->V, c->scales, c->w, 0.0, s.n, k, coef_dev));
    BK_TRY(bk_precond_apply_dev(c, c->w, c->z, s.n));
    BK_TRY(bk_dev_axpby(c, x, 1.0, c->z, x_zero ? 0.0 : 1.0, s.n));
  } else {
    BK_TRY(bk_launch_lincomb(c, c->V, c->scales, x, x_zero ? 0.0 : 1.0, s.n, k, coef_dev));
  }
  BK_CUDA(c, cudaStreamSynchronize(c->stream));  // coef_pinned is reused by the next cycle
  return BK_OK;
}

int bk_gmres_dev(bk_ctx* c, const OpDesc& op, const double* rhs, double* x, const bk_gmres_opts* o, int* converged,
                 int* iters, double* resnorm) {
  Solve s;
  BK_TRY(plan_solve(c, op, o, &s));
  c->stats.last_fused_bytes = 0;
  c->stats.last_fused_launches = 0;
  c->stats.last_fused_ms = 0.0;
  c->solve_count++;
  c->timing_now = c->timing && (c->solve_count % c->timing_every == 0);
  c->fused_timer.used = 0;  // drop what a failed solve left behind

  BK_CUDA(c, cudaMemsetAsync(x, 0, 8 * (size_t)s.n, c->stream));  // initially_zero = true (src/LinearSolver.jl:171)
  bool x_zero = true, conv = false;
  int total = 0;
  double beta = 0, res = 0.0;
  BK_TRY(init_residual(c, s, rhs, x, x_zero, &beta));
  const double tol = fmax(o->reltol * beta, o->abstol);
  // Single-pass classical Gram-Schmidt (north_star) can lose orthogonality on long cycles / tight tolerances, and the
  // Givens estimate |g[k+1]| then under-reports the residual (the reference's backend uses modified GS).  A cycle that ends
  // "converged" after >= 40 Krylov vectors or with reltol < 1e-9 is therefore verified against the TRUE residual
  // (the next cycle's initial residual); on failure the solve continues with CGS2 cycles from the current iterate.
  while (true) {
    res = beta;
    if (!(res > tol) || total >= s.maxiter || !(beta > 0.0)) {
      conv = res <= tol;
      break;
    }
    int k = 0;
    BK_TRY(cycle(c, s, beta, tol, &total, &k, &res));
    if (k > 0) {
      BK_TRY(update_solution(c, s, k, x, x_zero));
      x_zero = false;
    }
    conv = res <= tol;
    const bool verify = conv && s.orth == BK_ORTH_CGS && (k >= 40 || o->reltol < 1e-9) && total < s.maxiter;
    if (!verify && (conv || total >= s.maxiter || k == 0)) break;
    BK_TRY(init_residual(c, s, rhs, x, x_zero, &beta));
    if (verify) {
      if (beta <= 4.0 * tol) {  // rounding slack between the Givens recurrence and the recomputed residual
        res = beta;
        break;
      }
      s.orth = BK_ORTH_CGS2;
      c->stats.cgs_fallbacks++;
    }
  }
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  c->stats.total_precond_applies += c->pc_timer.harvest(c->stats.total_precond_ms);
  if (c->timing_now) {
    double ms = 0;
    c->fused_timer.harvest(ms);
    c->stats.last_fused_ms = ms;
    if (s.fuses_jvp) c->stats.total_fused_ms += ms;
  }
  if (converged) *converged = conv ? 1 : 0;
  if (iters) *iters = total;
  if (resnorm) *resnorm = res;
  return conv ? BK_OK : BK_NOT_CONVERGED;
}

// ------------------------------------------------------------------------------------------------ C ABI
static bk_gmres_opts default_opts() {
  bk_gmres_opts o;
  o.reltol = 1e-8;
  o.abstol = 0.0;
  o.restart = 200;
  o.maxiter = 100;
  o.pc_side = BK_SIDE_NONE;
  o.orth = BK_ORTH_CGS;
  o.fused = 1;
  o.reserved = 0;
  return o;
}

extern "C" int32_t bk_gmres(bk_ctx* c, const double* rhs, double* x, double a0, double a1, const bk_gmres_opts* opts,
                            int32_t* converged, int32_t* iters, double* resnorm) {
  BK_ENTER(c);
  BkRange nvtx_range("bk_gmres");
  BK_CHECK(c, c->have_state, "bk_jac_set_state must be called before bk_gmres");
  bk_gmres_opts o = opts ? *opts : default_opts();
  double *drhs, *dx;
  BK_TRY(bk_stage_in(c, rhs, c->N, 4, true, &drhs));
  BK_TRY(bk_stage_in(c, x, c->N, 5, false, &dx));
  BK_CHECK(c, drhs != dx, "bk_gmres: rhs and x must not alias");
  OpDesc op = bk_make_op(c, a0, a1);
  int cv = 0, it = 0;
  double rn = 0;
  int st = bk_gmres_dev(c, op, drhs, dx, &o, &cv, &it, &rn);
  if (st < 0) return st;
  if (converged) *converged = cv;
  if (iters) *iters = it;
  if (resnorm) *resnorm = rn;
  BK_TRY(bk_stage_out(c, x, c->N, dx));
  return st;
}

extern "C" int32_t bk_gmres2(bk_ctx* c, const double* rhs1, const double* rhs2, double* x1, double* x2, double a0, double a1,
                             const bk_gmres_opts* opts, int32_t* converged, int32_t iters[2]) {
  // src/LinearSolver.jl:15-19: two sequential solves with the same operator, flag1 & flag2, (it1, it2)
  int32_t c1 = 0, c2 = 0, i1 = 0, i2 = 0;
  int s1 = bk_gmres(c, rhs1, x1, a0, a1, opts, &c1, &i1, nullptr);
  if (s1 < 0) return s1;
  int s2 = bk_gmres(c, rhs2, x2, a0, a1, opts, &c2, &i2, nullptr);
  if (s2 < 0) return s2;
  if (converged) *converged = c1 & c2;
  if (iters) {
    iters[0] = i1;
    iters[1] = i2;
  }
  return (c1 & c2) ? BK_OK : BK_NOT_CONVERGED;
}
