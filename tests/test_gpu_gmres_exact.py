"""bk_gmres against exact GMRES(m): the long-double reference of tests/gmres_exact_oracle.py, iterate by iterate, with exact
iteration counts, every stopping rule and every restart path of the device driver.

Bounds.  eps = 2^-52.  beta0 is the norm of the initial residual on the side that carries the tolerance (Pl rhs with a left
preconditioner, rhs otherwise); after k columns rho_k is the exact minimal residual, x_k the exact iterate, Hbar_k the
(j+1) x j Hessenberg of the cycle in progress and y_k its least-squares solution (x_k = x_cycle + Pr V y_k).

* Residuals.  GMRES with a well-conditioned basis is backward stable: the computed iterate is the exact one of a system
  perturbed by O(k eps ||A||) per column.  So both the returned Givens estimate `resnorm` and the true residual of the
  returned x satisfy
      |r_k - rho_k| <= C_RES k eps beta0 mu_k,   mu_k = max(1, ||Hbar_k|| ||y_k|| / beta0),
  ||Hbar_k|| ||y_k|| standing for ||A|| ||x_k||.  C_RES = 16: one rounding for each of the ~13 stencil products that enter
  a column, one for the dot and one for the update, and the square root of the norm.
  With a preconditioner the operator and the preconditioner round one after the other, each at its own scale, so the
  backward error is relative to ||P|| ||A|| (the unpreconditioned operator) rather than to ||P A|| ~ ||Hbar_k||: mu_k and
  the iterate bound below carry alpha_k = max(1, ||P|| ||A|| / ||Hbar_k||).  ||P|| is the largest entry of the
  preconditioner's symbol; ||A|| <= |a0| + |a1| (max L1 + max |l + 2 nu u - 3 u^2|).  This is the floor of a composed
  step: for the 64 x 64 periodic SH, alpha ~ 1e5 and the unfused left and right solves do sit above the unscaled bound.
* Iterates.  The least-squares perturbation bound (Wedin) turns that backward error into
      ||x - x_k|| / ||x_k|| <= C_X k eps kappa_k (1 + kappa_k rho_k / (||Hbar_k|| ||y_k||)) pi_k,
  kappa_k = cond(Hbar_k) (the running maximum over the cycles of the run) and pi_k = max(1, ||Pr|| ||V y_k|| / ||x_k||) the
  amplification of a right preconditioner (1 without one).  C_X = 32: C_RES and a factor 2 for the rounding of Pr and
  of the lincomb that forms x.
* Direct solves.  Full-space GMRES (restart >= n) ends at the solution of the n x n system to C_X n eps kappa(A).

Worst observed ratios to these bounds over every comparison in this file, on an H100 80GB HBM3 at its 700 W power
limit: resnorm 0.058, true residual 0.0062, iterate 0.038 (the module fixture prints them at teardown).

Iteration counts are compared exactly.  `_gap_tol` places the tolerance at the geometric mean of two consecutive rho_k
whose ratio is >= 1.5: the device's residual would have to be off by a factor 1.22 to stop one column early or late,
which is ~1e10 times the residual bound above.
"""
import numpy as np
import pytest

import __graft_entry__ as g
from oracle import problems
from tests import gmres_exact_oracle as X

pytestmark = pytest.mark.gpu

EPS = X.EPS
C_RES, C_X = 16.0, 32.0
LX, LY = 8 * np.pi, 4 * np.pi / np.sqrt(3)
WORST = {"resnorm": 0.0, "true": 0.0, "x": 0.0}


@pytest.fixture(scope="module")
def bk():
    yield g.load_package()
    print("\nworst ratio to the bounds:", {k: round(float(v), 4) for k, v in WORST.items()})


def _sh_lmax(dims, lengths):
    """largest eigenvalue of L1 = (I + Lap)^2 with the Neumann closure: (1 - 4/hx^2 - 4/hy^2 (- 4/hz^2))^2 bounds it"""
    s = 1.0
    for n, L in zip(dims, lengths):
        s -= 4.0 / (2 * L / n) ** 2
    return s * s


def _shift(lmax, a1):
    """a0 for a0 I + a1 J with a spectrum in [0.3, 1.3] lmax (up to the O(1) diagonal of J): condition number ~5"""
    return 0.3 * lmax + 3.0 if a1 < 0 else 1.3 * lmax + 3.0


class Case:
    """one linear system on a context: the device handle J (a Jacobian or a bordered solver), its long-double map A,
    the preconditioner (device kind + long-double inverse) and the rhs"""

    def __init__(self, ctx, J, A, rhs, a0, a1, pc=None, anorm=None):
        self.ctx, self.J, self.A, self.rhs, self.a0, self.a1, self.pc, self.anorm = ctx, J, A, rhs, a0, a1, pc, anorm


def _solve(bk, case, side="none", **kw):
    ls = bk.GMRESB200(Pl=side == "left", Pr=side == "right", **kw)
    x, ok, it = ls(case.J, case.rhs, a0=case.a0, a1=case.a1)
    x = np.asarray(x)
    _check_cgs_claim(case, side, ls, x, ok, it)
    return x, ok, it, ls.last_resnorm


def _check_cgs_claim(case, side, ls, x, ok, it):
    """every single-pass CGS solve of this file that reports converged where the true-residual check applies (its last
    cycle has >= 40 columns or reltol < 1e-9, and iters < maxiter) has a true residual <= 4 tol"""
    if ls.orth != "cgs" or not ok or it == 0 or it >= ls.maxiter:
        return
    m = min(ls.restart, case.ctx.krylov_m, case.ctx.N)
    last = it - m * ((it - 1) // m)
    if not (ls.reltol < 1e-9 or last >= 40):
        return
    b = X.ld(case.rhs)
    tol = max(ls.reltol * float(X.nrm(case.pc(b) if side == "left" else b)), ls.abstol)
    assert _true_res(case, side, x) <= 4 * tol, ("converged above 4 tol", it, _true_res(case, side, x) / tol)


def _ref(case, side, restart, maxiter, reltol=0.0, abstol=0.0, keep_x=True, orth="cgs"):
    P = case.pc
    kw = dict(Pl=P) if side == "left" else (dict(Pr=P) if side == "right" else {})
    return X.gmres(case.A, case.rhs, reltol=reltol, abstol=abstol, restart=restart, krylov_m=case.ctx.krylov_m, maxiter=maxiter,
                   keep_x=keep_x, orth=orth, **kw)


def _true_res(case, side, x):
    r = X.ld(case.rhs) - case.A(X.ld(x))
    return float(X.nrm(case.pc(r) if side == "left" else r))


def _bounds(R, side, case, k, kappa):
    b0 = float(R.beta0)
    # preconditioned: A and P round separately, at the scale of ||P|| ||A|| rather than ||P A|| ~ ||Hbar||
    alpha = max(1.0, case.pc.norm * case.anorm / R.hnorm[k]) if side != "none" else 1.0
    mu = max(1.0, alpha * R.hnorm[k] * R.ynorm[k] / b0)
    res_b = C_RES * k * EPS * b0 * mu
    xk = R.xs[k]
    xn = float(X.nrm(xk))
    pi = max(1.0, case.pc.norm * float(X.nrm(R.z[k])) / xn) if side == "right" else 1.0
    x_b = C_X * k * EPS * kappa * (1.0 + kappa * float(R.rho[k]) / max(R.hnorm[k] * R.ynorm[k], 1e-300)) * pi * alpha
    return res_b, x_b, xn


def _check_iterate(R, side, case, k, kappa, x, rn=None):
    res_b, x_b, xn = _bounds(R, side, case, k, kappa)
    rho = float(R.rho[k])
    tr = _true_res(case, side, x)
    assert abs(tr - rho) <= res_b, ("true residual", k, tr, rho, res_b)
    WORST["true"] = max(WORST["true"], abs(tr - rho) / res_b)
    if rn is not None:
        assert abs(rn - rho) <= res_b, ("resnorm", k, rn, rho, res_b)
        WORST["resnorm"] = max(WORST["resnorm"], abs(rn - rho) / res_b)
    err = float(X.nrm(X.ld(x) - R.xs[k])) / xn
    assert err <= x_b, ("iterate", k, err, x_b)
    WORST["x"] = max(WORST["x"], err / x_b)


def _history(bk, case, K, side="none", orth="cgs", fused=True, restart=None, every=1):
    """device runs with maxiter = k for k = 1..K (every `every`-th, and K) against the reference's column k"""
    restart = restart or case.ctx.krylov_m
    big = case.ctx.N > 2_000_000
    R = _ref(case, side, restart, K, keep_x=not big)
    assert R.iters == K
    kappa = 1.0
    for k in range(1, K + 1):
        kappa = max(kappa, R.cond[k])
        if k % every and k != K:
            continue
        x, ok, it, rn = _solve(bk, case, side, reltol=0.0, abstol=0.0, restart=restart, maxiter=k, orth=orth, fused=fused)
        assert it == k and not ok
        if big and k != K:
            res_b, _, _ = _bounds_res_only(R, k)
            assert abs(rn - float(R.rho[k])) <= res_b, ("resnorm", k, rn, float(R.rho[k]), res_b)
            continue
        _check_iterate(R, side, case, k, kappa, x, rn)


def _bounds_res_only(R, k):
    b0 = float(R.beta0)
    return C_RES * k * EPS * b0 * max(1.0, R.hnorm[k] * R.ynorm[k] / b0), None, None


# ------------------------------------------------------------------------------------------------------------- problems
def _sh2d_case(bk, dims, a1, side="none", krylov_m=30, noise=0.1, seed=7, a0=None):
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    u = problems.sh2d_sol0(*dims, LX, LY) + noise * np.random.default_rng(1).standard_normal(sh.N)
    rhs = np.random.default_rng(seed).standard_normal(sh.N)
    a0 = _shift(_sh_lmax(dims, (LX, LY)), a1) if a0 is None else a0
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=krylov_m, params=(-0.1, 1.3))
    pc = None
    if side != "none":
        ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
        pc = X.dct_precond(dims, (LX, LY), 1.0)
    d = -0.1 + 2.6 * u - 3.0 * u**2
    anorm = abs(a0) + abs(a1) * (_sh_lmax(dims, (LX, LY)) + np.abs(d).max())
    return Case(ctx, ctx.jacobian(u), X.sh_op(sh, u, a0, a1), rhs, a0, a1, pc, anorm)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("orth", ["cgs", "cgs2"])
@pytest.mark.parametrize("a1", [1.0, -1.0])
@pytest.mark.parametrize("side", ["none", "left", "right"])
def test_history_sh2d_even_width(bk, side, a1, orth, fused):
    """k2_fused (nx even, no left preconditioner, fused) or the stand-alone apply + k2_dots, column by column"""
    _history(bk, _sh2d_case(bk, (16, 12), a1, side), 20, side, orth, fused)


@pytest.mark.parametrize("dims", [(258, 5), (64, 37), (15, 7), (95, 64)])
@pytest.mark.parametrize("side", ["none", "right"])
def test_history_sh2d_tile_edges(bk, dims, side):
    """rows of two TMA rows with a narrow last one (258), ny not a multiple of the tile height (37), odd nx (stand-alone
    apply + k2_dots)"""
    _history(bk, _sh2d_case(bk, dims, -1.0, side), 16, side)


@pytest.mark.parametrize("fused", [True, False])
def test_history_sh2d_bordered(bk, fused):
    """MatrixFreeBLS on N + 1 = 193 (odd: the pad element is read): k2_fused<E, true> when fused"""
    dims = (16, 12)
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    u = problems.sh2d_sol0(*dims, LX, LY)
    rng = np.random.default_rng(12)
    N = sh.N
    a, b, R, n = rng.standard_normal(N), rng.standard_normal(N), rng.standard_normal(N), 0.7
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=30, params=(-0.1, 1.3))
    J = ctx.jacobian(u)
    # the device solves [shift I + J, a; b'/N, 0.9]
    shift = _shift(_sh_lmax(dims, (LX, LY)), 1.0)
    A = X.bordered_op(X.sh_op(sh, u, shift, 1.0), [a], [b], [[0.9]], dotscale=1.0 / N)
    rhs = np.concatenate([R, [n]])
    Rf = X.gmres(A, rhs, reltol=0.0, restart=30, maxiter=16)
    case = Case(ctx, J, A, rhs, shift, 1.0)
    kappa = 1.0
    for k in range(1, 17):
        kappa = max(kappa, Rf.cond[k])
        ls = bk.GMRESB200(reltol=0.0, restart=30, maxiter=k, fused=fused)
        dX, dl, ok, it = bk.MatrixFreeBLSB200(ls)(J, a, b, 0.9, R, n, shift=shift, dotscale=1.0 / N)
        assert it == k and not ok
        _check_iterate(Rf, "none", case, k, kappa, np.concatenate([dX, [dl]]))


def test_history_sh3d_chan_cgl(bk):
    dims, L = (12, 10, 8), (4 * np.pi, 4 * np.pi, 3 * np.pi)
    sh = problems.SwiftHohenberg(dims, L, l=0.1, nu=1.2)
    u = problems.sh3d_sol0(*dims, *L)
    ctx = bk.Context(bk.BK_SH3D, dims, L, krylov_m=30, params=(0.1, 1.2))
    a0 = _shift(_sh_lmax(dims, L), -1.0)
    rhs = np.random.default_rng(9).standard_normal(sh.N)
    _history(bk, Case(ctx, ctx.jacobian(u), X.sh_op(sh, u, a0, -1.0), rhs, a0, -1.0), 16)

    n = 1000
    x = problems.chan_sol0(n) + 0.01 * np.random.default_rng(3).standard_normal(n)
    ctxc = bk.Context(bk.BK_CHAN, (n,), (1.0,), krylov_m=30, params=(3.3, 0.01))
    a0 = 1.3 * 4 * (n - 1) ** 2
    rhs = np.random.default_rng(10).standard_normal(n)
    _history(bk, Case(ctxc, ctxc.jacobian(x), X.chan_op(x, 3.3, 0.01, a0, 1.0), rhs, a0, 1.0), 16)

    gl = problems.GinzburgLandau2D(24, 12, np.pi, np.pi / 2, r=1.2)
    ug = 0.3 * np.random.default_rng(10).standard_normal(gl.N)
    ctxg = bk.Context(bk.BK_CGL2D, (24, 12), (np.pi, np.pi / 2), krylov_m=30, params=(1.2, 0.1, 1.0, -1.0, 1.0))
    a0 = 0.3 * 8 * max(24 / (2 * np.pi), 12 / np.pi) ** 2 + 10.0
    rg = np.random.default_rng(11).standard_normal(gl.N)
    _history(bk, Case(ctxg, ctxg.jacobian(ug), X.cgl_op(gl, ug, a0, -1.0), rg, a0, -1.0), 16)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("side,a1", [("none", -1.0), ("left", -1.0), ("right", -1.0), ("left", 1.0), ("right", 1.0)])
def test_history_sh2d_periodic(bk, side, a1, fused):
    """BK_SH2D_PERIODIC with BK_PC_SH_FFT: fused, the preconditioned operator of a step is one spectral pipeline on either
    side (fuses_pc); unfused, precond + apply or apply + precond"""
    from tests import sh_periodic_oracle as po
    dims = (64, 64)
    L = po.example_lengths(*dims)
    psh = po.PeriodicSH(dims, L, -0.15, 1.3)
    u = po.sol0(*dims, *L) + 0.05 * np.random.default_rng(0).standard_normal(psh.N)
    rhs = np.random.default_rng(7).standard_normal(psh.N)
    # unpreconditioned: a spectrum in [0.3, 1.3] max(L1); preconditioned: (a0 + a1 J) / (L1 + 1) in about [1, 3] up to sign
    a0 = _shift(float(psh.symbol.max()), a1) if side == "none" else -3.0 * a1
    ctx = bk.Context(bk.BK_SH2D_PERIODIC, dims, L, krylov_m=30, params=(-0.15, 1.3))
    pc = None
    if side != "none":
        ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
        pc = X.fft_precond(psh, 1.0)
    anorm = abs(a0) + abs(a1) * (float(psh.symbol.max()) + np.abs(-0.15 + 2.6 * u - 3.0 * u**2).max())
    _history(bk, Case(ctx, ctx.jacobian(u), X.periodic_sh_op(psh, u, a0, a1), rhs, a0, a1, pc, anorm), 16, side, fused=fused)


@pytest.mark.parametrize("a0", [5.0, 50.0])
def test_history_trapeze(bk, a0):
    """the Trapeze periodic-orbit functional over cGL (BK_POTRAP_CGL2D), N = 2 Nx Ny M + 1 = 1441"""
    Nx, Ny, M = 12, 6, 10
    gl = problems.GinzburgLandau2D(Nx, Ny, np.pi, np.pi / 2, r=1.3)
    rng = np.random.default_rng(5)
    NM = gl.N * M
    x = np.concatenate([0.3 * rng.standard_normal(NM), [6.1]])
    phi, xpi = rng.standard_normal(NM), rng.standard_normal(NM)
    rhs = rng.standard_normal(NM + 1)
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (Nx, Ny, M), (np.pi, np.pi / 2), krylov_m=30, params=(1.3, 0.1, 1.0, -1.0, 1.0))
    ctx.potrap_set_section(phi, xpi)
    _history(bk, Case(ctx, ctx.jacobian(x), X.trapeze_op(gl, x, phi, M, a0, 1.0), rhs, a0, 1.0), 16)


def _opnorm(A, n):
    """||A||_2 of a long-double map through its dense fp64 matrix (small n)"""
    return float(np.linalg.norm(X.dense(A, n).astype(np.float64), 2))


@pytest.mark.parametrize("side", ["left", "right"])
@pytest.mark.parametrize("problem", ["cgl_dst", "chan_tridiag", "trapeze_circulant"])
def test_history_other_preconditioners(bk, problem, side):
    """BK_PC_CGL_DST, BK_PC_CHAN_TRIDIAG and BK_PC_POTRAP_CIRC (inverse of its defining operator) on either side"""
    if problem == "cgl_dst":
        dims = (24, 12)
        gl = problems.GinzburgLandau2D(*dims, np.pi, np.pi / 2, r=1.2)
        u = 0.3 * np.random.default_rng(10).standard_normal(gl.N)
        ctx = bk.Context(bk.BK_CGL2D, dims, (np.pi, np.pi / 2), krylov_m=30, params=(1.2, 0.1, 1.0, -1.0, 1.0))
        ctx.precond_setup(bk.BK_PC_CGL_DST, 1.0, -1.0)
        A, pc, a0, a1, K = X.cgl_op(gl, u, 1.0, -1.0), X.dst_precond(gl, 1.0, -1.0), 1.0, -1.0, 16
        rhs = np.random.default_rng(11).standard_normal(gl.N)
    elif problem == "chan_tridiag":
        n = 1000
        u = problems.chan_sol0(n) + 0.01 * np.random.default_rng(3).standard_normal(n)
        ctx = bk.Context(bk.BK_CHAN, (n,), (1.0,), krylov_m=30, params=(3.3, 0.01))
        ctx.precond_setup(bk.BK_PC_CHAN_TRIDIAG)
        A, pc, a0, a1, K = X.chan_op(u, 3.3, 0.01), X.chan_precond(n), 0.0, 1.0, 6  # at the rounding floor after ~7 columns
        rhs = np.random.default_rng(10).standard_normal(n)
    else:
        Nx, Ny, M = 12, 6, 10
        gl = problems.GinzburgLandau2D(Nx, Ny, np.pi, np.pi / 2, r=1.3)
        rng = np.random.default_rng(5)
        NM = gl.N * M
        u = np.concatenate([0.3 * rng.standard_normal(NM), [6.1]])
        phi, xpi = rng.standard_normal(NM), rng.standard_normal(NM)
        rhs = rng.standard_normal(NM + 1)
        ctx = bk.Context(bk.BK_POTRAP_CGL2D, (Nx, Ny, M), (np.pi, np.pi / 2), krylov_m=30, params=(1.3, 0.1, 1.0, -1.0, 1.0))
        ctx.potrap_set_section(phi, xpi)
        ctx.precond_setup(bk.BK_PC_POTRAP_CIRC, 6.1)
        A, pc, a0, a1, K = X.trapeze_op(gl, u, phi, M), X.potrap_circ_precond(gl, M, 6.1), 0.0, 1.0, 16
    _history(bk, Case(ctx, ctx.jacobian(u), A, rhs, a0, a1, pc, _opnorm(A, ctx.N)), K, side)


def test_history_past_the_l2_resident_vectors(bk):
    """j beyond plan2's `keep` vectors, so that every ring pass also reads its evict_first part: chan at N = 4.85 M
    (keep = 0: one basis vector is 39 MB, more than half the L2) and SH2d 1024^2, unpreconditioned (keep = 3)"""
    n = 4_850_000
    x = problems.chan_sol0(n)
    ctx = bk.Context(bk.BK_CHAN, (n,), (1.0,), krylov_m=4, params=(3.3, 0.01))
    a0 = 1.3 * 4 * float(n - 1) ** 2
    rhs = np.random.default_rng(13).standard_normal(n)
    _history(bk, Case(ctx, ctx.jacobian(x), X.chan_op(x, 3.3, 0.01, a0, 1.0), rhs, a0, 1.0), 4)
    del ctx
    dims = (1024, 1024)
    case = _sh2d_case(bk, dims, -1.0, krylov_m=10, noise=0.0)
    # shifted to a condition number ~5: ten columns stay far above the rounding floor
    _history(bk, case, 10, every=3)


# ---------------------------------------------------------------------------------------------------- exact iteration counts
def _gap_tol(R, start=1, ratio=1.5):
    k, t = X.first_gap(R.rho, ratio=ratio, start=start)
    return k + 1, t


def _exact_count(bk, case, side="none", restart=None, maxiter=40, start=1, orth="cgs", fused=True):
    """the tolerance between two columns of the reference; device iters / converged / x against the reference's"""
    restart = restart or case.ctx.krylov_m
    H = _ref(case, side, restart, maxiter)
    stop, t = _gap_tol(H, start)
    reltol = t / float(H.beta0)
    R = _ref(case, side, restart, maxiter, reltol=reltol, orth=orth)
    assert R.converged and R.iters == stop
    x, ok, it, rn = _solve(bk, case, side, reltol=reltol, restart=restart, maxiter=maxiter, orth=orth, fused=fused)
    assert (ok, it) == (True, stop)
    kappa = max(H.cond[1:stop + 1])
    if R.checks == 0:  # with a true-residual check, resnorm is that residual
        _check_iterate(H, side, case, stop, kappa, x, rn)
    else:
        _check_iterate(H, side, case, stop, kappa, x)
    return R, x, it


@pytest.mark.parametrize("side", ["none", "left", "right"])
def test_exact_count_by_side(bk, side):
    """tol = reltol * ||Pl rhs|| with a left preconditioner: beta0 is the preconditioned residual's"""
    case = _sh2d_case(bk, (48, 32), -1.0, side, krylov_m=40, a0=_shift(_sh_lmax((48, 32), (LX, LY)), -1.0) / 8)
    _exact_count(bk, case, side, start=4)


def test_exact_count_restart_one_and_partial_cycles(bk):
    case = _sh2d_case(bk, (16, 12), 1.0, krylov_m=30, a0=3.0 * _sh_lmax((16, 12), (LX, LY)))
    R, _, _ = _exact_count(bk, case, restart=1, maxiter=60, start=3)
    assert R.cycles == list(range(R.iters))
    # restart 7, maxiter 23: the stop inside the fourth cycle (columns 22 or 23), and not converged at 23
    case = _sh2d_case(bk, (48, 32), -1.0, krylov_m=30)
    H = _ref(case, "none", 7, 23)
    assert H.cycles == [0, 7, 14, 21]
    kappa = max(H.cond[1:])
    for k in (21, 22):
        if float(H.rho[k]) / float(H.rho[k + 1]) >= 1.5:
            t = float(np.sqrt(H.rho[k] * H.rho[k + 1]))
            x, ok, it, rn = _solve(bk, case, reltol=t / float(H.beta0), restart=7, maxiter=23)
            assert (ok, it) == (True, k + 1)
            _check_iterate(H, "none", case, k + 1, kappa, x)
            break
    else:
        pytest.fail("no contraction >= 1.5 at the end of the fourth cycle")
    x, ok, it, rn = _solve(bk, case, reltol=0.5 * float(H.rho[23] / H.beta0), restart=7, maxiter=23)
    assert (ok, it) == (False, 23)
    _check_iterate(H, "none", case, 23, kappa, x, rn)


def test_restart_clamped_to_krylov_m_and_n(bk):
    """restart > krylov_m gives the bits of restart = krylov_m; restart > n those of restart = n, and full GMRES on a
    7 x 5 grid reaches A^-1 b to C_X n eps kappa"""
    case = _sh2d_case(bk, (16, 12), -1.0, krylov_m=10)
    a = _solve(bk, case, reltol=1e-10, restart=50, maxiter=35)
    b = _solve(bk, case, reltol=1e-10, restart=10, maxiter=35)
    assert a[1:] == b[1:] and np.array_equal(a[0], b[0])
    assert a[2] > 10  # the run restarted
    dims = (7, 5)
    case = _sh2d_case(bk, dims, -1.0, krylov_m=64, a0=3.0)
    n = case.ctx.N
    M = X.dense(case.A, n)
    xd = X.direct_solve(M, case.rhs)
    kappa = float(np.linalg.cond(M.astype(np.float64)))
    for maxiter in (n, 2 * n):
        st0 = case.ctx.stats()["kernel_launches"]
        a = _solve(bk, case, reltol=0.0, restart=200, maxiter=maxiter)
        st1 = case.ctx.stats()["kernel_launches"]
        b = _solve(bk, case, reltol=0.0, restart=n, maxiter=maxiter)
        st2 = case.ctx.stats()["kernel_launches"]
        assert a[1:] == b[1:] and np.array_equal(a[0], b[0]) and st1 - st0 == st2 - st1
        assert a[2] == maxiter and not a[1]
        err = float(X.nrm(X.ld(a[0]) - xd) / X.nrm(xd))
        assert err <= C_X * n * EPS * kappa, (maxiter, err, C_X * n * EPS * kappa)


# ---------------------------------------------------------------------------------------------------- stopping-rule edges
def test_zero_rhs_host_and_device(bk):
    case = _sh2d_case(bk, (16, 12), -1.0)
    for rhs in (np.zeros(case.ctx.N), case.ctx.to_device(np.zeros(case.ctx.N))):
        ls = bk.GMRESB200(reltol=1e-8, restart=30, maxiter=30)
        x, ok, it = ls(case.J, rhs, a0=case.a0, a1=case.a1)
        x = x.numpy() if hasattr(x, "numpy") else x
        assert ok and it == 0 and ls.last_resnorm == 0.0
        assert np.all(x == 0) and not np.any(np.signbit(x))


def test_abstol_dominates(bk):
    case = _sh2d_case(bk, (16, 12), -1.0)
    H = _ref(case, "none", 30, 30)
    stop, t = _gap_tol(H, start=5)
    reltol = 1e-3 * t / float(H.beta0)
    x, ok, it, rn = _solve(bk, case, reltol=reltol, abstol=t, restart=30, maxiter=30)
    assert (ok, it) == (True, stop)
    _check_iterate(H, "none", case, stop, max(H.cond[1:stop + 1]), x)


def test_zero_tolerances_run_to_maxiter_at_the_rounding_floor(bk):
    """reltol = abstol = 0: maxiter columns, not converged, x finite with its residual at the floor.  With one-column
    cycles, each restart's Givens estimate starts from the recomputed residual, so at the floor `resnorm` stays within a
    factor 1e3 of the true residual (a cycle that restarted from the previous estimate would drift orders below it)"""
    case = _sh2d_case(bk, (16, 12), 1.0, a0=3.0 * _sh_lmax((16, 12), (LX, LY)))
    for restart, maxiter in ((30, 60), (1, 120)):
        H = _ref(case, "none", restart, maxiter)
        x, ok, it, rn = _solve(bk, case, reltol=0.0, abstol=0.0, restart=restart, maxiter=maxiter)
        assert (ok, it) == (False, maxiter) and np.all(np.isfinite(x)) and np.isfinite(rn)
        res_b, _, _ = _bounds(H, "none", case, maxiter, 1.0)
        tr = _true_res(case, "none", x)
        assert tr <= res_b and float(H.rho[maxiter]) <= 1e-3 * res_b  # the reference is far below the floor
        if restart == 1:
            assert tr / 1e3 <= rn <= tr * 1e3 + res_b, (rn, tr)


def test_pure_shift_happy_breakdown(bk):
    """a1 = 0 and ||rhs|| a power of two: v'_1 = w - h s_0 v'_0 is exactly zero, so the exact-breakdown branch hk1 == 0
    ends the solve after one column although the speculative step after it divides by a zero norm"""
    for dims in ((16, 12), (15, 7)):
        case = _sh2d_case(bk, dims, 0.0, a0=3.0)
        rhs = np.zeros(case.ctx.N)
        rhs[np.random.default_rng(11).choice(case.ctx.N, 64, replace=False)] = np.random.default_rng(12).choice([-1.0, 1.0], 64)
        case.rhs = rhs
        for fused in (True, False):
            x, ok, it, rn = _solve(bk, case, reltol=1e-8, restart=30, maxiter=30, fused=fused)
            assert ok and it == 1 and rn == 0.0
            assert np.all(np.isfinite(x))
            assert np.max(np.abs(x - rhs / 3.0)) <= np.spacing(1.0 / 3.0)


def test_nan_rhs_returns_not_converged(bk):
    case = _sh2d_case(bk, (16, 12), -1.0)
    case.rhs = case.rhs.copy()
    case.rhs[5] = np.nan
    ls = bk.GMRESB200(reltol=1e-8, restart=30, maxiter=30)
    x, ok, it = ls(case.J, case.rhs, a0=case.a0, a1=case.a1)
    assert not ok and it == 0
    xout = np.empty(case.ctx.N)  # kept alive: the call writes x through this pointer
    st = case.ctx.lib.bk_gmres(case.ctx.handle, bk.lib.ptr(case.rhs), bk.lib.ptr(xout), case.a0, case.a1,
                               bk.lib.C.byref(ls.opts()), None, None, None)
    assert st == bk.lib.BK_NOT_CONVERGED


# --------------------------------------------------------------------------------------------- borders and block borders
@pytest.mark.parametrize("fused", [True, False])
def test_matrixfree_bordered_exact_count(bk, fused):
    dims = (16, 12)
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    u = problems.sh2d_sol0(*dims, LX, LY)
    rng = np.random.default_rng(14)
    N = sh.N
    a, b, R, n = rng.standard_normal(N), rng.standard_normal(N), rng.standard_normal(N), -0.4
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=40, params=(-0.1, 1.3))
    J = ctx.jacobian(u)
    shift = _shift(_sh_lmax(dims, (LX, LY)), 1.0) / 1.2
    A = X.bordered_op(X.sh_op(sh, u, shift, 1.0), [a], [b], [[0.9]], dotscale=1.0 / N)
    rhs = np.concatenate([R, [n]])
    H = X.gmres(A, rhs, reltol=0.0, restart=40, maxiter=40)
    stop, t = _gap_tol(H, start=4)
    ls = bk.GMRESB200(reltol=t / float(H.beta0), restart=40, maxiter=40, fused=fused)
    dX, dl, ok, it = bk.MatrixFreeBLSB200(ls)(J, a, b, 0.9, R, n, shift=shift, dotscale=1.0 / N)
    assert (ok, it) == (True, stop)
    _check_iterate(H, "none", Case(ctx, J, A, rhs, 0, 0), stop, max(H.cond[1:stop + 1]), np.concatenate([dX, [dl]]))


def test_block_bordered_m2_exact_count(bk):
    dims = (16, 12)
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    u = problems.sh2d_sol0(*dims, LX, LY)
    rng = np.random.default_rng(15)
    N = sh.N
    a = [rng.standard_normal(N) for _ in range(2)]
    b = [rng.standard_normal(N) for _ in range(2)]
    c = np.array([[1.1, 0.2], [-0.3, 0.8]])
    rhst, rhsb = rng.standard_normal(N), np.array([0.3, -0.6])
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=40, params=(-0.1, 1.3))
    J = ctx.jacobian(u)
    shift = _shift(_sh_lmax(dims, (LX, LY)), 1.0) / 1.2
    A = X.bordered_op(X.sh_op(sh, u, shift, 1.0), a, b, c, dotscale=1.0 / N)
    rhs = np.concatenate([rhst, rhsb])
    H = X.gmres(A, rhs, reltol=0.0, restart=40, maxiter=40)
    stop, t = _gap_tol(H, start=4)
    ls = bk.GMRESB200(reltol=t / float(H.beta0), restart=40, maxiter=40)
    uu, p, ok, it = bk.MatrixFreeBLSB200(ls).solve_block(J, tuple(a), tuple(b), c, rhst, rhsb, shift=shift, dotscale=1.0 / N)
    assert (ok, it) == (True, stop)
    _check_iterate(H, "none", Case(ctx, J, A, rhs, 0, 0), stop, max(H.cond[1:stop + 1]), np.concatenate([uu, p]))


# --------------------------------------------------------------------------------------------------------- the CGS check
def test_cgs_check_passes_on_a_long_converged_cycle(bk):
    """single-pass CGS converging after >= 40 columns with reltol >= 1e-9: the true residual is recomputed once (one more
    operator application, axpby and norm), accepted, and no CGS2 fallback is taken"""
    dims = (48, 32)
    case = _sh2d_case(bk, dims, -1.0, krylov_m=120, a0=_shift(_sh_lmax(dims, (LX, LY)), -1.0) / 30)
    H = _ref(case, "none", 120, 120)
    # this slowly converging system contracts by less than 1.5 per column past 40: a ratio 1.2 still leaves a margin of
    # 1.095, ~1e8 times the residual bound
    stop, t = _gap_tol(H, start=40, ratio=1.2)
    reltol = t / float(H.beta0)
    assert stop >= 41 and reltol >= 1e-9
    ctx = case.ctx
    st = lambda: ctx.stats()
    f0 = st()["cgs_fallbacks"]
    # launches of the same solve with maxiter = stop (no check: the cap is reached) and maxiter = stop - 1 (one column less)
    l0 = st()["kernel_launches"]
    x, ok, it, rn = _solve(bk, case, reltol=reltol, restart=120, maxiter=120)
    l1 = st()["kernel_launches"]
    xs, oks, its, _ = _solve(bk, case, reltol=reltol, restart=120, maxiter=stop)
    l2 = st()["kernel_launches"]
    _solve(bk, case, reltol=reltol, restart=120, maxiter=stop - 1)
    l3 = st()["kernel_launches"]
    assert (ok, it) == (True, stop) and (oks, its) == (True, stop)
    assert st()["cgs_fallbacks"] == f0
    assert np.array_equal(x, xs)  # the check does not touch x
    step = (l2 - l1) - (l3 - l2)   # the launches of one Arnoldi column
    xd = ctx.to_device(x)
    j0 = st()["kernel_launches"]
    case.J(xd)
    apply = st()["kernel_launches"] - j0
    # maxiter = 120 launched one speculative column more, then the check: apply, rhs - A x and the norm pass
    assert (l1 - l0) - (l2 - l1) == step + apply + 2
    tol = reltol * float(H.beta0)
    assert _true_res(case, "none", x) <= 4 * tol
    res_b, _, _ = _bounds(H, "none", case, stop, 1.0)
    assert abs(rn - _true_res(case, "none", x)) <= res_b  # resnorm is the recomputed residual


def _hexagon_case(bk):
    dims = (48, 32)
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    u = problems.sh2d_sol0(*dims, LX, LY) + 0.1 * np.random.default_rng(1).standard_normal(sh.N)
    rhs = np.random.default_rng(7).standard_normal(sh.N)
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=400, params=(-0.1, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    anorm = 1.0 + _sh_lmax(dims, (LX, LY)) + np.abs(-0.1 + 2.6 * u - 3.0 * u**2).max()
    return Case(ctx, ctx.jacobian(u), X.sh_op(sh, u, 1.0, 1.0), rhs, 1.0, 1.0, X.dct_precond(dims, (LX, LY), 1.0), anorm)


def test_cgs_check_falls_back_below_the_attainable_floor(bk):
    """reltol = 1e-13 on a right-DCT-preconditioned SH2d system: single-pass CGS claims convergence while the true
    residual is above 4 tol.  The check catches it, counts a CGS2 fallback, and the solve never reports a false converged"""
    case = _hexagon_case(bk)
    f0 = case.ctx.stats()["cgs_fallbacks"]
    x, ok, it, rn = _solve(bk, case, "right", reltol=1e-13, restart=400, maxiter=400)
    assert case.ctx.stats()["cgs_fallbacks"] == f0 + 1
    tol = 1e-13 * float(X.nrm(X.ld(case.rhs)))
    if ok:
        assert _true_res(case, "right", x) <= 4 * tol
    # with CGS2 from the start there is nothing to fall back from
    x2, ok2, it2, _ = _solve(bk, case, "right", reltol=1e-13, restart=400, maxiter=400, orth="cgs2")
    assert case.ctx.stats()["cgs_fallbacks"] == f0 + 1


def test_converged_cgs_solves_meet_four_tol(bk):
    """every single-pass CGS solve that reports converged where the check applies has a true residual <= 4 tol"""
    cases = [(_sh2d_case(bk, (48, 32), -1.0, "right", krylov_m=200, a0=1.0), "right"),
             (_sh2d_case(bk, (48, 32), -1.0, "left", krylov_m=200, a0=1.0), "left"),
             (_sh2d_case(bk, (64, 37), 1.0, krylov_m=200, a0=1.3 * _sh_lmax((64, 37), (LX, LY)) / 1.2), "none")]
    for case, side in cases:
        for reltol in (1e-10, 1e-12):
            x, ok, it, rn = _solve(bk, case, side, reltol=reltol, restart=200, maxiter=200)
            beta0 = float(X.nrm(case.pc(X.ld(case.rhs)) if side == "left" else X.ld(case.rhs)))
            if ok:
                assert _true_res(case, side, x) <= 4 * reltol * beta0, (side, reltol, it)


# ------------------------------------------------------------------------------------------------------------- bk_gmres2
def test_gmres2_one_converges_one_does_not(bk):
    case = _sh2d_case(bk, (16, 12), -1.0)
    r1 = 1e-3 * case.rhs
    r2 = np.random.default_rng(21).standard_normal(case.ctx.N)
    c1 = Case(case.ctx, case.J, case.A, r1, case.a0, case.a1)
    c2 = Case(case.ctx, case.J, case.A, r2, case.a0, case.a1)
    H1, H2 = _ref(c1, "none", 30, 30), _ref(c2, "none", 30, 30)
    stop, t = _gap_tol(H1, start=2)
    maxiter = stop + 1
    assert float(H2.rho[maxiter]) > 2 * t  # rhs2 is 1000 times larger: not converged at maxiter
    ls = bk.GMRESB200(reltol=0.0, abstol=t, restart=30, maxiter=maxiter)
    x1, x2, ok, its = ls(case.J, r1, r2, a0=case.a0, a1=case.a1)
    assert ok is False and its == (stop, maxiter)
    s1 = ls(case.J, r1, a0=case.a0, a1=case.a1)
    s2 = ls(case.J, r2, a0=case.a0, a1=case.a1)
    assert (s1[1], s1[2]) == (True, stop) and (s2[1], s2[2]) == (False, maxiter)
    assert np.array_equal(x1, s1[0]) and np.array_equal(x2, s2[0])
    _check_iterate(H1, "none", c1, stop, max(H1.cond[1:stop + 1]), x1)
    _check_iterate(H2, "none", c2, maxiter, max(H2.cond[1:maxiter + 1]), x2)


@pytest.mark.parametrize("transpose", [False, True])
def test_complex_context_exact_count(bk, transpose):
    """ComplexGMRESB200 on a BK_COMPLEX cGL context, ((a0 + i a0_imag) I - J) z = rhs with J and J': the real-equivalent
    2 N0 system, iteration count exact, solution and resnorm within the bounds"""
    dims = (24, 12)
    gl = problems.GinzburgLandau2D(*dims, np.pi, np.pi / 2, r=1.2)
    ug = 0.3 * np.random.default_rng(10).standard_normal(gl.N)
    a0 = 0.3 * 8 * max(24 / (2 * np.pi), 12 / np.pi) ** 2 + 10.0
    ctx = bk.Context(bk.BK_CGL2D, dims, (np.pi, np.pi / 2), krylov_m=40, params=(1.2, 0.1, 1.0, -1.0, 1.0), complex=True)
    z = np.random.default_rng(11).standard_normal(2 * gl.N)
    A = X.complex_op(X.cgl_op(gl, ug, transpose=transpose), gl.N, a0, -0.6, -1.0)
    case = Case(ctx, None, A, z, 0, 0)
    H = _ref(case, "none", 40, 40)
    stop, t = _gap_tol(H, start=4)
    ls = bk.ComplexGMRESB200(reltol=t / float(H.beta0), restart=40, maxiter=40)
    x, ok, it = ls(ctx.cjacobian(ug, transpose), z[:gl.N] + 1j * z[gl.N:], a0=complex(a0, -0.6), a1=-1.0)
    assert (ok, it) == (True, stop)
    _check_iterate(H, "none", case, stop, max(H.cond[1:stop + 1]), np.concatenate([x.real, x.imag]), ls.last_resnorm)
