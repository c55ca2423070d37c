"""Shift-invert eigensolver (bk_eigs_shift_invert through ShiftInvertB200) against spectra computed without the device: closed
forms in long double where J is diagonal in a known basis, dense LAPACK on the oracle's Jacobian otherwise.

The solver has two outer iterations around the same device kernels: a thick restart (Krylov-Schur with Ritz vectors) for the
symmetric kinds (SH2d, SH3d) and an explicitly restarted Arnoldi for the others (chan, cGL2d).  Each case runs its path on
purpose: a restart shows as more inner solves than the Krylov dimension (nops > krylovdim), the invariant-subspace exit as
fewer than the problem size.

Tolerances.  The inner GMRES stops at ||b - (J - sigma) x|| <= rho ||b||, so every application of the operator
(J - sigma)^-1 is off by at most rho ||(J - sigma)^-1|| = rho / delta, delta = min_i |lambda_i - sigma|.  The converged flag
certifies Ritz residuals below tol |theta|.  For a normal J, Bauer-Fike then bounds the error of theta = 1 / (lambda - sigma)
by tol |theta| + rho / delta, and lambda = sigma + 1 / theta turns it into
    |d lambda| <= tol |lambda - sigma| + rho |lambda - sigma|^2 / delta,
times the condition number kappa of the eigenvalue for a non-normal J.  The eigen-residual of a Ritz vector v (||v|| = 1),
J v - lambda v = -(J - sigma) r / theta with r the residual of the operator, is bounded by
    ||J - sigma|| (tol + rho |lambda - sigma| / delta).
rho stands for rho + eps ||J - sigma|| / delta, the rounding floor of the inner residual.  Both get a factor 10: the solver's residual estimate (|h_{m+1,m}| times the last component of the small eigenvector) stands for
the true residual, and J is applied in fp64 (eps ||J|| per application, far below the terms above).
"""
import types

import numpy as np
import pytest
import scipy.fft
import scipy.linalg

import __graft_entry__ as g
from oracle import problems, precond as oprecond

pytestmark = pytest.mark.gpu

EPS = float(np.finfo(np.float64).eps)
PI_LD = np.arccos(np.longdouble(-1))
SH_L, SH_NU, SH_C0 = 0.1, 1.2, 0.3
SH_COEF = SH_L + 2 * SH_NU * SH_C0 - 3 * SH_C0**2      # J = SH_COEF I - (I + Lap)^2 at the constant state SH_C0


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


# ------------------------------------------------------------------------------------------------------------- references
def _neumann_eigs_ld(n, L):
    """oracle.precond.neumann_eigs(n, 2 L / n) in long double: the Neumann Laplacian of oracle.problems in the DCT-II basis"""
    h = 2 * np.longdouble(L) / n
    mu = (2 * np.cos(PI_LD * np.arange(n, dtype=np.longdouble) / n) - 2) / h**2
    assert np.allclose(mu.astype(float), oprecond.neumann_eigs(n, 2 * L / n), rtol=1e-13, atol=1e-13)
    return mu


def _sh_const_spectrum(dims, L, coef=SH_COEF):
    """coef - (1 + sum_d mu_d)^2 for every DCT mode, long double, mode (k0, k1, ...) at flat index k0 + n0 k1 + ..."""
    t = np.longdouble(1)
    for d, (n, Li) in enumerate(zip(dims, L)):
        shape = [1] * len(dims)
        shape[len(dims) - 1 - d] = n
        t = t + _neumann_eigs_ld(n, Li).reshape(shape)
    return (np.longdouble(coef) - t**2).reshape(-1)


def _cgl_zero_spectrum(dims, L, r, nu):
    """cGL2d linearised at u = 0: [[Lap + r, -nu], [nu, Lap + r]], eigenvalues r + mu_k +- i nu with mu_k the eigenvalues of the
    Dirichlet Laplacian of oracle.problems (h = 2 L / n, modes sin(pi k i / (n + 1))), long double"""
    mu = 0
    for d, (n, Li) in enumerate(zip(dims, L)):
        h = 2 * np.longdouble(Li) / n
        e = (2 * np.cos(PI_LD * np.arange(1, n + 1, dtype=np.longdouble) / (n + 1)) - 2) / h**2
        mu = np.add.outer(mu, e) if d else e
    mu = np.asarray(mu).reshape(-1)
    return np.concatenate([(r + mu).astype(float) + 1j * nu, (r + mu).astype(float) - 1j * nu]), mu


def _dense(apply, n):
    return np.column_stack([apply(e) for e in np.eye(n)])


def _nearest(spec, sigma, k):
    return spec[np.argsort(np.abs(spec - sigma), kind="stable")[:k]]


def _pick_sigma(spec, nev):
    """A real shift above the rightmost eigenvalue (so J - sigma is definite for the symmetric kinds and the inner GMRES converges
    fast), a quarter of the spread of the wanted block away from it: the wanted eigenvalues are then the nev rightmost, and
    sigma is no closer to one of them than a fifth of the nev-th distance (well-conditioned inner solves)."""
    spec = np.asarray(spec, dtype=complex)
    re = np.sort(spec.real)[::-1]
    sigma = float(re[0] + 0.25 * max(re[0] - re[nev - 1], 1e-2))
    d = np.sort(np.abs(spec - sigma))
    # well posed: the nev-th and (nev+1)-th sigma-nearest are separated by far more than the value tolerance (< 1e-8 here)
    assert d[nev] - d[nev - 1] > 1e-6, (nev, d[: nev + 1])
    return sigma


def _bounds(lam, spec, sigma, tol, rho, kappa=1.0):
    """(value tolerance per eigenvalue, eigen-residual bound per eigenvalue) of the module docstring"""
    d = np.abs(np.asarray(lam) - sigma)
    delta = np.min(np.abs(spec - sigma))
    normJs = np.max(np.abs(spec - sigma))
    rho = rho + EPS * normJs / delta      # GMRES cannot push the true residual below eps ||J - sigma|| ||x|| ~ eps ||J - sigma|| / delta
    return 10 * kappa * (tol * d + rho * d**2 / delta), 10 * kappa * normJs * (tol + rho * d / delta)


def _projector_norms(Jd, lams):
    """the condition number of each eigenvalue in lams: ||P||_2 of the spectral projector X (Y^H X)^-1 Y^H onto its eigenspace
    (1 / |y^H x| for unit vectors of a simple eigenvalue), from scipy's left and right eigenvectors of the dense Jd"""
    w, yl, xr = scipy.linalg.eig(Jd, left=True, right=True)
    out = []
    for lam in lams:
        sel = np.abs(w - lam) < 1e-8 * max(1.0, abs(lam))
        X, Y = xr[:, sel], yl[:, sel]
        out.append(np.linalg.norm(X @ np.linalg.solve(Y.conj().T @ X, Y.conj().T), 2))
    return np.array(out)


def _match(vals, want):
    """vals and want as the same multiset, both in the solver's order (decreasing real part, then decreasing imaginary part)"""
    key = lambda z: (-round(z.real, 6), -z.imag)
    return np.array(sorted(vals, key=key)), np.array(sorted(want, key=key))


# ------------------------------------------------------------------------------------------------------------- 1. thick restart, closed form
SH_GRIDS = {
    "even": ((24, 14), (2.7 * np.pi, 1.9 * np.pi)),        # nx even: the fused JVP + dots kernels
    "odd": ((25, 14), (2.7 * np.pi, 1.9 * np.pi)),         # nx odd: apply + k2_dots
    "3d": ((10, 8, 6), (2.2 * np.pi, 1.7 * np.pi, 1.3 * np.pi)),
}
RHO = 1e-12


def _sh_ctx(bk, dims, L, params=(SH_L, SH_NU), m=60):
    ctx = bk.Context(bk.BK_SH2D if len(dims) == 2 else bk.BK_SH3D, dims, L, krylov_m=m, params=params)
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    return ctx


def _check_symmetric(vals, vecs, Js, want, spec, sigma, tol):
    """values against want (same order), real and sorted, eigen-residuals with the oracle's sparse Jacobian Js, orthonormal
    vectors"""
    dv, dr = _bounds(want, spec, sigma, tol, RHO)
    assert np.all(np.diff(vals.real) <= 0), vals
    assert np.all(vals.imag == 0), vals
    assert np.all(np.abs(vals.real - want) <= dv), (vals.real - want, dv)
    for k in range(len(vals)):
        v = vecs[:, k]
        res = np.linalg.norm(Js @ v - vals[k].real * v) / np.linalg.norm(v)
        assert res <= dr[k], (k, vals[k], res, dr[k])
    G = vecs.T @ vecs
    assert np.max(np.abs(G - np.eye(len(vals)))) < 1e-10, G   # CGS2 keeps Q orthonormal to O(m eps), Jacobi's S is orthogonal


def _check_operator_residual(vals, vecs, dims, spec, sigma, tol):
    """The converged flag's claim itself: the Ritz residual ||Op v - theta v|| with the EXACT operator Op = (J - sigma)^-1, applied
    in the DCT basis where it is diagonal, theta = 1 / (lambda - sigma), v unit.  The flag certifies |h_{m+1,m}| |s_last| <=
    tol |theta| for the computed operator, which is off the exact one by rho / delta (module docstring; rho with its rounding
    floor), times sqrt(m) for the symmetrised projected matrix standing for the computed one; a factor 2 on the certified part
    covers rounding.  A residual estimate that lags the factorisation it certifies (the h_{m+1,m} of an earlier cycle) lets
    the flag through before this holds."""
    delta = np.min(np.abs(spec - sigma))
    rho = RHO + EPS * np.max(np.abs(spec - sigma)) / delta
    shape = tuple(dims[::-1])
    for k in range(len(vals)):
        v = vecs[:, k] / np.linalg.norm(vecs[:, k])
        opv = scipy.fft.idctn(scipy.fft.dctn(v.reshape(shape), norm="ortho") / (spec.reshape(shape) - sigma), norm="ortho")
        theta = 1.0 / (vals[k].real - sigma)
        res = np.linalg.norm(opv.reshape(-1) - theta * v)
        assert res <= 2 * tol * abs(theta) + 10 * rho / delta, (k, vals[k], res, tol * abs(theta))


@pytest.mark.parametrize("nev", [1, 6, 12])
@pytest.mark.parametrize("grid", list(SH_GRIDS))
def test_thick_restart_constant_state_closed_form(bk, grid, nev):
    """SH at a constant state: J = coef I - (I + Lap)^2 is diagonal in the DCT basis.  Krylov dimension nev + 4 restarts (thick
    restart: arrow matrix, pkeep Ritz vectors rebuilt into Q2, residual estimate after a restart), nev + 12 restarts unless the
    gap is wide (nev = 1), 40 is the long run the others must agree with."""
    dims, L = SH_GRIDS[grid]
    spec = _sh_const_spectrum(dims, L).astype(float)
    sigma = _pick_sigma(spec, nev)
    want = np.sort(_nearest(spec, sigma, nev))[::-1]
    ctx = _sh_ctx(bk, dims, L)
    sh = problems.SwiftHohenberg(dims, L, l=SH_L, nu=SH_NU)
    u = np.full(sh.N, SH_C0)
    Js = sh.jac_sparse(u)
    J = ctx.jacobian(ctx.to_device(u))
    inner = bk.GMRESB200(reltol=RHO, restart=60, maxiter=600, Pr=True)
    tol = 1e-10
    runs = {}
    for kd in (nev + 4, nev + 12, 40):
        vals, vecs, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=kd, tol=tol, maxrestart=500)(J, nev, want_vectors=True)
        assert cv, (kd, vals, nops)
        if kd == nev + 4:
            assert nops > kd, (kd, nops)     # restarted
        _check_symmetric(vals, vecs, Js, want, spec, sigma, tol)
        _check_operator_residual(vals, vecs, dims, spec, sigma, tol)
        runs[kd] = vals.real
    dv, _ = _bounds(want, spec, sigma, tol, RHO)
    for kd in (nev + 4, nev + 12):
        assert np.all(np.abs(runs[kd] - runs[40]) <= 2 * dv), (kd, runs[kd] - runs[40])


# ------------------------------------------------------------------------------------------------------------- 2. thick restart, dense
def _hexagon_case():
    dims, L = (32, 20), (8 * np.pi, 4 * np.pi / np.sqrt(3))
    sh = problems.SwiftHohenberg(dims, L, l=-0.1, nu=1.3)
    u = problems.sh2d_sol0(*dims, *L)
    Js = sh.jac_sparse(u)
    spec = np.linalg.eigvalsh(Js.toarray())
    return dims, L, u, Js, spec


def test_thick_restart_hexagons_dense(bk):
    """SH2d at the hexagon state (not diagonal in any known basis): the nev = 5 sigma-nearest eigenvalues of eigh of the dense
    Jacobian, restarted (krylovdim 9) and in one long Krylov space (40)."""
    dims, L, u, Js, spec = _hexagon_case()
    nev, tol = 5, 1e-10
    sigma = _pick_sigma(spec, nev)
    want = np.sort(_nearest(spec, sigma, nev))[::-1]
    ctx = _sh_ctx(bk, dims, L, params=(-0.1, 1.3))
    J = ctx.jacobian(ctx.to_device(u))
    inner = bk.GMRESB200(reltol=RHO, restart=60, maxiter=600, Pr=True)
    for kd in (nev + 4, 40):
        vals, vecs, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=kd, tol=tol, maxrestart=500)(J, nev, want_vectors=True)
        assert cv, (kd, vals, nops)
        if kd < 40:
            assert nops > kd, nops
        _check_symmetric(vals, vecs, Js, want, spec, sigma, tol)


def test_thick_restart_sigma_between_close_eigenvalues(bk):
    """sigma at the midpoint of the two rightmost eigenvalues of a constant state (9e-4 apart, the third 1.9e-3 below sigma):
    the two are equally near, one on each side (theta = +-2 / gap), so the selection by |theta| keeps both and the final sort
    puts the upper one first.  The preconditioned operator has eigenvalues +-4.6e-4 on either side of 0 and the rest in
    (-1, 0): restarted GMRES(60) can stall there near 1e-6, which would move lambda by ~ (rho / delta) |lambda - sigma|^2 ~ 4e-10,
    so the inner GMRES gets a Krylov space of 200 (it converges unrestarted in about 120 iterations), and one solve with the
    same options shows that it reaches rho."""
    dims, L = (24, 16), (3.1 * np.pi, 2.3 * np.pi)
    spec = _sh_const_spectrum(dims, L).astype(float)
    top = np.sort(spec)[::-1]
    sigma = 0.5 * (top[0] + top[1])
    d = np.sort(np.abs(spec - sigma))
    assert d[2] > 3 * d[1], d[:3]                       # the pair stands apart from everything else
    want = top[:2]
    sh = problems.SwiftHohenberg(dims, L, l=SH_L, nu=SH_NU)
    u = np.full(sh.N, SH_C0)
    Js = sh.jac_sparse(u)
    ctx = _sh_ctx(bk, dims, L, m=200)
    J = ctx.jacobian(ctx.to_device(u))
    # J - sigma has condition ~ 2e5 here: two Gram-Schmidt passes keep GMRES's residual estimate that of the true residual
    inner = bk.GMRESB200(reltol=RHO, restart=200, maxiter=2000, Pr=True, orth="cgs2")
    b = np.random.default_rng(11).standard_normal(sh.N)
    x, ok, it = inner(J, ctx.to_device(b), a0=-sigma, a1=1.0)
    x = x.numpy()
    # true residual: GMRES's estimate plus the rounding floor eps ||J - sigma|| ||x||
    floor = EPS * np.max(np.abs(spec - sigma)) * np.linalg.norm(x)
    assert ok and np.linalg.norm(b - (Js @ x - sigma * x)) <= 10 * (RHO * np.linalg.norm(b) + floor), (ok, it)
    tol, kd = 1e-12, 4
    vals, vecs, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=kd, tol=tol, maxrestart=500)(J, 2, want_vectors=True)
    assert cv and nops > kd, (vals, nops)
    assert vals[0].real > sigma > vals[1].real, (vals, sigma)
    _check_symmetric(vals, vecs, Js, want, spec, sigma, tol)


# ------------------------------------------------------------------------------------------------------------- 3. double eigenvalue
@pytest.mark.parametrize("kd", [6, 40])
def test_double_eigenvalue_square_box(bk, kd):
    """Square box (nx = ny, Lx = Ly) at a constant state: modes (k, l) and (l, k) share an eigenvalue.  sigma next to such a
    double eigenvalue, nev = 2: both copies are the sigma-nearest.  Every returned pair must be an eigenpair, the two vectors
    independent, and the multiplicity that of the dense spectrum -- bifdiagram's nd detection counts it."""
    n, Lb = 16, 2.4 * np.pi
    dims, L = (n, n), (Lb, Lb)
    spec = _sh_const_spectrum(dims, L).astype(float)
    sh = problems.SwiftHohenberg(dims, L, l=SH_L, nu=SH_NU)
    u = np.full(sh.N, SH_C0)
    Js = sh.jac_sparse(u)
    dense = np.linalg.eigvalsh(Js.toarray())
    # the double eigenvalue nearest the top whose neighbours are at least 1e-3 away
    top = np.sort(spec)[::-1]
    lam2 = next(top[i] for i in range(1, 60) if top[i - 1] - top[i] < 1e-12 and (i < 2 or top[i - 2] - top[i] > 1e-3)
                and top[i] - top[i + 1] > 1e-3)
    assert np.sum(np.abs(dense - lam2) < 1e-9) == 2     # the dense spectrum has it twice as well
    gap = np.min(np.abs(spec[np.abs(spec - lam2) > 1e-9] - lam2))
    sigma = lam2 + 0.2 * gap
    ctx = _sh_ctx(bk, dims, L)
    J = ctx.jacobian(ctx.to_device(u))
    inner = bk.GMRESB200(reltol=RHO, restart=60, maxiter=600, Pr=True)
    tol = 1e-10
    vals, vecs, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=kd, tol=tol, maxrestart=500)(J, 2, want_vectors=True)
    assert cv, (vals, nops)
    if kd < 40:
        assert nops > kd, nops
    dv, dr = _bounds(np.array([lam2, lam2]), spec, sigma, tol, RHO)
    for k in range(2):
        v = vecs[:, k]
        res = np.linalg.norm(Js @ v - vals[k].real * v) / np.linalg.norm(v)
        assert res <= dr[k], (k, vals, res)
    assert np.sum(np.abs(vals.real - lam2) <= dv) == 2, (vals, lam2, np.sort(np.abs(spec - sigma))[:3])
    s = np.linalg.svd(vecs / np.linalg.norm(vecs, axis=0), compute_uv=False)
    assert s[-1] > 0.5, s


# ------------------------------------------------------------------------------------------------------------- 4. explicit restart
CGL_DIMS, CGL_L = (12, 8), (np.pi, np.pi / 2)
CGL_PARS = (1.8, 0.1, 0.3, -1.0, 1.0)                     # r, mu, nu, c3, c5: the two leading pairs r + mu_1,2 +- 0.3 i are unstable


def _cgl_ctx(bk, m=60):
    return bk.Context(bk.BK_CGL2D, CGL_DIMS, CGL_L, krylov_m=m, params=CGL_PARS)


def _cgl_oracle():
    return problems.GinzburgLandau2D(*CGL_DIMS, *CGL_L, r=CGL_PARS[0], mu=CGL_PARS[1], nu=CGL_PARS[2], c3=CGL_PARS[3], c5=CGL_PARS[4])


def _check_general(bk, J, Jd, vals, vecs, spec, sigma, tol, kappa, want=None):
    """values against the dense spectrum (the sigma-nearest unless want is given), the solver's order, the complex
    eigen-residual of every column completed by normalform._eigvec, and the two columns of a pair returned whole spanning its
    real invariant plane"""
    want = _nearest(spec, sigma, len(vals)) if want is None else want
    got, ref = _match(vals, want)
    assert np.all(np.abs(got - ref) <= _bounds(ref, spec, sigma, tol, RHO, kappa)[0]), (got, ref)
    assert all((a.real, a.imag) >= (b.real, b.imag) for a, b in zip(vals[:-1], vals[1:])), vals
    normJs = np.max(np.abs(spec - sigma))
    for k in range(len(vals)):
        w = bk.normalform._eigvec(J, vals, vecs, k)
        dr = _bounds([vals[k]], spec, sigma, tol, RHO, kappa)[1][0]
        if vals[k].imag != 0:    # the completion Im(w) = (alpha v - J v) / beta multiplies the error of v by 1 + ||J - alpha|| / |beta|
            dr *= 1 + 2 * normJs / abs(vals[k].imag)
        res = np.linalg.norm(Jd @ w - vals[k] * w) / np.linalg.norm(w)
        assert res <= dr, (k, vals[k], res, dr)
    for i in range(len(vals)):
        for j in range(i + 1, len(vals)):
            if vals[i].imag > 0 and abs(vals[j] - np.conj(vals[i])) < 1e-6 * abs(vals[i]):
                P = vecs[:, [i, j]] / np.linalg.norm(vecs[:, [i, j]], axis=0)
                assert np.linalg.svd(P, compute_uv=False)[-1] > 0.1, (i, j, vals[i])


def test_explicit_restart_cgl_zero_state_closed_form(bk):
    """cGL2d at u = 0: J is normal with eigenvalues r + mu_k +- i nu.  nev = 4 (two whole pairs), krylovdim 8: restarted."""
    spec, _ = _cgl_zero_spectrum(CGL_DIMS, CGL_L, CGL_PARS[0], CGL_PARS[2])
    gl = _cgl_oracle()
    u = np.zeros(gl.N)
    Jd = _dense(lambda e: gl.dF(u, e), gl.N)
    assert np.max(np.abs(np.sort_complex(np.linalg.eigvals(Jd)) - np.sort_complex(spec))) < 1e-10
    nev, kd, tol, sigma = 4, 8, 1e-10, 0.5
    d = np.sort(np.abs(spec - sigma))
    assert d[nev] > 1.5 * d[nev - 1], d[: nev + 1]
    ctx = _cgl_ctx(bk)
    J = ctx.jacobian(ctx.to_device(u))
    inner = bk.GMRESB200(reltol=RHO, restart=60, maxiter=2000, orth="cgs2")
    vals, vecs, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=kd, tol=tol, maxrestart=500)(J, nev, want_vectors=True)
    assert cv and nops > kd, (vals, nops)
    _check_general(bk, J, Jd, vals, vecs, spec, sigma, tol, 1.0)


def test_explicit_restart_cgl_random_state_dense(bk):
    """cGL2d at a random small-amplitude state on 12 x 8: non-normal J, values against scipy's eig of the dense Jacobian with
    each eigenvalue's condition number 1 / |y^H x| in the tolerance; restarted (krylovdim nev + 4)."""
    gl = _cgl_oracle()
    u = 0.1 * np.random.default_rng(5).standard_normal(gl.N)
    Jd = _dense(lambda e: gl.dF(u, e), gl.N)
    spec, yl, xr = scipy.linalg.eig(Jd, left=True, right=True)
    kappa_all = 1.0 / np.abs(np.sum(np.conj(yl) * xr, axis=0))       # columns of yl, xr have unit 2-norm
    nev, tol = 4, 1e-10
    sigma = _pick_sigma(spec, nev)
    kappa = float(np.max(kappa_all[np.argsort(np.abs(spec - sigma))[:nev]]))
    assert kappa < 1e3, kappa
    ctx = _cgl_ctx(bk)
    J = ctx.jacobian(ctx.to_device(u))
    inner = bk.GMRESB200(reltol=RHO, restart=60, maxiter=2000, orth="cgs2")
    for kd in (nev + 4, 40):
        vals, vecs, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=kd, tol=tol, maxrestart=500)(J, nev, want_vectors=True)
        assert cv, (kd, vals, nops)
        if kd < 40:
            assert nops > kd, nops
        _check_general(bk, J, Jd, vals, vecs, spec, sigma, tol, kappa)


def test_explicit_restart_nev_cuts_a_conjugate_pair(bk):
    """cGL2d at u = 0 with nev = 3: the third and fourth sigma-nearest eigenvalues are a conjugate pair, so nev cuts it.  The
    members' Ritz values are made exact conjugates and the tie rule (larger Im theta first) keeps the member with Im lambda < 0.
    Both leading pairs are unstable: the cut run counts 3 eigenvalues with Re > 0, all 3 complex, so a Hopf crossing of the cut
    pair changes (n_unstable, n_imag) by (1, 1), which events.get_bifurcation_type classifies as a Hopf point, not a branch
    point."""
    spec, _ = _cgl_zero_spectrum(CGL_DIMS, CGL_L, CGL_PARS[0], CGL_PARS[2])
    gl = _cgl_oracle()
    u = np.zeros(gl.N)
    Jd = _dense(lambda e: gl.dF(u, e), gl.N)
    sigma, tol = 0.5, 1e-10
    near = _nearest(spec, sigma, 4)
    assert abs(near[2] - np.conj(near[3])) < 1e-12 and near[2].imag != 0     # nev = 3 cuts a pair
    ctx = _cgl_ctx(bk)
    J = ctx.jacobian(ctx.to_device(u))
    inner = bk.GMRESB200(reltol=RHO, restart=60, maxiter=2000, orth="cgs2")
    for kd in (7, 40):
        vals, vecs, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=kd, tol=tol, maxrestart=500)(J, 3, want_vectors=True)
        assert cv, (kd, vals, nops)
        if kd < 40:
            assert nops > kd, nops
        cut = near[2].real
        member = [z for z in vals if abs(z.real - cut) < 1e-6]
        assert len(member) == 1 and member[0].imag < 0, vals
        _check_general(bk, J, Jd, vals, vecs, spec, sigma, tol, 1.0, want=np.array([near[0], near[1], member[0]]))
        assert abs(member[0] - near[2].real + 1j * abs(near[2].imag)) < 1e-9, member
        _, nu, ni = bk.palc.is_stable(types.SimpleNamespace(tol_stability=1e-8), vals)
        assert (nu, ni) == (3, 3), vals
        # the cut member crossing back to Re < 0 would leave (2, 2): the step is classified from (nu, ni) -> (2, 2)
        st = types.SimpleNamespace(n_unstable=(nu, 2), n_imag=(ni, 2), step=0, z_p=0.0, z_u=u, tau_p=0.0, tau_u=u)
        sp = bk.events.get_bifurcation_type(types.SimpleNamespace(normC=np.linalg.norm), st, "guess", (0.0, 1.0))
        assert sp.type == "hopf", sp.type


# ------------------------------------------------------------------------------------------------------------- 5. invariant subspace, start vectors
def test_invariant_subspace_chan(bk):
    """chan at n = 12: the two identity boundary rows give the eigenvalue 1 twice (geometric multiplicity 2), so in exact
    arithmetic every Krylov space has dimension <= 11.  In fp64 the second copy enters through rounding in the inner solves
    (their error is not confined to the Krylov space): with krylovdim = N = 12 one cycle of 12 inner solves spans the whole space
    and the 11 sigma-nearest eigenvalues come out with 1 twice, as in the dense spectrum."""
    n, pars = 12, (3.3, 0.01)
    x = problems.chan_sol0(n)
    Jd = _dense(lambda e: problems.chan_dF(x, e, *pars), n)
    spec = np.linalg.eigvals(Jd)
    assert np.sum(np.abs(spec - 1) < 1e-9) == 2
    want = np.sort(_nearest(spec, -30.0, 11).real)[::-1]
    ctx = bk.Context(bk.BK_CHAN, (n,), (1.0,), krylov_m=n, params=pars)
    J = ctx.jacobian(ctx.to_device(x))
    inner = bk.GMRESB200(reltol=1e-14, restart=n, maxiter=4 * n, orth="cgs2")
    sigma, tol = -30.0, 1e-10
    vals, vecs, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=n, tol=tol, maxrestart=1)(J, 11, want_vectors=True)
    assert cv and nops == n, (vals, nops)
    # J is not normal (identity boundary rows): the module's bound times the condition of each eigenvalue, the norm of its spectral
    # projector (the double eigenvalue 1 is semisimple: the projector onto its two-dimensional eigenspace)
    dv = _bounds(want, spec, sigma, tol, 1e-14, _projector_norms(Jd, want))[0]
    assert np.all(np.abs(vals.real - want) <= dv) and np.all(vals.imag == 0), (vals.real - want, dv)


def test_invariant_subspace_sh_full_krylov_space(bk):
    """SH2d on a 7 x 5 grid at a constant state with krylovdim = N = 35 (35 distinct eigenvalues): one cycle of exactly N inner
    solves spans the whole space and every eigenvalue comes out as the closed form says."""
    dims, L = (7, 5), (2.3, 1.9)
    spec = _sh_const_spectrum(dims, L).astype(float)
    N = spec.size
    ctx = _sh_ctx(bk, dims, L, m=N)
    u = np.full(N, SH_C0)
    J = ctx.jacobian(ctx.to_device(u))
    inner = bk.GMRESB200(reltol=RHO, restart=N, maxiter=20 * N, Pr=True)
    sigma, tol = 0.3, 1e-10
    vals, _, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=N, tol=tol, maxrestart=1)(J, N, want_vectors=False)
    assert np.min(np.diff(np.sort(spec))) > 1e-3
    assert cv and nops == N, (vals, nops)
    want = np.sort(spec)[::-1]
    assert np.all(np.abs(vals.real - want) <= _bounds(want, spec, sigma, tol, RHO)[0]), vals.real - want


def test_start_vector_exact_eigenvector(bk):
    """v0 = one DCT mode, an exact eigenvector of J at a constant state (||J|| ~ 1.5 on this coarse grid, so J v0 - lambda v0 is
    at the rounding floor): keff = 1.  nev = 1 converges to the mode's eigenvalue after one inner solve; nev = 2 is reported
    not converged, with NaN only in the slot that has no value."""
    dims, L = (8, 6), (8.3, 5.7)
    spec = _sh_const_spectrum(dims, L)
    kx, ky = 1, 2
    i, j = np.arange(dims[0]), np.arange(dims[1])
    v0 = (np.cos(np.pi * kx * (i + 0.5) / dims[0])[None, :] * np.cos(np.pi * ky * (j + 0.5) / dims[1])[:, None]).reshape(-1)
    lam = float(spec[kx + dims[0] * ky])
    ctx = bk.Context(bk.BK_SH2D, dims, L, krylov_m=48, params=(SH_L, SH_NU))
    J = ctx.jacobian(ctx.to_device(np.full(v0.size, SH_C0)))
    inner = bk.GMRESB200(reltol=RHO, restart=48, maxiter=480)
    eig = bk.ShiftInvertB200(0.3, inner, krylovdim=10, tol=1e-10, maxrestart=5)
    vals, vecs, cv, nops = eig(J, 1, v0=v0, want_vectors=True)
    assert cv and nops == 1 and abs(vals[0] - lam) < 1e-12, (vals, lam, nops)
    assert abs(abs(vecs[:, 0] @ v0) / np.linalg.norm(v0) - 1) < 1e-12
    vals, _, cv, nops = eig(J, 2, v0=v0)
    assert not cv and nops == 1, (vals, nops)
    assert abs(vals[0] - lam) < 1e-12 and np.isnan(vals[1].real), vals


def test_start_vector_host_and_device_same_bits(bk):
    dims, L, u, Js, spec = _hexagon_case()
    ctx = _sh_ctx(bk, dims, L, params=(-0.1, 1.3))
    J = ctx.jacobian(ctx.to_device(u))
    v0 = np.random.default_rng(3).standard_normal(u.size)
    eig = bk.ShiftInvertB200(0.1, bk.GMRESB200(reltol=1e-10, restart=60, maxiter=600, Pr=True), krylovdim=12, tol=1e-8,
                             maxrestart=50)
    a = eig(J, 4, v0=v0, want_vectors=True)
    b = eig(J, 4, v0=ctx.to_device(v0), want_vectors=True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and a[2:] == b[2:]


def test_transposed_jacobian_cgl(bk):
    """ShiftInvertB200 on a TransposedJacobian gives the eigenpairs of J': values of the dense eig, vectors eigenvectors of the
    dense transpose (and not of J, the state is non-normal)."""
    gl = _cgl_oracle()
    u = 0.1 * np.random.default_rng(5).standard_normal(gl.N)
    Jd = _dense(lambda e: gl.dF(u, e), gl.N)
    JdT = np.ascontiguousarray(Jd.T)
    spec, yl, xr = scipy.linalg.eig(JdT, left=True, right=True)
    nev, tol = 4, 1e-10
    sigma = _pick_sigma(spec, nev)
    kappa = float(np.max((1.0 / np.abs(np.sum(np.conj(yl) * xr, axis=0)))[np.argsort(np.abs(spec - sigma))[:nev]]))
    ctx = _cgl_ctx(bk)
    Jt = ctx.jacobian_adjoint(ctx.to_device(u))
    inner = bk.GMRESB200(reltol=RHO, restart=60, maxiter=2000, orth="cgs2")
    vals, vecs, cv, nops = bk.ShiftInvertB200(sigma, inner, krylovdim=nev + 4, tol=tol, maxrestart=500)(Jt, nev, want_vectors=True)
    assert cv, (vals, nops)
    _check_general(bk, Jt, JdT, vals, vecs, spec, sigma, tol, kappa)
    w = bk.normalform._eigvec(Jt, vals, vecs, 0)
    assert np.linalg.norm(Jd @ w - vals[0] * w) > 1e-6 * np.linalg.norm(w)


# ------------------------------------------------------------------------------------------------------------- 6. complex contexts
def test_complex_context_is_refused_before_any_launch(bk):
    """A BK_COMPLEX context's operator is the real-equivalent form of ((-sigma + i a0_imag) I + J): not symmetric, not mapped
    back by sigma + 1/theta, every eigenvalue twice.  bk_eigs_shift_invert refuses it with BK_ERR_ARG before launching anything.
    So it does a krylovdim above the context's krylov_m in a real context: the workspace is only grown after every check."""
    dims, L = (8, 6), (8.3, 5.7)
    for cplx, kd, refusal in ((True, 8, "BK_COMPLEX"), (False, 12, "krylov_m")):
        ctx = bk.Context(bk.BK_SH2D, dims, L, krylov_m=8, params=(SH_L, SH_NU), complex=cplx)
        J = ctx.cjacobian(np.full(ctx.N0, SH_C0)) if cplx else ctx.jacobian(np.full(ctx.N, SH_C0))
        ctx.sync()
        before = ctx.stats()["kernel_launches"]
        with pytest.raises(bk.BK200Error, match=refusal):
            bk.ShiftInvertB200(0.1, bk.GMRESB200(reltol=1e-10, restart=8, maxiter=80), krylovdim=kd)(J, 2)
        assert ctx.stats()["kernel_launches"] == before, refusal
