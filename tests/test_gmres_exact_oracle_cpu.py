"""The long-double GMRES reference (tests/gmres_exact_oracle.py) checked on the CPU: its operators and preconditioners
against the fp64 oracle, its residual history against oracle.krylov.gmres, full-space GMRES against a direct solve, and the
cycle / tolerance / iteration-count rules of libbk200's driver on hand-sized cases."""
import numpy as np
import pytest

from oracle import problems, krylov, precond as oprecond, bls as obls
from tests import gmres_exact_oracle as X

LX, LY = 8 * np.pi, 4 * np.pi / np.sqrt(3)
EPS = X.EPS


def _sh2d(dims, seed=1, noise=0.0):
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    u = problems.sh2d_sol0(*dims, LX, LY) + noise * np.random.default_rng(seed).standard_normal(sh.N)
    return sh, u


def _rel(a, b):
    a, b = np.asarray(a, dtype=X.LD), np.asarray(b, dtype=X.LD)
    return float(X.nrm(a - b) / X.nrm(b))


def test_long_double_is_80_bit():
    assert X.EPS_LD <= 1.1e-19
    assert X.LD(1) + X.LD(2.0 ** -63) != X.LD(1)


@pytest.mark.parametrize("dims", [(16, 12), (258, 5), (15, 7)])
def test_sh2d_operator_matches_fp64_oracle(dims):
    sh, u = _sh2d(dims, noise=0.1)
    v = np.random.default_rng(2).standard_normal(sh.N)
    A = X.sh_op(sh, u, a0=0.7, a1=-1.3)
    ref = 0.7 * v - 1.3 * sh.dF(u, v)
    # the fp64 oracle rounds each of ~13 products and sums per row: a few eps of ||L1|| ||v||
    scale = np.abs(sh.L1).max() * 13 * np.linalg.norm(v)
    assert float(X.nrm(A(X.ld(v)) - X.ld(ref))) <= 8 * EPS * scale


def test_sh3d_chan_cgl_operators_match_fp64_oracle():
    rng = np.random.default_rng(3)
    dims, L = (6, 5, 4), (np.pi, np.pi, np.pi)
    sh = problems.SwiftHohenberg(dims, L, l=0.1, nu=1.2)
    u = problems.sh3d_sol0(*dims, *L)
    v = rng.standard_normal(sh.N)
    scale = np.abs(sh.L1).max() * 25 * np.linalg.norm(v)
    assert float(X.nrm(X.sh_op(sh, u, 2.0, 1.0)(X.ld(v)) - X.ld(2.0 * v + sh.dF(u, v)))) <= 8 * EPS * scale
    n = 101
    x = problems.chan_sol0(n) + 0.01 * rng.standard_normal(n)
    v = rng.standard_normal(n)
    out = X.chan_op(x, 3.3, 0.01, a0=5.0)(X.ld(v))
    assert float(X.nrm(out - X.ld(5.0 * v + problems.chan_dF(x, v, 3.3, 0.01)))) <= 8 * EPS * 4 * (n - 1) ** 2 * np.linalg.norm(v)
    gl = problems.GinzburgLandau2D(12, 6, np.pi, np.pi / 2, r=1.2)
    ug, v = 0.3 * rng.standard_normal(gl.N), rng.standard_normal(gl.N)
    out = X.cgl_op(gl, ug, a0=60.0, a1=-1.0)(X.ld(v))
    assert float(X.nrm(out - X.ld(60.0 * v - gl.dF(ug, v)))) <= 8 * EPS * 8 * np.abs(gl.Delta).max() * np.linalg.norm(v)


@pytest.mark.parametrize("m", [1, 2])
def test_bordered_map_matches_fp64_oracle(m):
    sh, u = _sh2d((16, 12))
    rng = np.random.default_rng(4)
    N = sh.N
    a = [rng.standard_normal(N) for _ in range(m)]
    b = [rng.standard_normal(N) for _ in range(m)]
    c = rng.standard_normal((m, m))
    x = rng.standard_normal(N + m)
    A = X.bordered_op(X.sh_op(sh, u, a0=-2.0), a, b, c, dotscale=1.0 / N)
    ref = obls.MatrixFreeBLSmapBlock(lambda v: sh.dF(u, v), a, b, c, -2.0, lambda p, q: float(np.dot(p, q)) / N)(x)
    assert _rel(A(X.ld(x)), ref) <= 64 * EPS


@pytest.mark.parametrize("dims", [(16, 12), (48, 32), (7, 5)])
def test_dct_preconditioner_matches_fp64_oracle(dims):
    r = np.random.default_rng(5).standard_normal(dims[0] * dims[1])
    P = X.dct_precond(dims, (LX, LY), 1.0)
    ref = oprecond.dct_precond(dims, (LX, LY), 1.0)(r)
    # both transforms are orthonormal: the fp64 FFT-based DCT is accurate to a few eps log n
    assert _rel(P(X.ld(r)), ref) <= 16 * EPS * np.log2(dims[0] * dims[1])
    # and the long-double one is the exact inverse of L1 + I to long-double precision
    sh = problems.SwiftHohenberg(dims, (LX, LY))
    L1 = X.SparseLD(sh.L1)
    z = P(X.ld(r))
    assert _rel(L1(z) + z, r) <= 1e3 * X.EPS_LD * X.nrm(z) * np.abs(sh.L1).max() * 13 / np.linalg.norm(r)


@pytest.mark.parametrize("orth", ["cgs", "cgs2", "mgs"])
@pytest.mark.parametrize("side", ["none", "left", "right"])
def test_residual_history_matches_fp64_gmres(orth, side):
    """oracle.krylov.gmres (fp64) and the reference agree column by column within the fp64 rounding of the former:
    |rho64_k - rho_k| <= c k eps ||A|| ||x_k|| with c = 16 (a well-conditioned shifted operator, so no loss of
    orthogonality beyond that level in any of the three Gram-Schmidt variants)"""
    dims = (16, 12)
    sh, u = _sh2d(dims, noise=0.1)
    rhs = np.random.default_rng(7).standard_normal(sh.N)
    a0, a1 = 20.0, -1.0
    P64 = oprecond.dct_precond(dims, (LX, LY), 1.0) if side != "none" else None
    PL = X.dct_precond(dims, (LX, LY), 1.0) if side != "none" else None
    kw64 = dict(Pl=P64) if side == "left" else (dict(Pr=P64) if side == "right" else {})
    kwl = dict(Pl=PL) if side == "left" else (dict(Pr=PL) if side == "right" else {})
    hist = []
    krylov.gmres(krylov.axpy_op(lambda v: sh.dF(u, v), a0, a1), rhs, reltol=0.0, restart=30, maxiter=30, orth=orth,
                 history=hist, **kw64)
    R = X.gmres(X.sh_op(sh, u, a0, a1), rhs, reltol=0.0, restart=30, maxiter=30, **kwl)
    assert len(hist) == len(R.rho) == 31
    for k in range(1, 31):
        mu = max(1.0, R.hnorm[k] * R.ynorm[k] / float(R.beta0))
        assert abs(hist[k] - float(R.rho[k])) <= 16 * k * EPS * mu * float(R.beta0), (k, hist[k], float(R.rho[k]))


def test_full_space_gmres_reproduces_direct_solve():
    dims = (7, 5)
    sh, u = _sh2d(dims, noise=0.1)
    n = sh.N
    rhs = np.random.default_rng(8).standard_normal(n)
    A = X.sh_op(sh, u, a0=3.0, a1=-1.0)
    M = X.dense(A, n)
    xd = X.direct_solve(M, rhs)
    R = X.gmres(A, rhs, reltol=0.0, restart=500, krylov_m=500, maxiter=n)
    assert R.restart == n and R.iters == n and R.cycles == [0]
    kappa = np.linalg.cond(M.astype(np.float64))
    assert _rel(R.x, xd) <= 64 * n * X.EPS_LD * kappa
    assert float(R.rho[-1]) <= 64 * n * X.EPS_LD * kappa * float(R.beta0)


def test_cycle_rules_restart_one_partial_cycle_and_krylov_m_clamp():
    dims = (16, 12)
    sh, u = _sh2d(dims)
    rhs = np.random.default_rng(9).standard_normal(sh.N)
    A = X.sh_op(sh, u, a0=40.0, a1=-1.0)
    R1 = X.gmres(A, rhs, reltol=0.0, restart=1, maxiter=9)
    assert R1.restart == 1 and R1.cycles == list(range(9)) and R1.iters == 9 and not R1.converged
    # restart = 1 is steepest descent in the residual: each column the exact one-dimensional minimiser
    for k in range(1, 10):
        r = X.ld(rhs) - A(R1.xs[k - 1])
        Ar = A(r)
        x = R1.xs[k - 1] + (np.dot(Ar, r) / np.dot(Ar, Ar)) * r
        assert _rel(R1.xs[k], x) <= 1e-16
    R7 = X.gmres(A, rhs, reltol=0.0, restart=7, maxiter=23)
    assert R7.restart == 7 and R7.cycles == [0, 7, 14, 21] and R7.iters == 23 and len(R7.rho) == 24
    # a cycle restarts from the true residual of its start iterate: its first rho is that of restart = 1 from there
    r = X.ld(rhs) - A(R7.xs[7])
    Ar = A(r)
    assert abs(float(R7.rho[8] / X.nrm(r - (np.dot(Ar, r) / np.dot(Ar, Ar)) * Ar)) - 1.0) <= 1e-16
    # the cycle length is clamped to krylov_m and to n
    assert X.gmres(A, rhs, reltol=0.0, restart=50, krylov_m=10, maxiter=12).cycles == [0, 10]
    small = X.sh_op(*_sh2d((7, 5)), a0=3.0, a1=-1.0)
    assert X.gmres(small, np.ones(35), reltol=0.0, restart=200, maxiter=40).restart == 35


def test_tolerance_rules_reltol_abstol_and_left_preconditioned_beta0():
    dims = (16, 12)
    sh, u = _sh2d(dims, noise=0.1)
    rhs = np.random.default_rng(10).standard_normal(sh.N)
    A = X.sh_op(sh, u, a0=20.0, a1=-1.0)
    H = X.gmres(A, rhs, reltol=0.0, restart=60, maxiter=40)
    k, t = X.first_gap(H.rho)
    R = X.gmres(A, rhs, reltol=t / float(H.beta0), restart=60, maxiter=40)
    assert R.converged and R.iters == k + 1 and R.checks == 0
    # abstol dominating reltol * beta0: tol == abstol and the stop follows it
    k2, t2 = X.first_gap(H.rho, start=7)  # rho_7 / beta0 < 1e-8: a reltol 1e-3 below it is < 1e-9
    Ra = X.gmres(A, rhs, reltol=1e-3 * t2 / float(H.beta0), abstol=t2, restart=60, maxiter=40)
    assert float(Ra.tol) == t2 and Ra.converged and Ra.iters == k2 + 1
    assert Ra.checks == 1  # reltol < 1e-9 with single-pass CGS: the true residual is checked once
    # tol on the preconditioned side: beta0 = ||Pl rhs||
    P = X.dct_precond(dims, (LX, LY), 1.0)
    Rl = X.gmres(A, rhs, reltol=1e-6, restart=60, maxiter=40, Pl=P)
    assert float(Rl.beta0) == float(X.nrm(P(X.ld(rhs))))
    assert float(Rl.tol) == float(X.LD(1e-6) * Rl.beta0)
    # maxiter reached: iters == maxiter, not converged; rhs = 0: converged after no column, x == 0
    Rm = X.gmres(A, rhs, reltol=1e-12, restart=60, maxiter=5)
    assert Rm.iters == 5 and not Rm.converged
    R0 = X.gmres(A, np.zeros(sh.N), reltol=1e-8, restart=60, maxiter=5)
    assert R0.converged and R0.iters == 0 and not np.any(R0.x)


def test_pure_shift_happy_breakdown():
    dims = (16, 12)
    sh, u = _sh2d(dims)
    rhs = np.zeros(sh.N)
    rhs[np.random.default_rng(11).choice(sh.N, 64, replace=False)] = 1.0
    R = X.gmres(X.sh_op(sh, u, a0=3.0, a1=0.0), rhs, reltol=1e-8, restart=60, maxiter=40)
    assert R.converged and R.iters == 1
    assert np.array_equal(R.x.astype(np.float64), rhs / 3.0)


def test_periodic_sh_operator_and_fft_preconditioner_match_fp64_oracle():
    from tests import sh_periodic_oracle as po
    dims = (64, 64)
    L = po.example_lengths(*dims)
    psh = po.PeriodicSH(dims, L)
    rng = np.random.default_rng(16)
    u = po.sol0(*dims, *L) + 0.05 * rng.standard_normal(psh.N)
    v = rng.standard_normal(psh.N)
    out = X.periodic_sh_op(psh, u, a0=3.0, a1=-1.0)(X.ld(v))
    # the fp64 FFT is accurate to a few eps log2(N) of ||symbol|| ||v||
    assert float(X.nrm(out - X.ld(3.0 * v - psh.dF(u, v)))) <= 16 * EPS * np.log2(psh.N) * psh.symbol.max() * np.linalg.norm(v)
    P = X.fft_precond(psh, 1.0)
    assert _rel(P(X.ld(v)), psh.precond(1.0)(v)) <= 16 * EPS * np.log2(psh.N)
    assert P.norm == 1.0 / (psh.symbol.min() + 1.0)


def test_cgl_transpose_complex_and_trapeze_operators_match_fp64_oracle():
    from oracle import potrap as opotrap
    rng = np.random.default_rng(17)
    gl = problems.GinzburgLandau2D(6, 4, np.pi, np.pi / 2, r=1.2)
    u = 0.3 * rng.standard_normal(gl.N)
    Jd = np.stack([gl.dF(u, e) for e in np.eye(gl.N)], axis=1)
    scale = 8 * np.abs(gl.Delta).max()
    assert float(np.max(np.abs(X.dense(X.cgl_op(gl, u), gl.N) - X.ld(Jd)))) <= 8 * EPS * scale
    assert float(np.max(np.abs(X.dense(X.cgl_op(gl, u, transpose=True), gl.N) - X.ld(Jd.T)))) <= 8 * EPS * scale
    z = rng.standard_normal(2 * gl.N)
    a0, ai = 0.7, -1.9
    ref = np.concatenate([a0 * z[:gl.N] - ai * z[gl.N:] + Jd @ z[:gl.N], ai * z[:gl.N] + a0 * z[gl.N:] + Jd @ z[gl.N:]])
    out = X.complex_op(X.cgl_op(gl, u), gl.N, a0, ai)(X.ld(z))
    assert float(X.nrm(out - X.ld(ref))) <= 8 * EPS * scale * np.linalg.norm(z)
    M = 5
    NM = gl.N * M
    x = np.concatenate([0.3 * rng.standard_normal(NM), [6.1]])
    phi, xpi = rng.standard_normal(NM), rng.standard_normal(NM)
    dx = rng.standard_normal(NM + 1)
    tr = opotrap.Trapeze(gl.F, gl.dF, phi, xpi, M, gl.N)
    out = X.trapeze_op(gl, x, phi, M, a0=2.0)(X.ld(dx))
    assert float(X.nrm(out - X.ld(2.0 * dx + tr.jvp(x, dx)))) <= 16 * EPS * scale * 6.1 * np.linalg.norm(dx)


def test_dst_chan_and_circulant_preconditioners_match_fp64_oracle():
    rng = np.random.default_rng(18)
    gl = problems.GinzburgLandau2D(12, 6, np.pi, np.pi / 2, r=1.3)
    r = rng.standard_normal(gl.N)
    P = X.dst_precond(gl, -1.0, 1.0)
    P64 = oprecond.dst_helmholtz_precond(12, 6, np.pi, np.pi / 2, -1.0, 1.0)
    assert _rel(P(X.ld(r)), np.concatenate([P64(r[:gl.n]), P64(r[gl.n:])])) <= 16 * EPS * np.log2(gl.n)
    n = 101
    rc = rng.standard_normal(n)
    Pc = X.chan_precond(n)
    z = Pc(X.ld(rc))
    assert _rel(z, oprecond.chan_lu_precond(n)(rc)) <= 64 * EPS * n
    assert _rel(X.SparseLD(problems.chan_precond_matrix(n))(z), rc) <= 1e3 * X.EPS_LD * 4 * (n - 1) ** 2 * Pc.norm
    M, T = 6, 6.1
    gl = problems.GinzburgLandau2D(6, 4, np.pi, np.pi / 2, r=1.3)
    v = rng.standard_normal(gl.N * M + 1)
    Pt = X.potrap_circ_precond(gl, M, T)
    ref = oprecond.potrap_circulant_precond(6, 4, np.pi, np.pi / 2, M, T, 1.3, 1.0)(v)
    assert _rel(Pt(X.ld(v)), ref) <= 1e3 * EPS * Pt.norm
