"""GPU parity of the periodic spectral Swift-Hohenberg kind (BK_SH2D_PERIODIC), its FFT preconditioner (BK_PC_SH_FFT) and the
one-transform preconditioned Arnoldi operator against the NumPy restatement of examples/SH2d-fronts-cuda.jl
(tests/sh_periodic_oracle.py)."""
import ctypes as C

import numpy as np
import pytest

import __graft_entry__ as g
from oracle import krylov as okry
from tests import sh_periodic_oracle as po

pytestmark = pytest.mark.gpu
PAR = (-0.15, 1.3)   # (l, nu) of the example (:116)


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


def _rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300)


def _ctx(bk, dims, m=2, complex=False):
    L = po.example_lengths(*dims)
    return bk.Context(bk.BK_SH2D_PERIODIC, dims, L, krylov_m=m, params=PAR, complex=complex), po.PeriodicSH(dims, L, *PAR)


def _state(dims, seed=0):
    L = po.example_lengths(*dims)
    return po.sol0(*dims, *L) + 0.05 * np.random.default_rng(seed).standard_normal(dims[0] * dims[1])


@pytest.mark.parametrize("dims", [(64, 64), (128, 64), (64, 2048), (2048, 64), (512, 512), (1024, 256)])
def test_residual_and_jvp_vs_oracle(bk, dims):
    ctx, sh = _ctx(bk, dims)
    u = _state(dims, sum(dims))
    v = np.random.default_rng(7).standard_normal(ctx.N)
    F = ctx.residual(u)
    assert _rel(F, sh.F(u)) < 1e-12
    Fd = ctx.residual(ctx.to_device(u)).numpy()
    assert np.array_equal(Fd, F)                                         # host and device pointers: the same bits
    ctx.jacobian(u)
    outs = {}
    for a0, a1 in ((0.0, 1.0), (-0.1, 1.0), (0.7, -2.0)):
        ref = a0 * v + a1 * sh.dF(u, v)
        out = ctx.jvp(v, a0=a0, a1=a1)
        assert _rel(out, ref) < 1e-12, (a0, a1)
        assert np.array_equal(ctx.jvp(ctx.to_device(v), a0=a0, a1=a1).numpy(), out)
        outs[(a0, a1)] = out
    ctx.set_transpose(True)                                              # self-adjoint: J' v is J v, bit for bit
    for (a0, a1), out in outs.items():
        assert np.array_equal(ctx.jvp(v, a0=a0, a1=a1), out), (a0, a1)
    ctx.set_transpose(False)


@pytest.mark.parametrize("dims", [(64, 64), (256, 128), (128, 1024), (2048, 64)])
def test_fft_preconditioner_vs_oracle(bk, dims):
    ctx, sh = _ctx(bk, dims)
    r = np.random.default_rng(3).standard_normal(ctx.N)
    for a0 in (1.0, 0.25):
        ctx.precond_setup(bk.BK_PC_SH_FFT, a0)
        ref = sh.precond(a0)(r)
        assert _rel(ctx.precond_apply(r), ref) < 1e-11
        assert _rel(ctx.precond_apply(ctx.to_device(r)).numpy(), ref) < 1e-11
    # a device vector offset by one double (8-byte, not 16-byte aligned) gives the same answer and does not fault
    big_in, big_out = ctx.zeros(ctx.N + 2), ctx.zeros(ctx.N + 2)
    host = np.concatenate([[0.0], r, [0.0]])
    assert ctx.lib.bk_vec_upload(ctx.handle, big_in.dptr, host.ctypes.data, len(host)) == 0
    st = ctx.lib.bk_precond_apply(ctx.handle, C.c_void_p(big_in.dptr + 8), C.c_void_p(big_out.dptr + 8))
    assert st == 0, ctx.lib.bk_last_error(ctx.handle)
    assert _rel(big_out.numpy()[1:-1], sh.precond(0.25)(r)) < 1e-11


def test_fft_preconditioner_rejects_bad_setups(bk):
    ctx, _ = _ctx(bk, (64, 64))
    for a0 in (0.0, -1.0):
        with pytest.raises(bk.BK200Error, match="a0 must be > 0"):
            ctx.precond_setup(bk.BK_PC_SH_FFT, a0)
    with pytest.raises(bk.BK200Error, match="needs a Swift-Hohenberg context"):
        ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    neu = bk.Context(bk.BK_SH2D, (64, 64), (10.0, 10.0), krylov_m=2, params=PAR)
    with pytest.raises(bk.BK200Error, match="BK_SH2D_PERIODIC"):
        neu.precond_setup(bk.BK_PC_SH_FFT, 1.0)


@pytest.mark.parametrize("side", ["Pl", "Pr"])
def test_gmres_hexagon_jacobian_fused_and_unfused(bk, side):
    """GMRES on the Jacobian at the hexagon guess, 128 x 128, with the preconditioner on either side: fused = 1 runs one spectral
    pipeline per Arnoldi step, fused = 0 the separate operator and preconditioner; both against the oracle GMRES"""
    dims = (128, 128)
    ctx, sh = _ctx(bk, dims, m=60)
    ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
    u = _state(dims, 11)
    rhs = np.random.default_rng(12).standard_normal(ctx.N)
    J = ctx.jacobian(u)
    P = sh.precond(1.0)
    kw = {side: P}
    xo, cvo, ito = okry.gmres(lambda v: sh.dF(u, v), rhs, reltol=1e-10, restart=60, maxiter=300, **kw)
    assert cvo
    res = {}
    for fused in (True, False):
        ls = bk.GMRESB200(reltol=1e-10, restart=60, maxiter=300, fused=fused, **{side: True})
        x, cv, it = ls(J, rhs)
        assert cv and abs(it - ito) <= 2, (fused, it, ito)
        assert _rel(x, xo) < 1e-8, fused
        res[fused] = (x, it)
    assert _rel(res[True][0], res[False][0]) < 1e-10 and abs(res[True][1] - res[False][1]) <= 1
    # the one-transform path ran: at a fixed 20 Arnoldi steps (reltol 0) the fused solve launches 3 kernels fewer per step
    # (one spectral pipeline instead of the operator's and the preconditioner's)
    launches = {}
    for fused in (True, False):
        ls = bk.GMRESB200(reltol=0.0, restart=20, maxiter=20, fused=fused, **{side: True})
        before = ctx.stats()["kernel_launches"]
        _, _, it = ls(J, rhs)
        assert it == 20
        launches[fused] = ctx.stats()["kernel_launches"] - before
    assert launches[False] - launches[True] == 3 * 20, launches


def test_shift_invert_eigenvalues_vs_dense(bk):
    """sigma = 0.1, nev = 6 on 64 x 64 (the example's SHEigOp, :92-102) against eigvalsh of the dense Jacobian"""
    dims = (64, 64)
    ctx, sh = _ctx(bk, dims, m=80)
    ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
    u = _state(dims, 5)
    J = ctx.jacobian(u)
    ls = bk.GMRESB200(reltol=1e-12, restart=80, maxiter=400, Pl=True)
    vals, vecs, ok, _ = bk.ShiftInvertB200(0.1, ls, krylovdim=50, tol=1e-10)(J, 6, want_vectors=True)
    assert ok
    A = sh.jac_dense(u)
    ev = np.linalg.eigvalsh(A)
    ref = ev[np.argsort(np.abs(ev - 0.1))[:6]]
    assert np.allclose(np.sort(vals.real), np.sort(ref), atol=1e-7), (vals, ref)
    assert np.abs(vals.imag).max() == 0.0
    for k in range(6):
        v = vecs[:, k]
        assert np.linalg.norm(A @ v - vals[k].real * v) < 1e-6 * np.linalg.norm(v)


def test_complex_shifted_solve_vs_dense(bk):
    """BK_COMPLEX through the split-complex path: ((a0 + i b) I + J) z = r at 64 x 64 against the dense complex solve"""
    dims = (64, 64)
    ctx, sh = _ctx(bk, dims, m=120, complex=True)
    ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
    u = _state(dims, 9)
    rng = np.random.default_rng(10)
    r = rng.standard_normal(ctx.N0) + 1j * rng.standard_normal(ctx.N0)
    shift = complex(-0.1, 0.4)
    J = ctx.cjacobian(u)
    for fused in (True, False):
        ls = bk.ComplexGMRESB200(reltol=1e-12, restart=120, maxiter=600, Pl=True, fused=fused)
        z, cv, _ = ls(J, r, a0=shift)
        assert cv
        ref = np.linalg.solve(shift * np.eye(ctx.N0) + sh.jac_dense(u), r)
        assert np.linalg.norm(z - ref) < 1e-8 * np.linalg.norm(ref), fused


def test_newton_to_hexagons_and_deflated_front(bk):
    """the example end to end, part one (:112-139) at 128 x 128 with the lengths scaled by n / 512: Newton from sol0 to the
    hexagons (tol 1e-6, norminf, GMRES with Pl = L^-1, Krylov dimension 50), the same iteration over the oracle, then the deflated
    Newton from 0.4 u_hexa exp(-x^2/25) to a converged state away from the hexagons"""
    P = bk.palc
    dims = (128, 128)
    L = po.example_lengths(*dims)
    ctx, sh = _ctx(bk, dims, m=50)
    ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
    ls = bk.GMRESB200(reltol=1e-8, restart=50, maxiter=300, Pl=True)
    u0 = po.sol0(*dims, *L)
    prob = P.BifurcationProblemB200(ctx, ctx.to_device(u0), PAR, lens=0)
    hexa = P.newton(prob, ctx.to_device(u0), PAR[0], P.NewtonPar(tol=1e-6, max_iterations=10, linsolver=ls), P.norminf)
    assert hexa.converged
    uh = hexa.u.numpy()
    assert np.abs(sh.F(uh)).max() < 1e-6
    # the oracle's Newton with the oracle GMRES reaches the same state in as many iterations
    x, it = u0.copy(), 0
    while np.abs(sh.F(x)).max() > 1e-6 and it < 10:
        dx, cv, _ = okry.gmres(lambda v: sh.dF(x, v), sh.F(x), Pl=sh.precond(1.0), reltol=1e-8, restart=50, maxiter=300)
        x, it = x - dx, it + 1
    assert it == hexa.itnewton and np.abs(x - uh).max() < 1e-6 * max(1.0, np.abs(uh).max())
    D = bk.deflation
    dop = D.DeflationOperator(2, 1.0, [hexa.u])
    guess = po.front_guess(uh, *dims, L[0])
    sol = D.newton_deflated(prob, ctx.to_device(guess), PAR[0], dop, P.NewtonPar(tol=1e-6, max_iterations=250, linsolver=ls),
                            P.norminf)
    assert sol.converged
    uf = sol.u.numpy()
    assert np.abs(sh.F(uf)).max() < 1e-6 and np.abs(uf - uh).max() > 1e-2


def test_native_loop_bit_identical_to_the_plugin_loop(bk):
    """bk_palc_run on the new kind writes the same rows as the plugin-surface loop (128 x 128, 5 steps, BorderingBLS with
    check_precision off, the example's ContinuationPar)"""
    P = bk.palc
    dims = (128, 128)
    L = po.example_lengths(*dims)
    ctx, _ = _ctx(bk, dims, m=50)
    ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
    ls = bk.GMRESB200(reltol=1e-8, restart=50, maxiter=300, Pl=True)
    u0 = po.sol0(*dims, *L)
    mk = lambda u: P.BifurcationProblemB200(ctx, u, PAR, lens=0)
    hexa = P.newton(mk(ctx.to_device(u0)), ctx.to_device(u0), PAR[0], P.NewtonPar(tol=1e-6, max_iterations=10, linsolver=ls), P.norminf)
    assert hexa.converged
    cp = P.ContinuationPar(dsmin=0.001, dsmax=0.007, ds=-0.005, p_max=0.005, p_min=-1.0, max_steps=5,
                           newton_options=P.NewtonPar(tol=1e-6, max_iterations=15, linsolver=ls))
    alg = P.PALC(bls=bk.BorderingBLSB200(ls, check_precision=False))
    ref, st = P.continuation(mk(hexa.u), alg, cp, normC=P.norminf)
    rows, info = P.continuation_native(mk(hexa.u), alg, cp, normC=P.norminf)
    assert len(ref) == 6 and len(rows) == len(ref)
    for r, o in zip(rows, ref):
        for k in ("param", "x", "itnewton", "itlinear", "ds", "step"):
            assert r[k] == o[k], (k, r, o)
    assert np.array_equal(info["u"].numpy(), st.z_u.numpy())


def _oracle_shift_invert(N, P, sigma=0.1):
    """the oracle's SHEigOp: eigsh in shift-invert mode, (J - sigma I)^-1 by the oracle GMRES with Pl = (L1 + I)^-1"""
    import scipy.sparse.linalg as spl

    def eig(J, nev):
        A = spl.LinearOperator((N, N), matvec=J, dtype=np.float64)
        inv = lambda b: okry.gmres(lambda v: J(v) - sigma * v, b, Pl=P, reltol=1e-12, restart=100, maxiter=2000)[0]
        OPinv = spl.LinearOperator((N, N), matvec=inv, dtype=np.float64)
        vals = spl.eigsh(A, k=nev, sigma=sigma, OPinv=OPinv, which="LM", tol=1e-9, return_eigenvectors=False)
        return vals, None, True, 0
    return eig


def test_palc_branch_with_stability_vs_oracle(bk):
    """the example end to end, part two (:141-157) at 128 x 128: 10 PALC steps from the hexagons with
    BorderingBLS(check_precision = false), the example's ContinuationPar (ds -0.005, dsmin 0.001, dsmax 0.007, Newton tol 1e-6 /
    15 iterations, nev = 11, sigma = 0.1), stability computed on the device at every step; the same host logic over the oracle
    gives the same rows (param 1e-7, ||u|| 1e-6 relative, Newton iterations, unstable eigenvalue counts)"""
    from oracle import bls as obls, palc as opalc
    P = bk.palc
    dims = (128, 128)
    L = po.example_lengths(*dims)
    ctx, sh = _ctx(bk, dims, m=50)
    ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
    ls = bk.GMRESB200(reltol=1e-8, restart=50, maxiter=300, Pl=True)
    eig = bk.ShiftInvertB200(0.1, bk.GMRESB200(reltol=1e-12, restart=50, maxiter=1000, Pl=True), krylovdim=40, tol=1e-9)
    u0 = po.sol0(*dims, *L)
    kw = dict(dsmin=0.001, dsmax=0.007, ds=-0.005, p_max=0.005, p_min=-1.0, max_steps=10, nev=11, detect_bifurcation=1,
              tol_stability=1e-5)
    hexa = P.newton(P.BifurcationProblemB200(ctx, ctx.to_device(u0), PAR, lens=0), ctx.to_device(u0), PAR[0],
                    P.NewtonPar(tol=1e-6, max_iterations=10, linsolver=ls), P.norminf)
    assert hexa.converged
    cp = P.ContinuationPar(newton_options=P.NewtonPar(tol=1e-6, max_iterations=15, linsolver=ls, eigsolver=eig), **kw)
    rows, _ = P.continuation(P.BifurcationProblemB200(ctx, hexa.u, PAR, lens=0),   # records norm(u), :124
                             P.PALC(bls=bk.BorderingBLSB200(ls, check_precision=False)), cp, normC=P.norminf)
    Pc = sh.precond(1.0)
    ols = okry.GMRESIterativeSolvers(reltol=1e-8, restart=50, maxiter=300, N=sh.N, Pl=Pc)
    oprob = lambda u: opalc.Problem(F=lambda x, l: sh.F(x, l), J=lambda x, l: (lambda v: sh.dF(x, v, l)), u0=u, p0=PAR[0])
    ohexa = opalc.newton(oprob(u0), u0, PAR[0], opalc.NewtonPar(tol=1e-6, max_iterations=10, linsolver=ols), opalc.norminf)
    assert ohexa.converged and ohexa.itnewton == hexa.itnewton
    cpo = opalc.ContinuationPar(newton_options=opalc.NewtonPar(tol=1e-6, max_iterations=15, linsolver=ols,
                                                               eigsolver=_oracle_shift_invert(sh.N, Pc)), **kw)
    orows, _ = opalc.continuation(oprob(ohexa.u), opalc.PALC(bls=obls.BorderingBLS(ols, check_precision=False)), cpo,
                                  normC=opalc.norminf)
    assert len(rows) == len(orows) == 11
    for r, o in zip(rows, orows):
        assert abs(r["param"] - o["param"]) < 1e-7 and abs(r["x"] - o["x"]) < 1e-6 * o["x"], (r, o)
        assert r["itnewton"] == o["itnewton"] and r["n_unstable"] == o["n_unstable"] >= 0, (r, o)
