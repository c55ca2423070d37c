"""GPU tests of J' of the Trapeze functional (k_potrap_apply_tr), the transposed circulant preconditioner (k_potrap_time<true>) and
the folds of periodic orbits built on them (periodic.newton_fold_po / continuation_fold_po), against the sparse Trapeze Jacobian
of tests/potrap_sparse_oracle.py."""
import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import __graft_entry__ as g
from oracle import bls as obls, krylov, potrap as opotrap, problems
from tests import potrap_sparse_oracle as PS
from tests.test_host_logic_cpu import BlsAdapter

pytestmark = pytest.mark.gpu
L = (np.pi, np.pi / 2)


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


def _rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300)


def _setup(bk, dims, M, seed):
    """a potrap context at a non-trivial orbit-like state x (T = 6.3) with a random section, and the oracle's sparse J there"""
    pars = (1.3, 0.1, 1.0, -1.0, 1.0)
    gl = problems.GinzburgLandau2D(*dims, *L, r=pars[0], mu=pars[1], nu=pars[2], c3=pars[3], c5=pars[4])
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (*dims, M), L, krylov_m=80, params=pars)
    rng = np.random.default_rng(seed)
    ph = gl.phi11()
    t = np.linspace(0, 2 * np.pi, M + 1)[:M]
    x = np.concatenate([np.concatenate([0.8 * np.cos(s) * ph, 0.8 * np.sin(s) * ph]) + 0.05 * rng.standard_normal(gl.N) for s in t]
                       + [np.array([6.3])])
    phi = rng.standard_normal(gl.N * M) / np.sqrt(gl.N * M)
    ctx.potrap_set_section(phi, x[:-1])
    return ctx, gl, x, phi, PS.cgl_po_jacobian(gl, x, M, phi), rng


@pytest.mark.parametrize("dims,M", [((16, 12), 10), ((41, 21), 30)], ids=["16x12x10", "41x21x30"])
def test_adjoint_identity_and_oracle(bk, dims, M):
    """<w, a0 v + a1 J v> = <a0 w + a1 J' w, v> to 1e-13 relative; J'w = the oracle's transpose to 1e-12; host and device
    vectors give the same bits, and so do two calls; the J' handle selects J' for its call only"""
    ctx, gl, x, phi, Jsp, rng = _setup(bk, dims, M, 1)
    Jt = ctx.jacobian_adjoint(x)
    for a0 in (0.0, 1.0):
        v, w = rng.standard_normal(ctx.N), rng.standard_normal(ctx.N)
        jv = ctx.jacobian(x)(v) if a0 == 0.0 else ctx.jvp(v, a0=a0, a1=0.7)
        ctx.set_transpose(True)
        jtw = ctx.jvp(w, a0=a0, a1=0.7 if a0 else 1.0)
        jtw_dev = ctx.jvp(ctx.to_device(w), a0=a0, a1=0.7 if a0 else 1.0).numpy()
        jtw2 = ctx.jvp(w, a0=a0, a1=0.7 if a0 else 1.0)
        ctx.set_transpose(False)
        a1 = 0.7 if a0 else 1.0
        lhs, rhs = np.dot(w, jv), np.dot(jtw, v)
        assert abs(lhs - rhs) < 1e-13 * np.linalg.norm(w) * np.linalg.norm(jv), (lhs, rhs)
        ref = a0 * w + a1 * (Jsp.T @ w)
        assert _rel(jtw, ref) < 1e-12
        assert np.array_equal(jtw, jtw_dev) and np.array_equal(jtw, jtw2)
    ctx.jacobian(x)
    assert _rel(Jt(w), Jsp.T @ w) < 1e-12          # the handle switches J' on for the call only
    assert _rel(ctx.jvp(v), Jsp @ v) < 1e-12


def test_gmres_with_the_adjoint_and_its_preconditioner(bk):
    """J' x = b by right-preconditioned GMRES (P'^-1 of the circulant preconditioner) has a residual below 1e-8 against the
    oracle's transpose; <P'^-1 a, b> = <a, P^-1 b>; with the transpose off, the preconditioner and a J solve after a J' solve give
    the bits of a context that never selected J'"""
    dims, M = (16, 12), 10
    ctx, gl, x, phi, Jsp, rng = _setup(bk, dims, M, 2)
    ctx.precond_setup(bk.BK_PC_POTRAP_CIRC, float(x[-1]))
    a, b = rng.standard_normal(ctx.N), rng.standard_normal(ctx.N)
    Pa_fresh = ctx.precond_apply(a)
    ctx.set_transpose(True)
    Pta = ctx.precond_apply(a)
    ctx.set_transpose(False)
    Pb = ctx.precond_apply(b)
    assert abs(np.dot(Pta, b) - np.dot(a, Pb)) < 1e-12 * np.linalg.norm(Pta) * np.linalg.norm(b)
    assert np.array_equal(ctx.precond_apply(a), Pa_fresh)
    P = PS.potrap_circulant_matrix(*dims, *L, M, float(x[-1]), gl.r, gl.nu)
    assert _rel(P.T @ Pta, a) < 1e-12 and _rel(P @ Pb, b) < 1e-12
    ls = bk.GMRESB200(reltol=1e-11, restart=80, maxiter=800, Pr=True, orth="cgs2")
    Jt = ctx.jacobian_adjoint(x)
    y, cv, it_t = ls(Jt, b)
    assert cv and np.linalg.norm(Jsp.T @ y - b) < 1e-8 * np.linalg.norm(b), it_t
    # no leak: the J solve after the J' solve equals the J solve of a fresh context
    J = ctx.jacobian(x)
    z1, cv1, it1 = ls(J, b)
    ctx2, *_ = _setup(bk, dims, M, 2)
    ctx2.precond_setup(bk.BK_PC_POTRAP_CIRC, float(x[-1]))
    z2, cv2, it2 = ls(ctx2.jacobian(x), b)
    assert cv1 and np.array_equal(z1, z2) and it1 == it2
    print(f"J' solve at 16x12x10: {it_t} iterations with P'^-1")


def test_bordered_solves_with_the_adjoint(bk):
    """BorderingBLSB200 and MatrixFreeBLSB200 with the J' handle agree with the oracle's sparse bordered system to 1e-8"""
    dims, M = (16, 12), 10
    ctx, gl, x, phi, Jsp, rng = _setup(bk, dims, M, 3)
    ctx.precond_setup(bk.BK_PC_POTRAP_CIRC, float(x[-1]))
    N = ctx.N
    dR, dzu, R = rng.standard_normal(N), rng.standard_normal(N), rng.standard_normal(N)
    dzp, n = 0.8, -0.4
    A = sp.bmat([[Jsp.T, sp.csr_matrix(dR[:, None])], [sp.csr_matrix(dzu[None, :]), sp.csr_matrix([[dzp]])]]).tocsc()
    ref = spl.spsolve(A, np.concatenate([R, [n]]))
    ls = bk.GMRESB200(reltol=1e-12, restart=80, maxiter=800, Pr=True, orth="cgs2")
    for bls in (bk.BorderingBLSB200(ls, check_precision=False), bk.MatrixFreeBLSB200(ls)):
        dX, dl, cv, it = bls(ctx.jacobian_adjoint(x), dR, dzu, dzp, R, n)
        assert cv and _rel(dX, ref[:-1]) < 1e-8 and abs(dl - ref[-1]) < 1e-8 * max(1.0, abs(ref[-1])), (type(bls).__name__, it)


# ------------------------------------------------------------------------------------------------ folds of cycles
def _hopf_point(bk, dims):
    P = bk.palc
    r_hopf = problems.GinzburgLandau2D(*dims, *L).r_hopf()
    pars = [r_hopf, 0.1, 1.0, -1.0, 1.0]
    gl = problems.GinzburgLandau2D(*dims, *L, r=pars[0], mu=pars[1], nu=pars[2], c3=pars[3], c5=pars[4])
    ctx_vf = bk.Context(bk.BK_CGL2D, dims, L, krylov_m=200, params=pars)
    prob = P.BifurcationProblemB200(ctx_vf, ctx_vf.zeros(), pars, lens=0)
    ph = gl.phi11() / np.linalg.norm(gl.phi11())
    zeta = np.concatenate([ph, -1j * ph]) / np.sqrt(2)
    ls_vf = bk.GMRESB200(reltol=1e-12, restart=200, maxiter=2000, orth="cgs2")
    return bk.normalform.hopf_normal_form_at(prob, ctx_vf.zeros(), r_hopf, pars[2], zeta, zeta, ls_vf), pars, r_hopf


def _fold_branch(bk, dims, M, max_steps):
    P = bk.palc
    hp, pars, r_hopf = _hopf_point(bk, dims)
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (*dims, M), L, krylov_m=60, params=pars)
    trap = bk.periodic.TrapezeProblemB200(ctx, None, list(pars), lens=0, circulant=True)
    ls = bk.GMRESB200(reltol=1e-10, restart=60, maxiter=600, Pr=True, orth="cgs2")
    cp = P.ContinuationPar(dsmin=1e-4, dsmax=0.05, ds=0.01, p_min=r_hopf - 3.0, p_max=r_hopf + 1.0, max_steps=max_steps,
                           newton_options=P.NewtonPar(tol=1e-9, max_iterations=15, linsolver=ls))
    br, _, _, _ = bk.periodic.continuation_from_hopf_point(hp, cp, trap, with_events=True)
    folds = [i for i, s in enumerate(br.specialpoint) if s.type == "fold" and s.param < r_hopf - 0.05]
    return trap, br, folds, ls, pars, r_hopf


def _oracle_check(gl_at, x0, p0, sol, tau, M):
    """F = 0 by the oracle with the section of the guess (phi = F(x0_i, p0) / M, xpi = x0), and sigma of the oracle's sparse
    bordered system [J a; b' 0] [v; sigma] = [0; 1] at the device's fold, a = b = tau / |tau|"""
    gl0 = gl_at(p0)
    Ns = gl0.N
    phi = np.concatenate([gl0.F(x0[i * Ns:(i + 1) * Ns]) / M for i in range(M)])
    gl = gl_at(sol.p)
    x = sol.u.numpy()
    F = opotrap.Trapeze(gl.F, gl.dF, phi, x0[:-1], M, Ns).residual(x)
    return np.max(np.abs(F)), _sigma(PS.cgl_po_jacobian(gl, x, M, phi), tau)


def _sigma(J, tau):
    """sigma of [J e; e' 0] [v; sigma] = [0; 1], e = tau / |tau|: zero exactly where J is singular, whatever the border"""
    e = tau / np.linalg.norm(tau)
    A = sp.bmat([[J, sp.csr_matrix(e[:, None])], [sp.csr_matrix(e[None, :]), None]]).tocsc()
    return spl.spsolve(A, np.concatenate([np.zeros(len(tau)), [1.0]]))[-1]


def test_fold_of_cycles_at_16x12x10(bk):
    """the branch from the Hopf point at 16 x 12, M = 10, with fold detection by monotony: newton_fold_po converges from the
    recorded fold, its parameter lies within the turning of the rows around it, F = 0 and sigma = 0 by the oracle (sigma of a
    bordered system with any generic border vanishes exactly where J is singular)"""
    dims, M = (16, 12), 10
    trap, br, folds, ls, pars, r_hopf = _fold_branch(bk, dims, M, 60)
    print("16x12x10 branch:", len(br.rows), "rows, folds", [(br.specialpoint[i].param, br.specialpoint[i].idx) for i in folds])
    assert folds, [s.type for s in br.specialpoint]
    ind = folds[0]
    spt = br.specialpoint[ind]
    x0 = spt.x.numpy()
    tau = spt.tau_u.numpy()
    opts = bk.palc.NewtonPar(tol=1e-9, max_iterations=15, linsolver=ls)
    sol = bk.periodic.newton_fold_po(trap, br, ind, opts, bk.BorderingBLSB200(ls, check_precision=False))
    print("newton_fold_po:", sol.p, sol.residuals, sol.itlinear)
    assert sol.converged
    k = spt.idx
    params = [r["param"] for r in br.rows[k - 1: k + 2]]
    # the fold is the extremum of r along the branch: at or beyond the turning row, within the width of the turn
    assert params[1] == min(params) and min(params) - (max(params) - min(params)) <= sol.p <= min(params) + 1e-9, (params, sol.p)
    gl_at = lambda p: problems.GinzburgLandau2D(*dims, *L, r=p, mu=pars[1], nu=pars[2], c3=pars[3], c5=pars[4])
    fmax, sigma = _oracle_check(gl_at, x0, spt.param, sol, tau, M)
    assert fmax < 1e-8 and abs(sigma) < 1e-8, (fmax, sigma)


def test_fold_of_cycles_at_the_example_size(bk):
    """examples/cGL2d.jl at 41 x 21, M = 30: the branch from the Hopf point finds a fold of cycles, newton_fold_po converges,
    continuation_fold_po runs 5 steps in c5 with F = 0 (oracle, section of the guess) and sigma = 0 on each, and an independent
    newton_fold_po at the last c5 gives the same r to 1e-6"""
    dims, M = (41, 21), 30
    trap, br, folds, ls, pars, r_hopf = _fold_branch(bk, dims, M, 80)
    print("41x21x30 branch:", len(br.rows), "rows, folds", [(br.specialpoint[i].param, br.specialpoint[i].idx) for i in folds])
    assert folds, [s.type for s in br.specialpoint]
    ind = folds[0]
    opts = bk.palc.NewtonPar(tol=1e-8, max_iterations=15, linsolver=ls)
    bls = bk.BorderingBLSB200(ls, check_precision=False)
    sol = bk.periodic.newton_fold_po(trap, br, ind, opts, bls)
    print("newton_fold_po:", sol.p, sol.residuals, sol.itlinear)
    assert sol.converged
    cp = bk.palc.ContinuationPar(dsmin=1e-4, dsmax=0.05, ds=0.02, p_min=0.5, p_max=2.0, max_steps=5,
                                 newton_options=bk.palc.NewtonPar(tol=1e-8, max_iterations=10))
    pts = []
    curve = bk.periodic.continuation_fold_po(trap, br, ind, 4, cp, bls,
                                             callback=lambda st: pts.append((st.z_p, st.z_u.p, st.z_u.u.numpy())) or True)
    print("fold curve (c5, r):", list(zip(curve.p2, curve.p1)))
    assert len(curve.rows) >= 6
    spt = br.specialpoint[ind]
    x0 = spt.x.numpy()
    Ns = 2 * dims[0] * dims[1]
    gl0 = problems.GinzburgLandau2D(*dims, *L, r=spt.param, mu=pars[1], nu=pars[2], c3=pars[3], c5=pars[4])
    phi = np.concatenate([gl0.F(x0[i * Ns:(i + 1) * Ns]) / M for i in range(M)])
    tau = spt.tau_u.numpy()
    for c5, r, x in pts:
        gl = problems.GinzburgLandau2D(*dims, *L, r=r, mu=pars[1], nu=pars[2], c3=pars[3], c5=c5)
        fmax = np.max(np.abs(opotrap.Trapeze(gl.F, gl.dF, phi, x0[:-1], M, Ns).residual(x)))
        sigma = _sigma(PS.cgl_po_jacobian(gl, x, M, phi), tau)
        print(f"c5 = {c5:.6f}  r = {r:.9f}  max|F| = {fmax:.2e}  sigma = {sigma:.2e}")
        assert fmax < 1e-7 and abs(sigma) < 1e-6, (c5, r, fmax, sigma)
    c5_last, r_last = curve.p2[-1], curve.p1[-1]
    trap.params[4] = c5_last
    sol2 = bk.periodic.newton_fold_po(trap, br, ind, opts, bls)
    trap.params[4] = pars[4]
    assert sol2.converged and abs(sol2.p - r_last) < 1e-6, (sol2.p, r_last)


# ------------------------------------------------------------------------------------------------ adjoint eigenvectors
def test_adjoint_eigenvector_of_the_normal_form_at_a_non_normal_state(bk):
    """normalform._adjoint_vector on a device cGL2d problem (prob.Jt with ShiftInvertB200): at a patterned state, where J is not
    normal, ζ★ is the eigenvector of J' (dense NumPy) for conj(λ), not that of J"""
    dims = (12, 8)
    pars = (0.8, 0.1, 1.0, -1.0, 1.0)
    gl = problems.GinzburgLandau2D(*dims, *L, r=pars[0], mu=pars[1], nu=pars[2], c3=pars[3], c5=pars[4])
    ctx = bk.Context(bk.BK_CGL2D, dims, L, krylov_m=120, params=pars)
    prob = bk.palc.BifurcationProblemB200(ctx, ctx.zeros(), pars, lens=0)
    assert hasattr(prob, "Jt") and not hasattr(bk.palc.BifurcationProblemB200(
        bk.Context(bk.BK_CHAN, (50,), krylov_m=4, params=(3.3, 0.01)), None, (3.3, 0.01)), "Jt")
    ph = gl.phi11()
    rng = np.random.default_rng(4)
    x0 = np.concatenate([0.6 * ph, 0.3 * ph * np.cos(np.arange(gl.n) % dims[0] * 0.4)]) + 0.05 * rng.standard_normal(gl.N)
    Jd = np.column_stack([gl.dF(x0, e) for e in np.eye(gl.N)])
    ev = np.linalg.eigvals(Jd)
    cos = lambda a, b: abs(np.vdot(a, b)) / (np.linalg.norm(a) * np.linalg.norm(b))
    ls = bk.GMRESB200(reltol=1e-12, restart=120, maxiter=1200, orth="cgs2")
    lam = ev[np.argmax(ev.real)]                                   # the rightmost pair (this J has no real eigenvalue)
    eig = bk.ShiftInvertB200(float(lam.real) + 0.05, ls, krylovdim=40, tol=1e-10, maxrestart=30)
    vec = np.asarray(bk.normalform._adjoint_vector(prob, ctx.to_device(x0), pars[0], lam, eig, 4))
    wt, vt = np.linalg.eig(Jd.T)
    w, vr = np.linalg.eig(Jd)
    ref = vt[:, np.argmin(np.abs(wt - np.conj(lam)))]
    right = max(cos(vec, vr[:, np.argmin(np.abs(w - m))]) for m in (lam, np.conj(lam)))   # 0.9952 for the exact ζ★ here
    print(f"lambda = {lam}: cos(zeta*, J' eigenvector) = {cos(vec, ref):.15f}, max cos(zeta*, J eigenvectors) = {right:.6f}")
    assert cos(vec, ref) > 1 - 1e-8
    assert right < 0.999


# ------------------------------------------------------------------------------------------------ device against a host twin
class _HostFoldTrap:
    """Host twin of periodic.TrapezeProblemB200 for the fold of cycles: oracle.potrap.Trapeze for F, the sparse oracle for J and
    J', the section in NumPy (the twin pattern of test_gpu_hopf_po.py)"""

    @staticmethod
    def make(bk, gl_at, M, pars):
        base = bk.periodic.TrapezeProblemB200

        class Twin(base):
            def __init__(self):
                base.__init__(self, None, None, list(pars), 0, M=M)
                self.phi = self.xpi = None

            def gl(self, p):
                q = list(self.params)
                q[self.lens] = p
                return gl_at(*q)

            def _set(self, p):
                self.cur = self.gl(p)

            def F(self, x, p, out=None):
                g_ = self.gl(p)
                r = opotrap.Trapeze(g_.F, g_.dF, self.phi, self.xpi, M, g_.N).residual(x)
                if out is not None:
                    out[...] = r
                    return out
                return r

            def J(self, x, p):
                return PS.cgl_po_jacobian(self.gl(p), x, M, self.phi)

            def Jt(self, x, p):
                return self.J(x, p).T.tocsr()

            def update_section(self, x, scale):
                g_ = self.cur
                self.phi = np.concatenate([scale * g_.F(x[i * g_.N:(i + 1) * g_.N]) for i in range(M)])
                self.xpi = x[:-1].copy()
        return Twin()


def _host_branch(bk, br, ind):
    """the branch with the fold's state and tangent as host arrays"""
    from dataclasses import replace
    sps = list(br.specialpoint)
    sps[ind] = replace(sps[ind], x=sps[ind].x.numpy(), tau_u=sps[ind].tau_u.numpy())
    return bk.events.Branch(rows=br.rows, specialpoint=sps)


def test_newton_fold_po_parity_with_the_host_twin(bk):
    """16 x 12, M = 10: newton_fold_po on the device and on the host twin (the oracle's Trapeze residual, the sparse oracle's J and
    J', direct sparse solves) from the same recorded fold agree in r to 1e-7 with equal Newton counts"""
    dims, M = (16, 12), 10
    trap, br, folds, ls, pars, r_hopf = _fold_branch(bk, dims, M, 60)
    assert folds
    ind = folds[0]
    lsd = bk.GMRESB200(reltol=1e-12, restart=60, maxiter=1200, Pr=True, orth="cgs2")
    opts = bk.palc.NewtonPar(tol=1e-9, max_iterations=15, linsolver=lsd)
    dev = bk.periodic.newton_fold_po(trap, br, ind, opts, bk.BorderingBLSB200(lsd, check_precision=False))
    gl_at = lambda r, mu, nu, c3, c5: problems.GinzburgLandau2D(*dims, *L, r=r, mu=mu, nu=nu, c3=c3, c5=c5)
    host = _HostFoldTrap.make(bk, gl_at, M, pars)
    hls = krylov.DefaultLS()
    hsol = bk.periodic.newton_fold_po(host, _host_branch(bk, br, ind), ind, bk.palc.NewtonPar(tol=1e-9, max_iterations=15, linsolver=hls),
                                      BlsAdapter(obls.BorderingBLS(hls, check_precision=False)))
    print("device:", dev.p, dev.itnewton, dev.residuals, " host:", hsol.p, hsol.itnewton, hsol.residuals)
    assert dev.converged and hsol.converged
    assert abs(dev.p - hsol.p) < 1e-7 and dev.itnewton == hsol.itnewton
    x, xh = dev.u.numpy(), hsol.u
    assert np.max(np.abs(x - xh)) < 1e-6 * np.max(np.abs(xh))


# ------------------------------------------------------------------------------------------------ Floquet classification
def test_floquet_reports_the_fold_as_a_branch_point(bk):
    """16 x 12, M = 10, detect_bifurcation = 3 with the Floquet eigensolver (tol_stability = 1e-4): the real multiplier that crosses
    1 at the fold of cycles makes it a "bp" (src/Bifurcations.jl:70-150).  The bisection's end points lie on both sides of the turn,
    where r is larger than at the fold, so the interval [lo, hi] holds the Newton fold up to the turn's quadratic depth: lo - (hi - lo)
    <= r_fold <= hi"""
    P = bk.palc
    dims, M = (16, 12), 10
    hp, pars, r_hopf = _hopf_point(bk, dims)
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (*dims, M), L, krylov_m=60, params=pars)
    trap = bk.periodic.TrapezeProblemB200(ctx, None, list(pars), lens=0, circulant=True)
    ls = bk.GMRESB200(reltol=1e-10, restart=60, maxiter=600, Pr=True, orth="cgs2")
    ctx_vf = bk.Context(bk.BK_CGL2D, dims, L, krylov_m=40, params=pars)
    lsf = bk.GMRESB200(reltol=1e-10, restart=40, maxiter=80, Pr=True, orth="cgs2")
    fl = bk.floquet.FloquetQaDB200(ctx_vf, lsf, M, eigsolver=bk.floquet.ArnoldiLMB200(krylovdim=30, tol=1e-8, maxrestart=10))
    cp = P.ContinuationPar(dsmin=1e-4, dsmax=0.05, ds=0.01, p_min=r_hopf - 3.0, p_max=r_hopf + 1.0, max_steps=40, nev=4,
                           detect_bifurcation=3, tol_stability=1e-4,
                           newton_options=P.NewtonPar(tol=1e-9, max_iterations=15, linsolver=ls))
    br, _, _, _ = bk.periodic.continuation_from_hopf_point(hp, cp, trap, floquet=fl, with_events=True)
    print("n_unstable along the branch:", [(round(r["param"], 5), r["n_unstable"]) for r in br.rows])
    print("special points:", [(s.type, s.param, s.interval, s.status) for s in br.specialpoint])
    bps = [i for i, s in enumerate(br.specialpoint) if s.type == "bp" and s.param < r_hopf - 0.05]
    assert bps, [s.type for s in br.specialpoint]
    sol = bk.periodic.newton_fold_po(trap, br, bps[0], P.NewtonPar(tol=1e-9, max_iterations=15, linsolver=ls),
                                     bk.BorderingBLSB200(ls, check_precision=False))
    lo, hi = br.specialpoint[bps[0]].interval
    print("bp interval", (lo, hi), "Newton fold", sol.p)
    assert sol.converged and lo - (hi - lo) <= sol.p <= hi, (lo, hi, sol.p)
