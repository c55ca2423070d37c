"""GPU tests of bk_potrap_update_section, the Hopf normal form on cGL2d (normalform.hopf_normal_form / hopf_normal_form_at)
and periodic-orbit branches switched from the Hopf point (periodic.py), with device vectors, against the NumPy oracle and a
host twin of the Trapeze problem."""
import numpy as np
import pytest

import __graft_entry__ as g
from oracle import krylov, bls as obls, potrap as opotrap, precond as oprecond, problems
from tests import jets_oracle as JO
from tests.test_host_logic_cpu import BlsAdapter

pytestmark = pytest.mark.gpu
L = (np.pi, np.pi / 2)


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


def _rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300)


def _gl(dims, pars):
    return problems.GinzburgLandau2D(*dims, *L, r=pars[0], mu=pars[1], nu=pars[2], c3=pars[3], c5=pars[4])


# ------------------------------------------------------------------------------------------------ bk_potrap_update_section
def test_update_section_on_the_device(bk):
    """phi_i = scale F(x_i) (oracle) and xpi = x without the period; host and device x give the same bits; the PO residual
    after the update equals the residual after bk_potrap_set_section with the same phi and xpi; bad arguments: BK_ERR_ARG."""
    nx, ny, M = 24, 12, 8
    pars = (1.3, 0.1, 1.0, -1.0, 1.0)
    gl = _gl((nx, ny), pars)
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (nx, ny, M), L, krylov_m=8, params=pars)
    ctx_vf = bk.Context(bk.BK_CGL2D, (nx, ny), L, krylov_m=4, params=pars)
    N, Ns = ctx.N, gl.N
    rng = np.random.default_rng(11)
    x = rng.standard_normal(N)
    x[-1] = 6.1
    probe = [rng.standard_normal(N) for _ in range(3)]
    for scale in (1.0 / M, 1.0):
        phi_ref = np.concatenate([scale * gl.F(x[i * Ns:(i + 1) * Ns]) for i in range(M)])
        tr = opotrap.Trapeze(gl.F, gl.dF, phi_ref, x[:-1], M, Ns)
        y = x + 0.01 * rng.standard_normal(N)
        outs = []
        for xin in (x, ctx.to_device(x)):
            ctx.potrap_update_section(xin, scale)
            J = ctx.jacobian(y)
            outs.append(np.concatenate([ctx.residual(y), [J(v)[-1] for v in probe]]))   # last JVP row = <v, phi>
        assert np.array_equal(outs[0], outs[1])
        assert abs(outs[0][-4] - tr.residual(y)[-1]) < 1e-13 * np.linalg.norm(phi_ref) * np.linalg.norm(y)
        for v, got in zip(probe, outs[0][-3:]):
            assert abs(got - np.dot(v[:-1], phi_ref)) < 1e-13 * np.linalg.norm(phi_ref) * np.linalg.norm(v)
        assert _rel(outs[0][:-3], tr.residual(y)) < 1e-12
        # the same phi from the vector-field kernels, through bk_potrap_set_section
        phi_dev = np.concatenate([scale * ctx_vf.residual(x[i * Ns:(i + 1) * Ns]) for i in range(M)])
        assert _rel(phi_dev, phi_ref) < 1e-13
        ctx.potrap_set_section(phi_dev, x[:-1])
        assert _rel(ctx.residual(y), outs[0][:-3]) < 1e-14
    lib = ctx.lib
    assert lib.bk_potrap_update_section(ctx.handle, None, 1.0) == -1
    assert lib.bk_potrap_update_section(ctx_vf.handle, x.ctypes.data, 1.0) == -1
    assert lib.bk_potrap_update_section(None, x.ctypes.data, 1.0) == -1


# ------------------------------------------------------------------------------------------------ Hopf normal form
@pytest.fixture(scope="module")
def hopf_branch(bk):
    """the trivial cGL2d 41 x 21 branch through its first Hopf point (set-up of test_hopf_point_located_by_bisection_on_device)"""
    P, E = bk.palc, bk.events
    dims = (41, 21)
    r_hopf = problems.GinzburgLandau2D(*dims, *L).r_hopf()
    pars = (r_hopf - 0.3, 0.1, 1.0, -1.0, 1.0)
    ctx = bk.Context(bk.BK_CGL2D, dims, L, krylov_m=120, params=pars)
    inner = bk.GMRESB200(reltol=1e-10, restart=120, maxiter=600, orth="cgs2")
    eig = bk.ShiftInvertB200(0.5, inner, krylovdim=40, tol=1e-8, maxrestart=30)
    ls = bk.GMRESB200(reltol=1e-10, restart=120, maxiter=240)
    nopts = P.NewtonPar(tol=1e-9, max_iterations=10, linsolver=ls, eigsolver=eig)
    cp = P.ContinuationPar(dsmin=1e-4, dsmax=0.05, ds=0.01, p_min=r_hopf - 0.5, p_max=r_hopf + 0.3, max_steps=60, newton_options=nopts,
                           detect_bifurcation=3, n_inversion=6, nev=4, tol_stability=1e-8)
    prob = P.BifurcationProblemB200(ctx, ctx.zeros(), pars, lens=0, record=lambda v: v.norminf())
    alg = P.PALC(bls=bk.MatrixFreeBLSB200(ls))
    br = E.continuation(prob, alg, cp, normC=P.norminf)
    ind = next(i for i, s in enumerate(br.specialpoint) if s.type == "hopf")
    return dict(it=P.ContIterable(prob, alg, cp, P.norminf), br=br, ind=ind, r_hopf=r_hopf, pars=pars, dims=dims)


def test_hopf_normal_form_at_the_analytic_hopf_point(bk, hopf_branch):
    """At the trivial state J = Lap + (r + iν) on A = u1 + i u2.  With φ the discrete first Dirichlet mode and A = c φ, the
    projection of -(c3 + iμ)|A|^2 A onto φ is -(c3 + iμ) |c|^2 c Σφ⁴ / Σφ²; the quadratic terms vanish at A = 0, so Ψ110 and Ψ200
    do not contribute.  ζ = (φ, ∓iφ) / (√2 |φ|) gives A = √2 w φ / |φ| (up to conjugation) for x = 2 Re(w ζ), hence
    dw/dt = (iω + (r - r_hopf)) w + 2(-c3 + iμ) (Σφ⁴ / (Σφ²)^2) |w|^2 w for ω > 0: a = 1 and b = 2(-c3 + iμ) Σφ⁴ / (Σφ²)^2.
    Stuart-Landau is the one-point case (b / 2 = -c3 + iμ, test/normal_forms/testNF.jl:441).  c3 = -1: Re b > 0, subcritical."""
    h = hopf_branch
    hp = bk.normalform.hopf_normal_form(h["it"], h["br"], h["ind"])
    _, mu, nu, c3, _ = h["pars"]
    phi = _gl(h["dims"], h["pars"]).phi11()
    S = np.sum(phi**4) / np.sum(phi**2) ** 2
    assert abs(hp.omega - nu) < 1e-6 and abs(hp.p - h["r_hopf"]) < 1e-5
    assert abs(hp.nf["a"] - 1) < 1e-6, hp.nf["a"]
    assert abs(hp.nf["b"] - 2 * (-c3 + 1j * mu) * S) < 1e-6 * abs(hp.nf["b"]), (hp.nf["b"], 2 * (-c3 + 1j * mu) * S)
    assert hp.type == "SubCritical"


def test_hopf_normal_form_at_a_patterned_state_matches_dense_numpy(bk):
    """hopf_normal_form_at on cGL2d 24 x 12 at a patterned state that is not an equilibrium, against a dense NumPy restatement of
    __hopf_normal_form (NormalForms.jl:1009-1076) with np.linalg.solve, the 2iω shift included: a, b, Ψ001, Ψ110, Ψ200.  The
    quadratic terms do not vanish here, so this exercises the complex solve.  Both sides take central differences with δ = 1e-4:
    F is linear in r, so they are exact up to rounding."""
    dims = (24, 12)
    pars = (0.8, 0.1, 1.0, -1.0, 1.0)
    gl = _gl(dims, pars)
    N = gl.N
    ctx = bk.Context(bk.BK_CGL2D, dims, L, krylov_m=300, params=pars)
    prob = bk.palc.BifurcationProblemB200(ctx, ctx.zeros(), pars, lens=0, delta=1e-4)
    rng = np.random.default_rng(4)
    ph = gl.phi11()
    x0 = np.concatenate([0.6 * ph, 0.3 * ph * np.cos(np.arange(gl.n) % dims[0] * 0.4)]) + 0.05 * rng.standard_normal(N)
    zeta = rng.standard_normal(N) + 1j * rng.standard_normal(N)
    zeta /= np.linalg.norm(zeta)
    zeta_ad = rng.standard_normal(N) + 1j * rng.standard_normal(N)
    zeta_ad /= np.vdot(zeta, zeta_ad)
    omega, p, d = 1.3, pars[0], 1e-4
    ls = bk.GMRESB200(reltol=1e-13, restart=300, maxiter=3000, orth="cgs2")
    hp = bk.normalform.hopf_normal_form_at(prob, ctx.to_device(x0), p, omega, zeta, zeta_ad, ls)
    # dense restatement
    Jd = lambda r: np.column_stack([gl.dF(x0, e, r) for e in np.eye(N)])
    L0 = Jd(p)

    def d2c(a, b):
        f = lambda u, v: JO.cgl_d2F(x0, u, v, gl.mu, gl.c3, gl.c5)
        return f(a.real, b.real) - f(a.imag, b.imag) + 1j * (f(a.real, b.imag) + f(a.imag, b.real))

    def d3c(a, b, c):
        out = 0
        for ka, pa in ((1, a.real), (1j, a.imag)):
            for kb, pb in ((1, b.real), (1j, b.imag)):
                for kc, pc in ((1, c.real), (1j, c.imag)):
                    out = out + ka * kb * kc * JO.cgl_d3F(x0, pa, pb, pc, gl.mu, gl.c3, gl.c5)
        return out
    R01 = (gl.F(x0, p + d) - gl.F(x0, p - d)) / (2 * d)
    P001 = np.linalg.solve(L0, -R01)
    av = (Jd(p + d) - Jd(p - d)) @ zeta / (2 * d) + d2c(zeta, P001 + 0j)
    a = np.vdot(av, zeta_ad)
    P200 = np.linalg.solve(2j * omega * np.eye(N) - L0, d2c(zeta, zeta) / 2)
    P110 = np.linalg.solve(L0, -np.real(d2c(zeta, np.conj(zeta))))
    bv = d2c(zeta, P110 + 0j) + d2c(np.conj(zeta), P200) + d3c(zeta, zeta, np.conj(zeta)) / 2
    b = np.vdot(bv, zeta_ad)
    nf = hp.nf
    assert _rel(nf["Psi001"], P001) < 1e-8 and _rel(nf["Psi110"], P110) < 1e-8 and _rel(nf["Psi200"], P200) < 1e-8
    assert abs(nf["a"] - a) < 1e-8 * abs(a) and abs(nf["b"] - b) < 1e-8 * abs(b), (nf["a"], a, nf["b"], b)


# ------------------------------------------------------------------------------------------------ periodic orbits
def test_branch_switching_from_the_hopf_point_on_the_device(bk, hopf_branch):
    """continuation_from_hopf at the size of examples/cGL2d.jl (41 x 21, M = 30, N = 51 661), 15 steps, the branch on the device:
    every orbit satisfies the oracle's Trapeze residual with the section of the guess (update_section_every_step = 0); the
    Hopf point is subcritical, so the first orbits lie at r < r_hopf; the first orbit's period and amplitude agree with the
    predictor's guess to first order; Floquet on the first orbit has one multiplier within 1e-4 of 1 (the phase) and, as
    theory predicts for the orbits born at a subcritical Hopf point, exactly one outside the unit circle."""
    P = bk.palc
    h = hopf_branch
    nx, ny = h["dims"]
    M = 30
    pars = list(h["pars"])
    gl = _gl(h["dims"], pars)
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (nx, ny, M), L, krylov_m=60, params=pars)
    assert ctx.N == 51661
    trap = bk.periodic.TrapezeProblemB200(ctx, None, pars, lens=0, circulant=True)
    ls = bk.GMRESB200(reltol=1e-8, restart=60, maxiter=300, Pr=True, orth="cgs2")
    cp = P.ContinuationPar(dsmin=1e-4, dsmax=0.03, ds=0.01, p_min=h["r_hopf"] - 1.0, p_max=h["r_hopf"] + 1.0, max_steps=15,
                           newton_options=P.NewtonPar(tol=1e-8, max_iterations=15, linsolver=ls))
    orbits = []
    rows, st, hp, pred = bk.periodic.continuation_from_hopf(h["it"], h["br"], h["ind"], cp, trap,
                                                            callback=lambda s: orbits.append((s.z_p, s.z_u.numpy())))
    assert hp.type == "SubCritical" and pred.p < hp.p and len(rows) >= 10
    guess = trap.u0.numpy()
    Ns = gl.N
    phi = np.concatenate([gl.F(guess[i * Ns:(i + 1) * Ns], pred.p) for i in range(M)])
    for r, x in orbits:
        tr = opotrap.Trapeze(lambda u: gl.F(u, r), lambda u, du: gl.dF(u, du, r), phi, guess[:-1], M, Ns)
        assert np.max(np.abs(tr.residual(x))) < 1e-7, r
    assert all(r < h["r_hopf"] for r, _ in orbits[:3])
    x1 = orbits[0][1]
    assert abs(x1[-1] - pred.period) < 0.05 * pred.period
    amp_guess = np.max(np.abs(guess[:-1]))
    assert abs(rows[0]["x"]["amplitude"] - amp_guess) < 0.2 * amp_guess
    # Floquet multipliers of the first orbit
    ctx_vf = bk.Context(bk.BK_CGL2D, (nx, ny), L, krylov_m=40, params=pars)
    lsf = bk.GMRESB200(reltol=1e-10, restart=40, maxiter=80, Pr=True, orth="cgs2")
    fl = bk.floquet.FloquetQaDB200(ctx_vf, lsf, M, eigsolver=bk.floquet.ArnoldiLMB200(krylovdim=30, tol=1e-8, maxrestart=10))
    q = list(pars)
    q[0] = orbits[0][0]
    ctx_vf.set_params(q)
    bk.floquet.cgl_shifted_precond(ctx_vf, x1[-1], M, q[0])
    sig, _, cv, info = fl(ctx.to_device(x1), 4)
    mu = np.abs(info["multipliers"])
    print("Floquet multipliers of the first orbit:", info["multipliers"])
    assert cv
    assert np.min(np.abs(info["multipliers"] - 1)) < 1e-4
    assert int(np.sum(mu > 1 + 1e-4)) == 1


class _HostTrap:
    """Host twin of periodic.TrapezeProblemB200 for cGL2d: oracle.potrap.Trapeze over oracle.problems.GinzburgLandau2D, the
    oracle's circulant preconditioner, the section in NumPy"""

    @staticmethod
    def make(bk, gl, M, pars, every):
        base = bk.periodic.TrapezeProblemB200
        Ns = gl.N

        class Twin(base):
            def __init__(self):
                base.__init__(self, None, None, list(pars), 0, update_section_every_step=every, circulant=True, M=M)
                self.tr = opotrap.Trapeze(None, None, np.zeros(Ns * M), np.zeros(Ns * M), M, Ns)
                self.Po = None

            def _set(self, p):
                self.r = p
                self.tr.F = lambda u: gl.F(u, p)
                self.tr.dF = lambda u, du: gl.dF(u, du, p)

            def F(self, x, p, out=None):
                self._set(p)
                res = self.tr.residual(x)
                if out is not None:
                    out[...] = res
                    return out
                return res

            def J(self, x, p):
                self.last_state, self.last_p = x, p
                self._set(p)
                tr = self.tr
                F, dF = tr.F, tr.dF
                return lambda v: opotrap.Trapeze(F, dF, tr.phi, tr.xpi, M, Ns).jvp(x, v)

            def update_section(self, x, scale):
                self.tr.phi = np.concatenate([scale * self.tr.F(x[i * Ns:(i + 1) * Ns]) for i in range(M)])
                self.tr.xpi = x[:-1].copy()

            def setup_precond(self, x):
                self.Po = oprecond.potrap_circulant_precond(gl.Nx, gl.Ny, gl.lx, gl.ly, M, float(x[-1]), self.r, gl.nu)
        return Twin()


def test_po_branch_parity_with_the_host_twin(bk):
    """cGL2d 16 x 12, M = 10: the same Hopf normal form (computed on the device at the analytic point, ζ = ζ★ = (φ, -iφ) / (√2 |φ|))
    continued on the device and on the host twin (oracle Trapeze, oracle GMRES with the oracle's circulant preconditioner):
    rows (param, period, amplitude) agree to 1e-6 with equal Newton counts, with the section kept and updated every step."""
    P = bk.palc
    dims, M = (16, 12), 10
    r_hopf = problems.GinzburgLandau2D(*dims, *L).r_hopf()
    pars = [r_hopf, 0.1, 1.0, -1.0, 1.0]
    gl = _gl(dims, pars)
    ctx_vf = bk.Context(bk.BK_CGL2D, dims, L, krylov_m=200, params=pars)
    prob = P.BifurcationProblemB200(ctx_vf, ctx_vf.zeros(), pars, lens=0)
    ph = gl.phi11() / np.linalg.norm(gl.phi11())
    zeta = np.concatenate([ph, -1j * ph]) / np.sqrt(2)
    ls_vf = bk.GMRESB200(reltol=1e-12, restart=200, maxiter=2000, orth="cgs2")
    hp = bk.normalform.hopf_normal_form_at(prob, ctx_vf.zeros(), r_hopf, pars[2], zeta, zeta, ls_vf)
    for every in (0, 1):
        ctx = bk.Context(bk.BK_POTRAP_CGL2D, (*dims, M), L, krylov_m=60, params=pars)
        dev = bk.periodic.TrapezeProblemB200(ctx, None, list(pars), lens=0, update_section_every_step=every, circulant=True)
        host = _HostTrap.make(bk, gl, M, pars, every)
        cp = lambda ls: P.ContinuationPar(dsmin=1e-4, dsmax=0.03, ds=0.01, p_min=r_hopf - 1.0, p_max=r_hopf + 1.0, max_steps=8,
                                          newton_options=P.NewtonPar(tol=1e-9, max_iterations=15, linsolver=ls))
        ls_d = bk.GMRESB200(reltol=1e-11, restart=60, maxiter=600, Pr=True, orth="cgs2")
        rd, _, _, _ = bk.periodic.continuation_from_hopf_point(hp, cp(ls_d), dev)

        class HostLS:  # the oracle GMRES with the twin's current circulant preconditioner
            def __call__(self, J, rhs, rhs2=None, a0=0.0, a1=1.0):
                return krylov.GMRESIterativeSolvers(reltol=1e-11, restart=60, maxiter=600, Pr=host.Po, orth="cgs2")(J, rhs, rhs2, a0=a0,
                                                                                                              a1=a1)
        ls_h = HostLS()
        rh, _, _, _ = bk.periodic.continuation_from_hopf_point(hp, cp(ls_h), host,
                                                               bls=BlsAdapter(obls.BorderingBLS(ls_h, check_precision=False)))
        assert len(rd) == len(rh) >= 6
        for a, b in zip(rd, rh):
            assert abs(a["param"] - b["param"]) < 1e-6 and abs(a["x"]["period"] - b["x"]["period"]) < 1e-6
            assert abs(a["x"]["amplitude"] - b["x"]["amplitude"]) < 1e-6 and a["itnewton"] == b["itnewton"], (a, b)
        assert dev.section_updates == host.section_updates == (0 if every == 0 else len(rd) - 2)
