"""CPU tests of the Hopf normal form, its predictor and the periodic-orbit branches started from it (normalform.py,
periodic.py) on host arrays: the Stuart-Landau values of the reference's test/normal_forms/testNF.jl:369-450, the complex
jets composed from real ones, the Trapeze orbits of Stuart-Landau against their closed form, the section hook, and the sm_90a
code of the section kernel (read with cuobjdump, no GPU needed)."""
import numpy as np
import pytest

import __graft_entry__ as g
from oracle import krylov, bls as obls, potrap, problems
from tests import jets_oracle as JO, sass_reader as SR
from tests.test_codim2_curves_cpu import NumpyProblem2
from tests.test_host_logic_cpu import BlsAdapter, DenseComplexProblem, _dense_cls
from tests.test_normal_form_cpu import dense_eig

SL = dict(r=-0.1, mu=0.132, nu=1.0, c3=1.123, c5=0.2)   # par_sl, testNF.jl:417


def Fsl(u, q):
    """Fsl2!, testNF.jl:371-381 (the one-point cGL vector field)"""
    r, mu, nu, c3, c5 = q
    u1, u2 = u
    ua = u1**2 + u2**2
    return np.array([r * u1 - nu * u2 - ua * (c3 * u1 - mu * u2) - c5 * ua**2 * u1,
                     r * u2 + nu * u1 - ua * (c3 * u2 + mu * u1) - c5 * ua**2 * u2])


def JFsl(u, q):
    """JFsl2, testNF.jl:385-413"""
    r, mu, nu, c3, c5 = q
    u1, u2 = u
    a = u1**2 + u2**2
    return np.array([[r - c3 * (3 * u1**2 + u2**2) + 2 * mu * u1 * u2 - c5 * a * (5 * u1**2 + u2**2),
                      -nu - 2 * c3 * u1 * u2 + mu * (u1**2 + 3 * u2**2) - 4 * c5 * a * u1 * u2],
                     [nu - 2 * c3 * u1 * u2 - mu * (3 * u1**2 + u2**2) - 4 * c5 * a * u1 * u2,
                      r - c3 * (u1**2 + 3 * u2**2) - 2 * mu * u1 * u2 - c5 * a * (u1**2 + 5 * u2**2)]])


class SLProblem(NumpyProblem2):
    """Stuart-Landau with its jets (tests/jets_oracle.py: cGL on one point) and J'"""

    def d2F(self, x, p, a, b):
        q = self._par(p)
        return JO.cgl_d2F(x, a, b, q[1], q[3], q[4])

    def d3F(self, x, p, a, b, c):
        q = self._par(p)
        return JO.cgl_d3F(x, a, b, c, q[1], q[3], q[4])


def _sl_branch(save_eigenvectors):
    """testNF.jl:418-423: ContinuationPar(dsmin = 0.001, dsmax = 0.02, ds = 0.01, p_max = 0.1, p_min = -0.3), PALC(),
    normC = norminf, from r = -0.1"""
    bk = g.load_package()
    P = bk.palc
    prob = SLProblem(Fsl, JFsl, np.zeros(2), list(SL.values()), 0)
    nopts = P.NewtonPar(tol=1e-12, linsolver=krylov.DefaultLS(), eigsolver=dense_eig)
    cp = P.ContinuationPar(dsmin=0.001, dsmax=0.02, ds=0.01, p_max=0.1, p_min=-0.3, detect_bifurcation=3, newton_options=nopts,
                           save_eigenvectors=save_eigenvectors)
    alg = P.PALC(bls=BlsAdapter(obls.MatrixBLS()))
    br = bk.events.continuation(prob, alg, cp, normC=P.norminf)
    ind = next(i for i, s in enumerate(br.specialpoint) if s.type == "hopf")
    return bk, prob, cp, br, ind, P.ContIterable(prob, alg, cp, P.norminf)


@pytest.mark.parametrize("saved", [True, False], ids=["saved_eigenvectors", "recomputed"])
def test_stuart_landau_hopf_normal_form(saved):
    """testNF.jl:437-448: a ≈ 1 (atol 1e-9) and b / 2 ≈ -c3 + iμ (atol 1e-14), with the branch's eigenvectors and with
    eigenvectors recomputed at the point; c3 > 0 makes the point supercritical."""
    bk, prob, cp, br, ind, it = _sl_branch(saved)
    assert abs(br.specialpoint[ind].param) < 1e-2 and br.specialpoint[ind].delta == (2, 2)   # r_hopf = 0, located coarsely
    assert ("eigenvecs" in br.eig[0]) == saved
    cprob = DenseComplexProblem(prob.J)
    hp = bk.normalform.hopf_normal_form(it, br, ind, cprob=cprob, cls=_dense_cls)
    nf = hp.nf
    assert abs(nf["a"] - 1) < 1e-9, nf["a"]
    assert abs(nf["b"] / 2 - (-SL["c3"] + 1j * SL["mu"])) < 1e-14, nf["b"]
    assert hp.type == "SuperCritical" and abs(abs(hp.omega) - SL["nu"]) < 1e-8
    assert abs(np.vdot(hp.zeta, hp.zeta_ad) - 1) < 1e-14
    short = bk.normalform.hopf_normal_form(it, br, ind, detailed=False)
    assert short.type == "?" and short.nf["a"] is None
    pred = bk.normalform.predictor(short, 0.01, ampfactor=0.3)                # the guess without a, b (NormalForms.jl:1258-1266)
    assert pred.amp == 0.6 and pred.p == short.p + 0.01 and pred.dsfactor == 1.0


# ------------------------------------------------------------------------------------------------ complex jets
def _pair_jets(u, mu, c3, c5):
    """the real-multilinear cGL jets written as polynomials in the split components (u1, u2) of every argument, so complex
    components give the complex-multilinear extension directly"""
    n = len(u) // 2
    A = (u[:n], u[n:])
    s = lambda x, y: 2 * (x[0] * y[0] + x[1] * y[1])
    pr = lambda v: (v[:n], v[n:])
    out = lambda t3, t5: np.concatenate([-(c3 * t3[0] - mu * t3[1]) - c5 * t5[0], -(c3 * t3[1] + mu * t3[0]) - c5 * t5[1]])

    def d2(a, b):
        a, b = pr(a), pr(b)
        ss, sa, sb, sab = s(A, A) / 2, s(A, a), s(A, b), s(a, b)
        t3 = [sab * A[k] + sa * b[k] + sb * a[k] for k in (0, 1)]
        t5 = [2 * (sa * sb + ss * sab) * A[k] + 2 * ss * (sa * b[k] + sb * a[k]) for k in (0, 1)]
        return out(t3, t5)

    def d3(a, b, c):
        a, b, c = pr(a), pr(b), pr(c)
        ss, sa, sb, sc = s(A, A) / 2, s(A, a), s(A, b), s(A, c)
        sab, sac, sbc = s(a, b), s(a, c), s(b, c)
        t3 = [sab * c[k] + sac * b[k] + sbc * a[k] for k in (0, 1)]
        t5 = [2 * (sab * sc + sac * sb + sbc * sa) * A[k] + 2 * (sa * sb + ss * sab) * c[k] + 2 * (sa * sc + ss * sac) * b[k]
              + 2 * (sb * sc + ss * sbc) * a[k] for k in (0, 1)]
        return out(t3, t5)
    return d2, d3


def test_complex_jets_are_composed_from_real_ones():
    """d2Fc / d3Fc on cGL2d 9 x 7 against the complex-multilinear evaluation of the NumPy jets and against central
    differences of the complexified dF (the complex form is linear in each argument)"""
    bk = g.load_package()
    nf = bk.normalform
    gl = problems.GinzburgLandau2D(9, 7, np.pi, np.pi / 2, r=0.5, mu=0.1, nu=1.0, c3=-1.0, c5=1.0)
    par = [gl.r, gl.mu, gl.nu, gl.c3, gl.c5]

    prob = SLProblem(lambda x, q: gl.F(x), lambda x, q: None, np.zeros(gl.N), par, 0)
    rng = np.random.default_rng(3)
    u = 0.7 * rng.standard_normal(gl.N)
    a, b, c = (rng.standard_normal(gl.N) + 1j * rng.standard_normal(gl.N) for _ in range(3))
    d2, d3 = _pair_jets(u, gl.mu, gl.c3, gl.c5)
    rel = lambda x, y: np.linalg.norm(x - y) / np.linalg.norm(y)
    assert rel(nf.d2Fc(prob, u, gl.r, a, b), d2(a, b)) < 1e-14
    assert rel(nf.d3Fc(prob, u, gl.r, a, b, c), d3(a, b, c)) < 1e-14
    aa = nf.d2Fc(prob, u, gl.r, a, np.conj(a))                              # d2F[a, conj a] is real up to rounding
    assert np.abs(aa.imag).max() < 1e-14 * np.abs(aa.real).max()
    h = 1e-5
    dFc = lambda x, v: gl.dF(x, v.real) + 1j * gl.dF(x, v.imag)
    fd2 = sum(k * (dFc(u + h * part, a) - dFc(u - h * part, a)) / (2 * h) for k, part in ((1, b.real), (1j, b.imag)))
    assert rel(nf.d2Fc(prob, u, gl.r, a, b), fd2) < 1e-7
    fd3 = sum(k * (nf.d2Fc(prob, u + h * part, gl.r, a, b) - nf.d2Fc(prob, u - h * part, gl.r, a, b)) / (2 * h)
              for k, part in ((1, c.real), (1j, c.imag)))
    assert rel(nf.d3Fc(prob, u, gl.r, a, b, c), fd3) < 1e-7
    real = rng.standard_normal(gl.N)                                         # real arguments: one real call
    assert np.array_equal(nf.d2Fc(prob, u, gl.r, real, real), JO.cgl_d2F(u, real, real, gl.mu, gl.c3, gl.c5) + 0j)


# ------------------------------------------------------------------------------------------------ orbits from the Hopf point
class HostTrap:
    """Host twin of periodic.TrapezeProblemB200: the same update / record logic over oracle.potrap.Trapeze and Stuart-Landau"""

    @staticmethod
    def make(bk, M, every):
        base = bk.periodic.TrapezeProblemB200

        class Twin(base):
            def __init__(self):
                base.__init__(self, None, None, list(SL.values()), 0, update_section_every_step=every, M=M)
                self.tr = potrap.Trapeze(None, None, np.zeros(2 * M), np.zeros(2 * M), M, 2)

            def _bind(self, p):
                q = list(self.params)
                q[self.lens] = p
                self.tr.F = lambda u: Fsl(u, q)
                self.tr.dF = lambda u, du: JFsl(u, q) @ du
                return q

            def _set(self, p):
                self.cur = self._bind(p)

            def F(self, x, p, out=None):
                self._bind(p)
                r = self.tr.residual(x)
                if out is not None:
                    out[...] = r
                    return out
                return r

            def J(self, x, p):
                self.last_state, self.last_p = x, p
                self._bind(p)
                return np.column_stack([self.tr.jvp(x, e) for e in np.eye(len(x))])

            def update_section(self, x, scale):
                F = self.tr.F
                self.tr.phi = np.concatenate([scale * F(u) for u in x[:-1].reshape(M, 2)])
                self.tr.xpi = x[:-1].copy()
        return Twin()


def _po_branch(every, M=10, steps=8):
    bk, prob, cp, br, ind, it = _sl_branch(False)
    P = bk.palc
    trap = HostTrap.make(bk, M, every)
    ls = krylov.DefaultLS()
    cpo = P.ContinuationPar(dsmin=1e-4, dsmax=0.02, ds=0.01, p_min=-0.3, p_max=0.3, max_steps=steps,
                            newton_options=P.NewtonPar(tol=1e-11, max_iterations=15, linsolver=ls))
    seen = []

    def cb(st):
        x = np.array(st.z_u)
        seen.append((st.step, st.z_p, x, trap.tr.phi.copy(), trap.tr.xpi.copy(), trap.section_updates))

    rows, st, hp, pred = bk.periodic.continuation_from_hopf(
        it, br, ind, cpo, trap, cprob=DenseComplexProblem(prob.J), cls=_dense_cls,
        bls=BlsAdapter(obls.BorderingBLS(ls, check_precision=False)), callback=cb)
    return bk, trap, rows, st, hp, pred, seen


@pytest.mark.parametrize("every", [0, 1])
def test_stuart_landau_orbits_from_the_hopf_point_are_discrete_circles(every):
    """With the mesh step T/M and M-1 cyclic rows (oracle/potrap.py) the discrete orbit of Stuart-Landau is a circle of radius ρ
    with r - c3 ρ^2 - c5 ρ^4 = 0, run at Ω = ν - μ ρ^2 with T = 2 M tan(π / (M - 1)) / Ω: consecutive slices turn by 2π/(M-1)
    and z_i - z_{i-1} = (h/2) iΩ (z_i + z_{i-1}) gives tan(π/(M-1)) = h Ω / 2.  Every row of the branch switched from the Hopf
    point matches it; c3 > 0 makes the Hopf point supercritical, so the orbits and the predictor lie at r > r_hopf."""
    M = 10
    bk, trap, rows, st, hp, pred, seen = _po_branch(every, M)
    assert hp.type == "SuperCritical" and pred.p > hp.p and pred.dsfactor == 1.0
    assert len(rows) >= 8 and all(r["param"] > hp.p for r in rows)
    c3, c5, mu, nu = SL["c3"], SL["c5"], SL["mu"], SL["nu"]
    for step, r, x, _, _, _ in seen:
        u = x[:-1].reshape(M, 2)
        rho = np.hypot(u[:, 0], u[:, 1])
        assert np.ptp(rho) < 1e-10, (step, rho)
        rho = rho.mean()
        assert abs(r - c3 * rho**2 - c5 * rho**4) < 1e-10, step
        assert abs(x[-1] - 2 * M * np.tan(np.pi / (M - 1)) / (nu - mu * rho**2)) < 1e-9, step
        assert np.abs(u[-1] - u[0]).max() < 1e-12
    assert [r["x"]["period"] for r in rows] == [s[2][-1] for s in seen]
    assert trap.section_updates == (0 if every == 0 else len(rows) - 2)


def test_section_hook_after_accepted_steps():
    """update!(wrap, iter, state) with update_section_every_step = 1 (PeriodicOrbits.jl:156-169): the start and the first step
    keep the section of re_make (phi_i = F(x_i) at the predictor's parameter, xpi = the guess); after every later accepted step
    phi_i = F(x_i) / M at that step's parameter and xpi = the orbit of that step (the reference calls the hook before it counts
    the step, and mod_counter(0, 1) is false)."""
    M = 10
    bk, trap, rows, st, hp, pred, seen = _po_branch(1, M, steps=5)
    phi0, xpi0 = seen[0][3], seen[0][4]
    assert np.array_equal(seen[1][3], phi0) and np.array_equal(seen[1][4], xpi0)
    g0 = xpi0.reshape(M, 2)
    assert np.allclose(phi0, np.concatenate([Fsl(v, [pred.p] + list(SL.values())[1:]) for v in g0]), rtol=0, atol=1e-15)
    for step, r, x, phi, xpi, n in seen[2:]:
        q = [r] + list(SL.values())[1:]
        ref = np.concatenate([Fsl(v, q) / M for v in x[:-1].reshape(M, 2)])
        assert np.allclose(phi, ref, rtol=1e-15, atol=1e-17) and np.array_equal(xpi, x[:-1]) and n == step - 1


# ------------------------------------------------------------------------------------------------ sm_90a code
def test_section_kernel_is_in_the_sm_90a_code_without_local_memory():
    cnt = SR.mnemonics()
    sec = {k: c for k, c in cnt.items() if "k_potrap_section" in k}
    assert len(sec) == 1
    c = next(iter(sec.values()))
    assert c["LDL"] == 0 and c["STL"] == 0 and c["DFMA"] + c["DMUL"] >= 10, dict(c)
    assert "arch = sm_90a" in SR.cuobjdump("-sass")
