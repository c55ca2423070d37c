"""CPU tests of the simple-branch-point normal form and branch switching (bifurcationkit.jl_b200/normalform.py) on host arrays,
pinned to the reference's test/normal_forms/testNF.jl; the NumPy jets of tests/jets_oracle.py against finite differences of the
oracle's dF; and the sm_90a code of the jet kernels (read with cuobjdump, no GPU needed)."""
import dataclasses
import re

import numpy as np
import pytest

import __graft_entry__ as g
from oracle import krylov, bls as obls, problems
from tests import jets_oracle as JO, sass_reader as SR
from tests.sh_periodic_oracle import PeriodicSH
from tests.test_codim2_curves_cpu import NumpyProblem2
from tests.test_host_logic_cpu import BlsAdapter


def _rel(a, b):
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


# ------------------------------------------------------------------------------------------------ 1. the NumPy jets
def _jet_cases():
    rng = np.random.default_rng(7)
    n = 40
    alpha, beta = 3.3, 0.01
    yield "chan", n, (lambda u, d: problems.chan_dF(u, d, alpha, beta)), \
        (lambda u, a, b: JO.chan_d2F(u, a, b, alpha, beta)), (lambda u, a, b, c: JO.chan_d3F(u, a, b, c, alpha, beta)), \
        problems.chan_sol0(n) + 0.5 * rng.standard_normal(n)
    for dims, L in (((24, 18), (2.3 * np.pi, 1.7 * np.pi)), ((10, 8, 6), (1.3 * np.pi, 1.1 * np.pi, 0.9 * np.pi))):
        sh = problems.SwiftHohenberg(dims, L, l=-0.1, nu=1.3)
        yield f"sh{len(dims)}d", sh.N, sh.dF, (lambda u, a, b, nu=sh.nu: JO.sh_d2F(u, a, b, nu)), JO.sh_d3F, rng.standard_normal(sh.N)
    ps = PeriodicSH((16, 8), (4 * np.pi, 2 * np.pi), l=-0.15, nu=1.3)
    yield "sh2d_periodic", ps.N, ps.dF, (lambda u, a, b: JO.sh_d2F(u, a, b, ps.nu)), JO.sh_d3F, rng.standard_normal(ps.N)
    gl = problems.GinzburgLandau2D(12, 7, np.pi, np.pi / 2, r=0.5, mu=0.1, nu=1.0, c3=-1.0, c5=1.0)
    yield "cgl2d", gl.N, gl.dF, (lambda u, a, b: JO.cgl_d2F(u, a, b, gl.mu, gl.c3, gl.c5)), \
        (lambda u, a, b, c: JO.cgl_d3F(u, a, b, c, gl.mu, gl.c3, gl.c5)), 0.7 * rng.standard_normal(gl.N)


@pytest.mark.parametrize("case", list(_jet_cases()), ids=lambda c: c[0])
def test_numpy_jets_are_the_derivatives_of_the_oracle_dF(case):
    """d2F[a, b] = d/dt dF(u + t b)[a] and d3F[a, b, c] = d/dt d2F(u + t c)[a, b], central differences at t = 0"""
    _, N, dF, d2F, d3F, u = case
    rng = np.random.default_rng(1)
    a, b, c = (rng.standard_normal(N) for _ in range(3))
    h = 1e-5
    fd2 = (dF(u + h * b, a) - dF(u - h * b, a)) / (2 * h)
    assert _rel(d2F(u, a, b), fd2) < 1e-6
    fd3 = (d2F(u + h * c, a, b) - d2F(u - h * c, a, b)) / (2 * h)
    assert _rel(d3F(u, a, b, c), fd3) < 1e-6
    assert _rel(d2F(u, a, b), d2F(u, b, a)) < 1e-14 and _rel(d3F(u, a, b, c), d3F(u, c, a, b)) < 1e-14


# ------------------------------------------------------------------------------------------------ testNF.jl problem
MU, NU, X2, X3, GAMMA = range(5)


def Fbp(x, q):
    """test/normal_forms/testNF.jl:8-9"""
    return np.array([x[0] * (3.23 * q[MU] - q[X2] * x[0] + q[X3] * x[0] ** 2) + x[1], -x[1] + q[GAMMA] * x[0] ** 2])


def Jbp(x, q):
    """testNF.jl:11-18"""
    return np.array([[3.23 * q[MU] - 2 * q[X2] * x[0] + 3 * q[X3] * x[0] ** 2, 1.0], [2 * q[GAMMA] * x[0], -1.0]])


class BpProblem(NumpyProblem2):
    """Fbp with its second and third differentials in x"""

    def d2F(self, x, p, a, b):
        q = self._par(p)
        return np.array([(-2 * q[X2] + 6 * q[X3] * x[0]) * a[0] * b[0], 2 * q[GAMMA] * a[0] * b[0]])

    def d3F(self, x, p, a, b, c):
        return np.array([6 * self._par(p)[X3] * a[0] * b[0] * c[0], 0.0])


def dense_eig(J, nev):
    """DefaultEig (src/EigSolver.jl:31-50) with eigenvectors: decreasing real part, vectors as columns"""
    vals, vecs = np.linalg.eig(np.asarray(J))
    k = np.argsort(-vals.real, kind="stable")[:nev]
    return vals[k], vecs[:, k], True, 1


def _setup(par, u0=(0.0, 0.0), tangent="secant", **kw):
    """testNF.jl:22-25: opts_br, PALC(), normC = norminf"""
    bk = g.load_package()
    P = bk.palc
    nopts = P.NewtonPar(tol=1e-14, linsolver=krylov.DefaultLS(), eigsolver=dense_eig)
    cp = P.ContinuationPar(**{**dict(dsmin=0.001, dsmax=0.05, ds=0.01, p_max=0.4, p_min=-0.5, detect_bifurcation=3,
                                     newton_options=nopts, max_steps=100, n_inversion=8), **kw})
    prob = BpProblem(Fbp, Jbp, np.array(u0), par, MU)
    alg = P.PALC(tangent=tangent, bls=BlsAdapter(obls.MatrixBLS()))
    br = bk.events.continuation(prob, alg, cp, normC=P.norminf)
    return bk, prob, alg, cp, br, P.ContIterable(prob, alg, cp, P.norminf)


def test_transcritical_with_given_kernel_vectors():
    """testNF.jl:20-49: gamma = 4.4323, ζs = [1, 0], ζs_ad = [1, 1], the point's parameter set to 0"""
    par = [-0.2, 0.0, 1.12, 0.234, 4.4323]
    bk, prob, alg, cp, br, it = _setup(par)
    bp0 = br.specialpoint[0]
    assert bp0.type == "bp" and bp0.interval[0] < 0 < bp0.interval[1]
    br.specialpoint[0] = dataclasses.replace(bp0, param=0.0)
    nfm = bk.normalform
    bp = nfm.get_normal_form1d(it, br, 0, zeta=[1.0, 0.0], zeta_ad=[1.0, 1.0], bls=alg.bls)
    nf = bp.nf
    assert np.allclose(nf["Psi20"], [0.0, 2 * par[GAMMA]], rtol=1e-8, atol=1e-12)
    assert abs(nf["a01"]) < 1e-10
    assert abs(nf["b11"] - 3.23) < 1e-10
    assert abs(nf["b20"] / 2 - (-par[X2] + par[GAMMA])) < 1e-10
    assert abs(nf["b30"] / 6 - par[X3]) < 1e-10
    assert bp.type == "Transcritical"
    assert np.linalg.norm(nfm.predictor(bp, 0.1).x0) < 1e-10


def test_transcritical_recomputed_eigenvectors_and_branch_switching():
    """testNF.jl:60-86: gamma = 0, eigen-elements recomputed at the point; aBS with p_max = 0.2, ds = 0.01, max_steps = 14 gives a
    branch of 12 points with eigenvalues"""
    par = [-0.2, 0.0, 1.12, 0.234, 0.0]
    bk, prob, alg, cp, br, it = _setup(par)
    nfm = bk.normalform
    bp = nfm.get_normal_form1d(it, br, 0, bls=alg.bls)
    nf = bp.nf
    assert abs(nf["a01"]) < 1e-10 and abs(nf["b11"] - 3.23) < 1e-10
    assert abs(nf["b20"] / 2 + 1.12) < 1e-10 and abs(nf["b30"] / 6 - 0.234) < 1e-10
    out = nfm.continuation_from_bp(br, 0, prob, alg, dataclasses.replace(cp, p_max=0.2, ds=0.01, max_steps=14), normC=bk.palc.norminf)
    br2, bp2 = out
    assert bp2.type == "Transcritical"
    assert len(br2.rows) == 12 and len(br2.eig) == 12
    assert prob.u0.tolist() == [0.0, 0.0] and prob.p0 == -0.2                         # the caller's problem is untouched
    # the new branch is the non-trivial one, 3.23 mu - 1.12 x + 0.234 x^2 = 0, y = 0; its first step crosses the branch point
    # (n_unstable 1 -> 0), which the bisection locates again, as get_normal_form(br2, 1) of testNF.jl:80 expects
    assert [s.type for s in br2.specialpoint] == ["bp", "endpoint"] and br2.specialpoint[0].idx == 1
    assert all(r["param"] > bp2.p for r in br2.rows[2:]) and br2.rows[-1]["param"] == 0.2
    st = br2.state
    assert np.linalg.norm(Fbp(st.z_u, prob._par(st.z_p))) < 1e-12 and abs(st.z_u[0]) > 0.1


def test_transcritical_from_the_non_trivial_branch():
    """testNF.jl:97-105: x3 = 1, start on the non-trivial branch, n_inversion = 10"""
    par = [-0.2, 0.0, 1.12, 1.0, 0.0]
    bk, prob, alg, cp, br, it = _setup(par, u0=(-0.5, 0.0), n_inversion=10)
    nf = bk.normalform.get_normal_form1d(it, br, 0, bls=alg.bls).nf
    assert abs(nf["a01"]) < 1e-6
    assert abs(nf["b11"] - 3.23) < 1e-10
    assert abs(nf["b20"] / 2 + par[X2]) < 1e-6
    assert abs(nf["b30"] / 6 - par[X3]) < 1e-10


def test_bordered_tangent_case_and_branch_switching():
    """testNF.jl:115-138: x2 = 0, x3 = -1, gamma = 1.422, PALC(tangent = Bordered()); aBS with max_steps = 19, ds = 0.001,
    dsmax = 0.01, detect_bifurcation = 2"""
    par = [-0.2, 0.0, 0.0, -1.0, 1.422]
    bk, prob, alg, cp, br, it = _setup(par, tangent="bordered")
    nfm = bk.normalform
    bp = nfm.get_normal_form1d(it, br, 0, bls=alg.bls)
    nf = bp.nf
    assert abs(nf["a01"]) < 1e-10 and abs(nf["a02"]) < 1e-10
    assert abs(nf["b11"] - 3.23) < 1e-10
    assert abs(nf["b20"] / 2 - par[GAMMA]) < 1e-4
    assert abs(nf["b30"] / 6 - par[X3]) < 1e-10
    assert np.max(np.abs(nfm.predictor(bp, 0.1).x0)) < 1e-6
    br2, _ = nfm.continuation_from_bp(br, 0, prob, alg, dataclasses.replace(cp, max_steps=19, dsmax=0.01, ds=0.001, detect_bifurcation=2),
                                      normC=bk.palc.norminf)
    assert br2.state.converged and [r["step"] for r in br2.rows] == list(range(len(br2.rows)))
    assert len(br2.rows) == 20
    for row in br2.rows:
        assert row["itnewton"] <= cp.newton_options.max_iterations


def test_pitchfork_predictor_and_branch_switching():
    """x2 = gamma = 0, x3 = -1: a supercritical pitchfork at mu = 0 whose bifurcated branch is x^2 = 3.23 mu, y = 0.  The predictor
    picks mu > 0 (b11 b30 < 0) with amplitude sqrt(-6 ds b11 / b30) (src/NormalForms.jl:457-487)"""
    par = [-0.2, 0.0, 0.0, -1.0, 0.0]
    bk, prob, alg, cp, br, it = _setup(par)
    nfm = bk.normalform
    bp = nfm.get_normal_form1d(it, br, 0, bls=alg.bls)
    assert bp.type == "Pitchfork" and abs(bp.nf["b30"] / 6 + 1) < 1e-10 and abs(bp.nf["b20"]) < 1e-10
    pred = nfm.predictor(bp, 0.01)
    assert pred.dsfactor == 1.0 and abs(pred.amp - np.sqrt(6 * 0.01 * 3.23 / 6)) < 1e-8
    br2, _ = nfm.continuation_from_bp(br, 0, prob, alg, dataclasses.replace(cp, p_max=0.2, max_steps=10), normC=bk.palc.norminf)
    st = br2.state
    assert st.z_p > bp.p and abs(st.z_u[0] ** 2 - 3.23 * st.z_p) < 1e-10 and abs(st.z_u[1]) < 1e-12


def test_rejections_follow_the_reference():
    """continuation(br, ind_bif) (src/bifdiagram/BranchSwitching.jl:107-160): a hopf point is an error, a kernel of dimension 2
    goes to multicontinuation (not implemented here), a Fold has no predictor and gives nothing"""
    bk = g.load_package()
    P, E, nfm = bk.palc, bk.events, bk.normalform
    _, prob, alg, cp, br, _ = _setup([-0.2, 0.0, 1.12, 0.234, 0.0])
    sp = br.specialpoint[0]
    br.specialpoint.append(dataclasses.replace(sp, type="hopf", delta=(2, 2)))
    br.specialpoint.append(dataclasses.replace(sp, type="nd", delta=(2, 0)))
    with pytest.raises(ValueError, match="hopf"):
        nfm.continuation_from_bp(br, len(br.specialpoint) - 2, prob, alg, cp, normC=P.norminf)
    with pytest.raises(NotImplementedError, match="multicontinuation"):
        nfm.continuation_from_bp(br, len(br.specialpoint) - 1, prob, alg, cp, normC=P.norminf)
    # a fold of x' = r + x - x^3 detected as a branch point by its eigenvalue: a01 = 1, so the normal form is a Fold
    Ff = lambda x, q: q[0] + x - x**3
    Jf = lambda x, q: np.diag(1 - 3 * x**2)

    class FoldProblem(NumpyProblem2):
        def d2F(self, x, p, a, b):
            return -6 * x * a * b

        def d3F(self, x, p, a, b, c):
            return -6 * a * b * c

    nopts = P.NewtonPar(tol=1e-12, linsolver=krylov.DefaultLS(), eigsolver=dense_eig)
    cpf = P.ContinuationPar(dsmin=0.001, dsmax=0.05, ds=-0.01, p_max=1.0, p_min=-1.0, detect_bifurcation=3, newton_options=nopts,
                            max_steps=200, n_inversion=6, detect_fold=False)
    pf = FoldProblem(Ff, Jf, np.array([1.2]), [0.5], 0)
    brf = E.continuation(pf, alg, cpf, normC=P.norminf)
    i = next(k for k, s in enumerate(brf.specialpoint) if s.type == "bp")
    assert abs(brf.specialpoint[i].param + 2 / (3 * np.sqrt(3))) < 1e-3
    assert nfm.get_normal_form1d(P.ContIterable(pf, alg, cpf, P.norminf), brf, i, bls=alg.bls).type == "Fold"
    assert nfm.continuation_from_bp(brf, i, pf, alg, cpf, normC=P.norminf) is None
    with pytest.raises(NotImplementedError, match="_predictor"):
        nfm.predictor(nfm.BranchPointNF("BranchPoint", np.zeros(1), 0.0, None, 0.0, np.ones(1), np.ones(1), {}), 0.1)


# ------------------------------------------------------------------------------------------------ 7. the jet kernels in SASS
def test_jet_kernels_are_in_the_sm_90a_code_without_local_memory():
    cnt = SR.mnemonics()
    jets = {k: c for k, c in cnt.items() if re.match(r"_Z5k_jetILi[23]E", k)}
    assert len(jets) == 2, sorted(cnt)[:5]
    for k, c in jets.items():
        assert c["LDL"] == 0 and c["STL"] == 0 and c["DFMA"] + c["DMUL"] >= 10, (k, dict(c))
