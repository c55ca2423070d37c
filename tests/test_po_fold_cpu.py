"""CPU tests of the folds of periodic orbits (periodic.continuation_po_events, newton_fold_po, continuation_fold_po) on a host twin
of the Trapeze problem: the sparse Trapeze Jacobian of tests/potrap_sparse_oracle.py against the Trapeze JVP, the fold of cycles
of Stuart-Landau against its closed form, and the sm_90a code of the J' kernels (read with cuobjdump, no GPU needed)."""
import numpy as np
import pytest

import __graft_entry__ as g
from oracle import krylov, bls as obls, potrap, problems
from tests import potrap_sparse_oracle as PS, sass_reader as SR
from tests.test_hopf_po_cpu import Fsl, JFsl, SLProblem
from tests.test_host_logic_cpu import BlsAdapter, DenseComplexProblem, _dense_cls
from tests.test_normal_form_cpu import dense_eig

SUB = dict(r=-0.1, mu=0.132, nu=1.0, c3=-1.0, c5=1.0)   # c3 < 0 < c5: subcritical Hopf point, a fold of cycles at r* = -c3^2 / (4 c5)
M = 10


def _jvp_columns(tr, x):
    return np.column_stack([tr.jvp(x, e) for e in np.eye(len(x))])


def test_sparse_oracle_matches_the_trapeze_jvp():
    """po_jacobian_sparse (analytic period column) equals the Trapeze JVP column by column, on cGL 6 x 4 with M = 5 and on
    Stuart-Landau with M = 10"""
    rng = np.random.default_rng(5)
    gl = problems.GinzburgLandau2D(6, 4, np.pi, np.pi / 2, r=0.7, mu=0.1, nu=1.0, c3=-1.0, c5=1.0)
    m = 5
    x = rng.standard_normal(gl.N * m + 1)
    x[-1] = 4.2
    phi = rng.standard_normal(gl.N * m)
    J = PS.cgl_po_jacobian(gl, x, m, phi).toarray()
    ref = _jvp_columns(potrap.Trapeze(gl.F, gl.dF, phi, np.zeros_like(phi), m, gl.N), x)
    assert np.abs(J - ref).max() < 1e-12 * np.abs(ref).max()
    q = list(SUB.values())
    y = rng.standard_normal(2 * M + 1)
    y[-1] = 6.0
    phs = rng.standard_normal(2 * M)
    Js = PS.po_jacobian_sparse(lambda u: JFsl(u, q), lambda u: Fsl(u, q), y, M, 2, phs).toarray()
    refs = _jvp_columns(potrap.Trapeze(lambda u: Fsl(u, q), lambda u, du: JFsl(u, q) @ du, phs, np.zeros(2 * M), M, 2), y)
    assert np.abs(Js - refs).max() < 1e-13 * np.abs(refs).max()


class SLTrap:
    """Host twin of periodic.TrapezeProblemB200 over Stuart-Landau: oracle.potrap.Trapeze for F, the sparse oracle for J and J'"""

    @staticmethod
    def make(bk, params):
        base = bk.periodic.TrapezeProblemB200

        class Twin(base):
            def __init__(self):
                base.__init__(self, None, None, list(params), 0, M=M)
                self.tr = potrap.Trapeze(None, None, np.zeros(2 * M), np.zeros(2 * M), M, 2)

            def _set(self, p):
                q = list(self.params)
                q[self.lens] = p
                self.q = q
                self.tr.F = lambda u: Fsl(u, q)
                self.tr.dF = lambda u, du: JFsl(u, q) @ du

            def F(self, x, p, out=None):
                self._set(p)
                r = self.tr.residual(x)
                if out is not None:
                    out[...] = r
                    return out
                return r

            def J(self, x, p):
                self.last_state, self.last_p = x, p
                self._set(p)
                q = self.q
                return PS.po_jacobian_sparse(lambda u: JFsl(u, q), lambda u: Fsl(u, q), x, M, 2, self.tr.phi)

            def Jt(self, x, p):
                return self.J(x, p).T.tocsr()

            def update_section(self, x, scale):
                F = self.tr.F
                self.tr.phi = np.concatenate([scale * F(u) for u in x[:-1].reshape(M, 2)])
                self.tr.xpi = x[:-1].copy()
        return Twin()


@pytest.fixture(scope="module")
def sl_fold():
    """the trivial branch of subcritical Stuart-Landau through its Hopf point at r = 0, the orbit branch switched from it with
    fold detection by parameter monotony, and the fold it records"""
    bk = g.load_package()
    P = bk.palc
    prob = SLProblem(Fsl, JFsl, np.zeros(2), list(SUB.values()), 0)
    nopts = P.NewtonPar(tol=1e-12, linsolver=krylov.DefaultLS(), eigsolver=dense_eig)
    cp = P.ContinuationPar(dsmin=0.001, dsmax=0.02, ds=0.01, p_max=0.1, p_min=-0.3, detect_bifurcation=3, newton_options=nopts)
    alg = P.PALC(bls=BlsAdapter(obls.MatrixBLS()))
    br = bk.events.continuation(prob, alg, cp, normC=P.norminf)
    ind = next(i for i, s in enumerate(br.specialpoint) if s.type == "hopf")
    it = P.ContIterable(prob, alg, cp, P.norminf)
    trap = SLTrap.make(bk, list(SUB.values()))
    ls = krylov.DefaultLS()
    cpo = P.ContinuationPar(dsmin=1e-4, dsmax=0.05, ds=0.01, p_min=-0.5, p_max=0.3, max_steps=40,
                            newton_options=P.NewtonPar(tol=1e-11, max_iterations=15, linsolver=ls))
    bpo, st, hp, pred = bk.periodic.continuation_from_hopf(it, br, ind, cpo, trap, cprob=DenseComplexProblem(prob.J), cls=_dense_cls,
                                                          bls=BlsAdapter(obls.BorderingBLS(ls, check_precision=False)),
                                                          with_events=True)
    # the first rows may turn next to the Hopf point, where the orbits shrink to the equilibrium: the fold of cycles is the
    # turning point away from it (the example, too, picks its fold by index, examples/cGL2d.jl:351)
    folds = [i for i, s in enumerate(bpo.specialpoint) if s.type == "fold" and s.param < -0.1]
    return dict(bk=bk, trap=trap, br=bpo, hp=hp, folds=folds, ls=ls)


def _closed_form(c3, c5):
    r = -c3**2 / (4 * c5)
    rho2 = -c3 / (2 * c5)
    T = 2 * M * np.tan(np.pi / (M - 1)) / (SUB["nu"] - SUB["mu"] * rho2)
    return r, rho2, T


def test_the_branch_from_the_subcritical_hopf_point_records_a_fold(sl_fold):
    br = sl_fold["br"]
    assert sl_fold["hp"].type == "SubCritical"
    assert len(sl_fold["folds"]) == 1
    sp0 = br.specialpoint[sl_fold["folds"][0]]
    r_star = _closed_form(SUB["c3"], SUB["c5"])[0]
    params = [row["param"] for row in br.rows]
    k = sp0.idx
    assert params[k] == min(params[k - 1: k + 2]) and min(params) >= r_star - 1e-12     # the turning row; no orbit below r*
    assert sp0.tau_u is not None and len(sp0.tau_u) == 2 * M + 1


def test_newton_fold_po_gives_the_closed_form_fold(sl_fold):
    """r* = -c3^2 / (4 c5), rho*^2 = -c3 / (2 c5), T* = 2 M tan(pi / (M - 1)) / (nu - mu rho*^2)"""
    bk, trap = sl_fold["bk"], sl_fold["trap"]
    P = bk.palc
    opts = P.NewtonPar(tol=1e-12, max_iterations=15, linsolver=sl_fold["ls"])
    sol = bk.periodic.newton_fold_po(trap, sl_fold["br"], sl_fold["folds"][0], opts, BlsAdapter(obls.MatrixBLS()))
    assert sol.converged, sol.residuals
    r, rho2, T = _closed_form(SUB["c3"], SUB["c5"])
    u = sol.u[:-1].reshape(M, 2)
    assert abs(sol.p - r) < 1e-10, sol.p
    assert np.abs(np.sum(u**2, axis=1) - rho2).max() < 1e-10
    assert abs(sol.u[-1] - T) < 1e-9
    with pytest.raises(ValueError):
        bk.periodic.fold_point(sl_fold["br"], len(sl_fold["br"].specialpoint) - 1)   # the endpoint


def test_continuation_fold_po_follows_the_closed_form_in_c5(sl_fold):
    """the fold of cycles continued in c5: r = -c3^2 / (4 c5) on every row"""
    bk, trap = sl_fold["bk"], sl_fold["trap"]
    P = bk.palc
    cp = P.ContinuationPar(dsmin=1e-4, dsmax=0.05, ds=0.02, p_min=0.5, p_max=3.0, max_steps=10,
                           newton_options=P.NewtonPar(tol=1e-12, max_iterations=10))
    curve = bk.periodic.continuation_fold_po(trap, sl_fold["br"], sl_fold["folds"][0], 4, cp, BlsAdapter(obls.MatrixBLS()))
    assert len(curve.rows) >= 9
    for p1, c5 in zip(curve.p1, curve.p2):
        assert abs(p1 - _closed_form(SUB["c3"], c5)[0]) < 1e-9, (p1, c5)
    assert trap.params[4] == SUB["c5"]


# ------------------------------------------------------------------------------------------------ sm_90a code
def test_adjoint_kernels_are_in_the_sm_90a_code():
    """k_potrap_apply_tr uses no local memory.  k_potrap_time<true> (the transposed solve), like k_potrap_time<false>, keeps its
    four per-thread arrays of BK_PO_KMAX double2 (the time DFT of one spatial mode) in local memory: it has exactly the forward
    kernel's stack frame, 4096 bytes, with no spills (ptxas reports LOCAL:0, i.e. no spill space) and the same register count"""
    cnt = SR.mnemonics()
    tr = [c for k, c in cnt.items() if "k_potrap_apply_tr" in k]
    assert len(tr) == 1
    assert tr[0]["LDL"] == 0 and tr[0]["STL"] == 0 and tr[0]["DFMA"] + tr[0]["DMUL"] >= 20, dict(tr[0])
    time_tr = [c for k, c in cnt.items() if "k_potrap_timeILb1E" in k]   # mangled k_potrap_time<true>
    time = [c for k, c in cnt.items() if "k_potrap_timeILb0E" in k]
    assert len(time_tr) == 1 and len(time) == 1
    assert "arch = sm_90a" in SR.cuobjdump("-sass")
    usage = SR.resources()
    fwd = next(v for k, v in usage.items() if "k_potrap_timeILb0E" in k)
    trn = next(v for k, v in usage.items() if "k_potrap_timeILb1E" in k)
    app = next(v for k, v in usage.items() if "k_potrap_apply_tr" in k)
    assert trn == fwd and fwd.stack == 4096 and fwd.local == 0, (trn, fwd)
    assert app.stack == 0 and app.local == 0, app
