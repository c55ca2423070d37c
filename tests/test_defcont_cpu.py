"""CPU tests of deflated continuation (defcont.py) and of the fused deflation formulas (deflation.fused_values): the reference's
known answers of test/continuation/simple_continuation.jl:381-431 on host vectors; M and dM from the moments against the
composed loop, with the moments restated on the host in long double; the closed-form autodiff derivative against a complex
step; and the sm_90a code of the deflation-moment kernels (read with cuobjdump, no GPU needed)."""
import collections
import re

import numpy as np
import pytest

import __graft_entry__ as g
from oracle import krylov
from tests import sass_reader as SR
from tests.test_normal_form_cpu import dense_eig


class HostProblem:
    """a scalar-parameter problem on host arrays, with the record u[0] so that rows give the point itself"""

    def __init__(self, F, J, u0, p0):
        self.F_, self.J_, self.u0, self.p0 = F, J, u0, p0
        self.delta = float(np.sqrt(np.finfo(float).eps))
        self.record = lambda x: float(x[0])

    def F(self, x, p, out=None):
        r = self.F_(x, p)
        if out is not None:
            out[...] = r
            return out
        return r

    def J(self, x, p):
        return self.J_(x, p)


def _opts(P, **kw):
    """the `opts` of simple_continuation.jl:126 with the changes of the DefCont calls"""
    base = dict(dsmax=0.051, dsmin=1e-3, ds=0.001, max_steps=140, p_min=-3.0, detect_bifurcation=3)
    nkw = kw.pop("newton", {})
    base.update(kw)
    return P.ContinuationPar(**base, newton_options=P.NewtonPar(tol=1e-8, linsolver=krylov.DefaultLS(), eigsolver=dense_eig, **nkw))


def test_defcont_f_simple_saves_only_solutions():
    """simple_continuation.jl:390-411: F_simple with DeflationOperator(2, 0.001, [[0]]) and a seeded perturbation; every saved
    point of every branch is a solution (norminf(F) < tol), as the reference asserts"""
    bk = g.load_package()
    P, D, DC = bk.palc, bk.deflation, bk.defcont
    F = lambda x, p: p * x + x**3 / 3 + 0.01
    J = lambda x, p: np.diag(p + x**2)
    prob = HostProblem(F, J, np.array([0.0]), 0.5)
    rng = np.random.default_rng(0)
    alg = DC.DefCont(deflation_operator=D.DeflationOperator(2, 0.001, [np.array([0.0])]),
                     perturb_solution=lambda x, p, idb: x + 0.1 * rng.random(len(x)))
    cp = _opts(P, ds=-0.001, max_steps=800, newton=dict(max_iterations=6))
    res = DC.continuation(prob, alg, cp, normC=P.norminf, callback_newton=P.cbMaxNorm(1e3), save_sol_every_step=0)
    assert len(res.branches) >= 2
    nsaved = 0
    for br in res.branches:
        for s in br.sol:
            assert P.norminf(F(s["x"], s["p"])) < cp.newton_options.tol
            nsaved += 1
        for r in br.rows:                       # the recorded points too: u[0] solves the scalar equation
            assert abs(F(np.array([r["x"]]), r["param"])[0]) < 1e-7
    assert nsaved >= len(res.branches)


def _f2_run(perturb):
    bk = g.load_package()
    P, D, DC = bk.palc, bk.deflation, bk.defcont
    F = lambda u, p: -u * (p + u * (2 - 5 * u)) * (p - 0.15 - u * (2 + 20 * u))

    def J(u, p):
        a, b = p + u * (2 - 5 * u), p - 0.15 - u * (2 + 20 * u)
        return np.diag(-(a * b) - u * ((2 - 10 * u) * b + a * (-2 - 40 * u)))

    prob = HostProblem(F, J, np.array([0.0]), 0.3)
    per_step = collections.Counter()        # branches continued at each parameter value

    def push(defop, x, p):
        per_step[p] += 1
        defop.push(x)

    kw = dict(perturb_solution=perturb) if perturb else {}
    alg = DC.DefCont(deflation_operator=D.DeflationOperator(2, 0.001, [np.array([0.0]), np.array([0.05])]), max_branches=6,
                     update_deflation_op=push, **kw)
    cp = _opts(P, dsmin=1e-4, ds=-0.002, max_steps=800, p_min=-0.8, newton=dict(max_iterations=15))
    res = DC.continuation(prob, alg, cp, callback_newton=P.cbMaxNorm(1e6))
    curves = [lambda u, p: abs(u), lambda u, p: abs(p + u * (2 - 5 * u)), lambda u, p: abs(p - 0.15 - u * (2 + 20 * u))]
    found = set()
    for br in res.branches:
        for r in br.rows:
            d = [c(r["x"], r["param"]) for c in curves]
            assert min(d) < 1e-6, (r["x"], r["param"], d)
            found.add(int(np.argmin(d)))
    assert len(per_step) > 500 and max(per_step.values()) <= 6
    assert len(res.sol) == sum(s.isactive for s in res.states) <= 6
    return found, res


def test_defcont_f2_as_the_reference_calls_it():
    """simple_continuation.jl:417-423: F2 = -u (p + u (2 - 5u)) (p - 0.15 - u (2 + 20u)) with roots [[0], [0.05]],
    max_branches = 6, ds = -0.002, p_min = -0.8, no perturbation.  Every branch starts from roots[1] = 0 (:162-163), and every
    search for a new solution starts exactly on the deflated root u = 0, where M = 1/0 (the reference's residual is NaN): only
    u = 0 is followed.  Every saved point lies on a solution curve; no more than 6 branches are ever active."""
    found, res = _f2_run(None)
    assert found == {0}
    assert [s.isactive for s in res.states] == [True, False]    # the second copy of the start dies on the first step


def test_defcont_f2_with_a_perturbation_finds_the_three_curves():
    """the same run with the seeded perturbation of the F_simple call (x + 0.1 rand): every saved point lies on u = 0,
    p = -u (2 - 5u) or p = 0.15 + u (2 + 20u), each curve is found, no more than 6 branches are ever active"""
    rng = np.random.default_rng(1)
    found, res = _f2_run(lambda x, p, idb: x + 0.1 * rng.random(len(x)))
    assert found == {0, 1, 2}


# ------------------------------------------------------------------------------------------------ the fused formulas
def _moments_ld(u, roots, dirs):
    """bk_deflation_moments restated in long double"""
    L = np.longdouble
    u = u.astype(L)
    d = [u - r.astype(L) for r in roots]
    h = [x.astype(L) for x in dirs]
    s = np.array([np.dot(x, x) for x in d], dtype=L)
    m = np.array([np.max(np.abs(x)) for x in d], dtype=L)
    t = np.array([[np.dot(x, y) for y in h] for x in d], dtype=L).reshape(len(roots), len(dirs))
    q = np.array([[np.dot(a, b) for b in h] for a in h], dtype=L).reshape(len(dirs), len(dirs))
    return s, m, t, q


def _case(seed, n=200, nroots=7, scale=1.0):
    rng = np.random.default_rng(seed)
    u = rng.standard_normal(n)
    roots = [u + scale * rng.standard_normal(n) for _ in range(nroots)]
    dirs = [rng.standard_normal(n), rng.standard_normal(n)]
    return u, roots, dirs


@pytest.mark.parametrize("acc", ["prod", "mean"])
@pytest.mark.parametrize("power", [1, 2])
def test_fused_m_and_forward_difference_against_the_composed_loop(acc, power):
    """M to 1e-14 relative.  The forward differences differ by the rounding of the two M(u + delta h): the composed loop rounds
    u + delta h entry by entry (relative error eps max|u| / |d_i| in each s_i), the fused form rounds s_i + 2 delta t_i +
    delta^2 q (relative error ~ eps); through M that is at most 4 p eps M (1 + max|u| / min|d_i|) per root, divided by delta."""
    bk = g.load_package()
    D = bk.deflation
    eps = np.finfo(float).eps
    for seed in range(4):
        u, roots, dirs = _case(seed)
        op = D.DeflationOperator(power, 0.5, roots, accumulator=acc)
        s, m, t, q = _moments_ld(u, roots, dirs)
        M, dM = D.fused_values(power, 0.5, acc, s.astype(float), t.astype(float), q.astype(float), op.delta)
        Mc = op(u)
        assert abs(M - Mc) <= 1e-14 * abs(Mc)
        dmin = min(np.linalg.norm(u - r) for r in roots)
        bound = 4 * power * len(roots) * eps * abs(Mc) * (1 + np.max(np.abs(u)) / dmin) / op.delta
        for a, h in enumerate(dirs):
            assert abs(dM[a] - op.dM(u, h)) <= bound, (a, dM[a], op.dM(u, h), bound)


@pytest.mark.parametrize("acc", ["prod", "mean"])
def test_autodiff_derivative_against_a_complex_step(acc):
    """the closed form of autodiff = true on the moments, and on the composed path, against Im M(u + i eps h) / eps"""
    bk = g.load_package()
    D = bk.deflation
    for seed in range(3):
        u, roots, dirs = _case(10 + seed, nroots=5)
        for power in (1, 2, 3):
            def Mc(z):
                vals = [1.0 / np.dot(z - r, z - r) ** power + 0.3 for r in roots]
                out = vals[0]
                for v in vals[1:]:
                    out = out * v if acc == "prod" else out + v
                return out / len(vals) if acc == "mean" else out
            s, m, t, q = _moments_ld(u, roots, dirs)
            _, dM = D.fused_values(power, 0.3, acc, s.astype(float), t.astype(float), q.astype(float), autodiff=True)
            op = D.DeflationOperator(power, 0.3, roots, accumulator=acc, autodiff=True)
            for a, h in enumerate(dirs):
                ref = (Mc(u + 1e-30j * h)).imag / 1e-30
                assert abs(dM[a] - ref) <= 1e-12 * abs(ref), (power, a, dM[a], ref)
                assert abs(op.dM(u, h) - ref) <= 1e-12 * abs(ref)


def test_host_vectors_and_custom_distances_take_the_composed_loop():
    """fused=True on host vectors, or with a distance other than the prefix dot, is the composed loop bit for bit"""
    bk = g.load_package()
    D = bk.deflation
    u, roots, dirs = _case(3)
    ref = D.DeflationOperator(2, 1.0, roots)
    for op in (D.DeflationOperator(2, 1.0, roots, fused=True),
               D.DeflationOperator(2, 1.0, roots, dot=lambda x, y: float(np.dot(x, y)), fused=True)):
        assert not op.runs_fused(u)
        assert op(u) == ref(u) and op.dM(u, dirs[0]) == ref.dM(u, dirs[0])
    pre = D.DeflationOperator(2, 1.0, roots, dot=D.PrefixDot(150))
    sub = D.DeflationOperator(2, 1.0, [r[:150].copy() for r in roots])
    assert pre(u) == sub(u[:150].copy())


def test_newton_callback_stops_and_marks_unconverged():
    """palc.newton's callback (src/Newton.jl:87,108,111): cbMaxNorm stops the iteration once the residual reaches maxres; with
    no callback the iterates are unchanged"""
    bk = g.load_package()
    P = bk.palc
    prob = HostProblem(lambda x, p: x**3 - p, lambda x, p: np.diag(3 * x**2), np.array([3.0]), 1.0)
    opts = P.NewtonPar(tol=1e-12, max_iterations=30, linsolver=krylov.DefaultLS())
    a = P.newton(prob, prob.u0, 1.0, opts)
    b = P.newton(prob, prob.u0, 1.0, opts, callback=P.cbMaxNorm(1e6))
    assert a.converged and b.converged and a.residuals == b.residuals
    c = P.newton(prob, prob.u0, 1.0, opts, callback=P.cbMaxNorm(1.0))
    assert not c.converged and c.itnewton == 0


# ------------------------------------------------------------------------------------------------ the kernels in SASS
def test_deflation_moment_kernels_are_in_the_sm_90a_code_without_local_memory():
    cnt = SR.mnemonics()
    mom = {k: c for k, c in cnt.items() if re.match(r"_Z19k_deflation_momentsILi(0|1|2)E", k)}
    assert len(mom) == 3, sorted(cnt)[:5]                     # 0, 1 and 2 directions
    for k, c in mom.items():
        assert c["LDL"] == 0 and c["STL"] == 0 and c["DFMA"] >= 4 and c["SHFL"] >= 5, (k, dict(c))
    assert any("k_deflation_moments_fold" in k for k in cnt)
    usage = {k: u for k, u in SR.resources().items() if "k_deflation_moments" in k}
    assert all(u.stack == 0 for u in usage.values()) and len(usage) == 4, usage
