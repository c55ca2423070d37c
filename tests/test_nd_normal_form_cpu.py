"""CPU tests of the normal form of branch points with an N-dimensional kernel and of branch switching from them
(normalform.get_normal_formNd, predictor_nd, multicontinuation) on host problems, pinned to the reference's
test/normal_forms/testNF.jl:172-366; the N-border oracle of tests/nd_normal_form_oracle.py; the generic contraction helper
against numpy.einsum; and the sm_90a code of the jet-moment kernels (read with cuobjdump, no GPU needed).

Tolerances are the reference's 1e-10, except where noted."""
import dataclasses
import re

import numpy as np
import pytest

import __graft_entry__ as g
from oracle import krylov, bls as obls
from tests import nd_normal_form_oracle as NO, sass_reader as SR
from tests.test_codim2_curves_cpu import NumpyProblem2
from tests.test_host_logic_cpu import BlsAdapter
from tests.test_normal_form_cpu import dense_eig


class DenseBlockBLS:
    """solve_block on the assembled (n + m) bordered matrix by least squares.  Where the two-border system is singular (kernels of
    dimension > 2) the solution is defined up to its null space only; `drift` adds that much of every null vector to the
    minimum-norm solution, as an iterative solver may, and get_normal_formNd must project it away"""

    def __init__(self, drift=0.0):
        self.drift = drift

    def solve_block(self, J, a, b, c, rhst, rhsb, shift=None):
        n, m = len(rhst), len(a)
        A = np.zeros((n + m, n + m))
        A[:n, :n] = np.asarray(J)
        A[:n, n:] = np.column_stack(a)
        A[n:, :n] = np.vstack(b)
        A[n:, n:] = c
        sol = np.linalg.lstsq(A, np.concatenate([rhst, rhsb]), rcond=None)[0]
        _, sv, vt = np.linalg.svd(A)
        for v in vt[sv < 1e-12 * sv[0]]:
            sol = sol + self.drift * v
        return sol[:n], sol[n:], True, 1


class JetProblem(NumpyProblem2):
    """a host problem with its jets in x: d2F(x, params, a, b), d3F(x, params, a, b, c)"""

    def __init__(self, F, J, d2, d3, u0, params, lens):
        super().__init__(F, J, u0, params, lens)
        self.d2, self.d3 = d2, d3

    def d2F(self, x, p, a, b):
        return self.d2(x, self._par(p), a, b)

    def d3F(self, x, p, a, b, c):
        return self.d3(x, self._par(p), a, b, c)


def _branch(prob, **kw):
    """testNF.jl opts_br: the branch of prob with detect_bifurcation = 3, dense eigen-solves, PALC with a MatrixBLS"""
    bk = g.load_package()
    P = bk.palc
    nopts = P.NewtonPar(tol=1e-14, linsolver=krylov.DefaultLS(), eigsolver=dense_eig)
    cp = P.ContinuationPar(**{**dict(dsmin=0.001, dsmax=0.05, ds=0.01, p_max=0.4, p_min=-0.5, detect_bifurcation=3,
                                     newton_options=nopts, max_steps=100, n_inversion=8), **kw})
    alg = P.PALC(bls=BlsAdapter(obls.MatrixBLS()))
    br = bk.events.continuation(prob, alg, cp, normC=P.norminf)
    return bk, alg, cp, br, P.ContIterable(prob, alg, cp, P.norminf)


def _nd_point(br):
    i = next(k for k, s in enumerate(br.specialpoint) if s.type == "nd")
    return i, br.specialpoint[i]


def _symmetrize(t):
    """the mean over the permutations of the last axes of each row t[i]"""
    import itertools
    n = t.ndim - 1
    return np.mean([np.transpose(t, (0,) + tuple(1 + q for q in perm)) for perm in itertools.permutations(range(n))], axis=0)


# ------------------------------------------------------------------------------------------------ testNF.jl:172-222
@pytest.mark.parametrize("give_ad", [True, False])
def test_reduced_form_problem_gives_back_its_coefficients(give_ad):
    """The problem x' = reduced form of a random normal form (a01 = a02 = 0, b11 = P^-1 diag(-1, -0.123) P, symmetric b20 and
    b30): its branch point at mu = 0 has that normal form, with the adjoint basis given or computed from J'"""
    bk = g.load_package()
    nfm = bk.normalform
    rng = np.random.default_rng(11)
    Pm = rng.random((2, 2))
    nf = dict(a01=np.zeros(2), a02=np.zeros(2), b11=np.linalg.solve(Pm, np.diag([-1.0, -0.123]) @ Pm),
              b20=_symmetrize(rng.random((2, 2, 2))), b30=_symmetrize(rng.random((2, 2, 2, 2))))
    vf = nfm.NdBranchPointNF(np.zeros(2), 0.0, None, 0.0, [np.array([1.0, 0]), np.array([0, 1.0])], None, nf, "none")
    prob = JetProblem(lambda x, q: vf.reduced_form(x, q[0]), lambda x, q: vf.reduced_jacobian(x, q[0]),
                      lambda x, q, a, b: np.einsum("ijk,j,k->i", nf["b20"], a, b),
                      lambda x, q, a, b, c: np.einsum("ijkl,j,k,l->i", nf["b30"], a, b, c), np.zeros(2), [-0.1], 0)
    bk, alg, cp, br, it = _branch(prob, dsmax=0.01)
    i, pt = _nd_point(br)
    assert abs(pt.delta[0]) == 2
    br.specialpoint[i] = dataclasses.replace(pt, param=0.0)                          # @reset br.specialpoint[1].param = 0.
    bp = nfm.get_normal_formNd(it, br, i, zetas=[[1, 0.0], [0, 1.0]], zetas_ad=[[1, 0.0], [0, 1.0]] if give_ad else None,
                               bls=DenseBlockBLS())
    for k in ("a01", "b11", "b20", "b30"):
        assert np.max(np.abs(bp.nf[k] - nf[k])) < 1e-10, (k, bp.nf[k], nf[k])
    assert bp.nf["b20"].shape == (2, 2, 2) and bp.nf["b30"].shape == (2, 2, 2, 2)


# ------------------------------------------------------------------------------------------------ testNF.jl:224-287
def _fbp2d(q):
    al, g_, A, B, C = q["alpha"], q["gamma"], q["A"], q["B"], q["C"]

    def F(x, par):
        mu = par[0]
        return np.array([al * x[0] * (3.23 * mu + A * x[0] ** 2 + B * x[1] ** 2) + x[2],
                         al * x[1] * (3.23 * mu + C * x[0] ** 2 + A * x[1] ** 2),
                         -x[2] + g_ * (x[0] ** 3 + x[1] ** 2)])

    def J(x, par):
        mu = par[0]
        return np.array([[al * (3.23 * mu + 3 * A * x[0] ** 2 + B * x[1] ** 2), 2 * al * B * x[0] * x[1], 1.0],
                         [2 * al * C * x[0] * x[1], al * (3.23 * mu + C * x[0] ** 2 + 3 * A * x[1] ** 2), 0.0],
                         [3 * g_ * x[0] ** 2, 2 * g_ * x[1], -1.0]])

    def d2(x, par, a, b):
        return np.array([al * (6 * A * x[0] * a[0] * b[0] + 2 * B * (x[0] * a[1] * b[1] + x[1] * (a[0] * b[1] + a[1] * b[0]))),
                         al * (6 * A * x[1] * a[1] * b[1] + 2 * C * (x[1] * a[0] * b[0] + x[0] * (a[0] * b[1] + a[1] * b[0]))),
                         g_ * (6 * x[0] * a[0] * b[0] + 2 * a[1] * b[1])])

    def d3(x, par, a, b, c):
        s = lambda i, j, k: a[i] * b[j] * c[k] + a[i] * b[k] * c[j] + a[j] * b[i] * c[k] + a[j] * b[k] * c[i] + \
            a[k] * b[i] * c[j] + a[k] * b[j] * c[i]
        return np.array([al * (6 * A * a[0] * b[0] * c[0] + 2 * B * s(0, 1, 1) / 2),
                         al * (6 * A * a[1] * b[1] * c[1] + 2 * C * s(1, 0, 0) / 2),
                         6 * g_ * a[0] * b[0] * c[0]])
    return F, J, d2, d3


@pytest.mark.parametrize("gamma", [0.0, 10.0])
def test_fbp2d_normal_form(gamma):
    """Every value testNF.jl:277-285 asserts, and the reduced form (a02 set to 0) against Fbp2d + gamma (x1^3 + x2^2, 0) at
    mu = 0 (< 1e-9, :274); the N-border oracle gives the same tensors"""
    q = dict(alpha=-1.0, gamma=gamma, A=0.123, B=0.234, C=0.456)
    F, J, d2, d3 = _fbp2d(q)
    prob = JetProblem(F, J, d2, d3, np.zeros(3), [-0.2], 0)
    bk, alg, cp, br, it = _branch(prob)
    i, pt = _nd_point(br)
    assert abs(pt.delta[0]) == 2
    br.specialpoint[i] = dataclasses.replace(pt, param=0.0)
    nfm = bk.normalform
    bp = nfm.get_normal_formNd(it, br, i, zetas=[[1, 0, 0.0], [0, 1, 0.0]], zetas_ad=[[1, 0, 1.0], [0, 1.0, 0]], bls=DenseBlockBLS())
    nf = bp.nf
    al, A, B, C = q["alpha"], q["A"], q["B"], q["C"]
    assert np.allclose(bp.zetas[0], [1, 0, 0]) and np.allclose(bp.zetas[1], [0, 1, 0])
    assert abs(nf["b30"][0, 0, 0, 0] / 6 - (al * A + gamma)) < 1e-10
    assert abs(nf["b30"][0, 0, 1, 1] / 2 - al * B) < 1e-10
    assert abs(nf["b30"][0, 0, 0, 1] / 2) < 1e-10
    assert abs(nf["b30"][1, 0, 0, 1] / 2 - al * C) < 1e-10
    assert np.max(np.abs(nf["b20"][:, :, 0])) < 1e-10
    assert np.max(np.abs(nf["b20"][0] / 2 - [[0, 0], [0, gamma]])) < 1e-10
    assert np.max(np.abs(nf["b11"] - al * 3.23 * np.eye(2))) < 1e-10
    assert np.max(np.abs(nf["a01"])) < 1e-10
    assert bp.type == "2-d"
    nf["a02"][:] = 0
    for x in (np.concatenate([np.random.default_rng(2).random(2), [0.0]]), np.array([1.0, 0, 0]), np.array([0, 1.0, 0])):
        o1 = bp.reduced_form(x[:2], 0.0)
        o2 = F(x, [0.0])[:2] + gamma * np.array([x[0] ** 3 + x[1] ** 2, 0])
        assert np.max(np.abs(o1 - o2)) < 1e-9
    assert np.allclose(bp(np.array([0.5, -2.0]), 0.2), [0.5, -2.0, 0.0])
    ref = NO.nd_normal_form(lambda x, p: F(x, [p]), lambda p: J(np.zeros(3), [p]), lambda a, b: d2(np.zeros(3), [0.0], a, b),
                            lambda a, b, c: d3(np.zeros(3), [0.0], a, b, c), np.zeros(3), 0.0, prob.delta,
                            bp.zetas, bp.zetas_ad)
    for k in ("a01", "b11", "b20", "b30"):
        assert np.max(np.abs(ref[k] - nf[k])) < 1e-10, k
    # the adjoint basis recomputed from J' (the problem is not symmetric) gives the same normal form
    bp2 = nfm.get_normal_formNd(it, br, i, zetas=[[1, 0, 0.0], [0, 1, 0.0]], bls=DenseBlockBLS())
    for k in ("a01", "b11", "b20", "b30"):
        assert np.max(np.abs(bp2.nf[k] - nf[k])) < 1e-10, k


# ------------------------------------------------------------------------------------------------ testNF.jl:326-366
D6 = dict(a=0.3, b=1.5, c=2.9)


def _fbpD6(x, mu, a=D6["a"], b=D6["b"], c=D6["c"]):
    return np.array([mu * x[0] + (a * x[1] * x[2] - b * x[0] ** 3 - c * (x[1] ** 2 + x[2] ** 2) * x[0]),
                     mu * x[1] + (a * x[0] * x[2] - b * x[1] ** 3 - c * (x[2] ** 2 + x[0] ** 2) * x[1]),
                     mu * x[2] + (a * x[0] * x[1] - b * x[2] ** 3 - c * (x[1] ** 2 + x[0] ** 2) * x[2])])


def _d6_problem():
    a, b, c = D6["a"], D6["b"], D6["c"]
    T2 = np.zeros((3, 3, 3))
    T3 = np.zeros((3, 3, 3, 3))
    for i in range(3):
        j, k = [m for m in range(3) if m != i]
        T2[i, j, k] = T2[i, k, j] = a
        T3[i, i, i, i] = -6 * b
        for m in (j, k):
            for perm in ((i, m, m), (m, i, m), (m, m, i)):
                T3[(i,) + perm] = -2 * c
    # F = mu x + T2[x, x] / 2 + T3[x, x, x] / 6, so J = mu I + T2[x] + T3[x, x] / 2
    J = lambda x, q: q[0] * np.eye(3) + np.einsum("ijk,k->ij", T2, x) + np.einsum("ijkl,k,l->ij", T3, x, x) / 2
    d2 = lambda x, q, u, v: np.einsum("ijk,j,k->i", T2, u, v) + np.einsum("ijkl,j,k,l->i", T3, u, v, x)
    d3 = lambda x, q, u, v, w: np.einsum("ijkl,j,k,l->i", T3, u, v, w)
    return JetProblem(lambda x, q: _fbpD6(x, q[0]), J, d2, d3, np.zeros(3), [-0.2], 0)


def test_d6_normal_form_and_multicontinuation():
    """testNF.jl:333-357: a01 = 0, b11 = I, b30[1,1,1,1] / 6 = -b, b30[1,1,2,2] / 2 = -c, b20[1,2,3] = a; the reduced form equals
    FbpD6 at mu = 0.001 to 1e-12; every branch multicontinuation gives solves FbpD6"""
    bk = g.load_package()
    nfm, P = bk.normalform, bk.palc
    prob = _d6_problem()
    bk, alg, cp, br, it = _branch(prob, n_inversion=6, ds=0.001)
    i, pt = _nd_point(br)
    assert abs(pt.delta[0]) == 3
    eye = [[1, 0, 0.0], [0, 1, 0.0], [0, 0, 1.0]]
    bp = nfm.get_normal_formNd(it, br, i, zetas=eye, bls=DenseBlockBLS())
    nf = bp.nf
    assert np.all(nf["a01"] == 0)
    assert np.max(np.abs(nf["b11"] - np.eye(3))) < 1e-7   # central differences of J = mu I with delta = sqrt(eps)
    assert abs(nf["b30"][0, 0, 0, 0] / 6 + D6["b"]) < 1e-10
    assert abs(nf["b30"][0, 0, 1, 1] / 2 + D6["c"]) < 1e-10
    assert abs(nf["b20"][0, 1, 2] - D6["a"]) < 1e-10
    x0 = np.random.default_rng(5).random(3)
    # b11 = I only to the rounding of its central difference (~1e-9), which 0.001 |x| scales down to below 1e-11
    assert np.max(np.abs(_fbpD6(x0, 0.001) - bp.reduced_form(x0, 0.001))) < 1e-11
    # the oracle's three-border solves give the same tensors
    ref = NO.nd_normal_form(prob.F, lambda p: prob.J(np.zeros(3), p), lambda u, v: prob.d2F(np.zeros(3), bp.p, u, v),
                            lambda u, v, w: prob.d3F(np.zeros(3), bp.p, u, v, w), np.zeros(3), bp.p, prob.delta, bp.zetas,
                            bp.zetas_ad)
    for k in ("a01", "b11", "b20", "b30"):
        assert np.max(np.abs(ref[k] - nf[k])) < 1e-10, k
    states = []
    cp2 = dataclasses.replace(cp, n_inversion=4, dsmax=0.005, ds=0.001, max_steps=12, p_max=1.0, detect_bifurcation=0)
    out = nfm.multicontinuation(br, i, prob, alg, cp2, normC=P.norminf, bpnf=bp,
                                callback=lambda st: states.append((st.z_u.copy(), st.z_p)) or True)
    assert len(out) >= 2 and all(b is bp for _, b in out)
    assert len(states) >= 10 * len(out)
    for u, mu in states:
        assert np.max(np.abs(_fbpD6(u, mu))) < 1e-12
    nontrivial = [br2 for br2, _ in out if np.max(np.abs(br2.state.z_u)) > 1e-3]
    assert len(nontrivial) == len(out)
    print(f"D6: {len(out)} branches")


def test_gram_projection_of_a_three_dimensional_kernel():
    """A kernel of dimension 3 whose singular solves have components outside the kernel (x4 = 0 is slaved to x1..x3): the
    two-border solves (minimum norm, then projected to <ζ_i, ψ> = 0) give the oracle's three-border tensors"""
    bk = g.load_package()
    nfm = bk.normalform
    rng = np.random.default_rng(3)
    T2 = _symmetrize(rng.standard_normal((4, 4, 4)))
    T3 = _symmetrize(rng.standard_normal((4, 4, 4, 4)))
    D = np.diag([1.0, 1.0, 1.0, 0.0])
    L = np.diag([0.0, 0.0, 0.0, -1.0])

    def F(x, q):
        return q[0] * D @ x + L @ x + np.einsum("ijk,j,k->i", T2, x, x) / 2 + np.einsum("ijkl,j,k,l->i", T3, x, x, x) / 6

    J = lambda x, q: q[0] * D + L + np.einsum("ijk,k->ij", T2, x) + np.einsum("ijkl,k,l->ij", T3, x, x) / 2
    d2 = lambda x, q, u, v: np.einsum("ijk,j,k->i", T2, u, v) + np.einsum("ijkl,j,k,l->i", T3, u, v, x)
    d3 = lambda x, q, u, v, w: np.einsum("ijkl,j,k,l->i", T3, u, v, w)
    prob = JetProblem(F, J, d2, d3, np.zeros(4), [-0.2], 0)
    bk, alg, cp, br, it = _branch(prob, n_inversion=6, ds=0.001, max_steps=40)
    i, pt = _nd_point(br)
    assert abs(pt.delta[0]) == 3
    br.specialpoint[i] = dataclasses.replace(pt, param=0.0, x=np.zeros(4))
    Z = [[1, 0, 0, 0.0], [0, 1, 0, 0.0], [0, 0, 1, 0.0]]
    bp = nfm.get_normal_formNd(it, br, i, zetas=Z, zetas_ad=Z, bls=DenseBlockBLS(drift=0.7))
    x0 = np.zeros(4)
    ref = NO.nd_normal_form(lambda x, p: F(x, [p]), lambda p: J(x0, [p]), lambda u, v: d2(x0, [0.0], u, v), lambda u, v, w: d3(x0, [0.0], u, v, w), x0, 0.0,
                            prob.delta, bp.zetas, bp.zetas_ad)
    assert np.max(np.abs(ref["b30"])) > 1.0
    for k in ("a01", "b11", "b20", "b30"):
        assert np.max(np.abs(ref[k] - bp.nf[k])) < 1e-10, k


# ------------------------------------------------------------------------------------------------ predictor_nd
def test_predictor_finds_the_closed_form_roots_reproducibly():
    """Two decoupled pitchforks x_i' = dp x_i - x_i^3: nine roots (0, ±sqrt(dp))^2 after the point, the trivial one before; the
    same generator seed gives the same roots in the same order.  dp = 0.5 puts the roots at the scale of the vertex guesses
    {-1, 0, 1}^2; deflated Newton from those guesses is not bound to find every root of a smaller-scale equation (at dp = 0.04
    it finds 3 to 4 of the 9), in the reference as here"""
    nfm = g.load_package().normalform
    b30 = np.zeros((2, 2, 2, 2))
    b30[0, 0, 0, 0] = b30[1, 1, 1, 1] = -6.0
    nf = dict(a01=np.zeros(2), a02=np.zeros(2), b11=np.eye(2), b20=np.zeros((2, 2, 2)), b30=b30)
    bp = nfm.NdBranchPointNF(np.zeros(2), 0.0, None, 0.0, [np.array([1.0, 0]), np.array([0, 1.0])], None, nf, "2-d")
    dp = 0.5
    before, after = nfm.predictor_nd(bp, dp, rng=np.random.default_rng(3), nbfailures=10)
    assert len(before) == 1 and np.all(before[0] == 0)
    s = np.sqrt(dp)
    want = sorted((a, b) for a in (-s, 0.0, s) for b in (-s, 0.0, s))
    got = sorted(tuple(np.round(r, 12) + 0.0) for r in after)
    assert len(after) == 9 and np.allclose(got, want, atol=1e-12), got
    assert np.all(after[0] == 0)
    before2, after2 = nfm.predictor_nd(bp, dp, rng=np.random.default_rng(3), nbfailures=10)
    assert len(after2) == len(after) and all(np.array_equal(a, b) for a, b in zip(after, after2))


# ------------------------------------------------------------------------------------------------ the contraction helper
def test_composed_contractions_match_einsum():
    """jet_moments_composed (a jet call and a dot product per tuple, the path of host problems) against numpy.einsum on a problem
    whose jets are the contractions of random tensors"""
    nfm = g.load_package().normalform
    rng = np.random.default_rng(4)
    n, nvec = 7, 5
    T2, T3 = rng.standard_normal((n, n, n)), rng.standard_normal((n, n, n, n))
    prob = JetProblem(None, None, lambda x, q, a, b: np.einsum("ijk,j,k->i", T2, a, b),
                      lambda x, q, a, b, c: np.einsum("ijkl,j,k,l->i", T3, a, b, c), np.zeros(n), [0.0], 0)
    Vm = rng.standard_normal((nvec, n))
    idx2 = rng.integers(0, nvec, (20, 3))
    idx3 = rng.integers(0, nvec, (15, 4))
    idx2[0] = (1, 1, 1)
    got = nfm.jet_moments(prob, np.zeros(n), 0.0, list(Vm), idx2, idx3)
    m2 = np.einsum("ap,pqr,bq,cr->abc", Vm, T2, Vm, Vm)
    m3 = np.einsum("ap,pqrs,bq,cr,ds->abcd", Vm, T3, Vm, Vm, Vm)
    want = np.concatenate([m2[tuple(idx2.T)], m3[tuple(idx3.T)]])
    assert np.max(np.abs(got - want)) < 1e-12 * np.max(np.abs(want))
    assert len(nfm.jet_moments(prob, np.zeros(n), 0.0, list(Vm))) == 0


def test_continuation_from_bp_points_to_multicontinuation():
    bk = g.load_package()
    prob = _d6_problem()
    bk, alg, cp, br, it = _branch(prob, n_inversion=6, ds=0.001)
    i, _ = _nd_point(br)
    with pytest.raises(NotImplementedError, match="normalform.multicontinuation"):
        bk.normalform.continuation_from_bp(br, i, prob, alg, cp, normC=bk.palc.norminf)


# ------------------------------------------------------------------------------------------------ the moment kernels in SASS
def test_jet_moment_kernels_are_in_the_sm_90a_code_without_local_memory():
    cnt = SR.mnemonics()
    mom = {k: c for k, c in cnt.items() if re.match(r"_Z13k_jet_momentsILi(1|2|4)E", k)}
    assert len(mom) == 3, sorted(cnt)[:5]                     # chan, the SH kinds, cGL2d
    for k, c in mom.items():
        assert c["LDL"] == 0 and c["STL"] == 0 and c["DFMA"] >= 4 and c["LDS"] >= 3, (k, dict(c))
    assert any("k_jet_moments_fold" in k for k in cnt)
    usage = {k: u for k, u in SR.resources().items() if "k_jet_moments" in k}
    assert all(u.stack == 0 for u in usage.values()) and len(usage) == 4, usage
