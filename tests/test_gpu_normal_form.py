"""GPU tests of bk_d2f / bk_d3f against the NumPy jets (tests/jets_oracle.py) and finite differences of bk_jvp / bk_d2f; the
simple-branch-point normal form (normalform.get_normal_form1d) at the closed-form branch points of the trivial Swift-Hohenberg
state; and branch switching (normalform.continuation_from_bp) from one of them, all with device vectors."""
import dataclasses

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

import __graft_entry__ as g
from oracle import problems
from tests import jets_oracle as JO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


def _rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300)


# ------------------------------------------------------------------------------------------------ jets
CGL_PAR = (0.5, 0.1, 1.0, -1.0, 1.0)   # (r, mu, nu, c3, c5)


def _jet_case(bk, name, dims):
    """(context, N, jets (u, a, b) -> d2F and (u, a, b, c) -> d3F of the NumPy restatement, a state u)"""
    rng = np.random.default_rng(int(np.prod(dims)))
    if name == "chan":
        alpha, beta = 3.3, 0.01
        ctx = bk.Context(bk.BK_CHAN, dims, (1.0,), krylov_m=4, params=(alpha, beta))
        u = problems.chan_sol0(dims[0]) + 0.5 * rng.standard_normal(ctx.N)
        return ctx, (lambda u, a, b: JO.chan_d2F(u, a, b, alpha, beta)), (lambda u, a, b, c: JO.chan_d3F(u, a, b, c, alpha, beta)), u
    if name == "cgl2d":
        ctx = bk.Context(bk.BK_CGL2D, dims, (np.pi, np.pi / 2), krylov_m=4, params=CGL_PAR)
        r, mu, nu, c3, c5 = CGL_PAR
        return ctx, (lambda u, a, b: JO.cgl_d2F(u, a, b, mu, c3, c5)), (lambda u, a, b, c: JO.cgl_d3F(u, a, b, c, mu, c3, c5)), \
            0.7 * rng.standard_normal(ctx.N)
    kind = {"sh2d": bk.BK_SH2D, "sh3d": bk.BK_SH3D, "sh2d_periodic": bk.BK_SH2D_PERIODIC}[name]
    ctx = bk.Context(kind, dims, (2.3 * np.pi, 1.7 * np.pi, 0.9 * np.pi)[: len(dims)], krylov_m=4, params=(-0.1, 1.3))
    return ctx, (lambda u, a, b: JO.sh_d2F(u, a, b, 1.3)), JO.sh_d3F, rng.standard_normal(ctx.N)


JET_CASES = [("chan", (1000,)), ("sh2d", (95, 64)), ("sh2d", (256, 128)), ("sh3d", (32, 24, 16)), ("sh2d_periodic", (128, 64)),
             ("cgl2d", (24, 12)), ("cgl2d", (512, 512))]


@pytest.mark.parametrize("name,dims", JET_CASES)
def test_jets_match_the_numpy_restatement_and_finite_differences(bk, name, dims):
    ctx, d2F, d3F, u = _jet_case(bk, name, dims)
    rng = np.random.default_rng(3)
    a, b, c = (rng.standard_normal(ctx.N) for _ in range(3))
    j2, j3 = ctx.d2f(u, a, b), ctx.d3f(u, a, b, c)
    assert _rel(j2, d2F(u, a, b)) < 1e-12 and _rel(j3, d3F(u, a, b, c)) < 1e-12
    # symmetric in their arguments
    assert _rel(ctx.d2f(u, b, a), j2) < 1e-14
    assert _rel(ctx.d3f(u, c, a, b), j3) < 1e-14 and _rel(ctx.d3f(u, b, c, a), j3) < 1e-14
    # d2F = d/dt J(u + t b) a and d3F = d/dt d2F(u + t c)[a, b] by central differences of bk_jvp and bk_d2f.  Chan's JVP carries
    # the Laplacian (n - 1)^2 (a[i-1] - 2 a[i] + a[i+1]) ~ 1e6 beside alpha Nl'(u) a ~ 1: its rounding, not the jet, would set the
    # difference quotient's error at a small step, so chan differentiates the JVP with a larger one
    h = 1e-3 if name == "chan" else 1e-5
    fd2 = (ctx.jacobian(u + h * b)(a) - ctx.jacobian(u - h * b)(a)) / (2 * h)
    h = 1e-5
    assert _rel(j2, fd2) < 1e-6
    fd3 = (ctx.d2f(u + h * c, a, b) - ctx.d2f(u - h * c, a, b)) / (2 * h)
    assert _rel(j3, fd3) < 1e-6
    # host and device pointers give the same bits
    du, da, db, dc = (ctx.to_device(v) for v in (u, a, b, c))
    assert np.array_equal(ctx.d2f(du, da, db).numpy(), j2) and np.array_equal(ctx.d3f(du, da, db, dc).numpy(), j3)
    out = ctx.zeros()
    ctx.d2f(u, a, b, out=out)
    assert np.array_equal(out.numpy(), j2)


def test_jets_are_refused_for_potrap_and_complex_contexts(bk):
    """BK_POTRAP_CGL2D has no jets and a BK_COMPLEX context's vectors are not states: BK_ERR_ARG before any launch"""
    cases = [bk.Context(bk.BK_POTRAP_CGL2D, (8, 6, 5), (np.pi, np.pi / 2), krylov_m=4, params=CGL_PAR),
             bk.Context(bk.BK_SH2D, (16, 12), (1.0, 1.0), krylov_m=4, params=(-0.1, 1.3), complex=True)]
    for ctx in cases:
        x = np.zeros(ctx.N0)
        before = ctx.stats()["kernel_launches"]
        with pytest.raises(bk.BK200Error, match="d2F / d3F"):
            ctx.d2f(x, x, x, out=np.zeros(ctx.N0))
        with pytest.raises(bk.BK200Error, match="d2F / d3F"):
            ctx.d3f(x, x, x, x, out=np.zeros(ctx.N0))
        assert ctx.stats()["kernel_launches"] == before


# ------------------------------------------------------------------------------------------------ normal form on the trivial SH state
def _dct_eigs(n, L):
    """eigenvalues of the Neumann-closure second difference (examples/SH2d-fronts.jl:13-29), DCT-II modes k = 0..n-1"""
    h = 2 * L / n
    return -(2 - 2 * np.cos(np.pi * np.arange(n) / n)) / h**2


def _crossing(dims, lengths):
    """J(0, l) = -L1 + l I has the eigenvalues l - (1 + sum_d lambda_d)^2 over the DCT modes: the first crossing l*, its mode and
    the gap to the next one"""
    lam = np.zeros(())
    for n, L in zip(dims, lengths):
        lam = np.add.outer(lam, _dct_eigs(n, L)) if lam.ndim else _dct_eigs(n, L)
    m = (1 + lam) ** 2
    order = np.argsort(m, axis=None)
    return m.flat[order[0]], np.unravel_index(order[0], m.shape), m.flat[order[1]] - m.flat[order[0]]


def _sh_trivial(bk, dims, lengths):
    """trivial branch of SH (nu = 1.3) in l through its first crossing, detect_bifurcation = 3, DCT-preconditioned solvers"""
    P, E = bk.palc, bk.events
    lstar, mode, gap = _crossing(dims, lengths)
    kind = bk.BK_SH2D if len(dims) == 2 else bk.BK_SH3D
    ctx = bk.Context(kind, dims, lengths, krylov_m=100, params=(lstar - 0.01, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(reltol=1e-11, restart=100, maxiter=300, Pl=True, orth="cgs2")
    eig = bk.ShiftInvertB200(0.05, ls, krylovdim=40, tol=1e-11, maxrestart=30)
    nopts = P.NewtonPar(tol=1e-10, max_iterations=10, linsolver=ls, eigsolver=eig)
    # steps of at most 0.002 sqrt(2) in l, so the step that crosses l* stays clear of p_max and the bisection runs
    cp = P.ContinuationPar(dsmin=1e-5, dsmax=0.002, ds=0.002, p_min=lstar - 0.011, p_max=lstar + 0.8 * gap, max_steps=40, nev=4,
                           newton_options=nopts, detect_bifurcation=3, n_inversion=8)
    prob = P.BifurcationProblemB200(ctx, ctx.zeros(), (lstar - 0.01, 1.3), lens=0, record=lambda v: v.norminf())
    alg = P.PALC(bls=bk.MatrixFreeBLSB200(ls))
    br = E.continuation(prob, alg, cp, normC=P.norminf)
    return P, ctx, prob, alg, cp, br, lstar, mode


def _b30_reference(dims, lengths, zeta, lstar):
    """b30 = <d3F(ζ,ζ,ζ) + 3 d2F(ζ, Ψ20), ζ> with Ψ20 from a sparse direct solve of [J ζ; ζ' 0] (J = the oracle's sparse
    Jacobian at u = 0, l = l*) and the NumPy jets"""
    sh = problems.SwiftHohenberg(dims, lengths, l=lstar, nu=1.3)
    u = np.zeros(sh.N)
    z = zeta / np.linalg.norm(zeta)
    A = sp.bmat([[sh.jac_sparse(u), sp.csc_matrix(z[:, None])], [sp.csc_matrix(z[None, :]), None]]).tocsc()
    b2v = JO.sh_d2F(u, z, z, 1.3)
    rhs = -b2v + np.dot(b2v, z) * z
    psi20 = spla.spsolve(A, np.concatenate([rhs, [0.0]]))[:-1]
    return np.dot(JO.sh_d3F(u, z, z, z) + 3 * JO.sh_d2F(u, z, psi20, 1.3), z)


NF_CASES = [((48, 36), (2.3 * np.pi, 1.7 * np.pi), (2, 3)), ((256, 192), (2.3 * np.pi, 1.7 * np.pi), (2, 3)),
            ((24, 20, 16), (1.3 * np.pi, 1.1 * np.pi, 0.9 * np.pi), (1, 2, 0))]


def _check_normal_form(bk, dims, lengths, mode):
    P, ctx, prob, alg, cp, br, lstar, found = _sh_trivial(bk, dims, lengths)
    assert tuple(int(k) for k in found) == mode            # (x, y[, z]) index of the critical DCT mode
    bps = [s for s in br.specialpoint if s.type == "bp"]
    assert len(bps) == 1, [(s.type, s.param) for s in br.specialpoint]
    i = br.specialpoint.index(bps[0])
    bifpt = br.specialpoint[i]
    assert bifpt.interval[0] <= lstar <= bifpt.interval[1] and bifpt.status == "converged"
    it = P.ContIterable(prob, alg, cp, P.norminf)
    bp = bk.normalform.get_normal_form1d(it, br, i)
    nf = bp.nf
    assert abs(nf["a01"]) < 1e-12
    assert abs(nf["b11"] - 1) < 1e-6
    assert abs(nf["b20"]) < 1e-6 * abs(nf["b30"])
    assert bp.type == "Pitchfork"
    ref = _b30_reference(dims, lengths, bp.zeta.numpy(), bp.p)
    assert abs(nf["b30"] - ref) < 1e-6 * abs(ref), (nf["b30"], ref)
    return P, ctx, prob, alg, cp, br, i, bp, lstar


@pytest.mark.parametrize("dims,lengths,mode", NF_CASES)
def test_normal_form_at_a_closed_form_branch_point(bk, dims, lengths, mode):
    """The trivial state of SH (Neumann FD) loses stability to one product of DCT modes at l* = (1 + lambda_x + lambda_y)^2; the
    normal form there is a pitchfork with b11 = 1, b20 = 0 and b30 from a direct solve"""
    _check_normal_form(bk, dims, lengths, mode)


def test_branch_switching_on_the_device(bk):
    """aBS from the 48 x 36 point: the branch lies on the side the predictor chose (b11 b30 > 0: l < l*), every state solves the
    oracle's sparse residual, and the first one points along the kernel vector"""
    dims, lengths, mode = NF_CASES[0]
    P, ctx, prob, alg, cp, br, i, bp, lstar = _check_normal_form(bk, dims, lengths, mode)
    states = []
    cp2 = dataclasses.replace(cp, detect_bifurcation=0, ds=0.0005, dsmax=0.001, max_steps=15, p_min=lstar - 0.1)
    nsaved = len(next(e["eigenvals"] for e in br.eig if e["step"] == br.specialpoint[i].idx))
    br2, bp2 = bk.normalform.continuation_from_bp(br, i, prob, alg, cp2, normC=P.norminf, nev=nsaved,
                                                  callback=lambda st: states.append((st.z_u.numpy(), st.z_p)) or True)
    assert bp2.type == "Pitchfork" and len(br2.rows) == 16
    sh = problems.SwiftHohenberg(dims, lengths, nu=1.3)
    for u, l in states:
        assert np.max(np.abs(sh.F(u, l))) < 10 * cp.newton_options.tol
    assert all(l < bp2.p for _, l in states[1:])
    z = bp2.zeta.numpy()
    u1 = states[1][0]
    assert np.dot(u1, z) / np.linalg.norm(u1) > 0.99
    b11, b30 = bp2.nf["b11"], bp2.nf["b30"]
    ratios = [float(np.dot(u, u) / (6 * abs(l - bp2.p) * b11 / b30)) for u, l in states[1:6]]
    print(f"aBS 48x36: |u|^2 / (6 |l - l*| b11 / b30) on the first rows = {np.round(ratios, 4).tolist()}")
