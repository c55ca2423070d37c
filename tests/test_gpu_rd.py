"""BK_RD on the device: residual, J, J', jets and moments against the NumPy restatement (tests/rd_oracle.py), the cGL2d model
written as RD terms against the BK_CGL2D kind, the BK_PC_RD preconditioner, complex shifted solves, and the pd-1d example
(examples/pd-1d.jl) through continuation, Hopf detection and the Hopf normal form."""
import gc

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spl

import __graft_entry__ as g
from oracle import problems
from tests import jets_oracle as JO
from tests import rd_oracle as RO

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


def _rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / np.linalg.norm(np.asarray(b))


def _random_model(rng, fields, bc, ndims, nterms=12, nparams=3):
    terms = []
    for t in range(nterms):
        deg = int(rng.integers(0, 6))
        fe = [0] * fields
        for _ in range(deg):
            fe[int(rng.integers(0, fields))] += 1
        pe = {int(k): int(rng.integers(-2, 3)) for k in rng.choice(nparams, size=2, replace=False)}
        terms.append((t % fields, float(rng.uniform(-1, 1)), pe, fe))
    diffusion = [(float(rng.uniform(0.2, 1.5)), {int(rng.integers(0, nparams)): 1}) for _ in range(fields)]
    return dict(fields=fields, bc=bc, diffusion=diffusion, terms=terms, nparams=nparams, ndims=ndims)


CASES = [(1, "neumann", (97,)), (3, "dirichlet", (151,)), (2, "neumann", (151, 100)), (4, "dirichlet", (97, 64)),
         (1, "dirichlet", (64, 48)), (2, "dirichlet", (100,))]


def _setup(bk, fields, bc, dims, seed=0):
    rng = np.random.default_rng(seed + 17 * fields + len(dims))
    m = _random_model(rng, fields, bc, len(dims))
    lengths = (3.0, 2.0)[:len(dims)]
    params = tuple(rng.uniform(0.6, 1.4, size=m["nparams"]))
    ctx = bk.Context(bk.BK_RD, dims, lengths, krylov_m=40, model=bk.ReactionDiffusion(**m), params=params)
    orc = RO.RD(**m, dims=dims, lengths=lengths, params=params)
    return ctx, orc, rng


@pytest.mark.parametrize("fields,bc,dims", CASES)
def test_residual_jvp_and_adjoint_against_the_oracle(bk, fields, bc, dims):
    ctx, orc, rng = _setup(bk, fields, bc, dims)
    N = orc.N
    assert ctx.N == N
    u, v, w = (0.6 * rng.standard_normal(N) for _ in range(3))
    assert _rel(ctx.residual(u), orc.F_(u)) < 1e-12
    J = ctx.jacobian(u)
    assert _rel(J(v), orc.dF(u, v)) < 1e-12
    assert _rel(ctx.jvp(v, a0=0.7, a1=-1.3), 0.7 * v - 1.3 * orc.dF(u, v)) < 1e-12
    JT = ctx.jacobian_adjoint(u)
    jtw = JT(w)
    assert _rel(jtw, orc.JT(u, w)) < 1e-12
    lhs, rhs = np.dot(w, J(v)), np.dot(jtw, v)
    assert abs(lhs - rhs) < 1e-12 * np.linalg.norm(w) * np.linalg.norm(orc.dF(u, v)) * 10
    # host and device pointers give the same bits
    du, dv = ctx.to_device(u), ctx.to_device(v)
    assert np.array_equal(ctx.residual(du).numpy(), ctx.residual(u))
    ctx.jacobian(du)
    assert np.array_equal(ctx.jvp(dv).numpy(), ctx.jvp(v))
    # jets
    a, b, c = (rng.standard_normal(N) for _ in range(3))
    assert _rel(ctx.d2f(u, a, b), orc.d2F(u, a, b)) < 1e-12
    assert _rel(ctx.d3f(u, a, b, c), orc.d3F(u, a, b, c)) < 1e-12
    assert np.array_equal(ctx.d2f(du, ctx.to_device(a), ctx.to_device(b)).numpy(), ctx.d2f(u, a, b))


def test_jet_moments_against_the_composed_jets(bk):
    ctx, orc, rng = _setup(bk, 3, "neumann", (61, 40))
    N = orc.N
    u = 0.5 * rng.standard_normal(N)
    vecs = [rng.standard_normal(N) for _ in range(4)]
    idx2 = [(0, 1, 2), (3, 3, 1), (2, 0, 0)]
    idx3 = [(1, 0, 2, 3), (0, 0, 0, 0)]
    out = ctx.jet_moments(u, vecs, idx2, idx3)
    ref2 = [np.dot(vecs[i], ctx.d2f(u, vecs[j], vecs[k])) for i, j, k in idx2]
    ref3 = [np.dot(vecs[i], ctx.d3f(u, vecs[j], vecs[k], vecs[l])) for i, j, k, l in idx3]
    ref = np.array(ref2 + ref3)
    assert np.max(np.abs(out - ref) / np.abs(ref)) < 1e-11
    dev = ctx.jet_moments(ctx.to_device(u), [ctx.to_device(x) for x in vecs], idx2, idx3)
    assert np.array_equal(dev, out)


CGL_PARS = (0.7, 0.1, 1.0, -1.0, 1.0)


def test_cgl_as_rd_terms_matches_the_cgl2d_kind(bk):
    dims, L = (48, 33), (3.0, 1.5)
    m = RO.cgl_model()
    rd = bk.Context(bk.BK_RD, dims, L, krylov_m=20, model=bk.ReactionDiffusion(**m), params=CGL_PARS)
    cg = bk.Context(bk.BK_CGL2D, dims, L, krylov_m=20, params=CGL_PARS)
    gl = problems.GinzburgLandau2D(*dims, *L, *CGL_PARS)
    rng = np.random.default_rng(3)
    N = gl.N
    u, v, a, b, c = (0.7 * rng.standard_normal(N) for _ in range(5))
    assert _rel(rd.residual(u), cg.residual(u)) < 1e-12 and _rel(rd.residual(u), gl.F(u)) < 1e-12
    rd.jacobian(u), cg.jacobian(u)
    assert _rel(rd.jvp(v, a0=0.3, a1=1.1), cg.jvp(v, a0=0.3, a1=1.1)) < 1e-12
    assert _rel(rd.jacobian_adjoint(u)(v), cg.jacobian_adjoint(u)(v)) < 1e-12
    _, mu, _, c3, c5 = CGL_PARS
    assert _rel(rd.d2f(u, a, b), cg.d2f(u, a, b)) < 1e-12 and _rel(rd.d2f(u, a, b), JO.cgl_d2F(u, a, b, mu, c3, c5)) < 1e-12
    assert _rel(rd.d3f(u, a, b, c), cg.d3f(u, a, b, c)) < 1e-12
    vecs = [a, b, c]
    idx2, idx3 = [(0, 1, 2), (2, 2, 0)], [(0, 1, 2, 0), (1, 1, 1, 1)]
    mr, mc = rd.jet_moments(u, vecs, idx2, idx3), cg.jet_moments(u, vecs, idx2, idx3)
    assert np.max(np.abs(mr - mc) / np.abs(mc)) < 1e-12


@pytest.mark.parametrize("bc,dims", [("neumann", (128,)), ("neumann", (97,)), ("dirichlet", (64, 40)), ("neumann", (128, 96))])
def test_rd_preconditioner_against_a_sparse_solve(bk, bc, dims):
    ctx, orc, rng = _setup(bk, 2, bc, dims, seed=5)
    a0, a1 = 1.3, -0.8
    ctx.precond_setup(bk.BK_PC_RD, a0, a1)
    r = rng.standard_normal(orc.N)
    A = (a0 * sp.identity(orc.N) + a1 * orc.Delta).tocsc()
    assert _rel(ctx.precond_apply(r), spl.spsolve(A, r)) < 1e-11
    with pytest.raises(bk.BK200Error, match="vanishes"):   # the constant mode of the Neumann Laplacian; every mode at a0 = a1 = 0
        ctx.precond_setup(bk.BK_PC_RD, 0.0, 1.0 if bc == "neumann" else 0.0)


def test_a_refused_rd_preconditioner_leaves_the_previous_one_intact(bk):
    """Dirichlet, D_0 = p_1, D_1 = p_0: at p = (0, 2) the set-up (0, 1) passes field 0 and fails field 1 (its symbol is 0); the
    preconditioner set up before is applied with the same bits afterwards"""
    m = dict(fields=2, bc="dirichlet", diffusion=[(1.0, {1: 1}), (1.0, {0: 1})], terms=[(0, 1.0, {}, [1, 1])], nparams=2, ndims=2)
    ctx = bk.Context(bk.BK_RD, (40, 30), (2.0, 1.0), krylov_m=10, model=bk.ReactionDiffusion(**m), params=(1.0, 1.0))
    ctx.precond_setup(bk.BK_PC_RD, 1.0, -0.5)
    r = np.random.default_rng(2).standard_normal(ctx.N)
    x1 = ctx.precond_apply(r)
    ctx.set_params((0.0, 2.0))
    with pytest.raises(bk.BK200Error, match="vanishes"):
        ctx.precond_setup(bk.BK_PC_RD, 0.0, 1.0)
    assert np.array_equal(ctx.precond_apply(r), x1)


def test_rd_params_need_the_whole_tuple(bk):
    ctx = _pd_ctx(bk, -0.6)
    with pytest.raises(bk.BK200Error, match="nparams"):
        ctx.set_params((1.0, -1.0))


def test_complex_shifted_solve_against_dense_algebra(bk):
    dims, L = (20, 12), (2.0, 1.0)
    m = RO.cgl_model()
    cctx = bk.Context(bk.BK_RD, dims, L, krylov_m=200, model=bk.ReactionDiffusion(**m), params=CGL_PARS, complex=True)
    orc = RO.RD(**m, dims=dims, lengths=L, params=CGL_PARS)
    rng = np.random.default_rng(9)
    u = 0.5 * rng.standard_normal(orc.N)
    rhs = rng.standard_normal(orc.N) + 1j * rng.standard_normal(orc.N)
    shift = 0.4 - 1.7j
    J = cctx.cjacobian(u)
    x, ok, _ = bk.ComplexGMRESB200(reltol=1e-12, restart=200, maxiter=2000, orth="cgs2")(J, rhs, a0=shift, a1=-1.0)
    Jd = orc.J(u).toarray()
    ref = np.linalg.solve(shift * np.eye(orc.N) - Jd, rhs)
    assert ok and _rel(x, ref) < 1e-9


# ------------------------------------------------------------------------------------------------ pd-1d (examples/pd-1d.jl)
PD_N, PD_LX = 100, 3 * np.pi / 2


def _pd_params(C):
    p = list(RO.PD1D_PARAMS)
    p[5] = C
    return tuple(p)


def _pd_u0():
    X = np.linspace(-PD_LX, PD_LX, PD_N)
    return np.concatenate([np.cos(2 * X)] * 2)


def _pd_oracle(C):
    return RO.RD(**RO.pd1d_model(), dims=(PD_N,), lengths=(PD_LX,), params=_pd_params(C))


def _pd_ctx(bk, C, **kw):
    return bk.Context(bk.BK_RD, (PD_N,), (PD_LX,), krylov_m=200, model=bk.ReactionDiffusion(**RO.pd1d_model()), params=_pd_params(C),
                      **kw)


def test_pd1d_residual_is_the_example_F(bk):
    """Fbr of examples/pd-1d.jl written out: f, g and blockdiag(D Δ, Δ) with the clamp-closure Δ"""
    ctx = _pd_ctx(bk, -0.6)
    u = _pd_u0() + 0.1 * np.random.default_rng(1).standard_normal(2 * PD_N)
    eta, a, b, H, D, C = RO.PD1D_PARAMS
    uu, vv = u[:PD_N], u[PD_N:]
    Lap = RO.lap1d(PD_N, PD_LX, "neumann")
    ref = np.concatenate([eta * (uu + a * vv - C * uu * vv - uu * vv**2) + D * (Lap @ uu),
                          eta * (H * uu + b * vv + C * uu * vv + uu * vv**2) + Lap @ vv])
    assert _rel(ctx.residual(u), ref) < 1e-13


def test_gmres_with_the_rd_preconditioner_converges_on_the_pd1d_jacobian(bk):
    ctx = _pd_ctx(bk, -0.6)
    P = bk.palc
    ls = bk.GMRESB200(reltol=1e-11, restart=200, maxiter=400)
    prob = P.BifurcationProblemB200(ctx, _pd_u0(), _pd_params(-0.6), lens=5)
    sol = P.newton(prob, _pd_u0(), -0.6, P.NewtonPar(tol=1e-10, max_iterations=30, linsolver=ls), normN=P.norminf)
    assert sol.converged
    ctx.precond_setup(bk.BK_PC_RD, -1.0, 1.0)
    rhs = np.random.default_rng(2).standard_normal(2 * PD_N)
    J = ctx.jacobian(sol.u)
    x, ok, it = bk.GMRESB200(reltol=1e-10, restart=60, maxiter=200, Pr=True)(J, rhs)
    ref = spl.spsolve(_pd_oracle(-0.6).J(np.asarray(sol.u)).tocsc(), rhs)
    assert ok and _rel(x, ref) < 1e-8, it


@pytest.fixture(scope="module")
def pd_branch(bk):
    """examples/pd-1d.jl:65-75: the branch in C from C = -0.2 with the example's ContinuationPar (p_min = -1.8, max_steps = 370),
    the eigen-solver EigArpack(0.5, :LM) as shift-invert about 0.5 with nev = 21.  The eigenvectors are saved with the branch, as
    ContinuationPar's default does in the reference: recomputing ind_ev + 2 eigenpairs about 0.5 would return the real
    eigenvalues nearer 0.5 than the Hopf pair"""
    P, E = bk.palc, bk.events
    ctx = _pd_ctx(bk, -0.2)
    ls = bk.GMRESB200(reltol=1e-11, restart=200, maxiter=400)
    inner = bk.GMRESB200(reltol=1e-11, restart=200, maxiter=400)
    eig = bk.ShiftInvertB200(0.5, inner, tol=1e-9, maxrestart=40)
    nopts = P.NewtonPar(tol=1e-9, max_iterations=3200, linsolver=ls, eigsolver=eig)
    cp = P.ContinuationPar(dsmax=0.051, ds=-0.001, p_min=-1.8, detect_bifurcation=3, nev=21, newton_options=nopts, max_steps=370,
                           n_inversion=10, max_bisection_steps=25, save_eigenvectors=True)
    prob = P.BifurcationProblemB200(ctx, ctx.to_device(_pd_u0()), _pd_params(-0.2), lens=5, record=lambda v: v.norminf())
    alg = P.PALC(bls=bk.MatrixFreeBLSB200(ls))
    br = E.continuation(prob, alg, cp, normC=P.norminf)
    return dict(br=br, it=P.ContIterable(prob, alg, cp, P.norminf), ctx=ctx)


def _oscillatory_unstable(C, u):
    """the oracle's count of eigenvalues with Re > 0 and Im != 0 on its own steady state at C (Newton from u), dense spectrum"""
    o = _pd_oracle(C)
    for _ in range(30):
        r = o.F_(u)
        if np.max(np.abs(r)) < 1e-12:
            break
        u = u - spl.spsolve(o.J(u).tocsc(), r)
    ev = np.linalg.eigvals(o.J(u).toarray())
    return int(np.sum((ev.real > 0) & (np.abs(ev.imag) > 1e-8)))


def test_pd1d_branch_reports_hopf_points_at_the_oracle_crossing(bk, pd_branch):
    """Every Hopf point the branch reports: the oracle's dense spectrum changes its count of oscillatory unstable eigenvalues between
    the branch rows on either side of the point; the crossing, bisected on the oracle to 1e-10, and the located parameter both lie
    in the bisection interval the branch reports.  The example's branch crosses at C = -0.862, -0.978 and -1.235."""
    br = pd_branch["br"]
    hopfs = [s for s in br.specialpoint if s.type == "hopf"]
    assert len(hopfs) >= 3, [(s.type, s.param) for s in br.specialpoint]
    par = {r["step"]: r["param"] for r in br.rows}
    slack = 1e-6
    for h in hopfs:
        lo, hi = min(h.interval), max(h.interval)
        u = np.asarray(h.x.numpy() if hasattr(h.x, "numpy") else h.x)
        a, b = par[h.idx - 1], par.get(h.idx + 1, par[h.idx])
        na, nb = _oscillatory_unstable(a, u), _oscillatory_unstable(b, u)
        assert na != nb, (h.param, a, b, na, nb)
        while abs(b - a) > 1e-10:
            c = 0.5 * (a + b)
            a, b = (c, b) if _oscillatory_unstable(c, u) == na else (a, c)
        c_star = 0.5 * (a + b)
        assert lo - slack <= c_star <= hi + slack, (c_star, h.interval, h.param)
        assert lo - slack <= h.param <= hi + slack, (h.param, h.interval)


def test_pd1d_hopf_normal_form_against_dense_numpy(bk, pd_branch):
    """get_normal_form(br, 1) (examples/pd-1d.jl:77): ω, a and b (Re b: the first Lyapunov coefficient) against a dense restatement
    of __hopf_normal_form at the device's point, with the dense eigenvectors (b does not depend on the phase of ζ)"""
    br, it = pd_branch["br"], pd_branch["it"]
    ind = next(i for i, s in enumerate(br.specialpoint) if s.type == "hopf")
    hp = bk.normalform.hopf_normal_form(it, br, ind)
    x0 = np.asarray(hp.x0.numpy() if hasattr(hp.x0, "numpy") else hp.x0)
    p = hp.p
    o = _pd_oracle(p)
    L0 = o.J(x0).toarray()
    ev, W = np.linalg.eig(L0)
    k = int(np.argmin(np.abs(ev.real) + 10 * (ev.imag <= 0)))
    lam = ev[k]
    assert abs(hp.omega - lam.imag) < 1e-6 * abs(lam.imag), (hp.omega, lam)
    zeta = W[:, k] / np.linalg.norm(W[:, k])
    evT, WT = np.linalg.eig(L0.T)
    zad = WT[:, int(np.argmin(np.abs(evT - np.conj(lam))))]
    zad = zad / np.vdot(zeta, zad)
    d2 = lambda a, b: o.d2F(x0, a, b)
    d3 = lambda a, b, c: o.d3F(x0, a, b, c)

    def d2c(a, b):
        return d2(a.real, b.real) - d2(a.imag, b.imag) + 1j * (d2(a.real, b.imag) + d2(a.imag, b.real))

    def d3c(a, b, c):
        out = 0
        for ka, pa in ((1, a.real), (1j, a.imag)):
            for kb, pb in ((1, b.real), (1j, b.imag)):
                for kc, pc in ((1, c.real), (1j, c.imag)):
                    out = out + ka * kb * kc * d3(pa, pb, pc)
        return out
    d = it.prob.delta
    R01 = (_pd_oracle(p + d).F_(x0) - _pd_oracle(p - d).F_(x0)) / (2 * d)
    P001 = np.linalg.solve(L0, -R01)
    av = (_pd_oracle(p + d).J(x0).toarray() - _pd_oracle(p - d).J(x0).toarray()) @ zeta / (2 * d) + d2c(zeta, P001 + 0j)
    a = np.vdot(av, zad)
    P200 = np.linalg.solve(2j * lam.imag * np.eye(len(x0)) - L0, d2c(zeta, zeta) / 2)
    P110 = np.linalg.solve(L0, -np.real(d2c(zeta, np.conj(zeta))))
    b = np.vdot(d2c(zeta, P110 + 0j) + d2c(np.conj(zeta), P200) + d3c(zeta, zeta, np.conj(zeta)) / 2, zad)
    assert abs(hp.nf["a"] - a) < 1e-5 * abs(a), (hp.nf["a"], a)
    assert abs(hp.nf["b"] - b) < 1e-5 * abs(b), (hp.nf["b"], b)


def test_pd1d_native_loop_is_bit_identical_to_the_plugin_loop(bk):
    P = bk.palc
    ctx = _pd_ctx(bk, -0.2)
    ls = bk.GMRESB200(reltol=1e-11, restart=200, maxiter=400)
    cp = P.ContinuationPar(dsmax=0.051, ds=-0.001, p_min=-1.8, max_steps=30,
                           newton_options=P.NewtonPar(tol=1e-9, max_iterations=30, linsolver=ls))
    alg = P.PALC(bls=bk.MatrixFreeBLSB200(ls))
    mk = lambda: P.BifurcationProblemB200(ctx, ctx.to_device(_pd_u0()), _pd_params(-0.2), lens=5)
    ref, st = P.continuation(mk(), alg, cp, normC=P.norminf)
    rows, info = P.continuation_native(mk(), alg, cp, normC=P.norminf)
    assert len(ref) > 10 and len(rows) == len(ref)
    for r, q in zip(rows, ref):
        assert all(r[k] == q[k] for k in q), (r, q)
    assert np.array_equal(info["u"].numpy(), st.z_u.numpy())
    # the run leaves the caller's parameter tuple, and everything computed from it, as it was: the context gives the bits of a
    # fresh context at the same params
    fresh = _pd_ctx(bk, -0.2)
    rng = np.random.default_rng(6)
    u, a, b = _pd_u0() + 0.1 * rng.standard_normal(2 * PD_N), rng.standard_normal(2 * PD_N), rng.standard_normal(2 * PD_N)
    assert ctx.params == fresh.params
    assert np.array_equal(ctx.residual(u), fresh.residual(u))
    assert np.array_equal(ctx.d2f(u, a, b), fresh.d2f(u, a, b))
    assert np.array_equal(ctx.jet_moments(u, [a, b], [(0, 1, 1)]), fresh.jet_moments(u, [a, b], [(0, 1, 1)]))
    assert np.array_equal(ctx.replicate().residual(u), ctx.residual(u))


def test_gray_scott_512_newton_with_the_rd_preconditioner(bk):
    """a user-size 2-D model: Gray-Scott at 512^2 (N = 524 288), Newton-GMRES right-preconditioned by BK_PC_RD"""
    m = RO.gray_scott_model()
    dims, L = (512, 512), (1.25, 1.25)
    pars = (2e-5, 1e-5, 0.04, 0.06)
    ctx = bk.Context(bk.BK_RD, dims, L, krylov_m=60, model=bk.ReactionDiffusion(**m), params=pars)
    n = dims[0] * dims[1]
    x = np.linspace(-1, 1, dims[0])
    X, Y = np.meshgrid(x, x, indexing="xy")
    bump = 0.2 * np.exp(-20 * (X**2 + Y**2)).ravel()
    u0 = np.concatenate([1 - 0.5 * bump, 0.25 * bump])
    P = bk.palc
    ctx.precond_setup(bk.BK_PC_RD, -0.07, 1.0)
    ls = bk.GMRESB200(reltol=1e-8, restart=60, maxiter=600, Pr=True)
    prob = P.BifurcationProblemB200(ctx, ctx.to_device(u0), pars, lens=2)
    sol = P.newton(prob, ctx.to_device(u0), pars[2], P.NewtonPar(tol=1e-9, max_iterations=30, linsolver=ls), normN=P.norminf)
    assert sol.converged, sol.residuals
    uh = sol.u.numpy()
    assert np.max(np.abs(RO.RD(**m, dims=dims, lengths=L, params=pars).F_(uh))) < 1e-9 * 1.01
    assert n == len(uh) // 2


def test_replicate_gives_the_same_bits_and_contexts_free_their_memory(bk):
    import torch
    ctx, orc, rng = _setup(bk, 2, "neumann", (128, 64))
    ctx.precond_setup(bk.BK_PC_RD, 1.0, -1.0)
    u, v = 0.5 * rng.standard_normal(orc.N), rng.standard_normal(orc.N)
    rep = ctx.replicate()
    assert np.array_equal(rep.residual(u), ctx.residual(u))
    ctx.jacobian(u), rep.jacobian(u)
    ls = bk.GMRESB200(reltol=1e-10, restart=40, maxiter=200, Pr=True)
    x1, _, _ = ls(ctx.jacobian(u), v, a0=1.0, a1=-0.1)
    x2, _, _ = ls(rep.jacobian(u), v, a0=1.0, a1=-0.1)
    assert np.array_equal(x1, x2)
    del ctx, rep
    gc.collect()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(5):
        c, o, r = _setup(bk, 3, "dirichlet", (256, 256))
        c.precond_setup(bk.BK_PC_RD, 1.0, -1.0)
        c.d2f(r.standard_normal(o.N), r.standard_normal(o.N), r.standard_normal(o.N))
        c.close()
        del c
        gc.collect()
    assert torch.cuda.mem_get_info()[0] >= free0 - (16 << 20)
