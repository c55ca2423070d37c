"""GPU tests of bk_deflation_moments (Context.deflation_moments), of the fused deflation operator and of deflated continuation
(defcont.py): the kernel against NumPy in long double and against the composed bk_vec_* path on chan, SH2d and cGL2d vectors,
near a root, host/device bit-identity, split invariance and every refusal; DeflatedProblemCustomLS fused against composed on the
three Chan solutions; DefCont on Chan against its host twin; DefCont on SH2d fronts checked by the oracle's residual."""
import ctypes as C

import numpy as np
import pytest
import scipy.sparse as sp

import __graft_entry__ as g
from oracle import problems, krylov

pytestmark = pytest.mark.gpu
LX, LY = 8 * np.pi, 4 * np.pi / np.sqrt(3)


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


def _ctx(bk, kind):
    if kind == "chan":
        return bk.Context(bk.BK_CHAN, (1000,), (1.0,), krylov_m=4, params=(3.3, 0.01))
    if kind == "sh2d":
        return bk.Context(bk.BK_SH2D, (128, 64), (LX, LY), krylov_m=4, params=(-0.1, 1.3))
    return bk.Context(bk.BK_CGL2D, (41, 21), (np.pi, np.pi / 2), krylov_m=4, params=(0.5, 0.1, 1.0, -1.0, 1.0))


def _ld(u, roots, dirs, n):
    L = np.longdouble
    u = u[:n].astype(L)
    d = [u - r[:n].astype(L) for r in roots]
    h = [x[:n].astype(L) for x in dirs]
    s = np.array([np.dot(x, x) for x in d])
    m = np.array([np.max(np.abs(x)) for x in d])
    t = np.array([[np.dot(x, y) for y in h] for x in d]).reshape(len(roots), len(dirs))
    q = np.array([[np.dot(a, b) for b in h] for a in h]).reshape(len(dirs), len(dirs))
    return s, m, t, q


def _vectors(N, nroots, seed, scale=1.0):
    rng = np.random.default_rng(seed)
    u = rng.standard_normal(N)
    return u, [u + scale * rng.standard_normal(N) for _ in range(nroots)], [rng.standard_normal(N) for _ in range(2)]


@pytest.mark.parametrize("kind", ["chan", "sh2d", "cgl2d"])
@pytest.mark.parametrize("nroots", [1, 7, 64, 130])
@pytest.mark.parametrize("ndir", [0, 1, 2])
def test_kernel_against_long_double_and_the_composed_path(bk, kind, nroots, ndir):
    ctx = _ctx(bk, kind)
    N = ctx.N0
    u, roots, dirs = _vectors(N, nroots, 100 * nroots + ndir)
    dirs = dirs[:ndir]
    du, dr, dh = ctx.to_device(u), [ctx.to_device(r) for r in roots], [ctx.to_device(h) for h in dirs]
    for n in (N, N - 1 - N // 3):                                  # the whole vectors and a prefix
        s, m, t, q = ctx.deflation_moments(du, dr, dh, n)
        S, M, T, Q = _ld(u, roots, dirs, n)
        assert np.all(np.abs(s - S) <= 1e-13 * S)
        assert np.array_equal(m, M.astype(float))                  # the max is exact
        hn = [np.linalg.norm(h[:n]) for h in dirs]
        for a in range(ndir):
            assert np.all(np.abs(t[:, a] - T[:, a]) <= 1e-13 * np.sqrt(S) * hn[a])
            for b in range(ndir):
                assert abs(q[a, b] - Q[a, b]) <= 1e-13 * hn[a] * hn[b] and q[a, b] == q[b, a]
        if n == N:                                                 # the composed loop: copy + axpby + dot / norminf per root
            for i in (0, nroots - 1):
                d = du.copy().axpby_(-1.0, dr[i], 1.0)
                assert abs(s[i] - d.dot(d)) <= 1e-12 * s[i] and m[i] == d.norminf()
                for a in range(ndir):
                    assert abs(t[i, a] - d.dot(dh[a])) <= 1e-12 * np.sqrt(s[i]) * hn[a]


@pytest.mark.parametrize("kind", ["chan", "sh2d", "cgl2d"])
def test_near_a_root_the_distance_keeps_its_relative_accuracy(bk, kind):
    """u within 1e-7 of a root: s = |u - r|^2 ~ 1e-14 N while <u, u> ~ N; the expanded form would keep no digit of s"""
    ctx = _ctx(bk, kind)
    u, roots, dirs = _vectors(ctx.N0, 3, 7, scale=1e-7)
    s, m, t, _ = ctx.deflation_moments(ctx.to_device(u), [ctx.to_device(r) for r in roots], [ctx.to_device(dirs[0])])
    S, M, T, _ = _ld(u, roots, dirs[:1], ctx.N0)
    exact = np.array([np.sum((u.astype(np.longdouble) - r) ** 2) for r in roots])  # u - r is exact in double here
    assert np.all(np.abs(s - S) <= 1e-13 * S) and np.all(np.abs(s - exact) <= 1e-13 * exact)
    assert np.array_equal(m, M.astype(float))


def test_host_device_bits_split_invariance_and_ndir_independence(bk):
    ctx = _ctx(bk, "sh2d")
    u, roots, dirs = _vectors(ctx.N0, 130, 3)
    du, dr, dh = ctx.to_device(u), [ctx.to_device(r) for r in roots], [ctx.to_device(h) for h in dirs]
    dev = ctx.deflation_moments(du, dr, dh)
    host = ctx.deflation_moments(u, roots, dirs)
    mixed = ctx.deflation_moments(u, dr, [dirs[0], dh[1]])
    for a, b in zip(dev, host):
        assert np.array_equal(a, b)
    for a, b in zip(dev, mixed):
        assert np.array_equal(a, b)
    # a root's values are the same alone, in another group, and with fewer directions
    for i in (0, 5, 63, 64, 129):
        one = ctx.deflation_moments(du, [dr[i]], dh)
        assert one[0][0] == dev[0][i] and one[1][0] == dev[1][i] and np.array_equal(one[2][0], dev[2][i])
        none = ctx.deflation_moments(du, [dr[i]])
        assert none[0][0] == dev[0][i] and none[1][0] == dev[1][i]
    sub = ctx.deflation_moments(du, dr[60:70], dh)
    assert np.array_equal(sub[0], dev[0][60:70]) and np.array_equal(sub[2], dev[2][60:70])


def test_every_refusal(bk):
    ctx = _ctx(bk, "chan")
    lib, h = ctx.lib, ctx.handle
    u = ctx.to_device(np.ones(ctx.N0))
    r = ctx.to_device(np.zeros(ctx.N0))
    out = np.zeros(64 * 4 + 3)
    op = out.ctypes.data_as(C.POINTER(C.c_double))
    roots = (C.c_void_p * 65)(*([r.dptr] * 65))
    dirs = (C.c_void_p * 2)(u.dptr, r.dptr)
    call = lambda uu, nr, rr, nd, dd, n, o=op: lib.bk_deflation_moments(h, uu, nr, rr, nd, dd, n, o)
    assert call(u.dptr, 1, roots, 2, dirs, ctx.N0) == 0
    launches = ctx.stats()["kernel_launches"]
    bad = [(u.dptr, 0, roots, 0, None, ctx.N0), (u.dptr, 65, roots, 0, None, ctx.N0), (u.dptr, 1, roots, -1, None, ctx.N0),
           (u.dptr, 1, roots, 3, dirs, ctx.N0), (u.dptr, 1, roots, 0, None, 0), (u.dptr, 1, roots, 0, None, ctx.N0 + 1),
           (None, 1, roots, 0, None, ctx.N0), (u.dptr, 1, None, 0, None, ctx.N0), (u.dptr, 1, roots, 1, None, ctx.N0),
           (u.dptr, 1, (C.c_void_p * 1)(None), 0, None, ctx.N0), (u.dptr, 1, roots, 2, (C.c_void_p * 2)(u.dptr, None), ctx.N0)]
    for args in bad:
        assert call(*args) == -1, args                           # BK_ERR_ARG
    assert call(u.dptr, 1, roots, 0, None, ctx.N0, None) == -1     # null out
    assert ctx.stats()["kernel_launches"] == launches            # refused before any launch
    cctx = bk.Context(bk.BK_CGL2D, (41, 21), (np.pi, np.pi / 2), krylov_m=4, params=(0.5, 0.1, 1.0, -1.0, 1.0), complex=True)
    cu = cctx.to_device(np.ones(cctx.N))
    assert cctx.lib.bk_deflation_moments(cctx.handle, cu.dptr, 1, (C.c_void_p * 1)(cu.dptr), 0, None, 100, op) == -1
    with pytest.raises(bk.BK200Error):
        ctx.deflation_moments(u, [])


# ------------------------------------------------------------------------------------------------ the fused operator
def _chan(bk, n=101, alpha=3.3):
    P = bk.palc
    ctx = bk.Context(bk.BK_CHAN, (n,), (1.0,), krylov_m=n, params=(alpha, 0.01))
    ctx.precond_setup(bk.BK_PC_CHAN_TRIDIAG)
    ls = bk.GMRESB200(reltol=1e-10, restart=n, maxiter=n, Pl=True, orth="cgs2")
    prob = P.BifurcationProblemB200(ctx, ctx.to_device(problems.chan_sol0(n)), (alpha, 0.01), lens=0)
    return ctx, ls, prob


def test_custom_linear_solver_fused_and_composed_give_the_same_iterates(bk):
    """the three Chan solutions at alpha = 3.3 (max u = 0.77197, 5.97988, 12.85103) by deflated Newton with the fused operator
    and with the composed loop: the same iteration counts and iterates to rounding"""
    P, D = bk.palc, bk.deflation
    ctx, ls, prob = _chan(bk)
    opts = P.NewtonPar(tol=1e-9, max_iterations=100, linsolver=ls)
    s0 = P.newton(prob, prob.u0, 3.3, opts, P.norminf)
    tops = {}
    for fused in (False, True):
        op = D.DeflationOperator(2, 1.0, [s0.u], fused=fused)
        g1 = s0.u.copy().scale_(4.0)
        s1 = D.newton_deflated(prob, g1, 3.3, op, opts, P.norminf)
        op.push(s1.u)
        s2 = D.newton_deflated(prob, s0.u.copy().scale_(8.0), 3.3, op, opts, P.norminf)
        assert s1.converged and s2.converged
        tops[fused] = (s1, s2)
    for a, b in zip(tops[False], tops[True]):
        assert a.itnewton == b.itnewton
        assert np.allclose(a.residuals, b.residuals, rtol=1e-5, atol=1e-12)
        assert np.max(np.abs(a.u.numpy() - b.u.numpy())) <= 1e-9 * np.max(np.abs(a.u.numpy()))
    got = sorted([float(np.max(s0.u.numpy()))] + [float(np.max(s.u.numpy())) for s in tops[True]])
    assert np.allclose(got, [0.77197, 5.97988, 12.85103], atol=1e-4)
    # host roots with a device u take the composed loop (they would be uploaded on every call)
    host_roots = D.DeflationOperator(2, 1.0, [s0.u.numpy()], fused=True)
    assert not host_roots.runs_fused(s0.u) and D.DeflationOperator(2, 1.0, [s0.u], fused=True).runs_fused(s0.u)
    # the fused jvp of the deflated problem against the composed one
    dp_f = D.DeflatedProblem(prob, D.DeflationOperator(2, 1.0, [s0.u], fused=True))
    dp_c = D.DeflatedProblem(prob, D.DeflationOperator(2, 1.0, [s0.u]))
    x, v = tops[True][0].u, ctx.to_device(np.random.default_rng(0).standard_normal(ctx.N))
    a, b = dp_f.jvp(x, 3.3, v).numpy(), dp_c.jvp(x, 3.3, v).numpy()
    assert np.linalg.norm(a - b) <= 1e-6 * np.linalg.norm(b)


class _HostChan:
    """the host twin: chan F of the oracle and its sparse Jacobian"""

    def __init__(self, u0, p0, n=101):
        self.u0, self.p0, self.n = u0, p0, n
        self.delta = float(np.sqrt(np.finfo(float).eps))
        self.record = lambda x: float(np.linalg.norm(x))

    def F(self, x, p, out=None):
        r = problems.chan_F(x, p, 0.01)
        if out is not None:
            out[...] = r
            return out
        return r

    def J(self, x, p):
        return sp.csr_matrix(np.column_stack([problems.chan_dF(x, e, p, 0.01) for e in np.eye(self.n)]))


def test_defcont_on_chan_against_its_host_twin(bk):
    P, DC, D = bk.palc, bk.defcont, bk.deflation
    ctx, ls, prob = _chan(bk, alpha=3.0)
    opts = P.NewtonPar(tol=1e-9, max_iterations=20, linsolver=ls)
    s0 = P.newton(prob, prob.u0, 3.0, opts, P.norminf)
    assert s0.converged
    cp = P.ContinuationPar(ds=0.05, p_min=2.5, p_max=3.6, max_steps=6, newton_options=opts)
    scale = lambda x, p, idb: x.copy().scale_(4.0) if hasattr(x, "dptr") else 4.0 * x
    alg = DC.DefCont(deflation_operator=D.DeflationOperator(2, 1.0, [s0.u]), perturb_solution=scale, max_branches=5)
    dev = DC.continuation(prob, alg, cp, normC=P.norminf, save_sol_every_step=1)
    hprob = _HostChan(s0.u.numpy(), 3.0)
    hcp = P.ContinuationPar(ds=0.05, p_min=2.5, p_max=3.6, max_steps=6,
                            newton_options=P.NewtonPar(tol=1e-9, max_iterations=20, linsolver=krylov.DefaultLS()))
    halg = DC.DefCont(deflation_operator=D.DeflationOperator(2, 1.0, [s0.u.numpy()]), perturb_solution=scale, max_branches=5)
    host = DC.continuation(hprob, halg, hcp, normC=P.norminf, save_sol_every_step=1)
    assert len(dev.branches) == len(host.branches) >= 2
    assert [s.isactive for s in dev.states] == [s.isactive for s in host.states]
    for a, b in zip(dev.branches, host.branches):
        assert len(a.rows) == len(b.rows) and len(a.sol) == len(b.sol)
        for ra, rb in zip(a.rows, b.rows):
            assert ra["step"] == rb["step"] and abs(ra["param"] - rb["param"]) <= 1e-12
            assert abs(ra["x"] - rb["x"]) <= 1e-8 * abs(rb["x"])
        for sa, sb in zip(a.sol, b.sol):
            assert P.norminf(problems.chan_F(sa["x"].numpy(), sa["p"], 0.01)) < 1e-8


def test_defcont_on_sh2d_fronts(bk):
    """examples/SH2d-fronts.jl:168-180 at 128 x 64: DeflationOperator(2, 1, [hexagons]), a seeded perturbation (the localized
    front envelope of :75 on the branch point plus 0.01 rand), a few branches and steps: every saved point solves F = 0 by the
    oracle's sparse residual, and the branches are pairwise distinct by more than tol"""
    P, DC, D = bk.palc, bk.defcont, bk.deflation
    dims = (128, 64)
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=100, params=(-0.1, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(reltol=1e-5, restart=100, maxiter=100, N=ctx.N, Pr=True)
    sol0 = ctx.to_device(problems.sh2d_sol0(*dims, LX, LY))
    prob = P.BifurcationProblemB200(ctx, sol0, (-0.1, 1.3), lens=0)
    opts = P.NewtonPar(tol=1e-8, max_iterations=20, linsolver=ls)
    hexa = P.newton(prob, sol0, -0.1, opts, P.norminf)
    assert hexa.converged
    rng = np.random.default_rng(0)

    def perturb(x, p, idb):
        return ctx.to_device(problems.sh2d_front_guess(x.numpy(), *dims, LX, LY) + 0.01 * rng.random(ctx.N))

    cp = P.ContinuationPar(dsmin=1e-4, dsmax=5e-3, ds=-2e-3, p_min=-1.0, p_max=0.0, max_steps=3, newton_options=opts)
    alg = DC.DefCont(deflation_operator=D.DeflationOperator(2, 1.0, [hexa.u]), perturb_solution=perturb, max_iter_defop=3,
                     max_branches=3)
    res = DC.continuation(prob, alg, cp, normC=P.norminf)
    assert len(res.branches) >= 2
    by_p = {}
    for k, br in enumerate(res.branches):
        for s in br.sol:
            sh = problems.SwiftHohenberg(dims, (LX, LY), l=s["p"], nu=1.3)
            x = s["x"].numpy()
            assert np.max(np.abs(sh.F(x, s["p"]))) < 1e-7
            by_p.setdefault(s["p"], []).append((k, x))
    pairs = 0
    for xs in by_p.values():                     # points of different branches at the same parameter
        for i in range(len(xs)):
            for j in range(i):
                if xs[i][0] != xs[j][0]:
                    assert np.max(np.abs(xs[i][1] - xs[j][1])) > opts.tol
                    pairs += 1
    assert pairs >= 1
