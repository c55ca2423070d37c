"""GPU tests of the one-pass jet contractions (bk_jet_moments) against the composed path (bk_d2f / bk_d3f + bk_vec_dot) and the
NumPy jets; and of the normal form of branch points with a 2- and 3-dimensional kernel (normalform.get_normal_formNd) and branch
switching from them (normalform.multicontinuation) on the trivial Swift-Hohenberg state of square and cubic Neumann boxes, whose
kernels are pairs / triples of DCT modes, against the N-border oracle of tests/nd_normal_form_oracle.py."""
import numpy as np
import pytest

import __graft_entry__ as g
from oracle import problems
from tests import jets_oracle as JO
from tests import nd_normal_form_oracle as NO
from tests.test_gpu_normal_form import CGL_PAR, _dct_eigs, _jet_case

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


# ------------------------------------------------------------------------------------------------ the moments kernel
MOM_CASES = [("chan", (1000,)), ("sh2d", (96, 64)), ("sh2d", (95, 63)), ("sh3d", (32, 24, 16)), ("sh2d_periodic", (128, 64)),
             ("cgl2d", (24, 12)), ("cgl2d", (256, 128))]


def _tuples(rng, nvec, n2, n3):
    idx2, idx3 = rng.integers(0, nvec, (n2, 3)), rng.integers(0, nvec, (n3, 4))
    idx2[0], idx2[1], idx3[0] = (0, 0, 0), (nvec - 1, 2, 2), (1, 1, 1, 1)       # repeated indices
    return idx2, idx3


@pytest.mark.parametrize("name,dims", MOM_CASES)
def test_moments_match_the_composed_path(bk, name, dims):
    """every contraction within 1e-12 of the composed path and of the NumPy jets, relative to the sum of |terms|; host and device
    inputs give the same bits, and so do two calls"""
    ctx, d2F, d3F, u = _jet_case(bk, name, dims)
    nfm = bk.normalform
    rng = np.random.default_rng(17)
    nvec = 9
    vecs = [rng.standard_normal(ctx.N) for _ in range(nvec)]
    idx2, idx3 = _tuples(rng, nvec, 40, 30)
    got = ctx.jet_moments(u, vecs, idx2, idx3)
    want, scale = NO.moments(lambda a, b: d2F(u, a, b), lambda a, b, c: d3F(u, a, b, c), vecs, idx2, idx3)
    assert np.all(np.abs(got - want) <= 1e-12 * scale), np.max(np.abs(got - want) / scale)
    du, dvecs = ctx.to_device(u), [ctx.to_device(v) for v in vecs]
    prob = bk.palc.BifurcationProblemB200(ctx, du, ctx.params, lens=0)
    composed = nfm.jet_moments_composed(prob, du, ctx.params[0], dvecs, idx2, idx3)
    assert np.all(np.abs(got - composed) <= 1e-12 * scale)
    dev = ctx.jet_moments(du, dvecs, idx2, idx3)
    assert np.array_equal(dev, got) and np.array_equal(ctx.jet_moments(du, dvecs, idx2, idx3), dev)
    mixed = ctx.jet_moments(du, vecs[:4] + dvecs[4:], idx2, idx3)
    assert np.array_equal(mixed, got)
    assert np.array_equal(nfm.jet_moments(prob, du, ctx.params[0], dvecs, idx2, idx3), dev)   # the problem's one-pass path


@pytest.mark.parametrize("nvec,n2,n3", [(6, 6000, 4000), (150, 300, 200)])
def test_moments_split_long_lists(bk, nvec, n2, n3):
    """Context.jet_moments splits lists longer than BK_JET_MOMENTS_MAX_TUPLES into several calls, and more than
    BK_JET_MOMENTS_MAX_VEC vectors into groups of tuples that need at most that many"""
    ctx, d2F, d3F, u = _jet_case(bk, "sh2d", (64, 48))
    rng = np.random.default_rng(2)
    vecs = [rng.standard_normal(ctx.N) for _ in range(nvec)]
    idx2, idx3 = _tuples(rng, nvec, n2, n3)
    before = ctx.stats()["kernel_launches"]
    got = ctx.jet_moments(u, vecs, idx2, idx3)
    calls = (ctx.stats()["kernel_launches"] - before) // 2
    want, scale = NO.moments(lambda a, b: d2F(u, a, b), lambda a, b, c: d3F(u, a, b, c), vecs, idx2, idx3)
    assert len(got) == n2 + n3 and np.all(np.abs(got - want) <= 1e-12 * scale)
    assert calls >= (2 if nvec <= 64 else -(-nvec // 64))


def test_moments_refusals_come_before_any_launch(bk):
    cases = [bk.Context(bk.BK_POTRAP_CGL2D, (8, 6, 5), (np.pi, np.pi / 2), krylov_m=4, params=CGL_PAR),
             bk.Context(bk.BK_SH2D, (16, 12), (1.0, 1.0), krylov_m=4, params=(-0.1, 1.3), complex=True)]
    for ctx in cases:
        x = np.zeros(ctx.N0)
        before = ctx.stats()["kernel_launches"]
        with pytest.raises(bk.BK200Error, match="d2F / d3F"):
            ctx.jet_moments(x, [x, x], [(0, 1, 1)])
        assert ctx.stats()["kernel_launches"] == before
    ctx = bk.Context(bk.BK_SH2D, (16, 12), (1.0, 1.0), krylov_m=4, params=(-0.1, 1.3))
    x = np.zeros(ctx.N)
    lib = ctx.lib
    before = ctx.stats()["kernel_launches"]
    bad = [(lambda: ctx.jet_moments(x, [x, x], [(0, 2, 1)]), "index out of range"),
           (lambda: ctx.jet_moments(x, [x, x], (), [(0, 1, 1, -1)]), "index out of range"),
           (lambda: ctx.jet_moments(x, [], [(0, 0, 0)]), "nvec out of range"),
           (lambda: ctx.jet_moments(x, [x, None], [(0, 1, 1)]), "null vector"),
           (lambda: ctx.jet_moments(None, [x, x], [(0, 1, 1)]), "null argument")]
    for call, msg in bad:
        with pytest.raises(bk.BK200Error, match=msg):
            call()
    import ctypes as C
    pv = (C.c_void_p * 65)(*([x.ctypes.data] * 65))
    idx = np.zeros(3, dtype=np.int32)
    out = np.zeros(1)
    st = lib.bk_jet_moments(ctx.handle, x.ctypes.data, 65, pv, 1, idx.ctypes.data_as(C.POINTER(C.c_int32)), 0, None,
                            out.ctypes.data_as(C.POINTER(C.c_double)))
    assert st < 0 and b"nvec out of range" in lib.bk_last_error(ctx.handle)
    idx = np.zeros(3 * 8193, dtype=np.int32)
    out = np.zeros(8193)
    st = lib.bk_jet_moments(ctx.handle, x.ctypes.data, 1, pv, 8193, idx.ctypes.data_as(C.POINTER(C.c_int32)), 0, None,
                            out.ctypes.data_as(C.POINTER(C.c_double)))
    assert st < 0 and b"too many tuples" in lib.bk_last_error(ctx.handle)
    assert ctx.stats()["kernel_launches"] == before


# ------------------------------------------------------------------------------------------------ the trivial SH state
def _dct_mode(dims, ks):
    """the DCT-II mode of the Neumann second difference with indices ks, as a state vector (x fastest)"""
    v = np.ones(())
    for n, k in zip(dims, ks):
        c = np.cos(np.pi * k * (np.arange(n) + 0.5) / n)
        v = np.multiply.outer(c, v) if v.ndim else c
    return v.ravel()


def _crossing_multi(dims, lengths):
    """l* of the first crossing of the trivial state, every DCT mode that crosses there, and the gap to the next one"""
    lam = None
    for n, L in zip(dims, lengths):
        e = _dct_eigs(n, L)
        lam = e if lam is None else np.add.outer(lam, e)
    m = ((1 + lam) ** 2).ravel()
    order = np.argsort(m, kind="stable")
    k = int(np.sum(np.abs(m - m[order[0]]) <= 1e-9 * max(1.0, m[order[0]])))
    modes = [tuple(int(q) for q in np.unravel_index(i, lam.shape)) for i in order[:k]]
    return m[order[0]], modes, m[order[k]] - m[order[0]]


def _sh_setup(bk, dims, lengths, lstart):
    P = bk.palc
    kind = bk.BK_SH2D if len(dims) == 2 else bk.BK_SH3D
    ctx = bk.Context(kind, dims, lengths, krylov_m=100, params=(lstart, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(reltol=1e-11, restart=100, maxiter=300, Pl=True, orth="cgs2")
    eig = bk.ShiftInvertB200(0.05, ls, krylovdim=40, tol=1e-11, maxrestart=30)
    nopts = P.NewtonPar(tol=1e-10, max_iterations=10, linsolver=ls, eigsolver=eig)
    prob = P.BifurcationProblemB200(ctx, ctx.zeros(), (lstart, 1.3), lens=0, record=lambda v: v.norminf())
    alg = P.PALC(bls=bk.MatrixFreeBLSB200(ls))
    return P, ctx, prob, alg, nopts


def _point_at(bk, ctx, lstar, N, nev=6):
    """a branch holding one specialpoint of kernel dimension N at the analytic l* on the trivial state (the reference's tests
    `@reset br.specialpoint[1].param`), with its eigenvalues"""
    E = bk.events
    sp = E.SpecialPoint(type="nd", idx=0, param=lstar, norm=0.0, step=0, status="converged", delta=(N, 0), ind_ev=N,
                        interval=(lstar, lstar), x=ctx.zeros(), tau_p=1.0, tau_u=ctx.zeros())
    return E.Branch(specialpoint=[sp], eig=[dict(eigenvals=np.zeros(nev, dtype=complex), step=0)])


def _oracle(dims, lengths, bp, delta):
    sh = lambda p: problems.SwiftHohenberg(dims, lengths, l=p, nu=1.3)
    u = np.zeros(sh(bp.p).N)
    host = lambda v: v.numpy() if hasattr(v, "numpy") else np.asarray(v)
    return NO.nd_normal_form(lambda x, p: sh(p).F(x, p), lambda p: sh(p).jac_sparse(u), lambda a, b: JO.sh_d2F(u, a, b, 1.3),
                             lambda a, b, c: JO.sh_d3F(u, a, b, c), u, bp.p, delta, [host(z) for z in bp.zetas],
                             [host(z) for z in bp.zetas_ad])


def _check_against_oracle(bp, ref, N):
    nf = bp.nf
    scale = np.max(np.abs(ref["b30"]))
    assert scale > 0
    assert np.max(np.abs(nf["b30"] - ref["b30"])) < 1e-6 * scale, (nf["b30"], ref["b30"])
    assert np.max(np.abs(nf["b20"] - ref["b20"])) < 1e-6 * max(scale, np.max(np.abs(ref["b20"])))
    assert np.max(np.abs(nf["a01"])) < 1e-12 and np.max(np.abs(nf["a02"])) < 1e-6
    assert np.max(np.abs(nf["b11"] - np.eye(N))) < 1e-6
    assert nf["b30"].shape == (N,) * 4


SQUARE = ((48, 48), (2.3 * np.pi, 2.3 * np.pi))


def test_square_box_has_one_nd_point(bk):
    """The trivial branch through l* of the 48 x 48 square: the crossing of the pair (2, 4) / (4, 2) is one nd point with
    delta (2, 0) and l* inside its interval"""
    dims, lengths = SQUARE
    lstar, modes, gap = _crossing_multi(dims, lengths)
    assert sorted(modes) == [(2, 4), (4, 2)] and abs(lstar - 0.0035283) < 1e-6
    P, ctx, prob, alg, nopts = _sh_setup(bk, dims, lengths, lstar - 0.01)
    cp = P.ContinuationPar(dsmin=1e-5, dsmax=0.002, ds=0.002, p_min=lstar - 0.011, p_max=lstar + 0.8 * gap, max_steps=40, nev=6,
                           newton_options=nopts, detect_bifurcation=3, n_inversion=8)
    br = bk.events.continuation(prob, alg, cp, normC=P.norminf)
    found = [(s.type, s.param, s.delta) for s in br.specialpoint if s.type != "endpoint"]
    print(f"48x48 square: special points {found}")
    assert len(found) == 1 and found[0][0] == "nd" and found[0][2] == (2, 0), found
    sp = br.specialpoint[0]
    assert sp.interval[0] <= lstar <= sp.interval[1]


@pytest.mark.parametrize("given", [True, False], ids=["dct_modes", "recomputed"])
def test_square_box_normal_form(bk, given):
    """get_normal_formNd at the analytic 48 x 48 point, with ζs the DCT modes or recomputed by the shift-invert eigensolver:
    b20, b30 match the oracle run on the same ζs / ζ★s to 1e-6, a01 = a02 = 0 and b11 = I"""
    dims, lengths = SQUARE
    lstar, modes, gap = _crossing_multi(dims, lengths)
    P, ctx, prob, alg, nopts = _sh_setup(bk, dims, lengths, lstar)
    cp = P.ContinuationPar(nev=6, newton_options=nopts)
    br = _point_at(bk, ctx, lstar, 2)
    it = P.ContIterable(prob, alg, cp, P.norminf)
    zetas = [_dct_mode(dims, m) for m in modes] if given else None
    bp = bk.normalform.get_normal_formNd(it, br, 0, zetas=zetas)
    assert bp.type == "2-d" and len(bp.zetas) == 2
    _check_against_oracle(bp, _oracle(dims, lengths, bp, prob.delta), 2)


def test_cube_three_dimensional_kernel(bk):
    """24^3 cube of side 1.3 pi: the modes (1, 1, 2) and its permutations cross together, N = 3.  With ζs given, the tensors
    match the oracle's three-border direct solves: the two-border device solves, projected, give the N-border solution"""
    dims, lengths = (24, 24, 24), (1.3 * np.pi,) * 3
    lstar, modes, gap = _crossing_multi(dims, lengths)
    assert len(modes) == 3 and sorted(sorted(m) for m in modes) == [[1, 1, 2]] * 3
    P, ctx, prob, alg, nopts = _sh_setup(bk, dims, lengths, lstar)
    cp = P.ContinuationPar(nev=6, newton_options=nopts)
    br = _point_at(bk, ctx, lstar, 3)
    it = P.ContIterable(prob, alg, cp, P.norminf)
    bp = bk.normalform.get_normal_formNd(it, br, 0, zetas=[_dct_mode(dims, m) for m in modes])
    _check_against_oracle(bp, _oracle(dims, lengths, bp, prob.delta), 3)


def test_multicontinuation_on_the_square(bk):
    """Branch switching at the 48 x 48 point: every state of every branch solves the oracle's sparse residual to 10x the Newton
    tolerance, the first points are pairwise distinct, and the x <-> y swap of the box (ζ₁ <-> ζ₂) maps every root of the
    reduced equation to a root"""
    dims, lengths = SQUARE
    lstar, modes, gap = _crossing_multi(dims, lengths)
    P, ctx, prob, alg, nopts = _sh_setup(bk, dims, lengths, lstar)
    cp = P.ContinuationPar(dsmin=1e-5, dsmax=0.002, ds=0.001, p_min=lstar - 0.05, p_max=lstar + 0.05, max_steps=4, nev=6,
                           newton_options=nopts, detect_bifurcation=0)
    br = _point_at(bk, ctx, lstar, 2)
    it = P.ContIterable(prob, alg, cp, P.norminf)
    nfm = bk.normalform
    bp = nfm.get_normal_formNd(it, br, 0, zetas=[_dct_mode(dims, m) for m in modes])
    before, after = nfm.predictor_nd(bp, cp.ds)
    for roots, dp in ((before, -cp.ds), (after, cp.ds)):
        for r in roots:
            assert np.max(np.abs(bp.reduced_form(r[::-1], dp))) < 1e-9, (r, bp.reduced_form(r[::-1], dp))
    first = nfm.get_first_points_on_branch(bp, (before, after), prob, cp, normN=P.norminf)
    for pts in (first.before, first.after):
        host = [v.numpy() for v in pts]
        for a in range(len(host)):
            for b in range(a):
                assert np.max(np.abs(host[a] - host[b])) > 1e-6
    states = []
    out = nfm.multicontinuation(br, 0, prob, alg, cp, normC=P.norminf, bpnf=bp, solfromRE=(before, after),
                                callback=lambda st: states.append((st.z_u.numpy(), st.z_p)) or True)
    print(f"multicontinuation 48x48: {len(before)} / {len(after)} roots of the reduced equation before / after l*, "
          f"{len(first.before)} / {len(first.after)} corrected points, {len(out)} branches")
    assert len(out) == len(first.before) + len(first.after) - 2 and len(out) >= 1
    sh = problems.SwiftHohenberg(dims, lengths, nu=1.3)
    assert len(states) >= 2 * len(out)
    for u, l in states:
        assert np.max(np.abs(sh.F(u, l))) < 10 * nopts.tol


def _spectral_nf(ps, lstar, zetas, zetas_ad, nu):
    """b20, b30 of the trivial periodic SH state restated in Fourier space, where J = l* - L1 is diagonal: the singular solves
    divide by the symbol off the kernel modes and leave those modes at 0 (⟨ζ_i, w⟩ = 0)"""
    sym = lstar - ps.symbol
    inv = np.divide(1.0, sym, out=np.zeros_like(sym), where=np.abs(sym) > 1e-9)
    solve = lambda r: ps.apply_symbol(r, inv)
    E = lambda r: r - sum(np.dot(r, za) * z for z, za in zip(zetas, zetas_ad))
    d2 = lambda a, b: 2 * nu * a * b
    N = len(zetas)
    w = {(a, b): solve(E(d2(zetas[a], zetas[b]))) for a in range(N) for b in range(N)}
    b20 = np.array([[[np.dot(zetas_ad[i], d2(zetas[j], zetas[k])) for k in range(N)] for j in range(N)] for i in range(N)])
    b30 = np.zeros((N,) * 4)
    for i in range(N):
        for j in range(N):
            for k in range(N):
                for l in range(N):
                    v = (-6 * zetas[j] * zetas[k] * zetas[l] - d2(zetas[j], w[l, k]) - d2(zetas[k], w[l, j])
                         - d2(zetas[l], w[k, j]))
                    b30[i, j, k, l] = np.dot(zetas_ad[i], v)
    return dict(b20=b20, b30=b30)


def test_periodic_box_four_dimensional_kernel(bk):
    """Periodic SH2d 64^2 on lx = ly = 2 pi: the wavenumbers |k| = 1 -- cos x, sin x, cos y, sin y -- cross together at l* = 0,
    N = 4.  With those ζs given, the tensors match the spectral restatement; the two-border device solves (FFT-preconditioned
    GMRES) leave two kernel directions free, which the Gram projection removes"""
    import warnings
    from tests.sh_periodic_oracle import PeriodicSH
    dims, lengths = (64, 64), (2 * np.pi, 2 * np.pi)
    ps = PeriodicSH(dims, lengths, l=0.0, nu=1.3)
    lstar = float(ps.symbol.min())
    assert lstar == 0.0 and int(np.sum(ps.symbol == lstar)) == 4
    P = bk.palc
    ctx = bk.Context(bk.BK_SH2D_PERIODIC, dims, lengths, krylov_m=100, params=(lstar, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
    ls = bk.GMRESB200(reltol=1e-11, restart=100, maxiter=300, Pl=True, orth="cgs2")
    nopts = P.NewtonPar(tol=1e-10, max_iterations=10, linsolver=ls)
    prob = P.BifurcationProblemB200(ctx, ctx.zeros(), (lstar, 1.3), lens=0)
    cp = P.ContinuationPar(nev=8, newton_options=nopts)
    it = P.ContIterable(prob, P.PALC(bls=bk.MatrixFreeBLSB200(ls)), cp, P.norminf)
    br = _point_at(bk, ctx, lstar, 4, nev=8)
    X = -lengths[0] + 2 * lengths[0] / dims[0] * np.arange(dims[0])
    Y = -lengths[1] + 2 * lengths[1] / dims[1] * np.arange(dims[1])
    one = np.ones((dims[1], dims[0]))
    zetas = [(f(X)[None, :] * one).ravel() for f in (np.cos, np.sin)] + [(f(Y)[:, None] * one).ravel() for f in (np.cos, np.sin)]
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        bp = bk.normalform.get_normal_formNd(it, br, 0, zetas=zetas)
    print(f"periodic 64^2, N = 4: {len(caught)} solver warnings {[str(c.message) for c in caught]}")
    assert bp.type == "4-d"
    ref = _spectral_nf(ps, lstar, [z.numpy() for z in bp.zetas], [z.numpy() for z in bp.zetas_ad], 1.3)
    _check_against_oracle(bp, ref, 4)
