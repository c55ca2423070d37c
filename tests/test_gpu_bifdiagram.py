"""GPU tests of the automatic bifurcation diagram (bifurcationkit.jl_b200/bifdiagram.py): sibling branches continued at once, each
on its own replicated context, give the bits of the sequential composition on one context; every saved state solves the
oracle's residual; the contexts are bounded and their memory comes back.  On the 48 x 48 square of test_gpu_nd_normal_form.py
(an nd point, delta (2, 0)) and on the set-up of examples/SH2d-fronts.jl (151 x 100)."""
import gc
import threading

import numpy as np
import pytest

import __graft_entry__ as g
from oracle import problems
from tests.test_gpu_nd_normal_form import SQUARE, _crossing_multi, _sh_setup

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


def _host(v):
    return None if v is None else (v.numpy() if hasattr(v, "numpy") else np.asarray(v))


def _same_branch(a, b):
    """rows, special points (with their states) and final state identical, bit for bit"""
    assert a.rows == b.rows
    assert len(a.specialpoint) == len(b.specialpoint)
    for s, t in zip(a.specialpoint, b.specialpoint):
        for f in ("type", "idx", "param", "norm", "step", "status", "delta", "ind_ev", "interval", "tau_p", "precision"):
            assert getattr(s, f) == getattr(t, f), f
        for f in ("x", "tau_u"):
            assert np.array_equal(_host(getattr(s, f)), _host(getattr(t, f))), f
    assert np.array_equal(a.state.z_u.numpy(), b.state.z_u.numpy()) and a.state.z_p == b.state.z_p


def _states(node):
    """every device state the diagram keeps below node: the special points' states and each branch's final state"""
    for c in node.child:
        yield c.gamma.state.z_u, c.gamma.state.z_p
        for s in c.gamma.specialpoint:
            if s.x is not None:
                yield s.x, s.param
        yield from _states(c)


def _children(P, cp_root, **kw):
    return lambda x, p, lvl: cp_root if lvl <= 1 else P.ContinuationPar(**{**vars(cp_root), **kw})


@pytest.fixture(scope="module")
def square(bk):
    """the trivial branch of the 48 x 48 square through its nd point (test_square_box_has_one_nd_point)"""
    dims, lengths = SQUARE
    lstar, modes, gap = _crossing_multi(dims, lengths)
    P, ctx, prob, alg, nopts = _sh_setup(bk, dims, lengths, lstar - 0.01)
    cp = P.ContinuationPar(dsmin=1e-5, dsmax=0.002, ds=0.002, p_min=lstar - 0.011, p_max=lstar + 0.8 * gap, max_steps=40, nev=6,
                           newton_options=nopts, detect_bifurcation=3, n_inversion=8)
    br = bk.events.continuation(prob, alg, cp, normC=P.norminf)
    options = _children(P, cp, ds=0.001, p_min=lstar - 0.05, p_max=lstar + 0.05, max_steps=4)
    return P, ctx, prob, alg, br, options


def test_square_diagram_is_the_sequential_composition(bk, square):
    """Level 2 from the nd point at l ~ 0.0035 (delta (2, 0)): the children are the branches multicontinuation gives there; with
    max_workers = 4 and 1 their rows, special points and states are those of the explicit calls on the one context, bit for bit;
    every saved state solves the oracle's sparse residual to 1e-8"""
    P, ctx, prob, alg, br, options = square
    D, nfm = bk.bifdiagram, bk.normalform
    i = next(k for k, s in enumerate(br.specialpoint) if s.type == "nd")
    pt = br.specialpoint[i]
    assert pt.delta == (2, 0) and abs(pt.param - 0.0035283) < 1e-3
    cp = options(pt.x, pt.param, 2)
    ref = nfm.multicontinuation(br, i, prob, alg, cp, normC=P.norminf, nev=cp.nev, ampfactor=1.0)
    assert len(ref) >= 1
    for workers in (4, 1):
        d = D.bifurcationdiagram_from(prob, br, 2, options, alg, normC=P.norminf, max_workers=workers)
        assert d.failures == [] and [c.code for c in d.child] == [i] * len(ref)
        for c, (b, nf) in zip(d.child, ref):
            _same_branch(c.gamma, b)
            assert c.nf.type == nf.type == "2-d"
            assert all(z.ctx is ctx for z in c.nf.zetas) and c.gamma.state.z_u.ctx is ctx   # moved onto the diagram's context
        sh = problems.SwiftHohenberg(*SQUARE, nu=1.3)
        n = 0
        for u, p in _states(d):
            assert np.max(np.abs(sh.F(u.numpy(), p))) <= 1e-8
            n += 1
        print(f"48x48 diagram, max_workers = {workers}: {len(d.child)} branches, {n} states checked")


def test_square_contexts_are_bounded_and_memory_comes_back(bk, square, monkeypatch):
    """The live-context count never exceeds max_workers + 1 (counted around Context.__init__ / close); once the diagram and its
    context are dropped, free device memory is back within 1 MB"""
    import torch
    P, ctx0, prob0, alg, br, options = square
    lock, live, peak = threading.Lock(), [0], [0]
    init, close = bk.Context.__init__, bk.Context.close

    def counted_init(self, *a, **k):
        init(self, *a, **k)
        with lock:
            live[0] += 1
            peak[0] = max(peak[0], live[0])

    def counted_close(self):
        if getattr(self, "handle", None):
            with lock:
                live[0] -= 1
        close(self)
    monkeypatch.setattr(bk.Context, "__init__", counted_init)
    monkeypatch.setattr(bk.Context, "close", counted_close)
    torch.cuda.synchronize()
    gc.collect()
    free0 = torch.cuda.mem_get_info()[0]
    ctx = ctx0.replicate()                     # the diagram's own context, reading the branch of ctx0
    prob = P.BifurcationProblemB200(ctx, ctx.zeros(), prob0.params, lens=0, record=prob0.record)
    for workers in (2, 1):
        peak[0] = live[0]
        d = bk.bifdiagram.bifurcationdiagram_from(prob, br, 2, options, alg, normC=P.norminf, max_workers=workers)
        assert len(d.child) >= 1 and peak[0] <= workers + 1   # the units' contexts and the diagram's
        del d
    assert live[0] == 1
    del prob
    ctx.close()
    gc.collect()
    torch.cuda.synchronize()
    free1 = torch.cuda.mem_get_info()[0]
    print(f"peak live contexts {peak[0]} (the diagram's included), free memory before {free0 / 2**20:.1f} MiB after "
          f"{free1 / 2**20:.1f} MiB")
    assert live[0] == 0 and abs(free1 - free0) <= 2**20


# ------------------------------------------------------------------------------------------------ examples/SH2d-fronts.jl
FRONTS = ((151, 100), (8 * np.pi, 4 * np.pi / np.sqrt(3)))


def test_sh2d_fronts_diagram(bk):
    """examples/SH2d-fronts.jl:8-11 and its optionsCont (:143-152), level 2, from a short hexagon branch (max_steps 20 instead of
    146, children 10): the diagram completes, every state solves the oracle's residual, and max_workers = 1 gives the bits of the
    default"""
    P = bk.palc
    dims, lengths = FRONTS
    ctx = bk.Context(bk.BK_SH2D, dims, lengths, krylov_m=100, params=(-0.1, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(reltol=1e-11, restart=100, maxiter=300, Pl=True, orth="cgs2")
    eig = bk.ShiftInvertB200(0.1, ls, krylovdim=40, tol=1e-11, maxrestart=30)              # EigArpack(0.1, :LM)
    prob = P.BifurcationProblemB200(ctx, ctx.to_device(problems.sh2d_sol0(*dims, *lengths)), (-0.1, 1.3), lens=0,
                                    record=lambda v: v.norminf())
    hexa = P.newton(prob, prob.u0, -0.1, P.NewtonPar(tol=1e-8, max_iterations=20, linsolver=ls), P.norminf)
    assert hexa.converged
    prob.u0 = hexa.u
    optcont = P.ContinuationPar(dsmin=1e-4, dsmax=0.005, ds=-0.001, p_max=0.0, p_min=-1.0, max_steps=20, detect_bifurcation=3,
                                nev=10, n_inversion=6, newton_options=P.NewtonPar(tol=1e-9, max_iterations=15, linsolver=ls,
                                                                                  eigsolver=eig))

    def options(x, p, lvl):                                                                 # optionsCont
        if lvl <= 1:
            return optcont
        return P.ContinuationPar(**{**vars(optcont), **dict(detect_bifurcation=3, ds=0.001, a=0.75, max_steps=10)})
    alg = P.PALC(bls=bk.MatrixFreeBLSB200(ls))
    d = bk.bifdiagram.bifurcationdiagram(prob, alg, 2, options, normC=P.norminf)
    one = bk.bifdiagram.bifurcationdiagram_from(prob, d.gamma, 2, options, alg, normC=P.norminf, max_workers=1)
    sh = problems.SwiftHohenberg(dims, lengths, nu=1.3)
    pts = [(s.type, s.param, s.delta) for s in d.gamma.specialpoint]
    print(f"SH2d fronts 151x100: root special points {pts}, {len(d.child)} children, failures {d.failures}")
    assert [c.code for c in one.child] == [c.code for c in d.child]
    assert [(f[0], f[1]) for f in one.failures] == [(f[0], f[1]) for f in d.failures]
    for a, b in zip(d.child, one.child):
        _same_branch(a.gamma, b.gamma)
    for u, p in _states(d):
        assert np.max(np.abs(sh.F(u.numpy(), p))) <= 1e-8


# ------------------------------------------------------------------------------------------------ several units at once
def test_three_units_at_once_give_the_bits_of_one_at_a_time(bk, monkeypatch):
    """The trivial SH2d state on the 151 x 100 domain of examples/SH2d-fronts.jl, its branch up to the third crossing (two bp
    points after the start, so two units): with max_workers = 4 at least two units run at once, never more than max_workers + 1 contexts live, and
    every child's rows, special points and states equal those of max_workers = 1, in the same order"""
    from tests.test_gpu_normal_form import _dct_eigs
    P = bk.palc
    dims, lengths = FRONTS
    lam = np.add.outer(_dct_eigs(dims[0], lengths[0]), _dct_eigs(dims[1], lengths[1]))
    m = np.unique(np.round(((1 + lam) ** 2).ravel(), 12))
    l0, l1 = m[0] - 0.01, 0.5 * (m[2] + m[3])
    _, ctx, prob, alg, nopts = _sh_setup(bk, dims, lengths, l0)
    step = min(0.002, (l1 - l0) / 30)
    cp = P.ContinuationPar(dsmin=1e-6, dsmax=step, ds=step, p_min=l0 - 1e-3, p_max=l1, max_steps=200, nev=8, newton_options=nopts,
                           detect_bifurcation=3, n_inversion=8)
    br = bk.events.continuation(prob, alg, cp, normC=P.norminf)
    units = [i for i, s in enumerate(br.specialpoint) if s.step > 1 and s.type in ("bp", "nd")]
    assert len(units) >= 2, [(s.type, s.param, s.delta) for s in br.specialpoint]
    options = _children(P, cp, ds=step / 2, max_steps=4, p_min=l0 - 0.05, p_max=l1 + 0.05)

    lock, live, peak, running, most = threading.Lock(), [1], [1], [0], [0]
    init, close, branch_at = bk.Context.__init__, bk.Context.close, bk.bifdiagram._branch_at

    def counted_init(self, *a, **k):
        init(self, *a, **k)
        with lock:
            live[0] += 1
            peak[0] = max(peak[0], live[0])

    def counted_close(self):
        if getattr(self, "handle", None):
            with lock:
                live[0] -= 1
        close(self)

    def counted_unit(*a, **k):
        with lock:
            running[0] += 1
            most[0] = max(most[0], running[0])
        try:
            return branch_at(*a, **k)
        finally:
            with lock:
                running[0] -= 1
    monkeypatch.setattr(bk.Context, "__init__", counted_init)
    monkeypatch.setattr(bk.Context, "close", counted_close)
    monkeypatch.setattr(bk.bifdiagram, "_branch_at", counted_unit)
    d4 = bk.bifdiagram.bifurcationdiagram_from(prob, br, 2, options, alg, normC=P.norminf, max_workers=4)
    peak4, most4 = peak[0], most[0]
    peak[0], most[0] = live[0], 0
    d1 = bk.bifdiagram.bifurcationdiagram_from(prob, br, 2, options, alg, normC=P.norminf, max_workers=1)
    print(f"151x100 trivial state: {len(units)} units, {len(d4.child)} children, at most {most4} units and {peak4} contexts "
          f"at once with max_workers = 4, {most[0]} / {peak[0]} with 1")
    assert most4 >= 2 and peak4 <= 4 + 1 and most[0] == 1 and peak[0] <= 2
    assert d4.failures == [] == d1.failures and len(d4.child) >= len(units)
    assert [c.code for c in d4.child] == [c.code for c in d1.child]
    for a, b in zip(d4.child, d1.child):
        _same_branch(a.gamma, b.gamma)
        assert a.nf.type == b.nf.type and a.nf.p == b.nf.p
    sh = problems.SwiftHohenberg(dims, lengths, nu=1.3)
    for u, p in _states(d4):
        assert np.max(np.abs(sh.F(u.numpy(), p))) <= 1e-8
