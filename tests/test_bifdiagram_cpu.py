"""CPU tests of the automatic bifurcation diagram (bifurcationkit.jl_b200/bifdiagram.py) on host problems with the oracle's dense
solvers, pinned to the reference's test/normal_forms/testNF.jl diagrams (:96-99, :149-152, :291-310, :327-363): the tree's shape,
the branching rule, bit-identity with an explicit sequential recursion, failures recorded on their node, and Context /
BifurcationProblemB200.replicate against a fake library (no GPU needed)."""
import ctypes as C
import dataclasses
import threading

import numpy as np
from numpy.polynomial import Polynomial
import pytest

import __graft_entry__ as g
from oracle import krylov, bls as obls
from tests.test_host_logic_cpu import BlsAdapter
from tests.test_normal_form_cpu import BpProblem, Fbp, Jbp, dense_eig, MU
from tests.test_nd_normal_form_cpu import DenseBlockBLS, JetProblem, _d6_problem, _fbp2d


def _opts(**kw):
    """testNF.jl opts_br"""
    P = g.load_package().palc
    nopts = P.NewtonPar(tol=1e-14, linsolver=krylov.DefaultLS(), eigsolver=dense_eig)
    return P.ContinuationPar(**{**dict(dsmin=0.001, dsmax=0.05, ds=0.01, p_max=0.4, p_min=-0.5, detect_bifurcation=3,
                                       newton_options=nopts, max_steps=100, n_inversion=8), **kw})


def _tol(cp, tol):
    return dataclasses.replace(cp, newton_options=dataclasses.replace(cp.newton_options, tol=tol))


class BothBLS(BlsAdapter):
    """the bordered solver of both normal forms: MatrixBLS for the 1-d form, the dense block solve for the N-d form"""

    def __init__(self):
        super().__init__(obls.MatrixBLS())

    def solve_block(self, *args, **kw):
        return DenseBlockBLS().solve_block(*args, **kw)


def _alg():
    return g.load_package().palc.PALC(bls=BlsAdapter(obls.MatrixBLS()))


def _secbif_problem():
    """testNF.jl:291-293: FbpSecBif(u, p) = -u (p + u (2 - 5u)) (p - 0.15 - u (2 + 20u)), with its jets"""
    poly = lambda q: Polynomial([0, -1]) * Polynomial([q[0], 2, -5]) * Polynomial([q[0] - 0.15, -2, -20])
    return JetProblem(lambda u, q: poly(q)(u), lambda u, q: np.array([[poly(q).deriv(1)(u[0])]]),
                      lambda u, q, a, b: poly(q).deriv(2)(u[0]) * a * b,
                      lambda u, q, a, b, c: poly(q).deriv(3)(u[0]) * a * b * c, np.zeros(1), [-0.2], 0)


SECBIF = dict(p_min=-1.0, p_max=0.3, ds=0.001, dsmax=0.005, n_inversion=8, dsmin_bisection=1e-18, tol_bisection_eigenvalue=1e-11,
              max_bisection_steps=20)
D6 = dict(p_min=-0.25, p_max=0.4, ds=0.001, dsmax=0.005, n_inversion=4, dsmin_bisection=1e-18, tol_bisection_eigenvalue=1e-11,
          max_bisection_steps=20)


# ------------------------------------------------------------------------------------------------ the sequential composition
def _sequential(prob, alg, br, maxlevel, options, normC, lvl=1, halfbranch=False, **kw):
    """bifurcationdiagram! (src/bifdiagram/BifurcationDiagram.jl:157-231) written out with events.continuation's branch,
    continuation_from_bp and multicontinuation, one call after another: [(index, Branch, normal form, children)]"""
    nfm = g.load_package().normalform
    if lvl >= maxlevel:
        return []
    out = []
    for ind, pt in enumerate(br.specialpoint):
        if pt.step <= 1 or pt.type not in ("bp", "nd"):
            continue
        cp0 = options(pt.x, pt.param, lvl + 1)

        def branch(dsfactor=1.0, ampfactor=1.0):
            cp = dataclasses.replace(cp0, ds=cp0.ds * dsfactor)
            if abs(pt.delta[0]) > 1:
                return nfm.multicontinuation(br, ind, prob, alg, cp, normC=normC, nev=cp.nev, ampfactor=ampfactor, **kw)
            return nfm.continuation_from_bp(br, ind, prob, alg, cp, normC=normC, nev=cp.nev, ampfactor=ampfactor, **kw)
        kids = branch()
        if kids is None:
            continue
        if not isinstance(kids, list):
            kids = [kids]
            if not halfbranch and kids[0][1].type == "Transcritical":
                kids.append(branch(dsfactor=-1.0))
            if not halfbranch and kids[-1][1].type == "Pitchfork":
                kids.append(branch(ampfactor=-1.0))
        out += [(ind, b, nf, None) for b, nf in kids]
    return [(ind, b, nf, _sequential(prob, alg, b, maxlevel, options, normC, lvl + 1, halfbranch, **kw)) for ind, b, nf, _ in out]


def _same_branch(a, b):
    """rows, special points (with their states) and final state identical, bit for bit"""
    assert a.rows == b.rows
    assert len(a.specialpoint) == len(b.specialpoint)
    for s, t in zip(a.specialpoint, b.specialpoint):
        for f in ("type", "idx", "param", "norm", "step", "status", "delta", "ind_ev", "interval", "tau_p", "precision"):
            assert getattr(s, f) == getattr(t, f), f
        for f in ("x", "tau_u"):
            assert (getattr(s, f) is None) == (getattr(t, f) is None) and np.array_equal(getattr(s, f), getattr(t, f)), f
    assert np.array_equal(a.state.z_u, b.state.z_u) and a.state.z_p == b.state.z_p


def _same_tree(node, seq):
    assert [c.code for c in node.child] == [ind for ind, *_ in seq]
    for c, (ind, b, nf, kids) in zip(node.child, seq):
        _same_branch(c.gamma, b)
        assert c.nf.type == nf.type and c.nf.p == nf.p
        _same_tree(c, kids)


def _shape(node):
    return [(c.code, _shape(c)) for c in node.child]


# ------------------------------------------------------------------------------------------------ testNF.jl:96-99
def test_transcritical_diagram_has_both_directions():
    """The root has one bp; the Transcritical normal form gives two children (ds and -ds); every state of the children solves
    F = 0; halfbranch keeps the first"""
    bk = g.load_package()
    D, P = bk.bifdiagram, bk.palc
    prob = BpProblem(Fbp, Jbp, np.zeros(2), [-0.2, 0.0, 1.12, 0.234, 4.4323], MU)
    cp = _tol(_opts(p_min=-0.2, p_max=0.2, ds=0.01, max_steps=15), 1e-12)
    states, lock = [], threading.Lock()

    def keep(st):
        with lock:
            states.append((st.z_u.copy(), st.z_p))
    d = D.bifurcationdiagram(prob, _alg(), 2, cp, normC=P.norminf, callback=keep)
    assert [s.type for s in d.gamma.specialpoint] == ["bp", "endpoint"]
    assert D.size(d) == 3 and D.level(d) == 1 and D.hasbranch(d) and d.code is None and d.failures == []
    assert [c.code for c in d.child] == [0, 0] and all(c.level == 2 and c.nf.type == "Transcritical" for c in d.child)
    assert d.child[0].nf is not d.child[1].nf
    # the two branches leave the point on opposite sides of the parameter
    p0 = d.child[0].nf.p
    assert d.child[0].gamma.rows[-1]["param"] == 0.2 and d.child[1].gamma.rows[-1]["param"] == -0.2
    assert all(c.gamma.rows[-1]["x"] > 0.2 for c in d.child) and all(abs(c.nf.p - p0) == 0 for c in d.child)
    assert len(states) == len(d.gamma.rows) + sum(len(c.gamma.rows) for c in d.child)   # the root branch gets the callback too
    for u, p in states:
        assert np.max(np.abs(Fbp(u, prob._par(p)))) < 1e-10
    half = D.bifurcationdiagram(prob, _alg(), 2, cp, normC=P.norminf, halfbranch=True)
    assert D.size(half) == 2
    _same_branch(half.child[0].gamma, d.child[0].gamma)


# ------------------------------------------------------------------------------------------------ testNF.jl:149-152
def test_pitchfork_diagram_has_both_amplitudes():
    """prob_pf of testNF.jl:117-119 with gamma = 0 (with its gamma = 1.422 the normal form is Transcritical, b20 / 2 = gamma), the
    options of :149-152: two Pitchfork children with ampfactor +1 and -1, whose first points have x[1] of opposite signs; one
    child with halfbranch"""
    bk = g.load_package()
    D, P = bk.bifdiagram, bk.palc
    prob = BpProblem(Fbp, Jbp, np.zeros(2), [-0.2, 0.0, 0.0, -1.0, 0.0], MU, record=lambda x: float(x[0]))
    cp = _tol(_opts(p_min=-1.0, p_max=0.5, ds=0.01, dsmax=0.05, n_inversion=6, max_bisection_steps=30, max_steps=15), 1e-12)
    d = D.bifurcationdiagram(prob, _alg(), 2, cp, normC=P.norminf)
    assert [(c.code, c.nf.type) for c in d.child] == [(0, "Pitchfork"), (0, "Pitchfork")]
    x1 = [c.gamma.rows[1]["x"] for c in d.child]
    assert x1[0] * x1[1] < 0 and abs(x1[0] + x1[1]) < 1e-12
    half = D.bifurcationdiagram(prob, _alg(), 2, cp, normC=P.norminf, halfbranch=True)
    assert len(half.child) == 1
    _same_branch(half.child[0].gamma, d.child[0].gamma)


# ------------------------------------------------------------------------------------------------ testNF.jl:291-310
def test_secondary_bifurcations_are_branched_from_level_three():
    """FbpSecBif: at level 2 the children's own bp points are recorded but not branched; at level 3 they are, and every grandchild
    equals continuation_from_bp called on its parent with the same arguments"""
    bk = g.load_package()
    D, P, nfm = bk.bifdiagram, bk.palc, bk.normalform
    prob, alg, cp = _secbif_problem(), _alg(), _opts(**SECBIF)
    d2 = D.bifurcationdiagram(prob, alg, 2, cp, normC=P.norminf)
    assert [s.type for s in d2.gamma.specialpoint] == ["bp", "bp", "endpoint"]
    assert [c.code for c in d2.child] == [0, 0, 1, 1]
    assert any(s.type == "bp" and s.step > 1 for c in d2.child for s in c.gamma.specialpoint)
    assert all(c.child == [] for c in d2.child)
    d3 = D.bifurcationdiagram(prob, alg, 3, cp, normC=P.norminf)
    assert D.size(d3) > D.size(d2) == 5
    grand = 0
    for c in d3.child:
        _same_branch(c.gamma, d2.child[d3.child.index(c)].gamma)
        for k in c.child:
            pt = c.gamma.specialpoint[k.code]
            first = next(j for j in c.child if j.code == k.code)   # the second branch: -ds (Transcritical), ampfactor -1 (Pitchfork)
            ds, amp = (1.0, 1.0) if k is first else ((-1.0, 1.0) if first.nf.type == "Transcritical" else (1.0, -1.0))
            br, nf = nfm.continuation_from_bp(c.gamma, k.code, prob, alg, dataclasses.replace(cp, ds=cp.ds * ds), normC=P.norminf,
                                              nev=cp.nev, ampfactor=amp)
            _same_branch(k.gamma, br)
            assert k.nf.type == nf.type and k.nf.p == pt.param and k.level == 3
            grand += 1
    assert grand == D.size(d3) - 5


# ------------------------------------------------------------------------------------------------ an nd point
def test_nd_point_goes_through_multicontinuation():
    """Fbp2d (testNF.jl:224-287, gamma = 10): the diagram sends its nd point to multicontinuation, and its children are the
    branches that call gives with the same arguments, in the same order"""
    bk = g.load_package()
    D, P, nfm = bk.bifdiagram, bk.palc, bk.normalform
    F, J, d2, d3 = _fbp2d(dict(alpha=-1.0, gamma=10.0, A=0.123, B=0.234, C=0.456))
    prob = JetProblem(F, J, d2, d3, np.zeros(3), [-0.2], 0)
    alg = _alg()
    cp = _opts(p_max=0.2)
    child = dataclasses.replace(cp, max_steps=12, dsmax=0.01, ds=0.005)
    d = D.bifurcationdiagram(prob, alg, 2, lambda x, p, lvl: cp if lvl == 1 else child, normC=P.norminf, bls=BothBLS())
    i = next(k for k, s in enumerate(d.gamma.specialpoint) if s.type == "nd")
    assert abs(d.gamma.specialpoint[i].delta[0]) == 2
    mine = D.get_branches_from_BP(d, i)
    ref = nfm.multicontinuation(d.gamma, i, prob, alg, child, normC=P.norminf, nev=child.nev, ampfactor=1.0, bls=BothBLS())
    assert len(mine) == len(ref) >= 1
    for k, (br, nf) in zip(mine, ref):
        _same_branch(k.gamma, br)
        assert k.code == i and k.nf.type == nf.type == "2-d"
        for a, b in zip(k.nf.zetas, nf.zetas):
            assert np.array_equal(a, b)


# ------------------------------------------------------------------------------------------------ testNF.jl:327-363
def test_d6_diagram_shape_and_getters():
    """FbpD6 at level 3 with the options of :359-361: the tree the explicit calls give, get_branch and get_branches_from_BP"""
    bk = g.load_package()
    D, P = bk.bifdiagram, bk.palc
    prob, alg, cp = _d6_problem(), _alg(), _opts(**D6)
    d = D.bifurcationdiagram(prob, alg, 3, lambda x, p, lvl: cp, normC=P.norminf, bls=BothBLS())
    seq = _sequential(prob, alg, d.gamma, 3, lambda x, p, lvl: cp, P.norminf, bls=BothBLS())
    assert _shape(d) == [(ind, [(i2, _shape_seq(k2)) for i2, _, _, k2 in kids]) for ind, _, _, kids in seq]
    assert [s.type for s in d.gamma.specialpoint] == ["nd", "endpoint"] and len(d.child) >= 2
    assert D.get_branch(d, (1,)) is d.child[1] and d[1] is d.child[1] and d[1, 0] is d.child[1].child[0]
    assert D.get_branch(d, ()) is d
    assert D.get_branches_from_BP(d, 0) == d.child
    assert D.size(d) == 1 + sum(D.size(c) for c in d.child) and D.size(d, (1,)) == 1 + len(d.child[1].child)
    assert all(c.level == 2 and c.nf.type == "3-d" for c in d.child)


def _shape_seq(kids):
    return [(i, _shape_seq(k)) for i, _, _, k in kids]


# ------------------------------------------------------------------------------------------------ bit-identity
@pytest.mark.parametrize("case", ["secbif", "d6"])
def test_concurrent_diagram_equals_the_sequential_composition(case):
    """max_workers = 4 against the explicit sequential recursion: every branch's rows, special points and states identical, in the
    same child order, at every level"""
    bk = g.load_package()
    D, P = bk.bifdiagram, bk.palc
    if case == "secbif":
        prob, kw, cp = _secbif_problem(), {}, _opts(**SECBIF)
    else:
        prob, kw, cp = _d6_problem(), dict(bls=BothBLS()), _opts(**D6)
    alg = _alg()
    d = D.bifurcationdiagram(prob, alg, 3, cp, normC=P.norminf, max_workers=4, **kw)
    seq = _sequential(prob, alg, d.gamma, 3, lambda x, p, lvl: cp, P.norminf, **kw)
    _same_tree(d, seq)
    one = D.bifurcationdiagram(prob, alg, 3, cp, normC=P.norminf, max_workers=1, **kw)
    _same_tree(one, seq)


# ------------------------------------------------------------------------------------------------ failures
def test_a_failing_unit_is_recorded_and_its_siblings_complete():
    """FbpSecBif: an exception raised while branching at the first bp, and a corrector that cannot converge at the second (one
    Newton iteration allowed, tolerance 0): the first is recorded on the node with its point and parameter, the second gives
    branches that end at their first step, and the rest of the tree goes on"""
    bk = g.load_package()
    D, P = bk.bifdiagram, bk.palc
    prob, alg, cp = _secbif_problem(), _alg(), _opts(**SECBIF)
    ref = D.bifurcationdiagram(prob, alg, 2, cp, normC=P.norminf)
    p_first = ref.gamma.specialpoint[0].param

    def options(x, p, lvl):
        if lvl == 2 and p == p_first:
            raise RuntimeError("injected")
        return cp
    d = D.bifurcationdiagram(prob, alg, 2, options, normC=P.norminf, max_workers=2)
    assert len(d.failures) == 1
    ind, p, err = d.failures[0]
    assert ind == 0 and p == p_first and isinstance(err, RuntimeError) and str(err) == "injected"
    assert [c.code for c in d.child] == [1, 1]
    for c, r in zip(d.child, [c for c in ref.child if c.code == 1]):
        _same_branch(c.gamma, r.gamma)

    # the exception comes after the first Transcritical branch: that branch is kept, as the reference's add! before the throw
    calls = []

    def second_fails(x, p, lvl):
        if lvl == 2 and p == p_first:
            calls.append(p)
            if len(calls) == 2:
                raise ValueError("second")
        return cp
    d = D.bifurcationdiagram(prob, alg, 2, second_fails, normC=P.norminf)
    assert [c.code for c in d.child] == [0, 1, 1] and [f[0] for f in d.failures] == [0]
    _same_branch(d.child[0].gamma, ref.child[0].gamma)

    # a corrector that cannot converge: no exception, the branches stop where the reference's would
    bad = _tol(dataclasses.replace(cp, newton_options=dataclasses.replace(cp.newton_options, max_iterations=1)), 0.0)
    d = D.bifurcationdiagram(prob, alg, 2, lambda x, p, lvl: cp if lvl == 1 else bad, normC=P.norminf)
    assert d.failures == [] and [c.code for c in d.child] == [0, 0, 1, 1]
    assert all(len(c.gamma.rows) <= 2 for c in d.child)


# ------------------------------------------------------------------------------------------------ replication
class _FakeLib:
    """the ctypes functions Context, DeviceVec and BifurcationProblemB200 call, recording their arguments"""

    def __init__(self):
        self.calls, self.next = [], 0x1000

    def _h(self, ref):
        self.next += 0x100
        ref._obj.value = self.next

    def bk_ctx_create(self, device, kind, d, L, m, h):
        self._h(h)
        self.calls.append(("create", device, kind, tuple(d), tuple(L), m))
        return 0

    def bk_problem_size(self, h):
        return 48 * 48

    bk_state_size = bk_problem_size

    def bk_jac_set_transpose(self, h, on):
        return 0

    def bk_set_params(self, h, p, n):
        self.calls.append(("params", h.value, tuple(p[i] for i in range(n))))
        return 0

    def bk_precond_setup(self, h, kind, a0, a1):
        self.calls.append(("precond", h.value, kind, a0, a1))
        return 0

    def bk_vec_alloc(self, h, n, out):
        self._h(out)
        return 0

    def bk_vec_copy(self, h, dst, src, n):
        self.calls.append(("copy", h.value, dst, src, n))
        return 0

    def bk_vec_free(self, h, p):
        return 0

    def bk_ctx_destroy(self, h):
        self.calls.append(("destroy", h.value))
        return 0


def test_replicate_keeps_every_creation_argument_and_the_preconditioner_set_up(monkeypatch):
    bk = g.load_package()
    fake = _FakeLib()
    monkeypatch.setattr(bk.lib, "load", lambda: fake)
    ctx = bk.Context(bk.BK_SH2D, (48, 48), (7.2, 7.2), krylov_m=40, device=0, params=(-0.1, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0, -1.0)
    ctx.set_params((0.2, 1.3))
    ctx.precond_setup(bk.BK_PC_CGL_DST, 2.0, 1.0)
    ctx.set_params((0.3, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 3.0, 1.0)     # replaces the first set-up of its kind
    ctx.set_params((0.4, 1.3))
    ctx.pin_host = True
    assert ctx.precond_calls == [(bk.BK_PC_CGL_DST, 2.0, 1.0, (0.2, 1.3)), (bk.BK_PC_SH_DCT, 3.0, 1.0, (0.3, 1.3))]
    n0 = len(fake.calls)
    new = ctx.replicate()
    h = new.handle.value
    assert h != ctx.handle.value
    # each set-up is replayed at the params it was made with, then the context's current params are set
    assert fake.calls[n0:] == [("create", 0, bk.BK_SH2D, (48, 48, 1), (7.2, 7.2, 1.0), 40), ("params", h, (0.4, 1.3)),
                               ("params", h, (0.2, 1.3)), ("precond", h, bk.BK_PC_CGL_DST, 2.0, 1.0),
                               ("params", h, (0.3, 1.3)), ("precond", h, bk.BK_PC_SH_DCT, 3.0, 1.0), ("params", h, (0.4, 1.3))]
    assert (new.kind, new.dims, new.lengths, new.krylov_m, new.params, new.complex) == \
        (ctx.kind, ctx.dims, ctx.lengths, ctx.krylov_m, ctx.params, ctx.complex)
    assert new.precond_calls == ctx.precond_calls and new.pin_host
    cctx = bk.Context(bk.BK_SH2D, (48, 48), (7.2, 7.2), krylov_m=40, complex=True)
    n0 = len(fake.calls)
    assert cctx.replicate().complex and fake.calls[n0][2] == bk.BK_SH2D | bk.BK_COMPLEX

    u0 = ctx.zeros()
    rec = lambda x: 1.0
    prob = bk.palc.BifurcationProblemB200(ctx, u0, [-0.1, 1.3], lens=0, record=rec, delta=1e-7)
    n0 = len(fake.calls)
    rep = prob.replicate()
    assert rep.ctx is not ctx and rep.ctx.handle.value != ctx.handle.value
    assert fake.calls[n0][0] == "create" and ("copy", rep.ctx.handle.value, rep.u0.dptr, u0.dptr, u0.n) in fake.calls[n0:]
    assert rep.params == prob.params and rep.params is not prob.params
    assert (rep.lens, rep.record, rep.delta, rep.p0) == (0, rec, 1e-7, -0.1)
    on = prob.replicate(new)
    assert on.ctx is new and fake.calls[-1] == ("copy", new.handle.value, on.u0.dptr, u0.dptr, u0.n)
    host = np.arange(3.0)
    hp = bk.palc.BifurcationProblemB200(ctx, host, [-0.1, 1.3]).replicate(new)
    assert np.array_equal(hp.u0, host) and hp.u0 is not host

    class Sub(bk.palc.BifurcationProblemB200):
        pass
    with pytest.raises(NotImplementedError, match="Sub is not supported"):
        Sub(ctx, host, [-0.1, 1.3]).replicate(new)


# ------------------------------------------------------------------------------------------------ threads, cycles, keywords
def test_vector_lock_is_reentrant_for_a_collection_on_its_own_thread(monkeypatch):
    """A cyclic collection that runs on the thread holding a context's vector lock, and finalises a DeviceVec of that context,
    frees it instead of waiting forever on the lock"""
    import gc
    bk = g.load_package()
    fake = _FakeLib()
    freed = []
    fake.bk_vec_free = lambda h, p: freed.append(p) or 0
    monkeypatch.setattr(bk.lib, "load", lambda: fake)
    ctx = bk.Context(bk.BK_SH2D, (48, 48), (7.2, 7.2), krylov_m=40)
    done = []

    class Holder:
        pass

    def run():
        with ctx._vec_lock:
            h = Holder()
            h.me, h.v = h, bk.DeviceVec(ctx, 4)      # a DeviceVec only the cyclic collector can free
            p = h.v.dptr
            del h
            gc.collect()
            bk.DeviceVec(ctx, 4)
            done.append(p in freed)
    t = threading.Thread(target=run, daemon=True)
    t.start()
    t.join(10)
    assert not t.is_alive() and done == [True]


def test_a_failure_kept_on_a_node_leaves_no_reference_cycle():
    """Dropping a diagram with a failing unit frees the tree by reference counting: the failure keeps its traceback as text, not
    its frames (which hold the node)"""
    import gc
    import weakref
    bk = g.load_package()
    D, P = bk.bifdiagram, bk.palc
    prob, alg, cp = _secbif_problem(), _alg(), _opts(**SECBIF)

    calls = []

    def options(x, p, lvl):
        calls.append(lvl)
        if calls.count(2) == 1 and lvl == 2:
            raise RuntimeError("injected")
        return cp
    gc.disable()
    try:
        d = D.bifurcationdiagram(prob, alg, 2, options, normC=P.norminf, max_workers=1)
        assert len(d.failures) >= 1
        err = d.failures[0][2]
        assert str(err) == "injected" and err.__traceback__ is None and "_branch_at" in err.__notes__[0]
        refs = [weakref.ref(d)] + [weakref.ref(c) for c in d.child] + [weakref.ref(c.gamma) for c in d.child]
        del d
        assert all(r() is None for r in refs)
    finally:
        gc.enable()


def test_keywords_follow_the_reference(monkeypatch):
    """A keyword neither branch-switching call takes is refused, usedeflation = true is refused, a given nev wins over the options'
    and the root branch gets the callback"""
    import functools
    bk = g.load_package()
    D, P, nfm = bk.bifdiagram, bk.palc, bk.normalform
    prob, alg = BpProblem(Fbp, Jbp, np.zeros(2), [-0.2, 0.0, 1.12, 0.234, 4.4323], MU), _alg()
    cp = _tol(_opts(p_min=-0.2, p_max=0.2, ds=0.01, max_steps=15), 1e-12)
    with pytest.raises(TypeError, match="bsl"):
        D.bifurcationdiagram(prob, alg, 2, cp, normC=P.norminf, bsl=None)
    with pytest.raises(NotImplementedError, match="usedeflation"):
        D.bifurcationdiagram(prob, alg, 2, cp, normC=P.norminf, usedeflation=True)
    seen = []
    orig = nfm.continuation_from_bp

    @functools.wraps(orig)
    def spy(*a, **kw):
        seen.append(kw)
        return orig(*a, **kw)
    monkeypatch.setattr(nfm, "continuation_from_bp", spy)
    rows = []
    d = D.bifurcationdiagram(prob, alg, 2, cp, normC=P.norminf, usedeflation=False, nev=2, callback=lambda st: rows.append(st.z_p))
    assert [k["nev"] for k in seen] == [2, 2] and [k["ampfactor"] for k in seen] == [1.0, 1.0]
    assert len(rows) == len(d.gamma.rows) + sum(len(c.gamma.rows) for c in d.child)
