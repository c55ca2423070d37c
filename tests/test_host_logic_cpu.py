"""CPU tests of the product's HOST logic (bifurcationkit.jl_b200/palc.py, segments.py): the continuation loop is
driven with NumPy vectors and NumPy solvers (duck-typed problem; the oracle is only the checker), and the multi-GPU
row exchange runs on world_size-2 gloo."""
import os
import sys

import numpy as np
import pytest

import __graft_entry__ as g
from oracle import krylov, bls as obls, palc as opalc, problems

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class NumpyProblem:
    """Duck-typed stand-in for BifurcationProblemB200 on host arrays."""

    def __init__(self, F, J, u0, p0, record=None):
        self.F_, self.J_, self.u0, self.p0 = F, J, u0, p0
        self.delta = float(np.sqrt(np.finfo(float).eps))
        self.record = record or (lambda x: float(np.linalg.norm(x)))

    def F(self, x, p, out=None):
        r = self.F_(x, p)
        if out is not None:
            out[...] = r
            return out
        return r

    def J(self, x, p):
        return self.J_(x, p)


class BlsAdapter:
    """product calling convention (dotscale=) -> oracle solver (dotp=)"""

    def __init__(self, inner):
        self.inner = inner

    def __call__(self, J, dR, dzu, dzp, R, n, xiu=1.0, xip=1.0, shift=None, dotscale=1.0):
        N = len(R)
        return self.inner(J, dR, dzu, dzp, R, n, xiu, xip, shift=shift, dotp=lambda a, b: dotscale * float(np.dot(a, b)),
                          apply_xiu=lambda row: row * dotscale)


def _fold_problem():
    F = lambda x, r: r + x - x**3
    J = lambda x, r: np.diag(1 - 3 * x**2)
    return F, J


@pytest.mark.parametrize("tangent", ["secant", "bordered"])
def test_product_host_loop_matches_oracle(tangent):
    """Same branch, row by row, as the oracle on test-cont-non-vector.jl:22-45 (param[end] == -1)."""
    bk = g.load_package()
    P = bk.palc
    F, J = _fold_problem()
    ls = krylov.DefaultLS()
    kw = dict(dsmin=0.001, dsmax=0.07, ds=-0.02, p_max=4.1, p_min=-1.0, max_steps=150)
    orows, _ = opalc.continuation(opalc.Problem(F=F, J=J, u0=np.array([0.8]), p0=1.0, record=lambda x: x[0]),
                                  opalc.PALC(tangent=tangent, bls=obls.MatrixBLS()),
                                  opalc.ContinuationPar(newton_options=opalc.NewtonPar(tol=1e-8, linsolver=ls), **kw))
    rows, st = P.continuation(NumpyProblem(F, J, np.array([0.8]), 1.0, record=lambda x: x[0]),
                              P.PALC(tangent=tangent, bls=BlsAdapter(obls.MatrixBLS())),
                              P.ContinuationPar(newton_options=P.NewtonPar(tol=1e-8, linsolver=ls), **kw))
    assert rows[-1]["param"] == -1.0
    assert len(rows) == len(orows)
    for r, o in zip(rows, orows):
        assert abs(r["param"] - o["param"]) < 1e-12 and abs(r["x"] - o["x"]) < 1e-12 and r["itnewton"] == o["itnewton"]
    assert st.nfail == 0 and st.work_newton == sum(r["itnewton"] for r in rows)


def test_step_size_control_and_rejection():
    bk = g.load_package()
    P = bk.palc
    cp = P.ContinuationPar(dsmin=1e-3, dsmax=0.1, a=0.5, newton_options=P.NewtonPar(max_iterations=10))
    assert np.isclose(P.step_size_control(0.01, True, 2, cp)[0], 0.01 * (1 + 0.5 * 0.8**2))
    assert P.step_size_control(-0.01, False, 10, cp) == (-0.005, False)
    assert P.step_size_control(1e-3, False, 10, cp)[1] is True
    # an initial guess that cannot converge raises like the reference (src/Continuation.jl:375-379)
    F = lambda x, p: np.exp(x) + 0 * p  # no root: Newton walks x <- x - 1 forever
    J = lambda x, p: np.diag(np.exp(x))
    prob = NumpyProblem(F, J, np.array([1.0]), 0.0)
    with pytest.raises(RuntimeError):
        P.continuation(prob, P.PALC(bls=BlsAdapter(obls.MatrixBLS())),
                       P.ContinuationPar(newton_options=P.NewtonPar(tol=1e-10, max_iterations=5, linsolver=krylov.DefaultLS())))


def test_two_point_start_continues_the_same_curve():
    """Segment seeding (SURVEY 8e): a run started from two consecutive scout points traces the same curve."""
    bk = g.load_package()
    P = bk.palc
    n = 31
    beta = 0.01
    F = lambda x, a: problems.chan_F(x, a, beta)
    def Jd(x, a):
        E = np.eye(n)
        return np.column_stack([problems.chan_dF(x, E[:, k], a, beta) for k in range(n)])
    ls = krylov.DefaultLS()
    mk = lambda ms: P.ContinuationPar(dsmin=0.01, dsmax=0.2, ds=0.01, p_max=4.2, p_min=-1.0, max_steps=ms,
                                      newton_options=P.NewtonPar(tol=1e-10, max_iterations=10, linsolver=ls))
    alg = P.PALC(bls=BlsAdapter(obls.MatrixBLS()))
    stride = 6
    grab = bk.segments.SeedGrabber(1, stride, lambda v: v.copy())
    full, _ = P.continuation(NumpyProblem(F, Jd, problems.chan_sol0(n), 3.3), alg, mk(2 * stride))
    P.continuation(NumpyProblem(F, Jd, problems.chan_sol0(n), 3.3), alg, mk(stride + 1), callback=grab)
    u0, p0, u1, p1 = grab.pair()
    assert abs(p0 - full[stride]["param"]) < 1e-14
    resid = []
    seg, _ = P.continuation(NumpyProblem(F, Jd, u0, p0), alg, mk(stride), u1=u1, p1=p1,
                            callback=lambda st: resid.append(np.linalg.norm(F(st.z_u, st.z_p))) or True)
    assert seg[0]["param"] == p0 and len(seg) == stride + 1
    assert max(resid) < 1e-9                              # every segment point solves F(x, alpha) = 0
    fx = np.array([r["x"] for r in full]); fp = np.array([r["param"] for r in full])
    assert np.all(np.diff(fx) > 0) and np.all(np.diff([r["x"] for r in seg]) > 0)   # same direction along the branch
    for r in seg:                                          # and lies on the scout curve ||x||(alpha) (coarse interpolation)
        if fx[0] <= r["x"] <= fx[-1]:
            assert abs(np.interp(r["x"], fx, fp) - r["param"]) < 2e-2


def _chan_window_setup(bk, n=31):
    P = bk.palc
    beta = 0.01
    F = lambda x, a: problems.chan_F(x, a, beta)

    def Jd(x, a):
        E = np.eye(n)
        return np.column_stack([problems.chan_dF(x, E[:, k], a, beta) for k in range(n)])

    ls = krylov.DefaultLS()
    mk = lambda tol, dsmax, ds: P.ContinuationPar(dsmin=0.005, dsmax=dsmax, ds=ds, p_max=4.2, p_min=-1.0, max_steps=400,
                                                  newton_options=P.NewtonPar(tol=tol, max_iterations=10, linsolver=ls))
    alg = P.PALC(bls=BlsAdapter(obls.MatrixBLS()))
    make_prob = lambda u, p: NumpyProblem(F, Jd, u, p)
    return P, F, make_prob, alg, mk


def _window_job(bk, rank, world, s_total=3.0):
    """What one rank of bench.py --gpus N does: replicated cheap scout over the window, partition by predicted cost,
    full-accuracy chunk through the two-point start."""
    P, F, make_prob, alg, mk = _chan_window_setup(bk)
    sc = bk.segments.run_scout(P, make_prob(problems.chan_sol0(31), 3.3), alg, mk(1e-4, 0.15, 0.05), P.norm2, s_total,
                               lambda v: v.copy(), margin=0.3)
    b = bk.segments.partition_by_cost(sc.cost, world)
    rows, st, trk = bk.segments.run_chunk(P, make_prob, alg, mk(1e-10, 0.05, 0.05), P.norm2, sc, b[rank], b[rank + 1], s_total,
                                          rank, rank == len(b) - 2)
    return sc, b, rows, F


def test_window_partition_traces_the_single_gpu_curve():
    """SURVEY 8e parity: the union of the chunks (started from loose scout seeds) lies on the curve the single run
    computes over the same arclength window -- compared by distance to the polyline, not row by row."""
    bk = g.load_package()
    P, F, make_prob, alg, mk = _chan_window_setup(bk)
    s_total = 3.0
    trk = bk.segments.ArcTracker(P.V, alg.theta, 0.0, s_total)
    full, _ = P.continuation(make_prob(problems.chan_sol0(31), 3.3), alg, mk(1e-10, 0.05, 0.05), callback=trk)
    ref = np.array([[r["param"], r["x"]] for r in full])
    assert abs(trk.s - s_total) < 0.06 and len(full) > 40
    # the same run a little further: the chunks measure arclength along their own polylines, so the window's end differs by O(ds)
    longer, _ = P.continuation(make_prob(problems.chan_sol0(31), 3.3), alg, mk(1e-10, 0.05, 0.05),
                               callback=bk.segments.ArcTracker(P.V, alg.theta, 0.0, s_total + 0.4))
    ref_long = np.array([[r["param"], r["x"]] for r in longer])
    for world in (1, 2, 4):
        merged = []
        for rank in range(world):
            sc, b, rows, _ = _window_job(bk, rank, world, s_total)
            assert len(sc.points) < 0.5 * len(full)                      # the scout is much coarser than the run itself
            assert len(rows) >= 1
            merged += [[r["param"], r["x"]] for r in rows]
        merged = np.array(merged)
        assert bk.segments.curve_distance(merged, ref_long) < 2e-3, world  # on the same curve (chords of the polyline: O(ds^2))
        assert bk.segments.curve_distance(ref, merged) < 2e-2, world      # and covering the whole window
        assert abs(len(merged) - len(full)) <= 4 * world                  # about the same number of steps: identical work


def test_partition_by_cost_is_balanced_and_contiguous():
    bk = g.load_package()
    cost = [0.0] + [1.0] * 10 + [5.0] * 10 + [1.0] * 10
    b = bk.segments.partition_by_cost(cost, 4)
    assert b[0] == 0 and b[-1] == 30 and all(x < y for x, y in zip(b[:-1], b[1:]))
    loads = [sum(cost[b[r] + 1: b[r + 1] + 1]) for r in range(4)]
    assert max(loads) <= 1.5 * sum(cost) / 4
    assert bk.segments.partition_by_cost([0.0, 1.0, 1.0], 8) == [0, 1, 2]   # more ranks than intervals


def _gloo_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    import __graft_entry__ as gg
    bk = gg.load_package()
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rows = [dict(param=-0.1 - 0.01 * (rank * 3 + i), x=1.0 + rank + 0.1 * i, itnewton=2, itlinear=40 + i) for i in range(4 - rank)]
    gathered = bk.segments.all_gather_rows(rows, 5, dist, torch, "cpu")
    merged = bk.segments.merge_branch(gathered)
    # the round-2 scheme end to end on 2 processes: replicated scout, cost partition, chunk, all_gather of the rows
    sc, b, wrows, F = _window_job(bk, rank, world)
    wg = bk.segments.all_gather_rows(wrows, 120, dist, torch, "cpu")
    wmerged = bk.segments.merge_chunks(wg)
    q.put((rank, gathered.shape, merged.tolist(), wmerged[:, :2].tolist(), b))
    dist.barrier()
    dist.destroy_process_group()


def test_all_gather_rows_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + (os.getpid() % 2000)
    ps = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = [q.get(timeout=180) for _ in ps]
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    res.sort()
    assert res[0][1] == (2, 5, 4) and res[0][2] == res[1][2]      # every rank assembles the same branch
    assert res[0][3] == res[1][3] and res[0][4] == res[1][4]       # same partition, same merged window on both ranks
    w = np.array(res[0][3])
    assert len(w) > 40 and np.all(np.diff(w[:, 1]) > 0)            # one monotone sweep along the Chan branch, no gap / overlap
    merged = np.array(res[0][2])
    assert merged.shape == (4 + 3 - 1, 4)                           # rank-1 segment starts at rank-0's last point (-0.13): dropped once
    assert np.all(np.diff(merged[:, 0]) < 0)


# ------------------------------------------------------------------------------------------------ Floquet (SURVEY 8f.1)
class NumpyVF:
    """Duck-typed vector-field context (what floquet.py needs of a BK_CGL2D Context) on the NumPy cGL operator."""

    def __init__(self, gl):
        self.gl, self.u = gl, None

    def jacobian(self, u):
        self.u = np.array(u)
        return self

    def jvp(self, v, a0=0.0, a1=1.0):
        return a0 * np.asarray(v) + a1 * self.gl.dF(self.u, np.asarray(v))


def _dense_shifted_solver(gl):
    def ls(J, rhs, a0=0.0, a1=1.0):
        A = a0 * np.eye(gl.N) + a1 * np.column_stack([gl.dF(J.u, e) for e in np.eye(gl.N)])
        return np.linalg.solve(A, rhs), True, 1
    return ls


def test_floquet_host_logic_matches_oracle():
    """FloquetQaDB200 / ArnoldiLMB200 driven with NumPy vectors against oracle.floquet (Floquet.jl:285-316, 59-85)."""
    from oracle import floquet as ofl
    bk = g.load_package()
    nx, ny, M = 6, 5, 9
    gl = problems.GinzburgLandau2D(nx, ny, np.pi, np.pi / 2, r=1.3)
    N = gl.N
    ph = gl.phi11()
    x = np.concatenate([np.concatenate([0.5 * ph * np.cos(2 * np.pi * k / M), 0.5 * ph * np.sin(2 * np.pi * k / M)]) for k in range(M)] + [np.array([6.4])])
    jac = lambda u: np.column_stack([gl.dF(u, e) for e in np.eye(N)])
    mono = ofl.monodromy_dense(jac, x, M, N)
    fl = bk.floquet.FloquetQaDB200(NumpyVF(gl), _dense_shifted_solver(gl), M, eigsolver=bk.floquet.ArnoldiLMB200(krylovdim=40, tol=1e-10))
    v = np.random.default_rng(5).standard_normal(N)
    assert np.allclose(fl.monodromy(x, v), mono @ v, rtol=1e-10, atol=1e-12)
    assert fl.solves == M - 1
    sig, vecs, cv, info = fl(x, 4)
    ref, _ = ofl.floquet_exponents(np.linalg.eigvals(mono))
    ref4 = ref[np.argsort(-np.abs(np.exp(ref)))][:4]      # the 4 multipliers of largest modulus ...
    ref4 = ref4[np.argsort(-ref4.real, kind="stable")]      # ... as exponents by decreasing real part
    assert cv and np.allclose(np.sort(sig.real)[::-1], np.sort(ref4.real)[::-1], rtol=1e-7, atol=1e-9)
    assert np.all(np.diff(sig.real) <= 1e-12)
    mu = info["multipliers"]
    for k in range(4):                                       # Ritz pairs really are eigenpairs of the monodromy
        z = vecs[k][0] + 1j * vecs[k][1]
        assert np.linalg.norm(mono @ z - mu[k] * z) < 1e-7 * abs(mu[k]) * np.linalg.norm(z)
    sl = fl.extract_eigenvector(x, vecs[0][0])
    assert len(sl) == M and np.allclose(sl[M - 2], mono @ vecs[0][0], rtol=1e-9, atol=1e-12)


# ------------------------------------------------------------------------------------------------ events (SURVEY 8f.2)
def _default_eig(J, nev):
    """DefaultEig (src/EigSolver.jl:31-50): dense spectrum, decreasing real part, first nev."""
    vals = np.linalg.eigvals(np.asarray(J))
    vals = vals[np.argsort(-vals.real, kind="stable")]
    return vals[:nev], None, True, 1


def _check_branch(br, cp, E):
    """`testBranch` of test/continuation/test_bif_detection.jl:19-55 (the parts that do not need br.sol)."""
    for i, row in enumerate(br.rows):
        assert row["step"] == i == br.eig[i]["step"]
        stable, nu, ni = E.is_stable(cp, br.eig[i]["eigenvals"])
        assert row["n_unstable"] == nu and row["stable"] == stable
    for bp in br.specialpoint:
        if bp.type == "endpoint":
            continue
        i = bp.idx
        nb = [br.rows[k]["n_unstable"] for k in (i - 1, i, i + 1) if 0 <= k < len(br.rows)]
        assert len(set(nb)) > 1                      # states marked as bifurcation points sit next to a change of n_unstable
        assert bp.interval[0] <= bp.param <= bp.interval[1]
        assert bp.param == br.rows[i]["param"]


def test_bifurcation_detection_and_bisection_known_answers():
    """test/continuation/test_bif_detection.jl:57-100: F = -x + lambda L x - x^3 on the trivial branch; bifurcation points at
    lambda = 1 / L_ii = 1,2,3,4,5 (multiplicity 1..5), 6, 6.5, 6.75, 6.875; located by bisection to 3e-3, from above."""
    bk = g.load_package()
    P, E = bk.palc, bk.events
    Ld = np.array([1.0 / ii for ii in range(1, 6) for _ in range(ii)] + [1 / 6.0, 1 / 6.5, 1 / 6.75, 1 / 6.875])
    F = lambda x, lam: -x + lam * Ld * x - x**3
    J = lambda x, lam: np.diag(lam * Ld - 3 * x**2 - 1.0)
    true_pts = np.array([1, 2, 3, 4, 5, 6, 6.5, 6.75, 6.875])
    dims = [1, 2, 3, 4, 5, 1, 1, 1, 1]
    nopts = P.NewtonPar(linsolver=krylov.DefaultLS(), eigsolver=_default_eig)
    mk = lambda **kw: P.ContinuationPar(**{**dict(p_min=-1.0, p_max=10.0, ds=0.1, max_steps=150, detect_bifurcation=3, newton_options=nopts), **kw})
    prob = lambda p0=0.0: NumpyProblem(F, J, np.zeros(len(Ld)), p0)
    alg = P.PALC(bls=BlsAdapter(obls.MatrixBLS()))
    # br1: default n_inversion = 2
    cp1 = mk()
    br1 = E.continuation(prob(), alg, cp1)
    _check_branch(br1, cp1, E)
    assert [abs(bp.delta[0]) for bp in br1.specialpoint if bp.type != "endpoint"] == dims
    assert br1.specialpoint[-1].type == "endpoint"
    # br2: n_inversion = 4, tol_bisection_eigenvalue = 1e-7 (:77-87)
    cp2 = mk(p_max=10.3, n_inversion=4, tol_bisection_eigenvalue=1e-7)
    br2 = E.continuation(prob(), alg, cp2)
    _check_branch(br2, cp2, E)
    pts = np.array([bp.param for bp in br2.specialpoint if bp.type != "endpoint"])
    assert len(pts) == len(true_pts)
    assert list(pts) > list(true_pts)                 # the reference's `specialpoint2 > specialpoints`
    assert np.max(np.abs(pts - true_pts)) < 3e-3
    assert [abs(bp.delta[0]) for bp in br2.specialpoint if bp.type != "endpoint"] == dims
    assert all(bp.type == ("bp" if d == 1 else "nd") for bp, d in zip(br2.specialpoint, dims))
    # br3: bisection "fails" (n_inversion = 8 cannot be reached within max_bisection_steps): intervals still valid (:90-92)
    cp3 = mk(p_max=10.3, n_inversion=8, tol_bisection_eigenvalue=1e-7)
    _check_branch(E.continuation(prob(), alg, cp3), cp3, E)
    # br4: coming from above with a huge step and a single bisection step (:94-97)
    cp4 = mk(p_max=1.95, n_inversion=8, ds=0.7, dsmax=1.5, max_bisection_steps=1)
    _check_branch(E.continuation(prob(0.95), alg, cp4), cp4, E)


def test_eigen_request_follows_the_reference_from_the_first_step():
    """compute_eigenvalues (src/Utils.jl:78-79) asks for max(n_unstable + 5, nev) eigenvalues, also while n_unstable is still
    -1: with nev = 1, palc.continuation asks for 4 at the start, as events.continuation does, and fills n_imag alike."""
    bk = g.load_package()
    P, E = bk.palc, bk.events
    F, J = _fold_problem()
    asked = {"palc": [], "events": []}

    def mk(who):
        eig = lambda Jm, nev: asked[who].append(nev) or _default_eig(Jm, nev)
        return P.ContinuationPar(dsmin=0.001, dsmax=0.07, ds=-0.02, p_max=4.1, p_min=-1.0, max_steps=30, nev=1, detect_bifurcation=1,
                                 newton_options=P.NewtonPar(tol=1e-8, linsolver=krylov.DefaultLS(), eigsolver=eig))

    alg = P.PALC(bls=BlsAdapter(obls.MatrixBLS()))
    rows, st = P.continuation(NumpyProblem(F, J, np.array([0.8]), 1.0), alg, mk("palc"))
    br = E.continuation(NumpyProblem(F, J, np.array([0.8]), 1.0), alg, mk("events"))
    assert asked["palc"][:2] == [4, 4] and asked["palc"] == asked["events"]
    assert [r["n_unstable"] for r in rows] == [r["n_unstable"] for r in br.rows]
    assert st.n_imag == br.state.n_imag == (0, 0)


def test_fold_and_hopf_detection_two_dimensional_field():
    """test/continuation/test_bif_detection.jl:113-143: 2-d field with folds and Hopf points; detect_bifurcation = 3,
    n_inversion = 6.  The branch invariants of `testBranch` hold and a Hopf point is found with a complex pair crossing."""
    bk = g.load_package()
    P, E = bk.palc, bk.events
    k = 3

    def F(X, p1):
        x, y = X
        return np.array([p1 + x - y - x**k / k, p1 + y + x - 2 * y**k / k])

    def J(X, p1):
        x, y = X
        return np.array([[1 - x ** (k - 1), -1.0], [1.0, 1 - 2 * y ** (k - 1)]])

    nopts = P.NewtonPar(max_iterations=5, linsolver=krylov.DefaultLS(), eigsolver=_default_eig)
    cp = P.ContinuationPar(dsmax=0.1, ds=0.001, max_steps=135, p_min=-3.0, p_max=4.0, newton_options=nopts, detect_bifurcation=3,
                           n_inversion=6, dsmin_bisection=1e-9, max_bisection_steps=15, nev=2)
    br = E.continuation(NumpyProblem(F, J, -2 * np.ones(2), -3.0, record=lambda x: x[0]), P.PALC(bls=BlsAdapter(obls.MatrixBLS())), cp)
    _check_branch(br, cp, E)
    types = [bp.type for bp in br.specialpoint]
    assert types[-1] == "endpoint" and "hopf" in types
    hopf = [bp for bp in br.specialpoint if bp.type == "hopf"]
    assert len(hopf) == 2 and abs(hopf[0].param + hopf[1].param) < 1e-4 and abs(abs(hopf[0].param) - 0.95385) < 1e-4
    for bp in hopf:
        assert abs(bp.delta[0]) == 2 and abs(bp.delta[1]) == 2 and bp.status == "converged"
        assert bp.interval[1] - bp.interval[0] < 1e-4
    # the field is odd-symmetric: the real eigenvalue crossings (folds of this branch) come in +- pairs
    bps = sorted(bp.param for bp in br.specialpoint if bp.type == "bp")
    assert len(bps) == 4 and abs(bps[0] + bps[3]) < 1e-5 and abs(bps[1] + bps[2]) < 2e-3
    # without eigenvalues, folds are found from the parameter's monotony (detect_bifurcation < 2)
    cp0 = P.ContinuationPar(dsmax=0.1, ds=0.001, max_steps=135, p_min=-3.0, p_max=4.0, newton_options=nopts, detect_bifurcation=0)
    br0 = E.continuation(NumpyProblem(F, J, -2 * np.ones(2), -3.0, record=lambda x: x[0]), P.PALC(bls=BlsAdapter(obls.MatrixBLS())), cp0)
    folds = [bp for bp in br0.specialpoint if bp.type == "fold"]
    assert len(folds) == 4
    for bp in folds:
        i = bp.idx
        assert (br0.rows[i + 1]["param"] - br0.rows[i]["param"]) * (br0.rows[i]["param"] - br0.rows[i - 1]["param"]) < 0


# ------------------------------------------------------------------------------------------------ deflation (SURVEY 8f.4)
def test_deflation_operator_problem_and_custom_linear_solver():
    """test/newton/test_newton.jl:54-168: value of the deflation factor, Jacobian of M(u) F(u) against finite differences,
    the Sherman-Morrison custom solver against a dense solve, deflated Newton finds the other root, two-guess Newton."""
    bk = g.load_package()
    P, D = bk.palc, bk.deflation
    rng = np.random.default_rng(7)
    # value of the factor (:70-87)
    for acc in ("prod", "mean"):
        op = D.DeflationOperator(2, 1.0, [rng.random(2) for _ in range(3)], accumulator=acc)
        x0 = rng.random(2)
        vals = [op.alpha + np.linalg.norm(x0 - r) ** (-2 * op.power) for r in op.roots]
        ref = np.prod(vals) if acc == "prod" else np.mean(vals)
        assert np.isclose(op(x0), ref, rtol=1e-8)
    # Jacobian-vector product and custom linear solver (:125-143), F4def = (x - 1)(x - 2)
    F = lambda x, p: (x - 1.0) * (x - 2.0)
    J = lambda x, p: np.diag(2 * x - 3.0)
    n = 3
    op = D.DeflationOperator(2, 1.0, [1 + 0.01 * rng.random(n) for _ in range(3)])
    prob = NumpyProblem(F, J, np.array([0.1] * n), None)
    jprob = NumpyProblem(F, lambda x, p: (lambda dx, A=J(x, p): A @ dx), np.array([0.1] * n), None)  # J as an operator
    dp, dpj = D.DeflatedProblem(prob, op), D.DeflatedProblem(jprob, op)
    sol, rhs = rng.random(n), rng.random(n)
    fd = lambda f, x: np.column_stack([(f(x + 1e-6 * e) - f(x - 1e-6 * e)) / 2e-6 for e in np.eye(len(x))])
    Jfd = fd(lambda z: dp.F(z, None), sol)
    assert np.allclose(dpj.jvp(sol, None, rhs), Jfd @ rhs, rtol=1e-5)
    h, ok, its = D.DeflatedProblemCustomLS(krylov.DefaultLS())(dp.J(sol, None), rhs)
    assert ok and np.allclose(h, np.linalg.solve(Jfd, rhs), rtol=1e-5)
    # deflated Newton avoids the known root (:146-149)
    for acc in ("prod", "mean"):
        op1 = D.DeflationOperator(2, 1.0, [np.array([1.0])], accumulator=acc)
        p1 = NumpyProblem(F, J, np.array([0.1]), None)
        s = D.newton_deflated(p1, p1.u0, None, op1, P.NewtonPar(linsolver=krylov.DefaultLS()))
        assert s.converged and np.isclose(s.u[0], 2.0, atol=1e-8)
    # newton(prob, x0, x1, ...) (:160-168)
    s1, s0, flag = D.newton_two_guesses(NumpyProblem(F, J, np.array([0.1]), None), np.array([1.2]), np.array([2.1]), None,
                                        P.NewtonPar(linsolver=krylov.DefaultLS()))
    assert flag and np.isclose(s0.u[0], 1.0) and np.isclose(s1.u[0], 2.0)


def test_deflated_newton_finds_the_three_chan_solutions():
    """The Chan/Bratu problem of examples/chan.jl at alpha = 3.3 sits on the S-shaped part of its branch: three solutions.
    Plain Newton from sol0 finds the lower one; deflating it (and then the next) gives the other two."""
    bk = g.load_package()
    P, D = bk.palc, bk.deflation
    n = 101
    F = lambda x, a: problems.chan_F(x, a, 0.01)
    J = lambda x, a: np.column_stack([problems.chan_dF(x, e, a, 0.01) for e in np.eye(n)])
    prob = NumpyProblem(F, J, problems.chan_sol0(n), 3.3)
    opts = P.NewtonPar(tol=1e-9, max_iterations=100, linsolver=krylov.DefaultLS())
    s0 = P.newton(prob, prob.u0, 3.3, opts, P.norminf)
    op = D.DeflationOperator(2, 1.0, [s0.u])
    s1 = D.newton_deflated(prob, 4.0 * s0.u, 3.3, op, opts, P.norminf)
    op.push(s1.u)
    s2 = D.newton_deflated(prob, 8.0 * s0.u, 3.3, op, opts, P.norminf)
    assert s0.converged and s1.converged and s2.converged
    tops = sorted(float(np.max(s.u)) for s in (s0, s1, s2))
    assert np.allclose(tops, [0.77197, 5.97988, 12.85103], atol=1e-4)
    for s in (s0, s1, s2):
        assert P.norminf(F(s.u, 3.3)) < 1e-8                  # roots of F itself, not only of M F


# ------------------------------------------------------------------------------------------------ Fold minimally augmented (SURVEY 8f.3)
def test_newton_fold_known_answers():
    """newton_fold (src/codim2/MinAugFold.jl:15-146,201-222) on host arrays with the oracle's bordered solver:
    (i) F = r + x - x^3 (test/continuation/test-cont-non-vector.jl:22-45): folds at x = +-1/sqrt(3), r = -+2/(3 sqrt 3);
    (ii) a 2-D self-adjoint system with an analytic fold; (iii) the Chan problem (examples/chan.jl): the located point has a
    singular Jacobian and sits at the turning point of the continuation branch."""
    bk = g.load_package()
    P = bk.palc
    bls = BlsAdapter(obls.MatrixBLS())
    opts = P.NewtonPar(tol=1e-10, max_iterations=12, linsolver=krylov.DefaultLS())
    # (i)
    F = lambda x, r: r + x - x**3
    J = lambda x, r: np.diag(1 - 3 * x**2)
    sol = bk.codim2.newton_fold(NumpyProblem(F, J, np.array([0.5]), -0.3), np.array([0.5]), -0.3, np.array([1.0]), np.array([1.0]), opts, bls)
    assert sol.converged, sol.residuals
    assert abs(sol.u[0] - 1 / np.sqrt(3)) < 1e-7 and abs(sol.p + 2 / (3 * np.sqrt(3))) < 1e-7 and abs(sol.sigma) < 1e-9
    # (ii) x1: fold of p + x1 - x1^3 coupled symmetrically to a damped x2
    F2 = lambda x, p: np.array([p + x[0] - x[0]**3 + 0.1 * x[1], 0.1 * x[0] - 2.0 * x[1]])
    J2 = lambda x, p: np.array([[1 - 3 * x[0]**2, 0.1], [0.1, -2.0]])
    s2 = bk.codim2.newton_fold(NumpyProblem(F2, J2, np.array([0.55, 0.03]), -0.35), np.array([0.55, 0.03]), -0.35, np.array([1.0, 0.0]),
                               np.array([1.0, 0.0]), opts, bls)
    assert s2.converged, s2.residuals
    assert abs(np.linalg.det(J2(s2.u, s2.p))) < 1e-8 and np.linalg.norm(F2(s2.u, s2.p)) < 1e-9
    # (iii) Chan: continuation through the fold, then refine the turning point
    n, beta = 31, 0.01
    Fc = lambda x, a: problems.chan_F(x, a, beta)
    Jc = lambda x, a: np.column_stack([problems.chan_dF(x, np.eye(n)[:, k], a, beta) for k in range(n)])
    pts = []
    cp = P.ContinuationPar(dsmin=0.005, dsmax=0.1, ds=0.05, p_max=4.3, p_min=-1.0, max_steps=120,
                           newton_options=P.NewtonPar(tol=1e-10, max_iterations=10, linsolver=krylov.DefaultLS()))
    rows, _ = P.continuation(NumpyProblem(Fc, Jc, problems.chan_sol0(n), 3.3), P.PALC(bls=bls), cp,
                             callback=lambda st: pts.append((st.z_u.copy(), st.z_p, st.tau_u.copy())) or True)
    ps = [p for _, p, _ in pts]
    k = next(i for i in range(1, len(ps) - 1) if ps[i] > ps[i + 1])  # first turning point of the S-shaped branch
    assert 0 < k < len(pts) - 1
    x0, p0, tau = pts[k]
    s3 = bk.codim2.newton_fold(NumpyProblem(Fc, Jc, x0, p0), x0, p0, tau / np.linalg.norm(tau), tau / np.linalg.norm(tau), opts, bls)
    assert s3.converged, s3.residuals
    sv = np.linalg.svd(Jc(s3.u, s3.p), compute_uv=False)
    assert sv[-1] < 1e-6 * sv[0] and np.linalg.norm(Fc(s3.u, s3.p)) < 1e-8
    assert p0 - 1e-9 <= s3.p < p0 + 0.02                          # the true fold lies at or just beyond the largest computed parameter


# ------------------------------------------------------------------------------------------------ Hopf minimally augmented (SURVEY 8f.3)
class DenseComplexProblem:
    """cprob of codim2.HopfMinAug on dense matrices: J(x, p, transpose) -> callable on complex vectors"""

    class Jc:
        def __init__(self, M):
            self.M = M

        def __call__(self, z):
            return self.M @ z

    def __init__(self, Jfun):
        self.Jfun = Jfun

    def J(self, x, p, transpose=False):
        M = np.asarray(self.Jfun(x, p), dtype=float)
        return self.Jc(M.T.copy() if transpose else M)


def _dense_cls(Jc, rhs, a0=0.0, a1=1.0):
    n = Jc.M.shape[0]
    return np.linalg.solve(a0 * np.eye(n) + a1 * Jc.M, rhs), True, 1


def _dense_ls2(J, r1, r2):
    return np.linalg.solve(J, r1), np.linalg.solve(J, r2), True, (1, 1)


def test_hopf_border_known_answer_complex():
    """The complex bordered system of the Hopf MA functional, test/linear_solvers/test_linear.jl:324-351:
    J = [0 1 0; -1 0 0; 0 0 1], lambda = 1.01 x (its eigenvalue i), borders w (null vector of J' - conj(lambda)) and v:
    the bordering elimination of codim2.HopfMinAug._border equals the explicit solve of [J - lambda I, w; v^H, 0] [x; s] = [0; 1]."""
    bk = g.load_package()
    J = np.array([[0.0, 1.0, 0.0], [-1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    vals, vecs = np.linalg.eig(J)
    k = int(np.argmin(abs(vals - 1j)))
    lam, v = vals[k], vecs[:, k]
    valt, vect = np.linalg.eig(J.T)
    w = vect[:, int(np.argmin(abs(valt + 1j)))]
    assert abs(np.linalg.det(J - lam * np.eye(3))) < 1e-12
    lam = 1.01 * lam
    J0 = np.block([[J - lam * np.eye(3), w[:, None]], [np.conj(v)[None, :], np.zeros((1, 1))]])
    rhs = np.zeros(4, dtype=complex)
    rhs[-1] = 1
    explicit = np.linalg.solve(J0, rhs)
    ma = bk.codim2.HopfMinAug(None, None, w, v, None, _dense_cls)
    x, s = ma._border(DenseComplexProblem.Jc(J), -lam, w, v)
    assert np.allclose(x, explicit[:-1], rtol=1e-10, atol=1e-12) and abs(s - explicit[-1]) < 1e-10 * abs(s)


def test_newton_hopf_known_answers():
    """newton_hopf (src/codim2/MinAugHopf.jl:19-188,258-283) on host arrays with dense solvers:
    (i) Brusselator x' = a - (b+1) x + x^2 y, y' = b x - x^2 y: Hopf at b = 1 + a^2 with omega = a, equilibrium (a, b/a) moving
    with the parameter (non-zero d_pF, sigma_x); (ii) cGL 2-D on 9 x 7 (examples/cGL2d.jl): trivial state, r = -lambda_1(Delta),
    omega = nu, null vectors phi_11 x (1, -i)."""
    bk = g.load_package()
    P = bk.palc
    opts = P.NewtonPar(tol=1e-9, max_iterations=15, linsolver=krylov.DefaultLS())
    a = 1.3
    F = lambda x, b: np.array([a - (b + 1) * x[0] + x[0] ** 2 * x[1], b * x[0] - x[0] ** 2 * x[1]])
    J = lambda x, b: np.array([[-(b + 1) + 2 * x[0] * x[1], x[0] ** 2], [b - 2 * x[0] * x[1], -x[0] ** 2]])
    bH = 1 + a * a
    x0 = np.array([a, (bH + 0.2) / a]) + 0.01
    vals, vecs = np.linalg.eig(J(x0, bH + 0.2))
    k = int(np.argmax(vals.imag))
    valt, vect = np.linalg.eig(J(x0, bH + 0.2).T)
    kt = int(np.argmin(valt.imag))
    sol = bk.codim2.newton_hopf(NumpyProblem(F, J, x0, bH + 0.2), DenseComplexProblem(J), x0, bH + 0.2, vals[k].imag,
                                vecs[:, k], vect[:, kt], opts, _dense_ls2, _dense_cls)
    assert sol.converged, sol.residuals
    assert abs(sol.p - bH) < 1e-7 and abs(sol.omega - a) < 1e-7 and np.allclose(sol.u, [a, bH / a], atol=1e-7)
    ev = np.linalg.eigvals(J(sol.u, sol.p))
    assert np.max(abs(ev.real)) < 1e-6
    # (ii)
    gl = problems.GinzburgLandau2D(9, 7, 1.0, 0.8)
    n = gl.N
    Fg = lambda u, r: gl.F(u, r)
    Jg = lambda u, r: np.column_stack([gl.dF(u, np.eye(n)[:, j], r) for j in range(n)])
    rng = np.random.default_rng(3)
    phi = gl.phi11()
    zeta = np.concatenate([phi, -1j * phi]) + 0.05 * (rng.standard_normal(n) + 1j * rng.standard_normal(n))
    u0 = 1e-3 * rng.standard_normal(n)
    s2 = bk.codim2.newton_hopf(NumpyProblem(Fg, Jg, u0, gl.r_hopf() + 0.3), DenseComplexProblem(Jg), u0, gl.r_hopf() + 0.3, gl.nu + 0.2,
                               zeta, zeta.copy(), opts, _dense_ls2, _dense_cls)
    assert s2.converged, s2.residuals
    assert abs(s2.p - gl.r_hopf()) < 1e-7 and abs(s2.omega - gl.nu) < 1e-7 and np.linalg.norm(s2.u) < 1e-8


# ------------------------------------------------------------------------------------------------ bothside (SURVEY 8e: the reference's own split)
def _bothside_setup(bk):
    P = bk.palc
    F = lambda x, r: r + x - x**3
    J = lambda x, r: np.diag(1 - 3 * x**2)
    ls = krylov.DefaultLS()
    cp = P.ContinuationPar(dsmin=0.001, dsmax=0.07, ds=0.02, p_max=1.5, p_min=-1.0, max_steps=150,
                           newton_options=P.NewtonPar(tol=1e-10, linsolver=ls))
    mk = lambda: NumpyProblem(F, J, np.array([0.8]), 0.2, record=lambda x: x[0])
    return P, mk, P.PALC(bls=BlsAdapter(obls.MatrixBLS())), cp


def test_bothside_merge_single_process():
    """continuation(...; bothside = true) (src/Continuation.jl:687-700) + _merge (src/Results.jl:464-489) on r + x - x^3 started
    in the middle of the branch: one monotone sweep of x from the p_min end to the p_max end, start point listed twice"""
    bk = g.load_package()
    P, mk, alg, cp = _bothside_setup(bk)
    merged, _ = bk.segments.continuation_bothside(P, mk, alg, cp, P.norm2)
    fwd, _ = P.continuation(mk(), alg, cp)
    cpb = P.ContinuationPar(**{**cp.__dict__, "ds": -cp.ds})
    bwd, _ = P.continuation(mk(), alg, cpb)
    assert len(merged) == len(fwd) + len(bwd)
    assert {merged[0, 0], merged[-1, 0]} == {-1.0, 1.5}                 # both parameter bounds are reached, one per direction
    k = len(bwd)
    assert merged[k - 1, 0] == merged[k, 0] == 0.2 and merged[k - 1, 1] == merged[k, 1]   # the common start point, twice
    x = np.delete(merged[:, 1], k)
    assert np.all(np.diff(x) > 0) or np.all(np.diff(x) < 0)             # one sweep along the curve, no gap and no overlap
    assert np.max(np.abs(merged[:, 0] + merged[:, 1] - merged[:, 1] ** 3)) < 1e-9
    # merge_bothside orders whatever ends coincide (src/Results.jl:470-487)
    a = np.array([[0.0, 0.0, 0, 0], [1.0, 1.0, 0, 0]])
    b = np.array([[0.0, 0.0, 0, 0], [-1.0, -1.0, 0, 0]])
    M = bk.segments.merge_bothside
    assert M(a, b)[:, 0].tolist() == [-1.0, 0.0, 0.0, 1.0] and M(a, b[::-1])[:, 0].tolist() == [-1.0, 0.0, 0.0, 1.0]
    assert M(a[::-1], b)[:, 0].tolist() == [1.0, 0.0, 0.0, -1.0] and M(a, np.zeros((0, 4))).tolist() == a.tolist()


def _bothside_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    import __graft_entry__ as gg
    bk = gg.load_package()
    dist.init_process_group("gloo", rank=rank, world_size=world)
    P, mk, alg, cp = _bothside_setup(bk)
    merged, mine = bk.segments.continuation_bothside(P, mk, alg, cp, P.norm2, dist=dist, torch=torch, device="cpu")
    q.put((rank, merged.tolist(), len(mine), mine[1]["param"] if len(mine) > 1 else None))
    dist.barrier()
    dist.destroy_process_group()


def test_bothside_two_ranks_gloo():
    """one direction per rank, all_gather of the rows, the same merged branch on both ranks and the same as one process computes"""
    import torch.multiprocessing as mp
    bk = g.load_package()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + (os.getpid() % 2000)
    ps = [ctx.Process(target=_bothside_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=180) for _ in ps)
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    P, mk, alg, cp = _bothside_setup(bk)
    single, _ = bk.segments.continuation_bothside(P, mk, alg, cp, P.norm2)
    assert res[0][1] == res[1][1] and np.array_equal(np.array(res[0][1]), single)
    assert res[0][3] > 0.2 and res[1][3] < 0.2 and res[0][2] + res[1][2] == len(single)   # rank 0 went up, rank 1 down


# ------------------------------------------------------------------------------------------------ speculative step sizes (a multi-rank run of ONE branch)
def _spec_setup(bk):
    """r + x - x^3 from the upper branch with a corrector that often fails (3 Newton iterations, large steps): many rejected steps"""
    P = bk.palc
    F = lambda x, r: r + x - x**3
    J = lambda x, r: np.diag(1 - 3 * x**2)
    ls = krylov.DefaultLS()
    cp = P.ContinuationPar(dsmin=0.002, dsmax=0.6, ds=-0.4, p_max=4.1, p_min=-1.0, max_steps=40, a=1.0,
                           newton_options=P.NewtonPar(tol=1e-10, max_iterations=3, linsolver=ls))
    mk = lambda: NumpyProblem(F, J, np.array([1.3247179572447460]), 1.0, record=lambda x: x[0])
    return P, mk, P.PALC(bls=BlsAdapter(obls.MatrixBLS())), cp


def _spec_worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    sys.path.insert(0, ROOT)
    import torch
    import torch.distributed as dist
    import __graft_entry__ as gg
    bk = gg.load_package()
    dist.init_process_group("gloo", rank=rank, world_size=world)
    P, mk, alg, cp = _spec_setup(bk)
    rows, st, info = bk.segments.continuation_speculative(P, mk(), alg, cp, P.norm2, dist, torch, "cpu")
    q.put((rank, [[r[k] for k in ("param", "x", "itnewton", "itlinear", "ds", "step")] for r in rows], st.nfail, st.work_newton, st.stop, info))
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("world", [2, 3])
def test_speculative_step_sizes_reproduce_the_sequential_branch(world):
    """segments.continuation_speculative on `world` gloo ranks: rows, rejected-step count, corrector work and the stop flag equal the
    single-process palc.continuation exactly; the rejected attempts no longer cost rounds."""
    import torch.multiprocessing as mp
    bk = g.load_package()
    P, mk, alg, cp = _spec_setup(bk)
    ref, st = P.continuation(mk(), alg, cp)
    assert st.nfail >= 2                                              # the setup does reject steps
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 33500 + (os.getpid() % 2000) + world
    ps = [ctx.Process(target=_spec_worker, args=(r, world, port, q)) for r in range(world)]
    for p in ps:
        p.start()
    res = sorted(q.get(timeout=240) for _ in ps)
    for p in ps:
        p.join(timeout=60)
        assert p.exitcode == 0
    want = [[r[k] for k in ("param", "x", "itnewton", "itlinear", "ds", "step")] for r in ref]
    for rank, rows, nfail, wn, stop, info in res:
        assert rows == want, (rank, len(rows), len(want))               # bit for bit
        assert nfail == st.nfail and wn == st.work_newton and stop == st.stop
        assert info["attempts"] == st.nfail + st.step                   # every attempt of the sequential loop, rejected or accepted
        assert info["rounds"] < info["attempts"]                        # at least one rejection was absorbed by a speculative rank
    assert res[0][5] == res[-1][5]
