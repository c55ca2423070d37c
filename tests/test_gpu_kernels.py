"""GPU parity tests proper: CUDA path (through the C ABI) vs the NumPy oracle on the same seeded inputs.
Tolerances: stencil kernels 1e-12 relative (fp64, different summation order only); solves 1e-8 relative
(the class the reference's own tests use, test/linear_solvers/test_linear.jl:120-122)."""
import numpy as np
import pytest

import __graft_entry__ as g
from oracle import problems, krylov, bls as obls, potrap as opotrap

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def bk():
    return g.load_package()


def _rel(a, b):
    return np.linalg.norm(np.asarray(a) - np.asarray(b)) / max(np.linalg.norm(b), 1e-300)


LX, LY = 8 * np.pi, 4 * np.pi / np.sqrt(3)


@pytest.mark.parametrize("dims", [(64, 32), (151, 100), (7, 5), (130, 67), (256, 256)])
def test_sh2d_residual_jvp(bk, dims):
    Nx, Ny = dims
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    rng = np.random.default_rng(1)
    u = problems.sh2d_sol0(Nx, Ny, LX, LY) + 0.1 * rng.standard_normal(sh.N)
    v = rng.standard_normal(sh.N)
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=8, params=(-0.1, 1.3))
    assert _rel(ctx.residual(u), sh.F(u)) < 1e-12
    J = ctx.jacobian(u)
    assert _rel(J(v), sh.dF(u, v)) < 1e-12
    assert _rel(ctx.jvp(v, a0=0.1, a1=0.9), 0.1 * v + 0.9 * sh.dF(u, v)) < 1e-12
    # device-resident path gives the same bits as the host-pointer path
    ud, vd = ctx.to_device(u), ctx.to_device(v)
    assert np.array_equal(ctx.residual(ud).numpy(), ctx.residual(u))
    assert np.array_equal(ctx.jvp(vd).numpy(), ctx.jvp(v))
    # parameter change is seen by the residual but J keeps its snapshot
    ctx.set_params((-0.3, 1.1))
    assert _rel(ctx.residual(u), sh.F(u, l=-0.3) + (1.1 - 1.3) * u**2) < 1e-12
    assert _rel(J(v), sh.dF(u, v)) < 1e-12


@pytest.mark.parametrize("dims", [(22, 22, 22), (33, 9, 17), (64, 32, 16)])
def test_sh3d_residual_jvp(bk, dims):
    L = (np.pi, np.pi, np.pi)
    sh = problems.SwiftHohenberg(dims, L, l=0.1, nu=1.2)
    rng = np.random.default_rng(2)
    u = problems.sh3d_sol0(*dims, *L) + 0.05 * rng.standard_normal(sh.N)
    v = rng.standard_normal(sh.N)
    ctx = bk.Context(bk.BK_SH3D, dims, L, krylov_m=8, params=(0.1, 1.2))
    assert _rel(ctx.residual(u), sh.F(u)) < 1e-12
    assert _rel(ctx.jacobian(u)(v), sh.dF(u, v)) < 1e-12


def test_chan_residual_jvp(bk):
    for n in (101, 1000):
        rng = np.random.default_rng(3)
        x = problems.chan_sol0(n) + 0.01 * rng.standard_normal(n)
        dx = rng.standard_normal(n)
        ctx = bk.Context(bk.BK_CHAN, (n,), (1.0,), krylov_m=8, params=(3.3, 0.01))
        assert _rel(ctx.residual(x), problems.chan_F(x, 3.3, 0.01)) < 1e-13
        assert _rel(ctx.jacobian(x)(dx), problems.chan_dF(x, dx, 3.3, 0.01)) < 1e-13


def test_cgl_residual_jvp(bk):
    for dims in ((41, 21), (64, 48)):
        gl = problems.GinzburgLandau2D(dims[0], dims[1], np.pi, np.pi / 2, r=1.2)
        rng = np.random.default_rng(4)
        u, du = 0.3 * rng.standard_normal(gl.N), rng.standard_normal(gl.N)
        ctx = bk.Context(bk.BK_CGL2D, dims, (np.pi, np.pi / 2), krylov_m=8, params=(1.2, 0.1, 1.0, -1.0, 1.0))
        assert _rel(ctx.residual(u), gl.F(u)) < 1e-12
        assert _rel(ctx.jacobian(u)(du), gl.dF(u, du)) < 1e-12


def test_potrap_residual_jvp(bk):
    Nx, Ny, M = 24, 12, 7
    gl = problems.GinzburgLandau2D(Nx, Ny, np.pi, np.pi / 2, r=1.3)
    rng = np.random.default_rng(5)
    NM = gl.N * M
    x = np.concatenate([0.3 * rng.standard_normal(NM), [6.1]])
    dx = np.concatenate([rng.standard_normal(NM), [0.7]])
    phi, xpi = rng.standard_normal(NM), rng.standard_normal(NM)
    tr = opotrap.Trapeze(gl.F, gl.dF, phi, xpi, M, gl.N)
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (Nx, Ny, M), (np.pi, np.pi / 2), krylov_m=8, params=(1.3, 0.1, 1.0, -1.0, 1.0))
    assert ctx.N == NM + 1
    ctx.potrap_set_section(phi, xpi)
    assert _rel(ctx.residual(x), tr.residual(x)) < 1e-12
    assert _rel(ctx.jacobian(x)(dx), tr.jvp(x, dx)) < 1e-12


def test_vector_algebra(bk):
    ctx = bk.Context(bk.BK_CHAN, (100003,), (1.0,), krylov_m=4, params=(3.3, 0.01))
    rng = np.random.default_rng(6)
    a, b, c = (rng.standard_normal(ctx.N) for _ in range(3))
    A, B, Cv = ctx.to_device(a), ctx.to_device(b), ctx.to_device(c)
    assert abs(A.dot(B) - a @ b) < 1e-9 * np.linalg.norm(a) * np.linalg.norm(b)
    assert abs(A.norm() - np.linalg.norm(a)) < 1e-12 * np.linalg.norm(a)
    assert A.norminf() == np.max(np.abs(a))
    assert abs(A.diffdot(B, Cv) - (a - b) @ c) < 1e-9 * np.linalg.norm(a - b) * np.linalg.norm(c)
    Y = B.copy().axpby_(0.3, A, -1.7)
    assert np.allclose(Y.numpy(), 0.3 * a - 1.7 * b, rtol=1e-15, atol=1e-15)
    assert np.allclose(A.copy().scale_(2.5).numpy(), 2.5 * a)
    assert np.all(A.copy().zero_().numpy() == 0)
    # reductions are deterministic (last-block scheme, no atomics on data)
    assert A.dot(B) == A.dot(B)


def _gmres_sh2d_vs_oracle(bk, dims, fused, orth):
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    u = problems.sh2d_sol0(*dims, LX, LY)
    rng = np.random.default_rng(7)
    rhs = rng.standard_normal(sh.N)
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=80, params=(-0.1, 1.3))
    J = ctx.jacobian(u)
    ols = krylov.GMRESIterativeSolvers(reltol=1e-10, restart=80, maxiter=80)
    ls = bk.GMRESB200(reltol=1e-10, restart=80, maxiter=80, orth=orth, fused=fused)
    for a0, a1 in ((3000.0, -1.0), (0.0, 1.0)):  # (3000 I - J): condition number ~4; J alone: not solvable in 80 its
        xo, oko, ito = ols(lambda v: sh.dF(u, v), rhs, a0=a0, a1=a1)
        x, ok, it = ls(J, rhs, a0=a0, a1=a1)
        assert ok == oko
        assert oko == (a0 != 0.0)
        if oko:
            assert abs(it - ito) <= 2, (it, ito)
            assert _rel(x, xo) < 1e-8
            # true residual
            A = a0 * np.eye(1)[0, 0]
            r = rhs - (a0 * x + a1 * sh.dF(u, x))
            assert np.linalg.norm(r) <= 1e-9 * np.linalg.norm(rhs)
        else:
            assert it == 80  # maxiter reached, never throws
        # device-resident rhs
        xd, okd, itd = ls(J, ctx.to_device(rhs), a0=a0, a1=a1)
        assert itd == it and np.array_equal(xd.numpy(), x)
        if dims[0] % 2:  # an odd nx has no fused Arnoldi kernel: fused=True and fused=False run the same kernels
            xf, okf, itf = bk.GMRESB200(reltol=1e-10, restart=80, maxiter=80, orth=orth, fused=not fused)(J, rhs, a0=a0, a1=a1)
            assert okf == ok and itf == it and np.array_equal(xf, x)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("orth", ["cgs", "cgs2"])
def test_gmres_sh2d_vs_oracle(bk, fused, orth):
    _gmres_sh2d_vs_oracle(bk, (96, 64), fused, orth)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("orth", ["cgs", "cgs2"])
def test_gmres_sh2d_odd_width_vs_oracle(bk, fused, orth):
    _gmres_sh2d_vs_oracle(bk, (95, 64), fused, orth)


def test_gmres_restart_and_maxiter(bk):
    dims = (64, 32)
    sh = problems.SwiftHohenberg(dims, (LX, LY))
    u = problems.sh2d_sol0(*dims, LX, LY)
    rhs = np.random.default_rng(8).standard_normal(sh.N)
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=20, params=(-0.1, 1.3))
    J = ctx.jacobian(u)
    x, ok, it = bk.GMRESB200(reltol=1e-9, restart=10, maxiter=400)(J, rhs, a0=3.0, a1=-1.0)
    xo, oko, ito = krylov.GMRESIterativeSolvers(reltol=1e-9, restart=10, maxiter=400)(lambda v: sh.dF(u, v), rhs, a0=3.0, a1=-1.0)
    assert ok and oko and abs(it - ito) <= 3
    assert _rel(x, xo) < 1e-7
    x, ok, it = bk.GMRESB200(reltol=1e-14, restart=20, maxiter=5)(J, rhs, a0=3.0, a1=-1.0)
    assert (not ok) and it == 5  # never throws on non-convergence (src/LinearSolver.jl:202-205)


def test_gmres_sh3d_and_generic_ops(bk):
    # SH3d (stand-alone 3-D stencil), chan and cGL (generic operator path)
    dims, L = (24, 20, 16), (4 * np.pi, 4 * np.pi, 3 * np.pi)  # h ~ 1: (shifted) operator is well conditioned
    sh = problems.SwiftHohenberg(dims, L, l=0.1, nu=1.2)
    u = problems.sh3d_sol0(*dims, *L)
    rhs = np.random.default_rng(9).standard_normal(sh.N)
    ctx = bk.Context(bk.BK_SH3D, dims, L, krylov_m=100, params=(0.1, 1.2))
    x, ok, it = bk.GMRESB200(reltol=1e-10, restart=100, maxiter=100)(ctx.jacobian(u), rhs, a0=40.0, a1=-1.0)
    xo, oko, ito = krylov.GMRESIterativeSolvers(reltol=1e-10, restart=100, maxiter=100)(lambda v: sh.dF(u, v), rhs, a0=40.0, a1=-1.0)
    assert ok and oko, (ok, oko, it, ito)
    assert abs(it - ito) <= 2 and _rel(x, xo) < 1e-8, (it, ito, _rel(x, xo))
    gl = problems.GinzburgLandau2D(24, 12, np.pi, np.pi / 2, r=1.2)
    ug = 0.3 * np.random.default_rng(10).standard_normal(gl.N)
    rg = np.random.default_rng(11).standard_normal(gl.N)
    ctx2 = bk.Context(bk.BK_CGL2D, (24, 12), (np.pi, np.pi / 2), krylov_m=200, params=(1.2, 0.1, 1.0, -1.0, 1.0))
    x, ok, it = bk.GMRESB200(reltol=1e-10, restart=200, maxiter=200)(ctx2.jacobian(ug), rg, a0=60.0, a1=-1.0)
    xo, oko, ito = krylov.GMRESIterativeSolvers(reltol=1e-10, restart=200, maxiter=200)(lambda v: gl.dF(ug, v), rg, a0=60.0, a1=-1.0)
    assert ok and oko, (ok, oko, it, ito)
    assert abs(it - ito) <= 2 and _rel(x, xo) < 1e-8, (it, ito, _rel(x, xo))


def test_bls_map_and_bordered_solvers(bk):
    """test/linear_solvers/test_linear.jl:71-85,172-244 restated on the SH2d Jacobian."""
    dims = (48, 32)
    sh = problems.SwiftHohenberg(dims, (LX, LY))
    u = problems.sh2d_sol0(*dims, LX, LY)
    rng = np.random.default_rng(12)
    N = sh.N
    a, b, R = rng.standard_normal(N), rng.standard_normal(N), rng.standard_normal(N)
    c, n = 0.37, -0.81
    x = rng.standard_normal(N + 1)
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=400, params=(-0.1, 1.3))
    J = ctx.jacobian(u)
    Jd = sh.jac_sparse(u).toarray()
    for shift in (None, 2.5):
        m = obls.MatrixFreeBLSmap(Jd, a, b, c, shift, lambda p, q: np.dot(p, q) / N)
        assert _rel(bk.bls_map(J, a, b, c, x, shift=shift, dotscale=1.0 / N), m(x)) < 1e-12
    # bordered solves on the shifted (well conditioned) operator  (shift I + J) with shift = -3
    shift, xiu, xip, dzp = -3.0, 0.5, 0.5, 0.9
    A = np.zeros((N + 1, N + 1))
    A[:N, :N] = Jd + shift * np.eye(N)
    A[:N, N] = a
    A[N, :N] = xiu * b / N
    A[N, N] = xip * dzp
    ref = np.linalg.solve(A, np.concatenate([R, [n]]))
    ls = bk.GMRESB200(reltol=1e-12, restart=400, maxiter=400, orth="cgs2")  # cond(J - 3I) ~ 200 on this grid  # 1e-12 needs re-orthogonalisation
    for solver in (bk.BorderingBLSB200(ls, check_precision=False), bk.BorderingBLSB200(ls, check_precision=True, k=2),
                   bk.MatrixFreeBLSB200(ls)):
        dX, dl, ok, it = solver(J, a, b, dzp, R, n, xiu, xip, shift=shift, dotscale=1.0 / N)
        assert ok, type(solver)
        assert _rel(dX, ref[:N]) < 1e-8 and abs(dl - ref[N]) < 1e-8 * max(1, abs(ref[N])), type(solver)
        # device-resident arguments
        dXd, dld, okd, _ = solver(J, ctx.to_device(a), ctx.to_device(b), dzp, ctx.to_device(R), n, xiu, xip,
                                  shift=shift, dotscale=1.0 / N)
        assert _rel(dXd.numpy(), ref[:N]) < 1e-8 and abs(dld - ref[N]) < 1e-8 * max(1, abs(ref[N]))


@pytest.mark.parametrize("fused", [2, 1, 0])
@pytest.mark.parametrize("side", ["none", "right", "left"])
def test_gmres_sh3d_fused_and_unfused_paths_agree_with_oracle(bk, fused, side):
    """3-D: stand-alone JVP + TMA-ring dots against the oracle, with the DCT preconditioner on either side.  There is no fused
    3-D kernel, so every value of `fused` gives the same bits and iteration count as the default fused = 1."""
    from oracle import precond as oprecond
    dims, L = (32, 16, 16), (4 * np.pi, 2 * np.pi, 2 * np.pi)
    sh = problems.SwiftHohenberg(dims, L, l=0.1, nu=1.2)
    u = problems.sh3d_sol0(*dims, *L)
    rhs = np.random.default_rng(31).standard_normal(sh.N)
    Pinv = oprecond.dct_precond(dims, L, 1.0)
    kw = {"none": {}, "right": dict(Pr=Pinv), "left": dict(Pl=Pinv)}[side]
    a0, a1 = 40.0, -1.0  # shifted operator: definite, converges for every variant
    xo, oko, ito = krylov.GMRESIterativeSolvers(reltol=1e-9, restart=120, maxiter=120, **kw)(lambda v: sh.dF(u, v), rhs, a0=a0, a1=a1)
    ctx = bk.Context(bk.BK_SH3D, dims, L, krylov_m=120, params=(0.1, 1.2))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    J = ctx.jacobian(u)
    solve = lambda fused: bk.GMRESB200(reltol=1e-9, restart=120, maxiter=120, fused=fused, Pr=side == "right", Pl=side == "left")(
        J, rhs, a0=a0, a1=a1)
    x, ok, it = solve(fused)
    assert ok and oko, (ok, oko, it, ito)
    assert abs(it - ito) <= 3 and _rel(x, xo) < 1e-7, (it, ito, _rel(x, xo))
    x1, ok1, it1 = solve(1)
    assert ok1 and it1 == it and np.array_equal(x1, x), (it1, it)


@pytest.mark.parametrize("N", [4849664, 4849664 + 1, 2424832 + 777])
def test_gmres_many_waves_of_tall_tiles(bk, N):
    """Regression: vectors long enough that the TMA-ring kernels run several waves of 8-row tiles (18944 rows of 256 =
    4 waves of 592 CTAs).  Before the consumers fenced their shared-memory reads against the async-proxy refill of a ring
    stage, a few tiles per launch were overwritten while still being read: GMRES stalled at ~0.17 and its recursive
    residual estimate disagreed with the true residual (tools/k2check/k2_check.cu isolates the kernels)."""
    ctx = bk.Context(bk.BK_CHAN, (N,), (1.0,), krylov_m=40, params=(3.3, 0.01))
    rng = np.random.default_rng(1)
    u = 0.1 * rng.standard_normal(N)
    b = rng.standard_normal(N)
    J = ctx.jacobian(ctx.to_device(u))
    rhs = ctx.to_device(b)
    a0 = -0.4 * float(N - 1) ** 2  # a0 I + J: moderately conditioned, ~34 iterations to 1e-9
    for orth in ("cgs", "cgs2"):
        ls = bk.GMRESB200(reltol=1e-9, restart=40, maxiter=40, orth=orth)
        x, ok, it = ls(J, rhs, a0=a0)
        true = np.linalg.norm(ctx.jvp(x, a0=a0).numpy() - b) / np.linalg.norm(b)
        est = ls.last_resnorm / np.linalg.norm(b)
        assert ok and it <= 38, (orth, it, est, true)
        assert true < 2e-9 and abs(true - est) < 1e-3 * est + 1e-12, (orth, est, true)


def test_gmres_two_right_hand_sides(bk):
    """S2 (src/LinearSolver.jl:15-19): ls(J, rhs1, rhs2) -> (x1, x2, flag1 & flag2, (it1, it2)) through bk_gmres2, host and device
    vectors, against two single solves and the oracle."""
    from oracle import precond as oprecond
    dims = (128, 64)
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    rng = np.random.default_rng(11)
    u = problems.sh2d_sol0(*dims, LX, LY)
    r1, r2 = rng.standard_normal(sh.N), rng.standard_normal(sh.N)
    ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=80, params=(-0.1, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(reltol=1e-9, restart=80, maxiter=80, Pr=True, orth="cgs2")
    J = ctx.jacobian(u)
    x1, x2, ok, (it1, it2) = ls(J, r1, r2, a0=1.5, a1=-1.0)
    y1, ok1, j1 = ls(J, r1, a0=1.5, a1=-1.0)
    y2, ok2, j2 = ls(J, r2, a0=1.5, a1=-1.0)
    assert ok and ok1 and ok2 and (it1, it2) == (j1, j2)
    assert np.array_equal(x1, y1) and np.array_equal(x2, y2)
    Pinv = oprecond.dct_precond(dims, (LX, LY), 1.0)
    ols = krylov.GMRESIterativeSolvers(reltol=1e-9, restart=80, maxiter=80, Pr=Pinv)
    o1, o2, oko, _ = ols(lambda v: sh.dF(u, v), r1, r2, a0=1.5, a1=-1.0)
    assert oko and _rel(x1, o1) < 1e-7 and _rel(x2, o2) < 1e-7
    d1, d2, okd, itd = ls(ctx.jacobian(ctx.to_device(u)), ctx.to_device(r1), ctx.to_device(r2), a0=1.5, a1=-1.0)
    assert okd and np.array_equal(d1.numpy(), x1) and np.array_equal(d2.numpy(), x2)


def test_two_contexts_with_different_krylov_dimensions_interleaved(bk):
    """cudaFuncAttributeMaxDynamicSharedMemorySize belongs to (device, kernel), not to a context: a context with a small Krylov
    dimension used between two solves of a large one must not shrink the large one's grant (found by the Hopf refinement, which
    alternates between a real and a complexified context)."""
    rng = np.random.default_rng(21)
    dims = (64, 32)
    sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
    u = problems.sh2d_sol0(*dims, LX, LY)
    rhs = rng.standard_normal(sh.N)
    big = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=400, params=(-0.1, 1.3))
    big.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(reltol=1e-9, restart=400, maxiter=400, Pr=True)
    x1, cv1, it1 = ls(big.jacobian(u), rhs)
    small = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=10, params=(-0.1, 1.3))
    small.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    bk.GMRESB200(reltol=1e-3, restart=10, maxiter=20, Pr=True)(small.jacobian(u), rhs)
    x2, cv2, it2 = ls(big.jacobian(u), rhs)
    assert cv1 and cv2 and it1 == it2 and np.array_equal(x1, x2)


@pytest.mark.parametrize("kind", ["sh2d", "cgl", "sh2d_odd"])
def test_block_bordered_solvers(bk, kind):
    """solve_bls_block with two borders (src/LinearBorderSolver.jl:173-206 BorderingBLS, :440-450 MatrixFreeBLS over the tuple
    map :366-389; exercised with random borders by test/linear_solvers/test_linear.jl:300-320): device path vs the oracle's
    restatement and vs the explicit (N + 2) x (N + 2) dense solve; also m = 1 against the scalar-border entry points, bit for bit."""
    rng = np.random.default_rng(31)
    # bordering: residual tolerance 1e-12 x cond(J) = 3e3 (Swift-Hohenberg near its pattern-forming modes), Schur elimination on top.
    # matrix-free: cond of the bordered matrix is 2e4, a relative residual of 1e-12 is below what fp64 attains there (the solve
    # stagnates at an error of 2e-11); the reference's own test of this call only asserts convergence (test_linear.jl:318-320)
    TOLB, TOLM = 1e-7, 1e-6
    if kind == "cgl":
        gl = problems.GinzburgLandau2D(24, 12, np.pi, np.pi / 2, r=1.2)
        N, u, dF = gl.N, 0.3 * rng.standard_normal(gl.N), gl.dF
        ctx = bk.Context(bk.BK_CGL2D, (24, 12), (np.pi, np.pi / 2), krylov_m=300, params=(1.2, 0.1, 1.0, -1.0, 1.0))
        ls = bk.GMRESB200(reltol=1e-12, restart=300, maxiter=900, orth="cgs2")
    else:
        dims = (32, 16) if kind == "sh2d" else (15, 9)          # odd N: the (N + 2)-vectors use the pad element behind them
        sh = problems.SwiftHohenberg(dims, (LX, LY), l=-0.1, nu=1.3)
        N, u, dF = sh.N, problems.sh2d_sol0(*dims, LX, LY) + 0.1 * rng.standard_normal(sh.N), sh.dF
        # Krylov dimension >= N + 2: no restarts.  J + 0.3 I is indefinite here and GMRES(200) stagnates on it (measured: full GMRES
        # needs 211-222 iterations for 1e-8..1e-12, GMRES(200) 500+ and GMRES(100) does not get below 1e-7 in 600)
        ctx = bk.Context(bk.BK_SH2D, dims, (LX, LY), krylov_m=560, params=(-0.1, 1.3))
        ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
        ls = bk.GMRESB200(reltol=1e-12, restart=560, maxiter=1120, Pr=True, orth="cgs2")
    lm = bk.GMRESB200(reltol=1e-10, restart=ls.restart, maxiter=ls.maxiter, Pr=ls.Pr, orth="cgs2")
    Jd = np.column_stack([dF(u, np.eye(N)[:, j]) for j in range(N)])
    a = (rng.standard_normal(N), rng.standard_normal(N))
    b = (rng.standard_normal(N), rng.standard_normal(N))
    c = rng.standard_normal((2, 2))
    rhst, rhsb = rng.standard_normal(N), rng.standard_normal(2)
    J = ctx.jacobian(u)
    for shift in (None, 0.3):
        sv = 0.0 if shift is None else shift
        A = np.block([[Jd + sv * np.eye(N), np.column_stack(a)], [np.vstack(b), c]])
        ex = np.linalg.solve(A, np.concatenate([rhst, rhsb]))
        x = rng.standard_normal(N + 2)
        assert _rel(bk.bls_map_block(J, a, b, c, x, shift=shift), A @ x) < 1e-12
        assert _rel(bk.bls_map_block(J, a, b, c, x, shift=shift), obls.MatrixFreeBLSmapBlock(Jd, a, b, c, shift, np.dot)(x)) < 1e-12
        # one border is the block form with m = 1, bit for bit
        x1 = x[:N + 1]
        assert np.array_equal(bk.bls_map(J, a[0], b[0], c[0, 0], x1, shift=shift, dotscale=1.0 / N),
                              bk.bls_map_block(J, (a[0],), (b[0],), [[c[0, 0]]], x1, shift=shift, dotscale=1.0 / N))
        ub, pb, cvb, itb = bk.BorderingBLSB200(ls).solve_block(J, a, b, c, rhst, rhsb, shift=shift)
        assert cvb and _rel(ub, ex[:N]) < TOLB and _rel(pb, ex[N:]) < TOLB and len(itb) == 3, (cvb, itb, _rel(ub, ex[:N]), _rel(pb, ex[N:]))
        um, pm, cvm, itm = bk.MatrixFreeBLSB200(lm).solve_block(J, a, b, c, rhst, rhsb, shift=shift)
        assert cvm and _rel(um, ex[:N]) < TOLM and _rel(pm, ex[N:]) < TOLM, (cvm, itm, _rel(um, ex[:N]), _rel(pm, ex[N:]))
        # normalised dot product (dotp = <.,.> / N) only rescales the border rows
        A2 = A.copy()
        A2[N:, :N] /= N
        ex2 = np.linalg.solve(A2, np.concatenate([rhst, rhsb]))
        u2, p2, cv2, _ = bk.MatrixFreeBLSB200(lm).solve_block(J, a, b, c, rhst, rhsb, shift=shift, dotscale=1.0 / N)
        assert cv2 and _rel(u2, ex2[:N]) < TOLM and _rel(p2, ex2[N:]) < TOLM, (cv2, _rel(u2, ex2[:N]), _rel(p2, ex2[N:]))
    # m = 1 block form == scalar-border entry points
    u1, p1, cv1, _ = bk.MatrixFreeBLSB200(lm).solve_block(J, (a[0],), (b[0],), [[0.7]], rhst, [rhsb[0]])
    us, ps, cvs, _ = bk.MatrixFreeBLSB200(lm)(J, a[0], b[0], 0.7, rhst, rhsb[0])
    assert cv1 and cvs and np.array_equal(u1, us) and p1[0] == ps
    # device-resident vectors give the same result
    ad, bd = tuple(ctx.to_device(v) for v in a), tuple(ctx.to_device(v) for v in b)
    ud, pd_, cvd, _ = bk.MatrixFreeBLSB200(lm).solve_block(J, ad, bd, c, ctx.to_device(rhst), rhsb)
    A = np.block([[Jd, np.column_stack(a)], [np.vstack(b), c]])
    ex = np.linalg.solve(A, np.concatenate([rhst, rhsb]))
    assert cvd and _rel(ud.numpy(), ex[:N]) < TOLM and _rel(pd_, ex[N:]) < TOLM
    with pytest.raises(AssertionError):
        bk.BorderingBLSB200(ls).solve_block(J, a, b[:1], c, rhst, rhsb)
