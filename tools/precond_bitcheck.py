"""Writes the result of every preconditioner path on seeded inputs as .npy files, so that two builds can be compared bit for bit:

   python tools/precond_bitcheck.py --out DIR [--root TREE]
   cmp DIR_A/x.npy DIR_B/x.npy   (for every file)

TREE is the repository whose build is loaded (default: the one holding this script); the script uses the public API only, so it
runs against any build of the library.  Cases: BK_PC_SH_DCT in 2-D and 3-D at power-of-two, mixed and odd sizes on aligned
vectors and on vectors offset by one double; the border entries of right-preconditioned matrix-free bordered solves (one border
and a block of two), which a plain application never has; BK_COMPLEX contexts; BK_PC_CGL_DST on cGL2d and Trapeze contexts;
BK_PC_POTRAP_CIRC with J' off and on; BK_PC_CHAN_TRIDIAG; BK_PC_SH_FFT with a right-preconditioned periodic GMRES solve.  The
BK_PC_SH_DCT cases run again in a child process under BK_FFT_NO_FAST=1 (general kernel everywhere; files nofast_*).

The Krylov drivers (files krylov_*) write x, iters, resnorm and converged of each GMRES solve, the eigenvalues, eigenvectors,
nconv and nops of each shift-invert solve, and the bk_get_stats counters after each call.  GMRES: SH2d with an even nx (k2_fused)
and an odd nx (apply + k2_dots), CGS and CGS2, restart below the iteration count, Pl and Pr with BK_PC_SH_DCT, one border and a
block of two, a solve whose CGS check falls back to CGS2, a BK_COMPLEX solve with an imaginary shift, and periodic SH2d with
BK_PC_SH_FFT on each side, fused and not.  Eigensolver: SH2d thick restart and cGL2d explicit restart with restarts forced,
eigenvectors to host and to device memory, and a given start vector.

The problem kernels (files problems_*) write their outputs and the bk_get_stats counters after each call, on host and on device
vectors: residual and JVP (a0 != 0, a1 != 1) of chan, SH2d (odd and even nx), SH3d, periodic SH2d, cGL2d (J and J'), BK_COMPLEX
cGL2d with an imaginary shift (J and J'), and Trapeze (J and J' after a section is set, reading the F-cache that
bk_jac_set_state fills); bls_map / bls_map_block on cGL2d and Trapeze contexts; d2F / d3F of every kind with jets; jet moments
of chan, SH2d and cGL2d, with more than 64 vectors and more than 8192 tuples; deflation moments with 0, 1 and 2 directions,
1, 5, 64 and 70 roots, and a prefix n < N0; and potrap_update_section at scale 1/M and 1, each followed by a residual."""
import argparse
import ctypes as C
import importlib.util
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import problems  # noqa: E402

SH_DCT_2D = [(1024, 1024), (151, 100), (62, 64), (64, 62), (256, 128)]
SH_DCT_3D = [(64, 64, 64), (48, 32, 16)]
SH_PAR = (-0.1, 1.3)
CGL_PAR = (1.2, 0.1, 1.0, -1.0, 1.0)


def load(root):
    spec = importlib.util.spec_from_file_location("bitcheck_graft_entry", os.path.join(root, "__graft_entry__.py"))
    ge = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ge)
    return ge.load_package()


class Dump:
    def __init__(self, out, prefix):
        self.out, self.prefix = out, prefix
        os.makedirs(out, exist_ok=True)

    def __call__(self, name, a):
        np.save(os.path.join(self.out, self.prefix + name + ".npy"), np.asarray(a, dtype=np.float64))


def applications(bk, ctx, r, name, dump):
    """host vectors (staged, aligned), device vectors, and device vectors offset by 8 bytes (in and out, then in only)"""
    dump(name + "_host", ctx.precond_apply(r))
    dump(name + "_dev", ctx.precond_apply(ctx.to_device(r)).numpy())
    n = ctx.N
    big_in, big_out = ctx.zeros(n + 2), ctx.zeros(n + 2)
    host = np.concatenate([[0.0], r, [0.0]])
    assert ctx.lib.bk_vec_upload(ctx.handle, big_in.dptr, host.ctypes.data, len(host)) == 0
    for tag, shift_out in (("off8", 8), ("off8in", 0)):
        big_out.zero_()
        st = ctx.lib.bk_precond_apply(ctx.handle, C.c_void_p(big_in.dptr + 8), C.c_void_p(big_out.dptr + shift_out))
        assert st == 0, ctx.lib.bk_last_error(ctx.handle)
        dump(f"{name}_{tag}", big_out.numpy())


def bordered(bk, ctx, u, rng, name, dump, restart=30):
    """right-preconditioned matrix-free bordered solves at u: N + 1 (one border) and N + 2 (a block of two) unknowns"""
    N = ctx.N
    ls = bk.GMRESB200(reltol=1e-12, restart=restart, maxiter=restart, Pr=True)
    J = ctx.jacobian(u)
    dR, dzu, R = rng.standard_normal(N), rng.standard_normal(N), rng.standard_normal(N)
    dX, dl, _, it = bk.MatrixFreeBLSB200(ls)(J, dR, dzu, 0.8, R, -0.4, shift=-0.5, dotscale=1.0 / N)
    dump(name + "_bls1", np.concatenate([dX, [dl, it]]))
    a = (rng.standard_normal(N), rng.standard_normal(N))
    b = (rng.standard_normal(N), rng.standard_normal(N))
    x, p, _, it = bk.MatrixFreeBLSB200(ls).solve_block(J, a, b, [[0.9, 0.1], [-0.2, 1.1]], R, [0.3, -0.7], shift=-0.5,
                                                        dotscale=1.0 / N)
    dump(name + "_bls2", np.concatenate([x, p, [it]]))


def sh_dct(bk, dump):
    for dims in SH_DCT_2D + SH_DCT_3D:
        kind = bk.BK_SH2D if len(dims) == 2 else bk.BK_SH3D
        L = (8 * np.pi, 4 * np.pi / np.sqrt(3)) if len(dims) == 2 else (np.pi, 1.3 * np.pi, 0.7 * np.pi)
        ctx = bk.Context(kind, dims, L, krylov_m=30, params=SH_PAR)
        rng = np.random.default_rng(sum(dims))
        name = "sh_dct_" + "x".join(map(str, dims))
        for shift in (1.0, 0.25):
            ctx.precond_setup(bk.BK_PC_SH_DCT, shift)
            applications(bk, ctx, rng.standard_normal(ctx.N), f"{name}_s{shift}", dump)
        if dims in ((256, 128), (151, 100), (48, 32, 16)):
            bordered(bk, ctx, 0.3 * rng.standard_normal(ctx.N), rng, name, dump)
        ctx.close()
    ctx = bk.Context(bk.BK_SH2D, (256, 128), (8 * np.pi, 4 * np.pi), krylov_m=2, params=SH_PAR, complex=True)
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    applications(bk, ctx, np.random.default_rng(1).standard_normal(ctx.N), "sh_dct_complex_256x128", dump)
    ctx.close()


def others(bk, dump):
    rng = np.random.default_rng(7)
    for dims in ((41, 21), (512, 512)):
        ctx = bk.Context(bk.BK_CGL2D, dims, (0.5 * np.pi, np.pi), krylov_m=30, params=CGL_PAR)
        ctx.precond_setup(bk.BK_PC_CGL_DST, 1.0, -0.05)
        name = "cgl_dst_" + "x".join(map(str, dims))
        applications(bk, ctx, rng.standard_normal(ctx.N), name, dump)
        bordered(bk, ctx, 0.3 * rng.standard_normal(ctx.N), rng, name, dump)
        ctx.close()
    ctx = bk.Context(bk.BK_CGL2D, (24, 12), (np.pi, np.pi / 2), krylov_m=2, params=CGL_PAR, complex=True)
    ctx.precond_setup(bk.BK_PC_CGL_DST, -1.0, 1.0)
    applications(bk, ctx, rng.standard_normal(ctx.N), "cgl_dst_complex_24x12", dump)
    ctx.close()
    for dims, M in (((16, 12), 10), ((41, 21), 30)):
        ctx = bk.Context(bk.BK_POTRAP_CGL2D, (*dims, M), (np.pi, np.pi / 2), krylov_m=30, params=(1.3,) + CGL_PAR[1:])
        name = f"potrap_{dims[0]}x{dims[1]}x{M}"
        r = rng.standard_normal(ctx.N)
        ctx.precond_setup(bk.BK_PC_CGL_DST, 1.0, -0.05)
        applications(bk, ctx, r, name + "_cgl_dst", dump)
        ctx.precond_setup(bk.BK_PC_POTRAP_CIRC, 6.3)
        applications(bk, ctx, r, name + "_circ", dump)
        ctx.set_transpose(True)
        applications(bk, ctx, r, name + "_circ_tr", dump)
        ctx.set_transpose(False)
        x = 0.1 * rng.standard_normal(ctx.N)
        x[-1] = 6.3
        ctx.potrap_set_section(rng.standard_normal(ctx.N - 1) / np.sqrt(ctx.N), x[:-1])
        bordered(bk, ctx, x, rng, name + "_circ", dump)
        ctx.close()
    ctx = bk.Context(bk.BK_CHAN, (1000,), krylov_m=2, params=(3.3, 0.01))
    ctx.precond_setup(bk.BK_PC_CHAN_TRIDIAG)
    applications(bk, ctx, rng.standard_normal(ctx.N), "chan_tridiag_1000", dump)
    ctx.close()
    for dims in ((256, 128), (64, 2048)):
        ctx = bk.Context(bk.BK_SH2D_PERIODIC, dims, (8 * np.pi, 4 * np.pi), krylov_m=40, params=(-0.15, 1.3))
        name = "sh_fft_" + "x".join(map(str, dims))
        for a0 in (1.0, 0.25):
            ctx.precond_setup(bk.BK_PC_SH_FFT, a0)
            applications(bk, ctx, rng.standard_normal(ctx.N), f"{name}_a{a0}", dump)
        u = 0.3 * rng.standard_normal(ctx.N)
        bordered(bk, ctx, u, rng, name, dump)
        J, rhs = ctx.jacobian(u), rng.standard_normal(ctx.N)
        for fused in (True, False):
            x, _, it = bk.GMRESB200(reltol=1e-12, restart=40, maxiter=40, Pr=True, fused=fused)(J, rhs)
            dump(f"{name}_gmres_fused{int(fused)}", np.concatenate([x, [it]]))
        ctx.close()


def counters(ctx, name, dump):
    """the bk_get_stats counters (not the timers) after a call"""
    dump(name + "_stats", [v for k, v in ctx.stats().items() if not k.endswith("_ms")])


def gmres(bk, ctx, J, rhs, name, dump, a0=0.0, a1=1.0, **kw):
    ls = bk.GMRESB200(**kw)
    x, cv, it = ls(J, rhs, a0=a0, a1=a1)
    dump(name, np.concatenate([x, [it, ls.last_resnorm, cv]]))
    counters(ctx, name, dump)


def eigs(bk, ctx, sigma, inner, nev, kd, maxrestart, name, dump, v0=None, device=False):
    """bk_eigs_shift_invert with the eigenvectors written to host memory or to a device vector"""
    re, im = np.zeros(nev), np.zeros(nev)
    vecs = ctx.zeros(nev * ctx.N) if device else np.zeros(nev * ctx.N)
    nconv, nops = C.c_int32(), C.c_int32()
    dp = C.POINTER(C.c_double)
    st = ctx.lib.bk_eigs_shift_invert(ctx.handle, sigma, nev, kd, 1e-8, maxrestart, C.byref(inner.opts()), C.c_void_p(
        bk.lib.ptr(v0)), re.ctypes.data_as(dp), im.ctypes.data_as(dp), C.c_void_p(bk.lib.ptr(vecs)), C.byref(nconv), C.byref(nops))
    assert st >= 0, ctx.lib.bk_last_error(ctx.handle)
    dump(name, np.concatenate([re, im, vecs.numpy() if device else vecs, [st, nconv.value, nops.value]]))
    counters(ctx, name, dump)


def krylov(bk, dump):
    L = (8 * np.pi, 4 * np.pi / np.sqrt(3))
    rng = np.random.default_rng(11)
    for dims in ((256, 128), (255, 96)):  # k2_fused; the stand-alone apply + k2_dots
        ctx = bk.Context(bk.BK_SH2D, dims, L, krylov_m=60, params=SH_PAR)
        u = problems.sh2d_sol0(*dims, *L) + 0.1 * rng.standard_normal(ctx.N)
        J, rhs = ctx.jacobian(u), rng.standard_normal(ctx.N)
        name = "krylov_sh2d_" + "x".join(map(str, dims))
        a0 = 0.3 * (1 - 4 / (2 * L[0] / dims[0]) ** 2 - 4 / (2 * L[1] / dims[1]) ** 2) ** 2 + 3.0  # condition number ~5
        for orth in ("cgs", "cgs2"):  # reltol < 1e-9: every converged CGS cycle is checked against the true residual
            gmres(bk, ctx, J, rhs, f"{name}_{orth}", dump, a0, -1.0, reltol=1e-10, restart=60, maxiter=200, orth=orth)
        gmres(bk, ctx, J, rhs, name + "_restart7", dump, a0, -1.0, reltol=1e-10, restart=7, maxiter=200)
        ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
        for side in ("Pl", "Pr"):
            gmres(bk, ctx, J, rhs, f"{name}_{side}", dump, 1.0, 1.0, reltol=1e-10, restart=60, maxiter=200, **{side: True})
        bordered(bk, ctx, u, rng, name, dump)
        counters(ctx, name + "_bls", dump)
        ctx.close()
    dims = (48, 32)  # reltol 1e-13 is below what single-pass CGS attains here: the CGS check fails once and CGS2 takes over
    ctx = bk.Context(bk.BK_SH2D, dims, L, krylov_m=400, params=SH_PAR)
    u = problems.sh2d_sol0(*dims, *L) + 0.1 * np.random.default_rng(1).standard_normal(ctx.N)
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    gmres(bk, ctx, ctx.jacobian(u), np.random.default_rng(7).standard_normal(ctx.N), "krylov_cgs_fallback", dump, 1.0, 1.0,
          reltol=1e-13, restart=400, maxiter=400, Pr=True)
    ctx.close()
    ctx = bk.Context(bk.BK_SH2D, (64, 48), L, krylov_m=60, params=SH_PAR, complex=True)
    J = ctx.cjacobian(0.3 * rng.standard_normal(ctx.N0))
    rhs = rng.standard_normal(ctx.N0) + 1j * rng.standard_normal(ctx.N0)
    ls = bk.ComplexGMRESB200(reltol=1e-10, restart=60, maxiter=300, orth="cgs2")
    x, cv, it = ls(J, rhs, a0=complex(2.0, -0.7), a1=-1.0)
    dump("krylov_complex", np.concatenate([x.real, x.imag, [it, ls.last_resnorm, cv]]))
    counters(ctx, "krylov_complex", dump)
    ctx.close()
    ctx = bk.Context(bk.BK_SH2D_PERIODIC, (128, 128), (8 * np.pi, 8 * np.pi), krylov_m=40, params=(-0.15, 1.3))
    J, rhs = ctx.jacobian(0.3 * rng.standard_normal(ctx.N)), rng.standard_normal(ctx.N)
    ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
    for side in ("Pl", "Pr"):
        for fused in (True, False):
            gmres(bk, ctx, J, rhs, f"krylov_sh_fft_{side}_fused{int(fused)}", dump, reltol=1e-12, restart=40, maxiter=80,
                  fused=fused, **{side: True})
    ctx.close()

    dims = (64, 48)
    ctx = bk.Context(bk.BK_SH2D, dims, L, krylov_m=60, params=SH_PAR)
    ctx.jacobian(problems.sh2d_sol0(*dims, *L))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    inner = bk.GMRESB200(reltol=1e-10, restart=60, maxiter=600, Pr=True)
    v0 = rng.standard_normal(ctx.N)
    eigs(bk, ctx, 0.1, inner, 4, 10, 40, "krylov_eigs_thick", dump)  # krylovdim 10: restarted
    eigs(bk, ctx, 0.1, inner, 4, 10, 40, "krylov_eigs_thick_dev", dump, device=True)
    eigs(bk, ctx, 0.1, inner, 4, 10, 40, "krylov_eigs_thick_v0", dump, v0=v0)
    eigs(bk, ctx, 0.1, inner, 4, 10, 40, "krylov_eigs_thick_v0dev", dump, v0=ctx.to_device(v0), device=True)
    ctx.close()
    ctx = bk.Context(bk.BK_CGL2D, (12, 8), (np.pi, np.pi / 2), krylov_m=60, params=(1.8, 0.1, 0.3, -1.0, 1.0))
    ctx.jacobian(0.1 * np.random.default_rng(5).standard_normal(ctx.N))
    inner = bk.GMRESB200(reltol=1e-12, restart=60, maxiter=2000, orth="cgs2")
    v0 = rng.standard_normal(ctx.N)
    eigs(bk, ctx, 0.5, inner, 4, 8, 200, "krylov_eigs_explicit", dump)  # krylovdim 8: restarted
    eigs(bk, ctx, 0.5, inner, 4, 8, 200, "krylov_eigs_explicit_dev", dump, device=True)
    eigs(bk, ctx, 0.5, inner, 4, 8, 200, "krylov_eigs_explicit_v0", dump, v0=v0)
    ctx.close()


def problem_kernels(bk, dump):
    rng = np.random.default_rng(13)

    def both(ctx, name, f, v):
        """f on a host vector and on a device vector, then the counters"""
        dump(name + "_host", f(v))
        dump(name + "_dev", f(ctx.to_device(v)).numpy())
        counters(ctx, name, dump)

    def res_jvp(ctx, name, u, n=None):
        n = ctx.N if n is None else n
        both(ctx, name + "_res", ctx.residual, u)
        ctx.jacobian(u)
        both(ctx, name + "_jvp", lambda v: ctx.jvp(v, a0=0.7, a1=-1.3), rng.standard_normal(n))

    def jets(ctx, name):
        u, a, b, c = (rng.standard_normal(ctx.N0) for _ in range(4))
        dump(name + "_d2f_host", ctx.d2f(u, a, b))
        dump(name + "_d3f_host", ctx.d3f(u, a, b, c))
        du, da, db, dc = (ctx.to_device(x) for x in (u, a, b, c))
        dump(name + "_d2f_dev", ctx.d2f(du, da, db).numpy())
        dump(name + "_d3f_dev", ctx.d3f(du, da, db, dc).numpy())
        counters(ctx, name + "_jets", dump)

    def moments(ctx, name, nvec):
        u = 0.5 * rng.standard_normal(ctx.N0)
        vecs = [rng.standard_normal(ctx.N0) for _ in range(nvec)]
        idx2, idx3 = rng.integers(0, nvec, (40, 3)), rng.integers(0, nvec, (30, 4))
        dump(name + "_mom_host", ctx.jet_moments(u, vecs, idx2, idx3))
        dump(name + "_mom_dev", ctx.jet_moments(ctx.to_device(u), [ctx.to_device(v) for v in vecs], idx2, idx3))
        counters(ctx, name + "_mom", dump)

    L2 = (8 * np.pi, 4 * np.pi / np.sqrt(3))
    ctx = bk.Context(bk.BK_CHAN, (1000,), (1.0,), krylov_m=4, params=(3.3, 0.01))
    res_jvp(ctx, "problems_chan", 0.3 * rng.standard_normal(ctx.N))
    jets(ctx, "problems_chan")
    moments(ctx, "problems_chan", 5)
    ctx.close()
    for dims in ((96, 64), (95, 64)):
        ctx = bk.Context(bk.BK_SH2D, dims, L2, krylov_m=4, params=SH_PAR)
        name = "problems_sh2d_" + "x".join(map(str, dims))
        res_jvp(ctx, name, 0.3 * rng.standard_normal(ctx.N))
        jets(ctx, name)
        ctx.close()
    ctx = bk.Context(bk.BK_SH2D, (64, 48), L2, krylov_m=4, params=SH_PAR)
    moments(ctx, "problems_sh2d_64x48", 70)  # more than BK_JET_MOMENTS_MAX_VEC vectors: several calls
    u, vecs = rng.standard_normal(ctx.N0), [rng.standard_normal(ctx.N0) for _ in range(8)]
    dump("problems_sh2d_mom_tuples", ctx.jet_moments(u, vecs, rng.integers(0, 8, (6000, 3)), rng.integers(0, 8, (4000, 4))))
    counters(ctx, "problems_sh2d_mom_tuples", dump)
    ctx.close()
    ctx = bk.Context(bk.BK_SH3D, (24, 20, 16), (np.pi, 1.3 * np.pi, 0.7 * np.pi), krylov_m=4, params=(0.1, 1.2))
    res_jvp(ctx, "problems_sh3d", 0.3 * rng.standard_normal(ctx.N))
    jets(ctx, "problems_sh3d")
    ctx.close()
    ctx = bk.Context(bk.BK_SH2D_PERIODIC, (128, 64), (8 * np.pi, 4 * np.pi), krylov_m=4, params=(-0.15, 1.3))
    res_jvp(ctx, "problems_sh_periodic", 0.3 * rng.standard_normal(ctx.N))
    jets(ctx, "problems_sh_periodic")
    ctx.close()
    ctx = bk.Context(bk.BK_CGL2D, (41, 21), (0.5 * np.pi, np.pi), krylov_m=4, params=CGL_PAR)
    u = 0.3 * rng.standard_normal(ctx.N)
    res_jvp(ctx, "problems_cgl", u)
    ctx.set_transpose(True)
    both(ctx, "problems_cgl_jvp_tr", lambda v: ctx.jvp(v, a0=0.7, a1=-1.3), rng.standard_normal(ctx.N))
    ctx.set_transpose(False)
    jets(ctx, "problems_cgl")
    moments(ctx, "problems_cgl", 6)
    J, N = ctx.jacobian(u), ctx.N
    a, b = rng.standard_normal(N), rng.standard_normal(N)
    dump("problems_cgl_bls1", bk.bls_map(J, a, b, 0.8, rng.standard_normal(N + 1), shift=-0.5, dotscale=1.0 / N))
    ab = (rng.standard_normal(N), rng.standard_normal(N))
    dump("problems_cgl_bls2", bk.bls_map_block(J, ab, (a, b), [[0.9, 0.1], [-0.2, 1.1]], rng.standard_normal(N + 2), shift=-0.5,
                                                dotscale=1.0 / N))
    counters(ctx, "problems_cgl_bls", dump)
    ctx.close()
    ctx = bk.Context(bk.BK_CGL2D, (24, 12), (np.pi, np.pi / 2), krylov_m=4, params=CGL_PAR, complex=True)
    u = 0.3 * rng.standard_normal(ctx.N0)
    both(ctx, "problems_cgl_complex_res", ctx.residual, u)
    ctx.jacobian(u)
    ctx.set_shift_imag(-0.6)
    for tr in (False, True):
        ctx.set_transpose(tr)
        both(ctx, f"problems_cgl_complex_jvp_tr{int(tr)}", lambda v: ctx.jvp(v, a0=0.7, a1=-1.3), rng.standard_normal(ctx.N))
    ctx.close()

    M = 10
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (16, 12, M), (np.pi, np.pi / 2), krylov_m=4, params=(1.3,) + CGL_PAR[1:])
    n = ctx.N - 1
    x = 0.1 * rng.standard_normal(ctx.N)
    x[-1] = 6.3
    ctx.potrap_set_section(rng.standard_normal(n) / np.sqrt(ctx.N), x[:-1])
    res_jvp(ctx, "problems_potrap", x)  # the JVP reads the F-cache filled by bk_jac_set_state
    ctx.set_transpose(True)
    both(ctx, "problems_potrap_jvp_tr", lambda v: ctx.jvp(v, a0=0.7, a1=-1.3), rng.standard_normal(ctx.N))
    ctx.set_transpose(False)
    J = ctx.jacobian(x)
    a, b = rng.standard_normal(ctx.N), rng.standard_normal(ctx.N)
    dump("problems_potrap_bls1", bk.bls_map(J, a, b, 0.8, rng.standard_normal(ctx.N + 1), shift=-0.5, dotscale=1.0 / ctx.N))
    ab = (rng.standard_normal(ctx.N), rng.standard_normal(ctx.N))
    dump("problems_potrap_bls2", bk.bls_map_block(J, ab, (a, b), [[0.9, 0.1], [-0.2, 1.1]], rng.standard_normal(ctx.N + 2),
                                                  shift=-0.5, dotscale=1.0 / ctx.N))
    counters(ctx, "problems_potrap_bls", dump)
    for scale in (1.0 / M, 1.0):
        for tag, xs in (("host", x), ("dev", ctx.to_device(x))):
            ctx.potrap_update_section(xs, scale)
            dump(f"problems_potrap_section_{scale:.2f}_{tag}", ctx.residual(x))
            counters(ctx, f"problems_potrap_section_{scale:.2f}_{tag}", dump)
    ctx.close()

    ctx = bk.Context(bk.BK_CHAN, (5000,), (1.0,), krylov_m=4, params=(3.3, 0.01))
    u = rng.standard_normal(ctx.N0)
    for nroots in (1, 5, 64, 70):
        roots = [u + 0.1 * rng.standard_normal(ctx.N0) for _ in range(nroots)]
        for ndir in (0, 1, 2):
            dirs = [rng.standard_normal(ctx.N0) for _ in range(ndir)]
            for n in (ctx.N0, 3001):
                name = f"problems_defl_r{nroots}_d{ndir}_n{n}"
                dump(name + "_host", np.concatenate([np.ravel(a) for a in ctx.deflation_moments(u, roots, dirs, n)]))
                dev = ctx.deflation_moments(ctx.to_device(u), [ctx.to_device(r) for r in roots], [ctx.to_device(h) for h in dirs], n)
                dump(name + "_dev", np.concatenate([np.ravel(a) for a in dev]))
                counters(ctx, name, dump)
    ctx.close()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--out", required=True)
    ap.add_argument("--root", default=ROOT)
    ap.add_argument("--sh-dct-only", action="store_true", help=argparse.SUPPRESS)  # the BK_FFT_NO_FAST child
    a = ap.parse_args()
    bk = load(os.path.abspath(a.root))
    if a.sh_dct_only:
        sh_dct(bk, Dump(a.out, "nofast_"))
        return
    sh_dct(bk, Dump(a.out, ""))
    others(bk, Dump(a.out, ""))
    krylov(bk, Dump(a.out, ""))
    problem_kernels(bk, Dump(a.out, ""))
    env = dict(os.environ, BK_FFT_NO_FAST="1")  # read once per process by the library
    subprocess.run([sys.executable, os.path.abspath(__file__), "--out", a.out, "--root", a.root, "--sh-dct-only"], env=env, check=True)
    print(f"{len(os.listdir(a.out))} files in {a.out}")


if __name__ == "__main__":
    main()
