"""Cost of the folds of periodic orbits of cGL2d (periodic.newton_fold_po), in the same run:
  - J and J' of the Trapeze functional per application (bk_jvp with the transpose off / on), from CUDA events on the library's
    stream over 200 launches that rotate through 4 input and 4 output device vectors, at 41 x 21 x 30 (examples/cGL2d.jl) and at
    512^2 x 30, with their algorithmic bytes: both read the input, the state, the F cache and the section and write the output,
    40 N bytes (J reads the input twice, in its slice kernel and in its phase kernel; J' reads it once);
  - GMRES iterations of J' x = b preconditioned on the right with P'^-1 (what the library applies while J' is selected) against
    the un-transposed P^-1, at the fold orbit of 41 x 21 x 30: the oracle's GMRES (oracle/krylov.py) over the device operator and
    the device preconditioner, the only difference being the preconditioner;
  - the wall time of newton_fold_po at 41 x 21 x 30 from the fold recorded on the branch switched from the Hopf point, between
    two device synchronises;
  - the card's name and power limit.
Prints one JSON object.  Usage: python tools/po_fold_cost.py"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import __graft_entry__ as g  # noqa: E402
from oracle import krylov, problems  # noqa: E402

bk = g.load_package()
P = bk.palc
L = (np.pi, np.pi / 2)
M = 30
PARS = (1.3, 0.1, 1.0, -1.0, 1.0)


def orbit_like(gl, T, seed=0):
    """M slices of a rotating first Dirichlet mode with noise, and the period T"""
    rng = np.random.default_rng(seed)
    ph = gl.phi11()
    t = np.linspace(0, 2 * np.pi, M + 1)[:M]
    return np.concatenate([np.concatenate([0.8 * np.cos(s) * ph, 0.8 * np.sin(s) * ph]) + 0.05 * rng.standard_normal(gl.N) for s in t]
                          + [np.array([T])])


def per_application(nx, ny, reps=200, nbuf=4):
    gl = problems.GinzburgLandau2D(nx, ny, *L, r=PARS[0], mu=PARS[1], nu=PARS[2], c3=PARS[3], c5=PARS[4])
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (nx, ny, M), L, krylov_m=4, params=PARS)
    x = orbit_like(gl, 6.3)
    ctx.potrap_update_section(ctx.to_device(x), 1.0 / M)
    ctx.jacobian(ctx.to_device(x))
    rng = np.random.default_rng(1)
    ins = [ctx.to_device(rng.standard_normal(ctx.N)) for _ in range(nbuf)]
    outs = [ctx.zeros() for _ in range(nbuf)]
    stream = torch.cuda.ExternalStream(ctx.lib.bk_stream(ctx.handle))
    res = {}
    for name, tr in (("J", False), ("Jt", True)):
        ctx.set_transpose(tr)
        for k in range(20):
            ctx.jvp(ins[k % nbuf], outs[k % nbuf])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for k in range(reps):
            ctx.jvp(ins[k % nbuf], outs[(k + 1) % nbuf])
        e1.record(stream)
        e1.synchronize()
        res[name + "_us"] = e0.elapsed_time(e1) * 1e3 / reps
    ctx.set_transpose(False)
    nbytes = 40 * ctx.N
    res.update(grid=f"{nx}x{ny}x{M}", N=ctx.N, algorithmic_bytes=nbytes,
               J_GBps=nbytes / (res["J_us"] * 1e-6) / 1e9, Jt_GBps=nbytes / (res["Jt_us"] * 1e-6) / 1e9,
               launches_per_application=dict(J=2, Jt=1))
    return res


def fold_cost(nx=41, ny=21):
    gl0 = problems.GinzburgLandau2D(nx, ny, *L)
    r_hopf = gl0.r_hopf()
    pars = [r_hopf, 0.1, 1.0, -1.0, 1.0]
    ctx_vf = bk.Context(bk.BK_CGL2D, (nx, ny), L, krylov_m=200, params=pars)
    prob = P.BifurcationProblemB200(ctx_vf, ctx_vf.zeros(), pars, lens=0)
    ph = gl0.phi11() / np.linalg.norm(gl0.phi11())
    zeta = np.concatenate([ph, -1j * ph]) / np.sqrt(2)
    hp = bk.normalform.hopf_normal_form_at(prob, ctx_vf.zeros(), r_hopf, 1.0, zeta, zeta,
                                           bk.GMRESB200(reltol=1e-12, restart=200, maxiter=2000, orth="cgs2"))
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (nx, ny, M), L, krylov_m=60, params=pars)
    trap = bk.periodic.TrapezeProblemB200(ctx, None, list(pars), lens=0, circulant=True)
    ls = bk.GMRESB200(reltol=1e-10, restart=60, maxiter=600, Pr=True, orth="cgs2")
    cp = P.ContinuationPar(dsmin=1e-4, dsmax=0.05, ds=0.01, p_min=r_hopf - 3.0, p_max=r_hopf + 1.0, max_steps=80,
                           newton_options=P.NewtonPar(tol=1e-9, max_iterations=15, linsolver=ls))
    br, _, _, _ = bk.periodic.continuation_from_hopf_point(hp, cp, trap, with_events=True)
    ind = next(i for i, s in enumerate(br.specialpoint) if s.type == "fold" and s.param < r_hopf - 0.05)
    opts = P.NewtonPar(tol=1e-8, max_iterations=15, linsolver=ls)
    bls = bk.BorderingBLSB200(ls, check_precision=False)
    ctx.sync()
    t = time.perf_counter()
    sol = bk.periodic.newton_fold_po(trap, br, ind, opts, bls)
    ctx.sync()
    wall = time.perf_counter() - t
    # J' x = b at the fold orbit: P'^-1 against P^-1, the same oracle GMRES over the device operator
    x = sol.u
    trap._set(sol.p)
    trap.setup_precond(x)
    Jt = trap.Jt(x, sol.p)
    b = np.random.default_rng(2).standard_normal(ctx.N)

    def pc(transpose):
        def apply(v):
            ctx.set_transpose(transpose)
            try:
                return ctx.precond_apply(np.ascontiguousarray(v))
            finally:
                ctx.set_transpose(False)
        return apply
    iters = {}
    for name, tr in (("Pt", True), ("P", False)):
        _, cv, it = krylov.GMRESIterativeSolvers(reltol=1e-10, restart=60, maxiter=1200, Pr=pc(tr), orth="cgs2")(
            lambda v: Jt(np.ascontiguousarray(v)), b)
        iters[name] = dict(iterations=int(np.sum(it)), converged=bool(cv))
    _, cvd, itd = ls(Jt, b)
    return dict(grid=f"{nx}x{ny}x{M}", N=ctx.N, branch_rows=len(br.rows), fold_guess_param=br.specialpoint[ind].param,
                newton_fold_po=dict(wall_s=wall, converged=sol.converged, p=sol.p, itnewton=sol.itnewton, itlinear=sol.itlinear,
                                    residuals=sol.residuals),
                adjoint_gmres_reltol_1e10=dict(oracle_gmres=iters, device_gmres_with_Pt=dict(iterations=int(itd), converged=bool(cvd))))


if __name__ == "__main__":
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out = dict(card=smi, per_application=[per_application(41, 21), per_application(512, 512)], fold=fold_cost())
    print(json.dumps(out, indent=1))
