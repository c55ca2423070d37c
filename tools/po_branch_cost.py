"""Cost of a periodic-orbit branch switched from the first Hopf point of cGL2d (periodic.continuation_from_hopf_point), at the
grid of examples/cGL2d.jl (41 x 21, M = 30) and at 512^2 x 30 (config 4 of BASELINE.json):
  - wall time per continuation step (the time between two converged steps, each read after a device synchronise), with the
    Newton and GMRES iterations of each step, and the share of that time spent in the Floquet eigen-solve
    (FloquetEigB200, contpar.detect_bifurcation = 1);
  - bk_potrap_update_section per call from CUDA events on the library's stream over 200 calls on a device orbit, with its
    algorithmic bytes (read x, write phi and xpi, then read both for <phi, xpi>: 40 (N - 1));
  - the card's name and power limit, read in the same run.
The Hopf normal form is computed at the analytic Hopf point r = -lambda_1 of the trivial state with ζ = ζ★ = (φ, -iφ) / (√2 |φ|).
Prints one JSON object.  Usage: python tools/po_branch_cost.py [steps_small] [steps_large]"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import __graft_entry__ as g  # noqa: E402
from oracle import problems  # noqa: E402

bk = g.load_package()
P = bk.palc
L = (np.pi, np.pi / 2)
M = 30


class TimedFloquet:
    """a FloquetQaDB200 whose calls are timed, each between two device synchronises (FloquetEigB200 reads .ctx and calls it)"""

    def __init__(self, fl, ctx_po):
        self.fl, self.ctx, self.ctx_po, self.seconds = fl, fl.ctx, ctx_po, 0.0

    def __call__(self, x, nev):
        self.ctx_po.sync()
        t = time.perf_counter()
        out = self.fl(x, nev)
        self.ctx.sync()
        self.seconds += time.perf_counter() - t
        return out


def branch(nx, ny, steps, reltol, newton_tol):
    gl0 = problems.GinzburgLandau2D(nx, ny, *L)
    r_hopf = gl0.r_hopf()
    pars = [r_hopf, 0.1, 1.0, -1.0, 1.0]
    ctx_vf = bk.Context(bk.BK_CGL2D, (nx, ny), L, krylov_m=40, params=pars)
    prob = P.BifurcationProblemB200(ctx_vf, ctx_vf.zeros(), pars, lens=0)
    ph = gl0.phi11() / np.linalg.norm(gl0.phi11())
    zeta = np.concatenate([ph, -1j * ph]) / np.sqrt(2)
    ls_vf = bk.GMRESB200(reltol=1e-10, restart=40, maxiter=400, orth="cgs2")
    hp = bk.normalform.hopf_normal_form_at(prob, ctx_vf.zeros(), r_hopf, 1.0, zeta, zeta, ls_vf)
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (nx, ny, M), L, krylov_m=60, params=pars)
    trap = bk.periodic.TrapezeProblemB200(ctx, None, list(pars), lens=0, circulant=True)
    ls = bk.GMRESB200(reltol=reltol, restart=60, maxiter=300, Pr=True, orth="cgs2")
    cp = P.ContinuationPar(dsmin=1e-4, dsmax=0.03, ds=0.01, p_min=r_hopf - 1.0, p_max=r_hopf + 1.0, max_steps=steps, nev=2,
                           detect_bifurcation=1, tol_stability=1e-5,
                           newton_options=P.NewtonPar(tol=newton_tol, max_iterations=15, linsolver=ls))
    lsf = bk.GMRESB200(reltol=1e-8, restart=40, maxiter=80, Pr=True, orth="cgs2")
    fl = bk.floquet.FloquetQaDB200(ctx_vf, lsf, M, eigsolver=bk.floquet.ArnoldiLMB200(krylovdim=12, tol=1e-4, maxrestart=2))
    tfl = TimedFloquet(fl, ctx)
    marks = []

    def cb(st):
        ctx.sync()
        marks.append((time.perf_counter(), tfl.seconds))
    rows, st, _, pred = bk.periodic.continuation_from_hopf_point(hp, cp, trap, floquet=tfl, callback=cb)
    per_step = [dict(wall_s=marks[k][0] - marks[k - 1][0], floquet_s=marks[k][1] - marks[k - 1][1], itnewton=rows[k]["itnewton"],
                     itlinear=rows[k]["itlinear"], param=rows[k]["param"], period=rows[k]["x"]["period"],
                     n_unstable=rows[k]["n_unstable"]) for k in range(1, len(rows))]
    wall = sum(s["wall_s"] for s in per_step)
    flo = sum(s["floquet_s"] for s in per_step)
    # bk_potrap_update_section on the last orbit
    x = st.z_u
    stream = torch.cuda.ExternalStream(ctx.lib.bk_stream(ctx.handle))
    for _ in range(10):
        ctx.potrap_update_section(x, 1.0 / M)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 200
    e0.record(stream)
    for _ in range(reps):
        ctx.potrap_update_section(x, 1.0 / M)
    e1.record(stream)
    e1.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    nbytes = 40 * (ctx.N - 1)
    return dict(grid=f"{nx}x{ny}x{M}", N=ctx.N, steps=len(per_step), hopf_type=hp.type, predictor_p=pred.p,
                mean_step_s=wall / max(len(per_step), 1), floquet_share=flo / wall if wall > 0 else None,
                per_step=per_step, update_section_us=us, update_section_bytes=nbytes,
                update_section_GBps=nbytes / (us * 1e-6) / 1e9,
                note="update_section time is the whole call: the section kernel, the <phi, xpi> reduction and its download")


if __name__ == "__main__":
    small = int(sys.argv[1]) if len(sys.argv) > 1 else 10
    large = int(sys.argv[2]) if len(sys.argv) > 2 else 3
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    out = dict(card=smi, sizes=[branch(41, 21, small, 1e-6, 1e-8), branch(512, 512, large, 1e-4, 1e-6)])
    print(json.dumps(out, indent=1))
