"""GPU check, a candidate for tests/test_gpu_palc.py: events.py (detect_bifurcation = 3) with device vectors.
cGL2d trivial branch u = 0 continued in r: eigenvalues r + lambda_k(Lap) +- i nu, so the first Hopf point is analytic,
r_hopf = -lambda_1 (examples/cGL2d.jl:120-135 finds it at r ~ 1.14 on 41 x 21).  Expected: one special point of type hopf,
delta = (2, 2), |param - r_hopf| below the bisection interval."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as g
from oracle import problems
bk = g.load_package(); P, E = bk.palc, bk.events
dims = (41, 21); L = (np.pi, np.pi / 2)
gl = problems.GinzburgLandau2D(*dims, *L)
r_hopf = gl.r_hopf()
ctx = bk.Context(bk.BK_CGL2D, dims, L, krylov_m=120, params=(r_hopf - 0.3, 0.1, 1.0, -1.0, 1.0))
inner = bk.GMRESB200(reltol=1e-10, restart=120, maxiter=600, orth="cgs2")
eig = bk.ShiftInvertB200(0.5, inner, krylovdim=40, tol=1e-8, maxrestart=30)
ls = bk.GMRESB200(reltol=1e-10, restart=120, maxiter=240)
nopts = P.NewtonPar(tol=1e-9, max_iterations=10, linsolver=ls, eigsolver=eig)
cp = P.ContinuationPar(dsmin=1e-4, dsmax=0.05, ds=0.01, p_min=r_hopf - 0.5, p_max=r_hopf + 0.3, max_steps=60, newton_options=nopts,
                       detect_bifurcation=3, n_inversion=6, nev=4, tol_stability=1e-8)
prob = P.BifurcationProblemB200(ctx, ctx.zeros(), (r_hopf - 0.3, 0.1, 1.0, -1.0, 1.0), lens=0, record=lambda v: v.norminf())
br = E.continuation(prob, P.PALC(bls=bk.MatrixFreeBLSB200(ls)), cp, normC=P.norminf, verbose=True)
pts = [(bp.type, bp.param, bp.delta, bp.status, bp.interval) for bp in br.specialpoint]
print(pts, "r_hopf", r_hopf)
h = [bp for bp in br.specialpoint if bp.type == "hopf"]
assert len(h) >= 1 and abs(h[0].param - r_hopf) < 1e-3 and tuple(map(abs, h[0].delta)) == (2, 2), pts
print("EVENTS GPU CHECK OK")
