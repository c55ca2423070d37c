"""GPU check, a candidate for a GPU test: deflation.py with device vectors.  Same case as
tests/test_host_logic_cpu.py::test_deflated_newton_finds_the_three_chan_solutions (Chan problem, alpha = 3.3, three solutions
with max u = 0.77197, 5.97988, 12.85103), linear solves = GMRESB200 with Pl = lu(P) (examples/chan.jl:108-111), two-rhs call."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as g
bk = g.load_package(); P, D = bk.palc, bk.deflation
n = 101
ctx = bk.Context(bk.BK_CHAN, (n,), (1.0,), krylov_m=n, params=(3.3, 0.01))
ctx.precond_setup(bk.BK_PC_CHAN_TRIDIAG)
ls = bk.GMRESB200(reltol=1e-10, restart=n, maxiter=n, Pl=True, orth="cgs2")
i = np.arange(1, n + 1)
sol0 = (i - 1) * (n - i) / n**2 + 0.1
prob = P.BifurcationProblemB200(ctx, ctx.to_device(sol0), (3.3, 0.01), lens=0)
opts = P.NewtonPar(tol=1e-9, max_iterations=100, linsolver=ls)
s0 = P.newton(prob, prob.u0, 3.3, opts, P.norminf)
op = D.DeflationOperator(2, 1.0, [s0.u])
g1 = s0.u.copy(); g1.scale_(4.0)
s1 = D.newton_deflated(prob, g1, 3.3, op, opts, P.norminf)
op.push(s1.u)
g2 = s0.u.copy(); g2.scale_(8.0)
s2 = D.newton_deflated(prob, g2, 3.3, op, opts, P.norminf)
tops = sorted(float(np.max(s.u.numpy())) for s in (s0, s1, s2))
print(tops, [s.converged for s in (s0, s1, s2)], [s.itnewton for s in (s0, s1, s2)])
assert np.allclose(tops, [0.77197, 5.97988, 12.85103], atol=1e-4)
print("DEFLATION GPU CHECK OK")
