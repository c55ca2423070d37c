"""Launches every stand-alone kernel of the path once or twice at BASELINE.json's config sizes, for one `ncu --set full` row per kernel:
K1/K2 stencils of the four problems, BLAS-1 / reductions, the general transform kernel."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import __graft_entry__ as g
import bench
bk = g.load_package()
rng = np.random.default_rng(0)
# SH2d 1024^2: k2_apply<8,0/1>, k_reduce<0,1,2>, k_axpby, k_scale
n = 1024
c = bk.Context(bk.BK_SH2D, (n, n), bench.domain(n), krylov_m=8, params=bench.PAR)
u = c.to_device(bench.sol0(n)); v = c.to_device(rng.standard_normal(c.N)); out = c.zeros()
for _ in range(2):
    c.residual(u, out); J = c.jacobian(u); c.jvp(v, out)
    v.dot(u); v.norminf(); v.diffdot(u, out); out.axpby_(0.5, v, 1.0); out.scale_(0.9)
x, ok, it = bk.GMRESB200(reltol=1e-30, restart=6, maxiter=6)(J, v)   # k_lincomb at the end of the cycle
c.sync(); del c
# SH3d 128^3: k_sh_apply<3,*>
c = bk.Context(bk.BK_SH3D, (128, 128, 128), (np.pi * 128 / 22,) * 3, krylov_m=4, params=(0.1, 1.2))
u = c.to_device(rng.standard_normal(c.N) * 0.1); v = c.to_device(rng.standard_normal(c.N)); out = c.zeros()
for _ in range(2):
    c.residual(u, out); c.jacobian(u); c.jvp(v, out)
c.sync(); del c
# cGL 512^2: k_cgl_apply + the general transform kernel (DST-I, L = 1026)
c = bk.Context(bk.BK_CGL2D, (512, 512), (np.pi, np.pi / 2), krylov_m=4, params=(1.2, 0.1, 1.0, -1.0, 1.0))
u = c.to_device(rng.standard_normal(c.N) * 0.1); v = c.to_device(rng.standard_normal(c.N)); out = c.zeros()
c.precond_setup(bk.BK_PC_CGL_DST, 1.0, -0.05)
for _ in range(2):
    c.residual(u, out); c.jacobian(u); c.jvp(v, out); c.precond_apply(v, out)
c.sync(); del c
# Trapeze 512^2 x 30: k_potrap_apply, k_potrap_section (the F-cache), k_potrap_phase
M = 30
c = bk.Context(bk.BK_POTRAP_CGL2D, (512, 512, M), (np.pi, np.pi / 2), krylov_m=4, params=(1.2, 0.1, 1.0, -1.0, 1.0))
x = c.to_device(np.concatenate([rng.standard_normal(c.N - 1) * 0.1, [6.3]])); v = c.to_device(rng.standard_normal(c.N)); out = c.zeros()
phi = np.zeros(c.N - 1); phi[:100] = 0.1
c.potrap_set_section(phi, np.zeros(c.N - 1))
for _ in range(2):
    c.residual(x, out); c.jacobian(x); c.jvp(v, out)
c.sync()
print("kernel tour done")
