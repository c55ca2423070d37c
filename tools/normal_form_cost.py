"""Cost of the simple-branch-point normal form on the device: SH2d 1024^2 (Neumann FD, lengths (2.3 pi, 1.7 pi), nu = 1.3) at the
closed-form branch point of its trivial state, l* = (1 + lambda_x + lambda_y)^2 of the first DCT mode to cross.
  - wall time of normalform.get_normal_form1d, split into the eigen-solve, the two bordered solves and the rest (jets, the
    central differences in the parameter and the vector algebra), each part ended by a device synchronise;
  - bk_d2f / bk_d3f kernel time from CUDA events over many launches on device vectors, and the kernel alone from torch.profiler,
    with the algorithmic bytes of include/bk200.h (32 N for d2F and SH d3F) as GB/s;
  - the card's name and power limit, read in the same run.
Prints one JSON object."""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import __graft_entry__ as g  # noqa: E402

bk = g.load_package()
P, E, NF = bk.palc, bk.events, bk.normalform
n = int(sys.argv[1]) if len(sys.argv) > 1 else 1024
dims, lengths, nu = (n, n), (2.3 * np.pi, 1.7 * np.pi), 1.3


def crossing():
    lam = [-(2 - 2 * np.cos(np.pi * np.arange(m) / m)) / (2 * L / m) ** 2 for m, L in zip(dims, lengths)]
    return float(np.min((1 + np.add.outer(lam[0], lam[1])) ** 2))


class Timed:
    """wraps a solver: accumulated wall time of its calls, each ended by a device synchronise"""

    def __init__(self, ctx, fn):
        self.ctx, self.fn, self.s = ctx, fn, 0.0

    def __call__(self, *a, **k):
        t = time.perf_counter()
        out = self.fn(*a, **k)
        self.ctx.sync()
        self.s += time.perf_counter() - t
        return out


lstar = crossing()
ctx = bk.Context(bk.BK_SH2D, dims, lengths, krylov_m=100, params=(lstar, nu))
ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
ls = bk.GMRESB200(reltol=1e-10, restart=100, maxiter=300, Pl=True, orth="cgs2")
eig = bk.ShiftInvertB200(0.05, ls, krylovdim=40, tol=1e-10, maxrestart=30)
prob = P.BifurcationProblemB200(ctx, ctx.zeros(), (lstar, nu), lens=0)
# the branch point as events.continuation records it on the trivial branch: state 0, the eigenvalues there, ind_ev = 1
vals, _, _, _ = eig(prob.J(prob.u0, lstar), 4)
br = E.Branch(specialpoint=[E.SpecialPoint(type="bp", idx=0, param=lstar, norm=0.0, step=0, status="converged", delta=(1, 0), ind_ev=1,
                                           interval=(lstar, lstar), x=prob.u0, tau_p=1.0, tau_u=ctx.zeros().zero_())],
              eig=[dict(eigenvals=vals, step=0)])
teig, tbls = Timed(ctx, lambda J, nev: eig(J, nev, want_vectors=True)), Timed(ctx, bk.MatrixFreeBLSB200(ls))
cp = P.ContinuationPar(newton_options=P.NewtonPar(tol=1e-10, linsolver=ls, eigsolver=teig), nev=4)
it = P.ContIterable(prob, P.PALC(bls=tbls), cp, P.norminf)
NF.get_normal_form1d(it, br, 0, bls=tbls)           # warm-up: modules, shared-memory grants, pools
teig.s = tbls.s = 0.0
ctx.sync()
t0 = time.perf_counter()
bp = NF.get_normal_form1d(it, br, 0, bls=tbls)
ctx.sync()
total = time.perf_counter() - t0

N = ctx.N
rng = np.random.default_rng(0)
# four sets of (u, a, b, c, out), 160 MB in all, used in turn: each launch reads what the previous ones evicted from the 50 MB L2
sets = [[ctx.to_device(rng.standard_normal(N)) for _ in range(5)] for _ in range(4)]
turn = [0]


def nxt():
    turn[0] = (turn[0] + 1) % len(sets)
    return sets[turn[0]]
stream = torch.cuda.ExternalStream(ctx.lib.bk_stream(ctx.handle))


def ev_ms(fn, reps=200, warm=10):
    for _ in range(warm):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ctx.sync()
    e0.record(stream)
    for _ in range(reps):
        fn()
    e1.record(stream)
    ctx.sync()
    return e0.elapsed_time(e1) / reps


d2 = lambda: (lambda u, a, b, c, out: ctx.d2f(u, a, b, out))(*nxt())
d3 = lambda: (lambda u, a, b, c, out: ctx.d3f(u, a, b, c, out))(*nxt())
ms2, ms3 = ev_ms(d2), ev_ms(d3)
from torch.profiler import profile, ProfilerActivity  # noqa: E402
with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
    for _ in range(100):
        d2()
        d3()
    ctx.sync()
kern = {}
for e in prof.events():
    if "k_jet" in e.name:
        key = "d2f" if ("ILi2E" in e.name or "k_jet<2>" in e.name) else "d3f"
        kern.setdefault(key, []).append(e.device_time if hasattr(e, "device_time") else e.cuda_time)
kern_us = {k: float(np.median(v)) for k, v in kern.items()}
smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
bytes_ = 32 * N
print(json.dumps({
    "card": smi, "grid": f"{n}x{n}", "N": N, "l_star": lstar, "type": bp.type,
    "b11": bp.nf["b11"], "b20": bp.nf["b20"], "b30": bp.nf["b30"],
    "normal_form_s": total, "eigen_solve_s": teig.s, "bordered_solves_s": tbls.s, "jets_and_differences_s": total - teig.s - tbls.s,
    "d2f_event_us": ms2 * 1e3, "d3f_event_us": ms3 * 1e3,
    "d2f_event_GBps": bytes_ / (ms2 * 1e-3) / 1e9, "d3f_event_GBps": bytes_ / (ms3 * 1e-3) / 1e9,
    "d2f_kernel_us": kern_us.get("d2f"), "d3f_kernel_us": kern_us.get("d3f"),
    "d2f_kernel_GBps": bytes_ / (kern_us["d2f"] * 1e-6) / 1e9 if "d2f" in kern_us else None,
    "d3f_kernel_GBps": bytes_ / (kern_us["d3f"] * 1e-6) / 1e9 if "d3f" in kern_us else None,
}), flush=True)
