"""Cost of the deflation scalars on the device at the bench's size: SH2d 1024^2 on the bench's domain (bench.domain), u the
localized front guess of examples/SH2d-fronts.jl:75 on sol0, and n in {1, 8, 40} roots taken as u plus 0.01 rand (seeded).

  - One M(u) plus two dM(u).h (what DeflatedProblemCustomLS needs per Newton iteration), fused (one bk_deflation_moments call
    with both directions) against composed (the copy + axpby + dot loop per root, and the forward differences through it), in
    alternating rounds timed with CUDA events on the context's stream.  Algorithmic bytes from the shapes: the fused pass reads
    u, h1, h2 and every root once, 8 N (n + 3); the composed path moves 56 N per root and M, 40 N more per dM, 280 N n + 80 N.
    Launches are the library's own count.
  - The kernel pair alone: torch.profiler (CUDA activities) over 20 fused calls, the mean device time of k_deflation_moments and of
    k_deflation_moments_fold per call, and the main kernel's algorithmic bytes over its own time against the data sheet's
    3.35 TB/s.
  - One deflated Newton iteration (newton_deflated, one step of GMRES(100) reltol 1e-5 with the DCT preconditioner, as the
    bench), both ways, with the time spent in the deflation operator (each call ended by a device synchronise) and its share.

The card's name and power limit are read in the same run.  Prints one JSON object."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import __graft_entry__ as g  # noqa: E402
import bench  # noqa: E402
from oracle import problems  # noqa: E402

bk = g.load_package()
P, D = bk.palc, bk.deflation


class DeflationClock:
    """wall time inside the outermost DeflationOperator calls, each ended by a device synchronise"""

    def __init__(self, ctx):
        self.ctx, self.s, self.depth, self.on = ctx, 0.0, 0, False
        for name in ("__call__", "dM", "values"):
            setattr(D.DeflationOperator, name, self.wrap(getattr(D.DeflationOperator, name)))

    def wrap(self, fn):
        def timed(*a, **k):
            if self.depth or not self.on:
                return fn(*a, **k)
            self.depth += 1
            t = time.perf_counter()
            try:
                return fn(*a, **k)
            finally:
                self.ctx.sync()
                self.s += time.perf_counter() - t
                self.depth -= 1
        return timed


def kernel_times(fn, calls=20):
    """mean device time per call of the two deflation-moment kernels, from torch.profiler's CUDA activities"""
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            fn()
        torch.cuda.synchronize()
    out = {"main_us": 0.0, "fold_us": 0.0, "calls": calls}
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        t = e.cuda_time_total if t is None else t
        if "k_deflation_moments_fold" in e.key:
            out["fold_us"] += t / calls
        elif "k_deflation_moments" in e.key:
            out["main_us"] += t / calls
    return out


def main(rounds=7):
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    n = 1024
    L = bench.domain(n)
    ctx = bk.Context(bk.BK_SH2D, (n, n), L, krylov_m=bench.GMRES["restart"], params=bench.PAR)
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(N=n * n, Pr=True, **bench.GMRES)
    N = ctx.N
    rng = np.random.default_rng(0)
    u0 = problems.sh2d_front_guess(problems.sh2d_sol0(n, n, *L), n, n, *L)
    u = ctx.to_device(u0)
    h = [ctx.to_device(rng.standard_normal(N)) for _ in range(2)]
    allroots = [ctx.to_device(u0 + 0.01 * rng.random(N)) for _ in range(40)]
    prob = P.BifurcationProblemB200(ctx, u, bench.PAR, lens=0)
    stream = torch.cuda.ExternalStream(ctx.lib.bk_stream(ctx.handle))
    clock = DeflationClock(ctx)
    cases = []
    for nr in (1, 8, 40):
        roots = allroots[:nr]
        ops = {"fused": D.DeflationOperator(2, 1.0, roots, fused=True), "composed": D.DeflationOperator(2, 1.0, roots)}
        run = {"fused": lambda: ops["fused"].values(u, h),
               "composed": lambda: (ops["composed"](u), ops["composed"].dM(u, h[0]), ops["composed"].dM(u, h[1]))}
        vals = {k: f() for k, f in run.items()}          # warm-up, and the values of both
        times = {k: [] for k in run}
        launches = {}
        for r in range(rounds):
            for k in ("fused", "composed"):
                l0 = ctx.stats()["kernel_launches"]
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record(stream)
                run[k]()
                b.record(stream)
                b.synchronize()
                times[k].append(a.elapsed_time(b) * 1e3)
                launches[k] = ctx.stats()["kernel_launches"] - l0
        med = {k: float(np.median(v)) for k, v in times.items()}
        by = {"fused": 8 * N * (nr + 3), "composed": 280 * N * nr + 80 * N}
        kern = kernel_times(lambda: run["fused"]())
        kern["GBps"] = by["fused"] / kern["main_us"] / 1e3
        kern["share_of_3350_GBps"] = kern["GBps"] / 3350.0
        Mf, dMf = vals["fused"]
        Mc, dM1, dM2 = vals["composed"]
        # one deflated Newton iteration each way
        newton = {}
        for k in ("fused", "composed"):
            opts = P.NewtonPar(tol=0.0, max_iterations=1, linsolver=ls)
            D.newton_deflated(prob, u, bench.PAR[0], ops[k], opts, P.norminf)        # warm-up
            clock.s, clock.on = 0.0, True
            t = time.perf_counter()
            D.newton_deflated(prob, u, bench.PAR[0], ops[k], opts, P.norminf)
            ctx.sync()
            tot = time.perf_counter() - t
            clock.on = False
            newton[k] = dict(iteration_ms=tot * 1e3, deflation_ms=clock.s * 1e3, deflation_share=clock.s / tot)
        cases.append(dict(nroots=nr, rounds=rounds, us_median={k: med[k] for k in med},
                          us_min={k: float(np.min(v)) for k, v in times.items()}, launches=launches, bytes=by,
                          GBps={k: by[k] / med[k] / 1e3 for k in med}, speedup=med["composed"] / med["fused"],
                          M_rel_diff=abs(Mf - Mc) / abs(Mc),
                          dM_rel_diff=max(abs(dMf[0] - dM1) / abs(dM1), abs(dMf[1] - dM2) / abs(dM2)),
                          kernel=kern, newton=newton))
    print(json.dumps(dict(gpu=gpu, N=N, dims=[n, n], lengths=list(L), cases=cases)))


if __name__ == "__main__":
    main()
