"""What the BK_RD kind costs on the GPU, at 1024^2 with 2 fields (the cGL2d reaction written as RD terms, tests/rd_oracle.py):

* per-launch device time of the RD residual and JVP kernels (CUDA events on the context's stream around >= 200 launches on
  rotated device buffers) and their algorithmic bandwidth: residual 16 N bytes (read u, write F), JVP 24 N (read v and u, write
  the result), N = 2 Nx Ny counting both fields;
* microseconds per GMRES iteration of the same unpreconditioned solve (200 Arnoldi steps, restart 40) on the RD context and on a
  BK_CGL2D context of the same grid and parameters: what the generic kernel costs next to the hand-written one.

Prints one JSON line with the card's name and power limit, read in the same run.  Needs a GPU."""
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def launch_time(ctx, fn, bufs, reps):
    """mean device milliseconds per call of fn(buffer) over reps calls on rotated buffers, events on the context's stream"""
    import torch
    st = torch.cuda.ExternalStream(ctx.lib.bk_stream(ctx.handle))
    for b in bufs:
        fn(b)
    ctx.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for i in range(reps):
        fn(bufs[i % len(bufs)])
    e1.record(st)
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    import __graft_entry__ as g
    from tests import rd_oracle as RO
    bk = g.load_package()
    dims, L = (1024, 1024), (8.0, 8.0)
    pars = (0.7, 0.1, 1.0, -1.0, 1.0)
    rd = bk.Context(bk.BK_RD, dims, L, krylov_m=40, model=bk.ReactionDiffusion(**RO.cgl_model()), params=pars)
    cg = bk.Context(bk.BK_CGL2D, dims, L, krylov_m=40, params=pars)
    N = rd.N
    rng = np.random.default_rng(0)
    host = [0.5 * rng.standard_normal(N) for _ in range(4)]
    reps = 400
    out = {"card": card(), "dims": list(dims), "fields": 2, "N": N, "reps": reps}
    for name, ctx in (("rd", rd), ("cgl2d", cg)):
        bufs = [ctx.to_device(h) for h in host]
        outs = [ctx.zeros() for _ in host]
        ctx.jacobian(bufs[0])
        k = iter(range(1 << 30))
        res = lambda b: ctx.lib.bk_residual(ctx.handle, b.dptr, outs[next(k) % len(outs)].dptr)
        jvp = lambda b: ctx.lib.bk_jvp(ctx.handle, b.dptr, outs[next(k) % len(outs)].dptr, 0.3, 1.0)
        t_res, t_jvp = launch_time(ctx, res, bufs, reps), launch_time(ctx, jvp, bufs, reps)
        out[f"{name}_residual_us"] = round(1e3 * t_res, 2)
        out[f"{name}_residual_GBps"] = round(16 * N / (t_res * 1e-3) / 1e9, 1)
        out[f"{name}_jvp_us"] = round(1e3 * t_jvp, 2)
        out[f"{name}_jvp_GBps"] = round(24 * N / (t_jvp * 1e-3) / 1e9, 1)
        J = ctx.jacobian(bufs[0])
        ls = bk.GMRESB200(reltol=1e-30, restart=40, maxiter=200)
        rhs = bufs[1]
        ls(J, rhs, a0=1.0, a1=-0.01)   # warm-up
        ctx.sync()
        t0 = time.perf_counter()
        _, _, it = ls(J, rhs, a0=1.0, a1=-0.01)
        ctx.sync()
        out[f"{name}_gmres_iters"] = it
        out[f"{name}_gmres_us_per_iter"] = round(1e6 * (time.perf_counter() - t0) / it, 2)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
