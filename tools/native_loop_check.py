#!/usr/bin/env python
"""bk_palc_run (all-native PALC loop) vs the plugin-surface loop (palc.continuation) on one context: are the branches
bit-identical, and what does the host-language dispatch between the kernels cost?  Wall clock around each loop with a
stream synchronise on both sides (this compares two HOST loops over the same kernels; it is not a bench.py number).

  python tools/native_loop_check.py [--grid 1024] [--steps 30] [--out native_loop_check.json]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402
import bench as B  # noqa: E402  (workload definition only: domain, start vectors, solver settings)


def run(n, steps):
    bk = g.load_package()
    P = bk.palc
    t0 = time.perf_counter()
    ctx, ls, u_front = B.gpu_setup(bk, n, 0)
    setup_s = time.perf_counter() - t0
    cp = P.ContinuationPar(max_steps=steps, newton_options=P.NewtonPar(tol=1e-9, max_iterations=15, linsolver=ls), **B.CONT)
    alg = P.PALC(bls=bk.MatrixFreeBLSB200(ls))
    mk = lambda: P.BifurcationProblemB200(ctx, u_front, list(B.PAR), lens=0)
    out = {"grid": n, "steps": steps, "setup_s": round(setup_s, 2)}
    P.continuation(mk(), alg, P.ContinuationPar(max_steps=3, newton_options=cp.newton_options, **B.CONT), normC=P.norminf)  # warm-up
    res = {}
    for name, fn in (("plugin_loop", lambda: P.continuation(mk(), alg, cp, normC=P.norminf)),
                     ("native_loop", lambda: P.continuation_native(mk(), alg, cp, normC=P.norminf)),
                     ("plugin_loop_again", lambda: P.continuation(mk(), alg, cp, normC=P.norminf)),
                     ("native_loop_again", lambda: P.continuation_native(mk(), alg, cp, normC=P.norminf))):
        ctx.sync()
        s0 = ctx.stats()
        t0 = time.perf_counter()
        rows, info = fn()
        ctx.sync()
        dt = time.perf_counter() - t0
        s1 = ctx.stats()
        res[name] = rows
        out[name] = {"seconds": dt, "rows": len(rows), "steps_per_s": (len(rows) - 1) / dt,
                     "kernel_launches": s1["kernel_launches"] - s0["kernel_launches"],
                     "itlinear": int(sum(r["itlinear"] for r in rows)), "itnewton": int(sum(r["itnewton"] for r in rows))}
    keys = ("param", "x", "itnewton", "itlinear", "ds", "step")
    a, b = res["plugin_loop"], res["native_loop"]
    out["rows_equal_length"] = len(a) == len(b)
    out["max_abs_row_difference"] = float(max(abs(r[k] - o[k]) for r, o in zip(a, b) for k in keys)) if a and b else None
    out["bit_identical"] = bool(len(a) == len(b) and all(r[k] == o[k] for r, o in zip(a, b) for k in keys))
    out["plugin_loop_repeatable"] = bool(all(r[k] == o[k] for r, o in zip(a, res["plugin_loop_again"]) for k in keys))
    out["native_loop_repeatable"] = bool(all(r[k] == o[k] for r, o in zip(b, res["native_loop_again"]) for k in keys))
    out["last_row"] = {k: float(b[-1][k]) for k in keys}
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--grid", type=int, nargs="+", default=[1024])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--out", default="native_loop_check.json")
    args = ap.parse_args()
    os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
    outs = []
    for n in args.grid:
        outs.append(run(n, args.steps))
        print(json.dumps(outs[-1]), flush=True)
        with open(args.out, "w") as f:
            json.dump(outs, f, indent=1)
