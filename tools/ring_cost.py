"""Fixed cost per launch and streaming rate of the ring kernels k2_fused<E,true> + k2_update<E> on the bench path:
SH2d 1024^2, fp64, bordered (MatrixFreeBLSB200), DCT preconditioner on the right, fused JVP+Arnoldi, CGS,
reltol = 1e-30 so that a GMRES cycle runs exactly m Arnoldi steps.

  python tools/ring_cost.py [--out FILE]             # CUDA-event sweep m = 10, 20, ..., 100 + HBM copy peak
  python tools/ring_cost.py --profile [--out FILE]   # one torch.profiler run: per-kernel durations and launch gaps

Sweep: the library's event pairs around each ring kernel (Context.set_timing) give the pair's time T(m) of a cycle of m steps;
step k has j = k + 1 basis vectors, so T(m) = A m + B m (m + 1) / 2 with A = a_fused + a_update (fixed cost per launch pair)
and B = b_fused + b_update (cost per basis vector).  The two kernels each stream one 8N-byte vector per j, so 16 MB / B is the
pair's streaming rate at 1024^2.  Note that an event record between two launches serialises them (no PDL overlap): A
includes the launch latency that PDL hides inside GMRES.
Profile: the same cycle once at m = 100 under torch.profiler; each kernel's duration is fitted as a + b j, and the gaps
between consecutive kernels (start of one minus end of the previous, negative when PDL overlaps them) are summarised per
kernel pair.  Profile in its own invocation: tracing slows the host."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as g  # noqa: E402

N1 = 1024
PAR = (-0.1, 1.3)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits", "-i", "0"],
                       capture_output=True, text=True).stdout.strip().split(",")
    return {"name": torch.cuda.get_device_name(0), "power_limit_w": float(q[1]) if len(q) > 1 else None,
            "sm_max_mhz": float(q[2]) if len(q) > 2 else None}


def hbm_peak_gbs(nbytes=1 << 30, reps=20):
    """device-to-device copy of nbytes: (read + write) bytes over CUDA-event time, best of reps"""
    import torch
    a = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    b = torch.empty_like(a)
    for _ in range(3):
        b.copy_(a)
    best = float("inf")
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        b.copy_(a)
        e1.record()
        e1.synchronize()
        best = min(best, e0.elapsed_time(e1))
    return 2 * nbytes / (best * 1e-3) / 1e9


def setup(m_max=100):
    bk = g.load_package()
    s = N1 / 256.0
    lx, ly = 8 * np.pi * s, 4 * np.pi / np.sqrt(3) * s  # bench.py's domain at 1024^2
    ctx = bk.Context(bk.BK_SH2D, (N1, N1), (lx, ly), krylov_m=m_max, params=PAR)
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    X = -lx + 2 * lx / N1 * np.arange(N1)
    Y = -ly + 2 * ly / N1 * np.arange(N1)
    u = (np.cos(X)[None, :] + np.cos(X / 2)[None, :] * np.cos(np.sqrt(3) * Y / 2)[:, None]).reshape(-1)
    rng = np.random.default_rng(1234)
    N = N1 * N1
    J = ctx.jacobian(ctx.to_device(0.5 * u))
    vecs = [ctx.to_device(rng.standard_normal(N)) for _ in range(3)]
    return bk, ctx, J, vecs


def solve(bk, ctx, J, vecs, m):
    dR, dzu, R = vecs
    ls = bk.GMRESB200(reltol=1e-30, restart=m, maxiter=m, Pr=True)
    _, _, _, it = bk.MatrixFreeBLSB200(ls)(J, dR, dzu, 0.7, R, 0.3, 0.5, 0.5, dotscale=1.0 / (N1 * N1))
    ctx.sync()
    return it


def sweep(reps=5):
    bk, ctx, J, vecs = setup()
    ctx.set_timing(True)
    ms = list(range(10, 101, 10))
    for m in (10, 100):  # warm-up of every launch shape
        solve(bk, ctx, J, vecs, m)
    rows = []
    for m in ms:
        t, its = [], set()
        for _ in range(reps):
            its.add(solve(bk, ctx, J, vecs, m))
            t.append(ctx.stats()["last_fused_ms"])
        rows.append({"m": m, "iters": sorted(its), "pair_ms_median": float(np.median(t)), "pair_ms_all": t})
    Tm = np.array([r["pair_ms_median"] for r in rows]) * 1e3  # us
    M = np.array(ms, dtype=float)
    (A, B), res, *_ = np.linalg.lstsq(np.stack([M, M * (M + 1) / 2], 1), Tm, rcond=None)
    peak = hbm_peak_gbs()
    vec_bytes = 8 * N1 * N1
    return {"tool": "ring_cost sweep", "grid": f"{N1}x{N1}", "card": card(), "rows": rows,
            "fit": {"model": "T(m) = A m + B m (m+1)/2 [us], A = a_fused + a_update, B = b_fused + b_update",
                    "A_us_per_launch_pair": float(A), "B_us_per_basis_vector": float(B),
                    "rms_residual_us": float(np.sqrt(np.mean((np.stack([M, M * (M + 1) / 2], 1) @ [A, B] - Tm) ** 2))),
                    "streaming_GBps": 2 * vec_bytes / (B * 1e-6) / 1e9},
            "hbm_copy_peak_GBps": peak,
            "streaming_over_copy_peak": 2 * vec_bytes / (B * 1e-6) / 1e9 / peak}


def profile(m=100):
    import torch
    from torch.profiler import ProfilerActivity, profile as tprofile
    bk, ctx, J, vecs = setup()
    solve(bk, ctx, J, vecs, m)
    solve(bk, ctx, J, vecs, m)
    with tempfile.TemporaryDirectory() as td:
        with tprofile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            solve(bk, ctx, J, vecs, m)
            torch.cuda.synchronize()
        path = os.path.join(td, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))["traceEvents"]
    ks = sorted([e for e in ev if e.get("cat") == "kernel"], key=lambda e: e["ts"])
    short = lambda nm: nm.split("(")[0].replace("void ", "")
    fused = [k for k in ks if "k2_fused" in k["name"]]
    first = ks.index(fused[0])
    upd = [k for k in ks[first:] if "k2_update" in k["name"]]
    n = min(len(fused), len(upd))
    fused, upd = fused[:n], upd[:n]
    j = np.arange(1, n + 1, dtype=float)
    out = {"tool": "ring_cost profile", "grid": f"{N1}x{N1}", "m": m, "steps_seen": n, "card": card(), "kernels": {}}
    for name, lst in (("k2_fused", fused), ("k2_update", upd)):
        d = np.array([k["dur"] for k in lst], dtype=float)
        b, a = np.polyfit(j, d, 1)
        out["kernels"][name] = {"instance": short(lst[0]["name"]), "a_us": float(a), "b_us_per_j": float(b),
                                "streaming_GBps": 8 * N1 * N1 / (b * 1e-6) / 1e9, "dur_us_j1_10_50_100":
                                [float(d[k]) for k in (0, 9, 49, 99) if k < n], "total_ms": float(d.sum() / 1e3)}
    gaps = {}
    for p, q in zip(ks[first:], ks[first + 1:]):
        key = short(p["name"]) + " -> " + short(q["name"])
        gaps.setdefault(key, []).append(q["ts"] - (p["ts"] + p["dur"]))
    out["gaps_us"] = {k: {"n": len(v), "median": float(np.median(v)), "min": float(np.min(v)), "max": float(np.max(v))}
                      for k, v in gaps.items() if len(v) >= 10}
    span = ks[-1]["ts"] + ks[-1]["dur"] - ks[first]["ts"]
    busy = {}
    for k in ks[first:]:
        busy[short(k["name"])] = busy.get(short(k["name"]), 0.0) + k["dur"]
    out["cycle_span_ms"] = span / 1e3
    out["kernel_ms"] = {k: v / 1e3 for k, v in sorted(busy.items(), key=lambda x: -x[1])}
    return out


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("ring_cost: no CUDA device")
    t0 = time.time()
    r = profile() if a.profile else sweep()
    r["wall_s"] = time.time() - t0
    s = json.dumps(r, indent=1)
    print(s)
    if a.out:
        with open(a.out, "w") as f:
            f.write(s + "\n")
