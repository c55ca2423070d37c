"""Cost of the normal form of a branch point with an N-dimensional kernel on the device (normalform.get_normal_formNd), at the
closed-form crossing of the trivial Swift-Hohenberg state (nu = 1.3, Neumann FD) in two boxes at the bench's mesh width
h = pi / 16 (DESIGN.md §7 workload note):
  - square 1024^2, lx = ly = 32 pi: the DCT pair (25, 59) / (59, 25) crosses first, N = 2;
  - cube 128^3, lx = ly = lz = 4 pi: (8, 0, 0) and its permutations, N = 3.
For each: the wall time of get_normal_formNd with ζs recomputed by the shift-invert eigensolver, split into the eigen-solves, the
bordered solves and the contractions (each part ended by a device synchronise); then the contractions it made, by the one-pass
kernel (bk_jet_moments) against the composed path (bk_d2f / bk_d3f + bk_vec_dot per tuple) in alternating rounds timed with
CUDA events on the context's stream, with the launches and algorithmic bytes of both from the shapes.  The card's name and power
limit are read in the same run.  Prints one JSON object."""
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
NU = 1.3


def crossing(dims, lengths):
    lam = None
    for n, L in zip(dims, lengths):
        e = -(2 - 2 * np.cos(np.pi * np.arange(n) / n)) / (2 * L / n) ** 2
        lam = e if lam is None else np.add.outer(lam, e)
    m = ((1 + lam) ** 2).ravel()
    order = np.argsort(m, kind="stable")
    k = int(np.sum(np.abs(m - m[order[0]]) <= 1e-12 * max(1.0, m[order[0]])))
    return float(m[order[0]]), [tuple(int(q) for q in np.unravel_index(i, lam.shape)) for i in order[:k]]


class Timed:
    """accumulated wall time of calls of fn, each ended by a device synchronise"""

    def __init__(self, ctx, fn):
        self.ctx, self.fn, self.s, self.calls = ctx, fn, 0.0, 0

    def __call__(self, *a, **k):
        t = time.perf_counter()
        out = self.fn(*a, **k)
        self.ctx.sync()
        self.s += time.perf_counter() - t
        self.calls += 1
        return out


def case(name, dims, lengths, rounds):
    lstar, modes = crossing(dims, lengths)
    N = len(modes)
    kind = bk.BK_SH2D if len(dims) == 2 else bk.BK_SH3D
    ctx = bk.Context(kind, dims, lengths, krylov_m=100, params=(lstar, NU))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(reltol=1e-10, restart=100, maxiter=300, Pl=True, orth="cgs2")
    eig = bk.ShiftInvertB200(0.05, ls, krylovdim=40, tol=1e-10, maxrestart=30)
    prob = P.BifurcationProblemB200(ctx, ctx.zeros(), (lstar, NU), lens=0)
    nev = 2 * N + 2
    vals, _, _, _ = eig(prob.J(prob.u0, lstar), nev)
    br = E.Branch(specialpoint=[E.SpecialPoint(type="nd", idx=0, param=lstar, norm=0.0, step=0, status="converged", delta=(N, 0),
                                               ind_ev=N, interval=(lstar, lstar), x=prob.u0, tau_p=1.0, tau_u=ctx.zeros())],
                  eig=[dict(eigenvals=vals, step=0)])
    teig = Timed(ctx, lambda J, k: eig(J, k, want_vectors=True))
    bls = bk.MatrixFreeBLSB200(ls)
    bls.solve_block = tbls = Timed(ctx, bls.solve_block)
    calls = []
    one_pass = prob.jet_moments

    def record(*a):
        calls.append(a)
        return one_pass(*a)
    prob.jet_moments = tmom = Timed(ctx, record)
    cp = P.ContinuationPar(newton_options=P.NewtonPar(tol=1e-10, linsolver=ls, eigsolver=teig), nev=nev)
    it = P.ContIterable(prob, P.PALC(bls=bls), cp, P.norminf)
    NF.get_normal_formNd(it, br, 0, bls=bls)                      # warm-up: modules, shared-memory grants, pools
    for t in (teig, tbls, tmom):
        t.s, t.calls = 0.0, 0
    calls.clear()
    t0 = time.perf_counter()
    bp = NF.get_normal_formNd(it, br, 0, bls=bls)
    ctx.sync()
    total = time.perf_counter() - t0
    x, p, vecs, idx2, idx3 = calls[0]
    n2, n3, nvec, N0 = len(idx2), len(idx3), len(vecs), ctx.N0
    G = min(-(-N0 // 256), 8 * torch.cuda.get_device_properties(0).multi_processor_count)   # bk_reduce_grid of the points
    # alternating rounds of the two paths on the same inputs, CUDA events on the context's stream
    stream = torch.cuda.ExternalStream(ctx.lib.bk_stream(ctx.handle))
    times = {"kernel": [], "composed": []}
    for r in range(rounds):
        for path in ("kernel", "composed"):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            m = one_pass(x, p, vecs, idx2, idx3) if path == "kernel" else NF.jet_moments_composed(prob, x, p, vecs, idx2, idx3)
            b.record(stream)
            b.synchronize()
            times[path].append(a.elapsed_time(b))
            if r == 0:
                scale = np.max(np.abs(m))
                if path == "kernel":
                    mk = m
                else:
                    diff = float(np.max(np.abs(m - mk)) / scale)
    kb = 8 * N0 * (nvec + 1) + 2 * 8 * (n2 + n3) * G
    cb = 8 * N0 * (6 * n2 + 7 * n3)
    med = {k: float(np.median(v)) for k, v in times.items()}
    return dict(case=name, dims=list(dims), lengths_over_pi=[L / np.pi for L in lengths], N0=N0, kernel_dim=N, modes=modes,
                lstar=lstar, type=bp.type, b30_norm=float(np.max(np.abs(bp.nf["b30"]))),
                normal_form_s=dict(total=total, eigen=teig.s, bordered=tbls.s, bordered_solves=tbls.calls, contractions=tmom.s,
                                   rest=total - teig.s - tbls.s - tmom.s),
                contractions=dict(n2=n2, n3=n3, nvec=nvec, rounds=rounds, kernel_ms_median=med["kernel"],
                                  composed_ms_median=med["composed"], speedup=med["composed"] / med["kernel"],
                                  kernel_launches=2, composed_launches=2 * (n2 + n3), kernel_bytes=kb, composed_bytes=cb,
                                  kernel_GBps=kb / med["kernel"] / 1e6, composed_GBps=cb / med["composed"] / 1e6,
                                  max_rel_diff=diff))


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = dict(gpu=gpu, cases=[case("square", (1024, 1024), (32 * np.pi,) * 2, 5),
                               case("cube", (128, 128, 128), (4 * np.pi,) * 3, 3)])
    print(json.dumps(out))


if __name__ == "__main__":
    main()
