"""Wall time of a level-2 automatic bifurcation diagram (bifdiagram.py) with its sibling branches continued one at a time
(max_workers = 1) and four at a time (max_workers = 4), on the trivial Swift-Hohenberg state of three grids:

  - 48 x 48 on the square of tests/test_gpu_nd_normal_form.py (lx = ly = 2.3 pi), the root branch through its first crossing;
  - 151 x 100 on the domain of examples/SH2d-fronts.jl (lx = 8 pi, ly = 4 pi / sqrt(3)), the root branch through its first
    four crossings;
  - 512 x 512 on the bench's domain scaling (bench.domain), the root branch through its first two crossings, started closer
    to them and with larger steps (`--cross`, `--lead`, `--root-steps` set these per grid: each root step at 512^2 costs an
    eigen-solve of several seconds).

The root branch is computed once per grid (detect_bifurcation = 3, shift-invert eigensolver, GMRES(100) with the DCT
preconditioner); each child is continued for `--child-steps` steps with detection on.  The two settings alternate, each run
ended by a device synchronise, and the median of `--reps` runs is reported, with the number of units (special points branched),
of children, the peak number of live contexts (the diagram's included), the lowest free device memory seen during the run
(sampled every 5 ms) and the card's name and power limit read in the same run.  Prints one JSON object."""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402
import __graft_entry__ as g  # noqa: E402
import bench  # noqa: E402
from tests.test_gpu_normal_form import _dct_eigs  # noqa: E402

bk = g.load_package()
P, D = bk.palc, bk.bifdiagram


def crossings(dims, lengths, k):
    """the first k distinct values of l where a DCT mode of the trivial state crosses"""
    lam = np.add.outer(_dct_eigs(dims[0], lengths[0]), _dct_eigs(dims[1], lengths[1]))
    m = np.unique(np.round(((1 + lam) ** 2).ravel(), 12))
    return m[: k + 1]


def case(dims, lengths, ncross, child_steps, lead=0.01, root_steps=30):
    """the root branch from l* - lead to midway between crossings ncross and ncross + 1, in steps of at most 1/root_steps of
    that interval"""
    ls_m = 100
    m = crossings(dims, lengths, ncross)
    l0, l1 = m[0] - lead, 0.5 * (m[ncross - 1] + m[ncross])
    ctx = bk.Context(bk.BK_SH2D, dims, lengths, krylov_m=ls_m, params=(l0, 1.3))
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(reltol=1e-11, restart=ls_m, maxiter=300, Pl=True, orth="cgs2")
    eig = bk.ShiftInvertB200(0.05, ls, krylovdim=40, tol=1e-11, maxrestart=30)
    nopts = P.NewtonPar(tol=1e-10, max_iterations=10, linsolver=ls, eigsolver=eig)
    prob = P.BifurcationProblemB200(ctx, ctx.zeros(), (l0, 1.3), lens=0, record=lambda v: v.norminf())
    alg = P.PALC(bls=bk.MatrixFreeBLSB200(ls))
    step = min(0.002, (l1 - l0) / root_steps)
    cp = P.ContinuationPar(dsmin=1e-6, dsmax=step, ds=step, p_min=l0 - 1e-3, p_max=l1, max_steps=200, nev=8, newton_options=nopts,
                           detect_bifurcation=3, n_inversion=8)
    br = bk.events.continuation(prob, alg, cp, normC=P.norminf,
                                callback=lambda st: print(f"root step {st.step} l = {st.z_p:.6g}", file=sys.stderr, flush=True))
    child = P.ContinuationPar(**{**vars(cp), **dict(ds=step / 2, max_steps=child_steps, p_min=l0 - 0.05, p_max=l1 + 0.05)})
    return ctx, prob, alg, br, (lambda x, p, lvl: cp if lvl <= 1 else child)


class Watch:
    """live contexts (around Context.__init__ / close) and the lowest free device memory, sampled every 5 ms"""

    def __init__(self):
        self.lock, self.live, self.peak, self.low, self.on = threading.Lock(), 0, 0, None, False
        init, close = bk.Context.__init__, bk.Context.close
        w = self

        def counted_init(ctx, *a, **k):
            init(ctx, *a, **k)
            with w.lock:
                w.live += 1
                w.peak = max(w.peak, w.live)

        def counted_close(ctx):
            if getattr(ctx, "handle", None):
                with w.lock:
                    w.live -= 1
            close(ctx)
        bk.Context.__init__, bk.Context.close = counted_init, counted_close

    def _sample(self):
        while self.on:
            f = torch.cuda.mem_get_info()[0]
            self.low = f if self.low is None else min(self.low, f)
            time.sleep(0.005)

    def __enter__(self):
        self.peak, self.low, self.on = self.live, None, True
        self.t = threading.Thread(target=self._sample)
        self.t.start()
        return self

    def __exit__(self, *exc):
        self.on = False
        self.t.join()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--child-steps", type=int, default=10)
    ap.add_argument("--grids", default="48,151,512")
    ap.add_argument("--cross", default="48:1,151:4,512:2", help="crossings of the root branch per grid")
    ap.add_argument("--lead", default="48:0.01,151:0.01,512:0.0005", help="how far before the first crossing the root starts")
    ap.add_argument("--root-steps", default="48:30,151:30,512:8", help="the root's largest step = its interval / this")
    args = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out = dict(gpu=q.stdout.strip(), reps=args.reps, child_steps=args.child_steps, cases=[])
    cross, lead, nroot = (dict(kv.split(":") for kv in a.split(",")) for a in (args.cross, args.lead, args.root_steps))
    setups = {"48": ((48, 48), (2.3 * np.pi, 2.3 * np.pi)), "151": ((151, 100), (8 * np.pi, 4 * np.pi / np.sqrt(3))),
              "512": ((512, 512), bench.domain(512))}
    watch = Watch()
    for key in args.grids.split(","):
        (dims, lengths), ncross = setups[key], int(cross[key])
        t0 = time.perf_counter()
        ctx, prob, alg, br, options = case(dims, lengths, ncross, args.child_steps, float(lead[key]), int(nroot[key]))
        t_root = time.perf_counter() - t0
        units = [i for i, s in enumerate(br.specialpoint) if s.step > 1 and s.type in ("bp", "nd")]
        res = {1: [], 4: []}
        info = {}
        for r in range(args.reps):
            for w in ((1, 4) if r % 2 == 0 else (4, 1)):
                torch.cuda.synchronize()
                free0 = torch.cuda.mem_get_info()[0]
                with watch:
                    t0 = time.perf_counter()
                    d = D.bifurcationdiagram_from(prob, br, 2, options, alg, normC=P.norminf, max_workers=w)
                    ctx.sync()
                    torch.cuda.synchronize()
                    res[w].append(time.perf_counter() - t0)
                info[w] = dict(children=len(d.child), failures=len(d.failures), peak_contexts=watch.peak,
                               peak_device_mib=(free0 - watch.low) / 2**20 if watch.low is not None else None)
                del d
        row = dict(dims=dims, lengths=[float(x) for x in lengths], root_steps=len(br.rows), root_s=t_root,
                   special=[(s.type, s.param, s.delta) for s in br.specialpoint], units=len(units),
                   wall_s={w: float(np.median(v)) for w, v in res.items()}, runs_s=res, info=info)
        row["speedup"] = row["wall_s"][1] / row["wall_s"][4]
        out["cases"].append(row)
        print(json.dumps(row, default=float), file=sys.stderr, flush=True)
        ctx.close()
    print(json.dumps(out, default=float))


if __name__ == "__main__":
    main()
