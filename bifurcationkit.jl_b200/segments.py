"""Multi-GPU partition of a branch by continuation step (SURVEY 8e).

PALC is a sequential recurrence (src/Continuation.jl:458-504), so one branch is cut into segments: rank r
advances `steps` continuation steps from a seed pair (z_a, z_b) = two consecutive points of a scout run, using the
reference's two-point start (iterate_from_two_points, src/Continuation.jl:408-456; same mechanism as branch
switching, src/bifdiagram/BranchSwitching.jl:8-44).  State vectors are replicated; the only collective is an
all_gather of the per-step rows (lambda, ||u||, itnewton, itlinear), 32 B per step.
"""
import numpy as np

ROW = ("param", "x", "itnewton", "itlinear")


def seed_steps(rank, stride):
    """Scout step indices whose states seed rank `rank` (first point, second point)."""
    return rank * stride, rank * stride + 1


class SeedGrabber:
    """Continuation callback that keeps the states at the scout steps this rank needs and stops the scout there."""

    def __init__(self, rank, stride, copy):
        self.a, self.b = seed_steps(rank, stride)
        self.copy, self.seeds = copy, {}
        self.last = []  # the two most recent scout points: fallback seeds if the branch ends before step b

    def __call__(self, st):
        if st.step in (self.a, self.b):
            self.seeds[st.step] = (self.copy(st.z_u), st.z_p)
        self.last = (self.last + [(st.step, self.copy(st.z_u), st.z_p)])[-2:]  # a device copy per scout step: negligible
        return st.step < self.b

    def pair(self):
        if self.a in self.seeds and self.b in self.seeds:
            (u0, p0), (u1, p1) = self.seeds[self.a], self.seeds[self.b]
            return u0, p0, u1, p1
        # the scout stopped early (parameter bound reached / ds < dsmin): seed from its last two points
        (_, u0, p0), (_, u1, p1) = self.last
        return u0, p0, u1, p1


def segment_starts(rank, world, steps, subs=4):
    """Interleaved partition of a window of world*steps scout steps into world*nsub sub-segments of `sub` steps:
    rank r owns sub-segments g = s*world + r (s = 0..nsub-1), i.e. every rank samples the whole window, so that hard
    stretches of the branch (folds of the snaking region: rejected steps) are spread over the ranks.
    Returns [(scout_step_of_first_seed, nsteps), ...]."""
    sub = max(1, steps // subs)
    out, left, s = [], steps, 0
    while left > 0:
        k = min(sub, left)
        out.append(((s * world + rank) * sub, k))
        left -= k
        s += 1
    return out


class MultiSeedGrabber:
    """Scout callback collecting the seed pairs (steps a, a+1) of several sub-segments; stops after the last one."""

    def __init__(self, starts, copy):
        self.want = sorted(set(a for a, _ in starts) | set(a + 1 for a, _ in starts))
        self.stop_at = self.want[-1]
        self.copy, self.seeds, self.last = copy, {}, []

    def __call__(self, st):
        if st.step in self.want:
            self.seeds[st.step] = (self.copy(st.z_u), st.z_p)
        self.last = (self.last + [(st.step, self.copy(st.z_u), st.z_p)])[-2:]
        return st.step < self.stop_at

    def pair(self, a):
        if a in self.seeds and a + 1 in self.seeds:
            (u0, p0), (u1, p1) = self.seeds[a], self.seeds[a + 1]
            return u0, p0, u1, p1
        (_, u0, p0), (_, u1, p1) = self.last  # the scout ended early: seed from its last two points
        return u0, p0, u1, p1


def rows_to_array(rows, nrows):
    """Fixed-size (nrows, 4) array for the collective; unused rows are NaN."""
    R = np.full((nrows, len(ROW)), np.nan)
    for i, r in enumerate(rows[:nrows]):
        R[i] = [r[k] for k in ROW]
    return R


def all_gather_rows(rows, nrows, dist, torch, device):
    """The path's only collective: every rank receives every rank's rows.  Returns (world, nrows, 4) ndarray."""
    t = torch.tensor(rows_to_array(rows, nrows), dtype=torch.float64, device=device)
    out = [torch.zeros_like(t) for _ in range(dist.get_world_size())]
    dist.all_gather(out, t)
    return np.stack([o.cpu().numpy() for o in out])


def merge_branch(gathered):
    """Concatenate the segments in rank order (the `_cat!` order of src/Results.jl:436-459), dropping padding and each
    segment's first row when it repeats the previous segment's last seed point."""
    out = []
    for seg in gathered:
        seg = seg[~np.isnan(seg[:, 0])]
        if out and len(seg) and abs(seg[0, 0] - out[-1][-1, 0]) < 1e-12:
            seg = seg[1:]
        if len(seg):
            out.append(seg)
    return np.concatenate(out) if out else np.zeros((0, len(ROW)))


# ======================================================================================================================
# Round 2: one branch WINDOW of fixed arclength, the same for every number of GPUs (strong scaling), partitioned by
# predicted cost from a cheap scout that is itself part of the timed job.
#
#   window   : the curve from the start point over the PALC arclength S (theta-norm chord length, src/continuation/Palc.jl:1-41)
#   scout    : the same PALC iteration with loose tolerances and larger steps (a seed generator, not a result): every rank
#              runs it itself, deterministically -- the library's reductions have a fixed order -- so no state ever crosses
#              NVLink; it records the points z_j, their arclength positions sigma_j and a cost proxy
#   partition: contiguous chunks of scout intervals with equal predicted cost, one per rank
#   chunk    : full-accuracy PALC from the seed pair (z_i, z_{i+1}) through the reference's two-point start
#              (iterate_from_two_points, src/Continuation.jl:408-456) until the curve passes the next rank's seed
#   collective: all_gather of the rows (lambda, ||u||, itnewton, itlinear) only, as before
# ======================================================================================================================
def _chord(V, theta, z_u, z_p, w_u, w_p):
    """theta-norm of (z - w): sqrt(theta/N ||z_u - w_u||^2 + (1 - theta) (z_p - w_p)^2), two reductions"""
    n = len(z_u)
    d2 = V.diffdot(z_u, w_u, z_u) - V.diffdot(z_u, w_u, w_u)
    return float(np.sqrt(max(0.0, theta * d2 / n + (1.0 - theta) * (z_p - w_p) ** 2)))


class ArcTracker:
    """Continuation callback: accumulates the chord arclength of the accepted steps and stops at `s_stop`."""

    def __init__(self, V, theta, s0=0.0, s_stop=np.inf, on_point=None):
        self.V, self.theta, self.s, self.s_stop, self.on_point = V, theta, float(s0), s_stop, on_point
        self.sigma = []

    def __call__(self, st):
        if st.step > 0:
            self.s += _chord(self.V, self.theta, st.z_u, st.z_p, st.zold_u, st.zold_p)
        self.sigma.append(self.s)
        keep = True
        if self.on_point is not None:
            r = self.on_point(st, self.s)
            keep = True if r is None else bool(r)
        return keep and self.s < self.s_stop


class Scout:
    """Seed points of the window: points[j] = (u, p), sigma[j] = arclength position, cost[j] = predicted cost of the
    full-accuracy run between point j-1 and j."""

    def __init__(self):
        self.points, self.sigma, self.cost, self.rows = [], [], [], []


def run_scout(P, prob, alg, cp_scout, normC, s_total, copy, margin=0.0, wrap_callback=None):
    """Loose continuation from the start point over arclength s_total (+ margin); returns a Scout."""
    V = P.V
    sc = Scout()

    def on_point(st, s):
        sc.points.append((copy(st.z_u), st.z_p))
        return True

    trk = ArcTracker(V, alg.theta, 0.0, s_total + margin, on_point)
    cb = wrap_callback(trk) if wrap_callback else trk  # e.g. bench.py's per-step CUDA-event timer
    rows, st = P.continuation(prob, alg, cp_scout, normC=normC, callback=cb)
    sc.sigma = list(trk.sigma)
    sc.rows = rows[: len(sc.sigma)]
    # cost proxy of the interval ending at point j: its arclength (= number of full-accuracy steps at dsmax) weighted by
    # the Krylov work the scout needed there (+ a constant for the per-step overhead)
    sc.cost = [0.0] + [(sc.sigma[j] - sc.sigma[j - 1]) * (20.0 + sc.rows[j]["itlinear"] / max(1, sc.rows[j]["itnewton"]))
                       for j in range(1, len(sc.sigma))]
    return sc


def partition_by_cost(cost, world, min_points=2):
    """Boundaries b[0] = 0 < b[1] < ... < b[world] = J over the scout intervals 1..J such that every chunk
    (b[r], b[r+1]] carries about the same cost and at least one interval.  Pure function (unit-tested on CPU)."""
    J = len(cost) - 1
    world = max(1, min(world, J))
    c = np.cumsum(np.asarray(cost, dtype=float))
    tot = c[-1] if c[-1] > 0 else 1.0
    b = [0]
    for r in range(1, world):
        j = int(np.searchsorted(c, tot * r / world))
        j = min(max(j, b[-1] + 1), J - (world - r))
        b.append(j)
    b.append(J)
    return b


def run_chunk(P, make_prob, alg, cp, normC, sc, i0, i1, s_total, rank, last, wrap_callback=None):
    """Full-accuracy PALC over the scout intervals (i0, i1]: two-point start from (z_i0, z_i0+1) -- rank 0 starts from the true
    start point the usual way -- until the curve passes seed i1 (or, for the last rank, the end of the window).
    Returns (rows, state); rows[0] (the seed itself) is dropped for rank > 0."""
    V, theta = P.V, alg.theta
    u0, p0 = sc.points[i0]
    prob = make_prob(u0, p0)
    end_u, end_p = sc.points[i1]
    # tangent of the scout polyline at the end seed (towards increasing arclength)
    nb_u, nb_p = sc.points[i1 - 1]
    s_end, s_start = sc.sigma[i1], sc.sigma[i0]
    near = s_end - 2.5 * (s_end - sc.sigma[i1 - 1])

    def passed(st, s):
        if last:
            return s < s_total
        if s < near:
            return True
        # projection of (z - z_end) on the end tangent (z_end - z_prev) in the theta inner product
        n = len(st.z_u)
        du = V.diffdot(st.z_u, end_u, end_u) - V.diffdot(st.z_u, end_u, nb_u)
        proj = theta * du / n + (1.0 - theta) * (st.z_p - end_p) * (end_p - nb_p)
        return proj < 0.0

    trk = ArcTracker(V, theta, s_start, np.inf, passed)
    cb = wrap_callback(trk) if wrap_callback else trk
    if rank == 0 and i0 == 0:
        rows, st = P.continuation(prob, alg, cp, normC=normC, callback=cb)
        return rows, st, trk
    u1, p1 = sc.points[i0 + 1]
    rows, st = P.continuation(prob, alg, cp, normC=normC, u1=u1, p1=p1, callback=cb)
    return rows[1:], st, trk


def merge_chunks(gathered):
    """Rank-ordered concatenation of the gathered (world, nrows, 4) rows, padding dropped."""
    out = [seg[~np.isnan(seg[:, 0])] for seg in gathered]
    out = [s for s in out if len(s)]
    return np.concatenate(out) if out else np.zeros((0, len(ROW)))


def curve_distance(branch, ref):
    """max over the points of `branch` of the distance to the polyline `ref` in the (lambda, x) plane, both columns scaled
    by the extent of `ref` -- the arclength-interpolation parity check of SURVEY 8e (segment boundaries and adaptive ds
    change WHICH points are computed, not the curve)."""
    a = np.asarray(branch)[:, :2].astype(float)
    b = np.asarray(ref)[:, :2].astype(float)
    sc = np.maximum(b.max(0) - b.min(0), 1e-300)
    a, b = a / sc, b / sc
    worst = 0.0
    for p in a:
        d = np.inf
        for q0, q1 in zip(b[:-1], b[1:]):
            v = q1 - q0
            t = 0.0 if not np.any(v) else min(1.0, max(0.0, float(np.dot(p - q0, v) / np.dot(v, v))))
            d = min(d, float(np.linalg.norm(p - (q0 + t * v))))
        worst = max(worst, d)
    return worst


# ======================================================================================================================
# bothside = true: the one split of a continuation job the reference itself offers (src/Continuation.jl:687-700): two
# independent iterators from the same start point, ds and -ds, merged by _merge (src/Results.jl:464-489).  On two GPUs each
# direction runs on its own device (replicated start state, nothing crosses NVLink), the rows are all_gathered and every rank
# assembles the same branch.
# ======================================================================================================================
def merge_bothside(fwd, bwd, tol=1e-6):
    """_merge(resfwd, resbwd): both runs start on the same point, so the merged branch is the backward run reversed followed
    by the forward run (`_cat!(_reverse(br2), br1)`, src/Results.jl:476-478) -- the start point appears twice, as in the
    reference -- with the steps renumbered along the merged branch.  fwd / bwd: (n, >= 2) arrays or lists of row dicts."""
    arr = lambda rows: rows_to_array(rows, len(rows)) if len(rows) and isinstance(rows[0], dict) else np.asarray(rows, dtype=float)
    f, b = arr(fwd), arr(bwd)
    f, b = f[~np.isnan(f[:, 0])], b[~np.isnan(b[:, 0])]
    if not len(b):
        return f
    if not len(f):
        return b[::-1]
    same = lambda r, s: max(abs(r[0] - s[0]), abs(r[1] - s[1])) < tol
    if same(f[0], b[0]):
        return np.concatenate([b[::-1], f])
    if same(f[0], b[-1]):
        return np.concatenate([b, f])
    if same(f[-1], b[0]):
        return np.concatenate([f, b])
    return np.concatenate([f, b[::-1]])


def continuation_bothside(P, make_prob, alg, contpar, normC, dist=None, torch=None, device="cpu", nrows=None):
    """continuation(prob, alg, contpar; bothside = true).  make_prob() -> a fresh problem (the reference deep-copies the iterator:
    some problems are changed in place).  Without `dist` (or world 1) both directions run here, one after the other; with a
    process group of >= 2 ranks, rank 0 runs ds, rank 1 runs -ds (further ranks idle), the rows are all_gathered and merged on
    every rank.  Returns (merged (n, 4) array of (param, x, itnewton, itlinear), this rank's own rows)."""
    import copy
    world = dist.get_world_size() if dist is not None else 1
    rank = dist.get_rank() if dist is not None else 0

    def run(sign):
        cp = copy.copy(contpar)
        cp.ds = sign * contpar.ds
        return P.continuation(make_prob(), alg, cp, normC=normC)[0]

    if world == 1:
        fwd, bwd = run(1.0), run(-1.0)
        return merge_bothside(fwd, bwd), fwd + bwd
    mine = run(1.0) if rank == 0 else (run(-1.0) if rank == 1 else [])
    nrows = nrows or contpar.max_steps + 8
    gathered = all_gather_rows(mine, nrows, dist, torch, device)
    return merge_bothside(gathered[0], gathered[1]), mine


# ======================================================================================================================
# Speculative step sizes: a multi-GPU scheme that computes the SAME branch as one GPU, point for point.
#
# PALC is a sequential recurrence, but one part of it is predictable: when the corrector fails, the reference halves ds and
# corrects again from the same point with the same tangent (step_size_control!, src/continuation/Contbase.jl:79-88) -- and a
# failing corrector is the expensive kind (all max_iterations Newton steps).  With the state replicated on every rank, rank r
# runs the corrector for the r-times-halved step at the same time; the first rank (in the order the sequential loop would try
# them) that converged wins, its corrected point is broadcast (N + 1 doubles), and every rank moves on from it with the step
# size the sequential loop would have had.  Accepted points, rows and counters equal the single-process run exactly (same
# inputs, deterministic kernels); what changes is the wall time of the rejected attempts.
# ======================================================================================================================
def continuation_speculative(P, prob, alg, contpar, normC, dist, torch, device="cpu", callback=None, to_host=None, from_host=None):
    """palc.continuation(prob, alg, contpar, normC) over the ranks of `dist` with speculative step sizes.  Every rank returns the
    same (rows, state, info); info = dict(rounds, attempts, wasted): corrector rounds actually waited for, corrector attempts the
    sequential loop makes, attempts computed but not needed.  to_host(v) -> ndarray / from_host(a, like) -> vector move the accepted
    point through the collective (defaults: ndarray as is, DeviceVec through .numpy() / ctx.to_device)."""
    V = P.V
    world, rank = dist.get_world_size(), dist.get_rank()
    to_host = to_host or (lambda v: v.numpy() if hasattr(v, "numpy") else np.asarray(v))
    from_host = from_host or (lambda a, like: like.ctx.to_device(a) if hasattr(like, "ctx") else np.array(a))
    it = P.ContIterable(prob, alg, contpar, normC)
    st = it.start()                                              # start-up: replicated, deterministic
    rows, info = [], dict(rounds=0, attempts=0, wasted=0)

    def save():
        rows.append(dict(param=st.z_p, x=prob.record(st.z_u), itnewton=st.itnewton, itlinear=st.itlinear, ds=st.ds, step=st.step,
                         n_unstable=-1))
        if callback is not None and callback(st) is False:
            st.stop = True

    save()
    n = len(st.z_u)
    while it.done(st):
        # the step sizes the sequential loop would try one after the other from this point: d_0 = ds, d_{r+1} = halve(d_r)
        trial, d, dead = [], st.ds, False
        for _ in range(world):
            trial.append(None if dead else d)
            if not dead:
                d, dead = P.step_size_control(d, False, 0, contpar)
        mine = trial[rank]
        res = np.zeros(4)                                        # (valid, converged, itnewton, itlinear)
        sol = None
        if mine is not None:
            V.copyto(st.zpred_u, st.z_u)
            V.axpby(st.zpred_u, mine, st.tau_u, 1.0)
            sol = it.correct(st, st.z_p + mine * st.tau_p, mine)
            res[:] = (1.0, float(sol.converged), sol.itnewton, sol.itlineartot)
        t = torch.tensor(res, dtype=torch.float64, device=device)
        allr = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(allr, t)
        allr = np.stack([a.cpu().numpy() for a in allr])
        info["rounds"] += 1
        win = next((r for r in range(world) if allr[r, 0] and allr[r, 1]), None)
        last = max(r for r in range(world) if allr[r, 0])        # last valid trial of this round
        upto = win if win is not None else last
        for r in range(upto + 1):                                # what the sequential loop would have run
            st.work_newton += int(allr[r, 2])
            st.work_linear += int(allr[r, 3])
            info["attempts"] += 1
        st.nfail += upto if win is not None else upto + 1
        info["wasted"] += int(np.sum(allr[:, 0])) - (upto + 1)
        if win is None:
            st.converged = False
            st.itnewton, st.itlinear = int(allr[last, 2]), int(allr[last, 3])
            st.ds, st.stop = P.step_size_control(trial[last], False, 0, contpar)  # the failed attempt with d_last: halve or stop
            continue
        # the winner's corrected point to every rank
        buf = np.zeros(n + 1)
        if rank == win:
            buf[:n], buf[n] = to_host(sol.u), sol.p
        tb = torch.tensor(buf, dtype=torch.float64, device=device)
        dist.broadcast(tb, src=win)
        buf = tb.cpu().numpy()
        it.accept(st, sol.u if rank == win else from_host(buf[:n], st.z_u), float(buf[n]))
        st.converged, st.itnewton, st.itlinear = True, int(allr[win, 2]), int(allr[win, 3])
        st.ds, st.stop = P.step_size_control(trial[win], True, st.itnewton, contpar)
        it.advance(st)
        if st.step <= contpar.max_steps:
            save()
    return rows, st, info
