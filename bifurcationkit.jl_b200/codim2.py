"""SURVEY section 8f.3: Fold and Hopf points by the minimally augmented (MA) formulation, as host orchestration over the
same C ABI -- every linear solve is a (bordered) solve through `bk_bls_*` / `bk_gmres`, every operator application a `bk_jvp`.

Mirror of src/codim2/MinAugFold.jl:
  FoldMinAug.residual      <->  (F::FoldMinimallyAugmentedFormulation)(x, p, params)            :15-39
  FoldMinAug.bordered_terms <-> _compute_bordered_vectors / _get_bordered_terms                   :55-104
  FoldMinAug.solve         <->  foldMALinearSolver, finite-difference branch (usehessian = false) :122-146
  FoldMinAug.update        <->  update!(probma, iter, state), test_bt_cusp                        :276-309, 551-575
  newton_fold              <->  newton_fold(prob, foldpointguess, par, eigenvec, eigenvec_ad, options; bdlinsolver)  :201-222
  MAProblem, MALinearSolver <-> FoldMAProblem, FoldLinearSolverMinAug                              :148-163
Swift-Hohenberg is self-adjoint (is_symmetric = true, examples/SH3d.jl:123), so J' = J and no adjoint kernel is needed (for
the Chan problem J' = J only up to the two boundary rows: the left null vector, hence sigma_x and sigma_p, are then approximate
and Newton on the MA system degrades to a quasi-Newton iteration that still converges to the same fold).

Mirror of src/codim2/MinAugHopf.jl:
  HopfMinAug.residual       <->  (H::HopfMinimallyAugmentedFormulation)(x, p, omega, params)      :19-40
  HopfMinAug.bordered_terms <->  __compute_bordered_vectors / _get_bordered_terms                 :59-104
  HopfMinAug.solve          <->  _hopf_MA_linear_solver, finite-difference branch                 :122-188
  HopfMinAug.update         <->  update!(probma, iter, state)                                     :323-367
  newton_hopf               <->  newton_hopf(prob, hopfpointguess, par, eigenvec, eigenvec_ad, options)  :258-283
  MAProblem, MALinearSolver <->  HopfMAProblem, HopfLinearSolverMinAug                            :190-205
The complex shifts (J - i omega, (J - i omega)^H = J' + i omega) are solved on a BK_COMPLEX context (include/bk200.h): split
complex vectors, GMRES on the real-equivalent system, J' from bk_jac_set_transpose.  The complex bordered systems
[A a; b^H 0] are eliminated by bordering on the host (one complex solve each, since their right-hand side is (0, 1));
complex vectors are NumPy arrays (a Hopf refinement is a handful of solves, not a hot loop), real ones keep their container.
"""
from dataclasses import dataclass
import math

import numpy as np

from .palc import V


def _apply(J, v):
    """apply(J, v) (src/Utils.jl:192): J may be a callable Jacobian object or a matrix"""
    return J(v) if callable(J) else J @ v


@dataclass
class FoldSolution:
    u: object
    p: float
    residuals: list
    converged: bool
    itnewton: int
    itlinear: int
    sigma: float


class FoldMinAug:
    """[F(x, p); sigma(x, p)] with sigma from  [J a; b' 0] [v; sigma] = [0; 1]  (Govaerts 2000: a ~ left, b ~ right null vector)."""

    # the MA state's BorderedVec.p <-> the scalar unknowns (p1,), and the residual's (sigma,) or a solve's (dp,) -> BorderedVec.p
    unpack = staticmethod(lambda zp: (zp,))
    pack = staticmethod(lambda sigma: sigma)
    copy_rhs = False   # MALinearSolver hands solve() the right-hand side itself

    def __init__(self, prob, a, b, bls, symmetric=True, norm=V.norm2):
        assert symmetric or hasattr(prob, "Jt"), "non-symmetric problem: prob.Jt(x, p) (jacobian_adjoint) is required"
        self.prob, self.a, self.b, self.bls, self.symmetric, self.norm = prob, V.copy(a), V.copy(b), bls, symmetric, norm
        self.problems = (prob,)      # the problems whose params[lens2] a curve sets
        self.zero = V.zeros_like(a)
        self.itlinear = 0
        self.BT, self.CP = 1.0, 1.0  # test functions of the Bogdanov-Takens / cusp events (MinAugFold.jl:421-423, 551-575)

    def _Jt(self, x, p):
        """jacobian_adjoint(prob, x, p) (has_adjoint) -- J itself for a self-adjoint problem (is_symmetric, MinAugFold.jl:96-100)"""
        return self.prob.J(x, p) if self.symmetric else self.prob.Jt(x, p)

    def _border(self, J, a, b):
        """linbdsolver(J, a, b, 0, zero, 1) -> (v, sigma): J v + a sigma = 0, <b, v> = 1"""
        v, sig, cv, it = self.bls(J, a, b, 0.0, self.zero, 1.0)
        self.itlinear += int(np.sum(it))
        return v, sig

    def residual(self, x, p):
        J = self.prob.J(x, p)
        _, sigma = self._border(J, self.a, self.b)
        return self.prob.F(x, p), sigma

    def bordered_terms(self, x, p):
        prob = self.prob
        eps = prob.delta
        J = prob.J(x, p)
        v, _ = self._border(J, self.a, self.b)
        w, _ = self._border(J if self.symmetric else self._Jt(x, p), self.b, self.a)   # adjoint system J' w + b sigma2 = 0, <a, w> = 1
        # d_p F and sigma_p = -<w, d_p(J v)> by centred differences (MinAugFold.jl:92-101)
        dpF = prob.F(x, p + eps)
        V.axpby(dpF, -1.0 / (2 * eps), prob.F(x, p - eps), 1.0 / (2 * eps))
        jp = _apply(prob.J(x, p + eps), v)
        jm = _apply(prob.J(x, p - eps), v)
        V.axpby(jp, -1.0 / (2 * eps), jm, 1.0 / (2 * eps))
        sigma_p = -V.dot(w, jp)
        return v, w, dpF, sigma_p

    def solve(self, x, p, rhsu, rhsp, cache=None):
        """foldMALinearSolver: [J d_pF; sigma_x' sigma_p] [dX; dp] = [rhsu; rhsp] with
        sigma_x = (J'(x) w - J'(x + eps v) w) / eps  (MinAugFold.jl:135-141).  `cache`: an object whose `.terms` keeps
        (d_pF, sigma_x, sigma_p) between the right-hand sides solved at the same (x, p)."""
        prob = self.prob
        eps = prob.delta
        if cache is not None and cache.terms is not None:
            dpF, sigma_x, sigma_p = cache.terms
        else:
            v, w, dpF, sigma_p = self.bordered_terms(x, p)
            xs = V.copy(x)
            V.axpby(xs, eps, v, 1.0)
            u1 = _apply(self._Jt(xs, p), w)
            sigma_x = _apply(self._Jt(x, p), w)
            V.axpby(sigma_x, -1.0 / eps, u1, 1.0 / eps)  # (u2 - u1) / eps
            if cache is not None:
                cache.terms = (dpF, sigma_x, sigma_p)
        J = prob.J(x, p)                                 # back to the linearisation at x (one state per context)
        dX, dp, cv, it = self.bls(J, dpF, sigma_x, sigma_p, rhsu, rhsp)
        self.itlinear += int(np.sum(it))
        return dX, dp, cv

    def update(self, x, p, keep_borders=False):
        """update!(probma, iter, state) (MinAugFold.jl:276-309) and test_bt_cusp (:551-575): after an accepted step the border
        vectors follow the null vectors, a <- w / ||w||, b <- v / ||v||; BT = <w / ||w||, v / ||v||>.  keep_borders: only the
        test function (inside an event bisection the reference leaves a, b alone, :287-289)."""
        J = self.prob.J(x, p)
        v, _ = self._border(J, self.a, self.b)
        w, _ = self._border(J if self.symmetric else self._Jt(x, p), self.b, self.a)
        V.scale(v, 1.0 / self.norm(v))
        V.scale(w, 1.0 / self.norm(w))
        if not keep_borders:
            V.copyto(self.a, w)
            V.copyto(self.b, v)
        self.BT = V.dot(w, v)
        return self.BT


def _newton_ma(ma, x0, q0, opts, resnorm):
    """src/Newton.jl:66-114 on the MA system of `ma` in the state (x, q), q = (p,) or (p, omega): ma.residual(x, *q) -> (F, *s),
    ma.solve(x, *q, F, *s) -> (dX, *dq, converged), resnorm(F, *s) -> the residual norm.  Returns (x, q, s, residuals, steps)."""
    x, q = V.copy(x0), [float(v) for v in q0]
    F, *s = ma.residual(x, *q)
    residuals = [resnorm(F, *s)]
    step = 0
    while step < opts.max_iterations and residuals[-1] > opts.tol:
        dX, *dq, _ = ma.solve(x, *q, F, *s)
        V.axpby(x, -1.0, dX, 1.0)
        q = [v - d for v, d in zip(q, dq)]
        F, *s = ma.residual(x, *q)
        residuals.append(resnorm(F, *s))
        step += 1
    return x, q, s, residuals, step


def newton_fold(prob, x0, p0, eigenvec, eigenvec_ad, opts, bls, normN=V.norm2, symmetric=True):
    """Newton on the MA system from the guess (x0, p0) with guesses for the right / left null vectors
    (newton_fold, MinAugFold.jl:201-222 + src/Newton.jl:66-114 on the bordered state)."""
    ma = FoldMinAug(prob, eigenvec_ad, eigenvec, bls, symmetric=symmetric)
    x, (p,), (sigma,), residuals, step = _newton_ma(ma, x0, (p0,), opts, lambda F, sigma: math.hypot(normN(F), abs(sigma)))
    return FoldSolution(x, p, residuals, residuals[-1] < opts.tol, step, ma.itlinear, sigma)


# ------------------------------------------------------------------------------------------------ Fold and Hopf curves in two parameters
class BorderedVec:
    """BorderedArray(u, p) (src/BorderedArrays.jl:23-70, 86-217) with the method set of a DeviceVec, so that the PALC host
    loop (palc.py) runs on the state of a minimally augmented problem unchanged: (x, p1) for Folds, (x, [p1, omega]) for Hopf
    points (hopf_point, MinAugHopf.jl:13).  u is a DeviceVec or an ndarray, p a float or a short ndarray."""

    def __init__(self, u, p):
        self.u = u
        self.p = float(p) if np.ndim(p) == 0 else np.array(p, dtype=np.float64)

    def __len__(self):                 # Base.length(b) = length(b.u) + length(b.p)   (:49-50)
        return len(self.u) + int(np.size(self.p))

    def copy(self):
        return BorderedVec(V.copy(self.u), self.p)

    def copyto(self, src):
        V.copyto(self.u, src.u)
        self.p = src.p if np.ndim(src.p) == 0 else src.p.copy()
        return self

    def zero_(self):                   # VI.zerovector!: exact zeros (0 * NaN would stay NaN)
        if hasattr(self.u, "zero_"):
            self.u.zero_()
        else:
            self.u[...] = 0.0
        self.p = 0.0 if np.ndim(self.p) == 0 else np.zeros_like(self.p)
        return self

    def scale_(self, a):
        V.scale(self.u, a)
        self.p = self.p * a
        return self

    def axpby_(self, a, x, b=1.0):     # VI.add!(y, x, a, b)
        V.axpby(self.u, a, x.u, b)
        self.p = a * x.p + b * self.p
        return self

    def dot(self, y):                  # VI.inner(a, b) = inner(a.u, b.u) + inner(a.p, b.p)   (:53)
        return V.dot(self.u, y.u) + float(np.sum(self.p * y.p))

    def norm(self):                    # :55-58
        return math.sqrt(V.norm2(self.u) ** 2 + float(np.sum(self.p * self.p)))

    def norminf(self):                 # :62
        from .palc import nanmax2
        return nanmax2(V.norminf(self.u), float(np.max(np.abs(self.p))))

    def diffdot(self, x0, tau):
        return V.diffdot(self.u, x0.u, tau.u) + float(np.sum((self.p - x0.p) * tau.p))


class _MAJacobian:
    """jacobian(MAProblem, z, p2): a handle on (z, p2).  `terms` keeps what ma.solve may share between the right-hand sides
    BorderingBLS solves with the handle (FoldMinAug: the bordered terms, which the reference recomputes per right-hand side)."""

    def __init__(self, pb, z, p2):
        self.pb, self.z, self.p2, self.terms = pb, z, p2, None


class MALinearSolver:
    """(foldl::FoldLinearSolverMinAug)(Jfold, rhs) / (hopfl::HopfLinearSolverMinAug)(Jhopf, rhs) -> (sol, converged, iters)
    (MinAugFold.jl:148-163, MinAugHopf.jl:190-205): ma.solve on the unpacked state and right-hand side."""

    def __call__(self, Jma, rhs):
        pb, ma = Jma.pb, Jma.pb.ma
        pb._set2(Jma.p2)
        it0 = ma.itlinear
        rhsu = V.copy(rhs.u) if ma.copy_rhs else rhs.u
        dX, *dq, cv = ma.solve(Jma.z.u, *ma.unpack(Jma.z.p), rhsu, *ma.unpack(rhs.p), cache=Jma)
        return BorderedVec(dX, ma.pack(*dq)), cv, ma.itlinear - it0


class MAProblem:
    """FoldMAProblem / HopfMAProblem: the minimally augmented system of `ma` ([F; sigma] for a FoldMinAug, [F; Re sigma; Im sigma]
    for a HopfMinAug) as a problem in the state z = BorderedVec(x, p1) or BorderedVec(x, [p1, omega]) with continuation parameter
    p2 = params[lens2] (continuation_fold, MinAugFold.jl:366-452; continuation_hopf, MinAugHopf.jl:425-522)."""

    def __init__(self, ma, lens2, z0, record=None):
        assert lens2 != ma.prob.lens, "Please choose 2 different parameters."
        self.ma, self.lens2, self.u0 = ma, lens2, z0
        self.p0 = float(ma.prob.params[lens2])
        self.delta = ma.prob.delta
        self.record = record or (lambda z: ma.unpack(z.p)[0])   # record_from_solution: p1 -- p2 is the row's param

    def _set2(self, p2):
        for prob in self.ma.problems:
            prob.params[self.lens2] = p2

    def F(self, z, p2, out=None):
        self._set2(p2)
        Fu, *s = self.ma.residual(z.u, *self.ma.unpack(z.p))
        if out is None:
            return BorderedVec(Fu, self.ma.pack(*s))
        V.copyto(out.u, Fu)
        out.p = self.ma.pack(*s)
        return out

    def J(self, z, p2):
        return _MAJacobian(self, z, p2)


class BorderingBLSHost:
    """BorderingBLS with check_precision = false (BEC, src/LinearBorderSolver.jl:125-144) over ANY linear solver and any vectors
    of the V interface: the `linear_algo` continuation_fold hands to PALC (MinAugFold.jl:446)."""

    def __init__(self, solver):
        self.solver = solver

    def __call__(self, J, dR, dzu, dzp, R, n, xiu=1.0, xip=1.0, shift=None, dotscale=1.0):
        assert shift is None
        x1, cv1, it1 = self.solver(J, R)
        dx, cv2, it2 = self.solver(J, dR)
        dl = (n - dotscale * V.dot(dzu, x1) * xiu) / (dzp * xip - dotscale * V.dot(dzu, dx) * xiu)
        V.axpby(x1, -dl, dx, 1.0)
        return x1, dl, bool(cv1 and cv2), (it1, it2)


@dataclass
class Codim2Point:
    """an entry of br.specialpoint on a codim-2 curve: type "bt" | "cusp", param = p2, p1, and the state of the located point"""
    type: str
    param: float
    p1: float
    step: int
    status: str      # converged | guess | guessL (locate_event!)
    interval: tuple
    x: object


def locate_event(it, _st, values_at, labels, indicator=None):
    """locate_event!(event, iter, state) (src/events/EventDetection.jl:28-235) for a ContinuousEvent whose indicator is the number of
    positive test functions (nb_signs): the bisection of events.bisection on that number, from the state `_st` just AFTER the
    event.  On return `_st` holds the located state (just after the event for an even number of reversals) and its predictor.
    values_at(st) -> tuple of test-function values at a state.  Returns (status, interval, label of the test function that changed
    at the last reversal)."""
    from . import events as E
    nb = indicator or (lambda vals: sum(1 for v in vals if v > 0))   # nb_signs: ContinuousEvent -> number of positive values;
    if abs(_st.ds) < it.contpar.dsmin:                                 # DiscreteEvent -> the value itself (EventDetection.jl:2-3)
        return "none", (0.0, 0.0), None
    seen = []                                 # (indicator, test-function values) at every state the bisection compares

    def count(s):
        vals = values_at(s)
        seen.append((nb(vals), vals))
        return seen[-1][0]

    status, interval, _, _ = E.bisection(it, _st, count)
    flips = [(a[1], b[1]) for a, b in zip(seen, seen[1:]) if a[0] != b[0]]
    if not flips:
        return status, interval, None
    prev, vals = flips[-1]
    changed = [k for k, (a_, b_) in enumerate(zip(prev, vals)) if ((a_ > 0) != (b_ > 0) if indicator is None else a_ != b_)]
    return status, interval, (labels[min(changed[0], len(labels) - 1)] if changed else None)


def _event(it, st, p2_prev, label, vals, values_at, labels, detect_event, indicator=None):
    """An event indicator of a codim-2 curve changed between the accepted point at p2_prev and the state `st`, whose test-function
    values are `vals` (label: the test function that changed).  detect_event = 1: a guess on the interval between the two points;
    > 1: located by locate_event(it, st, values_at, labels, indicator), after which `st` holds the located state, params[lens2]
    its p2 and `vals` its values_at.  Returns ((status, interval, label), or None where the bisection did not run; vals)."""
    from . import events as E
    if detect_event < 2:
        return ("guess", tuple(E.getinterval(p2_prev, st.z_p)), label), vals
    status, interval, lab = locate_event(it, st, values_at, labels, indicator)
    it.prob._set2(st.z_p)
    return (None if status == "none" else (status, tuple(interval), lab or label)), values_at(st)


def _continue_ma(pb, contpar, alg, normC, point, callback):
    """PALC on the MA problem `pb` in p2 = params[lens2] (MinAugFold.jl:446-457, MinAugHopf.jl:510-521): Newton linear solver
    MALinearSolver, outer bordered solver BorderingBLS(MALinearSolver, check_precision = false), no bifurcation detection on the
    MA system.  After every accepted point, with params[lens2] set to its p2: point(it, st), where False ends the curve, then the
    user's callback(st).  The parameter lists the curve writes are left as they were.  Returns (rows, state)."""
    from . import palc as P
    mls = MALinearSolver()
    no = contpar.newton_options
    cp = P.ContinuationPar(**{**contpar.__dict__, "newton_options": P.NewtonPar(tol=no.tol, max_iterations=no.max_iterations, linsolver=mls),
                              "detect_bifurcation": 0})
    alg = alg or P.PALC()
    alg = P.PALC(tangent=alg.tangent, theta=alg.theta, bls=BorderingBLSHost(mls))
    it = P.ContIterable(pb, alg, cp, normC)

    def cb(st):
        pb._set2(st.z_p)
        return point(it, st) is not False and (callback is None or callback(st))

    saved = [prob.params[pb.lens2] for prob in pb.ma.problems]
    try:
        return P.continuation(pb, alg, cp, normC=normC, callback=cb, it=it)
    finally:
        for prob, p2 in zip(pb.ma.problems, saved):
            prob.params[pb.lens2] = p2


@dataclass
class FoldCurve:
    rows: list      # palc rows: param = p2, x = record (default p1), itnewton, itlinear, ds, step
    p1: list        # the Fold curve (p1[k], p2[k])
    p2: list
    BT: list        # test function <w / ||w||, v / ||v||> at every point: zero at a Bogdanov-Takens point (test_bt_cusp)
    CP: list        # p2-component of the tangent, getp(state.tau) (test_bt_cusp): changes sign at a cusp, where p2 is extremal along the curve
    ma: object
    state: object
    specialpoint: list = None   # Codim2Point entries (detect_event > 0)


def test_zh(eigvals, tol_stability):
    """test_zh (MinAugFold.jl:533-543): Zero-Hopf test function on a Fold curve -- the number of eigenvalues of J(x, p) to the right
    of the (numerically) zero one with a positive imaginary part; a change between two points is a "zh" event"""
    if eigvals is None:
        return 1
    ev = np.asarray(eigvals)
    rho = float(np.min(np.abs(ev.real)))
    return int(np.sum((ev.real > rho) & (ev.imag > tol_stability)))


def continuation_fold(prob, x0, p1_0, lens2, eigenvec, eigenvec_ad, contpar, bls, alg=None, normC=V.norminf, symmetric=True,
                      update_minaug_every_step=1, record=None, callback=None, detect_event=0, eigsolver=None):
    """Codim-2 continuation of a Fold point in the parameters (p1 = params[prob.lens], p2 = params[lens2]):
    continuation_fold(prob, alg, foldpointguess, par, lens1, lens2, eigenvec, eigenvec_ad, options_cont; jacobian_ma = MinAug())
    (MinAugFold.jl:366-452).  PALC on the minimally augmented system, Newton linear solver = MALinearSolver over the
    bordered solver `bls` (bdlinsolver: MatrixFreeBLSB200 / BorderingBLSB200 on the device), outer bordered solver =
    BorderingBLS(that solver, check_precision = false), border vectors updated after every accepted step (update!), the
    Bogdanov-Takens and cusp test functions recorded along the curve.  detect_event = 1: a change of sign of a test function
    between two points is recorded as a special point ("bt" / "cusp", the event of :428-431); = 2: it is located by the reference's
    bisection (locate_event) with contpar.n_inversion / max_bisection_steps / dsmin_bisection, and the curve goes on from the
    located state, as in the reference.  eigsolver (J, nev) -> (eigenvalues, ...): eigenvalues of J along the curve (FoldEig, :577-590;
    contpar.nev of them) for the Zero-Hopf event "zh" (DiscreteEvent(1, test_zh), :431; recorded at the point after the change)."""
    from . import events as E
    ma = FoldMinAug(prob, eigenvec_ad, eigenvec, bls, symmetric=symmetric, norm=normC)
    pb = MAProblem(ma, lens2, BorderedVec(V.copy(x0), p1_0), record)
    curve = FoldCurve([], [], [], [], [], ma, None, [])
    zh_hist = []

    def values_at(s):   # test_bt_cusp at a state, the border vectors untouched
        pb._set2(s.z_p)
        return (ma.update(s.z_u.u, s.z_u.p, keep_borders=True), s.tau_p)

    def point(it, st):
        vals = (ma.update(st.z_u.u, st.z_u.p, keep_borders=st.step % update_minaug_every_step != 0), st.tau_p)
        if eigsolver is not None:
            zh = test_zh(eigsolver(prob.J(st.z_u.u, st.z_u.p), contpar.nev)[0], contpar.tol_stability)
            if detect_event > 0 and zh_hist and st.step > 0 and zh != zh_hist[-1]:
                curve.specialpoint.append(Codim2Point("zh", st.z_p, st.z_u.p, st.step, "guess", tuple(E.getinterval(curve.p2[-1], st.z_p)),
                                                      V.copy(st.z_u.u)))
            zh_hist.append(zh)
        if detect_event > 0 and curve.BT and st.step > 0:
            prev = (curve.BT[-1], curve.CP[-1])
            flips = [k for k in range(2) if (prev[k] > 0) != (vals[k] > 0)]
            if flips:
                found, vals = _event(it, st, curve.p2[-1], ("bt", "cusp")[flips[0]], vals, values_at, ("bt", "cusp"), detect_event)
                if found:
                    status, interval, label = found
                    curve.specialpoint.append(Codim2Point(label, st.z_p, st.z_u.p, st.step, status, interval, V.copy(st.z_u.u)))
        curve.p1.append(st.z_u.p)
        curve.p2.append(st.z_p)
        curve.BT.append(vals[0])
        curve.CP.append(vals[1])

    curve.rows, curve.state = _continue_ma(pb, contpar, alg, normC, point, callback)
    return curve


# ------------------------------------------------------------------------------------------------ Hopf
def _np(x):
    return x.numpy() if hasattr(x, "numpy") else np.asarray(x)


def _shifted(x, eps, d):
    """x + eps d for a real state x (NumPy array or DeviceVec) and a real NumPy direction d"""
    if hasattr(x, "ctx"):
        t = x.copy()
        t.axpby_(eps, x.ctx.to_device(d), 1.0)
        return t
    return x + eps * d


class ComplexProblemB200:
    """Complexified twin of a BifurcationProblemB200: the same stencil, grid and parameters on a BK_COMPLEX context.
    J(x, p, transpose) -> callable on complex vectors, consumable by ComplexGMRESB200."""

    def __init__(self, cctx, params, lens=0):
        assert cctx.complex
        self.ctx, self.params, self.lens = cctx, list(params), lens

    def J(self, x, p, transpose=False):
        q = list(self.params)
        q[self.lens] = p
        self.ctx.set_params(q)
        return self.ctx.cjacobian(x, transpose)


@dataclass
class HopfSolution:
    u: object
    p: float
    omega: float
    residuals: list
    converged: bool
    itnewton: int
    itlinear: int


class HopfMinAug:
    """[F(x, p); Re sigma; Im sigma](x, p, omega) with  [J - i omega, a; b^H, 0] [v; sigma] = [0; 1]
    (a ~ null vector of (J - i omega)^H, b ~ null vector of J - i omega)."""

    # the MA state's BorderedVec.p <-> (p1, omega), and the residual's (Re sigma, Im sigma) or a solve's (dp, domega) -> BorderedVec.p
    unpack = staticmethod(lambda zp: (float(zp[0]), float(zp[1])))
    pack = staticmethod(lambda sr, si: np.array([sr, si]))
    copy_rhs = True   # MALinearSolver hands solve() a copy of the right-hand side

    def __init__(self, prob, cprob, a, b, ls, cls, cbls=None):
        self.prob, self.cprob, self.ls, self.cls, self.cbls = prob, cprob, ls, cls, cbls
        self.problems = (prob, cprob)   # the problems whose params[lens2] a curve sets
        self.a, self.b = np.array(a, dtype=complex), np.array(b, dtype=complex)
        self.itlinear = 0

    def _border(self, Jc, shift, a, b):
        """(Jc + shift) v + a sigma = 0, <b, v> = 1 (linbdsolver(J, a, b, 0, zero, 1; shift), MinAugHopf.jl:17).  With a complex
        bordered solver `cbls(Jc, a, b, shift) -> (v, sigma, converged, iters)` (the reference's MatrixBLS / BorderingBLS on the
        bordered matrix, regular AT the Hopf point) that is one call; otherwise by bordering: y = (Jc + shift)^-1 a,
        sigma = -1 / <b, y>, v = -sigma y -- fine for an iterative solver next to the point, singular exactly on it."""
        if self.cbls is not None:
            v, sigma, cv, it = self.cbls(Jc, a, b, shift)
            self.itlinear += int(np.sum(it))
            return v, sigma
        y, cv, it = self.cls(Jc, a, a0=shift)
        self.itlinear += int(np.sum(it))
        sigma = -1.0 / np.vdot(b, y)
        return -sigma * y, sigma

    def residual(self, x, p, om):
        _, sigma = self._border(self.cprob.J(x, p), complex(0.0, -om), self.a, self.b)
        return self.prob.F(x, p), sigma.real, sigma.imag

    def bordered_terms(self, x, p, om):
        prob, cprob = self.prob, self.cprob
        eps = prob.delta
        v, _ = self._border(cprob.J(x, p), complex(0.0, -om), self.a, self.b)
        w, _ = self._border(cprob.J(x, p, transpose=True), complex(0.0, om), self.b, self.a)
        dpF = prob.F(x, p + eps)
        V.axpby(dpF, -1.0 / (2 * eps), prob.F(x, p - eps), 1.0 / (2 * eps))
        dpJv = (cprob.J(x, p + eps)(v) - cprob.J(x, p - eps)(v)) / (2 * eps)
        sigma_p = -np.vdot(w, dpJv)
        sigma_om = 1j * np.vdot(w, v)
        return v, w, dpF, sigma_p, sigma_om

    def solve(self, x, p, om, duu, dup, duom, cache=None):
        """_hopf_MA_linear_solver: [J dpF 0; sigma_x sigma_p sigma_om] [dX; dp; dom] = [duu; dup; duom].  `cache` is not used:
        the bordered terms are computed again for every right-hand side, as in the reference."""
        prob, cprob = self.prob, self.cprob
        eps = prob.delta
        v, w, dpF, sigma_p, sigma_om = self.bordered_terms(x, p, om)
        x1, x2, cv, it = self.ls(prob.J(x, p), duu, dpF)
        self.itlinear += int(np.sum(it))
        cw = np.conj(w)
        u1r = cprob.J(_shifted(x, eps, np.ascontiguousarray(v.real)), p, transpose=True)(cw)
        u1i = cprob.J(_shifted(x, eps, np.ascontiguousarray(v.imag)), p, transpose=True)(cw)
        u2 = cprob.J(x, p, transpose=True)(cw)
        sigma_x = -(u1r - u2) / eps + 1j * (-(u1i - u2) / eps)
        sxx1 = np.vdot(sigma_x, _np(x1))
        sxx2 = np.vdot(sigma_x, _np(x2))
        # the inner product conjugates its first argument: hence + Im(sxx2) and + Im(sxx1) (MinAugHopf.jl:180-186)
        LS = np.array([[(sigma_p - sxx2).real, sigma_om.real], [(sigma_p + sxx2).imag, sigma_om.imag]])
        rhs = np.array([dup - sxx1.real, duom + sxx1.imag])
        dp, dom = np.linalg.solve(LS, rhs)
        V.axpby(x1, -dp, x2, 1.0)
        return x1, float(dp), float(dom), cv

    def update(self, x, p, om):
        """update!(probma, iter, state) (MinAugHopf.jl:323-367): after an accepted step the border vectors follow the null
        vectors, a <- w / ||w||inf, b <- v / ||v||inf."""
        v, _ = self._border(self.cprob.J(x, p), complex(0.0, -om), self.a, self.b)
        w, _ = self._border(self.cprob.J(x, p, transpose=True), complex(0.0, om), self.b, self.a)
        self.a, self.b = w / float(np.max(np.abs(w))), v / float(np.max(np.abs(v)))


def newton_hopf(prob, cprob, x0, p0, omega0, eigenvec, eigenvec_ad, opts, ls, cls, normN=V.norm2, cbls=None):
    """Newton on the Hopf MA system from (x0, p0, omega0) with guesses for the i omega eigenvector and its adjoint
    (newton_hopf, MinAugHopf.jl:258-283 + src/Newton.jl:66-114 on the state (x, [p, omega]))."""
    ma = HopfMinAug(prob, cprob, eigenvec_ad, eigenvec, ls, cls, cbls)
    x, (p, om), _, residuals, step = _newton_ma(ma, x0, (p0, omega0), opts,
                                               lambda F, sr, si: math.sqrt(normN(F) ** 2 + sr * sr + si * si))
    return HopfSolution(x, p, om, residuals, residuals[-1] < opts.tol, step, ma.itlinear)


# ------------------------------------------------------------------------------------------------ Hopf curves in two parameters
@dataclass
class HopfCurve:
    rows: list
    p1: list        # the Hopf curve (p1[k], p2[k]) with the frequency omega[k]
    p2: list
    omega: list
    ma: object
    state: object
    stopped_at_bt: bool = False
    specialpoint: list = None   # Codim2Point entries: "zh" / "hh" (detect_event > 0 with an eigsolver)


def continuation_hopf(prob, cprob, x0, p1_0, omega0, lens2, eigenvec, eigenvec_ad, contpar, ls, cls, alg=None, normC=V.norminf,
                      update_minaug_every_step=1, record=None, callback=None, cbls=None, detect_event=0, eigsolver=None):
    """Codim-2 continuation of a Hopf point in (p1 = params[prob.lens], p2 = params[lens2]): continuation_hopf(prob, alg,
    hopfpointguess, par, lens1, lens2, eigenvec, eigenvec_ad, options_cont; jacobian_ma = MinAug()) (MinAugHopf.jl:425-522).
    PALC on the minimally augmented system in the state (x, [p1, omega]); Newton linear solver = MALinearSolver (one
    two-right-hand-side real solve + four complex shifted solves on the BK_COMPLEX twin `cprob`), outer bordered solver =
    BorderingBLS(that solver, check_precision = false); after every accepted step a <- w / ||w||, b <- v / ||v|| (update!,
    :323-367); the curve stops where omega -> 0 (Bogdanov-Takens, |omega| < 100 Newton tol).  With eigsolver (J, nev) -> (eigenvalues,
    ...) and detect_event > 0 the number of unstable eigenvalues of J along the curve is the reference's BifDetectEvent (:489-500,
    src/events/BifurcationDetection.jl:57-70; tol_stability raised to 10 x the Newton tolerance so that the Hopf pair itself does not
    count): a change is a Zero-Hopf ("zh", one real eigenvalue) or Hopf-Hopf ("hh", a second pair) point, recorded (1) or located by
    the event bisection (2).  The Bautin test function (first Lyapunov coefficient) needs normal forms and is not evaluated."""
    ma = HopfMinAug(prob, cprob, eigenvec_ad, eigenvec, ls, cls, cbls)
    pb = MAProblem(ma, lens2, BorderedVec(V.copy(x0), [p1_0, omega0]), record)
    curve = HopfCurve([], [], [], [], ma, None, specialpoint=[])
    tol = contpar.newton_options.tol
    tol_st = max(10 * tol, contpar.tol_stability)
    nhist = []

    def unstable_at(s):   # (n_unstable, n_imag) of J at the Hopf point of state s (is_stable, src/Bifurcations.jl:5-18)
        pb._set2(s.z_p)
        ev = np.asarray(eigsolver(prob.J(s.z_u.u, float(s.z_u.p[0])), contpar.nev)[0])
        un = ev.real > tol_st
        return (int(np.sum(un)), int(np.sum(un & (np.abs(ev.imag) > tol_st))))

    def point(it, st):
        if eigsolver is not None:
            nu = unstable_at(st)
            if detect_event > 0 and nhist and st.step > 0 and nu[0] != nhist[-1][0]:
                prev = nhist[-1]
                found, nu = _event(it, st, curve.p2[-1], None, nu, unstable_at, ("hh",), detect_event, indicator=lambda v: v[0])
                if found:
                    dn, di = abs(nu[0] - prev[0]), abs(nu[1] - prev[1])
                    curve.specialpoint.append(Codim2Point("zh" if dn == 1 else ("hh" if di == 2 else "nd"), st.z_p, ma.unpack(st.z_u.p)[0],
                                                          st.step, found[0], found[1], V.copy(st.z_u.u)))
            nhist.append(nu)
        p1, om = ma.unpack(st.z_u.p)
        if st.step % update_minaug_every_step == 0:
            ma.update(st.z_u.u, p1, om)
        curve.p1.append(p1)
        curve.p2.append(st.z_p)
        curve.omega.append(om)
        if abs(om) < 100 * tol:  # the frequency is null: not a Hopf point any more, the curve ends on a Bogdanov-Takens point
            curve.stopped_at_bt = True
            return False

    curve.rows, curve.state = _continue_ma(pb, contpar, alg, normC, point, callback)
    return curve
