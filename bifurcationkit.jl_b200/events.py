"""Bifurcation detection and location along a PALC branch (SURVEY 8f.2) -- host orchestration only.

What the reference does between two continuation steps when ``detect_bifurcation >= 2`` (src/Continuation.jl:506-560):
count unstable eigenvalues (``is_stable``, src/Bifurcations.jl:5-18), flag a change (``detect_bifurcation`` :21-28),
optionally locate it by bisection on the step size (``locate_bifurcation!`` :159-349, ``detect_bifurcation = 3``), classify
it from the change of (n_unstable, n_imag) (``get_bifurcation_type`` :70-150) and record a special point; folds by
parameter monotony when eigenvalues are not used (``locate_fold!`` :33-66).  The continuation steps, of the branch and of
the bisection, are those of ``palc.ContIterable`` -- the iterator ``palc.continuation`` runs -- so every linear solve and
eigen-solve still goes through the C ABI (``MatrixFreeBLSB200`` / ``BorderingBLSB200`` / ``ShiftInvertB200``).  The
bisection loop (``bisection``) also locates the events of codim-2 curves (``codim2.locate_event``).

State vectors are ``DeviceVec`` or ndarray through the ``V`` interface of palc.py; the three state copies the bisection keeps
(`before`, `after`, current) are device copies (4 vectors each).
"""
import copy as _copy
from dataclasses import dataclass, field

import numpy as np

from .palc import V, ContIterable, is_stable, _predict


# ------------------------------------------------------------------------------------------------ stability bookkeeping
def detect_bifurcation(st):
    """src/Bifurcations.jl:21-28"""
    n1, n2 = st.n_unstable
    if n1 == -1 or n2 == -1:
        return False
    return n1 != n2


def detect_fold(p1, p2, p3):
    """src/Bifurcations.jl:31"""
    return (p3 - p2) * (p2 - p1) < 0


def rightmost(ev):
    """src/Utils.jl:31: eigenvalues sorted by |real part|"""
    ev = np.asarray(ev, dtype=complex)
    return ev[np.argsort(np.abs(ev.real), kind="stable")]


def getinterval(a, b):
    return (min(a, b), max(a, b))


@dataclass
class SpecialPoint:
    """src/Results.jl SpecialPoint (fields the detection fills)"""
    type: str
    idx: int            # 0-based row of the branch holding the state recorded with the point
    param: float
    norm: float
    step: int
    status: str         # :guess, :guessL, :converged
    delta: tuple        # (change of n_unstable, change of n_imag)
    ind_ev: int
    interval: tuple
    x: object = None
    tau_p: float = 0.0
    precision: float = -1.0
    tau_u: object = None   # tangent at x (bifpt.τ.u), read by the Transcritical predictor (src/NormalForms.jl:410)


# ------------------------------------------------------------------------------------------------ state helpers
_VEC = ("z_u", "zold_u", "tau_u", "zpred_u")


def copy_state(st):
    """copy(state): src/Continuation.jl:196-212"""
    new = _copy.copy(st)
    for k in _VEC:
        setattr(new, k, V.copy(getattr(st, k)))
    return new


def copyto_state(dst, src):
    """copyto!(dest, src): src/Continuation.jl:214-240 (vectors copied into dst's own buffers)"""
    for k, v in vars(src).items():
        if k in _VEC:
            V.copyto(getattr(dst, k), v)
        else:
            setattr(dst, k, v)
    return dst


def _is_on_boundary(contpar, p):
    return p == contpar.p_min or p == contpar.p_max


# ------------------------------------------------------------------------------------------------ classification
def get_bifurcation_type(it, st, status, interval, floquet=False):
    """src/Bifurcations.jl:70-150 -> SpecialPoint (raises as the reference `throw`s when nothing changed)"""
    n_unstable, n_unstable_prev = st.n_unstable
    n_imag, n_imag_prev = st.n_imag
    ind_ev = n_unstable_prev if n_unstable < n_unstable_prev else n_unstable
    tp, known = "none", False
    dn, di = abs(n_unstable - n_unstable_prev), abs(n_imag - n_imag_prev)
    if dn == 1:
        tp = "bp" if di == 0 else (("pd" if floquet else "hopf") if di == 1 else "nd")
        known = True
    elif dn == 2:
        tp = ("ns" if floquet else "hopf") if di == 2 else "nd"
        known = True
    elif dn > 2:
        tp, known = "nd", True
    if dn < di:
        tp, known = "nd", True
    if st.n_unstable[0] * st.n_unstable[1] < 0 or st.n_imag[0] * st.n_imag[1] < 0:
        tp, known = "nd", True
    if not known:
        raise RuntimeError(f"We could not detect/identify the bifurcation point. (dn_unstable, dn_imag) = ({dn}, {di})")
    return SpecialPoint(type=tp, idx=st.step, param=st.z_p, norm=it.normC(st.z_u), step=st.step, status=status,
                        delta=(n_unstable - n_unstable_prev, n_imag - n_imag_prev), ind_ev=ind_ev, interval=tuple(interval),
                        x=V.copy(st.z_u), tau_p=st.tau_p, precision=abs(interval[1] - interval[0]), tau_u=V.copy(st.tau_u))


def locate_fold(rows, specialpoints, it, st):
    """src/Bifurcations.jl:33-66 (called before the current state is saved: rows[-1] is the previous point)"""
    cp = it.contpar
    if cp.detect_fold and len(rows) > 2 and detect_fold(rows[-3]["param"], rows[-2]["param"], rows[-1]["param"]):
        specialpoints.append(SpecialPoint(type="fold", idx=len(rows) - 2, param=st.z_p, norm=it.normC(st.z_u), step=len(rows) - 2,
                                          status="guess", delta=(0, 0), ind_ev=0, interval=(rows[-2]["param"], rows[-2]["param"]),
                                          x=V.copy(st.z_u), tau_p=st.tau_p, tau_u=V.copy(st.tau_u)))
        return True
    return False


# ------------------------------------------------------------------------------------------------ bisection
def bisection(it, _st, indicator, located=None):
    """The bisection on ds of locate_bifurcation! (src/Bifurcations.jl:159-349) and locate_event! (src/events/
    EventDetection.jl:28-235) from the state `_st` just after a change of `indicator(state)`: half a step back, then ds halved
    at every step and reversed at every change of the indicator, until contpar.n_inversion reversals, max_bisection_steps,
    dsmin_bisection or `located(state)`.  The steps are it.iterate without step-size control.  On return `_st` holds the
    located state (just after the point for an even number of reversals) and its predictor.  Returns (status in {converged,
    guess, guessL}, interval, the located state, the state on the other side of the point)."""
    cp = it.contpar
    marks = [indicator(_st)]
    after, st, before = copy_state(_st), copy_state(_st), copy_state(_st)
    st.in_bisection = True
    before.n_unstable = (before.n_unstable[1], before.n_unstable[0])   # `before` is the previous point until a reversal
    before.n_imag = (before.n_imag[1], before.n_imag[0])
    before.zold_p, before.z_p = before.z_p, before.zold_p
    st.ds *= -1
    st.step = 0
    st.stepsizecontrol = False
    interval = list(getinterval(st.z_p, st.zold_p))
    indinterval = 0 if interval[0] == st.z_p else 1
    n_inversion, alive = 0, True
    while st.converged and alive:      # a failed Newton step or the end of the branch ends the bisection
        marks.append(indicator(st))
        if marks[-1] == marks[-2]:
            st.ds /= 2                 # the point is still before the current state, keep going
        else:
            st.ds /= -2                # passed it: reverse
            n_inversion += 1
            indinterval = 1 - indinterval
        _predict(st)                   # update_predictor!
        copyto_state(after if n_inversion % 2 == 0 else before, st)
        if st.step > 0:
            interval[indinterval] = st.z_p
        if not (abs(st.ds) >= cp.dsmin_bisection and st.step < cp.max_bisection_steps and n_inversion < cp.n_inversion
                and not (located is not None and located(st))):
            break
        alive = it.iterate(st)
    if n_inversion % 2 == 0:
        status, here, there = ("converged" if n_inversion >= cp.n_inversion else "guess"), st, before
    else:
        status, here, there = "guessL", after, st
    for k in _VEC:
        V.copyto(getattr(_st, k), getattr(here, k))
    _st.z_p, _st.zold_p, _st.tau_p, _st.zpred_p = here.z_p, here.zold_p, here.tau_p, here.zpred_p
    _st.work_newton, _st.work_linear = st.work_newton, st.work_linear   # the bisection's corrector work is real work
    _predict(_st)                      # update_predictor!(_state, iter) with the outer ds
    return status, getinterval(st.z_p, (after if n_inversion % 2 else before).z_p), here, there


def locate_bifurcation(it, _st):
    """locate_bifurcation!(iter, state) (src/Bifurcations.jl:159-349): bisection on the number of unstable eigenvalues, which
    also stops at an eigenvalue within tol_bisection_eigenvalue of the imaginary axis; on return `_st` sits just after the
    bifurcation point (or is restored to `after`), status in {guess, guessL, converged, none}."""
    assert detect_bifurcation(_st), "No bifurcation detected for the state"
    cp = it.contpar
    n2, n1 = _st.n_unstable
    if n1 == -1 or n2 == -1 or abs(_st.ds) < cp.dsmin:
        return "none", (0.0, 0.0)
    status, interval, here, there = bisection(it, _st, lambda s: s.n_unstable[0],
                                              lambda s: abs(rightmost(s.eigvals).real[0]) < cp.tol_bisection_eigenvalue)
    _st.n_unstable = (here.n_unstable[0], there.n_unstable[0])
    _st.n_imag = (here.n_imag[0], there.n_imag[0])
    _st.eigvals, _st.eigvecs = here.eigvals, here.eigvecs
    return status, interval


# ------------------------------------------------------------------------------------------------ driver
@dataclass
class Branch:
    rows: list = field(default_factory=list)
    specialpoint: list = field(default_factory=list)
    eig: list = field(default_factory=list)
    state: object = None


def branch_row(prob, cp, st):
    """get_state_summary (src/Continuation.jl:259-272): the row a branch keeps for the state st"""
    stable, _, _ = is_stable(cp, st.eigvals)
    return dict(param=st.z_p, x=prob.record(st.z_u), itnewton=st.itnewton, itlinear=st.itlinear, ds=st.ds, step=st.step,
                n_unstable=st.n_unstable[0], n_imag=st.n_imag[0], stable=stable)


def continuation(prob, alg, contpar, normC=V.norm2, verbose=False, callback=None, floquet=False, u1=None, p1=None):
    """continuation(prob, PALC(...), ContinuationPar(detect_bifurcation = 0..3)) with special points
    (src/Continuation.jl:349-400 start-up, :506-575 loop): the loop of palc.continuation with the detection before each
    row is saved.  With (u1, p1) the branch starts from the two points (prob.u0, prob.p0), (u1, p1) (iterate_from_two_points,
    src/Continuation.jl:408-456), as branch switching does.  Returns a Branch (rows as palc.continuation + `n_imag`, `stable`;
    specialpoint list ends with the :endpoint)."""
    cp = contpar
    it = ContIterable(prob, alg, cp, normC)
    st = it.start(u1, p1)
    it.eigen(st)
    br = Branch(state=st)

    def save():
        br.rows.append(branch_row(prob, cp, st))
        if st.eigvals is not None:
            br.eig.append(dict(eigenvals=np.array(st.eigvals), step=st.step))
            if cp.save_eigenvectors and st.eigvecs is not None:
                br.eig[-1]["eigenvecs"] = np.array(st.eigvecs)
        if callback is not None and callback(st) is False:
            st.stop = True

    save()
    status = "guess"
    while it.iterate(st):
        if verbose:
            print(f"step {st.step} p={st.z_p:.6e} ds={st.ds:.3e} conv={st.converged} itn={st.itnewton} n_unstable={st.n_unstable}", flush=True)
        if not (st.converged and st.step <= cp.max_steps):
            continue
        if cp.detect_fold and cp.detect_bifurcation < 2:
            locate_fold(br.rows, br.specialpoint, it, st)
        if cp.detect_bifurcation > 1 and detect_bifurcation(st):
            interval = getinterval(st.zold_p, st.z_p)
            if cp.detect_bifurcation > 2 and not _is_on_boundary(cp, st.z_p):
                status, interval = locate_bifurcation(it, st)
            if detect_bifurcation(st):   # the bisection may have moved the state before the point
                bp = get_bifurcation_type(it, st, status, interval, floquet)
                if bp.type != "none":
                    br.specialpoint.append(bp)
                if verbose:
                    print(f"--> {bp.type} bifurcation point at p ~ {bp.param:.8g} in {bp.interval}, delta = {bp.delta}, {bp.status}", flush=True)
        save()
    br.specialpoint.append(SpecialPoint(type="endpoint", idx=len(br.rows) - 1, param=st.z_p, norm=normC(st.z_u), step=st.step,
                                        status="converged", delta=(0, 0), ind_ev=0, interval=(st.z_p, st.z_p)))
    return br
