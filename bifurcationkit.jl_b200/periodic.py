"""Branches of periodic orbits with the Trapeze functional, and branch switching to them from a Hopf point -- host
orchestration over the C ABI, like normalform.py.  The orbit x = [x_1 .. x_M; T] lives in a BK_POTRAP_CGL2D context
(include/bk200.h): its residual, Jacobian, bordered solves and time-circulant preconditioner are that context's kernels, and
the section of the phase condition is updated on the device by bk_potrap_update_section.

Mirror of the reference:
  TrapezeProblemB200      <->  PeriodicOrbitFunctionalTrap over Trapeze(...; update_section_every_step)
                                 src/periodicorbit/PeriodicOrbitTrapeze.jl:150-200, 1042-1050
  TrapezeProblemB200.update <->  update!(wrap, iter, state)              src/periodicorbit/PeriodicOrbits.jl:156-169
                                 with updatesection! (PeriodicOrbitTrapeze.jl:665-679) and mod_counter (src/Utils.jl:183)
  FloquetEigB200          <->  FloquetQaD as the eigensolver of the PO branch (PeriodicOrbitTrapeze.jl:960, 973-976)
  continuation_po         <->  continuation(trap::Trapeze, orbitguess, alg, opts)  PeriodicOrbitTrapeze.jl:955-1052
  continuation_from_hopf  <->  continuation(br, ind_hopf, opts, disc)    PeriodicOrbits.jl:395-410
  continuation_from_hopf_point <-> _continuation(hopfpt, ...)              PeriodicOrbits.jl:412-514, without usedeflation, with
                                 the orbit form of re_make (PeriodicOrbitTrapeze.jl:1056-1084)

  continuation_po_events  <->  the same continuation with event detection (src/Continuation.jl:506-575): folds of cycles by
                                 parameter monotony (detect_bifurcation < 2, :522-528) or from the Floquet multipliers
  fold_point              <->  fold_point(br, index)                     src/codim2/MinAugFold.jl:6-13
  newton_fold_po          <->  newton_fold(br_po, indfold; prob, bdlinsolver)  MinAugFold.jl:236-262, examples/cGL2d.jl:352-379
  continuation_fold_po    <->  continuation_fold(prob, br_po, indfold, lens2, opts)  MinAugFold.jl:369-452, 460ff,
                                 examples/cGL2d.jl:381-390
The folds of cycles need J' of the Trapeze functional: the context applies it (bk_jac_set_transpose) and its circulant
preconditioner then applies P'^-1, so every adjoint solve of the minimally augmented problem runs on the device.

Not here: branch switching at period-doubling or Neimark-Sacker points and their curves, usedeflation, shooting, collocation
and non-uniform time meshes.
"""
import ctypes as C
from dataclasses import replace
import math

import numpy as np

from . import lib as _l
from . import codim2, events
from .core import _chk, BorderingBLSB200, DeviceVec
from .floquet import cgl_shifted_precond, period
from .normalform import hopf_normal_form, predictor
from .palc import V, SQRT_EPS, BifurcationProblemB200, PALC, continuation


def mod_counter(step, every):
    """mod_counter(step, everyN) (src/Utils.jl:183-188)"""
    if step == 0 or every == 0:
        return False
    if every == 1:
        return True
    return step % every == 0


def amplitude(x):
    """max |x_i| over the slices (the period excluded)"""
    if isinstance(x, DeviceVec):
        res = C.c_double()
        _chk(x.ctx, x.ctx.lib.bk_vec_norminf(x.ctx.handle, x.dptr, x.n - 1, C.byref(res)))
        return res.value
    return float(np.max(np.abs(x[:-1])))


class TrapezeProblemB200(BifurcationProblemB200):
    """The Trapeze functional of a BK_POTRAP_CGL2D context as a continuation problem (PeriodicOrbitFunctionalTrap).

    M: number of time slices (the context's third dimension).  update_section_every_step: 0 (the reference's default) keeps the
    section; k > 0 updates it after every k-th converged step.  circulant: the Newton linear solver is preconditioned by
    BK_PC_POTRAP_CIRC, which is then set up at the period and parameters of the orbit guess and again at those of every
    converged point.  record: the period
    x[end] (PeriodicOrbitTrapeze.jl:1047) and the amplitude max |x_i| over the slices (examples/cGL2d.jl records
    maximum(solpo.u), the largest entry rather than the largest modulus)."""

    def __init__(self, ctx, u0, params, lens=0, update_section_every_step=0, circulant=False, delta=SQRT_EPS, M=None):
        super().__init__(ctx, u0, params, lens, record=self.record_po, delta=delta)
        self.M = int(ctx.dims[2]) if M is None else int(M)
        self.update_section_every_step, self.circulant = int(update_section_every_step), bool(circulant)
        self.last_state = self.last_p = None
        self.section_updates = 0

    @staticmethod
    def record_po(x):
        return dict(period=period(x), amplitude=amplitude(x))

    def J(self, x, p):
        self.last_state, self.last_p = x, p    # the orbit of the last Jacobian, for the Floquet eigensolver
        return super().J(x, p)

    def update_section(self, x, scale):
        """phi_i = scale F(x_i), xpi = x without the period, at the current params (bk_potrap_update_section)"""
        self.ctx.potrap_update_section(x, scale)

    def setup_precond(self, x):
        """BK_PC_POTRAP_CIRC at the period of x and the current params"""
        self.ctx.precond_setup(_l.BK_PC_POTRAP_CIRC, period(x))

    def update(self, st):
        """update!(wrap, iter, state) (PeriodicOrbits.jl:156-169) after a converged continuation step: the section when
        mod_counter(step, update_section_every_step), outside a bisection; then the circulant preconditioner.  The reference
        calls it before it counts the step, so `step` there is st.step - 1 here."""
        if st.step < 1 or not st.converged:
            return True
        if mod_counter(st.step - 1, self.update_section_every_step) and not st.in_bisection:
            self._set(st.z_p)
            self.update_section(st.z_u, 1.0 / self.M)
            self.section_updates += 1
        if self.circulant:
            self._set(st.z_p)
            self.setup_precond(st.z_u)
        return True


class FloquetEigB200:
    """The eigensolver of a periodic-orbit branch: ContIterable.eigen calls eig(prob.J(x, p), nev); this runs the Floquet
    solver `floquet` (floquet.FloquetQaDB200 over a BK_CGL2D context of the same grid) on the orbit of that Jacobian, with the
    vector field's params set to those of the orbit and its shifted preconditioner (floquet.cgl_shifted_precond) at the
    orbit's period.  Returns the Floquet exponents log(mu), so is_stable counts the multipliers outside the unit circle."""

    def __init__(self, trap, floquet):
        self.trap, self.floquet = trap, floquet

    def __call__(self, J, nev):
        trap, fl = self.trap, self.floquet
        q = list(trap.params)
        q[trap.lens] = trap.last_p
        fl.ctx.set_params(q)
        cgl_shifted_precond(fl.ctx, period(trap.last_state), trap.M, q[0])
        return fl(trap.last_state, nev)


def _po_setup(trap, orbitguess, alg, contpar, bls, floquet, callback):
    """what continuation(trap::Trapeze, ...) sets up before it continues: the bordered solver, the Floquet eigensolver, the
    start at the guess, the circulant preconditioner there and the section hook"""
    assert period(orbitguess) >= 0, "The guess for the period should be positive"
    ls = contpar.newton_options.linsolver
    alg = replace(alg, bls=bls or BorderingBLSB200(ls, check_precision=False))
    if contpar.detect_bifurcation > 0:
        assert floquet is not None, "detect_bifurcation > 0 needs a Floquet solver"
        contpar = replace(contpar, newton_options=replace(contpar.newton_options, eigsolver=FloquetEigB200(trap, floquet)))
    trap.u0, trap.p0 = orbitguess, float(trap.params[trap.lens])
    if trap.circulant:
        trap._set(trap.p0)
        trap.setup_precond(orbitguess)

    def hook(st):
        ok = trap.update(st)
        if callback is not None and callback(st) is False:
            return False
        return ok
    return alg, contpar, hook


def continuation_po(trap, orbitguess, alg, contpar, normC=V.norminf, bls=None, floquet=None, callback=None, verbose=False):
    """continuation(trap::Trapeze, orbitguess, alg, opts) (PeriodicOrbitTrapeze.jl:955-1052) on palc.continuation from the
    orbit guess at trap's parameter.  bls: the bordered solver, by default BorderingBLSB200(check_precision = False) over the
    Newton linear solver (:1050).  floquet: a floquet.FloquetQaDB200, the eigensolver when contpar.detect_bifurcation >= 1
    (:960, 973-976).  The section hook trap.update runs after every converged step, before `callback`.  Returns (rows, state):
    rows as palc.continuation, with x = dict(period, amplitude) and n_unstable from the Floquet exponents."""
    alg, contpar, hook = _po_setup(trap, orbitguess, alg, contpar, bls, floquet, callback)
    return continuation(trap, alg, contpar, normC, verbose=verbose, callback=hook)


def continuation_po_events(trap, orbitguess, alg, contpar, normC=V.norminf, bls=None, floquet=None, callback=None, verbose=False):
    """continuation_po with the special points of events.continuation: folds of cycles by parameter monotony when
    contpar.detect_bifurcation < 2 (contpar.detect_fold), otherwise from the change of the number of Floquet multipliers outside
    the unit circle, named bp / pd / ns (src/Continuation.jl:522-528, src/Bifurcations.jl:70-150); a fold of cycles, where one
    real multiplier crosses 1, is a "bp" there.  Same set-up, section hook and rows as continuation_po.  Returns an
    events.Branch (rows, specialpoint, state)."""
    alg, contpar, hook = _po_setup(trap, orbitguess, alg, contpar, bls, floquet, callback)
    return events.continuation(trap, alg, contpar, normC, verbose=verbose, callback=hook, floquet=True)


def fold_point(br, ind):
    """fold_point(br, index) (MinAugFold.jl:6-13): the state and parameter of br.specialpoint[ind], a fold / bp / nd point"""
    bp = br.specialpoint[ind]
    if bp.type not in ("bp", "nd", "fold"):
        raise ValueError(f"This should be a Fold / BP point.\nYou passed a {bp.type} point.")
    return V.copy(bp.x), float(bp.param)


def _fold_start(trap, br, ind, normN, update_section):
    """the guess of newton_fold(br, ind) (MinAugFold.jl:245-248) for an orbit: fold_point, eigenvec = τ.u / normN(τ.u),
    eigenvec_ad a copy; before that the section is updated at the guess and its parameter (updatesection!, scale 1/M,
    examples/cGL2d.jl:364) and the circulant preconditioner is set up there"""
    x0, p0 = fold_point(br, ind)
    tau = br.specialpoint[ind].tau_u
    assert tau is not None, "the special point carries no tangent (tau_u)"
    trap._set(p0)
    if update_section:
        trap.update_section(x0, 1.0 / trap.M)
    if trap.circulant:
        trap.setup_precond(x0)
    eigenvec = V.copy(tau)
    V.scale(eigenvec, 1.0 / normN(eigenvec))
    return x0, p0, eigenvec, V.copy(eigenvec)


def newton_fold_po(trap, br, ind, opts, bls, normN=V.norm2, update_section=True):
    """newton_fold(br_po, indfold; prob, options, bdlinsolver) (MinAugFold.jl:236-262) for a fold of cycles of the Trapeze
    branch br (continuation_po_events), as examples/cGL2d.jl:352-379 runs it: the section updated at the guess, then Newton on
    the minimally augmented Fold system with J' from the context (symmetric = False).  opts: NewtonPar whose linsolver is the
    GMRES of the bordered solves; bls: the bordered solver (BorderingBLSB200(ls, check_precision = False) in the example).
    Returns a codim2.FoldSolution (u = the orbit, p = the fold's parameter)."""
    x0, p0, ev, ev_ad = _fold_start(trap, br, ind, normN, update_section)
    return codim2.newton_fold(trap, x0, p0, ev, ev_ad, opts, bls, normN=normN, symmetric=False)


def continuation_fold_po(trap, br, ind, lens2, contpar, bls, normN=V.norm2, normC=V.norminf, update_section=True, callback=None,
                         **kw):
    """continuation_fold(prob, br_po, indfold, lens2, opts; jacobian_ma = MinAug(), bdlinsolver) (MinAugFold.jl:369-452, 460ff;
    examples/cGL2d.jl:381-390): the fold of cycles continued in (trap's parameter, params[lens2]) by codim2.continuation_fold with
    J' from the context, from the guess of newton_fold_po.  The section stays that of the guess along the curve, as in the
    reference; the circulant preconditioner is set up again at the period and parameters of every accepted point.  Other
    keywords go to codim2.continuation_fold.  Returns a codim2.FoldCurve."""
    x0, p0, ev, ev_ad = _fold_start(trap, br, ind, normN, update_section)

    def cb(st):
        if trap.circulant:
            trap.params[lens2] = st.z_p
            trap._set(st.z_u.p)
            trap.setup_precond(st.z_u.u)
        return True if callback is None else callback(st)
    return codim2.continuation_fold(trap, x0, p0, lens2, ev, ev_ad, contpar, bls, normC=normC, symmetric=False, callback=cb, **kw)


def continuation_from_hopf(it, br, ind_hopf, contpar, trap, ds=None, ampfactor=1.0, detailed=True, nev=None, cprob=None, cls=None,
                           **kw):
    """continuation(br, ind_hopf, opts, disc) (PeriodicOrbits.jl:395-410): the Hopf normal form of br.specialpoint[ind_hopf]
    (normalform.hopf_normal_form over the iterator `it` of the branch; nev, detailed, cprob, cls as there), then
    continuation_from_hopf_point.  Returns (rows, state, HopfNF, predictor)."""
    hp = hopf_normal_form(it, br, ind_hopf, nev=nev, detailed=detailed, cprob=cprob, cls=cls)
    return continuation_from_hopf_point(hp, contpar, trap, ds=ds, ampfactor=ampfactor, **kw)


def continuation_from_hopf_point(hp, contpar, trap, ds=None, ampfactor=1.0, alg=None, normC=V.norminf, bls=None, floquet=None,
                                 callback=None, verbose=False, with_events=False):
    """_continuation(hopfpt, prob, opts, disc) (PeriodicOrbits.jl:412-514) without usedeflation: the predictor of the HopfNF hp
    at ds (contpar.ds by default) and ampfactor, the guess orbit(t - ϕ) on the M times LinRange(0, 2π, M + 1)[1:M] with
    ϕ = atan(<ζr, ζr>, <ζi, ζr>) and the period |2π / ω|, the section of that guess (the orbit form of re_make: phi_i = F(x_i),
    xpi = the guess, at the predictor's parameter), then continuation_po from it (alg, normC, bls, floquet, callback as there).
    trap: a TrapezeProblemB200 whose lens is the Hopf point's parameter; its params are set to the predictor's, and a device
    problem keeps the branch on the device.  Returns (rows, state, hp, predictor); with with_events = True the continuation is
    continuation_po_events and `rows` is its events.Branch (folds of cycles among its special points)."""
    ds = contpar.ds if ds is None else ds
    pred = predictor(hp, ds, ampfactor)
    zr, zi = np.real(hp.zeta), np.imag(hp.zeta)
    phase = math.atan2(float(np.dot(zr, zr)), float(np.dot(zi, zr)))                     # :419
    M = trap.M
    ts = np.linspace(0.0, 2 * np.pi, M + 1)[:M]
    guess = np.concatenate([pred.orbit(t - phase) for t in ts] + [np.array([abs(2 * np.pi / pred.omega)])])
    if trap.ctx is not None:    # a device problem keeps the branch on the device
        guess = trap.ctx.to_device(guess)
    trap.params[trap.lens] = pred.p
    trap._set(pred.p)
    trap.update_section(guess, 1.0)                                                     # re_make(...; orbit), :1077-1080
    if with_events:
        br = continuation_po_events(trap, guess, alg or PALC(), contpar, normC, bls=bls, floquet=floquet, callback=callback,
                                    verbose=verbose)
        return br, br.state, hp, pred
    rows, st = continuation_po(trap, guess, alg or PALC(), contpar, normC, bls=bls, floquet=floquet, callback=callback,
                               verbose=verbose)
    return rows, st, hp, pred
