"""Normal form of a simple branch point and automatic branch switching (aBS) from it -- host orchestration over the C ABI,
like codim2.py.  Every linear solve is a bordered solve (`MatrixFreeBLSB200` by default), every eigen-solve the branch's
eigensolver, every second / third differential a `bk_d2f` / `bk_d3f` call (BifurcationProblemB200.d2F / d3F); host problems
bring their own d2F / d3F, J and, when not symmetric, Jt.

Mirror of the reference:
  get_normal_form1d      <->  get_normal_form1d, autodiff = false           src/NormalForms.jl:189-353
  (adjoint eigenvector)  <->  get_adjoint_basis(L★, λ::Number, eigsolver)    src/NormalForms.jl:31-49
  predictor              <->  predictor(::Transcritical / ::Pitchfork / ::Fold, ds)  src/NormalForms.jl:389-493
  continuation_from_bp   <->  continuation(br, ind_bif, options_cont)       src/bifdiagram/BranchSwitching.jl:74-198, :8-44

Not here: kernels of dimension > 1 (get_normal_formNd, multicontinuation), the generic BranchPoint predictor (_predictor,
src/NormalForms.jl:496-535), usedeflation, bothside and bifurcationdiagram; Hopf and higher codimension normal forms.
"""
import copy
from dataclasses import dataclass, replace
import math
import types
import warnings

import numpy as np

from .codim2 import _apply
from .core import DeviceVec, ShiftInvertB200, MatrixFreeBLSB200
from .palc import V, ContIterable
from . import events


@dataclass
class BranchPointNF:
    """Transcritical / Pitchfork / Fold / BranchPoint of src/NormalForms.jl:340-350 (fields of AbstractSimpleBranchPoint):
    the point (x0, p), the tangent there (tau_u, tau_p), the kernel vector zeta, the adjoint vector zeta_ad with
    <zeta, zeta_ad> = 1 and the coefficients of the reduced equation
    a01 dp + a02 dp^2 / 2 + b11 x dp + b20 x^2 / 2 + b30 x^3 / 6, plus Psi01 and Psi20."""
    type: str
    x0: object
    p: float
    tau_u: object
    tau_p: float
    zeta: object
    zeta_ad: object
    nf: dict
    bptype: str = "NA"   # BranchPoint only: NonQuadraticParameter when |a02| < tol_fold


def _like(x, a):
    """host array a -> the container type of x"""
    a = np.ascontiguousarray(np.real(a), dtype=np.float64)
    return x.ctx.to_device(a) if isinstance(x, DeviceVec) else a


def _eig(eigsolver, J, nev):
    """eigsolver(J, nev) with eigenvectors: (vals, vecs as columns)"""
    out = eigsolver(J, nev, want_vectors=True) if isinstance(eigsolver, ShiftInvertB200) else eigsolver(J, nev)
    return np.asarray(out[0]), out[1]


def _isapprox(a, b):
    """Julia's a ≈ b with the default rtol = sqrt(eps)"""
    return a == b or abs(a - b) <= math.sqrt(np.finfo(float).eps) * max(abs(a), abs(b))


def _E(x, zeta, zeta_ad):
    """E(x) = x - <x, zeta_ad> zeta, in place (src/NormalForms.jl:178)"""
    return V.axpby(x, -V.dot(x, zeta_ad), zeta, 1.0)


def _adjoint_vector(prob, x0, p, lam, eigsolver, nev):
    """get_adjoint_basis(L★, conj(λ), eigsolver; nev) (src/NormalForms.jl:31-49): the eigenvector of J' whose eigenvalue is
    closest to conj(λ).  J' is prob.Jt for host problems and J under bk_jac_set_transpose on the device."""
    if hasattr(prob, "Jt"):
        vals, vecs = _eig(eigsolver, prob.Jt(x0, p), nev)
    else:
        prob.ctx.set_transpose(True)
        try:
            vals, vecs = _eig(eigsolver, prob.J(x0, p), nev)
        finally:
            prob.ctx.set_transpose(False)
    i = int(np.argmin(np.abs(vals - np.conj(lam))))
    if abs(vals[i].real) > 1e-2:
        warnings.warn(f"The bifurcating eigenvalue is not that close to Re = 0. We found {vals[i].real} !≈ 0. "
                      "You can perhaps increase the argument `nev`.")
    return _like(x0, np.asarray(vecs)[:, i])


def _eigvals_at(br, bifpt):
    return next(e["eigenvals"] for e in br.eig if e["step"] == bifpt.idx)


def get_normal_form1d(it, br, ind_bif, nev=None, zeta=None, zeta_ad=None, bls=None, tol_fold=1e-3):
    """get_normal_form1d(prob, br, ind_bif; autodiff = false) (src/NormalForms.jl:189-353) for the branch `br` computed by
    events.continuation over the iterator `it` (its problem and Newton options).  `ind_bif` indexes br.specialpoint.  The
    parameter derivatives are central differences with prob.delta.  zeta / zeta_ad: the kernel and adjoint vectors (ζs, ζs_ad of
    the reference); otherwise the eigenpairs at the point are recomputed with newton_options.eigsolver.  bls: the bordered solver
    of the two singular systems, MatrixFreeBLSB200 over the Newton linear solver by default (J is singular there, so a bordering
    solver cannot be).  Returns a BranchPointNF."""
    prob, options = it.prob, it.contpar.newton_options
    bifpt = br.specialpoint[ind_bif]
    if bifpt.type not in ("bp", "fold"):
        raise ValueError("The provided index does not refer to a Branch Point with 1d kernel. "
                         f"The type of the bifurcation is {bifpt.type}.")
    if abs(bifpt.delta[0]) > 1:
        raise ValueError("We only provide normal form computation for simple bifurcation points e.g. when the kernel of the "
                         f"jacobian is 1d. Here, the dimension of the kernel is {abs(bifpt.delta[0])}.")
    bls = bls or MatrixFreeBLSB200(options.linsolver)
    x0, p, delta = bifpt.x, bifpt.param, prob.delta                                      # :223-230
    saved = np.asarray(_eigvals_at(br, bifpt))
    nev = len(saved) if nev is None else nev
    lam = float(np.real(saved[bifpt.ind_ev - 1]))                                        # :236 (ind_ev is 1-based)
    if zeta is None:                                                                     # :243-256
        nev_required = max(nev, bifpt.ind_ev + 2)
        vals, vecs = _eig(options.eigsolver, prob.J(x0, p), nev_required)
        if not _isapprox(vals[bifpt.ind_ev - 1], lam):
            raise RuntimeError(f"We did not find the correct eigenvalue {lam}. We found {vals}")
        zeta = _like(x0, np.asarray(vecs)[:, bifpt.ind_ev - 1])
    else:
        zeta = _like(x0, zeta) if isinstance(zeta, (list, np.ndarray)) else V.copy(zeta)
    V.scale(zeta, 1.0 / V.norm2(zeta))                                                   # scaleζ = norm, :257
    if zeta_ad is not None:                                                              # :260-272
        zeta_ad = _like(x0, zeta_ad) if isinstance(zeta_ad, (list, np.ndarray)) else V.copy(zeta_ad)
    elif getattr(prob, "symmetric", False):
        zeta_ad = V.copy(zeta)
    else:
        zeta_ad = _adjoint_vector(prob, x0, p, lam, options.eigsolver, nev)
    zz = V.dot(zeta, zeta_ad)
    if not abs(zz) > 1e-10:                                                              # :275-277
        raise RuntimeError(f"We got ζ⋅ζ★ = {zz}.\nThis dot product should not be zero.\n"
                           f"Perhaps, you can increase `nev` which is currently {nev}.")
    V.scale(zeta_ad, 1.0 / zz)

    R2 = lambda a, b: prob.d2F(x0, p, a, b)
    R3 = lambda a, b, c: prob.d3F(x0, p, a, b, c)
    dF = lambda q, v: _apply(prob.J(x0, q), v)

    def solve(rhs):  # bls(L, ζ★, ζ, 0, E(-rhs), 0): L is re-made before each solve (a device context keeps one Jacobian)
        r = V.scale(V.copy(rhs), -1.0)
        psi, _, cv, its = bls(prob.J(x0, p), zeta_ad, zeta, 0.0, _E(r, zeta, zeta_ad), 0.0)
        if not cv:
            warnings.warn(f"[Normal form] Linear solver for J did not converge. it = {its}")
        return psi

    def central(fp, fm):  # (fp - fm) / 2δ, in fp
        return V.scale(V.axpby(fp, -1.0, fm, 1.0), 1.0 / (2 * delta))

    Fp, F0, Fm = prob.F(x0, p + delta), prob.F(x0, p), prob.F(x0, p - delta)            # :293-297
    R02 = V.axpby(V.axpby(V.copy(Fp), -2.0, F0, 1.0), 1.0, Fm, 1.0)
    V.scale(R02, 1.0 / delta**2)
    R01 = central(Fp, Fm)
    a01 = V.dot(R01, zeta_ad)
    Psi01 = solve(R01)                                                                   # :303
    R11 = central(dF(p + delta, zeta), dF(p - delta, zeta))                              # :310-312
    b11 = V.dot(V.axpby(R11, 1.0, R2(zeta, Psi01), 1.0), zeta_ad)
    R11Psi = central(dF(p + delta, Psi01), dF(p - delta, Psi01))                         # :319-320
    a2v = V.axpby(V.axpby(R02, 2.0, R11Psi, 1.0), 1.0, R2(Psi01, Psi01), 1.0)
    a02 = V.dot(a2v, zeta_ad)
    b2v = R2(zeta, zeta)                                                                 # :328
    b20 = V.dot(b2v, zeta_ad)
    Psi20 = solve(b2v)                                                                   # :333
    b3v = V.axpby(R3(zeta, zeta, zeta), 3.0, R2(zeta, Psi20), 1.0)
    b30 = V.dot(b3v, zeta_ad)

    nf = dict(a01=a01, a02=a02, b11=b11, b20=b20, b30=b30, Psi01=Psi01, Psi20=Psi20)
    tp, bptype = "BranchPoint", "NA"                                                     # :340-350
    if max(abs(a01), abs(b11)) > 1e-10:
        if abs(a01) < tol_fold:
            tp = "Pitchfork" if 100 * abs(b20 / 2) < abs(b30 / 6) else "Transcritical"
        else:
            tp = "Fold"
    elif abs(a02) < tol_fold:
        bptype = "NonQuadraticParameter"
    return BranchPointNF(type=tp, x0=x0, p=p, tau_u=bifpt.tau_u, tau_p=bifpt.tau_p, zeta=zeta, zeta_ad=zeta_ad, nf=nf,
                         bptype=bptype)


def _comb(x, *terms):
    """x + sum(c v for (c, v) in terms), a new vector"""
    y = V.copy(x)
    for c, v in terms:
        V.axpby(y, c, v, 1.0)
    return y


def predictor(bp, ds, ampfactor=1.0):
    """predictor(bp, ds; ampfactor) (src/NormalForms.jl:389-493): a point (x1, p) on the bifurcated branch near bp, as a
    namespace with the reference's fields; None for a Fold."""
    nf = bp.nf
    if bp.type == "Transcritical":                                                       # :389-435
        b11, b20, Psi01 = nf["b11"], nf["b20"], nf["Psi01"]
        pnew = bp.p + ds
        amp = -2 * ds * b11 / b20 * ampfactor
        tu = bp.tau_u
        ntu = 0.0 if tu is None else V.norm2(tu)
        if ntu > 0 and abs(V.dot(bp.zeta, tu)) >= 0.9 * ntu:                             # the branch was the bifurcated one
            x1, xm1, x0 = _comb(bp.x0, (ds, Psi01)), V.copy(bp.x0), _comb(bp.x0, (ds / bp.tau_p, tu))
        else:
            x0 = V.copy(bp.x0)
            x1 = _comb(bp.x0, (amp, bp.zeta), (-ds, Psi01))
            xm1 = _comb(bp.x0, (-amp, bp.zeta), (ds, Psi01))
        if amp == 0:
            amp = abs(ds)
            warnings.warn(f"Singular normal form (`amp = 0`)!! Defaulting to `amp = {amp}`.")
        return types.SimpleNamespace(x0=x0, x1=x1, xm1=xm1, p=pnew, pm1=bp.p - ds, dsfactor=1.0, amp=amp, p0=bp.p)
    if bp.type == "Pitchfork":                                                           # :457-487
        b11, b30 = nf["b11"], nf["b30"]
        dsfactor = 1.0 if b11 * b30 < 0 else -1.0
        amp = ampfactor * math.sqrt(-6 * abs(ds) * dsfactor * b11 / b30)
        pnew = bp.p + abs(ds) * dsfactor
        if amp == 0:
            amp = abs(ds)
            warnings.warn(f"Singular normal form (`amp = 0`)!! Defaulting to `amp = {amp}`.")
        return types.SimpleNamespace(x0=bp.x0, x1=_comb(bp.x0, (amp, bp.zeta)), p=pnew, dsfactor=dsfactor, amp=amp,
                                     dp=pnew - bp.p)
    if bp.type == "Fold":                                                                # :489-492
        return None
    raise NotImplementedError("predictor for a BranchPoint: the generic `_predictor` scan of the reduced equation "
                              "(src/NormalForms.jl:496-535) is not implemented")


def continuation_from_bp(br, ind_bif, prob, alg, contpar, normC=V.norm2, ds=None, ampfactor=1.0, nev=None, use_normal_form=True,
                         bls=None, tol_fold=1e-3, callback=None, verbose=False):
    """continuation(br, ind_bif, options_cont; ampfactor, use_normal_form, nev) (src/bifdiagram/BranchSwitching.jl:74-198):
    automatic branch switching at the simple branch point br.specialpoint[ind_bif] of a branch of `prob` computed by
    events.continuation.  The new branch is continued with events.continuation (alg, contpar, normC) from the two points
    (x0, p0) and the predictor (x1, p1) (:8-44), with contpar.ds = |ds| sign(p1 - p0); `prob` and `contpar` are left as they
    are.  ds: the predictor's step, contpar.ds by default.  bls: the bordered solver of the normal form, alg.bls by default
    (get_bordered_linsolver(br), :84).  callback / verbose: as events.continuation.  Returns (Branch, BranchPointNF), or None at a
    Fold (:157-160)."""
    bifpt = br.specialpoint[ind_bif]
    if bifpt.type not in ("bp", "nd"):
        raise ValueError(f"You cannot branch from a :{bifpt.type} point using these arguments.")
    if abs(bifpt.delta[0]) > 1:
        raise NotImplementedError(f"branch switching at a point with a {abs(bifpt.delta[0])}-dimensional kernel "
                                  "(multicontinuation, src/bifdiagram/BranchSwitching.jl:234-330) is not implemented")
    ds = contpar.ds if ds is None else ds
    nev = contpar.nev if nev is None else nev
    it = ContIterable(prob, alg, contpar, normC)
    bp = get_normal_form1d(it, br, ind_bif, nev=nev, bls=bls or alg.bls, tol_fold=tol_fold)
    if not use_normal_form:
        pred = types.SimpleNamespace(x0=bp.x0, x1=_comb(bp.x0, (ampfactor, bp.zeta)), p=bp.p + ds, amp=ampfactor)
    else:
        pred = predictor(bp, ds, ampfactor)
    if pred is None:
        return None
    cp = replace(contpar, ds=abs(contpar.ds) * float(np.sign(pred.p - bp.p)))            # :18-20
    prob2 = copy.copy(prob)                                                              # re_make(prob; params = par0)
    prob2.u0, prob2.p0 = bp.x0, bp.p
    if hasattr(prob2, "params"):
        prob2.params = list(prob.params)
        prob2.params[prob.lens] = bp.p
    return events.continuation(prob2, alg, cp, normC, verbose=verbose, callback=callback, u1=pred.x1, p1=pred.p), bp
