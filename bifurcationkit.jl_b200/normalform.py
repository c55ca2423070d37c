"""Normal form of a simple branch point and automatic branch switching (aBS) from it -- host orchestration over the C ABI,
like codim2.py.  Every linear solve is a bordered solve (`MatrixFreeBLSB200` by default), every eigen-solve the branch's
eigensolver, every second / third differential a `bk_d2f` / `bk_d3f` call (BifurcationProblemB200.d2F / d3F); host problems
bring their own d2F / d3F, J and, when not symmetric, Jt.

Mirror of the reference:
  get_normal_form1d      <->  get_normal_form1d, autodiff = false           src/NormalForms.jl:189-353
  (adjoint eigenvector)  <->  get_adjoint_basis(L★, λ::Number, eigsolver)    src/NormalForms.jl:31-49
  predictor              <->  predictor(::Transcritical / ::Pitchfork / ::Fold, ds)  src/NormalForms.jl:389-493
  continuation_from_bp   <->  continuation(br, ind_bif, options_cont)       src/bifdiagram/BranchSwitching.jl:74-198, :8-44
  hopf_normal_form       <->  hopf_normal_form(prob, br, ind_hopf; autodiff = false)  src/NormalForms.jl:1102-1204
  hopf_normal_form_at    <->  __hopf_normal_form(prob, pt::Hopf, ls; autodiff = false) src/NormalForms.jl:1009-1076
  predictor (Hopf)       <->  predictor(hp::Hopf, ds)                       src/NormalForms.jl:1227-1281
  d2Fc / d3Fc            <->  d2Fc (src/Problems.jl:171-178): complex forms composed from real bk_d2f / bk_d3f calls

  get_normal_formNd      <->  get_normal_formNd, autodiff = false           src/NormalForms.jl:656-896
  (adjoint basis)        <->  get_adjoint_basis(L★, λs, eigsolver)          src/NormalForms.jl:1-24
  biorthogonalise        <->  biorthogonalise(ζs, ζ★s)                      src/NormalForms.jl:51-91
  NdBranchPointNF        <->  NdBranchPoint, its reduced form and bp(x, δp) src/NormalForms.jl:533-582
  predictor_nd           <->  predictor(bp::NdBranchPoint, δp)              src/NormalForms.jl:916-985
  multicontinuation      <->  multicontinuation(br, ind_bif, options_cont)  src/bifdiagram/BranchSwitching.jl:234-442
  get_first_points_on_branch <-> get_first_points_on_branch                  src/bifdiagram/BranchSwitching.jl:298-352

The Hopf normal form keeps its complex vectors (ζ, ζ★, Ψ200) as host arrays: it is a handful of solves at one point.
Branch switching from a Hopf point to periodic orbits is in periodic.py.  The N-dimensional normal form makes every inner
product of a jet with ζ★ᵢ in one `bk_jet_moments` pass (prob.jet_moments); host problems get the same contractions from a jet
call and a dot product per tuple (jet_moments_composed).

Not here: the generic BranchPoint predictor (_predictor, src/NormalForms.jl:496-535), usedeflation = false and bothside;
higher codimension normal forms.  bifurcationdiagram, which chains these calls, is bifdiagram.py.
"""
import itertools
from dataclasses import dataclass, replace
import math
import types
import warnings

import numpy as np
import scipy.linalg as sla

from .codim2 import _apply, ComplexProblemB200
from .core import Context, DeviceVec, ComplexGMRESB200, MatrixFreeBLSB200, eigsolve
from .deflation import DeflationOperator, newton_deflated_or_fail
from .palc import V, ContIterable, NewtonPar, re_make
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


def _given(x, z):
    """a vector given by the caller, as a new vector of the container of x: a list or host array through _like, else a copy"""
    return _like(x, z) if isinstance(z, (list, np.ndarray)) else V.copy(z)


def _eig(eigsolver, J, nev):
    """eigsolver(J, nev) with eigenvectors: (vals, vecs as columns)"""
    out = eigsolve(eigsolver, J, nev, True)
    return np.asarray(out[0]), out[1]


def _isapprox(a, b):
    """Julia's a ≈ b with the default rtol = sqrt(eps)"""
    return a == b or abs(a - b) <= math.sqrt(np.finfo(float).eps) * max(abs(a), abs(b))


def _eig_entry(br, bifpt, nev):
    """the br.eig entry saved at the special point bifpt, its eigenvalues as an array, and nev (their number when None)"""
    entry = next(e for e in br.eig if e["step"] == bifpt.idx)
    saved = np.asarray(entry["eigenvals"])
    return entry, saved, len(saved) if nev is None else nev


def _recomputed_eig(prob, x0, p, eigsolver, nev, k, expected):
    """the eigenpairs of J at (x0, p) recomputed with eigsolver (nev of them); raises unless eigenvalue k ≈ expected, the one
    saved with the branch"""
    vals, vecs = _eig(eigsolver, prob.J(x0, p), nev)
    if not _isapprox(vals[k], expected):
        raise RuntimeError(f"We did not find the correct eigenvalue {expected}. We found {vals}.\n"
                           "If you use aBS, pass a higher `nev` (number of eigenvalues) to be computed.")
    return vals, vecs


def _E(x, zeta, zeta_ad):
    """E(x) = x - <x, zeta_ad> zeta, in place (src/NormalForms.jl:178)"""
    return V.axpby(x, -V.dot(x, zeta_ad), zeta, 1.0)


def _host(x):
    """a vector as a host array"""
    return x.numpy() if isinstance(x, DeviceVec) else np.asarray(x)


def _capply(J, z):
    """apply(J, z) for a complex host vector z: J on the real and the imaginary part"""
    re = _host(_apply(J, np.ascontiguousarray(np.real(z), dtype=np.float64)))
    im = _host(_apply(J, np.ascontiguousarray(np.imag(z), dtype=np.float64)))
    return re + 1j * im


def _eigvec(J, vals, vecs, k):
    """geteigenvector(eigsolver, vecs, k) as a host array: a complex column as it is; a real-stored one (ShiftInvertB200 keeps a
    complex pair as real columns) is completed from one of its columns v, which lies in the pair's invariant subspace: with
    λ = α + iβ, v = Re(w) for an eigenvector w of λ, and J v = α Re(w) - β Im(w) gives Im(w) = (α v - J v) / β."""
    v = np.asarray(vecs)[:, k]
    lam = complex(vals[k])
    if np.iscomplexobj(v) or lam.imag == 0:
        return v
    return v + 1j * (lam.real * v - _host(_apply(J, np.ascontiguousarray(v)))) / lam.imag


def _adjoint_basis(prob, x0, p, lams, eigsolver, nev):
    """get_adjoint_basis(L★, λs, eigsolver; nev) (src/NormalForms.jl:1-24): from one eigen-solve of J', for each λ of `lams` in
    turn the eigenvector whose eigenvalue is closest to conj(λ), each eigenvalue used once.  J' is prob.Jt where the problem has
    it (host problems, device kinds with a J' kernel), else J under bk_jac_set_transpose.  A real λ gives a real vector of the
    container of x0, a complex λ a complex host array.  An eigenvalue found with |Re| > 1e-2 is warned of in the words of the
    reference's method for one λ (:31-49) or for a list."""
    def adjoint(J):
        vals, vecs = _eig(eigsolver, J, nev)
        free = np.array(vals, dtype=complex)
        out = []
        for lam in lams:
            i = int(np.argmin(np.abs(free - np.conj(lam))))
            free[i] = 1e9                                        # not used twice (:21)
            if abs(vals[i].real) > 1e-2 and len(lams) == 1:
                warnings.warn(f"The bifurcating eigenvalue is not that close to Re = 0. We found {vals[i].real} !≈ 0. "
                              "You can perhaps increase the argument `nev`.")
            elif abs(vals[i].real) > 1e-2:
                warnings.warn(f"Did not converge to the requested eigenvalues. We found {vals[i].real} !≈ 0. This might not "
                              "lead to precise normal form computation. You can perhaps increase the argument `nev`.")
            out.append(_like(x0, np.asarray(vecs)[:, i]) if np.imag(lam) == 0 else _eigvec(J, vals, vecs, i))
        return out
    if hasattr(prob, "Jt"):
        return adjoint(prob.Jt(x0, p))
    prob.ctx.set_transpose(True)
    try:
        return adjoint(prob.J(x0, p))
    finally:
        prob.ctx.set_transpose(False)


def _adjoint_vector(prob, x0, p, lam, eigsolver, nev):
    """get_adjoint_basis(L★, conj(λ), eigsolver; nev) (src/NormalForms.jl:31-49): the eigenvector of J' whose eigenvalue is
    closest to conj(λ) (_adjoint_basis for one λ)."""
    return _adjoint_basis(prob, x0, p, [lam], eigsolver, nev)[0]


def _adjoint_vectors(prob, x0, p, zetas, zetas_ad, lams, eigsolver, nev):
    """ζ★s of a branch point (src/NormalForms.jl:260-272, :737-748): zetas_ad as given, in the container of x0; copies of ζs
    for a symmetric problem; else the eigenvectors of J' for λs (_adjoint_basis), a complex one replaced by its real part"""
    if zetas_ad is not None:
        return [_given(x0, z) for z in zetas_ad]
    if getattr(prob, "symmetric", False):
        return [V.copy(z) for z in zetas]
    return [z if not np.iscomplexobj(z) else _like(x0, z) for z in _adjoint_basis(prob, x0, p, lams, eigsolver, nev)]


def _parameter_differences(prob, x0, p):
    """R01 = ∂F/∂p and R02 = ∂²F/∂p² at (x0, p) by central differences with prob.delta (src/NormalForms.jl:293-297), from
    F(p + δ), F(p), F(p - δ) in that order, and d_dp(v) = ∂(dF v)/∂p from J(p + δ) v and J(p - δ) v; each a new vector"""
    delta = prob.delta

    def central(fp, fm):  # (fp - fm) / 2δ, in fp
        return V.scale(V.axpby(fp, -1.0, fm, 1.0), 1.0 / (2 * delta))

    Fp, F0, Fm = prob.F(x0, p + delta), prob.F(x0, p), prob.F(x0, p - delta)
    R02 = V.axpby(V.axpby(V.copy(Fp), -2.0, F0, 1.0), 1.0, Fm, 1.0)   # before central overwrites Fp
    V.scale(R02, 1.0 / delta**2)
    R01 = central(Fp, Fm)
    return R01, R02, lambda v: central(_apply(prob.J(x0, p + delta), v), _apply(prob.J(x0, p - delta), v))


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
    x0, p = bifpt.x, bifpt.param                                                         # :223-230
    _, saved, nev = _eig_entry(br, bifpt, nev)
    k = bifpt.ind_ev - 1                                                                 # ind_ev is 1-based
    lam = float(np.real(saved[k]))                                                       # :236
    if zeta is None:                                                                     # :243-256
        _, vecs = _recomputed_eig(prob, x0, p, options.eigsolver, max(nev, bifpt.ind_ev + 2), k, lam)
        zeta = _like(x0, np.asarray(vecs)[:, k])
    else:
        zeta = _given(x0, zeta)
    V.scale(zeta, 1.0 / V.norm2(zeta))                                                   # scaleζ = norm, :257
    (zeta_ad,) = _adjoint_vectors(prob, x0, p, [zeta], None if zeta_ad is None else [zeta_ad], [lam], options.eigsolver,
                                  nev)                                                   # :260-272
    zz = V.dot(zeta, zeta_ad)
    if not abs(zz) > 1e-10:                                                              # :275-277
        raise RuntimeError(f"We got ζ⋅ζ★ = {zz}.\nThis dot product should not be zero.\n"
                           f"Perhaps, you can increase `nev` which is currently {nev}.")
    V.scale(zeta_ad, 1.0 / zz)

    R2 = lambda a, b: prob.d2F(x0, p, a, b)
    R3 = lambda a, b, c: prob.d3F(x0, p, a, b, c)

    def solve(rhs):  # bls(L, ζ★, ζ, 0, E(-rhs), 0): L is re-made before each solve (a device context keeps one Jacobian)
        r = V.scale(V.copy(rhs), -1.0)
        psi, _, cv, its = bls(prob.J(x0, p), zeta_ad, zeta, 0.0, _E(r, zeta, zeta_ad), 0.0)
        if not cv:
            warnings.warn(f"[Normal form] Linear solver for J did not converge. it = {its}")
        return psi

    R01, R02, d_dp = _parameter_differences(prob, x0, p)                                 # :293-297
    a01 = V.dot(R01, zeta_ad)
    Psi01 = solve(R01)                                                                   # :303
    R11 = d_dp(zeta)                                                                     # :310-312
    b11 = V.dot(V.axpby(R11, 1.0, R2(zeta, Psi01), 1.0), zeta_ad)
    R11Psi = d_dp(Psi01)                                                                 # :319-320
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


@dataclass
class HopfNF:
    """Hopf of src/NormalForms.jl (fields of the Hopf point): the point (x0, p), the frequency omega = Im λ, the eigenvector
    zeta of J for λ and the adjoint vector zeta_ad with <zeta, zeta_ad> = 1 (complex host arrays), and HopfNormalForm in `nf`:
    a, b of the reduced equation dA/dt = (iω + a dp) A + b A |A|^2, with Psi001, Psi110 (real host arrays) and Psi200 (complex);
    all None for detailed = False.  type: SuperCritical / SubCritical / Singular by the sign of Re b, ? without a, b."""
    type: str
    x0: object
    p: float
    omega: float
    zeta: object
    zeta_ad: object
    nf: dict


def _jet(f, x0, p, *vs):
    """the complex-multilinear extension of a real jet f(x0, p, v1, ..) (d2F / d3F) to complex host vectors, from real calls on
    their real and imaginary parts (d2Fc, src/Problems.jl:171-178); calls on an imaginary part that is zero are skipped"""
    parts = [(np.ascontiguousarray(np.real(v), dtype=np.float64), np.ascontiguousarray(np.imag(v), dtype=np.float64)) for v in vs]
    re = im = 0.0
    for pick in itertools.product((0, 1), repeat=len(vs)):
        if any(k and not np.any(parts[j][1]) for j, k in enumerate(pick)):
            continue
        val = _host(f(x0, p, *[parts[j][k] for j, k in enumerate(pick)]))
        n_im = sum(pick) % 4                                   # the factor i^n_im
        if n_im == 0:
            re = re + val
        elif n_im == 1:
            im = im + val
        elif n_im == 2:
            re = re - val
        else:
            im = im - val
    return re + 1j * im


def d2Fc(prob, x0, p, a, b):
    """d2F(x0, p)[a, b] for complex host vectors a, b (four real bk_d2f calls at most)"""
    return _jet(prob.d2F, x0, p, a, b)


def d3Fc(prob, x0, p, a, b, c):
    """d3F(x0, p)[a, b, c] for complex host vectors (eight real bk_d3f calls at most)"""
    return _jet(prob.d3F, x0, p, a, b, c)


def _complex_twin(prob):
    """ComplexProblemB200 and ComplexGMRESB200 on a BK_COMPLEX context of the device problem's grid (codim2.py)"""
    ctx = prob.ctx
    cctx = Context(**{**ctx._args, "complex": True}, params=ctx.params)
    return ComplexProblemB200(cctx, prob.params, prob.lens)


def hopf_normal_form_at(prob, x0, p, omega, zeta, zeta_ad, ls, cprob=None, cls=None):
    """__hopf_normal_form (src/NormalForms.jl:1009-1076) with autodiff = false: the parameter derivatives are central
    differences with prob.delta.  Psi001 and Psi110 come from real solves ls(J, rhs) (the Newton linear solver), Psi200 from
    (2iω - J) Psi200 = R20 solved by cls(cprob.J(x0, p), R20, a0 = 2iω, a1 = -1) on the complexified twin; for a device
    problem both default to a BK_COMPLEX context of its grid and ComplexGMRESB200 with ls's settings.  zeta, zeta_ad: complex
    host arrays.  Inner products are Julia's VI.inner(x, y) = Σ conj(x) y.  Returns a HopfNF."""
    delta = prob.delta
    zeta, zeta_ad = np.asarray(zeta, dtype=complex), np.asarray(zeta_ad, dtype=complex)
    czeta = np.conj(zeta)
    if cprob is None:
        cprob = _complex_twin(prob)
    if cls is None:
        cls = ComplexGMRESB200(reltol=ls.reltol, abstol=ls.abstol, restart=ls.restart, maxiter=ls.maxiter, Pl=ls.Pl, Pr=ls.Pr,
                               orth=ls.orth, fused=ls.fused)
    R2 = lambda a, b: d2Fc(prob, x0, p, a, b) / 2
    R3 = lambda a, b, c: d3Fc(prob, x0, p, a, b, c) / 6

    def solve(rhs, what):  # ls(L, rhs) with L re-made before the solve (a device context keeps one Jacobian)
        psi, cv, its = ls(prob.J(x0, p), _like(x0, rhs))
        if not cv:
            warnings.warn(f"[Hopf {what}] Linear solver for J did not converge. it = {its}")
        return _host(psi)

    R01 = (_host(prob.F(x0, p + delta)) - _host(prob.F(x0, p - delta))) / (2 * delta)       # :1036-1037
    Psi001 = solve(-R01, "Ψ001")                                                             # :1039
    av = (_capply(prob.J(x0, p + delta), zeta) - _capply(prob.J(x0, p - delta), zeta)) / (2 * delta)  # :1046-1047
    av = av + 2 * R2(zeta, Psi001)
    a = complex(np.vdot(av, zeta_ad))
    R20 = R2(zeta, zeta)                                                                     # :1053-1055
    Psi200, cv, its = cls(cprob.J(x0, p), R20, a0=complex(0.0, 2 * omega), a1=-1.0)
    if not cv:
        warnings.warn(f"[Hopf Ψ200] Linear solver for J did not converge. it = {its}")
    Psi200 = np.asarray(Psi200, dtype=complex)
    R20 = 2 * R2(zeta, czeta)                                                                # :1058-1060
    Psi110 = solve(-np.real(R20), "Ψ110")    # R2(ζ, conj ζ) is real: its imaginary part is rounding
    bv = 2 * R2(zeta, Psi110) + 2 * R2(czeta, Psi200) + 3 * R3(zeta, zeta, czeta)          # :1063-1064
    b = complex(np.vdot(bv, zeta_ad))
    tp = "SuperCritical" if b.real < 0 else ("SubCritical" if b.real > 0 else "Singular")    # :1068-1074
    return HopfNF(type=tp, x0=x0, p=p, omega=omega, zeta=zeta, zeta_ad=zeta_ad,
                  nf=dict(a=a, b=b, Psi001=Psi001, Psi110=Psi110, Psi200=Psi200))


def hopf_normal_form(it, br, ind_hopf, nev=None, zeta=None, zeta_ad=None, detailed=True, cprob=None, cls=None):
    """hopf_normal_form(prob, br, ind_hopf; autodiff = false, detailed) (src/NormalForms.jl:1102-1204) for the branch `br`
    computed by events.continuation over the iterator `it`.  λ is the saved eigenvalue ind_ev of the point and ω = Im λ.  zeta:
    the eigenvector of J for λ -- given, or the one saved with the branch (ContinuationPar.save_eigenvectors), or recomputed
    with newton_options.eigsolver; scaled by 1 / norm.  zeta_ad: the eigenvector of J' for the eigenvalue closest to conj(λ)
    (given, or computed as get_normal_form1d does), normalised by ζ★ ./= dot(ζ, ζ★).  cprob / cls: see hopf_normal_form_at.
    Returns a HopfNF; with detailed = False only the point, ω and ζ."""
    prob, options = it.prob, it.contpar.newton_options
    bifpt = br.specialpoint[ind_hopf]
    if bifpt.type != "hopf":
        raise ValueError("The provided index does not refer to a Hopf Point")
    x0, p = bifpt.x, bifpt.param
    entry, saved, nev = _eig_entry(br, bifpt, nev)
    k = bifpt.ind_ev - 1                                                                     # ind_ev is 1-based
    # :1138-1139.  λ is the member of the crossing pair with Im λ > 0 -- the one the reference's DefaultEig puts at ind_ev (it
    # lists a pair of equal real parts with the positive imaginary part second); the guess x0 + 2 Re(ζ A(t)) of the predictor
    # runs forward in time only for ω > 0.  Eigensolvers that list the other member first (ShiftInvertB200) give the same λ.
    lam = complex(saved[k])
    lam = lam if lam.imag >= 0 else lam.conjugate()
    omega = lam.imag
    closest = lambda vals: int(np.argmin(np.abs(np.asarray(vals) - lam)))
    if zeta is not None:
        zeta = np.array(zeta, dtype=complex)
    elif entry.get("eigenvecs") is not None:                                                 # :1150-1151
        zeta = _eigvec(prob.J(x0, p), saved, entry["eigenvecs"], closest(saved))
    else:                                                                                    # :1142-1148
        vals, vecs = _recomputed_eig(prob, x0, p, options.eigsolver, bifpt.ind_ev + 2, k, complex(saved[k]))
        zeta = _eigvec(prob.J(x0, p), vals, vecs, closest(vals))
    zeta = np.asarray(zeta, dtype=complex) / np.linalg.norm(zeta)                            # :1153
    if not detailed:                                                                         # :1155-1168
        nf = dict(a=None, b=None, Psi001=None, Psi110=None, Psi200=None)
        return HopfNF(type="?", x0=x0, p=p, omega=omega, zeta=zeta, zeta_ad=np.zeros_like(zeta), nf=nf)
    if zeta_ad is None:                                                                      # :1171-1173
        zeta_ad = _adjoint_vector(prob, x0, p, lam, options.eigsolver, nev)
    zeta_ad = np.array(zeta_ad, dtype=complex)
    zeta_ad /= np.vdot(zeta, zeta_ad)                                                        # :1186: ζ★ ./= dot(ζ, ζ★)
    if not _isapprox(np.vdot(zeta, zeta_ad), 1):
        raise RuntimeError("Error of precision in normalization")
    return hopf_normal_form_at(prob, x0, p, omega, zeta, zeta_ad, options.linsolver, cprob, cls)


def _hopf_predictor(hp, ds, ampfactor):
    """predictor(hp::Hopf, ds; ampfactor) (src/NormalForms.jl:1227-1281)"""
    nf = hp.nf
    x0 = _host(hp.x0)
    if nf["a"] is not None and nf["b"] is not None:
        a, b = nf["a"], nf["b"]
        if abs(b.real) < 1e-10:
            warnings.warn(f"The Lyapunov coefficient is nearly zero:\nb = {b}.\nThe Hopf predictor may be unreliable.")
        dsfactor = 1.0 if a.real * b.real < 0 else -1.0
        dsnew = abs(ds) * dsfactor
        pnew = hp.p + dsnew
        amp = ampfactor * math.sqrt(-dsnew * a.real / b.real)                               # a ds + b amp^2 = 0
        omega = hp.omega + (a.imag - b.imag * a.real / b.real) * ds
        Psi001, Psi110, Psi200 = nf["Psi001"], nf["Psi110"], nf["Psi200"]
    else:
        amp, omega, pnew, dsfactor = ampfactor, hp.omega, hp.p + ds, 1.0
        Psi001, Psi110, Psi200 = np.zeros_like(x0), np.zeros_like(hp.zeta), np.zeros_like(hp.zeta)

    def orbit(t):
        A = amp * complex(math.cos(t), math.sin(t))                                          # amp cis(t)
        return (x0 + 2 * np.real(hp.zeta * A) + ds * Psi001 + abs(A) ** 2 * np.real(Psi110)
                + 2 * np.real(A ** 2 * Psi200))
    return types.SimpleNamespace(orbit=orbit, Psi001=Psi001, amp=2 * amp, omega=omega, period=abs(2 * math.pi / omega), p=pnew,
                                 dsfactor=dsfactor)


def _comb(x, *terms):
    """x + sum(c v for (c, v) in terms), a new vector"""
    y = V.copy(x)
    for c, v in terms:
        V.axpby(y, c, v, 1.0)
    return y


def predictor(bp, ds, ampfactor=1.0):
    """predictor(bp, ds; ampfactor) (src/NormalForms.jl:389-493, :1227-1281): a point (x1, p) on the bifurcated branch near bp,
    or for a Hopf point the guess of the bifurcated periodic orbits, as a namespace with the reference's fields; None for a
    Fold."""
    if isinstance(bp, HopfNF):
        return _hopf_predictor(bp, ds, ampfactor)
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
        raise NotImplementedError(f"branch switching at a point with a {abs(bifpt.delta[0])}-dimensional kernel goes through "
                                  "normalform.multicontinuation (src/bifdiagram/BranchSwitching.jl:234-442)")
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
    sign = float(np.sign(pred.p - bp.p))                                                 # :18-20
    return _continue_from(prob, bp, alg, contpar, normC, pred.x1, pred.p, sign, callback, verbose), bp


def _continue_from(prob, bp, alg, contpar, normC, u1, p1, ds_sign, callback, verbose):
    """events.continuation (alg, contpar with ds = |contpar.ds| ds_sign, normC, callback, verbose) of re_make(prob; u0 = bp.x0,
    params = par0) from the two points (bp.x0, bp.p) and (u1, p1) (src/bifdiagram/BranchSwitching.jl:8-44)"""
    cp = replace(contpar, ds=abs(contpar.ds) * ds_sign)
    return events.continuation(re_make(prob, bp.x0, bp.p), alg, cp, normC, verbose=verbose, callback=callback, u1=u1, p1=p1)


# ------------------------------------------------------------------------------------------------ kernels of dimension N > 1
def jet_moments_composed(prob, x0, p, vecs, idx2=(), idx3=()):
    """<v_i, d2F(x0, p)[v_j, v_k]> for the rows (i, j, k) of idx2, then <v_i, d3F(x0, p)[v_j, v_k, v_l]> for the rows of idx3: one
    jet call and one dot product per tuple.  It serves problems that bring only d2F / d3F, and it is what the one-pass device
    contraction (prob.jet_moments, bk_jet_moments) is checked against."""
    idx2, idx3 = np.reshape(np.asarray(idx2, dtype=int), (-1, 3)), np.reshape(np.asarray(idx3, dtype=int), (-1, 4))
    out = [V.dot(vecs[i], prob.d2F(x0, p, vecs[j], vecs[k])) for i, j, k in idx2]
    out += [V.dot(vecs[i], prob.d3F(x0, p, vecs[j], vecs[k], vecs[l])) for i, j, k, l in idx3]
    return np.array(out, dtype=float)


def jet_moments(prob, x0, p, vecs, idx2=(), idx3=()):
    """the contractions of jet_moments_composed, in one pass over the vectors where the problem has it (prob.jet_moments)"""
    if hasattr(prob, "jet_moments"):
        return prob.jet_moments(x0, p, vecs, idx2, idx3)
    return jet_moments_composed(prob, x0, p, vecs, idx2, idx3)


def _lincomb(coefs, vecs):
    """sum_j coefs[j] vecs[j], a new vector of the container of vecs[0]"""
    y = V.zeros_like(vecs[0])
    for c, v in zip(coefs, vecs):
        if c != 0:
            V.axpby(y, float(c), v, 1.0)
    return y


def _gram(a, b):
    return np.array([[V.dot(x, y) for y in b] for x in a])


def biorthogonalise(zetas, zetas_ad):
    """biorthogonalise(ζs, ζ★s) (src/NormalForms.jl:51-91): ζ★s <- Q' ζ★s with Q = pinv(G), G_ij = <ζ_i, ζ★_j>; when G is then
    not the identity to 1e-5, the LU algorithm (G = P L U: ζs <- (P L)^-1 ζs, ζ★s <- U'^-1 ζ★s), which also changes ζs.
    Raises as the reference does when G is singular or the result is not biorthogonal."""
    assert len(zetas) == len(zetas_ad), "The Gram matrix is not square!"
    G = _gram(zetas, zetas_ad)
    if abs(np.linalg.det(G)) <= 1e-14:
        raise RuntimeError(f"The Gram matrix is not invertible! det(G) = {np.linalg.det(G)}, G =\n{G}\n"
                           "You can perhaps increase the argument `nev`.")
    Q = np.linalg.pinv(G)
    new_ad = [_lincomb(Q[:, i], zetas_ad) for i in range(len(zetas))]                  # (Q' ζ★s)_i = sum_j Q_ji ζ★_j
    if np.max(np.abs(_gram(zetas, new_ad) - np.eye(len(zetas)))) >= 1e-5:
        warnings.warn("Gram matrix not equal to identity. Switching to LU algorithm.\n This modifies the basis of right eigenvectors!")
        Pm, Lm, Um = sla.lu(G)
        M, Ui = np.linalg.inv(Pm @ Lm), np.linalg.inv(Um)
        zetas = [_lincomb(M[i], zetas) for i in range(len(zetas))]
        new_ad = [_lincomb(Ui[:, i], zetas_ad) for i in range(len(zetas))]
    G = _gram(zetas, new_ad)
    if not np.max(np.abs(G - np.eye(len(zetas)))) < 1e-5:
        raise RuntimeError("Failure in bi-orthogonalisation of the right / left eigenvectors.\nThe left eigenvectors do not form "
                           f"a basis.\nYou may want to increase `nev`, G =\n{G}")
    return zetas, new_ad


@dataclass
class NdBranchPointNF:
    """NdBranchPoint of src/NormalForms.jl:533-582 (fields of the point): (x0, p), the tangent (tau_u, tau_p), the kernel basis
    zetas and the adjoint basis zetas_ad with <ζ_i, ζ★_j> = δ_ij, and in `nf` the coefficients a01 (N), a02 (N), b11 (N x N), b20
    (N x N x N), b30 (N x N x N x N) of the reduced equation; type "N-d" or "NonQuadraticParameter" (:882)."""
    x0: object
    p: float
    tau_u: object
    tau_p: float
    zetas: list
    zetas_ad: list
    nf: dict
    type: str

    def reduced_form(self, x, dp):
        """bp(Val(:reducedForm), x, dp) (:541-574): a01 dp + dp b11 x + b20[x, x] / 2 + b30[x, x, x] / 6 (the a02 term carries the
        reference's factor 0 dp)"""
        nf, x = self.nf, np.asarray(x, dtype=float)
        if len(x) != len(self.zetas):
            raise ValueError(f"N = {len(self.zetas)} and length(x) = {len(x)} should match!")
        return (dp * nf["a01"] + dp * nf["b11"] @ x + np.einsum("ijk,j,k->i", nf["b20"], x, x) / 2
                + np.einsum("ijkl,j,k,l->i", nf["b30"], x, x, x) / 6)

    def reduced_jacobian(self, x, dp):
        """the derivative of reduced_form in x"""
        nf, x = self.nf, np.asarray(x, dtype=float)
        b20, b30 = nf["b20"], nf["b30"]
        return (dp * nf["b11"] + (np.einsum("imk,k->im", b20, x) + np.einsum("ijm,j->im", b20, x)) / 2
                + (np.einsum("imkl,k,l->im", b30, x, x) + np.einsum("ijml,j,l->im", b30, x, x)
                   + np.einsum("ijkm,j,k->im", b30, x, x)) / 6)

    def __call__(self, x, dp):
        """bp(x, δp) (:576-582): x0 + sum_i x_i ζ_i"""
        y = V.copy(self.x0)
        for xi, z in zip(x, self.zetas):
            V.axpby(y, float(xi), z, 1.0)
        return y


def get_normal_formNd(it, br, ind_bif, nev=None, zetas=None, zetas_ad=None, bls=None, tol_fold=1e-3):
    """get_normal_formNd(prob, br, id_bif; autodiff = false) (src/NormalForms.jl:656-896) at the point br.specialpoint[ind_bif],
    whose kernel has dimension N = |delta[0]| > 1, of the branch `br` computed by events.continuation over the iterator `it`.
    zetas: a basis of the kernel; otherwise the eigenvectors ind_ev - N + 1 .. ind_ev, saved with the branch or recomputed with
    newton_options.eigsolver; each is divided by its norm.  zetas_ad: the adjoint basis; otherwise ζs for a symmetric problem,
    else the eigenvectors of J' closest to conj(λs).  Both are biorthogonalised.  bls: the solver of the singular systems,
    through its solve_block with the borders (ζ★₁, ζ★₂; ζ₁, ζ₂) of the reference; MatrixFreeBLSB200 over the Newton linear
    solver by default.  For N > 2 that two-border system is singular (its kernel is span(ζ₃ .. ζ_N)), so each solution is
    projected to <ζ_i, ψ> = 0 for every i, the solution an N-border solve would give (DESIGN.md §2).  Every inner product of a
    jet with ζ★ᵢ goes through one `jet_moments` call: one kernel pass over the 2N + 1 + N(N+1)/2 vectors up to N = 9, several
    beyond (Context.jet_moments groups the tuples).  Returns an NdBranchPointNF."""
    prob, options = it.prob, it.contpar.newton_options
    bifpt = br.specialpoint[ind_bif]
    N = abs(bifpt.delta[0])
    if N < 2:
        raise ValueError(f"get_normal_formNd needs a kernel of dimension > 1, here {N}: use get_normal_form1d.")
    bls = bls or MatrixFreeBLSB200(options.linsolver)
    x0, p = bifpt.x, bifpt.param
    entry, rightEv, nev = _eig_entry(br, bifpt, nev)
    nev = max(2 * N, nev)                                                                # :680-681
    ind = list(range(bifpt.ind_ev - N, bifpt.ind_ev))                                    # indev-N+1:indev, 0-based
    lams = rightEv[ind]
    if zetas is None:                                                                    # :711-724
        if entry.get("eigenvecs") is not None:
            vecs = np.asarray(entry["eigenvecs"])
        else:
            vals, vecs = _eig(options.eigsolver, prob.J(x0, p), max(nev, len(rightEv)))
            if np.max(np.abs(vals[: len(rightEv)] - rightEv)) > it.contpar.tol_stability:
                warnings.warn(f"We did not find the correct eigenvalues. We found {vals[: len(rightEv)]} instead of {rightEv}.")
        zetas = [_like(x0, np.asarray(vecs)[:, i]) for i in ind]
    else:
        zetas = [_given(x0, z) for z in zetas]
    for z in zetas:                                                                      # scaleζ = norm, :729
        V.scale(z, 1.0 / V.norm2(z))
    zetas_ad = _adjoint_vectors(prob, x0, p, zetas, zetas_ad, lams, options.eigsolver, nev)   # :737-748
    zetas, zetas_ad = biorthogonalise(zetas, zetas_ad)                                   # :752

    gram_inv = np.linalg.inv(_gram(zetas, zetas)) if N > 2 else None

    def E(x):  # E_nd (:648-654): x - sum_i <x, ζ★_i> ζ_i, a new vector
        return _lincomb([1.0] + [-V.dot(x, za) for za in zetas_ad], [x] + zetas)

    def solve(rhs, what):  # solve_bls_block(bls, L, (ζ★₁, ζ★₂), (ζ₁, ζ₂), 0, rhs, 0) (:759-763), L re-made before each solve
        psi, _, cv, its = bls.solve_block(prob.J(x0, p), tuple(zetas_ad[:2]), tuple(zetas[:2]), np.zeros((2, 2)), rhs, np.zeros(2))
        if not cv:
            warnings.warn(f"[Normal form Nd {what}] linear solver did not converge. it = {its}")
        if gram_inv is not None:  # N > 2: the component in span(ζ₃ .. ζ_N) the two borders leave free, removed
            c = gram_inv @ np.array([V.dot(z, psi) for z in zetas])
            psi = _lincomb([1.0] + list(-c), [psi] + zetas)
        return psi

    R01, R02, d_dp = _parameter_differences(prob, x0, p)                                 # :774-780
    a01 = np.array([V.dot(R01, za) for za in zetas_ad])                                 # :782-784
    # The reference re-solves the Ψ01 system inside its jj loop (:798) and the wst system of each ordered pair inside its b30
    # loop (:844-857).  The device solver is deterministic, so one solve for Ψ01 gives the reference's numbers exactly, and so
    # does one wst solve per unordered pair {k, l} where d2F is symmetric bit for bit: the SH kinds and chan, whose pointwise
    # products commute.  For cGL2d (cgl_jet adds its terms in argument order) and host d2F the two orders agree to rounding.
    Psi01 = solve(V.scale(E(R01), -1.0), "Ψ01")
    R11 = [d_dp(z) for z in zetas]                                                       # :790-796
    R11Psi = d_dp(Psi01)                                                                 # :806-811 (the same for every jj)
    a2v = V.axpby(R02, 2.0, R11Psi, 1.0)
    pairs = [(k, l) for k in range(N) for l in range(k, N)]
    w = {kl: solve(E(prob.d2F(x0, p, zetas[kl[0]], zetas[kl[1]])), "wst") for kl in pairs}
    triples = [(j, k, l) for j in range(N) for k in range(N) for l in range(N) if j == k or j < k < l]   # :841
    # one contraction pass: vectors ζ★ (0..N-1), ζ (N..2N-1), Ψ01 (2N), w_{kl} (2N+1..)
    Z, ps = (lambda j: N + j), 2 * N
    W = {kl: 2 * N + 1 + n for n, kl in enumerate(pairs)}
    wid = lambda a, b: W[(min(a, b), max(a, b))]
    idx2, idx3, at = [], [], {}
    for i in range(N):
        for j, k in pairs:                                                               # b20, :820-828
            at["b20", i, j, k] = len(idx2); idx2.append((i, Z(j), Z(k)))
        for j in range(N):                                                               # b11: R2(ζ_j, Ψ01), :800
            at["b11", i, j] = len(idx2); idx2.append((i, Z(j), ps))
        at["a02", i] = len(idx2); idx2.append((i, ps, ps))                               # a02: R2(Ψ01, Ψ01), :812
        for j, k, l in triples:                                                          # b30, :842-857
            at["b3w", i, j, k, l] = len(idx2)
            idx2 += [(i, Z(j), wid(l, k)), (i, Z(k), wid(l, j)), (i, Z(l), wid(k, j))]
            at["b3", i, j, k, l] = len(idx3); idx3.append((i, Z(j), Z(k), Z(l)))
    vecs = list(zetas_ad) + list(zetas) + [Psi01] + [w[kl] for kl in pairs]
    m = jet_moments(prob, x0, p, vecs, idx2, idx3)
    m2, m3 = m[: len(idx2)], m[len(idx2):]

    b11 = np.zeros((N, N)); a02 = np.zeros(N)
    b20 = np.zeros((N, N, N)); b30 = np.zeros((N, N, N, N))
    for i in range(N):
        for j in range(N):
            b11[i, j] = V.dot(R11[j], zetas_ad[i]) + m2[at["b11", i, j]]
        a02[i] = V.dot(a2v, zetas_ad[i]) + m2[at["a02", i]]
        for j, k in pairs:
            b20[i, j, k] = b20[i, k, j] = m2[at["b20", i, j, k]]
        for j, k, l in triples:
            t = at["b3w", i, j, k, l]
            c = m3[at["b3", i, j, k, l]] - m2[t] - m2[t + 1] - m2[t + 2]
            for I in itertools.permutations((j, k, l)):
                b30[(i,) + I] = c
    nf = dict(a01=a01, a02=a02, b11=b11, b20=b20, b30=b30)
    tp = "NonQuadraticParameter" if max(np.max(np.abs(a01)), np.max(np.abs(a02)), np.max(np.abs(b11))) < tol_fold else f"{N}-d"
    return NdBranchPointNF(x0=x0, p=p, tau_u=bifpt.tau_u, tau_p=bifpt.tau_p, zetas=zetas, zetas_ad=zetas_ad, nf=nf, type=tp)


class _Dense:
    """a small dense Jacobian: apply(J, v) and its matrix"""

    def __init__(self, A):
        self.A = A

    def __call__(self, v):
        return self.A @ v


def _dense_solve(J, rhs, rhs2=None, a0=0.0, a1=1.0):
    """the linear solver of the reduced equation, in the one- and two-right-hand-side forms"""
    A = a0 * np.eye(len(rhs)) + a1 * J.A
    if rhs2 is None:
        return np.linalg.solve(A, rhs), True, 1
    x = np.linalg.solve(A, np.column_stack([rhs, rhs2]))
    return np.ascontiguousarray(x[:, 0]), np.ascontiguousarray(x[:, 1]), True, (1, 1)


class _ReducedProblem:
    """the reduced equation perturb(bp.reduced_form(x, dp)) = 0 as a host problem for newton_deflated, with the analytic Jacobian
    of the cubic (the reference differentiates it with ForwardDiff)"""

    def __init__(self, bp, perturb):
        self.bp, self.perturb = bp, perturb
        self.u0, self.p0, self.delta = np.zeros(len(bp.zetas)), 0.0, 1e-8

    def F(self, x, p, out=None):
        r = np.asarray(self.perturb(self.bp.reduced_form(x, p)), dtype=float)
        if out is not None:
            out[...] = r
            return out
        return r

    def J(self, x, p):
        return _Dense(self.bp.reduced_jacobian(x, p))


def predictor_nd(bp, dp, rng=None, ampfactor=1.0, nbfailures=50, maxiter=100, igs=None, amp_igs=1.0, normN=None,
                 perturb=lambda r: r, tol=1e-12):
    """predictor(bp::NdBranchPoint, δp) (src/NormalForms.jl:916-985): the zeros of the reduced equation at dp = -|δp| and +|δp|,
    by deflated Newton (DeflationOperator(2, 0.1, [0]) per side, newton_deflated with NewtonPar(tol, maxiter)) from the vertices
    of {-1, 0, 1}^N (scaled by amp_igs, or the guesses igs), then from random restarts until nbfailures of them fail.  rng: a
    numpy.random.Generator (default_rng(0) by default), so that the result is reproducible.  perturb is applied to the reduced
    residual, as the reference's.  The Jacobian is the analytic one of the cubic.  Returns (before, after): the roots found on
    each side, the trivial one first, each multiplied by ampfactor."""
    rng = np.random.default_rng(0) if rng is None else rng
    n = len(bp.zetas)
    normN = normN or (lambda v: float(np.max(np.abs(v))))
    opts = NewtonPar(tol=tol, max_iterations=maxiter, linsolver=_dense_solve)
    guesses = list(itertools.product((-1, 0, 1), repeat=n)) if igs is None else list(igs)

    def roots(ds):
        defop = DeflationOperator(2, 0.1, [np.zeros(n)])
        prob = _ReducedProblem(bp, perturb)
        u0 = rng.random(n) - 0.5
        for ci in guesses:                                                               # :954-964
            ci = np.asarray(ci, dtype=float)
            if np.linalg.norm(ci) > 0:
                u0 = ci * amp_igs
                sol = newton_deflated_or_fail(prob, u0, ds, defop, opts, normN)
                if sol.converged:
                    defop.push(ampfactor * sol.u)
        failures = 0
        while failures < nbfailures:                                                     # :966-976
            sol = newton_deflated_or_fail(prob, u0, ds, defop, opts, normN)
            if sol.converged:
                defop.push(ampfactor * sol.u)
            else:
                failures += 1
            u0 = sol.u + 0.1 * (rng.random(n) - 0.5)
        return defop.roots
    return roots(-abs(dp)), roots(abs(dp))


def get_first_points_on_branch(bp, solfromRE, prob, contpar, ds=None, max_iter_deflation=None, perturb_guess=lambda x: x,
                               normN=V.norm2):
    """get_first_points_on_branch(br, bpnf, solfromRE) (src/bifdiagram/BranchSwitching.jl:298-352): deflated Newton
    (newton_deflated: DeflatedProblemCustomLS around the Newton linear solver) on the full problem at p + |ds| from bp(root) for
    every root after the bifurcation point, then at p - |ds| for those before, each side with its own DeflationOperator(2, 1, []).
    Returns a namespace (before, after: the converged states, bpm = p - |ds|, bpp = p + |ds|)."""
    ds = abs(contpar.ds if ds is None else ds)
    optn = contpar.newton_options
    optnDf = replace(optn, max_iterations=min(50, 15 * optn.max_iterations) if max_iter_deflation is None else max_iter_deflation)
    before, after = solfromRE

    def side(roots, q):
        defop = DeflationOperator(2, 1.0, [])
        for xsol in roots:
            sol = newton_deflated_or_fail(prob, perturb_guess(bp(xsol, ds)), q, defop, optnDf, normN)
            if sol.converged:
                defop.push(sol.u)
        return defop.roots
    after = side(after, bp.p + ds)
    before = side(before, bp.p - ds)
    return types.SimpleNamespace(before=before, after=after, bpm=bp.p - ds, bpp=bp.p + ds)


def multicontinuation(br, ind_bif, prob, alg, contpar, normC=V.norm2, ds=None, ampfactor=1.0, nev=None, zetas=None, zetas_ad=None,
                      bpnf=None, solfromRE=None, bls=None, tol_fold=1e-3, rng=None, max_iter_deflation=None,
                      perturb_guess=lambda x: x, callback=None, verbose=False):
    """multicontinuation(br, ind_bif, options_cont) (src/bifdiagram/BranchSwitching.jl:234-442): automatic branch switching at the
    point br.specialpoint[ind_bif], whose kernel has dimension > 1, of a branch of `prob` computed by events.continuation.  The
    normal form (get_normal_formNd with nev, zetas, zetas_ad, bls, tol_fold; or the precomputed `bpnf`), the roots of its reduced
    equation at p ∓ |ds| (predictor_nd with ampfactor and rng; or `solfromRE` = (before, after)), their corrections on the full
    problem (get_first_points_on_branch), then one events.continuation (alg, contpar, normC) from the two points (x0, p) and
    (root, p ∓ |ds|) for every corrected root after the first, which is the trivial branch: contpar.ds = -|ds| before the point,
    +|ds| after it (:432-437).  ds: contpar.ds by default.  `prob` and `contpar` are left as they are.  Returns a list of
    (Branch, NdBranchPointNF)."""
    it = ContIterable(prob, alg, contpar, normC)
    bp = bpnf or get_normal_formNd(it, br, ind_bif, nev=contpar.nev if nev is None else nev, zetas=zetas, zetas_ad=zetas_ad,
                                   bls=bls, tol_fold=tol_fold)
    dp = abs(contpar.ds if ds is None else ds)
    roots = solfromRE or predictor_nd(bp, dp, rng=rng, ampfactor=ampfactor)
    first = get_first_points_on_branch(bp, roots, prob, contpar, dp, max_iter_deflation, perturb_guess, normN=normC)
    out = [(_continue_from(prob, bp, alg, contpar, normC, u, first.bpm, -1.0, callback, verbose), bp) for u in first.before[1:]]
    out += [(_continue_from(prob, bp, alg, contpar, normC, u, first.bpp, 1.0, callback, verbose), bp) for u in first.after[1:]]
    return out
