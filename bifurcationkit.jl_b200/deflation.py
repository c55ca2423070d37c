"""Deflated Newton (SURVEY 8f.4) -- host orchestration over the same C ABI.

* ``DeflationOperator``       <-> src/DeflationOperator.jl:50-170:  M(u) = prod_i (1 / <u - r_i, u - r_i>^p + alpha)
  (or the mean, ``accumulator="mean"``); ``dM(u, du)`` by the reference's forward difference (delta = 1e-8, :158-166).
* ``DeflatedProblem``         <-> :172-232:  residual M(u) F(u); its Jacobian handle is the triple (u, p, problem) (:215-217).
* ``DeflatedProblemCustomLS`` <-> :247-310:  Sherman-Morrison-type solve of  M(u) J h + F(u) dM(u).h = rhs  with the *two-rhs*
  call ``linsolve(Ju, rhs, Fu)`` (src/LinearSolver.jl:15-19 -> ``GMRESB200(J, rhs, rhs2)``), h = (h1 - z h2) / M(u),
  z = dM.h1 / (M(u) + dM.h2).
* ``newton_deflated``         <-> ``solve(prob, defOp, options)`` (:340-356);  ``newton_two_guesses`` <-> ``newton(prob, x0, x1, p0, options)``
  (:392-420), the variant the reference uses for branch switching seeds (examples/SH2d-fronts.jl:70-80 builds the localized
  fronts this way).

Vectors are ``DeviceVec`` or ndarray through ``palc.V``; one extra device vector of scratch, like the reference's ``tmp``.

``DeflationOperator(..., fused=True)`` takes every scalar of the operator from one ``bk_deflation_moments`` pass over u, the
directions and the roots (``Context.deflation_moments``) when u and the roots are ``DeviceVec``s and the distance is the dot product or its
prefix form (``PrefixDot``).  With s_i = <d_i, d_i>, t_ia = <d_i, h_a>, q_ab = <h_a, h_b>, d_i = u - r_i, the reference's
forward difference takes its distances at u + delta h as |d_i + delta h|^2 = s_i + 2 delta t_i + delta^2 q (``fused_values``);
``autodiff=True`` gives the derivative ForwardDiff computes (:161-163) in closed form.  Host vectors and other distances run the
composed loop; so does the default ``fused=False``, which keeps the reference's arithmetic bit for bit.
"""
import ctypes as C
import math

import numpy as np

from .core import DeviceVec, _chk
from .palc import V, NewtonPar, NonLinearSolution, newton
from dataclasses import replace as _replace


class PrefixDot:
    """dot(x[1:n], y[1:n]): the distance of examples/cGL2d.jl:192, which leaves the period of an orbit out"""

    def __init__(self, n):
        self.n = int(n)

    def __call__(self, x, y):
        if isinstance(x, np.ndarray):
            return float(np.dot(x[:self.n], y[:self.n]))
        out = C.c_double()
        _chk(x.ctx, x.ctx.lib.bk_vec_dot(x.ctx.handle, x.dptr, y.dptr, self.n, C.byref(out)))
        return out.value


def _term(s, power, alpha):
    return 1.0 / s ** power + alpha


def fused_values(power, alpha, accumulator, s, t=None, q=None, delta=1e-8, autodiff=False):
    """M(u) and dM(u).h_a for every direction a from the moments s[i], t[i, a], q[a, b] (bk_deflation_moments): the composed
    loop's formula on s_i, the forward difference (M(u + delta h_a) - M(u)) / delta with |d_i + delta h_a|^2 = s_i + 2 delta t_ia
    + delta^2 q_aa, or with autodiff the derivative of the dual-number evaluation: for m_i = 1 / s_i^p + alpha,
    m_i' = -p s_i^(p-1) (2 t_ia) / (s_i^p)^2, accumulated as (a, a') * (b, b') = (a b, a' b + a b') for "prod" and as a sum
    divided by the number of roots for "mean"."""
    prod = accumulator == "prod"

    def acc(vals):
        out = vals[0]
        for v in vals[1:]:
            out = out * v if prod else out + v
        return out / len(vals) if not prod else out

    s = [float(x) for x in s]
    M = acc([_term(x, power, alpha) for x in s])
    nd = 0 if t is None else np.shape(t)[1]
    dM = []
    for a in range(nd):
        ta = [float(x) for x in np.asarray(t)[:, a]]
        if autodiff:
            out, dout = None, None
            for si, ti in zip(s, ta):
                sp = si ** power
                m, dm = _term(si, power, alpha), -(power * si ** (power - 1) * (2.0 * ti)) / (sp * sp)
                if out is None:
                    out, dout = m, dm
                elif prod:
                    out, dout = out * m, dout * m + out * dm
                else:
                    out, dout = out + m, dout + dm
            dM.append(dout if prod else dout / len(s))
        else:
            qa = float(np.asarray(q)[a, a])
            Md = acc([_term(si + 2.0 * delta * ti + delta * delta * qa, power, alpha) for si, ti in zip(s, ta)])
            dM.append((Md - M) / delta)
    return M, dM


class DeflationOperator:
    def __init__(self, power, alpha, roots, dot=None, delta=1e-8, accumulator="prod", fused=False, autodiff=False):
        assert accumulator in ("prod", "mean")
        self.power, self.alpha, self.roots, self.delta, self.accumulator = power, float(alpha), list(roots), delta, accumulator
        self.dot = dot or V.dot
        self.fused, self.autodiff = fused, autodiff

    def copy(self):
        """copy(df) (:101): the same operator over a copy of the root list (the roots themselves are not copied)"""
        return DeflationOperator(self.power, self.alpha, self.roots, self.dot, self.delta, self.accumulator, self.fused,
                                 self.autodiff)

    def runs_fused(self, u):
        """whether the scalars at u come from one bk_deflation_moments pass: u and every root on the device (host roots would be
        uploaded on every call, which costs more than the composed loop saves)"""
        return (self.fused and isinstance(u, DeviceVec) and all(isinstance(r, DeviceVec) for r in self.roots)
                and (self.dot is V.dot or isinstance(self.dot, PrefixDot)))

    def moments(self, u, dirs=()):
        """(s, m, t, q) of Context.deflation_moments over this operator's roots and distance (runs_fused(u) must hold)"""
        return u.ctx.deflation_moments(u, self.roots, dirs, self.dot.n if isinstance(self.dot, PrefixDot) else None)

    def values(self, u, dirs=()):
        """M(u) and [dM(u).h for h in dirs]: one kernel pass where runs_fused(u), else the composed loop"""
        if not self.roots:
            return 1.0, [0.0] * len(dirs)
        if self.runs_fused(u):
            s, _, t, q = self.moments(u, dirs)
            return fused_values(self.power, self.alpha, self.accumulator, s, t, q, self.delta, self.autodiff)
        return self(u), [self.dM(u, h) for h in dirs]

    def _composed_moments(self, u, h):
        s, t = [], []
        tmp = V.copy(u)
        for r in self.roots:
            V.copyto(tmp, u)
            V.axpby(tmp, -1.0, r, 1.0)
            s.append(self.dot(tmp, tmp))
            t.append([self.dot(tmp, h)])
        return s, t

    def __len__(self):
        return len(self.roots)

    def __getitem__(self, i):
        return self.roots[i]

    def push(self, r):
        self.roots.append(r)

    def pop(self):
        return self.roots.pop()

    def __call__(self, u, tmp=None):
        """M(u) (:118-131)"""
        if not self.roots:
            return 1.0
        if self.runs_fused(u):
            return self.values(u)[0]
        tmp = V.copy(u) if tmp is None else tmp
        out = None
        for r in self.roots:
            V.copyto(tmp, u)
            V.axpby(tmp, -1.0, r, 1.0)
            m = 1.0 / self.dot(tmp, tmp) ** self.power + self.alpha
            out = m if out is None else (out * m if self.accumulator == "prod" else out + m)
        return out / len(self.roots) if self.accumulator == "mean" else out

    def dM(self, u, du, tmp=None, tmp2=None):
        """dM(u).du by forward difference (:158-166)"""
        if not self.roots:
            return 0.0
        if self.runs_fused(u):
            return self.values(u, (du,))[1][0]
        if self.autodiff:
            s, t = self._composed_moments(u, du)
            return fused_values(self.power, self.alpha, self.accumulator, s, t, autodiff=True)[1][0]
        tmp = V.copy(u) if tmp is None else V.copyto(tmp, u)
        V.axpby(tmp, self.delta, du, 1.0)
        return (self(tmp, tmp2) - self(u, tmp2)) / self.delta


class DeflatedProblem:
    """M(u) F(u) = 0 (:172-232), same duck type as BifurcationProblemB200 for palc.newton."""

    def __init__(self, prob, M):
        self.prob, self.M = prob, M
        self.u0, self.p0 = prob.u0, prob.p0
        self.delta = getattr(prob, "delta", 1e-8)
        self.record = getattr(prob, "record", None)

    def F(self, x, p, out=None):
        out = self.prob.F(x, p, out)
        return V.scale(out, self.M(x))

    def J(self, x, p):
        return (x, p, self)   # jacobian(dfp::DeflatedProblem{..., Val{:Custom}}, x, p)

    def jvp(self, x, p, du):
        """dF(u).du M(u) + F(u) dM(u).du (:193-207)"""
        J = self.prob.J(x, p)
        if self.M.runs_fused(x):
            Mx, (dMx,) = self.M.values(x, (du,))
            out = V.scale(J(du), Mx)
            if len(self.M):
                V.axpby(out, dMx, self.prob.F(x, p), 1.0)
            return out
        out = V.scale(J(du), self.M(x))
        if len(self.M):
            V.axpby(out, self.M.dM(x, du), self.prob.F(x, p), 1.0)
        return out


class DeflatedProblemCustomLS:
    """(:247-310)"""

    def __init__(self, solver):
        self.solver = solver

    def __call__(self, J, rhs):
        u, p, dp = J
        fused = dp.M.runs_fused(u)
        Fu = dp.prob.F(u, p)
        Mu = None if fused else dp.M(u)
        Ju = dp.prob.J(u, p)
        if len(dp.M) == 0:
            h1, ok, it1 = self.solver(Ju, rhs)
            return h1, ok, (it1, 0)
        h1, h2, ok, its = self.solver(Ju, rhs, Fu)   # two right-hand sides
        tmp = V.zeros_like(u)
        if fused:
            Mu, (z1, z2) = dp.M.values(u, (h1, h2))   # M(u), dM.h1, dM.h2 from one pass
        else:
            tmp2 = V.zeros_like(u)
            z1 = dp.M.dM(u, h1, tmp, tmp2)
            z2 = dp.M.dM(u, h2, tmp, tmp2)
        z = z1 / (Mu + z2)
        V.copyto(tmp, h1)
        V.axpby(tmp, -z, h2, 1.0)
        V.scale(tmp, 1.0 / Mu)
        return tmp, True, its


def newton_deflated(prob, x0, p, defop, opts, normN=V.norm2, callback=None):
    """solve(prob, defOp, options) (:340-356): Newton on M(u) F(u) with the custom linear solver around opts.linsolver."""
    dprob = DeflatedProblem(prob, defop)
    return newton(dprob, x0, p, _replace(opts, linsolver=DeflatedProblemCustomLS(opts.linsolver)), normN, callback)


def newton_deflated_or_fail(prob, x0, p, defop, opts, normN=V.norm2, callback=None):
    """newton_deflated, with a diverging run (iterates beyond float range, where the reference's cbMaxNorm(1e100) stops) or an
    iterate exactly on a deflated root (M(u) = 1 / 0, an infinite residual in the reference) returned as a failed solve from
    the guess"""
    try:
        return newton_deflated(prob, x0, p, defop, opts, normN, callback)
    except (ZeroDivisionError, OverflowError):
        return NonLinearSolution(V.copy(x0), p, [math.inf], False, 0, 0)


def newton_two_guesses(prob, x0, x1, p, opts, defop=None, normN=V.norm2):
    """newton(prob, x0, x1, p0, options, defOp) (:392-420) -> (sol1, sol0, ok): converge from x0, deflate that root, then
    converge from x1 to a different one."""
    defop = defop or DeflationOperator(2, 1.0, [])
    sol0 = newton(prob, x0, p, opts, normN)
    assert sol0.converged, "Newton did not converge to the trivial solution x0."
    defop.push(sol0.u)
    sol1 = newton_deflated(prob, x1, p, defop, _replace(opts, max_iterations=10 * opts.max_iterations), normN)  # (:401)
    return sol1, sol0, sol0.converged and sol1.converged
