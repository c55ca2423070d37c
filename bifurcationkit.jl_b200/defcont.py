"""Deflated continuation (src/DeflatedContinuation.jl:14-356) -- host orchestration over palc.ContIterable.

Every step moves the parameter by ds and continues each active branch with a deflated Newton solve from its current point,
deflated against the points the branches before it reached at this step; then, from each active branch, deflated Newton solves
from the (perturbed) branch point look for solutions not yet known, and each one found starts a new branch (Farrell, Beentjes
and Birkisson, "The computation of disconnected bifurcation diagrams", arXiv:1603.00809).  The branches of a snaking system,
such as the localized fronts of examples/SH2d-fronts.jl:168-180, coexist at every parameter value and are found this way.

One deliberate difference: the reference recomputes a branch's tangent and predictor around each deflated solve (getpredictor!,
:113,127), but nothing in deflated continuation reads them -- the solve starts from the branch point -- and with z_old.p set to
the new parameter the secant of a branch that does not move in u is 0/0.  They are left as the start-up made them.

The deflation operator is built with ``fused=True``: on device vectors M(u) and its derivatives in a deflated Newton iteration
come from one ``bk_deflation_moments`` pass, and so do the distances of a candidate to the known roots (the m_i / s_i of the
kernel for ``normC`` = norminf / norm2).
"""
from dataclasses import dataclass, field, replace as _replace
import math

from .deflation import DeflationOperator, newton_deflated_or_fail
from .events import Branch, branch_row, detect_bifurcation, get_bifurcation_type, getinterval
from .palc import PALC, V, ContIterable, re_make


def _perturb_solution(x, p, idb):
    return x


def _accept_solution(x, p):
    return True


def _update_deflation_op(defop, x, p):
    defop.push(x)


@dataclass
class DefCont:
    """DefCont (src/DeflatedContinuation.jl:14-33), jacobian = DeflatedProblemCustomLS()"""
    deflation_operator: DeflationOperator = None
    alg: PALC = field(default_factory=PALC)
    max_branches: int = 100
    seek_every_step: int = 1
    max_iter_defop: int = 5
    perturb_solution: object = _perturb_solution
    accept_solution: object = _accept_solution
    update_deflation_op: object = _update_deflation_op


@dataclass
class DCState:
    """DCState (:87-93): a branch's continuation state and whether the branch is still followed"""
    state: object
    isactive: bool = True


@dataclass
class DCBranch(Branch):
    """a branch of deflated continuation: the rows of events.continuation, its guess-type special points, and `sol`, the saved
    solutions dict(x, p, step) (every save_sol_every_step steps, and the last point of a branch that stops)"""
    sol: list = field(default_factory=list)


@dataclass
class DCResult:
    """DCResult (:60-71): the branches, and the final solutions of the branches still active"""
    branches: list
    sol: list
    states: list
    alg: DefCont


def distances(defop, u, others, normC):
    """[normC(u - r) for r in others]: from the m_i (norminf) or s_i (norm2) of one bk_deflation_moments pass where the operator
    runs fused at u, else by vector operations"""
    if others and defop.runs_fused(u) and normC in (V.norminf, V.norm2):
        s, m, _, _ = u.ctx.deflation_moments(u, others)
        return [float(x) for x in m] if normC is V.norminf else [math.sqrt(x) for x in s]
    out, tmp = [], V.copy(u)
    for r in others:
        V.copyto(tmp, u)
        V.axpby(tmp, -1.0, r, 1.0)
        out.append(normC(tmp))
    return out


def _new_branch(it, sol_every):
    """iterate(contIt) (the start-up of src/Continuation.jl:349-405) and ContResult(it, state): the first point of a branch"""
    st = it.start()
    it.eigen(st)
    br = DCBranch(state=st)
    _save(br, it, st, sol_every)
    return DCState(st), br


def _save(br, it, st, sol_every):
    """save! (src/Continuation.jl:280-304)"""
    br.rows.append(branch_row(it.prob, it.contpar, st))
    if sol_every > 0 and st.step % sol_every == 0:
        br.sol.append(dict(x=V.copy(st.z_u), p=st.z_p, step=st.step))


def continuation(prob, alg, contpar, normC=V.norm2, callback_newton=None, save_sol_every_step=1, verbosity=0):
    """continuation(prob, alg::DefCont, contParams) (:196-356) -> DCResult.  `save_sol_every_step` is the field of the
    reference's ContinuationPar (default 1); 0 saves the first point of each branch only, as the reference does (:238-239)."""
    cp = contpar
    opts = cp.newton_options
    alg = _replace(alg, max_iter_defop=alg.max_iter_defop * opts.max_iterations)   # (:223)
    if alg.deflation_operator is None or len(alg.deflation_operator) == 0:
        raise ValueError("You must provide at least one guess")
    defop = alg.deflation_operator.copy()
    defop.fused = True
    sol_every = save_sol_every_step if save_sol_every_step > 0 else 10 ** 14
    it = ContIterable(prob, alg.alg, cp, normC, callback_newton)

    # start-up (:157-166): every branch starts from iterate(contIt) with prob.u0 = roots[1]
    it.prob = re_make(prob, V.copy(defop.roots[0]), prob.p0)
    states, branches = [], []
    for _ in defop.roots:
        dcs, br = _new_branch(it, sol_every)
        states.append(dcs)
        branches.append(br)

    def update_branch(dcs, br, p):
        """updatebranch! (:100-153)"""
        if not dcs.isactive:
            return False, 0
        st = dcs.state
        sol = newton_deflated_or_fail(it.prob, st.z_u, p, defop, opts, normC, callback_newton)
        if sol.converged:
            V.copyto(st.z_u, sol.u)
            st.z_p = p
            st.zold_p = p
            alg.update_deflation_op(defop, sol.u, p)
            it.eigen(st)
            if cp.detect_bifurcation > 1 and detect_bifurcation(st):
                bp = get_bifurcation_type(it, st, "guess", getinterval(p, p - st.ds))
                if bp.type != "none":
                    bp.idx = len(br.rows)
                    br.specialpoint.append(bp)
            st.step += 1
            _save(br, it, st, sol_every)
        else:
            dcs.isactive = False
            br.sol.append(dict(x=V.copy(st.z_u), p=st.z_p, step=st.step))
        return sol.converged, sol.itnewton

    def new_solution(dcs, p, idb):
        """_DC_get_new_solution (:269-286)"""
        u0 = alg.perturb_solution(V.copy(dcs.state.z_u), p, idb)
        pb = re_make(it.prob, u0, p)
        sol = newton_deflated_or_fail(pb, u0, p, defop, _replace(opts, max_iterations=alg.max_iter_defop), normC, callback_newton)
        if sol.converged:
            sol.converged = normC(it.prob.F(sol.u, p)) < opts.tol     # the residual of the problem itself (:281)
        if sol.converged:
            d = distances(defop, sol.u, defop.roots + [dcs.state.z_u], normC)
            if len(d) > 1 and min(d[:-1]) < opts.tol:                    # a known root (:282)
                sol.converged = False
            sol.same = d[-1] < opts.tol                                  # the branch's own point (:334)
        return sol

    current = prob.p0
    nstep = 0
    while ((cp.p_min < current < cp.p_max) or nstep == 0) and nstep < cp.max_steps:
        current = min(max(current + cp.ds, cp.p_min), cp.p_max)        # clamp_predp
        defop.roots.clear()
        for idb, (dcs, br) in enumerate(zip(states, branches)):
            ok, itn = update_branch(dcs, br, current)
            if verbosity >= 2 and dcs.isactive:
                print(f"step {nstep} p={current:.6e}: branch {idb} in {itn} iterations", flush=True)
        nbrs = len(states)
        nactive = sum(d.isactive for d in states)
        if nstep % alg.seek_every_step == 0 and nactive < alg.max_branches:
            n_active = 0
            for idb in range(nbrs):                      # not the branches found at this step
                dcs = states[idb]
                if not (dcs.isactive and n_active < alg.max_branches):
                    continue
                n_active += 1
                success = True
                while success:
                    sol = new_solution(dcs, current, idb)
                    success = sol.converged
                    if success and sol.same:
                        if verbosity >= 1:
                            print("Same solution found for identical parameter value!!", flush=True)
                        success = False
                    if success and alg.accept_solution(sol.u, current):
                        if verbosity >= 1:
                            print(f"step {nstep} p={current:.6e}: new solution from branch {idb}", flush=True)
                        defop.roots.append(sol.u)
                        itn = ContIterable(re_make(it.prob, sol.u, current), alg.alg, cp, normC, callback_newton)
                        new, br = _new_branch(itn, sol_every)
                        new.isactive = n_active + 1 < alg.max_branches
                        states.append(new)
                        branches.append(br)
        nstep += 1
    return DCResult(branches, [d.state.z_u for d in states if d.isactive], states, alg)
