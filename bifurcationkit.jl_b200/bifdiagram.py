"""Automatic bifurcation diagrams (src/bifdiagram/BifurcationDiagram.jl:106-237) -- host orchestration over the branch switching
of normalform.py, like codim2.py and defcont.py.

Mirror of the reference:
  BifDiagNode              <->  BifDiagNode (:18-30), with from(γ) kept as `nf`
  get_branch               <->  get_branch(diagram, code) (:70-78); node[code] the same
  get_branches_from_BP     <->  get_branches_from_BP(diagram, indbif) (:80-104)
  size / level             <->  Base.size (:61-63), level (:34)
  bifurcationdiagram       <->  bifurcationdiagram(prob, alg, level, options) (:106-127)
  bifurcationdiagram_from  <->  bifurcationdiagram(prob, br, maxlevel, options) (:129-142)
  bifurcationdiagram_      <->  bifurcationdiagram!(prob, node, maxlevel, options) (:157-231)

The branching rule is the reference's: a special point is branched when its step is > 1 and its type is bp or nd; the child's
ContinuationPar is options(x, p, level + 1) with ds multiplied by the branch's dsfactor; a kernel of dimension 1 goes to
continuation_from_bp, a larger one to multicontinuation; a Transcritical point also gets the branch with ds -> -ds and a
Pitchfork the one with ampfactor -1, unless halfbranch; a Fold adds nothing.  An exception while branching at a point is
recorded on the node (`failures`) and the other points and the rest of the tree go on.

What differs is when the branches are computed.  The branches leaving one node are independent, so the work at each special
point -- its whole branch switching, including the second Transcritical / Pitchfork branch -- is one unit, and up to
`max_workers` units run at once on host threads (ctypes releases the GIL during every library call).  Each running unit has
its own Context, a `Context.replicate` of the problem's, with its own stream and workspace; every reduction of the library has
an order fixed by the grid, so a unit gives the bits it would give alone, and the children are added in the reference's order
whatever order the units end in.  A unit reads the parent branch's vectors from the diagram's context (synchronised before the
units start) with one device-to-device copy each; when it ends, every device vector its branches and normal forms keep is
copied onto the diagram's context and the unit's context is closed, so at most max_workers + 1 contexts exist at any time.
All calls on the diagram's context are made by the calling thread.  max_workers = 1 runs the same code one unit at a time.
Host problems (no `ctx`) take the same path, with a copy of the problem per unit.

Shared solver objects: every unit continues with shallow copies of the PALC, its bordered solver, the ContinuationPar, its
NewtonPar and their linear and eigen solvers (`_private`), since GMRESB200 writes `last_resnorm` during a call; the others
write nothing during a call.

Not here: usedeflation = true, diagrams of periodic orbits, plotting.
"""
from concurrent.futures import ThreadPoolExecutor, wait, FIRST_COMPLETED
import copy
import dataclasses
from dataclasses import dataclass, field, replace
import inspect
import traceback
import types

from .core import DeviceVec
from . import lib as _l
from .palc import V
from . import events, normalform


@dataclass
class BifDiagNode:
    """A node of the diagram: its recursion level, `code` = the index in the parent branch's specialpoint list of the point this
    branch starts from (None at the root), the branch `gamma` (events.Branch), the children, `nf` = the normal form the branch
    comes from (from(γ); None at the root) and `failures` = (special point index, parameter, exception) of every point whose
    branch switching raised."""
    level: int
    code: object
    gamma: object
    child: list = field(default_factory=list)
    nf: object = None
    failures: list = field(default_factory=list)

    def __getitem__(self, code):
        return get_branch(self, code if isinstance(code, tuple) else (code,))


def level(node):
    return node.level


def hasbranch(node):
    return node.gamma is not None


def size(node, code=()):
    """the number of branches in the tree below get_branch(node, code), itself included (:61-63)"""
    node = get_branch(node, code)
    return 1 + sum(size(c) for c in node.child)


def get_branch(node, code):
    """node.child[code[0]].child[code[1]]... (:70-78); indices are 0-based"""
    for i in code:
        node = node.child[i]
    return node


def get_branches_from_BP(node, ind):
    """the children of node that branch off its special point `ind` (0-based): those whose normal form sits at its parameter
    (:80-104)"""
    p = node.gamma.specialpoint[ind].param
    return [c for c in node.child if c.nf is not None and c.nf.p == p]


def _as_function(options):
    """options: a ContinuationPar or a callable (x, p, level) -> ContinuationPar (:129-135)"""
    return options if callable(options) else (lambda x, p, lvl: options)


def bifurcationdiagram(prob, alg, level, options, normC=V.norm2, halfbranch=False, verbose=False, max_workers=None, **kwargs):
    """bifurcationdiagram(prob, alg, level, options) (:106-127): the root branch by events.continuation with options(prob.u0,
    prob.params, 1), then the diagram below it up to `level` (bifurcationdiagram_).  kwargs go to the branch-switching calls
    (continuation_from_bp or multicontinuation, each receiving those it takes; a keyword neither takes is refused) and, where
    events.continuation takes them (callback), to the root branch, with verbose."""
    _check_kwargs(kwargs)
    opts = _as_function(options)
    root_kw = {k: v for k, v in kwargs.items() if k in ("callback",)}
    gamma = events.continuation(prob, alg, opts(prob.u0, prob.params, 1), normC, verbose=verbose, **root_kw)
    return bifurcationdiagram_from(prob, gamma, level, options, alg=alg, normC=normC, halfbranch=halfbranch, verbose=verbose,
                                   max_workers=max_workers, **kwargs)


def bifurcationdiagram_from(prob, br, maxlevel, options, alg, **kwargs):
    """bifurcationdiagram(prob, br, maxlevel, options) (:129-142): the diagram below the branch br of prob, whose branches are
    continued with alg (the reference takes it from br)"""
    if kwargs.get("verbose"):
        print("━" * 50 + "\n───▶ Automatic computation of bifurcation diagram\n", flush=True)
    return bifurcationdiagram_(prob, BifDiagNode(1, None, br), maxlevel, options, alg, **kwargs)


def bifurcationdiagram_(prob, node, maxlevel, options, alg, normC=V.norm2, halfbranch=False, verbose=False, max_workers=None,
                        code=(), **kwargs):
    """bifurcationdiagram!(prob, node, maxlevel, options) (:157-231): branch at every bp / nd point of node.gamma with step > 1,
    add the branches, continued with alg, as children in the reference's order, then recurse into each child, until the level
    maxlevel.  max_workers: how many special points are branched at once, min(their number, 4) by default.  Returns node."""
    _check_kwargs(kwargs)
    if node.level >= maxlevel or node.gamma is None:
        return node
    opts = _as_function(options)
    inds = [i for i, pt in enumerate(node.gamma.specialpoint) if pt.step > 1 and pt.type in ("bp", "nd")]   # :180-182

    def unit(ind, ctx):
        return _branch_at(prob, alg, node, ind, ctx, opts, normC, halfbranch, verbose, code, kwargs)

    workers = min(len(inds), 4) if max_workers is None else max_workers
    for ind, (kids, err) in zip(inds, _run_units(getattr(prob, "ctx", None), inds, unit, workers)):
        pt = node.gamma.specialpoint[ind]
        for br, nf in kids:
            node.child.append(BifDiagNode(node.level + 1, ind, br, nf=nf))
        if err is not None:                                                              # :206-208
            node.failures.append((ind, pt.param, _detached(err)))
            if verbose:
                print(f"Failed to compute new branch at p = {pt.param}: {err!r}", flush=True)
    for ii, nd in enumerate(node.child):
        bifurcationdiagram_(prob, nd, maxlevel, options, alg, normC=normC, halfbranch=halfbranch, verbose=verbose,
                            max_workers=max_workers, code=code + (ii,), **kwargs)
    return node


def _branch_at(prob, alg, node, ind, ctx, opts, normC, halfbranch, verbose, code, kwargs):
    """one unit: the branches off node.gamma.specialpoint[ind] on the context ctx (None for a host problem), as the loop body of
    :178-205.  Returns (list of (Branch, normal form), the exception that ended it or None); the branches computed before an
    exception are kept, as the reference's add! before it."""
    kids = []
    try:
        p = prob.replicate(ctx) if hasattr(prob, "replicate") else copy.copy(prob)
        br = _moved(node.gamma, ctx, {}, only=ind)
        pt = br.specialpoint[ind]
        lvl = node.level
        if verbose:
            print("─" * 80 + f"\n──▶ New branch, level = {lvl + 1}, dim(Kernel) = {abs(pt.delta[0])}, code = {code}, "
                  f"from bp #{ind} at p = {pt.param}, type = {pt.type}", flush=True)

        def letsbranch(dsfactor=1.0, ampfactor=1.0):                                    # :170-178
            a, cp = _private(alg, opts(pt.x, pt.param, lvl + 1))
            cp = replace(cp, ds=cp.ds * dsfactor)
            kw = {"nev": cp.nev, **kwargs, "normC": normC, "ampfactor": ampfactor}   # `nev = optscont.nev, kwargs..., ampfactor`
            if "bls" in kw:
                kw["bls"] = copy.copy(kw["bls"])
            if abs(pt.delta[0]) > 1:
                f = normalform.multicontinuation
                return f(br, ind, p, a, cp, **_accepted(f, kw))
            f = normalform.continuation_from_bp
            return f(br, ind, p, a, cp, **_accepted(f, kw))

        gamma = letsbranch()
        if gamma is None:                                                                # a Fold: no branch
            return kids, None
        if isinstance(gamma, list):                                                      # multicontinuation
            kids += gamma
            return kids, None
        kids.append(gamma)
        if verbose:
            print(f"────▶ From {gamma[1].type}", flush=True)
        if not halfbranch and gamma[1].type == "Transcritical":                          # :195-204
            gamma = letsbranch(dsfactor=-1.0)
            kids.append(gamma)
        if not halfbranch and gamma[1].type == "Pitchfork":
            gamma = letsbranch(ampfactor=-1.0)
            kids.append(gamma)
    except Exception as e:
        return kids, e
    return kids, None


_SWITCHING = (normalform.continuation_from_bp, normalform.multicontinuation)


def _check_kwargs(kwargs):
    """refuse what the branch-switching calls would not take: usedeflation = true (not supported here) and any keyword neither
    continuation_from_bp nor multicontinuation has (a misspelling would otherwise be ignored)"""
    if kwargs.pop("usedeflation", False):
        raise NotImplementedError("bifurcationdiagram: usedeflation = true is not supported")
    names = set().union(*(inspect.signature(f).parameters for f in _SWITCHING)) - {"br", "ind_bif", "prob", "alg", "contpar"}
    unknown = sorted(set(kwargs) - names)
    if unknown:
        raise TypeError(f"bifurcationdiagram: unexpected keyword argument(s) {unknown}")


def _detached(err):
    """err without a traceback, its traceback kept as text in a note: the unit's frames (and the frames that called them) hold
    the node, so a failure kept on the node with its traceback would make the whole tree, device vectors included, a
    reference cycle that only the cyclic collector frees.  The same for the exceptions it chains."""
    err.add_note("Traceback of the failed unit (most recent call last):\n" + "".join(traceback.format_tb(err.__traceback__)))
    todo, seen = [err], set()
    while todo:
        e = todo.pop()
        if e is None or id(e) in seen:
            continue
        seen.add(id(e))
        e.__traceback__ = None
        todo += [e.__cause__, e.__context__]
    return err


def _accepted(f, kw):
    names = inspect.signature(f).parameters
    return {k: v for k, v in kw.items() if k in names}


def _private(alg, cp):
    """shallow copies of the solver objects a unit uses -- the PALC, its bordered solver and that solver's linear solver, the
    ContinuationPar, its NewtonPar, the Newton linear solver and the eigensolver with its linear solver -- so that what one unit
    writes into a solver during a call (GMRESB200.last_resnorm) is not what another reads"""
    def cp1(obj, *attrs):
        obj = copy.copy(obj)
        for a in attrs:
            if getattr(obj, a, None) is not None:
                setattr(obj, a, copy.copy(getattr(obj, a)))
        return obj
    no = cp.newton_options
    no = replace(no, linsolver=copy.copy(no.linsolver), eigsolver=cp1(no.eigsolver, "ls"))
    return replace(alg, bls=cp1(alg.bls, "solver")), replace(cp, newton_options=no)


def _moved(obj, ctx, memo, only=None):
    """obj with every DeviceVec it holds (in lists, tuples, dicts, dataclasses, namespaces) replaced by a copy on ctx; None
    leaves obj as it is.  Shared vectors stay shared (memo).  only: for an events.Branch, copy the vectors of that one special
    point and of the saved eigen-elements, and share the rest."""
    if ctx is None:
        return obj
    key = id(obj)
    if key in memo:
        return memo[key]
    if isinstance(obj, DeviceVec):
        out = ctx.copy_from(obj)
    elif isinstance(obj, list):
        out = [_moved(v, ctx, memo) for v in obj]
    elif isinstance(obj, tuple):
        out = tuple(_moved(v, ctx, memo) for v in obj)
    elif isinstance(obj, dict):
        out = {k: _moved(v, ctx, memo) for k, v in obj.items()}
    elif only is not None and isinstance(obj, events.Branch):
        sp = list(obj.specialpoint)
        sp[only] = _moved(sp[only], ctx, memo)
        out = events.Branch(rows=obj.rows, specialpoint=sp, eig=_moved(obj.eig, ctx, memo), state=None)
    elif (dataclasses.is_dataclass(obj) and not isinstance(obj, type)) or isinstance(obj, types.SimpleNamespace):
        out = copy.copy(obj)
        for k, v in vars(obj).items():
            setattr(out, k, _moved(v, ctx, memo))
    else:
        out = obj
    memo[key] = out
    return out


def _out_of_memory(e):
    return "out of memory" in str(e) or "cudaErrorMemoryAllocation" in str(e)


def _run_units(root, inds, unit, max_workers):
    """unit(ind, ctx) for every ind, at most max_workers at once, each on a new root.replicate() (None when root is None) that is
    closed when its results have been moved onto root.  A context that cannot be created for lack of memory waits for a running
    unit to end; with none running the error is raised.  Returns the units' results in the order of inds."""
    if not inds:
        return []
    if root is not None:
        root.sync()   # the parent branch's vectors are read from the units' streams
    results, pending, running = {}, list(inds), {}
    pool = ThreadPoolExecutor(max(1, max_workers))
    try:
        while pending or running:
            while pending and len(running) < max(1, max_workers):
                try:
                    ctx = None if root is None else root.replicate()
                except _l.BK200Error as e:
                    if not running or not _out_of_memory(e):
                        raise
                    break
                ind = pending.pop(0)
                running[pool.submit(unit, ind, ctx)] = (ind, ctx)
            done, _ = wait(running, return_when=FIRST_COMPLETED)
            for fut in done:
                ind, ctx = running.pop(fut)
                try:
                    kids, err = fut.result()
                    if ctx is not None:
                        ctx.sync()
                        kids = _moved(kids, root, {})
                        root.sync()
                    results[ind] = (kids, err)
                finally:
                    if ctx is not None:
                        ctx.close()
    finally:
        for fut, (_, ctx) in running.items():   # after an error: let the other units end, then close their contexts
            fut.exception()
            if ctx is not None:
                ctx.close()
        pool.shutdown(wait=True)
    return [results[i] for i in inds]
