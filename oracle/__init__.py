"""CPU oracle for the PALC Newton-Krylov corrector path of BifurcationKit.jl.

TEST INFRASTRUCTURE ONLY.  This package is a NumPy/SciPy restatement of the
reference's algorithms on the hot path (SURVEY.md section 8a); it is imported only by
``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs, as the checker.  Nothing under
``bifurcationkit.jl_b200/`` imports it and the product path never falls back to it.

Parity status: the reference is pure Julia and ``julia`` is absent from this image,
and the Krylov arithmetic lives in un-vendored packages (IterativeSolvers.jl,
KrylovKit.jl, ArnoldiMethod.jl: Project.toml:45-57, no Manifest), so the
reference itself cannot be run here.  The oracle is pinned against every
known-answer test the reference holds for this path (tests/test_oracle_*.py
restate test/linear_solvers/test_linear.jl, test/continuation/*.jl,
test/newton/test_newton.jl, test/periodic_orbits_function_fd/test_potrap.jl);
GMRES *iterates* and iteration counts are "parity unpinned" (the reference's
own tests only pin solutions against dense solves).

All citations ``file:line`` are relative to the root of the BifurcationKit.jl source tree.
"""
