"""Numbers for the other BASELINE.json configs (kernel-level, CUDA-event timed):
  [1] SH2d 512^2 GMRES(100): fused JVP+Arnoldi GB/s          [4] cGL2d 512^2 Trapeze M=30: po_jvp GB/s, bordered MF GMRES it/s
  [5] SH3d 128^3: Newton to the pattern + shift-invert Arnoldi k=10 eigenpairs, s/eigensolve
  [6] periodic spectral SH2d, the reference GPU example at its own size (examples/SH2d-fronts-cuda.jl: 512^2, lx = 16 pi,
      ly = 8 pi / sqrt(3), (l, nu) = (-0.15, 1.3)): Newton to the hexagons, one GMRES(50) with Pl = (L1 + I)^-1 fused (one
      transform per Arnoldi step) and unfused at equal iteration counts, the same at 1024^2, with the card and its power limit
Prints one JSON object per config."""
import json, os, subprocess, sys, time
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import __graft_entry__ as g
import bench

bk = g.load_package(); P = bk.palc
which = sys.argv[1:] or ["1", "4", "5"]


def ev_time(ctx, fn, reps=20, warm=3):
    stream = torch.cuda.ExternalStream(ctx.lib.bk_stream(ctx.handle))
    for _ in range(warm): fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ctx.sync(); e0.record(stream)
    for _ in range(reps): fn()
    e1.record(stream); ctx.sync()
    return e0.elapsed_time(e1) / reps


if "1" in which:
    for n in (512, 1024):
        ctx = bk.Context(bk.BK_SH2D, (n, n), bench.domain(n), krylov_m=100, params=bench.PAR)
        u = ctx.to_device(bench.sol0(n)); rhs = ctx.to_device(np.random.default_rng(1234).standard_normal(n * n))
        J = ctx.jacobian(u); ls = bk.GMRESB200(reltol=1e-30, restart=100, maxiter=100)
        ctx.set_timing(True)
        for _ in range(3): ls(J, rhs)
        s = ctx.stats()
        print(json.dumps({"config": f"SH2d {n}^2 GMRES(100), no preconditioner", "fused_ms": s["last_fused_ms"], "fused_GB": s["last_fused_bytes"] / 1e9,
                          "fused_GBps": s["last_fused_bytes"] / 1e6 / s["last_fused_ms"], "frac_of_measured_peak": s["last_fused_bytes"] / 1e6 / s["last_fused_ms"] / bench.measured_peak()[0],
                          "jvp_us": ev_time(ctx, lambda: ctx.jvp(rhs, u)) * 1e3, "residual_us": ev_time(ctx, lambda: ctx.residual(rhs, u)) * 1e3}), flush=True)
        del ctx

if "4" in which:
    nx = ny = int(os.environ.get("BK_CGL_N", "512")); M = 30
    L = (np.pi, np.pi / 2)
    n = nx * ny
    hx, hy = 2 * L[0] / nx, 2 * L[1] / ny
    lam1 = -(2 - 2 * np.cos(np.pi / (nx + 1))) / hx**2 - (2 - 2 * np.cos(np.pi / (ny + 1))) / hy**2
    r = -lam1 - 0.01  # r_hopf - 0.01 as examples/cGL2d.jl:177 (r_hopf = -lambda_1(Lap), analytic: SURVEY 8d)
    pars = (r, 0.1, 1.0, -1.0, 1.0)
    ctx = bk.Context(bk.BK_POTRAP_CGL2D, (nx, ny, M), L, krylov_m=60, params=pars)
    i = np.arange(1, nx + 1); j = np.arange(1, ny + 1)
    phi11 = (np.sin(np.pi * i / (nx + 1))[None, :] * np.sin(np.pi * j / (ny + 1))[:, None]).reshape(-1)
    amp = 1.0  # orbit guess x_k = a phi11 [cos t_k; sin t_k], T = 2 pi (cf. cGL2d.jl:171-174)
    xs = np.concatenate([np.concatenate([amp * phi11 * np.cos(2 * np.pi * k / M), amp * phi11 * np.sin(2 * np.pi * k / M)]) for k in range(M)] + [np.array([2 * np.pi])])
    N = ctx.N
    x = ctx.to_device(xs)
    f1 = ctx.residual(x).numpy()[: 2 * n]
    phi = np.zeros(N - 1); phi[: 2 * n] = f1 / np.linalg.norm(f1)  # section through the first slice (cf. cGL2d.jl:177-181)
    ctx.potrap_set_section(phi, np.zeros(N - 1))
    dx = ctx.to_device(np.random.default_rng(0).standard_normal(N)); out = ctx.zeros()
    J = ctx.jacobian(x)
    t_res = ev_time(ctx, lambda: ctx.residual(x, out)); t_jvp = ev_time(ctx, lambda: ctx.jvp(dx, out))
    ctx.precond_setup(bk.BK_PC_POTRAP_CIRC, 2 * np.pi)  # time-circulant / DST preconditioner (stand-in for the example's ILU)
    t_pc = ev_time(ctx, lambda: ctx.precond_apply(dx, out), reps=5, warm=1)
    ls = bk.GMRESB200(reltol=float(os.environ.get("BK_PO_RELTOL", "1e-3")), restart=40, maxiter=50, Pr=True,
                      orth=os.environ.get("BK_PO_ORTH", "cgs2"))  # examples/cGL2d.jl:213: reltol 1e-3, restart 40, maxiter 50
    prob = P.BifurcationProblemB200(ctx, x, pars, lens=0)
    ctx.sync(); t0 = time.perf_counter()
    NT = float(os.environ.get('BK_PO_NEWTON_TOL', '1e-8' if nx <= 256 else '1e-6'))
    po = P.newton(prob, x, r, P.NewtonPar(tol=NT, max_iterations=20, linsolver=ls), P.norminf)
    ctx.sync(); t_newton = time.perf_counter() - t0
    upo = po.u.numpy()
    # one bordered matrix-free solve at the orbit (the PALC corrector's linear system)
    Jpo = ctx.jacobian(po.u)
    rhs = ctx.to_device(np.random.default_rng(1).standard_normal(N))
    tau = ctx.to_device(np.random.default_rng(2).standard_normal(N)); dR = ctx.to_device(np.random.default_rng(3).standard_normal(N))
    bls = bk.MatrixFreeBLSB200(ls)
    bls(Jpo, dR, tau, 0.7, rhs, 0.1, 0.5, 0.5, dotscale=1.0 / N)
    ctx.sync(); t0 = time.perf_counter()
    dX, dl, ok, it = bls(Jpo, dR, tau, 0.7, rhs, 0.1, 0.5, 0.5, dotscale=1.0 / N)
    ctx.sync(); t_solve = time.perf_counter() - t0
    # Floquet exponents of the orbit (SURVEY 8f.1): matrix-free monodromy = M-1 shifted JVPs + shifted GMRES solves
    floq = None
    if os.environ.get("BK_PO_FLOQUET", "1") == "1":
        try:
            ctx_vf = bk.Context(bk.BK_CGL2D, (nx, ny), L, krylov_m=40, params=pars)
            Tpo = float(upo[-1])
            bk.floquet.cgl_shifted_precond(ctx_vf, Tpo, M, r)
            lsf = bk.GMRESB200(reltol=1e-8, restart=40, maxiter=40, Pr=True)
            fl = bk.floquet.FloquetQaDB200(ctx_vf, lsf, M, eigsolver=bk.floquet.ArnoldiLMB200(krylovdim=int(os.environ.get("BK_FLOQUET_KDIM", "16")), tol=1e-6, maxrestart=2))
            ctx.sync(); ctx_vf.sync(); t0 = time.perf_counter()
            sig, _, cvf, info = fl(po.u, 3)
            ctx_vf.sync(); t_fl = time.perf_counter() - t0
            floq = {"exponents_sigma": [[float(z.real), float(z.imag)] for z in sig], "converged": bool(cvf), "seconds": t_fl,
                    "monodromy_applications": info["monodromy_applications"], "shifted_solves": info["solves"], "gmres_its": info["linear_its"]}
            del ctx_vf
        except Exception as e:  # keep the rest of the config line
            floq = {"error": str(e)[:200]}
    # continuation of the periodic orbit in r: PALC + MatrixFreeBLS (continuation_po with linear_algo = MatrixFreeBLS(ls))
    prob2 = P.BifurcationProblemB200(ctx, po.u, pars, lens=0, record=lambda v: v.norminf())
    cp = P.ContinuationPar(dsmin=1e-4, dsmax=0.03, ds=0.001, p_min=r - 1.0, p_max=2.5, max_steps=8,   # cGL2d.jl:197 opts_po_cont
                           newton_options=P.NewtonPar(tol=NT, max_iterations=15, linsolver=ls))
    print(json.dumps({"po_newton_residuals": po.residuals, "converged": po.converged, "linear_its": po.itlineartot}), flush=True)
    ctx.sync(); t0 = time.perf_counter()
    try:
        rows, st = P.continuation(prob2, P.PALC(bls=bls), cp, normC=P.norminf)
    except RuntimeError as e:
        print("continuation failed:", str(e)[:300], flush=True)
        rows = []
    ctx.sync(); t_cont = time.perf_counter() - t0
    print(json.dumps({"config": f"cGL2d {nx}^2 Trapeze M={M} (N={N}), matrix-free Newton + bordered MF solve, circulant/DST preconditioner",
                      "po_residual_ms": t_res, "po_jvp_ms": t_jvp, "po_jvp_GBps": 24 * N / 1e6 / t_jvp, "precond_ms": t_pc,
                      "po_newton": {"converged": po.converged, "its": po.itnewton, "linear_its": po.itlineartot, "seconds": t_newton,
                                    "period_T": float(upo[-1]), "max_abs_u": float(np.max(np.abs(upo[:-1])))},
                      "bordered_mf_solve_s": t_solve, "gmres_iters": it, "converged": ok, "floquet": floq,
                      "po_continuation": {"steps": len(rows) - 1, "seconds": t_cont, "rows": [[round(q["param"], 6), round(q["x"], 6), q["itnewton"], q["itlinear"]] for q in rows]}}), flush=True)
    del ctx, x, dx, out, rhs, tau, dR

if "5" in which:
    n3 = 128
    Lz = np.pi * n3 / 22.0  # mesh width of examples/SH3d.jl:69-70 (22^3 on pi)
    L3 = (Lz, Lz, Lz)
    ctx = bk.Context(bk.BK_SH3D, (n3, n3, n3), L3, krylov_m=150, params=(0.1, 1.2))
    X = -Lz + 2 * Lz / n3 * np.arange(n3)
    s0 = (np.cos(X)[None, None, :] * np.cos(X)[None, :, None] * np.ones(n3)[:, None, None])
    s0 = s0 - s0.min(); s0 = s0 / s0.max() * 1.2
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    ls = bk.GMRESB200(reltol=1e-9, restart=150, maxiter=150, Pr=True, orth="cgs2")  # rtol of examples/SH3d.jl:93
    ls_newton = bk.GMRESB200(reltol=1e-6, restart=150, maxiter=150, Pr=True)
    # Newton from the raw guess wanders at this domain size (many unstable directions); relax it first with the
    # semi-implicit gradient flow u <- u + (L1 + 1/dt + sigma)^-1 F(u) (same DCT solver, shift 4), then polish with Newton
    u_dev = ctx.to_device(s0.reshape(-1)); fbuf = ctx.zeros(); pbuf = ctx.zeros()
    ctx.precond_setup(bk.BK_PC_SH_DCT, 4.0)
    ctx.sync(); t0 = time.perf_counter()
    for _ in range(400):
        ctx.residual(u_dev, fbuf); ctx.precond_apply(fbuf, pbuf); u_dev.axpby_(1.0, pbuf, 1.0)
    relax_res = ctx.residual(u_dev, fbuf).norminf()
    ctx.sync(); t_relax = time.perf_counter() - t0
    ctx.precond_setup(bk.BK_PC_SH_DCT, 1.0)
    prob = P.BifurcationProblemB200(ctx, u_dev, (0.1, 1.2), lens=0)
    ctx.sync(); t0 = time.perf_counter()
    sol = P.newton(prob, prob.u0, 0.1, P.NewtonPar(tol=1e-8, max_iterations=30, linsolver=ls_newton), P.norminf)
    ctx.sync(); t_newton = time.perf_counter() - t0
    eig = bk.ShiftInvertB200(0.1, ls, krylovdim=40, tol=1e-8, maxrestart=5)
    J = ctx.jacobian(sol.u)
    ctx.sync(); t0 = time.perf_counter()
    vals, _, cv, nops = eig(J, 10)
    ctx.sync(); t_eig = time.perf_counter() - t0
    print(json.dumps({"config": f"SH3d {n3}^3, shift-invert Arnoldi k=10 (sigma=0.1, krylovdim 40, inner GMRES rtol 1e-9)", "newton_converged": sol.converged,
                      "relax_s": t_relax, "residual_after_relaxation": relax_res, "newton_its": sol.itnewton, "newton_linear_its": sol.itlineartot, "newton_s": t_newton, "residuals": sol.residuals[-3:],
                      "eig_s": t_eig, "eig_converged": cv, "inner_solves": nops, "eigenvalues": [float(v.real) for v in vals]}), flush=True)

if "6" in which:
    def card():
        try:
            q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                               capture_output=True, text=True, timeout=30).stdout.strip()
        except (OSError, subprocess.TimeoutExpired):
            q = ""
        return {"name": torch.cuda.get_device_name(), "nvidia_smi": q}

    PAR6 = (-0.15, 1.3)
    out = {"config": "periodic SH2d (examples/SH2d-fronts-cuda.jl), GMRES(50) with Pl = (L1 + I)^-1", "card": card(),
           "operator_bytes_per_arnoldi_step": {"fused": "64N", "unfused": "112N"}}
    for n in (512, 1024):
        lx, ly = 16 * np.pi * n / 512, 8 * np.pi / np.sqrt(3) * n / 512   # the example's domain at 512^2, scaled to keep sol0 periodic
        ctx = bk.Context(bk.BK_SH2D_PERIODIC, (n, n), (lx, ly), krylov_m=50, params=PAR6)
        ctx.precond_setup(bk.BK_PC_SH_FFT, 1.0)
        X = -lx + 2 * lx / n * np.arange(n); Y = -ly + 2 * ly / n * np.arange(n)
        u0 = (0.5 * (np.cos(X)[None, :] + np.cos(X / 2)[None, :] * np.cos(np.sqrt(3.0) * Y / 2)[:, None])).reshape(-1)
        ls = bk.GMRESB200(reltol=1e-8, restart=50, maxiter=300, Pl=True)
        prob = P.BifurcationProblemB200(ctx, ctx.to_device(u0), PAR6, lens=0)
        ctx.sync(); t0 = time.perf_counter()
        sol = P.newton(prob, prob.u0, PAR6[0], P.NewtonPar(tol=1e-6, max_iterations=10, linsolver=ls), P.norminf)
        ctx.sync(); t_newton = time.perf_counter() - t0
        J = ctx.jacobian(sol.u)
        rhs = ctx.to_device(np.random.default_rng(6).standard_normal(n * n))
        per = {"fused": {"us_per_iteration_rounds": []}, "unfused": {"us_per_iteration_rounds": []}}
        for _ in range(3):                # alternate the two variants; reltol 0: exactly 50 iterations (one cycle) either way
            for fused in (True, False):
                g50 = bk.GMRESB200(reltol=0.0, restart=50, maxiter=50, Pl=True, fused=fused)
                its = []
                ms = ev_time(ctx, lambda: its.append(g50(J, rhs)[2]), reps=10, warm=2)
                d = per["fused" if fused else "unfused"]
                d["iterations"] = its[-1]
                d["us_per_iteration_rounds"].append(ms * 1e3 / its[-1])
        for d in per.values():
            d["us_per_iteration"] = float(np.median(d["us_per_iteration_rounds"]))
        out[f"{n}^2"] = {"newton_converged": sol.converged, "newton_its": sol.itnewton, "newton_linear_its": sol.itlineartot,
                         "newton_s": t_newton, "norminf_u": float(sol.u.norminf()), "gmres50": per,
                         "fused_speedup": per["unfused"]["us_per_iteration"] / per["fused"]["us_per_iteration"]}
        del ctx, J, rhs, sol, prob
    print(json.dumps(out), flush=True)
