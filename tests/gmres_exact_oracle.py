"""GMRES(m) with libbk200's driver semantics, in 80-bit long double.  Test infrastructure only.

The fp64 oracle (oracle/krylov.py) is itself a rounded computation, so a device solve can only be held to it within the sum
of two rounding errors.  This module computes the iterates of exact GMRES(m) to ~1e-19 instead, so that a comparison with the
device measures the device's rounding alone.  It follows ``bk_gmres_dev`` (csrc/bk_krylov.cu) rule for rule:

1. ``tol = max(reltol * beta0, abstol)``, beta0 = ||Pl r0|| (the preconditioned initial residual when Pl is on);
2. ``x0 = 0``;
3. each cycle minimises ||Pl r_c - Pl A Pr V y|| over K_k(Pl A Pr, Pl r_c) and updates ``x += Pr V y``;
4. a cycle starts from the recomputed true residual and the solve stops as soon as that residual is <= tol;
5. ``iters`` counts Arnoldi columns, capped by ``maxiter`` (the last cycle may be partial);
6. the cycle length is ``min(restart, krylov_m, n)``;
7. when the solve runs single-pass CGS and a cycle ends converged with ``k >= 40`` columns or ``reltol < 1e-9`` (and
   ``iters < maxiter``), the true residual is recomputed and accepted when <= 4 tol.  In exact arithmetic the check always
   passes; the reference counts it (``checks``) so that a test can count the extra operator application.

The Krylov basis is orthogonalised by modified Gram-Schmidt applied twice, in long double.  Operators and preconditioners are
built from the fp64 oracle's coefficients (cast exactly: every fp64 value is a long double) and applied in long double:
SH2d / SH3d (Neumann, matrix-free through the sparse L1 rows, so 1024^2 stays cheap), chan, cGL and its transpose, the Trapeze
functional over cGL, periodic SH2d through separable DFT matrices, bordered maps with one or two borders, and the
real-equivalent 2 N0 map of a complex shift; the DCT, DST and FFT preconditioners through separable transform matrices, chan's
tridiagonal one by the Thomas algorithm and the Trapeze circulant one as the inverse of the operator that defines it.
"""
import numpy as np

LD = np.longdouble
EPS_LD = float(np.finfo(LD).eps)
EPS = float(np.finfo(np.float64).eps)
if not EPS_LD <= 1.1e-19:
    raise ImportError(f"gmres_exact_oracle needs 80-bit long double (eps <= 1.1e-19); this platform's is {EPS_LD:.3e}")


_PI_LD = LD(np.pi) + LD(1.2246467991473532e-16)  # pi to long-double precision: fp64 pi plus its fp64 remainder


def ld(a):
    """fp64 values cast exactly to long double"""
    return np.asarray(a, dtype=np.float64).astype(LD)


def nrm(v):
    return np.sqrt(np.dot(v, v))


# ---------------------------------------------------------------------------------------------------------------- operators
class SparseLD:
    """y = M x in long double for an fp64 scipy sparse M: each row summed in order over its stored entries."""

    def __init__(self, M):
        M = M.tocsr()
        M.sort_indices()
        assert np.all(np.diff(M.indptr) > 0), "every row needs a stored entry (reduceat)"
        self.data, self.indices, self.start = ld(M.data), M.indices, M.indptr[:-1]
        self.shape = M.shape

    def __call__(self, x):
        return np.add.reduceat(self.data * x[self.indices], self.start)


def sh_op(sh, u, a0=0.0, a1=1.0):
    """v -> a0 v + a1 (-L1 v + (l + 2 nu u - 3 u^2) v) for an oracle.problems.SwiftHohenberg (2-D or 3-D, Neumann)"""
    L1 = SparseLD(sh.L1)
    uu = ld(u)
    d = LD(sh.l) + LD(2.0) * LD(sh.nu) * uu - LD(3.0) * uu * uu
    a0, a1 = LD(a0), LD(a1)
    return lambda v: a0 * v + a1 * (d * v - L1(v))


def chan_op(u, alpha, beta, a0=0.0, a1=1.0):
    """v -> a0 v + a1 dF_chan(u) v (oracle.problems.chan_dF)"""
    n = len(u)
    x = ld(u)[1:-1]
    bb, s = LD(beta), LD(float((n - 1) ** 2))
    dn = LD(alpha) * (LD(1) - bb * x * x + LD(2) * LD(0.5) * x) / (LD(1) + bb * x * x) ** 2
    a0, a1 = LD(a0), LD(a1)

    def apply(v):
        out = np.empty_like(v)
        out[0], out[-1] = v[0], v[-1]
        out[1:-1] = (v[:-2] - LD(2) * v[1:-1] + v[2:]) * s + dn * v[1:-1]
        return a0 * v + a1 * out

    return apply


def _cgl_coefs(gl, u):
    n = gl.n
    u1, u2 = ld(u[:n]), ld(u[n:])
    mu, nu, c3, c5, r = (LD(t) for t in (gl.mu, gl.nu, gl.c3, gl.c5, gl.r))
    k11 = -5 * c5 * u1**4 + (-6 * c5 * u2**2 - 3 * c3) * u1**2 + 2 * mu * u1 * u2 - c5 * u2**4 - c3 * u2**2 + r
    k12 = -4 * c5 * u2 * u1**3 + mu * u1**2 + (-4 * c5 * u2**3 - 2 * c3 * u2) * u1 + 3 * u2**2 * mu - nu
    k21 = -4 * c5 * u2 * u1**3 - 3 * mu * u1**2 + (-4 * c5 * u2**3 - 2 * c3 * u2) * u1 - u2**2 * mu + nu
    k22 = -c5 * u1**4 + (-6 * c5 * u2**2 - c3) * u1**2 - 2 * mu * u1 * u2 - 5 * c5 * u2**4 - 3 * c3 * u2**2 + r
    ua = u1 * u1 + u2 * u2
    f = np.concatenate([r * u1 - nu * u2 - ua * (c3 * u1 - mu * u2) - c5 * ua * ua * u1,
                        r * u2 + nu * u1 - ua * (c3 * u2 + mu * u1) - c5 * ua * ua * u2])
    return k11, k12, k21, k22, f


def cgl_op(gl, u, a0=0.0, a1=1.0, transpose=False):
    """v -> a0 v + a1 dF(u) v (or dF(u)' v) for an oracle.problems.GinzburgLandau2D (Delta is symmetric)"""
    Delta = SparseLD(gl.Delta)
    n = gl.n
    k11, k12, k21, k22, _ = _cgl_coefs(gl, u)
    if transpose:
        k12, k21 = k21, k12
    a0, a1 = LD(a0), LD(a1)

    def apply(v):
        d1, d2 = v[:n], v[n:]
        return a0 * v + a1 * (np.concatenate([k11 * d1 + k12 * d2, k21 * d1 + k22 * d2]) + Delta(v))

    return apply


def trapeze_op(gl, x, phi, M, a0=0.0, a1=1.0):
    """v -> a0 v + a1 J_T(x) v, the Jacobian of the Trapeze functional over cGL (oracle.potrap.Trapeze.jvp): rows
    i = 0..M-2  (dv_i - dv_{i-1}) - h/2 (J_i dv_i + J_{i-1} dv_{i-1}) - dh/2 (F_i + F_{i-1}),  dv_{-1} = dv_{M-2};
    row M-1  dv_{M-1} - dv_0;  last entry <dv, phi>.  h = T / M, dh = dT / M."""
    N = gl.N
    T = LD(float(x[-1]))
    u = x[:-1].reshape(M, N)
    ops = [cgl_op(gl, u[i]) for i in range(M)]
    Fs = [_cgl_coefs(gl, u[i])[4] + SparseLD(gl.Delta)(ld(u[i])) for i in range(M)]
    ph = ld(phi)
    a0, a1 = LD(a0), LD(a1)
    h = T / M

    def apply(v):
        dv = v[:-1].reshape(M, N)
        dh = v[-1] / M
        out = np.empty_like(v)
        o = out[:-1].reshape(M, N)
        Js = [ops[i](dv[i]) for i in range(M - 1)]
        for i in range(M - 1):
            p = i - 1 if i > 0 else M - 2
            o[i] = (dv[i] - dv[p]) - h / 2 * (Js[i] + Js[p]) - dh / 2 * (Fs[i] + Fs[p])
        o[M - 1] = dv[M - 1] - dv[0]
        out[-1] = np.dot(v[:-1], ph)
        return a0 * v + a1 * out

    return apply


def complex_op(J, N0, a0=0.0, a0_imag=0.0, a1=1.0):
    """the real-equivalent 2 N0 map of ((a0 + i a0_imag) I + a1 J) on z = [x; y], J a real long-double map on N0-vectors"""
    a0, ai, a1 = LD(a0), LD(a0_imag), LD(a1)

    def apply(z):
        x, y = z[:N0], z[N0:]
        return np.concatenate([a0 * x - ai * y + a1 * J(x), ai * x + a0 * y + a1 * J(y)])

    return apply


def _dft_matrix(n):
    """F[j, k] = exp(-2 pi i j k / n) in complex long double"""
    jk = (np.arange(n)[:, None] * np.arange(n)[None, :]) % n
    ang = (LD(2) * _PI_LD / n) * jk.astype(LD)
    return np.cos(ang) - 1j * np.sin(ang).astype(np.clongdouble)


def periodic_symbol_apply(dims, sym):
    """r -> real(ifft2(fft2(r) * sym)) by separable long-double DFT matrices, sym (Ny, Nx) fp64 cast exactly"""
    Nx, Ny = dims
    Fx, Fy = _dft_matrix(Nx), _dft_matrix(Ny)
    s = ld(sym)

    def apply(r):
        U = Fy @ r.reshape(Ny, Nx).astype(np.clongdouble) @ Fx
        return np.real(np.conj(Fy) @ (U * s) @ np.conj(Fx)).reshape(-1) / LD(Nx * Ny)

    return apply


def periodic_sh_op(psh, u, a0=0.0, a1=1.0):
    """v -> a0 v + a1 (-L1 v + (l + 2 nu u - 3 u^2) v) for a tests.sh_periodic_oracle.PeriodicSH"""
    L1 = periodic_symbol_apply(psh.dims, psh.symbol)
    uu = ld(u)
    d = LD(psh.l) + LD(2.0) * LD(psh.nu) * uu - LD(3.0) * uu * uu
    a0, a1 = LD(a0), LD(a1)
    return lambda v: a0 * v + a1 * (d * v - L1(v))


def fft_precond(psh, shift=1.0):
    """r -> (L1 + shift I)^-1 r (PeriodicSH.precond, BK_PC_SH_FFT) with the fp64 symbol 1 / (symbol + shift)"""
    sym = 1.0 / (psh.symbol + shift)
    apply = periodic_symbol_apply(psh.dims, sym)
    apply.norm = float(np.max(np.abs(sym)))
    return apply


def bordered_op(A, a, b, c, dotscale=1.0):
    """x = [xu; xp] -> [A xu + sum_i xp_i a_i; c xp + dotscale <b_i, xu>] (oracle.bls.MatrixFreeBLSmapBlock, m = len(a)),
    A the long-double map of the N block (its shift included)"""
    a, b = [ld(t) for t in a], [ld(t) for t in b]
    m = len(a)
    C = ld(np.atleast_2d(c))
    ds = LD(dotscale)

    def apply(x):
        xu, xp = x[:-m], x[-m:]
        top = A(xu)
        for i in range(m):
            top = top + a[i] * xp[i]
        bot = C @ xp + ds * np.array([np.dot(b[i], xu) for i in range(m)], dtype=LD)
        return np.concatenate([top, bot])

    return apply


def dense(A, n):
    """the n x n long-double matrix of a linear map (small n only)"""
    I = np.eye(n, dtype=LD)
    return np.stack([A(I[:, j]) for j in range(n)], axis=1)


def direct_solve(M, b, steps=6):
    """M^-1 b in long double for a dense long-double M: an fp64 LU solve refined on long-double residuals (converges to
    long-double accuracy while cond(M) eps64 << 1)"""
    M64 = M.astype(np.float64)
    b = ld(b) if b.dtype != LD else b
    x = np.linalg.solve(M64, b.astype(np.float64)).astype(LD)
    for _ in range(steps):
        x = x + np.linalg.solve(M64, (b - M @ x).astype(np.float64)).astype(LD)
    return x


# ------------------------------------------------------------------------------------------------------- preconditioners
def dct2_matrix(n):
    """the orthonormal DCT-II matrix (scipy.fft.dct(type=2, norm='ortho') as C @ x) in long double"""
    k = np.arange(n, dtype=LD)[:, None]
    i = np.arange(n, dtype=LD)[None, :]
    C = np.cos(_PI_LD * k * (2 * i + 1) / (2 * n)) * np.sqrt(LD(2) / n)
    C[0] /= np.sqrt(LD(2))
    return C


def dct_precond(dims, lengths, shift=1.0):
    """r -> (L1 + shift I)^-1 r (oracle.precond.dct_precond) by separable long-double DCT matrices, 2-D"""
    from oracle import precond as oprecond
    assert len(dims) == 2
    Nx, Ny = dims
    Cx, Cy = dct2_matrix(Nx), dct2_matrix(Ny)
    sym = ld(oprecond.sh_symbol(dims, lengths, shift))

    def apply(r):
        R = Cy @ r.reshape(Ny, Nx) @ Cx.T
        return (Cy.T @ (R / sym) @ Cx).reshape(-1)

    apply.norm = float(1.0 / np.min(np.abs(oprecond.sh_symbol(dims, lengths, shift))))
    return apply


def dst1_matrix(n):
    """the orthonormal DST-I matrix (scipy.fft.dst(type=1, norm='ortho') as S @ x) in long double"""
    jk = (np.arange(1, n + 1)[:, None] * np.arange(1, n + 1)[None, :]) % (2 * (n + 1))
    return np.sin(_PI_LD * jk.astype(LD) / (n + 1)) * np.sqrt(LD(2) / (n + 1))


def dst_precond(gl, a0, a1):
    """BK_PC_CGL_DST: (a0 I + a1 Lap_dirichlet)^-1 on each n = Nx Ny component of a cGL vector (oracle.precond.
    dst_helmholtz_precond per component), by separable long-double DST-I matrices"""
    from oracle import precond as oprecond
    Nx, Ny, n = gl.Nx, gl.Ny, gl.n
    Sx, Sy = dst1_matrix(Nx), dst1_matrix(Ny)
    ex = oprecond.dirichlet_eigs(Nx, 2 * gl.lx / Nx)
    ey = oprecond.dirichlet_eigs(Ny, 2 * gl.ly / Ny)
    sym64 = a0 + a1 * (ex[None, :] + ey[:, None])
    sym = ld(sym64)

    def one(r):
        return (Sy @ ((Sy @ r.reshape(Ny, Nx) @ Sx) / sym) @ Sx).reshape(-1)

    def apply(r):
        return np.concatenate([one(r[i * n:(i + 1) * n]) for i in range(len(r) // n)])

    apply.norm = float(1.0 / np.min(np.abs(sym64)))
    return apply


def chan_precond(n):
    """BK_PC_CHAN_TRIDIAG: r -> P^-1 r with P the tridiagonal matrix of oracle.problems.chan_precond_matrix, by the Thomas
    algorithm in long double (P is diagonally dominant: no pivoting)"""
    from oracle import problems
    P = problems.chan_precond_matrix(n).toarray()
    lo, di, up = ld(np.r_[0.0, np.diag(P, -1)]), ld(np.diag(P)), ld(np.r_[np.diag(P, 1), 0.0])

    def apply(r):
        c, d = np.empty(n, dtype=LD), np.empty(n, dtype=LD)
        c[0], d[0] = up[0] / di[0], r[0] / di[0]
        for i in range(1, n):
            m = di[i] - lo[i] * c[i - 1]
            c[i] = up[i] / m
            d[i] = (r[i] - lo[i] * d[i - 1]) / m
        x = np.empty(n, dtype=LD)
        x[-1] = d[-1]
        for i in range(n - 2, -1, -1):
            x[i] = d[i] - c[i] * x[i + 1]
        return x

    apply.norm = float(np.linalg.norm(np.linalg.inv(P), 2))
    return apply


def potrap_circ_operator(gl, M, T):
    """the operator that BK_PC_POTRAP_CIRC inverts (oracle.precond.potrap_circulant_precond): the Trapeze Jacobian of cGL
    linearised at the trivial state, rows i = 0..M-2  A x_i - B x_{i-1} (x_{-1} = x_{M-2}), A = I - h/2 J0,
    B = I + h/2 J0, J0 = Lap_dirichlet + r + nu R; row M-1  x_{M-1} - x_0; identity on the period entry"""
    N, n = gl.N, gl.n
    lap = SparseLD(gl.lap)
    r, nu, h = LD(gl.r), LD(gl.nu), LD(T) / M

    def J0(v):
        v1, v2 = v[:n], v[n:]
        return np.concatenate([lap(v1) + r * v1 - nu * v2, lap(v2) + r * v2 + nu * v1])

    def apply(v):
        x = v[:-1].reshape(M, N)
        out = v.copy()
        o = out[:-1].reshape(M, N)
        Jx = [J0(x[i]) for i in range(M - 1)]
        for i in range(M - 1):
            p = i - 1 if i > 0 else M - 2
            o[i] = (x[i] - h / 2 * Jx[i]) - (x[p] + h / 2 * Jx[p])
        o[M - 1] = x[M - 1] - x[0]
        return out

    return apply


def potrap_circ_precond(gl, M, T):
    """BK_PC_POTRAP_CIRC from its definition: the long-double inverse of potrap_circ_operator (dense, small grids)"""
    import scipy.linalg as sla
    n = gl.N * M + 1
    C = dense(potrap_circ_operator(gl, M, T), n)
    C64 = C.astype(np.float64)
    lu = sla.lu_factor(C64)

    def apply(v):
        x = sla.lu_solve(lu, v.astype(np.float64)).astype(LD)
        for _ in range(4):  # refined on long-double residuals
            x = x + sla.lu_solve(lu, (v - C @ x).astype(np.float64)).astype(LD)
        return x

    apply.norm = float(np.linalg.norm(np.linalg.inv(C64), 2))
    return apply


def bordered_precond(P, m):
    """P on the N block, identity on the m border entries"""
    return lambda v: np.concatenate([P(v[:-m]), v[-m:]])


# ----------------------------------------------------------------------------------------------------------------- GMRES
class Result:
    pass


def gmres(A, b, *, reltol=1e-8, abstol=0.0, restart=200, krylov_m=None, maxiter=100, Pl=None, Pr=None, orth="cgs",
          keep_x=True):
    """GMRES(m) with libbk200's semantics (module docstring).  A, Pl, Pr: long-double maps (Pl / Pr apply the inverse).
    Returns a Result with
      x, converged, iters, tol, beta0, checks (true-residual checks of rule 7), restart (after rule 6);
      rho[k]    the exact minimal residual after k columns (rho[0] = beta0), on the side that carries tol;
      xs[k]     the iterate after k columns (if keep_x), xs[0] = 0;
      z[k]      V y of the cycle in progress after k columns (x_k = x_cycle + Pr z_k);
      cond[k]   the 2-norm condition number of the cycle's (j+1) x j Hessenberg after k columns, hnorm[k] its 2-norm,
                ynorm[k] the norm of its least-squares solution y;
      cycles    the column counts at which a cycle started."""
    Pl = Pl or (lambda v: v)
    Pr = Pr or (lambda v: v)
    b = ld(b) if b.dtype != LD else b
    n = len(b)
    m = min(restart, krylov_m if krylov_m is not None else restart, n)
    R = Result()
    R.restart = m
    R.rho, R.xs, R.z, R.cond, R.hnorm, R.ynorm, R.cycles = [], [], [], [], [], [], []
    R.checks = 0
    x = np.zeros(n, dtype=LD)
    x_zero = True
    total = 0
    first = True
    verify = False
    conv = False
    while True:
        r = Pl(b if x_zero else b - A(x))
        beta = nrm(r)
        if first:
            R.beta0 = beta
            R.tol = max(LD(reltol) * beta, LD(abstol))
            R.rho.append(beta)
            R.xs.append(x.copy())
            R.z.append(np.zeros(n, dtype=LD))
            R.cond.append(1.0)
            R.hnorm.append(0.0)
            R.ynorm.append(0.0)
            first = False
        tol = R.tol
        if verify:
            verify = False
            R.checks += 1
            assert beta <= 4 * tol, "exact GMRES failed its own true-residual check"
            conv = True
            break
        if not (beta > tol) or total >= maxiter or not (beta > 0):
            conv = beta <= tol
            break
        R.cycles.append(total)
        V = np.zeros((m + 1, n), dtype=LD)
        H = np.zeros((m + 1, m), dtype=LD)
        V[0] = r / beta
        k = 0
        res = beta
        xc = x.copy()
        while k < m and total < maxiter:
            w = Pl(A(Pr(V[k])))
            for _ in range(2):  # MGS, twice
                for i in range(k + 1):
                    h = np.dot(V[i], w)
                    H[i, k] += h
                    w = w - h * V[i]
            hk1 = nrm(w)
            # happy breakdown: the new direction is rounding noise of a column that already lies in the space
            if hk1 <= 64 * EPS_LD * nrm(H[: k + 1, k]):
                hk1 = LD(0)
            H[k + 1, k] = hk1
            if hk1 > 0:
                V[k + 1] = w / hk1
            k += 1
            total += 1
            Hk = H[: k + 1, :k]
            g = np.zeros(k + 1, dtype=LD)
            g[0] = beta
            Q, Rr = np.linalg.qr(Hk.astype(np.float64))  # fp64 only to start the long-double refinement below
            y = _lstsq_ld(Hk, g, Q, Rr)
            res = nrm(g - Hk @ y)
            zk = V[:k].T @ y
            R.rho.append(res)
            R.z.append(zk)
            sv = np.linalg.svd(Hk.astype(np.float64), compute_uv=False)
            R.cond.append(float(sv[0] / sv[-1]) if sv[-1] > 0 else np.inf)
            R.hnorm.append(float(sv[0]))
            R.ynorm.append(float(nrm(y)))
            if keep_x or res <= tol or total >= maxiter or hk1 == 0 or k == m:
                xk = xc + Pr(zk)
            R.xs.append(xk if keep_x else None)
            if res <= tol or hk1 == 0:
                break
        x = xk
        x_zero = False
        conv = res <= tol
        if conv and orth == "cgs" and (k >= 40 or reltol < 1e-9) and total < maxiter:
            verify = True
            continue
        if conv or total >= maxiter:
            break
    R.x, R.converged, R.iters = x, bool(conv), total
    if not keep_x:
        R.xs[-1] = x
    return R


def _lstsq_ld(H, g, Q, Rr):
    """min ||g - H y|| in long double: the fp64 QR solution refined by corrected semi-normal equations"""
    y = np.linalg.solve(Rr, Q.T @ g.astype(np.float64)).astype(LD)
    Rl = Rr.astype(LD)
    for _ in range(4):
        r = g - H @ y
        t = H.T @ r                                 # R^T R dy = H^T r
        s = _trisolve(Rl.T, t, lower=True)
        dy = _trisolve(Rl, s, lower=False)
        y = y + dy
    return y


def _trisolve(T, v, lower):
    n = len(v)
    out = np.zeros(n, dtype=LD)
    rng = range(n) if lower else range(n - 1, -1, -1)
    for i in rng:
        acc = v[i] - (T[i, :i] @ out[:i] if lower else T[i, i + 1:] @ out[i + 1:])
        out[i] = acc / T[i, i]
    return out


def first_gap(rho, ratio=1.5, start=1):
    """the first k >= start with rho[k] / rho[k+1] >= ratio, and the geometric mean of the two: a tolerance that ends the
    exact solve at column k + 1 with a margin of sqrt(ratio) either way"""
    for k in range(start, len(rho) - 1):
        if rho[k + 1] > 0 and rho[k] / rho[k + 1] >= ratio:
            return k, float(np.sqrt(rho[k] * rho[k + 1]))
    raise ValueError("no step with the requested contraction")
