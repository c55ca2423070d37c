"""The Trapeze Jacobian as a sparse matrix (po_jacobian_sparse, src/periodicorbit/PeriodicOrbitTrapeze.jl:469-486), with the
phase row and the period column -- the reference for J and J' of BK_POTRAP_CGL2D at any size.  Test infrastructure only.

Rows 0..M-2: (I - h/2 A_sl) x_sl + (-I - h/2 A_sp) x_sp with sp(0) = M-2 and h/2 = T/(2M), A_k = J_F(x_k); row M-1: x_{M-1} - x_0;
last row: phi'.  The period column is the analytic derivative -(f_sl + f_sp) / (2M), f_k = F(x_k), which is what the Trapeze JVP
(oracle/potrap.py, the device kernel) computes; the reference's line 476 takes a forward difference in T instead."""
import numpy as np
import scipy.sparse as sp


def po_jacobian_sparse(jac, F, x, M, N, phi):
    """jac(u) -> J_F(u) as an N x N sparse matrix, F(u) -> F(u); x = [x_0 .. x_{M-1}; T]; phi: the section (N M values)"""
    T = x[-1]
    u = x[:-1].reshape(M, N)
    h2 = T / (2 * M)
    I = sp.identity(N, format="csr")
    A = [sp.csr_matrix(jac(u[k])) for k in range(M - 1)]
    f = [F(u[k]) for k in range(M - 1)]
    blocks = [[None] * M for _ in range(M)]
    col = np.zeros(N * M)
    for sl in range(M - 1):
        spv = sl - 1 if sl > 0 else M - 2
        for k, blk in ((sl, I - h2 * A[sl]), (spv, -I - h2 * A[spv])):
            blocks[sl][k] = blk if blocks[sl][k] is None else blocks[sl][k] + blk
        col[sl * N:(sl + 1) * N] = -(f[sl] + f[spv]) / (2 * M)
    blocks[M - 1][M - 1] = I
    blocks[M - 1][0] = -I if M > 1 else None
    J = sp.bmat(blocks, format="csr")
    return sp.bmat([[J, sp.csr_matrix(col[:, None])], [sp.csr_matrix(np.asarray(phi)[None, :]), None]], format="csr")


def cgl_jac_sparse(gl, u, r=None):
    """J_F(u) of oracle.problems.GinzburgLandau2D as a sparse matrix: the Dirichlet Laplacian on both components plus the 2 x 2
    reaction block of dNL at every point"""
    n = gl.n
    e1 = np.concatenate([np.ones(n), np.zeros(n)])
    c1, c2 = gl.dNL(u, e1, r), gl.dNL(u, 1.0 - e1, r)    # [a11; a21] and [a12; a22]
    R = sp.bmat([[sp.diags(c1[:n]), sp.diags(c2[:n])], [sp.diags(c1[n:]), sp.diags(c2[n:])]])
    return (gl.Delta + R).tocsr()


def cgl_po_jacobian(gl, x, M, phi, r=None):
    return po_jacobian_sparse(lambda u: cgl_jac_sparse(gl, u, r), lambda u: gl.F(u, r), x, M, gl.N, phi)


def potrap_circulant_matrix(Nx, Ny, lx, ly, M, T, r, nu):
    """The matrix P whose inverse oracle.precond.potrap_circulant_precond applies: the Trapeze rows and the closure row of the
    cGL Jacobian at the trivial state (J0 = Lap_dirichlet + r + nu R on every slice), identity on the period"""
    from oracle import problems
    gl = problems.GinzburgLandau2D(Nx, Ny, lx, ly, r=r, mu=0.0, nu=nu, c3=0.0, c5=0.0)
    x = np.zeros(gl.N * M + 1)
    x[-1] = T
    P = po_jacobian_sparse(lambda u: cgl_jac_sparse(gl, u, r), lambda u: np.zeros(gl.N), x, M, gl.N, np.zeros(gl.N * M)).tolil()
    P[-1, -1] = 1.0
    return P.tocsr()
