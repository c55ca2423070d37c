"""NumPy / SciPy restatement of the normal form of a branch point with an N-dimensional kernel (get_normal_formNd,
src/NormalForms.jl:656-896, autodiff = false) for host arrays, the checker of normalform.get_normal_formNd.  Test infrastructure
only; the product never imports it.  It takes the biorthogonal bases as given and solves every singular system with the N-border
direct solve [J Z★; Z' 0] (sparse LU), whose solution satisfies <ζ_i, ψ> = 0 for every i; it loops over every index tuple, with no
cache and no symmetry shortcut.  Also: the contractions <v_i, d2F[v_j, v_k]> / <v_i, d3F[v_j, v_k, v_l]> with the sums of the
absolute values of their pointwise terms, which set the tolerance of a reordered sum."""
import numpy as np
import scipy.sparse as sp
import scipy.sparse.linalg as spla


def nd_normal_form(F, Jfun, d2F, d3F, x0, p, delta, zetas, zetas_ad):
    """F(x, p), Jfun(p) (the Jacobian at x0, sparse or dense), d2F(a, b), d3F(a, b, c) at (x0, p) -> dict a01, a02, b11, b20, b30"""
    N = len(zetas)
    Z, Za = np.column_stack(zetas), np.column_stack(zetas_ad)
    J = sp.csc_matrix(Jfun(p))
    lu = spla.splu(sp.bmat([[J, sp.csc_matrix(Za)], [sp.csc_matrix(Z.T), None]]).tocsc())
    E = lambda x: x - Z @ (Za.T @ x)
    solve = lambda r: lu.solve(np.concatenate([r, np.zeros(N)]))[:-N]
    Jp, Jm = sp.csc_matrix(Jfun(p + delta)), sp.csc_matrix(Jfun(p - delta))
    R01 = (F(x0, p + delta) - F(x0, p - delta)) / (2 * delta)
    R02 = (F(x0, p + delta) - 2 * F(x0, p) + F(x0, p - delta)) / delta**2
    a01 = Za.T @ R01
    psi01 = solve(-E(R01))
    b11 = np.array([[Za[:, i] @ ((Jp @ Z[:, j] - Jm @ Z[:, j]) / (2 * delta) + d2F(Z[:, j], psi01)) for j in range(N)]
                    for i in range(N)])
    a2v = R02 + 2 * (Jp @ psi01 - Jm @ psi01) / (2 * delta) + d2F(psi01, psi01)
    a02 = Za.T @ a2v
    b20 = np.zeros((N, N, N))
    b30 = np.zeros((N, N, N, N))
    w = lambda a, b: solve(E(d2F(Z[:, a], Z[:, b])))
    for j in range(N):
        for k in range(N):
            b20[:, j, k] = Za.T @ d2F(Z[:, j], Z[:, k])
            for l in range(N):
                b3v = (d3F(Z[:, j], Z[:, k], Z[:, l]) - d2F(Z[:, j], w(l, k)) - d2F(Z[:, k], w(l, j)) - d2F(Z[:, l], w(k, j)))
                b30[:, j, k, l] = Za.T @ b3v
    return dict(a01=a01, a02=a02, b11=b11, b20=b20, b30=b30)


def moments(d2F, d3F, vecs, idx2, idx3):
    """(values, sums of |terms|) of the contractions <v_i, d2F[v_j, v_k]> (rows of idx2) then <v_i, d3F[v_j, v_k, v_l]> (idx3)"""
    val, scale = [], []
    for i, j, k in np.reshape(idx2, (-1, 3)):
        t = vecs[i] * d2F(vecs[j], vecs[k])
        val.append(t.sum())
        scale.append(np.abs(t).sum())
    for i, j, k, l in np.reshape(idx3, (-1, 4)):
        t = vecs[i] * d3F(vecs[j], vecs[k], vecs[l])
        val.append(t.sum())
        scale.append(np.abs(t).sum())
    return np.array(val), np.array(scale)
