"""NumPy / SciPy restatement of the BK_RD problem kind (include/bk200.h): F_i(u) = D_i Lap u_i + R_i(u) on a 1-D or 2-D grid,
state [u_1; ..; u_F], with the kron-built Laplacians of the reference examples and the polynomial R evaluated term by term, and
its exact J, J', d2F and d3F.  Test infrastructure only: the product never imports it.

A model is given as the arguments of bk.ReactionDiffusion: fields, bc ("neumann" / "dirichlet"), diffusion (D or (scale, pexp)
per field), terms ((eq, scale, pexp, fexp) tuples, exponents as lists or {index: exponent} dicts), nparams, ndims."""
import itertools
import math

import numpy as np
import scipy.sparse as sp


def lap1d(n, l, bc):
    """the second-difference matrix with h = 2 l / n: Neumann = clamp closure (corner -1/h^2, examples/pd-1d.jl), Dirichlet =
    diagonal -2/h^2 everywhere (examples/cGL2d.jl:6-22)"""
    h = 2 * l / n
    D = sp.diags([np.ones(n - 1), -2 * np.ones(n), np.ones(n - 1)], [-1, 0, 1]).tolil() / h**2
    if bc == "neumann":
        D[0, 0] = D[n - 1, n - 1] = -1 / h**2
    return D.tocsr()


def laplacian(dims, lengths, bc):
    if len(dims) == 1:
        return lap1d(dims[0], lengths[0], bc)
    nx, ny = dims
    return (sp.kron(sp.identity(ny), lap1d(nx, lengths[0], bc)) + sp.kron(lap1d(ny, lengths[1], bc), sp.identity(nx))).tocsr()


def _exps(e, n):
    out = [0] * n
    for k, v in (e.items() if isinstance(e, dict) else enumerate(e)):
        out[int(k)] = int(v)
    return out


def _ff(a, k):
    """the falling factorial a (a - 1) .. (a - k + 1)"""
    return math.prod(a - q for q in range(k))


class RD:
    def __init__(self, fields, bc, diffusion, terms, nparams, ndims, dims, lengths, params):
        self.F, self.nd = fields, ndims
        self.dims = tuple(dims[:ndims])
        self.n = int(np.prod(self.dims))
        self.N = self.F * self.n
        self.bc = bc
        self.lap = laplacian(self.dims, lengths, bc)
        self.p = np.asarray(params, dtype=float)
        mono = lambda s, pe: s * np.prod([self.p[k] ** e for k, e in enumerate(_exps(pe, nparams)) if e != 0])
        self.D = [mono(*((d, ()) if np.isscalar(d) else d)) for d in diffusion]
        self.terms = [(eq, mono(s, pe), _exps(fe, fields)) for eq, s, pe, fe in terms]
        self.Delta = sp.block_diag([D * self.lap for D in self.D]).tocsr()

    def fields_of(self, u):
        return [u[i * self.n:(i + 1) * self.n] for i in range(self.F)]

    def _deriv(self, U, al, beta):
        """d^beta of prod_j u_j^al_j at the fields U (beta a multi-index)"""
        out = np.ones(self.n)
        for j in range(self.F):
            c = _ff(al[j], beta[j])
            if c == 0:
                return np.zeros(self.n)
            out = out * c * U[j] ** (al[j] - beta[j])
        return out

    def _jet(self, u, dirs):
        """sum over the terms of c_t sum_{k_1..k_m} d^m m_t / du_k1 .. du_km  dirs[0]_k1 .. dirs[m-1]_km  (m = len(dirs))"""
        U = self.fields_of(u)
        V = [self.fields_of(d) for d in dirs]
        out = [np.zeros(self.n) for _ in range(self.F)]
        for eq, c, al in self.terms:
            for ks in itertools.product(range(self.F), repeat=len(dirs)):
                beta = [ks.count(j) for j in range(self.F)]
                w = np.prod([V[a][k] for a, k in enumerate(ks)], axis=0) if dirs else 1.0
                out[eq] = out[eq] + c * self._deriv(U, al, beta) * w
        return np.concatenate(out)

    def R(self, u):
        return self._jet(u, [])

    def F_(self, u):
        return self.Delta @ u + self.R(u)

    def dR(self, u):
        """the reaction Jacobian as an F x F block of diagonal matrices"""
        U = self.fields_of(u)
        blocks = [[sp.csr_matrix((self.n, self.n)) for _ in range(self.F)] for _ in range(self.F)]
        for eq, c, al in self.terms:
            for k in range(self.F):
                beta = [1 if j == k else 0 for j in range(self.F)]
                blocks[eq][k] = blocks[eq][k] + sp.diags(c * self._deriv(U, al, beta))
        return sp.bmat(blocks).tocsr()

    def J(self, u):
        return (self.Delta + self.dR(u)).tocsr()

    def dF(self, u, v):
        return self.J(u) @ v

    def JT(self, u, w):
        return self.J(u).T @ w

    def d2F(self, u, a, b):
        return self._jet(u, [a, b])

    def d3F(self, u, a, b, c):
        return self._jet(u, [a, b, c])


# ---- models of the reference examples -------------------------------------------------------------------------------------
def pd1d_model():
    """examples/pd-1d.jl: f = η (u + a v - C u v - u v^2), g = η (H u + b v + C u v + u v^2), Δ = blockdiag(D Δ, Δ), Neumann;
    params (η, a, b, H, D, C)"""
    terms = [(0, 1.0, {0: 1}, [1, 0]), (0, 1.0, {0: 1, 1: 1}, [0, 1]), (0, -1.0, {0: 1, 5: 1}, [1, 1]), (0, -1.0, {0: 1}, [1, 2]),
             (1, 1.0, {0: 1, 3: 1}, [1, 0]), (1, 1.0, {0: 1, 2: 1}, [0, 1]), (1, 1.0, {0: 1, 5: 1}, [1, 1]), (1, 1.0, {0: 1}, [1, 2])]
    return dict(fields=2, bc="neumann", diffusion=[(1.0, {4: 1}), 1.0], terms=terms, nparams=6, ndims=1)


PD1D_PARAMS = (1.0, -1.0, -1.5, 3.0, 0.08, -0.6)   # η, a, b, H, D, C of examples/pd-1d.jl:54-55


def cgl_model():
    """the reaction of examples/cGL2d.jl:262-279 expanded into monomials, params (r, μ, ν, c3, c5), Dirichlet, D = 1:
    NL(A) = (r + iν) A - (c3 + iμ) |A|^2 A - c5 |A|^4 A with A = u1 + i u2"""
    r, mu, nu, c3, c5 = ({k: 1} for k in range(5))
    t = [(0, 1.0, r, [1, 0]), (0, -1.0, nu, [0, 1]), (0, -1.0, c3, [3, 0]), (0, -1.0, c3, [1, 2]), (0, 1.0, mu, [2, 1]),
         (0, 1.0, mu, [0, 3]), (0, -1.0, c5, [5, 0]), (0, -2.0, c5, [3, 2]), (0, -1.0, c5, [1, 4]),
         (1, 1.0, r, [0, 1]), (1, 1.0, nu, [1, 0]), (1, -1.0, c3, [2, 1]), (1, -1.0, c3, [0, 3]), (1, -1.0, mu, [3, 0]),
         (1, -1.0, mu, [1, 2]), (1, -1.0, c5, [4, 1]), (1, -2.0, c5, [2, 3]), (1, -1.0, c5, [0, 5])]
    return dict(fields=2, bc="dirichlet", diffusion=[1.0, 1.0], terms=t, nparams=5, ndims=2)


def gray_scott_model():
    """Gray-Scott: u_t = Du Δu - u v^2 + f (1 - u), v_t = Dv Δv + u v^2 - (f + k) v; params (Du, Dv, f, k), Neumann"""
    t = [(0, -1.0, {}, [1, 2]), (0, 1.0, {2: 1}, []), (0, -1.0, {2: 1}, [1, 0]),
         (1, 1.0, {}, [1, 2]), (1, -1.0, {2: 1}, [0, 1]), (1, -1.0, {3: 1}, [0, 1])]
    return dict(fields=2, bc="neumann", diffusion=[(1.0, {0: 1}), (1.0, {1: 1})], terms=t, nparams=4, ndims=2)
