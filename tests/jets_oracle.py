"""NumPy restatement of the second and third differentials of F in u (prob.VF.d2F / d3F, src/Problems.jl:107-110,165-183) for
the problem kinds of libbk200, the checker of bk_d2f / bk_d3f.  Test infrastructure only; the product never imports it.  The
linear parts of F (Laplacians, L1) drop out, so every jet is pointwise:
  Swift-Hohenberg (2-D, 3-D, periodic 2-D): F = -L1 u + l u + nu u^2 - u^3      d2F = (2 nu - 6 u) a b,  d3F = -6 a b c
  chan (examples/chan.jl:5-19, b = beta as oracle.problems.chan_F):             interior rows alpha Nl''(u) a b, alpha Nl'''(u) a b c
  cGL2d (examples/cGL2d.jl:262-279): NL(A) = (r + i nu) A - (c3 + i mu) |A|^2 A - c5 |A|^4 A, A = u1 + i u2, real-multilinear."""
import numpy as np


def sh_d2F(u, a, b, nu):
    return (2.0 * nu - 6.0 * u) * a * b


def sh_d3F(u, a, b, c):
    return -6.0 * a * b * c


def chan_d2Nl(x, b):
    """second derivative of chan_Nl(x, a = 1/2, b) = 1 + (x + x^2 / 2) / (1 + b x^2)"""
    h = 1.0 + b * x**2
    return (1.0 - 6.0 * b * x - 3.0 * b * x**2 + 2.0 * b**2 * x**3) / h**3


def chan_d3Nl(x, b):
    h = 1.0 + b * x**2
    return (-6.0 * b - 12.0 * b * x + 36.0 * b**2 * x**2 + 12.0 * b**2 * x**3 - 6.0 * b**3 * x**4) / h**4


def chan_d2F(u, a, b, alpha, beta):
    out = alpha * chan_d2Nl(u, beta) * a * b
    out[0] = out[-1] = 0.0
    return out


def chan_d3F(u, a, b, c, alpha, beta):
    out = alpha * chan_d3Nl(u, beta) * a * b * c
    out[0] = out[-1] = 0.0
    return out


def _cplx(v):
    n = len(v) // 2
    return v[:n] + 1j * v[n:]


def _split(z):
    return np.concatenate([z.real, z.imag])


def _s(x, y):
    """s_xy = D^2 |A|^2 [x, y] = 2 Re(x conj y)"""
    return 2.0 * np.real(x * np.conj(y))


def cgl_d2F(u, a, b, mu, c3, c5):
    A, a, b = _cplx(u), _cplx(a), _cplx(b)
    s, sa, sb, sab = np.abs(A) ** 2, _s(A, a), _s(A, b), _s(a, b)
    t3 = sab * A + sa * b + sb * a                                          # D^2(|A|^2 A)[a, b]
    t5 = 2 * (sa * sb + s * sab) * A + 2 * s * (sa * b + sb * a)             # D^2(|A|^4 A)[a, b]
    return _split(-(c3 + 1j * mu) * t3 - c5 * t5)


def cgl_d3F(u, a, b, c, mu, c3, c5):
    A, a, b, c = _cplx(u), _cplx(a), _cplx(b), _cplx(c)
    s, sa, sb, sc = np.abs(A) ** 2, _s(A, a), _s(A, b), _s(A, c)
    sab, sac, sbc = _s(a, b), _s(a, c), _s(b, c)
    t3 = sab * c + sac * b + sbc * a
    t5 = (2 * (sab * sc + sac * sb + sbc * sa) * A + 2 * (sa * sb + s * sab) * c + 2 * (sa * sc + s * sac) * b
          + 2 * (sb * sc + s * sbc) * a)
    return _split(-(c3 + 1j * mu) * t3 - c5 * t5)
