"""NumPy restatement of the reference's GPU Swift-Hohenberg example (examples/SH2d-fronts-cuda.jl) for the BK_SH2D_PERIODIC
tests: the spectral operator, F, dF, the FFT preconditioner and the initial guess.  Test infrastructure only; the product never
imports it.  Layout x fastest: flat index i + j Nx, arrays (Ny, Nx)."""
import numpy as np


def wavenumbers(n, L):
    """examples/SH2d-fronts-cuda.jl:48-49: signed frequencies 0..n/2, -n/2+1..-1, times pi / L"""
    k = np.concatenate([np.arange(0, n // 2 + 1), np.arange(n // 2 + 1, n) - n]).astype(np.float64)
    return np.pi * k / L


def example_lengths(Nx, Ny):
    """the example's domain (lx = 16 pi, ly = 8 pi / sqrt(3) at 512 x 512, :66-69) scaled by n / 512, which keeps sol0 periodic"""
    return 16 * np.pi * Nx / 512, 8 * np.pi / np.sqrt(3) * Ny / 512


class PeriodicSH:
    """The example's L has symbol (1 - kx^2 - ky^2)^2 + 1 = L1 + 1 (:50), so its F (:104-108),
    F = -L u + (l + 1) u + nu u^2 - u^3, is F = -L1 u + l u + nu u^2 - u^3."""

    def __init__(self, dims, lengths, l=-0.15, nu=1.3):
        self.dims, self.lengths = tuple(dims), tuple(lengths)
        Nx, Ny = self.dims
        kx, ky = wavenumbers(Nx, lengths[0]), wavenumbers(Ny, lengths[1])
        self.symbol = (1.0 - kx[None, :] ** 2 - ky[:, None] ** 2) ** 2   # symbol of L1, (Ny, Nx)
        self.N = Nx * Ny
        self.l, self.nu = l, nu

    def apply_symbol(self, u, sym):
        Nx, Ny = self.dims
        return np.real(np.fft.ifft2(np.fft.fft2(np.reshape(u, (Ny, Nx))) * sym)).reshape(-1)

    def L1(self, u):
        return self.apply_symbol(u, self.symbol)

    def F(self, u, l=None):
        l = self.l if l is None else l
        return -self.L1(u) + (l * u + self.nu * u**2 - u**3)

    def dF(self, u, du, l=None):
        l = self.l if l is None else l
        return -self.L1(du) + (l + 2.0 * self.nu * u - 3.0 * u**2) * du

    def precond(self, shift=1.0):
        """(L1 + shift I)^-1: the example's `L \\ r` is shift = 1 (:64)"""
        sym = 1.0 / (self.symbol + shift)
        return lambda r: self.apply_symbol(r, sym)

    def jac_dense(self, u, l=None):
        """J = -L1 + diag(l + 2 nu u - 3 u^2) as a dense matrix (small grids)"""
        l = self.l if l is None else l
        Nx, Ny = self.dims
        cols = np.real(np.fft.ifft2(np.fft.fft2(np.eye(self.N).reshape(self.N, Ny, Nx)) * self.symbol)).reshape(self.N, self.N)
        return -cols.T + np.diag(l + 2.0 * self.nu * u - 3.0 * u**2)


def sol0(Nx, Ny, lx, ly):
    """examples/SH2d-fronts-cuda.jl:71-74"""
    X = -lx + 2 * lx / Nx * np.arange(Nx)
    Y = -ly + 2 * ly / Ny * np.arange(Ny)
    return (0.5 * (np.cos(X)[None, :] + np.cos(X / 2)[None, :] * np.cos(np.sqrt(3.0) * Y / 2)[:, None])).reshape(-1)


def front_guess(u_hexa, Nx, Ny, lx):
    """examples/SH2d-fronts-cuda.jl:135: 0.4 u_hexa exp(-x^2 / 25)"""
    X = -lx + 2 * lx / Nx * np.arange(Nx)
    return 0.4 * u_hexa * np.tile(np.exp(-X**2 / 25.0), Ny)
