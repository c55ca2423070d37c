"""Periodic spectral Swift-Hohenberg (BK_SH2D_PERIODIC, BK_PC_SH_FFT) without a GPU: the NumPy restatement of
examples/SH2d-fronts-cuda.jl against the example's own formulas, the thread-by-thread model of the new transform modes
(tools/fftcheck/model.py: r2c pair split, packed half-spectrum, c2r, the fused y pass with its kx = 0 / Nyquist column pair)
against numpy.fft, and the bindings."""
import os
import sys

import numpy as np
import pytest

import __graft_entry__ as g
from tests import sh_periodic_oracle as po

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools", "fftcheck"))
import model  # noqa: E402


def test_constant_state_residual():
    """a constant u only sees the k = 0 symbol (1 - 0)^2 = 1: F = -u + l u + nu u^2 - u^3 = (l - 1) u + nu u^2 - u^3"""
    sh = po.PeriodicSH((64, 32), po.example_lengths(64, 32), l=-0.15, nu=1.3)
    for c in (0.3, -0.7):
        u = np.full(sh.N, c)
        assert np.allclose(sh.F(u), (sh.l - 1) * c + sh.nu * c**2 - c**3, atol=1e-13)


def test_fourier_mode_is_an_eigenvector_with_the_stated_symbol():
    """cos(pi (kx x / lx + ky y / ly)) is an eigenvector of L1 with eigenvalue (1 - (pi kx / lx)^2 - (pi ky / ly)^2)^2, and of
    the example's L with that value + 1"""
    Nx, Ny = 64, 32
    lx, ly = po.example_lengths(Nx, Ny)
    sh = po.PeriodicSH((Nx, Ny), (lx, ly))
    X = -lx + 2 * lx / Nx * np.arange(Nx)
    Y = -ly + 2 * ly / Ny * np.arange(Ny)
    for kx, ky in ((0, 0), (1, 0), (3, 2), (Nx // 2, 1), (5, Ny // 2)):
        v = np.cos(np.pi * (kx * X[None, :] / lx + ky * Y[:, None] / ly)).reshape(-1)
        lam = (1 - (np.pi * kx / lx) ** 2 - (np.pi * ky / ly) ** 2) ** 2
        assert np.allclose(sh.L1(v), lam * v, atol=1e-9 * max(1.0, lam))
        assert np.allclose(sh.precond(1.0)(v), v / (lam + 1), atol=1e-12)


def test_dF_is_the_derivative_of_F():
    Nx, Ny = 64, 64
    L = po.example_lengths(Nx, Ny)
    sh = po.PeriodicSH((Nx, Ny), L)
    rng = np.random.default_rng(1)
    u = po.sol0(Nx, Ny, *L) + 0.05 * rng.standard_normal(sh.N)
    du = rng.standard_normal(sh.N)
    eps = 1e-6
    fd = (sh.F(u + eps * du) - sh.F(u - eps * du)) / (2 * eps)
    assert np.linalg.norm(fd - sh.dF(u, du)) < 1e-7 * np.linalg.norm(sh.dF(u, du))
    J = po.PeriodicSH((16, 8), (2.0, 1.5)).jac_dense(np.linspace(-1, 1, 128))
    assert np.allclose(J, J.T, atol=1e-12)   # self-adjoint: the eigensolver takes its symmetric path


@pytest.mark.parametrize("n", [64, 128, 256, 512, 1024, 2048])
@pytest.mark.parametrize("E", [4, 8])
def test_periodic_transform_model_matches_numpy(n, E):
    """r2c (packed half-spectrum), c2r and the fused y pass of both column-pair kinds, thread by thread, to 1e-12 n"""
    rng = np.random.default_rng(n + E)
    pl = model.Plan(n, E)
    x1, x2 = rng.standard_normal(n), rng.standard_normal(n)
    P1, P2 = model.rfft_pair(pl, x1, x2)
    for x, P in ((x1, P1), (x2, P2)):
        R = np.fft.rfft(x)
        packed = np.empty(n)
        packed[0], packed[1] = R[0].real, R[n // 2].real
        packed[2::2], packed[3::2] = R[1:n // 2].real, R[1:n // 2].imag
        assert np.abs(P - packed).max() < 1e-12 * n
    y1, y2 = model.irfft_pair(pl, P1, P2)
    assert max(np.abs(y1 / n - x1).max(), np.abs(y2 / n - x2).max()) < 1e-12 * n
    # y pass: a complex column line (kx >= 1), and the kx = 0 / Nyquist pair of real lines with two even symbols
    ky = np.minimum(np.arange(n), n - np.arange(n))
    s0, sn = 1.0 / (1.0 + 0.01 * ky**2), 2.0 + np.cos(np.pi * ky / n)
    c0, c1 = rng.standard_normal(n), rng.standard_normal(n)
    a, b = model.periodic_y_pair(pl, c0, c1, s0 / n)
    z = np.fft.ifft(np.fft.fft(c0 + 1j * c1) * s0)
    assert max(np.abs(a - z.real).max(), np.abs(b - z.imag).max()) < 1e-12 * n
    a, b = model.periodic_y_pair(pl, c0, c1, s0 / n, sn / n)
    r0, rn = np.fft.ifft(np.fft.fft(c0) * s0).real, np.fft.ifft(np.fft.fft(c1) * sn).real
    assert max(np.abs(a - r0).max(), np.abs(b - rn).max()) < 1e-12 * n


@pytest.mark.parametrize("dims,E", [((64, 16), 4), ((16, 64), 8), ((32, 32), 8)])
def test_periodic_pipeline_model_matches_rfft2(dims, E):
    """the three passes together: irfft2(rfft2(u) * symbol) for the -L1 and (L1 + 1)^-1 symbols"""
    Nx, Ny = dims
    L = (3.0, 2.0)
    sh = po.PeriodicSH(dims, L)
    u = np.random.default_rng(Nx * Ny).standard_normal((Ny, Nx))
    half = sh.symbol[:, :Nx // 2 + 1]
    for sym in (-half, 1.0 / (half + 1.0)):
        ref = np.fft.irfft2(np.fft.rfft2(u) * sym, s=(Ny, Nx))
        assert np.abs(model.periodic_apply(u, sym, E) - ref).max() < 1e-12 * max(Nx, Ny) * max(1.0, np.abs(ref).max())


def test_bindings_expose_the_periodic_kind_and_preconditioner():
    bk = g.load_package()
    assert bk.BK_SH2D_PERIODIC == 6 and bk.lib.BK_SH2D_PERIODIC == 6
    assert bk.BK_PC_SH_FFT == 5 and bk.lib.BK_PC_SH_FFT == 5
    hdr = open(os.path.join(ROOT, "include", "bk200.h")).read()
    assert "BK_SH2D_PERIODIC = 6" in hdr and "BK_PC_SH_FFT = 5" in hdr
    jl = open(os.path.join(ROOT, "julia", "BK200.jl")).read()
    assert ":SH2D_PERIODIC => 6" in jl and ":SH_FFT => 5" in jl


@pytest.mark.parametrize("dims", [(96, 64), (64, 32), (4096, 64), (64, 100)])
def test_unsupported_sizes_are_rejected_before_any_device_work(dims):
    """BK_ERR_ARG with a message naming the limit, checked before the context touches a GPU"""
    bk = g.load_package()
    if not os.path.exists(bk.lib.LIB_PATH):
        bk.build()
    with pytest.raises(bk.BK200Error, match="powers of two from 64 to 2048"):
        bk.Context(bk.BK_SH2D_PERIODIC, dims, (10.0, 10.0), krylov_m=4)
