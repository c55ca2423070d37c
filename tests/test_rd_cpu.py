"""BK_RD without a GPU: the NumPy restatement (tests/rd_oracle.py) against finite differences and the existing cGL2d oracles, the
pd-1d F of examples/pd-1d.jl, the model checks that run before any device work, and the sm_90a code of the new kernels."""
import os

import numpy as np
import pytest

import __graft_entry__ as g
from oracle import problems
from tests import jets_oracle as JO
from tests import rd_oracle as RO
from tests import sass_reader as SR


def _rel(a, b):
    return np.linalg.norm(a - b) / np.linalg.norm(b)


MODEL = dict(fields=3, bc="neumann", diffusion=[(0.5, {0: 1}), 1.0, (2.0, {1: -1})], nparams=3, ndims=2,
             terms=[(0, 1.5, {0: 1}, [1, 0, 0]), (0, -1.0, {}, [2, 1, 0]), (1, 0.7, {2: 2}, [0, 1, 2]), (2, -0.3, {1: -2}, [5, 0, 0]),
                    (2, 1.0, {}, [1, 1, 1]), (1, 2.0, {0: 1, 2: 1}, [0, 0, 0]), (0, 0.4, {}, [0, 2, 3])])


@pytest.mark.parametrize("bc", ["neumann", "dirichlet"])
def test_oracle_derivatives_against_finite_differences(bc):
    o = RO.RD(**{**MODEL, "bc": bc}, dims=(9, 7), lengths=(1.5, 1.0), params=(1.1, 0.8, 1.3))
    rng = np.random.default_rng(0)
    u, a, b, c = (0.7 * rng.standard_normal(o.N) for _ in range(4))
    h = 1e-5
    fd = (o.F_(u + h * a) - o.F_(u - h * a)) / (2 * h)
    assert _rel(o.dF(u, a), fd) < 1e-8
    fd2 = (o.dF(u + h * b, a) - o.dF(u - h * b, a)) / (2 * h)
    assert _rel(o.d2F(u, a, b), fd2) < 1e-8
    fd3 = (o.d2F(u + h * c, a, b) - o.d2F(u - h * c, a, b)) / (2 * h)
    assert _rel(o.d3F(u, a, b, c), fd3) < 1e-8
    w = rng.standard_normal(o.N)
    assert abs(np.dot(w, o.dF(u, a)) - np.dot(o.JT(u, w), a)) < 1e-10 * np.linalg.norm(w) * np.linalg.norm(o.dF(u, a))


def test_cgl_written_as_rd_terms_is_the_cgl2d_oracle():
    dims, L, pars = (11, 8), (2.0, 1.0), (0.7, 0.1, 1.0, -1.0, 1.0)
    o = RO.RD(**RO.cgl_model(), dims=dims, lengths=L, params=pars)
    gl = problems.GinzburgLandau2D(*dims, *L, *pars)
    rng = np.random.default_rng(1)
    u, a, b, c = (rng.standard_normal(o.N) for _ in range(4))
    assert _rel(o.F_(u), gl.F(u)) < 1e-13
    assert _rel(o.dF(u, a), gl.dF(u, a)) < 1e-13
    _, mu, _, c3, c5 = pars
    assert _rel(o.d2F(u, a, b), JO.cgl_d2F(u, a, b, mu, c3, c5)) < 1e-13
    assert _rel(o.d3F(u, a, b, c), JO.cgl_d3F(u, a, b, c, mu, c3, c5)) < 1e-13


def test_pd1d_oracle_is_the_example_F():
    """examples/pd-1d.jl:6-7,47-55 with its parameters, N = 100, lx = 3π/2: Fbr = NL + blockdiag(D Δ, Δ) u"""
    N, lx = 100, 3 * np.pi / 2
    eta, a, b, H, D, C = RO.PD1D_PARAMS
    o = RO.RD(**RO.pd1d_model(), dims=(N,), lengths=(lx,), params=RO.PD1D_PARAMS)
    h = 2 * lx / N
    Lap = (np.diag(-2 * np.ones(N)) + np.diag(np.ones(N - 1), 1) + np.diag(np.ones(N - 1), -1)) / h**2
    Lap[0, 0] = Lap[-1, -1] = -1 / h**2
    X = np.linspace(-lx, lx, N)
    u = np.concatenate([np.cos(2 * X), np.cos(2 * X) + 0.1 * np.sin(X)])
    uu, vv = u[:N], u[N:]
    ref = np.concatenate([eta * (uu + a * vv - C * uu * vv - uu * vv**2) + D * Lap @ uu,
                          eta * (H * uu + b * vv + C * uu * vv + uu * vv**2) + Lap @ vv])
    assert _rel(o.F_(u), ref) < 1e-14


@pytest.fixture(scope="module")
def bk():
    bk = g.load_package()
    if not os.path.exists(bk.lib.LIB_PATH):
        bk.build()
    return bk


def _model(**kw):
    m = dict(fields=2, bc="neumann", diffusion=[1.0, 1.0], terms=[(0, 1.0, {0: 1}, [1, 1])], nparams=2, ndims=1)
    m.update(kw)
    return m


BAD = [
    (dict(fields=0, diffusion=[]), "fields must be 1 .. 4"),
    (dict(fields=5, diffusion=[1.0] * 5), "fields must be 1 .. 4"),
    (dict(ndims=3), "ndims must be 1 or 2"),
    (dict(bc=2), "bc must be"),
    (dict(nparams=9), "nparams must be 0 .. 8"),
    (dict(terms=[(0, 1.0, {}, [1, 0])] * 65), "nterms must be 0 .. 64"),
    (dict(terms=[(2, 1.0, {}, [1, 0])]), "equation index"),
    (dict(terms=[(-1, 1.0, {}, [1, 0])]), "equation index"),
    (dict(terms=[(0, 1.0, {0: 5}, [1, 0])]), "parameter exponent is outside"),
    (dict(terms=[(0, 1.0, {1: -5}, [1, 0])]), "parameter exponent is outside"),
    (dict(terms=[(0, 1.0, {3: 1}, [1, 0])]), "parameter index >= nparams"),
    (dict(terms=[(0, 1.0, {}, [6, 0])]), "field exponent is outside"),
    (dict(terms=[(0, 1.0, {}, [-1, 0])]), "field exponent is outside"),
    (dict(terms=[(0, 1.0, {}, [3, 3])]), "degree"),
    (dict(terms=[(0, 1.0, {}, [1, 0, 1])]), "field index >= fields"),
    (dict(diffusion=[(1.0, {0: 7}), 1.0]), "diffusion parameter exponent"),
    (dict(diffusion=[(1.0, {5: 1}), 1.0]), "diffusion coefficient reads a parameter index"),
    (dict(terms=[(0, float("nan"), {}, [1, 0])]), "scale is not finite"),
]


@pytest.mark.parametrize("kw,msg", BAD)
def test_malformed_models_are_refused_before_any_device_work(bk, kw, msg):
    """BK_ERR_ARG with a message, from checks that run before the context touches a GPU"""
    with pytest.raises(bk.BK200Error, match=msg):
        bk.Context(bk.BK_RD, (16,), (1.0,), krylov_m=4, model=bk.ReactionDiffusion(**_model(**kw)))


def test_dims_beyond_the_model_dimensions_and_unknown_boundary_conditions_are_refused(bk):
    with pytest.raises(bk.BK200Error, match="more grid dimensions than the model's ndims"):
        bk.Context(bk.BK_RD, (151, 100), (1.0, 1.0), krylov_m=4, model=bk.ReactionDiffusion(**_model()))
    with pytest.raises(bk.BK200Error, match="more grid dimensions than the model's ndims"):
        bk.Context(bk.BK_RD, (16, 16, 4), (1.0, 1.0, 1.0), krylov_m=4, model=bk.ReactionDiffusion(**_model(ndims=2)))
    with pytest.raises(bk.BK200Error, match="bc must be"):
        bk.ReactionDiffusion(**_model(bc="periodic"))


def test_plain_ctx_create_refuses_the_rd_kind(bk):
    with pytest.raises(bk.BK200Error, match="bk_rd_ctx_create"):
        bk.Context(bk.BK_RD, (16,), (1.0,), krylov_m=4)


def test_rd_kernels_are_in_the_sm_90a_cubin_without_local_memory():
    res = SR.resources()
    ops = SR.mnemonics()
    names = [k for k in res if any(s in k for s in ("k_rd_apply", "k_rd_jet", "k_rd_symbol_div"))]
    # residual / JVP / J' for 1-4 fields in 1-D and 2-D, d2F / d3F and the moments for 1-4 fields, the preconditioner's symbol
    assert len(names) == 24 + 8 + 4 + 1, sorted(names)
    for k in names:
        assert res[k].local == 0 and res[k].stack == 0, (k, res[k])
        assert "LDL" not in ops[k] and "STL" not in ops[k], k
