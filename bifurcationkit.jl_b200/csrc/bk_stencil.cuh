// bk_stencil.cuh -- device-side tile evaluators of the Swift-Hohenberg stencils (K1/K2) for the
// stand-alone apply kernel k_sh_apply (bk_problems.cu): every SH3d residual / JVP, and SH2d where the
// TMA-staged tile of bk_krylov_tma.cuh does not apply (odd nx or an input not 16-byte aligned).
//
// Swift-Hohenberg (examples/SH2d-fronts.jl:13-34,124-127; examples/SH3d.jl:16-53):
//   L1 = (I + Lap)^2 with the Neumann-closure Laplacian (corner diagonal -1/h^2) == two passes of
//   the 5-/7-point stencil with clamp-to-edge ghost cells (identity checked in tests/test_oracle_palc.py).
//   JVP:      out = a0 v + a1 ( -L1 v + (l + 2 nu u - 3 u^2) v )
//   residual: out = -L1 u + l u + nu u^2 - u^3
// One CTA evaluates a TX x TY x TZ tile: the input tile with a 2-cell halo is staged in shared
// memory (clamped loads), t = v + Lap v is formed on the tile with a 1-cell halo in shared memory,
// and every thread finishes EPT output points in registers.
#pragma once
#include "bk_common.cuh"

#define BK_EPT 8
#define BK_THREADS 256
#define BK_TILE (BK_EPT * BK_THREADS)  // 2048 points per CTA

template <int DIM>
struct ShTile;
template <>
struct ShTile<2> {
  static constexpr int TX = 64, TY = 32, TZ = 1, HZ = 0;
};
template <>
struct ShTile<3> {
  static constexpr int TX = 32, TY = 8, TZ = 8, HZ = 2;
};

template <int DIM>
struct ShSmem {
  using T = ShTile<DIM>;
  static constexpr int VX = T::TX + 4, VY = T::TY + 4, VZ = T::TZ + 2 * T::HZ;
  static constexpr int QX = T::TX + 2, QY = T::TY + 2, QZ = T::TZ + (DIM == 3 ? 2 : 0);
  static constexpr int V_ELEMS = VX * VY * VZ;
  static constexpr int Q_ELEMS = QX * QY * QZ;
  static constexpr size_t BYTES = sizeof(double) * (size_t)(V_ELEMS + Q_ELEMS);
};

__device__ __forceinline__ int bk_clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

// Decompose blockIdx.x into the tile origin.
template <int DIM>
__device__ __forceinline__ void sh_tile_origin(const OpDesc& op, int& x0, int& y0, int& z0) {
  using T = ShTile<DIM>;
  int tiles_x = (op.nx + T::TX - 1) / T::TX;
  int tiles_y = (op.ny + T::TY - 1) / T::TY;
  int b = blockIdx.x;
  int bx = b % tiles_x;
  int by = (b / tiles_x) % tiles_y;
  int bz = b / (tiles_x * tiles_y);
  x0 = bx * T::TX;
  y0 = by * T::TY;
  z0 = bz * T::TZ;
}
template <int DIM>
static inline int sh_num_tiles(int nx, int ny, int nz) {
  using T = ShTile<DIM>;
  return ((nx + T::TX - 1) / T::TX) * ((ny + T::TY - 1) / T::TY) * ((nz + T::TZ - 1) / T::TZ);
}

// MODE 0: JVP (a0 v + a1 J(u) v), MODE 1: residual F(v).
// Outputs, for the EPT points owned by this thread: val[e] and the global offset off[e] (-1 when the
// point lies outside the grid, val = 0).  smem must hold ShSmem<DIM>::BYTES.
template <int DIM, int MODE>
__device__ __forceinline__ void sh_tile_eval(const OpDesc& op, const double* __restrict__ in, double in_scale,
                                             double* smem, double (&val)[BK_EPT], long long (&off)[BK_EPT]) {
  using T = ShTile<DIM>;
  using S = ShSmem<DIM>;
  double* vs = smem;
  double* qs = smem + S::V_ELEMS;
  int x0, y0, z0;
  sh_tile_origin<DIM>(op, x0, y0, z0);
  const int nx = op.nx, ny = op.ny, nz = (DIM == 3 ? op.nz : 1);
  const long long sy = nx, sz = (long long)nx * ny;
  // 1. stage the input tile with a 2-cell halo, clamp-to-edge
  for (int q = threadIdx.x; q < S::V_ELEMS; q += BK_THREADS) {
    int i = q % S::VX, j = (q / S::VX) % S::VY, k = q / (S::VX * S::VY);
    int gx = bk_clampi(x0 - 2 + i, 0, nx - 1);
    int gy = bk_clampi(y0 - 2 + j, 0, ny - 1);
    int gz = (DIM == 3) ? bk_clampi(z0 - 2 + k, 0, nz - 1) : 0;
    vs[q] = in_scale * __ldg(in + gx + gy * sy + gz * sz);
  }
  __syncthreads();
  // 2. t = v + Lap v on the tile with a 1-cell halo; out-of-grid positions replicate the clamped in-grid value
  for (int q = threadIdx.x; q < S::Q_ELEMS; q += BK_THREADS) {
    int i = q % S::QX, j = (q / S::QX) % S::QY, k = q / (S::QX * S::QY);
    int ci = bk_clampi(x0 - 1 + i, 0, nx - 1) - (x0 - 2);
    int cj = bk_clampi(y0 - 1 + j, 0, ny - 1) - (y0 - 2);
    int ck = (DIM == 3) ? bk_clampi(z0 - 1 + k, 0, nz - 1) - (z0 - 2) : 0;
    const double* p = vs + ci + cj * S::VX + ck * (S::VX * S::VY);
    double c0 = p[0];
    double t = c0 + op.cx * (p[-1] - 2.0 * c0 + p[1]) + op.cy * (p[-S::VX] - 2.0 * c0 + p[S::VX]);
    if (DIM == 3) t += op.cz * (p[-S::VX * S::VY] - 2.0 * c0 + p[S::VX * S::VY]);
    qs[q] = t;
  }
  __syncthreads();
  // 3. finish the owned points
  const double l = op.par[0], nu = op.par[1];
#pragma unroll
  for (int e = 0; e < BK_EPT; ++e) {
    int q = threadIdx.x + e * BK_THREADS;
    int lx = q % T::TX, ly = (q / T::TX) % T::TY, lz = q / (T::TX * T::TY);
    int gx = x0 + lx, gy = y0 + ly, gz = z0 + lz;
    bool ok = gx < nx && gy < ny && gz < nz;
    if (ok) {
      const double* p = qs + (lx + 1) + (ly + 1) * S::QX + (DIM == 3 ? (lz + 1) * (S::QX * S::QY) : 0);
      double c0 = p[0];
      double l1v = c0 + op.cx * (p[-1] - 2.0 * c0 + p[1]) + op.cy * (p[-S::QX] - 2.0 * c0 + p[S::QX]);
      if (DIM == 3) l1v += op.cz * (p[-S::QX * S::QY] - 2.0 * c0 + p[S::QX * S::QY]);
      double v = vs[(lx + 2) + (ly + 2) * S::VX + (DIM == 3 ? (lz + 2) * (S::VX * S::VY) : 0)];
      long long g = gx + gy * sy + gz * sz;
      if (MODE == 0) {
        double uu = __ldg(op.u + g);
        double coef = l + uu * (2.0 * nu - 3.0 * uu);
        val[e] = op.a0 * v + op.a1 * (coef * v - l1v);
      } else {
        val[e] = v * (l + v * (nu - v)) - l1v;
      }
      off[e] = g;
    } else {
      val[e] = 0.0;
      off[e] = -1;
    }
  }
}
