// bk_krylov_tma.cuh -- second-generation Arnoldi kernels: the Krylov basis is streamed through a
// shared-memory ring by the TMA engine (cp.async.bulk + mbarrier), issued by a dedicated producer
// warp, while 8 consumer warps do the fp64 FMAs.  One CTA owns a tile of up to 8 rows x 256 columns
// (fused 2-D stencil) or a contiguous segment of up to 8 x 256 values (generic vectors); the tile
// height E is chosen on the host so that the grid fills every SM of the device in whole, balanced waves
// (a grid of 1.15 waves leaves most SMs idle during its last wave).
//
//   pass 1  k2_fused<E>  : w = a0 v + a1 J(u) v on a 256 x E tile (stencil from shared memory, halo 2),
//                          then h_i = <v_i, w>, i < j, with V_i tiles arriving through the ring.
//           k2_dots<E>   : same without the stencil (w read from memory).
//   pass 2  k2_update<E> : v' = w - sum_i g_i V_i, ||v'||^2.
// Reductions: warp shuffle -> per-CTA partial -> deterministic last-block sum (no atomics on data).
#pragma once
#include "bk_common.cuh"
#include "bk_async.cuh"

#define BK2_CONS 256
#define BK2_THREADS 288
#define BK2_EMAX 8
#define BK2_ROW 256

struct Tile2 {
  long long base;  // offset of (row 0, col 0) inside a vector
  int rs;          // row stride (elements)
  int rows;        // valid rows (<= E)
  int len;         // valid columns of rows 0..rows-2
  int last_len;    // valid columns of the last row
};

#define BK2_MAXSTAGES 8
struct Ring {
  unsigned long long full[BK2_MAXSTAGES];
  unsigned long long empty[BK2_MAXSTAGES];
};

__device__ __forceinline__ void ring_init(Ring* rg, int NS) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < NS; ++s) {
      mbar_init(&rg->full[s], 1);
      mbar_init(&rg->empty[s], 8);
    }
    fence_mbar_init();
  }
}

// Streams V_0..V_{j-1} restricted to the tile through the ring.  MODE 0: sred[i*8 + warp] = warp partial of
// <V_i, val>; MODE 1: val -= g_i V_i.  Called by all BK2_THREADS threads after a __syncthreads().
// REV: the basis is traversed from V_{j-1} down to V_0.  Pass 1 (dots) runs forward and pass 2 (update) backward, so each
// pass starts with the vectors the previous pass touched last, which may still be in the L2 (50 MB on an H100: the last few
// 8 MB basis vectors at 1024^2); with both passes forward the LRU order evicts exactly what is needed next.
// keep: the last `keep` vectors of the pass are read with L2 evict_last, all others with evict_first, so that the vectors the
// next pass starts with survive the rest of this pass and the kernels in between (plan2 sizes keep from the L2).
template <int E, int MODE, bool REV = false>
__device__ __forceinline__ void stream_basis(const Tile2& tl, const double* __restrict__ V, long long ld, int j, int keep,
                                             double* ring, int NS, Ring* rg, double (&val)[E], double* sred,
                                             const double* __restrict__ gcoef) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp == 8) {
    if (lane == 0) {
      fence_proxy_async_smem();  // the ring may alias memory written through the generic proxy (stencil scratch)
      const unsigned row_b = (unsigned)(((tl.len + 1) & ~1) * 8);
      const unsigned last_b = (unsigned)(((tl.last_len + 1) & ~1) * 8);
      const bool contiguous = (tl.rs == BK2_ROW) && (tl.len == BK2_ROW);
      const unsigned total = row_b * (unsigned)(tl.rows - 1) + last_b;
      const unsigned long long pol_first = l2_evict_first(), pol_last = l2_evict_last();
      for (int i = 0; i < j; ++i) {
        const int s = i % NS, round = i / NS;
        if (round > 0) mbar_wait(&rg->empty[s], (unsigned)((round - 1) & 1));
        mbar_arrive_expect_tx(&rg->full[s], total);
        const double* src = V + (long long)(REV ? j - 1 - i : i) * ld + tl.base;
        double* dst = ring + (size_t)s * (E * BK2_ROW);
        const unsigned long long pol = i >= j - keep ? pol_last : pol_first;
        if (contiguous) {
          bulk_g2s(dst, src, total, &rg->full[s], pol);
        } else {
          for (int r = 0; r < tl.rows - 1; ++r)
            bulk_g2s(dst + r * BK2_ROW, src + (long long)r * tl.rs, row_b, &rg->full[s], pol);
          bulk_g2s(dst + (tl.rows - 1) * BK2_ROW, src + (long long)(tl.rows - 1) * tl.rs, last_b, &rg->full[s], pol);
        }
      }
    }
  } else {
    const int t = threadIdx.x;
    if (MODE == 0) {
      // two basis vectors per trip: their warp reductions are independent shuffle chains that overlap
      for (int i = 0; i < j; i += 2) {
        const int s0 = i % NS, s1 = (i + 1) % NS;
        const bool two = (i + 1 < j);
        mbar_wait(&rg->full[s0], (unsigned)((i / NS) & 1));
        const double* st0 = ring + (size_t)s0 * (E * BK2_ROW) + t;
        double a0 = 0.0, a1 = 0.0;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int lim = (e == tl.rows - 1) ? tl.last_len : tl.len;
          if (e < tl.rows && t < lim) a0 = fma(st0[e * BK2_ROW], val[e], a0);
        }
        if (two) {
          mbar_wait(&rg->full[s1], (unsigned)(((i + 1) / NS) & 1));
          const double* st1 = ring + (size_t)s1 * (E * BK2_ROW) + t;
#pragma unroll
          for (int e = 0; e < E; ++e) {
            const int lim = (e == tl.rows - 1) ? tl.last_len : tl.len;
            if (e < tl.rows && t < lim) a1 = fma(st1[e * BK2_ROW], val[e], a1);
          }
        }
        consumer_release_fence();
        __syncwarp();
        if (lane == 0) {
          mbar_arrive(&rg->empty[s0]);
          if (two) mbar_arrive(&rg->empty[s1]);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
          a0 += __shfl_xor_sync(0xffffffffu, a0, o);
          a1 += __shfl_xor_sync(0xffffffffu, a1, o);
        }
        if (lane == 0) {
          sred[i * 8 + warp] = a0;
          if (two) sred[(i + 1) * 8 + warp] = a1;
        }
      }
    } else {
      for (int i = 0; i < j; ++i) {
        const int s = i % NS;
        mbar_wait(&rg->full[s], (unsigned)((i / NS) & 1));
        const double* st = ring + (size_t)s * (E * BK2_ROW) + t;
        const double g = __ldg(gcoef + (REV ? j - 1 - i : i));
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int lim = (e == tl.rows - 1) ? tl.last_len : tl.len;
          if (e < tl.rows && t < lim) val[e] = fma(-g, st[e * BK2_ROW], val[e]);
        }
        consumer_release_fence();
        __syncwarp();
        if (lane == 0) mbar_arrive(&rg->empty[s]);
      }
    }
  }
}

// per-CTA partials of the j dot products + deterministic last-block reduction -> hcol[i] = s_i * sum, gcoef[i] = hcol[i] * s_i
// With a border (bord != nullptr): row j of sred/partials carries <b, x_u>; the last CTA first forms
// w_p = bscale * sum + bc * x_p, stores it as w[N], and adds V_i[N] * w_p to every dot product (vectors have N+1 entries).
struct BorderFin {
  double bscale, bc, xp;
  double* w_tail;          // &w[N]
  const double* V_tail;    // &V[0*ld + N]
  long long ld;
};
__device__ __forceinline__ void dots_finish(int j, const double* sred, const double* __restrict__ scales,
                                            double* __restrict__ partials, unsigned int* counter, double* __restrict__ hcol,
                                            double* __restrict__ gcoef, int* s_flag, const BorderFin* bord = nullptr,
                                            double* s_wp = nullptr) {
  const int G = gridDim.x;
  const int jj = bord ? j + 1 : j;
  for (int i = threadIdx.x; i < jj; i += blockDim.x) {
    double t = 0.0;
#pragma unroll
    for (int k = 0; k < 8; ++k) t += sred[i * 8 + k];
    partials[(long long)i * G + blockIdx.x] = t;
  }
  if (bk_last_block(counter, s_flag)) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    double wp = 0.0;
    if (bord) {
      if (warp == 0) {
        double t = 0.0;
        for (int k = lane; k < G; k += 32) t += __ldcg(partials + (long long)j * G + k);
        t = bk_warp_sum(t);
        if (lane == 0) {
          *s_wp = bord->bscale * t + bord->bc * bord->xp;
          *bord->w_tail = *s_wp;
        }
      }
      __syncthreads();
      wp = *s_wp;
    }
    for (int i = warp; i < j; i += nw) {
      double t = 0.0;
      for (int k = lane; k < G; k += 32) t += __ldcg(partials + (long long)i * G + k);
      t = bk_warp_sum(t);
      if (lane == 0) {
        if (bord) t = fma(__ldg(bord->V_tail + (long long)i * bord->ld), wp, t);
        const double s = scales[i];
        const double h = s * t;
        hcol[i] = h;
        gcoef[i] = h * s;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ 2-D SH tile stencil
// Tile = 256 columns x E rows at (x0, y0); thread t < 256 owns column x0 + t.  scratch: vs[(E+4)][260] | qs[(E+2)][258].
template <int E>
struct Sh2Scratch {
  static constexpr int VX = BK2_ROW + 4, VY = E + 4, QX = BK2_ROW + 2, QY = E + 2;
  static constexpr int V_ELEMS = VX * VY, Q_ELEMS = QX * QY;
  static constexpr size_t BYTES = sizeof(double) * (size_t)(V_ELEMS + Q_ELEMS);
};

// BORDERED (MatrixFreeBLSmap, src/LinearBorderSolver.jl:312-325): val += x_p * a + shift * v, and *bsum accumulates this
// thread's share of <b, x_u>.
// The input tile (E + 4 rows, clamped at the grid edge) is staged by the TMA engine: one cp.async.bulk per row for the
// central 256 columns (16-byte aligned: x0 is a multiple of 256 and nx is even), issued by the producer lane and counted
// on `tbar`; the 2 + 2 halo columns of every row are clamped scalar loads by 4 (E + 4) threads.  The stencil is linear in
// v, so the deferred normalisation in_scale is applied to the results instead of the staged tile.
// Producer lane: one bulk copy per tile row (central 256 columns), counted on `tbar`.  Issued FIRST, before any L2 prefetch:
// the tile is on the critical path of the kernel.
template <int E>
__device__ __forceinline__ void sh2_tile_issue(const OpDesc& op, const double* __restrict__ in, int x0, int y0, double* scratch,
                                               unsigned long long* tbar) {
  using S = Sh2Scratch<E>;
  const int nx = op.nx, ny = op.ny;
  const int len = min(BK2_ROW, nx - x0);
  mbar_arrive_expect_tx(tbar, (unsigned)(len * 8) * (unsigned)S::VY);
#pragma unroll 1
  for (int jj = 0; jj < S::VY; ++jj) {
    int gy = y0 - 2 + jj;
    gy = gy < 0 ? 0 : (gy > ny - 1 ? ny - 1 : gy);
    bulk_g2s(scratch + jj * S::VX + 2, in + x0 + (long long)gy * nx, (unsigned)(len * 8), tbar);
  }
}

// RESID: the residual F(v) = -L1 v + l v + nu v^2 - v^3 (examples/SH2d-fronts.jl:31-34) instead of the JVP.
template <int E, bool BORDERED, bool RESID = false>
__device__ __forceinline__ void sh2_tile_eval(const OpDesc& op, const double* __restrict__ in, double in_scale, int x0, int y0,
                                              double* scratch, unsigned long long* tbar, double (&val)[E], double xp,
                                              double* bsum) {
  using S = Sh2Scratch<E>;
  double* vs = scratch;
  double* qs = scratch + S::V_ELEMS;
  const int nx = op.nx, ny = op.ny;
  const int len = min(BK2_ROW, nx - x0);
  const int t = threadIdx.x;
  const double l = op.par[0], nu = op.par[1];
  const int gx = x0 + t;
  const bool colok = t < BK2_ROW && gx < nx;
  const int rows = min(E, ny - y0);
  // Epilogue in sub-passes so that each issues E independent global loads before the first use (the first version mixed the
  // loads of u, a, b with the arithmetic row by row and stalled on each of them).  The u rows do not depend on the tile, so
  // their loads are issued before the tile wait and arrive while the tile and the q pass are in progress.
  double g[E];
  if (!RESID) {
#pragma unroll
    for (int e = 0; e < E; ++e) g[e] = (colok && e < rows) ? __ldg(op.u + gx + (long long)(y0 + e) * nx) : 0.0;
  }
  if (threadIdx.x < 4 * S::VY) {
    const int jj = threadIdx.x >> 2, h = threadIdx.x & 3;
    const int i = h < 2 ? h : len + h;  // 0, 1, len + 2, len + 3
    int gx = x0 - 2 + i, gy = y0 - 2 + jj;
    gx = gx < 0 ? 0 : (gx > nx - 1 ? nx - 1 : gx);
    gy = gy < 0 ? 0 : (gy > ny - 1 ? ny - 1 : gy);
    vs[jj * S::VX + i] = __ldg(in + gx + (long long)gy * nx);
  }
  mbar_wait(tbar, 0);
  __syncthreads();
  for (int q = threadIdx.x; q < S::Q_ELEMS; q += blockDim.x) {
    int i = q % S::QX, jj = q / S::QX;
    int cx = x0 - 1 + i, cy = y0 - 1 + jj;
    cx = (cx < 0 ? 0 : (cx > nx - 1 ? nx - 1 : cx)) - (x0 - 2);
    cy = (cy < 0 ? 0 : (cy > ny - 1 ? ny - 1 : cy)) - (y0 - 2);
    const double* p = vs + cx + cy * S::VX;
    const double c0 = p[0];
    qs[q] = c0 + op.cx * (p[-1] - 2.0 * c0 + p[1]) + op.cy * (p[-S::VX] - 2.0 * c0 + p[S::VX]);
  }
  __syncthreads();
#pragma unroll
  for (int e = 0; e < E; ++e) {
    double r = 0.0;
    if (colok && e < rows) {
      const double* p = qs + (t + 1) + (e + 1) * S::QX;
      const double c0 = p[0];
      const double l1v = in_scale * (c0 + op.cx * (p[-1] - 2.0 * c0 + p[1]) + op.cy * (p[-S::QX] - 2.0 * c0 + p[S::QX]));
      const double v = in_scale * vs[(t + 2) + (e + 2) * S::VX];
      if (RESID) {
        r = v * (l + v * (nu - v)) - l1v;
      } else {
        const double coef = l + g[e] * (2.0 * nu - 3.0 * g[e]);
        r = op.a0 * v + op.a1 * (coef * v - l1v);
        if (BORDERED) r += op.bshift * v;
      }
    }
    val[e] = r;
  }
  if (BORDERED) {
#pragma unroll
    for (int e = 0; e < E; ++e) g[e] = (colok && e < rows) ? __ldg(op.ba + gx + (long long)(y0 + e) * nx) : 0.0;
#pragma unroll
    for (int e = 0; e < E; ++e) val[e] = fma(xp, g[e], val[e]);
#pragma unroll
    for (int e = 0; e < E; ++e) g[e] = (colok && e < rows) ? __ldg(op.bb + gx + (long long)(y0 + e) * nx) : 0.0;
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (colok && e < rows) *bsum = fma(g[e], in_scale * vs[(t + 2) + (e + 2) * S::VX], *bsum);
  }
}

template <int E, bool BORDERED>
static __global__ void __launch_bounds__(BK2_THREADS, 4) k2_fused(OpDesc op, const double* __restrict__ in,
                                                                  const double* __restrict__ in_scale_ptr,
                                                                  double* __restrict__ w, const double* __restrict__ V,
                                                                  long long ld, int j, const double* __restrict__ scales,
                                                                  double* __restrict__ partials, unsigned int* counter,
                                                                  double* __restrict__ hcol, double* __restrict__ gcoef,
                                                                  int keep, int NS, int sred_off) {
  extern __shared__ __align__(128) double smem2[];
  __shared__ Ring rg;
  __shared__ __align__(8) unsigned long long tbar;
  __shared__ int s_flag;
  double* ring = smem2;
  double* sred = smem2 + sred_off;
  // barrier set-up and tile arithmetic overlap the tail of the previous kernel (PDL): nothing it wrote is read before the wait
  if (threadIdx.x == 0) mbar_init(&tbar, 1);
  ring_init(&rg, NS);
  const int tiles_x = (op.nx + BK2_ROW - 1) / BK2_ROW;
  const int x0 = (blockIdx.x % tiles_x) * BK2_ROW, y0 = (blockIdx.x / tiles_x) * E;
  double val[E];
  Tile2 tl;
  tl.base = x0 + (long long)y0 * op.nx;
  tl.rs = op.nx;
  tl.rows = min(E, op.ny - y0);
  tl.len = min(BK2_ROW, op.nx - x0);
  tl.last_len = tl.len;
  __syncthreads();  // barriers initialised before the producer lane arms them
  bk_pdl_sync();
  const double s = in_scale_ptr ? __ldg(in_scale_ptr) : 1.0;
  if (threadIdx.x == BK2_CONS) {
    sh2_tile_issue<E>(op, in, x0, y0, smem2, &tbar);
    // pull what the stencil epilogue will read into L2 while the tile is in flight.  No basis tiles: the first ones are still
    // in L2 from k2_update (evict_last), and prefetching more of them only competes with the prologue for HBM
    const unsigned row_b = (unsigned)(((tl.len + 1) & ~1) * 8);
    for (int r = 0; r < tl.rows; ++r) {
      const long long o = tl.base + (long long)r * tl.rs;
      bulk_prefetch_l2(op.u + o, row_b);
      if (BORDERED) {
        bulk_prefetch_l2(op.ba + o, row_b);
        bulk_prefetch_l2(op.bb + o, row_b);
      }
    }
  }
  const double xp = BORDERED ? s * __ldg(in + op.N) : 0.0;
  double bsum = 0.0;
  sh2_tile_eval<E, BORDERED>(op, in, s, x0, y0, smem2, &tbar, val, xp, &bsum);
  fence_proxy_async_smem();  // generic-proxy accesses to the scratch are ordered before the TMA writes that reuse it
  __syncthreads();           // scratch is dead, barriers are initialised: the ring takes over the shared memory
  stream_basis<E, 0>(tl, V, ld, j, keep, ring, NS, &rg, val, sred, nullptr);
  // w is stored after the basis stream (val is unchanged by it), so that it is still in L2 when k2_update reads it
  if (threadIdx.x < tl.len) {
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (e < tl.rows) w[tl.base + (long long)e * tl.rs + threadIdx.x] = val[e];
  }
  if (BORDERED) {
    __shared__ double s_wp;
    bsum = bk_warp_sum(bsum);  // bsum already carries the input scale (v = s * in)
    if ((threadIdx.x & 31) == 0 && threadIdx.x < BK2_CONS) sred[j * 8 + (threadIdx.x >> 5)] = bsum;
    __syncthreads();
    BorderFin bf;
    bf.bscale = op.bscale;
    bf.bc = op.bc;
    bf.xp = xp;
    bf.w_tail = w + op.N;
    bf.V_tail = V + op.N;
    bf.ld = ld;
    dots_finish(j, sred, scales, partials, counter, hcol, gcoef, &s_flag, &bf, &s_wp);
  } else {
    __syncthreads();
    dots_finish(j, sred, scales, partials, counter, hcol, gcoef, &s_flag);
  }
}

// Stand-alone K1 / K2 for the 2-D Swift-Hohenberg stencil on the same TMA-staged tile (MODE 0: out = a0 v + a1 J(u) v, 1: F(v)).
// 256 columns x E rows per CTA, 16-byte aligned bulk rows, no per-element div/mod in the load phase.
template <int E, int MODE>
static __global__ void __launch_bounds__(BK2_THREADS, 4) k2_apply(OpDesc op, const double* __restrict__ in,
                                                                  const double* __restrict__ in_scale_ptr, double* __restrict__ out) {
  extern __shared__ __align__(128) double smem2[];
  __shared__ __align__(8) unsigned long long tbar;
  if (threadIdx.x == 0) {
    mbar_init(&tbar, 1);
    fence_mbar_init();
  }
  const int tiles_x = (op.nx + BK2_ROW - 1) / BK2_ROW;
  const int x0 = (blockIdx.x % tiles_x) * BK2_ROW, y0 = (blockIdx.x / tiles_x) * E;
  const int rows = min(E, op.ny - y0), len = min(BK2_ROW, op.nx - x0);
  __syncthreads();
  const double s = in_scale_ptr ? __ldg(in_scale_ptr) : 1.0;
  if (threadIdx.x == BK2_CONS) {
    sh2_tile_issue<E>(op, in, x0, y0, smem2, &tbar);
    if (MODE == 0) {
      const unsigned row_b = (unsigned)(len * 8);
      for (int r = 0; r < rows; ++r) bulk_prefetch_l2(op.u + x0 + (long long)(y0 + r) * op.nx, row_b);
    }
  }
  double val[E];
  double bsum = 0.0;
  sh2_tile_eval<E, false, MODE == 1>(op, in, s, x0, y0, smem2, &tbar, val, 0.0, &bsum);
  if (threadIdx.x < len) {
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (e < rows) out[x0 + (long long)(y0 + e) * op.nx + threadIdx.x] = val[e];
  }
}

__device__ __forceinline__ Tile2 linear_tile(long long n, int E) {
  Tile2 tl;
  tl.base = (long long)blockIdx.x * (E * BK2_ROW);
  tl.rs = BK2_ROW;
  long long rem = n - tl.base;
  int rows = (int)((rem + BK2_ROW - 1) / BK2_ROW);
  tl.rows = rows < E ? rows : E;
  tl.len = BK2_ROW;
  long long lastrem = rem - (long long)(tl.rows - 1) * BK2_ROW;
  tl.last_len = lastrem < BK2_ROW ? (int)lastrem : BK2_ROW;
  if (tl.rows == 1) tl.len = tl.last_len;
  return tl;
}

template <int E>
static __global__ void __launch_bounds__(BK2_THREADS, 4) k2_dots(const double* __restrict__ w, long long n,
                                                                 const double* __restrict__ V, long long ld, int j,
                                                                 const double* __restrict__ scales,
                                                                 double* __restrict__ partials, unsigned int* counter,
                                                                 double* __restrict__ hcol, double* __restrict__ gcoef, int keep,
                                                                 int NS, int sred_off) {
  extern __shared__ __align__(128) double smem2[];
  __shared__ Ring rg;
  __shared__ int s_flag;
  double* ring = smem2;
  double* sred = smem2 + sred_off;
  ring_init(&rg, NS);
  const Tile2 tl = linear_tile(n, E);
  double val[E];
  bk_pdl_sync();  // after the barrier set-up: it overlaps the tail of the previous kernel
#pragma unroll
  for (int e = 0; e < E; ++e) {
    const int lim = (e == tl.rows - 1) ? tl.last_len : tl.len;
    val[e] = (threadIdx.x < BK2_ROW && e < tl.rows && (int)threadIdx.x < lim) ? w[tl.base + e * BK2_ROW + threadIdx.x] : 0.0;
  }
  __syncthreads();
  stream_basis<E, 0>(tl, V, ld, j, keep, ring, NS, &rg, val, sred, nullptr);
  __syncthreads();
  dots_finish(j, sred, scales, partials, counter, hcol, gcoef, &s_flag);
}

template <int E>
static __global__ void __launch_bounds__(BK2_THREADS, 4) k2_update(const double* w, long long n,  // w may alias vout
                                                                   const double* __restrict__ V, long long ld, int j,
                                                                   const double* __restrict__ gcoef, double* vout,
                                                                   double* __restrict__ partials, unsigned int* counter,
                                                                   double* __restrict__ h_out, double* __restrict__ scale_out,
                                                                   int keep, int NS) {
  extern __shared__ __align__(128) double smem2[];
  __shared__ Ring rg;
  __shared__ double s_w[9];
  __shared__ int s_flag;
  double* ring = smem2;
  ring_init(&rg, NS);
  const Tile2 tl = linear_tile(n, E);
  double val[E];
  const int t = threadIdx.x;
  bk_pdl_sync();  // after the barrier set-up: it overlaps the tail of the previous kernel
#pragma unroll
  for (int e = 0; e < E; ++e) {
    const int lim = (e == tl.rows - 1) ? tl.last_len : tl.len;
    val[e] = (t < BK2_ROW && e < tl.rows && t < lim) ? w[tl.base + e * BK2_ROW + t] : 0.0;
  }
  __syncthreads();
  stream_basis<E, 1, true>(tl, V, ld, j, keep, ring, NS, &rg, val, nullptr, gcoef);
  double acc = 0.0;
  if (t < BK2_ROW) {
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int lim = (e == tl.rows - 1) ? tl.last_len : tl.len;
      if (e < tl.rows && t < lim) {
        vout[tl.base + e * BK2_ROW + t] = val[e];
        acc = fma(val[e], val[e], acc);
      }
    }
  }
  acc = bk_warp_sum(acc);
  const int lane = t & 31, wid = t >> 5;
  if (lane == 0) s_w[wid] = acc;
  __syncthreads();
  if (t == 0) {
    double r = 0;
    for (int k = 0; k < 9; ++k) r += s_w[k];
    partials[blockIdx.x] = r;
  }
  if (bk_last_block(counter, &s_flag)) {
    double r = 0.0;
    for (int k = t; k < (int)gridDim.x; k += blockDim.x) r += __ldcg(partials + k);
    r = bk_warp_sum(r);
    if (lane == 0) s_w[wid] = r;
    __syncthreads();
    if (t == 0) {
      double q = 0;
      for (int k = 0; k < 9; ++k) q += s_w[k];
      const double h = sqrt(q);
      *h_out = h;
      *scale_out = 1.0 / h;
    }
  }
}
