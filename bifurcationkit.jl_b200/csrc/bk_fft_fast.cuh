// bk_fft_fast.cuh -- K6, third generation: register-resident DCT-II kernels for power-of-two line lengths 64..2048.
//
// The preconditioner of the Swift-Hohenberg examples, (L1 + shift I)^-1 with L1 = (I + Lap_Neumann)^2
// (examples/SH2d-fronts.jl:120-122, examples/SH3d.jl:88), is diagonal in the DCT-II basis (bk_precond.cu).  The second
// generation (radix-4 passes IN shared memory) was instruction-bound.  This version keeps the data in registers:
//
//  * TWO real lines form ONE complex line z = v1 + i v2 after Makhoul's reordering (v[m] = x[2m], v[n-1-m] = x[2m+1]).  In
//    the strided directions the two lines are neighbouring columns, so z is simply a 16-byte load.  One length-n complex FFT
//    gives both DCTs:  V1[k] = (Z[k] + conj Z[n-k]) / 2,  V2[k] = (Z[k] - conj Z[n-k]) / 2i,  C_p[k] = Re(w_k V_p[k]),
//    w_k = exp(-i pi k / 2n);  also  w_k V_p[k] = C_p[k] - i C_p[n-k].
//  * every thread owns E = 2^LOGE complex values; a pass of the decimation-in-frequency FFT has radix r <= E and runs E / r
//    butterflies per thread entirely in registers (compile-time twiddles W_32^j); between passes the line lives IN PLACE in
//    shared memory (butterfly (blk, b) of a pass with block length N_p = r M' touches positions blk N_p + a M' + b, a < r, and
//    writes the same positions), so n = 1024 needs two passes (32 x 32) and ONE exchange per FFT.  Z[k] ends at the
//    digit-reversed position pos(k); the inverse is the exact mirror (decimation in time, conjugate twiddles), so the fused
//    kernel (forward, divide by the operator symbol, inverse) never restores natural order;
//  * twiddles between passes come from per-pass tables that are contiguous in the butterfly position b; w_k and the 1-D
//    eigenvalues (lambda[k], lambda[n-k]) are stored in REGISTER-major order tab[reg * T + tau] (coalesced, broadcast across
//    the lanes of different line pairs);
//  * shared-memory slot of position i of pair pr:  (i + (i >> 2) + (i >> PB)) * PP + pr  (conflict-free for every pass in the
//    bank model tools/fftcheck/model.py + tools/fftcheck/padsearch.py).
//  * the periodic kind (BK_SH2D_PERIODIC) reuses the same FFT as a real 2-D transform: k_contig MODE 2 / 3 (x r2c / c2r, two
//    rows per complex line, packed half-spectrum, pointwise prologue / epilogue) and k_strided MODE 3 (y forward, periodic
//    symbol, inverse).
// Executable specification, thread by thread: tools/fftcheck/model.py (checked against scipy.fft).
// Device check + timing: tools/fftcheck/fft_check.cu.
#pragma once
#include "bk_common.cuh"
#include "bk_async.cuh"

namespace bkf {

// ------------------------------------------------------------------------------------------------ configuration
template <int LOGN_, int LOGE_>
struct Cfg {
  static constexpr int LOGN = LOGN_, LOGE = LOGE_;
  static constexpr int N = 1 << LOGN, E = 1 << LOGE, T = N / E;   // T threads per line pair
  static constexpr int F = LOGN / LOGE, RB = LOGN % LOGE;          // F full passes of radix E, then one of radix 2^RB
  static constexpr int NP = F + (RB ? 1 : 0);
  static constexpr int PP = (T >= 32) ? 2 : 64 / T;                // line pairs per CTA
  static constexpr int THREADS = T * PP;
  // second padding shift, chosen per (E, n) with the bank model (tools/fftcheck/model.py); 0 = none
  static constexpr int PB = LOGE == 5 ? (LOGN >= 10 ? 5 : 4) : LOGE == 4 ? 4 : LOGE == 3 ? ((LOGN == 9 || LOGN == 10) ? 3 : 0) : 0;
  __host__ __device__ static constexpr int pad(int i) { return i + (i >> 2) + (PB ? (i >> PB) : 0); }
  // resident threads per SM the register budget is sized for (launch bounds): few fat threads (E = 32: 255 registers) ... many thin ones
  static constexpr int TPSM = LOGE == 5 ? 256 : LOGE == 4 ? 512 : LOGE == 3 ? 768 : 1024;
  static constexpr int MINB = TPSM / THREADS > 0 ? TPSM / THREADS : 1;
  // the periodic r2c split and the periodic y pass hold twice the values across a barrier: one CTA per SM fewer, so the
  // instantiations the library launches (E = 4 below n = 1024, E = 8 from 1024 on; bk_precond.cu::fast_loge) do not spill
  // (tests/test_sass_periodic_cpu.py).  Other E, reachable only through BK_FFT_LOGE, still spill in some periodic modes
  // (e.g. k_strided MODE 3 at n = 512, E = 16; n = 2048, E = 4): correct, but not tuned.
  static constexpr int MINB_P = MINB > 1 ? MINB - 1 : 1;
  // padding of the NATURAL-order staging array of the contiguous kernels (scatter by register = digit-reversed k, then read
  // k = tau + T i): conflict-free choices from the same bank model (tools/fftcheck/padsearch.py)
  static constexpr int NB = LOGE == 2 ? (LOGN <= 6 ? 0 : LOGN <= 8 ? 4 : LOGN <= 10 ? 6 : 8)
                          : LOGE == 3 ? (LOGN <= 6 ? 0 : LOGN <= 9 ? 3 : 6)
                          : LOGE == 4 ? (LOGN <= 8 ? 0 : 4)
                                      : (LOGN <= 10 ? 0 : 5);
  __host__ __device__ static constexpr int padn(int k) { return k + (k >> 2) + (NB ? (k >> NB) : 0); }
  static constexpr int SLOTS_POS = pad(N - 1) + 1, SLOTS_NAT = padn(N - 1) + 1;
  static constexpr int SLOTS = SLOTS_POS > SLOTS_NAT ? SLOTS_POS : SLOTS_NAT;   // padded complex slots per pair
  static constexpr size_t SMEM_DATA = sizeof(double2) * (size_t)SLOTS * PP;
  __host__ __device__ static constexpr int logr(int p) { return p < F ? LOGE : RB; }
  __host__ __device__ static constexpr int logNp(int p) { return LOGN - LOGE * p; }       // block length before pass p
  __host__ __device__ static constexpr int logMp(int p) { return logNp(p) - logr(p); }     // butterfly stride of pass p
  __host__ __device__ static constexpr int tw_off(int p) {                                 // offset of pass p's twiddle table
    int o = 0;
    for (int q = 0; q < p; ++q) o += ((1 << logr(q)) - 1) << logMp(q);
    return o;
  }
  static constexpr int TW_TOTAL = tw_off(NP);
  // shared memory: work array | twiddles | w_k | (lambda[k], lambda[n-k]) -- the tables are copied in by the TMA engine
  static constexpr size_t SMEM = SMEM_DATA + sizeof(double2) * ((size_t)TW_TOTAL + N);          // forward / inverse kernels
  static constexpr size_t SMEM_FUSED = SMEM + sizeof(double2) * (size_t)N;                      // fused kernel
  static_assert(LOGN >= LOGE + 1 && LOGN <= 11, "line length out of range");
  static_assert(THREADS <= 1024, "CTA too large");
};

// position <-> frequency (digit reversal in units of LOGE bits, last digit RB bits)
template <class C>
__host__ __device__ inline int k_of_pos(int p) {
  int k = 0, sh = 0;
  for (int q = 0; q < C::NP; ++q) {
    const int d = (p >> C::logMp(q)) & ((1 << C::logr(q)) - 1);
    k |= d << sh;
    sh += C::logr(q);
  }
  return k;
}
template <class C>
__host__ __device__ inline int pos_of_k(int k) {
  int p = 0, sh = 0;
  for (int q = 0; q < C::NP; ++q) {
    const int d = (k >> sh) & ((1 << C::logr(q)) - 1);
    p |= d << C::logMp(q);
    sh += C::logr(q);
  }
  return p;
}
__host__ __device__ constexpr int brev_c(int j, int bits) {
  int r = 0;
  for (int b = 0; b < bits; ++b) r |= ((j >> b) & 1) << (bits - 1 - b);
  return r;
}

#ifdef __CUDACC__
// ------------------------------------------------------------------------------------------------ complex helpers
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(fma(a.x, b.x, -(a.y * b.y)), fma(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ double2 cmulc(double2 a, double2 b) {  // a * conj(b)
  return make_double2(fma(a.x, b.x, a.y * b.y), fma(a.y, b.x, -(a.x * b.y)));
}

#define BKF_C1 0.98078528040323043
#define BKF_S1 0.19509032201612825
#define BKF_C2 0.92387953251128674
#define BKF_S2 0.38268343236508978
#define BKF_C3 0.83146961230254524
#define BKF_S3 0.55557023301960218
#define BKF_C4 0.70710678118654752
// t * W_32^j (INV: t * conj(W_32^j)), j a compile-time constant after unrolling; W_32^j = cos(pi j/16) - i sin(pi j/16)
template <bool INV>
__device__ __forceinline__ double2 mul_w32(double2 t, int j) {
  double c, s;
  switch (j) {
    case 0: return t;
    case 8: return INV ? make_double2(-t.y, t.x) : make_double2(t.y, -t.x);
    case 4: {
      const double a = BKF_C4 * t.x, b = BKF_C4 * t.y;
      return INV ? make_double2(a - b, a + b) : make_double2(a + b, b - a);
    }
    case 12: {
      const double a = BKF_C4 * t.x, b = BKF_C4 * t.y;
      return INV ? make_double2(-a - b, a - b) : make_double2(b - a, -a - b);
    }
    case 1: c = BKF_C1; s = BKF_S1; break;
    case 2: c = BKF_C2; s = BKF_S2; break;
    case 3: c = BKF_C3; s = BKF_S3; break;
    case 5: c = BKF_S3; s = BKF_C3; break;
    case 6: c = BKF_S2; s = BKF_C2; break;
    case 7: c = BKF_S1; s = BKF_C1; break;
    case 9: c = -BKF_S1; s = BKF_C1; break;
    case 10: c = -BKF_S2; s = BKF_C2; break;
    case 11: c = -BKF_S3; s = BKF_C3; break;
    case 13: c = -BKF_C3; s = BKF_S3; break;
    case 14: c = -BKF_C2; s = BKF_S2; break;
    default: c = -BKF_C1; s = BKF_S1; break;  // 15
  }
  // forward: (x + i y)(c - i s) = (x c + y s) + i (y c - x s);  inverse: (x c - y s) + i (y c + x s)
  return INV ? make_double2(fma(t.x, c, -(t.y * s)), fma(t.y, c, t.x * s)) : make_double2(fma(t.x, c, t.y * s), fma(t.y, c, -(t.x * s)));
}

// in-register radix-R decimation in frequency on a[S0 .. S0+R-1]; output q lands at index S0 + brev(q)
template <int R, int S0, int ESZ>
__device__ __forceinline__ void bfly_fwd(double2 (&a)[ESZ]) {
  if constexpr (R >= 2) {
    constexpr int H = R / 2;
#pragma unroll
    for (int i = 0; i < H; ++i) {
      const double2 u = a[S0 + i], v = a[S0 + i + H];
      a[S0 + i] = cadd(u, v);
      a[S0 + i + H] = mul_w32<false>(csub(u, v), i * (32 / R));
    }
    bfly_fwd<H, S0, ESZ>(a);
    bfly_fwd<H, S0 + H, ESZ>(a);
  }
}
// mirror: input Y_q at index S0 + brev(q), output natural order, unnormalised inverse DFT
template <int R, int S0, int ESZ>
__device__ __forceinline__ void bfly_inv(double2 (&a)[ESZ]) {
  if constexpr (R >= 2) {
    constexpr int H = R / 2;
    bfly_inv<H, S0, ESZ>(a);
    bfly_inv<H, S0 + H, ESZ>(a);
#pragma unroll
    for (int i = 0; i < H; ++i) {
      const double2 u = a[S0 + i], t = mul_w32<true>(a[S0 + i + H], i * (32 / R));
      a[S0 + i] = cadd(u, t);
      a[S0 + i + H] = csub(u, t);
    }
  }
}

// ------------------------------------------------------------------------------------------------ tables / geometry
struct Tables {  // global memory (built on the host by build_tables)
  const double2* tw;    // per-pass contiguous forward twiddles  W_{N_p}^{b q} at tw_off(p) + (q-1) M' + b
  const double2* om;    // om[reg * T + tau]   = w_k          of the position the thread holds in register `reg` after the last pass
  const double2* lam2;  // lam2[reg * T + tau] = (lambda[k], lambda[(n-k) % n])
};
// Every table entry is read exactly once per line pair, by one thread: straight from global memory each read is an exposed L2
// round trip, and with few warps per SM nothing hides it.  The
// CTA therefore pulls its tables into shared memory with three bulk copies issued BEFORE griddepcontrol.wait -- the tables are
// constants, so the copies overlap the tail of the previous kernel -- and waits on the mbarrier just before the first use.
template <class C, bool FUSED>
__device__ __forceinline__ Tables stage_tables(const Tables& g, double2* sm, unsigned long long* bar) {
  Tables t;
  double2* stw = sm + (size_t)C::SLOTS * C::PP;
  double2* som = stw + C::TW_TOTAL;
  double2* slam = som + C::N;
  if (threadIdx.x == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
    constexpr unsigned twb = 16u * C::TW_TOTAL, nb = 16u * C::N;
    mbar_arrive_expect_tx(bar, twb + nb + (FUSED ? nb : 0u));
    if (twb) bulk_g2s(stw, g.tw, twb, bar);
    bulk_g2s(som, g.om, nb, bar);
    if (FUSED) bulk_g2s(slam, g.lam2, nb, bar);
  }
  t.tw = stw;
  t.om = som;
  t.lam2 = slam;
  return t;
}

struct Geom {
  long long es;   // element stride along the line (doubles); 1 for contiguous lines
  long long os;   // stride of the outer index
  int nb;         // extent of the batch index: strided lines: columns (contiguous, stride 1); contiguous lines: number of lines (stride os)
  int nouter;     // strided lines only: number of outer indices (blockIdx.y)
};

struct Symbol {
  const double* lam_b;  // eigenvalues along the batch (column) index
  const double* lam_o;  // eigenvalues along the outer index (may be NULL)
  double shift;         // out = in / ((1 + lam_line + lam_b + lam_o)^2 + shift)
  double scale;         // 1 / (2^d prod n): the forward kernels return 2 C, the inverse kernels n x
  const double* tail_src;  // optional pass-through of trailing (border) entries
  double* tail_dst;
  int tail_n;
  int neg;              // periodic kernel (MODE 3): 1 -> symbol -scale L1, 0 -> scale / (L1 + shift)
};

template <class C>
__device__ __forceinline__ int slot(int pos, int pr) { return C::pad(pos) * C::PP + pr; }

// position of register `reg` of thread tau in pass P (register index = u * r + j; j is the butterfly INPUT a for loads of a
// forward pass, and brev(output q) after the butterfly)
template <class C, int P>
__device__ __forceinline__ void pass_geom(int tau, int u, int& base, int& b) {
  constexpr int LM = C::logMp(P), LN = C::logNp(P);
  const int beta = tau + C::T * u;
  const int blk = beta >> LM;
  b = beta & ((1 << LM) - 1);
  base = (blk << LN) + b;
}

// ------------------------------------------------------------------------------------------------ the FFT itself
template <int R, int U, int NB, int ESZ>
__device__ __forceinline__ void bfly_all_fwd(double2 (&a)[ESZ]) {
  if constexpr (U < NB) {
    bfly_fwd<R, U * R, ESZ>(a);
    bfly_all_fwd<R, U + 1, NB, ESZ>(a);
  }
}
template <int R, int U, int NB, int ESZ>
__device__ __forceinline__ void bfly_all_inv(double2 (&a)[ESZ]) {
  if constexpr (U < NB) {
    bfly_inv<R, U * R, ESZ>(a);
    bfly_all_inv<R, U + 1, NB, ESZ>(a);
  }
}

// Forward passes P .. NP-1.  Entry (P = 0): a[i] = z[i * T + tau].  Exit: a[u * r + j] = Z at position
// ((tau + T u) << logr(NP-1)) + brev(j), r = radix of the last pass.
template <class C, int P>
__device__ __forceinline__ void fwd_passes(double2 (&a)[C::E], double2* sm, const Tables& tb, int tau, int pr) {
  constexpr int LR = C::logr(P), R = 1 << LR, NB = C::E / R, LM = C::logMp(P);
  if constexpr (P > 0) {
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      int base, b;
      pass_geom<C, P>(tau, u, base, b);
#pragma unroll
      for (int i = 0; i < R; ++i) a[u * R + i] = sm[slot<C>(base + (i << LM), pr)];
    }
  }
  bfly_all_fwd<R, 0, NB, C::E>(a);
  if constexpr (P < C::NP - 1) {
    const double2* tw = tb.tw + C::tw_off(P);
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      int base, b;
      pass_geom<C, P>(tau, u, base, b);
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const int q = brev_c(j, LR);
        double2 v = a[u * R + j];
        if (q > 0) v = cmul(v, tw[((q - 1) << LM) + b]);
        sm[slot<C>(base + (q << LM), pr)] = v;
      }
    }
    __syncthreads();
    fwd_passes<C, P + 1>(a, sm, tb, tau, pr);
  }
}

// Inverse passes P .. 0 (mirror of fwd_passes).  Entry (P = NP-1): registers as fwd_passes leaves them.
// Exit: a[i] = n * z[i * T + tau] (unnormalised inverse DFT).
template <class C, int P>
__device__ __forceinline__ void inv_passes(double2 (&a)[C::E], double2* sm, const Tables& tb, int tau, int pr) {
  constexpr int LR = C::logr(P), R = 1 << LR, NB = C::E / R, LM = C::logMp(P);
  if constexpr (P < C::NP - 1) {
    const double2* tw = tb.tw + C::tw_off(P);
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      int base, b;
      pass_geom<C, P>(tau, u, base, b);
#pragma unroll
      for (int j = 0; j < R; ++j) {
        const int q = brev_c(j, LR);
        double2 v = sm[slot<C>(base + (q << LM), pr)];
        if (q > 0) v = cmulc(v, tw[((q - 1) << LM) + b]);
        a[u * R + j] = v;
      }
    }
  }
  bfly_all_inv<R, 0, NB, C::E>(a);
  if constexpr (P > 0) {
#pragma unroll
    for (int u = 0; u < NB; ++u) {
      int base, b;
      pass_geom<C, P>(tau, u, base, b);
#pragma unroll
      for (int i = 0; i < R; ++i) sm[slot<C>(base + (i << LM), pr)] = a[u * R + i];
    }
    __syncthreads();
    inv_passes<C, P - 1>(a, sm, tb, tau, pr);
  }
}

// position held in register `reg` after the last forward pass
template <class C>
__device__ __forceinline__ int reg_pos(int tau, int reg) {
  constexpr int LR = C::logr(C::NP - 1), R = 1 << LR;
  const int u = reg >> LR, j = reg & (R - 1);
  return ((tau + C::T * u) << LR) + brev_c(j, LR);
}
// write Z in place so that every thread can read the partner Z[n-k]; caller syncs
template <class C>
__device__ __forceinline__ void park(const double2 (&a)[C::E], double2* sm, int tau, int pr) {
#pragma unroll
  for (int reg = 0; reg < C::E; ++reg) sm[slot<C>(reg_pos<C>(tau, reg), pr)] = a[reg];
}
template <class C>
__device__ __forceinline__ double2 partner(const double2* sm, int pos, int pr, int& k) {
  k = k_of_pos<C>(pos);
  const int nk = (C::N - k) & (C::N - 1);
  return sm[slot<C>(pos_of_k<C>(nk), pr)];
}
// row of the Makhoul-reordered element m:  v[m] = x[2m] (m < n/2),  v[m] = x[2n-1-2m] (m >= n/2)
template <class C>
__device__ __forceinline__ int row_of(int i, int tau) {
  const int m = i * C::T + tau;
  return (i < C::E / 2) ? 2 * m : 2 * C::N - 1 - 2 * m;
}

// ------------------------------------------------------------------------------------------------ strided lines (y, z)
template <class C>
__device__ __forceinline__ void strided_load(double2 (&a)[C::E], const double* __restrict__ base, long long es, int tau, bool v0,
                                             bool v1) {
  if (v1) {
#pragma unroll
    for (int i = 0; i < C::E; ++i) a[i] = __ldg(reinterpret_cast<const double2*>(base + (long long)row_of<C>(i, tau) * es));
  } else {
#pragma unroll
    for (int i = 0; i < C::E; ++i) a[i] = make_double2(v0 ? __ldg(base + (long long)row_of<C>(i, tau) * es) : 0.0, 0.0);
  }
}
template <class C>
__device__ __forceinline__ void strided_store(const double2 (&a)[C::E], double* __restrict__ base, long long es, int tau, bool v0,
                                              bool v1) {
  if (v1) {
#pragma unroll
    for (int i = 0; i < C::E; ++i) *reinterpret_cast<double2*>(base + (long long)row_of<C>(i, tau) * es) = a[i];
  } else if (v0) {
#pragma unroll
    for (int i = 0; i < C::E; ++i) base[(long long)row_of<C>(i, tau) * es] = a[i].x;
  }
}

#define BKF_BOUNDS(C, PERIODIC) __launch_bounds__(C::THREADS, (PERIODIC) ? C::MINB_P : C::MINB)

// 1 / x for 0 < x < 2^1000: hardware estimate + two Newton steps (no division slow path: its call frame spills)
__device__ __forceinline__ double rcp_nr(double x) {
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x));
  double e = fma(-x, r, 1.0);
  r = fma(r, e, r);
  e = fma(-x, r, 1.0);
  return fma(r, e, r);
}
// periodic symbol of one element, lam = lambda_x + lambda_y (eigenvalues of the periodic Laplacian, -k^2)
__device__ __forceinline__ double per_symbol(const Symbol& sy, double lam) {
  const double t = 1.0 + lam, l1 = t * t;
  return sy.neg ? -sy.scale * l1 : sy.scale * rcp_nr(l1 + sy.shift);
}

// MODE 0: forward (out = 2 C, natural k along the line), 1: inverse (out = n x from C), 2: forward, divide by the symbol, inverse
// MODE 3: periodic y pass of BK_SH2D_PERIODIC: forward FFT, multiply by the periodic symbol, inverse, natural order both ways.
//   The input rows are the packed half-spectra of k_contig MODE 2, so for q >= 1 the column pair (2q, 2q+1) is the complex line
//   of kx = q (one 16-byte load per element).  Pair (0, 1) holds two real lines, kx = 0 and kx = Nx/2, with symbols s0 and sn;
//   as the symbol is even in ky, Z'[k] = ((s0 + sn)/2) Z[k] + ((s0 - sn)/2) conj Z[-k] (one partner read).
template <class C, int MODE>
static __global__ void BKF_BOUNDS(C, MODE == 3) k_strided(const double* __restrict__ in, double* __restrict__ out, Geom g, Tables tbg, Symbol sy) {
  extern __shared__ __align__(128) double2 sm_fast[];
  __shared__ __align__(8) unsigned long long tbar;
  double2* sm = sm_fast;
  const Tables tb = stage_tables<C, MODE == 2 || MODE == 3>(tbg, sm, &tbar);
  const int tid = threadIdx.x, pr = tid % C::PP, tau = tid / C::PP;
  __syncthreads();  // the barrier is initialised before anybody waits on it
  bk_pdl_sync();
  const int col = (blockIdx.x * C::PP + pr) * 2, o = blockIdx.y;
  const bool v0 = col < g.nb, v1 = col + 1 < g.nb;
  const long long off = (long long)o * g.os + col;
  if ((MODE == 2 || MODE == 3) && sy.tail_n > 0 && blockIdx.x == 0 && blockIdx.y == 0 && tid < sy.tail_n)
    sy.tail_dst[tid] = sy.tail_src[tid];
  double2 a[C::E];
  if (MODE == 3) {
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      const double* p = in + off + (long long)(i * C::T + tau) * g.es;
      a[i] = v1 ? __ldg(reinterpret_cast<const double2*>(p)) : make_double2(v0 ? __ldg(p) : 0.0, 0.0);
    }
    mbar_wait(&tbar, 0);
    fwd_passes<C, 0>(a, sm, tb, tau, pr);
    const bool nyq = blockIdx.x == 0 && pr == 0;   // column pair (0, 1): kx = 0 and kx = Nx/2
    if (blockIdx.x == 0) {                          // CTA-uniform
      park<C>(a, sm, tau, pr);
      __syncthreads();
      if (nyq) {
        const double l0 = __ldg(sy.lam_b), ln = __ldg(sy.lam_b + (g.nb >> 1));
#pragma unroll
        for (int reg = 0; reg < C::E; ++reg) {
          int k;
          const double2 z = a[reg], zp = partner<C>(sm, reg_pos<C>(tau, reg), pr, k);
          const double ly = tb.lam2[reg * C::T + tau].x;
          const double s0 = per_symbol(sy, l0 + ly), sn = per_symbol(sy, ln + ly);
          const double hp = 0.5 * (s0 + sn), hm = 0.5 * (s0 - sn);
          a[reg] = make_double2(fma(hp, z.x, hm * zp.x), fma(hp, z.y, -(hm * zp.y)));
        }
      }
      __syncthreads();
    }
    if (!nyq) {
      const double lq = v0 ? __ldg(sy.lam_b + (col >> 1)) : 0.0;
#pragma unroll
      for (int reg = 0; reg < C::E; ++reg) {
        const double s = per_symbol(sy, lq + tb.lam2[reg * C::T + tau].x);
        a[reg] = make_double2(s * a[reg].x, s * a[reg].y);
      }
    }
    inv_passes<C, C::NP - 1>(a, sm, tb, tau, pr);
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      double* p = out + off + (long long)(i * C::T + tau) * g.es;
      if (v1) *reinterpret_cast<double2*>(p) = a[i];
      else if (v0) *p = a[i].x;
    }
    return;
  }
  if (MODE != 1) {
    strided_load<C>(a, in + off, g.es, tau, v0, v1);
    mbar_wait(&tbar, 0);
    fwd_passes<C, 0>(a, sm, tb, tau, pr);
    park<C>(a, sm, tau, pr);
    __syncthreads();
  }
  if (MODE == 0) {
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) {
      int k;
      const double2 z = a[reg], zp = partner<C>(sm, reg_pos<C>(tau, reg), pr, k);
      const double2 w = tb.om[reg * C::T + tau];
      const double sx = z.x + zp.x, sy_ = z.y - zp.y;   // Z + conj Zp
      const double dx = z.x - zp.x, dy = z.y + zp.y;    // Z - conj Zp
      // 2 C1 = Re(w (Z + conj Zp)),  2 C2 = Re(w (-i)(Z - conj Zp)) = w.x dy + w.y dx
      const double c1 = fma(w.x, sx, -(w.y * sy_)), c2 = fma(w.x, dy, w.y * dx);
      double* p = out + off + (long long)k * g.es;
      if (v1) *reinterpret_cast<double2*>(p) = make_double2(c1, c2);
      else if (v0) *p = c1;
    }
    return;
  }
  if (MODE == 1) {
    // D[k] = C1[k] + i C2[k] parked at pos(k); Zhat[k] = conj(w_k) ((D[k].x + D[n-k].y) + i (D[k].y - D[n-k].x)), D[n] = 0
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) {
      const int k = k_of_pos<C>(reg_pos<C>(tau, reg));
      const double* p = in + off + (long long)k * g.es;
      a[reg] = v1 ? __ldg(reinterpret_cast<const double2*>(p)) : make_double2(v0 ? __ldg(p) : 0.0, 0.0);
    }
    mbar_wait(&tbar, 0);
    park<C>(a, sm, tau, pr);
    __syncthreads();
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) {
      int k;
      double2 dn = partner<C>(sm, reg_pos<C>(tau, reg), pr, k);
      if (k == 0) dn = make_double2(0.0, 0.0);
      const double2 w = tb.om[reg * C::T + tau];
      a[reg] = cmulc(make_double2(a[reg].x + dn.y, a[reg].y - dn.x), w);
    }
    __syncthreads();
  }
  if (MODE == 2) {
    const double lo = sy.lam_o ? __ldg(sy.lam_o + o) : 0.0;
    const double cA = 1.0 + lo + (v0 ? __ldg(sy.lam_b + col) : 0.0), cB = 1.0 + lo + (v1 ? __ldg(sy.lam_b + col + 1) : 0.0);
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) {
      int k;
      const double2 z = a[reg], zp = partner<C>(sm, reg_pos<C>(tau, reg), pr, k);
      const double2 w = tb.om[reg * C::T + tau];
      const double2 l2 = tb.lam2[reg * C::T + tau];
      // A1 = w (Z + conj Zp) = 2 (C1[k] - i C1[n-k]),  A2 = w (-i)(Z - conj Zp) = 2 (C2[k] - i C2[n-k])
      const double2 A1 = cmul(make_double2(z.x + zp.x, z.y - zp.y), w);
      const double2 A2 = cmul(make_double2(z.y + zp.y, zp.x - z.x), w);
      double t = cA + l2.x;
      const double s1k = fma(t, t, sy.shift);
      t = cA + l2.y;
      const double s1n = fma(t, t, sy.shift);
      t = cB + l2.x;
      const double s2k = fma(t, t, sy.shift);
      t = cB + l2.y;
      const double s2n = fma(t, t, sy.shift);
      const double r1 = sy.scale * __drcp_rn(s1k * s1n), r2 = sy.scale * __drcp_rn(s2k * s2n);
      const double h1x = A1.x * (r1 * s1n), h1y = A1.y * (r1 * s1k);   // C1[k] / s1k,  -C1[n-k] / s1n
      const double h2x = A2.x * (r2 * s2n), h2y = A2.y * (r2 * s2k);
      a[reg] = cmulc(make_double2(h1x - h2y, h1y + h2x), w);            // conj(w) (h1 + i h2)
    }
    __syncthreads();
  }
  inv_passes<C, C::NP - 1>(a, sm, tb, tau, pr);
  strided_store<C>(a, out + off, g.es, tau, v0, v1);
}

// ------------------------------------------------------------------------------------------------ contiguous lines (x)
// MODE 0: forward, 1: inverse.  A CTA owns 2 PP consecutive lines (PP pairs).  The Makhoul side (x[2m], x[2n-1-2m]) is read /
// written straight from / to global memory (8-byte accesses at a 16-byte stride: the other half of every sector belongs to the
// mirror register of another thread of the same CTA, L1 / L2 merge them); the frequency side goes through a NATURAL-order
// shared-memory array with its own conflict-free padding, so that global accesses in k are fully coalesced.  (The first
// version staged whole rows in natural order and scattered into them by digit-reversed k: most of its shared-memory
// wavefronts were bank conflicts.)
template <class C>
__device__ __forceinline__ int nslot(int k, int pr) { return C::padn(k) * C::PP + pr; }

__device__ __forceinline__ double pw_c(const PerPw& pw, double u) { return fma(u, fma(-3.0, u, 2.0 * pw.nu), pw.l); }
__device__ __forceinline__ double pw_d(const PerPw& pw, double u) { return fma(pw.a1, pw.spc + pw_c(pw, u), pw.a0); }
// epilogue of the periodic c2r pass (PerPw, bk_common.cuh); v / u point at the row, m is the element
__device__ __forceinline__ double pw_out(const PerPw& pw, double y, const double* v, const double* u, int m, double s) {
  switch (pw.epi) {
    case PW_RESID: {
      const double x = __ldg(v + m);
      return fma(x, fma(x, pw.nu - x, pw.l), y);
    }
    case PW_JVP: return fma(fma(pw.a1, pw_c(pw, __ldg(u + m)), pw.a0), s * __ldg(v + m), y);
    case PW_FLEFT: return fma(-pw.a1 * s, __ldg(v + m), y);
    case PW_FRIGHT: return fma(pw_d(pw, __ldg(u + m)), y, -pw.a1 * s * __ldg(v + m));
    default: return y;
  }
}

// MODE 2 / 3: the x passes of BK_SH2D_PERIODIC.  Two neighbouring rows form one complex line z = r_A + i r_B (natural order, no
// Makhoul reordering), so one length-n FFT gives both real transforms: X_A[k] = (Z[k] + conj Z[n-k]) / 2,
// X_B[k] = (Z[k] - conj Z[n-k]) / 2i.  A row is stored as its packed half-spectrum [Re X0, Re X_{n/2}, Re X1, Im X1, ...,
// Re X_{n/2-1}, Im X_{n/2-1}] (n doubles).  MODE 2 (r2c) multiplies the input by the prologue of pw first; MODE 3 (c2r) rebuilds
// Z[k] = X_A[k] + i X_B[k] (X[n-k] = conj X[k]), inverts (n z) and applies the epilogue of pw.  The caller's vectors are only
// touched by 8-byte accesses, so they need no 16-byte alignment.
template <class C, int MODE>
static __global__ void BKF_BOUNDS(C, MODE == 2) k_contig(const double* __restrict__ in, double* __restrict__ out, Geom g, Tables tbg, PerPw pw) {
  extern __shared__ __align__(128) double2 sm_fast[];
  __shared__ __align__(8) unsigned long long tbar;
  double2* sm = sm_fast;
  const Tables tb = stage_tables<C, false>(tbg, sm, &tbar);
  const int tid = threadIdx.x, pr = tid % C::PP, tau = tid / C::PP;
  __syncthreads();
  bk_pdl_sync();
  const long long lineA = ((long long)blockIdx.x * C::PP + pr) * 2, lineB = lineA + 1;
  const bool vA = lineA < g.nb, vB = lineB < g.nb;
  const double* inA = in + lineA * g.os;
  const double* inB = in + lineB * g.os;
  double* outA = out + lineA * g.os;
  double* outB = out + lineB * g.os;
  double2 a[C::E];
  if (MODE == 2) {
    const double s = pw.sp ? __ldg(pw.sp) : 1.0;
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      const int m = i * C::T + tau;
      double xa = vA ? __ldg(inA + m) : 0.0, xb = vB ? __ldg(inB + m) : 0.0;
      if (pw.pro == PW_D) {
        xa *= vA ? pw_d(pw, __ldg(pw.u + lineA * g.os + m)) : 0.0;
        xb *= vB ? pw_d(pw, __ldg(pw.u + lineB * g.os + m)) : 0.0;
      }
      a[i] = make_double2(s * xa, s * xb);
    }
    mbar_wait(&tbar, 0);
    fwd_passes<C, 0>(a, sm, tb, tau, pr);
    park<C>(a, sm, tau, pr);
    __syncthreads();
    double2 b[C::E];
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) {
      int k;
      const double2 z = a[reg], zp = partner<C>(sm, reg_pos<C>(tau, reg), pr, k);
      // X_A = (Z + conj Zp) / 2,  X_B = (Z - conj Zp) / 2i;  a = (Re X_A, Re X_B), b = (Im X_A, Im X_B)
      a[reg] = make_double2(0.5 * (z.x + zp.x), 0.5 * (z.y + zp.y));
      b[reg] = make_double2(0.5 * (z.y - zp.y), 0.5 * (zp.x - z.x));
    }
    __syncthreads();  // every partner read is done: the natural-order array may overwrite the work array
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) {
      const int k = k_of_pos<C>(reg_pos<C>(tau, reg));
      if (k == 0) sm[nslot<C>(0, pr)] = a[reg];
      else if (k == C::N / 2) sm[nslot<C>(1, pr)] = a[reg];
      else if (k < C::N / 2) {
        sm[nslot<C>(2 * k, pr)] = a[reg];
        sm[nslot<C>(2 * k + 1, pr)] = b[reg];
      }
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      const int p = i * C::T + tau;
      const double2 d = sm[nslot<C>(p, pr)];
      if (vA) outA[p] = d.x;
      if (vB) outB[p] = d.y;
    }
    return;
  }
  if (MODE == 3) {
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      const int p = i * C::T + tau;
      sm[nslot<C>(p, pr)] = make_double2(vA ? __ldg(inA + p) : 0.0, vB ? __ldg(inB + p) : 0.0);
    }
    mbar_wait(&tbar, 0);
    __syncthreads();
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) {
      const int k = k_of_pos<C>(reg_pos<C>(tau, reg)), kk = k <= C::N / 2 ? k : C::N - k;
      double2 xa, xb;  // X_A[kk], X_B[kk] (x: A, y: B in the packed pairs)
      if (kk == 0 || kk == C::N / 2) {
        const double2 d = sm[nslot<C>(kk ? 1 : 0, pr)];
        xa = make_double2(d.x, 0.0);
        xb = make_double2(d.y, 0.0);
      } else {
        const double2 re = sm[nslot<C>(2 * kk, pr)], im = sm[nslot<C>(2 * kk + 1, pr)];
        xa = make_double2(re.x, k == kk ? im.x : -im.x);
        xb = make_double2(re.y, k == kk ? im.y : -im.y);
      }
      a[reg] = make_double2(xa.x - xb.y, xa.y + xb.x);  // Z = X_A + i X_B
    }
    __syncthreads();  // the natural-order array is dead: the inverse passes reuse the memory
    inv_passes<C, C::NP - 1>(a, sm, tb, tau, pr);
    const double s = pw.sp ? __ldg(pw.sp) : 1.0;
    const double* vrA = pw.v + lineA * g.os;
    const double* vrB = pw.v + lineB * g.os;
    const double* urA = pw.u ? pw.u + lineA * g.os : nullptr;
    const double* urB = pw.u ? pw.u + lineB * g.os : nullptr;
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      const int m = i * C::T + tau;
      if (vA) outA[m] = pw_out(pw, a[i].x, vrA, urA, m, s);
      if (vB) outB[m] = pw_out(pw, a[i].y, vrB, urB, m, s);
    }
    return;
  }
  if (MODE == 0) {
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      const int e = row_of<C>(i, tau);
      a[i] = make_double2(vA ? __ldg(inA + e) : 0.0, vB ? __ldg(inB + e) : 0.0);
    }
    mbar_wait(&tbar, 0);
    fwd_passes<C, 0>(a, sm, tb, tau, pr);
    park<C>(a, sm, tau, pr);
    __syncthreads();
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) {
      int k;
      const double2 z = a[reg], zp = partner<C>(sm, reg_pos<C>(tau, reg), pr, k);
      const double2 w = tb.om[reg * C::T + tau];
      const double sx = z.x + zp.x, sy_ = z.y - zp.y, dx = z.x - zp.x, dy = z.y + zp.y;
      a[reg] = make_double2(fma(w.x, sx, -(w.y * sy_)), fma(w.x, dy, w.y * dx));   // (2 C1[k], 2 C2[k])
    }
    __syncthreads();  // every partner read is done: the natural-order array may overwrite the work array
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) sm[nslot<C>(k_of_pos<C>(reg_pos<C>(tau, reg)), pr)] = a[reg];
    __syncthreads();
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      const int k = i * C::T + tau;
      const double2 d = sm[nslot<C>(k, pr)];
      if (vA) outA[k] = d.x;
      if (vB) outB[k] = d.y;
    }
  } else {
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      const int k = i * C::T + tau;
      sm[nslot<C>(k, pr)] = make_double2(vA ? __ldg(inA + k) : 0.0, vB ? __ldg(inB + k) : 0.0);
    }
    mbar_wait(&tbar, 0);
    __syncthreads();
    // Zhat[k] = conj(w_k) ((D[k].x + D[n-k].y) + i (D[k].y - D[n-k].x)),  D[k] = C1[k] + i C2[k],  D[n] = 0
#pragma unroll
    for (int reg = 0; reg < C::E; ++reg) {
      const int k = k_of_pos<C>(reg_pos<C>(tau, reg)), nk = (C::N - k) & (C::N - 1);
      const double2 w = tb.om[reg * C::T + tau];
      const double2 d = sm[nslot<C>(k, pr)];
      double2 dn = sm[nslot<C>(nk, pr)];
      if (k == 0) dn = make_double2(0.0, 0.0);
      a[reg] = cmulc(make_double2(d.x + dn.y, d.y - dn.x), w);
    }
    __syncthreads();  // the natural-order array is dead: the inverse passes reuse the memory
    inv_passes<C, C::NP - 1>(a, sm, tb, tau, pr);
#pragma unroll
    for (int i = 0; i < C::E; ++i) {
      const int e = row_of<C>(i, tau);
      if (vA) outA[e] = a[i].x;
      if (vB) outB[e] = a[i].y;
    }
  }
}
#endif  // __CUDACC__

// ------------------------------------------------------------------------------------------------ host: tables
// lam may be NULL (no eigenvalue table: forward / inverse kernels only)
template <class C>
static inline void build_tables(std::vector<double>& tw, std::vector<double>& om, std::vector<double>& lam2, const double* lam) {
  const long double PI = 3.14159265358979323846264338327950288L;
  tw.assign(2 * (size_t)C::TW_TOTAL, 0.0);
  for (int p = 0; p < C::NP - 1; ++p) {
    const int r = 1 << C::logr(p), M = 1 << C::logMp(p), Np = 1 << C::logNp(p);
    for (int q = 1; q < r; ++q)
      for (int b = 0; b < M; ++b) {
        const long double ang = -2.0L * PI * (long double)((long long)b * q % Np) / Np;
        const size_t i = (size_t)C::tw_off(p) + (size_t)(q - 1) * M + b;
        tw[2 * i] = (double)cosl(ang);
        tw[2 * i + 1] = (double)sinl(ang);
      }
  }
  om.assign(2 * (size_t)C::N, 0.0);
  lam2.assign(2 * (size_t)C::N, 0.0);
  const int LR = C::logr(C::NP - 1), R = 1 << LR;
  for (int reg = 0; reg < C::E; ++reg)
    for (int tau = 0; tau < C::T; ++tau) {
      const int u = reg >> LR, j = reg & (R - 1);
      const int pos = ((tau + C::T * u) << LR) + brev_c(j, LR);
      const int k = k_of_pos<C>(pos), nk = (C::N - k) & (C::N - 1);
      const size_t i = (size_t)reg * C::T + tau;
      om[2 * i] = (double)cosl(-PI * k / (2.0L * C::N));
      om[2 * i + 1] = (double)sinl(-PI * k / (2.0L * C::N));
      if (lam) {
        lam2[2 * i] = lam[k];
        lam2[2 * i + 1] = lam[nk];
      }
    }
}
}  // namespace bkf
