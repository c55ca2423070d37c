// bk_common.cuh -- context, operator descriptor and small device helpers shared by the
// libbk200 translation units.  sm_90a only.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string>
#include <unordered_map>
#include <vector>
#include "../../include/bk200.h"
#include <nvtx3/nvToolsExt.h>   // header-only NVTX v3: ranges around the ABI entry points (visible in nsys / ncu --nvtx)

struct BkRange {  // RAII range
  explicit BkRange(const char* name) { nvtxRangePushA(name); }
  ~BkRange() { nvtxRangePop(); }
};

#define BK_MAX_PAR 8
#define BK_NSM_FALLBACK 132

// Operator descriptor, passed BY VALUE to kernels.  Describes  out = a0*in + a1*J(u)*in  for the
// named PDE stencils, optionally bordered (MatrixFreeBLSmap, src/LinearBorderSolver.jl:299-335).
struct OpDesc {
  int kind;
  int nx, ny, nz;        // grid (potrap: nz = M time slices)
  double cx, cy, cz;     // 1/h^2
  double par[BK_MAX_PAR];
  const double* u;       // linearisation state (device)
  double a0, a1;         // a0 I + a1 J
  long long N;           // unknowns of the un-bordered problem
  // bordered map:  out.u = Op(x.u) + x.p * ba (+ bshift * x.u);  out.p = bscale*<bb, x.u> + bc * x.p
  int bordered;          // number of borders: 0, 1 or 2
  const double* ba;
  const double* bb;
  double bc, bshift, bscale;
  // second border of the block / tuple form (src/LinearBorderSolver.jl:338-389): x.p and out.p have two entries,
  //   out.u += x.p[1] ba2;   out.p = bscale [<bb, x.u>; <bb2, x.u>] + [bc bc01; bc10 bc11] x.p
  const double* ba2;
  const double* bb2;
  double bc01, bc10, bc11;
  // potrap extras
  const double* phi;     // section (length N-1)
  const double* fcache;  // F(x_i) cache, M slices (device)
  // complexified contexts (BK_COMPLEX): N = 2 N0, vectors are [re; im], operator ((a0 + i a0i) I + a1 J) with J real
  int cplx;
  double a0i;
  int transpose;         // J' instead of J (cGL2d: transposed reaction block; SH: self-adjoint)
};

// general-length transform plan (bk_fft_gen.cuh), passed by value to the kernels
namespace bkg {
#define BKG_MAXPASS 16
struct Plan {
  int n;                   // line length
  int L;                   // FFT length: 2n (DCT-II, even extension) or 2n + 2 (DST-I, odd extension)
  int npass;
  int radix[BKG_MAXPASS];  // Stockham radices (prime factors of L, 4 preferred over 2 x 2)
  const double2* wl;       // W_L^t = exp(-2 pi i t / L), t < L
  const double2* ph;       // exp(-i pi k / 2n), k < n (DCT-II pre/post twiddle)
  double dst_scale;        // sqrt(2 / (n + 1)) / 2
};
}  // namespace bkg

// Pointwise prologue / epilogue of the periodic spectral pipeline (BK_SH2D_PERIODIC, bk_fft_fast.cuh k_contig MODE 2 / 3).
// The x r2c pass reads s v (pro = PW_D: s v d(u)); the x c2r pass turns the spectral result y into the output:
//   PW_NONE  y                       (preconditioner)
//   PW_RESID y + l v + nu v^2 - v^3  (residual, v = u)
//   PW_JVP   y + (a0 + a1 c(u)) s v  (the symbol carries -a1 L1)
//   PW_FLEFT y - a1 s v              (P (a0 I + a1 J) v = P (d v) - a1 v)
//   PW_FRIGHT d(u) y - a1 s v        ((a0 I + a1 J) P v = d (P v) - a1 v)
// with c(u) = l + 2 nu u - 3 u^2,  d(u) = a0 + a1 (spc + c(u)),  s = *sp (1 when sp is NULL).
enum { PW_NONE = 0, PW_RESID = 1, PW_JVP = 2, PW_FLEFT = 3, PW_FRIGHT = 4 };
struct PerPw {
  int pro;               // 0: s v, 1 (PW_D): s v d(u)
  int epi;               // PW_*
  const double* v;       // operator input (the epilogue reads it again)
  const double* u;       // linearisation state
  const double* sp;      // device scalar s, may be NULL
  double a0, a1, l, nu;
  double spc;            // shift of the preconditioner (L1 + spc I)^-1
};
#define PW_D 1

// The transform of one dimension of the spectral preconditioners (bk_precond.cu line_setup / line_free)
struct Line {
  int n = 0;
  int type = 0;               // 0: DCT-II (Neumann), 1: DST-I (Dirichlet)
  double* lam = nullptr;      // 1-D eigenvalues of the Laplacian factor (natural order)
  // register-resident power-of-two kernels (bk_fft_fast.cuh): log2(n) or 0, and their tables
  int fast = 0;
  double2* ftw = nullptr;     // per-pass contiguous FFT twiddles
  double2* fom = nullptr;     // w_k = exp(-i pi k / 2n), register-major
  double2* flam2 = nullptr;   // (lambda[k], lambda[n-k]), register-major
  // general lengths (bk_fft_gen.cuh): the plan points at gwl / gph
  bkg::Plan plan = {};
  double2* gwl = nullptr;
  double2* gph = nullptr;
};

struct Precond {
  int kind = BK_PC_NONE;
  double a0 = 0, a1 = 0;
  Line line[3];
  double* work = nullptr;                           // scratch vector (N)
  double* work2 = nullptr;
  // chan tridiagonal LU factors
  double* tri = nullptr;
  // potrap circulant preconditioner
  double2* tdft = nullptr;   // exp(-2 pi i j / (M-1))
  double po_r = 0, po_nu = 0, po_T = 0;
  // BK_PC_RD: the diffusion coefficients at the params of the set-up
  double rd_diff[BK_RD_MAX_FIELDS] = {};
};

// What the host code needs to know about a problem kind.  N0 = fields * dims[0] * ... * dims[ndims - 1] + extra.
struct BkKindTraits {
  int ndims;        // grid dimensions that multiply into N0
  int fields;       // values per grid point
  int extra;        // unknowns behind the grid (the Trapeze period)
  bool jac_sym;     // J symmetric: the eigensolver runs its thick-restart branch
  bool has_jt;      // J' available (bk_jac_set_transpose)
  bool complex_ok;  // BK_COMPLEX allowed
  bool pow2_grid;   // Nx and Ny must be powers of two from 64 to 2048
  bool has_jets;    // d2F / d3F available (bk_d2f, bk_d3f)
};
const BkKindTraits* bk_kind_traits(int kind);  // nullptr for an unknown kind and for BK_RD, whose traits depend on its model

// BK_RD: the model's terms with their parameter monomials evaluated at one parameter tuple (bk_set_params), passed by value to
// the RD kernels (bk_problems.cu).  alpha packs the field exponents of a term, 3 bits per field.
struct RdTable {
  int nterms;
  int bc;  // BK_BC_*
  double diff[BK_RD_MAX_FIELDS];
  double coef[BK_RD_MAX_TERMS];
  int eq[BK_RD_MAX_TERMS];
  int alpha[BK_RD_MAX_TERMS];
};
static_assert(BK_RD_MAX_PAR == BK_MAX_PAR, "an RD model reads the context's parameter tuple");

// CUDA event pairs bracketing intervals on a stream, created on first use and reused from one harvest to the next.
struct BkEventTimer {
  std::vector<std::pair<cudaEvent_t, cudaEvent_t>> pairs;
  size_t used = 0;  // pairs begun since the last harvest
  void begin(cudaStream_t st) {
    if (used == pairs.size()) {
      cudaEvent_t a, b;
      cudaEventCreate(&a);
      cudaEventCreate(&b);
      pairs.push_back({a, b});
    }
    cudaEventRecord(pairs[used++].first, st);
  }
  void end(cudaStream_t st) { cudaEventRecord(pairs[used - 1].second, st); }
  // adds the milliseconds of every pair begun since the last harvest to ms and returns how many there were; the stream must
  // be idle.  A pair whose end was never recorded has no time and is not counted.
  long long harvest(double& ms) {
    long long k = 0;
    for (size_t i = 0; i < used; ++i) {
      float t = 0;
      if (cudaEventElapsedTime(&t, pairs[i].first, pairs[i].second) == cudaSuccess) {
        ms += t;
        ++k;
      }
    }
    used = 0;
    return k;
  }
  void destroy() {
    for (auto& p : pairs) {
      cudaEventDestroy(p.first);
      cudaEventDestroy(p.second);
    }
    pairs.clear();
    used = 0;
  }
};

struct bk_ctx {
  int device = 0;
  int nsm = BK_NSM_FALLBACK;
  long long l2_bytes = 0;     // L2 cache size of the device (plan2: how many basis vectors a ring pass keeps in L2)
  cudaStream_t stream = nullptr;
  int kind = 0;
  BkKindTraits kt = {};   // the kind's traits (bk_traits); BK_RD: from its model
  long long dims[3] = {1, 1, 1};
  double lengths[3] = {1, 1, 1};
  double par[BK_MAX_PAR] = {0};  // written only by bk_store_params
  long long N = 0;        // unknowns (BK_COMPLEX: 2 N0)
  long long N0 = 0;       // size of the real problem: length of the state u and of F(u)
  bool cplx = false;      // BK_COMPLEX context
  double shift_imag = 0;  // imaginary part of a0 (bk_jac_set_shift_imag)
  bool transpose = false; // bk_jac_set_transpose
  int m = 0;              // Krylov dimension capacity (basis holds m+1 vectors of length N+1)
  long long ld = 0;       // leading dimension of the basis (>= N+1, multiple of 32)
  // Jacobian state
  double* u_state = nullptr;
  double jpar[BK_MAX_PAR] = {0};
  bool have_state = false;
  // BK_RD: the model (its terms copied) and its table at par (residual, jets) and at jpar (the Jacobian)
  bk_rd_model rd_model = {};
  std::vector<bk_rd_term> rd_terms;
  RdTable rd_par = {}, rd_jpar = {};
  // potrap
  double* phi = nullptr;
  double* xpi = nullptr;
  double* fcache = nullptr;
  double phi_dot_xpi = 0;
  // Krylov workspace
  double* V = nullptr;        // (m+1) x ld, unnormalised basis vectors v'_i
  double* w = nullptr;        // ld
  double* z = nullptr;        // ld  (preconditioned vector)
  double* r = nullptr;        // ld
  double* scales = nullptr;   // m+2 : s_i = 1/||v'_i||
  double* gcoef = nullptr;    // m+2 : g_i = h_i * s_i (device), also lincomb coefficients
  double* hcols = nullptr;    // (m+1) x (m+4) device H columns
  double* hcols2 = nullptr;   // second-pass (CGS2) corrections
  double* h_pinned = nullptr; // pinned host mirror of hcols (+ hcols2 behind it)
  double* partials = nullptr; // (m+4) x Gmax
  int gmax = 0;
  unsigned int* counters = nullptr; // last-block tickets
  double* red_out = nullptr;  // small device buffer for scalar reductions (16 doubles)
  double* red_pinned = nullptr;
  double* coef_pinned = nullptr; // m+2
  std::vector<cudaEvent_t> events;
  // staging buffers for host-pointer arguments
  std::vector<double*> stage;  // each ld doubles
  double* host_pinned = nullptr; // pinned bounce buffer (ld doubles) for pageable host memory
  // generic temporaries for BLS/eigs
  std::vector<double*> tmp;
  // bk_jet_moments and bk_deflation_moments, lazily allocated and grown: staged host vectors (one row each), the tuples /
  // results / partials, and the pinned landing buffer of the results (BK_JET_MOMENTS_MAX_TUPLES doubles)
  double* mom_stage = nullptr;
  size_t mom_stage_cap = 0;  // bytes
  void* mom_work = nullptr;
  size_t mom_work_cap = 0;   // bytes
  double* mom_pinned = nullptr;
  // bk_vec_alloc pool: live allocations (ptr -> padded length) and the recycled free list
  std::unordered_map<double*, size_t> vec_live;
  std::vector<std::pair<size_t, double*>> vec_pool;
  // eigensolver workspace (lazily allocated)
  double* Q = nullptr;       // (qcap+1) x ld Arnoldi basis of the shift-invert operator
  double* Q2 = nullptr;      // second basis buffer for thick restarts
  int q2cap = 0;
  int qcap = 0;
  double* eig_dev = nullptr; // ones (qcap+2) | hcolA (qcap+2) | hcolB (qcap+2) | g (qcap+2) | coef (2*(qcap+2))
  double* eig_pinned = nullptr;
  Precond pc;
  bk_stats stats = {};
  bool timing = false;      // bk_set_timing: event pairs around the fused kernels / preconditioner applications
  int timing_every = 1;     // ... of every timing_every-th bk_gmres call only (event records sit between PDL launches: sampling keeps the overhead small)
  long long solve_count = 0;
  bool timing_now = false;  // decided per solve
  BkEventTimer fused_timer; // the Arnoldi kernels of one solve (bk_gmres_dev)
  BkEventTimer pc_timer;    // one pair per preconditioner application, read back at the end of a solve and in bk_get_stats
  // dynamic shared memory this context has already asked for, per kernel (first-level filter in front of bk_grant_smem)
  std::unordered_map<const void*, size_t> smem_attr;
  std::string err;
};

// ---- error helpers ---------------------------------------------------------------------------
int bk_fail(bk_ctx* c, int code, const char* what, const char* file, int line);
#define BK_CUDA(c, expr)                                                             \
  do {                                                                               \
    cudaError_t _e = (expr);                                                         \
    if (_e != cudaSuccess) return bk_fail((c), BK_ERR_CUDA, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)
#define BK_CHECK(c, cond, msg)                                                       \
  do {                                                                               \
    if (!(cond)) return bk_fail((c), BK_ERR_ARG, (msg), __FILE__, __LINE__);         \
  } while (0)
// first statement of every extern "C" entry point: a process may hold contexts on several GPUs (Context(device=...)),
// and kernel launches / cudaFuncSetAttribute / cudaMalloc all act on the CURRENT device
#define BK_ENTER(c)                                 \
  do {                                              \
    if (!(c)) return BK_ERR_ARG;                    \
    if (cudaSetDevice((c)->device) != cudaSuccess)  \
      return bk_fail((c), BK_ERR_CUDA, "cudaSetDevice failed", __FILE__, __LINE__); \
  } while (0)
#define BK_TRY(expr)                 \
  do {                               \
    int _s = (expr);                 \
    if (_s < 0) return _s;           \
  } while (0)

// ---- host-side internal API (cross-TU) ----------------------------------------------------------
static inline const BkKindTraits* bk_traits(const bk_ctx* c) { return &c->kt; }
// the one writer of c->par: sets its first n entries and what is derived from them (the BK_RD table rd_par)
void bk_store_params(bk_ctx* c, const double* p, int n);
// Grid of the 256-thread grid-stride kernels: one CTA per 256 values, at most 8 per SM.
static inline int bk_lin_grid(const bk_ctx* c, long long n) {
  long long g = (n + 255) / 256;
  long long cap = (long long)c->nsm * 8;
  return (int)(g < cap ? (g > 0 ? g : 1) : cap);
}
// Grid of the bk_grid_reduce kernels (k_reduce, k_tail, k_potrap_phase): bk_lin_grid, at most one CTA per partial-sum column.
// It fixes the summation order of every such reduction, and with it the rounding of the continuation (DESIGN.md §7).
static inline int bk_reduce_grid(const bk_ctx* c, long long n) {
  const int g = bk_lin_grid(c, n);
  return g < c->gmax ? g : c->gmax;
}
// 1/h^2 along dimension d, with h = 2 l / n in every example (SH2d-fronts.jl:14-15, SH3d.jl:18-20, cGL2d.jl:7-8)
static inline double bk_inv_h2(const bk_ctx* c, int d) {
  const double h = 2 * c->lengths[d] / c->dims[d];
  return 1.0 / (h * h);
}

bool bk_is_device_ptr(const void* p);
// Returns a device pointer for argument p (n doubles): p itself when device memory, else stage slot `slot`
// filled by H2D (when `in`).  For outputs call bk_stage_out afterwards.
int bk_stage_in(bk_ctx* c, const double* p, long long n, int slot, bool copy_in, double** dev);
int bk_stage_out(bk_ctx* c, double* p, long long n, const double* dev);

OpDesc bk_make_op(bk_ctx* c, double a0, double a1);
OpDesc bk_make_residual_op(bk_ctx* c);
int bk_launch_residual(bk_ctx* c, const double* u_dev, double* out_dev);
// out = a0*in*in_scale + a1*J*(in*in_scale) [+ bordered terms]; in_scale_ptr (device, may be NULL => 1)
int bk_launch_apply(bk_ctx* c, const OpDesc& op, const double* in_dev, const double* in_scale_ptr, double* out_dev);
int bk_potrap_refresh_cache(bk_ctx* c);

int bk_precond_apply_dev(bk_ctx* c, const double* in_dev, double* out_dev, long long n);
void line_free(Line& ln);

// BK_SH2D_PERIODIC (bk_precond.cu): transform tables and work buffers at bk_ctx_create, then the three-kernel spectral pipeline
// x r2c -> y (forward, symbol, inverse) -> x c2r for the residual, the JVP and the one-transform preconditioned operator
int bk_periodic_setup(bk_ctx* c);
int bk_periodic_residual(bk_ctx* c, const OpDesc& op, const double* u, double* out);
int bk_periodic_jvp(bk_ctx* c, const OpDesc& op, const double* in, const double* sp, double* out);
// left: P (a0 I + a1 J) v, right: (a0 I + a1 J) P v, P = (L1 + pc.a0 I)^-1 (BK_PC_SH_FFT); op unbordered and real
int bk_periodic_fused(bk_ctx* c, const OpDesc& op, const double* in, const double* sp, double* out, bool left);

// vector kernels (device pointers)
int bk_dev_axpby(bk_ctx* c, double* y, double a, const double* x, double b, long long n);
int bk_dev_scale(bk_ctx* c, double* x, double a, long long n);
int bk_dev_dot(bk_ctx* c, const double* x, const double* y, long long n, double* out_host);
int bk_dev_norminf(bk_ctx* c, const double* x, long long n, double* out_host);
int bk_dev_copy(bk_ctx* c, double* dst, const double* src, long long n);

// GMRES on device pointers; n = op.N (+1 if bordered)
int bk_gmres_dev(bk_ctx* c, const OpDesc& op, const double* rhs_dev, double* x_dev, const bk_gmres_opts* o,
                 int* converged, int* iters, double* resnorm);
// Arnoldi building blocks (used by the eigensolver): dots h_i = s_i <B_i, w> (also g_i = h_i s_i), update
// vout = w - sum g_i B_i with its norm -> *h_out, 1/norm -> *scale_out, and x = beta x + sum coef_i s_i B_i.
int bk_launch_dots(bk_ctx* c, const double* basis, const double* scales, const double* w, long long n, int j, double* hcol,
                   double* gcoef);
int bk_launch_update(bk_ctx* c, const double* basis, const double* gcoef, const double* w, long long n, int j, double* vout,
                     double* h_out, double* scale_out);
int bk_launch_lincomb(bk_ctx* c, const double* basis, const double* scales, double* x, double beta, long long n, int k,
                      const double* coef_dev);
int bk_tmp(bk_ctx* c, int slot, double** out);  // lazily allocated ld-sized temporaries

// grant `bytes` of dynamic shared memory to `kern` on the context's device.  cudaFuncAttributeMaxDynamicSharedMemorySize is a
// property of (device, kernel), shared by every context of the process: the grant only ever grows (bk_grant_smem keeps the
// process-wide maximum under a mutex -- a context with a smaller Krylov dimension must not shrink what another one needs),
// and the per-context map is just a lock-free first-level filter.
void bk_grant_smem(int device, const void* kern, size_t bytes);
template <typename K>
static inline void bk_ensure_smem(bk_ctx* c, K kern, size_t bytes) {
  size_t& cur = c->smem_attr[(const void*)kern];
  if (bytes > cur) {
    bk_grant_smem(c->device, (const void*)kern, bytes);
    cur = bytes;
  }
}

// ---- kernel launches on the context's stream ------------------------------------------------------------------------
#ifdef __CUDACC__
// launch kern on stream st.  With pdl (programmatic dependent launch) the kernel is launched while the previous one drains.
template <typename... KArgs, typename... Args>
static inline cudaError_t bk_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                                        Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  // BK_NO_PDL=1: plain stream order (diagnostics); read once, by whichever thread launches first (a static local's
  // initialisation is thread-safe, so contexts driven from several host threads do not race on it)
  static const int no_pdl = getenv("BK_NO_PDL") ? 1 : 0;
  cfg.numAttrs = pdl && !no_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, KArgs(args)...);
}
// grant `smem` bytes of dynamic shared memory to kern, launch it on the context's stream, check and count the launch
template <typename... KArgs, typename... Args>
static inline int bk_launch_ex(bk_ctx* c, bool pdl, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem,
                               Args&&... args) {
  if (smem) bk_ensure_smem(c, kern, smem);
  bk_launch_pdl(kern, grid, block, smem, c->stream, pdl, static_cast<Args&&>(args)...);
  BK_CUDA(c, cudaGetLastError());
  c->stats.kernel_launches++;
  return BK_OK;
}
// PDL launch: kern must begin with bk_pdl_sync
template <typename... KArgs, typename... Args>
static inline int bk_launch(bk_ctx* c, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, Args&&... args) {
  return bk_launch_ex(c, true, kern, grid, block, smem, static_cast<Args&&>(args)...);
}
// stream-ordered launch: kern starts once the previous kernel of the stream has finished
template <typename... KArgs, typename... Args>
static inline int bk_launch_ordered(bk_ctx* c, void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, Args&&... args) {
  return bk_launch_ex(c, false, kern, grid, block, smem, static_cast<Args&&>(args)...);
}
// first statement of every kernel launched through bk_launch: wait for the previous grid's memory, then let the next
// grid start launching (its CTAs block at their own wait)
__device__ __forceinline__ void bk_pdl_sync() {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
#endif

// ---- device helpers ---------------------------------------------------------------------------
#ifdef __CUDACC__
__device__ __forceinline__ double bk_warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// NaN-propagating max: fmax() drops NaN, which would turn an all-NaN residual into norminf = 0 ("converged").
// norm(x, Inf) of the reference returns NaN there and the step is rejected (src/continuation/Palc.jl:228-231).
__device__ __forceinline__ double bk_nanmax(double a, double b) { return (a != a) ? a : ((b != b) ? b : fmax(a, b)); }
__device__ __forceinline__ double bk_warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = bk_nanmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Grid-wide "last block done" ticket.  Returns true in exactly one block (the last to arrive),
// after all other blocks' prior global writes are visible.  Resets the counter for the next launch.
__device__ __forceinline__ bool bk_last_block(unsigned int* counter, int* s_flag) {
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned int t = atomicAdd(counter, 1u);
    int last = (t == gridDim.x * gridDim.y * gridDim.z - 1);
    if (last) *counter = 0u;
    *s_flag = last;
  }
  __syncthreads();
  bool last = (*s_flag != 0);
  if (last) __threadfence();
  return last;
}
template <bool MAX>
__device__ __forceinline__ double bk_red(double a, double b) { return MAX ? bk_nanmax(a, b) : a + b; }
// Deterministic two-level reduction of K <= 2 values per thread over a grid of 256-thread CTAs: sums, or bk_nanmax (MAX).
// Each CTA reduces its warps by shuffles, then folds the 8 warp results in order, starting from 0.0, into the partial
// partials[k * gridDim.x + blockIdx.x]; the last CTA to arrive folds the gridDim.x partials the same way.  Returns true in
// thread 0 of that CTA only, with the grid totals in v.  The order depends on the grid alone (bk_reduce_grid).
template <int K, bool MAX = false>
__device__ __forceinline__ bool bk_grid_reduce(double (&v)[K], double* __restrict__ partials, unsigned int* counter) {
  __shared__ double s_w[K][8];
  __shared__ int s_flag;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const double t = MAX ? bk_warp_max(v[k]) : bk_warp_sum(v[k]);
    if (lane == 0) s_w[k][wid] = t;
  }
  __syncthreads();
  if (threadIdx.x < K) {
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t = bk_red<MAX>(t, s_w[threadIdx.x][w]);
    partials[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = t;
  }
  if (!bk_last_block(counter, &s_flag)) return false;
  double t[K];
#pragma unroll
  for (int k = 0; k < K; ++k) t[k] = 0.0;
  for (int i = threadIdx.x; i < (int)gridDim.x; i += blockDim.x)
#pragma unroll
    for (int k = 0; k < K; ++k) t[k] = bk_red<MAX>(t[k], __ldcg(partials + (size_t)k * gridDim.x + i));
#pragma unroll
  for (int k = 0; k < K; ++k) {
    t[k] = MAX ? bk_warp_max(t[k]) : bk_warp_sum(t[k]);
    if (lane == 0) s_w[k][wid] = t[k];
  }
  __syncthreads();
  if (threadIdx.x != 0) return false;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    v[k] = 0.0;
    for (int w = 0; w < 8; ++w) v[k] = bk_red<MAX>(v[k], s_w[k][w]);
  }
  return true;
}
#endif
