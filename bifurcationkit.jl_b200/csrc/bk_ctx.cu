// bk_ctx.cu -- context life cycle, host<->device staging and the S11 vector algebra kernels
// (BorderedArray / VectorInterface methods of src/BorderedArrays.jl:30-35,53-70,79-217 for a
// device-resident state vector).
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <mutex>
#include <new>
#include "bk_common.cuh"

int bk_fail(bk_ctx* c, int code, const char* what, const char* file, int line) {
  if (c) {
    char buf[512];
    snprintf(buf, sizeof buf, "%s (%s:%d)", what, file, line);
    c->err = buf;
  }
  return code;
}

void bk_grant_smem(int device, const void* kern, size_t bytes) {
  static std::mutex mu;
  static std::map<std::pair<int, const void*>, size_t> granted;  // (device, kernel) -> largest size set so far
  std::lock_guard<std::mutex> lk(mu);
  size_t& cur = granted[{device, kern}];
  if (bytes <= cur) return;
  cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (bytes > 48 * 1024) cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
  cur = bytes;
}

bool bk_is_device_ptr(const void* p) {
  cudaPointerAttributes at;
  cudaError_t e = cudaPointerGetAttributes(&at, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

int bk_stage_in(bk_ctx* c, const double* p, long long n, int slot, bool copy_in, double** dev) {
  BK_CHECK(c, p != nullptr, "null vector argument");
  if (bk_is_device_ptr(p)) {
    *dev = const_cast<double*>(p);
    return BK_OK;
  }
  BK_CHECK(c, slot >= 0 && slot < 16, "bad stage slot");
  if ((int)c->stage.size() <= slot) c->stage.resize(slot + 1, nullptr);
  if (!c->stage[slot]) BK_CUDA(c, cudaMalloc(&c->stage[slot], sizeof(double) * (size_t)c->ld));
  BK_CHECK(c, n <= c->ld, "vector longer than the context's leading dimension");
  if (copy_in) {
    BK_CUDA(c, cudaMemcpyAsync(c->stage[slot], p, sizeof(double) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
    c->stats.h2d_bytes += 8 * n;
  }
  *dev = c->stage[slot];
  return BK_OK;
}

int bk_stage_out(bk_ctx* c, double* p, long long n, const double* dev) {
  if (p == dev) return BK_OK;
  BK_CUDA(c, cudaMemcpyAsync(p, dev, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  c->stats.d2h_bytes += 8 * n;
  return BK_OK;
}

int bk_tmp(bk_ctx* c, int slot, double** out) {
  if ((int)c->tmp.size() <= slot) c->tmp.resize(slot + 1, nullptr);
  if (!c->tmp[slot]) BK_CUDA(c, cudaMalloc(&c->tmp[slot], sizeof(double) * (size_t)c->ld));
  *out = c->tmp[slot];
  return BK_OK;
}

const BkKindTraits* bk_kind_traits(int kind) {
  //                                   ndims fields extra jac_sym has_jt complex_ok pow2_grid has_jets
  static const BkKindTraits table[] = {{0, 0, 0, false, false, false, false, false},  // 0: not a kind
                                       {1, 1, 0, false, false, true, false, true},     // BK_CHAN
                                       {2, 1, 0, true, true, true, false, true},       // BK_SH2D
                                       {3, 1, 0, true, true, true, false, true},       // BK_SH3D
                                       {2, 2, 0, false, true, true, false, true},      // BK_CGL2D
                                       {3, 2, 1, false, true, false, false, false},    // BK_POTRAP_CGL2D
                                       {2, 1, 0, true, true, true, true, true}};       // BK_SH2D_PERIODIC
  static_assert(BK_CHAN == 1 && BK_POTRAP_CGL2D == 5 && BK_SH2D_PERIODIC == 6, "the table is indexed by kind");
  if (kind < BK_CHAN || kind > BK_SH2D_PERIODIC) return nullptr;
  return &table[kind];
}

// The checks of an RD model (bk200.h), all before any device work
static int rd_validate(bk_ctx* c, const bk_rd_model* m) {
  BK_CHECK(c, m != nullptr, "bk_rd_ctx_create: null model");
  BK_CHECK(c, m->fields >= 1 && m->fields <= BK_RD_MAX_FIELDS, "BK_RD: fields must be 1 .. 4");
  BK_CHECK(c, m->ndims == 1 || m->ndims == 2, "BK_RD: ndims must be 1 or 2");
  BK_CHECK(c, m->bc == BK_BC_NEUMANN || m->bc == BK_BC_DIRICHLET, "BK_RD: bc must be BK_BC_NEUMANN or BK_BC_DIRICHLET");
  BK_CHECK(c, m->nparams >= 0 && m->nparams <= BK_RD_MAX_PAR, "BK_RD: nparams must be 0 .. 8");
  BK_CHECK(c, m->flags == 0 || m->flags == BK_COMPLEX, "BK_RD: flags must be 0 or BK_COMPLEX");
  BK_CHECK(c, m->nterms >= 0 && m->nterms <= BK_RD_MAX_TERMS, "BK_RD: nterms must be 0 .. 64");
  BK_CHECK(c, m->nterms == 0 || m->terms != nullptr, "BK_RD: null term list");
  auto pexp_ok = [&](const int32_t* e) {
    for (int k = 0; k < BK_RD_MAX_PAR; ++k) {
      if (e[k] < -BK_RD_MAX_PEXP || e[k] > BK_RD_MAX_PEXP) return 1;
      if (k >= m->nparams && e[k] != 0) return 2;
    }
    return 0;
  };
  for (int i = 0; i < m->fields; ++i) {
    const int e = pexp_ok(m->diff_pexp[i]);
    BK_CHECK(c, e != 1, "BK_RD: a diffusion parameter exponent is outside [-4, 4]");
    BK_CHECK(c, e != 2, "BK_RD: a diffusion coefficient reads a parameter index >= nparams");
    BK_CHECK(c, std::isfinite(m->diff_scale[i]), "BK_RD: a diffusion scale is not finite");
  }
  for (int t = 0; t < m->nterms; ++t) {
    const bk_rd_term& tm = m->terms[t];
    BK_CHECK(c, tm.eq >= 0 && tm.eq < m->fields, "BK_RD: a term's equation index is outside [0, fields)");
    BK_CHECK(c, std::isfinite(tm.scale), "BK_RD: a term's scale is not finite");
    const int e = pexp_ok(tm.pexp);
    BK_CHECK(c, e != 1, "BK_RD: a term's parameter exponent is outside [-4, 4]");
    BK_CHECK(c, e != 2, "BK_RD: a term reads a parameter index >= nparams");
    int deg = 0;
    for (int j = 0; j < BK_RD_MAX_FIELDS; ++j) {
      BK_CHECK(c, tm.fexp[j] >= 0 && tm.fexp[j] <= BK_RD_MAX_DEGREE, "BK_RD: a term's field exponent is outside [0, 5]");
      BK_CHECK(c, j < m->fields || tm.fexp[j] == 0, "BK_RD: a term has an exponent on a field index >= fields");
      deg += tm.fexp[j];
    }
    BK_CHECK(c, deg <= BK_RD_MAX_DEGREE, "BK_RD: a term's degree |alpha| is above 5");
  }
  return BK_OK;
}

// The RD table at the parameter tuple p: every parameter monomial evaluated, the field exponents packed 3 bits per field
static void rd_eval(const bk_ctx* c, const double* p, RdTable* t) {
  const bk_rd_model& m = c->rd_model;
  auto mono = [&](double s, const int32_t* e) {
    for (int k = 0; k < m.nparams; ++k) {
      for (int r = 0; r < e[k]; ++r) s *= p[k];
      for (int r = 0; r < -e[k]; ++r) s /= p[k];
    }
    return s;
  };
  *t = RdTable{};
  t->nterms = m.nterms;
  t->bc = m.bc;
  for (int i = 0; i < m.fields; ++i) t->diff[i] = mono(m.diff_scale[i], m.diff_pexp[i]);
  for (int k = 0; k < m.nterms; ++k) {
    const bk_rd_term& tm = c->rd_terms[k];
    t->coef[k] = mono(tm.scale, tm.pexp);
    t->eq[k] = tm.eq;
    int a = 0;
    for (int j = 0; j < m.fields; ++j) a |= tm.fexp[j] << (3 * j);
    t->alpha[k] = a;
  }
}

static int ctx_create(int32_t device, int32_t kind, const bk_rd_model* model, const int64_t dims[3], const double lengths[3],
                      int32_t krylov_m, bk_ctx** out) {
  if (!out) return BK_ERR_ARG;
  *out = nullptr;
  bk_ctx* c = new (std::nothrow) bk_ctx();
  if (!c) return BK_ERR_ARG;
  *out = c;  // returned even on failure so the caller can read bk_last_error
  c->device = device;
  c->cplx = (kind & BK_COMPLEX) != 0;
  kind &= ~BK_COMPLEX;
  c->kind = kind;
  for (int i = 0; i < 3; ++i) {
    c->dims[i] = dims ? (dims[i] > 0 ? dims[i] : 1) : 1;
    c->lengths[i] = lengths ? lengths[i] : 1.0;
  }
  if (kind == BK_RD) {
    BK_CHECK(c, model != nullptr, "BK_RD contexts are created by bk_rd_ctx_create (the model describes the problem)");
    BK_TRY(rd_validate(c, model));
    c->rd_model = *model;
    c->rd_terms.assign(model->terms, model->terms + model->nterms);
    c->rd_model.terms = c->rd_terms.data();
    for (int d = model->ndims; d < 3; ++d)
      BK_CHECK(c, c->dims[d] == 1, "BK_RD: dims has more grid dimensions than the model's ndims");
    //          ndims          fields         extra jac_sym              has_jt complex_ok pow2_grid has_jets
    c->kt = {model->ndims, model->fields, 0, model->fields == 1, true, true, false, true};
    rd_eval(c, c->par, &c->rd_par);
    c->rd_jpar = c->rd_par;
  } else {
    const BkKindTraits* kt = bk_kind_traits(kind);
    if (!kt) return bk_fail(c, BK_ERR_ARG, "unknown problem kind", __FILE__, __LINE__);
    c->kt = *kt;
  }
  const BkKindTraits* kt = &c->kt;
  if (kt->pow2_grid)
    for (int d = 0; d < 2; ++d) {
      const long long v = c->dims[d];
      BK_CHECK(c, v >= 64 && v <= 2048 && (v & (v - 1)) == 0,
               "BK_SH2D_PERIODIC: Nx and Ny must be powers of two from 64 to 2048");
    }
  long long n = kt->fields;
  for (int d = 0; d < kt->ndims; ++d) n *= c->dims[d];
  n += kt->extra;
  BK_CHECK(c, n >= 2, "problem too small");
  BK_CHECK(c, krylov_m >= 1 && krylov_m <= 1024, "krylov_m out of range");
  BK_CHECK(c, !c->cplx || kt->complex_ok, "BK_COMPLEX is not available for the periodic-orbit functional");
  c->N0 = n;
  if (c->cplx) n *= 2;  // [re; im]
  c->N = n;
  c->m = krylov_m;
  c->ld = ((n + 2 + 31) / 32) * 32;  // >= N + 2: bordered vectors (N+1) keep one zero pad element for even-sized TMA rows
  BK_CUDA(c, cudaSetDevice(device));
  cudaDeviceProp prop;
  BK_CUDA(c, cudaGetDeviceProperties(&prop, device));
  c->nsm = prop.multiProcessorCount;
  c->l2_bytes = prop.l2CacheSize;
  if (const char* e = getenv("BK_NSM")) {  // diagnostics: size grids and reductions as for a device with BK_NSM SMs
    const int v = atoi(e);
    if (v >= 1 && v <= 1024) c->nsm = v;
  }
  BK_CUDA(c, cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
  size_t ld = (size_t)c->ld, m = (size_t)c->m;
  BK_CUDA(c, cudaMalloc(&c->u_state, 8 * ld));
  BK_CUDA(c, cudaMalloc(&c->V, 8 * ld * (m + 1)));
  BK_CUDA(c, cudaMalloc(&c->w, 8 * ld));
  BK_CUDA(c, cudaMalloc(&c->z, 8 * ld));
  BK_CUDA(c, cudaMalloc(&c->r, 8 * ld));
  BK_CUDA(c, cudaMemset(c->u_state, 0, 8 * ld));
  BK_CUDA(c, cudaMemset(c->V, 0, 8 * ld * (m + 1)));
  BK_CUDA(c, cudaMemset(c->w, 0, 8 * ld));
  BK_CUDA(c, cudaMemset(c->z, 0, 8 * ld));
  BK_CUDA(c, cudaMemset(c->r, 0, 8 * ld));
  BK_CUDA(c, cudaMalloc(&c->scales, 8 * (m + 4)));
  BK_CUDA(c, cudaMalloc(&c->gcoef, 8 * (m + 4)));
  BK_CUDA(c, cudaMalloc(&c->hcols, 8 * (m + 1) * (m + 4)));
  BK_CUDA(c, cudaMalloc(&c->hcols2, 8 * (m + 1) * (m + 4)));
  BK_CUDA(c, cudaMemset(c->hcols, 0, 8 * (m + 1) * (m + 4)));
  BK_CUDA(c, cudaMemset(c->hcols2, 0, 8 * (m + 1) * (m + 4)));
  BK_CUDA(c, cudaMallocHost(&c->h_pinned, 2 * 8 * (m + 1) * (m + 4)));
  // number of partial-sum columns: one per CTA of the widest reduction grid
  long long g = (n + 2 + 255) / 256 + 8;  // worst case: one CTA per 256 values
  if (kind == BK_SH2D) {
    // the fused 2-D kernel tiles rows, not the flat vector: a narrow grid (nx << 256) has up to ceil(nx/256) * ny CTAs
    long long gf = ((c->dims[0] + 255) / 256) * c->dims[1] + 8;
    if (gf > g) g = gf;
  }
  if (g < 4 * c->nsm) g = 4 * c->nsm;
  c->gmax = (int)g;
  BK_CUDA(c, cudaMalloc(&c->partials, 8 * (m + 4) * (size_t)c->gmax));
  BK_CUDA(c, cudaMalloc(&c->counters, 64 * sizeof(unsigned int)));
  BK_CUDA(c, cudaMemset(c->counters, 0, 64 * sizeof(unsigned int)));
  BK_CUDA(c, cudaMalloc(&c->red_out, 8 * 16));
  BK_CUDA(c, cudaMallocHost(&c->red_pinned, 8 * 16));
  BK_CUDA(c, cudaMallocHost(&c->coef_pinned, 8 * (m + 4)));
  c->events.resize(m + 2);
  for (auto& e : c->events) BK_CUDA(c, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
  if (kind == BK_POTRAP_CGL2D) {
    BK_CUDA(c, cudaMalloc(&c->phi, 8 * ld));
    BK_CUDA(c, cudaMalloc(&c->xpi, 8 * ld));
    BK_CUDA(c, cudaMalloc(&c->fcache, 8 * ld));
    BK_CUDA(c, cudaMemset(c->phi, 0, 8 * ld));
    BK_CUDA(c, cudaMemset(c->xpi, 0, 8 * ld));
  }
  if (kind == BK_SH2D_PERIODIC) BK_TRY(bk_periodic_setup(c));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  return BK_OK;
}

extern "C" int32_t bk_ctx_create(int32_t device, int32_t kind, const int64_t dims[3], const double lengths[3],
                                 int32_t krylov_m, bk_ctx** out) {
  return ctx_create(device, kind, nullptr, dims, lengths, krylov_m, out);
}

extern "C" int32_t bk_rd_ctx_create(int32_t device, const bk_rd_model* model, const int64_t dims[3], const double lengths[3],
                                    int32_t krylov_m, bk_ctx** out) {
  return ctx_create(device, BK_RD | (model ? model->flags : 0), model, dims, lengths, krylov_m, out);
}

extern "C" int32_t bk_ctx_destroy(bk_ctx* c) {
  if (!c) return BK_OK;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  double* bufs[] = {c->u_state, c->V, c->w, c->z, c->r, c->scales, c->gcoef, c->hcols, c->hcols2, c->partials,
                    c->red_out, c->phi, c->xpi, c->fcache, c->pc.work, c->pc.work2, c->pc.tri, c->Q, c->Q2, c->eig_dev};
  for (double* b : bufs)
    if (b) cudaFree(b);
  for (Line& ln : c->pc.line) line_free(ln);
  if (c->pc.tdft) cudaFree(c->pc.tdft);
  if (c->counters) cudaFree(c->counters);
  for (auto& kv : c->vec_live) cudaFree(kv.first);
  for (double* b : c->stage)
    if (b) cudaFree(b);
  for (double* b : c->tmp)
    if (b) cudaFree(b);
  if (c->mom_stage) cudaFree(c->mom_stage);
  if (c->mom_work) cudaFree(c->mom_work);
  if (c->mom_pinned) cudaFreeHost(c->mom_pinned);
  if (c->h_pinned) cudaFreeHost(c->h_pinned);
  if (c->red_pinned) cudaFreeHost(c->red_pinned);
  if (c->coef_pinned) cudaFreeHost(c->coef_pinned);
  if (c->host_pinned) cudaFreeHost(c->host_pinned);
  if (c->eig_pinned) cudaFreeHost(c->eig_pinned);
  for (auto& e : c->events)
    if (e) cudaEventDestroy(e);
  c->fused_timer.destroy();
  c->pc_timer.destroy();
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
  return BK_OK;
}

extern "C" const char* bk_last_error(bk_ctx* c) { return c ? c->err.c_str() : "null context"; }
extern "C" int64_t bk_problem_size(bk_ctx* c) { return c ? c->N : 0; }
extern "C" int64_t bk_state_size(bk_ctx* c) { return c ? c->N0 : 0; }
void bk_store_params(bk_ctx* c, const double* p, int n) {
  for (int i = 0; i < n; ++i) c->par[i] = p[i];
  if (c->kind == BK_RD) rd_eval(c, c->par, &c->rd_par);
}
extern "C" int32_t bk_set_params(bk_ctx* c, const double* p, int32_t n) {
  BK_ENTER(c);
  BK_CHECK(c, p && n >= 0 && n <= BK_MAX_PAR, "bad params");
  BK_CHECK(c, c->kind != BK_RD || n >= c->rd_model.nparams, "BK_RD: bk_set_params needs the model's nparams values");
  bk_store_params(c, p, n);
  return BK_OK;
}
extern "C" int32_t bk_get_stats(bk_ctx* c, bk_stats* out) {
  BK_ENTER(c);
  if (!out) return BK_ERR_ARG;
  if (c->pc_timer.used) {
    BK_CUDA(c, cudaStreamSynchronize(c->stream));
    c->stats.total_precond_applies += c->pc_timer.harvest(c->stats.total_precond_ms);
  }
  *out = c->stats;
  return BK_OK;
}
extern "C" int32_t bk_set_timing(bk_ctx* c, int32_t on) {
  BK_ENTER(c);
  c->timing = on != 0;
  c->timing_every = on > 1 ? on : 1;  // on = k > 1: time every k-th solve
  c->timing_now = c->timing && c->timing_every == 1;
  return BK_OK;
}
extern "C" int32_t bk_sync(bk_ctx* c) {
  BK_ENTER(c);
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  return BK_OK;
}
extern "C" void* bk_stream(bk_ctx* c) { return c ? (void*)c->stream : nullptr; }

// ---- vectors -----------------------------------------------------------------------------------
extern "C" int32_t bk_vec_alloc(bk_ctx* c, int64_t n, double** out) {
  BK_ENTER(c);
  if (!out) return BK_ERR_ARG;
  BK_CHECK(c, n > 0, "bad length");
  BK_CUDA(c, cudaSetDevice(c->device));
  size_t len = ((size_t)n + 31) / 32 * 32;
  // pooled: cudaMalloc/cudaFree synchronise the device and cost far more than a continuation-step kernel;
  // freed vectors are recycled in stream order (every kernel of a context runs on its one stream)
  for (size_t i = 0; i < c->vec_pool.size(); ++i) {
    if (c->vec_pool[i].first == len) {
      *out = c->vec_pool[i].second;
      c->vec_pool[i] = c->vec_pool.back();
      c->vec_pool.pop_back();
      BK_CUDA(c, cudaMemsetAsync(*out, 0, 8 * len, c->stream));
      return BK_OK;
    }
  }
  BK_CUDA(c, cudaMalloc(out, 8 * len));
  c->vec_live[*out] = len;
  BK_CUDA(c, cudaMemsetAsync(*out, 0, 8 * len, c->stream));
  return BK_OK;
}
extern "C" int32_t bk_vec_free(bk_ctx* c, double* v) {
  BK_ENTER(c);
  if (v) {
    auto it = c->vec_live.find(v);
    BK_CHECK(c, it != c->vec_live.end(), "bk_vec_free: pointer was not allocated by bk_vec_alloc of this context");
    c->vec_pool.push_back({it->second, v});
  }
  return BK_OK;
}
// pinned host buffers for option-A callers (host-resident state): H2D/D2H at PCIe speed instead of the
// pageable-memory staging path
extern "C" int32_t bk_host_alloc(bk_ctx* c, int64_t n, double** out) {
  BK_ENTER(c);
  if (!out) return BK_ERR_ARG;
  BK_CHECK(c, n > 0, "bad length");
  BK_CUDA(c, cudaSetDevice(c->device));
  BK_CUDA(c, cudaHostAlloc((void**)out, 8 * (size_t)n, cudaHostAllocDefault));
  return BK_OK;
}
extern "C" int32_t bk_host_free(bk_ctx* c, double* p) {
  BK_ENTER(c);
  if (p) {
    BK_CUDA(c, cudaStreamSynchronize(c->stream));
    BK_CUDA(c, cudaFreeHost(p));
  }
  return BK_OK;
}
extern "C" int32_t bk_vec_upload(bk_ctx* c, double* dst, const double* src, int64_t n) {
  BK_ENTER(c);
  BK_CUDA(c, cudaMemcpyAsync(dst, src, 8 * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  c->stats.h2d_bytes += 8 * n;
  return BK_OK;
}
extern "C" int32_t bk_vec_download(bk_ctx* c, double* dst, const double* src, int64_t n) {
  BK_ENTER(c);
  BK_CUDA(c, cudaMemcpyAsync(dst, src, 8 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  c->stats.d2h_bytes += 8 * n;
  return BK_OK;
}

int bk_dev_copy(bk_ctx* c, double* dst, const double* src, long long n) {
  if (dst == src) return BK_OK;
  BK_CUDA(c, cudaMemcpyAsync(dst, src, 8 * (size_t)n, cudaMemcpyDeviceToDevice, c->stream));
  return BK_OK;
}

static __global__ void __launch_bounds__(256) k_axpby(double* __restrict__ y, double a, const double* __restrict__ x,
                                                      double b, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  if (b == 0.0) {
    for (; i < n; i += stride) y[i] = a * x[i];
  } else {
    for (; i < n; i += stride) y[i] = a * x[i] + b * y[i];
  }
}
static __global__ void __launch_bounds__(256) k_scale(double* __restrict__ x, double a, long long n) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < n; i += stride) x[i] *= a;
}

int bk_dev_axpby(bk_ctx* c, double* y, double a, const double* x, double b, long long n) {
  return bk_launch_ordered(c, k_axpby, bk_lin_grid(c, n), 256, 0, y, a, x, b, n);
}
int bk_dev_scale(bk_ctx* c, double* x, double a, long long n) {
  return bk_launch_ordered(c, k_scale, bk_lin_grid(c, n), 256, 0, x, a, n);
}

// mode 0: sum x*y ; 1: max |x| ; 2: sum (x - x0)*y
template <int MODE>
static __global__ void __launch_bounds__(256) k_reduce(const double* __restrict__ x, const double* __restrict__ y,
                                                       const double* __restrict__ x0, long long n,
                                                       double* __restrict__ partials, unsigned int* counter,
                                                       double* __restrict__ out) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  double acc[1] = {0.0};
  for (; i < n; i += stride) {
    if (MODE == 0) acc[0] = fma(x[i], y[i], acc[0]);
    if (MODE == 1) acc[0] = bk_nanmax(acc[0], fabs(x[i]));
    if (MODE == 2) acc[0] = fma(x[i] - x0[i], y[i], acc[0]);
  }
  if (bk_grid_reduce<1, MODE == 1>(acc, partials, counter)) out[0] = acc[0];
}

template <int MODE>
static int reduce_launch(bk_ctx* c, const double* x, const double* y, const double* x0, long long n, double* out_host) {
  BK_TRY(bk_launch_ordered(c, k_reduce<MODE>, bk_reduce_grid(c, n), 256, 0, x, y, x0, n, c->partials, c->counters + 8,
                           c->red_out));
  BK_CUDA(c, cudaMemcpyAsync(c->red_pinned, c->red_out, 8, cudaMemcpyDeviceToHost, c->stream));
  BK_CUDA(c, cudaStreamSynchronize(c->stream));
  *out_host = c->red_pinned[0];
  return BK_OK;
}
int bk_dev_dot(bk_ctx* c, const double* x, const double* y, long long n, double* out_host) {
  return reduce_launch<0>(c, x, y, nullptr, n, out_host);
}
int bk_dev_norminf(bk_ctx* c, const double* x, long long n, double* out_host) {
  return reduce_launch<1>(c, x, x, nullptr, n, out_host);
}

#define BK_DEVPTR(c, p) BK_CHECK(c, (p) && bk_is_device_ptr(p), "bk_vec_* needs device pointers from bk_vec_alloc")

extern "C" int32_t bk_vec_copy(bk_ctx* c, double* dst, const double* src, int64_t n) {
  BK_ENTER(c);
  BK_DEVPTR(c, dst);
  BK_DEVPTR(c, src);
  return bk_dev_copy(c, dst, src, n);
}
extern "C" int32_t bk_vec_zero(bk_ctx* c, double* x, int64_t n) {
  BK_ENTER(c);
  BK_DEVPTR(c, x);
  BK_CUDA(c, cudaMemsetAsync(x, 0, 8 * (size_t)n, c->stream));
  return BK_OK;
}
extern "C" int32_t bk_vec_scale(bk_ctx* c, double* x, double a, int64_t n) {
  BK_ENTER(c);
  BK_DEVPTR(c, x);
  return bk_dev_scale(c, x, a, n);
}
extern "C" int32_t bk_vec_axpby(bk_ctx* c, double* y, double a, const double* x, double b, int64_t n) {
  BK_ENTER(c);
  BK_DEVPTR(c, y);
  BK_DEVPTR(c, x);
  return bk_dev_axpby(c, y, a, x, b, n);
}
extern "C" int32_t bk_vec_dot(bk_ctx* c, const double* x, const double* y, int64_t n, double* out) {
  BK_ENTER(c);
  if (!out) return BK_ERR_ARG;
  BK_DEVPTR(c, x);
  BK_DEVPTR(c, y);
  return bk_dev_dot(c, x, y, n, out);
}
extern "C" int32_t bk_vec_norm2(bk_ctx* c, const double* x, int64_t n, double* out) {
  BK_ENTER(c);
  if (!out) return BK_ERR_ARG;
  BK_DEVPTR(c, x);
  double d = 0;
  BK_TRY(bk_dev_dot(c, x, x, n, &d));
  *out = sqrt(d);
  return BK_OK;
}
extern "C" int32_t bk_vec_norminf(bk_ctx* c, const double* x, int64_t n, double* out) {
  BK_ENTER(c);
  if (!out) return BK_ERR_ARG;
  BK_DEVPTR(c, x);
  return bk_dev_norminf(c, x, n, out);
}
extern "C" int32_t bk_vec_diffdot(bk_ctx* c, const double* x, const double* x0, const double* tau, int64_t n, double* out) {
  BK_ENTER(c);
  if (!out) return BK_ERR_ARG;
  BK_DEVPTR(c, x);
  BK_DEVPTR(c, x0);
  BK_DEVPTR(c, tau);
  return reduce_launch<2>(c, x, tau, x0, n, out);
}
