// C ABI of libtaiga_b200.so (declared in include/taiga_b200.h).  No exception crosses this boundary.
#include "../../include/taiga_b200.h"
#include "common.cuh"
#include "kernels.cuh"
#include "srs.cuh"
#include "capi_internal.cuh"

using namespace tb;

extern "C" {

const char* tb_version(void) { return "taiga_b200 0.1 (sm_90a)"; }

tb_status tb_ctx_create(int device, tb_ctx** out) {
  if (!out) return TB_ERR_INVALID;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || device < 0 || device >= count) { cudaGetLastError(); return TB_ERR_CUDA; }
  tb_ctx* ctx = new tb_ctx();
  try {
    TB_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    TB_CUDA(cudaGetDeviceProperties(&prop, device));
    // the library holds sm_90a code only, which no other compute capability can run
    if (prop.major != 9 || prop.minor != 0) throw tb::CudaError("libtaiga_b200 requires an sm_90 (H100) device (no fallback path exists)");
    ctx->c.device = device;
    ctx->c.sm_count = prop.multiProcessorCount;
    TB_CUDA(cudaStreamCreateWithFlags(&ctx->c.stream, cudaStreamNonBlocking));
    cudaMemPool_t pool;
    TB_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
    uint64_t thresh = UINT64_MAX;
    TB_CUDA(cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thresh));
    ctx->c.d_msm_adds = DevMem<unsigned long long>(1);
    TB_CUDA(cudaMemset(ctx->c.d_msm_adds.get(), 0, sizeof(unsigned long long)));
    build_twiddles<Fp>(&ctx->c);
    build_twiddles<Fq>(&ctx->c);
  } catch (const std::exception& e) {
    fprintf(stderr, "tb_ctx_create: %s\n", e.what());
    delete ctx; cudaGetLastError();
    return TB_ERR_CUDA;
  }
  *out = ctx;
  return TB_OK;
}

void tb_ctx_destroy(tb_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->c.device);
  delete ctx;
}
const char* tb_last_error(const tb_ctx* ctx) { return ctx ? ctx->c.last_error.c_str() : "null context"; }
tb_status tb_ctx_sync(tb_ctx* ctx) { TB_API_BEGIN(ctx) ctx->c.sync(); TB_API_END(ctx) }
uint64_t tb_ctx_stream(const tb_ctx* ctx) { return ctx ? (uint64_t)(uintptr_t)ctx->c.stream : 0; }
uint64_t tb_ctx_launch_count(const tb_ctx* ctx) { return ctx ? ctx->c.launches : 0; }

static const char* PROF_NAMES[PC_COUNT] = {"ntt", "msm_sort", "msm_accum", "msm_reduce", "quotient_gates", "quotient_finish", "ipa_fold", "transcript",
                                           "lookup_sort", "poly"};
int tb_prof_categories(void) { return PC_COUNT; }
const char* tb_prof_category_name(int i) { return (i >= 0 && i < PC_COUNT) ? PROF_NAMES[i] : ""; }
tb_status tb_prof_enable(tb_ctx* ctx, int on) {
  TB_API_BEGIN(ctx)
  ctx->c.sync();
  for (auto& r : ctx->c.prof_recs) { ctx->c.event_pool.push_back(r.a); ctx->c.event_pool.push_back(r.b); }
  ctx->c.prof_recs.clear();
  ctx->c.prof = on != 0;
  TB_API_END(ctx)
}
tb_status tb_prof_read(tb_ctx* ctx, double* ms_out, uint64_t* counts_out) {
  TB_API_BEGIN(ctx)
  ctx->c.sync();
  for (int i = 0; i < PC_COUNT; ++i) { ms_out[i] = 0; counts_out[i] = 0; }
  for (auto& r : ctx->c.prof_recs) {
    float ms = 0; TB_CUDA(cudaEventElapsedTime(&ms, r.a, r.b));
    ms_out[r.cat] += ms; counts_out[r.cat]++;
    ctx->c.event_pool.push_back(r.a); ctx->c.event_pool.push_back(r.b);
  }
  ctx->c.prof_recs.clear();
  TB_API_END(ctx)
}

// Montgomery multiplications executed per category since the last call (analytic counts per launch; the batched MSM's bucket
// additions are counted on the device and charged 6 multiplications each + the product tree)
tb_status tb_prof_work(tb_ctx* ctx, double* modmuls_out) {
  TB_API_BEGIN(ctx)
  ctx->c.sync();
  unsigned long long adds = 0;
  TB_CUDA(cudaMemcpy(&adds, ctx->c.d_msm_adds.get(), sizeof(adds), cudaMemcpyDeviceToHost));
  TB_CUDA(cudaMemset(ctx->c.d_msm_adds.get(), 0, sizeof(adds)));
  ctx->c.work[PC_MSM_ACCUM] += 6.4 * (double)adds;
  for (int i = 0; i < PC_COUNT; ++i) { modmuls_out[i] = ctx->c.work[i]; ctx->c.work[i] = 0; }
  TB_API_END(ctx)
}

}  // extern "C"

// ---------------------------------------------------------------- NTT
template <class F>
static void dev_ntt(Ctx* c, uint32_t logn, int inverse, int coset, uint32_t batch, const F* in, F* out, F* scratch) {
  NttHook<F> hook; hook.k = 0; hook.mod_bits = TW_LOG; hook.use_const = 0; hook.use_zeta = 1;
  F z = zeta_const<F>();
  if (!inverse) { hook.z1 = z; hook.z2 = z.sqr(); } else { hook.z1 = z.sqr(); hook.z2 = z; }
  long long stride = 1ll << logn;
  ntt_run<F>(c, (int)logn, inverse != 0, in, out, scratch, (int)batch, stride, stride, (coset && !inverse) ? &hook : nullptr,
             (coset && inverse) ? &hook : nullptr);
}

template <class F>
static void host_ntt(Ctx* c, uint32_t logn, int inverse, int coset, uint32_t batch, const uint8_t* in, uint8_t* out) {
  size_t n = (size_t)batch << logn;
  DevBuf<F> a(c, n), b(c, n), s(c, n);
  a.upload(in, n);
  fe_to_mont<F>(c, a.get(), n);
  dev_ntt<F>(c, logn, inverse, coset, batch, a.get(), b.get(), s.get());
  fe_from_mont<F>(c, b.get(), n);
  b.download(out, n);
  c->sync();
}

// ---------------------------------------------------------------- MSM
template <class B, class S>
static void dev_msm(Ctx* c, size_t n, uint32_t batch, const S* scalars, const Aff<B>* points, uint32_t window_bits, Aff<B>* out) {
  DevBuf<Xyzz<B>> acc(c, batch);
  MsmConfig cfg; cfg.c = (int)window_bits;
  msm_run<B, S>(c, scalars, (long long)n, points, 0, (int)n, (int)batch, cfg, acc.get());
  points_to_affine<B>(c, acc.get(), (int)batch, out);
}

template <class B, class S>
static void host_msm(Ctx* c, size_t n, uint32_t batch, const uint8_t* scalars, const uint8_t* points, uint32_t window_bits, uint8_t* out) {
  DevBuf<S> ds(c, n * batch);
  DevBuf<Aff<B>> dp(c, n), dout(c, batch);
  ds.upload(scalars, n * batch);
  dp.upload(points, n);
  fe_to_mont<S>(c, ds.get(), n * batch);
  fe_to_mont<B>(c, reinterpret_cast<B*>(dp.get()), 2 * n);
  dev_msm<B, S>(c, n, batch, ds.get(), dp.get(), window_bits, dout.get());
  fe_from_mont<B>(c, reinterpret_cast<B*>(dout.get()), 2 * (size_t)batch);
  dout.download(out, batch);
  c->sync();
}

extern "C" {

tb_status tb_ntt(tb_ctx* ctx, int field, uint32_t logn, int inverse, int coset, uint32_t batch, const uint8_t* in, uint8_t* out) {
  TB_API_BEGIN(ctx)
  TB_REQUIRE(in && out && batch >= 1 && logn >= 1 && logn <= 24, "tb_ntt arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  if (field == TB_FP) host_ntt<Fp>(&ctx->c, logn, inverse, coset, batch, in, out);
  else if (field == TB_FQ) host_ntt<Fq>(&ctx->c, logn, inverse, coset, batch, in, out);
  else throw std::invalid_argument("unknown field id");
  TB_API_END(ctx)
}

tb_status tb_msm(tb_ctx* ctx, int curve, size_t n, uint32_t batch, const uint8_t* scalars, const uint8_t* points, uint32_t window_bits,
                 uint8_t* out_points) {
  TB_API_BEGIN(ctx)
  TB_REQUIRE(scalars && points && out_points && n >= 1 && batch >= 1, "tb_msm arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  if (curve == TB_VESTA) host_msm<Fq, Fp>(&ctx->c, n, batch, scalars, points, window_bits, out_points);
  else if (curve == TB_PALLAS) host_msm<Fp, Fq>(&ctx->c, n, batch, scalars, points, window_bits, out_points);
  else throw std::invalid_argument("unknown curve id");
  TB_API_END(ctx)
}

tb_status tb_dev_to_mont(tb_ctx* ctx, int field, void* d, size_t n) {
  TB_API_BEGIN(ctx)
  if (field == TB_FP) fe_to_mont<Fp>(&ctx->c, (Fp*)d, n); else if (field == TB_FQ) fe_to_mont<Fq>(&ctx->c, (Fq*)d, n);
  else throw std::invalid_argument("unknown field id");
  TB_API_END(ctx)
}
tb_status tb_dev_from_mont(tb_ctx* ctx, int field, void* d, size_t n) {
  TB_API_BEGIN(ctx)
  if (field == TB_FP) fe_from_mont<Fp>(&ctx->c, (Fp*)d, n); else if (field == TB_FQ) fe_from_mont<Fq>(&ctx->c, (Fq*)d, n);
  else throw std::invalid_argument("unknown field id");
  TB_API_END(ctx)
}
tb_status tb_dev_ntt(tb_ctx* ctx, int field, uint32_t logn, int inverse, int coset, uint32_t batch, const void* d_in, void* d_out, void* d_scratch) {
  TB_API_BEGIN(ctx)
  TB_REQUIRE(d_in && d_out && batch >= 1 && logn >= 1 && logn <= 24, "tb_dev_ntt arguments");
  if (field == TB_FP) dev_ntt<Fp>(&ctx->c, logn, inverse, coset, batch, (const Fp*)d_in, (Fp*)d_out, (Fp*)d_scratch);
  else if (field == TB_FQ) dev_ntt<Fq>(&ctx->c, logn, inverse, coset, batch, (const Fq*)d_in, (Fq*)d_out, (Fq*)d_scratch);
  else throw std::invalid_argument("unknown field id");
  TB_API_END(ctx)
}
tb_status tb_dev_msm(tb_ctx* ctx, int curve, size_t n, uint32_t batch, const void* d_scalars, const void* d_points, uint32_t window_bits,
                     void* d_out_points) {
  TB_API_BEGIN(ctx)
  TB_REQUIRE(d_scalars && d_points && d_out_points && n >= 1 && batch >= 1, "tb_dev_msm arguments");
  if (curve == TB_VESTA) dev_msm<Fq, Fp>(&ctx->c, n, batch, (const Fp*)d_scalars, (const Aff<Fq>*)d_points, window_bits, (Aff<Fq>*)d_out_points);
  else if (curve == TB_PALLAS) dev_msm<Fp, Fq>(&ctx->c, n, batch, (const Fq*)d_scalars, (const Aff<Fp>*)d_points, window_bits, (Aff<Fp>*)d_out_points);
  else throw std::invalid_argument("unknown curve id");
  TB_API_END(ctx)
}

// ---------------------------------------------------------------- SRS
tb_status tb_srs_load(tb_ctx* ctx, uint32_t k, const uint8_t* g, const uint8_t* g_lagrange, const uint8_t* w, const uint8_t* u, tb_srs** out) {
  TB_API_BEGIN(ctx)
  TB_REQUIRE(out && g && g_lagrange && w && u && k >= 1 && k <= 20, "tb_srs_load arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  *out = reinterpret_cast<tb_srs*>(Srs::load(&ctx->c, k, g, g_lagrange, w, u));
  TB_API_END(ctx)
}
void tb_srs_free(tb_srs* srs) { delete reinterpret_cast<Srs*>(srs); }

tb_status tb_srs_commit(tb_ctx* ctx, const tb_srs* srs_, int lagrange, uint32_t batch, const uint8_t* scalars, const uint8_t* blinds, uint8_t* out_points) {
  TB_API_BEGIN(ctx)
  const Srs* srs = reinterpret_cast<const Srs*>(srs_);
  TB_REQUIRE(srs && scalars && out_points && batch >= 1, "tb_srs_commit arguments");
  Ctx* c = &ctx->c;
  size_t n = srs->n;
  DevBuf<Fp> ds(c, n * batch), db(c, batch);
  DevBuf<Aff<Fq>> dout(c, batch);
  ds.upload(scalars, n * batch);
  fe_to_mont<Fp>(c, ds.get(), n * batch);
  if (blinds) { db.upload(blinds, batch); fe_to_mont<Fp>(c, db.get(), batch); }
  srs->commit(c, lagrange != 0, ds.get(), (long long)n, (int)batch, blinds ? db.get() : nullptr, dout.get());
  fe_from_mont<Fq>(c, reinterpret_cast<Fq*>(dout.get()), 2 * (size_t)batch);
  dout.download(out_points, batch);
  c->sync();
  TB_API_END(ctx)
}

}  // extern "C"
