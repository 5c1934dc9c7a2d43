// Shared host-side plumbing for libtaiga_b200: context, error handling, stream-ordered device memory.
#pragma once
#include <algorithm>
#include <cstdlib>
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <stdexcept>
#include <string>
#include <map>
#include <utility>
#include <mutex>
#include <vector>
#include "curve.cuh"

namespace tb {

struct CudaError : std::runtime_error { using std::runtime_error::runtime_error; };
// the witness does not satisfy the circuit (halo2 Error::ConstraintSystemFailure class)
struct ConstraintError : std::runtime_error { using std::runtime_error::runtime_error; };

#define TB_CUDA(expr)                                                                                   \
  do {                                                                                                  \
    cudaError_t _e = (expr);                                                                            \
    if (_e != cudaSuccess)                                                                              \
      throw tb::CudaError(std::string(#expr) + " failed: " + cudaGetErrorString(_e) + " at " + __FILE__ + ":" + std::to_string(__LINE__)); \
  } while (0)

// Owner of one device allocation that outlives a call (SRS, proving key, context tables, workspaces): cudaMalloc / cudaFree,
// which no stream orders, since such an allocation may outlive the context whose stream made it.  DevBuf is the stream-ordered
// owner of per-call scratch.
template <class T> struct DevMem {
  DevMem() {}
  explicit DevMem(size_t count) { TB_CUDA(try_alloc(count)); }
  DevMem(const T* host, size_t count) : DevMem(count) { if (count) TB_CUDA(cudaMemcpy(p, host, count * sizeof(T), cudaMemcpyHostToDevice)); }
  explicit DevMem(const std::vector<T>& v) : DevMem(v.data(), v.size()) {}
  DevMem(const DevMem&) = delete; DevMem& operator=(const DevMem&) = delete;
  DevMem(DevMem&& o) noexcept : p(o.p), n(o.n) { o.p = nullptr; o.n = 0; }
  DevMem& operator=(DevMem&& o) noexcept { if (this != &o) { reset(); p = o.p; n = o.n; o.p = nullptr; o.n = 0; } return *this; }
  ~DevMem() { reset(); }
  void reset() { if (p) cudaFree(p); p = nullptr; n = 0; }
  // frees what this holds, then allocates `count` elements (at least one); returns the error instead of throwing it
  cudaError_t try_alloc(size_t count) {
    reset();
    cudaError_t e = cudaMalloc(reinterpret_cast<void**>(&p), std::max<size_t>(1, count) * sizeof(T));
    if (e == cudaSuccess) n = count; else p = nullptr;
    return e;
  }
  T* get() const { return p; }
  size_t size() const { return n; }
 private:
  T* p = nullptr; size_t n = 0;
};

// NTT twiddle tables: powers of the 2^24-th root of unity, two-level (SURVEY E.3; tables are 2 x 128 KiB per
// field and direction, L2 resident).  w_S^e = hi[e >> 12] * lo[e & 4095].
constexpr int TW_LOG = 24;
constexpr int TW_HALF = 12;
// w_S^e, S = 2^24: two-level tables (e = hi * 2^12 + lo) plus, for the circuit field, a flat table of the 2^full_log-th roots --
// every twiddle the k <= 19 prover NTTs and the quotient kernels ask for is then one 32-byte load instead of a load pair and a multiply
template <class F> struct TwiddleTables { F* lo = nullptr; F* hi = nullptr; F* full = nullptr; int full_log = 0; };
constexpr int TW_FULL_LOG = 19;

template <class F> struct FieldTables {
  TwiddleTables<F> fwd, inv;   // what the kernels take by value: views of `mem`
  DevMem<F> mem[2][3];         // [fwd, inv][lo, hi, full]
};

// kernel categories for the built-in CUDA-event profiler (bench.py's roofline / share-of-step numbers)
enum ProfCat { PC_NTT = 0, PC_MSM_SORT, PC_MSM_ACCUM, PC_MSM_REDUCE, PC_QUOT_GATES, PC_QUOT_FINISH, PC_IPA_FOLD, PC_TRANSCRIPT, PC_LOOKUP_SORT,
               PC_POLY, PC_COUNT };
struct ProfRec { int cat; cudaEvent_t a, b; };

// Integer from the environment (read on every call; only on host set-up paths).  A variable is read only if a test sets it
// to compare two shipped paths on the same input, or to reach a shipped path that the test's inputs would not reach:
// TB_MSM_BA_MIN_TERMS, TB_MSM_BA_ROUNDS, TB_MSM_BA_CHUNK (msm_batch.cu), TB_Q_SPLIT (prover.cu); TB_DEBUG prints the
// quotient's degree split at circuit load.  Every other launch choice is a constant of the code.
inline int tb_tune(const char* name, int dflt) { const char* e = getenv(name); return e ? atoi(e) : dflt; }

// Opt a kernel into more than 48 KB of dynamic shared memory on the current device.  The attribute belongs to the (function,
// device) pair, which every context of the device shares, and a kernel may need more on a later call (msm_sort_kernel's
// histogram grows with the window), so the attribute only ever grows, to the largest size a launch on the device asked for.
// The table is never destroyed: a thread of the host program may still launch while the process exits.
inline void opt_in_smem_device(int device, const void* kernel, size_t bytes) {
  static std::mutex* mu = new std::mutex;
  static auto* opted = new std::map<std::pair<int, const void*>, size_t>;
  std::lock_guard<std::mutex> lock(*mu);
  size_t& have = (*opted)[{device, kernel}];
  if (bytes > have) { TB_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes)); have = bytes; }
}

struct Ctx {
  int device = 0;
  cudaStream_t stream = nullptr;
  std::string last_error;
  FieldTables<Fp> tw_fp;
  FieldTables<Fq> tw_fq;
  int sm_count = 132;   // H100 SXM; tb_ctx_create reads the device's own count
  uint64_t launches = 0;  // kernels launched through this context (bench's gpu_launches)
  bool prof = false; std::vector<ProfRec> prof_recs; std::vector<cudaEvent_t> event_pool;
  // executed 255-bit Montgomery multiplications per kernel category (host-side accounting at every launch, for the integer-pipe
  // roofline of bench.py); the bucket additions of the batched MSM are counted on the device (they depend on the scalars)
  double work[PC_COUNT] = {0};
  DevMem<unsigned long long> d_msm_adds;
  // tb_ctx_create may fail part way: every step skips what was never created
  ~Ctx() {
    if (stream) cudaStreamSynchronize(stream);
    tw_fp = {}; tw_fq = {}; d_msm_adds.reset();
    for (cudaEvent_t e : event_pool) cudaEventDestroy(e);
    for (const ProfRec& r : prof_recs) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
    if (stream) cudaStreamDestroy(stream);
  }
  cudaEvent_t get_event() {
    cudaEvent_t e;
    if (!event_pool.empty()) { e = event_pool.back(); event_pool.pop_back(); return e; }
    TB_CUDA(cudaEventCreate(&e)); return e;
  }

  template <class T> T* alloc(size_t count) {
    void* p = nullptr;
    if (count == 0) count = 1;
    TB_CUDA(cudaMallocAsync(&p, count * sizeof(T), stream));
    return reinterpret_cast<T*>(p);
  }
  void free(void* p) { if (p) cudaFreeAsync(p, stream); }
  template <class K> void opt_in_smem(K kernel, size_t bytes) { opt_in_smem_device(device, reinterpret_cast<const void*>(kernel), bytes); }
  void sync() { TB_CUDA(cudaStreamSynchronize(stream)); }
};

// Every kernel of the library is launched here: on the context's stream, as clusters of `cluster` CTAs along x when
// cluster > 1, checked at once (so a failure names the kernel that failed) and counted in `launches`.
template <class... P, class... A>
void launch_cluster(Ctx* c, unsigned cluster, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
  cudaLaunchAttribute at = {};
  at.id = cudaLaunchAttributeClusterDimension; at.val.clusterDim.x = cluster; at.val.clusterDim.y = 1; at.val.clusterDim.z = 1;
  const cudaLaunchConfig_t cfg = {grid, block, smem, c->stream, &at, cluster > 1 ? 1u : 0u};
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, std::forward<A>(args)...);
  if (e == cudaSuccess) e = cudaGetLastError();   // or an error an earlier call left pending
  if (e != cudaSuccess) {
    const char* name = "?"; cudaFuncGetName(&name, kernel);
    throw CudaError(std::string("launch of ") + name + " failed: " + cudaGetErrorString(e));
  }
  c->launches++;
}
template <class... P, class... A> void launch(Ctx* c, void (*kernel)(P...), dim3 grid, dim3 block, size_t smem, A&&... args) {
  launch_cluster(c, 1, kernel, grid, block, smem, std::forward<A>(args)...);
}

// records a pair of CUDA events on the context's stream around a group of launches (only when profiling is on)
struct ProfScope {
  Ctx* c; int idx = -1;
  ProfScope(Ctx* ctx, int cat) : c(ctx) {
    if (!c->prof) return;
    ProfRec r; r.cat = cat; r.a = c->get_event(); r.b = c->get_event();
    cudaEventRecord(r.a, c->stream);
    idx = (int)c->prof_recs.size(); c->prof_recs.push_back(r);
  }
  ~ProfScope() { if (idx >= 0) cudaEventRecord(c->prof_recs[idx].b, c->stream); }
};

// RAII stream-ordered device buffer
template <class T> struct DevBuf {
  Ctx* ctx = nullptr; T* p = nullptr; size_t n = 0;
  DevBuf() {}
  DevBuf(Ctx* c, size_t count) : ctx(c), n(count) { p = c->alloc<T>(count); }
  DevBuf(const DevBuf&) = delete; DevBuf& operator=(const DevBuf&) = delete;
  DevBuf(DevBuf&& o) noexcept : ctx(o.ctx), p(o.p), n(o.n) { o.p = nullptr; }
  DevBuf& operator=(DevBuf&& o) noexcept { if (this != &o) { release(); ctx = o.ctx; p = o.p; n = o.n; o.p = nullptr; } return *this; }
  ~DevBuf() { release(); }
  void release() { if (p && ctx) ctx->free(p); p = nullptr; }
  T* get() const { return p; }
  void zero() { TB_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), ctx->stream)); }
  void upload(const void* host, size_t count) { TB_CUDA(cudaMemcpyAsync(p, host, count * sizeof(T), cudaMemcpyHostToDevice, ctx->stream)); }
  void download(void* host, size_t count) const { TB_CUDA(cudaMemcpyAsync(host, p, count * sizeof(T), cudaMemcpyDeviceToHost, ctx->stream)); }
};

template <class F> inline FieldTables<F>& field_tables(Ctx* c);
template <> inline FieldTables<Fp>& field_tables<Fp>(Ctx* c) { return c->tw_fp; }
template <> inline FieldTables<Fq>& field_tables<Fq>(Ctx* c) { return c->tw_fq; }

template <class F> inline F omega_k(int k) { F w = root_of_unity_2_32<F>(); for (int i = k; i < 32; ++i) w = w.sqr(); return w; }
template <class F> inline F delta_const() { return F::from_u32(5).pow_u64(1ull << 32); }  // pasta DELTA = 5^(2^32)

#ifdef __CUDACC__
// 128-bit vectorised global access of a field element (two LDG.128 / STG.128)
template <class F> __device__ __forceinline__ F ldg_fe(const F* p) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4 a = __ldg(q), b = __ldg(q + 1);
  F r; r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w; r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
  return r;
}
template <class F> __device__ __forceinline__ F ld_fe(const F* p) {
  const uint4* q = reinterpret_cast<const uint4*>(p);
  uint4 a = q[0], b = q[1];
  F r; r.l[0] = a.x; r.l[1] = a.y; r.l[2] = a.z; r.l[3] = a.w; r.l[4] = b.x; r.l[5] = b.y; r.l[6] = b.z; r.l[7] = b.w;
  return r;
}
template <class F> __device__ __forceinline__ void st_fe(F* p, const F& v) {
  uint4* q = reinterpret_cast<uint4*>(p);
  q[0] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
  q[1] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}
template <class F> __device__ __forceinline__ Aff<F> ldg_aff(const Aff<F>* p) {
  Aff<F> a; a.x = ldg_fe(&p->x); a.y = ldg_fe(&p->y); return a;
}
// w_S^e from the two-level table
template <class F> __device__ __forceinline__ F tw_pow2(const TwiddleTables<F>& t, uint32_t e) {
  F h = ldg_fe(t.hi + (e >> TW_HALF));
  uint32_t lo = e & ((1u << TW_HALF) - 1);
  if (lo) h = h * ldg_fe(t.lo + lo);
  return h;
}
template <class F> __device__ __forceinline__ F tw_pow(const TwiddleTables<F>& t, uint32_t e) {
  if (t.full && (e & ((1u << (TW_LOG - TW_FULL_LOG)) - 1)) == 0) return ldg_fe(t.full + (e >> (TW_LOG - TW_FULL_LOG)));
  return tw_pow2(t, e);
}
#endif

}  // namespace tb
