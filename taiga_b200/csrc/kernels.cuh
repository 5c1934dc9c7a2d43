// Declarations of the host-callable kernel drivers shared between translation units of libtaiga_b200.
#pragma once
#include "common.cuh"

namespace tb {

// ---------------------------------------------------------------- NTT (ntt.cu)
// Optional per-element scaling fused into the first load / last store of a transform:
//   v *= zeta^(idx mod 3)            (halo2 `distribute_powers_zeta`)           if use_zeta (z1 = zeta^1, z2 = zeta^2 or inverses)
//   v *= w_{2^mod_bits}^(idx * k)    (sub-coset shift, same direction as the transform's twiddles)   if k != 0
//   v *= c                                                                           if use_const
//   v *= table[idx]                  (all of the above precomputed per element: one multiplication, one coalesced load)   if table
template <class F> struct NttHook { int use_zeta; F z1, z2; uint32_t k; int mod_bits; int use_const; F c; const F* table = nullptr; };
// table[i] = what `hook` multiplies element i by, i < n (built once per circuit for the forward coset hooks)
template <class F> void ntt_hook_table(Ctx* ctx, const NttHook<F>& hook, bool inverse, F* table, int n);

template <class F>
void ntt_run(Ctx* ctx, int logn, bool inverse, const F* in, F* out, F* scratch, int batch, long long in_bstride,
             long long out_bstride, const NttHook<F>* pre, const NttHook<F>* post, int batch2 = 1, long long in_b2stride = 0,
             long long out_b2stride = 0);  // scratch must hold batch2 * batch * 2^logn elements
template <class F> void build_twiddles(Ctx* ctx);

// ---------------------------------------------------------------- MSM (msm.cu)
struct MsmConfig {
  int c = 0;             // window bits (0 = choose from N; a fixed-base table needs the c it was built with)
  int table_windows = 0;  // >0: `bases` is a fixed-base table [table_windows][table_stride] of 2^(c*w)*B_i and all windows share one bucket set
  int table_stride = 0;   // points per table window (>= N + n_extra); 0 = N
  int n_extra = 0;        // extra terms per MSM: scalar extra_scalars[k*n_extra + j] (Montgomery) times table point N + j
  const void* extra_scalars = nullptr;
  void* affine_out = nullptr;  // fixed-base mode: also write the K results normalised to affine (Aff<B>[K])
};
// K multi-scalar multiplications of N terms.  scalars: Montgomery form, item k at scalars + k*scalar_bstride.
// bases: affine Montgomery; item k at bases + k*base_bstride (0 = shared).  out: K XYZZ points.
template <class B, class S>
void msm_run(Ctx* ctx, const S* scalars, long long scalar_bstride, const Aff<B>* bases, long long base_bstride, int N, int K,
             const MsmConfig& cfg, Xyzz<B>* out);
// msm_batch.cu: throughput path for K fixed-base MSMs (shared-memory counting sort + batch-affine reduction rounds)
bool msm_batch_applicable(int N, int K, const MsmConfig& cfg, int c);
template <class B, class S>
void msm_batch_buckets(Ctx* ctx, const S* scalars, long long sstride, const Aff<B>* table, int N, int K, int c, int W, int table_stride, const S* extras, int n_extra,
                       Xyzz<B>* buckets);
// table[w][i] = 2^(c*w) * bases[i], w < windows  (one-off, at SRS load)
template <class B> void msm_build_tables(Ctx* ctx, const Aff<B>* bases, int N, int c, int windows, Aff<B>* table);
template <class B> void points_to_affine(Ctx* ctx, const Xyzz<B>* acc, int K, Aff<B>* out);

// ---------------------------------------------------------------- elementwise helpers (poly.cu)
template <class F> void fe_to_mont(Ctx* ctx, F* v, size_t n);     // canonical -> Montgomery, in place
template <class F> void fe_from_mont(Ctx* ctx, F* v, size_t n);   // Montgomery -> canonical, in place
void exclusive_scan_u32(Ctx* ctx, const uint32_t* in, uint32_t* out, size_t n);  // out has n+1 entries (last = total)

}  // namespace tb
