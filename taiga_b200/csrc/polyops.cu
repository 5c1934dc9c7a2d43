// Batched polynomial utilities of the prover: linear combination, Horner evaluation, Kate (synthetic) division,
// batch inversion, prefix products, inner products, power vectors, and a per-proof scalar interpreter.
// Replaces halo2_proofs `arithmetic::{eval_polynomial, kate_division, compute_inner_product}`, `BatchInvert` and the
// `Polynomial` +, * operators used by plonk::create_proof / multiopen / commitment (EXT; SURVEY.md §8a H4-H9).
#define TB_NOINLINE_MUL 0  // loop-structured kernels: small code, keep the multiply inline
#include <cooperative_groups.h>
#include "common.cuh"
#include "prover.cuh"

namespace tb {

constexpr int PO_THREADS = 256;

__global__ void poly_fma_kernel(Fp* out, long long out_stride, const Fp* s, long long s_stride, const Fp* in, long long in_stride, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= n) return;
  Fp sv = ld_fe(s + (long long)b * s_stride);
  Fp* o = out + (long long)b * out_stride + i;
  st_fe(o, ld_fe(o) * sv + ld_fe(in + (long long)b * in_stride + i));
}
void poly_fma(Ctx* c, Fp* out, long long out_stride, const Fp* s, long long s_stride, const Fp* in, long long in_stride, int n, int B) {
  ProfScope prof_scope(c, PC_POLY);
  launch(c, poly_fma_kernel, dim3((n + PO_THREADS - 1) / PO_THREADS, B), PO_THREADS, 0, out, out_stride, s, s_stride, in, in_stride, n);
}

__global__ void poly_scale_kernel(Fp* out, long long out_stride, const Fp* s, long long s_stride, const Fp* a, long long a_stride, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= n) return;
  st_fe(out + (long long)b * out_stride + i, ld_fe(a + (long long)b * a_stride + i) * ld_fe(s + (long long)b * s_stride));
}
void poly_scale(Ctx* c, Fp* out, long long out_stride, const Fp* s, long long s_stride, const Fp* a, long long a_stride, int n, int B) {
  launch(c, poly_scale_kernel, dim3((n + PO_THREADS - 1) / PO_THREADS, B), PO_THREADS, 0, out, out_stride, s, s_stride, a, a_stride, n);
}

__global__ void poly_copy_kernel(Fp* out, long long out_stride, const Fp* in, long long in_stride, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= n) return;
  st_fe(out + (long long)b * out_stride + i, ld_fe(in + (long long)b * in_stride + i));
}
void poly_copy(Ctx* c, Fp* out, long long out_stride, const Fp* in, long long in_stride, int n, int B) {
  launch(c, poly_copy_kernel, dim3((n + PO_THREADS - 1) / PO_THREADS, B), PO_THREADS, 0, out, out_stride, in, in_stride, n);
}

__global__ void poly_add_at_kernel(Fp* v, long long stride, int idx, const Fp* s, long long s_stride, int sign, int B) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  Fp* p = v + (long long)b * stride + idx;
  Fp sv = s[(long long)b * s_stride];
  *p = sign > 0 ? *p + sv : *p - sv;
}
void poly_add_at(Ctx* c, Fp* v, long long stride, int idx, const Fp* s, long long s_stride, int sign, int B) {
  launch(c, poly_add_at_kernel, (B + 31) / 32, 32, 0, v, stride, idx, s, s_stride, sign, B);
}

// ---- block-wide sum of field elements (256 threads); result valid in thread 0
__device__ __forceinline__ Fp shfl_down_fe(const Fp& v, int d) {
  Fp r;
#pragma unroll
  for (int i = 0; i < 8; ++i) r.l[i] = __shfl_down_sync(0xffffffffu, v.l[i], d);
  return r;
}
__device__ Fp block_sum_fe(Fp v, Fp* sm /* 8 */) {
  for (int d = 16; d >= 1; d >>= 1) v = v + shfl_down_fe(v, d);
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = lane < (int)(blockDim.x >> 5) ? sm[lane] : Fp::zero();
    for (int d = 4; d >= 1; d >>= 1) v = v + shfl_down_fe(v, d);
  }
  return v;
}

// Horner evaluation: each thread owns a contiguous chunk of m = n/256 coefficients
__global__ void __launch_bounds__(PO_THREADS) poly_eval_kernel(const EvalItem* __restrict__ items, const Fp* __restrict__ points, long long pt_stride,
                                                                Fp* __restrict__ evals, long long ev_stride, int n) {
  __shared__ Fp sm[8];
  int t = blockIdx.x, b = blockIdx.y;
  EvalItem it = items[t];
  const Fp* poly = it.base + (long long)b * it.bstride;
  Fp x = points[(long long)b * pt_stride + it.point];
  int m = n / PO_THREADS; if (m < 1) m = 1;
  int j = threadIdx.x;
  Fp acc = Fp::zero();
  if (j * m < n) {
    for (int i = m - 1; i >= 0; --i) acc = acc * x + ldg_fe(poly + j * m + i);
    // * x^(j*m)
    Fp xm = x; for (int s = 1; s < m; s <<= 1) xm = xm.sqr();   // m is a power of two
    Fp pw = Fp::one();
    for (int bit = 31 - __clz(j | 1); bit >= 0; --bit) { pw = pw.sqr(); if ((j >> bit) & 1) pw = pw * xm; }
    acc = acc * pw;
  }
  acc = block_sum_fe(acc, sm);
  if (threadIdx.x == 0) evals[(long long)b * ev_stride + t] = acc;
}
void poly_eval(Ctx* c, const EvalItem* d_items, int nitems, const Fp* points, long long pt_stride, Fp* evals, long long ev_stride, int n, int B) {
  ProfScope prof_scope(c, PC_POLY);
  if (nitems <= 0) return;
  TB_REQUIRE((n & (n - 1)) == 0, "poly_eval needs a power-of-two length");
  launch(c, poly_eval_kernel, dim3(nitems, B), PO_THREADS, 0, d_items, points, pt_stride, evals, ev_stride, n);
}

__global__ void __launch_bounds__(PO_THREADS) inner_product_kernel(Fp* out, long long out_stride, const Fp* a, long long a_stride, const Fp* bv,
                                                                    long long b_stride, int n) {
  __shared__ Fp sm[8];
  int b = blockIdx.x;
  Fp acc = Fp::zero();
  for (int i = threadIdx.x; i < n; i += PO_THREADS) acc = acc + ldg_fe(a + (long long)b * a_stride + i) * ldg_fe(bv + (long long)b * b_stride + i);
  acc = block_sum_fe(acc, sm);
  if (threadIdx.x == 0) out[(long long)b * out_stride] = acc;
}
void inner_product(Ctx* c, Fp* out, long long out_stride, const Fp* a, long long a_stride, const Fp* bvec, long long b_stride, int n, int B) {
  launch(c, inner_product_kernel, B, PO_THREADS, 0, out, out_stride, a, a_stride, bvec, b_stride, n);
}

__global__ void powers_kernel(Fp* out, long long out_stride, const Fp* x, long long x_stride, int n) {
  // thread j writes x^(16j .. 16j+15)
  int j = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  int i0 = j * 16;
  if (i0 >= n) return;
  Fp xv = x[(long long)b * x_stride];
  Fp pw = Fp::one();
  for (int bit = 31 - __clz(i0 | 1); bit >= 0; --bit) { pw = pw.sqr(); if ((i0 >> bit) & 1) pw = pw * xv; }
  Fp* o = out + (long long)b * out_stride + i0;
  for (int i = 0; i < 16 && i0 + i < n; ++i) { st_fe(o + i, pw); pw = pw * xv; }
}
void powers(Ctx* c, Fp* out, long long out_stride, const Fp* x, long long x_stride, int n, int B) {
  int threads = (n + 15) / 16;
  launch(c, powers_kernel, dim3((threads + 127) / 128, B), 128, 0, out, out_stride, x, x_stride, n);
}

// ---------------------------------------------------------------- Kate division (suffix linear recurrence q_j = a_{j+1} + z q_{j+1})
// One thread-block CLUSTER per polynomial: 8 CTAs x 512 threads cover n = 2^15 coefficients with 8 per thread, so the
// dependent chain is 8 (local Horner) + 9 (block suffix composition) + <= 7 (cluster composition over distributed shared
// memory) + 8 (replay with the incoming carry) multiply-adds, spread over 8 SMs -- it used to be 64 + 9 + 64 on one SM.
// The kernel is pure latency (one polynomial per proof per opening point).  Polynomials shorter than 4096 use a single CTA.
// KD_THREADS, KD_CLUSTER, KD_MAX_M and the length limit KD_MAX_N are in prover.cuh.
__global__ void __launch_bounds__(KD_THREADS) kate_div_kernel(Fp* out, long long out_stride, const Fp* in, long long in_stride, const Fp* zs,
                                                               long long z_stride, int n, int cs /* CTAs per polynomial */) {
  namespace cg = cooperative_groups;
  __shared__ uint4 kd_smem[(2 * KD_THREADS + 3) * 2];
  Fp* A = reinterpret_cast<Fp*>(kd_smem);       // additive part of the suffix map
  Fp* M = A + KD_THREADS;                        // multiplicative part
  Fp* summ = M + KD_THREADS;                     // [0], [1]: this CTA's (A, M) summary; [2]: carry into this CTA
  const int rank = cs > 1 ? (int)cg::this_cluster().block_rank() : 0;
  const int b = blockIdx.x / cs, t = threadIdx.x;
  const Fp* a = in + (long long)b * in_stride;
  Fp* q = out + (long long)b * out_stride;
  const Fp z = zs[(long long)b * z_stride];
  const int T = (n / cs) < KD_THREADS ? (n / cs) : KD_THREADS;   // active threads per CTA
  const int m = n / (cs * T);                                      // chunk per thread (powers of two, m <= KD_MAX_M)
  const int j0 = (rank * T + t) * m;                               // q indices [j0, j0 + m)
  Fp av[KD_MAX_M];
  Fp loc = Fp::zero(), zm = z;
  if (t < T) {
#pragma unroll
    for (int i = 0; i < KD_MAX_M; ++i) { int j = j0 + i + 1; av[i] = (i < m && j < n) ? ldg_fe(a + j) : Fp::zero(); }
#pragma unroll
    for (int i = KD_MAX_M - 1; i >= 0; --i) if (i < m) loc = av[i] + z * loc;
    for (int i = 1; i < m; i <<= 1) zm = zm.sqr();
    A[t] = loc; M[t] = zm;
  }
  __syncthreads();
  // suffix composition inside the CTA: carry into chunk t-1 is C_{t-1} = A_t + M_t * C_t
  for (int d = 1; d < T; d <<= 1) {
    Fp na, nm; const bool act = (t < T) && (t + d < T);
    if (act) { na = A[t] + M[t] * A[t + d]; nm = M[t] * M[t + d]; }
    __syncthreads();
    if (act) { A[t] = na; M[t] = nm; }
    __syncthreads();
  }
  // A[t]: value at the bottom of chunk t with zero carry into the top of this CTA; M[t] = z^(m (T - t))
  Fp cin = Fp::zero();
  if (cs > 1) {
    cg::cluster_group cluster = cg::this_cluster();
    if (t == 0) { summ[0] = A[0]; summ[1] = M[0]; }
    cluster.sync();
    if (t == 0) {
      Fp c = Fp::zero();
      for (int r = cs - 1; r > rank; --r) {
        const Fp* rs = cluster.map_shared_rank(summ, r);
        c = rs[0] + rs[1] * c;
      }
      summ[2] = c;
    }
    __syncthreads();
    cin = summ[2];
    cluster.sync();   // nobody leaves while its summary may still be read
  }
  if (t < T) {
    Fp cur = (t + 1 < T) ? A[t + 1] + M[t + 1] * cin : cin;
#pragma unroll
    for (int i = KD_MAX_M - 1; i >= 0; --i) if (i < m) { cur = av[i] + z * cur; st_fe(q + j0 + i, cur); }
  }
}
void poly_kate_div(Ctx* c, Fp* out, long long out_stride, const Fp* in, long long in_stride, const Fp* z, long long z_stride, int n, int B) {
  ProfScope prof_scope(c, PC_POLY);
  TB_REQUIRE((n & (n - 1)) == 0, "kate division needs a power-of-two length");
  TB_REQUIRE(n >= 1 && n <= KD_MAX_N, "kate division: polynomial too long for one cluster");
  const int cs = n >= KD_CLUSTER * KD_THREADS ? KD_CLUSTER : 1;
  launch_cluster(c, cs, kate_div_kernel, (unsigned)(B * cs), KD_THREADS, 0, out, out_stride, in, in_stride, z, z_stride, n, cs);
}

// ---------------------------------------------------------------- batch inversion (Montgomery trick, 16 elements per thread, zeros skipped)
constexpr int BI_CHUNK = 16;
__global__ void batch_inverse_kernel(Fp* v, size_t count) {
  size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  size_t i0 = t * BI_CHUNK;
  if (i0 >= count) return;
  int m = (int)((count - i0) < (size_t)BI_CHUNK ? (count - i0) : BI_CHUNK);
  Fp pre[BI_CHUNK];
  Fp acc = Fp::one();
  for (int i = 0; i < m; ++i) { pre[i] = acc; Fp x = ld_fe(v + i0 + i); if (!x.is_zero()) acc = acc * x; }
  acc = acc.inv();
  for (int i = m - 1; i >= 0; --i) {
    Fp x = ld_fe(v + i0 + i);
    if (x.is_zero()) continue;
    st_fe(v + i0 + i, acc * pre[i]);
    acc = acc * x;
  }
}
void batch_inverse(Ctx* c, Fp* v, size_t count) {
  if (!count) return;
  size_t threads = (count + BI_CHUNK - 1) / BI_CHUNK;
  launch(c, batch_inverse_kernel, (unsigned)((threads + 63) / 64), 64, 0, v, count);
}

// ---------------------------------------------------------------- exclusive prefix product
constexpr int PP_THREADS = 512;
__global__ void __launch_bounds__(PP_THREADS) prefix_product_kernel(Fp* out, const Fp* in, int n) {
  extern __shared__ uint4 pp_smem[];
  Fp* S = reinterpret_cast<Fp*>(pp_smem);
  int t = threadIdx.x;
  const Fp* a = in + (size_t)blockIdx.x * n;
  Fp* o = out + (size_t)blockIdx.x * n;
  int T = n < PP_THREADS ? n : PP_THREADS;
  int m = n / T;
  Fp loc = Fp::one();
  if (t < T) { for (int i = 0; i < m; ++i) loc = loc * ldg_fe(a + t * m + i); S[t] = loc; }
  __syncthreads();
  for (int d = 1; d < T; d <<= 1) {  // inclusive Hillis-Steele scan of chunk products
    Fp nv; bool act = (t < T) && (t >= d);
    if (act) nv = S[t - d] * S[t];
    __syncthreads();
    if (act) S[t] = nv;
    __syncthreads();
  }
  if (t < T) {
    Fp cur = t ? S[t - 1] : Fp::one();
    for (int i = 0; i < m; ++i) { Fp x = ldg_fe(a + t * m + i); st_fe(o + t * m + i, cur); cur = cur * x; }
  }
}
void prefix_product(Ctx* c, Fp* out, const Fp* in, int n, int count) {
  TB_REQUIRE((n & (n - 1)) == 0 && out != in, "prefix_product arguments");
  launch(c, prefix_product_kernel, count, PP_THREADS, PP_THREADS * 32, out, in, n);
}

// ---------------------------------------------------------------- per-proof scalar interpreter
__global__ void scalar_program_kernel(Fp* vars, long long stride, const ScalarInstr* __restrict__ prog, int ninstr, const Fp* __restrict__ consts, int B) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  Fp* v = vars + (long long)b * stride;
  for (int pc = 0; pc < ninstr; ++pc) {
    ScalarInstr in = prog[pc];
    Fp r;
    switch (in.op) {
      case S_MUL: r = v[in.a] * v[in.b]; break;
      case S_ADD: r = v[in.a] + v[in.b]; break;
      case S_SUB: r = v[in.a] - v[in.b]; break;
      case S_INV: r = v[in.a].inv(); break;
      case S_COPY: r = v[in.a]; break;
      case S_POW2K: r = v[in.a]; for (uint32_t i = 0; i < in.imm; ++i) r = r.sqr(); break;
      case S_CONST: r = consts[in.imm]; break;
      case S_NEG: r = v[in.a].neg(); break;
      case S_FMA: r = v[in.dst] * v[in.a] + v[in.b]; break;
      case S_POWI: r = v[in.a].pow_u64((uint64_t)in.imm); break;
      default: r = Fp::zero();
    }
    v[in.dst] = r;
  }
}
void scalar_program(Ctx* c, Fp* vars, long long stride, const ScalarInstr* d_prog, int ninstr, const Fp* d_consts, int B) {
  if (ninstr <= 0) return;
  launch(c, scalar_program_kernel, (B + 31) / 32, 32, 0, vars, stride, d_prog, ninstr, d_consts, B);
}

}  // namespace tb
