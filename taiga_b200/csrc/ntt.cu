// Radix-2 NTT / iNTT / coset NTT over the Pasta scalar fields for sm_90a.
//
// Replaces halo2_proofs `arithmetic::best_fft` and `EvaluationDomain::{lagrange_to_coeff, coeff_to_extended,
// extended_to_coeff}` (EXT, called under taiga_halo2/src/proof.rs:33-40; SURVEY.md §8a row H2).
//
// Decomposition (Stockham-style, no bit-reversal pass): N = R_1 * R_2 (* R_3).  Pass p runs a size-R_p transform on
// digit p of the index for T neighbouring "lanes" inside shared memory, multiplies by the inter-pass twiddle
// w_{N_p}^{k_p * m} and writes back; the last pass writes digit-reversed, so input and output are both in natural
// order.  Every pass streams the vector through HBM exactly once with 128-bit loads/stores of the 4x64-bit Montgomery
// limbs; lanes are chosen so each global access covers >=128 contiguous bytes.  Shared memory holds elements as
// two 16-byte halves (conflict-free LDS.128) with a one-element pad per row.
//
// Algorithmic bytes: 64*N per transform (read N*32, write N*32); passes = ceil(logN / 9) for logN > 11.
#define TB_NOINLINE_MUL 0  // loop-structured kernels: small code, keep the multiply inline
#include "common.cuh"
#include "kernels.cuh"

namespace tb {

constexpr int NTT_TILE_LOG = 10;  // elements per CTA tile (2^10 x 32 B = 32 KB of shared memory: 6 CTAs per SM; measured +1 % over 2^11 at small batches)
constexpr int NTT_THREADS = 256;

template <class F>
struct NttArgs {
  TwiddleTables<F> tw;
  int logn, r, sh, last, npass, pass;
  int rs[3];
  int logT;
  long long in_bstride, out_bstride;  // elements between batch items (blockIdx.y)
  long long in_b2stride, out_b2stride;  // second batch dimension (blockIdx.z), e.g. proofs
  NttHook<F> pre, post;
};

template <class F>
__device__ __forceinline__ F apply_hook(const NttHook<F>& h, const TwiddleTables<F>& tw, F v, uint32_t idx) {
  if (h.table) return v * ldg_fe(h.table + idx);
  if (h.use_zeta) { uint32_t m3 = idx % 3u; if (m3) v = v * (m3 == 1 ? h.z1 : h.z2); }
  if (h.k) {
    uint32_t e = (uint32_t)(((uint64_t)idx * h.k) & ((1ull << h.mod_bits) - 1)) << (TW_LOG - h.mod_bits);
    if (e) v = v * tw_pow(tw, e);
  }
  if (h.use_const) v = v * h.c;
  return v;
}

template <class F>
__global__ void __launch_bounds__(NTT_THREADS) ntt_pass_kernel(const F* __restrict__ in, F* __restrict__ out, const NttArgs<F> a) {
  extern __shared__ uint4 smem[];
  const int R = 1 << a.r, T = 1 << a.logT;
  const int stride = (T == 1) ? 1 : T + 1;
  uint4* slo = smem;
  uint4* shi = smem + R * stride;
  in += (long long)blockIdx.y * a.in_bstride + (long long)blockIdx.z * a.in_b2stride;
  out += (long long)blockIdx.y * a.out_bstride + (long long)blockIdx.z * a.out_b2stride;
  const uint32_t lane0 = blockIdx.x << a.logT;
  const int logn = a.logn;

  // position of element j of lane L in the (in-place) working layout
  auto pos_of = [&](uint32_t L, uint32_t j) -> uint32_t {
    if (!a.last) {
      uint32_t m = L & ((1u << a.sh) - 1), h = L >> a.sh;
      return (h << (a.sh + a.r)) | (j << a.sh) | m;
    }
    uint32_t base = 0, t = L; int s2 = logn;
    for (int q = 0; q < a.pass; ++q) { s2 -= a.rs[q]; base |= (t & ((1u << a.rs[q]) - 1)) << s2; t >>= a.rs[q]; }
    return base | j;
  };

  for (int e = threadIdx.x; e < R * T; e += NTT_THREADS) {
    uint32_t l, j;
    if (!a.last) { l = e & (T - 1); j = e >> a.logT; } else { j = e & (R - 1); l = e >> a.r; }
    uint32_t p = pos_of(lane0 + l, j);
    F v = ldg_fe(in + p);
    if (a.pass == 0) v = apply_hook(a.pre, a.tw, v, p);
    slo[j * stride + l] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]);
    shi[j * stride + l] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
  }
  __syncthreads();

  auto lds = [&](int idx) -> F {
    uint4 x = slo[idx], y = shi[idx]; F v;
    v.l[0] = x.x; v.l[1] = x.y; v.l[2] = x.z; v.l[3] = x.w; v.l[4] = y.x; v.l[5] = y.y; v.l[6] = y.z; v.l[7] = y.w; return v;
  };
  auto sts = [&](int idx, const F& v) {
    slo[idx] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]); shi[idx] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
  };

  // decimation-in-frequency stages: natural order in, bit-reversed order out
  for (int lh = a.r - 1; lh >= 0; --lh) {
    const int h = 1 << lh;
    for (int t = threadIdx.x; t < (R >> 1) * T; t += NTT_THREADS) {
      int l = t & (T - 1), bj = t >> a.logT;
      int off = bj & (h - 1), j0 = ((bj >> lh) << (lh + 1)) | off;
      int i0 = j0 * stride + l, i1 = (j0 + h) * stride + l;
      F x = lds(i0), y = lds(i1);
      F s = x + y, d = x - y;
      if (off) d = d * ldg_fe(a.tw.hi + ((uint32_t)off << (TW_HALF - 1 - lh)));  // w_{2h}^off = w_S^(off << (24-1-lh))
      sts(i0, s); sts(i1, d);
    }
    __syncthreads();
  }

  for (int e = threadIdx.x; e < R * T; e += NTT_THREADS) {
    uint32_t l = e & (T - 1), jo = e >> a.logT;
    uint32_t L = lane0 + l;
    F v = lds((int)(__brev(jo) >> (32 - a.r)) * stride + l);
    if (!a.last) {
      uint32_t m = L & ((1u << a.sh) - 1);
      uint32_t ex = (jo * m) << (logn - (a.sh + a.r));  // exponent of w_N
      if (ex) v = v * tw_pow(a.tw, ex << (TW_LOG - logn));
      st_fe(out + pos_of(L, jo), v);
    } else {
      uint32_t k = L | (jo << (logn - a.r));
      v = apply_hook(a.post, a.tw, v, k);
      st_fe(out + k, v);
    }
  }
}

static void ntt_plan(int logn, int* rs, int* npass) {
  if (logn <= NTT_TILE_LOG) { rs[0] = logn; *npass = 1; return; }
  int np = logn > 16 ? (logn + 8) / 9 : 2;
  int base = logn / np, rem = logn % np;
  for (int i = 0; i < np; ++i) rs[i] = base + (i < rem ? 1 : 0);
  *npass = np;
}

template <class F>
void ntt_run(Ctx* ctx, int logn, bool inverse, const F* in, F* out, F* scratch, int batch, long long in_bstride,
             long long out_bstride, const NttHook<F>* pre, const NttHook<F>* post, int batch2, long long in_b2stride, long long out_b2stride) {
  TB_REQUIRE(logn >= 1 && logn <= TW_LOG, "NTT size out of range");
  TB_REQUIRE(batch >= 1 && batch <= 65535 && batch2 >= 1 && batch2 <= 65535, "NTT batch out of range");
  ProfScope prof_scope(ctx, PC_NTT);
  { const double elems = (double)batch * batch2 * (double)(1ull << logn);
    const double hook = (pre ? (pre->table ? 1.0 : (pre->use_zeta ? 0.67 : 0.0) + (pre->k ? 1.0 : 0.0) + (pre->use_const ? 1.0 : 0.0)) : 0.0) +
                        ((post || inverse) ? 1.0 + (post && post->k ? 1.0 : 0.0) + (post && post->use_zeta ? 0.67 : 0.0) : 0.0);
    ctx->work[PC_NTT] += elems * (0.5 * logn + hook + (logn > 10 ? 1.0 : 0.0)); }   // butterflies + hooks + inter-pass twiddles
  ctx->opt_in_smem(ntt_pass_kernel<F>, 96 * 1024);
  NttArgs<F> a;
  a.tw = inverse ? field_tables<F>(ctx).inv : field_tables<F>(ctx).fwd;
  a.logn = logn;
  ntt_plan(logn, a.rs, &a.npass);
  NttHook<F> none; none.use_zeta = 0; none.k = 0; none.use_const = 0; none.mod_bits = TW_LOG;
  a.pre = pre ? *pre : none;
  a.post = post ? *post : none;
  if (inverse) {  // fold 1/N into the post hook
    F ninv = F::from_u32(1u << (logn > 30 ? 30 : logn)).inv();
    if (a.post.use_const) a.post.c = a.post.c * ninv; else { a.post.use_const = 1; a.post.c = ninv; }
  }
  TB_REQUIRE(a.npass == 1 || scratch != nullptr, "multi-pass NTT needs a scratch buffer");
  int sh = logn;
  for (int p = 0; p < a.npass; ++p) {
    a.pass = p; a.r = a.rs[p]; sh -= a.r; a.sh = sh; a.last = (p == a.npass - 1);
    int lanes_log = logn - a.r;
    a.logT = NTT_TILE_LOG - a.r < lanes_log ? NTT_TILE_LOG - a.r : lanes_log;
    if (a.logT < 0) a.logT = 0;
    const F* src = (p == 0) ? in : scratch;
    F* dst = a.last ? out : scratch;
    a.in_bstride = (p == 0) ? in_bstride : (long long)(1ll << logn);
    a.out_bstride = a.last ? out_bstride : (long long)(1ll << logn);
    a.in_b2stride = (p == 0) ? in_b2stride : (long long)batch * (1ll << logn);   // scratch is [batch2][batch][N]
    a.out_b2stride = a.last ? out_b2stride : (long long)batch * (1ll << logn);
    int R = 1 << a.r, T = 1 << a.logT;
    size_t smem = (size_t)R * (T == 1 ? 1 : T + 1) * 32;
    dim3 grid((1u << lanes_log) >> a.logT, batch, batch2);
    launch(ctx, ntt_pass_kernel<F>, grid, NTT_THREADS, smem, src, dst, a);
  }
}

template void ntt_run<Fp>(Ctx*, int, bool, const Fp*, Fp*, Fp*, int, long long, long long, const NttHook<Fp>*, const NttHook<Fp>*, int, long long, long long);
template void ntt_run<Fq>(Ctx*, int, bool, const Fq*, Fq*, Fq*, int, long long, long long, const NttHook<Fq>*, const NttHook<Fq>*, int, long long, long long);

template <class F>
__global__ void ntt_hook_table_kernel(NttHook<F> h, TwiddleTables<F> tw, F* table, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) st_fe(table + i, apply_hook(h, tw, F::one(), (uint32_t)i));
}
template <class F> void ntt_hook_table(Ctx* ctx, const NttHook<F>& hook, bool inverse, F* table, int n) {
  NttHook<F> h = hook; h.table = nullptr;
  launch(ctx, ntt_hook_table_kernel<F>, (n + 255) / 256, 256, 0, h, inverse ? field_tables<F>(ctx).inv : field_tables<F>(ctx).fwd, table, n);
}
template void ntt_hook_table<Fp>(Ctx*, const NttHook<Fp>&, bool, Fp*, int);
template void ntt_hook_table<Fq>(Ctx*, const NttHook<Fq>&, bool, Fq*, int);

// ---- twiddle table construction (host arithmetic with the same field code, uploaded once per context)
template <class F>
__global__ void tw_fill_kernel(TwiddleTables<F> t, F* full) {
  uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < (1u << TW_FULL_LOG)) st_fe(full + i, tw_pow2(t, i << (TW_LOG - TW_FULL_LOG)));
}

template <class F>
void build_twiddles(Ctx* ctx) {
  FieldTables<F>& ft = field_tables<F>(ctx);
  F w = omega_k<F>(TW_LOG), wi = w.inv();
  const int n = 1 << TW_HALF;
  std::vector<F> lo(n), hi(n);
  for (int dir = 0; dir < 2; ++dir) {
    F base = dir ? wi : w;
    F step = base; for (int i = 0; i < TW_HALF; ++i) step = step.sqr();
    lo[0] = F::one(); hi[0] = F::one();
    for (int i = 1; i < n; ++i) { lo[i] = lo[i - 1] * base; hi[i] = hi[i - 1] * step; }
    TwiddleTables<F>& t = dir ? ft.inv : ft.fwd;
    DevMem<F>* mem = ft.mem[dir];
    mem[0] = DevMem<F>(n); mem[1] = DevMem<F>(n);
    t.lo = mem[0].get(); t.hi = mem[1].get();
    // on the context's stream, ahead of tw_fill_kernel which reads them (that stream does not wait for the legacy default stream)
    TB_CUDA(cudaMemcpyAsync(t.lo, lo.data(), n * sizeof(F), cudaMemcpyHostToDevice, ctx->stream));
    TB_CUDA(cudaMemcpyAsync(t.hi, hi.data(), n * sizeof(F), cudaMemcpyHostToDevice, ctx->stream));
    if (F::params_id() == 0) {  // circuit field only: 2 x 16 MB per context
      mem[2] = DevMem<F>(size_t(1) << TW_FULL_LOG);
      launch(ctx, tw_fill_kernel<F>, (1u << TW_FULL_LOG) / 256, 256, 0, t, mem[2].get());
      TB_CUDA(cudaDeviceSynchronize());
      t.full = mem[2].get(); t.full_log = TW_FULL_LOG;
    }
  }
}
template void build_twiddles<Fp>(Ctx*);
template void build_twiddles<Fq>(Ctx*);

}  // namespace tb
