// Lookup-argument permutation on the device: sort of 255-bit keys + halo2's table arrangement.
// Replaces halo2_proofs `lookup::prover::permute_expression_pair` (EXT; SURVEY.md §8a row H5, App. A.0):
//   A' = ascending sort of the compressed inputs over the usable rows (canonical-integer order, pasta `Ord`);
//   S'_i = A'_i wherever A'_i starts a new run (consuming one copy of that table value); the remaining slots receive
//   the unused table values in ascending order, handed out from the LAST repeated row backwards (the BTreeMap / pop()
//   order of the reference), so the result is bit-identical to the CPU path, not merely a valid arrangement.
#define TB_NOINLINE_MUL 0  // loop-structured kernels: small code, keep the multiply inline
#include "common.cuh"
#include "prover.cuh"
#include "prover_kernels.cuh"

namespace tb {

constexpr int BS_TILE = 2048;     // keys per CTA tile in shared memory (64 KiB)
constexpr int BS_THREADS = 512;

// Montgomery -> canonical keys; rows >= usable become +infinity sentinels so they sort to the end
__global__ void lookup_keys_kernel(Fp* keys, const Fp* vals, int n, int usable) {
  int i = blockIdx.x * blockDim.x + threadIdx.x, a = blockIdx.y;
  if (i >= n) return;
  Fp v;
  if (i < usable) v = ld_fe(vals + (size_t)a * n + i).from_mont();
  else { for (int j = 0; j < 8; ++j) v.l[j] = 0xffffffffu; }
  st_fe(keys + (size_t)a * n + i, v);
}

__device__ __forceinline__ void cmp_swap(Fp& x, Fp& y, bool asc) {
  int c = Fp::cmp_raw(x, y);
  if ((c > 0) == asc && c != 0) { Fp t = x; x = y; y = t; }
}

// all (k, j) steps with k <= tile (first = 1), or the steps j = jstart..1 of one k (first = 0), inside shared memory
__global__ void __launch_bounds__(BS_THREADS) bitonic_local_kernel(Fp* keys, int n, int tile, int first, int kk, int jstart) {
  extern __shared__ uint4 bs_smem[];
  Fp* s = reinterpret_cast<Fp*>(bs_smem);
  Fp* base = keys + (size_t)blockIdx.y * n + (size_t)blockIdx.x * tile;
  int g0 = blockIdx.x * tile;
  for (int i = threadIdx.x; i < tile; i += BS_THREADS) s[i] = ld_fe(base + i);
  __syncthreads();
  int k0 = first ? 2 : kk, k1 = first ? tile : kk;
  for (int k = k0; k <= k1; k <<= 1) {
    for (int j = first ? (k >> 1) : jstart; j >= 1; j >>= 1) {
      for (int t = threadIdx.x; t < (tile >> 1); t += BS_THREADS) {
        int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // index with bit j clear
        bool asc = (((g0 + i) & k) == 0);
        Fp x = s[i], y = s[i | j];
        cmp_swap(x, y, asc);
        s[i] = x; s[i | j] = y;
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < tile; i += BS_THREADS) st_fe(base + i, s[i]);
}

__global__ void bitonic_global_kernel(Fp* keys, int n, int k, int j) {
  int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (n >> 1)) return;
  Fp* base = keys + (size_t)blockIdx.y * n;
  int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
  bool asc = ((i & k) == 0);
  Fp x = ld_fe(base + i), y = ld_fe(base + (i | j));
  int c = Fp::cmp_raw(x, y);
  if ((c > 0) == asc && c != 0) { st_fe(base + i, y); st_fe(base + (i | j), x); }
}

void sort_keys(Ctx* c, Fp* keys, int n, int arrays) {
  ProfScope prof_scope(c, PC_LOOKUP_SORT);
  TB_REQUIRE((n & (n - 1)) == 0, "sort needs a power-of-two length");
  c->opt_in_smem(bitonic_local_kernel, BS_TILE * 32);
  int tile = n < BS_TILE ? n : BS_TILE;
  dim3 lg(n / tile, arrays);
  launch(c, bitonic_local_kernel, lg, BS_THREADS, tile * 32, keys, n, tile, 1, 0, 0);
  for (int k = tile << 1; k <= n; k <<= 1) {
    for (int j = k >> 1; j >= tile; j >>= 1) {
      launch(c, bitonic_global_kernel, dim3((n / 2 + 255) / 256, arrays), 256, 0, keys, n, k, j);
    }
    launch(c, bitonic_local_kernel, lg, BS_THREADS, tile * 32, keys, n, tile, 0, k, tile >> 1);
  }
}

// ---------------------------------------------------------------- arrangement of the permuted table column
// one CTA per (proof, lookup).  A: sorted inputs (canonical, `usable` valid); T: sorted table (canonical).
// Writes S' (canonical) for rows < usable; scratch `left` holds the unused table values by rank.
__global__ void __launch_bounds__(LP_THREADS) lookup_arrange_kernel(const Fp* __restrict__ A_all, const Fp* __restrict__ T_all, Fp* __restrict__ left_all,
                                                                     Fp* __restrict__ S_all, int n, int usable, uint32_t* __restrict__ err) {
  __shared__ int sm[LP_THREADS];
  const Fp* A = A_all + (size_t)blockIdx.x * n;
  const Fp* T = T_all + (size_t)blockIdx.x * n;
  Fp* left = left_all + (size_t)blockIdx.x * n;
  Fp* S = S_all + (size_t)blockIdx.x * n;
  int t = threadIdx.x;
  int m = (usable + LP_THREADS - 1) / LP_THREADS;
  int i0 = t * m, i1 = min(usable, i0 + m);
  // unused table entries: T[i] unless it is the first copy of a value that occurs among the inputs
  int n_left = 0, n_first = 0, n_cons = 0;
  for (int i = i0; i < i1; ++i) {
    Fp v = ld_fe(T + i);
    bool firstT = (i == 0) || (ld_fe(T + i - 1) != v);
    bool cons = false;
    if (firstT) {  // binary search v in A[0, usable)
      int lo = 0, hi = usable;
      while (lo < hi) { int mid = (lo + hi) >> 1; if (Fp::cmp_raw(ld_fe(A + mid), v) < 0) lo = mid + 1; else hi = mid; }
      cons = (lo < usable) && (ld_fe(A + lo) == v);
    }
    n_left += cons ? 0 : 1; n_cons += cons ? 1 : 0;
    Fp a = ld_fe(A + i);
    n_first += ((i == 0) || (ld_fe(A + i - 1) != a)) ? 1 : 0;
  }
  int tot_left, tot_first, tot_cons;
  int off_left = block_excl_scan(n_left, sm, &tot_left);
  int off_rep = block_excl_scan((i1 > i0 ? i1 - i0 : 0) - n_first, sm, &tot_first);  // tot_first reused as total repeated
  int tot_rep = tot_first;
  (void)block_excl_scan(n_cons, sm, &tot_cons);
  // every distinct input value must consume one table copy (else Error::ConstraintSystemFailure)
  if (t == 0 && tot_cons != usable - tot_rep) err[blockIdx.x] = 1u;   // err: one flag per array = per (proof, lookup)
  if (tot_left != tot_rep) { if (t == 0) err[blockIdx.x] = 1u; return; }
  int r = off_left;
  for (int i = i0; i < i1; ++i) {
    Fp v = ld_fe(T + i);
    bool firstT = (i == 0) || (ld_fe(T + i - 1) != v);
    bool cons = false;
    if (firstT) {
      int lo = 0, hi = usable;
      while (lo < hi) { int mid = (lo + hi) >> 1; if (Fp::cmp_raw(ld_fe(A + mid), v) < 0) lo = mid + 1; else hi = mid; }
      cons = (lo < usable) && (ld_fe(A + lo) == v);
    }
    if (!cons) st_fe(left + r++, v);
  }
  __threadfence_block();
  __syncthreads();
  int rr = off_rep;
  for (int i = i0; i < i1; ++i) {
    Fp a = ld_fe(A + i);
    bool firstA = (i == 0) || (ld_fe(A + i - 1) != a);
    if (firstA) st_fe(S + i, a);
    else { st_fe(S + i, ld_fe(left + (tot_rep - 1 - rr))); ++rr; }
  }
}

void lookup_arrange(Ctx* c, const Fp* sortedA, const Fp* sortedT, Fp* scratch, Fp* S, int n, int usable, int arrays, uint32_t* d_err) {
  launch(c, lookup_arrange_kernel, arrays, LP_THREADS, 0, sortedA, sortedT, scratch, S, n, usable, d_err);
}

void lookup_keys(Ctx* c, Fp* keys, const Fp* vals, int n, int usable, int arrays) {
  launch(c, lookup_keys_kernel, dim3((n + 255) / 256, arrays), 256, 0, keys, vals, n, usable);
}

}  // namespace tb
