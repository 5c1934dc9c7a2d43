// Batched fixed-base MSM for many commitments at once (the throughput path of the prover: B proofs x columns MSMs per call).
//
// Replaces halo2_proofs `Params::{commit, commit_lagrange}` -> `arithmetic::best_multiexp` (EXT, called under
// taiga_halo2/src/proof.rs:33-40; SURVEY.md 8a row H1) for K MSMs that share the SRS basis.  The bases were
// premultiplied by 2^(c*w) at SRS load (srs.cuh), so the W windows of one MSM share ONE set of NB = 2^(c-1) buckets.
//
//   1. msm_sort_kernel      one CTA per MSM: signed c-bit digits of every scalar, bucket histogram and counting sort
//                           entirely in shared memory (no global atomics, no scan launches).  The scalars are staged
//                           through shared memory by TMA (cp.async.bulk.tensor, two-stage mbarrier pipeline).
//   2. msm_ba_round_kernel  R rounds of pairwise reduction inside every bucket with BATCH-AFFINE additions: a CTA takes
//                           2048 pairs, multiplies their denominators together (per-thread prefix products, then a
//                           product tree across the 256 threads in shared memory), inverts ONCE, and walks back.  An
//                           addition costs 6 field multiplications + ~1/2048 of an inversion instead of the 10 of the
//                           XYZZ mixed addition: the path is bound by the integer pipe (tools/modmul_bench.cu), so
//                           multiplications are what counts.  Round r halves every bucket: ceil(c/2^r) items are left,
//                           so the offsets of every round follow from the round-0 counts and are re-derived per CTA
//                           by a 4096-element shared-memory scan -- no per-round bookkeeping in global memory.
//   3. msm_ba_finish_kernel the (normally single) item left in every bucket becomes the XYZZ bucket sum that the
//                           two-level weighted bucket reduction of msm.cu consumes.
//
// Exceptional pairs (equal points, opposite points, the identity) are handled inside the batch: their denominator is
// replaced (2y for a doubling) or left out, so any input -- including the structured SRS of the tests -- is exact.  The
// forward kernel classifies every pair once and stores the kind beside the pair index; the backward kernel runs the plain
// addition and sends the rare kinds to a cold branch.
//
// The rounds spend HBM bytes (each round writes its items, ~330 B per pair addition) to save integer instructions; at the
// shapes of the prover they stream ~2 TB/s, so their layout matters: items are stored as x / y planes, and round 0 keeps the
// table indices of its pairs for the backward kernel.  DESIGN.md section 4.3 has the measured accounting.
#define TB_NOINLINE_MUL 0   // every loop of this file is rolled (small code): inline multiplies keep live values in registers instead of spilling them around calls
#include <cuda.h>
#include <algorithm>
#include <memory>
#include <type_traits>
#include "common.cuh"
#include "kernels.cuh"

namespace tb {

constexpr int BA_THREADS = 256;
constexpr int BA_M = 32;                        // pairs per thread of a round (16 is faster on sparse witness columns, slower on dense scalars: DESIGN §8)
constexpr int BA_BWD_MINB = 3;                  // resident CTAs per SM of the backward kernel
constexpr int BA_MAX_NB = 4096;
constexpr int SORT_THREADS = 1024;
constexpr int SORT_TILE = 1024;                 // scalars per pipeline stage (32 KB), one per thread
constexpr int SORT_BOX = 256;                   // scalars per TMA box (a box dimension is limited to 256)

// ---------------------------------------------------------------- small shared-memory helpers
// exclusive scan of v[0..n) in place (n <= 16 * blockDim.x), v[n] = total.  blockDim.x threads, tmp: 32 words.
__device__ __forceinline__ void block_scan_excl(uint32_t* v, int n, uint32_t* tmp) {
  const int T = blockDim.x, t = threadIdx.x, per = (n + T - 1) / T;
  const int b0 = t * per, b1 = min(n, b0 + per);
  uint32_t local = 0;
  for (int i = b0; i < b1; ++i) local += v[i];
  uint32_t incl = local;
  const int lane = t & 31, warp = t >> 5, nw = (T + 31) >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += o; }
  if (lane == 31) tmp[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = lane < nw ? tmp[lane] : 0u, wi = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) { uint32_t o = __shfl_up_sync(0xffffffffu, wi, d); if (lane >= d) wi += o; }
    if (lane < nw) tmp[lane] = wi - w;
    if (lane == nw - 1) v[n] = wi;
  }
  __syncthreads();
  uint32_t run = tmp[warp] + incl - local;
  for (int i = b0; i < b1; ++i) { uint32_t x = v[i]; v[i] = run; run += x; }
  __syncthreads();
}

// ---------------------------------------------------------------- TMA / mbarrier primitives (sm_90a PTX)
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
// bounded wait: a TMA that never lands must not hang the GPU box -- trap instead
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  for (uint32_t spin = 0; spin < (1u << 26); ++spin) {
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    if (done) return;
  }
  __trap();
}
// box (8 words, SORT_BOX scalars, 1 MSM) of the 3-D scalar tensor [K][N][8 x u32] -> shared memory
__device__ __forceinline__ void tma_load_tile(void* dst, const CUtensorMap* map, uint64_t* bar, int scalar0, int item) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
               ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(0), "r"(scalar0), "r"(item) : "memory");
}

// ---------------------------------------------------------------- 1. digits + counting sort, one CTA per MSM
// entries of MSM k: entries[k * cap0 + pos] = (w * table_stride + i) | sign << 31, grouped by bucket; counts[k * NB + b]
// CT > 0: window width known at compile time (the digit loop unrolls and the limbs stay in registers); CT = 0: generic
template <class S, int CT>
__global__ void __launch_bounds__(SORT_THREADS) msm_sort_kernel(const __grid_constant__ CUtensorMap smap, const S* __restrict__ extras, int N, int n_extra, int c_rt, int W_rt,
                                                                 int NB, int table_stride, uint32_t* __restrict__ counts, uint32_t* __restrict__ entries, long long cap0,
                                                                 unsigned long long* __restrict__ total_entries) {
  const int c = CT ? CT : c_rt, W = CT ? (256 + CT - 1) / CT : W_rt;
  extern __shared__ __align__(128) uint8_t sort_smem[];
  S* tile = reinterpret_cast<S*>(sort_smem);                                   // [2][SORT_TILE]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sort_smem + 2 * SORT_TILE * sizeof(S));   // [2], 8-byte aligned
  uint32_t* hist = reinterpret_cast<uint32_t*>(bars + 2);                       // [NB + 1]
  uint32_t* tmp = hist + NB + 1;                                                // [32]
  const int k = blockIdx.x, t = threadIdx.x;
  const uint32_t half = 1u << (c - 1);
  const int ntiles = (N + SORT_TILE - 1) / SORT_TILE;
  if (t == 0) { mbar_init(&bars[0], 1); mbar_init(&bars[1], 1); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  for (int b = t; b <= NB; b += SORT_THREADS) hist[b] = 0;
  __syncthreads();
  uint32_t* ent = entries + (long long)k * cap0;

  // `scatter` is a compile-time constant of each pass: the histogram pass issues its shared-memory atomics without waiting for a
  // return value (no scoreboard stall), only the scatter pass needs the old counter
  auto digits = [&](const S& sm, uint32_t idx, auto scatter_c) {
    constexpr bool scatter = decltype(scatter_c)::value;
    S s = sm.from_mont();
    if (s.is_zero()) return;
    uint32_t carry = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const int bit = w * c, limb = bit >> 5, off = bit & 31;
      uint64_t v64 = s.l[limb];
      if (limb + 1 < 8) v64 |= (uint64_t)s.l[limb + 1] << 32;
      uint32_t v = ((uint32_t)(v64 >> off) & ((1u << c) - 1)) + carry, neg = 0;
      if (v > half) { v = (1u << c) - v; neg = 1; carry = 1; } else carry = 0;
      if (v) {
        if (scatter) { const uint32_t pos = atomicAdd(&hist[v - 1], 1u); ent[pos] = (uint32_t)(w * table_stride + idx) | (neg << 31); }
        else atomicAdd(&hist[v - 1], 1u);
      }
    }
  };
  // two passes over the scalars (histogram, then scatter with the scanned histogram as cursors); tiles arrive by TMA
  auto issue = [&](int stage, int it) {   // thread 0: fill `stage` with scalars [it * SORT_TILE, (it + 1) * SORT_TILE) of MSM k
    const int s0 = it * SORT_TILE;
    int nbox = (N - s0 + SORT_BOX - 1) / SORT_BOX; if (nbox > SORT_TILE / SORT_BOX) nbox = SORT_TILE / SORT_BOX;
    mbar_expect_tx(&bars[stage], (uint32_t)(nbox * SORT_BOX * sizeof(S)));
    for (int j = 0; j < nbox; ++j) tma_load_tile(tile + stage * SORT_TILE + j * SORT_BOX, &smap, &bars[stage], s0 + j * SORT_BOX, k);
  };
  uint32_t phase[2] = {0, 0};
  for (int pass = 0; pass < 2; ++pass) {
    if (t == 0) issue(0, 0);
    for (int it = 0; it < ntiles; ++it) {
      const int st = it & 1;
      if (t == 0 && it + 1 < ntiles) issue(st ^ 1, it + 1);   // the other stage: its readers finished before the last barrier
      mbar_wait(&bars[st], phase[st]); phase[st] ^= 1;
      const int i = it * SORT_TILE + t;
      if (i < N) { if (pass) digits(tile[st * SORT_TILE + t], (uint32_t)i, std::true_type()); else digits(tile[st * SORT_TILE + t], (uint32_t)i, std::false_type()); }
      __syncthreads();   // everybody is done with stage st before it is refilled
    }
    if (t < n_extra) { const S ex = ldg_fe(extras + (long long)k * n_extra + t); if (pass) digits(ex, (uint32_t)(N + t), std::true_type()); else digits(ex, (uint32_t)(N + t), std::false_type()); }
    __syncthreads();
    if (pass == 0) {
      for (int b = t; b < NB; b += SORT_THREADS) counts[(long long)k * NB + b] = hist[b];
      __syncthreads();
      block_scan_excl(hist, NB, tmp);
      if (t == 0) atomicAdd(total_entries, (unsigned long long)hist[NB]);
    }
  }
}

// ---------------------------------------------------------------- 2. batch-affine pairwise reduction round
template <class F> __device__ __forceinline__ void sts_fe(uint4* lo, uint4* hi, int idx, const F& v) {
  lo[idx] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]); hi[idx] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]);
}
template <class F> __device__ __forceinline__ F lds_fe(const uint4* lo, const uint4* hi, int idx) {
  uint4 x = lo[idx], y = hi[idx]; F v;
  v.l[0] = x.x; v.l[1] = x.y; v.l[2] = x.z; v.l[3] = x.w; v.l[4] = y.x; v.l[5] = y.y; v.l[6] = y.z; v.l[7] = y.w; return v;
}

// pair kinds, found once by the forward kernel and stored in the top bits of meta[q] = in0 | kind << META_KIND_SHIFT
enum { PK_ADD = 0, PK_DBL, PK_COPY1, PK_COPY2, PK_INF };
constexpr int META_KIND_SHIFT = 28;
constexpr uint32_t META_IN0_MASK = (1u << META_KIND_SHIFT) - 1;

// what a round needs to know about one MSM: the bucket offsets of its input (round r) and output (round r + 1) items
struct RoundOffsets {
  uint32_t* off_cur; uint32_t* off_nxt; uint32_t n_next;
  __device__ __forceinline__ void build(uint8_t* smem, const uint32_t* __restrict__ counts0, int NB, int round) {
    off_cur = reinterpret_cast<uint32_t*>(smem); off_nxt = off_cur + (NB + 4);
    uint32_t* tmp = off_nxt + (NB + 4);
    for (int b = threadIdx.x; b < NB; b += blockDim.x) {
      const uint32_t c0 = counts0[b], cr = (c0 + ((1u << round) - 1)) >> round;
      off_cur[b] = cr; off_nxt[b] = (cr + 1) >> 1;
    }
    __syncthreads();
    block_scan_excl(off_cur, NB, tmp);
    block_scan_excl(off_nxt, NB, tmp);
    n_next = off_nxt[NB];
  }
  // output item q -> position of its first input, and whether a second input exists.  `hint`: a bucket at or before the one of q
  // (the previous item of the same thread): a few steps forward usually find it, a binary search takes over otherwise.
  __device__ __forceinline__ void locate(uint32_t q, int NB, uint32_t& in0, bool& two, int& hint) const {
    int lo = hint;   // invariant: off_nxt[lo] <= q
#pragma unroll 1
    for (int s = 0; s < 6 && off_nxt[lo + 1] <= q; ++s) ++lo;
    if (off_nxt[lo + 1] <= q) {
      int hi = NB;   // largest b with off_nxt[b] <= q
      while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (off_nxt[mid] <= q) lo = mid; else hi = mid; }
    }
    hint = lo;
    in0 = off_cur[lo] + 2 * (q - off_nxt[lo]);
    two = in0 + 1 < off_cur[lo + 1];
  }
};
constexpr size_t ba_off_bytes(int NB) { return (size_t)(2 * (NB + 4) + 32) * 4; }

// the items a round reads and writes, stored as two planes per MSM: x[0, cap) then y[0, cap).  The forward kernel reads the
// x plane only, two adjacent coordinates per pair.
template <class B> struct Planes {
  B* x; long long cap;
  __device__ __forceinline__ B ldx(uint32_t pos) const { return ldg_fe(x + pos); }
  __device__ __forceinline__ Aff<B> ld(uint32_t pos) const { Aff<B> p; p.x = ldg_fe(x + pos); p.y = ldg_fe(x + cap + pos); return p; }
  __device__ __forceinline__ void st(uint32_t pos, const Aff<B>& p) const { st_fe(x + pos, p.x); st_fe(x + cap + pos, p.y); }
};
// round 0 reads the window table through entries: e = (table index) | sign << 31
template <class B> __device__ __forceinline__ Aff<B> table_point(const Aff<B>* table, uint32_t e) {
  Aff<B> p = ldg_aff(table + (e & 0x7fffffffu));
  if (e >> 31) p.y = p.y.neg();
  return p;
}
// classification of a pair of two inputs whose x coordinates are equal or zero (the identity is (0, 0)), and its denominator
template <class B> __device__ __forceinline__ int classify_pair(const Aff<B>& p1, const Aff<B>& p2, B& den) {
  if (p2.is_inf()) return PK_COPY1;
  if (p1.is_inf()) return PK_COPY2;
  den = p2.x - p1.x;
  if (!den.is_zero()) return PK_ADD;
  if (p1.y == p2.y && !p1.y.is_zero()) { den = p1.y.dbl(); return PK_DBL; }
  return PK_INF;
}

// ---- 2.0 items per MSM after every round (n_items[k * (R + 1) + r] = sum_b ceil(c_b / 2^r)): lets the CTAs of a round that have
// nothing to do leave before they build any offsets (sparse witness columns leave most of the worst-case grid idle)
__global__ void __launch_bounds__(BA_THREADS) msm_ba_count_kernel(const uint32_t* __restrict__ counts0, int NB, int R, uint32_t* __restrict__ n_items) {
  __shared__ uint32_t red[BA_THREADS / 32];
  const int k = blockIdx.x, t = threadIdx.x;
  for (int r = 0; r <= R; ++r) {
    uint32_t s = 0;
    for (int b = t; b < NB; b += BA_THREADS) s += (counts0[(long long)k * NB + b] + ((1u << r) - 1)) >> r;
    for (int d = 16; d >= 1; d >>= 1) s += __shfl_down_sync(0xffffffffu, s, d);
    if ((t & 31) == 0) red[t >> 5] = s;
    __syncthreads();
    if (t == 0) { uint32_t tot = 0; for (int w = 0; w < BA_THREADS / 32; ++w) tot += red[w]; n_items[(long long)k * (R + 1) + r] = tot; }
    __syncthreads();
  }
}

// ---- 2a. forward: classify every pair, prefix products of the denominators (to global memory), product tree of the CTA (to
// global memory).  A CTA owns BA_M * BA_THREADS consecutive output items of one MSM; thread t owns items Q0 + i * BA_THREADS + t.
// Per item q it stores meta[q] = in0 | kind << META_KIND_SHIFT, and in round 0 the two signed table indices of the pair (eidx),
// so that the backward kernel neither searches nor classifies again and gathers the table points without the entries load.
template <class B, bool FIRST>
__global__ void __launch_bounds__(BA_THREADS) msm_ba_fwd_kernel(const uint32_t* __restrict__ counts0, int NB, int round, const uint32_t* __restrict__ entries,
                                                                 const Aff<B>* __restrict__ table, const B* __restrict__ items_in, long long cap_in, long long cap_out,
                                                                 B* __restrict__ pre, B* __restrict__ tree, uint32_t* __restrict__ meta, uint2* __restrict__ eidx,
                                                                 const uint32_t* __restrict__ n_items, int R) {
  extern __shared__ __align__(16) uint8_t ba_smem[];
  const int k = blockIdx.y, t = threadIdx.x;
  const uint32_t Q0 = blockIdx.x * (BA_M * BA_THREADS);
  if (Q0 >= n_items[(long long)k * (R + 1) + round + 1]) return;   // nothing of this MSM left for this CTA (uniform over the CTA)
  RoundOffsets ro; ro.build(ba_smem, counts0 + (long long)k * NB, NB, round);
  const uint32_t* ent_k = entries + (long long)k * cap_in;
  const Planes<B> in{const_cast<B*>(items_in) + 2 * (long long)k * cap_in, cap_in};
  B* pre_k = pre + 2 * (long long)k * cap_out;   // the y plane of this round's output (see msm_batch_buckets)
  uint32_t* meta_k = meta + (long long)k * cap_out;
  uint2* eidx_k = eidx + (long long)k * cap_out;
  B acc = B::one();
  int hint = 0;
#pragma unroll 1
  for (int i = 0; i < BA_M; ++i) {
    const uint32_t q = Q0 + (uint32_t)i * BA_THREADS + t;
    if (q >= ro.n_next) break;
    uint32_t in0; bool two; ro.locate(q, NB, in0, two, hint);
    st_fe(pre_k + q, acc);
    int kind = PK_COPY1;
    uint2 e = make_uint2(0, 0);
    if (FIRST) { e.x = __ldg(ent_k + in0); if (two) e.y = __ldg(ent_k + in0 + 1); eidx_k[q] = e; }
    if (two) {
      const B x1 = FIRST ? ldg_fe(&table[e.x & 0x7fffffffu].x) : in.ldx(in0), x2 = FIRST ? ldg_fe(&table[e.y & 0x7fffffffu].x) : in.ldx(in0 + 1);
      B den = x2 - x1;
      kind = PK_ADD;
      if (den.is_zero() || x1.is_zero() || x2.is_zero()) {   // equal x (doubling / cancellation) or possibly an identity (0, 0): classify on the full points
        const Aff<B> p1 = FIRST ? table_point(table, e.x) : in.ld(in0), p2 = FIRST ? table_point(table, e.y) : in.ld(in0 + 1);
        kind = classify_pair(p1, p2, den);
      }
      if (kind == PK_ADD || kind == PK_DBL) acc = acc * den;
    }
    meta_k[q] = in0 | (uint32_t)kind << META_KIND_SHIFT;
  }
  __syncthreads();   // the offset arrays are dead: the product tree (heap layout, nd[1] = root, leaves nd[BA_THREADS + t]) takes their place
  B* nd = reinterpret_cast<B*>(ba_smem);
  nd[BA_THREADS + t] = acc;
  __syncthreads();
  for (int w = BA_THREADS >> 1; w >= 1; w >>= 1) {
    if (t < w) nd[w + t] = nd[2 * (w + t)] * nd[2 * (w + t) + 1];
    __syncthreads();
  }
  B* tr = tree + ((long long)k * gridDim.x + blockIdx.x) * (2 * BA_THREADS);
  st_fe(tr + t, t ? nd[t] : B::one()); st_fe(tr + BA_THREADS + t, nd[BA_THREADS + t]);
}

// ---- 2b. the roots of all CTAs are inverted together, one per thread (every lane busy: nobody waits for a lone inversion)
template <class B>
__global__ void msm_ba_inv_kernel(B* __restrict__ tree, uint32_t n_trees) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_trees) return;
  B* root = tree + (size_t)i * (2 * BA_THREADS) + 1;
  st_fe(root, ld_fe(root).inv());
}

// ---- 2c. backward: push the inverted root down the tree, then walk every thread's pairs back and write the sums.
// BA_BWD_MINB resident CTAs per SM (80 registers): faster on H100 than 2 (more registers, fewer warps) or 4 (64 registers, spills).
template <class B, bool FIRST>
__global__ void __launch_bounds__(BA_THREADS, BA_BWD_MINB) msm_ba_bwd_kernel(const Aff<B>* __restrict__ table, const B* __restrict__ items_in, long long cap_in,
                                                                 B* __restrict__ items_out, long long cap_out, const B* __restrict__ tree,
                                                                 const uint32_t* __restrict__ meta, const uint2* __restrict__ eidx, const uint32_t* __restrict__ n_items, int round, int R) {
  extern __shared__ __align__(16) uint8_t ba_smem[];
  const int k = blockIdx.y, t = threadIdx.x;
  const uint32_t Q0 = blockIdx.x * (BA_M * BA_THREADS);
  const uint32_t n_next = n_items[(long long)k * (R + 1) + round + 1];
  if (Q0 >= n_next) return;
  B* nd = reinterpret_cast<B*>(ba_smem);   // [2 * BA_THREADS]
  { const B* tr = tree + ((long long)k * gridDim.x + blockIdx.x) * (2 * BA_THREADS);
    nd[t] = ld_fe(tr + t); nd[BA_THREADS + t] = ld_fe(tr + BA_THREADS + t); }
  __syncthreads();
  for (int w = 1; w < BA_THREADS; w <<= 1) {   // node i in [w, 2w) holds the inverse of its subtree product: inverse(child) = inverse(parent) * product(sibling)
    B child_inv;
    const int node = w + (t >> 1);
    if (t < 2 * w) child_inv = nd[node] * nd[2 * node + ((t & 1) ^ 1)];
    __syncthreads();
    if (t < 2 * w) nd[2 * node + (t & 1)] = child_inv;
    __syncthreads();
  }
  B inv_run = nd[BA_THREADS + t];   // 1 / (product of this thread's denominators)
  const Planes<B> in{const_cast<B*>(items_in) + 2 * (long long)k * cap_in, cap_in}, out{items_out + 2 * (long long)k * cap_out, cap_out};
  const uint32_t* meta_k = meta + (long long)k * cap_out;
  const uint2* eidx_k = eidx + (long long)k * cap_out;
  // the prefix products of the forward kernel sit in the y plane of the output: slot q is read (plain, coherent load) by this
  // thread before it writes out.y[q] over it
  const B* pre_k = out.x + cap_out;
  int last = BA_M - 1;
  while (last >= 0 && Q0 + (uint32_t)last * BA_THREADS + t >= n_next) --last;
#pragma unroll 1
  for (int i = last; i >= 0; --i) {
    const uint32_t q = Q0 + (uint32_t)i * BA_THREADS + t;
    const uint32_t mt = __ldg(meta_k + q);
    const uint2 e = FIRST ? __ldg(eidx_k + q) : make_uint2(0, 0);   // round 0: loaded beside meta, one load before the table gather
    const uint32_t in0 = mt & META_IN0_MASK, kind = mt >> META_KIND_SHIFT;
    const Aff<B> p1 = FIRST ? table_point(table, e.x) : in.ld(in0);
    Aff<B> r;
    if (kind <= PK_DBL) {   // an addition (the common case) or, rarely, a doubling: lambda = num / den
      Aff<B> p2 = p1;
      B num, den;
      if (kind == PK_ADD) { p2 = FIRST ? table_point(table, e.y) : in.ld(in0 + 1); num = p2.y - p1.y; den = p2.x - p1.x; }
      else { const B x2 = p1.x.sqr(); num = x2.dbl() + x2; den = p1.y.dbl(); }
      const B dinv = inv_run * ld_fe(pre_k + q);   // 1 / den
      inv_run = inv_run * den;
      const B lam = num * dinv;
      r.x = lam.sqr() - p1.x - p2.x;
      r.y = lam * (p1.x - r.x) - p1.y;
    } else {   // rare: the identity, a pair that cancels, a bucket's odd item out
      r = p1;
      if (kind == PK_COPY2) r = FIRST ? table_point(table, e.y) : in.ld(in0 + 1);
      else if (kind == PK_INF) r = Aff<B>::inf();
    }
    out.st(q, r);
  }
}

// ---------------------------------------------------------------- 3. what is left in every bucket -> XYZZ bucket sums
template <class B>
__global__ void __launch_bounds__(BA_THREADS) msm_ba_finish_kernel(const uint32_t* __restrict__ counts0, int NB, int round, const B* __restrict__ items, long long cap,
                                                                    Xyzz<B>* __restrict__ buckets) {
  extern __shared__ __align__(16) uint8_t fin_smem[];
  uint32_t* off = reinterpret_cast<uint32_t*>(fin_smem);   // [NB + 1]
  uint32_t* tmp = off + NB + 4;
  const int k = blockIdx.y, t = threadIdx.x;
  for (int b = t; b < NB; b += BA_THREADS) { uint32_t c0 = counts0[(long long)k * NB + b]; off[b] = (c0 + ((1u << round) - 1)) >> round; }
  __syncthreads();
  block_scan_excl(off, NB, tmp);
  const int b = blockIdx.x * BA_THREADS + t;
  if (b >= NB) return;
  Xyzz<B> acc = Xyzz<B>::inf();
  const Planes<B> it{const_cast<B*>(items) + 2 * (long long)k * cap, cap};
  for (uint32_t p = off[b]; p < off[b + 1]; ++p) acc.add_affine(it.ld(p));
  buckets[(long long)k * NB + b] = acc;
}

// ---------------------------------------------------------------- host driver
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn encode_tiled_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr; cudaDriverEntryPointQueryResult qr;
    TB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr));
    if (qr != cudaDriverEntryPointSuccess || !p) throw CudaError("cuTensorMapEncodeTiled is not available from this driver");
    fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// one reduction round = forward, root inversion, backward
template <class B, bool FIRST>
static void launch_round(Ctx* ctx, dim3 grid, size_t fwd_smem, size_t bwd_smem, const uint32_t* counts, int NB, int r, const uint32_t* entries, const Aff<B>* table, const B* in,
                         long long cap_in, B* out, long long cap_out, B* pre, B* tree, uint32_t* meta, uint2* eidx, const uint32_t* n_items, int R, uint32_t n_trees) {
  ctx->opt_in_smem(msm_ba_fwd_kernel<B, FIRST>, fwd_smem);
  ctx->opt_in_smem(msm_ba_bwd_kernel<B, FIRST>, bwd_smem);
  launch(ctx, msm_ba_fwd_kernel<B, FIRST>, grid, BA_THREADS, fwd_smem, counts, NB, r, entries, table, in, cap_in, cap_out, pre, tree, meta, eidx, n_items, R);
  launch(ctx, msm_ba_inv_kernel<B>, (n_trees + 63) / 64, 64, 0, tree, n_trees);
  launch(ctx, msm_ba_bwd_kernel<B, FIRST>, grid, BA_THREADS, bwd_smem, table, in, cap_in, out, cap_out, tree, meta, eidx, n_items, r, R);
}

bool msm_batch_applicable(int N, int K, const MsmConfig& cfg, int c) {
  if (cfg.table_windows <= 0 || (1 << (c - 1)) > BA_MAX_NB || c < 6) return false;
  const long long min_terms = tb_tune("TB_MSM_BA_MIN_TERMS", 1 << 21);
  return (long long)N * K >= min_terms;
}

// bucket sums of K fixed-base MSMs (all windows of an MSM share NB buckets): buckets[k * NB + b], XYZZ
template <class B, class S>
void msm_batch_buckets(Ctx* ctx, const S* scalars, long long sstride, const Aff<B>* table, int N, int K, int c, int W, int table_stride, const S* extras, int n_extra,
                       Xyzz<B>* buckets) {
  const int NB = 1 << (c - 1);
  TB_REQUIRE(((uintptr_t)scalars & 15) == 0 && (sstride * (long long)sizeof(S)) % 16 == 0, "scalar vectors must be 16-byte aligned for TMA");
  const long long cap0 = (long long)(N + n_extra) * W;
  std::vector<long long> cap(1, cap0);
  const int R = tb_tune("TB_MSM_BA_ROUNDS", 10);
  TB_REQUIRE(R >= 1 && R <= 20, "TB_MSM_BA_ROUNDS out of range");
  for (int r = 0; r < R; ++r) cap.push_back((cap.back() + NB + 1) / 2);
  TB_REQUIRE(cap0 <= (long long)META_IN0_MASK + 1, "too many MSM entries for the pair index of meta");
  // MSMs per chunk: one wave of the sort kernel (one 1024-thread CTA per SM).  A chunk's temporaries take ~36 MB per MSM
  // from the stream-ordered pool, which keeps them cached: ~4.8 GB per proving stream on H100 at this size.
  const int Kc_max = tb_tune("TB_MSM_BA_CHUNK", ctx->sm_count);
  const int Kc = K < Kc_max ? K : Kc_max;
  DevBuf<uint32_t> counts(ctx, (size_t)Kc * NB), entries(ctx, (size_t)Kc * cap0);
  // round items as x / y planes (2 * cap field elements per MSM).  The prefix products of a round live in the y plane of its
  // output until the backward kernel overwrites them (each slot is read, then written, by the same thread).  itB is free
  // during round 0 and holds its table indices (8 B per output item, a quarter of a field element).
  const size_t eidx_fe = ((size_t)Kc * cap[1] + 3) / 4;
  DevBuf<B> itA(ctx, (size_t)Kc * 2 * cap[1]), itB(ctx, std::max(R > 1 ? (size_t)(Kc * 2 * cap[2]) : (size_t)0, eidx_fe));
  uint2* eidx = reinterpret_cast<uint2*>(itB.get());
  const size_t sort_smem = 2 * SORT_TILE * sizeof(S) + 16 + (size_t)(NB + 1 + 32) * 4 + 16;
  const size_t fwd_smem = std::max(ba_off_bytes(NB), (size_t)2 * BA_THREADS * sizeof(B));
  const size_t bwd_smem = (size_t)2 * BA_THREADS * sizeof(B);
  const size_t fin_smem = (size_t)(NB + 4 + 32) * 4;
  ctx->opt_in_smem(msm_sort_kernel<S, 13>, sort_smem);
  ctx->opt_in_smem(msm_sort_kernel<S, 0>, sort_smem);
  ctx->opt_in_smem(msm_ba_finish_kernel<B>, fin_smem);
  const long long pairs_per_cta = (long long)BA_M * BA_THREADS;
  const unsigned ctas1 = (unsigned)((cap[1] + pairs_per_cta - 1) / pairs_per_cta);
  DevBuf<B> tree(ctx, (size_t)Kc * ctas1 * 2 * BA_THREADS);
  DevBuf<uint32_t> meta(ctx, (size_t)Kc * cap[1]), n_items(ctx, (size_t)Kc * (R + 1));
  for (int k0 = 0; k0 < K; k0 += Kc) {
    const int kc = K - k0 < Kc ? K - k0 : Kc;
    { ProfScope ps(ctx, PC_MSM_SORT);
      // 3-D tensor over the scalar vectors of this chunk: [kc][N][8 x u32], box = 8 x SORT_BOX x 1
      CUtensorMap smap;
      const cuuint64_t dims[3] = {8, (cuuint64_t)N, (cuuint64_t)kc};
      const cuuint64_t strides[2] = {sizeof(S), (cuuint64_t)sstride * sizeof(S)};
      const cuuint32_t box[3] = {8, SORT_BOX, 1}, estr[3] = {1, 1, 1};
      CUresult cr = encode_tiled_fn()(&smap, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<S*>(scalars + (long long)k0 * sstride), dims, strides, box, estr,
                                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
      if (cr != CUDA_SUCCESS) throw CudaError("cuTensorMapEncodeTiled failed for the scalar tensor (" + std::to_string((int)cr) + ")");
      const S* ex = extras ? extras + (long long)k0 * n_extra : nullptr;
      if (c == 13) launch(ctx, msm_sort_kernel<S, 13>, kc, SORT_THREADS, sort_smem, smap, ex, N, extras ? n_extra : 0, c, W, NB, table_stride, counts.get(), entries.get(), cap0, ctx->d_msm_adds.get());
      else launch(ctx, msm_sort_kernel<S, 0>, kc, SORT_THREADS, sort_smem, smap, ex, N, extras ? n_extra : 0, c, W, NB, table_stride, counts.get(), entries.get(), cap0, ctx->d_msm_adds.get()); }
    { ProfScope ps(ctx, PC_MSM_ACCUM);
      launch(ctx, msm_ba_count_kernel, kc, BA_THREADS, 0, counts.get(), NB, R, n_items.get());
      for (int r = 0; r < R; ++r) {
        const B* in = (r & 1) ? itA.get() : itB.get();   // round r reads what round r-1 wrote (r = 0 reads the entries)
        B* out = (r & 1) ? itB.get() : itA.get();
        const unsigned gx = (unsigned)((cap[r + 1] + pairs_per_cta - 1) / pairs_per_cta);
        dim3 grid(gx, kc);
        const uint32_t n_trees = gx * (uint32_t)kc;
        (r == 0 ? launch_round<B, true> : launch_round<B, false>)(ctx, grid, fwd_smem, bwd_smem, counts.get(), NB, r, entries.get(), table, in, r == 0 ? cap0 : cap[r], out,
                                                                  cap[r + 1], out + cap[r + 1], tree.get(), meta.get(), eidx, n_items.get(), R, n_trees);
      }
      const B* last = (R & 1) ? itA.get() : itB.get();
      launch(ctx, msm_ba_finish_kernel<B>, dim3((NB + BA_THREADS - 1) / BA_THREADS, kc), BA_THREADS, fin_smem, counts.get(), NB, R, last, cap[R], buckets + (size_t)k0 * NB); }
  }
}

template void msm_batch_buckets<Fq, Fp>(Ctx*, const Fp*, long long, const Aff<Fq>*, int, int, int, int, int, const Fp*, int, Xyzz<Fq>*);
template void msm_batch_buckets<Fp, Fq>(Ctx*, const Fq*, long long, const Aff<Fp>*, int, int, int, int, int, const Fq*, int, Xyzz<Fp>*);

}  // namespace tb
