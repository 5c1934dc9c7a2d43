// Pippenger multi-scalar multiplication over the Pasta curves for sm_90a.
//
// Replaces halo2_proofs `arithmetic::best_multiexp` and `Params::{commit, commit_lagrange}` (EXT, called under
// taiga_halo2/src/proof.rs:33-40; SURVEY.md §8a row H1, App. E.4).  Two modes share one pipeline:
//   * variable-base (standalone sweep, IPA rounds): W = ceil(256/c) windows, one bucket set per window;
//   * fixed-base (every commitment of the prover: bases are the SRS `g` / `g_lagrange`): the bases were premultiplied
//     by 2^(c*w) at SRS load, so all windows share ONE bucket set and the final Horner over windows disappears.
// Pipeline: signed-digit extraction + bucket histogram -> exclusive scan -> scatter of (point index, sign) into
// bucket-sorted order -> bucket accumulation (one thread per <=64-entry unit, XYZZ mixed adds; oversized buckets are
// split into units and combined by a CTA with warp-shuffle reduction) -> per-window running-sum reduction (segments,
// warp-shuffle tree) -> Horner over windows.
//
// Algorithmic bytes: 96*N per MSM (64 B affine base + 32 B scalar); fixed-base batched: 64*N*W (tables) + 32*N*K.
#include <memory>
#include "common.cuh"
#include "kernels.cuh"

namespace tb {

constexpr int MSM_CHUNK_MAX = 64;  // max entries accumulated by one thread (adaptive: chosen so the accumulation fills the GPU)
constexpr int MSM_UNITS_PER_SM = 2048;       // accumulation units aimed at per SM when choosing the chunk
constexpr int MSM_SUB_WARPS_PER_SM = 16;     // warps per SM the sub-warp combine aims at when choosing its lanes per bucket
constexpr int MSM_SEG = 8;         // buckets per thread in the running-sum reduction
constexpr uint32_t MSM_HEAVY_UNITS = 1024;  // buckets with more units than this get a whole CTA (e.g. the top window of a variable-base MSM)

// variable-base window from the MSM length (fixed-base callers pass the c their tables were built with)
static int msm_default_window(int n) {
  int lg = 0; while ((1 << (lg + 1)) <= n) ++lg;
  int c = lg - 4;
  if (c < 4) c = 4;
  if (c > 16) c = 16;
  return c;
}

__device__ __forceinline__ uint32_t window_bits(const uint32_t* s, int bit, int c) {
  int limb = bit >> 5, off = bit & 31;
  uint64_t v = s[limb];
  if (limb + 1 < 8) v |= (uint64_t)s[limb + 1] << 32;
  return (uint32_t)(v >> off) & ((1u << c) - 1);
}

// MODE 0: histogram, MODE 1: scatter
template <class S, int MODE>
__global__ void msm_digits_kernel(const S* __restrict__ scalars, long long sstride, int N, int c, int W, int NB, int wsep,
                                  int table_mode, int table_stride, const S* __restrict__ extras, int n_extra,
                                  uint32_t* __restrict__ counts_or_cursor, uint32_t* __restrict__ entries) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int k = blockIdx.y;
  if (i >= N + n_extra) return;
  // terms N .. N+n_extra-1 are the extra (scalar, base) pairs appended to the fixed-base table (blind * w, value * u)
  S s = (i < N ? ldg_fe(scalars + (long long)k * sstride + i) : ldg_fe(extras + (long long)k * n_extra + (i - N))).from_mont();
  if (s.is_zero()) return;
  const uint32_t half = 1u << (c - 1);
  uint32_t carry = 0;
  for (int w = 0; w < W; ++w) {
    uint32_t v = window_bits(s.l, w * c, c) + carry;
    uint32_t neg = 0;
    if (v > half) { v = (1u << c) - v; neg = 1; carry = 1; } else carry = 0;
    if (v) {
      uint32_t b = ((uint32_t)k * wsep + (wsep > 1 ? w : 0)) * NB + (v - 1);
      if (MODE == 0) atomicAdd(&counts_or_cursor[b], 1u);
      else {
        uint32_t pos = atomicAdd(&counts_or_cursor[b], 1u);
        entries[pos] = (table_mode ? (uint32_t)(w * table_stride + i) : (uint32_t)i) | (neg << 31);
      }
    }
  }
}

// units (chunks of <= chunk entries) per bucket; buckets too large for the sub-warp combine go to the mid list (one warp
// each), oversized ones to the heavy list (one CTA each)
__global__ void msm_units_kernel(const uint32_t* __restrict__ offs, uint32_t nb_total, uint32_t chunk_log, uint32_t sub_units, uint32_t* __restrict__ unit_count,
                                 uint32_t* __restrict__ mid, uint32_t* __restrict__ heavy, uint32_t* __restrict__ n_lists /* [0] mid, [1] heavy */) {
  uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= nb_total) return;
  uint32_t cnt = offs[b + 1] - offs[b];
  uint32_t uc = (cnt + (1u << chunk_log) - 1) >> chunk_log;
  unit_count[b] = uc;
  if (uc > MSM_HEAVY_UNITS) heavy[atomicAdd(n_lists + 1, 1u)] = b;
  else if (uc > sub_units) mid[atomicAdd(n_lists, 1u)] = b;
}

template <class B>
__global__ void __launch_bounds__(128, 4) msm_accum_kernel(const Aff<B>* __restrict__ bases, long long base_bstride, uint32_t buckets_per_item,
                                 const uint32_t* __restrict__ offs, const uint32_t* __restrict__ unit_off, uint32_t nb_total, uint32_t chunk,
                                 const uint32_t* __restrict__ entries, Xyzz<B>* __restrict__ partial) {
  uint32_t u = blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= unit_off[nb_total]) return;
  // largest b with unit_off[b] <= u
  uint32_t lo = 0, hi = nb_total;
  while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (unit_off[mid] <= u) lo = mid; else hi = mid; }
  uint32_t b = lo, j = u - unit_off[b];
  uint32_t beg = offs[b] + j * chunk, end = offs[b + 1];
  if (end > beg + chunk) end = beg + chunk;
  const Aff<B>* pts = bases + (long long)(b / buckets_per_item) * base_bstride;
  Xyzz<B> acc = Xyzz<B>::inf();
  for (uint32_t e = beg; e < end; ++e) {
    uint32_t pl = __ldg(entries + e);
    Aff<B> p = ldg_aff(pts + (pl & 0x7fffffffu));
    if (pl >> 31) p.y = p.y.neg();
    acc.add_affine(p);
  }
  partial[u] = acc;
}

template <class B> __device__ __forceinline__ Xyzz<B> shfl_down_pt(const Xyzz<B>& p, int delta) {
  Xyzz<B> r;
  const uint32_t* src = reinterpret_cast<const uint32_t*>(&p);
  uint32_t* dst = reinterpret_cast<uint32_t*>(&r);
#pragma unroll
  for (int i = 0; i < 32; ++i) dst[i] = __shfl_down_sync(0xffffffffu, src[i], delta);
  return r;
}

// sum over a 256-thread CTA; result valid in thread 0
template <class B> __device__ Xyzz<B> block_reduce_pt(Xyzz<B> v, Xyzz<B>* sm /* 8 slots */) {
  for (int d = 16; d >= 1; d >>= 1) { Xyzz<B> o = shfl_down_pt(v, d); v.add(o); }
  int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) sm[warp] = v;
  __syncthreads();
  if (warp == 0) {
    v = (lane < (int)(blockDim.x >> 5)) ? sm[lane] : Xyzz<B>::inf();
    for (int d = 4; d >= 1; d >>= 1) { Xyzz<B> o = shfl_down_pt(v, d); v.add(o); }
  }
  return v;
}

// one warp per mid-list bucket (grid-stride): sum the partial results of its units (warp-shuffle tree)
template <class B>
__global__ void __launch_bounds__(256) msm_combine_kernel(const uint32_t* __restrict__ mid, const uint32_t* __restrict__ n_mid, const uint32_t* __restrict__ unit_off,
                                                           const Xyzz<B>* __restrict__ partial, Xyzz<B>* __restrict__ buckets) {
  const uint32_t lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5, nm = *n_mid;
  for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < nm; w += nw) {
    const uint32_t b = mid[w], u0 = unit_off[b], u1 = unit_off[b + 1];
    Xyzz<B> acc = Xyzz<B>::inf();
    for (uint32_t u = u0 + lane; u < u1; u += 32) acc.add(partial[u]);
    for (int d = 16; d >= 1; d >>= 1) { Xyzz<B> o = shfl_down_pt(acc, d); acc.add(o); }
    if (lane == 0) buckets[b] = acc;
  }
}

// 2^lpb_log lanes per bucket (1, 2, .. 32): every add a warp issues costs the same whether 1 or 32 of its lanes are live, so a
// full warp per bucket spends as many issue slots on the tree as the accumulation itself when buckets hold ~10 units.  The
// host picks the narrowest group that still leaves a few warps per SM sub-partition; buckets with more than 4 * lanes units are
// left to the warp / heavy kernels.
template <class B>
__global__ void __launch_bounds__(128) msm_combine_sub_kernel(const uint32_t* __restrict__ unit_off, const Xyzz<B>* __restrict__ partial, uint32_t nb_total,
                                                               uint32_t lpb_log, Xyzz<B>* __restrict__ buckets) {
  const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x, lpb = 1u << lpb_log;
  const uint32_t b = gt >> lpb_log, l = gt & (lpb - 1);
  uint32_t u0 = 0, u1 = 0;
  if (b < nb_total) { u0 = unit_off[b]; u1 = unit_off[b + 1]; }
  const bool mine = b < nb_total && (u1 - u0) <= (4u << lpb_log);
  Xyzz<B> acc = Xyzz<B>::inf();
  if (mine) for (uint32_t u = u0 + l; u < u1; u += lpb) acc.add(partial[u]);
  for (uint32_t d = lpb >> 1; d >= 1; d >>= 1) {
    Xyzz<B> o;
    { const uint32_t* src = reinterpret_cast<const uint32_t*>(&acc); uint32_t* dst = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int i = 0; i < 32; ++i) dst[i] = __shfl_down_sync(0xffffffffu, src[i], d, lpb); }
    if (l < d) acc.add(o);
  }
  if (mine && l == 0) buckets[b] = acc;
}

// one CTA per oversized bucket (grid-stride over the heavy list)
template <class B>
__global__ void __launch_bounds__(256) msm_combine_heavy_kernel(const uint32_t* __restrict__ heavy, const uint32_t* __restrict__ n_heavy,
                                                                 const uint32_t* __restrict__ unit_off, const Xyzz<B>* __restrict__ partial,
                                                                 Xyzz<B>* __restrict__ buckets) {
  __shared__ Xyzz<B> sm[8];
  const uint32_t nh = *n_heavy;
  for (uint32_t h = blockIdx.x; h < nh; h += gridDim.x) {
    uint32_t b = heavy[h], u0 = unit_off[b], u1 = unit_off[b + 1];
    Xyzz<B> acc = Xyzz<B>::inf();
    for (uint32_t u = u0 + threadIdx.x; u < u1; u += blockDim.x) acc.add(partial[u]);
    acc = block_reduce_pt(acc, sm);
    if (threadIdx.x == 0) buckets[b] = acc;
    __syncthreads();
  }
}

// running-sum reduction of one segment of `seg` buckets: sum_b (b+1) * bucket_b restricted to the segment
template <class B>
__global__ void __launch_bounds__(128) msm_segsum_kernel(const Xyzz<B>* __restrict__ buckets, int NB, int seg, int nt, uint32_t groups,
                                                          Xyzz<B>* __restrict__ seg_out) {
  uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= groups * (uint32_t)nt) return;
  uint32_t g = id / nt, t = id % nt;
  const Xyzz<B>* bk = buckets + (size_t)g * NB + (size_t)t * seg;
  Xyzz<B> run = Xyzz<B>::inf(), acc = Xyzz<B>::inf();
  for (int j = seg - 1; j >= 0; --j) { run.add(bk[j]); acc.add(run); }
  // + (t*seg) * run
  uint32_t m = t * seg;
  if (m && !run.is_inf()) {
    Xyzz<B> r = Xyzz<B>::inf();
    for (int bit = 31 - __clz(m); bit >= 0; --bit) { r = r.dbl(); if ((m >> bit) & 1) r.add(run); }
    acc.add(r);
  }
  seg_out[id] = acc;
}

// fused variant for nt <= 256 segments (<= 2 warps per SM sub-partition, so the latency-bound chains run at full issue rate): one CTA per bucket set does the running sums AND the tree; thread 0 optionally
// normalises to affine (saves two launches and a global round trip per commitment)
template <class B>
__global__ void __launch_bounds__(256) msm_bucket_reduce_kernel(const Xyzz<B>* __restrict__ buckets, int NB, int seg, int nt,
                                                                   Xyzz<B>* __restrict__ out, Aff<B>* __restrict__ aff_out) {
  __shared__ Xyzz<B> sm[32];
  const uint32_t g = blockIdx.x, t = threadIdx.x;
  Xyzz<B> acc = Xyzz<B>::inf();
  if ((int)t < nt) {
    const Xyzz<B>* bk = buckets + (size_t)g * NB + (size_t)t * seg;
    Xyzz<B> run = Xyzz<B>::inf();
    for (int j = seg - 1; j >= 0; --j) { run.add(bk[j]); acc.add(run); }
    uint32_t m = t * seg;
    if (m && !run.is_inf()) {
      Xyzz<B> r = Xyzz<B>::inf();
      for (int bit = 31 - __clz(m); bit >= 0; --bit) { r = r.dbl(); if ((m >> bit) & 1) r.add(run); }
      acc.add(r);
    }
  }
  for (int d = 16; d >= 1; d >>= 1) { Xyzz<B> o = shfl_down_pt(acc, d); acc.add(o); }
  const int warp = t >> 5, lane = t & 31, nwarps = (blockDim.x + 31) >> 5;
  if (lane == 0) sm[warp] = acc;
  __syncthreads();
  if (warp == 0) {
    acc = lane < nwarps ? sm[lane] : Xyzz<B>::inf();
    for (int d = 16; d >= 1; d >>= 1) { Xyzz<B> o = shfl_down_pt(acc, d); acc.add(o); }
    if (lane == 0) { out[g] = acc; if (aff_out) aff_out[g] = acc.to_affine(); }
  }
}

// ---- weighted bucket sum for one window set, two-level: b = hi * S + lo (S = 2^s_log columns, H = NB / S rows)
//   sum_b (b+1) B_b = sum_lo (lo+1) C_lo + S * sum_hi hi * R_hi,   C_lo = sum_hi B[hi][lo],  R_hi = sum_lo B[hi][lo]
// and sum_j (j+1) C_j = sum_j Suffix_j(C), sum_j j R_j = sum_{j>=1} Suffix_j(R).  Every step is a tree: the dependent chain is
// ~27 point additions (line sums 8, suffix scan 6, tree 6, 6 doublings, 1) against ~46 for running sums + a 12-bit scalar
// multiple per thread + a block tree -- these kernels are pure latency (one launch per commitment / IPA round).
//
// kernel 1: the S column sums and H row sums of every group, 16 lanes per line
template <class B>
__global__ void __launch_bounds__(128) msm_linesum_kernel(const Xyzz<B>* __restrict__ buckets, int NB, int s_log, uint32_t groups,
                                                           Xyzz<B>* __restrict__ lines) {
  const int S = 1 << s_log, H = NB >> s_log, nl = S + H;
  const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x, line = gt >> 4, l = gt & 15;
  const bool live = line < groups * (uint32_t)nl;
  Xyzz<B> acc = Xyzz<B>::inf();
  if (live) {
    const uint32_t g = line / nl, L = line % nl;
    const Xyzz<B>* bk = buckets + (size_t)g * NB;
    if ((int)L < S) { for (int hi = l; hi < H; hi += 16) acc.add(bk[(size_t)hi * S + L]); }
    else { const Xyzz<B>* row = bk + (size_t)(L - S) * S; for (int lo = l; lo < S; lo += 16) acc.add(row[lo]); }
  }
  for (int d = 8; d >= 1; d >>= 1) {
    Xyzz<B> o;
    { const uint32_t* src = reinterpret_cast<const uint32_t*>(&acc); uint32_t* dst = reinterpret_cast<uint32_t*>(&o);
#pragma unroll
      for (int i = 0; i < 32; ++i) dst[i] = __shfl_down_sync(0xffffffffu, src[i], d, 16); }
    if ((int)l < d) acc.add(o);
  }
  if (live && l == 0) lines[line] = acc;
}
// kernel 2: one CTA per group, blockDim = 2 * max(S, H): suffix scans of the two line vectors, their totals, the final
// combination and (optionally) the normalisation to affine
template <class B>
__global__ void __launch_bounds__(256) msm_weighted_kernel(const Xyzz<B>* __restrict__ lines, int s_log, int h_log, Xyzz<B>* __restrict__ out, Aff<B>* __restrict__ aff_out) {
  extern __shared__ uint4 mw_smem[];
  Xyzz<B>* sm = reinterpret_cast<Xyzz<B>*>(mw_smem);
  const int S = 1 << s_log, H = 1 << h_log, half = blockDim.x >> 1;
  const int part = threadIdx.x >= (unsigned)half, j = threadIdx.x - part * half, len = part ? H : S;
  const Xyzz<B>* src = lines + (size_t)blockIdx.x * (S + H) + (part ? S : 0);
  Xyzz<B>* v = sm + part * half;
  Xyzz<B> acc = j < len ? src[j] : Xyzz<B>::inf();
  v[j] = acc;
  __syncthreads();
  for (int d = 1; d < half; d <<= 1) {   // suffix scan (Hillis-Steele)
    const bool act = j + d < len;
    Xyzz<B> o;
    if (act) o = v[j + d];
    __syncthreads();
    if (act) { acc.add(o); v[j] = acc; }
    __syncthreads();
  }
  if (part && j == 0) v[0] = Xyzz<B>::inf();   // rows are weighted hi, not hi + 1
  __syncthreads();
  for (int d = half >> 1; d >= 1; d >>= 1) {   // totals of the suffixes
    if (j < d) { Xyzz<B> a = v[j]; a.add(v[j + d]); v[j] = a; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    Xyzz<B> r = sm[half];
    for (int i = 0; i < s_log; ++i) r = r.dbl();
    r.add(sm[0]);
    out[blockIdx.x] = r;
    if (aff_out) aff_out[blockIdx.x] = r.to_affine();
  }
}

template <class B>
__global__ void __launch_bounds__(256) msm_window_kernel(const Xyzz<B>* __restrict__ seg_out, int nt, Xyzz<B>* __restrict__ win_out) {
  __shared__ Xyzz<B> sm[8];
  uint32_t g = blockIdx.x;
  Xyzz<B> acc = Xyzz<B>::inf();
  for (int t = threadIdx.x; t < nt; t += blockDim.x) acc.add(seg_out[(size_t)g * nt + t]);
  acc = block_reduce_pt(acc, sm);
  if (threadIdx.x == 0) win_out[g] = acc;
}

template <class B>
__global__ void msm_horner_kernel(const Xyzz<B>* __restrict__ win, int wsep, int c, int K, Xyzz<B>* __restrict__ out) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= K) return;
  Xyzz<B> acc = win[(size_t)k * wsep + wsep - 1];
  for (int w = wsep - 2; w >= 0; --w) {
    for (int i = 0; i < c; ++i) acc = acc.dbl();
    acc.add(win[(size_t)k * wsep + w]);
  }
  out[k] = acc;
}

template <class B, class S>
void msm_run(Ctx* ctx, const S* scalars, long long scalar_bstride, const Aff<B>* bases, long long base_bstride, int N, int K,
             const MsmConfig& cfg_in, Xyzz<B>* out) {
  TB_REQUIRE(N >= 1 && K >= 1 && K <= 65535, "MSM shape out of range");
  const bool table_mode = cfg_in.table_windows > 0;
  int c = cfg_in.c ? cfg_in.c : msm_default_window(N);
  TB_REQUIRE(c >= 2 && c <= 20, "MSM window out of range");
  const int W = (256 + c - 1) / c;
  if (table_mode) TB_REQUIRE(cfg_in.table_windows >= W, "fixed-base table has too few windows");
  const int NB = 1 << (c - 1);
  const int wsep = table_mode ? 1 : W;
  const uint64_t nb_total64 = (uint64_t)K * wsep * NB;
  const int n_extra = table_mode ? cfg_in.n_extra : 0;
  const int table_stride = table_mode ? (cfg_in.table_stride ? cfg_in.table_stride : N) : 0;
  const uint64_t max_entries = (uint64_t)K * (N + n_extra) * W;
  TB_REQUIRE(nb_total64 < (1ull << 31) && max_entries < (1ull << 32) && (uint64_t)(N + 2) * (table_mode ? W : 1) < (1ull << 31), "MSM too large");
  const uint32_t nb_total = (uint32_t)nb_total64;
  cudaStream_t st = ctx->stream;

  DevBuf<Xyzz<B>> buckets(ctx, nb_total);
  ctx->work[PC_MSM_SORT] += 2.0 * (double)K * (N + n_extra);                      // two passes of from_mont over the scalars
  ctx->work[PC_MSM_REDUCE] += (double)K * wsep * NB * 30.0;                       // ~2 full XYZZ additions (14 M) per bucket + the weighted tail
  std::unique_ptr<ProfScope> ps;
  if (msm_batch_applicable(N, K, cfg_in, c)) {
    // throughput path: shared-memory counting sort per MSM + batch-affine pairwise reduction (msm_batch.cu)
    msm_batch_buckets<B, S>(ctx, scalars, scalar_bstride, bases, N, K, c, W, table_stride, reinterpret_cast<const S*>(cfg_in.extra_scalars), n_extra, buckets.get());
  } else {
    DevBuf<uint32_t> counts(ctx, nb_total), offs(ctx, nb_total + 1), cursor(ctx, nb_total), entries(ctx, max_entries);
    ps.reset(new ProfScope(ctx, PC_MSM_SORT));
    counts.zero();
    dim3 dg((N + n_extra + 255) / 256, K);
    const S* extras = reinterpret_cast<const S*>(cfg_in.extra_scalars);
    launch(ctx, msm_digits_kernel<S, 0>, dg, 256, 0, scalars, scalar_bstride, N, c, W, NB, wsep, table_mode, table_stride, extras, n_extra, counts.get(), nullptr);
    exclusive_scan_u32(ctx, counts.get(), offs.get(), nb_total);
    TB_CUDA(cudaMemcpyAsync(cursor.get(), offs.get(), nb_total * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
    launch(ctx, msm_digits_kernel<S, 1>, dg, 256, 0, scalars, scalar_bstride, N, c, W, NB, wsep, table_mode, table_stride, extras, n_extra, cursor.get(), entries.get());

    // adaptive chunk: aim at ~4 waves of 512 threads per SM so that small batches still fill the machine
    uint32_t chunk_log = 3;
    { const uint64_t target_units = (uint64_t)MSM_UNITS_PER_SM * (uint64_t)ctx->sm_count;
      while ((1u << chunk_log) < (uint32_t)MSM_CHUNK_MAX && (max_entries >> chunk_log) > target_units) ++chunk_log; }
    const uint64_t max_units = nb_total64 + (max_entries >> chunk_log) + 1;
    const uint64_t max_heavy = (max_entries >> chunk_log) / MSM_HEAVY_UNITS + 1;
    // three disjoint classes of buckets: <= 4 * lanes units (a group of `lanes` threads), <= 1024 units (one warp), more (one
    // CTA each).  lanes: as wide as keeps ~4 warps per SM sub-partition busy, no wider than the average bucket needs.
    uint32_t lpb_log = 0;
    { const uint64_t avg_units = ((max_entries >> chunk_log) + nb_total64 - 1) / nb_total64;
      const uint64_t warps_target = (uint64_t)MSM_SUB_WARPS_PER_SM * (uint64_t)ctx->sm_count;
      while (lpb_log < 5 && ((nb_total64 << (lpb_log + 1)) >> 5) <= warps_target && (1ull << lpb_log) < avg_units) ++lpb_log; }
    const uint32_t sub_units = 4u << lpb_log;
    uint64_t max_mid = (max_entries >> chunk_log) / sub_units + 1;   // buckets with more than sub_units * chunk entries
    if (max_mid > nb_total64) max_mid = nb_total64;
    DevBuf<uint32_t> unit_count(ctx, nb_total), unit_off(ctx, nb_total + 1), mid(ctx, max_mid), heavy(ctx, max_heavy), n_lists(ctx, 2);
    n_lists.zero();
    launch(ctx, msm_units_kernel, (nb_total + 255) / 256, 256, 0, offs.get(), nb_total, chunk_log, sub_units, unit_count.get(), mid.get(), heavy.get(), n_lists.get());
    exclusive_scan_u32(ctx, unit_count.get(), unit_off.get(), nb_total);
    DevBuf<Xyzz<B>> partial(ctx, max_units);
    ctx->work[PC_MSM_ACCUM] += 10.5 * (double)max_entries * 0.97;                 // XYZZ mixed additions (upper bound: every digit non-zero)
    ps.reset(); ps.reset(new ProfScope(ctx, PC_MSM_ACCUM));
    launch(ctx, msm_accum_kernel<B>, (unsigned)((max_units + 127) / 128), 128, 0, bases, base_bstride, (uint32_t)wsep * NB, offs.get(), unit_off.get(), nb_total,
           1u << chunk_log, entries.get(), partial.get());
    ps.reset(); ps.reset(new ProfScope(ctx, PC_MSM_REDUCE));
    launch(ctx, msm_combine_sub_kernel<B>, (unsigned)((((uint64_t)nb_total << lpb_log) + 127) / 128), 128, 0, unit_off.get(), partial.get(), nb_total, lpb_log,
           buckets.get());
    { uint64_t g = (max_mid + 7) / 8, cap = 4ull * (uint64_t)ctx->sm_count;   // e.g. a witness column that is mostly small values
      launch(ctx, msm_combine_kernel<B>, (unsigned)(g < cap ? g : cap), 256, 0, mid.get(), n_lists.get(), unit_off.get(), partial.get(), buckets.get()); }
    if ((max_entries >> chunk_log) > MSM_HEAVY_UNITS)  // e.g. the top window of a variable-base MSM, or a witness column that is mostly ones
      launch(ctx, msm_combine_heavy_kernel<B>, (unsigned)(max_heavy < 296 ? max_heavy : 296), 256, 0, heavy.get(), n_lists.get() + 1, unit_off.get(), partial.get(), buckets.get());
    ps.reset();
  }
  ps.reset(new ProfScope(ctx, PC_MSM_REDUCE));

  const int seg = NB < MSM_SEG ? NB : MSM_SEG;
  const int nt = NB / seg;
  const uint32_t groups = (uint32_t)K * wsep;
  Aff<B>* const aff_out = reinterpret_cast<Aff<B>*>(cfg_in.affine_out);
  if (wsep == 1 && NB < 64) {
    int threads = ((nt + 31) / 32) * 32;
    launch(ctx, msm_bucket_reduce_kernel<B>, groups, threads, 0, buckets.get(), NB, seg, nt, out, aff_out);
    return;
  }
  if (wsep == 1) {
    const int lb = c - 1, s_log = (lb + 1) / 2, h_log = lb - s_log;
    const int nl = (1 << s_log) + (1 << h_log), threads = 2 << s_log;
    TB_REQUIRE(threads <= 256, "fixed-base window too wide for the weighted-sum kernel (c <= 15)");
    DevBuf<Xyzz<B>> lines(ctx, (size_t)groups * nl);
    launch(ctx, msm_linesum_kernel<B>, (unsigned)(((uint64_t)groups * nl * 16 + 127) / 128), 128, 0, buckets.get(), NB, s_log, groups, lines.get());
    const size_t smem = (size_t)threads * sizeof(Xyzz<B>);
    if (smem > 48 * 1024) {
      ctx->opt_in_smem(msm_weighted_kernel<B>, 128 * 1024);
    }
    launch(ctx, msm_weighted_kernel<B>, groups, threads, smem, lines.get(), s_log, h_log, out, aff_out);
    return;
  }
  DevBuf<Xyzz<B>> seg_out(ctx, (size_t)groups * nt), win(ctx, groups);
  launch(ctx, msm_segsum_kernel<B>, (groups * nt + 127) / 128, 128, 0, buckets.get(), NB, seg, nt, groups, seg_out.get());
  launch(ctx, msm_window_kernel<B>, groups, 256, 0, seg_out.get(), nt, win.get());
  launch(ctx, msm_horner_kernel<B>, (K + 31) / 32, 32, 0, win.get(), wsep, c, K, out);
}

template void msm_run<Fq, Fp>(Ctx*, const Fp*, long long, const Aff<Fq>*, long long, int, int, const MsmConfig&, Xyzz<Fq>*);
template void msm_run<Fp, Fq>(Ctx*, const Fq*, long long, const Aff<Fp>*, long long, int, int, const MsmConfig&, Xyzz<Fp>*);

// ---------------------------------------------------------------- fixed-base tables
template <class B>
__global__ void msm_table_step_kernel(const Aff<B>* __restrict__ prev, Aff<B>* __restrict__ next, int N, int c) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  Xyzz<B> p = Xyzz<B>::from_affine(prev[i]);
  for (int j = 0; j < c; ++j) p = p.dbl();
  next[i] = p.to_affine();
}

template <class B>
void msm_build_tables(Ctx* ctx, const Aff<B>* bases, int N, int c, int windows, Aff<B>* table) {
  TB_CUDA(cudaMemcpyAsync(table, bases, (size_t)N * sizeof(Aff<B>), cudaMemcpyDeviceToDevice, ctx->stream));
  for (int w = 1; w < windows; ++w) {
    launch(ctx, msm_table_step_kernel<B>, (N + 127) / 128, 128, 0, table + (size_t)(w - 1) * N, table + (size_t)w * N, N, c);
  }
}
template void msm_build_tables<Fq>(Ctx*, const Aff<Fq>*, int, int, int, Aff<Fq>*);
template void msm_build_tables<Fp>(Ctx*, const Aff<Fp>*, int, int, int, Aff<Fp>*);

template <class B>
__global__ void points_to_affine_kernel(const Xyzz<B>* __restrict__ acc, int K, Aff<B>* __restrict__ out) {
  int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < K) out[k] = acc[k].to_affine();
}
template <class B> void points_to_affine(Ctx* ctx, const Xyzz<B>* acc, int K, Aff<B>* out) {
  launch(ctx, points_to_affine_kernel<B>, (K + 31) / 32, 32, 0, acc, K, out);
}
template void points_to_affine<Fq>(Ctx*, const Xyzz<Fq>*, int, Aff<Fq>*);
template void points_to_affine<Fp>(Ctx*, const Xyzz<Fp>*, int, Aff<Fp>*);

}  // namespace tb
