// Batched witness check: halo2's MockProver::run(k, circuit, instance).verify() for B witnesses of one circuit, on the device.
//
// Each failure MockProver (and circuits_random.satisfied) can name here is found without building a proof:
//   gates   every gate part of the quotient's plan runs once on the Lagrange domain (n rows instead of the quotient's 16
//           sub-cosets of n rows); a row < usable fails iff some part's y-fold is non-zero there.  Only the rows that go into
//           the report are then evaluated constraint by constraint, with one-constraint programs on the same interpreter;
//   lookups inputs and tables compressed with theta as the prover does, table keys sorted, every input key binary-searched;
//   copies  every permutation cell compared with its sigma-successor, exactly.
// y and theta are drawn per proof from the caller's seed, so a failing gate row or lookup input goes unreported with
// probability at most about (constraints + lookup width) / p per row; the seed must be unpredictable to whoever wrote the
// witness.  Advice rows >= usable are overwritten with PRF values (MockProver's poisoned cells).
#define TB_NOINLINE_MUL 0  // loop-structured kernels: small code, keep the multiply inline
#include <algorithm>
#include <array>
#include "capi_internal.cuh"
#include "prover_kernels.cuh"
#include "circuit.cuh"

namespace tb {

// fail[a][row] = the canonical key keysA[a][row] is not among sortedT[a][0, usable)   (a = proof * L + lookup)
__global__ void check_lookup_kernel(const Fp* __restrict__ keysA, const Fp* __restrict__ sortedT, uint8_t* __restrict__ fail, int n, int usable) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x;
  const size_t a = blockIdx.y;
  if (row >= usable) return;
  const Fp* T = sortedT + a * n;
  const Fp v = ld_fe(keysA + a * n + row);
  int lo = 0, hi = usable;
  while (lo < hi) { int mid = (lo + hi) >> 1; if (Fp::cmp_raw(ld_fe(T + mid), v) < 0) lo = mid + 1; else hi = mid; }
  fail[a * usable + row] = (lo < usable && ld_fe(T + lo) == v) ? 0 : 1;
}

struct CopyCells {
  const Fp* adv; long long adv_pstride; const Fp* inst; long long inst_pstride; const Fp* fix;   // Lagrange values (Montgomery)
  const int2* cols; const uint32_t* next; int n, usable, P;
  __device__ Fp at(int b, int col, int row) const {
    const int2 c = cols[col];
    const Fp* base = c.x == TB_COL_ADVICE ? adv + b * adv_pstride : c.x == TB_COL_INSTANCE ? inst + b * inst_pstride : fix;
    return ld_fe(base + (size_t)c.y * n + row);
  }
};
// fail[b][p][row] = cell (p, row) differs from its sigma-successor
__global__ void check_copy_kernel(CopyCells c, uint8_t* __restrict__ fail) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x, p = blockIdx.y, b = blockIdx.z;
  if (row >= c.usable) return;
  const uint32_t q = c.next[(size_t)p * c.n + row];
  fail[((size_t)b * c.P + p) * c.usable + row] = c.at(b, p, row) != c.at(b, (int)(q / c.n), (int)(q % c.n)) ? 1 : 0;
}

struct Report {
  const Fp* gate; int nparts; long long part_stride;   // [part][B][n] y-folds
  const uint8_t* lk_fail; const uint8_t* cp_fail; const uint32_t* next; int L, P, n, usable, M;
  uint64_t* counts;                                    // [B][3]
  uint32_t* rows; tb_failure* lrec; tb_failure* crec;  // [B][M]: the first failing gate rows, lookup and copy records
};
// the positions i < N with flag(i), in order: emit(k, i) for the k-th one while k < M; returns how many there are
template <class Flag, class Emit> __device__ int compact(int N, int M, int* sm, Flag flag, Emit emit) {
  const int m = (N + LP_THREADS - 1) / LP_THREADS, i0 = min(N, (int)threadIdx.x * m), i1 = min(N, i0 + m);
  int cnt = 0;
  for (int i = i0; i < i1; ++i) cnt += flag(i) ? 1 : 0;
  int total;
  int k = block_excl_scan(cnt, sm, &total);
  for (int i = i0; i < i1 && k < M; ++i) if (flag(i)) emit(k++, i);
  return total;
}
// one CTA per proof
__global__ void __launch_bounds__(LP_THREADS) check_report_kernel(Report r) {
  __shared__ int sm[LP_THREADS];
  const int b = blockIdx.x, U = r.usable, M = r.M;
  const size_t o = (size_t)b * M;
  const int g = compact(r.nparts ? U : 0, M, sm,
      [&](int i) { for (int p = 0; p < r.nparts; ++p) if (!ld_fe(r.gate + p * r.part_stride + (size_t)b * r.n + i).is_zero()) return true; return false; },
      [&](int k, int i) { r.rows[o + k] = (uint32_t)i; });
  const uint8_t* lf = r.lk_fail + (size_t)b * r.L * U;
  const int l = compact(r.L * U, M, sm, [&](int i) { return lf[i] != 0; },
      [&](int k, int i) { r.lrec[o + k] = tb_failure{TB_FAIL_LOOKUP, (uint32_t)(i / U), (uint32_t)(i % U), 0, 0}; });
  const uint8_t* cf = r.cp_fail + (size_t)b * r.P * U;
  const int c = compact(r.P * U, M, sm, [&](int i) { return cf[i] != 0; },
      [&](int k, int i) { const uint32_t q = r.next[(size_t)(i / U) * r.n + i % U];
                          r.crec[o + k] = tb_failure{TB_FAIL_COPY, (uint32_t)(i / U), (uint32_t)(i % U), q / r.n, q % r.n}; });
  if (threadIdx.x == 0) { uint64_t* cn = r.counts + (size_t)b * 3; cn[0] = (uint64_t)g; cn[1] = (uint64_t)l; cn[2] = (uint64_t)c; }
}

// one thread per proof: gate records by (row, constraint), then the lookup and the copy records, the first M of them
__global__ void check_assemble_kernel(const uint64_t* __restrict__ counts, const uint32_t* __restrict__ rows, const uint8_t* __restrict__ nonzero, int J,
                                      const tb_failure* __restrict__ lrec, const tb_failure* __restrict__ crec, int M, tb_failure* __restrict__ out, int B) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const uint64_t* cn = counts + (size_t)b * 3;
  const size_t o = (size_t)b * M;
  int k = 0;
  for (int s = 0; s < (int)min((uint64_t)M, cn[0]) && k < M; ++s)
    for (int j = 0; j < J && k < M; ++j)
      if (nonzero[(o + s) * J + j]) out[o + k++] = tb_failure{TB_FAIL_GATE, (uint32_t)j, rows[o + s], 0, 0};
  for (int i = 0; i < (int)min((uint64_t)M, cn[1]) && k < M; ++i) out[o + k++] = lrec[o + i];
  for (int i = 0; i < (int)min((uint64_t)M, cn[2]) && k < M; ++i) out[o + k++] = crec[o + i];
  for (; k < M; ++k) out[o + k] = tb_failure{0, 0, 0, 0, 0};
}

// What a check needs beyond the proving key, built once per key on its first check: the sigma-successor map and the
// one-constraint programs on the device.  Callers that only prove never pay for either.
static void check_prepare(const Circuit& C) {
  std::lock_guard<std::mutex> lk(C.mu);
  if (C.check_ready) return;
  const size_t n = C.n, cells = (size_t)C.P * n;
  if (C.P) {
    // sigma(p, r) = delta^q omega^s names cell (q, s): sort the values of all cells, then look every sigma value up
    std::vector<std::pair<std::array<uint32_t, 8>, uint32_t>> ids(cells);
    Fp d = Fp::one();
    for (uint32_t q = 0; q < C.P; ++q) {
      Fp v = d;
      for (size_t s = 0; s < n; ++s) { auto& e = ids[q * n + s]; std::copy(v.l, v.l + 8, e.first.begin()); e.second = (uint32_t)(q * n + s); v = v * C.omega; }
      d = d * C.delta;
    }
    std::sort(ids.begin(), ids.end());
    std::vector<Fp> sig(cells);
    TB_CUDA(cudaMemcpy(sig.data(), C.sig_vals.get(), cells * sizeof(Fp), cudaMemcpyDeviceToHost));
    std::vector<uint32_t> next(cells);
    for (size_t i = 0; i < cells; ++i) {
      std::pair<std::array<uint32_t, 8>, uint32_t> key; std::copy(sig[i].l, sig[i].l + 8, key.first.begin()); key.second = 0;
      auto it = std::lower_bound(ids.begin(), ids.end(), key);
      TB_REQUIRE(it != ids.end() && it->first == key.first, "a sigma value of the proving key is not a cell of the permutation columns");
      next[i] = it->second;
    }
    C.sig_next = DevMem<uint32_t>(next);
  }
  std::vector<QInstr> code; std::vector<int2> table; int nregs = 1;
  for (const GateProgram& p : C.plan.single) {
    table.push_back(make_int2((int)code.size(), (int)p.code.size()));
    code.insert(code.end(), p.code.begin(), p.code.end());
    nregs = std::max(nregs, p.nregs);
  }
  C.single_code = DevMem<QInstr>(code); C.single_table = DevMem<int2>(table); C.single_nregs = nregs;
  C.check_ready = true;
}

static void check_batch(Ctx* ctx, const Circuit& C, int B, const uint8_t* advice, const uint8_t* instance, const uint32_t* instance_len,
                        const uint8_t* seed, int M, uint64_t* counts_out, tb_failure* failures_out) {
  const size_t n = C.n; const long long nn = (long long)n;
  const int na = C.na, ni = C.ni, L = C.L, P = C.P, U = (int)C.usable, J = (int)C.plan.num_constraints;
  const int ni1 = std::max(1, ni), L1 = std::max(1, L), P1 = std::max(1, P);
  instance_total(C, instance_len);
  check_prepare(C);
  ProveWs* claimed = C.claim_workspace(ctx, B, true);
  TB_REQUIRE(claimed != nullptr, "this proving key / context / batch size is already checking on another thread (a tb_ctx is bound to one thread)");
  struct BusyGuard { std::atomic<int>& f; ~BusyGuard() { f.store(0); } } guard{claimed->busy};
  WsAlloc ws{ctx, C, claimed->blocks};

  // ---- the witness, and per proof theta, y and y^i (0 <= i < J + 2: the gaps of the gate folds)
  const int V_THETA = 0, V_Y = 1, V_YTAB = 2, YTAB = J + 2, NV = V_YTAB + YTAB;
  WBuf<Fp> vars = ws.buf<Fp>((size_t)B * NV);
  WBuf<Fp> inst = ws.buf<Fp>((size_t)B * ni1 * n), adv = ws.buf<Fp>((size_t)B * na * n);
  upload_witness(ctx, C, B, advice, instance, instance_len, seed, 0, R_CHECK_ROWS, inst.get(), adv.get());
  prf_fill(ctx, seed, 0, R_CHECK_THETA, 0, vars.get() + V_THETA, NV, 1, 1, B);
  prf_fill(ctx, seed, 0, R_CHECK_Y, 0, vars.get() + V_Y, NV, 1, 1, B);
  powers(ctx, vars.get() + V_YTAB, NV, vars.get() + V_Y, NV, YTAB, B);
  QData qd; memset(&qd, 0, sizeof(qd));
  qd.adv = adv.get(); qd.adv_pstride = (long long)na * nn; qd.inst = inst.get(); qd.inst_pstride = (long long)ni1 * nn;
  qd.fix = C.fixed_vals.get(); qd.R = 1; qd.k1 = 0; qd.consts = C.consts.get();
  qd.chal = vars.get(); qd.chal_stride = NV; qd.y_slot = V_Y; qd.theta_slot = V_THETA; qd.ytab_slot = V_YTAB; qd.n = (int)n; qd.lk_pstride = (long long)L1 * nn;

  // ---- gates: every part of the plan on the Lagrange domain, folds [part][B][n]
  const std::vector<QProgram>& hi = C.gate_parts[B >= 8];
  const std::vector<QProgram>* lo = C.plan.split ? &C.gate_parts_lo[B >= 8] : nullptr;
  const int NP = J ? (int)(hi.size() + (lo ? lo->size() : 0)) : 0;
  WBuf<Fp> gate = ws.buf<Fp>((size_t)std::max(1, NP) * B * n);
  if (J) {
    qd.gate_out = gate.get(); qd.gate_pstride = nn;
    q_run_parts(ctx, hi, qd, (long long)B * nn, B);
    if (lo) { qd.gate_out = gate.get() + hi.size() * B * n; q_run_parts(ctx, *lo, qd, (long long)B * nn, B); }
    qd.gate_out = nullptr;
  }
  // ---- lookups: compressed inputs and tables, table keys sorted, every input searched
  WBuf<uint8_t> lk_fail = ws.buf<uint8_t>((size_t)B * L1 * U);
  if (L) {
    WBuf<Fp> lkA = ws.buf<Fp>((size_t)B * L * n), lkS = ws.buf<Fp>((size_t)B * L * n), keysA = ws.buf<Fp>((size_t)B * L * n), keysS = ws.buf<Fp>((size_t)B * L * n);
    qd.lkA = lkA.get(); qd.lkS = lkS.get();
    q_run(ctx, C.prog_lookups, qd, B);
    lookup_keys(ctx, keysA.get(), lkA.get(), (int)n, U, B * L);
    lookup_keys(ctx, keysS.get(), lkS.get(), (int)n, U, B * L);
    sort_keys(ctx, keysS.get(), (int)n, B * L);
    launch(ctx, check_lookup_kernel, dim3((U + 255) / 256, B * L), 256, 0, keysA.get(), keysS.get(), lk_fail.get(), (int)n, U);
  }
  // ---- copies
  WBuf<uint8_t> cp_fail = ws.buf<uint8_t>((size_t)B * P1 * U);
  if (P) {
    CopyCells cc = {adv.get(), (long long)na * nn, inst.get(), (long long)ni1 * nn, C.fixed_vals.get(), C.d_perm.get(), C.sig_next.get(), (int)n, U, P};
    launch(ctx, check_copy_kernel, dim3((U + 255) / 256, P, B), 256, 0, cc, cp_fail.get());
  }
  // ---- report: counts and records compacted per proof, the listed gate rows evaluated constraint by constraint
  const size_t counts_bytes = (size_t)B * 3 * sizeof(uint64_t), fail_bytes = (size_t)B * M * sizeof(tb_failure);
  WBuf<uint8_t> out = ws.buf<uint8_t>(counts_bytes + fail_bytes);
  uint64_t* d_counts = reinterpret_cast<uint64_t*>(out.get());
  tb_failure* d_fail = reinterpret_cast<tb_failure*>(out.get() + counts_bytes);
  WBuf<uint32_t> rows = ws.buf<uint32_t>((size_t)B * M);
  WBuf<tb_failure> lrec = ws.buf<tb_failure>((size_t)B * M), crec = ws.buf<tb_failure>((size_t)B * M);
  WBuf<uint8_t> nonzero = ws.buf<uint8_t>((size_t)B * M * std::max(1, J));
  Report r = {gate.get(), NP, (long long)B * nn, lk_fail.get(), cp_fail.get(), C.sig_next.get(), L, P, (int)n, U, M, d_counts, rows.get(), lrec.get(), crec.get()};
  launch(ctx, check_report_kernel, B, LP_THREADS, 0, r);
  q_run_rows(ctx, C.single_code.get(), C.single_table.get(), J, C.single_nregs, qd, rows.get(), d_counts, 3, M, nonzero.get(), B);
  launch(ctx, check_assemble_kernel, (B + 63) / 64, 64, 0, d_counts, rows.get(), nonzero.get(), J, lrec.get(), crec.get(), M, d_fail, B);

  // ---- download (the only host synchronisation of the call)
  std::vector<uint8_t> host(counts_bytes + fail_bytes);
  TB_CUDA(cudaMemcpyAsync(host.data(), out.get(), host.size(), cudaMemcpyDeviceToHost, ctx->stream));
  ctx->sync();
  memcpy(counts_out, host.data(), counts_bytes);
  if (M) memcpy(failures_out, host.data() + counts_bytes, fail_bytes);
}

}  // namespace tb

using namespace tb;

extern "C" tb_status tb_check_batch(tb_ctx* ctx, const tb_pk* pk, uint32_t n_proofs, const uint8_t* advice, const uint8_t* instance,
                                    const uint32_t* instance_len, const uint8_t seed[32], uint32_t max_failures, uint64_t* counts_out,
                                    tb_failure* failures_out) {
  TB_API_BEGIN(ctx)
  const Circuit* C = reinterpret_cast<const Circuit*>(pk);
  TB_REQUIRE(C && n_proofs >= 1 && advice && seed && counts_out && (failures_out || max_failures == 0) && (C->ni == 0 || (instance && instance_len)),
             "tb_check_batch arguments");
  TB_REQUIRE((uint64_t)n_proofs * std::max<uint32_t>(1, std::max(C->L, C->P)) <= 65535 && max_failures <= (1u << 16), "batch too large for one call");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  check_batch(&ctx->c, *C, (int)n_proofs, advice, instance, instance_len, seed, (int)max_failures, counts_out, failures_out);
  TB_API_END(ctx)
}
