// Batched PLONKish / IPA prover: host orchestration of the sm_90a kernels for B independent proofs of one circuit.
//
// Drop-in for the body of `Proof::create` (taiga_halo2/src/proof.rs:25-42), i.e. halo2_proofs
// `plonk::create_proof` + `poly::multiopen::create_proof` + `poly::commitment::create_proof` (EXT; SURVEY.md App. A),
// after the Rust side has run `synthesize` and handed over the advice table.  Everything between the upload of the
// advice table and the download of the proof bytes stays on the device: commitments (fixed-base Pippenger), NTTs,
// lookup sort, grand products, quotient evaluation tiled by sub-coset, multiopen, the 15 IPA rounds and the
// Fiat-Shamir transcript.  Proof bytes are bit-identical to oracle/plonk.cpp for the same seed.
#include <algorithm>
#include <cstdlib>
#include <map>
#include <memory>
#include <set>
#include "capi_internal.cuh"
#include "prover_kernels.cuh"
#include "circuit.cuh"

namespace tb {

static NttHook<Fp> coset_hook(const Circuit& C, int k1, bool inverse) {
  NttHook<Fp> h; h.use_const = 0; h.mod_bits = C.ext_k; h.k = (uint32_t)k1;
  if (!inverse) { h.use_zeta = 1; h.z1 = C.zeta; h.z2 = C.zeta.sqr(); h.table = C.coset_pre.get() + (size_t)k1 * C.n; }
  else { h.use_zeta = 0; h.z1 = Fp::one(); h.z2 = Fp::one(); }
  return h;
}
// polys [count][n] -> cosets [count][R][n] (sub-coset major)
static void to_cosets(Ctx* ctx, const Circuit& C, const Fp* polys, Fp* cosets, Fp* scratch, int count) {
  if (!count) return;
  for (int k1 = 0; k1 < C.R; ++k1) {
    NttHook<Fp> h = coset_hook(C, k1, false);
    ntt_run<Fp>(ctx, (int)C.k, false, polys, cosets + (size_t)k1 * C.n, scratch, count, (long long)C.n, (long long)C.R * C.n, &h, nullptr);
  }
}

static Circuit* circuit_load(Ctx* ctx, const Srs* srs, const tb_cs_desc* cs, const uint8_t* fixed, const uint8_t* sigma) {
  TB_REQUIRE(cs->k == srs->k, "circuit k must match the SRS");
  gate_desc_check(cs);
  std::unique_ptr<Circuit> Cp(new Circuit());
  Circuit& C = *Cp;
  C.srs = srs;
  C.k = cs->k; C.n = size_t(1) << C.k; C.na = cs->num_advice; C.nf = cs->num_fixed; C.ni = cs->num_instance; C.degree = cs->cs_degree; C.bf = cs->blinding_factors;
  TB_REQUIRE(C.n > C.bf + 2, "too few rows");
  C.usable = C.n - (C.bf + 1);
  C.P = cs->num_perm_columns; C.L = cs->num_lookups; C.chunk = C.degree - 2; C.nsets = C.P ? (C.P + C.chunk - 1) / C.chunk : 0;
  C.pieces = C.degree - 1;
  C.ext_k = C.k; while ((size_t(1) << C.ext_k) < C.n * C.pieces) C.ext_k++;
  TB_REQUIRE(C.ext_k <= TW_LOG, "extended domain too large");
  C.R = 1 << (C.ext_k - C.k);
  C.aq.assign(cs->advice_queries, cs->advice_queries + cs->num_advice_queries);
  C.fq.assign(cs->fixed_queries, cs->fixed_queries + cs->num_fixed_queries);
  C.iq.assign(cs->instance_queries, cs->instance_queries + cs->num_instance_queries);
  C.perm.assign(cs->perm_columns, cs->perm_columns + C.P);
  memcpy(C.vk_repr.l, cs->vk_transcript_repr, 32);

  C.delta = delta_const<Fp>(); C.zeta = zeta_const<Fp>(); C.omega = omega_k<Fp>((int)C.k);
  C.r_inv = Fp::from_u32((uint32_t)C.R).inv();
  for (int s = 0; s < PERM_MAX_SETS; ++s) C.delta_c0[s] = C.delta.pow_u64((uint64_t)s * C.chunk);
  Fp w_ext = omega_k<Fp>(C.ext_k);
  { Fp zn = C.zeta.pow_u64(C.n), step = w_ext.pow_u64(C.n), cur = zn;
    for (int k1 = 0; k1 < C.R; ++k1) { C.t_inv.push_back((cur - Fp::one()).inv()); cur = cur * step; }
    std::vector<Fp> wr(C.R); Fp wri = step.inv(); wr[0] = Fp::one(); for (int e = 1; e < C.R; ++e) wr[e] = wr[e - 1] * wri;
    C.wr_inv = DevMem<Fp>(wr); }

  size_t n = C.n;
  // constants -> Montgomery
  for (uint32_t i = 0; i < cs->num_constants; ++i) { Fp v; memcpy(v.l, cs->constants + 32 * (size_t)i, 32); C.consts_host.push_back(v.to_mont()); }
  C.consts = DevMem<Fp>(C.consts_host);
  { std::vector<int2> pc; for (auto& c : C.perm) pc.push_back(make_int2((int)c.kind, (int)c.index)); C.d_perm = DevMem<int2>(pc); }

  { // per-element factors of the forward coset hooks (one multiplication per coefficient instead of up to two and a table walk);
    // ntt_hook_table computes them from the hook without its table
    C.coset_pre = DevMem<Fp>((size_t)C.R * n);
    for (int k1 = 0; k1 < C.R; ++k1) { NttHook<Fp> h = coset_hook(C, k1, false); ntt_hook_table<Fp>(ctx, h, false, C.coset_pre.get() + (size_t)k1 * n, (int)n); }
    ctx->sync();
  }
  DevBuf<Fp> scratch(ctx, std::max<size_t>(3, std::max<size_t>(C.nf, C.P)) * n);
  auto load_cols = [&](const uint8_t* src, size_t cnt, DevMem<Fp>& vals, DevMem<Fp>& polys, DevMem<Fp>& cosets) {
    vals = DevMem<Fp>(cnt * n); polys = DevMem<Fp>(cnt * n); cosets = DevMem<Fp>(cnt * C.R * n);
    if (!cnt) return;
    TB_CUDA(cudaMemcpyAsync(vals.get(), src, cnt * n * 32, cudaMemcpyHostToDevice, ctx->stream));
    fe_to_mont<Fp>(ctx, vals.get(), cnt * n);
    ntt_run<Fp>(ctx, (int)C.k, true, vals.get(), polys.get(), scratch.get(), (int)cnt, (long long)n, (long long)n, nullptr, nullptr);
    to_cosets(ctx, C, polys.get(), cosets.get(), scratch.get(), (int)cnt);
  };
  load_cols(fixed, C.nf, C.fixed_vals, C.fixed_polys, C.fixed_cosets);
  load_cols(sigma, C.P, C.sig_vals, C.sig_polys, C.sig_cosets);
  // l0, l_last, l_blind
  { std::vector<Fp> lag(3 * n, Fp::zero());
    lag[0] = Fp::one(); lag[n + (n - C.bf - 1)] = Fp::one();
    for (size_t r = n - C.bf; r < n; ++r) lag[2 * n + r] = Fp::one();
    DevBuf<Fp> lv(ctx, 3 * n), lp(ctx, 3 * n), lc(ctx, 3 * (size_t)C.R * n);
    lv.upload(lag.data(), 3 * n);
    ntt_run<Fp>(ctx, (int)C.k, true, lv.get(), lp.get(), scratch.get(), 3, (long long)n, (long long)n, nullptr, nullptr);
    to_cosets(ctx, C, lp.get(), lc.get(), scratch.get(), 3);
    C.l0 = DevMem<Fp>((size_t)C.R * n); C.l_last = DevMem<Fp>((size_t)C.R * n); C.l_blind = DevMem<Fp>((size_t)C.R * n);
    size_t sz = (size_t)C.R * n * sizeof(Fp);
    TB_CUDA(cudaMemcpyAsync(C.l0.get(), lc.get(), sz, cudaMemcpyDeviceToDevice, ctx->stream));
    TB_CUDA(cudaMemcpyAsync(C.l_last.get(), lc.get() + (size_t)C.R * n, sz, cudaMemcpyDeviceToDevice, ctx->stream));
    TB_CUDA(cudaMemcpyAsync(C.l_blind.get(), lc.get() + 2 * (size_t)C.R * n, sz, cudaMemcpyDeviceToDevice, ctx->stream));
    ctx->sync(); }

  // expression programs
  { GatePlan g = gate_plan(cs, C.R, tb_tune("TB_Q_SPLIT", 1) != 0);
    C.num_constraints = g.num_constraints; C.t_pl = g.t_pl; C.split = g.split;
    for (int big = 0; big < 2; ++big) {
      for (auto& p : g.gate_parts[big]) C.gate_parts[big].emplace_back(std::move(p));
      for (auto& p : g.gate_parts_lo[big]) C.gate_parts_lo[big].emplace_back(std::move(p));
    }
    C.prog_lookups = QProgram(std::move(g.lookups));
    if (getenv("TB_DEBUG")) {
      fprintf(stderr, "[tb] circuit k=%u degree=%u: %u constraints, %zu of degree <= %d (%d of %d instructions): split %s\n", C.k, C.degree, cs->num_constraints,
              g.num_lo, C.R / 2, g.lo_instr, g.all_instr, C.split ? "on" : "off");
      for (auto* m : {C.gate_parts, C.gate_parts_lo})
        for (int big = 0; big < 2; ++big) if (!m[big].empty()) {
          fprintf(stderr, "[tb]   %s %d parts:", m == C.gate_parts ? "all/high" : "low", GatePlan::nparts[big]); for (auto& qp : m[big]) fprintf(stderr, " %zu/%d", qp.prog.code.size(), qp.prog.nregs); fprintf(stderr, "\n"); }
    } }

  // ---- evaluation section order (plonk/prover.rs) and multiopen query order
  int last_rot = -(int)(C.bf + 1);
  for (auto& q : C.iq) C.evals.push_back({{PK_INST, (int)q.column}, q.rotation});
  for (auto& q : C.aq) C.evals.push_back({{PK_ADV, (int)q.column}, q.rotation});
  for (auto& q : C.fq) C.evals.push_back({{PK_FIXED, (int)q.column}, q.rotation});
  C.evals.push_back({{PK_RANDOM, 0}, 0});
  for (uint32_t c = 0; c < C.P; ++c) C.evals.push_back({{PK_SIG, (int)c}, 0});
  for (uint32_t s = 0; s < C.nsets; ++s) {
    C.evals.push_back({{PK_PZ, (int)s}, 0}); C.evals.push_back({{PK_PZ, (int)s}, 1});
    if (s + 1 < C.nsets) C.evals.push_back({{PK_PZ, (int)s}, last_rot});
  }
  for (uint32_t l = 0; l < C.L; ++l) {
    C.evals.push_back({{PK_LZ, (int)l}, 0}); C.evals.push_back({{PK_LZ, (int)l}, 1}); C.evals.push_back({{PK_LPIN, (int)l}, 0});
    C.evals.push_back({{PK_LPIN, (int)l}, -1}); C.evals.push_back({{PK_LPTAB, (int)l}, 0});
  }
  for (auto& q : C.iq) C.queries.push_back({{PK_INST, (int)q.column}, q.rotation});
  for (auto& q : C.aq) C.queries.push_back({{PK_ADV, (int)q.column}, q.rotation});
  for (uint32_t s = 0; s < C.nsets; ++s) { C.queries.push_back({{PK_PZ, (int)s}, 0}); C.queries.push_back({{PK_PZ, (int)s}, 1}); }
  for (int s = (int)C.nsets - 1; s >= 0; --s) if (s + 1 < (int)C.nsets) C.queries.push_back({{PK_PZ, s}, last_rot});
  for (uint32_t l = 0; l < C.L; ++l) {
    C.queries.push_back({{PK_LZ, (int)l}, 0}); C.queries.push_back({{PK_LPIN, (int)l}, 0}); C.queries.push_back({{PK_LPTAB, (int)l}, 0});
    C.queries.push_back({{PK_LPIN, (int)l}, -1}); C.queries.push_back({{PK_LZ, (int)l}, 1});
  }
  for (auto& q : C.fq) C.queries.push_back({{PK_FIXED, (int)q.column}, q.rotation});
  for (uint32_t c = 0; c < C.P; ++c) C.queries.push_back({{PK_SIG, (int)c}, 0});
  C.queries.push_back({{PK_H, 0}, 0});
  C.queries.push_back({{PK_RANDOM, 0}, 0});
  // multiopen::construct_intermediate_sets (points identified by rotation; sets ordered by first appearance)
  { std::map<int, int> point_index; std::vector<std::set<int>> prots;
    for (auto& q : C.queries) {
      if (!point_index.count(q.rot)) { int idx = (int)point_index.size(); point_index[q.rot] = idx; C.rots.push_back(q.rot); }
      size_t pos = 0; for (; pos < C.uniq.size(); ++pos) if (C.uniq[pos] == q.poly) break;
      if (pos == C.uniq.size()) { C.uniq.push_back(q.poly); prots.emplace_back(); }
      prots[pos].insert(point_index[q.rot]);
    }
    std::map<std::set<int>, int> set_index;
    for (size_t c = 0; c < C.uniq.size(); ++c) {
      if (!set_index.count(prots[c])) { int idx = (int)set_index.size(); set_index[prots[c]] = idx; }
      C.uniq_set.push_back(set_index[prots[c]]);
    }
    C.point_sets.resize(set_index.size());
    for (auto& kv : set_index) for (int pi : kv.first) C.point_sets[kv.second].push_back(C.rots[pi]); }
  for (auto& e : C.evals) if (std::find(C.rots.begin(), C.rots.end(), e.rot) == C.rots.end()) C.rots.push_back(e.rot);
  uint32_t commits = C.na + 3 * C.L + C.nsets + 1 + C.pieces;
  C.proof_len = 32 * (commits + (uint32_t)C.evals.size() + 1 + (uint32_t)C.point_sets.size() + 1 + 2 * C.k + 2);
  return Cp.release();
}

// ---------------------------------------------------------------- IPA kernels (s-vector form, SURVEY App. E.5)
// After j rounds the folded generators are G'_i = sum_q s_j(q) g[i + m q] (m = n >> j), so L_j / R_j are fixed-base MSMs over
// the ORIGINAL generators with scalars p'[.] * s(t): no generator folding, no variable-base MSM, no Horner over windows.
//   cL[t] = p'[half + i] * s[t]  if i <  half      cR[t] = p'[i - half] * s[t]  if i >= half      (i = t mod m, half = m/2)
__global__ void ipa_round_scalars_kernel(const Fp* __restrict__ pprime, const Fp* __restrict__ sfull, Fp* __restrict__ cLR, int n, int m) {
  int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (t >= n) return;
  int i = t & (m - 1), half = m >> 1;
  const Fp* pp = pprime + (size_t)b * n;
  Fp s = ld_fe(sfull + (size_t)b * n + t);
  Fp* out = cLR + (size_t)b * 2 * n;
  if (i < half) { st_fe(out + t, ld_fe(pp + half + i) * s); st_fe(out + n + t, Fp::zero()); }
  else { st_fe(out + t, Fp::zero()); st_fe(out + n + t, ld_fe(pp + i - half) * s); }
}
// p'[i] += p'[i+half] / u ; b[i] += b[i+half] * u  (i < half);  s[t] *= u for t with bit log2(half) set
__global__ void ipa_fold_kernel(Fp* p, Fp* bv, Fp* sfull, int n, int half, const Fp* vars, long long vstride, int u_slot, int uinv_slot) {
  int t = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (t >= n) return;
  Fp u = vars[(long long)b * vstride + u_slot];
  if (t & half) { Fp* sp = sfull + (size_t)b * n + t; st_fe(sp, ld_fe(sp) * u); }
  if (t < half) {
    Fp ui = vars[(long long)b * vstride + uinv_slot];
    Fp* pb = p + (size_t)b * n; Fp* bb = bv + (size_t)b * n;
    st_fe(pb + t, ld_fe(pb + t) + ld_fe(pb + t + half) * ui);
    st_fe(bb + t, ld_fe(bb + t) + ld_fe(bb + t + half) * u);
  }
}
// extras[b][0] = {lr, vl*z}, extras[b][1] = {rr, vr*z}   (multipliers of the SRS points w and u)
__global__ void ipa_extras_kernel(Fp* ex, const Fp* vars, long long vstride, int lr, int rr, int vl, int vr, int z, int B) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  const Fp* v = vars + (long long)b * vstride;
  Fp* e = ex + (size_t)b * 4;
  e[0] = v[lr]; e[1] = v[vl] * v[z]; e[2] = v[rr]; e[3] = v[vr] * v[z];
}
__global__ void fill_const_kernel(Fp* v, size_t count, Fp val) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) st_fe(v + i, val);
}

// ---------------------------------------------------------------- the prover
struct VarAlloc {
  int next = 0;
  int one(int cnt = 1) { int r = next; next += cnt; return r; }
};
struct Prog {
  std::vector<ScalarInstr> ins;
  void op(int o, int dst, int a = 0, int b = 0, uint32_t imm = 0) { ScalarInstr i; i.op = (uint16_t)o; i.dst = (uint16_t)dst; i.a = (uint16_t)a; i.b = (uint16_t)b; i.imm = imm; ins.push_back(i); }
};
// Persistent per-(circuit, batch size) device workspace: the same sequence of requests returns the same pointers on every
// call, so item tables / scalar programs that embed them are uploaded once and no allocation or host sync happens later.
template <class T> struct WBuf {
  T* p = nullptr; size_t n = 0; Ctx* ctx = nullptr;
  T* get() const { return p; }
  void zero() { TB_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), ctx->stream)); }
};
struct WsAlloc {
  Ctx* ctx; const Circuit& C; std::vector<DevMem<uint8_t>>& blocks; size_t cur = 0;
  template <class T> WBuf<T> buf(size_t count) {
    size_t bytes = std::max<size_t>(1, count) * sizeof(T);
    if (cur == blocks.size()) blocks.emplace_back();
    if (blocks[cur].size() < bytes) {   // try_alloc frees the smaller block first
      cudaError_t e = blocks[cur].try_alloc(bytes);
      if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); C.release_idle(ctx->device); e = blocks[cur].try_alloc(bytes); }
      TB_CUDA(e);
    }
    WBuf<T> w; w.p = reinterpret_cast<T*>(blocks[cur].get()); w.n = count; w.ctx = ctx; ++cur;
    return w;
  }
};

static void prove_batch(Ctx* ctx, const Circuit& C, int B, const uint8_t* advice_host, const uint8_t* instance_host, const uint32_t* instance_len,
                        const uint8_t* seed, uint32_t proof0, uint8_t* proofs_out, size_t proof_stride) {
  const Srs& srs = *C.srs;
  const size_t n = C.n; const long long nn = (long long)n; const int k = (int)C.k; const int na = C.na, ni = C.ni, L = C.L, nsets = C.nsets, P = C.P, bf = C.bf;
  const int ni1 = std::max(1, ni), L1 = std::max(1, L), ns1 = std::max(1, nsets);
  // all per-proof polynomials that are taken to the extended cosets live in ONE buffer [B][NC][n] so that each sub-coset
  // needs a single batched NTT launch: advice | instance | permutation Z | lookup Z | A' | S'
  const int NC = na + ni + nsets + 3 * L;
  const int O_ADV = 0, O_INST = na, O_PZ = na + ni, O_LZ = na + ni + nsets, O_LPIN = O_LZ + L, O_LPTAB = O_LZ + 2 * L;
  const long long PS = (long long)NC * nn;   // per-proof stride of the merged buffers
  cudaStream_t st = ctx->stream;
  size_t inst_total = 0;
  for (int c = 0; c < ni; ++c) { TB_REQUIRE(instance_len[c] <= C.usable, "InstanceTooLarge"); inst_total += instance_len[c]; }
  ProveWs* claimed = C.claim_workspace(ctx, B);
  TB_REQUIRE(claimed != nullptr, "this proving key / context / batch size is already proving on another thread (a tb_ctx is bound to one thread)");
  ProveWs& pws = *claimed;
  struct BusyGuard { std::atomic<int>& f; ~BusyGuard() { f.store(0); } } guard{pws.busy};
  WsAlloc ws{ctx, C, pws.blocks};
  std::vector<DevMem<uint8_t>>& tables = pws.tables;
  size_t table_cur = 0;
  // uploads a small host table once per (circuit, context, B); later calls reuse the device copy.  The contents follow from the
  // circuit and B alone; they are still compared with what was uploaded (a cheap guard should a table come to depend on anything
  // else) and refreshed in stream order if they differ.
  auto cached_upload = [&](const void* host, size_t bytes) -> void* {
    const uint8_t* hb = static_cast<const uint8_t*>(host);
    if (table_cur == tables.size()) {
      tables.emplace_back(std::max<size_t>(16, bytes));
      TB_CUDA(cudaMemcpy(tables.back().get(), host, bytes, cudaMemcpyHostToDevice));
      pws.table_bytes.emplace_back(hb, hb + bytes);
    } else {
      std::vector<uint8_t>& old = pws.table_bytes[table_cur];
      if (old.size() != bytes || memcmp(old.data(), host, bytes) != 0) {
        if (old.size() < bytes) tables[table_cur] = DevMem<uint8_t>(bytes);
        old.assign(hb, hb + bytes);
        TB_CUDA(cudaMemcpyAsync(tables[table_cur].get(), old.data(), bytes, cudaMemcpyHostToDevice, st));
      }
    }
    return tables[table_cur++].get();
  };

  // ---- per-proof scalar variables
  VarAlloc va;
  const int V_ONE = va.one(), V_THETA = va.one(), V_BETA = va.one(), V_GAMMA = va.one(), V_Y = va.one(), V_X = va.one(), V_XN = va.one();
  const int V_X1 = va.one(), V_X2 = va.one(), V_X3 = va.one(), V_X4 = va.one(), V_XI = va.one(), V_Z = va.one();
  const int V_PT = va.one((int)C.rots.size());
  const int V_ADV_BLIND = va.one(na), V_LPIN_BLIND = va.one(L1), V_LPTAB_BLIND = va.one(L1), V_PZ_BLIND = va.one(ns1), V_LZ_BLIND = va.one(L1);
  const int V_RANDOM_BLIND = va.one(), V_H_BLINDS = va.one(C.pieces), V_H_BLIND = va.one(), V_QPRIME_BLIND = va.one();
  const int nps = (int)C.point_sets.size();
  const int V_QBLIND = va.one(nps), V_P_BLIND = va.one(), V_S_BLIND = va.one(), V_F = va.one();
  const int V_S_AT = va.one(), V_V = va.one(), V_LR = va.one(), V_RR = va.one(), V_VL = va.one(), V_VR = va.one();
  const int V_U = va.one(), V_UINV = va.one(), V_T0 = va.one(), V_C = va.one();
  const int YTAB = (int)(C.num_constraints + C.t_pl) + 2;
  const int V_YTAB = va.one(YTAB);   // y^i, 0 <= i < YTAB: gap-aware folds of the gate programs and the weights that combine them
  const int NV = va.next;
  WBuf<Fp> vars = ws.buf<Fp>((size_t)B * NV);
  vars.zero();
  std::vector<Fp> hconsts = {Fp::one(), C.omega, C.omega.inv()};
  Fp* dconsts = reinterpret_cast<Fp*>(cached_upload(hconsts.data(), hconsts.size() * sizeof(Fp)));
  auto run_prog = [&](Prog& p) {
    if (p.ins.empty()) return;
    ScalarInstr* d = reinterpret_cast<ScalarInstr*>(cached_upload(p.ins.data(), p.ins.size() * sizeof(ScalarInstr)));
    scalar_program(ctx, vars.get(), NV, d, (int)p.ins.size(), dconsts, B);
    p.ins.clear();
  };
  { Prog p; p.op(S_CONST, V_ONE, 0, 0, 0); run_prog(p); }
  auto VP = [&](int slot) { return vars.get() + slot; };  // pointer to slot of proof 0, stride NV

  Transcripts tr; tr.init(ctx, B, C.proof_len, C.vk_repr);
  WBuf<Fp> scratch = ws.buf<Fp>((size_t)B * std::max({NC, (int)C.pieces, 4}) * n);
  WBuf<Fp> polys = ws.buf<Fp>((size_t)B * NC * n), cosets = ws.buf<Fp>((size_t)B * NC * n);
  WBuf<Aff<Fq>> pts = ws.buf<Aff<Fq>>((size_t)B * std::max({na + ni, 2 * L1, ns1 + L1, (int)C.pieces, 2}));
  WBuf<Fp> blinds = ws.buf<Fp>((size_t)B * std::max({na + ni, 2 * L1, ns1 + L1, (int)C.pieces, 4}));
  WBuf<uint32_t> derr = ws.buf<uint32_t>((size_t)B * L1); derr.zero();   // one flag per (proof, lookup)

  // ---- instance + advice columns (commit_lagrange): one batched fixed-base MSM call for both
  // (the vanishing argument's random polynomial is committed over `g`, a different table: separate call)
  WBuf<Fp> first = ws.buf<Fp>((size_t)B * (ni + na) * n);
  WBuf<Fp> inst_vals; inst_vals.p = first.get(); inst_vals.n = (size_t)B * ni * n; inst_vals.ctx = ctx;
  WBuf<Fp> adv_vals; adv_vals.p = first.get() + (size_t)B * ni * n; adv_vals.n = (size_t)B * na * n; adv_vals.ctx = ctx;
  Fp* const inst_polys = polys.get() + (size_t)O_INST * n;
  if (ni) inst_vals.zero();
  if (ni) {
    size_t off = 0;
    for (int c = 0; c < ni; ++c) {
      if (instance_len[c])
        TB_CUDA(cudaMemcpy2DAsync(inst_vals.get() + (size_t)c * n, (size_t)ni * n * 32, instance_host + 32 * off, inst_total * 32, (size_t)instance_len[c] * 32, B,
                                  cudaMemcpyHostToDevice, st));
      off += instance_len[c];
    }
    fe_to_mont<Fp>(ctx, inst_vals.get(), (size_t)B * ni * n);
    launch(ctx, fill_const_kernel, (B * ni + 63) / 64, 64, 0, blinds.get(), (size_t)B * ni, Fp::one());
  }
  // ---- advice columns: upload, blinding rows, commit, iNTT
  Fp* const adv_polys = polys.get() + (size_t)O_ADV * n;
  TB_CUDA(cudaMemcpyAsync(adv_vals.get(), advice_host, (size_t)B * na * n * 32, cudaMemcpyDefault, st));  // host or device pointer
  fe_to_mont<Fp>(ctx, adv_vals.get(), (size_t)B * na * n);
  for (int c = 0; c < na; ++c)
    prf_fill(ctx, seed, proof0, R_ADVICE_ROWS, (uint32_t)(c * (bf + 1)), adv_vals.get() + (size_t)c * n + C.usable, (long long)na * nn, 1, bf + 1, B);
  prf_fill(ctx, seed, proof0, R_ADVICE_BLIND, 0, VP(V_ADV_BLIND), NV, 1, na, B);
  poly_copy(ctx, blinds.get() + (size_t)B * ni, na, VP(V_ADV_BLIND), NV, na, B);
  srs.commit(ctx, true, first.get(), nn, B * (ni + na), blinds.get(), pts.get());   // [B*ni instance | B*na advice]
  if (ni) {
    tr.points(pts.get(), ni, ni, false);
    ntt_run<Fp>(ctx, k, true, inst_vals.get(), inst_polys, scratch.get(), ni, nn, nn, nullptr, nullptr, B, (long long)ni * nn, PS);
  }
  tr.points(pts.get() + (size_t)B * ni, na, na, true);
  ntt_run<Fp>(ctx, k, true, adv_vals.get(), adv_polys, scratch.get(), na, nn, nn, nullptr, nullptr, B, (long long)na * nn, PS);
  tr.squeeze(VP(V_THETA), NV, 1);

  // ---- lookups: compress (Lagrange domain), sort, arrange, blind, commit A', S'
  WBuf<Fp> lkA = ws.buf<Fp>((size_t)B * L1 * n), lkS = ws.buf<Fp>((size_t)B * L1 * n), lperm = ws.buf<Fp>((size_t)2 * B * L1 * n);
  WBuf<Fp> lpin; lpin.p = lperm.get(); lpin.n = (size_t)B * L1 * n; lpin.ctx = ctx;
  WBuf<Fp> lptab; lptab.p = lperm.get() + (size_t)B * L * n; lptab.n = (size_t)B * L1 * n; lptab.ctx = ctx;   // adjacent: one commitment call
  Fp* const lpin_polys = polys.get() + (size_t)O_LPIN * n; Fp* const lptab_polys = polys.get() + (size_t)O_LPTAB * n;
  QData qd; memset(&qd, 0, sizeof(qd));
  qd.consts = C.consts.get(); qd.chal = vars.get(); qd.chal_stride = NV; qd.y_slot = V_Y; qd.theta_slot = V_THETA; qd.ytab_slot = V_YTAB;
  qd.n = (int)n; qd.lk_pstride = (long long)L1 * nn;
  if (L) {
    qd.adv = adv_vals.get(); qd.adv_pstride = (long long)na * nn; qd.inst = inst_vals.get(); qd.inst_pstride = (long long)ni1 * nn;
    qd.fix = C.fixed_vals.get(); qd.R = 1; qd.k1 = 0; qd.gate_out = nullptr; qd.lkA = lkA.get(); qd.lkS = lkS.get();
    q_run(ctx, C.prog_lookups, qd, B);
    WBuf<Fp> keysA = ws.buf<Fp>((size_t)B * L * n), keysS = ws.buf<Fp>((size_t)B * L * n), left = ws.buf<Fp>((size_t)B * L * n);
    lookup_keys(ctx, keysA.get(), lkA.get(), (int)n, (int)C.usable, B * L);
    lookup_keys(ctx, keysS.get(), lkS.get(), (int)n, (int)C.usable, B * L);
    sort_keys(ctx, keysA.get(), (int)n, B * L);
    sort_keys(ctx, keysS.get(), (int)n, B * L);
    lookup_arrange(ctx, keysA.get(), keysS.get(), left.get(), lptab.get(), (int)n, (int)C.usable, B * L, derr.get());  // error flag read back with the proofs
    TB_CUDA(cudaMemcpyAsync(lpin.get(), keysA.get(), (size_t)B * L * n * 32, cudaMemcpyDeviceToDevice, st));
    fe_to_mont<Fp>(ctx, lpin.get(), (size_t)B * L * n);
    fe_to_mont<Fp>(ctx, lptab.get(), (size_t)B * L * n);
    for (int l = 0; l < L; ++l) {
      prf_fill(ctx, seed, proof0, R_LK_IN_ROWS, (uint32_t)(l * (bf + 1)), lpin.get() + (size_t)l * n + C.usable, (long long)L * nn, 1, bf + 1, B);
      prf_fill(ctx, seed, proof0, R_LK_TAB_ROWS, (uint32_t)(l * (bf + 1)), lptab.get() + (size_t)l * n + C.usable, (long long)L * nn, 1, bf + 1, B);
    }
    prf_fill(ctx, seed, proof0, R_LK_IN_BLIND, 0, VP(V_LPIN_BLIND), NV, 1, L, B);
    prf_fill(ctx, seed, proof0, R_LK_TAB_BLIND, 0, VP(V_LPTAB_BLIND), NV, 1, L, B);
    // commit in transcript order: per lookup A' then S'
    poly_copy(ctx, blinds.get(), L, VP(V_LPIN_BLIND), NV, L, B);
    poly_copy(ctx, blinds.get() + (size_t)B * L, L, VP(V_LPTAB_BLIND), NV, L, B);
    srs.commit(ctx, true, lperm.get(), nn, 2 * B * L, blinds.get(), pts.get());   // [B*L A' | B*L S']
    for (int l = 0; l < L; ++l) { tr.points(pts.get() + l, L, 1, true); tr.points(pts.get() + (size_t)B * L + l, L, 1, true); }
    ntt_run<Fp>(ctx, k, true, lpin.get(), lpin_polys, scratch.get(), L, nn, nn, nullptr, nullptr, B, (long long)L * nn, PS);
    ntt_run<Fp>(ctx, k, true, lptab.get(), lptab_polys, scratch.get(), L, nn, nn, nullptr, nullptr, B, (long long)L * nn, PS);
  }
  tr.squeeze(VP(V_BETA), NV, 1);
  tr.squeeze(VP(V_GAMMA), NV, 1);

  // ---- permutation grand products
  Fp* const pz_polys = polys.get() + (size_t)O_PZ * n;
  const size_t gp = (size_t)std::max(ns1, L1);
  WBuf<Fp> gnum = ws.buf<Fp>((size_t)B * gp * n), gden = ws.buf<Fp>((size_t)B * gp * n), gz = ws.buf<Fp>((size_t)B * (ns1 + L1) * n);
  Fp* const gz_lk = gz.get() + (size_t)B * nsets * n;   // lookup Z vectors directly after the permutation Z vectors: one commitment call
  if (nsets) {
    PermFrac pf; memset(&pf, 0, sizeof(pf));
    pf.adv = adv_vals.get(); pf.adv_pstride = (long long)na * nn; pf.inst = inst_vals.get(); pf.inst_pstride = (long long)ni1 * nn; pf.fix = C.fixed_vals.get();
    pf.sig = C.sig_vals.get(); pf.perm_cols = C.d_perm.get(); pf.P = P; pf.chunk = C.chunk; pf.nsets = nsets; pf.chal = vars.get(); pf.chal_stride = NV;
    pf.beta_slot = V_BETA; pf.gamma_slot = V_GAMMA; pf.delta = C.delta; pf.omega = C.omega; memcpy(pf.delta_c0, C.delta_c0, sizeof(pf.delta_c0));
    pf.tw = ctx->tw_fp.fwd; pf.num = gnum.get(); pf.den = gden.get(); pf.pstride = (long long)nsets * nn; pf.n = (int)n; pf.k = k;
    perm_fractions(ctx, pf, B);
    batch_inverse(ctx, gden.get(), (size_t)B * nsets * n);
    vec_mul(ctx, gnum.get(), gden.get(), (size_t)B * nsets * n);
    prefix_product(ctx, gz.get(), gnum.get(), (int)n, B * nsets);
    perm_chain(ctx, gz.get(), (long long)nsets * nn, nsets, (int)n, (int)(n - bf - 1), B);
    for (int s = 0; s < nsets; ++s)
      prf_fill(ctx, seed, proof0, R_PERM_ROWS, (uint32_t)(s * bf), gz.get() + (size_t)s * n + (n - bf), (long long)nsets * nn, 1, bf, B);
    prf_fill(ctx, seed, proof0, R_PERM_BLIND, 0, VP(V_PZ_BLIND), NV, 1, nsets, B);
    poly_copy(ctx, blinds.get(), nsets, VP(V_PZ_BLIND), NV, nsets, B);
  }
  // ---- lookup grand products
  Fp* const lz_polys = polys.get() + (size_t)O_LZ * n;
  if (L) {
    lookup_fractions(ctx, lkA.get(), lkS.get(), lpin.get(), lptab.get(), gnum.get(), gden.get(), (long long)L * nn, L, (int)n, vars.get(), NV, V_BETA, V_GAMMA, B);
    batch_inverse(ctx, gden.get(), (size_t)B * L * n);
    vec_mul(ctx, gnum.get(), gden.get(), (size_t)B * L * n);
    prefix_product(ctx, gz_lk, gnum.get(), (int)n, B * L);
    for (int l = 0; l < L; ++l)
      prf_fill(ctx, seed, proof0, R_LKZ_ROWS, (uint32_t)(l * bf), gz_lk + (size_t)l * n + (n - bf), (long long)L * nn, 1, bf, B);
    prf_fill(ctx, seed, proof0, R_LKZ_BLIND, 0, VP(V_LZ_BLIND), NV, 1, L, B);
    poly_copy(ctx, blinds.get() + (size_t)B * nsets, L, VP(V_LZ_BLIND), NV, L, B);
  }
  if (nsets + L) {
    srs.commit(ctx, true, gz.get(), nn, B * (nsets + L), blinds.get(), pts.get());   // [B*nsets permutation Z | B*L lookup Z]
    if (nsets) {
      tr.points(pts.get(), nsets, nsets, true);
      ntt_run<Fp>(ctx, k, true, gz.get(), pz_polys, scratch.get(), nsets, nn, nn, nullptr, nullptr, B, (long long)nsets * nn, PS);
    }
    if (L) {
      tr.points(pts.get() + (size_t)B * nsets, L, L, true);
      ntt_run<Fp>(ctx, k, true, gz_lk, lz_polys, scratch.get(), L, nn, nn, nullptr, nullptr, B, (long long)L * nn, PS);
    }
  }
  // ---- vanishing argument: random polynomial
  WBuf<Fp> random_poly = ws.buf<Fp>((size_t)B * n);
  prf_fill(ctx, seed, proof0, R_RANDOM_POLY, 0, random_poly.get(), nn, 1, (int)n, B);
  prf_fill(ctx, seed, proof0, R_RANDOM_BLIND, 0, VP(V_RANDOM_BLIND), NV, 1, 1, B);
  poly_copy(ctx, blinds.get(), 1, VP(V_RANDOM_BLIND), NV, 1, B);
  srs.commit(ctx, false, random_poly.get(), nn, B, blinds.get(), pts.get());
  tr.points(pts.get(), 1, 1, true);
  tr.squeeze(VP(V_Y), NV, 1);

  // ---- quotient, tiled by sub-coset (SURVEY E.3)
  const int R = C.R;
  // Constraint-parallel split of the gate program.  More parts = shorter per-thread chains (latency at small batches) AND
  // fewer live temporaries per part = smaller shared-memory register file = higher occupancy (ncu: 6 warps/SM with one
  // 26-register program vs 20 warps/SM with eight <=11-register parts), for ~15% more instructions in total.
  const std::vector<QProgram>& gprogs = C.gate_parts[B >= 8];
  const std::vector<QProgram>* lprogs = C.split ? &C.gate_parts_lo[B >= 8] : nullptr;
  { Prog p; p.op(S_CONST, V_YTAB, 0, 0, 0); p.op(S_COPY, V_YTAB + 1, V_Y);
    for (int i = 2; i < YTAB; ++i) p.op(S_MUL, V_YTAB + i, V_YTAB + i - 1, V_Y);
    run_prog(p); }
  const int J = (int)C.num_constraints;
  WBuf<Fp> hext = ws.buf<Fp>((size_t)B * R * n), hcoef = ws.buf<Fp>((size_t)B * C.pieces * n);
  { WBuf<Fp> c_lkA = ws.buf<Fp>((size_t)B * L1 * n), c_lkS = ws.buf<Fp>((size_t)B * L1 * n), gate = ws.buf<Fp>((size_t)Q_MAX_PARTS * B * n), V = ws.buf<Fp>((size_t)B * R * n);
    const int Rlo = C.split ? R / 2 : 0;
    // ---- low-degree constraints: every second sub-coset only.  Their sum H_lo is interpolated (Rlo * n coefficients) and divided by
    // X^n - 1 in coefficient form, H_lo = q_lo (X^n - 1) + r_lo; q_lo goes straight into h, r_lo (n coefficients) joins the numerator
    // of the high-degree part as one more polynomial on every sub-coset.  The column cosets computed here are kept for the second pass.
    WBuf<Fp> keep, elo, vlo, clo, qlo, rlo_poly, rlo_coset;
    if (C.split) {
      keep = ws.buf<Fp>((size_t)Rlo * B * NC * n); elo = ws.buf<Fp>((size_t)B * Rlo * n); vlo = ws.buf<Fp>((size_t)B * Rlo * n); clo = ws.buf<Fp>((size_t)B * Rlo * n);
      qlo = ws.buf<Fp>((size_t)B * Rlo * n); rlo_poly = ws.buf<Fp>((size_t)B * n); rlo_coset = ws.buf<Fp>((size_t)B * n);
      int gexp[Q_MAX_PARTS] = {0};
      for (size_t p = 0; p < lprogs->size(); ++p) gexp[p] = J - 1 - (*lprogs)[p].prog.last + (int)C.t_pl;
      for (int kq = 0; kq < Rlo; ++kq) {
        const int k1 = 2 * kq;
        Fp* ck = keep.get() + (size_t)kq * B * NC * n;
        NttHook<Fp> h = coset_hook(C, k1, false);
        ntt_run<Fp>(ctx, k, false, polys.get(), ck, scratch.get(), B * NC, nn, nn, &h, nullptr);
        qd.adv = ck + (size_t)O_ADV * n; qd.adv_pstride = PS; qd.inst = ck + (size_t)O_INST * n; qd.inst_pstride = PS;
        qd.fix = C.fixed_cosets.get(); qd.R = R; qd.k1 = k1; qd.lkA = c_lkA.get(); qd.lkS = c_lkS.get();
        qd.gate_out = gate.get(); qd.gate_pstride = nn;
        q_run_parts(ctx, *lprogs, qd, (long long)B * nn, B);
        q_combine(ctx, gate.get(), (int)lprogs->size(), (long long)B * nn, gexp, vars.get(), NV, V_YTAB, elo.get() + (size_t)kq * n, (long long)Rlo * nn, (int)n, B);
      }
      for (int kq = 0; kq < Rlo; ++kq) {   // interpolation on the coset zeta * <w_ext^2>: same two steps as extended_to_coeff, with R / 2 sub-cosets
        NttHook<Fp> h = coset_hook(C, 2 * kq, true);
        ntt_run<Fp>(ctx, k, true, elo.get() + (size_t)kq * n, vlo.get() + (size_t)kq * n, scratch.get(), B, (long long)Rlo * nn, (long long)Rlo * nn, nullptr, &h);
      }
      h_cross(ctx, vlo.get(), (long long)Rlo * nn, clo.get(), (long long)Rlo * nn, (int)n, Rlo, Rlo, C.wr_inv.get(), 2, Fp::from_u32((uint32_t)Rlo).inv(), C.zeta.sqr(), B);
      q_lo_split(ctx, clo.get(), (long long)Rlo * nn, Rlo, rlo_poly.get(), nn, qlo.get(), (long long)Rlo * nn, (int)n, B);
    }
    int gexp_hi[Q_MAX_PARTS] = {0};
    for (size_t p = 0; p < gprogs.size(); ++p) gexp_hi[p] = J - 1 - gprogs[p].prog.last;
    for (int k1 = 0; k1 < R; ++k1) {
      NttHook<Fp> h = coset_hook(C, k1, false);
      Fp* ck = cosets.get();
      if (C.split && (k1 & 1) == 0) ck = keep.get() + (size_t)(k1 / 2) * B * NC * n;   // computed in the first pass
      else ntt_run<Fp>(ctx, k, false, polys.get(), ck, scratch.get(), B * NC, nn, nn, &h, nullptr);
      if (C.split) ntt_run<Fp>(ctx, k, false, rlo_poly.get(), rlo_coset.get(), scratch.get(), B, nn, nn, &h, nullptr);
      Fp* const c_adv = ck + (size_t)O_ADV * n; Fp* const c_inst = ck + (size_t)O_INST * n; Fp* const c_pz = ck + (size_t)O_PZ * n;
      Fp* const c_lz = ck + (size_t)O_LZ * n; Fp* const c_lpin = ck + (size_t)O_LPIN * n; Fp* const c_lptab = ck + (size_t)O_LPTAB * n;
      qd.adv = c_adv; qd.adv_pstride = PS; qd.inst = c_inst; qd.inst_pstride = PS;
      qd.fix = C.fixed_cosets.get(); qd.R = R; qd.k1 = k1; qd.lkA = c_lkA.get(); qd.lkS = c_lkS.get();
      qd.gate_out = gate.get(); qd.gate_pstride = nn;
      q_run_parts(ctx, gprogs, qd, (long long)B * nn, B);
      if (L) { qd.gate_out = nullptr; q_run(ctx, C.prog_lookups, qd, B); }
      QFinish f; memset(&f, 0, sizeof(f));
      f.gate = gate.get(); f.nparts = (int)gprogs.size(); f.gate_part_stride = (long long)B * nn; f.ytab_slot = V_YTAB; memcpy(f.gexp, gexp_hi, sizeof(gexp_hi));
      f.rlo = C.split ? rlo_coset.get() : nullptr; f.rlo_pstride = nn;
      f.adv = c_adv; f.adv_pstride = PS; f.inst = c_inst; f.inst_pstride = PS;
      f.fix = C.fixed_cosets.get(); f.sig = C.sig_cosets.get(); f.R = R; f.k1 = k1; f.l0 = C.l0.get(); f.l_last = C.l_last.get(); f.l_blind = C.l_blind.get();
      f.pz = c_pz; f.pz_pstride = PS; f.lz = c_lz; f.lpin = c_lpin; f.lptab = c_lptab; f.lk_pstride = PS; f.lkc_pstride = (long long)L1 * nn;
      f.lkA = c_lkA.get(); f.lkS = c_lkS.get(); f.perm_cols = C.d_perm.get(); f.P = P; f.chunk = C.chunk; f.nsets = nsets; f.L = L; f.bf = bf;
      f.chal = vars.get(); f.chal_stride = NV; f.y_slot = V_Y; f.beta_slot = V_BETA; f.gamma_slot = V_GAMMA;
      f.delta = C.delta; f.zeta = C.zeta; f.t_inv = C.t_inv[k1]; memcpy(f.delta_c0, C.delta_c0, sizeof(f.delta_c0)); f.tw = ctx->tw_fp.fwd;
      f.ext_k = C.ext_k; f.k = k; f.out = hext.get(); f.out_pstride = (long long)R * nn; f.n = (int)n;
      q_finish(ctx, f, B);
    }
    // extended_to_coeff: per sub-coset iNTT with w_ext^(-i*k1) (step A), then the size-R cross transform (step B)
    for (int k1 = 0; k1 < R; ++k1) {
      NttHook<Fp> h = coset_hook(C, k1, true);
      ntt_run<Fp>(ctx, k, true, hext.get() + (size_t)k1 * n, V.get() + (size_t)k1 * n, scratch.get(), B, (long long)R * nn, (long long)R * nn, nullptr, &h);
    }
    h_cross(ctx, V.get(), (long long)R * nn, hcoef.get(), (long long)C.pieces * nn, (int)n, R, (int)C.pieces, C.wr_inv.get(), 1, C.r_inv, C.zeta.sqr(), B);
    if (C.split) q_add_blocks(ctx, hcoef.get(), (long long)C.pieces * nn, qlo.get(), (long long)Rlo * nn, Rlo - 1, (int)n, B);   // + H_lo div (X^n - 1)
  }
  prf_fill(ctx, seed, proof0, R_H_BLIND, 0, VP(V_H_BLINDS), NV, 1, (int)C.pieces, B);
  poly_copy(ctx, blinds.get(), C.pieces, VP(V_H_BLINDS), NV, C.pieces, B);
  srs.commit(ctx, false, hcoef.get(), nn, B * (int)C.pieces, blinds.get(), pts.get());
  tr.points(pts.get(), C.pieces, C.pieces, true);
  tr.squeeze(VP(V_X), NV, 1);

  // ---- evaluation points, h(X) = sum xn^i h_i, blinds
  WBuf<Fp> h_poly = ws.buf<Fp>((size_t)B * n);
  { Prog p;
    p.op(S_POW2K, V_XN, V_X, 0, (uint32_t)k);
    for (size_t i = 0; i < C.rots.size(); ++i) {
      int rot = C.rots[i], dst = V_PT + (int)i;
      p.op(S_COPY, dst, V_X);
      if (rot) { p.op(S_CONST, V_T0, 0, 0, rot > 0 ? 1 : 2); for (int r = 0; r < std::abs(rot); ++r) p.op(S_MUL, dst, dst, V_T0); }
    }
    p.op(S_SUB, V_H_BLIND, V_H_BLIND, V_H_BLIND);
    for (int i = (int)C.pieces - 1; i >= 0; --i) p.op(S_FMA, V_H_BLIND, V_XN, V_H_BLINDS + i);
    run_prog(p); }
  h_poly.zero();
  for (int i = (int)C.pieces - 1; i >= 0; --i) poly_fma(ctx, h_poly.get(), nn, VP(V_XN), NV, hcoef.get() + (size_t)i * n, (long long)C.pieces * nn, (int)n, B);

  auto rot_slot = [&](int rot) { return V_PT + (int)(std::find(C.rots.begin(), C.rots.end(), rot) - C.rots.begin()); };
  auto mk_item = [](const Fp* base, long long bstride, int point) { EvalItem it; it.base = base; it.bstride = bstride; it.point = point; it.pad = 0; return it; };
  struct PRef { const Fp* base; long long bstride; int blind_slot; };
  auto poly_ref = [&](const PolyId& id) -> PRef {
    switch (id.kind) {
      case PK_INST: return {inst_polys + (size_t)id.idx * n, PS, V_ONE};
      case PK_ADV: return {adv_polys + (size_t)id.idx * n, PS, V_ADV_BLIND + id.idx};
      case PK_PZ: return {pz_polys + (size_t)id.idx * n, PS, V_PZ_BLIND + id.idx};
      case PK_LZ: return {lz_polys + (size_t)id.idx * n, PS, V_LZ_BLIND + id.idx};
      case PK_LPIN: return {lpin_polys + (size_t)id.idx * n, PS, V_LPIN_BLIND + id.idx};
      case PK_LPTAB: return {lptab_polys + (size_t)id.idx * n, PS, V_LPTAB_BLIND + id.idx};
      case PK_FIXED: return {C.fixed_polys.get() + (size_t)id.idx * n, 0, V_ONE};
      case PK_SIG: return {C.sig_polys.get() + (size_t)id.idx * n, 0, V_ONE};
      case PK_H: return {h_poly.get(), nn, V_H_BLIND};
      default: return {random_poly.get(), nn, V_RANDOM_BLIND};
    }
  };
  { std::vector<EvalItem> items;
    for (auto& e : C.evals) { PRef r = poly_ref(e.poly); items.push_back(mk_item(r.base, r.bstride, rot_slot(e.rot))); }
    const EvalItem* ditems = reinterpret_cast<const EvalItem*>(cached_upload(items.data(), items.size() * sizeof(EvalItem)));
    WBuf<Fp> ev = ws.buf<Fp>((size_t)B * items.size());
    poly_eval(ctx, ditems, (int)items.size(), vars.get(), NV, ev.get(), (long long)items.size(), (int)n, B);
    tr.scalars(ev.get(), (long long)items.size(), (int)items.size(), true); }

  // ---- multiopen
  tr.squeeze(VP(V_X1), NV, 1);
  tr.squeeze(VP(V_X2), NV, 1);
  WBuf<Fp> q_polys = ws.buf<Fp>((size_t)B * nps * n), q_prime = ws.buf<Fp>((size_t)B * n), kd_a = ws.buf<Fp>((size_t)B * n), kd_b = ws.buf<Fp>((size_t)B * n);
  { std::vector<char> started(nps, 0); Prog p;
    for (int s = 0; s < nps; ++s) p.op(S_SUB, V_QBLIND + s, V_QBLIND + s, V_QBLIND + s);
    for (size_t c = 0; c < C.uniq.size(); ++c) {
      PRef r = poly_ref(C.uniq[c]); int s = C.uniq_set[c];
      Fp* q = q_polys.get() + (size_t)s * n;
      if (!started[s]) { poly_copy(ctx, q, (long long)nps * nn, r.base, r.bstride, (int)n, B); started[s] = 1; }
      else poly_fma(ctx, q, (long long)nps * nn, VP(V_X1), NV, r.base, r.bstride, (int)n, B);
      p.op(S_FMA, V_QBLIND + s, V_X1, r.blind_slot);
    }
    run_prog(p); }
  for (int s = 0; s < nps; ++s) {
    const Fp* cur = q_polys.get() + (size_t)s * n; long long cur_stride = (long long)nps * nn;
    Fp* bufs[2] = {kd_a.get(), kd_b.get()}; int w = 0;
    for (int rot : C.point_sets[s]) {
      poly_kate_div(ctx, bufs[w], nn, cur, cur_stride, VP(rot_slot(rot)), NV, (int)n, B);
      cur = bufs[w]; cur_stride = nn; w ^= 1;
    }
    if (s == 0) poly_copy(ctx, q_prime.get(), nn, cur, cur_stride, (int)n, B);
    else poly_fma(ctx, q_prime.get(), nn, VP(V_X2), NV, cur, cur_stride, (int)n, B);
  }
  prf_fill(ctx, seed, proof0, R_QPRIME_BLIND, 0, VP(V_QPRIME_BLIND), NV, 1, 1, B);
  poly_copy(ctx, blinds.get(), 1, VP(V_QPRIME_BLIND), NV, 1, B);
  srs.commit(ctx, false, q_prime.get(), nn, B, blinds.get(), pts.get());
  tr.points(pts.get(), 1, 1, true);
  tr.squeeze(VP(V_X3), NV, 1);
  { std::vector<EvalItem> items;
    for (int s = 0; s < nps; ++s) items.push_back(mk_item(q_polys.get() + (size_t)s * n, (long long)nps * nn, V_X3));
    const EvalItem* ditems = reinterpret_cast<const EvalItem*>(cached_upload(items.data(), items.size() * sizeof(EvalItem)));
    WBuf<Fp> ev = ws.buf<Fp>((size_t)B * nps);
    poly_eval(ctx, ditems, nps, vars.get(), NV, ev.get(), nps, (int)n, B);
    tr.scalars(ev.get(), nps, nps, true); }
  tr.squeeze(VP(V_X4), NV, 1);
  // p(X) = ((q' x4 + q_0) x4 + q_1) ... ; same for the blinds
  WBuf<Fp> pprime = ws.buf<Fp>((size_t)B * n), bvec = ws.buf<Fp>((size_t)B * n), s_poly = ws.buf<Fp>((size_t)B * n);
  Fp* p_poly = q_prime.get();
  { Prog p; p.op(S_COPY, V_P_BLIND, V_QPRIME_BLIND);
    for (int s = 0; s < nps; ++s) { poly_fma(ctx, p_poly, nn, VP(V_X4), NV, q_polys.get() + (size_t)s * n, (long long)nps * nn, (int)n, B); p.op(S_FMA, V_P_BLIND, V_X4, V_QBLIND + s); }
    run_prog(p); }

  // ---- inner product argument (poly/commitment/prover.rs), s-vector form
  prf_fill(ctx, seed, proof0, R_S_POLY, 0, s_poly.get(), nn, 1, (int)n, B);
  prf_fill(ctx, seed, proof0, R_S_BLIND, 0, VP(V_S_BLIND), NV, 1, 1, B);
  auto eval_one = [&](const Fp* poly, int out_slot) {
    EvalItem it = mk_item(poly, nn, V_X3);
    const EvalItem* d = reinterpret_cast<const EvalItem*>(cached_upload(&it, sizeof(it)));
    poly_eval(ctx, d, 1, vars.get(), NV, VP(out_slot), NV, (int)n, B);
  };
  eval_one(s_poly.get(), V_S_AT);
  poly_add_at(ctx, s_poly.get(), nn, 0, VP(V_S_AT), NV, -1, B);
  poly_copy(ctx, blinds.get(), 1, VP(V_S_BLIND), NV, 1, B);
  srs.commit(ctx, false, s_poly.get(), nn, B, blinds.get(), pts.get());
  tr.points(pts.get(), 1, 1, true);
  tr.squeeze(VP(V_XI), NV, 1);
  tr.squeeze(VP(V_Z), NV, 1);
  poly_copy(ctx, pprime.get(), nn, s_poly.get(), nn, (int)n, B);
  poly_fma(ctx, pprime.get(), nn, VP(V_XI), NV, p_poly, nn, (int)n, B);
  eval_one(pprime.get(), V_V);
  poly_add_at(ctx, pprime.get(), nn, 0, VP(V_V), NV, -1, B);
  { Prog p; p.op(S_MUL, V_F, V_S_BLIND, V_XI); p.op(S_ADD, V_F, V_F, V_P_BLIND); run_prog(p); }
  powers(ctx, bvec.get(), nn, VP(V_X3), NV, (int)n, B);
  WBuf<Fp> sfull = ws.buf<Fp>((size_t)B * n), cLR = ws.buf<Fp>((size_t)B * 2 * n), ex = ws.buf<Fp>((size_t)B * 4);
  WBuf<Xyzz<Fq>> accLR = ws.buf<Xyzz<Fq>>((size_t)B * 2);
  WBuf<Aff<Fq>> ptLR = ws.buf<Aff<Fq>>((size_t)B * 2);
  launch(ctx, fill_const_kernel, (unsigned)(((size_t)B * n + 255) / 256), 256, 0, sfull.get(), (size_t)B * n, Fp::one());
  Prog round_prog;  // identical every round
  round_prog.op(S_INV, V_UINV, V_U); round_prog.op(S_MUL, V_T0, V_LR, V_UINV); round_prog.op(S_ADD, V_F, V_F, V_T0);
  round_prog.op(S_MUL, V_T0, V_RR, V_U); round_prog.op(S_ADD, V_F, V_F, V_T0);
  const ScalarInstr* d_round = reinterpret_cast<const ScalarInstr*>(cached_upload(round_prog.ins.data(), round_prog.ins.size() * sizeof(ScalarInstr)));
  for (int j = 0; j < k; ++j) {
    int m = (int)(n >> j), half = m >> 1;
    { ProfScope fold_scope(ctx, PC_IPA_FOLD);
      launch(ctx, ipa_round_scalars_kernel, dim3((unsigned)((n + 255) / 256), B), 256, 0, pprime.get(), sfull.get(), cLR.get(), (int)n, m); }
    inner_product(ctx, VP(V_VL), NV, pprime.get() + half, nn, bvec.get(), nn, half, B);
    inner_product(ctx, VP(V_VR), NV, pprime.get(), nn, bvec.get() + half, nn, half, B);
    prf_fill(ctx, seed, proof0, R_IPA_L, (uint32_t)j, VP(V_LR), NV, 1, 1, B);
    prf_fill(ctx, seed, proof0, R_IPA_R, (uint32_t)j, VP(V_RR), NV, 1, 1, B);
    launch(ctx, ipa_extras_kernel, (B + 31) / 32, 32, 0, ex.get(), vars.get(), NV, V_LR, V_RR, V_VL, V_VR, V_Z, B);
    // L_j, R_j = <cL | cR, g> + l_rand * w + (value * z) * u : one batched fixed-base MSM, K = 2 per proof
    srs.commit_xyzz(ctx, false, cLR.get(), nn, 2 * B, ex.get(), 2, accLR.get(), ptLR.get());
    tr.points(ptLR.get(), 2, 2, true);
    tr.squeeze(VP(V_U), NV, 1);
    scalar_program(ctx, vars.get(), NV, d_round, (int)round_prog.ins.size(), dconsts, B);
    { ProfScope fold_scope(ctx, PC_IPA_FOLD);
      launch(ctx, ipa_fold_kernel, dim3((unsigned)((n + 255) / 256), B), 256, 0, pprime.get(), bvec.get(), sfull.get(), (int)n, half, vars.get(), NV, V_U, V_UINV); }
  }
  poly_copy(ctx, VP(V_C), NV, pprime.get(), nn, 1, B);
  tr.scalars(VP(V_C), NV, 1, true);
  tr.scalars(VP(V_F), NV, 1, true);

  // ---- download (the only host synchronisation of the call)
  std::vector<TrState> hst(B);
  std::vector<uint32_t> herr((size_t)B * L1, 0);
  TB_CUDA(cudaMemcpyAsync(hst.data(), tr.states.get(), (size_t)B * sizeof(TrState), cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaMemcpyAsync(herr.data(), derr.get(), herr.size() * 4, cudaMemcpyDeviceToHost, st));
  TB_CUDA(cudaMemcpy2DAsync(proofs_out, proof_stride, tr.proofs.get(), C.proof_len, C.proof_len, B, cudaMemcpyDeviceToHost, st));
  ctx->sync();
  for (int b = 0; b < B; ++b) for (int l = 0; l < L; ++l)
    if (herr[(size_t)b * L + l])
      throw ConstraintError("proof " + std::to_string(b) + " of the batch (index " + std::to_string(proof0 + (uint32_t)b) + "): an input of lookup " + std::to_string(l) +
                            " is not contained in its table (ConstraintSystemFailure)");
  for (int b = 0; b < B; ++b) {
    if (hst[b].error & TR_ERR_INFINITY) throw std::runtime_error("cannot write points at infinity to the transcript");
    if (hst[b].error || hst[b].proof_len != C.proof_len) throw std::runtime_error("internal error: proof length mismatch");
  }
}

}  // namespace tb

using namespace tb;

extern "C" {

tb_status tb_circuit_load(tb_ctx* ctx, const tb_srs* srs, const tb_cs_desc* cs, const uint8_t* fixed_values, const uint8_t* sigma_values, tb_pk** out) {
  TB_API_BEGIN(ctx)
  TB_REQUIRE(srs && cs && out && (fixed_values || cs->num_fixed == 0) && (sigma_values || cs->num_perm_columns == 0), "tb_circuit_load arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  *out = reinterpret_cast<tb_pk*>(circuit_load(&ctx->c, reinterpret_cast<const Srs*>(srs), cs, fixed_values, sigma_values));
  TB_API_END(ctx)
}
void tb_pk_free(tb_pk* pk) { delete reinterpret_cast<Circuit*>(pk); }

// keygen_vk on the device: commit_lagrange(column, Blind::default() = 1) of every fixed and sigma column
tb_status tb_pk_commitments(tb_ctx* ctx, const tb_pk* pk, uint8_t* fixed_commitments, uint8_t* sigma_commitments) {
  TB_API_BEGIN(ctx)
  const Circuit* C = reinterpret_cast<const Circuit*>(pk);
  TB_REQUIRE(C && (fixed_commitments || C->nf == 0) && (sigma_commitments || C->P == 0), "tb_pk_commitments arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  Ctx* c = &ctx->c;
  for (int which = 0; which < 2; ++which) {
    int cnt = which ? (int)C->P : (int)C->nf;
    if (!cnt) continue;
    DevBuf<Fp> ones(c, cnt);
    DevBuf<Aff<Fq>> pts(c, cnt);
    std::vector<Fp> h(cnt, Fp::one());
    ones.upload(h.data(), cnt);
    C->srs->commit(c, true, which ? C->sig_vals.get() : C->fixed_vals.get(), (long long)C->n, cnt, ones.get(), pts.get());
    fe_from_mont<Fq>(c, reinterpret_cast<Fq*>(pts.get()), 2 * (size_t)cnt);
    pts.download(which ? sigma_commitments : fixed_commitments, cnt);
    c->sync();
  }
  TB_API_END(ctx)
}
size_t tb_pk_proof_len(const tb_pk* pk) { return pk ? reinterpret_cast<const Circuit*>(pk)->proof_len : 0; }

tb_status tb_prove_batch(tb_ctx* ctx, const tb_pk* pk, uint32_t n_proofs, const uint8_t* advice, const uint8_t* instance, const uint32_t* instance_len,
                         const uint8_t seed[32], uint32_t first_proof_index, uint8_t* proofs_out, size_t proof_stride) {
  TB_API_BEGIN(ctx)
  const Circuit* C = reinterpret_cast<const Circuit*>(pk);
  TB_REQUIRE(C && n_proofs >= 1 && advice && seed && proofs_out && proof_stride >= C->proof_len && (C->ni == 0 || (instance && instance_len)), "tb_prove_batch arguments");
  TB_REQUIRE((uint64_t)n_proofs * std::max<uint32_t>(C->na, C->pieces) <= 65535, "batch too large for one call");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  prove_batch(&ctx->c, *C, (int)n_proofs, advice, instance, instance_len, seed, first_proof_index, proofs_out, proof_stride);
  TB_API_END(ctx)
}

}  // extern "C"
