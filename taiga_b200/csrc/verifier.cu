// Batched verifier (SURVEY.md §8f-3): the transcript of every proof is replayed by one function (replay.cuh), on the host for
// proofs in host memory and on the device for proofs in device memory; the two multi-scalar multiplications of the final IPA
// check run on the device for the whole batch.
//
// Replaces halo2_proofs `plonk::verify_proof` with `SingleVerifier` as called by `Proof::verify`
// (taiga_halo2/src/proof.rs:45-54; serial loop over proofs in ShieldedPartialTxBundle::execute, transaction.rs:246-257).
// Accept iff   sum_i coef_i * C_i  +  xi*S  +  sum_j (u_j^-1 L_j + u_j R_j)  -  sum_t (c s_t + [t=0] v) g_t  -  (c b z) U  -  f W  ==  O
// where the C_i are every commitment of the proof, of the verifying key and of the instance, with the multiopen
// coefficients (SURVEY App. A.2/A.4).  The g-term is one fixed-base MSM over the SRS tables, the rest (W and U included) a
// ~100-term variable-base MSM per proof.  The batch verifier (tb_batch_verifier) sums these checks with random weights over
// any number of proofs and circuits: one shared g-term, one variable-base MSM per call.
#define TB_NOINLINE_MUL 1
#include <algorithm>
#include <cstdlib>
#include "capi_internal.cuh"
#include "circuit.cuh"
#include "replay.cuh"
#include "transcript.cuh"

namespace tb {

// One thread per point: the 32 bytes at in + (i / npts) * stride + off[i % npts] (off = nullptr: at in + stride * i), decoded
// as decompress_point decodes them.  out[i] = the point in Montgomery form (the identity for 32 zero bytes), ok[i] = 1 iff
// the encoding is canonical and on the curve (out[i] = the identity otherwise).
__global__ void decompress_kernel(const uint8_t* __restrict__ in, size_t stride, const uint32_t* __restrict__ off, int npts, size_t count,
                                  Aff<Fq>* __restrict__ out, uint8_t* __restrict__ ok) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const uint8_t* b = off ? in + (i / npts) * stride + off[i % npts] : in + stride * i;
  Aff<Fq> p;
  bool good = decompress_point(b, p);
  out[i] = good ? p.to_mont() : Aff<Fq>::inf();
  ok[i] = good ? 1 : 0;
}
static void decompress(Ctx* ctx, const uint8_t* d_in, size_t stride, const uint32_t* d_off, int npts, size_t count, Aff<Fq>* d_out, uint8_t* d_ok) {
  if (!count) return;
  ProfScope scope(ctx, PC_TRANSCRIPT);
  launch(ctx, decompress_kernel, (unsigned)((count + 127) / 128), 128, 0, d_in, stride, d_off, npts, count, d_out, d_ok);
}

// ok[p] = 1 iff a[p] + b[p] is the identity and (alive = nullptr or) alive[p] != 0
__global__ void verify_final_kernel(const Xyzz<Fq>* a, const Xyzz<Fq>* b, uint8_t* ok, int K, const uint8_t* alive) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= K) return;
  Xyzz<Fq> s = a[p]; s.add(b[p]);
  ok[p] = (s.is_inf() && (!alive || alive[p])) ? 1 : 0;
}

// commit_lagrange(column, Blind::default()) of `count` columns of n values at `vals` ([count][n], Montgomery): the points,
// Montgomery, on the device at `out`
static void commit_columns_dev(Ctx* ctx, const Srs& srs, const Fp* vals, int count, Aff<Fq>* out) {
  if (!count) return;
  DevBuf<Fp> ones(ctx, count);
  launch(ctx, fill_const_kernel, (unsigned)((count + 127) / 128), 128, 0, ones.get(), (size_t)count, Fp::one());
  srs.commit(ctx, true, vals, (long long)srs.n, count, ones.get(), out);
}
// the same, on the host
static std::vector<Aff<Fq>> commit_columns(Ctx* ctx, const Srs& srs, const Fp* vals, int count) {
  std::vector<Aff<Fq>> out(count, Aff<Fq>::inf());
  if (!count) return out;
  DevBuf<Aff<Fq>> pts(ctx, count);
  commit_columns_dev(ctx, srs, vals, count, pts.get());
  pts.download(out.data(), count); ctx->sync();
  return out;
}

// The ReplayShape of a shape with its tables packed in `blob`: until bind(base) its pointers are offsets into the blob, so
// one copy of the blob (host or device) serves the replay.  Building it checks, once per call, what the replay relies on:
// every evaluation it reads exists, the points lie at the offsets it reads them from, and it pushes exactly M terms.
struct ReplayPlan {
  ReplayShape v;
  std::vector<uint8_t> blob;
  template <class T> const T* put(const T* p, size_t n) {
    const size_t off = (blob.size() + 15) & ~size_t(15);
    blob.resize(off + std::max<size_t>(1, n) * sizeof(T));
    if (n) memcpy(blob.data() + off, p, n * sizeof(T));
    return reinterpret_cast<const T*>(off);
  }
  template <class T> const T* put(const std::vector<T>& x) { return put(x.data(), x.size()); }
  template <class T> static const T* at(const uint8_t* base, const T* off) { return reinterpret_cast<const T*>(base + reinterpret_cast<uintptr_t>(off)); }
  ReplayShape bind(const uint8_t* base) const {
    ReplayShape s = v;
    s.rots = at(base, s.rots); s.evpos = at(base, s.evpos); s.uniq = at(base, s.uniq); s.ps_off = at(base, s.ps_off); s.ps_rot = at(base, s.ps_rot);
    s.perm_kind = at(base, s.perm_kind); s.perm_idx = at(base, s.perm_idx); s.progs = at(base, s.progs); s.code = at(base, s.code); s.consts = at(base, s.consts);
    return s;
  }
};
static_assert((int)PK_INST == RP_INST && (int)PK_ADV == RP_ADV && (int)PK_PZ == RP_PZ && (int)PK_LZ == RP_LZ && (int)PK_LPIN == RP_LPIN && (int)PK_LPTAB == RP_LPTAB && (int)PK_FIXED == RP_FIXED &&
              (int)PK_SIG == RP_SIG && (int)PK_H == RP_H && (int)PK_RANDOM == RP_RANDOM, "replay.cuh numbers polynomials as circuit.cuh does");

static ReplayPlan replay_plan(const Shape& C) {
  auto internal = [](bool cond, const char* what) { if (!cond) throw std::logic_error(std::string("internal error: ") + what); };
  ReplayPlan R; ReplayShape& v = R.v;
  v.k = (int)C.k; v.na = (int)C.na; v.ni = (int)C.ni; v.L = (int)C.L; v.nsets = (int)C.nsets; v.P = (int)C.P; v.bf = (int)C.bf; v.pieces = (int)C.pieces;
  v.chunk = (int)C.chunk; v.nevals = (int)C.evals.size(); v.nuniq = (int)C.uniq.size(); v.nps = (int)C.point_sets.size(); v.npts = (int)C.point_offsets.size();
  v.proof_len = C.proof_len;
  v.vk_repr = C.vk_repr; v.omega = C.omega; v.omega_inv = C.omega.inv(); v.n_inv = Fp::from_u32((uint32_t)C.n).inv(); v.delta = C.delta;
  for (int s = 0; s < PERM_MAX_SETS; ++s) v.delta_c0[s] = C.delta_c0[s];
  // (poly, rotation) -> evaluation, dense
  const int counts[RP_KINDS] = {v.ni, v.na, v.nsets, v.L, v.L, v.L, (int)C.nf, v.P, 1, 1};
  int npoly = 0;
  for (int kd = 0; kd < RP_KINDS; ++kd) { v.poly_base[kd] = npoly; npoly += counts[kd]; }
  const std::vector<int>& rots = C.rots; v.nrots = (int)rots.size();
  auto rot_index = [&](int rot) { return (int)(std::find(rots.begin(), rots.end(), rot) - rots.begin()); };
  std::vector<int> evpos((size_t)npoly * v.nrots, -1);
  for (const auto& kv : C.eval_pos) {
    const int r = rot_index(kv.first.second);
    internal(r < v.nrots && kv.first.first.idx < counts[kv.first.first.kind], "an evaluation outside the replay's table");
    evpos[(size_t)(v.poly_base[kv.first.first.kind] + kv.first.first.idx) * v.nrots + r] = kv.second;
  }
  auto need = [&](int kind, int idx, int rot) {
    const int r = rot_index(rot);
    internal(idx >= 0 && idx < counts[kind] && r < v.nrots && evpos[(size_t)(v.poly_base[kind] + idx) * v.nrots + r] >= 0, "a query without an evaluation");
  };
  // the multiopen's commitments and point sets
  const int na = v.na, L = v.L, nsets = v.nsets, commits = na + 3 * L + nsets + 1 + v.pieces;
  std::vector<RpUniq> uniq; int nh = 0;
  for (int c = 0; c < v.nuniq; ++c) {
    const PolyId& id = C.uniq[c]; const int s = C.uniq_set[c];
    int src = -1;
    switch (id.kind) {
      case PK_ADV: src = id.idx; break;
      case PK_LPIN: src = na + 2 * id.idx; break;
      case PK_LPTAB: src = na + 2 * id.idx + 1; break;
      case PK_PZ: src = na + 2 * L + id.idx; break;
      case PK_LZ: src = na + 2 * L + nsets + id.idx; break;
      case PK_RANDOM: src = na + 2 * L + nsets + L; break;
      case PK_H: src = na + 2 * L + nsets + L + 1; ++nh; break;
      default: break;
    }
    uniq.push_back({id.kind, id.idx, s, src});
    for (int rot : C.point_sets[s]) need(id.kind, id.idx, rot);
  }
  std::vector<int> ps_off(1, 0), ps_rot; int max_set = 1;
  for (const auto& ps : C.point_sets) { ps_rot.insert(ps_rot.end(), ps.begin(), ps.end()); ps_off.push_back((int)ps_rot.size()); max_set = std::max(max_set, (int)ps.size()); }
  // the arguments' reads
  std::vector<int> perm_kind, perm_idx;
  for (int c = 0; c < v.P; ++c) {
    const PolyId id = column_poly(C.perm[c]);
    perm_kind.push_back(id.kind); perm_idx.push_back(id.idx);
    need(id.kind, id.idx, 0); need(PK_SIG, c, 0);
  }
  for (int s = 0; s < nsets; ++s) { need(PK_PZ, s, 0); need(PK_PZ, s, 1); if (s + 1 < nsets) need(PK_PZ, s, -(v.bf + 1)); }
  for (int l = 0; l < L; ++l) { need(PK_LZ, l, 0); need(PK_LZ, l, 1); need(PK_LPIN, l, 0); need(PK_LPIN, l, -1); need(PK_LPTAB, l, 0); }
  need(PK_H, 0, 0);
  // the gate programs, then the lookup program, with every column query they read
  std::vector<RpProgram> progs; std::vector<QInstr> code; int max_regs = 0;
  auto add = [&](const GateProgram& g) {
    progs.push_back({(int)code.size(), (int)g.code.size(), g.nregs, g.last});
    max_regs = std::max(max_regs, g.nregs);
    for (const QInstr& in : g.code) {
      const int kinds[2] = {(int)((in.w0 >> 16) & 0xff), (int)(in.w0 >> 24)}; const uint32_t vals[2] = {in.a, in.b};
      for (int o = 0; o < 2; ++o)
        if (kinds[o] == K_ADV || kinds[o] == K_FIX || kinds[o] == K_INST)
          need(kinds[o] == K_ADV ? PK_ADV : kinds[o] == K_FIX ? PK_FIXED : PK_INST, (int)(vals[o] >> 8), (int)(vals[o] & 255u) - 128);
      code.push_back(in);
    }
  };
  for (const auto* parts : {&C.plan.gate_parts[0], &C.plan.gate_parts_lo[0]})
    for (const GateProgram& g : *parts) add(g);
  v.ngates = (int)progs.size();
  add(C.plan.lookups);
  v.J = (int)C.plan.num_constraints; v.nypow = v.J + (int)C.plan.t_pl + 2;
  // the proof's layout: the commitments, the evaluations, q', the multiopen evaluations u, S, then k (L, R) pairs and (c, f)
  { std::vector<uint32_t> off; uint32_t pos = 0;
    for (int i = 0; i < commits; ++i, pos += 32) off.push_back(pos);
    pos += 32 * v.nevals; off.push_back(pos); pos += 32 + 32 * v.nps; off.push_back(pos); pos += 32;
    for (int j = 0; j < 2 * v.k; ++j, pos += 32) off.push_back(pos);
    pos += 64;
    internal(off == C.point_offsets && pos == C.proof_len, "proof point offsets"); }
  // every committed polynomial (h in its pieces), q', S, the L_j and R_j, W and U
  v.M = v.nuniq - 1 + v.pieces + 2 + 2 * v.k + 2;
  internal(nh == 1, "verifier term count");
  v.rots = R.put(rots); v.evpos = R.put(evpos); v.uniq = R.put(uniq); v.ps_off = R.put(ps_off); v.ps_rot = R.put(ps_rot);
  v.perm_kind = R.put(perm_kind); v.perm_idx = R.put(perm_idx); v.progs = R.put(progs); v.code = R.put(code); v.consts = R.put(C.consts_host);
  // scratch per proof
  int s = 0;
  auto carve = [&](int count) { const int at = s; s += std::max(1, count); return at; };
  v.s_ev = carve(v.nevals + 1); v.s_regs = carve(max_regs + 2); v.s_ypow = carve(v.nypow); v.s_lka = carve(L); v.s_lkt = carve(L);
  v.s_qev = carve(ps_off.back()); v.s_coef = carve(v.nuniq); v.s_cur = carve(v.nps); v.s_u = carve(v.nps); v.s_x4 = carve(v.nps + 1); v.s_ptsx = carve(max_set);
  v.scratch = s;
  return R;
}

// One thread per proof: replay_proof over device memory.  A proof rejected during its replay gets alive[p] = 0 and, when
// batch_alive is given, sets *batch_alive = 0.
constexpr int RP_THREADS = 32;
__global__ void __launch_bounds__(RP_THREADS) replay_kernel(const ReplayShape S, int K, const uint8_t* __restrict__ proofs, size_t stride, size_t len,
                                                            const uint8_t* __restrict__ inst, size_t inst_total, const Aff<Fq>* __restrict__ dec,
                                                            const uint8_t* __restrict__ dec_ok, const Aff<Fq>* __restrict__ inst_comm,
                                                            const Aff<Fq>* __restrict__ fixed, const Aff<Fq>* __restrict__ sigma, const Aff<Fq>* __restrict__ wu,
                                                            Fp* __restrict__ scratch, Aff<Fq>* __restrict__ pts, Fp* __restrict__ sc, Fp* __restrict__ us,
                                                            Fp* __restrict__ ab, uint8_t* __restrict__ alive, uint8_t* batch_alive) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= K) return;
  const ReplayIn in = {proofs + (size_t)p * stride, len, dec + (size_t)p * S.npts, dec_ok + (size_t)p * S.npts, inst + 32 * inst_total * p, inst_total,
                       inst_comm + (size_t)p * S.ni, fixed, sigma, wu[0], wu[1]};
  const ReplayOut out = {pts + (size_t)p * S.M, sc + (size_t)p * S.M, us + (size_t)p * S.k, ab + 2 * p};
  const bool good = replay_proof(S, in, scratch + (size_t)p * S.scratch, out);
  alive[p] = good ? 1 : 0;
  if (!good && batch_alive) *batch_alive = 0;
}

// What the transcript replay of K proofs leaves on the device for their final IPA checks.  Proof p's M variable-base terms
// are pts / sc at [p * M, (p + 1) * M), the last two W and U with their scalars -f and -c*b*z; us[p] = the kk IPA challenges
// u_j and ab[p] = (-c, -v), the coefficients of its g-term.  alive[p] = 0 for a proof rejected during the replay (a read that
// fails, an identity absorbed, a non-canonical scalar or instance value, trailing bytes); its terms are the identity times 0,
// its ab 0.
struct DevReplay {
  int M = 0;
  DevBuf<Aff<Fq>> pts; DevBuf<Fp> sc, us, ab; DevBuf<uint8_t> alive;
};

// Replays the transcripts of K proofs of proof_len == C.proof_len bytes (proof p at proofs + p * proof_stride, in device
// memory iff on_device) of the circuit of shape C, whose fixed / sigma commitments are `fixed` / `sigma` (Montgomery).
// Every point is decoded and every instance column committed on the device first.  Proofs in host memory are copied to the
// device for that, and are then replayed on the host after one wait, the results uploaded; proofs in device memory are
// replayed by replay_kernel, enqueued without waiting, which also clears *batch_alive (when given) for a rejected proof.
// Returns whether a host replay rejected a proof.
static bool replay_batch(Ctx* ctx, bool on_device, const Shape& C, const Srs& srs, const std::vector<Aff<Fq>>& fixed, const std::vector<Aff<Fq>>& sigma,
                         int K, const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs, size_t proof_stride, size_t proof_len,
                         DevReplay& r, uint8_t* batch_alive) {
  const int kk = (int)C.k, ni = C.ni;
  const size_t inst_total = instance_total(C, instance_len);
  // the shape's tables, the point offsets and, for the device replay, the key's commitments: one upload
  ReplayPlan plan = replay_plan(C);
  const uint32_t* o_off = plan.put(C.point_offsets);
  const Aff<Fq>* o_fixed = on_device ? plan.put(fixed) : nullptr; const Aff<Fq>* o_sigma = on_device ? plan.put(sigma) : nullptr;
  DevBuf<uint8_t> d_blob(ctx, plan.blob.size());
  d_blob.upload(plan.blob.data(), plan.blob.size());
  const ReplayShape S = plan.bind(on_device ? d_blob.get() : plan.blob.data());
  const int npts = S.npts;
  // ---- every point of the batch, decoded on the device: [K][npts]
  DevBuf<uint8_t> staged;
  if (!on_device) {
    staged = DevBuf<uint8_t>(ctx, (size_t)K * proof_len);
    TB_CUDA(cudaMemcpy2DAsync(staged.get(), proof_len, proofs, proof_stride, proof_len, K, cudaMemcpyHostToDevice, ctx->stream));
  }
  DevBuf<Aff<Fq>> dec(ctx, (size_t)K * npts); DevBuf<uint8_t> dec_ok(ctx, (size_t)K * npts);
  decompress(ctx, on_device ? proofs : staged.get(), on_device ? proof_stride : proof_len, ReplayPlan::at(d_blob.get(), o_off), npts, (size_t)K * npts,
             dec.get(), dec_ok.get());
  // ---- instance commitments for the whole batch: [K][ni]
  DevBuf<Aff<Fq>> inst_comm(ctx, (size_t)K * ni);
  if (ni) {
    DevBuf<Fp> iv(ctx, (size_t)K * ni * C.n);
    upload_instance(ctx, C, K, instance, instance_len, iv.get());
    commit_columns_dev(ctx, srs, iv.get(), K * ni, inst_comm.get());
  }
  // ---- per proof: the shared replay
  r.M = S.M;
  r.pts = DevBuf<Aff<Fq>>(ctx, (size_t)K * S.M); r.sc = DevBuf<Fp>(ctx, (size_t)K * S.M); r.us = DevBuf<Fp>(ctx, (size_t)K * kk);
  r.ab = DevBuf<Fp>(ctx, (size_t)K * 2); r.alive = DevBuf<uint8_t>(ctx, K);
  if (on_device) {
    DevBuf<Fp> scratch(ctx, (size_t)K * S.scratch);
    ProfScope scope(ctx, PC_TRANSCRIPT);
    launch(ctx, replay_kernel, (unsigned)((K + RP_THREADS - 1) / RP_THREADS), RP_THREADS, 0, S, K, proofs, proof_stride, proof_len, instance, inst_total,
           dec.get(), dec_ok.get(), inst_comm.get(), ReplayPlan::at(d_blob.get(), o_fixed), ReplayPlan::at(d_blob.get(), o_sigma), srs.wu.get(), scratch.get(),
           r.pts.get(), r.sc.get(), r.us.get(), r.ab.get(), r.alive.get(), batch_alive);
    return false;
  }
  std::vector<Aff<Fq>> h_dec(dec.n), h_inst(inst_comm.n); std::vector<uint8_t> h_ok(dec_ok.n);
  dec.download(h_dec.data(), h_dec.size()); dec_ok.download(h_ok.data(), h_ok.size());
  if (ni) inst_comm.download(h_inst.data(), h_inst.size());
  ctx->sync();
  std::vector<Aff<Fq>> pts((size_t)K * S.M, Aff<Fq>::inf());
  std::vector<Fp> sc((size_t)K * S.M, Fp::zero()), us((size_t)K * kk, Fp::zero()), ab((size_t)K * 2, Fp::zero()), scratch(S.scratch);
  std::vector<uint8_t> alive(K);
  for (int p = 0; p < K; ++p) {
    const ReplayIn in = {proofs + (size_t)p * proof_stride, proof_len, h_dec.data() + (size_t)p * npts, h_ok.data() + (size_t)p * npts,
                         instance + 32 * inst_total * p, inst_total, h_inst.data() + (size_t)p * ni, fixed.data(), sigma.data(), srs.w_host, srs.u_host};
    const ReplayOut out = {pts.data() + (size_t)p * S.M, sc.data() + (size_t)p * S.M, us.data() + (size_t)p * kk, ab.data() + 2 * p};
    alive[p] = replay_proof(S, in, scratch.data(), out) ? 1 : 0;
  }
  r.pts.upload(pts.data(), pts.size()); r.sc.upload(sc.data(), sc.size()); r.us.upload(us.data(), us.size()); r.ab.upload(ab.data(), ab.size());
  r.alive.upload(alive.data(), K);
  return std::find(alive.begin(), alive.end(), 0) != alive.end();
}

// K proofs of the circuit of shape C, each checked on its own: the replay, then both MSMs of every proof's final check for
// the whole batch on the device (each proof its own g-term), then the identity test.  d_ok[p] = 1 iff proof p passes its
// replay and its check; written in stream order.
static void verify_batch(Ctx* ctx, bool on_device, const Shape& C, const Srs& srs, const std::vector<Aff<Fq>>& fixed, const std::vector<Aff<Fq>>& sigma,
                         int K, const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs, size_t proof_stride, size_t proof_len,
                         uint8_t* d_ok) {
  const size_t n = C.n;
  DevReplay r;
  replay_batch(ctx, on_device, C, srs, fixed, sigma, K, instance, instance_len, proofs, proof_stride, proof_len, r, nullptr);
  DevBuf<Fp> d_gs(ctx, (size_t)K * n); DevBuf<Xyzz<Fq>> acc_v(ctx, K), acc_g(ctx, K);
  d_gs.zero();
  msm_run<Fq, Fp>(ctx, r.sc.get(), r.M, r.pts.get(), r.M, r.M, K, MsmConfig(), acc_v.get());
  batch_g_scalars(ctx, d_gs.get(), r.us.get(), r.ab.get(), (int)C.k, K, 1);
  srs.commit_xyzz(ctx, false, d_gs.get(), (long long)n, K, nullptr, 0, acc_g.get());
  launch(ctx, verify_final_kernel, (K + 31) / 32, 32, 0, acc_v.get(), acc_g.get(), d_ok, K, (const uint8_t*)r.alive.get());
}

// The same for proofs in host memory, waited for: the verdicts at ok_out on the host.  A proof_len other than the shape's
// gives 0 for every proof, nothing decoded.
static void verify_batch_host(Ctx* ctx, const Shape& C, const Srs& srs, const std::vector<Aff<Fq>>& fixed, const std::vector<Aff<Fq>>& sigma, int K,
                              const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs, size_t proof_stride, size_t proof_len,
                              uint8_t* ok_out) {
  memset(ok_out, 0, K);
  if (proof_len != C.proof_len) return;   // no proof of this length is accepted
  DevBuf<uint8_t> d_ok(ctx, K);
  verify_batch(ctx, false, C, srs, fixed, sigma, K, instance, instance_len, proofs, proof_stride, proof_len, d_ok.get());
  d_ok.download(ok_out, K); ctx->sync();
}

// ---------------------------------------------------------------- batch verifier (tb_batch_verifier)
// halo2's BatchVerifier: proof j's final-check sum is weighted by rho_j = PRF(seed, j, R_BATCH_WEIGHT, 0) and the weighted sums
// of every proof added are added up, so one test for the identity decides the whole batch.  All proofs commit over one SRS,
// so their g-terms share `g` (n scalars); everything else of a call's proofs goes through one variable-base MSM whose result
// is added into `acc`.  `next` is the j of the next proof; `rejected`: a proof was rejected before its final check on the host,
// `alive` = 0: one was rejected during a device replay.
struct BatchVerifier {
  const Srs* srs = nullptr; int device = 0; uint8_t seed[32];
  uint64_t next = 0;
  bool rejected = false;
  bool broken = false;      // an add failed after it began changing g / acc: only tb_batch_verifier_free is allowed
  bool finalized = false;
  const Ctx* pending = nullptr;   // the context whose stream may still hold device adds (compared, never dereferenced)
  DevMem<Fp> g;             // [n] sum_p rho_p (-c_p s_{p,t} - [t = 0] v_p), Montgomery
  DevMem<Xyzz<Fq>> acc;     // [1] sum_p rho_p (every variable-base term of proof p, W and U included)
  DevMem<uint8_t> alive;    // [1] 1 until a device replay rejects a proof
};

// Before `ctx` works on the batch: device adds another context enqueued must have run.  That context may be closed by now,
// so the whole device is waited for; a batch that stays on one context never waits here.
static void batch_claim(const Ctx* ctx, BatchVerifier& bv) {
  if (bv.pending && bv.pending != ctx) TB_CUDA(cudaDeviceSynchronize());
  bv.pending = nullptr;
}

// Per proof p of a call (one CTA each): its M variable-base scalars and ab[p], the coefficients of its g-term, times rho_p
__global__ void batch_weights_kernel(const Fp* __restrict__ rho, Fp* __restrict__ sc, int M, Fp* __restrict__ ab) {
  const int p = blockIdx.x;
  const Fp w = ldg_fe(rho + p);
  if (threadIdx.x < 2) { Fp* a = ab + 2 * p + threadIdx.x; st_fe(a, ld_fe(a) * w); }
  for (int i = threadIdx.x; i < M; i += blockDim.x) { Fp* s = sc + (size_t)p * M + i; st_fe(s, ld_fe(s) * w); }
}

__global__ void batch_acc_kernel(Xyzz<Fq>* acc, const Xyzz<Fq>* add) {
  Xyzz<Fq> s = *acc; s.add(*add); *acc = s;
}

// G[g][t] += sum_{p in group g} (a_p s_{p,t} + [t = 0] b_p), s_{p,t} = prod_j u_{p,j}^{bit_(kk-1-j)(t)}, (a_p, b_p) = ab[p],
// group g = proofs [g * group, min((g + 1) * group, K)).  With t = hi * 2^lb + lo (lb = min(kk, BG_LOG)), s_{p,t} = H_p(hi) *
// L_p(lo), H over the top kk - lb bits, L over the low lb bits.  One CTA per (hi, g): for BG_PROOFS proofs at a time it writes
// a_p H_p(hi) into entry 0 of a table in shared memory and doubles the table lb times (entries [m, 2m) = entries [0, m) times
// the u of bit log2(m)), which leaves a_p s_{p,t} in entry lo; each thread then adds its entries.  One product per (proof, t),
// plus ~(kk - lb)/2 per (proof, CTA) for H.
constexpr int BG_LOG = 8, BG_THREADS = 1 << BG_LOG, BG_PROOFS = 4;
__global__ void __launch_bounds__(BG_THREADS) batch_g_scalars_kernel(Fp* __restrict__ G, const Fp* __restrict__ us, const Fp* __restrict__ ab, int kk, int K,
                                                                     int group) {
  __shared__ Fp tab[BG_PROOFS][BG_THREADS];
  const int lb = kk < BG_LOG ? kk : BG_LOG, lo = threadIdx.x;
  const uint32_t hi = blockIdx.x;
  const int p_end = min(K, (int)(blockIdx.y + 1) * group);
  Fp acc = Fp::zero();
  for (int p0 = blockIdx.y * group; p0 < p_end; p0 += BG_PROOFS) {
    const int np = p_end - p0 < BG_PROOFS ? p_end - p0 : BG_PROOFS;
    if (lo < np) {
      const Fp* u = us + (size_t)(p0 + lo) * kk;
      Fp h = ldg_fe(ab + 2 * (p0 + lo));
      for (int j = 0; j < kk - lb; ++j) if ((hi >> (kk - lb - 1 - j)) & 1) h = h * ldg_fe(u + j);
      tab[lo][0] = h;
    }
    __syncthreads();
    for (int b = 0; b < lb; ++b) {
      for (int e = threadIdx.x; e < (np << b); e += BG_THREADS) {
        const int q = e >> b, i = e & ((1 << b) - 1);
        tab[q][(1 << b) + i] = tab[q][i] * ldg_fe(us + (size_t)(p0 + q) * kk + kk - 1 - b);
      }
      __syncthreads();
    }
    if (lo < (1 << lb)) for (int q = 0; q < np; ++q) acc = acc + tab[q][lo];
    if (hi == 0 && lo == 0) for (int q = 0; q < np; ++q) acc = acc + ldg_fe(ab + 2 * (p0 + q) + 1);
    __syncthreads();
  }
  if (lo < (1 << lb)) { Fp* g = G + ((size_t)blockIdx.y << kk) + ((size_t)hi << lb) + lo; st_fe(g, ld_fe(g) + acc); }
}

void batch_g_scalars(Ctx* ctx, Fp* G, const Fp* us, const Fp* ab, int kk, int K, int group) {
  TB_REQUIRE(kk >= 1 && kk <= 30 && K >= 1 && group >= 1 && (K - 1) / group < 65535, "batch_g_scalars shape");
  const int lb = kk < BG_LOG ? kk : BG_LOG;
  ProfScope scope(ctx, PC_IPA_FOLD);
  ctx->work[PC_IPA_FOLD] += (double)K * (double)(1ull << kk) * (1.0 + 0.5 * (kk - lb) / (1 << lb));
  launch(ctx, batch_g_scalars_kernel, dim3(1u << (kk - lb), (unsigned)((K - 1) / group + 1)), BG_THREADS, 0, G, us, ab, kk, K, group);
}

// Adds K replayed proofs (device terms pts / sc, M per proof, us, ab) of a circuit of k rows to the batch: their weights
// rho_{j0 + p}, their terms through one variable-base MSM into bv.acc, their g-terms into bv.g.  sc and ab are scaled in place.
static void batch_fold(Ctx* ctx, BatchVerifier& bv, uint32_t j0, int K, int M, int kk, const Aff<Fq>* pts, Fp* sc, const Fp* us, Fp* ab) {
  DevBuf<Fp> d_rho(ctx, K); DevBuf<Xyzz<Fq>> part(ctx, 1);
  { ProfScope scope(ctx, PC_IPA_FOLD);
    prf_fill(ctx, bv.seed, j0, R_BATCH_WEIGHT, 0, d_rho.get(), 1, 1, 1, K);
    ctx->work[PC_IPA_FOLD] += (double)K * (M + 2);
    launch(ctx, batch_weights_kernel, K, 128, 0, d_rho.get(), sc, M, ab); }
  msm_run<Fq, Fp>(ctx, sc, 0, pts, 0, K * M, 1, MsmConfig(), part.get());
  { ProfScope scope(ctx, PC_MSM_REDUCE);
    launch(ctx, batch_acc_kernel, 1, 1, 0, bv.acc.get(), part.get()); }
  batch_g_scalars(ctx, bv.g.get(), us, ab, kk, K, K);
}

// The proofs of one tb_batch_verifier_add (host memory) or tb_dev_batch_verifier_add (device memory): the replay, then
// batch_fold.  A host add does nothing once a proof was rejected, folds nothing when its replay rejects a proof, and waits
// for its work.  A device add folds every proof (a rejected one clears bv.alive and adds nothing: its terms and g-term
// coefficients are 0) and returns without waiting.
static void batch_add(Ctx* ctx, bool on_device, BatchVerifier& bv, const Shape& C, const Srs& srs, const std::vector<Aff<Fq>>& fixed,
                      const std::vector<Aff<Fq>>& sigma, int K, const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs,
                      size_t proof_stride, size_t proof_len) {
  const uint32_t j0 = (uint32_t)bv.next;
  batch_claim(ctx, bv);
  if (proof_len != C.proof_len) bv.rejected = true;   // no proof of this length is accepted: nothing is decoded
  else if (on_device || !bv.rejected) {
    bv.broken = on_device;   // the device replay writes bv.alive
    DevReplay r;
    if (replay_batch(ctx, on_device, C, srs, fixed, sigma, K, instance, instance_len, proofs, proof_stride, proof_len, r, on_device ? bv.alive.get() : nullptr))
      bv.rejected = true;
    else {
      bv.broken = true;
      batch_fold(ctx, bv, j0, K, r.M, (int)C.k, r.pts.get(), r.sc.get(), r.us.get(), r.ab.get());
      if (on_device) bv.pending = ctx;
      else ctx->sync();   // the batch may be used from another context (stream) next
      bv.broken = false;
    }
  }
  bv.next += (uint64_t)K;
}

// 1 iff no device replay rejected a proof and the weighted sum of every final check added is the identity: g through the
// SRS's fixed-base tables, plus acc
static uint8_t batch_finalize(Ctx* ctx, BatchVerifier& bv) {
  batch_claim(ctx, bv);
  DevBuf<Xyzz<Fq>> acc_g(ctx, 1); DevBuf<uint8_t> d_ok(ctx, 1);
  bv.srs->commit_xyzz(ctx, false, bv.g.get(), (long long)bv.srs->n, 1, nullptr, 0, acc_g.get());
  launch(ctx, verify_final_kernel, 1, 32, 0, bv.acc.get(), acc_g.get(), d_ok.get(), 1, (const uint8_t*)bv.alive.get());
  uint8_t ok = 0;
  d_ok.download(&ok, 1); ctx->sync();
  return ok;
}

// The verifying key of a proving key: commit_lagrange(column, Blind::default()) of every fixed and sigma column, computed on
// first use and kept with the key.
static const Circuit& pk_commitments(Ctx* ctx, const Circuit& C) {
  std::lock_guard<std::mutex> vk_lock(C.mu);
  if (C.vk_fixed.size() != (size_t)C.nf || C.vk_sigma.size() != (size_t)C.P) {
    C.vk_fixed = commit_columns(ctx, *C.srs, C.fixed_vals.get(), (int)C.nf);
    C.vk_sigma = commit_columns(ctx, *C.srs, C.sig_vals.get(), (int)C.P);
  }
  return C;
}

// Montgomery points -> 64 bytes each: canonical affine x || y, 64 zero bytes = the identity (the inverse of parse_commitments)
static void store_commitments(const std::vector<Aff<Fq>>& pts, uint8_t* b) {
  for (const Aff<Fq>& p : pts) { Aff<Fq> c = p.from_mont(); memcpy(b, c.x.l, 32); memcpy(b + 32, c.y.l, 32); b += 64; }
}

// cnt commitments of 64 bytes (canonical affine x || y, 64 zero bytes = the identity) -> Montgomery points; refuses a
// coordinate >= q and a point off the curve
static std::vector<Aff<Fq>> parse_commitments(const uint8_t* b, size_t cnt, const char* what) {
  std::vector<Aff<Fq>> out(cnt, Aff<Fq>::inf());
  for (size_t i = 0; i < cnt; ++i, b += 64) {
    bool zero = true; for (int j = 0; j < 64; ++j) zero &= b[j] == 0;
    if (zero) continue;
    Aff<Fq> p;
    TB_REQUIRE(canonical<Fq>(b, p.x) && canonical<Fq>(b + 32, p.y), std::string(what) + " commitment " + std::to_string(i) + ": a coordinate is not below q");
    TB_REQUIRE(p.y.sqr() == p.x.sqr() * p.x + Fq::from_u32(5), std::string(what) + " commitment " + std::to_string(i) + " is not on the curve");
    out[i] = p;
  }
  return out;
}

// Refuses (TB_ERR_INVALID, "<what> arguments") a verifier call of no proofs or more than 4096, without proofs, with rows
// shorter than proof_len or without the instance values of a circuit that has instance columns; and what instance_total
// refuses.  Every verifier entry point checks this before it changes or launches anything.
static void require_proofs(const Shape& C, uint32_t n_proofs, const void* instance, const uint32_t* instance_len, const void* proofs, size_t proof_stride,
                           size_t proof_len, const char* what) {
  TB_REQUIRE(n_proofs >= 1 && n_proofs <= 4096 && proofs && proof_stride >= proof_len && (C.ni == 0 || (instance && instance_len)),
             std::string(what) + " arguments");
  instance_total(C, instance_len);
}

// Refuses (TB_ERR_INVALID) an add of n_proofs proofs over `srs` on `ctx` that the batch cannot take, before the batch changes
static void require_batch(const Ctx& ctx, const BatchVerifier& bv, const Srs* srs, uint32_t n_proofs, const char* what) {
  TB_REQUIRE(!bv.finalized, std::string(what) + " after tb_batch_verifier_finalize");
  TB_REQUIRE(!bv.broken, "an earlier tb_batch_verifier_add failed part way: the batch can only be freed");
  TB_REQUIRE(srs == bv.srs, "the verifying key refers to another SRS than the batch");
  TB_REQUIRE(ctx.device == bv.device, "the context is on another device than the batch");
  TB_REQUIRE(bv.next + n_proofs <= (1ull << 32), "a batch holds at most 2^32 proofs");
}

}  // namespace tb

using namespace tb;
extern "C" {

tb_status tb_verify_batch(tb_ctx* ctx, const tb_pk* pk, uint32_t n_proofs, const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs,
                          size_t proof_stride, size_t proof_len, uint8_t* ok_out) {
  TB_API_BEGIN(ctx)
  const Circuit* C = reinterpret_cast<const Circuit*>(pk);
  TB_REQUIRE(C && ok_out, "tb_verify_batch arguments");
  require_proofs(*C, n_proofs, instance, instance_len, proofs, proof_stride, proof_len, "tb_verify_batch");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  pk_commitments(&ctx->c, *C);
  verify_batch_host(&ctx->c, *C, *C->srs, C->vk_fixed, C->vk_sigma, (int)n_proofs, instance, instance_len, proofs, proof_stride, proof_len, ok_out);
  TB_API_END(ctx)
}

// keygen_vk on the device: commit_lagrange(column, Blind::default() = 1) of every fixed and sigma column
tb_status tb_pk_commitments(tb_ctx* ctx, const tb_pk* pk, uint8_t* fixed_commitments, uint8_t* sigma_commitments) {
  TB_API_BEGIN(ctx)
  const Circuit* C = reinterpret_cast<const Circuit*>(pk);
  TB_REQUIRE(C && (fixed_commitments || C->nf == 0) && (sigma_commitments || C->P == 0), "tb_pk_commitments arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  pk_commitments(&ctx->c, *C);
  store_commitments(C->vk_fixed, fixed_commitments);
  store_commitments(C->vk_sigma, sigma_commitments);
  TB_API_END(ctx)
}

tb_status tb_vk_load(tb_ctx* ctx, const tb_srs* srs_, const tb_cs_desc* cs, const uint8_t* fixed_commitments, const uint8_t* sigma_commitments, tb_vk** out) {
  TB_API_BEGIN(ctx)
  const Srs* srs = reinterpret_cast<const Srs*>(srs_);
  TB_REQUIRE(srs && cs && out && (fixed_commitments || cs->num_fixed == 0) && (sigma_commitments || cs->num_perm_columns == 0), "tb_vk_load arguments");
  // the verifier combines the gate programs the same way whether the quotient's degree split is on or not
  std::unique_ptr<VerifyingKey> vk(new VerifyingKey{shape_build(cs, srs->k, true), srs, {}, {}});
  vk->fixed = parse_commitments(fixed_commitments, vk->shape.nf, "fixed");
  vk->sigma = parse_commitments(sigma_commitments, vk->shape.P, "sigma");
  *out = reinterpret_cast<tb_vk*>(vk.release());
  TB_API_END(ctx)
}
void tb_vk_free(tb_vk* vk) { delete reinterpret_cast<VerifyingKey*>(vk); }
size_t tb_vk_proof_len(const tb_vk* vk) { return vk ? reinterpret_cast<const VerifyingKey*>(vk)->shape.proof_len : 0; }

tb_status tb_verify_batch_vk(tb_ctx* ctx, const tb_vk* vk_, uint32_t n_proofs, const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs,
                             size_t proof_stride, size_t proof_len, uint8_t* ok_out) {
  TB_API_BEGIN(ctx)
  const VerifyingKey* vk = reinterpret_cast<const VerifyingKey*>(vk_);
  TB_REQUIRE(vk && ok_out, "tb_verify_batch_vk arguments");
  require_proofs(vk->shape, n_proofs, instance, instance_len, proofs, proof_stride, proof_len, "tb_verify_batch_vk");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  verify_batch_host(&ctx->c, vk->shape, *vk->srs, vk->fixed, vk->sigma, (int)n_proofs, instance, instance_len, proofs, proof_stride, proof_len, ok_out);
  TB_API_END(ctx)
}

tb_status tb_dev_verify_batch_vk(tb_ctx* ctx, const tb_vk* vk_, uint32_t n_proofs, const void* d_instance, const uint32_t* instance_len,
                                 const void* d_proofs, size_t proof_stride, size_t proof_len, void* d_ok_out) {
  TB_API_BEGIN(ctx)
  const VerifyingKey* vk = reinterpret_cast<const VerifyingKey*>(vk_);
  TB_REQUIRE(vk && d_ok_out, "tb_dev_verify_batch_vk arguments");
  require_proofs(vk->shape, n_proofs, d_instance, instance_len, d_proofs, proof_stride, proof_len, "tb_dev_verify_batch_vk");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  require_device_memory(ctx->c, {d_proofs, d_ok_out, vk->shape.ni ? d_instance : nullptr}, "tb_dev_verify_batch_vk");
  if (proof_len != vk->shape.proof_len)   // no proof of this length is accepted: nothing is decoded
    TB_CUDA(cudaMemsetAsync(d_ok_out, 0, n_proofs, ctx->c.stream));
  else
    verify_batch(&ctx->c, true, vk->shape, *vk->srs, vk->fixed, vk->sigma, (int)n_proofs, static_cast<const uint8_t*>(d_instance), instance_len,
                 static_cast<const uint8_t*>(d_proofs), proof_stride, proof_len, static_cast<uint8_t*>(d_ok_out));
  TB_API_END(ctx)
}

tb_status tb_batch_verifier_create(tb_ctx* ctx, const tb_srs* srs_, const uint8_t seed[32], tb_batch_verifier** out) {
  TB_API_BEGIN(ctx)
  const Srs* srs = reinterpret_cast<const Srs*>(srs_);
  TB_REQUIRE(srs && seed && out, "tb_batch_verifier_create arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  std::unique_ptr<BatchVerifier> bv(new BatchVerifier());
  bv->srs = srs; bv->device = ctx->c.device; memcpy(bv->seed, seed, 32);
  bv->g = DevMem<Fp>(srs->n);
  bv->acc = DevMem<Xyzz<Fq>>(1);
  // zero bytes: the scalar 0 (Montgomery) and the XYZZ identity
  TB_CUDA(cudaMemsetAsync(bv->g.get(), 0, srs->n * sizeof(Fp), ctx->c.stream));
  TB_CUDA(cudaMemsetAsync(bv->acc.get(), 0, sizeof(Xyzz<Fq>), ctx->c.stream));
  bv->alive = DevMem<uint8_t>(1);
  TB_CUDA(cudaMemsetAsync(bv->alive.get(), 1, 1, ctx->c.stream));
  ctx->c.sync();
  *out = reinterpret_cast<tb_batch_verifier*>(bv.release());
  TB_API_END(ctx)
}

tb_status tb_batch_verifier_add(tb_ctx* ctx, tb_batch_verifier* bv_, const tb_vk* vk_, uint32_t n_proofs, const uint8_t* instance,
                                const uint32_t* instance_len, const uint8_t* proofs, size_t proof_stride, size_t proof_len) {
  TB_API_BEGIN(ctx)
  BatchVerifier* bv = reinterpret_cast<BatchVerifier*>(bv_);
  const VerifyingKey* vk = reinterpret_cast<const VerifyingKey*>(vk_);
  TB_REQUIRE(bv && vk, "tb_batch_verifier_add arguments");
  require_proofs(vk->shape, n_proofs, instance, instance_len, proofs, proof_stride, proof_len, "tb_batch_verifier_add");
  require_batch(ctx->c, *bv, vk->srs, n_proofs, "tb_batch_verifier_add");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  batch_add(&ctx->c, false, *bv, vk->shape, *vk->srs, vk->fixed, vk->sigma, (int)n_proofs, instance, instance_len, proofs, proof_stride, proof_len);
  TB_API_END(ctx)
}

tb_status tb_dev_batch_verifier_add(tb_ctx* ctx, tb_batch_verifier* bv_, const tb_vk* vk_, uint32_t n_proofs, const void* d_instance,
                                    const uint32_t* instance_len, const void* d_proofs, size_t proof_stride, size_t proof_len) {
  TB_API_BEGIN(ctx)
  BatchVerifier* bv = reinterpret_cast<BatchVerifier*>(bv_);
  const VerifyingKey* vk = reinterpret_cast<const VerifyingKey*>(vk_);
  TB_REQUIRE(bv && vk, "tb_dev_batch_verifier_add arguments");
  require_proofs(vk->shape, n_proofs, d_instance, instance_len, d_proofs, proof_stride, proof_len, "tb_dev_batch_verifier_add");
  require_batch(ctx->c, *bv, vk->srs, n_proofs, "tb_dev_batch_verifier_add");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  require_device_memory(ctx->c, {d_proofs, vk->shape.ni ? d_instance : nullptr}, "tb_dev_batch_verifier_add");
  batch_add(&ctx->c, true, *bv, vk->shape, *vk->srs, vk->fixed, vk->sigma, (int)n_proofs, static_cast<const uint8_t*>(d_instance), instance_len,
            static_cast<const uint8_t*>(d_proofs), proof_stride, proof_len);
  TB_API_END(ctx)
}

tb_status tb_batch_verifier_finalize(tb_ctx* ctx, tb_batch_verifier* bv_, uint8_t* ok_out) {
  TB_API_BEGIN(ctx)
  BatchVerifier* bv = reinterpret_cast<BatchVerifier*>(bv_);
  TB_REQUIRE(bv && ok_out, "tb_batch_verifier_finalize arguments");
  TB_REQUIRE(!bv->finalized, "tb_batch_verifier_finalize after tb_batch_verifier_finalize");
  TB_REQUIRE(!bv->broken, "an earlier tb_batch_verifier_add failed part way: the batch can only be freed");
  TB_REQUIRE(ctx->c.device == bv->device, "the context is on another device than the batch");
  bv->finalized = true;
  *ok_out = 0;
  TB_CUDA(cudaSetDevice(ctx->c.device));
  if (!bv->rejected) *ok_out = batch_finalize(&ctx->c, *bv);
  TB_API_END(ctx)
}

void tb_batch_verifier_free(tb_batch_verifier* bv) { delete reinterpret_cast<BatchVerifier*>(bv); }

tb_status tb_decompress(tb_ctx* ctx, size_t n, const uint8_t* in, uint8_t* out, uint8_t* ok) {
  TB_API_BEGIN(ctx)
  TB_REQUIRE(in && out && ok && n >= 1, "tb_decompress arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  Ctx* c = &ctx->c;
  DevBuf<uint8_t> d_in(c, 32 * n), d_ok(c, n); DevBuf<Aff<Fq>> d_out(c, n);
  d_in.upload(in, 32 * n);
  decompress(c, d_in.get(), 32, nullptr, 1, n, d_out.get(), d_ok.get());
  fe_from_mont<Fq>(c, reinterpret_cast<Fq*>(d_out.get()), 2 * n);
  d_out.download(out, n); d_ok.download(ok, n);
  c->sync();
  TB_API_END(ctx)
}

}  // extern "C"
