// Batched verifier (SURVEY.md §8f-3): the transcript is replayed on the host, the two multi-scalar multiplications of
// the final IPA check run on the device for the whole batch.
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

// the transcript replayed over the bytes of one proof; `bad` once a read failed or the identity was absorbed.  The points
// were decoded before the replay (pts / pts_ok: this proof's points in transcript order, at the offsets `offsets`).
struct VTranscript : Transcript {
  const uint8_t* rd; size_t len, pos = 0; bool bad = false;
  const Aff<Fq>* pts; const uint8_t* pts_ok; const std::vector<uint32_t>& offsets; size_t ipt = 0;
  VTranscript(const uint8_t* p, size_t n, const Fp& vk_repr, const Aff<Fq>* pts, const uint8_t* pts_ok, const std::vector<uint32_t>& offsets)
      : rd(p), len(n), pts(pts), pts_ok(pts_ok), offsets(offsets) { start(vk_repr); }
  void common_point(const Aff<Fq>& p) { if (!absorb_point(p.from_mont())) bad = true; }
  bool read_point(Aff<Fq>& p) {
    if (pos + 32 > len || ipt >= offsets.size()) { bad = true; return false; }
    if (offsets[ipt] != pos) throw std::logic_error("internal error: proof point offsets");
    if (!pts_ok[ipt]) { bad = true; return false; }
    p = pts[ipt++]; pos += 32;
    if (!absorb_point(p.from_mont())) bad = true;
    return !bad;
  }
  bool read_scalar(Fp& s) {
    if (pos + 32 > len || !canonical<Fp>(rd + pos, s)) { bad = true; return false; }
    pos += 32; absorb_scalar(s.from_mont()); return true;
  }
};

__global__ void verify_final_kernel(const Xyzz<Fq>* a, const Xyzz<Fq>* b, uint8_t* ok, int K) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= K) return;
  Xyzz<Fq> s = a[p]; s.add(b[p]);
  ok[p] = s.is_inf() ? 1 : 0;
}

// the proof's evaluations at x (C.evals order, then the expected h(x)), as argument.cuh reads them
struct EvalView {
  const Shape& C; const std::vector<Fp>& ev; int last_rot;
  Fp at(const PolyId& poly, int rot) const { return ev[C.eval_index(poly, rot)]; }
  Fp perm_col(int c) const { return at(column_poly(C.perm[c]), 0); }
  Fp sigma(int c) const { return at({PK_SIG, c}, 0); }
  Fp z(int s) const { return at({PK_PZ, s}, 0); }
  Fp z_next(int s) const { return at({PK_PZ, s}, 1); }
  Fp z_last(int s) const { return at({PK_PZ, s}, last_rot); }
};

// commit_lagrange(column, Blind::default()) of `count` columns of n values at `vals` ([count][n], Montgomery): the points,
// Montgomery, on the host
static std::vector<Aff<Fq>> commit_columns(Ctx* ctx, const Srs& srs, const Fp* vals, int count) {
  std::vector<Aff<Fq>> out(count, Aff<Fq>::inf());
  if (!count) return out;
  DevBuf<Fp> ones(ctx, count); DevBuf<Aff<Fq>> pts(ctx, count);
  std::vector<Fp> h(count, Fp::one()); ones.upload(h.data(), count);
  srs.commit(ctx, true, vals, (long long)srs.n, count, ones.get(), pts.get());
  pts.download(out.data(), count); ctx->sync();
  return out;
}

// What the transcript replay of K proofs leaves for their final IPA checks.  Proof p's M variable-base terms are pts / sc at
// [p * M, (p + 1) * M), the last two W and U with their scalars -f and -c*b*z; us[p] = the kk IPA challenges u_j and
// ab[p] = (-c, -v), the coefficients of its g-term.  alive[p] = 0 for a proof rejected during the replay (a read that fails,
// an identity absorbed, a non-canonical scalar or instance value, trailing bytes); its terms are the identity times 0, its ab 0.
struct Replay {
  int M = 0;
  std::vector<Aff<Fq>> pts; std::vector<Fp> sc, us, ab; std::vector<char> alive;
};

// Replays the transcripts of K proofs of proof_len == C.proof_len bytes of the circuit of shape C, whose fixed / sigma
// commitments are `vk_fixed` / `vk_sigma` (Montgomery).  Every point is decoded and every instance column committed on the
// device first.
static void replay_batch(Ctx* ctx, const Shape& C, const Srs& srs, const std::vector<Aff<Fq>>& vk_fixed, const std::vector<Aff<Fq>>& vk_sigma, int K,
                         const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs, size_t proof_stride, size_t proof_len, Replay& rep) {
  const size_t n = C.n; const int kk = (int)C.k, na = C.na, ni = C.ni, L = C.L, nsets = C.nsets, P = C.P, bf = C.bf, pieces = C.pieces;
  const size_t inst_total = instance_total(C, instance_len);
  // ---- every point of the batch, decoded on the device: [K][npts]
  const int npts = (int)C.point_offsets.size();
  std::vector<Aff<Fq>> dec((size_t)K * npts);
  std::vector<uint8_t> dec_ok((size_t)K * npts);
  { DevBuf<uint8_t> d_proofs(ctx, (size_t)K * proof_len), d_ok(ctx, dec_ok.size()); DevBuf<uint32_t> d_off(ctx, npts); DevBuf<Aff<Fq>> d_pts(ctx, dec.size());
    TB_CUDA(cudaMemcpy2DAsync(d_proofs.get(), proof_len, proofs, proof_stride, proof_len, K, cudaMemcpyHostToDevice, ctx->stream));
    d_off.upload(C.point_offsets.data(), npts);
    decompress(ctx, d_proofs.get(), proof_len, d_off.get(), npts, dec.size(), d_pts.get(), d_ok.get());
    d_pts.download(dec.data(), dec.size()); d_ok.download(dec_ok.data(), dec_ok.size()); ctx->sync(); }
  // ---- instance commitments for the whole batch: [K][ni]
  std::vector<Aff<Fq>> inst_comm;
  if (ni) {
    DevBuf<Fp> iv(ctx, (size_t)K * ni * n);
    upload_instance(ctx, C, K, instance, instance_len, iv.get());
    inst_comm = commit_columns(ctx, srs, iv.get(), K * ni);
  }
  // ---- per proof: replay the transcript, accumulate (scalar, point) pairs
  const int nps = (int)C.point_sets.size();
  // variable-base terms per proof: every committed polynomial (h in its pieces), q', S, the L_j and R_j, W and U
  rep.M = (int)C.uniq.size() - 1 + pieces + 2 + 2 * kk + 2;
  rep.pts.assign((size_t)K * rep.M, Aff<Fq>::inf());
  rep.sc.assign((size_t)K * rep.M, Fp::zero()); rep.us.assign((size_t)K * kk, Fp::zero()); rep.ab.assign((size_t)K * 2, Fp::zero());
  rep.alive.assign(K, 0);
  const Fp one = Fp::one();
  const int last_rot = -(bf + 1);
  Fp omega = C.omega, omega_inv = C.omega.inv(), n_inv = Fp::from_u32((uint32_t)n).inv();
  auto rot_pow = [&](int rot) { Fp r = one; const Fp& w = rot >= 0 ? omega : omega_inv; for (int i = 0; i < std::abs(rot); ++i) r = r * w; return r; };
  for (int p = 0; p < K; ++p) {
    VTranscript tr(proofs + (size_t)p * proof_stride, proof_len, C.vk_repr, dec.data() + (size_t)p * npts, dec_ok.data() + (size_t)p * npts, C.point_offsets);
    bool ok = true;
    const uint8_t* ib = instance + 32 * inst_total * p;
    for (size_t i = 0; i < inst_total && ok; ++i) { Fp t; ok = canonical<Fp>(ib + 32 * i, t); }
    if (!ok) continue;
    // commitment table for this proof: id -> point
    std::map<PolyId, Aff<Fq>> comm;
    for (int c = 0; c < ni; ++c) { comm[{PK_INST, c}] = inst_comm[(size_t)p * ni + c]; tr.common_point(inst_comm[(size_t)p * ni + c]); }
    auto rp = [&](PolyId id) { Aff<Fq> pt; if (!tr.read_point(pt)) return false; comm[id] = pt; return true; };
    for (int c = 0; c < na && ok; ++c) ok = rp({PK_ADV, c});
    Fp theta = tr.squeeze();
    for (int l = 0; l < L && ok; ++l) ok = rp({PK_LPIN, l}) && rp({PK_LPTAB, l});
    Fp beta = tr.squeeze(), gamma = tr.squeeze();
    for (int s = 0; s < nsets && ok; ++s) ok = rp({PK_PZ, s});
    for (int l = 0; l < L && ok; ++l) ok = rp({PK_LZ, l});
    ok = ok && rp({PK_RANDOM, 0});
    Fp y = tr.squeeze();
    std::vector<Aff<Fq>> hpts(pieces);
    for (int i = 0; i < pieces && ok; ++i) ok = tr.read_point(hpts[i]);
    Fp x = tr.squeeze();
    if (!ok) continue;
    // evaluations, in the prover's order (C.evals); the last entry is set to the expected h(x) below
    std::vector<Fp> ev(C.evals.size() + 1, Fp::zero());
    for (size_t i = 0; i < C.evals.size() && ok; ++i) ok = tr.read_scalar(ev[i]);
    if (!ok) continue;
    const EvalView view{C, ev, last_rot};
    // expected h(x)
    Fp xn = x; for (int i = 0; i < kk; ++i) xn = xn.sqr();
    auto l_at = [&](int rot) { Fp wi = rot_pow(rot); return (xn - one) * n_inv * wi * (x - wi).inv(); };
    Fp l_last = l_at(last_rot), l_blind = Fp::zero(), l_0 = l_at(0);
    for (int r = -bf; r <= -1; ++r) l_blind = l_blind + l_at(r);
    // the circuit's programs at x: the gates as the quotient combines its parts (sum_p y^(J - 1 - last_p) S_p), and the lookups
    const int J = (int)C.plan.num_constraints;
    std::vector<Fp> ypow(J + C.plan.t_pl + 2, one), lk_a(L), lk_t(L);
    for (size_t i = 1; i < ypow.size(); ++i) ypow[i] = ypow[i - 1] * y;
    auto at_x = [&](int kind, int col, int rot) { return view.at({kind == K_ADV ? PK_ADV : kind == K_FIX ? PK_FIXED : PK_INST, col}, rot); };
    PointMachine<decltype(at_x)> m{at_x, C.consts_host.data(), ypow.data(), theta, lk_a.data(), lk_t.data()};
    Fp acc = Fp::zero();
    for (const auto* parts : {&C.plan.gate_parts[0], &C.plan.gate_parts_lo[0]})
      for (const GateProgram& g : *parts) acc = acc + ypow[J - 1 - g.last] * m.run(g);
    m.run(C.plan.lookups);
    const ArgPoint at = {y, beta, gamma, l_0, l_last, one - (l_last + l_blind)};
    acc = perm_fold(acc, view, at, nsets, (int)C.chunk, P, C.delta, C.delta_c0, x);
    for (int l = 0; l < L; ++l)
      acc = lookup_fold(acc, at, view.at({PK_LZ, l}, 0), view.at({PK_LZ, l}, 1), view.at({PK_LPIN, l}, 0), view.at({PK_LPIN, l}, -1), view.at({PK_LPTAB, l}, 0),
                        lk_a[l], lk_t[l]);
    ev[C.eval_index({PK_H, 0}, 0)] = acc * (xn - one).inv();
    // ---- multiopen
    Fp x1 = tr.squeeze(), x2 = tr.squeeze();
    std::vector<std::vector<Fp>> q_evals(nps);
    for (int s = 0; s < nps; ++s) q_evals[s].assign(C.point_sets[s].size(), Fp::zero());
    std::map<PolyId, Fp> coef_in_set;   // coefficient of each commitment inside its q_commitment (power of x1)
    { std::vector<Fp> cur(nps, one); std::vector<char> started(nps, 0);
      // q_comm[s] = (...(C_first * x1 + C_2) * x1 + ...) : walk backwards so each commitment gets x1^(#later ones in its set)
      for (int c = (int)C.uniq.size() - 1; c >= 0; --c) { int s = C.uniq_set[c]; coef_in_set[C.uniq[c]] = cur[s]; cur[s] = cur[s] * x1; }
      for (size_t c = 0; c < C.uniq.size(); ++c) {
        int s = C.uniq_set[c];
        for (size_t pi = 0; pi < C.point_sets[s].size(); ++pi) q_evals[s][pi] = q_evals[s][pi] * x1 + view.at(C.uniq[c], C.point_sets[s][pi]);
      } }
    Aff<Fq> q_prime; ok = ok && tr.read_point(q_prime);
    Fp x3 = tr.squeeze();
    std::vector<Fp> u(nps); for (auto& e : u) ok = ok && tr.read_scalar(e);
    if (!ok) continue;
    Fp msm_eval = Fp::zero();
    for (int s = 0; s < nps; ++s) {
      size_t m = C.point_sets[s].size();
      std::vector<Fp> ptsx(m); for (size_t i = 0; i < m; ++i) ptsx[i] = x * rot_pow(C.point_sets[s][i]);
      Fp r_eval = Fp::zero();
      for (size_t i = 0; i < m; ++i) { Fp num = one, den = one; for (size_t j = 0; j < m; ++j) if (j != i) { num = num * (x3 - ptsx[j]); den = den * (ptsx[i] - ptsx[j]); } r_eval = r_eval + q_evals[s][i] * num * den.inv(); }
      Fp e = u[s] - r_eval;
      for (size_t i = 0; i < m; ++i) e = e * (x3 - ptsx[i]).inv();
      msm_eval = msm_eval * x2 + e;
    }
    Fp x4 = tr.squeeze();
    std::vector<Fp> x4pow(nps + 1, one); for (int i = 1; i <= nps; ++i) x4pow[i] = x4pow[i - 1] * x4;
    Fp v = msm_eval * x4pow[nps];
    for (int s = 0; s < nps; ++s) v = v + u[s] * x4pow[nps - 1 - s];
    // ---- IPA part of the transcript
    Aff<Fq> s_comm; ok = ok && tr.read_point(s_comm);
    Fp xi = tr.squeeze(), z = tr.squeeze();
    std::vector<Aff<Fq>> Ls(kk), Rs(kk); std::vector<Fp> uj(kk);
    for (int j = 0; j < kk && ok; ++j) { ok = tr.read_point(Ls[j]) && tr.read_point(Rs[j]); uj[j] = tr.squeeze(); }
    Fp cc, ff; ok = ok && tr.read_scalar(cc) && tr.read_scalar(ff);
    if (!ok || tr.bad || tr.pos != proof_len) continue;
    Fp b = one; { Fp cur = x3; for (int j = kk - 1; j >= 0; --j) { b = b * (one + uj[j] * cur); cur = cur * cur; } }
    // ---- variable-base terms
    Aff<Fq>* pp = rep.pts.data() + (size_t)p * rep.M; Fp* ss = rep.sc.data() + (size_t)p * rep.M; int w = 0;
    auto push = [&](const Aff<Fq>& pt, const Fp& sc) { pp[w] = pt; ss[w] = sc; ++w; };
    for (size_t c = 0; c < C.uniq.size(); ++c) {
      const PolyId& id = C.uniq[c]; Fp coef = coef_in_set[id] * x4pow[nps - 1 - C.uniq_set[c]];
      if (id.kind == PK_H) { Fp cur = coef; for (int i = 0; i < pieces; ++i) { push(hpts[i], cur); cur = cur * xn; } }
      else if (id.kind == PK_FIXED) push(vk_fixed[id.idx], coef);
      else if (id.kind == PK_SIG) push(vk_sigma[id.idx], coef);
      else push(comm[id], coef);
    }
    push(q_prime, x4pow[nps]);
    push(s_comm, xi);
    for (int j = 0; j < kk; ++j) { push(Ls[j], uj[j].inv()); push(Rs[j], uj[j]); }
    push(srs.w_host, ff.neg());
    push(srs.u_host, (cc * b * z).neg());
    if (w != rep.M) throw std::logic_error("internal error: verifier term count");
    for (int j = 0; j < kk; ++j) rep.us[(size_t)p * kk + j] = uj[j];
    rep.ab[2 * p] = cc.neg(); rep.ab[2 * p + 1] = v.neg();
    rep.alive[p] = 1;
  }
}

// n_proofs proofs of the circuit of shape C, each checked on its own: the replay, then both MSMs of every proof's final
// check for the whole batch on the device (each proof its own g-term), then the identity test
static void verify_batch(Ctx* ctx, const Shape& C, const Srs& srs, const std::vector<Aff<Fq>>& vk_fixed, const std::vector<Aff<Fq>>& vk_sigma, int K,
                         const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs, size_t proof_stride, size_t proof_len, uint8_t* ok_out) {
  const size_t n = C.n;
  instance_total(C, instance_len);
  for (int p = 0; p < K; ++p) ok_out[p] = 0;
  if (proof_len != C.proof_len) return;   // no proof of this length is accepted
  Replay r;
  replay_batch(ctx, C, srs, vk_fixed, vk_sigma, K, instance, instance_len, proofs, proof_stride, proof_len, r);
  DevBuf<Aff<Fq>> d_pts(ctx, r.pts.size()); DevBuf<Fp> d_sc(ctx, r.sc.size()), d_us(ctx, r.us.size()), d_ab(ctx, r.ab.size()), d_gs(ctx, (size_t)K * n);
  DevBuf<Xyzz<Fq>> acc_v(ctx, K), acc_g(ctx, K); DevBuf<uint8_t> d_ok(ctx, K);
  d_pts.upload(r.pts.data(), r.pts.size()); d_sc.upload(r.sc.data(), r.sc.size()); d_us.upload(r.us.data(), r.us.size()); d_ab.upload(r.ab.data(), r.ab.size());
  d_gs.zero();
  msm_run<Fq, Fp>(ctx, d_sc.get(), r.M, d_pts.get(), r.M, r.M, K, MsmConfig(), acc_v.get());
  batch_g_scalars(ctx, d_gs.get(), d_us.get(), d_ab.get(), (int)C.k, K, 1);
  srs.commit_xyzz(ctx, false, d_gs.get(), (long long)n, K, nullptr, 0, acc_g.get());
  launch(ctx, verify_final_kernel, (K + 31) / 32, 32, 0, acc_v.get(), acc_g.get(), d_ok.get(), K);
  std::vector<uint8_t> hok(K);
  d_ok.download(hok.data(), K); ctx->sync();
  for (int p = 0; p < K; ++p) ok_out[p] = (r.alive[p] && hok[p]) ? 1 : 0;
}

// ---------------------------------------------------------------- batch verifier (tb_batch_verifier)
// halo2's BatchVerifier: proof j's final-check sum is weighted by rho_j = PRF(seed, j, R_BATCH_WEIGHT, 0) and the weighted sums
// of every proof added are added up, so one test for the identity decides the whole batch.  All proofs commit over one SRS,
// so their g-terms share `g` (n scalars); everything else of a call's proofs goes through one variable-base MSM whose result
// is added into `acc`.  `next` is the j of the next proof; `rejected`: a proof was rejected before its final check.
struct BatchVerifier {
  const Srs* srs = nullptr; int device = 0; uint8_t seed[32];
  uint64_t next = 0;
  bool rejected = false;
  bool broken = false;      // an add failed after it began changing g / acc: only tb_batch_verifier_free is allowed
  bool finalized = false;
  DevMem<Fp> g;             // [n] sum_p rho_p (-c_p s_{p,t} - [t = 0] v_p), Montgomery
  DevMem<Xyzz<Fq>> acc;     // [1] sum_p rho_p (every variable-base term of proof p, W and U included)
};

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

// The proofs of one tb_batch_verifier_add: replay, then (unless a proof was rejected) their weights, their terms through one
// variable-base MSM into bv.acc, and their g-terms into bv.g.
static void batch_add(Ctx* ctx, BatchVerifier& bv, const VerifyingKey& vk, int K, const uint8_t* instance, const uint32_t* instance_len,
                      const uint8_t* proofs, size_t proof_stride, size_t proof_len) {
  const Shape& C = vk.shape;
  const uint32_t j0 = (uint32_t)bv.next;
  if (!bv.rejected && proof_len != C.proof_len) bv.rejected = true;   // no proof of this length is accepted
  if (!bv.rejected) {
    Replay r;
    replay_batch(ctx, C, *vk.srs, vk.fixed, vk.sigma, K, instance, instance_len, proofs, proof_stride, proof_len, r);
    if (std::find(r.alive.begin(), r.alive.end(), 0) != r.alive.end()) bv.rejected = true;
    else {
      const size_t N = (size_t)K * r.M;
      DevBuf<Aff<Fq>> d_pts(ctx, N); DevBuf<Fp> d_sc(ctx, N), d_us(ctx, r.us.size()), d_rho(ctx, K), d_ab(ctx, r.ab.size());
      DevBuf<Xyzz<Fq>> part(ctx, 1);
      d_pts.upload(r.pts.data(), N); d_sc.upload(r.sc.data(), N); d_us.upload(r.us.data(), r.us.size()); d_ab.upload(r.ab.data(), r.ab.size());
      bv.broken = true;
      { ProfScope scope(ctx, PC_IPA_FOLD);
        prf_fill(ctx, bv.seed, j0, R_BATCH_WEIGHT, 0, d_rho.get(), 1, 1, 1, K);
        ctx->work[PC_IPA_FOLD] += (double)K * (r.M + 2);
        launch(ctx, batch_weights_kernel, K, 128, 0, d_rho.get(), d_sc.get(), r.M, d_ab.get()); }
      msm_run<Fq, Fp>(ctx, d_sc.get(), 0, d_pts.get(), 0, (int)N, 1, MsmConfig(), part.get());
      { ProfScope scope(ctx, PC_MSM_REDUCE);
        launch(ctx, batch_acc_kernel, 1, 1, 0, bv.acc.get(), part.get()); }
      batch_g_scalars(ctx, bv.g.get(), d_us.get(), d_ab.get(), (int)C.k, K, K);
      ctx->sync();   // the batch may be used from another context (stream) next
      bv.broken = false;
    }
  }
  bv.next += (uint64_t)K;
}

// 1 iff the weighted sum of every final check added is the identity: g through the SRS's fixed-base tables, plus acc
static uint8_t batch_finalize(Ctx* ctx, const BatchVerifier& bv) {
  DevBuf<Xyzz<Fq>> acc_g(ctx, 1); DevBuf<uint8_t> d_ok(ctx, 1);
  bv.srs->commit_xyzz(ctx, false, bv.g.get(), (long long)bv.srs->n, 1, nullptr, 0, acc_g.get());
  launch(ctx, verify_final_kernel, 1, 32, 0, bv.acc.get(), acc_g.get(), d_ok.get(), 1);
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

}  // namespace tb

using namespace tb;
extern "C" {

tb_status tb_verify_batch(tb_ctx* ctx, const tb_pk* pk, uint32_t n_proofs, const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs,
                          size_t proof_stride, size_t proof_len, uint8_t* ok_out) {
  TB_API_BEGIN(ctx)
  const Circuit* C = reinterpret_cast<const Circuit*>(pk);
  TB_REQUIRE(C && n_proofs >= 1 && n_proofs <= 4096 && proofs && ok_out && proof_stride >= proof_len && (C->ni == 0 || (instance && instance_len)), "tb_verify_batch arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  pk_commitments(&ctx->c, *C);
  verify_batch(&ctx->c, *C, *C->srs, C->vk_fixed, C->vk_sigma, (int)n_proofs, instance, instance_len, proofs, proof_stride, proof_len, ok_out);
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
  TB_REQUIRE(vk && n_proofs >= 1 && n_proofs <= 4096 && proofs && ok_out && proof_stride >= proof_len && (vk->shape.ni == 0 || (instance && instance_len)),
             "tb_verify_batch_vk arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  verify_batch(&ctx->c, vk->shape, *vk->srs, vk->fixed, vk->sigma, (int)n_proofs, instance, instance_len, proofs, proof_stride, proof_len, ok_out);
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
  ctx->c.sync();
  *out = reinterpret_cast<tb_batch_verifier*>(bv.release());
  TB_API_END(ctx)
}

tb_status tb_batch_verifier_add(tb_ctx* ctx, tb_batch_verifier* bv_, const tb_vk* vk_, uint32_t n_proofs, const uint8_t* instance,
                                const uint32_t* instance_len, const uint8_t* proofs, size_t proof_stride, size_t proof_len) {
  TB_API_BEGIN(ctx)
  BatchVerifier* bv = reinterpret_cast<BatchVerifier*>(bv_);
  const VerifyingKey* vk = reinterpret_cast<const VerifyingKey*>(vk_);
  // every refusal comes before the batch changes
  TB_REQUIRE(bv && vk && n_proofs >= 1 && n_proofs <= 4096 && proofs && proof_stride >= proof_len && (vk->shape.ni == 0 || (instance && instance_len)),
             "tb_batch_verifier_add arguments");
  TB_REQUIRE(!bv->finalized, "tb_batch_verifier_add after tb_batch_verifier_finalize");
  TB_REQUIRE(!bv->broken, "an earlier tb_batch_verifier_add failed part way: the batch can only be freed");
  TB_REQUIRE(vk->srs == bv->srs, "the verifying key refers to another SRS than the batch");
  TB_REQUIRE(ctx->c.device == bv->device, "the context is on another device than the batch");
  TB_REQUIRE(bv->next + n_proofs <= (1ull << 32), "a batch holds at most 2^32 proofs");
  instance_total(vk->shape, instance_len);
  TB_CUDA(cudaSetDevice(ctx->c.device));
  batch_add(&ctx->c, *bv, *vk, (int)n_proofs, instance, instance_len, proofs, proof_stride, proof_len);
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
