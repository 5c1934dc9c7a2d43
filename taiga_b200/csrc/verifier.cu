// Batched verifier (SURVEY.md §8f-3): the transcript is replayed on the host, the two multi-scalar multiplications of
// the final IPA check run on the device for the whole batch.
//
// Replaces halo2_proofs `plonk::verify_proof` with `SingleVerifier` as called by `Proof::verify`
// (taiga_halo2/src/proof.rs:45-54; serial loop over proofs in ShieldedPartialTxBundle::execute, transaction.rs:246-257).
// Accept iff   sum_i coef_i * C_i  +  xi*S  +  sum_j (u_j^-1 L_j + u_j R_j)  -  sum_t (c s_t + [t=0] v) g_t  -  (c b z) U  -  f W  ==  O
// where the C_i are every commitment of the proof, of the verifying key and of the instance, with the multiopen
// coefficients (SURVEY App. A.2/A.4).  The g-term is one fixed-base MSM over the SRS tables (U and W are its two extra
// table columns), the rest a ~100-term variable-base MSM per proof.
#define TB_NOINLINE_MUL 1
#include <algorithm>
#include <cstdlib>
#include "capi_internal.cuh"
#include "circuit.cuh"
#include "transcript.cuh"

namespace tb {

// the transcript replayed over the bytes of one proof; `bad` once a read failed or the identity was absorbed
struct VTranscript : Transcript {
  const uint8_t* rd; size_t len, pos = 0; bool bad = false;
  VTranscript(const uint8_t* p, size_t n, const Fp& vk_repr) : rd(p), len(n) { start(vk_repr); }
  void common_point(const Aff<Fq>& p) { if (!absorb_point(p.from_mont())) bad = true; }
  bool read_point(Aff<Fq>& p) {
    Aff<Fq> c;
    if (pos + 32 > len || !decompress_point(rd + pos, c)) { bad = true; return false; }
    pos += 32;
    if (!absorb_point(c)) bad = true;
    p = c.to_mont(); return !bad;
  }
  bool read_scalar(Fp& s) {
    if (pos + 32 > len || !canonical<Fp>(rd + pos, s)) { bad = true; return false; }
    pos += 32; absorb_scalar(s.from_mont()); return true;
  }
};

// out[k][t] = -(c_k * s_t),  s_t = prod_j u_{k,j}^{bit_(kk-1-j)(t)};  t = 0 additionally gets -v_k
__global__ void verify_g_scalars_kernel(const Fp* __restrict__ us, const Fp* __restrict__ cv, Fp* __restrict__ out, int kk, int n) {
  int t = blockIdx.x * blockDim.x + threadIdx.x, p = blockIdx.y;
  if (t >= n) return;
  Fp s = cv[2 * p];
  for (int j = 0; j < kk; ++j) if ((t >> (kk - 1 - j)) & 1) s = s * us[(size_t)p * kk + j];
  if (t == 0) s = s + cv[2 * p + 1];
  st_fe(out + (size_t)p * n + t, s.neg());
}
__global__ void verify_final_kernel(const Xyzz<Fq>* a, const Xyzz<Fq>* b, uint8_t* ok, int K) {
  int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= K) return;
  Xyzz<Fq> s = a[p]; s.add(b[p]);
  ok[p] = s.is_inf() ? 1 : 0;
}

// the proof's evaluations at x, as argument.cuh reads them
struct EvalView {
  const Circuit& C; std::map<std::pair<PolyId, int>, Fp>& ev; int last_rot;
  Fp perm_col(int c) const { const tb_column& col = C.perm[c]; return ev[{{col.kind == TB_COL_ADVICE ? PK_ADV : col.kind == TB_COL_FIXED ? PK_FIXED : PK_INST, (int)col.index}, 0}]; }
  Fp sigma(int c) const { return ev[{{PK_SIG, c}, 0}]; }
  Fp z(int s) const { return ev[{{PK_PZ, s}, 0}]; }
  Fp z_next(int s) const { return ev[{{PK_PZ, s}, 1}]; }
  Fp z_last(int s) const { return ev[{{PK_PZ, s}, last_rot}]; }
};

static void verify_batch(Ctx* ctx, const Circuit& C, int K, const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs, size_t proof_stride,
                         size_t proof_len, uint8_t* ok_out) {
  const Srs& srs = *C.srs;
  const size_t n = C.n; const int kk = (int)C.k, na = C.na, ni = C.ni, L = C.L, nsets = C.nsets, P = C.P, bf = C.bf, nf = C.nf, pieces = C.pieces;
  cudaStream_t st = ctx->stream;
  size_t inst_total = 0; for (int c = 0; c < ni; ++c) inst_total += instance_len[c];
  for (int p = 0; p < K; ++p) ok_out[p] = 0;
  // ---- verifying-key commitments (computed once per circuit, cached)
  std::unique_lock<std::mutex> vk_lock(C.mu);
  if (C.vk_fixed.size() != (size_t)nf || C.vk_sigma.size() != (size_t)P) {
    for (int which = 0; which < 2; ++which) {
      int cnt = which ? P : nf;
      std::vector<Aff<Fq>>& dst = which ? C.vk_sigma : C.vk_fixed;
      dst.assign(cnt, Aff<Fq>::inf());
      if (!cnt) continue;
      DevBuf<Fp> ones(ctx, cnt); DevBuf<Aff<Fq>> pts(ctx, cnt);
      std::vector<Fp> h(cnt, Fp::one()); ones.upload(h.data(), cnt);
      srs.commit(ctx, true, which ? C.sig_vals.get() : C.fixed_vals.get(), (long long)n, cnt, ones.get(), pts.get());
      pts.download(dst.data(), cnt); ctx->sync();
    }
  }
  vk_lock.unlock();
  // ---- instance commitments for the whole batch: commit_lagrange(instance, Blind::default())
  std::vector<Aff<Fq>> inst_comm((size_t)K * std::max(1, ni), Aff<Fq>::inf());
  if (ni) {
    DevBuf<Fp> iv(ctx, (size_t)K * ni * n), ones(ctx, (size_t)K * ni); DevBuf<Aff<Fq>> pts(ctx, (size_t)K * ni);
    iv.zero();
    size_t off = 0;
    for (int c = 0; c < ni; ++c) {
      TB_REQUIRE(instance_len[c] <= C.usable, "InstanceTooLarge");
      if (instance_len[c])
        TB_CUDA(cudaMemcpy2DAsync(iv.get() + (size_t)c * n, (size_t)ni * n * 32, instance + 32 * off, inst_total * 32, (size_t)instance_len[c] * 32, K, cudaMemcpyHostToDevice, st));
      off += instance_len[c];
    }
    fe_to_mont<Fp>(ctx, iv.get(), (size_t)K * ni * n);
    std::vector<Fp> h((size_t)K * ni, Fp::one()); ones.upload(h.data(), h.size());
    srs.commit(ctx, true, iv.get(), (long long)n, K * ni, ones.get(), pts.get());
    pts.download(inst_comm.data(), (size_t)K * ni); ctx->sync();
  }
  // ---- per proof: replay the transcript, accumulate (scalar, point) pairs
  const int nps = (int)C.point_sets.size();
  const int M = ni + na + 3 * L + nsets + 1 + pieces + nf + P + 2 + 2 * kk;   // variable-base terms per proof
  int Mpad = 32; while (Mpad < M) Mpad *= 2;
  std::vector<Aff<Fq>> vpts((size_t)K * Mpad, Aff<Fq>::inf());
  std::vector<Fp> vsc((size_t)K * Mpad, Fp::zero()), us((size_t)K * kk, Fp::zero()), cv((size_t)K * 2, Fp::zero()), extras((size_t)K * 2, Fp::zero());
  std::vector<char> alive(K, 0);
  const Fp one = Fp::one();
  const int last_rot = -(bf + 1);
  Fp omega = C.omega, omega_inv = C.omega.inv(), n_inv = Fp::from_u32((uint32_t)n).inv();
  auto rot_pow = [&](int rot) { Fp r = one; const Fp& w = rot >= 0 ? omega : omega_inv; for (int i = 0; i < std::abs(rot); ++i) r = r * w; return r; };
  for (int p = 0; p < K; ++p) {
    VTranscript tr(proofs + (size_t)p * proof_stride, proof_len, C.vk_repr);
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
    // evaluations, in the prover's order (C.evals)
    std::map<std::pair<PolyId, int>, Fp> ev;
    for (auto& e : C.evals) {
      Fp v; if (!tr.read_scalar(v)) { ok = false; break; }
      ev[{e.poly, e.rot}] = v;
    }
    if (!ok) continue;
    // expected h(x)
    Fp xn = x; for (int i = 0; i < kk; ++i) xn = xn.sqr();
    auto l_at = [&](int rot) { Fp wi = rot_pow(rot); return (xn - one) * n_inv * wi * (x - wi).inv(); };
    Fp l_last = l_at(last_rot), l_blind = Fp::zero(), l_0 = l_at(0);
    for (int r = -bf; r <= -1; ++r) l_blind = l_blind + l_at(r);
    // the circuit's programs at x: the gates as the quotient combines its parts (sum_p y^(J - 1 - last_p) S_p), and the lookups
    const int J = (int)C.num_constraints;
    std::vector<Fp> ypow(J + C.t_pl + 2, one), lk_a(L), lk_t(L);
    for (size_t i = 1; i < ypow.size(); ++i) ypow[i] = ypow[i - 1] * y;
    auto at_x = [&](int kind, int col, int rot) { return ev[{{kind == K_ADV ? PK_ADV : kind == K_FIX ? PK_FIXED : PK_INST, col}, rot}]; };
    PointMachine<decltype(at_x)> m{at_x, C.consts_host.data(), ypow.data(), theta, lk_a.data(), lk_t.data()};
    Fp acc = Fp::zero();
    for (const auto* parts : {&C.gate_parts[0], &C.gate_parts_lo[0]})
      for (const QProgram& qp : *parts) acc = acc + ypow[J - 1 - qp.prog.last] * m.run(qp.prog);
    m.run(C.prog_lookups.prog);
    const ArgPoint at = {y, beta, gamma, l_0, l_last, one - (l_last + l_blind)};
    acc = perm_fold(acc, EvalView{C, ev, last_rot}, at, nsets, (int)C.chunk, P, C.delta, C.delta_c0, x);
    for (int l = 0; l < L; ++l)
      acc = lookup_fold(acc, at, ev[{{PK_LZ, l}, 0}], ev[{{PK_LZ, l}, 1}], ev[{{PK_LPIN, l}, 0}], ev[{{PK_LPIN, l}, -1}], ev[{{PK_LPTAB, l}, 0}], lk_a[l], lk_t[l]);
    ev[{{PK_H, 0}, 0}] = acc * (xn - one).inv();
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
        for (size_t pi = 0; pi < C.point_sets[s].size(); ++pi) {
          auto it = ev.find({C.uniq[c], C.point_sets[s][pi]});
          if (it == ev.end()) { ok = false; break; }
          q_evals[s][pi] = q_evals[s][pi] * x1 + it->second;
        }
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
    Aff<Fq>* pp = vpts.data() + (size_t)p * Mpad; Fp* ss = vsc.data() + (size_t)p * Mpad; int w = 0;
    auto push = [&](const Aff<Fq>& pt, const Fp& sc) { pp[w] = pt; ss[w] = sc; ++w; };
    for (size_t c = 0; c < C.uniq.size(); ++c) {
      const PolyId& id = C.uniq[c]; Fp coef = coef_in_set[id] * x4pow[nps - 1 - C.uniq_set[c]];
      if (id.kind == PK_H) { Fp cur = coef; for (int i = 0; i < pieces; ++i) { push(hpts[i], cur); cur = cur * xn; } }
      else if (id.kind == PK_FIXED) push(C.vk_fixed[id.idx], coef);
      else if (id.kind == PK_SIG) push(C.vk_sigma[id.idx], coef);
      else push(comm[id], coef);
    }
    push(q_prime, x4pow[nps]);
    push(s_comm, xi);
    for (int j = 0; j < kk; ++j) { push(Ls[j], uj[j].inv()); push(Rs[j], uj[j]); }
    if (w > Mpad) throw std::runtime_error("internal error: verifier term count");
    for (int j = 0; j < kk; ++j) us[(size_t)p * kk + j] = uj[j];
    cv[2 * p] = cc; cv[2 * p + 1] = v;
    extras[2 * p] = ff.neg();                    // * W
    extras[2 * p + 1] = (cc * b * z).neg();      // * U
    alive[p] = 1;
  }
  // ---- device: both MSMs for the whole batch, then the identity test
  DevBuf<Aff<Fq>> d_pts(ctx, vpts.size()); DevBuf<Fp> d_sc(ctx, vsc.size()), d_us(ctx, us.size()), d_cv(ctx, cv.size()), d_ex(ctx, extras.size()), d_gs(ctx, (size_t)K * n);
  DevBuf<Xyzz<Fq>> acc_v(ctx, K), acc_g(ctx, K); DevBuf<uint8_t> d_ok(ctx, K);
  d_pts.upload(vpts.data(), vpts.size()); d_sc.upload(vsc.data(), vsc.size()); d_us.upload(us.data(), us.size()); d_cv.upload(cv.data(), cv.size());
  d_ex.upload(extras.data(), extras.size());
  MsmConfig cfg;
  msm_run<Fq, Fp>(ctx, d_sc.get(), (long long)Mpad, d_pts.get(), (long long)Mpad, Mpad, K, cfg, acc_v.get());
  launch(ctx, verify_g_scalars_kernel, dim3((unsigned)((n + 255) / 256), K), 256, 0, d_us.get(), d_cv.get(), d_gs.get(), kk, (int)n);
  srs.commit_xyzz(ctx, false, d_gs.get(), (long long)n, K, d_ex.get(), 2, acc_g.get());
  launch(ctx, verify_final_kernel, (K + 31) / 32, 32, 0, acc_v.get(), acc_g.get(), d_ok.get(), K);
  std::vector<uint8_t> hok(K);
  d_ok.download(hok.data(), K); ctx->sync();
  for (int p = 0; p < K; ++p) ok_out[p] = (alive[p] && hok[p]) ? 1 : 0;
}

}  // namespace tb

using namespace tb;
extern "C" tb_status tb_verify_batch(tb_ctx* ctx, const tb_pk* pk, uint32_t n_proofs, const uint8_t* instance, const uint32_t* instance_len, const uint8_t* proofs,
                                     size_t proof_stride, size_t proof_len, uint8_t* ok_out) {
  TB_API_BEGIN(ctx)
  const Circuit* C = reinterpret_cast<const Circuit*>(pk);
  TB_REQUIRE(C && n_proofs >= 1 && n_proofs <= 4096 && proofs && ok_out && proof_stride >= proof_len && (C->ni == 0 || (instance && instance_len)), "tb_verify_batch arguments");
  TB_CUDA(cudaSetDevice(ctx->c.device));
  verify_batch(&ctx->c, *C, (int)n_proofs, instance, instance_len, proofs, proof_stride, proof_len, ok_out);
  TB_API_END(ctx)
}
