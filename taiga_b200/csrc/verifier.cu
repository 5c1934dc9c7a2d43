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

namespace tb {

// ---------------------------------------------------------------- host BLAKE2b (transcript replay)
struct HostBlake2b {
  uint64_t h[8], t = 0; uint8_t buf[128]; size_t buflen = 0;
  static uint64_t rotr(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }
  explicit HostBlake2b(const char* personal16) {
    static const uint64_t iv[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                                   0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
    memcpy(h, iv, 64); h[0] ^= 0x01010040ULL;
    uint64_t p[2]; memcpy(p, personal16, 16); h[6] ^= p[0]; h[7] ^= p[1];
  }
  void compress(const uint8_t* block, bool last) {
    static const uint64_t iv[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                                   0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
    static const uint8_t S[12][16] = {
        {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
        {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
        {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
        {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
        {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
        {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};
    uint64_t m[16], v[16];
    memcpy(m, block, 128);
    for (int i = 0; i < 8; ++i) { v[i] = h[i]; v[i + 8] = iv[i]; }
    v[12] ^= t; if (last) v[14] = ~v[14];
    auto G = [&](int a, int b, int c, int d, uint64_t x, uint64_t y) {
      v[a] = v[a] + v[b] + x; v[d] = rotr(v[d] ^ v[a], 32); v[c] = v[c] + v[d]; v[b] = rotr(v[b] ^ v[c], 24);
      v[a] = v[a] + v[b] + y; v[d] = rotr(v[d] ^ v[a], 16); v[c] = v[c] + v[d]; v[b] = rotr(v[b] ^ v[c], 63);
    };
    for (int r = 0; r < 12; ++r) {
      const uint8_t* s = S[r];
      G(0, 4, 8, 12, m[s[0]], m[s[1]]); G(1, 5, 9, 13, m[s[2]], m[s[3]]); G(2, 6, 10, 14, m[s[4]], m[s[5]]); G(3, 7, 11, 15, m[s[6]], m[s[7]]);
      G(0, 5, 10, 15, m[s[8]], m[s[9]]); G(1, 6, 11, 12, m[s[10]], m[s[11]]); G(2, 7, 8, 13, m[s[12]], m[s[13]]); G(3, 4, 9, 14, m[s[14]], m[s[15]]);
    }
    for (int i = 0; i < 8; ++i) h[i] ^= v[i] ^ v[i + 8];
  }
  void update(const void* data, size_t len) {
    const uint8_t* p = (const uint8_t*)data;
    while (len) {
      if (buflen == 128) { t += 128; compress(buf, false); buflen = 0; }
      size_t take = std::min(len, (size_t)128 - buflen);
      memcpy(buf + buflen, p, take); buflen += take; p += take; len -= take;
    }
  }
  void digest(uint8_t* out) const {
    HostBlake2b c = *this;
    c.t += c.buflen; memset(c.buf + c.buflen, 0, 128 - c.buflen); c.compress(c.buf, true);
    memcpy(out, c.h, 64);
  }
};

template <class F> static bool canonical(const uint8_t* b, F& out) {  // 32 LE bytes < modulus -> Montgomery
  F raw; memcpy(raw.l, b, 32);
  F m; for (int i = 0; i < 8; ++i) m.l[i] = F::modulus_limb(i);
  if (F::cmp_raw(raw, m) >= 0) return false;
  out = raw.to_mont(); return true;
}
static Fp wide_reduce(const uint8_t* d64) {  // Challenge255: 64 LE bytes mod p
  Fp lo, hi; memcpy(lo.l, d64, 32); memcpy(hi.l, d64 + 32, 32);
  Fp r2 = Fp::r2();
  return r2 * lo + r2 * (r2 * hi);
}
// Tonelli-Shanks in Fq (2-adicity 32)
static bool fq_sqrt(const Fq& a, Fq& out) {
  if (a.is_zero()) { out = a; return true; }
  uint32_t q[8]; for (int i = 0; i < 8; ++i) q[i] = Fq::modulus_limb(i);
  q[0] -= 1;                                    // m - 1 = 2^32 * odd
  uint32_t odd[8]; for (int i = 0; i < 7; ++i) odd[i] = q[i + 1]; odd[7] = 0;
  uint32_t h[8];                                // (odd + 1) / 2
  { uint64_t c = 1; for (int i = 0; i < 8; ++i) { c += odd[i]; h[i] = (uint32_t)c; c >>= 32; }
    for (int i = 0; i < 8; ++i) h[i] = (h[i] >> 1) | (i < 7 ? (h[i + 1] << 31) : 0); }
  Fq c = root_of_unity_2_32<Fq>(), t = a.pow(odd, 8), r = a.pow(h, 8);
  int m = 32;
  Fq one = Fq::one();
  while (t != one) {
    int i = 0; Fq t2 = t;
    while (t2 != one) { t2 = t2.sqr(); if (++i == m) return false; }
    Fq b = c; for (int j = 0; j < m - i - 1; ++j) b = b.sqr();
    m = i; c = b.sqr(); t = t * c; r = r * b;
  }
  out = r; return true;
}
static bool decompress(const uint8_t* b, Aff<Fq>& out) {  // pasta encoding: x LE, bit 255 = parity of y; identity = zeros
  uint8_t t[32]; memcpy(t, b, 32);
  int sign = t[31] >> 7; t[31] &= 0x7f;
  bool allz = true; for (int i = 0; i < 32; ++i) allz &= (t[i] == 0);
  if (allz && !sign) { out = Aff<Fq>::inf(); return true; }
  Fq x; if (!canonical<Fq>(t, x)) return false;
  Fq y; if (!fq_sqrt(x.sqr() * x + Fq::from_u32(5), y)) return false;
  if ((int)(y.from_mont().l[0] & 1) != sign) y = y.neg();
  out.x = x; out.y = y; return true;
}

struct VTranscript {
  HostBlake2b st; const uint8_t* rd; size_t len, pos = 0; bool bad = false;
  VTranscript(const uint8_t* p, size_t n) : st("Halo2-Transcript"), rd(p), len(n) {}
  void common_point(const Aff<Fq>& p) {
    if (p.is_inf()) { bad = true; return; }
    uint8_t b[65]; b[0] = 1; Fq x = p.x.from_mont(), y = p.y.from_mont(); memcpy(b + 1, x.l, 32); memcpy(b + 33, y.l, 32); st.update(b, 65);
  }
  void common_scalar(const Fp& s) { uint8_t b[33]; b[0] = 2; Fp c = s.from_mont(); memcpy(b + 1, c.l, 32); st.update(b, 33); }
  Fp squeeze() { uint8_t z = 0; st.update(&z, 1); uint8_t d[64]; st.digest(d); return wide_reduce(d); }
  bool read_point(Aff<Fq>& p) {
    if (pos + 32 > len || !decompress(rd + pos, p)) { bad = true; return false; }
    pos += 32; common_point(p); return !bad;
  }
  bool read_scalar(Fp& s) {
    if (pos + 32 > len || !canonical<Fp>(rd + pos, s)) { bad = true; return false; }
    pos += 32; common_scalar(s); return true;
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

static Fp eval_expr(const Circuit& C, uint32_t root, std::vector<Fp>& memo, std::vector<char>& done, const std::vector<Fp>& adv, const std::vector<Fp>& fix,
                    const std::vector<Fp>& inst) {
  if (done[root]) return memo[root];
  const tb_expr_node& nd = C.nodes[root];
  Fp r;
  switch (nd.op) {
    case TB_EX_CONST: { Fp c; memcpy(c.l, C.consts_bytes.data() + 32 * nd.a, 32); r = c.to_mont(); break; }
    case TB_EX_ADVICE: r = adv[nd.a]; break;
    case TB_EX_FIXED: r = fix[nd.a]; break;
    case TB_EX_INSTANCE: r = inst[nd.a]; break;
    case TB_EX_NEG: r = eval_expr(C, nd.a, memo, done, adv, fix, inst).neg(); break;
    case TB_EX_ADD: r = eval_expr(C, nd.a, memo, done, adv, fix, inst) + eval_expr(C, nd.b, memo, done, adv, fix, inst); break;
    case TB_EX_MUL: r = eval_expr(C, nd.a, memo, done, adv, fix, inst) * eval_expr(C, nd.b, memo, done, adv, fix, inst); break;
    default: { Fp c; memcpy(c.l, C.consts_bytes.data() + 32 * nd.b, 32); r = eval_expr(C, nd.a, memo, done, adv, fix, inst) * c.to_mont(); }
  }
  memo[root] = r; done[root] = 1;
  return r;
}

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
    VTranscript tr(proofs + (size_t)p * proof_stride, proof_len);
    { Fp repr = C.vk_repr.to_mont(); tr.common_scalar(repr); }
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
    std::vector<Fp> adv_ev, fix_ev, inst_ev;
    for (auto& e : C.evals) {
      Fp v; if (!tr.read_scalar(v)) { ok = false; break; }
      ev[{e.poly, e.rot}] = v;
    }
    if (!ok) continue;
    for (auto& q : C.iq) inst_ev.push_back(ev[{{PK_INST, (int)q.column}, q.rotation}]);
    for (auto& q : C.aq) adv_ev.push_back(ev[{{PK_ADV, (int)q.column}, q.rotation}]);
    for (auto& q : C.fq) fix_ev.push_back(ev[{{PK_FIXED, (int)q.column}, q.rotation}]);
    // expected h(x)
    Fp xn = x; for (int i = 0; i < kk; ++i) xn = xn.sqr();
    auto l_at = [&](int rot) { Fp wi = rot_pow(rot); return (xn - one) * n_inv * wi * (x - wi).inv(); };
    Fp l_last = l_at(last_rot), l_blind = Fp::zero(), l_0 = l_at(0);
    for (int r = -bf; r <= -1; ++r) l_blind = l_blind + l_at(r);
    std::vector<Fp> memo(C.nodes.size()); std::vector<char> done(C.nodes.size(), 0);
    Fp acc = Fp::zero();
    for (uint32_t r : C.roots) acc = acc * y + eval_expr(C, r, memo, done, adv_ev, fix_ev, inst_ev);
    Fp active = one - (l_last + l_blind);
    auto col_eval = [&](const tb_column& c) { return ev[{{c.kind == TB_COL_ADVICE ? PK_ADV : c.kind == TB_COL_FIXED ? PK_FIXED : PK_INST, (int)c.index}, 0}]; };
    if (nsets) {
      auto pz = [&](int s, int rot) { return ev[{{PK_PZ, s}, rot}]; };
      acc = acc * y + l_0 * (one - pz(0, 0));
      acc = acc * y + (pz(nsets - 1, 0).sqr() - pz(nsets - 1, 0)) * l_last;
      for (int s = 1; s < nsets; ++s) acc = acc * y + (pz(s, 0) - pz(s - 1, last_rot)) * l_0;
      for (int s = 0; s < nsets; ++s) {
        int c0 = s * (int)C.chunk, c1 = std::min(P, c0 + (int)C.chunk);
        Fp left = pz(s, 1), right = pz(s, 0), cd = beta * x * C.delta_c0[s];
        for (int c = c0; c < c1; ++c) {
          Fp e = col_eval(C.perm[c]);
          left = left * (e + beta * ev[{{PK_SIG, c}, 0}] + gamma); right = right * (e + cd + gamma); cd = cd * C.delta;
        }
        acc = acc * y + (left - right) * active;
      }
    }
    for (int l = 0; l < L; ++l) {
      Fp a = Fp::zero(), t = Fp::zero();
      for (uint32_t r : C.lk_in[l]) a = a * theta + eval_expr(C, r, memo, done, adv_ev, fix_ev, inst_ev);
      for (uint32_t r : C.lk_tab[l]) t = t * theta + eval_expr(C, r, memo, done, adv_ev, fix_ev, inst_ev);
      Fp z = ev[{{PK_LZ, l}, 0}], zn = ev[{{PK_LZ, l}, 1}], ap = ev[{{PK_LPIN, l}, 0}], am = ev[{{PK_LPIN, l}, -1}], sp = ev[{{PK_LPTAB, l}, 0}];
      acc = acc * y + l_0 * (one - z);
      acc = acc * y + l_last * (z.sqr() - z);
      acc = acc * y + (zn * (ap + beta) * (sp + gamma) - z * (a + beta) * (t + gamma)) * active;
      acc = acc * y + l_0 * (ap - sp);
      acc = acc * y + (ap - sp) * (ap - am) * active;
    }
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
