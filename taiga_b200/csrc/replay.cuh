// The transcript replay of one proof for its final IPA check: one source that the host verifier and the device verifier
// (replay_kernel) of verifier.cu, and the CPU tests (plain g++), all compile.
//
// halo2_proofs plonk::verify_proof up to the IPA's final check (EXT; SURVEY.md App. A.2/A.4): the transcript over the
// proof's bytes, the gate, permutation and lookup constraints at x (gates.cuh, argument.cuh) for the expected h(x), the
// multiopen algebra, and the variable-base terms of the check.  The circuit comes as a ReplayShape: a flat view of its Shape
// (pointers and counts, no container), valid on whichever side its tables live.
#pragma once
#include "argument.cuh"
#include "gates.cuh"
#include "transcript.cuh"

namespace tb {

constexpr int RP_KINDS = 10;   // PolyKind (circuit.cuh): PK_INST .. PK_RANDOM
enum RpKind { RP_INST = 0, RP_ADV, RP_PZ, RP_LZ, RP_LPIN, RP_LPTAB, RP_FIXED, RP_SIG, RP_H, RP_RANDOM };

// a committed polynomial of the multiopen (Shape::uniq): its kind and index, its point set, and for a commitment read from
// the proof the index of its point among the proof's points (for h: the first piece)
struct RpUniq { int kind, idx, set, src; };
// one gate or lookup program: code at [off, off + len), `last` as GateProgram::last
struct RpProgram { int off, len, nregs, last; };

struct ReplayShape {
  int k, na, ni, L, nsets, P, bf, pieces, chunk;
  int nevals, nuniq, nps, npts, ngates, nrots, J, nypow, M;   // J constraints; nypow = J + permutation / lookup terms + 2
  uint32_t proof_len;
  Fp vk_repr, omega, omega_inv, n_inv, delta;   // vk_repr canonical, the rest Montgomery
  Fp delta_c0[PERM_MAX_SETS];
  int poly_base[RP_KINDS];       // (kind, idx) -> kind's base + idx, a dense number of every polynomial
  const int* rots;               // [nrots] every rotation the evaluations are read at
  const int* evpos;              // [poly][nrots] position of the evaluation in the proof (nevals for h at 0), -1 for none
  const RpUniq* uniq;            // [nuniq]
  const int* ps_off;             // [nps + 1] point set s holds the rotations ps_rot[ps_off[s] .. ps_off[s + 1])
  const int* ps_rot;
  const int* perm_kind;          // [P] RP_ADV / RP_FIXED / RP_INST of permutation column c
  const int* perm_idx;
  const RpProgram* progs;        // [ngates + 1] the gate programs, then the lookup program
  const QInstr* code;
  const Fp* consts;              // Montgomery
  // per-proof scratch, in field elements: its offsets and size
  int s_ev, s_regs, s_ypow, s_lka, s_lkt, s_qev, s_coef, s_cur, s_u, s_x4, s_ptsx, scratch;
};

// What one proof's replay reads besides the shape.  Points are Montgomery affine; the proof's points were decoded before
// (pts[i] / pts_ok[i]: its i-th point in transcript order).  inst: the proof's instance values, 32 canonical bytes each.
struct ReplayIn {
  const uint8_t* proof; size_t len;
  const Aff<Fq>* pts; const uint8_t* pts_ok;
  const uint8_t* inst; size_t inst_total;
  const Aff<Fq>* inst_comm;      // [ni]
  const Aff<Fq>* fixed; const Aff<Fq>* sigma;
  Aff<Fq> w, u;                  // the SRS's W and U
};
// What the final check needs: M variable-base terms (pts, sc), the k IPA challenges us and ab = (-c, -v), the coefficients
// of the g-term
struct ReplayOut { Aff<Fq>* pts; Fp* sc; Fp* us; Fp* ab; };

TB_HD int rp_eval_pos(const ReplayShape& S, int kind, int idx, int rot) {
  int r = 0;
  while (r + 1 < S.nrots && S.rots[r] != rot) ++r;   // present: the view's builder checks every lookup the replay makes
  return S.evpos[(S.poly_base[kind] + idx) * S.nrots + r];
}

// the transcript over one proof's bytes; `bad` once a read failed or the identity was absorbed
struct ProofReader : Transcript {
  const uint8_t* rd; size_t len, pos; const Aff<Fq>* pts; const uint8_t* pts_ok; int npts, ipt; bool bad;
  TB_HD void common_point(const Aff<Fq>& p) { if (!absorb_point(p.from_mont())) bad = true; }
  TB_HD bool read_point() {
    if (pos + 32 > len || ipt >= npts || !pts_ok[ipt]) { bad = true; return false; }
    pos += 32;
    if (!absorb_point(pts[ipt++].from_mont())) bad = true;
    return !bad;
  }
  TB_HD bool read_scalar(Fp& s) {
    if (pos + 32 > len || !canonical<Fp>(rd + pos, s)) { bad = true; return false; }
    pos += 32; absorb_scalar(s.from_mont()); return true;
  }
};

// the proof's evaluations as argument.cuh reads them
struct RpEvals {
  const ReplayShape& S; const Fp* ev;
  TB_HD Fp at(int kind, int idx, int rot) const { return ev[rp_eval_pos(S, kind, idx, rot)]; }
  TB_HD Fp perm_col(int c) const { return at(S.perm_kind[c], S.perm_idx[c], 0); }
  TB_HD Fp sigma(int c) const { return at(RP_SIG, c, 0); }
  TB_HD Fp z(int s) const { return at(RP_PZ, s, 0); }
  TB_HD Fp z_next(int s) const { return at(RP_PZ, s, 1); }
  TB_HD Fp z_last(int s) const { return at(RP_PZ, s, -(S.bf + 1)); }
};

TB_HD Fp rp_rot_pow(const ReplayShape& S, int rot) {
  Fp r = Fp::one();
  const Fp w = rot >= 0 ? S.omega : S.omega_inv;
  for (int i = 0; i < (rot >= 0 ? rot : -rot); ++i) r = r * w;
  return r;
}

// Replays one proof: true and its terms in `out` if the proof reaches its final check; false (the terms the identity times
// 0, us and ab 0) for a read past the end, a point that does not decode, the identity absorbed, a scalar or instance value
// >= p, or trailing bytes.  `scratch` holds S.scratch field elements.
TB_HD bool replay_proof(const ReplayShape& S, const ReplayIn& in, Fp* scratch, const ReplayOut& out) {
  const int kk = S.k, nps = S.nps;
  const Fp one = Fp::one();
  for (int i = 0; i < S.M; ++i) { out.pts[i] = Aff<Fq>::inf(); out.sc[i] = Fp::zero(); }
  for (int j = 0; j < kk; ++j) out.us[j] = Fp::zero();
  out.ab[0] = Fp::zero(); out.ab[1] = Fp::zero();
  for (size_t i = 0; i < in.inst_total; ++i) { Fp t; if (!canonical<Fp>(in.inst + 32 * i, t)) return false; }
  ProofReader tr;
  tr.start(S.vk_repr);
  tr.rd = in.proof; tr.len = in.len; tr.pos = 0; tr.pts = in.pts; tr.pts_ok = in.pts_ok; tr.npts = S.npts; tr.ipt = 0; tr.bad = false;
  for (int c = 0; c < S.ni; ++c) tr.common_point(in.inst_comm[c]);
  // the commitments: advice, the lookups' permuted input and table, the permutation and lookup products, the random
  // polynomial, h in its pieces (their points are in.pts[0 ..) in this order, as RpUniq::src names them)
  bool ok = true;
  for (int c = 0; c < S.na && ok; ++c) ok = tr.read_point();
  const Fp theta = tr.squeeze();
  for (int l = 0; l < 2 * S.L && ok; ++l) ok = tr.read_point();
  const Fp beta = tr.squeeze(), gamma = tr.squeeze();
  for (int s = 0; s < S.nsets && ok; ++s) ok = tr.read_point();
  for (int l = 0; l < S.L && ok; ++l) ok = tr.read_point();
  ok = ok && tr.read_point();
  const Fp y = tr.squeeze();
  for (int i = 0; i < S.pieces && ok; ++i) ok = tr.read_point();
  const Fp x = tr.squeeze();
  if (!ok) return false;
  // the evaluations in transcript order; ev[nevals] is set to the expected h(x) below
  Fp* ev = scratch + S.s_ev;
  for (int i = 0; i < S.nevals && ok; ++i) ok = tr.read_scalar(ev[i]);
  if (!ok) return false;
  const RpEvals view{S, ev};
  // expected h(x)
  Fp xn = x; for (int i = 0; i < kk; ++i) xn = xn.sqr();
  const Fp n_inv = S.n_inv;
  auto l_at = [&](int rot) { Fp wi = rp_rot_pow(S, rot); return (xn - one) * n_inv * wi * (x - wi).inv(); };
  const int last_rot = -(S.bf + 1);
  Fp l_last = l_at(last_rot), l_blind = Fp::zero(), l_0 = l_at(0);
  for (int r = -S.bf; r <= -1; ++r) l_blind = l_blind + l_at(r);
  // the circuit's programs at x: the gates as the quotient combines its parts (sum_p y^(J - 1 - last_p) S_p), and the lookups
  Fp* ypow = scratch + S.s_ypow;
  Fp* lk_a = scratch + S.s_lka; Fp* lk_t = scratch + S.s_lkt;
  ypow[0] = one;
  for (int i = 1; i < S.nypow; ++i) ypow[i] = ypow[i - 1] * y;
  auto at_x = [&](int kind, int col, int rot) { return view.at(kind == K_ADV ? RP_ADV : kind == K_FIX ? RP_FIXED : RP_INST, col, rot); };
  PointMachine<decltype(at_x)> m{at_x, S.consts, ypow, theta, lk_a, lk_t};
  m.regs = scratch + S.s_regs;
  const int J = S.J;
  Fp acc = Fp::zero();
  for (int g = 0; g < S.ngates; ++g) {
    const RpProgram& p = S.progs[g];
    acc = acc + ypow[J - 1 - p.last] * m.run(S.code + p.off, p.len, p.nregs);
  }
  { const RpProgram& p = S.progs[S.ngates]; m.run(S.code + p.off, p.len, p.nregs); }
  const ArgPoint at = {y, beta, gamma, l_0, l_last, one - (l_last + l_blind)};
  acc = perm_fold(acc, view, at, S.nsets, S.chunk, S.P, S.delta, S.delta_c0, x);
  for (int l = 0; l < S.L; ++l)
    acc = lookup_fold(acc, at, view.at(RP_LZ, l, 0), view.at(RP_LZ, l, 1), view.at(RP_LPIN, l, 0), view.at(RP_LPIN, l, -1), view.at(RP_LPTAB, l, 0),
                      lk_a[l], lk_t[l]);
  ev[S.nevals] = acc * (xn - one).inv();
  // ---- multiopen
  const Fp x1 = tr.squeeze(), x2 = tr.squeeze();
  Fp* q_evals = scratch + S.s_qev;   // [ps_off[nps]]: set s's evaluations at its points
  Fp* coef = scratch + S.s_coef;     // [nuniq] coefficient of each commitment inside its q_commitment (a power of x1)
  Fp* cur = scratch + S.s_cur;
  for (int i = 0; i < S.ps_off[nps]; ++i) q_evals[i] = Fp::zero();
  for (int s = 0; s < nps; ++s) cur[s] = one;
  // q_comm[s] = (...(C_first * x1 + C_2) * x1 + ...) : walk backwards so each commitment gets x1^(#later ones in its set)
  for (int c = S.nuniq - 1; c >= 0; --c) { const int s = S.uniq[c].set; coef[c] = cur[s]; cur[s] = cur[s] * x1; }
  for (int c = 0; c < S.nuniq; ++c) {
    const RpUniq& q = S.uniq[c];
    for (int i = S.ps_off[q.set]; i < S.ps_off[q.set + 1]; ++i) q_evals[i] = q_evals[i] * x1 + view.at(q.kind, q.idx, S.ps_rot[i]);
  }
  ok = tr.read_point();
  const int i_qprime = tr.ipt - 1;
  const Fp x3 = tr.squeeze();
  Fp* u = scratch + S.s_u;
  for (int s = 0; s < nps; ++s) ok = ok && tr.read_scalar(u[s]);
  if (!ok) return false;
  Fp msm_eval = Fp::zero();
  Fp* ptsx = scratch + S.s_ptsx;
  for (int s = 0; s < nps; ++s) {
    const int m0 = S.ps_off[s], np = S.ps_off[s + 1] - m0;
    for (int i = 0; i < np; ++i) ptsx[i] = x * rp_rot_pow(S, S.ps_rot[m0 + i]);
    Fp r_eval = Fp::zero();
    for (int i = 0; i < np; ++i) {
      Fp num = one, den = one;
      for (int j = 0; j < np; ++j) if (j != i) { num = num * (x3 - ptsx[j]); den = den * (ptsx[i] - ptsx[j]); }
      r_eval = r_eval + q_evals[m0 + i] * num * den.inv();
    }
    Fp e = u[s] - r_eval;
    for (int i = 0; i < np; ++i) e = e * (x3 - ptsx[i]).inv();
    msm_eval = msm_eval * x2 + e;
  }
  const Fp x4 = tr.squeeze();
  Fp* x4pow = scratch + S.s_x4;
  x4pow[0] = one; for (int i = 1; i <= nps; ++i) x4pow[i] = x4pow[i - 1] * x4;
  Fp v = msm_eval * x4pow[nps];
  for (int s = 0; s < nps; ++s) v = v + u[s] * x4pow[nps - 1 - s];
  // ---- IPA part of the transcript
  ok = tr.read_point();
  const int i_s = tr.ipt - 1;
  const Fp xi = tr.squeeze(), z = tr.squeeze();
  for (int j = 0; j < kk && ok; ++j) { ok = tr.read_point() && tr.read_point(); out.us[j] = tr.squeeze(); }
  Fp cc, ff; ok = ok && tr.read_scalar(cc) && tr.read_scalar(ff);
  if (!ok || tr.bad || tr.pos != in.len) { for (int j = 0; j < kk; ++j) out.us[j] = Fp::zero(); return false; }
  Fp b = one; { Fp c = x3; for (int j = kk - 1; j >= 0; --j) { b = b * (one + out.us[j] * c); c = c * c; } }
  // ---- variable-base terms: every committed polynomial (h in its pieces), q', S, the L_j and R_j, W and U
  int w = 0;
  auto push = [&](const Aff<Fq>& pt, const Fp& sc) { out.pts[w] = pt; out.sc[w] = sc; ++w; };
  for (int c = 0; c < S.nuniq; ++c) {
    const RpUniq& q = S.uniq[c];
    const Fp cf = coef[c] * x4pow[nps - 1 - q.set];
    if (q.kind == RP_H) { Fp t = cf; for (int i = 0; i < S.pieces; ++i) { push(in.pts[q.src + i], t); t = t * xn; } }
    else if (q.kind == RP_FIXED) push(in.fixed[q.idx], cf);
    else if (q.kind == RP_SIG) push(in.sigma[q.idx], cf);
    else if (q.kind == RP_INST) push(in.inst_comm[q.idx], cf);
    else push(in.pts[q.src], cf);
  }
  push(in.pts[i_qprime], x4pow[nps]);
  push(in.pts[i_s], xi);
  for (int j = 0; j < kk; ++j) { push(in.pts[i_s + 1 + 2 * j], out.us[j].inv()); push(in.pts[i_s + 2 + 2 * j], out.us[j]); }
  push(in.w, ff.neg());
  push(in.u, (cc * b * z).neg());
  out.ab[0] = cc.neg(); out.ab[1] = v.neg();
  return true;
}

}  // namespace tb
