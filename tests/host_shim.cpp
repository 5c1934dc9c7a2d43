// Host instantiation of the product's __host__ __device__ field/curve arithmetic, transcript, argument terms and gate
// programs (taiga_b200/csrc/*.cuh), so the same source the kernels compile can be checked on a CPU-only box against the oracle.
#include <cstdio>
#include <cstring>
#include "../taiga_b200/csrc/argument.cuh"
#include "../taiga_b200/csrc/gates.cuh"
#include "../taiga_b200/csrc/transcript.cuh"
using namespace tb;
template <class F> static void fop(int op, const uint8_t* a, const uint8_t* b, uint8_t* o) {
  F x, y, r; memcpy(&x, a, 32); memcpy(&y, b, 32);
  x = x.to_mont(); y = y.to_mont();
  switch (op) { case 0: r = x + y; break; case 1: r = x - y; break; case 2: r = x * y; break; case 3: r = x.inv(); break; case 4: r = x.neg(); break; default: r = x.sqr(); }
  r = r.from_mont(); memcpy(o, &r, 32);
}
template <class F> static Aff<F> ld(const uint8_t* p) { Aff<F> a; memcpy(&a, p, 64); a.x = a.x.to_mont(); a.y = a.y.to_mont(); return a; }
template <class F> static void st(const Aff<F>& a, uint8_t* p) { Aff<F> b; b.x = a.x.from_mont(); b.y = a.y.from_mont(); memcpy(p, &b, 64); }
template <class F> static void pop(int op, const uint8_t* a, const uint8_t* b, uint8_t* o) {
  Aff<F> pa = ld<F>(a); Xyzz<F> r;
  if (op == 0) { r = Xyzz<F>::from_affine(pa); r.add_affine(ld<F>(b)); }
  else if (op == 1) { uint32_t k[8]; memcpy(k, b, 32); r = scalar_mul(pa, k); }
  else if (op == 2) { r = Xyzz<F>::from_affine(pa).dbl(); }
  else if (op == 3) { r = Xyzz<F>::from_affine(pa).dbl(); Xyzz<F> s = Xyzz<F>::from_affine(ld<F>(b)).dbl(); s.add_affine(ld<F>(b)); r.add(s); }  // 2a + 3b
  else { r = Xyzz<F>::dbl_affine(pa); }
  st(r.to_affine(), o);
}
extern "C" {
void hs_field(int f, int op, const uint8_t* a, const uint8_t* b, uint8_t* o) { if (f == 0) fop<Fp>(op, a, b, o); else fop<Fq>(op, a, b, o); }
void hs_point(int c, int op, const uint8_t* a, const uint8_t* b, uint8_t* o) { if (c == 0) pop<Fq>(op, a, b, o); else pop<Fp>(op, a, b, o); }
// BLAKE2b-512 of data fed in nchunks pieces of the given lengths
void hs_blake2b(const char* personal16, const uint8_t* data, const int* chunks, int nchunks, uint8_t* out64) {
  Blake2b h; h.init(personal16);
  for (int i = 0; i < nchunks; ++i) { h.update(data, chunks[i]); data += chunks[i]; }
  uint64_t d[8]; h.finish(d); memcpy(out64, d, 64);
}
// transcript started from vk_repr, then ops[i] = 'P' (64 bytes x || y), 'S' (32 bytes) or 'Z' (a squeeze, 32 bytes out);
// values canonical.  Returns the index of a point the transcript refused, or -1.
int hs_transcript(const uint8_t* vk_repr, const char* ops, int nops, const uint8_t* in, uint8_t* out) {
  Transcript tr; Fp v; memcpy(v.l, vk_repr, 32); tr.start(v);
  for (int i = 0; i < nops; ++i) {
    if (ops[i] == 'P') { Aff<Fq> p; memcpy(&p, in, 64); in += 64; if (!tr.absorb_point(p)) return i; }
    else if (ops[i] == 'S') { memcpy(v.l, in, 32); in += 32; tr.absorb_scalar(v); }
    else { v = tr.squeeze().from_mont(); memcpy(out, v.l, 32); out += 32; }
  }
  return -1;
}
void hs_prf(const uint8_t* seed32, uint32_t proof, uint32_t tag, uint32_t idx, uint8_t* out) {
  uint32_t s[8]; memcpy(s, seed32, 32);
  Fp v = prf_scalar(s, proof, tag, idx).from_mont(); memcpy(out, v.l, 32);
}
void hs_compress(const uint8_t* xy, uint8_t* out) { Aff<Fq> p; memcpy(&p, xy, 64); uint32_t w[8]; compress_point(p, w); memcpy(out, w, 32); }
int hs_decompress(const uint8_t* b, uint8_t* xy) { Aff<Fq> p; if (!decompress_point(b, p)) return 0; memcpy(xy, &p, 64); return 1; }
// a scalar of the proof; on success out = the value back from Montgomery form
int hs_scalar(const uint8_t* b, uint8_t* out) { Fp v; if (!canonical<Fp>(b, v)) return 0; v = v.from_mont(); memcpy(out, v.l, 32); return 1; }
}

// ---------------------------------------------------------------- argument.cuh; every value canonical, 32 bytes
static Fp fe(const uint8_t* b) { Fp v; memcpy(v.l, b, 32); return v.to_mont(); }
static void put(const Fp& v, uint8_t* out) { Fp c = v.from_mont(); memcpy(out, c.l, 32); }
// permutation column c is vals[kind[c]][index[c]] (kinds advice, fixed, instance); zs is [set][X, wX, w^-(bf+1) X]
struct ShimView {
  const int* kind; const int* index; const uint8_t* vals[3]; const uint8_t* sig; const uint8_t* zs;
  Fp perm_col(int c) const { return fe(vals[kind[c]] + 32 * index[c]); }
  Fp sigma(int c) const { return fe(sig + 32 * c); }
  Fp z(int s) const { return fe(zs + 96 * s); }
  Fp z_next(int s) const { return fe(zs + 96 * s + 32); }
  Fp z_last(int s) const { return fe(zs + 96 * s + 64); }
};
extern "C" {
// out = [prod with sigma, prod with the identity] of set s, both products started at one
void hs_perm_set(const int* kind, const int* index, const uint8_t* adv, const uint8_t* fix, const uint8_t* inst, const uint8_t* sig, int s, int chunk, int ncols,
                 const uint8_t* beta, const uint8_t* gamma, const uint8_t* delta, const uint8_t* cd, uint8_t* out) {
  ShimView v = {kind, index, {adv, fix, inst}, sig, nullptr};
  Fp with_sigma = Fp::one(), with_id = Fp::one();
  perm_set_products(v, s, chunk, ncols, fe(beta), fe(gamma), fe(delta), fe(cd), with_sigma, with_id);
  put(with_sigma, out); put(with_id, out + 32);
}
// acc after the permutation terms and L lookups' terms; pt = acc, x, y, beta, gamma, l0, l_last, active;
// lk = [L][z, z_next, ap, ap_prev, sp, a, s]
void hs_arg_fold(const uint8_t* pt, const uint8_t* delta, const int* kind, const int* index, const uint8_t* adv, const uint8_t* fix, const uint8_t* inst,
                 const uint8_t* sig, const uint8_t* zs, int nsets, int chunk, int ncols, int L, const uint8_t* lk, uint8_t* out) {
  ShimView v = {kind, index, {adv, fix, inst}, sig, zs};
  Fp d = fe(delta), delta_c0[PERM_MAX_SETS];
  for (int s = 0; s < PERM_MAX_SETS; ++s) delta_c0[s] = d.pow_u64((uint64_t)s * chunk);
  const ArgPoint at = {fe(pt + 64), fe(pt + 96), fe(pt + 128), fe(pt + 160), fe(pt + 192), fe(pt + 224)};
  Fp acc = perm_fold(fe(pt), v, at, nsets, chunk, ncols, d, delta_c0, fe(pt + 32));
  for (int l = 0; l < L; ++l, lk += 224)
    acc = lookup_fold(acc, at, fe(lk), fe(lk + 32), fe(lk + 64), fe(lk + 96), fe(lk + 128), fe(lk + 160), fe(lk + 192));
  put(acc, out);
}
uint32_t hs_arg_terms(uint32_t nsets, uint32_t L) { return perm_lookup_terms(nsets, L); }
}

// ---------------------------------------------------------------- gates.cuh
static GatePlan g_plan;   // the plan of the last hs_gate_plan
extern "C" {
// checks cs and plans its programs for R sub-cosets: 1, or 0 with the rejection's message in err
int hs_gate_plan(const tb_cs_desc* cs, int R, int allow_split, char* err, int cap) {
  try { gate_desc_check(cs); g_plan = gate_plan(cs, R, allow_split != 0); return 1; }
  catch (const std::invalid_argument& e) { snprintf(err, cap, "%s", e.what()); return 0; }
}
int hs_gate_split() { return g_plan.split; }
uint32_t hs_gate_t_pl() { return g_plan.t_pl; }
static const std::vector<GateProgram>& programs(int which) { return which < 2 ? g_plan.gate_parts[which] : g_plan.gate_parts_lo[which - 2]; }
// list `which` (0, 1: gate_parts[big]; 2, 3: gate_parts_lo[big]; 4: the lookup program): with p < 0 the number of programs,
// else program p's instruction count, its code (4 words per instruction, up to cap instructions) and meta = [nregs, last]
int hs_gate_program(int which, int p, uint32_t* code, int cap, int* meta) {
  if (p < 0) return which == 4 ? 1 : (int)programs(which).size();
  const GateProgram& g = which == 4 ? g_plan.lookups : programs(which)[p];
  for (int i = 0; i < (int)g.code.size() && i < cap; ++i) memcpy(code + 4 * i, &g.code[i], 16);
  meta[0] = g.nregs; meta[1] = g.last;
  return (int)g.code.size();
}
// The planned programs at one point; adv / fix / inst hold one value per query of the description.  gate = sum_p
// y^(J - 1 - last_p) S_p over gate_parts[big] and gate_parts_lo[big]; lk = [L][compressed inputs, table].  Returns the
// number of leaves read that match no query.
int hs_gate_eval(const tb_cs_desc* cs, int big, const uint8_t* adv, const uint8_t* fix, const uint8_t* inst, const uint8_t* y, const uint8_t* theta,
                 uint8_t* gate, uint8_t* lk) {
  std::vector<Fp> consts;
  for (uint32_t i = 0; i < cs->num_constants; ++i) consts.push_back(fe(cs->constants + 32 * (size_t)i));
  int unmatched = 0;
  auto at = [&](int kind, int col, int rot) {
    const tb_query* q = kind == K_ADV ? cs->advice_queries : kind == K_FIX ? cs->fixed_queries : cs->instance_queries;
    const uint32_t nq = kind == K_ADV ? cs->num_advice_queries : kind == K_FIX ? cs->num_fixed_queries : cs->num_instance_queries;
    const uint8_t* v = kind == K_ADV ? adv : kind == K_FIX ? fix : inst;
    for (uint32_t i = 0; i < nq; ++i) if ((int)q[i].column == col && q[i].rotation == rot) return fe(v + 32 * (size_t)i);
    ++unmatched; return Fp::zero();
  };
  const int J = (int)cs->num_constraints;
  std::vector<Fp> ypow(J + g_plan.t_pl + 2, Fp::one()), a(cs->num_lookups), t(cs->num_lookups);
  for (size_t i = 1; i < ypow.size(); ++i) ypow[i] = ypow[i - 1] * fe(y);
  PointMachine<decltype(at)> m{at, consts.data(), ypow.data(), fe(theta), a.data(), t.data()};
  Fp acc = Fp::zero();
  for (const auto* parts : {&g_plan.gate_parts[big], &g_plan.gate_parts_lo[big]})
    for (const GateProgram& p : *parts) acc = acc + ypow[J - 1 - p.last] * m.run(p);
  m.run(g_plan.lookups);
  put(acc, gate);
  for (uint32_t l = 0; l < cs->num_lookups; ++l) { put(a[l], lk + 64 * l); put(t[l], lk + 64 * l + 32); }
  return unmatched;
}
void hs_constraint_degrees(const tb_cs_desc* cs, int* out) { std::vector<int> d = q_constraint_degrees(cs); for (size_t j = 0; j < d.size(); ++j) out[j] = d[j]; }
}
