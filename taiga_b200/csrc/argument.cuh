// The constraint terms of the permutation and lookup arguments: one source that the quotient and grand-product
// kernels (quotient_finish.cu), the host verifier (verifier.cu) and the CPU tests (tests/host_shim.cpp, plain g++) all
// compile.
//
// halo2_proofs plonk/permutation and plonk/lookup (EXT; SURVEY.md App. A.4).  After the gate constraints the quotient
// numerator folds, acc = acc * y + term, first the permutation terms (perm_fold), then five terms per lookup
// (lookup_fold).  The prover evaluates them on the extended cosets, the verifier at x from the proof's evaluations.
// Each caller passes a view that says where its values come from:
//   v.perm_col(c), v.sigma(c)         permutation column c and its sigma polynomial at X
//   v.z(s), v.z_next(s), v.z_last(s)  the grand product of set s at X, wX and w^-(bf+1) X  (perm_fold only)
#pragma once
#include "field.cuh"
// The templates below also take host-only views (the verifier's): nv_exec_check_disable keeps nvcc from warning about
// the device side of those instantiations, which is never generated.

namespace tb {

constexpr int PERM_MAX_SETS = 16;   // permutation sets of a circuit: sizes the per-set tables delta^(s * chunk)

// the values at X that the terms share; active = 1 - (l_last + l_blind)
struct ArgPoint { Fp y, beta, gamma, l0, l_last, active; };

// terms folded after the gate constraints: l0 (1 - z_0), l_last (z_last^2 - z_last), one link per pair of sets and one
// product per set, then five per lookup
TB_HD constexpr uint32_t perm_lookup_terms(uint32_t nsets, uint32_t L) { return (nsets ? 2 + (nsets - 1) + nsets : 0) + 5 * L; }

// Permutation set s, columns [s * chunk, min((s + 1) * chunk, ncols)):
//   with_sigma *= prod_c (v_c + beta sigma_c + gamma),  with_id *= prod_c (v_c + beta delta^c X + gamma)
// where cd = beta delta^(s * chunk) X (delta^c X is the identity permutation of column c).
#pragma nv_exec_check_disable
template <class V>
TB_HD void perm_set_products(const V& v, int s, int chunk, int ncols, const Fp& beta, const Fp& gamma, const Fp& delta, Fp cd, Fp& with_sigma, Fp& with_id) {
  const int c0 = s * chunk, c1 = c0 + chunk < ncols ? c0 + chunk : ncols;
  for (int c = c0; c < c1; ++c) {
    const Fp val = v.perm_col(c);
    with_sigma = with_sigma * (val + beta * v.sigma(c) + gamma);
    with_id = with_id * (val + cd + gamma);
    cd = cd * delta;
  }
}

// The permutation terms at X folded onto acc: l0 (1 - z_0(X)), l_last (z_{nsets-1}(X)^2 - z_{nsets-1}(X)),
// l0 (z_s(X) - z_{s-1}(w^-(bf+1) X)) for s >= 1, then per set active (z_s(wX) prod_sigma - z_s(X) prod_id).
// delta_c0[s] = delta^(s * chunk).
#pragma nv_exec_check_disable
template <class V>
TB_HD Fp perm_fold(Fp acc, const V& v, const ArgPoint& p, int nsets, int chunk, int ncols, const Fp& delta, const Fp* delta_c0, const Fp& x) {
  if (!nsets) return acc;
  acc = acc * p.y + p.l0 * (Fp::one() - v.z(0));
  { const Fp zl = v.z(nsets - 1); acc = acc * p.y + p.l_last * (zl * zl - zl); }
  for (int s = 1; s < nsets; ++s) acc = acc * p.y + p.l0 * (v.z(s) - v.z_last(s - 1));
  for (int s = 0; s < nsets; ++s) {
    Fp left = v.z_next(s), right = v.z(s);
    perm_set_products(v, s, chunk, ncols, p.beta, p.gamma, delta, p.beta * delta_c0[s] * x, left, right);
    acc = acc * p.y + (left - right) * p.active;
  }
  return acc;
}

// (a + beta)(s + gamma): the lookup grand product's factor of the compressed input and table (numerator) and of the
// permuted A', S' (denominator)
TB_HD Fp lookup_factor(const Fp& a, const Fp& s, const Fp& beta, const Fp& gamma) { return (a + beta) * (s + gamma); }

// The five terms of one lookup at X folded onto acc, given Z(X), Z(wX), A'(X), A'(w^-1 X), S'(X) and the compressed
// input a and table s at X
TB_HD Fp lookup_fold(Fp acc, const ArgPoint& p, const Fp& z, const Fp& z_next, const Fp& ap, const Fp& ap_prev, const Fp& sp, const Fp& a, const Fp& s) {
  acc = acc * p.y + p.l0 * (Fp::one() - z);
  acc = acc * p.y + p.l_last * (z * z - z);
  acc = acc * p.y + (z_next * lookup_factor(ap, sp, p.beta, p.gamma) - z * lookup_factor(a, s, p.beta, p.gamma)) * p.active;
  acc = acc * p.y + p.l0 * (ap - sp);
  acc = acc * p.y + (ap - sp) * (ap - ap_prev) * p.active;
  return acc;
}

}  // namespace tb
