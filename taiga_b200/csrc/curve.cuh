// Pasta curve arithmetic (y^2 = x^3 + 5, a = 0) for sm_90a.  Accumulators are kept in extended Jacobian
// ("XYZZ": x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2) so that the hot mixed addition costs 8M+2S and needs no inversion
// (SURVEY.md App. E.2).  Affine points are 64 bytes (x||y, Montgomery limbs on device); identity = (0,0), the
// encoding `vesta::Affine` uses (EXT pasta_curves).  Replaces pasta_curves' group arithmetic as used by
// halo2_proofs `best_multiexp` / `Params::commit*` under taiga_halo2/src/proof.rs:33-40.
#pragma once
#include "field.cuh"

namespace tb {

template <class F>
struct alignas(16) Aff {
  F x, y;
  TB_HD bool is_inf() const { return x.is_zero() && y.is_zero(); }
  static TB_HD Aff inf() { Aff a; a.x = F::zero(); a.y = F::zero(); return a; }
  TB_HD Aff neg() const { Aff a; a.x = x; a.y = y.neg(); return a; }
  TB_HD Aff to_mont() const { Aff a; a.x = x.to_mont(); a.y = y.to_mont(); return a; }
  TB_HD Aff from_mont() const { Aff a; a.x = x.from_mont(); a.y = y.from_mont(); return a; }
};

template <class F>
struct alignas(16) Xyzz {
  F X, Y, ZZ, ZZZ;  // identity: ZZ == 0

  static TB_HD Xyzz inf() { Xyzz p; p.X = F::zero(); p.Y = F::zero(); p.ZZ = F::zero(); p.ZZZ = F::zero(); return p; }
  TB_HD bool is_inf() const { return ZZ.is_zero(); }
  static TB_HD Xyzz from_affine(const Aff<F>& a) {
    if (a.is_inf()) return inf();
    Xyzz p; p.X = a.x; p.Y = a.y; p.ZZ = F::one(); p.ZZZ = F::one(); return p;
  }
  // 2*(affine point): mdbl-2008-s-1
  static TB_HD Xyzz dbl_affine(const Aff<F>& a) {
    if (a.is_inf() || a.y.is_zero()) return inf();
    Xyzz r;
    F U = a.y.dbl(), V = U.sqr(), W = U * V, S = a.x * V;
    F x2 = a.x.sqr(), M = x2.dbl() + x2;
    r.X = M.sqr() - S.dbl();
    r.Y = M * (S - r.X) - W * a.y;
    r.ZZ = V; r.ZZZ = W;
    return r;
  }
  // dbl-2008-s-1
  TB_HD Xyzz dbl() const {
    if (is_inf() || Y.is_zero()) return inf();
    Xyzz r;
    F U = Y.dbl(), V, x2;
    F::mul2(U, U, X, X, V, x2);
    F W, S;
    F::mul2(U, V, X, V, W, S);
    F M = x2.dbl() + x2;
    r.X = M.sqr() - S.dbl();
    F t1, t2;
    F::mul2(M, S - r.X, W, Y, t1, t2);
    r.Y = t1 - t2;
    F::mul2(V, ZZ, W, ZZZ, r.ZZ, r.ZZZ);
    return r;
  }
  // this += affine (madd-2008-s), with all exceptional cases handled; the ten multiplies are issued as five
  // independent pairs (F::mul2)
  TB_HD void add_affine(const Aff<F>& b) {
    if (b.is_inf()) return;
    if (is_inf()) { *this = from_affine(b); return; }
    F U2, S2;
    F::mul2(b.x, ZZ, b.y, ZZZ, U2, S2);
    F Pp = U2 - X, R = S2 - Y;
    if (Pp.is_zero()) {
      if (R.is_zero()) *this = dbl_affine(b); else *this = inf();
      return;
    }
    F PP, RR;
    F::mul2(Pp, Pp, R, R, PP, RR);
    F PPP, Qq;
    F::mul2(Pp, PP, X, PP, PPP, Qq);
    F X3 = RR - PPP - Qq.dbl();
    F t1, t2;
    F::mul2(R, Qq - X3, Y, PPP, t1, t2);
    Y = t1 - t2;
    X = X3;
    F::mul2(ZZ, PP, ZZZ, PPP, ZZ, ZZZ);
  }
  // this += b (add-2008-s); fourteen multiplies as seven independent pairs
  TB_HD void add(const Xyzz& b) {
    if (b.is_inf()) return;
    if (is_inf()) { *this = b; return; }
    F U1, U2, S1, S2;
    F::mul2(X, b.ZZ, b.X, ZZ, U1, U2);
    F::mul2(Y, b.ZZZ, b.Y, ZZZ, S1, S2);
    F Pp = U2 - U1, R = S2 - S1;
    if (Pp.is_zero()) {
      if (R.is_zero()) *this = dbl(); else *this = inf();
      return;
    }
    F PP, RR;
    F::mul2(Pp, Pp, R, R, PP, RR);
    F PPP, Qq;
    F::mul2(Pp, PP, U1, PP, PPP, Qq);
    F X3 = RR - PPP - Qq.dbl();
    F t1, t2;
    F::mul2(R, Qq - X3, S1, PPP, t1, t2);
    Y = t1 - t2;
    X = X3;
    F z2, z3;
    F::mul2(ZZ, b.ZZ, ZZZ, b.ZZZ, z2, z3);
    F::mul2(z2, PP, z3, PPP, ZZ, ZZZ);
  }
  TB_HD Xyzz neg() const { Xyzz r = *this; r.Y = Y.neg(); return r; }
  // one field inversion
  TB_HD Aff<F> to_affine() const {
    if (is_inf()) return Aff<F>::inf();
    F iz3 = ZZZ.inv();            // 1/Z^3
    F izz = (ZZ * iz3).sqr();     // (Z^2/Z^3)^2 = 1/Z^2
    Aff<F> a; a.x = X * izz; a.y = Y * iz3; return a;
  }
};

// [k]P for a canonical (non-Montgomery) 256-bit scalar given as 8 LE limbs; 4-bit fixed windows.
template <class F>
TB_HD Xyzz<F> scalar_mul(const Aff<F>& p, const uint32_t* k) {
  Xyzz<F> tab[15];
  tab[0] = Xyzz<F>::from_affine(p);
  for (int i = 1; i < 15; ++i) { tab[i] = tab[i - 1]; tab[i].add_affine(p); }
  Xyzz<F> acc = Xyzz<F>::inf();
  for (int w = 63; w >= 0; --w) {
    acc = acc.dbl().dbl().dbl().dbl();
    uint32_t d = (k[w >> 3] >> ((w & 7) * 4)) & 15;
    if (d) acc.add(tab[d - 1]);
  }
  return acc;
}

}  // namespace tb
