// Pasta field arithmetic for sm_90a: 8x32-bit limbs, Montgomery form (R = 2^256), values always in [0, m).
// Memory format is 4x u64 little-endian = the same 32 bytes Rust's `Fp([u64;4])` holds, so a warp reading 32
// consecutive elements issues two fully coalesced 128-bit loads per thread (SURVEY.md App. E.1).
//
// The reduction exploits the Pasta moduli (SURVEY.md App. B.1 / E.1): m = 1 (mod 2^32) so the Montgomery quotient
// digit is simply -t0, limb 0 of m is 1, limbs 4..6 are 0 and limb 7 is 2^30, so each reduction row costs three
// real multiply-adds plus a shift.
//
// Replaces (on device) pasta_curves `Fp`/`Fq` as used by halo2_proofs under taiga_halo2/src/proof.rs:33-40.
#pragma once
#include <cstdint>
#include <stdexcept>
#include <string>

#ifdef __CUDACC__
#define TB_HD __host__ __device__ __forceinline__
#else
#define TB_HD inline
#endif
#define TB_REQUIRE(cond, msg) do { if (!(cond)) throw std::invalid_argument(std::string(msg) + " (" #cond ")"); } while (0)

namespace tb {

struct FpParams {  // Pallas base field = Vesta scalar field = circuit field
  static TB_HD constexpr uint32_t m(int i) {
    return i == 0 ? 0x00000001u : i == 1 ? 0x992d30edu : i == 2 ? 0x094cf91bu : i == 3 ? 0x224698fcu : i == 7 ? 0x40000000u : 0u;
  }
  static TB_HD constexpr bool m30(int i) { return i <= 4 || i == 8; }   // non-zero 30-bit limbs of the modulus
  // R mod p, R^2 mod p (SURVEY B.1)
  static TB_HD constexpr uint32_t r(int i) {
    return i == 0 ? 0xfffffffdu : i == 1 ? 0x34786d38u : i == 2 ? 0xe41914adu : i == 3 ? 0x992c350bu : i == 7 ? 0x3fffffffu : 0xffffffffu;
  }
  static TB_HD constexpr uint32_t r2(int i) {
    return i == 0 ? 0x0000000fu : i == 1 ? 0x8c78ecb3u : i == 2 ? 0x8b0de0e7u : i == 3 ? 0xd7d30dbdu : i == 4 ? 0xc3c95d18u : i == 5 ? 0x7797a99bu : i == 6 ? 0x7b9cb714u : 0x096d41afu;
  }
  // R^3 mod p (for the Montgomery inverse: (aR)^-1 * R^3 * R^-1 = a^-1 R)
  static TB_HD constexpr uint32_t r3(int i) {
    return i == 0 ? 0x3a9e10f9u : i == 1 ? 0xf185a599u : i == 2 ? 0x6ac5b1d1u : i == 3 ? 0xf6a68f3bu : i == 4 ? 0x353fd42cu : i == 5 ? 0xdf8d1014u : i == 6 ? 0x2d2d9910u : 0x2ae30922u;
  }
  static constexpr int id = 0;
};
struct FqParams {  // Vesta base field = Pallas scalar field
  static TB_HD constexpr uint32_t m(int i) {
    return i == 0 ? 0x00000001u : i == 1 ? 0x8c46eb21u : i == 2 ? 0x0994a8ddu : i == 3 ? 0x224698fcu : i == 7 ? 0x40000000u : 0u;
  }
  static TB_HD constexpr bool m30(int i) { return i <= 4 || i == 8; }
  static TB_HD constexpr uint32_t r(int i) {
    return i == 0 ? 0xfffffffdu : i == 1 ? 0x5b2b3e9cu : i == 2 ? 0xe3420567u : i == 3 ? 0x992c350bu : i == 7 ? 0x3fffffffu : 0xffffffffu;
  }
  static TB_HD constexpr uint32_t r2(int i) {
    return i == 0 ? 0x0000000fu : i == 1 ? 0xfc9678ffu : i == 2 ? 0x891a16e3u : i == 3 ? 0x67bb433du : i == 4 ? 0x04ccf590u : i == 5 ? 0x7fae2310u : i == 6 ? 0x7ccfdaa9u : 0x096d41afu;
  }
  static TB_HD constexpr uint32_t r3(int i) {
    return i == 0 ? 0x249dae4cu : i == 1 ? 0x008b421cu : i == 2 ? 0xdba41326u : i == 3 ? 0xe13bda50u : i == 4 ? 0x8e15cb63u : i == 5 ? 0x88fececbu : i == 6 ? 0x6e6792c8u : 0x07dd97a0u;
  }
  static constexpr int id = 1;
};


#ifndef TB_NOINLINE_MUL
#define TB_NOINLINE_MUL 1
#endif
#if defined(__CUDA_ARCH__) && !defined(TB_PORTABLE_FIELD)
#define TB_PTX_FIELD 1
// Montgomery product on the FMA pipe.  The GPU issues IMAD on the fma pipe and IADD3 on the alu pipe, each at one warp
// instruction per two cycles per sub-partition; a product whose carries are resolved with add-with-carry chains is
// alu-bound at ~2x its IMAD count.  Here the running sum T is kept as two
// interleaved accumulators, T = X + Y * 2^32: the products a[2k] * bi land on the 64-bit slots of X and a[2k+1] * bi on
// those of Y, so `mad.lo.cc / madc.hi.cc` pairs fuse into IMAD.WIDE.U32(.X) with the carry travelling in a predicate
// -- no alu instruction per product.  Dividing by 2^32 after a reduction row swaps the roles: X' = Y, Y' = X >> 64, and
// the odd limb X[1] is added at the bottom of X'.  (Restated from the published even/odd CIOS technique used by GPU
// big-number libraries; verified against big-integer arithmetic in scratch simulation and tests/test_host_arith.py +
// the GPU field tests.)  Each asm block is self-contained with respect to the carry flag.
//
// first row: X = a_even * b0, Y = a_odd * b0
__device__ __forceinline__ void tb_eo_first(uint32_t* X, uint32_t* Y, const uint32_t* a, uint32_t bi) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    uint64_t p = (uint64_t)a[2 * k] * bi, q = (uint64_t)a[2 * k + 1] * bi;
    X[2 * k] = (uint32_t)p; X[2 * k + 1] = (uint32_t)(p >> 32);
    Y[2 * k] = (uint32_t)q; Y[2 * k + 1] = (uint32_t)(q >> 32);
  }
}
// row i > 0.  In: X (old even accumulator, X[0] == 0 after its reduction), Y (old odd).  Out: X' = Y + X[1] + a_even * bi
// (returned in Y's registers), Y' = (X >> 64) + a_odd * bi (+ carries) returned in N.
__device__ __forceinline__ void tb_eo_row(uint32_t* Y /* in: old Y, out: new X */, uint32_t* N /* out: new Y */, const uint32_t* X /* old X */,
                                          const uint32_t* a, uint32_t bi) {
  asm("add.cc.u32 %0, %0, %9;\n\t"
      "madc.lo.cc.u32 %1, %16, %20, %10;\n\t"
      "madc.hi.cc.u32 %2, %16, %20, %11;\n\t"
      "madc.lo.cc.u32 %3, %17, %20, %12;\n\t"
      "madc.hi.cc.u32 %4, %17, %20, %13;\n\t"
      "madc.lo.cc.u32 %5, %18, %20, %14;\n\t"
      "madc.hi.cc.u32 %6, %18, %20, %15;\n\t"
      "madc.lo.cc.u32 %7, %19, %20, 0;\n\t"
      "madc.hi.u32 %8, %19, %20, 0;"
      : "+r"(Y[0]), "=&r"(N[0]), "=&r"(N[1]), "=&r"(N[2]), "=&r"(N[3]), "=&r"(N[4]), "=&r"(N[5]), "=&r"(N[6]), "=&r"(N[7])
      : "r"(X[1]), "r"(X[2]), "r"(X[3]), "r"(X[4]), "r"(X[5]), "r"(X[6]), "r"(X[7]), "r"(a[1]), "r"(a[3]), "r"(a[5]), "r"(a[7]), "r"(bi));
  asm("mad.lo.cc.u32 %0, %9, %13, %0;\n\t"
      "madc.hi.cc.u32 %1, %9, %13, %1;\n\t"
      "madc.lo.cc.u32 %2, %10, %13, %2;\n\t"
      "madc.hi.cc.u32 %3, %10, %13, %3;\n\t"
      "madc.lo.cc.u32 %4, %11, %13, %4;\n\t"
      "madc.hi.cc.u32 %5, %11, %13, %5;\n\t"
      "madc.lo.cc.u32 %6, %12, %13, %6;\n\t"
      "madc.hi.cc.u32 %7, %12, %13, %7;\n\t"
      "addc.u32 %8, %8, 0;"
      : "+r"(Y[0]), "+r"(Y[1]), "+r"(Y[2]), "+r"(Y[3]), "+r"(Y[4]), "+r"(Y[5]), "+r"(Y[6]), "+r"(Y[7]), "+r"(N[7])
      : "r"(a[0]), "r"(a[2]), "r"(a[4]), "r"(a[6]), "r"(bi));
}
// Pasta reduction row: mi = -X[0] (since -m^-1 = -1 mod 2^32); T += mi * m with m = 1 + m1 2^32 + m2 2^64 + m3 2^96 + m7 2^224.
// Odd limbs (m1, m3, 0, m7) go to Y, even limbs (1, m2, 0, 0) to X; afterwards X[0] == 0.
__device__ __forceinline__ void tb_eo_red(uint32_t* X, uint32_t* Y, uint32_t m1, uint32_t m2, uint32_t m3, uint32_t m7) {
  const uint32_t mi = 0u - X[0];
  asm("mad.lo.cc.u32 %0, %8, %9, %0;\n\t"
      "madc.hi.cc.u32 %1, %8, %9, %1;\n\t"
      "madc.lo.cc.u32 %2, %8, %10, %2;\n\t"
      "madc.hi.cc.u32 %3, %8, %10, %3;\n\t"
      "addc.cc.u32 %4, %4, 0;\n\t"
      "addc.cc.u32 %5, %5, 0;\n\t"
      "madc.lo.cc.u32 %6, %8, %11, %6;\n\t"
      "madc.hi.u32 %7, %8, %11, %7;"
      : "+r"(Y[0]), "+r"(Y[1]), "+r"(Y[2]), "+r"(Y[3]), "+r"(Y[4]), "+r"(Y[5]), "+r"(Y[6]), "+r"(Y[7])
      : "r"(mi), "r"(m1), "r"(m3), "r"(m7));
  asm("add.cc.u32 %0, %0, %9;\n\t"
      "addc.cc.u32 %1, %1, 0;\n\t"
      "madc.lo.cc.u32 %2, %9, %10, %2;\n\t"
      "madc.hi.cc.u32 %3, %9, %10, %3;\n\t"
      "addc.cc.u32 %4, %4, 0;\n\t"
      "addc.cc.u32 %5, %5, 0;\n\t"
      "addc.cc.u32 %6, %6, 0;\n\t"
      "addc.cc.u32 %7, %7, 0;\n\t"
      "addc.u32 %8, %8, 0;"
      : "+r"(X[0]), "+r"(X[1]), "+r"(X[2]), "+r"(X[3]), "+r"(X[4]), "+r"(X[5]), "+r"(X[6]), "+r"(X[7]), "+r"(Y[7])
      : "r"(mi), "r"(m2));
}
// result = Y + (X >> 32)   (< 2m)
__device__ __forceinline__ void tb_eo_merge(uint32_t* r, const uint32_t* X, const uint32_t* Y) {
  asm("add.cc.u32 %0, %8, %16;\n\t"
      "addc.cc.u32 %1, %9, %17;\n\t"
      "addc.cc.u32 %2, %10, %18;\n\t"
      "addc.cc.u32 %3, %11, %19;\n\t"
      "addc.cc.u32 %4, %12, %20;\n\t"
      "addc.cc.u32 %5, %13, %21;\n\t"
      "addc.cc.u32 %6, %14, %22;\n\t"
      "addc.u32 %7, %15, 0;"
      : "=&r"(r[0]), "=&r"(r[1]), "=&r"(r[2]), "=&r"(r[3]), "=&r"(r[4]), "=&r"(r[5]), "=&r"(r[6]), "=&r"(r[7])
      : "r"(Y[0]), "r"(Y[1]), "r"(Y[2]), "r"(Y[3]), "r"(Y[4]), "r"(Y[5]), "r"(Y[6]), "r"(Y[7]),
        "r"(X[1]), "r"(X[2]), "r"(X[3]), "r"(X[4]), "r"(X[5]), "r"(X[6]), "r"(X[7]));
}
#endif

template <class P>
struct alignas(16) Fe {
  uint32_t l[8];

  static TB_HD constexpr int params_id() { return P::id; }
  static TB_HD constexpr uint32_t modulus_limb(int i) { return P::m(i); }
  static TB_HD Fe zero() { Fe z;
#pragma unroll
    for (int i = 0; i < 8; ++i) z.l[i] = 0; return z; }
  static TB_HD Fe one() { Fe o;
#pragma unroll
    for (int i = 0; i < 8; ++i) o.l[i] = P::r(i); return o; }
  static TB_HD Fe r2() { Fe o;
#pragma unroll
    for (int i = 0; i < 8; ++i) o.l[i] = P::r2(i); return o; }
  static TB_HD Fe raw_one() { Fe o = zero(); o.l[0] = 1; return o; }

  TB_HD bool is_zero() const { uint32_t a = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) a |= l[i]; return a == 0; }
  TB_HD bool operator==(const Fe& o) const { uint32_t a = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) a |= l[i] ^ o.l[i]; return a == 0; }
  TB_HD bool operator!=(const Fe& o) const { return !(*this == o); }

  // r = a - m if a >= m (a < 2m)
  static TB_HD void cond_sub(uint32_t* a) {
#ifdef TB_PTX_FIELD
    uint32_t t[8], br;
    asm("sub.cc.u32 %0, %9, %17;\n\t"
        "subc.cc.u32 %1, %10, %18;\n\t"
        "subc.cc.u32 %2, %11, %19;\n\t"
        "subc.cc.u32 %3, %12, %20;\n\t"
        "subc.cc.u32 %4, %13, 0;\n\t"
        "subc.cc.u32 %5, %14, 0;\n\t"
        "subc.cc.u32 %6, %15, 0;\n\t"
        "subc.cc.u32 %7, %16, %21;\n\t"
        "subc.u32 %8, 0, 0;"
        : "=r"(t[0]), "=r"(t[1]), "=r"(t[2]), "=r"(t[3]), "=r"(t[4]), "=r"(t[5]), "=r"(t[6]), "=r"(t[7]), "=r"(br)
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]), "r"(P::m(0)), "r"(P::m(1)), "r"(P::m(2)), "r"(P::m(3)), "r"(P::m(7)));
#pragma unroll
    for (int i = 0; i < 8; ++i) a[i] = br ? a[i] : t[i];
    return;
#else
    uint32_t t[8]; uint64_t br = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { uint64_t d = (uint64_t)a[i] - P::m(i) - br; t[i] = (uint32_t)d; br = (d >> 32) & 1; }
    if (!br) {
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = t[i];
    }
#endif
  }
  friend TB_HD Fe operator+(const Fe& a, const Fe& b) {
#ifdef TB_PTX_FIELD
    Fe r;
    asm("add.cc.u32 %0, %8, %16;\n\t"
        "addc.cc.u32 %1, %9, %17;\n\t"
        "addc.cc.u32 %2, %10, %18;\n\t"
        "addc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\t"
        "addc.cc.u32 %5, %13, %21;\n\t"
        "addc.cc.u32 %6, %14, %22;\n\t"
        "addc.u32 %7, %15, %23;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7])
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
          "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
    cond_sub(r.l);
    return r;
#else
    Fe r; uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { c += (uint64_t)a.l[i] + b.l[i]; r.l[i] = (uint32_t)c; c >>= 32; }
    cond_sub(r.l);  // a+b < 2m < 2^256: no carry out
    return r;
#endif
  }
  friend TB_HD Fe operator-(const Fe& a, const Fe& b) {
#ifdef TB_PTX_FIELD
    Fe r; uint32_t br;
    asm("sub.cc.u32 %0, %9, %17;\n\t"
        "subc.cc.u32 %1, %10, %18;\n\t"
        "subc.cc.u32 %2, %11, %19;\n\t"
        "subc.cc.u32 %3, %12, %20;\n\t"
        "subc.cc.u32 %4, %13, %21;\n\t"
        "subc.cc.u32 %5, %14, %22;\n\t"
        "subc.cc.u32 %6, %15, %23;\n\t"
        "subc.cc.u32 %7, %16, %24;\n\t"
        "subc.u32 %8, 0, 0;"
        : "=r"(r.l[0]), "=r"(r.l[1]), "=r"(r.l[2]), "=r"(r.l[3]), "=r"(r.l[4]), "=r"(r.l[5]), "=r"(r.l[6]), "=r"(r.l[7]), "=r"(br)
        : "r"(a.l[0]), "r"(a.l[1]), "r"(a.l[2]), "r"(a.l[3]), "r"(a.l[4]), "r"(a.l[5]), "r"(a.l[6]), "r"(a.l[7]),
          "r"(b.l[0]), "r"(b.l[1]), "r"(b.l[2]), "r"(b.l[3]), "r"(b.l[4]), "r"(b.l[5]), "r"(b.l[6]), "r"(b.l[7]));
    // br = 0xffffffff on borrow: add m back
    asm("add.cc.u32 %0, %0, %8;\n\t"
        "addc.cc.u32 %1, %1, %9;\n\t"
        "addc.cc.u32 %2, %2, %10;\n\t"
        "addc.cc.u32 %3, %3, %11;\n\t"
        "addc.cc.u32 %4, %4, 0;\n\t"
        "addc.cc.u32 %5, %5, 0;\n\t"
        "addc.cc.u32 %6, %6, 0;\n\t"
        "addc.u32 %7, %7, %12;"
        : "+r"(r.l[0]), "+r"(r.l[1]), "+r"(r.l[2]), "+r"(r.l[3]), "+r"(r.l[4]), "+r"(r.l[5]), "+r"(r.l[6]), "+r"(r.l[7])
        : "r"(br & P::m(0)), "r"(br & P::m(1)), "r"(br & P::m(2)), "r"(br & P::m(3)), "r"(br & P::m(7)));
    return r;
#else
    Fe r; uint64_t br = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { uint64_t d = (uint64_t)a.l[i] - b.l[i] - br; r.l[i] = (uint32_t)d; br = (d >> 32) & 1; }
    uint32_t mask = (uint32_t)0 - (uint32_t)br; uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) { c += (uint64_t)r.l[i] + (P::m(i) & mask); r.l[i] = (uint32_t)c; c >>= 32; }
    return r;
#endif
  }
  TB_HD Fe neg() const { return zero() - *this; }
  TB_HD Fe dbl() const { return *this + *this; }

  // Montgomery product a*b*R^-1 mod m (CIOS, 32-bit limbs, Pasta-specific reduction row)
#ifdef TB_PTX_FIELD
  // Out-of-line Montgomery product.  The EC formulas call the multiply 10-14 times each; fully inlined they are
  // ~100 KB of SASS per kernel and ncu showed `no_instruction` (instruction-cache miss) as the top stall of the MSM
  // kernels.  As a real function (operands and result travel in registers) the hot kernels fit the 32 KB L1.5 I-cache.
  static __device__ __noinline__ Fe mul_call(Fe a, Fe b) { return mul_body(a, b); }
  // Two independent products per call: the two carry chains interleave, doubling the instruction-level parallelism of
  // the (latency-bound) EC formulas, whose multiplies come in independent pairs.
  struct Pair { Fe a, b; };
  static __device__ __noinline__ Pair mul2_call(Fe a, Fe b, Fe c, Fe d) {
    static_assert(P::m(0) == 1 && P::m(4) == 0 && P::m(5) == 0 && P::m(6) == 0, "Pasta-shaped modulus expected");
    uint32_t X[8], Y[8], U[8], V[8];
    tb_eo_first(X, Y, a.l, b.l[0]);
    tb_eo_first(U, V, c.l, d.l[0]);
    tb_eo_red(X, Y, P::m(1), P::m(2), P::m(3), P::m(7));
    tb_eo_red(U, V, P::m(1), P::m(2), P::m(3), P::m(7));
#pragma unroll
    for (int i = 1; i < 8; ++i) {
      uint32_t N[8], W[8];
      tb_eo_row(Y, N, X, a.l, b.l[i]);
      tb_eo_row(V, W, U, c.l, d.l[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) { X[j] = Y[j]; Y[j] = N[j]; U[j] = V[j]; V[j] = W[j]; }
      tb_eo_red(X, Y, P::m(1), P::m(2), P::m(3), P::m(7));
      tb_eo_red(U, V, P::m(1), P::m(2), P::m(3), P::m(7));
    }
    Pair r;
    tb_eo_merge(r.a.l, X, Y);
    tb_eo_merge(r.b.l, U, V);
    cond_sub(r.a.l); cond_sub(r.b.l);
    return r;
  }
#endif
  // (x*y, z*w)
  static TB_HD void mul2(const Fe& x, const Fe& y, const Fe& z, const Fe& w, Fe& r1, Fe& r2) {
#if defined(TB_PTX_FIELD) && TB_NOINLINE_MUL
    Pair p = mul2_call(x, y, z, w); r1 = p.a; r2 = p.b;
#else
    r1 = x * y; r2 = z * w;
#endif
  }
  friend TB_HD Fe operator*(const Fe& a, const Fe& b) {
#if defined(TB_PTX_FIELD) && TB_NOINLINE_MUL
    return mul_call(a, b);
#else
    return mul_body(a, b);
#endif
  }
  static TB_HD Fe mul_body(const Fe& a, const Fe& b) {
#ifdef TB_PTX_FIELD
    // requires a < m (any 256-bit b): invariant T < 2m after every row
    static_assert(P::m(0) == 1 && P::m(4) == 0 && P::m(5) == 0 && P::m(6) == 0, "Pasta-shaped modulus expected");
    uint32_t X[8], Y[8];
    tb_eo_first(X, Y, a.l, b.l[0]);
    tb_eo_red(X, Y, P::m(1), P::m(2), P::m(3), P::m(7));
#pragma unroll
    for (int i = 1; i < 8; ++i) {
      uint32_t N[8];
      tb_eo_row(Y, N, X, a.l, b.l[i]);
#pragma unroll
      for (int j = 0; j < 8; ++j) { X[j] = Y[j]; Y[j] = N[j]; }
      tb_eo_red(X, Y, P::m(1), P::m(2), P::m(3), P::m(7));
    }
    Fe r;
    tb_eo_merge(r.l, X, Y);
    cond_sub(r.l);
    return r;
#else
    uint32_t t[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) t[i] = 0;
    uint32_t t8 = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      uint64_t c = 0;
      const uint32_t bi = b.l[i];
#pragma unroll
      for (int j = 0; j < 8; ++j) { c += (uint64_t)a.l[j] * bi + t[j]; t[j] = (uint32_t)c; c >>= 32; }
      c += t8; t8 = (uint32_t)c; uint32_t t9 = (uint32_t)(c >> 32);
      // reduction row: q = -t0 (since -m^-1 = -1 mod 2^32); t = (t + q*m) >> 32
      const uint32_t q = 0u - t[0];
      c = (t[0] != 0) ? 1 : 0;  // (t0 + q*1) >> 32
      c += (uint64_t)q * P::m(1) + t[1]; t[0] = (uint32_t)c; c >>= 32;
      c += (uint64_t)q * P::m(2) + t[2]; t[1] = (uint32_t)c; c >>= 32;
      c += (uint64_t)q * P::m(3) + t[3]; t[2] = (uint32_t)c; c >>= 32;
      c += t[4]; t[3] = (uint32_t)c; c >>= 32;
      c += t[5]; t[4] = (uint32_t)c; c >>= 32;
      c += t[6]; t[5] = (uint32_t)c; c >>= 32;
      c += ((uint64_t)q << 30) + t[7]; t[6] = (uint32_t)c; c >>= 32;  // q * 2^30 at limb 7
      c += t8; t[7] = (uint32_t)c; t8 = t9 + (uint32_t)(c >> 32);
    }
    Fe r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.l[i] = t[i];
    cond_sub(r.l);  // result < 2m, t8 == 0
    return r;
#endif
  }
  TB_HD Fe sqr() const { return (*this) * (*this); }

  TB_HD Fe to_mont() const { return (*this) * r2(); }        // canonical -> Montgomery
  TB_HD Fe from_mont() const { return (*this) * raw_one(); }  // Montgomery -> canonical

  static TB_HD Fe from_u32(uint32_t v) { Fe a = zero(); a.l[0] = v; return a.to_mont(); }

  // exponent as 8 LE 32-bit limbs
  TB_HD Fe pow(const uint32_t* e, int nlimbs) const {
    Fe acc = one();
    for (int i = nlimbs - 1; i >= 0; --i)
      for (int b = 31; b >= 0; --b) { acc = acc.sqr(); if ((e[i] >> b) & 1) acc = acc * (*this); }
    return acc;
  }
  TB_HD Fe pow_u64(uint64_t e) const { uint32_t w[2] = {(uint32_t)e, (uint32_t)(e >> 32)}; return pow(w, 2); }
  // Inversion (0 -> 0) by Bernstein-Yang "divsteps" in batches of 30 (the safegcd recurrence as used by variable-time modular
  // inversion libraries): the low 30 bits of (f, g) decide 30 division steps and their 2x2 transition matrix, which is then
  // applied to the full 9 x 30-bit signed limbs of (f, g) and, modulo p, to the Bezout coefficients (d, e).  ~18 batches of
  // ~300 instructions replace the ~700 shift/subtract steps (~20k instructions, branchy) of the binary extended Euclid that
  // stood here: the single-thread latency of every normalisation to affine and of the batched-inversion root drops ~4x.
  // The Pasta moduli are 1 mod 2^32, so the "make divisible by 2^30" correction needs no multiplication by p^-1.
  // Checked on the host against big-integer arithmetic (tests/test_host_arith.py) and by every GPU parity test.
  static TB_HD int ctz32(uint32_t x) {
#ifdef __CUDA_ARCH__
    return __clz(__brev(x));
#else
    return __builtin_ctz(x);
#endif
  }
  TB_HD Fe inv() const {
    if (is_zero()) return zero();
    constexpr int32_t M30 = (int32_t)((1u << 30) - 1);
    int32_t f[9], g[9], d[9], e[9], p[9];
    {  // p and x (the stored limbs as an integer; for a Montgomery value x = aR) in 30-bit limbs
      uint32_t pm[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) pm[i] = P::m(i);
      split30(pm, p); split30(l, g);
#pragma unroll
      for (int i = 0; i < 9; ++i) { f[i] = p[i]; d[i] = 0; e[i] = 0; }
      e[0] = 1;
    }
    int32_t eta = -1;
    for (int it = 0; it < 26; ++it) {   // 590 divsteps bound the 256-bit case: 20 batches; the loop leaves as soon as g == 0
      // ---- 30 divsteps on the low words
      int32_t u = 1, v = 0, q = 0, r = 1;
      { uint32_t fl = (uint32_t)f[0] | ((uint32_t)f[1] << 30), gl = (uint32_t)g[0] | ((uint32_t)g[1] << 30);
        int i = 30;
        for (;;) {
          int zeros = ctz32(gl | (0xffffffffu << i));
          gl >>= zeros; u = (int32_t)((uint32_t)u << zeros); v = (int32_t)((uint32_t)v << zeros); eta -= zeros; i -= zeros;
          if (i == 0) break;
          if (eta < 0) {
            eta = -eta;
            uint32_t tf = fl; fl = gl; gl = 0u - tf;
            int32_t tu = u; u = q; q = -tu;
            int32_t tv = v; v = r; r = -tv;
          }
          const int limit = (eta + 1) > i ? i : (eta + 1);
          const uint32_t m = (0xffffffffu >> (32 - (limit > 6 ? 6 : limit)));
          const uint32_t w = (fl * gl * (fl * fl - 2u)) & m;   // -g / f mod 2^min(limit, 6)
          gl += fl * w; q += u * (int32_t)w; r += v * (int32_t)w;
        } }
      // ---- (d, e) <- (u d + v e, q d + r e) / 2^30  (mod p)
      { const int32_t sd = d[8] >> 31, se = e[8] >> 31;
        int32_t md = (u & sd) + (v & se), me = (q & sd) + (r & se);
        int64_t cd = (int64_t)u * d[0] + (int64_t)v * e[0], ce = (int64_t)q * d[0] + (int64_t)r * e[0];
        md -= ((int32_t)(uint32_t)cd + md) & M30;   // p^-1 = 1 (mod 2^30)
        me -= ((int32_t)(uint32_t)ce + me) & M30;
        cd += (int64_t)p[0] * md; ce += (int64_t)p[0] * me;
        cd >>= 30; ce >>= 30;
#pragma unroll
        for (int i = 1; i < 9; ++i) {
          cd += (int64_t)u * d[i] + (int64_t)v * e[i]; ce += (int64_t)q * d[i] + (int64_t)r * e[i];
          if (P::m30(i)) { cd += (int64_t)p[i] * md; ce += (int64_t)p[i] * me; }
          d[i - 1] = (int32_t)cd & M30; cd >>= 30;
          e[i - 1] = (int32_t)ce & M30; ce >>= 30;
        }
        d[8] = (int32_t)cd; e[8] = (int32_t)ce; }
      // ---- (f, g) <- (u f + v g, q f + r g) / 2^30
      { int64_t cf = (int64_t)u * f[0] + (int64_t)v * g[0], cg = (int64_t)q * f[0] + (int64_t)r * g[0];
        cf >>= 30; cg >>= 30;
        int32_t nz = 0;
#pragma unroll
        for (int i = 1; i < 9; ++i) {
          cf += (int64_t)u * f[i] + (int64_t)v * g[i]; cg += (int64_t)q * f[i] + (int64_t)r * g[i];
          f[i - 1] = (int32_t)cf & M30; cf >>= 30;
          g[i - 1] = (int32_t)cg & M30; cg >>= 30;
          nz |= g[i - 1];
        }
        f[8] = (int32_t)cf; g[8] = (int32_t)cg;
        if ((nz | g[8]) == 0) break; }
    }
    // f = +-1, d * x = f (mod p), d in (-2p, p): fix the sign, bring into [0, p)
    if (f[8] < 0) {
#pragma unroll
      for (int i = 0; i < 9; ++i) d[i] = -d[i];
    }
#pragma unroll
    for (int rep = 0; rep < 3; ++rep) {   // carry-normalise (first round), then add p while negative (at most twice)
      const int32_t add = (rep > 0 && d[8] < 0) ? -1 : 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) { d[i] += p[i] & add; d[i + 1] += d[i] >> 30; d[i] &= M30; }
      d[8] += p[8] & add;
    }
    Fe y; join30(d, y.l);
    cond_sub(y.l); cond_sub(y.l);
    Fe r3c;
#pragma unroll
    for (int i = 0; i < 8; ++i) r3c.l[i] = P::r3(i);
    return y * r3c;   // x^-1 * R^3 * R^-1: Montgomery form of a^-1 when x = aR
  }
  // 8 x 32-bit <-> 9 x 30-bit limbs (non-negative values)
  static TB_HD void split30(const uint32_t* a, int32_t* o) {
#pragma unroll
    for (int i = 0; i < 9; ++i) {
      const int bit = 30 * i, w = bit >> 5, sh = bit & 31;
      uint64_t v = a[w];
      if (w + 1 < 8) v |= (uint64_t)a[w + 1] << 32;
      o[i] = (int32_t)((uint32_t)(v >> sh) & ((1u << 30) - 1));
    }
  }
  static TB_HD void join30(const int32_t* a, uint32_t* o) {   // limbs 0..7 in [0, 2^30), limb 8 small and non-negative
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int bit = 32 * j, i = bit / 30, sh = bit - 30 * i;   // out word j = bits [32j, 32j + 32): limbs i, i+1 (and i+2 when sh > 28)
      uint64_t v = (uint64_t)(uint32_t)a[i] >> sh;
      v |= (uint64_t)(uint32_t)a[i + 1] << (30 - sh);
      if (i + 2 < 9) v |= (uint64_t)(uint32_t)a[i + 2] << (60 - sh);
      o[j] = (uint32_t)v;
    }
  }
  // canonical-integer comparison of two canonical (non-Montgomery) values
  static TB_HD int cmp_raw(const Fe& a, const Fe& b) {
    for (int i = 7; i >= 0; --i) { if (a.l[i] < b.l[i]) return -1; if (a.l[i] > b.l[i]) return 1; }
    return 0;
  }
};

typedef Fe<FpParams> Fp;
typedef Fe<FqParams> Fq;

// 2^32-th roots of unity (pasta_curves ROOT_OF_UNITY; SURVEY B.1), canonical 32-bit LE limbs
template <class F> TB_HD F root_of_unity_2_32();
template <> TB_HD Fp root_of_unity_2_32<Fp>() {
  Fp r; const uint32_t v[8] = {0xd87ea32fu, 0xbdad6fabu, 0xb7bb7584u, 0xea322bf2u, 0x0561f81au, 0x36212083u, 0xac30ebdau, 0x2bce74deu};
  for (int i = 0; i < 8; ++i) r.l[i] = v[i]; return r.to_mont();
}
template <> TB_HD Fq root_of_unity_2_32<Fq>() {
  Fq r; const uint32_t v[8] = {0x02b6d05fu, 0xa70e2c11u, 0xc106f049u, 0x9bb97ea3u, 0x492ae26eu, 0x9e5c4dfdu, 0x746d3f58u, 0x2de6a9b8u};
  for (int i = 0; i < 8; ++i) r.l[i] = v[i]; return r.to_mont();
}
template <class F> TB_HD F zeta_const();  // pasta_curves ZETA (cube root of unity; halo2 coset shift)
template <> TB_HD Fp zeta_const<Fp>() {
  Fp r; const uint32_t v[8] = {0xfdfe4ab9u, 0x1dad5ebdu, 0x37ad3149u, 0x1d1f8bd2u, 0x57aab1b0u, 0x2caad5dcu, 0x4acdba71u, 0x12ccca83u};
  for (int i = 0; i < 8; ++i) r.l[i] = v[i]; return r.to_mont();
}
template <> TB_HD Fq zeta_const<Fq>() {
  Fq r; const uint32_t v[8] = {0x50aa0e4fu, 0x2aa9d2e0u, 0x47c033afu, 0x0fed467du, 0x1cf70f5au, 0x511db4d8u, 0x283e528eu, 0x06819a58u};
  for (int i = 0; i < 8; ++i) r.l[i] = v[i]; return r.to_mont();
}

}  // namespace tb
