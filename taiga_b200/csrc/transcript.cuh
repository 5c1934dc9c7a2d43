// The Fiat-Shamir transcript of a proof, its point encoding and the blinding PRF: one source that the device prover
// (transcript.cu), the host verifier (verifier.cu) and the CPU tests (tests/host_shim.cpp, plain g++) all compile.
//
// Transcript: halo2_proofs `Blake2bWrite` / `Blake2bRead<_, vesta::Affine, Challenge255<_>>` (EXT; instantiated at
// taiga_halo2/src/proof.rs:32).  A streaming BLAKE2b-512 state (personal "Halo2-Transcript") absorbs 0x01||x||y for a
// point, 0x02||repr for a scalar, and a squeeze absorbs 0x00, then reduces the 64-byte digest mod p (SURVEY.md App. A.3).
//
// The blinding PRF replaces the caller's `RngCore` (proof.rs:30): every random scalar of proof i is
// BLAKE2b-512(personal "TaigaB200-Blind\0", seed || i || tag || index) reduced mod p, reproducible on the CPU oracle.
#pragma once
#include <cstring>
#include "curve.cuh"

namespace tb {

// ---------------------------------------------------------------- BLAKE2b-512 (RFC 7693)
// Each table is defined once; the device reads a copy of it in constant memory.
struct Blake2bIv { uint64_t w[8]; };
struct Blake2bSigma { uint8_t r[12][16]; };   // byte-aligned, as the device loads it
static constexpr Blake2bIv b2b_iv_host = {{0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                                           0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL}};
static constexpr Blake2bSigma b2b_sigma_host = {
    {{0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
     {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
     {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
     {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
     {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
     {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}}};
#ifdef __CUDACC__
static __constant__ Blake2bIv b2b_iv_dev = b2b_iv_host;
static __constant__ Blake2bSigma b2b_sigma_dev = b2b_sigma_host;
#endif
#ifdef __CUDA_ARCH__
#define TB_B2B(table) b2b_##table##_dev
#else
#define TB_B2B(table) b2b_##table##_host
#endif
TB_HD uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

// h ^= the compression of block m; t = bytes hashed so far including this block, last = final block
TB_HD void b2b_compress(uint64_t* h, const uint64_t* m, uint64_t t, bool last) {
  uint64_t v[16];
  for (int i = 0; i < 8; ++i) { v[i] = h[i]; v[i + 8] = TB_B2B(iv).w[i]; }
  v[12] ^= t;
  if (last) v[14] = ~v[14];
#define TB_G(a, b, c, d, x, y)                                                                         \
  v[a] = v[a] + v[b] + (x); v[d] = rotr64(v[d] ^ v[a], 32); v[c] = v[c] + v[d]; v[b] = rotr64(v[b] ^ v[c], 24); \
  v[a] = v[a] + v[b] + (y); v[d] = rotr64(v[d] ^ v[a], 16); v[c] = v[c] + v[d]; v[b] = rotr64(v[b] ^ v[c], 63);
  for (int r = 0; r < 12; ++r) {
    const uint8_t* s = TB_B2B(sigma).r[r];
    TB_G(0, 4, 8, 12, m[s[0]], m[s[1]]) TB_G(1, 5, 9, 13, m[s[2]], m[s[3]]) TB_G(2, 6, 10, 14, m[s[4]], m[s[5]]) TB_G(3, 7, 11, 15, m[s[6]], m[s[7]])
    TB_G(0, 5, 10, 15, m[s[8]], m[s[9]]) TB_G(1, 6, 11, 12, m[s[10]], m[s[11]]) TB_G(2, 7, 8, 13, m[s[12]], m[s[13]]) TB_G(3, 4, 9, 14, m[s[14]], m[s[15]])
  }
#undef TB_G
  for (int i = 0; i < 8; ++i) h[i] ^= v[i] ^ v[i + 8];
}

// chaining value for a 64-byte digest, no key, 16-byte personalisation
TB_HD void b2b_init(uint64_t* h, const char* personal16) {
  for (int i = 0; i < 8; ++i) h[i] = TB_B2B(iv).w[i];
  h[0] ^= 0x01010040ULL;  // digest 64, fanout 1, depth 1
  uint64_t p0 = 0, p1 = 0;
  for (int i = 0; i < 8; ++i) { p0 |= (uint64_t)(uint8_t)personal16[i] << (8 * i); p1 |= (uint64_t)(uint8_t)personal16[8 + i] << (8 * i); }
  h[6] ^= p0; h[7] ^= p1;
}
#undef TB_B2B

struct Blake2b {
  uint64_t h[8], t; alignas(8) uint8_t buf[128]; uint32_t buflen;   // t: bytes of the blocks compressed so far
  TB_HD void init(const char* personal16) { b2b_init(h, personal16); t = 0; buflen = 0; }
  // a full block is compressed only when more data arrives: the last block must be compressed as the final one
  TB_HD void update(const uint8_t* data, int len) {
    for (int i = 0; i < len; ++i) {
      if (buflen == 128) { t += 128; b2b_compress(h, reinterpret_cast<const uint64_t*>(buf), t, false); buflen = 0; }
      buf[buflen++] = data[i];
    }
  }
  // digest of everything absorbed so far; the state goes on absorbing
  TB_HD void finish(uint64_t* out) const {
    uint64_t blk[16];
    uint8_t* bb = reinterpret_cast<uint8_t*>(blk);
    for (int i = 0; i < 128; ++i) bb[i] = i < (int)buflen ? buf[i] : 0;
    for (int i = 0; i < 8; ++i) out[i] = h[i];
    b2b_compress(out, blk, t + buflen, true);
  }
};

// 64-byte digest (8 LE words) -> field element in Montgomery form: lo + hi * 2^256 (mod p)
TB_HD Fp reduce_wide(const uint64_t* d) {
  Fp lo, hi;
  memcpy(lo.l, d, 32); memcpy(hi.l, d + 4, 32);
  Fp r2 = Fp::r2();
  return r2 * lo + r2 * (r2 * hi);  // the reduced operand goes first: Fe::operator* needs a < m, b may be any 256-bit value
}

// ---------------------------------------------------------------- transcript
// Absorbs canonical values (what halo2 hashes is their `to_repr()`); challenges come out in Montgomery form.
struct Transcript {
  Blake2b hash;
  // the state every proof of a circuit starts from: common_scalar of the verifying key's representative
  TB_HD void start(const Fp& vk_repr) { hash.init("Halo2-Transcript"); absorb_scalar(vk_repr); }
  // halo2 refuses to hash the identity ("cannot write points at infinity to the transcript"): false, nothing absorbed
  TB_HD bool absorb_point(const Aff<Fq>& p) {
    if (p.is_inf()) return false;
    uint8_t pre = 1;
    hash.update(&pre, 1);
    hash.update(reinterpret_cast<const uint8_t*>(p.x.l), 32);
    hash.update(reinterpret_cast<const uint8_t*>(p.y.l), 32);
    return true;
  }
  TB_HD void absorb_scalar(const Fp& v) {
    uint8_t pre = 2;
    hash.update(&pre, 1);
    hash.update(reinterpret_cast<const uint8_t*>(v.l), 32);
  }
  TB_HD Fp squeeze() {
    uint8_t z = 0;
    hash.update(&z, 1);
    uint64_t d[8];
    hash.finish(d);
    return reduce_wide(d);
  }
};

// ---------------------------------------------------------------- encodings of the proof bytes (pasta_curves)
// A point in canonical coordinates <-> x little-endian with the parity of y in bit 255; the identity is 32 zero bytes.
TB_HD void compress_point(const Aff<Fq>& p, uint32_t* out) {
  for (int j = 0; j < 8; ++j) out[j] = p.x.l[j];
  out[7] |= (p.y.l[0] & 1u) << 31;
}

// 32 LE bytes -> Montgomery form; false unless the value is below the modulus
template <class F> TB_HD bool canonical(const uint8_t* b, F& out) {
  F raw; memcpy(raw.l, b, 32);
  F m; for (int i = 0; i < 8; ++i) m.l[i] = F::modulus_limb(i);
  if (F::cmp_raw(raw, m) >= 0) return false;
  out = raw.to_mont(); return true;
}
// square root in Fq (2-adicity 32) by Tonelli-Shanks; false if a is not a square
TB_HD bool tonelli_shanks(const Fq& a, Fq& out) {
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
// the inverse of compress_point; false for x >= q, an x off the curve, and x = 0 with the sign bit set (5 is not a square).
// The verifier decodes a batch's points with it on the device (decompress_kernel, verifier.cu).
TB_HD bool decompress_point(const uint8_t* b, Aff<Fq>& out) {
  uint8_t t[32]; memcpy(t, b, 32);
  int sign = t[31] >> 7; t[31] &= 0x7f;
  bool allz = true; for (int i = 0; i < 32; ++i) allz &= (t[i] == 0);
  if (allz && !sign) { out = Aff<Fq>::inf(); return true; }
  Fq x; if (!canonical<Fq>(t, x)) return false;
  Fq y; if (!tonelli_shanks(x.sqr() * x + Fq::from_u32(5), y)) return false;
  y = y.from_mont();
  if ((int)(y.l[0] & 1) != sign) y = y.neg();
  memcpy(out.x.l, t, 32); out.y = y; return true;
}

// ---------------------------------------------------------------- blinding PRF
// BLAKE2b-512("TaigaB200-Blind\0", seed || proof || tag || idx as 4 LE bytes each, then 4 zero bytes) mod p: one 48-byte block
TB_HD Fp prf_scalar(const uint32_t* seed8, uint32_t proof, uint32_t tag, uint32_t idx) {
  uint64_t h[8];
  b2b_init(h, "TaigaB200-Blind\0");
  uint64_t m[16];
  for (int i = 0; i < 4; ++i) m[i] = (uint64_t)seed8[2 * i] | ((uint64_t)seed8[2 * i + 1] << 32);
  m[4] = (uint64_t)proof | ((uint64_t)tag << 32);
  m[5] = (uint64_t)idx;
  for (int i = 6; i < 16; ++i) m[i] = 0;
  b2b_compress(h, m, 48, true);
  return reduce_wide(h);
}

}  // namespace tb
