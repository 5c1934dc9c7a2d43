// Host instantiation of the product's __host__ __device__ field/curve arithmetic and transcript (taiga_b200/csrc/*.cuh),
// so the same source the kernels compile can be checked on a CPU-only box against the oracle.
#include <cstring>
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
