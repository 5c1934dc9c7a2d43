// Device-side Fiat-Shamir transcript and blinding PRF.
//
// Replaces halo2_proofs `transcript::Blake2bWrite<_, vesta::Affine, Challenge255<_>>` (EXT; instantiated at
// taiga_halo2/src/proof.rs:32) so that a whole batch of proofs advances through its ~40 challenge points without a
// host round trip: one thread per proof keeps a streaming BLAKE2b-512 state (personal "Halo2-Transcript"), absorbs
// 0x01||x||y for points, 0x02||repr for scalars and squeezes 0x00 -> 64-byte digest -> wide reduction mod p
// (SURVEY.md App. A.3).  Proof bytes (32-byte compressed points / scalars) are appended on the device.
//
// The blinding PRF replaces the caller's `RngCore` (proof.rs:30): every random scalar of proof i is
// BLAKE2b-512(personal "TaigaB200-Blind\0", seed || i || tag || index) reduced mod p, reproducible on the CPU oracle.
#define TB_NOINLINE_MUL 0  // loop-structured kernels: small code, keep the multiply inline
#include "common.cuh"
#include "prover.cuh"

namespace tb {

__device__ __constant__ uint64_t B2B_IV[8] = {0x6a09e667f3bcc908ULL, 0xbb67ae8584caa73bULL, 0x3c6ef372fe94f82bULL, 0xa54ff53a5f1d36f1ULL,
                                              0x510e527fade682d1ULL, 0x9b05688c2b3e6c1fULL, 0x1f83d9abfb41bd6bULL, 0x5be0cd19137e2179ULL};
__device__ __constant__ uint8_t B2B_SIGMA[12][16] = {
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3},
    {11, 8, 12, 0, 5, 2, 15, 13, 10, 14, 3, 6, 7, 1, 9, 4}, {7, 9, 3, 1, 13, 12, 11, 14, 2, 6, 5, 10, 4, 0, 15, 8},
    {9, 0, 5, 7, 2, 4, 10, 15, 14, 1, 11, 12, 6, 8, 3, 13}, {2, 12, 6, 10, 0, 11, 8, 3, 4, 13, 7, 5, 15, 14, 1, 9},
    {12, 5, 1, 15, 14, 13, 4, 10, 0, 7, 6, 3, 9, 2, 8, 11}, {13, 11, 7, 14, 12, 1, 3, 9, 5, 0, 15, 4, 8, 6, 2, 10},
    {6, 15, 14, 9, 11, 3, 0, 8, 12, 2, 13, 7, 1, 4, 10, 5}, {10, 2, 8, 4, 7, 6, 1, 5, 15, 11, 9, 14, 3, 12, 13, 0},
    {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15}, {14, 10, 4, 8, 9, 15, 13, 6, 1, 12, 0, 2, 11, 7, 5, 3}};

__device__ __forceinline__ uint64_t rotr64(uint64_t x, int n) { return (x >> n) | (x << (64 - n)); }

__device__ void b2b_compress(uint64_t* h, const uint64_t* m, uint64_t t, bool last) {
  uint64_t v[16];
  for (int i = 0; i < 8; ++i) { v[i] = h[i]; v[i + 8] = B2B_IV[i]; }
  v[12] ^= t;
  if (last) v[14] = ~v[14];
#define TB_G(a, b, c, d, x, y)                                                                         \
  v[a] = v[a] + v[b] + (x); v[d] = rotr64(v[d] ^ v[a], 32); v[c] = v[c] + v[d]; v[b] = rotr64(v[b] ^ v[c], 24); \
  v[a] = v[a] + v[b] + (y); v[d] = rotr64(v[d] ^ v[a], 16); v[c] = v[c] + v[d]; v[b] = rotr64(v[b] ^ v[c], 63);
  for (int r = 0; r < 12; ++r) {
    const uint8_t* s = B2B_SIGMA[r];
    TB_G(0, 4, 8, 12, m[s[0]], m[s[1]]) TB_G(1, 5, 9, 13, m[s[2]], m[s[3]]) TB_G(2, 6, 10, 14, m[s[4]], m[s[5]]) TB_G(3, 7, 11, 15, m[s[6]], m[s[7]])
    TB_G(0, 5, 10, 15, m[s[8]], m[s[9]]) TB_G(1, 6, 11, 12, m[s[10]], m[s[11]]) TB_G(2, 7, 8, 13, m[s[12]], m[s[13]]) TB_G(3, 4, 9, 14, m[s[14]], m[s[15]])
  }
#undef TB_G
  for (int i = 0; i < 8; ++i) h[i] ^= v[i] ^ v[i + 8];
}

__device__ void b2b_init(uint64_t* h, const char* personal16) {
  for (int i = 0; i < 8; ++i) h[i] = B2B_IV[i];
  h[0] ^= 0x01010040ULL;  // digest 64, fanout 1, depth 1
  uint64_t p0 = 0, p1 = 0;
  for (int i = 0; i < 8; ++i) { p0 |= (uint64_t)(uint8_t)personal16[i] << (8 * i); p1 |= (uint64_t)(uint8_t)personal16[8 + i] << (8 * i); }
  h[6] ^= p0; h[7] ^= p1;
}

__device__ void tr_update(TrState& s, const uint8_t* data, int len) {
  for (int i = 0; i < len; ++i) {
    if (s.buflen == 128) { s.t += 128; b2b_compress(s.h, reinterpret_cast<const uint64_t*>(s.buf), s.t, false); s.buflen = 0; }
    s.buf[s.buflen++] = data[i];
  }
}

// 64-byte digest (as 16 LE 32-bit words) -> field element in Montgomery form: lo + hi * 2^256 (mod p)
__device__ Fp reduce_wide(const uint32_t* w) {
  Fp lo, hi;
  for (int i = 0; i < 8; ++i) { lo.l[i] = w[i]; hi.l[i] = w[8 + i]; }
  Fp r2 = Fp::r2();
  return r2 * lo + r2 * (r2 * hi);  // the reduced operand goes first: Fe::operator* needs a < m, b may be any 256-bit value
}

__device__ Fp tr_squeeze_one(TrState& s) {
  uint8_t z = 0;
  tr_update(s, &z, 1);
  uint64_t h[8]; for (int i = 0; i < 8; ++i) h[i] = s.h[i];
  uint64_t blk[16];
  uint8_t* bb = reinterpret_cast<uint8_t*>(blk);
  for (int i = 0; i < 128; ++i) bb[i] = i < (int)s.buflen ? s.buf[i] : 0;
  b2b_compress(h, blk, s.t + s.buflen, true);
  return reduce_wide(reinterpret_cast<const uint32_t*>(h));
}

__global__ void tr_init_kernel(TrState* st, int B, Fp vk_repr_canonical) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  TrState s;
  b2b_init(s.h, "Halo2-Transcript");
  s.t = 0; s.buflen = 0; s.proof_len = 0; s.error = 0; s.pad = 0;
  uint8_t pre = 2;
  tr_update(s, &pre, 1);
  tr_update(s, reinterpret_cast<const uint8_t*>(vk_repr_canonical.l), 32);
  st[b] = s;
}

// absorb `count` affine points (Montgomery) per proof; write != 0 also appends the 32-byte compressed encoding
__global__ void tr_points_kernel(TrState* st, uint8_t* proofs, uint32_t cap, int B, const Aff<Fq>* pts, long long stride, int count, int write) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  TrState s = st[b];
  for (int i = 0; i < count; ++i) {
    Aff<Fq> p = pts[(long long)b * stride + i];
    if (p.is_inf()) { s.error |= TR_ERR_INFINITY; continue; }  // "cannot write points at infinity to the transcript"
    Fq x = p.x.from_mont(), y = p.y.from_mont();
    uint8_t pre = 1;
    tr_update(s, &pre, 1);
    tr_update(s, reinterpret_cast<const uint8_t*>(x.l), 32);
    tr_update(s, reinterpret_cast<const uint8_t*>(y.l), 32);
    if (write) {
      if (s.proof_len + 32 > cap) { s.error |= TR_ERR_OVERFLOW; continue; }
      uint32_t* out = reinterpret_cast<uint32_t*>(proofs + (size_t)b * cap + s.proof_len);
      for (int j = 0; j < 8; ++j) out[j] = x.l[j];
      out[7] |= (y.l[0] & 1u) << 31;
      s.proof_len += 32;
    }
  }
  st[b] = s;
}

__global__ void tr_scalars_kernel(TrState* st, uint8_t* proofs, uint32_t cap, int B, const Fp* sc, long long stride, int count, int write) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  TrState s = st[b];
  for (int i = 0; i < count; ++i) {
    Fp v = sc[(long long)b * stride + i].from_mont();
    uint8_t pre = 2;
    tr_update(s, &pre, 1);
    tr_update(s, reinterpret_cast<const uint8_t*>(v.l), 32);
    if (write) {
      if (s.proof_len + 32 > cap) { s.error |= TR_ERR_OVERFLOW; continue; }
      uint32_t* out = reinterpret_cast<uint32_t*>(proofs + (size_t)b * cap + s.proof_len);
      for (int j = 0; j < 8; ++j) out[j] = v.l[j];
      s.proof_len += 32;
    }
  }
  st[b] = s;
}

__global__ void tr_squeeze_kernel(TrState* st, int B, Fp* out, long long stride, int count) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  TrState s = st[b];
  for (int i = 0; i < count; ++i) out[(long long)b * stride + i] = tr_squeeze_one(s);
  st[b] = s;
}

void Transcripts::init(Ctx* c, int B_, uint32_t cap_, const Fp& vk_repr_canonical) {
  ctx = c; B = B_; cap = cap_;
  states = DevBuf<TrState>(c, B);
  proofs = DevBuf<uint8_t>(c, (size_t)B * cap);
  proofs.zero();
  launch(c, tr_init_kernel, (B + 31) / 32, 32, 0, states.get(), B, vk_repr_canonical);
}
void Transcripts::points(const Aff<Fq>* pts, long long stride, int count, bool write) {
  ProfScope prof_scope(ctx, PC_TRANSCRIPT);
  launch(ctx, tr_points_kernel, (B + 31) / 32, 32, 0, states.get(), proofs.get(), cap, B, pts, stride, count, write ? 1 : 0);
}
void Transcripts::scalars(const Fp* sc, long long stride, int count, bool write) {
  ProfScope prof_scope(ctx, PC_TRANSCRIPT);
  launch(ctx, tr_scalars_kernel, (B + 31) / 32, 32, 0, states.get(), proofs.get(), cap, B, sc, stride, count, write ? 1 : 0);
}
void Transcripts::squeeze(Fp* out, long long stride, int count) {
  ProfScope prof_scope(ctx, PC_TRANSCRIPT);
  launch(ctx, tr_squeeze_kernel, (B + 31) / 32, 32, 0, states.get(), B, out, stride, count);
}

// ---------------------------------------------------------------- blinding PRF
__device__ Fp prf_scalar(const uint32_t* seed8, uint32_t proof, uint32_t tag, uint32_t idx) {
  uint64_t h[8];
  b2b_init(h, "TaigaB200-Blind\0");
  uint64_t m[16];
  for (int i = 0; i < 4; ++i) m[i] = (uint64_t)seed8[2 * i] | ((uint64_t)seed8[2 * i + 1] << 32);
  m[4] = (uint64_t)proof | ((uint64_t)tag << 32);
  m[5] = (uint64_t)idx;
  for (int i = 6; i < 16; ++i) m[i] = 0;
  b2b_compress(h, m, 48, true);
  return reduce_wide(reinterpret_cast<const uint32_t*>(h));
}

struct SeedArg { uint32_t w[8]; };
// out[b*stride + i*elem_stride] = PRF(seed, proof0 + b, tag, idx0 + i), i < count
__global__ void prf_fill_kernel(SeedArg seed, uint32_t proof0, uint32_t tag, uint32_t idx0, Fp* out, long long stride, long long elem_stride, int count, int B) {
  long long id = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (long long)B * count) return;
  int b = (int)(id / count), i = (int)(id % count);
  st_fe(out + (long long)b * stride + (long long)i * elem_stride, prf_scalar(seed.w, proof0 + b, tag, idx0 + i));
}

void prf_fill(Ctx* c, const uint8_t* seed32, uint32_t proof0, uint32_t tag, uint32_t idx0, Fp* out, long long stride, long long elem_stride, int count, int B) {
  if (count <= 0) return;
  SeedArg s; memcpy(s.w, seed32, 32);
  long long total = (long long)B * count;
  launch(c, prf_fill_kernel, (unsigned)((total + 127) / 128), 128, 0, s, proof0, tag, idx0, out, stride, elem_stride, count, B);
}

}  // namespace tb
