// Device side of the Fiat-Shamir transcript and the blinding PRF (formats in transcript.cuh).
//
// A whole batch of proofs advances through its ~40 challenge points without a host round trip: one thread per proof
// keeps its transcript state, and the proof bytes (32-byte compressed points / scalars) are appended on the device.
#define TB_NOINLINE_MUL 0  // loop-structured kernels: small code, keep the multiply inline
#include "common.cuh"
#include "prover.cuh"

namespace tb {

__global__ void tr_init_kernel(TrState* st, int B, Fp vk_repr_canonical) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  TrState s;
  s.tr.start(vk_repr_canonical); s.proof_len = 0; s.error = 0;
  st[b] = s;
}

// absorb `count` affine points (Montgomery) per proof; write != 0 also appends the 32-byte compressed encoding
__global__ void tr_points_kernel(TrState* st, uint8_t* proofs, uint32_t cap, int B, const Aff<Fq>* pts, long long stride, int count, int write) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  TrState s = st[b];
  for (int i = 0; i < count; ++i) {
    Aff<Fq> p = pts[(long long)b * stride + i].from_mont();
    if (!s.tr.absorb_point(p)) { s.error |= TR_ERR_INFINITY; continue; }
    if (write) {
      if (s.proof_len + 32 > cap) { s.error |= TR_ERR_OVERFLOW; continue; }
      compress_point(p, reinterpret_cast<uint32_t*>(proofs + (size_t)b * cap + s.proof_len));
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
    s.tr.absorb_scalar(v);
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
  for (int i = 0; i < count; ++i) out[(long long)b * stride + i] = s.tr.squeeze();
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
