// Internal declarations of the batched PLONKish/IPA prover engine (transcript.cu, polyops.cu, lookup.cu,
// quotient.cu, prover.cu).  Unit of work: B independent proofs of the SAME circuit, device resident from the moment
// the advice tables are uploaded until the proof bytes come back (SURVEY.md §7 design stance).
#pragma once
#include <cstring>
#include "../../include/taiga_b200.h"
#include "common.cuh"
#include "kernels.cuh"
#include "srs.cuh"
#include "transcript.cuh"

namespace tb {

// ---------------------------------------------------------------- transcript.cu
enum { TR_ERR_INFINITY = 1, TR_ERR_OVERFLOW = 2 };
struct TrState { Transcript tr; uint32_t proof_len, error; };
struct Transcripts {
  Ctx* ctx = nullptr; int B = 0; uint32_t cap = 0;
  DevBuf<TrState> states; DevBuf<uint8_t> proofs;
  void init(Ctx* c, int B, uint32_t cap, const Fp& vk_repr_canonical);
  void points(const Aff<Fq>* pts, long long stride, int count, bool write);   // common_point / write_point
  void scalars(const Fp* sc, long long stride, int count, bool write);        // common_scalar / write_scalar
  void squeeze(Fp* out, long long stride, int count);                         // squeeze_challenge_scalar
};
// blinding PRF tags (must match oracle/plonk.cpp RndTag)
enum RndTag { R_ADVICE_ROWS = 1, R_ADVICE_BLIND, R_LK_IN_ROWS, R_LK_TAB_ROWS, R_LK_IN_BLIND, R_LK_TAB_BLIND, R_PERM_ROWS, R_PERM_BLIND,
              R_LKZ_ROWS, R_LKZ_BLIND, R_RANDOM_POLY, R_RANDOM_BLIND, R_H_BLIND, R_QPRIME_BLIND, R_S_POLY, R_S_BLIND, R_IPA_L, R_IPA_R };
void prf_fill(Ctx* c, const uint8_t* seed32, uint32_t proof0, uint32_t tag, uint32_t idx0, Fp* out, long long stride, long long elem_stride,
              int count, int B);

// ---------------------------------------------------------------- polyops.cu  (all batched over B proofs; strides in elements)
// out[b][i] = out[b][i] * s[b*s_stride] + in[b][i]      (in_stride may be 0 = shared polynomial)
void poly_fma(Ctx* c, Fp* out, long long out_stride, const Fp* s, long long s_stride, const Fp* in, long long in_stride, int n, int B);
// out[b][i] = a[b][i] * s[b*s_stride]
void poly_scale(Ctx* c, Fp* out, long long out_stride, const Fp* s, long long s_stride, const Fp* a, long long a_stride, int n, int B);
void poly_copy(Ctx* c, Fp* out, long long out_stride, const Fp* in, long long in_stride, int n, int B);
// v[b*stride + idx] += sign * s[b*s_stride]   (sign = +1 / -1)
void poly_add_at(Ctx* c, Fp* v, long long stride, int idx, const Fp* s, long long s_stride, int sign, int B);
struct EvalItem { const Fp* base; long long bstride; int point; int pad; };
// evals[b*ev_stride + t] = poly_t(points[b*pt_stride + items[t].point]),  poly_t = items[t].base + b*items[t].bstride, n coefficients
void poly_eval(Ctx* c, const EvalItem* d_items, int nitems, const Fp* points, long long pt_stride, Fp* evals, long long ev_stride, int n, int B);
// out[b] = quotient of (in[b](X) - in[b](z_b)) / (X - z_b), zero padded to n coefficients (halo2 kate_division + resize)
void poly_kate_div(Ctx* c, Fp* out, long long out_stride, const Fp* in, long long in_stride, const Fp* z, long long z_stride, int n, int B);
void batch_inverse(Ctx* c, Fp* v, size_t count);  // elementwise, 0 -> 0
// out[b][0] = 1, out[b][i] = prod_{j<i} in[b][j]   (count independent vectors of n; n a power of two)
void prefix_product(Ctx* c, Fp* out, const Fp* in, int n, int count);
// out[b] = sum_i a[b][i] * bvec[b][i]
void inner_product(Ctx* c, Fp* out, long long out_stride, const Fp* a, long long a_stride, const Fp* bvec, long long b_stride, int n, int B);
// out[b][i] = x[b]^i
void powers(Ctx* c, Fp* out, long long out_stride, const Fp* x, long long x_stride, int n, int B);

// ---------------------------------------------------------------- generic small per-proof scalar programs (prover.cu)
// One thread per proof runs a tiny field program over a per-proof scratch vector (challenges, blinds, evaluation points).
enum ScalarOp { S_MUL = 0, S_ADD, S_SUB, S_INV, S_COPY, S_POW2K /* dst = a^(2^imm) */, S_CONST /* dst = consts[imm] */, S_NEG, S_FMA /* dst = dst*a + b */, S_POWI /* dst = a^imm */ };
struct ScalarInstr { uint16_t op, dst, a, b; uint32_t imm; };
void scalar_program(Ctx* c, Fp* vars, long long stride, const ScalarInstr* d_prog, int ninstr, const Fp* d_consts, int B);

}  // namespace tb
