// Declarations for lookup.cu and quotient.cu (kernel drivers used by prover.cu).
#pragma once
#include "argument.cuh"
#include "gates.cuh"
#include "prover.cuh"

namespace tb {

// ---------------------------------------------------------------- lookup.cu
void lookup_keys(Ctx* c, Fp* keys, const Fp* vals, int n, int usable, int arrays);      // Montgomery -> canonical sort keys (+ sentinels)
void sort_keys(Ctx* c, Fp* keys, int n, int arrays);                                      // ascending, canonical-integer order
void lookup_arrange(Ctx* c, const Fp* sortedA, const Fp* sortedT, Fp* scratch, Fp* S, int n, int usable, int arrays, uint32_t* d_err);

// ---------------------------------------------------------------- quotient.cu
// Row-parallel interpreter of the programs of gates.cuh.  Temporaries live in a shared-memory register file laid out
// [reg][thread] as two 16-byte halves; leaves (column queries, constants) are read straight from global memory.
struct QProgram {           // compiled once per circuit (host), resident on the device
  GateProgram prog; DevMem<QInstr> dev;
  QProgram() {}
  explicit QProgram(GateProgram&& p) : prog(std::move(p)) { if (!prog.code.empty()) dev = DevMem<QInstr>(prog.code); }
};
struct QPartList { const QInstr* prog[Q_MAX_PARTS]; int ninstr[Q_MAX_PARTS]; int nparts; long long part_stride; };

struct QData {
  const Fp* adv; long long adv_pstride;     // [B][num_advice][n]
  const Fp* inst; long long inst_pstride;   // [B][num_instance][n]
  const Fp* fix; int R; int k1;             // [num_fixed][R][n]  (R = 1: Lagrange values)
  const Fp* consts;                         // Montgomery
  const Fp* chal; long long chal_stride; int y_slot, theta_slot, ytab_slot;   // chal[ytab_slot + i] = y^i (0 <= i <= constraints + permutation / lookup terms)
  Fp* gate_out; long long gate_pstride;     // [B][n]
  Fp* lkA; Fp* lkS; long long lk_pstride;   // [B][L][n]
  int n;
};
void q_run(Ctx* c, const QProgram& prog, const QData& d, int B);
void q_run_parts(Ctx* c, const std::vector<QProgram>& progs, QData d, long long part_stride, int B);

// permutation + lookup terms of the quotient, folded onto the gate accumulator, times 1/(X^n - 1) (constant per sub-coset)
struct QFinish {
  const Fp* gate;          // [nparts][B][n] partial Horner sums of the gate constraints
  int nparts; long long gate_part_stride; int ytab_slot; int gexp[Q_MAX_PARTS];   // numerator += chal[ytab_slot + gexp[p]] * gate[p]
  const Fp* rlo; long long rlo_pstride;   // remainder of the low-degree numerator modulo X^n - 1 on this sub-coset (or null): added before the division
  const Fp* adv; long long adv_pstride; const Fp* inst; long long inst_pstride;   // sub-coset evaluations
  const Fp* fix; const Fp* sig; int R; int k1;      // [nf][R][n], [P][R][n]
  const Fp* l0; const Fp* l_last; const Fp* l_blind; // [R][n]
  const Fp* pz; long long pz_pstride;                // [B][nsets][n]
  const Fp* lz; const Fp* lpin; const Fp* lptab; long long lk_pstride;  // per-proof stride of the three (merged coset buffer)
  long long lkc_pstride;                             // per-proof stride of lkA / lkS
  const Fp* lkA; const Fp* lkS;                      // [B][L][n] compressed input / table on this sub-coset
  const int2* perm_cols; int P; int chunk; int nsets; int L; int bf;
  const Fp* chal; long long chal_stride; int y_slot, beta_slot, gamma_slot;
  Fp delta; Fp zeta; Fp t_inv;                       // DELTA, ZETA, 1/((zeta w^k1)^n - 1)
  Fp delta_c0[PERM_MAX_SETS];                        // DELTA^(s*chunk) per permutation set
  TwiddleTables<Fp> tw;                              // forward tables
  int ext_k; int k;
  Fp* out; long long out_pstride;                    // H[b][k1][row]  (out + b*out_pstride + k1*n + row)
  int n;
};
void q_finish(Ctx* c, const QFinish& f, int B);

// extended_to_coeff step B: size-R inverse transform across sub-cosets + zeta^-i, keeps `pieces` * n coefficients
void h_cross(Ctx* c, const Fp* V, long long v_pstride, Fp* hcoef, long long h_pstride, int n, int R, int pieces, const Fp* d_wr_inv /* R * wr_step */,
             int wr_step, Fp r_inv, Fp zeta_inv, int B);
// low-degree numerator (SURVEY 8a H3, evaluated on every second sub-coset only):
//   out[b][k][row] = sum_p chal[b][ytab_slot + gexp[p]] * gate[p][b][row]      (combination of the low programs on one sub-coset)
void q_combine(Ctx* c, const Fp* gate, int nparts, long long part_stride, const int* gexp, const Fp* chal, long long chal_stride, int ytab_slot, Fp* out, long long out_pstride,
               int n, int B);
//   c[b][j][i], j < m: coefficients of H_lo.  r[b][i] = sum_j c[b][j][i] (= H_lo mod X^n - 1);  q[b][j][i] = sum_{t > j} c[b][t][i], j < m - 1 (= H_lo div X^n - 1)
void q_lo_split(Ctx* c, const Fp* coef, long long c_pstride, int m, Fp* r, long long r_pstride, Fp* q, long long q_pstride, int n, int B);
// h[b][j][i] += q[b][j][i], j < m
void q_add_blocks(Ctx* c, Fp* h, long long h_pstride, const Fp* q, long long q_pstride, int m, int n, int B);

// grand products (permutation / lookup)
struct PermFrac {
  const Fp* adv; long long adv_pstride; const Fp* inst; long long inst_pstride; const Fp* fix;   // Lagrange values
  const Fp* sig;                     // [P][n] sigma values
  const int2* perm_cols; int P; int chunk; int nsets;
  const Fp* chal; long long chal_stride; int beta_slot, gamma_slot;
  Fp delta, omega;
  Fp delta_c0[PERM_MAX_SETS];
  TwiddleTables<Fp> tw;
  Fp* num; Fp* den; long long pstride;   // [B][nsets][n]
  int n; int k;
};
void perm_fractions(Ctx* c, const PermFrac& p, int B);
// a[i] *= b[i]
void vec_mul(Ctx* c, Fp* a, const Fp* b, size_t count);
// z[b][s][i] *= carry, where carry_s = prod_{s' < s} zlocal[b][s'][u]; applied in place (u = last usable row)
void perm_chain(Ctx* c, Fp* z, long long pstride, int nsets, int n, int u, int B);
// lookup: den = (A'+beta)(S'+gamma), num = (A+beta)(S+gamma)
void lookup_fractions(Ctx* c, const Fp* A, const Fp* S, const Fp* Ap, const Fp* Sp, Fp* num, Fp* den, long long pstride, int L, int n,
                      const Fp* chal, long long chal_stride, int beta_slot, int gamma_slot, int B);

}  // namespace tb
