// Row-parallel evaluation of the PLONKish gate / lookup / permutation constraint polynomial (the quotient numerator)
// and the grand-product helpers, for sm_90a.
//
// Replaces the h(X) construction of halo2_proofs `plonk::create_proof` + `vanishing::Argument::construct`,
// `permutation::Argument::commit` and `lookup::Argument::commit_product` (EXT; SURVEY.md §8a rows H3-H5, App. A.1
// step 8, App. E.3/E.6).  The extended domain is never materialised per column: for each of the R = 2^(ext_k-k)
// sub-cosets zeta*w_ext^k1*<w> the per-proof columns are NTT'd onto that sub-coset (n rows), every constraint is
// evaluated one thread per row, and the result is scaled by the (constant on the sub-coset) 1/(X^n - 1).
//
// Algorithmic bytes per sub-coset row: 32*(C+1), C = distinct column-cosets read (SURVEY §8d).
#define TB_NOINLINE_MUL 0  // loop-structured kernels: small code, keep the multiply inline
#include "common.cuh"
#include "prover_kernels.cuh"

namespace tb {

// ---------------------------------------------------------------- interpreter kernel
// One thread per (row, constraint part).  ALL values, including the running folds, live in the shared-memory register file
// [nregs + 2][T] x 32 B (slot nregs = the y / theta fold accumulator, slot nregs + 1 = the group / table fold): the loop carries
// no 256-bit value in registers, which kept the compiler from shuffling 16-24 registers on every interpreted instruction
// (ncu source view of the previous version: 30 % of the executed instructions were MOV / CS2R / SEL / BRA).
// `pl` is indexed by blockIdx.z: __grid_constant__ keeps those loads in the parameter bank, where ptxas would otherwise copy the
// part list to the stack of every thread.
struct QRowMachine {   // gate_interp's machine: one row of one proof; register r lives at [r * T] of the two halves
  const uint4* __restrict__ prog; uint4* rlo; uint4* rhi; int T, row, b;
  const Fp* adv; const Fp* inst; const Fp* chal; const QData& d;
  __device__ QInstr instr(int pc) const { const uint4 w = __ldg(prog + pc); QInstr i; i.w0 = w.x; i.a = w.y; i.b = w.z; i.pad = w.w; return i; }
  __device__ int slot(int r) const { return r * T; }
  __device__ Fp get(int i) const { const uint4 x = rlo[i], z = rhi[i]; Fp v;
    v.l[0] = x.x; v.l[1] = x.y; v.l[2] = x.z; v.l[3] = x.w; v.l[4] = z.x; v.l[5] = z.y; v.l[6] = z.z; v.l[7] = z.w; return v; }
  __device__ void set(int i, const Fp& v) const {
    rlo[i] = make_uint4(v.l[0], v.l[1], v.l[2], v.l[3]); rhi[i] = make_uint4(v.l[4], v.l[5], v.l[6], v.l[7]); }
  __device__ Fp leaf(int kind, uint32_t v) const {   // one load for either kind of leaf
    const Fp* p;
    if (kind == K_CONST) p = d.consts + v;
    else { const int rot = (int)(v & 255u) - 128; const size_t col = v >> 8;
      const Fp* base = kind == K_ADV ? adv + col * d.n : kind == K_INST ? inst + col * d.n : d.fix + (col * d.R + d.k1) * d.n;
      p = base + ((row + rot + d.n) & (d.n - 1)); }
    return ldg_fe(p);
  }
  __device__ const Fp& ypow(uint32_t gap) const { return chal[d.ytab_slot + gap]; }
  __device__ const Fp& theta() const { return chal[d.theta_slot]; }
  __device__ void lk_store(uint32_t l, const Fp& a, const Fp& s) const { const size_t o = (size_t)b * d.lk_pstride + (size_t)l * d.n + row; st_fe(d.lkA + o, a); st_fe(d.lkS + o, s); }
};
__global__ void __launch_bounds__(128) q_interp_kernel(const __grid_constant__ QPartList pl, int nregs, QData d) {
  const uint4* __restrict__ prog = reinterpret_cast<const uint4*>(pl.prog[blockIdx.z]);
  const int ninstr = pl.ninstr[blockIdx.z];
  extern __shared__ uint4 q_smem[];
  const int T = blockDim.x, tid = threadIdx.x;
  uint4* rlo = q_smem + tid;
  uint4* rhi = q_smem + (size_t)(nregs + 2) * T + tid;
  const int row = blockIdx.x * T + tid, b = blockIdx.y;
  if (row >= d.n) return;
  QRowMachine m = {prog, rlo, rhi, T, row, b, d.adv + (long long)b * d.adv_pstride, d.inst + (long long)b * d.inst_pstride, d.chal + (long long)b * d.chal_stride, d};
  gate_interp(m, nregs, ninstr);
  if (d.gate_out) st_fe(d.gate_out + (long long)blockIdx.z * pl.part_stride + (long long)b * d.gate_pstride + row, m.get(m.slot(nregs)));
}

// The same interpreter on listed rows: thread (s, b) of program blockIdx.z evaluates row rows[b * M + s], s < min(M, nrows[b])
__global__ void __launch_bounds__(128) q_interp_rows_kernel(const QInstr* __restrict__ code, const int2* __restrict__ table, int nregs, QData d,
                                                            const uint32_t* __restrict__ rows, const uint64_t* __restrict__ nrows, long long nrows_stride, int M,
                                                            uint8_t* __restrict__ nonzero) {
  extern __shared__ uint4 q_smem[];
  const int T = blockDim.x, tid = threadIdx.x, s = blockIdx.x * T + tid, b = blockIdx.y, j = blockIdx.z;
  if ((uint64_t)s >= min((uint64_t)M, nrows[(long long)b * nrows_stride])) return;
  const int2 e = table[j];
  const int row = (int)rows[(size_t)b * M + s];
  QRowMachine m = {reinterpret_cast<const uint4*>(code + e.x), q_smem + tid, q_smem + (size_t)(nregs + 2) * T + tid, T, row, b,
                   d.adv + (long long)b * d.adv_pstride, d.inst + (long long)b * d.inst_pstride, d.chal + (long long)b * d.chal_stride, d};
  gate_interp(m, nregs, e.y);
  nonzero[((size_t)b * M + s) * gridDim.z + j] = m.get(m.slot(nregs)).is_zero() ? 0 : 1;
}

static double program_muls(const QProgram& p) {   // field multiplications per evaluated row
  double m = 0;
  for (const QInstr& in : p.prog.code) { const int op = in.w0 & 0xff; m += (op == Q_MUL || op == Q_FOLD_Y || op == Q_FOLD_A || op == Q_FOLD_S || op == Q_GFOLD) ? 1.0 : op == Q_GEND ? 2.0 : 0.0; }
  return m;
}
static void q_launch(Ctx* c, const QPartList& pl, int nregs, const QData& d, int B) {
  ProfScope prof_scope(c, PC_QUOT_GATES);
  c->opt_in_smem(q_interp_kernel, 96 * 1024);
  // T threads evaluate T rows; the register file [nregs + 2][T] x 32 B lives in shared memory
  int T = (96 * 1024) / ((nregs + 2) * 32);
  T = T >= 128 ? 128 : (T / 16) * 16;
  TB_REQUIRE(T >= 16 && T <= 128, "constraint program register file does not fit shared memory");
  while (T > d.n && T > 1) T >>= 1;
  const size_t smem = (size_t)(nregs + 2) * T * 32;
  launch(c, q_interp_kernel, dim3((d.n + T - 1) / T, B, pl.nparts), T, smem, pl, nregs, d);
}
void q_run(Ctx* c, const QProgram& prog, const QData& d, int B) {
  QPartList pl; memset(&pl, 0, sizeof(pl));
  pl.prog[0] = prog.dev.get(); pl.ninstr[0] = (int)prog.prog.code.size(); pl.nparts = 1; pl.part_stride = 0;
  c->work[PC_QUOT_GATES] += program_muls(prog) * (double)d.n * B;
  q_launch(c, pl, prog.prog.nregs, d, B);
}
void q_run_parts(Ctx* c, const std::vector<QProgram>& progs, QData d, long long part_stride, int B) {
  QPartList pl; memset(&pl, 0, sizeof(pl));
  int nregs = 1;
  pl.nparts = (int)progs.size(); pl.part_stride = part_stride;
  for (int p = 0; p < pl.nparts; ++p) c->work[PC_QUOT_GATES] += program_muls(progs[p]) * (double)d.n * B;
  for (int p = 0; p < pl.nparts; ++p) { pl.prog[p] = progs[p].dev.get(); pl.ninstr[p] = (int)progs[p].prog.code.size(); nregs = nregs > progs[p].prog.nregs ? nregs : progs[p].prog.nregs; }
  q_launch(c, pl, nregs, d, B);
}
void q_run_rows(Ctx* c, const QInstr* code, const int2* table, int nprogs, int nregs, const QData& d, const uint32_t* rows, const uint64_t* nrows,
                long long nrows_stride, int M, uint8_t* nonzero, int B) {
  if (M == 0 || nprogs == 0) return;
  ProfScope prof_scope(c, PC_QUOT_GATES);
  c->opt_in_smem(q_interp_rows_kernel, 96 * 1024);
  int T = (96 * 1024) / ((nregs + 2) * 32);   // as q_launch: the register file fits 96 KiB
  T = T >= 128 ? 128 : (T / 16) * 16;
  while (T > 32 && T / 2 >= M) T >>= 1;        // few listed rows: small CTAs
  const size_t smem = (size_t)(nregs + 2) * T * 32;
  launch(c, q_interp_rows_kernel, dim3((M + T - 1) / T, B, nprogs), T, smem, code, table, nregs, d, rows, nrows, nrows_stride, M, nonzero);
}

}  // namespace tb
