// Permutation / lookup terms of the quotient, the size-R cross transform of extended_to_coeff and the grand-product
// helpers (second half of the h(X) construction; see quotient.cu for the gate interpreter).  These kernels have many
// distinct multiply sites, so the field multiply is called out of line here (instruction-cache footprint).
#define TB_NOINLINE_MUL 1
#include "common.cuh"
#include "prover_kernels.cuh"

namespace tb {

// One row of one proof on one sub-coset of the extended domain, or of the Lagrange values (R = 1, k1 = 0): the view
// through which argument.cuh reads the permutation columns, the sigma polynomials and (q_finish only) the permutation
// grand products.  Fixed and sigma columns are [col][R][n], the other columns [col][n]; rows wrap around.
struct RowView {
  const Fp* adv; const Fp* inst; const Fp* fix; const Fp* sig; const int2* cols; const Fp* pz;
  int R, k1, n, row, last_rot;
  __device__ __forceinline__ Fp perm_col(int c) const {
    const int2 col = cols[c];
    return col.x == TB_COL_ADVICE ? ldg_fe(adv + (size_t)col.y * n + row)
         : col.x == TB_COL_FIXED ? ldg_fe(fix + ((size_t)col.y * R + k1) * n + row) : ldg_fe(inst + (size_t)col.y * n + row);
  }
  __device__ __forceinline__ Fp sigma(int c) const { return ldg_fe(sig + ((size_t)c * R + k1) * n + row); }
  __device__ __forceinline__ Fp z(int s) const { return ldg_fe(pz + (size_t)s * n + row); }
  __device__ __forceinline__ Fp z_next(int s) const { return ldg_fe(pz + (size_t)s * n + ((row + 1) & (n - 1))); }
  __device__ __forceinline__ Fp z_last(int s) const { return ldg_fe(pz + (size_t)s * n + ((row + last_rot + n) & (n - 1))); }
};

// ---------------------------------------------------------------- permutation + lookup terms, vanishing division
__global__ void __launch_bounds__(128) q_finish_kernel(QFinish f) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (row >= f.n) return;
  const int n = f.n, nm = n - 1;
  const Fp* chal = f.chal + (long long)b * f.chal_stride;
  const Fp y = chal[f.y_slot], beta = chal[f.beta_slot], gamma = chal[f.gamma_slot];
  const size_t crow = (size_t)f.k1 * n + row;
  Fp acc = Fp::zero();   // gate programs: sum_p y^(J - 1 - last_p) S_p
  for (int p = 0; p < f.nparts; ++p) acc = acc + chal[f.ytab_slot + f.gexp[p]] * ldg_fe(f.gate + (size_t)p * f.gate_part_stride + (size_t)b * n + row);
  const Fp ll = ldg_fe(f.l_last + crow);
  const ArgPoint at = {y, beta, gamma, ldg_fe(f.l0 + crow), ll, Fp::one() - (ll + ldg_fe(f.l_blind + crow))};
  if (f.nsets) {   // without a permutation, X and its twiddle loads are not needed
    const RowView v = {f.adv + (long long)b * f.adv_pstride, f.inst + (long long)b * f.inst_pstride, f.fix, f.sig, f.perm_cols, f.pz + (long long)b * f.pz_pstride,
                       f.R, f.k1, n, row, -(f.bf + 1)};
    const Fp x = f.zeta * tw_pow(f.tw, (uint32_t)(f.k1 + f.R * row) << (TW_LOG - f.ext_k));   // zeta * w_ext^(k1 + R*row)
    acc = perm_fold(acc, v, at, f.nsets, f.chunk, f.P, f.delta, f.delta_c0, x);
  }
  for (int l = 0; l < f.L; ++l) {
    size_t o = (size_t)b * f.lk_pstride + (size_t)l * n, oc = (size_t)b * f.lkc_pstride + (size_t)l * n;
    Fp z = ldg_fe(f.lz + o + row), zn = ldg_fe(f.lz + o + ((row + 1) & nm));
    Fp ap = ldg_fe(f.lpin + o + row), apm = ldg_fe(f.lpin + o + ((row - 1 + n) & nm)), sp = ldg_fe(f.lptab + o + row);
    Fp a = ldg_fe(f.lkA + oc + row), t = ldg_fe(f.lkS + oc + row);
    acc = lookup_fold(acc, at, z, zn, ap, apm, sp, a, t);
  }
  if (f.rlo) acc = acc + ldg_fe(f.rlo + (long long)b * f.rlo_pstride + row);   // low-degree numerator modulo X^n - 1 (its quotient is added in coefficient form)
  st_fe(f.out + (long long)b * f.out_pstride + crow, acc * f.t_inv);
}

void q_finish(Ctx* c, const QFinish& f, int B) {
  ProfScope prof_scope(c, PC_QUOT_FINISH);
  c->work[PC_QUOT_FINISH] += (double)f.n * B * (3.0 * f.P + 6.0 * f.nsets + 16.0 * f.L + 2.0 * f.nparts + 8.0);   // permutation products, lookup terms, y folds
  launch(c, q_finish_kernel, dim3((f.n + 127) / 128, B), 128, 0, f);
}

// ---------------------------------------------------------------- extended_to_coeff, step B
__global__ void h_cross_kernel(const Fp* __restrict__ V, long long v_pstride, Fp* __restrict__ hcoef, long long h_pstride, int n, int R, int pieces,
                               const Fp* __restrict__ wr_inv, int wr_step, Fp r_inv, Fp zeta_inv) {
  int i2 = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i2 >= n) return;
  const Fp* v = V + (long long)b * v_pstride;
  Fp zi2 = zeta_inv.sqr();
  for (int i1 = 0; i1 < pieces; ++i1) {
    Fp acc = Fp::zero();
    for (int k1 = 0; k1 < R; ++k1) {
      Fp x = ldg_fe(v + (size_t)k1 * n + i2);
      int e = (i1 * k1) & (R - 1);
      acc = acc + (e ? x * ldg_fe(wr_inv + e * wr_step) : x);
    }
    acc = acc * r_inv;
    uint32_t m3 = (uint32_t)((size_t)i1 * n + i2) % 3u;
    if (m3) acc = acc * (m3 == 1 ? zeta_inv : zi2);
    st_fe(hcoef + (long long)b * h_pstride + (size_t)i1 * n + i2, acc);
  }
}
void h_cross(Ctx* c, const Fp* V, long long v_pstride, Fp* hcoef, long long h_pstride, int n, int R, int pieces, const Fp* d_wr_inv, int wr_step, Fp r_inv,
             Fp zeta_inv, int B) {
  launch(c, h_cross_kernel, dim3((n + 127) / 128, B), 128, 0, V, v_pstride, hcoef, h_pstride, n, R, pieces, d_wr_inv, wr_step, r_inv, zeta_inv);
}

// ---------------------------------------------------------------- low-degree part of the numerator (evaluated on every second sub-coset)
struct QCombineArgs { int gexp[Q_MAX_PARTS]; };
__global__ void q_combine_kernel(const Fp* __restrict__ gate, int nparts, long long part_stride, QCombineArgs a, const Fp* __restrict__ chal, long long chal_stride, int ytab_slot,
                                 Fp* __restrict__ out, long long out_pstride, int n) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (row >= n) return;
  const Fp* ch = chal + (long long)b * chal_stride;
  Fp acc = Fp::zero();
  for (int p = 0; p < nparts; ++p) acc = acc + ch[ytab_slot + a.gexp[p]] * ldg_fe(gate + (size_t)p * part_stride + (size_t)b * n + row);
  st_fe(out + (long long)b * out_pstride + row, acc);
}
void q_combine(Ctx* c, const Fp* gate, int nparts, long long part_stride, const int* gexp, const Fp* chal, long long chal_stride, int ytab_slot, Fp* out, long long out_pstride,
               int n, int B) {
  ProfScope prof_scope(c, PC_QUOT_FINISH);
  QCombineArgs a; for (int p = 0; p < Q_MAX_PARTS; ++p) a.gexp[p] = p < nparts ? gexp[p] : 0;
  c->work[PC_QUOT_FINISH] += (double)n * B * nparts;
  launch(c, q_combine_kernel, dim3((n + 127) / 128, B), 128, 0, gate, nparts, part_stride, a, chal, chal_stride, ytab_slot, out, out_pstride, n);
}
__global__ void q_lo_split_kernel(const Fp* __restrict__ coef, long long c_pstride, int m, Fp* __restrict__ r, long long r_pstride, Fp* __restrict__ q, long long q_pstride, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= n) return;
  const Fp* cb = coef + (long long)b * c_pstride;
  Fp run = Fp::zero();
  for (int j = m - 1; j >= 1; --j) { run = run + ldg_fe(cb + (size_t)j * n + i); st_fe(q + (long long)b * q_pstride + (size_t)(j - 1) * n + i, run); }   // q_{j-1} = sum_{t >= j} c_t
  st_fe(r + (long long)b * r_pstride + i, run + ldg_fe(cb + i));
}
void q_lo_split(Ctx* c, const Fp* coef, long long c_pstride, int m, Fp* r, long long r_pstride, Fp* q, long long q_pstride, int n, int B) {
  launch(c, q_lo_split_kernel, dim3((n + 127) / 128, B), 128, 0, coef, c_pstride, m, r, r_pstride, q, q_pstride, n);
}
__global__ void q_add_blocks_kernel(Fp* __restrict__ h, long long h_pstride, const Fp* __restrict__ q, long long q_pstride, int count) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (i >= count) return;
  Fp* hp = h + (long long)b * h_pstride + i;
  st_fe(hp, ld_fe(hp) + ldg_fe(q + (long long)b * q_pstride + i));
}
void q_add_blocks(Ctx* c, Fp* h, long long h_pstride, const Fp* q, long long q_pstride, int m, int n, int B) {
  const int count = m * n;
  launch(c, q_add_blocks_kernel, dim3((count + 255) / 256, B), 256, 0, h, h_pstride, q, q_pstride, count);
}

// ---------------------------------------------------------------- grand products
__global__ void perm_fractions_kernel(PermFrac p) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y, b = blockIdx.z;
  if (row >= p.n) return;
  const int n = p.n;
  const Fp* chal = p.chal + (long long)b * p.chal_stride;
  const Fp beta = chal[p.beta_slot], gamma = chal[p.gamma_slot];
  const RowView v = {p.adv + (long long)b * p.adv_pstride, p.inst + (long long)b * p.inst_pstride, p.fix, p.sig, p.perm_cols, nullptr, 1, 0, n, row, 0};
  Fp num = Fp::one(), den = Fp::one();
  perm_set_products(v, s, p.chunk, p.P, beta, gamma, p.delta, p.delta_c0[s] * tw_pow(p.tw, (uint32_t)row << (TW_LOG - p.k)) * beta, den, num);   // X = omega^row
  size_t o = (size_t)b * p.pstride + (size_t)s * n + row;
  st_fe(p.num + o, num); st_fe(p.den + o, den);
}
void perm_fractions(Ctx* c, const PermFrac& p, int B) {
  if (!p.nsets) return;
  launch(c, perm_fractions_kernel, dim3((p.n + 127) / 128, p.nsets, B), 128, 0, p);
}

__global__ void vec_mul_kernel(Fp* a, const Fp* b, size_t count) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < count) st_fe(a + i, ld_fe(a + i) * ld_fe(b + i));
}
void vec_mul(Ctx* c, Fp* a, const Fp* b, size_t count) {
  if (!count) return;
  launch(c, vec_mul_kernel, (unsigned)((count + 255) / 256), 256, 0, a, b, count);
}

__global__ void perm_carry_kernel(const Fp* z, long long pstride, int nsets, int n, int u, Fp* carries, int B) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  Fp carry = Fp::one();
  for (int s = 0; s < nsets; ++s) { carries[(size_t)b * nsets + s] = carry; carry = carry * z[(long long)b * pstride + (size_t)s * n + u]; }
}
__global__ void perm_scale_kernel(Fp* z, long long pstride, int nsets, int n, const Fp* carries) {
  int row = blockIdx.x * blockDim.x + threadIdx.x, s = blockIdx.y, b = blockIdx.z;
  if (row >= n || s == 0) return;
  Fp* p = z + (long long)b * pstride + (size_t)s * n + row;
  st_fe(p, ld_fe(p) * carries[(size_t)b * nsets + s]);
}
void perm_chain(Ctx* c, Fp* z, long long pstride, int nsets, int n, int u, int B) {
  if (nsets <= 1) return;
  DevBuf<Fp> carries(c, (size_t)B * nsets);
  launch(c, perm_carry_kernel, (B + 31) / 32, 32, 0, z, pstride, nsets, n, u, carries.get(), B);
  launch(c, perm_scale_kernel, dim3((n + 255) / 256, nsets, B), 256, 0, z, pstride, nsets, n, carries.get());
}

__global__ void lookup_fractions_kernel(const Fp* A, const Fp* S, const Fp* Ap, const Fp* Sp, Fp* num, Fp* den, long long pstride, int n,
                                        const Fp* chal, long long chal_stride, int beta_slot, int gamma_slot) {
  int row = blockIdx.x * blockDim.x + threadIdx.x, l = blockIdx.y, b = blockIdx.z;
  if (row >= n) return;
  const Fp beta = chal[(long long)b * chal_stride + beta_slot], gamma = chal[(long long)b * chal_stride + gamma_slot];
  size_t o = (size_t)b * pstride + (size_t)l * n + row;
  st_fe(den + o, lookup_factor(ld_fe(Ap + o), ld_fe(Sp + o), beta, gamma));
  st_fe(num + o, lookup_factor(ld_fe(A + o), ld_fe(S + o), beta, gamma));
}
void lookup_fractions(Ctx* c, const Fp* A, const Fp* S, const Fp* Ap, const Fp* Sp, Fp* num, Fp* den, long long pstride, int L, int n,
                      const Fp* chal, long long chal_stride, int beta_slot, int gamma_slot, int B) {
  if (!L) return;
  launch(c, lookup_fractions_kernel, dim3((n + 255) / 256, L, B), 256, 0, A, S, Ap, Sp, num, den, pstride, n, chal, chal_stride, beta_slot, gamma_slot);
}

}  // namespace tb
