// Permutation / lookup terms of the quotient, the size-R cross transform of extended_to_coeff and the grand-product
// helpers (second half of the h(X) construction; see quotient.cu for the gate interpreter).  These kernels have many
// distinct multiply sites, so the field multiply is called out of line here (instruction-cache footprint).
#define TB_NOINLINE_MUL 1
#include "common.cuh"
#include "prover_kernels.cuh"

namespace tb {

// ---------------------------------------------------------------- permutation + lookup terms, vanishing division
__global__ void __launch_bounds__(128) q_finish_kernel(QFinish f) {
  const int row = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
  if (row >= f.n) return;
  const int n = f.n, nm = n - 1;
  const Fp* chal = f.chal + (long long)b * f.chal_stride;
  const Fp y = chal[f.y_slot], beta = chal[f.beta_slot], gamma = chal[f.gamma_slot];
  const Fp one = Fp::one();
  const size_t crow = (size_t)f.k1 * n + row;
  Fp acc = Fp::zero();   // gate programs: sum_p y^(J - 1 - last_p) S_p
  for (int p = 0; p < f.nparts; ++p) acc = acc + chal[f.ytab_slot + f.gexp[p]] * ldg_fe(f.gate + (size_t)p * f.gate_part_stride + (size_t)b * n + row);
  const Fp l0 = ldg_fe(f.l0 + crow), ll = ldg_fe(f.l_last + crow);
  const Fp active = one - (ll + ldg_fe(f.l_blind + crow));
  const Fp* adv = f.adv + (long long)b * f.adv_pstride;
  const Fp* inst = f.inst + (long long)b * f.inst_pstride;
  if (f.nsets) {
    const Fp* pz = f.pz + (long long)b * f.pz_pstride;
    const int last_rot = -(f.bf + 1);
    acc = acc * y + l0 * (one - ldg_fe(pz + row));
    { Fp zl = ldg_fe(pz + (size_t)(f.nsets - 1) * n + row); acc = acc * y + ll * (zl * zl - zl); }
    for (int s = 1; s < f.nsets; ++s)
      acc = acc * y + l0 * (ldg_fe(pz + (size_t)s * n + row) - ldg_fe(pz + (size_t)(s - 1) * n + ((row + last_rot + n) & nm)));
    // X on this sub-coset: zeta * w_ext^(k1 + R*row)
    Fp xcur = f.zeta * tw_pow(f.tw, (uint32_t)(f.k1 + f.R * row) << (TW_LOG - f.ext_k));
    for (int s = 0; s < f.nsets; ++s) {
      int c0 = s * f.chunk, c1 = c0 + f.chunk < f.P ? c0 + f.chunk : f.P;
      Fp left = ldg_fe(pz + (size_t)s * n + ((row + 1) & nm)), right = ldg_fe(pz + (size_t)s * n + row);
      Fp cd = beta * f.delta_c0[s] * xcur;
      for (int cidx = c0; cidx < c1; ++cidx) {
        int2 col = f.perm_cols[cidx];
        Fp val = col.x == TB_COL_ADVICE ? ldg_fe(adv + (size_t)col.y * n + row)
               : col.x == TB_COL_FIXED ? ldg_fe(f.fix + ((size_t)col.y * f.R + f.k1) * n + row) : ldg_fe(inst + (size_t)col.y * n + row);
        left = left * (val + beta * ldg_fe(f.sig + ((size_t)cidx * f.R + f.k1) * n + row) + gamma);
        right = right * (val + cd + gamma);
        cd = cd * f.delta;
      }
      acc = acc * y + (left - right) * active;
    }
  }
  for (int l = 0; l < f.L; ++l) {
    size_t o = (size_t)b * f.lk_pstride + (size_t)l * n, oc = (size_t)b * f.lkc_pstride + (size_t)l * n;
    Fp z = ldg_fe(f.lz + o + row), zn = ldg_fe(f.lz + o + ((row + 1) & nm));
    Fp ap = ldg_fe(f.lpin + o + row), apm = ldg_fe(f.lpin + o + ((row - 1 + n) & nm)), sp = ldg_fe(f.lptab + o + row);
    Fp a = ldg_fe(f.lkA + oc + row), t = ldg_fe(f.lkS + oc + row);
    acc = acc * y + l0 * (one - z);
    acc = acc * y + ll * (z * z - z);
    acc = acc * y + (zn * (ap + beta) * (sp + gamma) - z * (a + beta) * (t + gamma)) * active;
    acc = acc * y + l0 * (ap - sp);
    acc = acc * y + (ap - sp) * (ap - apm) * active;
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
  const Fp* adv = p.adv + (long long)b * p.adv_pstride;
  const Fp* inst = p.inst + (long long)b * p.inst_pstride;
  int c0 = s * p.chunk, c1 = c0 + p.chunk < p.P ? c0 + p.chunk : p.P;
  Fp num = Fp::one(), den = Fp::one();
  Fp dw = p.delta_c0[s] * tw_pow(p.tw, (uint32_t)row << (TW_LOG - p.k)) * beta;  // delta^c * omega^row * beta
  for (int cidx = c0; cidx < c1; ++cidx) {
    int2 col = p.perm_cols[cidx];
    Fp val = col.x == TB_COL_ADVICE ? ldg_fe(adv + (size_t)col.y * n + row)
           : col.x == TB_COL_FIXED ? ldg_fe(p.fix + (size_t)col.y * n + row) : ldg_fe(inst + (size_t)col.y * n + row);
    den = den * (beta * ldg_fe(p.sig + (size_t)cidx * n + row) + gamma + val);
    num = num * (dw + gamma + val);
    dw = dw * p.delta;
  }
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
  st_fe(den + o, (beta + ld_fe(Ap + o)) * (gamma + ld_fe(Sp + o)));
  st_fe(num + o, (ld_fe(A + o) + beta) * (ld_fe(S + o) + gamma));
}
void lookup_fractions(Ctx* c, const Fp* A, const Fp* S, const Fp* Ap, const Fp* Sp, Fp* num, Fp* den, long long pstride, int L, int n,
                      const Fp* chal, long long chal_stride, int beta_slot, int gamma_slot, int B) {
  if (!L) return;
  launch(c, lookup_fractions_kernel, dim3((n + 255) / 256, L, B), 256, 0, A, S, Ap, Sp, num, den, pstride, n, chal, chal_stride, beta_slot, gamma_slot);
}

}  // namespace tb
