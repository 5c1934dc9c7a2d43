// Device-resident structured reference string with fixed-base window tables.
// Replaces halo2_proofs `poly::commitment::Params<vesta::Affine>` (EXT) as loaded by SETUP_PARAMS_MAP
// (taiga_halo2/src/constant.rs:128-139) and its `commit` / `commit_lagrange` methods (SURVEY.md §8a H1, App. E.4).
#pragma once
#include <memory>
#include "common.cuh"
#include "kernels.cuh"

namespace tb {

struct Srs {
  uint32_t k = 0; size_t n = 0;
  int c = 13, W = 20;                       // fixed-base window bits / number of table windows
  DevMem<Aff<Fq>> g;                         // [n]   (device, Montgomery)
  DevMem<Aff<Fq>> g_lagrange;                // [n]
  DevMem<Aff<Fq>> tab_g;                     // [W][n+2]  2^(c*w) * {g[0..n), w, u}
  DevMem<Aff<Fq>> tab_gl;                    // [W][n+2]  same with g_lagrange
  DevMem<Aff<Fq>> wu;                        // [2] = {w, u}
  Aff<Fq> w_host, u_host;                    // Montgomery

  static Srs* load(Ctx* ctx, uint32_t k, const uint8_t* g, const uint8_t* gl, const uint8_t* w, const uint8_t* u) {
    std::unique_ptr<Srs> s(new Srs());
    s->k = k; s->n = size_t(1) << k;
    // 13 at k = 15: 4096 buckets per MSM, 20 table windows (measured best of 11/12/13/16 at k = 15)
    int c = (int)k - 2; if (c < 4) c = 4; if (c > 13) c = 13;
    s->c = c; s->W = (256 + c - 1) / c;
    size_t n = s->n;
    s->g = DevMem<Aff<Fq>>(n);
    s->g_lagrange = DevMem<Aff<Fq>>(n);
    s->tab_g = DevMem<Aff<Fq>>((size_t)s->W * (n + 2));
    s->tab_gl = DevMem<Aff<Fq>>((size_t)s->W * (n + 2));
    s->wu = DevMem<Aff<Fq>>(2);
    TB_CUDA(cudaMemcpyAsync(s->g.get(), g, n * 64, cudaMemcpyHostToDevice, ctx->stream));
    TB_CUDA(cudaMemcpyAsync(s->g_lagrange.get(), gl, n * 64, cudaMemcpyHostToDevice, ctx->stream));
    TB_CUDA(cudaMemcpyAsync(s->wu.get(), w, 64, cudaMemcpyHostToDevice, ctx->stream));
    TB_CUDA(cudaMemcpyAsync(s->wu.get() + 1, u, 64, cudaMemcpyHostToDevice, ctx->stream));
    fe_to_mont<Fq>(ctx, reinterpret_cast<Fq*>(s->g.get()), 2 * n);
    fe_to_mont<Fq>(ctx, reinterpret_cast<Fq*>(s->g_lagrange.get()), 2 * n);
    fe_to_mont<Fq>(ctx, reinterpret_cast<Fq*>(s->wu.get()), 4);
    { // window 0 of each table: the basis followed by w and u (the extra terms every commitment / IPA round adds)
      DevBuf<Aff<Fq>> b0(ctx, n + 2);
      for (int t = 0; t < 2; ++t) {
        TB_CUDA(cudaMemcpyAsync(b0.get(), (t ? s->g_lagrange : s->g).get(), n * sizeof(Aff<Fq>), cudaMemcpyDeviceToDevice, ctx->stream));
        TB_CUDA(cudaMemcpyAsync(b0.get() + n, s->wu.get(), 2 * sizeof(Aff<Fq>), cudaMemcpyDeviceToDevice, ctx->stream));
        msm_build_tables<Fq>(ctx, b0.get(), (int)n + 2, c, s->W, (t ? s->tab_gl : s->tab_g).get());
      }
    }
    Aff<Fq> h[2];
    TB_CUDA(cudaMemcpyAsync(h, s->wu.get(), sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
    ctx->sync();
    s->w_host = h[0]; s->u_host = h[1];
    return s.release();
  }

  // acc[k] = MSM(scalars_k, basis) + sum_j extras[k][j] * {w, u}[j] via the fixed-base tables (no normalisation)
  void commit_xyzz(Ctx* c_, bool lagrange, const Fp* scalars, long long stride, int K, const Fp* extras, int n_extra, Xyzz<Fq>* acc,
                   Aff<Fq>* affine_out = nullptr) const {
    MsmConfig cfg; cfg.c = c; cfg.table_windows = W; cfg.table_stride = (int)n + 2; cfg.n_extra = extras ? n_extra : 0; cfg.extra_scalars = extras;
    cfg.affine_out = affine_out;
    msm_run<Fq, Fp>(c_, scalars, stride, (lagrange ? tab_gl : tab_g).get(), 0, (int)n, K, cfg, acc);
  }
  // out[k] = affine(MSM(scalars_k, basis) + blinds[k] * w)      (Params::commit / commit_lagrange)
  void commit(Ctx* c_, bool lagrange, const Fp* scalars, long long stride, int K, const Fp* blinds, Aff<Fq>* out) const {
    DevBuf<Xyzz<Fq>> acc(c_, K);
    commit_xyzz(c_, lagrange, scalars, stride, K, blinds, 1, acc.get(), out);
  }
};

}  // namespace tb
