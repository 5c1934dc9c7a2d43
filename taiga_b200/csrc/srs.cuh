// Device-resident structured reference string with fixed-base window tables.
// Replaces halo2_proofs `poly::commitment::Params<vesta::Affine>` (EXT) as loaded by SETUP_PARAMS_MAP
// (taiga_halo2/src/constant.rs:128-139) and its `commit` / `commit_lagrange` methods (SURVEY.md §8a H1, App. E.4).
#pragma once
#include "common.cuh"
#include "kernels.cuh"

namespace tb {

struct Srs {
  Ctx* ctx = nullptr;
  uint32_t k = 0; size_t n = 0;
  int c = 13, W = 20;                       // fixed-base window bits / number of table windows
  Aff<Fq>* g = nullptr;                      // [n]   (device, Montgomery)
  Aff<Fq>* g_lagrange = nullptr;             // [n]
  Aff<Fq>* tab_g = nullptr;                  // [W][n+2]  2^(c*w) * {g[0..n), w, u}
  Aff<Fq>* tab_gl = nullptr;                 // [W][n+2]  same with g_lagrange
  Aff<Fq>* wu = nullptr;                     // [2] = {w, u}
  Aff<Fq> w_host, u_host;                    // Montgomery

  static Srs* load(Ctx* ctx, uint32_t k, const uint8_t* g, const uint8_t* gl, const uint8_t* w, const uint8_t* u) {
    Srs* s = new Srs();
    s->ctx = ctx; s->k = k; s->n = size_t(1) << k;
    // 13 at k = 15: 4096 buckets per MSM, 20 table windows (measured best of 11/12/13/16 at k = 15)
    int c = (int)k - 2; if (c < 4) c = 4; if (c > 13) c = 13;
    s->c = c; s->W = (256 + c - 1) / c;
    size_t n = s->n;
    try {
      TB_CUDA(cudaMalloc(&s->g, n * sizeof(Aff<Fq>)));
      TB_CUDA(cudaMalloc(&s->g_lagrange, n * sizeof(Aff<Fq>)));
      TB_CUDA(cudaMalloc(&s->tab_g, (size_t)s->W * (n + 2) * sizeof(Aff<Fq>)));
      TB_CUDA(cudaMalloc(&s->tab_gl, (size_t)s->W * (n + 2) * sizeof(Aff<Fq>)));
      TB_CUDA(cudaMalloc(&s->wu, 2 * sizeof(Aff<Fq>)));
      TB_CUDA(cudaMemcpyAsync(s->g, g, n * 64, cudaMemcpyHostToDevice, ctx->stream));
      TB_CUDA(cudaMemcpyAsync(s->g_lagrange, gl, n * 64, cudaMemcpyHostToDevice, ctx->stream));
      TB_CUDA(cudaMemcpyAsync(s->wu, w, 64, cudaMemcpyHostToDevice, ctx->stream));
      TB_CUDA(cudaMemcpyAsync(s->wu + 1, u, 64, cudaMemcpyHostToDevice, ctx->stream));
      fe_to_mont<Fq>(ctx, reinterpret_cast<Fq*>(s->g), 2 * n);
      fe_to_mont<Fq>(ctx, reinterpret_cast<Fq*>(s->g_lagrange), 2 * n);
      fe_to_mont<Fq>(ctx, reinterpret_cast<Fq*>(s->wu), 4);
      { // window 0 of each table: the basis followed by w and u (the extra terms every commitment / IPA round adds)
        DevBuf<Aff<Fq>> b0(ctx, n + 2);
        for (int t = 0; t < 2; ++t) {
          TB_CUDA(cudaMemcpyAsync(b0.get(), t ? s->g_lagrange : s->g, n * sizeof(Aff<Fq>), cudaMemcpyDeviceToDevice, ctx->stream));
          TB_CUDA(cudaMemcpyAsync(b0.get() + n, s->wu, 2 * sizeof(Aff<Fq>), cudaMemcpyDeviceToDevice, ctx->stream));
          msm_build_tables<Fq>(ctx, b0.get(), (int)n + 2, c, s->W, t ? s->tab_gl : s->tab_g);
        }
      }
      Aff<Fq> h[2];
      TB_CUDA(cudaMemcpyAsync(h, s->wu, sizeof(h), cudaMemcpyDeviceToHost, ctx->stream));
      ctx->sync();
      s->w_host = h[0]; s->u_host = h[1];
    } catch (...) { delete s; throw; }
    return s;
  }
  ~Srs() { cudaFree(g); cudaFree(g_lagrange); cudaFree(tab_g); cudaFree(tab_gl); cudaFree(wu); }

  // acc[k] = MSM(scalars_k, basis) + sum_j extras[k][j] * {w, u}[j] via the fixed-base tables (no normalisation)
  void commit_xyzz(Ctx* c_, bool lagrange, const Fp* scalars, long long stride, int K, const Fp* extras, int n_extra, Xyzz<Fq>* acc,
                   Aff<Fq>* affine_out = nullptr) const {
    MsmConfig cfg; cfg.c = c; cfg.table_windows = W; cfg.table_stride = (int)n + 2; cfg.n_extra = extras ? n_extra : 0; cfg.extra_scalars = extras;
    cfg.affine_out = affine_out;
    msm_run<Fq, Fp>(c_, scalars, stride, lagrange ? tab_gl : tab_g, 0, (int)n, K, cfg, acc);
  }
  // out[k] = affine(MSM(scalars_k, basis) + blinds[k] * w)      (Params::commit / commit_lagrange)
  void commit(Ctx* c_, bool lagrange, const Fp* scalars, long long stride, int K, const Fp* blinds, Aff<Fq>* out) const {
    DevBuf<Xyzz<Fq>> acc(c_, K);
    commit_xyzz(c_, lagrange, scalars, stride, K, blinds, 1, acc.get(), out);
  }
};

}  // namespace tb
