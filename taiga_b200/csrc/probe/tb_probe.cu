// libtaiga_b200_probe.so: plain C entry points over the prover's internal kernel drivers (polyops.cu, lookup.cu), so that the
// test-suite can run each of them on its own, at any size, against a big-integer reference (tests/test_gpu_poly_lookup.py).
//
// It is linked against libtaiga_b200.so and calls that library's compiled drivers; it launches nothing and allocates
// nothing itself.  Every pointer is a caller-owned device buffer in the driver's own layout (Montgomery form except where a
// driver says canonical), and every size and stride is passed through unchanged.  Not public ABI: include/taiga_b200.h
// does not declare these, and they may change with the drivers.
#include "../capi_internal.cuh"
#include "../prover_kernels.cuh"

using namespace tb;

#define FP(p) reinterpret_cast<Fp*>(p)
#define CFP(p) reinterpret_cast<const Fp*>(p)

extern "C" {

tb_status tbp_poly_fma(tb_ctx* ctx, void* out, long long out_stride, const void* s, long long s_stride, const void* in, long long in_stride, int n, int B) {
  TB_API_BEGIN(ctx) poly_fma(&ctx->c, FP(out), out_stride, CFP(s), s_stride, CFP(in), in_stride, n, B); TB_API_END(ctx)
}
tb_status tbp_poly_scale(tb_ctx* ctx, void* out, long long out_stride, const void* s, long long s_stride, const void* a, long long a_stride, int n, int B) {
  TB_API_BEGIN(ctx) poly_scale(&ctx->c, FP(out), out_stride, CFP(s), s_stride, CFP(a), a_stride, n, B); TB_API_END(ctx)
}
tb_status tbp_poly_copy(tb_ctx* ctx, void* out, long long out_stride, const void* in, long long in_stride, int n, int B) {
  TB_API_BEGIN(ctx) poly_copy(&ctx->c, FP(out), out_stride, CFP(in), in_stride, n, B); TB_API_END(ctx)
}
tb_status tbp_poly_add_at(tb_ctx* ctx, void* v, long long stride, int idx, const void* s, long long s_stride, int sign, int B) {
  TB_API_BEGIN(ctx) poly_add_at(&ctx->c, FP(v), stride, idx, CFP(s), s_stride, sign, B); TB_API_END(ctx)
}
// items: a device array of `nitems` EvalItem {const Fp* base; long long bstride; int point; int pad;}
tb_status tbp_poly_eval(tb_ctx* ctx, const void* items, int nitems, const void* points, long long pt_stride, void* evals, long long ev_stride, int n, int B) {
  TB_API_BEGIN(ctx)
  poly_eval(&ctx->c, reinterpret_cast<const EvalItem*>(items), nitems, CFP(points), pt_stride, FP(evals), ev_stride, n, B);
  TB_API_END(ctx)
}
tb_status tbp_poly_kate_div(tb_ctx* ctx, void* out, long long out_stride, const void* in, long long in_stride, const void* z, long long z_stride, int n, int B) {
  TB_API_BEGIN(ctx) poly_kate_div(&ctx->c, FP(out), out_stride, CFP(in), in_stride, CFP(z), z_stride, n, B); TB_API_END(ctx)
}
tb_status tbp_batch_inverse(tb_ctx* ctx, void* v, size_t count) {
  TB_API_BEGIN(ctx) batch_inverse(&ctx->c, FP(v), count); TB_API_END(ctx)
}
tb_status tbp_prefix_product(tb_ctx* ctx, void* out, const void* in, int n, int count) {
  TB_API_BEGIN(ctx) prefix_product(&ctx->c, FP(out), CFP(in), n, count); TB_API_END(ctx)
}
tb_status tbp_inner_product(tb_ctx* ctx, void* out, long long out_stride, const void* a, long long a_stride, const void* b, long long b_stride, int n, int B) {
  TB_API_BEGIN(ctx) inner_product(&ctx->c, FP(out), out_stride, CFP(a), a_stride, CFP(b), b_stride, n, B); TB_API_END(ctx)
}
tb_status tbp_powers(tb_ctx* ctx, void* out, long long out_stride, const void* x, long long x_stride, int n, int B) {
  TB_API_BEGIN(ctx) powers(&ctx->c, FP(out), out_stride, CFP(x), x_stride, n, B); TB_API_END(ctx)
}
// prog: a device array of `ninstr` ScalarInstr {uint16_t op, dst, a, b; uint32_t imm;}; consts: Montgomery
tb_status tbp_scalar_program(tb_ctx* ctx, void* vars, long long stride, const void* prog, int ninstr, const void* consts, int B) {
  TB_API_BEGIN(ctx)
  scalar_program(&ctx->c, FP(vars), stride, reinterpret_cast<const ScalarInstr*>(prog), ninstr, CFP(consts), B);
  TB_API_END(ctx)
}
// keys (canonical, rows >= usable set to the all-ones sentinel) from Montgomery values: `arrays` arrays of n
tb_status tbp_lookup_keys(tb_ctx* ctx, void* keys, const void* vals, int n, int usable, int arrays) {
  TB_API_BEGIN(ctx) lookup_keys(&ctx->c, FP(keys), CFP(vals), n, usable, arrays); TB_API_END(ctx)
}
tb_status tbp_sort_keys(tb_ctx* ctx, void* keys, int n, int arrays) {
  TB_API_BEGIN(ctx) sort_keys(&ctx->c, FP(keys), n, arrays); TB_API_END(ctx)
}
// err: one uint32 flag per array, set to 1 (never cleared) when the array's inputs are not all in its table
tb_status tbp_lookup_arrange(tb_ctx* ctx, const void* sorted_a, const void* sorted_t, void* scratch, void* s, int n, int usable, int arrays, void* err) {
  TB_API_BEGIN(ctx)
  lookup_arrange(&ctx->c, CFP(sorted_a), CFP(sorted_t), FP(scratch), FP(s), n, usable, arrays, reinterpret_cast<uint32_t*>(err));
  TB_API_END(ctx)
}
// the batch verifier's g-term (verifier.cu): G (2^kk scalars) += the terms of K proofs, us [K][kk], ab [K][2]
tb_status tbp_batch_g_scalars(tb_ctx* ctx, void* G, const void* us, const void* ab, int kk, int K) {
  TB_API_BEGIN(ctx) batch_g_scalars(&ctx->c, FP(G), CFP(us), CFP(ab), kk, K, K); TB_API_END(ctx)
}
// the same driver with the proofs in groups of `group` (1: the per-proof verifier's call): G [ceil(K / group)][2^kk]
tb_status tbp_batch_g_scalars_grouped(tb_ctx* ctx, void* G, const void* us, const void* ab, int kk, int K, int group) {
  TB_API_BEGIN(ctx) batch_g_scalars(&ctx->c, FP(G), CFP(us), CFP(ab), kk, K, group); TB_API_END(ctx)
}

}  // extern "C"
