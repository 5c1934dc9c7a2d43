// Elementwise field-vector kernels and small utilities (exclusive scan) for libtaiga_b200.
#define TB_NOINLINE_MUL 0  // loop-structured kernels: small code, keep the multiply inline
#include "common.cuh"
#include "kernels.cuh"

namespace tb {

template <class F, int DIR>
__global__ void fe_convert_kernel(F* v, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  F x = ld_fe(v + i);
  st_fe(v + i, DIR ? x.to_mont() : x.from_mont());
}
template <class F> void fe_to_mont(Ctx* ctx, F* v, size_t n) {
  if (!n) return;
  launch(ctx, fe_convert_kernel<F, 1>, (unsigned)((n + 255) / 256), 256, 0, v, n);
}
template <class F> void fe_from_mont(Ctx* ctx, F* v, size_t n) {
  if (!n) return;
  launch(ctx, fe_convert_kernel<F, 0>, (unsigned)((n + 255) / 256), 256, 0, v, n);
}
template void fe_to_mont<Fp>(Ctx*, Fp*, size_t);
template void fe_to_mont<Fq>(Ctx*, Fq*, size_t);
template void fe_from_mont<Fp>(Ctx*, Fp*, size_t);
template void fe_from_mont<Fq>(Ctx*, Fq*, size_t);

// ---------------------------------------------------------------- exclusive scan (u32)
constexpr int SCAN_THREADS = 256, SCAN_ITEMS = 8, SCAN_BLOCK = SCAN_THREADS * SCAN_ITEMS;

__global__ void __launch_bounds__(SCAN_THREADS) scan_block_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out,
                                                                   uint32_t* __restrict__ sums, size_t n) {
  __shared__ uint32_t warp_sums[SCAN_THREADS / 32];
  size_t base = (size_t)blockIdx.x * SCAN_BLOCK + (size_t)threadIdx.x * SCAN_ITEMS;
  uint32_t v[SCAN_ITEMS], local = 0;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) { v[i] = (base + i < n) ? in[base + i] : 0u; local += v[i]; }
  uint32_t incl = local;
  int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, d); if (lane >= d) incl += t; }
  if (lane == 31) warp_sums[warp] = incl;
  __syncthreads();
  if (warp == 0) {
    uint32_t w = lane < SCAN_THREADS / 32 ? warp_sums[lane] : 0u, wi = w;
#pragma unroll
    for (int d = 1; d < 8; d <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, wi, d); if (lane >= d) wi += t; }
    if (lane < SCAN_THREADS / 32) warp_sums[lane] = wi - w;  // exclusive warp offsets
    if (lane == SCAN_THREADS / 32 - 1) sums[blockIdx.x] = wi;
  }
  __syncthreads();
  uint32_t run = warp_sums[warp] + incl - local;
#pragma unroll
  for (int i = 0; i < SCAN_ITEMS; ++i) { if (base + i < n) out[base + i] = run; run += v[i]; }
}

__global__ void scan_add_kernel(uint32_t* __restrict__ out, const uint32_t* __restrict__ block_offs, size_t n) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] += block_offs[i / SCAN_BLOCK];
}

void exclusive_scan_u32(Ctx* ctx, const uint32_t* in, uint32_t* out, size_t n) {
  size_t nblocks = (n + SCAN_BLOCK - 1) / SCAN_BLOCK;
  if (nblocks == 0) { TB_CUDA(cudaMemsetAsync(out, 0, sizeof(uint32_t), ctx->stream)); return; }
  DevBuf<uint32_t> sums(ctx, nblocks);
  launch(ctx, scan_block_kernel, (unsigned)nblocks, SCAN_THREADS, 0, in, out, sums.get(), n);
  if (nblocks == 1) {
    TB_CUDA(cudaMemcpyAsync(out + n, sums.get(), sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
    return;
  }
  DevBuf<uint32_t> offs(ctx, nblocks + 1);
  exclusive_scan_u32(ctx, sums.get(), offs.get(), nblocks);
  launch(ctx, scan_add_kernel, (unsigned)((n + 255) / 256), 256, 0, out, offs.get(), n);
  TB_CUDA(cudaMemcpyAsync(out + n, offs.get() + nblocks, sizeof(uint32_t), cudaMemcpyDeviceToDevice, ctx->stream));
}

}  // namespace tb
