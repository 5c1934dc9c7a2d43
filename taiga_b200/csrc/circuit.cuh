// What the prover and the verifier know of one circuit: its shape (host only, derived from the tb_cs_desc), the
// device-resident proving key built on it (tb_pk), and the verifying key (tb_vk: the shape plus the fixed and sigma
// commitments).  Shared by shape.cu, prover.cu and verifier.cu.
#pragma once
#include <atomic>
#include <map>
#include <mutex>
#include <set>
#include <memory>
#include <vector>
#include "prover_kernels.cuh"

namespace tb {

enum PolyKind { PK_INST = 0, PK_ADV, PK_PZ, PK_LZ, PK_LPIN, PK_LPTAB, PK_FIXED, PK_SIG, PK_H, PK_RANDOM };
struct PolyId { int kind, idx; bool operator<(const PolyId& o) const { return kind != o.kind ? kind < o.kind : idx < o.idx; } bool operator==(const PolyId& o) const { return kind == o.kind && idx == o.idx; } };
struct QueryRef { PolyId poly; int rot; };
inline PolyId column_poly(const tb_column& col) { return {col.kind == TB_COL_ADVICE ? PK_ADV : col.kind == TB_COL_FIXED ? PK_FIXED : PK_INST, (int)col.index}; }
// Scratch of one (context, batch size) pair: device blocks in request order and the small tables uploaded on first use.
// A tb_pk may be shared by several contexts (= host threads); each gets its own workspace, and a second thread entering
// with the SAME context and batch size while a call is in flight is refused (TB_ERR_INVALID) instead of corrupting it.
// `busy` covers the host call only.  A device call (tb_dev_prove_batch) returns with its work still queued: `idle` is recorded
// on the context's stream after that work, and the workspace is not freed before it has completed.  Two calls on the same
// context need no more than that (stream order keeps them apart); a host call waits for its stream, so `idle` has then passed.
struct ProveWs {
  std::vector<DevMem<uint8_t>> blocks, tables; std::vector<std::vector<uint8_t>> table_bytes; std::atomic<int> busy{0};
  Ctx::Event idle;
};

// Everything the description fixes, built once by shape_build: sizes, domain constants, the compiled programs and the
// order of the proof's elements.  Host memory only and nothing per row, so a verifying key costs kilobytes.
struct Shape {
  uint32_t k, na, nf, ni, degree, bf, P, L, chunk, nsets, pieces; int ext_k, R; size_t n, usable;
  std::vector<tb_query> aq, fq, iq; std::vector<tb_column> perm;
  std::vector<Fp> consts_host;   // the constants (Montgomery) the gate programs read
  Fp vk_repr;  // canonical
  GatePlan plan;                 // the programs of gate_plan (gates.cuh)
  std::vector<Fp> t_inv; Fp delta, zeta, omega, r_inv;
  Fp delta_c0[PERM_MAX_SETS];
  // evaluation / multiopen structure
  std::vector<QueryRef> evals;            // transcript order of the evaluation section
  // (poly, rotation) -> its position in `evals` (the last one, should a query repeat); (PK_H, 0) -> evals.size(), where the
  // verifier keeps the h(x) it expects.  Every permutation column has its rotation-0 query (shape_build refuses it otherwise).
  std::map<std::pair<PolyId, int>, int> eval_pos;
  int eval_index(const PolyId& poly, int rot) const {
    auto it = eval_pos.find({poly, rot});
    if (it == eval_pos.end()) throw std::logic_error("internal error: a query without an evaluation");
    return it->second;
  }
  std::vector<QueryRef> queries;          // multiopen query order
  std::vector<int> rots;                  // distinct rotations (evaluation points), in order of first appearance in `queries`
  std::vector<PolyId> uniq; std::vector<int> uniq_set; std::vector<std::vector<int>> point_sets;
  uint32_t proof_len;
  std::vector<uint32_t> point_offsets;    // byte offset of every point of a proof, in transcript order
};
// checks the description (gate_desc_check, k == srs_k) and derives its shape; `allow_split`: the quotient's degree split
Shape shape_build(const tb_cs_desc* cs, uint32_t srs_k, bool allow_split);

struct Circuit : Shape {
  const Srs* srs;
  // device tables
  DevMem<Fp> fixed_vals, fixed_polys, fixed_cosets, sig_vals, sig_polys, sig_cosets;
  DevMem<Fp> l0, l_last, l_blind, consts, wr_inv;
  DevMem<Fp> coset_pre;   // [R][n]: zeta^(i mod 3) * w_ext^(i * k1), the factor the forward coset NTT applies to coefficient i for sub-coset k1
  DevMem<int2> d_perm;
  // the programs of `plan` with their device copies
  QProgram prog_lookups;
  std::vector<QProgram> gate_parts[2], gate_parts_lo[2];
  // persistent per-batch-size workspace and cached small tables (see prove_batch)
  mutable std::mutex mu;                                                   // guards the two caches below
  mutable std::map<std::pair<const Ctx*, int>, std::unique_ptr<ProveWs>> ws;
  mutable std::vector<Aff<Fq>> vk_fixed, vk_sigma;   // verifying-key commitments (Montgomery, host), filled on first verification
  // what tb_check_batch adds, built on its first call (check.cu): the sigma-successor of every permutation cell as a cell index
  // q * n + r ([P][n]), and the one-constraint programs of plan.single concatenated, with (offset, instructions) per constraint
  mutable DevMem<uint32_t> sig_next;
  mutable DevMem<QInstr> single_code; mutable DevMem<int2> single_table; mutable int single_nregs = 0; mutable bool check_ready = false;
  explicit Circuit(Shape&& s) : Shape(std::move(s)) {}
  // tb_pk_free: the workspaces' device calls may still be queued; their memory is freed only after each has completed
  ~Circuit() {
    for (auto& w : ws) try { w.second->idle.wait(); } catch (const CudaError&) {}
  }
  // the workspace of (context, batch size), marked busy; nullptr if a call is already using it.  Claiming under the lock
  // lets release_idle() free every workspace that is not marked.  Checks (`check`) keep workspaces apart from proofs: their
  // buffers differ, and sharing would reallocate on every switch between the two.
  ProveWs* claim_workspace(const Ctx* c, int B, bool check = false) const {
    std::lock_guard<std::mutex> lk(mu);
    auto& slot = ws[std::make_pair(c, check ? -B : B)];
    if (!slot) slot.reset(new ProveWs());
    return slot->busy.exchange(1) == 0 ? slot.get() : nullptr;
  }
  // Out of device memory on `device` (the calling context's): frees the workspaces no call is using (other batch sizes, other
  // contexts) and what the stream-ordered pool keeps cached, so that scratch kept for earlier calls does not make a new batch size fail.
  // A workspace whose last device call is still queued or running is kept: `busy` is cleared only after `idle` is recorded, so
  // under the lock a workspace that is not busy has its last call's mark in `idle`.
  void release_idle(int device) const {
    TB_CUDA(cudaDeviceSynchronize());
    {
      std::lock_guard<std::mutex> lk(mu);
      for (auto it = ws.begin(); it != ws.end();) {
        if (it->second->busy.load() != 0 || !it->second->idle.done()) { ++it; continue; }
        it = ws.erase(it);
      }
    }
    cudaMemPool_t pool;
    TB_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
    TB_CUDA(cudaMemPoolTrimTo(pool, 0));
  }
};

// Persistent per-(circuit, batch size) device workspace: the same sequence of requests returns the same pointers on every
// call, so item tables / scalar programs that embed them are uploaded once and no allocation or host sync happens later.
template <class T> struct WBuf {
  T* p = nullptr; size_t n = 0; Ctx* ctx = nullptr;
  T* get() const { return p; }
  void zero() { TB_CUDA(cudaMemsetAsync(p, 0, n * sizeof(T), ctx->stream)); }
};
struct WsAlloc {
  Ctx* ctx; const Circuit& C; std::vector<DevMem<uint8_t>>& blocks; size_t cur = 0;
  template <class T> WBuf<T> buf(size_t count) {
    size_t bytes = std::max<size_t>(1, count) * sizeof(T);
    if (cur == blocks.size()) blocks.emplace_back();
    if (blocks[cur].size() < bytes) {   // try_alloc frees the smaller block first
      cudaError_t e = blocks[cur].try_alloc(bytes);
      if (e == cudaErrorMemoryAllocation) { cudaGetLastError(); C.release_idle(ctx->device); e = blocks[cur].try_alloc(bytes); }
      TB_CUDA(e);
    }
    WBuf<T> w; w.p = reinterpret_cast<T*>(blocks[cur].get()); w.n = count; w.ctx = ctx; ++cur;
    return w;
  }
};


// sum(instance_len); refuses an instance column longer than the usable rows (InstanceTooLarge)
size_t instance_total(const Shape& C, const uint32_t* instance_len);
// The instance columns of B proofs on the device in Montgomery form (Lagrange basis), [B][ni][n] zero past instance_len;
// `instance` (a host or device pointer) holds each proof's sum(instance_len) values column after column; refuses what
// instance_total refuses.  Shared by the prover, the check and the verifier.
void upload_instance(Ctx* ctx, const Shape& C, int B, const uint8_t* instance, const uint32_t* instance_len, Fp* dst);
// The witness of B proofs on the device in Montgomery form (Lagrange basis), shared by the prover and the check: the
// instance columns as upload_instance leaves them, advice [B][na][n] (host or device pointer) whose rows >= usable are
// overwritten with PRF(seed, proof0 + b, rows_tag, c * (bf + 1) + r - usable).
void upload_witness(Ctx* ctx, const Circuit& C, int B, const uint8_t* advice, const uint8_t* instance, const uint32_t* instance_len,
                    const uint8_t* seed, uint32_t proof0, uint32_t rows_tag, Fp* inst_vals, Fp* adv_vals);

// tb_vk: what Proof::verify needs of a circuit.  The commitments are Montgomery affine points, the identity (0, 0).
struct VerifyingKey {
  Shape shape;
  const Srs* srs;
  std::vector<Aff<Fq>> fixed, sigma;
};

}  // namespace tb
