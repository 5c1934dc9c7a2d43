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
// Scratch of one (context, batch size) pair: device blocks in request order and the small tables uploaded on first use.
// A tb_pk may be shared by several contexts (= host threads); each gets its own workspace, and a second thread entering
// with the SAME context and batch size while a call is in flight is refused (TB_ERR_INVALID) instead of corrupting it.
struct ProveWs { std::vector<DevMem<uint8_t>> blocks, tables; std::vector<std::vector<uint8_t>> table_bytes; std::atomic<int> busy{0}; };

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
  explicit Circuit(Shape&& s) : Shape(std::move(s)) {}
  // the workspace of (context, batch size), marked busy; nullptr if a call is already using it.  Claiming under the lock
  // lets release_idle() free every workspace that is not marked.
  ProveWs* claim_workspace(const Ctx* c, int B) const {
    std::lock_guard<std::mutex> lk(mu);
    auto& slot = ws[std::make_pair(c, B)];
    if (!slot) slot.reset(new ProveWs());
    return slot->busy.exchange(1) == 0 ? slot.get() : nullptr;
  }
  // Out of device memory on `device` (the calling context's): frees the workspaces no call is using (other batch sizes, other
  // contexts) and what the stream-ordered pool keeps cached, so that scratch kept for earlier calls does not make a new batch size fail.
  void release_idle(int device) const {
    TB_CUDA(cudaDeviceSynchronize());
    {
      std::lock_guard<std::mutex> lk(mu);
      for (auto it = ws.begin(); it != ws.end();) {
        if (it->second->busy.load() != 0) { ++it; continue; }
        it = ws.erase(it);
      }
    }
    cudaMemPool_t pool;
    TB_CUDA(cudaDeviceGetDefaultMemPool(&pool, device));
    TB_CUDA(cudaMemPoolTrimTo(pool, 0));
  }
};

// tb_vk: what Proof::verify needs of a circuit.  The commitments are Montgomery affine points, the identity (0, 0).
struct VerifyingKey {
  Shape shape;
  const Srs* srs;
  std::vector<Aff<Fq>> fixed, sigma;
};

}  // namespace tb
