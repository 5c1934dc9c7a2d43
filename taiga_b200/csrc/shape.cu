// The shape of a circuit (circuit.cuh): everything tb_circuit_load and tb_vk_load derive from a tb_cs_desc, on the host.
#include <algorithm>
#include <map>
#include <set>
#include "circuit.cuh"

namespace tb {

Shape shape_build(const tb_cs_desc* cs, uint32_t srs_k, bool allow_split) {
  TB_REQUIRE(cs->k == srs_k, "circuit k must match the SRS");
  gate_desc_check(cs);
  Shape C;
  C.k = cs->k; C.n = size_t(1) << C.k; C.na = cs->num_advice; C.nf = cs->num_fixed; C.ni = cs->num_instance; C.degree = cs->cs_degree; C.bf = cs->blinding_factors;
  TB_REQUIRE(C.n > C.bf + 2, "too few rows");
  C.usable = C.n - (C.bf + 1);
  C.P = cs->num_perm_columns; C.L = cs->num_lookups; C.chunk = C.degree - 2; C.nsets = C.P ? (C.P + C.chunk - 1) / C.chunk : 0;
  C.pieces = C.degree - 1;
  C.ext_k = C.k; while ((size_t(1) << C.ext_k) < C.n * C.pieces) C.ext_k++;
  TB_REQUIRE(C.ext_k <= TW_LOG, "extended domain too large");
  C.R = 1 << (C.ext_k - C.k);
  C.aq.assign(cs->advice_queries, cs->advice_queries + cs->num_advice_queries);
  C.fq.assign(cs->fixed_queries, cs->fixed_queries + cs->num_fixed_queries);
  C.iq.assign(cs->instance_queries, cs->instance_queries + cs->num_instance_queries);
  C.perm.assign(cs->perm_columns, cs->perm_columns + C.P);
  memcpy(C.vk_repr.l, cs->vk_transcript_repr, 32);

  C.delta = delta_const<Fp>(); C.zeta = zeta_const<Fp>(); C.omega = omega_k<Fp>((int)C.k);
  C.r_inv = Fp::from_u32((uint32_t)C.R).inv();
  for (int s = 0; s < PERM_MAX_SETS; ++s) C.delta_c0[s] = C.delta.pow_u64((uint64_t)s * C.chunk);
  { Fp zn = C.zeta.pow_u64(C.n), step = omega_k<Fp>(C.ext_k).pow_u64(C.n), cur = zn;
    for (int k1 = 0; k1 < C.R; ++k1) { C.t_inv.push_back((cur - Fp::one()).inv()); cur = cur * step; } }
  // constants -> Montgomery
  for (uint32_t i = 0; i < cs->num_constants; ++i) { Fp v; memcpy(v.l, cs->constants + 32 * (size_t)i, 32); C.consts_host.push_back(v.to_mont()); }
  C.plan = gate_plan(cs, C.R, allow_split);

  // ---- evaluation section order (plonk/prover.rs) and multiopen query order
  int last_rot = -(int)(C.bf + 1);
  for (auto& q : C.iq) C.evals.push_back({{PK_INST, (int)q.column}, q.rotation});
  for (auto& q : C.aq) C.evals.push_back({{PK_ADV, (int)q.column}, q.rotation});
  for (auto& q : C.fq) C.evals.push_back({{PK_FIXED, (int)q.column}, q.rotation});
  C.evals.push_back({{PK_RANDOM, 0}, 0});
  for (uint32_t c = 0; c < C.P; ++c) C.evals.push_back({{PK_SIG, (int)c}, 0});
  for (uint32_t s = 0; s < C.nsets; ++s) {
    C.evals.push_back({{PK_PZ, (int)s}, 0}); C.evals.push_back({{PK_PZ, (int)s}, 1});
    if (s + 1 < C.nsets) C.evals.push_back({{PK_PZ, (int)s}, last_rot});
  }
  for (uint32_t l = 0; l < C.L; ++l) {
    C.evals.push_back({{PK_LZ, (int)l}, 0}); C.evals.push_back({{PK_LZ, (int)l}, 1}); C.evals.push_back({{PK_LPIN, (int)l}, 0});
    C.evals.push_back({{PK_LPIN, (int)l}, -1}); C.evals.push_back({{PK_LPTAB, (int)l}, 0});
  }
  for (size_t i = 0; i < C.evals.size(); ++i) C.eval_pos[{C.evals[i].poly, C.evals[i].rot}] = (int)i;
  C.eval_pos[{{PK_H, 0}, 0}] = (int)C.evals.size();
  // the permutation argument reads every column at X: without that query its copy constraints would not bind the column
  for (uint32_t c = 0; c < C.P; ++c) {
    static const char* kinds[] = {"advice", "fixed", "instance"};
    TB_REQUIRE(C.eval_pos.count({column_poly(C.perm[c]), 0}), "permutation column " + std::to_string(c) + " (" + kinds[C.perm[c].kind] + " column " +
               std::to_string(C.perm[c].index) + ") has no rotation-0 query");
  }
  for (auto& q : C.iq) C.queries.push_back({{PK_INST, (int)q.column}, q.rotation});
  for (auto& q : C.aq) C.queries.push_back({{PK_ADV, (int)q.column}, q.rotation});
  for (uint32_t s = 0; s < C.nsets; ++s) { C.queries.push_back({{PK_PZ, (int)s}, 0}); C.queries.push_back({{PK_PZ, (int)s}, 1}); }
  for (int s = (int)C.nsets - 1; s >= 0; --s) if (s + 1 < (int)C.nsets) C.queries.push_back({{PK_PZ, s}, last_rot});
  for (uint32_t l = 0; l < C.L; ++l) {
    C.queries.push_back({{PK_LZ, (int)l}, 0}); C.queries.push_back({{PK_LPIN, (int)l}, 0}); C.queries.push_back({{PK_LPTAB, (int)l}, 0});
    C.queries.push_back({{PK_LPIN, (int)l}, -1}); C.queries.push_back({{PK_LZ, (int)l}, 1});
  }
  for (auto& q : C.fq) C.queries.push_back({{PK_FIXED, (int)q.column}, q.rotation});
  for (uint32_t c = 0; c < C.P; ++c) C.queries.push_back({{PK_SIG, (int)c}, 0});
  C.queries.push_back({{PK_H, 0}, 0});
  C.queries.push_back({{PK_RANDOM, 0}, 0});
  // multiopen::construct_intermediate_sets (points identified by rotation; sets ordered by first appearance)
  { std::map<int, int> point_index; std::vector<std::set<int>> prots;
    for (auto& q : C.queries) {
      if (!point_index.count(q.rot)) { int idx = (int)point_index.size(); point_index[q.rot] = idx; C.rots.push_back(q.rot); }
      size_t pos = 0; for (; pos < C.uniq.size(); ++pos) if (C.uniq[pos] == q.poly) break;
      if (pos == C.uniq.size()) { C.uniq.push_back(q.poly); prots.emplace_back(); }
      prots[pos].insert(point_index[q.rot]);
    }
    std::map<std::set<int>, int> set_index;
    for (size_t c = 0; c < C.uniq.size(); ++c) {
      if (!set_index.count(prots[c])) { int idx = (int)set_index.size(); set_index[prots[c]] = idx; }
      C.uniq_set.push_back(set_index[prots[c]]);
    }
    C.point_sets.resize(set_index.size());
    for (auto& kv : set_index) for (int pi : kv.first) C.point_sets[kv.second].push_back(C.rots[pi]); }
  for (auto& e : C.evals) if (std::find(C.rots.begin(), C.rots.end(), e.rot) == C.rots.end()) C.rots.push_back(e.rot);
  // ---- proof layout: the commitments, the evaluations, q', the multiopen evaluations u, S, then k (L, R) pairs and (c, f)
  const uint32_t commits = C.na + 3 * C.L + C.nsets + 1 + C.pieces, nevals = (uint32_t)C.evals.size(), nps = (uint32_t)C.point_sets.size();
  for (uint32_t i = 0; i < commits; ++i) C.point_offsets.push_back(32 * i);
  C.point_offsets.push_back(32 * (commits + nevals));
  C.point_offsets.push_back(32 * (commits + nevals + 1 + nps));
  for (uint32_t j = 0; j < 2 * C.k; ++j) C.point_offsets.push_back(32 * (commits + nevals + 2 + nps + j));
  C.proof_len = 32 * (commits + nevals + 1 + nps + 1 + 2 * C.k + 2);
  return C;
}

}  // namespace tb
