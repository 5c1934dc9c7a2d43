// The gate and lookup expressions of a circuit compiled to register-allocated instruction lists (SURVEY.md App. E.6), and
// the one loop that runs them: on every sub-coset row in the quotient kernel (quotient.cu), at x in the host verifier
// (verifier.cu) and in the CPU tests (tests/host_shim.cpp, plain g++).  Callers pass a machine, as argument.cuh's views.
#pragma once
#include <vector>
#include "../../include/taiga_b200.h"
#include "argument.cuh"

namespace tb {

enum QOp { Q_MOV = 0, Q_NEG, Q_ADD, Q_SUB, Q_MUL, Q_FOLD_Y, Q_LK_BEGIN, Q_FOLD_A, Q_FOLD_S, Q_LK_STORE, Q_GBEGIN, Q_GFOLD, Q_GEND };
enum QKind { K_REG = 0, K_ADV, K_FIX, K_INST, K_CONST };
struct alignas(16) QInstr { uint32_t w0; uint32_t a, b, pad; };  // w0 = op | dst << 8 | akind << 16 | bkind << 24 (one 128-bit load)
inline QInstr q_make(int op, int dst, int ak, uint32_t a, int bk, uint32_t b) { QInstr i; i.w0 = op | (dst << 8) | (ak << 16) | (bk << 24); i.a = a; i.b = b; i.pad = 0; return i; }
constexpr int Q_MAX_PARTS = 8;

// Gate programs fold their constraints with y, gap-aware: program p yields S_p = sum_{j in p} y^(last_p - j) e_j, so any
// set of programs combines as sum_p y^(J - 1 - last_p) S_p, whatever subset of the J constraints each one holds.
struct GateProgram { std::vector<QInstr> code; int nregs = 0; int last = -1; };   // last: the last constraint it folds

// A constraint list is compiled as a sequence of ITEMS.  Consecutive constraints of one gate usually share their selector
// factor, root_j = S * X_j: since  acc <- acc * y + S * X_j  over such a run equals  acc * y^len + S * (Horner of the X_j in y),
// the run is evaluated as a group with len + 1 multiplications instead of 2 * len (the result is the same field element, so
// the proof bytes do not change).  A program may hold any subset of the constraints: every fold multiplies by y^(gap to the
// previous constraint of the program), read from a per-proof table of powers of y.
struct Item { bool group; uint32_t root; uint32_t S; std::vector<uint32_t> xs; std::vector<uint32_t> pos; };   // pos: constraint index of every element
inline std::vector<Item> build_items(const tb_cs_desc* cs, const std::vector<uint32_t>& idx) {
  std::vector<Item> items;
  auto factors = [&](uint32_t r, uint32_t* f) -> int { const tb_expr_node& nd = cs->nodes[r]; if (nd.op != TB_EX_MUL) return 0; f[0] = nd.a; f[1] = nd.b; return nd.a == nd.b ? 1 : 2; };
  size_t i = 0;
  while (i < idx.size()) {
    uint32_t f[2]; int nf = factors(cs->constraint_roots[idx[i]], f);
    size_t j = i + 1;
    while (nf && j < idx.size()) {
      uint32_t g[2]; int ng = factors(cs->constraint_roots[idx[j]], g);
      uint32_t keep[2]; int nk = 0;
      for (int x = 0; x < nf; ++x) for (int y = 0; y < ng; ++y) if (f[x] == g[y]) { keep[nk++] = f[x]; break; }
      if (!nk) break;
      nf = nk; f[0] = keep[0]; if (nk > 1) f[1] = keep[1];
      ++j;
    }
    Item it; it.S = 0; it.root = 0;
    if (j - i >= 2) {
      it.group = true; it.S = f[0];
      for (size_t q = i; q < j; ++q) { const tb_expr_node& nd = cs->nodes[cs->constraint_roots[idx[q]]]; it.xs.push_back(nd.a == it.S ? nd.b : nd.a); it.pos.push_back(idx[q]); }
    } else {
      it.group = false; it.root = cs->constraint_roots[idx[i]]; it.pos.push_back(idx[i]); j = i + 1;
    }
    items.push_back(it);
    i = j;
  }
  return items;
}

struct Compiler {
  const tb_cs_desc* cs;
  std::vector<int> refc;          // remaining uses per node
  std::vector<int> reg_of;        // register holding node value (-1 = none)
  std::vector<int> free_regs; int next_reg = 0, max_regs = 0;
  std::vector<QInstr> code;
  struct Opnd { int kind; uint32_t v; int node; };

  explicit Compiler(const tb_cs_desc* c) : cs(c), refc(c->num_nodes, 0), reg_of(c->num_nodes, -1) {}
  void count(uint32_t node, std::vector<char>& seen) {
    refc[node]++;
    if (seen[node]) return;
    seen[node] = 1;
    const tb_expr_node& nd = cs->nodes[node];
    if (nd.op == TB_EX_NEG || nd.op == TB_EX_SCALE) count(nd.a, seen);
    else if (nd.op == TB_EX_ADD || nd.op == TB_EX_MUL) { count(nd.a, seen); count(nd.b, seen); }
  }
  int alloc() {
    int r;
    if (!free_regs.empty()) { r = free_regs.back(); free_regs.pop_back(); } else r = next_reg++;
    if (next_reg > max_regs) max_regs = next_reg;
    return r;
  }
  void release(const Opnd& o) {
    if (o.node < 0) return;
    if (--refc[o.node] == 0 && reg_of[o.node] >= 0) { free_regs.push_back(reg_of[o.node]); reg_of[o.node] = -1; }
  }
  static uint32_t leaf(const tb_query& q) {   // column << 8 | (rotation + 128): the kernel needs no query table
    TB_REQUIRE(q.rotation >= -128 && q.rotation < 128 && q.column < (1u << 24), "query rotation / column out of the encodable range");
    return (q.column << 8) | (uint32_t)(q.rotation + 128);
  }
  bool is_two(uint32_t const_index) const {
    const uint8_t* c = cs->constants + 32 * (size_t)const_index;
    if (c[0] != 2) return false;
    for (int i = 1; i < 32; ++i) if (c[i]) return false;
    return true;
  }
  Opnd emit(uint32_t node) {
    const tb_expr_node& nd = cs->nodes[node];
    switch (nd.op) {
      case TB_EX_CONST: return {K_CONST, nd.a, (int)node};
      case TB_EX_ADVICE: return {K_ADV, leaf(cs->advice_queries[nd.a]), (int)node};
      case TB_EX_FIXED: return {K_FIX, leaf(cs->fixed_queries[nd.a]), (int)node};
      case TB_EX_INSTANCE: return {K_INST, leaf(cs->instance_queries[nd.a]), (int)node};
      default: break;
    }
    if (reg_of[node] >= 0) return {K_REG, (uint32_t)reg_of[node], (int)node};
    int op; Opnd oa, ob; bool binary = true;
    if (nd.op == TB_EX_NEG) { oa = emit(nd.a); ob = {K_CONST, 0, -1}; op = Q_NEG; binary = false; }
    else if (nd.op == TB_EX_SCALE) {
      oa = emit(nd.a);
      if (is_two(nd.b)) { ob = oa; ob.node = -1; op = Q_ADD; }   // 2 x = x + x: an addition instead of a multiplication
      else { ob = {K_CONST, nd.b, -1}; op = Q_MUL; }
    }
    else if (nd.op == TB_EX_MUL) { oa = emit(nd.a); ob = emit(nd.b); op = Q_MUL; }
    else {  // ADD, with a - b peephole when the negation is used only here
      const tb_expr_node& na = cs->nodes[nd.a]; const tb_expr_node& nb = cs->nodes[nd.b];
      if (nb.op == TB_EX_NEG && refc[nd.b] == 1 && reg_of[nd.b] < 0) {
        oa = emit(nd.a); refc[nd.b]--; ob = emit(nb.a); op = Q_SUB;
      } else if (na.op == TB_EX_NEG && refc[nd.a] == 1 && reg_of[nd.a] < 0) {
        oa = emit(nd.b); refc[nd.a]--; ob = emit(na.a); op = Q_SUB;
      } else { oa = emit(nd.a); ob = emit(nd.b); op = Q_ADD; }
    }
    // operands of leaves carry node ids only for refcounting; leaves hold no register
    release(oa); if (binary) release(ob);
    int r = alloc();
    code.push_back(q_make(op, r, oa.kind, oa.v, ob.kind, ob.v));
    reg_of[node] = r;
    return {K_REG, (uint32_t)r, (int)node};
  }
  // the constraints `idx` (ascending) folded with y; returns the index of the last one
  int compile_constraints(const std::vector<uint32_t>& idx) {
    std::vector<Item> items = build_items(cs, idx);
    std::vector<char> seen(cs->num_nodes, 0);
    for (auto& it : items) {
      if (!it.group) count(it.root, seen);
      else { count(it.S, seen); for (uint32_t x : it.xs) count(x, seen); }
    }
    int prev = -1;
    for (auto& it : items) {
      if (!it.group) {
        Opnd o = emit(it.root);
        code.push_back(q_make(Q_FOLD_Y, 0, o.kind, o.v, K_CONST, prev < 0 ? 1u : (uint32_t)((int)it.pos[0] - prev))); release(o);
        prev = (int)it.pos[0];
        continue;
      }
      for (size_t j = 0; j < it.xs.size(); ++j) {
        Opnd o = emit(it.xs[j]);
        code.push_back(q_make(j == 0 ? Q_GBEGIN : Q_GFOLD, 0, o.kind, o.v, K_CONST, j == 0 ? 0u : it.pos[j] - it.pos[j - 1])); release(o);
      }
      Opnd os = emit(it.S);
      code.push_back(q_make(Q_GEND, 0, os.kind, os.v, K_CONST, prev < 0 ? 1u : (uint32_t)((int)it.pos.back() - prev))); release(os);
      prev = (int)it.pos.back();
    }
    return prev;
  }
};
inline void finish_program(Compiler& c, GateProgram* out) {
  out->code = c.code; out->nregs = c.max_regs < 1 ? 1 : c.max_regs;
  TB_REQUIRE(out->nregs <= 48, "constraint expressions need too many live temporaries");
}

// polynomial degree of every constraint (a column query counts 1): decides which sub-cosets a constraint must be evaluated on
inline std::vector<int> q_constraint_degrees(const tb_cs_desc* cs) {
  std::vector<int> deg(cs->num_nodes, -1);
  for (uint32_t i = 0; i < cs->num_nodes; ++i) {   // nodes are in topological order (gate_desc_check)
    const tb_expr_node& nd = cs->nodes[i];
    switch (nd.op) {
      case TB_EX_CONST: deg[i] = 0; break;
      case TB_EX_ADVICE: case TB_EX_FIXED: case TB_EX_INSTANCE: deg[i] = 1; break;
      case TB_EX_NEG: case TB_EX_SCALE: deg[i] = deg[nd.a]; break;
      case TB_EX_ADD: deg[i] = deg[nd.a] > deg[nd.b] ? deg[nd.a] : deg[nd.b]; break;
      default: deg[i] = deg[nd.a] + deg[nd.b]; break;
    }
  }
  std::vector<int> out(cs->num_constraints);
  for (uint32_t j = 0; j < cs->num_constraints; ++j) out[j] = deg[cs->constraint_roots[j]];
  return out;
}
// The (sorted) constraint subset `subset` split into `parts` groups of similar cost, one program each (row-parallel AND
// constraint-parallel evaluation).
inline void q_compile_gates_split(const tb_cs_desc* cs, const std::vector<uint32_t>& subset, int parts, std::vector<GateProgram>* out) {
  // cost of a root = instructions of its stand-alone program; contiguous (within the subset) groups with roughly equal cumulative cost
  std::vector<size_t> cost(subset.size());
  size_t total = 0;
  for (size_t i = 0; i < subset.size(); ++i) {
    Compiler c(cs); std::vector<char> seen(cs->num_nodes, 0);
    c.count(cs->constraint_roots[subset[i]], seen);
    Compiler::Opnd o = c.emit(cs->constraint_roots[subset[i]]); (void)o;
    cost[i] = c.code.size() + 1; total += cost[i];
  }
  if (parts > (int)subset.size()) parts = subset.empty() ? 1 : (int)subset.size();
  out->clear();
  size_t r0 = 0, acc = 0;
  for (int p = 0; p < parts; ++p) {
    size_t r1 = r0;
    const size_t target = total * (p + 1) / parts;
    while (r1 < subset.size() && (acc < target || p == parts - 1)) acc += cost[r1++];
    if (p == parts - 1) r1 = subset.size();
    Compiler c(cs);
    const int last = c.compile_constraints(std::vector<uint32_t>(subset.begin() + r0, subset.begin() + r1));
    out->emplace_back();
    finish_program(c, &out->back());
    out->back().last = last;
    r0 = r1;
  }
}
// every lookup's inputs and table expressions compressed with theta: Q_LK_STORE l leaves the inputs in ACC, the table in G
inline void q_compile_lookups(const tb_cs_desc* cs, GateProgram* out) {
  Compiler c(cs);
  std::vector<char> seen(cs->num_nodes, 0);
  for (uint32_t l = 0; l < cs->num_lookups; ++l)
    for (uint32_t e = 0; e < cs->lookups[l].num_exprs; ++e) { c.count(cs->lookups[l].input_roots[e], seen); c.count(cs->lookups[l].table_roots[e], seen); }
  for (uint32_t l = 0; l < cs->num_lookups; ++l) {
    c.code.push_back(q_make(Q_LK_BEGIN, 0, K_CONST, 0, K_CONST, 0));
    for (uint32_t e = 0; e < cs->lookups[l].num_exprs; ++e) {
      Compiler::Opnd o = c.emit(cs->lookups[l].input_roots[e]);
      c.code.push_back(q_make(Q_FOLD_A, 0, o.kind, o.v, K_CONST, 0)); c.release(o);
    }
    for (uint32_t e = 0; e < cs->lookups[l].num_exprs; ++e) {
      Compiler::Opnd o = c.emit(cs->lookups[l].table_roots[e]);
      c.code.push_back(q_make(Q_FOLD_S, 0, o.kind, o.v, K_CONST, 0)); c.release(o);
    }
    c.code.push_back(q_make(Q_LK_STORE, 0, K_CONST, l, K_CONST, 0));
  }
  finish_program(c, out);
}

// The description comes across the ABI: reject anything that would make the compiler recurse without end or an
// interpreter read out of bounds (forward references, cycles, stray constant / query / column indices).
inline void gate_desc_check(const tb_cs_desc* cs) {
  TB_REQUIRE(cs->cs_degree >= 3 && cs->num_perm_columns <= PERM_MAX_SETS * (cs->cs_degree - 2), "unsupported constraint system shape");
  for (uint32_t l = 0; l < cs->num_lookups; ++l) {
    TB_REQUIRE(cs->lookups && cs->lookups[l].num_exprs >= 1 && cs->lookups[l].input_roots && cs->lookups[l].table_roots, "a lookup needs at least one expression pair");
    for (uint32_t e = 0; e < cs->lookups[l].num_exprs; ++e) {
      TB_REQUIRE(cs->lookups[l].input_roots[e] < cs->num_nodes, "lookup input root out of range");
      TB_REQUIRE(cs->lookups[l].table_roots[e] < cs->num_nodes, "lookup table root out of range");
    }
  }
  for (uint32_t i = 0; i < cs->num_advice_queries; ++i) TB_REQUIRE(cs->advice_queries[i].column < cs->num_advice, "advice query column out of range");
  for (uint32_t i = 0; i < cs->num_fixed_queries; ++i) TB_REQUIRE(cs->fixed_queries[i].column < cs->num_fixed, "fixed query column out of range");
  for (uint32_t i = 0; i < cs->num_instance_queries; ++i) TB_REQUIRE(cs->instance_queries[i].column < cs->num_instance, "instance query column out of range");
  for (uint32_t i = 0; i < cs->num_nodes; ++i) {
    const tb_expr_node& nd = cs->nodes[i];
    TB_REQUIRE(nd.op <= TB_EX_SCALE, "bad expression node");
    switch (nd.op) {
      case TB_EX_CONST: TB_REQUIRE(nd.a < cs->num_constants, "expression constant index out of range"); break;
      case TB_EX_ADVICE: TB_REQUIRE(nd.a < cs->num_advice_queries, "expression advice query index out of range"); break;
      case TB_EX_FIXED: TB_REQUIRE(nd.a < cs->num_fixed_queries, "expression fixed query index out of range"); break;
      case TB_EX_INSTANCE: TB_REQUIRE(nd.a < cs->num_instance_queries, "expression instance query index out of range"); break;
      case TB_EX_NEG: TB_REQUIRE(nd.a < i, "expression nodes must be in topological order"); break;
      case TB_EX_SCALE: TB_REQUIRE(nd.a < i && nd.b < cs->num_constants, "bad SCALE node"); break;
      default: TB_REQUIRE(nd.a < i && nd.b < i, "expression nodes must be in topological order"); break;
    }
  }
  for (uint32_t j = 0; j < cs->num_constraints; ++j) TB_REQUIRE(cs->constraint_roots[j] < cs->num_nodes, "constraint root out of range");
  for (const tb_column* pc = cs->perm_columns; pc < cs->perm_columns + cs->num_perm_columns; ++pc) {
    TB_REQUIRE(pc->kind <= TB_COL_INSTANCE, "permutation column kind out of range");
    TB_REQUIRE(pc->index < (pc->kind == TB_COL_ADVICE ? cs->num_advice : pc->kind == TB_COL_FIXED ? cs->num_fixed : cs->num_instance), "permutation column index out of range");
  }
  TB_REQUIRE(cs->blinding_factors >= 1 && cs->num_advice >= 1, "unsupported constraint system shape");
}
// The programs of a checked description whose quotient runs on R sub-cosets.  Gate programs come in nparts[big] parts,
// big = (batch size >= 8): small batches run more, shorter programs (latency), large ones fewer (less duplicated work).
// `gate_parts` holds the constraints evaluated on every sub-coset (all of them when the circuit is not split),
// `gate_parts_lo` the low-degree ones (degree <= R / 2) that are evaluated on every second sub-coset only.
struct GatePlan {
  static constexpr int nparts[2] = {8, 4};
  uint32_t num_constraints = 0, t_pl = 0; bool split = false;   // t_pl: permutation + lookup terms folded after the gates
  size_t num_lo = 0; int lo_instr = 0, all_instr = 0;   // what decided the split: low-degree constraints, instructions of them / of all
  std::vector<GateProgram> gate_parts[2], gate_parts_lo[2]; GateProgram lookups;
};
// Degree split: a constraint of degree <= R / 2 is a polynomial of fewer than (R / 2) * n coefficients, so the sum of all such
// constraints is fixed by its values on every second sub-coset; only the high-degree constraints (and the permutation /
// lookup terms) need all R sub-cosets.  Worth it when the low class carries a good part of the arithmetic (and allowed).
inline GatePlan gate_plan(const tb_cs_desc* cs, int R, bool allow_split) {
  GatePlan g; g.num_constraints = cs->num_constraints;
  const uint32_t chunk = cs->cs_degree - 2, P = cs->num_perm_columns;
  g.t_pl = perm_lookup_terms(P ? (P + chunk - 1) / chunk : 0, cs->num_lookups);
  std::vector<int> deg = q_constraint_degrees(cs);
  std::vector<uint32_t> all, lo, hi;
  for (uint32_t j = 0; j < cs->num_constraints; ++j) { all.push_back(j); ((R >= 4 && deg[j] <= R / 2) ? lo : hi).push_back(j); }
  { std::vector<GateProgram> t_all, t_lo;
    q_compile_gates_split(cs, all, 1, &t_all); q_compile_gates_split(cs, lo, 1, &t_lo);
    g.num_lo = lo.size(); g.lo_instr = (int)t_lo[0].code.size(); g.all_instr = (int)t_all[0].code.size();
    g.split = allow_split && R >= 4 && !lo.empty() && !hi.empty() && g.lo_instr * 10 >= g.all_instr * 3; }
  for (int big = 0; big < 2; ++big) {
    q_compile_gates_split(cs, g.split ? hi : all, GatePlan::nparts[big], &g.gate_parts[big]);
    if (g.split) q_compile_gates_split(cs, lo, GatePlan::nparts[big], &g.gate_parts_lo[big]);
  }
  q_compile_lookups(cs, &g.lookups);
  return g;
}

// One program on one point; ACC holds its result at the end.  The machine m says where values come from:
//   m.instr(pc); m.slot(r), where register r lives (ACC = nregs, the y / theta fold; G = nregs + 1, the group / table
//   fold); m.get(slot), m.set(slot, v); m.leaf(kind, v), constant v (K_CONST, Montgomery) or the column query
//   v = column << 8 | (rotation + 128); m.ypow(gap) = y^gap; m.theta(); m.lk_store(l, inputs, table).
// nv_exec_check_disable: as in argument.cuh, for the host-only machines.
#pragma nv_exec_check_disable
template <class M> TB_HD Fp gate_operand(M& m, int kind, uint32_t v) { return kind == K_REG ? m.get(m.slot((int)v)) : m.leaf(kind, v); }
#pragma nv_exec_check_disable
template <class M> TB_HD void gate_interp(M& m, int nregs, int ninstr) {
  const int ACC = m.slot(nregs), G = m.slot(nregs + 1);
  m.set(ACC, Fp::zero()); m.set(G, Fp::zero());
  QInstr in = m.instr(0);
  for (int pc = 0; pc < ninstr; ++pc) {
    const uint32_t w0 = in.w0, ia = in.a, ib = in.b;
    if (pc + 1 < ninstr) in = m.instr(pc + 1);   // next instruction word in flight while this one executes
    const int op = w0 & 0xff, ak = (w0 >> 16) & 0xff, bk = w0 >> 24;
    int dst = m.slot((w0 >> 8) & 0xff);
    Fp r;
    switch (op) {
      case Q_MOV: r = gate_operand(m, ak, ia); break;
      case Q_NEG: r = gate_operand(m, ak, ia).neg(); break;
      case Q_ADD: r = gate_operand(m, ak, ia) + gate_operand(m, bk, ib); break;
      case Q_SUB: r = gate_operand(m, ak, ia) - gate_operand(m, bk, ib); break;
      case Q_MUL: r = gate_operand(m, ak, ia) * gate_operand(m, bk, ib); break;
      case Q_FOLD_Y: r = m.get(ACC) * m.ypow(ib) + gate_operand(m, ak, ia); dst = ACC; break;   // acc = acc * y^gap + e
      case Q_FOLD_A: r = m.get(ACC) * m.theta() + gate_operand(m, ak, ia); dst = ACC; break;
      case Q_FOLD_S: r = m.get(G) * m.theta() + gate_operand(m, ak, ia); dst = G; break;
      case Q_GFOLD: r = m.get(G) * m.ypow(ib) + gate_operand(m, ak, ia); dst = G; break;
      case Q_GBEGIN: r = gate_operand(m, ak, ia); dst = G; break;
      case Q_GEND: r = m.get(ACC) * m.ypow(ib) + gate_operand(m, ak, ia) * m.get(G); dst = ACC; break;   // acc = acc * y^gap + S * g
      case Q_LK_BEGIN: r = Fp::zero(); m.set(G, r); dst = ACC; break;
      case Q_LK_STORE: m.lk_store(ia, m.get(ACC), m.get(G)); continue;
      default: continue;
    }
    m.set(dst, r);
  }
}

// The host machine (the verifier at x, the CPU tests): at(kind, column, rotation) is a column query's value, ypows[i] = y^i
template <class At> struct PointMachine {
  At at; const Fp* consts; const Fp* ypows; Fp th; Fp* lk_a; Fp* lk_s;
  const GateProgram* p = nullptr; std::vector<Fp> regs;
  QInstr instr(int pc) const { return pc < (int)p->code.size() ? p->code[pc] : QInstr{}; }   // gate_interp reads instruction 0 of an empty program
  int slot(int r) const { return r; }
  Fp get(int i) const { return regs[i]; } void set(int i, const Fp& v) { regs[i] = v; }
  Fp leaf(int kind, uint32_t v) const { return kind == K_CONST ? consts[v] : at(kind, (int)(v >> 8), (int)(v & 255u) - 128); }
  const Fp& ypow(uint32_t gap) const { return ypows[gap]; } const Fp& theta() const { return th; }
  void lk_store(uint32_t l, const Fp& a, const Fp& s) { lk_a[l] = a; lk_s[l] = s; }
  Fp run(const GateProgram& prog) { p = &prog; regs.assign(prog.nregs + 2, Fp::zero()); gate_interp(*this, prog.nregs, (int)prog.code.size()); return regs[prog.nregs]; }
};

}  // namespace tb
