// Minimal C++ caller of the host-side mirror (include/taiga_b200.hpp): a one-gate PLONKish circuit
//     q * (a * b - c) = 0,  public c            (k = 5, 3 advice + 1 instance + 1 selector, no lookups,
// a, b, c, instance in the permutation with the identity wiring except c[0] <-> instance[0]), proved and verified with
// Proof::create / Proof::verify (through a VerifyingKey) as a Taiga caller would (proof.rs:25-54).  Field arithmetic for the key material comes
// from the library's own header in host mode.  Without an H100 it must fail loudly: there is no CPU fallback (that path and
// the build are what tests/test_abi.py checks; the proving path itself is covered through the same C ABI by tests/test_gpu_*.py).
//
//   g++ -std=c++17 -I include examples/prove_cpp.cpp -L taiga_b200 -ltaiga_b200 -Wl,-rpath,$PWD/taiga_b200 -o /tmp/prove_cpp
#include <cstdio>
#include <string>
#include <vector>

#define TB_PORTABLE_FIELD 1
#include "../taiga_b200/csrc/curve.cuh"
#include "taiga_b200.hpp"

using namespace taiga_b200;
using tb::Fp;

static FieldBytes to_bytes(const Fp& v) {
  Fp c = v.from_mont();
  FieldBytes b;
  for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) b[4 * i + j] = (uint8_t)(c.l[i] >> (8 * j));
  return b;
}
static Fp small(uint32_t v) { return Fp::from_u32(v); }

// omega_k = ROOT_OF_UNITY^(2^(32-k)), ROOT_OF_UNITY = 5^((p-1)/2^32)   (pasta_curves Fp constants)
static Fp omega_of(uint32_t k) {
  const uint32_t t[8] = {0x992d30edu, 0x094cf91bu, 0x224698fcu, 0, 0, 0, 0x40000000u, 0};   // (p - 1) >> 32
  Fp root = Fp::one(), base = small(5);
  for (int limb = 7; limb >= 0; --limb) for (int bit = 31; bit >= 0; --bit) { root = root.sqr(); if ((t[limb] >> bit) & 1) root = root * base; }
  for (uint32_t i = 0; i < 32 - k; ++i) root = root.sqr();
  return root;
}
static PointBytes point_bytes(const tb::Aff<tb::Fq>& a) {
  PointBytes out;
  tb::Fq x = a.x.from_mont(), y = a.y.from_mont();
  for (int i = 0; i < 8; ++i) for (int j = 0; j < 4; ++j) { out[4 * i + j] = (uint8_t)(x.l[i] >> (8 * j)); out[32 + 4 * i + j] = (uint8_t)(y.l[i] >> (8 * j)); }
  return out;
}
static PointBytes mul_generator(const Fp& scalar) {
  tb::Aff<tb::Fq> G;   // Vesta generator (-1, 2)
  G.x = tb::Fq::one().neg(); G.y = tb::Fq::from_u32(2);
  Fp c = scalar.from_mont();
  return point_bytes(tb::scalar_mul(G, c.l).to_affine());
}
static void build_srs(uint32_t k, const Fp& omega, std::vector<uint8_t>& g, std::vector<uint8_t>& gl, PointBytes& W, PointBytes& U) {
  const uint32_t n = 1u << k;
  const Fp s = small(0x5eed5eedu) * small(0x0badc0deu) + small(7);
  Fp sn = s;
  for (uint32_t i = 0; i < k; ++i) sn = sn.sqr();                       // s^n
  const Fp num = (sn - Fp::one()) * small(n).inv();                     // (s^n - 1) / n
  Fp sj = Fp::one(), wi = Fp::one();
  for (uint32_t i = 0; i < n; ++i) {
    PointBytes a = mul_generator(sj), b = mul_generator(wi * num * (s - wi).inv());
    std::memcpy(&g[64 * i], a.data(), 64); std::memcpy(&gl[64 * i], b.data(), 64);
    sj = sj * s; wi = wi * omega;
  }
  W = mul_generator(small(0x77777777u) * small(0x12345u));
  U = mul_generator(small(0x33333333u) * small(0x54321u));
}

int main(int argc, char** argv) {
  try {
    const uint32_t k = 5, n = 1u << k;
    const Fp omega = omega_of(k);
    std::vector<uint8_t> g(64 * n), gl(64 * n);
    PointBytes W{}, U{};
    // ---- a throw-away SRS with the structure Params::new produces: g_lagrange is the Lagrange-basis image of g, i.e.
    // sum_i v_i * g_lagrange[i] == sum_j c_j * g[j] whenever c = iNTT(v).  Here g[j] = [s^j] G for a fixed scalar s (fine for
    // an example, worthless as a commitment key), hence g_lagrange[i] = [L_i(s)] G with
    // L_i(s) = omega^i (s^n - 1) / (n (s - omega^i)); w = [s_w] G, u = [s_u] G.
    build_srs(k, omega, g, gl, W, U);
    if (argc > 2 && std::string(argv[1]) == "--dump-srs") {   // lets tests/test_abi.py check the construction on a CPU-only box
      FILE* f = std::fopen(argv[2], "wb");
      if (!f) return 3;
      std::fwrite(g.data(), 1, g.size(), f); std::fwrite(gl.data(), 1, gl.size(), f); std::fwrite(W.data(), 1, 64, f); std::fwrite(U.data(), 1, 64, f);
      std::fclose(f);
    }
    Context ctx(0);   // throws without a usable sm_90 device
    Params params(ctx, k, g.data(), gl.data(), W, U);

    // ---- constraint system
    ConstraintSystem cs;
    cs.k = k; cs.num_advice = 3; cs.num_fixed = 1; cs.num_instance = 1;
    cs.cs_degree = 3; cs.blinding_factors = 5;   // max(3, 1 query per column) + 2
    for (uint32_t c = 0; c < 3; ++c) cs.advice_queries.push_back(tb_query{c, 0});
    cs.fixed_queries.push_back(tb_query{0, 0});
    cs.instance_queries.push_back(tb_query{0, 0});
    for (uint32_t c = 0; c < 3; ++c) cs.perm_columns.push_back(tb_column{TB_COL_ADVICE, c});
    cs.perm_columns.push_back(tb_column{TB_COL_INSTANCE, 0});
    uint32_t a = cs.add_node(TB_EX_ADVICE, 0), b = cs.add_node(TB_EX_ADVICE, 1), c = cs.add_node(TB_EX_ADVICE, 2), q = cs.add_node(TB_EX_FIXED, 0);
    uint32_t ab = cs.add_node(TB_EX_MUL, a, b), nc = cs.add_node(TB_EX_NEG, c), d = cs.add_node(TB_EX_ADD, ab, nc);
    cs.constraint_roots.push_back(cs.add_node(TB_EX_MUL, q, d));

    // ---- key material: selector on row 0; sigma = identity (delta^col * omega^row) with c[0] <-> instance[0] swapped
    std::vector<uint8_t> fixed(32 * n, 0), sigma(32 * n * 4);
    { FieldBytes one = to_bytes(Fp::one()); std::memcpy(&fixed[0], one.data(), 32); }
    Fp delta = small(5);
    for (int i = 0; i < 32; ++i) delta = delta.sqr();
    std::vector<Fp> sig(4 * n);
    Fp dc = Fp::one();
    for (uint32_t col = 0; col < 4; ++col) { Fp w = dc; for (uint32_t r = 0; r < n; ++r) { sig[col * n + r] = w; w = w * omega; } dc = dc * delta; }
    std::swap(sig[2 * n + 0], sig[3 * n + 0]);
    for (size_t i = 0; i < sig.size(); ++i) { FieldBytes v = to_bytes(sig[i]); std::memcpy(&sigma[32 * i], v.data(), 32); }
    ProvingKey pk(params, cs, fixed.data(), sigma.data());

    // ---- witness: 3 * 7 = 21 on row 0
    std::vector<uint8_t> advice(32 * n * 3, 0);
    FieldBytes three = to_bytes(small(3)), seven = to_bytes(small(7)), twentyone = to_bytes(small(21));
    std::memcpy(&advice[0], three.data(), 32); std::memcpy(&advice[32 * n], seven.data(), 32); std::memcpy(&advice[64 * n], twentyone.data(), 32);
    std::vector<std::vector<FieldBytes>> instance = {{twentyone}};
    std::array<uint8_t, 32> seed{};   // a real caller draws this from its RNG (proof.rs:30)

    Proof proof = Proof::create(pk, params, AdviceTable{advice.data()}, instance, seed);
    // a verifier holds the verifying key only: the constraint system and the commitments keygen_vk made
    std::vector<PointBytes> fixed_commitments, sigma_commitments;
    pk.commitments(fixed_commitments, sigma_commitments);
    VerifyingKey vk(params, cs, fixed_commitments, sigma_commitments);
    proof.verify(vk, params, instance);
    std::printf("proof of %zu bytes created and verified; kernels launched: %llu\n", proof.inner().size(), (unsigned long long)ctx.launch_count());
    instance[0][0] = seven;
    try { proof.verify(vk, params, instance); std::printf("ERROR: wrong instance accepted\n"); return 2; }
    catch (const Error& e) { std::printf("wrong instance rejected: %s (%s)\n", e.what(), e.kind()); }
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "taiga_b200 error [%s, status %d]: %s\n", e.kind(), e.status(), e.what());
    return 1;
  }
}
