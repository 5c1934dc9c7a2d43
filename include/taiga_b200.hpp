// C++ host-side mirror of the reference's interface for the proving path, over the C ABI of taiga_b200.h.
//
// The reference is Rust (taiga_halo2); its seam is
//     Proof::create(pk, params, circuit, instance, rng) -> Result<Proof, plonk::Error>      taiga_halo2/src/proof.rs:25-42
//     Proof::verify(&self, vk, params, instance)        -> Result<(), plonk::Error>         taiga_halo2/src/proof.rs:45-54
// with `params` / `pk` living in process-wide lazies (SETUP_PARAMS_MAP, COMPLIANCE_PROVING_KEY: constant.rs:128-153).
// This header keeps those names, argument meanings and the error behaviour (every failure is a typed exception, the
// counterpart of `Err(plonk::Error)`; nothing is silently downgraded, and there is no CPU fallback) for C++ callers and
// as the model for the Rust shim of INTEGRATION.md.  Header only; link with -ltaiga_b200.
#pragma once
#include <array>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "taiga_b200.h"

namespace taiga_b200 {

using FieldBytes = std::array<uint8_t, 32>;   // canonical little-endian field element (ff::PrimeField::to_repr)
using PointBytes = std::array<uint8_t, 64>;   // affine x || y, identity = all zero

// plonk::Error as seen through the C ABI.  `status` is the tb_status; kind() names the halo2 variant it mirrors.
class Error : public std::runtime_error {
 public:
  Error(tb_status status, const std::string& what) : std::runtime_error(what), status_(status) {}
  tb_status status() const { return status_; }
  // TB_ERR_CONSTRAINT <-> plonk::Error::ConstraintSystemFailure; TB_ERR_INVALID <-> InstanceTooLarge / malformed call;
  // everything else (no device, CUDA failure) has no halo2 counterpart and maps to Error::Synthesis-class failures.
  const char* kind() const {
    switch (status_) {
      case TB_ERR_CONSTRAINT: return "ConstraintSystemFailure";
      case TB_ERR_INVALID: return "InvalidArgument";
      default: return "BackendFailure";
    }
  }

 private:
  tb_status status_;
};

// One GPU + one stream.  Bound to the creating host thread, like the reference's single-threaded callers
// (shielded_ptx.rs:107-125); use one Context per worker thread.
class Context {
 public:
  explicit Context(int device = 0) {
    tb_ctx* c = nullptr;
    tb_status st = tb_ctx_create(device, &c);
    if (st != TB_OK) {
      std::string msg = c ? tb_last_error(c) : "tb_ctx_create failed (no CUDA device? the library has no CPU fallback)";
      if (c) tb_ctx_destroy(c);
      throw Error(st, msg);
    }
    ctx_.reset(c);
  }
  tb_ctx* get() const { return ctx_.get(); }
  void check(tb_status st) const {
    if (st != TB_OK) throw Error(st, tb_last_error(ctx_.get()));
  }
  uint64_t launch_count() const { return tb_ctx_launch_count(ctx_.get()); }

 private:
  struct Del { void operator()(tb_ctx* c) const { tb_ctx_destroy(c); } };
  std::unique_ptr<tb_ctx, Del> ctx_;
};

// poly::commitment::Params<vesta::Affine> (an entry of SETUP_PARAMS_MAP, constant.rs:128-139), resident on the device
// together with its fixed-base window tables.
class Params {
 public:
  // g, g_lagrange: 2^k affine points each (the decompressed contents of taiga_halo2/params/params_<k>); w, u: one point
  Params(const Context& ctx, uint32_t k, const uint8_t* g, const uint8_t* g_lagrange, const PointBytes& w, const PointBytes& u) : ctx_(&ctx), k_(k) {
    tb_srs* s = nullptr;
    ctx.check(tb_srs_load(ctx.get(), k, g, g_lagrange, w.data(), u.data(), &s));
    srs_.reset(s);
  }
  uint32_t k() const { return k_; }
  const tb_srs* get() const { return srs_.get(); }
  const Context& context() const { return *ctx_; }
  // Params::commit / commit_lagrange: MSM(scalars, basis) + blind * w
  PointBytes commit(const uint8_t* scalars, const FieldBytes* blind, bool lagrange) const {
    PointBytes out{};
    ctx_->check(tb_srs_commit(ctx_->get(), srs_.get(), lagrange ? 1 : 0, 1, scalars, blind ? blind->data() : nullptr, out.data()));
    return out;
  }

 private:
  struct Del { void operator()(tb_srs* s) const { tb_srs_free(s); } };
  const Context* ctx_;
  uint32_t k_;
  std::unique_ptr<tb_srs, Del> srs_;
};

// Owning builder of tb_cs_desc: what the shim reads out of `pk.get_vk().cs()` (ConstraintSystem<Fp>) once per circuit.
struct ConstraintSystem {
  uint32_t k = 0, num_advice = 0, num_fixed = 0, num_instance = 0, cs_degree = 0, blinding_factors = 0;
  std::vector<tb_query> advice_queries, fixed_queries, instance_queries;
  std::vector<tb_column> perm_columns;
  std::vector<FieldBytes> constants;
  std::vector<tb_expr_node> nodes;
  std::vector<uint32_t> constraint_roots;
  std::vector<std::pair<std::vector<uint32_t>, std::vector<uint32_t>>> lookups;   // (input roots, table roots)
  FieldBytes vk_transcript_repr{};

  uint32_t add_constant(const FieldBytes& c) { constants.push_back(c); return (uint32_t)constants.size() - 1; }
  uint32_t add_node(uint32_t op, uint32_t a, uint32_t b = 0) { nodes.push_back(tb_expr_node{op, a, b}); return (uint32_t)nodes.size() - 1; }

  // the flat view handed to tb_circuit_load; valid while *this and `lk` are alive and unchanged
  tb_cs_desc view(std::vector<tb_lookup>& lk) const {
    lk.clear();
    for (const auto& l : lookups) {
      if (l.first.size() != l.second.size()) throw Error(TB_ERR_INVALID, "lookup argument: input and table expression counts differ");
      lk.push_back(tb_lookup{(uint32_t)l.first.size(), l.first.data(), l.second.data()});
    }
    tb_cs_desc d;
    std::memset(&d, 0, sizeof(d));
    d.k = k; d.num_advice = num_advice; d.num_fixed = num_fixed; d.num_instance = num_instance;
    d.cs_degree = cs_degree; d.blinding_factors = blinding_factors;
    d.num_advice_queries = (uint32_t)advice_queries.size(); d.advice_queries = advice_queries.data();
    d.num_fixed_queries = (uint32_t)fixed_queries.size(); d.fixed_queries = fixed_queries.data();
    d.num_instance_queries = (uint32_t)instance_queries.size(); d.instance_queries = instance_queries.data();
    d.num_perm_columns = (uint32_t)perm_columns.size(); d.perm_columns = perm_columns.data();
    d.num_constants = (uint32_t)constants.size(); d.constants = constants.empty() ? nullptr : constants[0].data();
    d.num_nodes = (uint32_t)nodes.size(); d.nodes = nodes.data();
    d.num_constraints = (uint32_t)constraint_roots.size(); d.constraint_roots = constraint_roots.data();
    d.num_lookups = (uint32_t)lk.size(); d.lookups = lk.data();
    std::memcpy(d.vk_transcript_repr, vk_transcript_repr.data(), 32);
    return d;
  }
};

// ProvingKey<vesta::Affine> (COMPLIANCE_PROVING_KEY / TRIVIAL_RESOURCE_LOGIC_PK): fixed and sigma polynomials, their
// extended cosets and the compiled constraint programs, resident on the device.  Proof::verify also accepts it in place of
// the VerifyingKey.
class ProvingKey {
 public:
  // fixed_values: num_fixed x 2^k, sigma_values: perm_columns x 2^k field elements (Lagrange basis, column-major)
  ProvingKey(const Params& params, const ConstraintSystem& cs, const uint8_t* fixed_values, const uint8_t* sigma_values)
      : params_(&params), num_advice_(cs.num_advice), num_instance_(cs.num_instance), k_(cs.k), num_fixed_(cs.num_fixed),
        num_perm_((uint32_t)cs.perm_columns.size()) {
    std::vector<tb_lookup> lk;
    tb_cs_desc d = cs.view(lk);
    tb_pk* p = nullptr;
    params.context().check(tb_circuit_load(params.context().get(), params.get(), &d, fixed_values, sigma_values, &p));
    pk_.reset(p);
  }
  const tb_pk* get() const { return pk_.get(); }
  const Params& params() const { return *params_; }
  size_t proof_len() const { return tb_pk_proof_len(pk_.get()); }
  uint32_t num_advice() const { return num_advice_; }
  uint32_t num_instance() const { return num_instance_; }
  size_t rows() const { return (size_t)1 << k_; }
  // keygen_vk: vk.fixed_commitments and vk.permutation.commitments (constant.rs:150)
  void commitments(std::vector<PointBytes>& fixed, std::vector<PointBytes>& sigma) const {
    fixed.assign(num_fixed_, PointBytes{});
    sigma.assign(num_perm_, PointBytes{});
    params_->context().check(tb_pk_commitments(params_->context().get(), pk_.get(), fixed.empty() ? nullptr : fixed[0].data(),
                                               sigma.empty() ? nullptr : sigma[0].data()));
  }

 private:
  struct Del { void operator()(tb_pk* p) const { tb_pk_free(p); } };
  const Params* params_;
  uint32_t num_advice_, num_instance_, k_, num_fixed_, num_perm_;
  std::unique_ptr<tb_pk, Del> pk_;
};

// VerifyingKey<vesta::Affine> as Proof::verify uses it (proof.rs:45-54): the constraint system and the fixed and
// permutation commitments, no proving-key table.  Built from what a verifier receives (ResourceLogicVerifyingInfo carries
// the vk, taiga_api.rs:110); host memory only.
class VerifyingKey {
 public:
  VerifyingKey(const Params& params, const ConstraintSystem& cs, const std::vector<PointBytes>& fixed_commitments,
               const std::vector<PointBytes>& sigma_commitments)
      : params_(&params), num_instance_(cs.num_instance) {
    if (fixed_commitments.size() != cs.num_fixed || sigma_commitments.size() != cs.perm_columns.size())
      throw Error(TB_ERR_INVALID, "one commitment per fixed and per permutation column is required");
    std::vector<tb_lookup> lk;
    tb_cs_desc d = cs.view(lk);
    tb_vk* v = nullptr;
    params.context().check(tb_vk_load(params.context().get(), params.get(), &d, fixed_commitments.empty() ? nullptr : fixed_commitments[0].data(),
                                      sigma_commitments.empty() ? nullptr : sigma_commitments[0].data(), &v));
    vk_.reset(v);
  }
  const tb_vk* get() const { return vk_.get(); }
  const Params& params() const { return *params_; }
  size_t proof_len() const { return tb_vk_proof_len(vk_.get()); }
  uint32_t num_instance() const { return num_instance_; }
  // Proof::verify for n proofs already in device memory of the context's device (tb_dev_verify_batch_vk): proof i at
  // d_proofs + i * proof_stride, instance values as canonical bytes, d_ok[i] written in stream order.  Returns without waiting.
  void verify_batch_device(uint32_t n, const void* d_instance, const std::vector<uint32_t>& instance_len, const void* d_proofs, size_t proof_stride,
                           void* d_ok) const {
    params_->context().check(tb_dev_verify_batch_vk(params_->context().get(), vk_.get(), n, d_instance, instance_len.empty() ? nullptr : instance_len.data(),
                                                    d_proofs, proof_stride, proof_len(), d_ok));
  }

 private:
  struct Del { void operator()(tb_vk* v) const { tb_vk_free(v); } };
  const Params* params_;
  uint32_t num_instance_;
  std::unique_ptr<tb_vk, Del> vk_;
};

// The witness of one proof: what `Circuit::synthesize` assigned (after batch_invert_assigned), num_advice x 2^k elements.
struct AdviceTable {
  const uint8_t* data;   // host or device pointer
};

// One failure MockProver::verify() would report (halo2's VerifyFailure): a constraint not zero on a row (Gate), a lookup input
// missing from its table (Lookup), or a copied cell that differs from its successor in the permutation (Permutation).
struct VerifyFailure {
  enum Kind { Gate = TB_FAIL_GATE, Lookup = TB_FAIL_LOOKUP, Permutation = TB_FAIL_COPY };
  Kind kind;
  uint32_t index;        // constraint (position in constraint_roots), lookup, or permutation column position
  uint32_t row;
  uint32_t other_column, other_row;   // Permutation: the cell's successor
};
// The outcome of checking one witness: the exact counts (rows with a failing constraint, failing lookup inputs, failing copy
// cells) and the first failures in MockProver's order.  passed() iff all counts are 0.
struct CheckResult {
  uint64_t gate_rows = 0, lookup_inputs = 0, copy_cells = 0;
  std::vector<VerifyFailure> failures;
  bool passed() const { return gate_rows == 0 && lookup_inputs == 0 && copy_cells == 0; }
};

// `Proof(Vec<u8>)`, proof.rs:19-22
class Proof {
 public:
  Proof() = default;
  explicit Proof(std::vector<uint8_t> bytes) : bytes_(std::move(bytes)) {}
  const std::vector<uint8_t>& inner() const { return bytes_; }

  // SECURITY: every blinding scalar of proof i is a PRF of (rng_seed, proof_index + i).  A (seed, index) pair must NEVER be used for
  // two different witnesses -- reusing it reuses all blinding scalars and leaks witness data.  Draw a fresh 32-byte seed from the
  // caller's RNG for every call (what the Rust shim does, rust/halo2_proofs_patch/src/gpu.rs) or advance proof_index.
  // Proof::create (proof.rs:25-42).  `instance`: one vector per instance column (&[&[pallas::Base]]); `rng_seed`: 32 bytes
  // the caller draws from its RNG (the reference passes `impl RngCore`), from which every blinding scalar is derived.
  // Throws Error (kind() == "ConstraintSystemFailure" for a lookup input outside its table).
  static Proof create(const ProvingKey& pk, const Params& params, const AdviceTable& circuit,
                      const std::vector<std::vector<FieldBytes>>& instance, const std::array<uint8_t, 32>& rng_seed, uint32_t proof_index = 0) {
    std::vector<Proof> out = create_batch(pk, params, &circuit, 1, {instance}, rng_seed, proof_index);
    return std::move(out[0]);
  }

  // Batched sibling (plonk::create_proof already takes slices of circuits): n proofs of one circuit in one device pass.
  // `circuits` points at n advice tables stored contiguously when n > 1 (circuits[0].data is the base address).
  static std::vector<Proof> create_batch(const ProvingKey& pk, const Params& params, const AdviceTable* circuits, uint32_t n,
                                         const std::vector<std::vector<std::vector<FieldBytes>>>& instances,
                                         const std::array<uint8_t, 32>& rng_seed, uint32_t first_proof_index = 0) {
    if (&pk.params() != &params) throw Error(TB_ERR_INVALID, "proving key was built for different Params");
    if (n == 0 || instances.size() != n) throw Error(TB_ERR_INVALID, "one instance per proof is required");
    std::vector<uint32_t> lens;
    std::vector<uint8_t> inst = flatten(instances, pk.num_instance(), lens);
    const size_t plen = pk.proof_len();
    std::vector<uint8_t> buf(plen * n);
    const Context& ctx = params.context();
    ctx.check(tb_prove_batch(ctx.get(), pk.get(), n, circuits[0].data, inst.data(), lens.data(), rng_seed.data(), first_proof_index, buf.data(), plen));
    std::vector<Proof> out;
    for (uint32_t i = 0; i < n; ++i) out.emplace_back(std::vector<uint8_t>(buf.begin() + i * plen, buf.begin() + (i + 1) * plen));
    return out;
  }

  // create_batch into device memory of the context's device (tb_dev_prove_batch): n advice tables at d_advice, the instance
  // values of each proof (canonical bytes, columns concatenated) at d_instance, proof i written at d_proofs + i * proof_stride
  // and its status at d_status[i] (TB_PROVED, 1 + l for a lookup l input outside its table, TB_PROVE_INTERNAL; a record whose
  // status is not TB_PROVED is zeros).  Returns without waiting: read the status from d_status after the context's stream has
  // passed the call.  Throws Error for a refused call (nothing is enqueued).  The seed rules of create apply.
  static void create_batch_device(const ProvingKey& pk, const Params& params, uint32_t n, const void* d_advice, const void* d_instance,
                                  const std::vector<uint32_t>& instance_len, const std::array<uint8_t, 32>& rng_seed, uint32_t first_proof_index,
                                  void* d_proofs, size_t proof_stride, uint32_t* d_status) {
    if (&pk.params() != &params) throw Error(TB_ERR_INVALID, "proving key was built for different Params");
    const Context& ctx = params.context();
    ctx.check(tb_dev_prove_batch(ctx.get(), pk.get(), n, d_advice, d_instance, instance_len.empty() ? nullptr : instance_len.data(), rng_seed.data(),
                                 first_proof_index, d_proofs, proof_stride, d_status));
  }

  // MockProver::run(k, circuit, instance).verify() for n witnesses, without proving (verify_transparently).  `circuits` and
  // `instances` as in create_batch.  `seed` must be unpredictable to whoever wrote the witnesses: gates and lookups are tested
  // through random combinations drawn from it (a failure escapes with probability about (constraints + lookup width) / p).
  static std::vector<CheckResult> check_batch(const ProvingKey& pk, const Params& params, const AdviceTable* circuits, uint32_t n,
                                              const std::vector<std::vector<std::vector<FieldBytes>>>& instances,
                                              const std::array<uint8_t, 32>& seed, uint32_t max_failures = 16) {
    if (&pk.params() != &params) throw Error(TB_ERR_INVALID, "proving key was built for different Params");
    if (n == 0 || instances.size() != n) throw Error(TB_ERR_INVALID, "one instance per witness is required");
    std::vector<uint32_t> lens;
    std::vector<uint8_t> inst = flatten(instances, pk.num_instance(), lens);
    std::vector<uint64_t> counts(3 * (size_t)n);
    std::vector<tb_failure> recs((size_t)n * max_failures);
    const Context& ctx = params.context();
    ctx.check(tb_check_batch(ctx.get(), pk.get(), n, circuits[0].data, inst.data(), lens.data(), seed.data(), max_failures, counts.data(),
                             max_failures ? recs.data() : nullptr));
    std::vector<CheckResult> out(n);
    for (uint32_t i = 0; i < n; ++i) {
      out[i].gate_rows = counts[3 * i]; out[i].lookup_inputs = counts[3 * i + 1]; out[i].copy_cells = counts[3 * i + 2];
      for (uint32_t j = 0; j < max_failures; ++j) {
        const tb_failure& f = recs[(size_t)i * max_failures + j];
        if (f.kind) out[i].failures.push_back(VerifyFailure{static_cast<VerifyFailure::Kind>(f.kind), f.index, f.row, f.other_column, f.other_row});
      }
    }
    return out;
  }

  // Proof::verify (proof.rs:45-54): returns normally iff accepted, throws Error("ConstraintSystemFailure") otherwise --
  // `Result<(), plonk::Error>` in the reference.  `vk` is the VerifyingKey, or the ProvingKey of the circuit.
  void verify(const VerifyingKey& vk, const Params& params, const std::vector<std::vector<FieldBytes>>& instance) const {
    std::vector<bool> ok = verify_batch(vk, params, {*this}, {instance});
    if (!ok[0]) throw Error(TB_ERR_CONSTRAINT, "proof rejected");
  }
  void verify(const ProvingKey& vk, const Params& params, const std::vector<std::vector<FieldBytes>>& instance) const {
    std::vector<bool> ok = verify_batch(vk, params, {*this}, {instance});
    if (!ok[0]) throw Error(TB_ERR_CONSTRAINT, "proof rejected");
  }
  static std::vector<bool> verify_batch(const VerifyingKey& vk, const Params& params, const std::vector<Proof>& proofs,
                                        const std::vector<std::vector<std::vector<FieldBytes>>>& instances) {
    return verify_with(params, proofs, instances, vk.num_instance(), [&](uint32_t n, const uint8_t* inst, const uint32_t* lens, const uint8_t* buf, size_t plen, uint8_t* ok) {
      return tb_verify_batch_vk(params.context().get(), vk.get(), n, inst, lens, buf, plen, plen, ok);
    });
  }
  static std::vector<bool> verify_batch(const ProvingKey& vk, const Params& params, const std::vector<Proof>& proofs,
                                        const std::vector<std::vector<std::vector<FieldBytes>>>& instances) {
    return verify_with(params, proofs, instances, vk.num_instance(), [&](uint32_t n, const uint8_t* inst, const uint32_t* lens, const uint8_t* buf, size_t plen, uint8_t* ok) {
      return tb_verify_batch(params.context().get(), vk.get(), n, inst, lens, buf, plen, plen, ok);
    });
  }

 private:
  template <class Call>
  static std::vector<bool> verify_with(const Params& params, const std::vector<Proof>& proofs, const std::vector<std::vector<std::vector<FieldBytes>>>& instances,
                                       uint32_t num_instance, Call call) {
    const uint32_t n = (uint32_t)proofs.size();
    if (n == 0 || instances.size() != n) throw Error(TB_ERR_INVALID, "one instance per proof is required");
    std::vector<uint32_t> lens;
    std::vector<uint8_t> inst = flatten(instances, num_instance, lens);
    const size_t plen = proofs[0].bytes_.size();
    std::vector<uint8_t> buf(plen * n), ok(n, 0);
    for (uint32_t i = 0; i < n; ++i) {
      if (proofs[i].bytes_.size() != plen) throw Error(TB_ERR_INVALID, "proofs of one circuit have one length");
      std::memcpy(buf.data() + i * plen, proofs[i].bytes_.data(), plen);
    }
    params.context().check(call(n, inst.data(), lens.data(), buf.data(), plen, ok.data()));
    return std::vector<bool>(ok.begin(), ok.end());
  }
  // per proof the instance columns concatenated; every proof of a batch must use the same column lengths
  static std::vector<uint8_t> flatten(const std::vector<std::vector<std::vector<FieldBytes>>>& instances, uint32_t num_instance,
                                      std::vector<uint32_t>& lens) {
    std::vector<uint8_t> out;
    lens.assign(num_instance, 0);
    for (size_t p = 0; p < instances.size(); ++p) {
      if (instances[p].size() != num_instance) throw Error(TB_ERR_INVALID, "wrong number of instance columns");
      for (uint32_t c = 0; c < num_instance; ++c) {
        const auto& col = instances[p][c];
        if (p == 0) lens[c] = (uint32_t)col.size();
        else if (lens[c] != col.size()) throw Error(TB_ERR_INVALID, "instance column lengths differ inside a batch");
        for (const FieldBytes& v : col) out.insert(out.end(), v.begin(), v.end());
      }
    }
    return out;
  }
  std::vector<uint8_t> bytes_;
  friend class BatchVerifier;
};

// plonk::BatchVerifier: proofs of any circuits over one Params, one verdict.  add_proof / add_proofs queue nothing on the host:
// each call replays its proofs and folds their random-weighted final checks into the batch on the device; finalize() runs
// the one remaining MSM and returns true iff every proof added would verify on its own.  `seed` draws the weights and must
// be unpredictable to whoever made the proofs (a batch holding a bad proof is then accepted with probability at most 1/p):
// draw a fresh one per batch.  finalize() consumes the batch.  Throws Error for a refused call (a key built for other
// Params, a call after finalize) and for device failures; a proof that does not even decode is not an error, it makes
// finalize() return false.
class BatchVerifier {
 public:
  BatchVerifier(const Params& params, const std::array<uint8_t, 32>& seed) : params_(&params) {
    tb_batch_verifier* b = nullptr;
    params.context().check(tb_batch_verifier_create(params.context().get(), params.get(), seed.data(), &b));
    bv_.reset(b);
  }
  void add_proof(const VerifyingKey& vk, const std::vector<std::vector<FieldBytes>>& instance, const Proof& proof) {
    add_proofs(vk, {proof}, {instance});
  }
  // `instances[i]`: one vector per instance column of proof i; at most 4096 proofs per call
  void add_proofs(const VerifyingKey& vk, const std::vector<Proof>& proofs, const std::vector<std::vector<std::vector<FieldBytes>>>& instances) {
    if (&vk.params() != params_) throw Error(TB_ERR_INVALID, "verifying key was built for different Params");
    Proof::verify_with(*params_, proofs, instances, vk.num_instance(), [&](uint32_t n, const uint8_t* inst, const uint32_t* lens, const uint8_t* buf, size_t plen, uint8_t*) {
      return tb_batch_verifier_add(params_->context().get(), bv_.get(), vk.get(), n, inst, lens, buf, plen, plen);
    });
  }
  // n proofs already in device memory (tb_dev_batch_verifier_add, layouts as VerifyingKey::verify_batch_device); returns
  // without waiting
  void add_proofs_device(const VerifyingKey& vk, uint32_t n, const void* d_instance, const std::vector<uint32_t>& instance_len, const void* d_proofs,
                         size_t proof_stride) {
    params_->context().check(tb_dev_batch_verifier_add(params_->context().get(), bv_.get(), vk.get(), n, d_instance,
                                                       instance_len.empty() ? nullptr : instance_len.data(), d_proofs, proof_stride, vk.proof_len()));
  }
  bool finalize() {
    uint8_t ok = 0;
    params_->context().check(tb_batch_verifier_finalize(params_->context().get(), bv_.get(), &ok));
    return ok == 1;
  }

 private:
  struct Del { void operator()(tb_batch_verifier* b) const { tb_batch_verifier_free(b); } };
  const Params* params_;
  std::unique_ptr<tb_batch_verifier, Del> bv_;
};

}  // namespace taiga_b200
