//! halo2_proofs/src/plonk/gpu.rs of the patched fork: everything of `plonk::create_proof` AFTER witness synthesis runs in
//! libtaiga_b200.so (C ABI: include/taiga_b200.h).  Taiga reaches it through `Proof::create`
//! (taiga_halo2/src/proof.rs:25-42) without any change to taiga_halo2.
//!
//! NOT compiled in the build image (no cargo); written against zcash/halo2 0.3 + the crate-private fields a fork can read.
#![cfg(feature = "gpu")]
#![allow(non_camel_case_types, non_upper_case_globals, dead_code)]

use std::collections::HashMap;
use std::sync::Mutex;

use ff::PrimeField;
use group::Curve;
use pasta_curves::arithmetic::CurveAffine;
use pasta_curves::{pallas, vesta};
use rand_core::RngCore;

use super::{Any, ConstraintSystem, Error, Expression, ProvingKey, VerifyingKey};
use crate::poly::commitment::Params;
use crate::poly::{LagrangeCoeff, Polynomial};
use crate::transcript::{EncodedChallenge, TranscriptWrite};

mod tb {
    include!(concat!(env!("OUT_DIR"), "/tb.rs"));
}

type F = pallas::Base; // circuit field = vesta::Scalar

fn affine_bytes(p: &vesta::Affine) -> [u8; 64] {
    // 64 bytes x || y, identity = zeros (the convention of taiga_b200.h)
    let mut o = [0u8; 64];
    if let Some(c) = Option::<pasta_curves::arithmetic::Coordinates<vesta::Affine>>::from(p.coordinates()) {
        o[..32].copy_from_slice(c.x().to_repr().as_ref());
        o[32..].copy_from_slice(c.y().to_repr().as_ref());
    }
    o
}

fn last_error(ctx: *mut tb::tb_ctx) -> String {
    unsafe { std::ffi::CStr::from_ptr(tb::tb_last_error(ctx)).to_string_lossy().into_owned() }
}

/// Device-resident `Params<vesta::Affine>` (the entries of SETUP_PARAMS_MAP, taiga_halo2/src/constant.rs:128-139).
/// A tb_ctx is bound to one host thread: the mutex serialises callers the way the reference's sequential loop does.
pub struct GpuParams {
    ctx: Mutex<*mut tb::tb_ctx>,
    srs: *mut tb::tb_srs,
    k: u32,
}
unsafe impl Send for GpuParams {}
unsafe impl Sync for GpuParams {}

impl GpuParams {
    pub fn new(params: &Params<vesta::Affine>, device: i32) -> Result<Self, Error> {
        let mut ctx = std::ptr::null_mut();
        if unsafe { tb::tb_ctx_create(device, &mut ctx) } != 0 {
            return Err(Error::Synthesis); // no usable sm_90 device: there is no CPU fallback behind this feature
        }
        let g: Vec<u8> = params.g.iter().flat_map(affine_bytes).collect(); // crate-private fields, reachable in the fork
        let gl: Vec<u8> = params.g_lagrange.iter().flat_map(affine_bytes).collect();
        let (w, u) = (affine_bytes(&params.w), affine_bytes(&params.u));
        let mut srs = std::ptr::null_mut();
        let st = unsafe { tb::tb_srs_load(ctx, params.k, g.as_ptr(), gl.as_ptr(), w.as_ptr(), u.as_ptr(), &mut srs) };
        if st != 0 {
            eprintln!("tb_srs_load: {}", last_error(ctx));
            return Err(Error::Synthesis);
        }
        Ok(GpuParams { ctx: Mutex::new(ctx), srs, k: params.k })
    }
}

impl Drop for GpuParams {
    fn drop(&mut self) {
        unsafe {
            tb::tb_srs_free(self.srs);
            tb::tb_ctx_destroy(*self.ctx.lock().unwrap());
        }
    }
}

/// Flattening of `Expression<F>` into the topologically ordered DAG of tb_cs_desc (taiga_b200.h).
#[derive(Default)]
struct Flat {
    nodes: Vec<tb::tb_expr_node>,
    consts: Vec<[u8; 32]>,
    const_ix: HashMap<[u8; 32], u32>,
    memo: HashMap<String, u32>, // structural sharing keyed by Debug (cheap: done once per circuit)
}

impl Flat {
    fn constant(&mut self, c: F) -> u32 {
        let mut r = [0u8; 32];
        r.copy_from_slice(c.to_repr().as_ref());
        if let Some(&i) = self.const_ix.get(&r) {
            return i;
        }
        self.consts.push(r);
        self.const_ix.insert(r, (self.consts.len() - 1) as u32);
        (self.consts.len() - 1) as u32
    }
    fn push(&mut self, op: u32, a: u32, b: u32) -> u32 {
        self.nodes.push(tb::tb_expr_node { op, a, b });
        (self.nodes.len() - 1) as u32
    }
    fn expr(&mut self, e: &Expression<F>) -> u32 {
        let key = format!("{:?}", e);
        if let Some(&n) = self.memo.get(&key) {
            return n;
        }
        let n = match e {
            Expression::Constant(c) => {
                let i = self.constant(*c);
                self.push(tb::TB_EX_CONST, i, 0)
            }
            Expression::Selector(_) => unreachable!("selectors are fixed columns after keygen (compress_selectors)"),
            Expression::Fixed { query_index, .. } => self.push(tb::TB_EX_FIXED, *query_index as u32, 0),
            Expression::Advice { query_index, .. } => self.push(tb::TB_EX_ADVICE, *query_index as u32, 0),
            Expression::Instance { query_index, .. } => self.push(tb::TB_EX_INSTANCE, *query_index as u32, 0),
            Expression::Negated(a) => {
                let a = self.expr(a);
                self.push(tb::TB_EX_NEG, a, 0)
            }
            Expression::Sum(a, b) => {
                let (a, b) = (self.expr(a), self.expr(b));
                self.push(tb::TB_EX_ADD, a, b)
            }
            Expression::Product(a, b) => {
                let (a, b) = (self.expr(a), self.expr(b));
                self.push(tb::TB_EX_MUL, a, b)
            }
            Expression::Scaled(a, c) => {
                let a = self.expr(a);
                let c = self.constant(*c);
                self.push(tb::TB_EX_SCALE, a, c)
            }
        };
        self.memo.insert(key, n);
        n
    }
}

/// Calls `f` with the tb_cs_desc of `vk.cs()` (the description is valid only inside the call: it points into locals).
fn with_desc<R>(k: u32, vk: &VerifyingKey<vesta::Affine>, f: impl FnOnce(&tb::tb_cs_desc) -> R) -> R {
    let cs: &ConstraintSystem<F> = vk.cs();
    let q = |col: usize, rot: i32| tb::tb_query { column: col as u32, rotation: rot };
    let aq: Vec<_> = cs.advice_queries.iter().map(|(c, r)| q(c.index(), r.0)).collect();
    let fq: Vec<_> = cs.fixed_queries.iter().map(|(c, r)| q(c.index(), r.0)).collect();
    let iq: Vec<_> = cs.instance_queries.iter().map(|(c, r)| q(c.index(), r.0)).collect();
    let perm: Vec<_> = cs
        .permutation
        .get_columns()
        .iter()
        .map(|c| tb::tb_column {
            kind: match c.column_type() {
                Any::Advice => tb::TB_COL_ADVICE,
                Any::Fixed => tb::TB_COL_FIXED,
                Any::Instance => tb::TB_COL_INSTANCE,
            },
            index: c.index() as u32,
        })
        .collect();
    let mut flat = Flat::default();
    let roots: Vec<u32> = cs.gates.iter().flat_map(|g| g.polynomials().iter()).map(|p| flat.expr(p)).collect();
    let lk_roots: Vec<(Vec<u32>, Vec<u32>)> = cs
        .lookups
        .iter()
        .map(|l| (l.input_expressions.iter().map(|e| flat.expr(e)).collect(), l.table_expressions.iter().map(|e| flat.expr(e)).collect()))
        .collect();
    let lookups: Vec<tb::tb_lookup> = lk_roots
        .iter()
        .map(|(i, t)| tb::tb_lookup { num_exprs: i.len() as u32, input_roots: i.as_ptr(), table_roots: t.as_ptr() })
        .collect();
    let consts: Vec<u8> = flat.consts.iter().flatten().copied().collect();
    let mut repr = [0u8; 32];
    repr.copy_from_slice(vk.transcript_repr.to_repr().as_ref());
    let desc = tb::tb_cs_desc {
        k,
        num_advice: cs.num_advice_columns as u32,
        num_fixed: cs.num_fixed_columns as u32,
        num_instance: cs.num_instance_columns as u32,
        cs_degree: cs.degree() as u32,
        blinding_factors: cs.blinding_factors() as u32,
        num_advice_queries: aq.len() as u32,
        advice_queries: aq.as_ptr(),
        num_fixed_queries: fq.len() as u32,
        fixed_queries: fq.as_ptr(),
        num_instance_queries: iq.len() as u32,
        instance_queries: iq.as_ptr(),
        num_perm_columns: perm.len() as u32,
        perm_columns: perm.as_ptr(),
        num_constants: flat.consts.len() as u32,
        constants: consts.as_ptr(),
        num_nodes: flat.nodes.len() as u32,
        nodes: flat.nodes.as_ptr(),
        num_constraints: roots.len() as u32,
        constraint_roots: roots.as_ptr(),
        num_lookups: lookups.len() as u32,
        lookups: lookups.as_ptr(),
        vk_transcript_repr: repr,
    };
    f(&desc)
}

/// Device-resident proving key of one circuit (COMPLIANCE_PROVING_KEY, constant.rs:145-152;
/// TRIVIAL_RESOURCE_LOGIC_PK, resource_logic_examples.rs:50-61).
pub struct GpuProvingKey {
    pk: *mut tb::tb_pk,
    proof_len: usize,
    num_advice: usize,
}
unsafe impl Send for GpuProvingKey {}
unsafe impl Sync for GpuProvingKey {}

impl GpuProvingKey {
    pub fn new(gp: &GpuParams, pk: &ProvingKey<vesta::Affine>) -> Result<Self, Error> {
        let cs: &ConstraintSystem<F> = pk.get_vk().cs();
        let n = 1usize << gp.k;
        let col_bytes = |cols: &[Polynomial<F, LagrangeCoeff>]| -> Vec<u8> {
            cols.iter().flat_map(|c| c.iter().flat_map(|v| v.to_repr().as_ref().to_vec())).collect()
        };
        let fixed = col_bytes(&pk.fixed_values);
        let sigma = col_bytes(&pk.permutation.permutations);
        debug_assert_eq!(fixed.len(), cs.num_fixed_columns * n * 32);
        let mut out = std::ptr::null_mut();
        let ctx = gp.ctx.lock().unwrap();
        let st = with_desc(gp.k, pk.get_vk(), |desc| unsafe { tb::tb_circuit_load(*ctx, gp.srs, desc, fixed.as_ptr(), sigma.as_ptr(), &mut out) });
        if st != 0 {
            eprintln!("tb_circuit_load: {}", last_error(*ctx));
            return Err(Error::Synthesis);
        }
        Ok(GpuProvingKey { pk: out, proof_len: unsafe { tb::tb_pk_proof_len(out) }, num_advice: cs.num_advice_columns })
    }
}

/// The verifying key of one circuit on the host (what `Proof::verify` takes, proof.rs:45-54): built from a
/// `VerifyingKey` alone, e.g. the one inside `ResourceLogicVerifyingInfo` (taiga_api.rs:110), with no proving key.
pub struct GpuVerifyingKey {
    vk: *mut tb::tb_vk,
}
unsafe impl Send for GpuVerifyingKey {}
unsafe impl Sync for GpuVerifyingKey {}

impl GpuVerifyingKey {
    pub fn new(gp: &GpuParams, vk: &VerifyingKey<vesta::Affine>) -> Result<Self, Error> {
        let fixed: Vec<u8> = vk.fixed_commitments().iter().flat_map(affine_bytes).collect();
        let sigma: Vec<u8> = vk.permutation().commitments().iter().flat_map(affine_bytes).collect();
        let mut out = std::ptr::null_mut();
        let ctx = gp.ctx.lock().unwrap();
        let st = with_desc(gp.k, vk, |desc| unsafe { tb::tb_vk_load(*ctx, gp.srs, desc, fixed.as_ptr(), sigma.as_ptr(), &mut out) });
        if st != 0 {
            eprintln!("tb_vk_load: {}", last_error(*ctx));
            return Err(Error::Synthesis);
        }
        Ok(GpuVerifyingKey { vk: out })
    }
}

impl Drop for GpuVerifyingKey {
    fn drop(&mut self) {
        unsafe { tb::tb_vk_free(self.vk) }
    }
}

impl Drop for GpuProvingKey {
    fn drop(&mut self) {
        unsafe { tb::tb_pk_free(self.pk) }
    }
}

fn map_status(st: i32, ctx: *mut tb::tb_ctx) -> Error {
    match st as u32 {
        tb::TB_ERR_CONSTRAINT => Error::ConstraintSystemFailure, // a lookup input is missing from its table
        tb::TB_ERR_INVALID => Error::InstanceTooLarge,           // or a malformed call: see the message
        _ => {
            eprintln!("libtaiga_b200: {}", last_error(ctx));
            Error::Synthesis
        }
    }
}

/// The new tail of `plonk::create_proof`: `advice[p]` is the table `synthesize` produced for proof p (after
/// batch_invert_assigned), `instances[p]` its instance columns.  One call proves all of them (the reference passes one;
/// a batched `ShieldedPartialTransaction::build` passes 2P resp. 4P).  Proof bytes are appended to the transcripts exactly
/// as `Blake2bWrite::finalize` would have produced them.
pub fn create_proofs_gpu(
    gp: &GpuParams,
    gpk: &GpuProvingKey,
    advice: &[Vec<Polynomial<F, LagrangeCoeff>>],
    instances: &[&[&[F]]],
    mut rng: impl RngCore,
    first_proof_index: u32,
) -> Result<Vec<Vec<u8>>, Error> {
    let n_proofs = advice.len();
    let mut adv = Vec::with_capacity(n_proofs * gpk.num_advice * (32 << gp.k));
    for table in advice {
        for col in table {
            for v in col.iter() {
                adv.extend_from_slice(v.to_repr().as_ref());
            }
        }
    }
    let inst_len: Vec<u32> = instances[0].iter().map(|c| c.len() as u32).collect();
    let mut inst = Vec::new();
    for proof in instances {
        for col in proof.iter() {
            for v in col.iter() {
                inst.extend_from_slice(v.to_repr().as_ref());
            }
        }
    }
    let mut seed = [0u8; 32];
    rng.fill_bytes(&mut seed); // the only use of the caller's RNG (proof.rs:30): blinding scalars derive from (seed, proof index)
    let mut out = vec![0u8; n_proofs * gpk.proof_len];
    let ctx = gp.ctx.lock().unwrap();
    let st = unsafe {
        tb::tb_prove_batch(*ctx, gpk.pk, n_proofs as u32, adv.as_ptr(), inst.as_ptr(), inst_len.as_ptr(), seed.as_ptr(), first_proof_index, out.as_mut_ptr(), gpk.proof_len)
    };
    if st != 0 {
        return Err(map_status(st, *ctx));
    }
    Ok(out.chunks(gpk.proof_len).map(|c| c.to_vec()).collect())
}

/// Body of `plonk::create_proof` with the "gpu" feature, for the single-circuit call Taiga makes:
/// ```ignore
/// // (unchanged) synthesize each circuit into a WitnessCollection, then batch_invert_assigned -> advice: Vec<Polynomial<F, LagrangeCoeff>>
/// let proofs = gpu::create_proofs_gpu(gpu_params(params), gpu_pk(pk), &[advice], &[instances[0]], rng, 0)?;
/// transcript.write_raw(&proofs[0])?;          // small helper on Blake2bWrite: append bytes without hashing; the GPU ran the transcript
/// Ok(())
/// ```
/// `gpu_params` / `gpu_pk` are `lazy_static` caches keyed by the address of `params` / `pk`, mirroring SETUP_PARAMS_MAP and
/// COMPLIANCE_PROVING_KEY (constant.rs:128-152).
pub fn _doc_anchor() {}

/// The instance columns of every proof, concatenated, and the column lengths (those of the first proof).
fn flatten_instances(instances: &[&[&[F]]]) -> (Vec<u8>, Vec<u32>) {
    let inst_len: Vec<u32> = instances[0].iter().map(|c| c.len() as u32).collect();
    let mut inst = Vec::new();
    for proof in instances {
        for col in proof.iter() {
            for v in col.iter() {
                inst.extend_from_slice(v.to_repr().as_ref());
            }
        }
    }
    (inst, inst_len)
}

/// Runs one of the two batched verifiers (`call` gets ctx, n, instance, instance_len, proofs, proof_len, ok).
fn verify_with(
    gp: &GpuParams,
    instances: &[&[&[F]]],
    proofs: &[&[u8]],
    call: impl FnOnce(*mut tb::tb_ctx, u32, *const u8, *const u32, *const u8, usize, *mut u8) -> i32,
) -> Result<Vec<bool>, Error> {
    let (inst, inst_len) = flatten_instances(instances);
    let plen = proofs[0].len();
    let flat: Vec<u8> = proofs.iter().flat_map(|p| p.iter().copied()).collect();
    let mut ok = vec![0u8; proofs.len()];
    let ctx = gp.ctx.lock().unwrap();
    let st = call(*ctx, proofs.len() as u32, inst.as_ptr(), inst_len.as_ptr(), flat.as_ptr(), plen, ok.as_mut_ptr());
    if st != 0 {
        return Err(map_status(st, *ctx));
    }
    Ok(ok.into_iter().map(|b| b == 1).collect())
}

/// `Proof::verify` for many proofs of one circuit (shielded_ptx.rs:137-153 loops them one by one, 35 ms each on CPU).
pub fn verify_batch_gpu(gp: &GpuParams, gpk: &GpuProvingKey, instances: &[&[&[F]]], proofs: &[&[u8]]) -> Result<Vec<bool>, Error> {
    verify_with(gp, instances, proofs, |ctx, n, inst, lens, flat, plen, ok| unsafe { tb::tb_verify_batch(ctx, gpk.pk, n, inst, lens, flat, plen, plen, ok) })
}

/// The same verdicts from the verifying key alone: what a node that checks partial transactions holds.
pub fn verify_batch_gpu_vk(gp: &GpuParams, gvk: &GpuVerifyingKey, instances: &[&[&[F]]], proofs: &[&[u8]]) -> Result<Vec<bool>, Error> {
    verify_with(gp, instances, proofs, |ctx, n, inst, lens, flat, plen, ok| unsafe { tb::tb_verify_batch_vk(ctx, gvk.vk, n, inst, lens, flat, plen, plen, ok) })
}

/// `plonk::BatchVerifier` on the device (tb_batch_verifier_*; the FFI declarations come from taiga_b200.h through bindgen):
/// proofs of any circuits over `gp`'s SRS, one verdict.  Each `add_proofs` call replays its proofs and folds their
/// random-weighted final checks into the batch on the device; `finalize` runs the one remaining MSM.  The weights come from a
/// seed drawn from `rng` at `new`, which must be unpredictable to whoever made the proofs (then a batch that holds a bad proof is
/// accepted with probability at most 1/p).  Replaces the serial `verify_proof` loop of ShieldedPartialTxBundle::execute
/// (transaction.rs:246-257, shielded_ptx.rs:137-153): see INTEGRATION.md.
pub struct GpuBatchVerifier<'a> {
    gp: &'a GpuParams,
    bv: *mut tb::tb_batch_verifier,
}

impl<'a> GpuBatchVerifier<'a> {
    pub fn new(gp: &'a GpuParams, mut rng: impl RngCore) -> Result<Self, Error> {
        let mut seed = [0u8; 32];
        rng.fill_bytes(&mut seed);
        let mut bv = std::ptr::null_mut();
        let ctx = gp.ctx.lock().unwrap();
        let st = unsafe { tb::tb_batch_verifier_create(*ctx, gp.srs, seed.as_ptr(), &mut bv) };
        if st != 0 {
            return Err(map_status(st, *ctx));
        }
        Ok(GpuBatchVerifier { gp, bv })
    }

    /// `add_proof` for each of `proofs` (one circuit, at most 4096 per call).  A proof that does not even decode is not an
    /// error: it makes `finalize` return false.
    pub fn add_proofs(&mut self, gvk: &GpuVerifyingKey, instances: &[&[&[F]]], proofs: &[&[u8]]) -> Result<(), Error> {
        let bv = self.bv;
        verify_with(self.gp, instances, proofs, |ctx, n, inst, lens, flat, plen, _ok| unsafe {
            tb::tb_batch_verifier_add(ctx, bv, gvk.vk, n, inst, lens, flat, plen, plen)
        })
        .map(|_| ())
    }

    pub fn add_proof(&mut self, gvk: &GpuVerifyingKey, instance: &[&[F]], proof: &[u8]) -> Result<(), Error> {
        self.add_proofs(gvk, &[instance], &[proof])
    }

    /// true iff every proof added would pass `Proof::verify` (halo2's `BatchVerifier::finalize`; an empty batch is true)
    pub fn finalize(self) -> Result<bool, Error> {
        let mut ok = 0u8;
        let ctx = self.gp.ctx.lock().unwrap();
        let st = unsafe { tb::tb_batch_verifier_finalize(*ctx, self.bv, &mut ok) };
        if st != 0 {
            return Err(map_status(st, *ctx));
        }
        Ok(ok == 1)
    }
}

impl Drop for GpuBatchVerifier<'_> {
    fn drop(&mut self) {
        unsafe { tb::tb_batch_verifier_free(self.bv) }
    }
}
