"""GPU: the batch verifier (tb_batch_verifier, lib.BatchVerifier), halo2's BatchVerifier: one verdict for any number of
proofs of any circuits over one SRS, from the random-weighted sum of their final IPA checks.

* Honest proofs of every shape the repository proves (mini circuits, boundary shapes, random seeds, both Taiga shapes at
  k = 15 in calls of 1, 64 and 65, Compliance and VP proofs in one batch, the golden proofs) are accepted, and so is the
  empty batch.
* Every soundness input of tests/soundness_cases.py (each one-element mutant of a proof, and the proofs of witnesses that
  break one gate or copy) makes the batch it sits in reject, wherever it sits: first, middle, last, or in a later call than
  the honest proofs; tb_verify_batch_vk rejects the same proof.
* A cancelling pair: the final scalar f of one proof + 1 and of another - 1 gives final-check sums -W and +W, which an
  unweighted sum would accept; the batch rejects it in one call, across two calls and across the two Taiga circuits, under
  three seeds.
* More than one call's limit (4160 proofs), refusals that leave the batch as it was, and ProverService.verify_ptx_batch.
* The g-term kernel on its own through the test probe, against a Python big-integer sum, with all proofs in one group (the
  batch verifier) and with one proof per group (the per-proof verifier)."""
import ctypes
import os
import random

import numpy as np
import pytest

import soundness_cases as sc
from conftest import GOLDEN
from taiga_b200 import circuits_mini as cm
from taiga_b200 import circuits_random as cr
from taiga_b200 import circuits_taiga as ct
from taiga_b200 import lib, ptx

from test_gpu_poly_lookup import Probe, addr, expect
from test_gpu_verifier_soundness import PROVE_SHAPES, stack
from test_verifier_soundness import MUTANT_SHAPES, SEED, mutant_shape

pytestmark = pytest.mark.gpu

P = cr.P
MINI = [(6, False, 2), (7, True, 1), (6, False, 0), (9, True, 2), (12, False, 1)]
RANDOM = [("boundary", name) for name, _ in cr.BOUNDARY] + [("seed", s) for s in range(8)]
GOLDEN_K6_SEED = bytes((7 * i + 1) & 0xFF for i in range(32))
SEEDS = [bytes(range(32)), bytes([0xA5] * 32), bytes(range(200, 232))]


@pytest.fixture(scope="module")
def srs_for(gpu_ctx, oracle_cpu):
    """k -> (synthetic SRS arrays, device SRS)"""
    cache = {}

    def get(k):
        if k not in cache:
            s = oracle_cpu.synthetic_srs(k, seed=k)
            cache[k] = (s, gpu_ctx.load_srs(k, s["g"], s["g_lagrange"], s["w"], s["u"]))
        return cache[k]
    yield get
    for _, g in cache.values():
        g.close()


def _honest(kd, make, pk, n, w0=400):
    adv, inst, lens = stack(kd, [make(w0 + b) for b in range(n)])
    return pk.prove_batch(adv, inst, lens, SEED), inst, lens


def run(srs, seed, adds):
    """finalize() of a new batch after add(vk, instance, lens, proofs) of each item of `adds`"""
    bv = lib.BatchVerifier(srs, seed)
    try:
        for vk, inst, lens, proofs in adds:
            bv.add(vk, inst, lens, proofs)
        return bv.finalize()
    finally:
        bv.close()


def shift_f(proof, d):
    """the proof with its last scalar f (absorbed last: nothing else depends on it) replaced by f + d mod p"""
    v = (int.from_bytes(proof[-32:], "little") + d) % P
    return proof[:-32] + v.to_bytes(32, "little")


@pytest.fixture(scope="module")
def small(srs_for):
    """the k = 6 standard PLONK shape: (device SRS, pk, vk, 64 honest proofs, their instances, lens)"""
    kd, make = cm.standard_plonk(k=6, n_lookups=2)
    _, gsrs = srs_for(6)
    pk = gsrs.load_circuit(kd)
    vk = pk.verifying_key()
    proofs, inst, lens = _honest(kd, make, pk, 64)
    yield gsrs, pk, vk, proofs, inst, lens
    vk.close()
    pk.close()


@pytest.fixture(scope="module")
def taiga(gpu_srs):
    """both Taiga shapes at k = 15: {compliance: (kd, pk, vk, 65 proofs, instances, lens, golden proof, its instance)}"""
    out = {}
    for compliance in (True, False):
        kd, make = ct.build(compliance)
        pk = gpu_srs.load_circuit(kd)
        wit = [kd.witness_arrays(make(40 + w)) for w in range(4)]
        adv = np.stack([wit[b % 4][0] for b in range(65)])
        inst = np.stack([wit[b % 4][1] for b in range(65)])
        proofs = pk.prove_batch(adv, inst, wit[0][2], bytes(range(100, 132)))
        golden = open(os.path.join(GOLDEN, "proof_k15_compliance_shape.bin" if compliance else "proof_k15_vp_shape.bin"), "rb").read()
        out[compliance] = (kd, pk, pk.verifying_key(), proofs, inst, wit[0][2], golden, wit[1][1][None])
    yield out
    for v in out.values():
        v[2].close()
        v[1].close()


# ---------------------------------------------------------------- honest batches
def test_empty_batch_accepts(srs_for):
    _, gsrs = srs_for(6)
    assert run(gsrs, SEEDS[0], []) is True


@pytest.mark.parametrize("k,wide,nl", MINI)
def test_mini_circuits_accepted(srs_for, k, wide, nl):
    kd, make = cm.standard_plonk(k=k, wide=wide, n_lookups=nl)
    _, gsrs = srs_for(k)
    pk = gsrs.load_circuit(kd)
    vk = pk.verifying_key()
    proofs, inst, lens = _honest(kd, make, pk, 3)
    assert run(gsrs, SEEDS[0], [(vk, inst, lens, proofs)])
    assert run(gsrs, SEEDS[1], [(vk, inst[:1], lens, proofs[:1]), (vk, inst[1:], lens, proofs[1:])])
    bad = bytearray(proofs[1])
    bad[len(bad) // 2] ^= 1
    assert not run(gsrs, SEEDS[0], [(vk, inst, lens, [proofs[0], bytes(bad), proofs[2]])])
    if (k, wide, nl) == (6, False, 2):   # the golden proof: witness 100, proof index 5
        _, inst1, lens1 = kd.witness_arrays(make(100))
        golden = open(os.path.join(GOLDEN, "proof_k6_plonk.bin"), "rb").read()
        assert run(gsrs, SEEDS[2], [(vk, inst, lens, proofs), (vk, inst1[None], lens1, [golden])])
    vk.close()
    pk.close()


@pytest.mark.parametrize("which", RANDOM, ids=["%s-%s" % w for w in RANDOM])
def test_random_and_boundary_shapes_accepted(srs_for, which):
    kind, v = which
    kd, make = cr.boundary(v) if kind == "boundary" else cr.random_shape(v)
    _, gsrs = srs_for(kd.k)
    pk = gsrs.load_circuit(kd)
    vk = pk.verifying_key()
    proofs, inst, lens = _honest(kd, make, pk, 2, w0=11)
    assert run(gsrs, SEEDS[0], [(vk, inst, lens, proofs)])
    a, e = dict((n, (s_, t)) for n, s_, t in cr.proof_sections(kd))["evaluations"]
    bad = bytearray(proofs[0])
    bad[(a + e) // 2] ^= 1
    assert not run(gsrs, SEEDS[0], [(vk, inst, lens, [bytes(bad), proofs[1]])])
    vk.close()
    pk.close()


def test_taiga_shapes_in_calls_of_1_64_65_mixed(gpu_srs, taiga):
    c, v = taiga[True], taiga[False]
    adds = []
    for B in (1, 64, 65):
        for kd, pk, vk, proofs, inst, lens, _, _ in (c, v):
            adds.append((vk, inst[:B], lens, proofs[:B]))
    adds += [(c[2], c[7], c[5], [c[6]]), (v[2], v[7], v[5], [v[6]])]   # the golden proofs
    assert run(gpu_srs, SEEDS[0], adds)
    assert run(gpu_srs, SEEDS[1], [(v[2], v[4], v[5], v[3]), (c[2], c[4], c[5], c[3])])
    bad = bytearray(v[3][33])
    bad[100] ^= 1
    assert not run(gpu_srs, SEEDS[0], [(c[2], c[4], c[5], c[3]), (v[2], v[4], v[5], v[3][:33] + [bytes(bad)] + v[3][34:])])


@pytest.mark.parametrize("seed", range(5))
def test_honest_batches_accept_under_any_seed(small, seed):
    gsrs, pk, vk, proofs, inst, lens = small
    s = random.Random(seed).randbytes(32)
    assert run(gsrs, s, [(vk, inst[:20], lens, proofs[:20]), (vk, inst[20:], lens, proofs[20:])])


# ---------------------------------------------------------------- soundness inputs
@pytest.fixture(scope="module")
def keys(srs_for):
    cache = {}

    def get(name):
        if name not in cache:
            kd, make = mutant_shape(name)
            _, gsrs = srs_for(kd.k)
            pk = gsrs.load_circuit(kd)
            cache[name] = (kd, make, gsrs, pk, pk.verifying_key())
        return cache[name]
    yield get
    for v in cache.values():
        v[4].close()
        v[3].close()


PLACEMENTS = ["first", "middle", "last", "later call"]


def placed(vk, honest, bad, where):
    """adds with `bad` = (proof, instance row) alone among the honest (proof, instance row) pairs, at `where`"""
    def call(items):
        return (vk, np.stack([i for _, i in items]), None, [p for p, _ in items])
    h = list(honest)
    if where == "first":
        calls = [[bad] + h]
    elif where == "middle":
        calls = [h[:len(h) // 2] + [bad] + h[len(h) // 2:]]
    elif where == "last":
        calls = [h + [bad]]
    else:
        calls = [h[:2], [bad], h[2:]]
    return [call(c) for c in calls if c]


def batch_verdict(gsrs, lens, adds, seed=SEEDS[0]):
    return run(gsrs, seed, [(vk, inst, lens, proofs) for vk, inst, _, proofs in adds])


@pytest.mark.parametrize("name", MUTANT_SHAPES)
def test_every_mutant_rejects_its_batch(keys, name):
    kd, make, gsrs, pk, vk = keys(name)
    proofs, inst, lens = _honest(kd, make, pk, 4)
    honest = list(zip(proofs[1:], inst[1:]))
    muts = sc.mutants(kd, proofs[0], proofs[1])
    same = [m for m in muts if len(m[3]) == len(proofs[0])]
    assert vk.verify_batch(np.stack([inst[0]] * len(same)), lens, [m for _, _, _, m in same]) == [False] * len(same)
    seen = set()
    for i, (label, section, kind, m) in enumerate(same):
        wheres = [PLACEMENTS[i % 4]]
        if (section, kind) not in seen:   # one mutant of every (section, kind) in every placement
            seen.add((section, kind))
            wheres = PLACEMENTS
        for where in wheres:
            assert not batch_verdict(gsrs, lens, placed(vk, honest, (m, inst[0]), where)), "%s: %s, %s, accepted" % (name, label, where)
    # a proof of another length, in a call of its own between honest calls
    for label, _, _, m in muts:
        if len(m) != len(proofs[0]):
            assert vk.verify_batch(inst[:1], lens, [m]) == [False]
            adds = [(vk, inst[1:3], lens, proofs[1:3]), (vk, inst[:1], lens, [m]), (vk, inst[3:], lens, proofs[3:])]
            assert not run(gsrs, SEEDS[0], adds), "%s: %s accepted" % (name, label)
    assert batch_verdict(gsrs, lens, [(vk, inst, None, proofs)])


@pytest.mark.parametrize("name", PROVE_SHAPES)
def test_false_statements_reject_their_batch(keys, name):
    kd, make, gsrs, pk, vk = keys(name)
    bad = [(label, asg) for label, asg in sc.violations(kd, make, 5) if not label.startswith("lookup")]
    adv, inst, lens = stack(kd, [make(100 + i) for i in range(3)] + [a for _, a in bad])
    proofs = pk.prove_batch(adv, inst, lens, SEED)
    honest = list(zip(proofs[:3], inst[:3]))
    assert vk.verify_batch(inst[3:], lens, proofs[3:]) == [False] * len(bad)
    for i, (label, _) in enumerate(bad):
        for where in PLACEMENTS:
            assert not batch_verdict(gsrs, lens, placed(vk, honest, (proofs[3 + i], inst[3 + i]), where)), "%s: %s, %s, accepted" % (name, label, where)


@pytest.mark.parametrize("seed", SEEDS, ids=["seed%d" % i for i in range(len(SEEDS))])
def test_cancelling_pair_is_rejected(small, gpu_srs, taiga, seed):
    """f + 1 and f - 1 in two proofs: final-check sums -W and +W, whose unweighted sum is the identity"""
    gsrs, pk, vk, proofs, inst, lens = small
    up, down = shift_f(proofs[1], 1), shift_f(proofs[3], -1)
    assert vk.verify_batch(inst[:4], lens, [proofs[0], up, proofs[2], down]) == [True, False, True, False]
    assert not run(gsrs, seed, [(vk, inst[:4], lens, [proofs[0], up, proofs[2], down])])
    assert not run(gsrs, seed, [(vk, inst[:2], lens, [proofs[0], up]), (vk, inst[2:4], lens, [proofs[2], down])])
    assert run(gsrs, seed, [(vk, inst[:4], lens, proofs[:4])])
    c, v = taiga[True], taiga[False]
    c_up, v_down = shift_f(c[3][0], 1), shift_f(v[3][1], -1)
    assert c[2].verify_batch(c[4][:1], c[5], [c_up]) == [False] and v[2].verify_batch(v[4][1:2], v[5], [v_down]) == [False]
    assert not run(gpu_srs, seed, [(c[2], c[4][:1], c[5], [c_up]), (v[2], v[4][:2], v[5], [v[3][0], v_down])])


def test_more_than_one_calls_limit(small):
    gsrs, pk, vk, proofs, inst, lens = small
    assert run(gsrs, SEEDS[0], [(vk, inst, lens, proofs)] * 65)
    bad = list(proofs)
    bad[4100 - 64 * 64] = shift_f(proofs[4100 - 64 * 64], 1)   # proof 4100 of the batch: item 4 of the 65th call
    assert not run(gsrs, SEEDS[0], [(vk, inst, lens, proofs)] * 64 + [(vk, inst, lens, bad)])


# ---------------------------------------------------------------- refusals
def _add_raw(ctx, bv, vk, inst, lens, proofs, stride, plen, n=None):
    K = len(proofs) if n is None else n
    buf = np.zeros(max(1, len(proofs) * max(stride, plen)), np.uint8)   # the last record is read in full
    for i, p in enumerate(proofs):
        w = min(stride, len(p))
        buf[i * stride:i * stride + w] = np.frombuffer(p[:w], np.uint8)
    inst = np.ascontiguousarray(inst, dtype=np.uint8)
    lens = np.ascontiguousarray(lens, dtype=np.uint32)
    return ctx._lib.tb_batch_verifier_add(ctx._h, bv._h, vk._h, K, inst.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p),
                                          buf.ctypes.data_as(ctypes.c_void_p), stride, plen)


def test_refusals_leave_the_batch_as_it_was(gpu_ctx, small, srs_for, oracle_cpu):
    gsrs, pk, vk, proofs, inst, lens = small
    kd = pk.keydata
    s6, _ = srs_for(6)
    other_srs = gpu_ctx.load_srs(6, s6["g"], s6["g_lagrange"], s6["w"], s6["u"])   # the same points, another SRS
    f, sg = pk.commitments()
    other_vk = other_srs.load_verifying_key(kd, f, sg)
    plen = len(proofs[0])
    usable = kd.n - (kd.blinding_factors + 1)
    long_lens = np.array([usable + 1] + list(lens[1:]), np.uint32)
    cases = [("a vk on another SRS", lambda bv: _add_raw(gpu_ctx, bv, other_vk, inst[:2], lens, proofs[:2], plen, plen)),
             ("no proof", lambda bv: _add_raw(gpu_ctx, bv, vk, inst[:1], lens, proofs[:1], plen, plen, n=0)),
             ("4097 proofs", lambda bv: _add_raw(gpu_ctx, bv, vk, np.stack([inst[0]] * 4097), lens, [proofs[0]] * 4097, plen, plen)),
             ("stride < proof_len", lambda bv: _add_raw(gpu_ctx, bv, vk, inst[:2], lens, proofs[:2], plen - 32, plen)),
             ("instance too long", lambda bv: _add_raw(gpu_ctx, bv, vk, np.zeros((1, 32 * int(long_lens.sum())), np.uint8), long_lens, proofs[:1], plen, plen))]
    for want in (True, False):
        bv = lib.BatchVerifier(gsrs, SEEDS[1])
        bv.add(vk, inst[:3], lens, proofs[:3] if want else [proofs[0], shift_f(proofs[1], 1), proofs[2]])
        for what, call in cases:
            assert call(bv) == lib.TB_ERR_INVALID, what
        bv.add(vk, inst[3:6], lens, proofs[3:6])
        for what, call in cases:
            assert call(bv) == lib.TB_ERR_INVALID, what
        assert bv.finalize() is want
        assert _add_raw(gpu_ctx, bv, vk, inst[:1], lens, proofs[:1], plen, plen) == lib.TB_ERR_INVALID
        with pytest.raises(lib.TaigaB200Error, match="after tb_batch_verifier_finalize") as e:
            bv.finalize()
        assert e.value.status == lib.TB_ERR_INVALID
        bv.close()
    assert run(gsrs, SEEDS[0], [(vk, inst, lens, proofs)])    # the context keeps working
    assert vk.verify_batch(inst[:2], lens, proofs[:2]) == [True, True]
    other_vk.close()
    other_srs.close()


def test_a_batch_moves_between_contexts(small):
    gsrs, pk, vk, proofs, inst, lens = small
    other = lib.Context(0)
    bv = lib.BatchVerifier(gsrs, SEEDS[2])
    bv.add(vk, inst[:10], lens, proofs[:10])
    bv.add(vk, inst[10:], lens, proofs[10:], ctx=other)
    assert bv.finalize(ctx=other)
    bv.close()
    other.close()


# ---------------------------------------------------------------- ProverService
def test_verify_ptx_batch(srs_fixture):
    svc = ptx.ProverService(0, srs_fixture, c_workers=1, v_workers=1)
    base = svc.synthesize_ptx(2, wseed=9)
    wit = {"c_adv": np.concatenate([base["c_adv"]] * 4), "c_inst": np.concatenate([base["c_inst"]] * 4), "c_len": base["c_len"],
           "v_adv": np.concatenate([base["v_adv"]] * 4), "v_inst": np.concatenate([base["v_inst"]] * 4), "v_len": base["v_len"]}
    seed = bytes(range(60, 92))
    pc, pv = svc.build_ptx_batch(wit, seed)
    assert svc.verify_ptx_batch(pc, pv, wit, bytes(range(32))) == (True, [True] * 8)
    bad = bytearray(pv[5 * ptx.VP_PER_PTX + 2])
    bad[len(bad) // 2] ^= 1
    pv2 = pv[:5 * ptx.VP_PER_PTX + 2] + [bytes(bad)] + pv[5 * ptx.VP_PER_PTX + 3:]
    assert svc.verify_ptx_batch(pc, pv2, wit, bytes(range(32))) == (False, [True] * 5 + [False] + [True] * 2)
    assert svc.verify_ptx_batch(pc, [shift_f(p, 1) if i == 21 else p for i, p in enumerate(pv)], wit, bytes(range(32))) == (False, [True] * 5 + [False] + [True] * 2)


# ---------------------------------------------------------------- the g-term kernel
def g_ref(G, us, ab, k):
    """G[t] + sum_p (a_p s_{p,t} + [t = 0] b_p), s_{p,t} = prod_j u_{p,j}^{bit_(k-1-j)(t)}"""
    out = list(G)
    for u, (a, b) in zip(us, ab):
        s = [a]
        for j in reversed(range(k)):      # u_(k-1) multiplies bit 0 of t, ..., u_0 the top bit
            s = s + [x * u[j] % P for x in s]
        out = [x + y for x, y in zip(out, s)]
        out[0] += b
    return [x % P for x in out]


@pytest.mark.parametrize("K", [1, 3, 64])
@pytest.mark.parametrize("k", [1, 2, 7, 8, 9, 15, 16])
def test_g_scalars_kernel(gpu_ctx, k, K):
    probe = Probe(gpu_ctx)
    so = probe.so
    so.tbp_batch_g_scalars.restype = ctypes.c_int
    so.tbp_batch_g_scalars.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int, ctypes.c_int]
    rnd = random.Random(k * 100 + K)
    n = 1 << k
    edge = [0, 1, P - 1]

    def field():
        return edge[rnd.randrange(3)] if rnd.random() < 0.1 else rnd.randrange(P)
    G = [rnd.randrange(P) for _ in range(n)]
    d_G = probe.put(G)
    want = G
    for call in range(2):
        us = [[field() for _ in range(k)] for _ in range(K)]
        ab = [(field(), field()) for _ in range(K)]
        d_us, d_ab = probe.put([x for u in us for x in u]), probe.put([x for p in ab for x in p])
        probe.run("tbp_batch_g_scalars", addr(d_G), addr(d_us), addr(d_ab), k, K)
        want = g_ref(want, us, ab, k)
        expect("batch_g_scalars k=%d K=%d, call %d" % (k, K, call), probe.get(d_G), want)
        assert probe.get(d_us) == [x for u in us for x in u]
    # the same driver with one proof per group (the per-proof verifier): proof p's terms added into row p of [K][n] alone
    so.tbp_batch_g_scalars_grouped.restype = ctypes.c_int
    so.tbp_batch_g_scalars_grouped.argtypes = [ctypes.c_void_p] * 4 + [ctypes.c_int] * 3
    rows = [[rnd.randrange(P) for _ in range(n)] for _ in range(K)]
    d_rows = probe.put([x for r in rows for x in r])
    us = [[field() for _ in range(k)] for _ in range(K)]
    ab = [(field(), field()) for _ in range(K)]
    d_us, d_ab = probe.put([x for u in us for x in u]), probe.put([x for p in ab for x in p])
    probe.run("tbp_batch_g_scalars_grouped", addr(d_rows), addr(d_us), addr(d_ab), k, K, 1)
    got = probe.get(d_rows)
    for p in range(K):
        expect("batch_g_scalars k=%d K=%d, one proof per group, proof %d" % (k, K, p), got[p * n:(p + 1) * n], g_ref(rows[p], us[p:p + 1], ab[p:p + 1], k))
