"""GPU: the CUDA prover on false statements and the device verifier (tb_verify_batch) on inputs it must reject, against the
oracles (the same inputs test_verifier_soundness.py checks on the CPU; tests/soundness_cases.py makes them).

* Witnesses that break one gate, copy or instance copy are proved in batches of 2 and 9 (B >= 8 selects the other
  quotient program set) next to honest ones; every proof equals the oracle's byte for byte.  On split_mixed_degrees this
  is the only input under which the remainder r_lo of the low-degree quotient is not zero.  The device verifier accepts
  exactly the honest slots.
* A witness that breaks a lookup is refused with ConstraintSystemFailure naming its slot.
* Every one-element mutant of a proof goes through one verify_batch call; the verdicts equal the C++ oracle's.
* Batch sizes 1, 31, 32, 33, 4096 and 4097, a proof stride wider than the proof, instance lengths and values the
  verifier must refuse or reject, and keys that differ in one fixed cell or one copy."""
import copy
import ctypes
import random

import numpy as np
import pytest

import soundness_cases as sc
from taiga_b200 import circuits_random as cr
from taiga_b200 import circuits_taiga as ct
from taiga_b200 import lib

from test_verifier_soundness import MUTANT_SHAPES, SEED, mutant_shape

pytestmark = pytest.mark.gpu

PROVE_SHAPES = [s for s in MUTANT_SHAPES if s != "standard_plonk"] + ["split_mixed_degrees"]


@pytest.fixture(scope="module")
def keys(gpu_ctx, oracle_cpu):
    """name -> (kd, make, oracle key, device key); one device SRS per k."""
    srs_cache, cache = {}, {}

    def get(name):
        if name not in cache:
            kd, make = mutant_shape(name)
            if kd.k not in srs_cache:
                s = oracle_cpu.synthetic_srs(kd.k, seed=kd.k)
                srs_cache[kd.k] = (s, gpu_ctx.load_srs(kd.k, s["g"], s["g_lagrange"], s["w"], s["u"]))
            srs, gsrs = srs_cache[kd.k]
            cache[name] = (kd, make, oracle_cpu.OracleKey(kd, srs), gsrs.load_circuit(kd))
        return cache[name]
    yield get
    for v in cache.values():
        v[3].close()
    for _, g in srs_cache.values():
        g.close()


def stack(kd, asgs):
    wit = [kd.witness_arrays(a) for a in asgs]
    lens = wit[0][2]
    assert all((w[2] == lens).all() for w in wit)
    return np.stack([w[0] for w in wit]), np.stack([w[1] for w in wit]), lens


def where_differs(kd, got, want):
    i = next(i for i in range(min(len(got), len(want))) if got[i] != want[i])
    return "first differing byte %d: %s" % (i, cr.section_of(kd, i))


@pytest.mark.parametrize("B", [2, 9])
@pytest.mark.parametrize("name", PROVE_SHAPES)
def test_false_statements_prove_like_the_oracle_and_are_rejected(keys, monkeypatch, capfd, name, B):
    kd, make, okey, pk = keys(name)
    if name == "split_mixed_degrees":   # the shape exists to run the degree split: the first with r_lo != 0
        assert "split on" in _split_report(keys, name, monkeypatch, capfd)
    bad = [(label, asg) for label, asg in sc.violations(kd, make, 5) if not label.startswith("lookup")]
    assert bad, name
    # batches of exactly B: B - 1 violations and one honest witness at a position that moves from batch to batch
    slots = []
    for c, i in enumerate(range(0, len(bad), B - 1)):
        batch = bad[i:i + B - 1]
        batch.insert(c % (len(batch) + 1), ("honest", make(100 + c)))
        batch += [("honest", make(200 + c * B + j)) for j in range(B - len(batch))]
        slots += batch
    for first in range(0, len(slots), B):
        batch = slots[first:first + B]
        adv, inst, lens = stack(kd, [a for _, a in batch])
        proofs = pk.prove_batch(adv, inst, lens, SEED, first_proof_index=first)
        for b, (label, _) in enumerate(batch):
            ref = okey.prove(adv[b], inst[b], lens, SEED, proof_index=first + b)
            if proofs[b] != ref:
                pytest.fail("%s B=%d %s: the proof differs from the oracle's, %s" % (name, B, label, where_differs(kd, proofs[b], ref)))
        verdicts = pk.verify_batch(inst, lens, proofs)
        assert verdicts == [label == "honest" for label, _ in batch], "%s B=%d: %s" % (name, B, list(zip([l for l, _ in batch], verdicts)))


def _split_report(keys, name, monkeypatch, capfd):
    """TB_DEBUG's report of the quotient split of a fresh load of the shape's key."""
    kd, _, _, pk = keys(name)
    monkeypatch.setenv("TB_DEBUG", "1")
    capfd.readouterr()
    again = pk.srs.load_circuit(kd)
    err = capfd.readouterr().err
    monkeypatch.delenv("TB_DEBUG")
    again.close()
    return err


@pytest.mark.parametrize("name,lookup", [("lookups4_wide", 0), ("lookups4_wide", 1), ("lookups4_wide", 2), ("no_gates", 2)],
                         ids=["4-pairs", "table-degree-2", "input-degree-3", "full-row"])
def test_lookup_violations_are_refused(keys, name, lookup):
    kd, make, okey, pk = keys(name)
    d = cr.describe(kd)
    if name == "lookups4_wide":
        assert (d["lookup_pairs"][lookup], d["table_degrees"][lookup], d["input_degrees"][lookup]) == [(4, 1, 2), (1, 2, 2), (2, 1, 3)][lookup]
    else:
        assert d["full_row_lookup"] and lookup == len(kd.cs.lookups) - 1
    label, asg = next(c for c in sc.violations(kd, make, 5) if c[0] == "lookup%d" % lookup)
    B, slot = 5, 1 + lookup
    asgs = [make(200 + b) for b in range(B)]
    asgs[slot] = asg
    adv, inst, lens = stack(kd, asgs)
    with pytest.raises(lib.ConstraintSystemFailure) as e:
        pk.prove_batch(adv, inst, lens, SEED, first_proof_index=10)
    msg = str(e.value)
    assert "proof %d of the batch (index %d)" % (slot, 10 + slot) in msg and "lookup %d " % lookup in msg, msg
    adv, inst, lens = stack(kd, [make(300 + b) for b in range(B)])
    proofs = pk.prove_batch(adv, inst, lens, SEED, first_proof_index=10)
    for b in range(B):
        assert proofs[b] == okey.prove(adv[b], inst[b], lens, SEED, proof_index=10 + b), "%s: honest proof %d after the refusal" % (name, b)


def _honest(kd, make, pk, n, first=0):
    adv, inst, lens = stack(kd, [make(400 + b) for b in range(n)])
    return pk.prove_batch(adv, inst, lens, SEED, first_proof_index=first), inst, lens


@pytest.mark.parametrize("name", MUTANT_SHAPES)
def test_every_mutant_in_one_call_matches_the_oracle(keys, name):
    kd, make, okey, pk = keys(name)
    (proof, other), inst, lens = _honest(kd, make, pk, 2)
    muts = sc.mutants(kd, proof, other)
    same = [m for m in muts if len(m[3]) == len(proof)]
    batch = [proof] + [m for _, _, _, m in same]
    batch.insert(len(batch) // 2, proof)
    batch.append(proof)
    labels = ["honest"] + [lbl for lbl, _, _, _ in same]
    labels.insert(len(labels) // 2, "honest")
    labels.append("honest")
    want = [okey.verify(inst[0], lens, p) == 0 for p in batch]
    assert sum(want) == 3, "%s: the oracle accepts a mutant" % name
    insts = np.stack([inst[0]] * len(batch))
    got = pk.verify_batch(insts, lens, batch)
    wrong = [lbl for lbl, g, w in zip(labels, got, want) if g != w]
    assert got == want, "%s: %d verdicts differ from the oracle's, e.g. %s" % (name, sum(g != w for g, w in zip(got, want)), wrong[:8])
    for label, _, _, m in muts:
        if len(m) != len(proof):
            assert okey.verify(inst[0], lens, m) != 0
            assert _verify_raw(pk, inst[:1], lens, [m], len(m), len(m)) == [False], "%s: %s accepted" % (name, label)
    # a stride wider than the proof, with garbage in the gap, changes nothing
    wide = _verify_raw(pk, insts, lens, batch, len(proof) + 40, len(proof), garbage=True)
    assert wide == want, name


def _verify_raw(pk, inst, lens, proofs, stride, plen, garbage=False):
    """tb_verify_batch through ctypes: -> verdicts, or the status when the call is refused."""
    K = len(proofs)
    buf = np.frombuffer(random.Random(stride).randbytes(K * stride), np.uint8).copy() if garbage else np.zeros(K * stride, np.uint8)
    for i, p in enumerate(proofs):
        buf[i * stride:i * stride + len(p)] = np.frombuffer(p, np.uint8)
    inst = np.ascontiguousarray(inst, dtype=np.uint8)
    lens = np.ascontiguousarray(lens, dtype=np.uint32)
    ok = np.zeros(max(K, 1), np.uint8)
    ctx = pk.ctx
    st = ctx._lib.tb_verify_batch(ctx._h, pk._h, K, inst.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p),
                                  buf.ctypes.data_as(ctypes.c_void_p), stride, plen, ok.ctypes.data_as(ctypes.c_void_p))
    if st != lib.TB_OK:
        return st
    return [bool(v) for v in ok[:K]]


def test_batch_sizes_and_argument_edges(keys):
    kd, make, okey, pk = keys("standard_plonk")
    proofs, inst, lens = _honest(kd, make, pk, 4)
    muts = [m for _, _, kind, m in sc.mutants(kd, proofs[0], proofs[1]) if kind in ("negated", "other", "v+1", "x+q", "v+p", "identity")]
    pool = list(zip(proofs, inst)) + [(m, inst[0]) for m in random.Random(1).sample(muts, 12)]   # (proof, its instance)
    alone = [pk.verify_batch(i[None], lens, [p])[0] for p, i in pool]
    assert alone == [True] * 4 + [False] * 12
    r = random.Random(2)
    for K in (1, 31, 32, 33, 4096):
        pick = [r.randrange(len(pool)) for _ in range(K)]
        got = pk.verify_batch(np.stack([pool[i][1] for i in pick]), lens, [pool[i][0] for i in pick])
        assert got == [alone[i] for i in pick], "K=%d" % K
    # more than 4096 proofs are refused, and the context verifies afterwards
    big = np.stack([inst[0]] * 4097)
    assert _verify_raw(pk, big, lens, [proofs[0]] * 4097, len(proofs[0]), len(proofs[0])) == lib.TB_ERR_INVALID
    assert pk.verify_batch(inst[:2], lens, proofs[:2]) == [True, True]
    # an instance column longer than the usable rows is refused
    usable = kd.n - (kd.blinding_factors + 1)
    long_inst = np.zeros((1, 32 * (usable + 1)), np.uint8)
    assert _verify_raw(pk, long_inst, np.array([usable + 1], np.uint32), proofs[:1], len(proofs[0]), len(proofs[0])) == lib.TB_ERR_INVALID
    assert pk.verify_batch(inst[:2], lens, proofs[:2]) == [True, True]
    # an instance value written as v + p: the same value mod p, rejected by both verifiers
    noncanon = inst[:1].copy()
    v = int.from_bytes(noncanon[0, :32].tobytes(), "little") + cr.P
    assert v < 1 << 256
    noncanon[0, :32] = np.frombuffer(v.to_bytes(32, "little"), np.uint8)
    assert pk.verify_batch(noncanon, lens, proofs[:1]) == [False]
    assert okey.verify(noncanon[0], lens, proofs[0]) != 0


def test_instance_moved_between_columns_is_rejected(keys):
    kd, make, okey, pk = keys("three_instance")
    proofs, inst, lens = _honest(kd, make, pk, 1)
    assert pk.verify_batch(inst, lens, proofs) == [True]
    moved = lens.copy()
    moved[0] -= 1
    moved[1] += 1
    assert moved.sum() == lens.sum()
    assert pk.verify_batch(inst, moved, proofs) == [False]
    assert okey.verify(inst[0], moved, proofs[0]) != 0


@pytest.mark.parametrize("what", ["fixed", "sigma"])
def test_key_differing_in_one_cell_rejects(keys, what):
    """The same circuit description and transcript representation, one fixed value or one copy different: reject."""
    kd, make, okey, pk = keys("sets16_deg3")
    proofs, inst, lens = _honest(kd, make, pk, 1)
    kd2 = copy.copy(kd)
    if what == "fixed":
        kd2.fixed = kd.fixed.copy()
        kd2.fixed[0, 1, 0] ^= 1
    else:                     # two cells exchange their successors: two cycles merge or one splits
        kd2.sigma = kd.sigma.copy()
        kd2.sigma[[0, 1], 0] = kd.sigma[[1, 0], 0]
    pk2 = pk.srs.load_circuit(kd2)
    try:
        assert pk2.verify_batch(inst, lens, proofs) == [False]
        assert pk.verify_batch(inst, lens, proofs) == [True]
    finally:
        pk2.close()


def test_k15_compliance_mutants_and_violation(gpu_srs, oracle_cpu, srs_fixture):
    """The reference's size: one mutant per (section, kind) and a broken copy, against the C++ oracle verifier."""
    kd, make = ct.build(True)
    okey = oracle_cpu.OracleKey(kd, srs_fixture)
    pk = gpu_srs.load_circuit(kd)
    asg = make(50)
    for col, row in [cell for pair in asg.copies for cell in pair if cell[0].kind == 0][:4]:
        broken = make(50)      # an advice cell of a copy, plus one: a copy breaks (a lookup may break too: then the next cell)
        broken.advice[col.index][row] = (broken.advice[col.index].get(row, 0) + 1) % cr.P
        adv, inst, lens = stack(kd, [asg, make(51), broken])
        try:
            ref = okey.prove(adv[2], inst[2], lens, SEED, proof_index=2)
            break
        except RuntimeError:
            continue
    proofs = pk.prove_batch(adv, inst, lens, SEED, first_proof_index=0)
    assert proofs[2] == ref, "the proof of a broken copy differs from the oracle's"
    assert okey.verify(inst[2], lens, proofs[2]) != 0
    seen, batch = set(), []
    for label, section, kind, m in sc.mutants(kd, proofs[0], proofs[1]):
        if (section, kind) not in seen and len(m) == len(proofs[0]):
            seen.add((section, kind))
            batch.append((label, m))
    want = [okey.verify(inst[0], lens, m) == 0 for _, m in batch]
    assert not any(want)
    got = pk.verify_batch(np.stack([inst[0]] * (len(batch) + 1) + [inst[1]]), lens, [proofs[0]] + [m for _, m in batch] + [proofs[1]])
    assert got == [True] + want + [True], [lbl for (lbl, _), g in zip(batch, got[1:]) if g]
    assert pk.verify_batch(inst[1:], lens, proofs[1:]) == [True, False]
    pk.close()
