"""GPU: verification from the verifying key alone (tb_vk_load / tb_verify_batch_vk) and the batched point decoder
(tb_decompress, the kernel that decodes every point of a batch before the transcripts are replayed).

* Decoding: the device decoder gives verifier_py's point and verdict on every chunk of the golden proofs, on x + q aliases,
  negative zero, the identity with and without the sign bit, x off the curve, and 10 000 random points of both parities.
* Every shape the repository proves on the GPU (mini circuits, boundary shapes, random seeds, both Taiga shapes at k = 15
  in batches of 1, 64 and 65) and the golden proofs are accepted, with the verdicts of tb_verify_batch.
* The soundness inputs of tests/soundness_cases.py get the verdicts of tb_verify_batch, the C++ oracle and verifier_py,
  and a proof's verdict does not depend on the rest of its batch.
* A vk made of the proving key's commitments, kept as bytes, verifies on a fresh context after the key and its context
  are gone; a vk with two fixed commitments swapped, one sigma commitment replaced or another transcript representation
  rejects every proof; malformed commitments and descriptions (among them an equality-enabled column without its
  rotation-0 query) are refused and the context keeps working."""
import copy
import ctypes
import os
import random

import numpy as np
import pytest

import soundness_cases as sc
from conftest import GOLDEN
from oracle import verifier_py as vp
from taiga_b200 import circuits_mini as cm
from taiga_b200 import circuits_random as cr
from taiga_b200 import circuits_taiga as ct
from taiga_b200 import lib
from taiga_b200.circuit import TbCsDesc, TbQuery

from test_gpu_verifier_soundness import PROVE_SHAPES, stack
from test_verifier_soundness import MUTANT_SHAPES, SEED, References, mutant_shape
from test_vk_host import encodings_of, ref_decode

pytestmark = pytest.mark.gpu

MINI = [(6, False, 2), (7, True, 1), (6, False, 0), (9, True, 2), (12, False, 1)]
RANDOM = [("boundary", name) for name, _ in cr.BOUNDARY] + [("seed", s) for s in range(8)]
GOLDEN_K6_SEED = bytes((7 * i + 1) & 0xFF for i in range(32))


@pytest.fixture(scope="module")
def srs_for(gpu_ctx, oracle_cpu):
    """k -> (synthetic SRS arrays, device SRS); the SRS every GPU test of a small shape uses (seed = k)."""
    cache = {}

    def get(k):
        if k not in cache:
            s = oracle_cpu.synthetic_srs(k, seed=k)
            cache[k] = (s, gpu_ctx.load_srs(k, s["g"], s["g_lagrange"], s["w"], s["u"]))
        return cache[k]
    yield get
    for _, g in cache.values():
        g.close()


def _verify_raw(ctx, fn, h, inst, lens, proofs, stride, plen):
    """tb_verify_batch / tb_verify_batch_vk through ctypes: -> verdicts, or the status when the call is refused."""
    K = len(proofs)
    buf = np.zeros(K * stride, np.uint8)
    for i, p in enumerate(proofs):
        buf[i * stride:i * stride + len(p)] = np.frombuffer(p, np.uint8)
    inst = np.ascontiguousarray(inst, dtype=np.uint8)
    lens = np.ascontiguousarray(lens, dtype=np.uint32)
    ok = np.zeros(max(K, 1), np.uint8)
    st = getattr(ctx._lib, fn)(ctx._h, h, K, inst.ctypes.data_as(ctypes.c_void_p), lens.ctypes.data_as(ctypes.c_void_p),
                               buf.ctypes.data_as(ctypes.c_void_p), stride, plen, ok.ctypes.data_as(ctypes.c_void_p))
    return [bool(v) for v in ok[:K]] if st == lib.TB_OK else st


def both(pk, vk, inst, lens, proofs):
    """verdicts of the proving-key and the verifying-key verifier, which must agree"""
    a, b = pk.verify_batch(inst, lens, proofs), vk.verify_batch(inst, lens, proofs)
    assert a == b, "tb_verify_batch %s, tb_verify_batch_vk %s" % (a, b)
    return b


def _honest(kd, make, pk, n, first=0, w0=400):
    adv, inst, lens = stack(kd, [make(w0 + b) for b in range(n)])
    return pk.prove_batch(adv, inst, lens, SEED, first_proof_index=first), inst, lens


# ---------------------------------------------------------------- decoding
def _device_decode(ctx, encs):
    pts, ok = ctx.decompress(np.frombuffer(b"".join(encs), np.uint8))
    out = []
    for p, good in zip(pts, ok):
        if not good:
            assert not p.any()
            out.append("reject")
            continue
        x, y = int.from_bytes(p[:32].tobytes(), "little"), int.from_bytes(p[32:].tobytes(), "little")
        out.append(None if x == 0 and y == 0 else (x, y))
    return out


def test_decoder_matches_verifier_py(gpu_ctx):
    encs = []
    for name in ("proof_k6_plonk.bin", "proof_k15_compliance_shape.bin", "proof_k15_vp_shape.bin"):
        proof = open(os.path.join(GOLDEN, name), "rb").read()
        for off in range(0, len(proof), 32):
            encs += encodings_of(proof[off:off + 32])
    encs += [bytes(32), (1 << 255).to_bytes(32, "little"), (vp.Q | 1 << 255).to_bytes(32, "little"), vp.Q.to_bytes(32, "little"),
             ((1 << 255) - 1).to_bytes(32, "little"), bytes([0xFF] * 32)]
    got = _device_decode(gpu_ctx, encs)
    want = [ref_decode(e) for e in encs]
    bad = [(e.hex(), g, w) for e, g, w in zip(encs, got, want) if g != w]
    assert not bad, "%d of %d encodings decode differently, e.g. %s" % (len(bad), len(encs), bad[:3])
    assert got[-6] is None and all(g == "reject" for g in got[-5:])
    assert sum(w == "reject" for w in want) > 1000 and sum(isinstance(w, tuple) for w in want) > 400


def test_decoder_on_random_points_of_both_parities(gpu_ctx):
    rnd = random.Random(11)
    xs = []
    while len(xs) < 5000:
        x = rnd.randrange(vp.Q)
        if pow(x ** 3 + 5, (vp.Q - 1) // 2, vp.Q) == 1:
            xs.append(x)
    encs = [(x | s << 255).to_bytes(32, "little") for x in xs for s in (0, 1)]
    got = _device_decode(gpu_ctx, encs)
    assert got == [ref_decode(e) for e in encs]
    for e, p in zip(encs, got):
        assert p[1] & 1 == e[31] >> 7 and (p[1] ** 2 - p[0] ** 3 - 5) % vp.Q == 0


# ---------------------------------------------------------------- every shape proved on the GPU
@pytest.mark.parametrize("k,wide,nl", MINI)
def test_mini_circuits_accepted(srs_for, k, wide, nl):
    kd, make = cm.standard_plonk(k=k, wide=wide, n_lookups=nl)
    _, gsrs = srs_for(k)
    pk = gsrs.load_circuit(kd)
    vk = pk.verifying_key()
    assert vk.proof_len == pk.proof_len == kd.proof_size()
    proofs, inst, lens = _honest(kd, make, pk, 3)
    assert both(pk, vk, inst, lens, proofs) == [True] * 3
    bad = bytearray(proofs[1])
    bad[len(bad) // 2] ^= 1
    assert both(pk, vk, inst, lens, [proofs[0], bytes(bad), proofs[2]]) == [True, False, True]
    if (k, wide, nl) == (6, False, 2):   # the golden proof: witness 100, proof index 5
        adv, inst1, lens1 = kd.witness_arrays(make(100))
        golden = open(os.path.join(GOLDEN, "proof_k6_plonk.bin"), "rb").read()
        assert pk.prove_batch(adv[None], inst1[None], lens1, GOLDEN_K6_SEED, first_proof_index=5)[0] == golden
        assert both(pk, vk, inst1[None], lens1, [golden]) == [True]
    vk.close()
    pk.close()


@pytest.mark.parametrize("which", RANDOM, ids=["%s-%s" % w for w in RANDOM])
def test_random_and_boundary_shapes_accepted(srs_for, which):
    kind, v = which
    kd, make = cr.boundary(v) if kind == "boundary" else cr.random_shape(v)
    _, gsrs = srs_for(kd.k)
    pk = gsrs.load_circuit(kd)
    f, s = pk.commitments()
    vk = gsrs.load_verifying_key(kd, f, s)
    proofs, inst, lens = _honest(kd, make, pk, 2, w0=11)
    assert both(pk, vk, inst, lens, proofs) == [True, True]
    a, e = dict((n, (s_, t)) for n, s_, t in cr.proof_sections(kd))["evaluations"]
    bad = bytearray(proofs[0])
    bad[(a + e) // 2] ^= 1
    assert both(pk, vk, inst, lens, [bytes(bad), proofs[1]]) == [False, True]
    vk.close()
    pk.close()


@pytest.mark.parametrize("compliance", [True, False], ids=["compliance", "vp"])
def test_taiga_shapes_in_batches_of_1_64_65(gpu_srs, compliance):
    kd, make = ct.build(compliance)
    pk = gpu_srs.load_circuit(kd)
    vk = pk.verifying_key()
    wit = [kd.witness_arrays(make(40 + w)) for w in range(4)]
    adv = np.stack([wit[b % 4][0] for b in range(65)])
    inst = np.stack([wit[b % 4][1] for b in range(65)])
    lens = wit[0][2]
    proofs = pk.prove_batch(adv, inst, lens, bytes(range(100, 132)))
    assert len(set(proofs)) == 65
    for B in (1, 64, 65):
        assert both(pk, vk, inst[:B], lens, proofs[:B]) == [True] * B, B
    bad = bytearray(proofs[33])
    bad[100] ^= 1
    mixed = proofs[:33] + [bytes(bad)] + proofs[34:]
    assert both(pk, vk, inst, lens, mixed) == [b != 33 for b in range(65)]
    # the golden proof of the shape: witness 41, proof index 1
    golden = open(os.path.join(GOLDEN, "proof_k15_compliance_shape.bin" if compliance else "proof_k15_vp_shape.bin"), "rb").read()
    assert both(pk, vk, wit[1][1][None], lens, [golden]) == [True]
    vk.close()
    pk.close()


# ---------------------------------------------------------------- soundness inputs
@pytest.fixture(scope="module")
def keys(srs_for, oracle_cpu):
    """name -> (kd, make, References, proving key, verifying key)"""
    cache = {}

    def get(name):
        if name not in cache:
            kd, make = mutant_shape(name)
            _, gsrs = srs_for(kd.k)
            pk = gsrs.load_circuit(kd)
            cache[name] = (kd, make, References(oracle_cpu, kd), pk, pk.verifying_key())
        return cache[name]
    yield get
    for v in cache.values():
        v[4].close()
        v[3].close()


@pytest.mark.parametrize("name", MUTANT_SHAPES)
def test_mutants_get_the_verdicts_of_every_verifier(keys, name):
    kd, make, ref, pk, vk = keys(name)
    (proof, other), inst, lens = _honest(kd, make, pk, 2)
    muts = sc.mutants(kd, proof, other)
    same = [m for m in muts if len(m[3]) == len(proof)]
    batch = [proof] + [m for _, _, _, m in same] + [proof]
    labels = ["honest"] + [lbl for lbl, _, _, _ in same] + ["honest"]
    insts = np.stack([inst[0]] * len(batch))
    got = both(pk, vk, insts, lens, batch)
    want = [ref.key.verify(inst[0], lens, p) == 0 for p in batch]
    wrong = [lbl for lbl, g, w in zip(labels, got, want) if g != w]
    assert got == want and sum(got) == 2, "%s: verdicts differ from the oracle's: %s" % (name, wrong[:8])
    # verifier_py on one mutant of every (section, kind), in this process (no fork of a process that holds a CUDA context)
    seen, py = set(), []
    for i, (label, section, kind, m) in enumerate(same):
        if (section, kind) not in seen:
            seen.add((section, kind))
            py.append(i + 1)
    assert [got[i] for i in py] == [ref.py_verify(inst[0], lens, batch[i]) for i in py], name
    # a proof one byte or 32 bytes too short or too long is rejected by both, on its own
    for label, _, _, m in muts:
        if len(m) != len(proof):
            for fn, h in (("tb_verify_batch", pk._h), ("tb_verify_batch_vk", vk._h)):
                assert _verify_raw(pk.ctx, fn, h, inst[:1], lens, [m], len(m), len(m)) == [False], "%s %s: %s accepted" % (name, fn, label)
            assert not ref.py_verify(inst[0], lens, m)
    # each verdict is the proof's own: random sub-batches give the verdicts of one big batch
    r = random.Random(name)
    for K in (1, 7, 33):
        pick = [r.randrange(len(batch)) for _ in range(K)]
        assert vk.verify_batch(np.stack([inst[0]] * K), lens, [batch[i] for i in pick]) == [got[i] for i in pick], (name, K)


@pytest.mark.parametrize("name", PROVE_SHAPES)
def test_false_statements_rejected(keys, name):
    kd, make, ref, pk, vk = keys(name)
    bad = [(label, asg) for label, asg in sc.violations(kd, make, 5) if not label.startswith("lookup")]
    batch = [("honest", make(100))] + bad + [("honest", make(101))]
    adv, inst, lens = stack(kd, [a for _, a in batch])
    proofs = pk.prove_batch(adv, inst, lens, SEED, first_proof_index=0)
    assert both(pk, vk, inst, lens, proofs) == [label == "honest" for label, _ in batch], name
    for (label, _), p, i in zip(batch, proofs, inst):
        if label != "honest":
            assert not ref.py_verify(i, lens, p), "%s %s: verifier_py accepts" % (name, label)


def test_instances_the_verifier_must_refuse_or_reject(keys):
    kd, make, ref, pk, vk = keys("three_instance")
    proofs, inst, lens = _honest(kd, make, pk, 2)
    assert both(pk, vk, inst, lens, proofs) == [True, True]
    moved = lens.copy()
    moved[0] -= 1
    moved[1] += 1
    assert both(pk, vk, inst, moved, proofs) == [False, False]
    noncanon = inst.copy()
    v = int.from_bytes(noncanon[0, :32].tobytes(), "little") + cr.P
    noncanon[0, :32] = np.frombuffer(v.to_bytes(32, "little"), np.uint8)
    assert both(pk, vk, noncanon, lens, proofs) == [False, True]
    usable = kd.n - (kd.blinding_factors + 1)
    long_lens = lens.copy()
    long_lens[0] = usable + 1
    long_inst = np.zeros((1, 32 * int(long_lens.sum())), np.uint8)
    for fn, h in (("tb_verify_batch", pk._h), ("tb_verify_batch_vk", vk._h)):
        assert _verify_raw(pk.ctx, fn, h, long_inst, long_lens, proofs[:1], len(proofs[0]), len(proofs[0])) == lib.TB_ERR_INVALID
        assert _verify_raw(pk.ctx, fn, h, np.stack([inst[0]] * 4097), lens, [proofs[0]] * 4097, len(proofs[0]), len(proofs[0])) == lib.TB_ERR_INVALID
    assert vk.verify_batch(inst, lens, proofs) == [True, True]


# ---------------------------------------------------------------- the verifying key itself
def test_vk_outlives_the_proving_key_and_its_context(oracle_cpu):
    kd, make = cm.standard_plonk(k=7, wide=True, n_lookups=1)
    s = oracle_cpu.synthetic_srs(7, seed=7)
    ctx1 = lib.Context(0)
    srs1 = ctx1.load_srs(7, s["g"], s["g_lagrange"], s["w"], s["u"])
    pk = srs1.load_circuit(kd)
    proofs, inst, lens = _honest(kd, make, pk, 3)
    f, sg = pk.commitments()
    f, sg = f.tobytes(), sg.tobytes()
    pk.close()
    srs1.close()
    ctx1.close()
    ctx2 = lib.Context(0)
    srs2 = ctx2.load_srs(7, s["g"], s["g_lagrange"], s["w"], s["u"])
    kd2 = copy.copy(kd)    # the vk reads the description only: no fixed or sigma value
    kd2.fixed, kd2.sigma = np.zeros_like(kd.fixed), np.zeros_like(kd.sigma)
    vk = srs2.load_verifying_key(kd2, np.frombuffer(f, np.uint8).reshape(-1, 64), np.frombuffer(sg, np.uint8).reshape(-1, 64))
    assert vk.verify_batch(inst, lens, proofs) == [True] * 3
    bad = bytearray(proofs[2])
    bad[-40] ^= 1
    assert vk.verify_batch(inst, lens, proofs[:2] + [bytes(bad)]) == [True, True, False]
    ok = oracle_cpu.OracleKey(kd, s).commitments()
    assert ok[0].tobytes() == f and ok[1].tobytes() == sg
    vk.close()
    srs2.close()
    ctx2.close()


def _with_desc(kd, **changes):
    """a shallow copy of kd whose descriptor differs in `changes` (vk_transcript_repr: a byte string)"""
    d = TbCsDesc.from_buffer_copy(kd.desc)
    for k, v in changes.items():
        if k == "vk_transcript_repr":
            d.vk_transcript_repr = (ctypes.c_uint8 * 32)(*v)
        else:
            setattr(d, k, v)
    kd2 = copy.copy(kd)
    kd2.desc = d
    return kd2


def _negate(pt):
    y = int.from_bytes(pt[32:].tobytes(), "little")
    out = pt.copy()
    out[32:] = np.frombuffer(((vp.Q - y) % vp.Q).to_bytes(32, "little"), np.uint8)
    return out


def test_wrong_vk_rejects_every_proof(srs_for):
    kd, make = cm.standard_plonk(k=6, n_lookups=2)
    _, gsrs = srs_for(6)
    pk = gsrs.load_circuit(kd)
    proofs, inst, lens = _honest(kd, make, pk, 3)
    f, s = pk.commitments()
    i, j = next((i, j) for i in range(len(f)) for j in range(i + 1, len(f)) if f[i].tobytes() != f[j].tobytes())
    swapped = f.copy()
    swapped[[i, j]] = f[[j, i]]
    sig = s.copy()
    sig[1] = _negate(s[1])
    repr_ = bytearray(bytes(kd.desc.vk_transcript_repr))
    repr_[0] ^= 1
    right = gsrs.load_verifying_key(kd, f, s)
    assert right.verify_batch(inst, lens, proofs) == [True] * 3
    for what, vk in (("fixed commitments %d and %d swapped" % (i, j), gsrs.load_verifying_key(kd, swapped, s)),
                     ("sigma commitment 1 negated", gsrs.load_verifying_key(kd, f, sig)),
                     ("another transcript representation", gsrs.load_verifying_key(_with_desc(kd, vk_transcript_repr=bytes(repr_)), f, s))):
        assert vk.verify_batch(inst, lens, proofs) == [False] * 3, what
        vk.close()
    right.close()
    pk.close()


def test_refused_loads_leave_the_context_usable(srs_for):
    kd, make = cm.standard_plonk(k=6, n_lookups=2)
    _, gsrs = srs_for(6)
    _, gsrs7 = srs_for(7)
    pk = gsrs.load_circuit(kd)
    proofs, inst, lens = _honest(kd, make, pk, 2)
    f, s = pk.commitments()
    c = next(i for i in range(len(f)) if f[i].any())
    off_curve = f.copy()
    y = int.from_bytes(f[c, 32:].tobytes(), "little")
    off_curve[c, 32:] = np.frombuffer(((y + 1) % vp.Q).to_bytes(32, "little"), np.uint8)
    x_alias = f.copy()       # x + q: the same x mod q, not canonical
    x_alias[c, :32] = np.frombuffer((int.from_bytes(f[c, :32].tobytes(), "little") + vp.Q).to_bytes(32, "little"), np.uint8)
    y_alias = s.copy()
    y_alias[0, 32:] = np.frombuffer((int.from_bytes(s[0, 32:].tobytes(), "little") + vp.Q).to_bytes(32, "little"), np.uint8)
    cases = [("off-curve fixed commitment", lambda: gsrs.load_verifying_key(kd, off_curve, s), "not on the curve"),
             ("x >= q", lambda: gsrs.load_verifying_key(kd, x_alias, s), "not below q"),
             ("y >= q", lambda: gsrs.load_verifying_key(kd, f, y_alias), "not below q"),
             ("k of another SRS", lambda: gsrs7.load_verifying_key(kd, f, s), "circuit k must match the SRS"),
             ("malformed description", lambda: gsrs.load_verifying_key(_with_desc(kd, cs_degree=2), f, s), "unsupported constraint system shape"),
             ("constraint root out of range", lambda: gsrs.load_verifying_key(_with_desc(kd, num_nodes=0), f, s), "out of range")]
    for what, load, msg in cases:
        with pytest.raises(lib.TaigaB200Error) as e:
            load()
        assert e.value.status == lib.TB_ERR_INVALID and msg in str(e.value), (what, str(e.value))
        vk = gsrs.load_verifying_key(kd, f, s)
        assert vk.verify_batch(inst, lens, proofs) == [True, True], what
        vk.close()
    pk.close()


def test_permutation_column_without_rotation_0_query_refused(srs_for):
    """halo2's enable_equality queries the column at rotation 0, and the permutation argument reads the column there: a
    descriptor that moves that query to another rotation is refused by both loads, naming the column."""
    kd, make = cm.standard_plonk(k=6, n_lookups=2)
    _, gsrs = srs_for(6)
    pk = gsrs.load_circuit(kd)
    proofs, inst, lens = _honest(kd, make, pk, 2)
    f, s = pk.commitments()
    col = kd.desc.perm_columns[0]
    field = ("advice", "fixed", "instance")[col.kind] + "_queries"
    qs = [(q.column, q.rotation) for q in getattr(kd.desc, field)[:getattr(kd.desc, "num_" + field)]]
    i = qs.index((col.index, 0))
    rot = max(r for c, r in qs if c == col.index) + 1     # a rotation the column has no other query at
    moved = (TbQuery * len(qs))(*[TbQuery(c, rot if j == i else r) for j, (c, r) in enumerate(qs)])
    bad = _with_desc(kd, **{field: moved})
    bad.moved_queries = moved
    for what, load in (("load_verifying_key", lambda: gsrs.load_verifying_key(bad, f, s)), ("load_circuit", lambda: gsrs.load_circuit(bad))):
        with pytest.raises(lib.TaigaB200Error) as e:
            load()
        assert e.value.status == lib.TB_ERR_INVALID and "permutation column 0 (" in str(e.value) and "has no rotation-0 query" in str(e.value), (what, str(e.value))
    vk = gsrs.load_verifying_key(kd, f, s)
    assert both(pk, vk, inst, lens, proofs) == [True, True]
    vk.close()
    pk.close()
