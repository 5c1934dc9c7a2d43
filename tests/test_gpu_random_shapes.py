"""GPU parity on random and boundary constraint systems (taiga_b200/circuits_random.py; the same shapes and seeds the CPU
file test_random_shapes_oracle.py proves on the oracle).  For every shape the CUDA prover's keygen commitments and proofs
of two distinct witnesses must equal the oracle's byte for byte; a mismatch is reported by proof section.  Each shape is
proved once more under one set of tuning knobs, and shapes beyond the supported envelope (three shapes, and a circuit with
more rows than the Kate division divides) must be refused at load."""
import numpy as np
import pytest

from taiga_b200 import circuits_random as cr
from taiga_b200 import lib
from taiga_b200.circuit import Assignment, CircuitKeyData, ConstraintSystem

from test_random_shapes_oracle import SHAPES, shape

pytestmark = pytest.mark.gpu

# the knob sets of test_tuning_knobs_do_not_change_results, plus the quotient without the degree split
KNOB_SETS = [{"TB_MSM_BA_MIN_TERMS": "0"}, {"TB_MSM_BA_MIN_TERMS": "0", "TB_MSM_BA_ROUNDS": "2", "TB_MSM_BA_CHUNK": "3"}, {"TB_Q_SPLIT": "0"}]
SPLIT_SHAPE = ("boundary", "split_mixed_degrees")


@pytest.fixture(scope="module")
def srs_for(gpu_ctx, oracle_cpu):
    cache = {}

    def get(k):
        if k not in cache:
            s = oracle_cpu.synthetic_srs(k, seed=k)
            cache[k] = (s, gpu_ctx.load_srs(k, s["g"], s["g_lagrange"], s["w"], s["u"]))
        return cache[k]
    yield get
    for _, g in cache.values():
        g.close()


def first_difference(kd, got, want):
    if len(got) != len(want):
        return "length %d, the oracle's is %d" % (len(got), len(want))
    i = next(i for i in range(len(want)) if got[i] != want[i])
    return "first differing byte %d: %s" % (i, cr.section_of(kd, i))


@pytest.mark.parametrize("i,which", list(enumerate(SHAPES)), ids=["%s-%s" % w for w in SHAPES])
def test_shape_proofs_bit_identical(gpu_ctx, oracle_cpu, srs_for, monkeypatch, capfd, i, which):
    kd, make = shape(which)
    d = cr.describe(kd)
    srs, gsrs = srs_for(kd.k)
    okey = oracle_cpu.OracleKey(kd, srs)
    if which == SPLIT_SHAPE:   # this shape exists to turn on the low / high degree split of the quotient programs
        monkeypatch.setenv("TB_DEBUG", "1")
        capfd.readouterr()
    pk = gsrs.load_circuit(kd)
    if which == SPLIT_SHAPE:
        err = capfd.readouterr().err
        monkeypatch.delenv("TB_DEBUG")
        assert "split on" in err, "%s: the degree split stayed off:\n%s" % (d["id"], err)
    assert pk.proof_len == kd.proof_size(), d["id"]
    gf, gs = pk.commitments()
    of, os_ = okey.commitments()
    assert gf.tobytes() == of.tobytes() and gs.tobytes() == os_.tobytes(), "%s: keygen commitments differ from the oracle's" % d["id"]

    wit = [kd.witness_arrays(make(w)) for w in (11, 12)]
    adv, inst, lens = np.stack([w[0] for w in wit]), np.stack([w[1] for w in wit]), wit[0][2]
    seed = bytes((5 * j + 3) & 0xFF for j in range(32))
    proofs = pk.prove_batch(adv, inst, lens, seed, first_proof_index=3)
    assert proofs[0] != proofs[1]
    for b in range(2):
        ref = okey.prove(wit[b][0], wit[b][1], lens, seed, proof_index=3 + b)
        if proofs[b] != ref:
            pytest.fail("%s: proof %d differs from the oracle, %s" % (d["id"], b, first_difference(kd, proofs[b], ref)))
    assert pk.verify_batch(inst, lens, proofs) == [True, True], d["id"]
    a, e = dict((n, (s, t)) for n, s, t in cr.proof_sections(kd))["evaluations"]
    bad = bytearray(proofs[0])
    bad[(a + e) // 2] ^= 1
    assert pk.verify_batch(inst, lens, [bytes(bad), proofs[1]]) == [False, True], d["id"]

    knobs = KNOB_SETS[i % len(KNOB_SETS)]
    for k_, v_ in knobs.items():
        monkeypatch.setenv(k_, v_)
    again = gsrs.load_circuit(kd).prove_batch(adv, inst, lens, seed, first_proof_index=3)   # TB_Q_SPLIT is read at load
    for b in range(2):
        if again[b] != proofs[b]:
            pytest.fail("%s under %s: proof %d changed, %s" % (d["id"], knobs, b, first_difference(kd, again[b], proofs[b])))


def _too_many_perm_columns(k):
    """Degree 3 (one column per permutation set) with 17 equality-enabled columns: one set more than the prover supports."""
    cs = ConstraintSystem()
    for _ in range(17):
        cs.enable_equality(cs.advice_column())
    return CircuitKeyData(cs, k, Assignment(cs, k), name="perm17")


def _rotation(k, rot):
    cs = ConstraintSystem()
    a, b, q = cs.advice_column(), cs.advice_column(), cs.selector()
    cs.create_gate("far", [cs.query(q) * (cs.query(a, rot) - cs.query(b))])
    return CircuitKeyData(cs, k, Assignment(cs, k), name="rot%d" % rot)


@pytest.mark.parametrize("build", [_too_many_perm_columns, lambda k: _rotation(k, 128), lambda k: _rotation(k, -129)],
                         ids=["perm_columns_17_at_degree_3", "rotation_128", "rotation_-129"])
def test_shapes_beyond_the_envelope_are_refused(gpu_ctx, oracle_cpu, srs_for, build):
    """tb_circuit_load refuses the shape with TB_ERR_INVALID, and the context proves a valid shape afterwards."""
    kd_ok, make = cr.boundary("deg4")
    srs, gsrs = srs_for(kd_ok.k)
    kd = build(kd_ok.k)
    assert kd.degree == 3
    with pytest.raises(lib.TaigaB200Error) as e:
        gsrs.load_circuit(kd)
    assert e.value.status == lib.TB_ERR_INVALID, str(e.value)
    adv, inst, lens = kd_ok.witness_arrays(make(4))
    seed = bytes(range(32))
    proof = gsrs.load_circuit(kd_ok).prove_batch(adv[None], inst[None], lens, seed, first_proof_index=9)[0]
    assert proof == oracle_cpu.OracleKey(kd_ok, srs).prove(adv, inst, lens, seed, proof_index=9)


def test_circuit_beyond_the_kate_division_is_refused_at_load(gpu_ctx, oracle_cpu, srs_for, srs_fixture):
    """k = 16: the multiopen's Kate division divides at most 2^15 coefficients, so tb_circuit_load refuses the circuit
    (TB_ERR_INVALID, naming the limit) instead of tb_prove_batch failing after the rest of the proof.  The refusal comes
    before the SRS's points are read, so the k = 15 fixture's points, repeated to 2^16, stand in for a k = 16 SRS."""
    s = srs_fixture
    g16 = gpu_ctx.load_srs(16, np.concatenate([s["g"], s["g"]]), np.concatenate([s["g_lagrange"], s["g_lagrange"]]), s["w"], s["u"])
    try:
        with pytest.raises(lib.TaigaB200Error) as e:
            g16.load_circuit(_rotation(16, 1))
        assert e.value.status == lib.TB_ERR_INVALID, str(e.value)
        assert "Kate division" in str(e.value) and str(1 << 15) in str(e.value), str(e.value)
    finally:
        g16.close()
    kd_ok, make = cr.boundary("deg4")
    srs, gsrs = srs_for(kd_ok.k)
    adv, inst, lens = kd_ok.witness_arrays(make(4))
    seed = bytes(range(32))
    proof = gsrs.load_circuit(kd_ok).prove_batch(adv[None], inst[None], lens, seed, first_proof_index=9)[0]
    assert proof == oracle_cpu.OracleKey(kd_ok, srs).prove(adv, inst, lens, seed, proof_index=9)
