"""CPU: what both reference verifiers must reject (tests/soundness_cases.py makes the inputs).

Every one-element mutant of a proof -- non-canonical encodings of the same point or scalar, the identity, negative zero,
an x off the curve, a negated point, a slot of another proof, a wrong length -- goes through the C++ oracle verifier;
the encoding mutants and one value mutant per (section, kind) go through the independent verifier_py as well.  Proofs
the oracle prover makes of witnesses that break one gate, copy or instance copy must be rejected by both; a witness that
breaks a lookup is refused by the prover itself.  test_gpu_verifier_soundness.py sends the same inputs through the CUDA
prover and the device verifier."""
import multiprocessing

import pytest

import soundness_cases as sc
from oracle import verifier_py as vp
from taiga_b200 import circuits_mini as cm
from taiga_b200 import circuits_random as cr

from test_random_shapes_oracle import instance_columns, shape, srs_for

MUTANT_SHAPES = ["standard_plonk", "sets16_deg3", "three_instance", "rotations_3", "lookups4_wide", "no_perm_no_lookup", "no_instance",
                 "deg18_R32"]
VIOLATION_SHAPES = [("boundary", name) for name, _ in cr.BOUNDARY] + [("seed", s) for s in range(10)]
SEED = bytes((7 * j + 1) & 0xFF for j in range(32))


def mutant_shape(name):
    return cm.standard_plonk(k=6, n_lookups=2) if name == "standard_plonk" else cr.boundary(name)


class References:
    """The C++ oracle and verifier_py for one circuit (verifier_py's n-term MSM over g reuses points decoded once)."""

    def __init__(self, oracle_cpu, kd):
        self.kd, self.srs = kd, srs_for(oracle_cpu, kd.k)
        self.key = oracle_cpu.OracleKey(kd, self.srs)
        self.fc, self.sc = self.key.commitments()
        self._g = None

    def _msm_g(self, scalars):
        if self._g is None:
            self._g = [vp._from_affine(b) for b in self.srs["g"]]
        return vp.msm(scalars, self._g)

    def prove(self, asg, index):
        adv, inst, lens = self.kd.witness_arrays(asg)
        return self.key.prove(adv, inst, lens, SEED, proof_index=index), inst, lens

    def py_verify(self, inst, lens, proof):
        return vp.verify(self.kd, self.srs, self.fc, self.sc, instance_columns(self.kd, inst, lens), proof, msm_big=self._msm_g)

    def py_verify_all(self, inst, lens, proofs):
        """verifier_py's verdicts on many proofs, in forked worker processes (each verdict costs tens of milliseconds)."""
        global _FORKED
        _FORKED = (self, inst, lens, proofs)
        with multiprocessing.get_context("fork").Pool(min(8, multiprocessing.cpu_count())) as pool:
            return pool.map(_py_verify_forked, range(len(proofs)), chunksize=8)


_FORKED = None


def _py_verify_forked(i):
    ref, inst, lens, proofs = _FORKED
    return ref.py_verify(inst, lens, proofs[i])


@pytest.mark.parametrize("name", MUTANT_SHAPES)
def test_every_proof_mutant_is_rejected(oracle_cpu, name):
    kd, make = mutant_shape(name)
    ref = References(oracle_cpu, kd)
    proof, inst, lens = ref.prove(make(2), 0)
    other, _, _ = ref.prove(make(3), 1)
    assert ref.key.verify(inst, lens, proof) == 0 and ref.py_verify(inst, lens, proof), "%s: the honest proof is rejected" % name
    sc.check_point_mutants(kd, proof)
    muts = sc.mutants(kd, proof, other)
    kinds = {kind for _, _, kind, _ in muts}
    assert kinds == set(sc.ENCODING_KINDS + sc.VALUE_KINDS), "%s: mutant kinds %s" % (name, sorted(kinds))

    accepted = [label for label, _, _, m in muts if ref.key.verify(inst, lens, m) == 0]
    assert not accepted, "%s: the oracle verifier accepts %d of %d mutants: %s" % (name, len(accepted), len(muts), accepted[:10])
    sampled, py = set(), []
    for label, section, kind, m in muts:
        if kind in sc.ENCODING_KINDS or (section, kind) not in sampled:
            sampled.add((section, kind))
            py.append((label, m))
    assert sampled == {(s, k) for _, s, k, _ in muts}
    accepted = [label for (label, _), ok in zip(py, ref.py_verify_all(inst, lens, [m for _, m in py])) if ok]
    assert not accepted, "%s: verifier_py accepts %d of %d mutants: %s" % (name, len(accepted), len(py), accepted[:10])


@pytest.mark.parametrize("which", VIOLATION_SHAPES, ids=["%s-%s" % w for w in VIOLATION_SHAPES])
def test_proofs_of_false_statements_are_rejected(oracle_cpu, which):
    kd, make = shape(which)
    ref = References(oracle_cpu, kd)
    cases = sc.violations(kd, make, 5)
    assert cases, "%s: no violation found" % kd.name
    for i, (label, asg) in enumerate(cases):
        if label.startswith("lookup"):
            with pytest.raises(RuntimeError, match="rc=3"):
                ref.prove(asg, i)
            continue
        proof, inst, lens = ref.prove(asg, i)
        assert ref.key.verify(inst, lens, proof) != 0, "%s %s: the oracle verifier accepts the proof" % (kd.name, label)
        assert not ref.py_verify(inst, lens, proof), "%s %s: verifier_py accepts the proof" % (kd.name, label)


def test_violation_kinds_cover_the_boundary_shapes():
    """Each kind of broken constraint is made for at least one pinned shape, so a helper that stops finding one fails here."""
    labels = set()
    for name, _ in cr.BOUNDARY:
        kd, make = cr.boundary(name)
        labels |= {label.split("-", 1)[-1] if label.startswith("gate") else label for label, _ in sc.violations(kd, make, 5)}
    want = {"out-first", "out-last", "copy-in-set", "copy-across-sets", "instance-copy", "constant-copy", "fixed-copy", "lookup0", "lookup4"}
    assert want <= labels, sorted(want - labels)
    assert any(x.startswith("read-rot-") for x in labels) and any(x.startswith("read-rot+") for x in labels), sorted(labels)
