"""CPU: random and boundary constraint systems (taiga_b200/circuits_random.py) through the oracle prover, the oracle verifier
and the independent pure-Python verifier.  Every shape must be satisfiable by construction (checked by a plain mock prover
first, so a generator mistake is not mistaken for a prover mistake), prove, have the proof length the key data predicts,
and be accepted by both verifiers, which must reject a flipped commitment byte and a flipped evaluation byte.  The same
shapes and seeds are proved on the GPU by test_gpu_random_shapes.py."""
import pytest

from oracle import verifier_py as vp
from taiga_b200 import circuits_random as cr

SEEDS = list(range(30))
SHAPES = [("boundary", name) for name, _ in cr.BOUNDARY] + [("seed", s) for s in SEEDS]
_SRS = {}


def shape(which):
    kind, v = which
    return cr.boundary(v) if kind == "boundary" else cr.random_shape(v)


def srs_for(oracle_cpu, k):
    if k not in _SRS:
        _SRS[k] = oracle_cpu.synthetic_srs(k, seed=k)
    return _SRS[k]


def instance_columns(kd, inst, lens):
    """The instance bytes as one list of ints per column (witness_arrays reports lens = [0] when there is no column)."""
    cols, off = [], 0
    for ln in lens[:kd.cs.num_instance]:
        cols.append([int.from_bytes(inst[32 * (off + i):32 * (off + i + 1)].tobytes(), "little") for i in range(int(ln))])
        off += int(ln)
    return cols


@pytest.mark.parametrize("which", SHAPES, ids=["%s-%s" % w for w in SHAPES])
def test_shape_proves_and_verifies_on_the_oracle(oracle_cpu, which):
    kd, make = shape(which)
    d = cr.describe(kd)
    asg = make(5)
    why = cr.satisfied(kd, asg)
    assert why is None, "%s: the generator made an unsatisfying witness: %s" % (d["id"], why)
    srs = srs_for(oracle_cpu, kd.k)
    key = oracle_cpu.OracleKey(kd, srs)
    adv, inst, lens = kd.witness_arrays(asg)
    proof = key.prove(adv, inst, lens, bytes(range(32)), proof_index=3)
    assert len(proof) == kd.proof_size(), d["id"]
    assert key.verify(inst, lens, proof) == 0, "%s: the oracle verifier rejects the oracle's proof" % d["id"]
    fc, sc = key.commitments()
    cols = instance_columns(kd, inst, lens)
    assert vp.verify(kd, srs, fc, sc, cols, proof), "%s: verifier_py rejects the oracle's proof" % d["id"]
    sections = {name: (a, b) for name, a, b in cr.proof_sections(kd)}
    assert sections["IPA"][1] == len(proof)
    for name in ("advice commitments", "evaluations"):
        a, b = sections[name]
        bad = bytearray(proof)
        bad[(a + b) // 2] ^= 1
        assert key.verify(inst, lens, bytes(bad)) != 0, "%s: oracle verifier accepts a flipped byte in the %s" % (d["id"], name)
        assert not vp.verify(kd, srs, fc, sc, cols, bytes(bad)), "%s: verifier_py accepts a flipped byte in the %s" % (d["id"], name)


def test_mock_prover_rejects_broken_witnesses():
    """The mock prover is what keeps generator mistakes out of the prover tests: it must see a broken gate, lookup and copy."""
    kd, make = cr.boundary("deg8")
    assert cr.satisfied(kd, make(2)) is None
    m = kd.random_shape["m"]                              # the first gate's first enabled row
    found = [cr.satisfied(kd, _bump(make(2), c, m)) for c in range(kd.cs.num_advice)]
    assert any(f and f.startswith("gate g0") for f in found), found
    kd, make = cr.boundary("lookups4_wide")               # one gate on one row: the first lookup window follows it
    rs = kd.random_shape
    row = rs["m"] + (2 * rs["m"] + 1) * len(rs["gates"]) * rs["gate_rows"]
    found = [cr.satisfied(kd, _bump(make(2), c, row + x)) for c in range(kd.cs.num_advice) for x in range(-rs["m"], rs["m"] + 1)]
    assert any(f and f.startswith("lookup 0") for f in found), found
    kd, make = cr.boundary("sets16_deg3")
    asg = make(2)
    col, row = next(cell for pair in asg.copies for cell in pair if cell[0].kind == 0)
    assert cr.satisfied(kd, _bump(asg, col.index, row)).startswith("copy")


def _bump(asg, col, row):
    asg.advice[col][row] = (asg.advice[col].get(row, 0) + 1) % cr.P
    return asg


def test_witness_structure_does_not_depend_on_the_witness_seed():
    """Keygen takes fixed columns and copies from make(1); every other witness must share them, or its proofs are of another circuit."""
    for which in [("boundary", n) for n, _ in cr.BOUNDARY[:6]] + [("seed", s) for s in range(5)]:
        kd, make = shape(which)
        a, b = make(1), make(7)
        assert a.fixed == b.fixed and a.copies == b.copies, which
        assert [len(c) for c in a.instance] == [len(c) for c in b.instance]


def test_boundary_shapes_cover_the_untested_paths():
    """Each bullet of the coverage list is met by at least one pinned shape, so dropping or weakening one fails here."""
    ds = {name: cr.describe(cr.boundary(name)[0]) for name, _ in cr.BOUNDARY}
    D = list(ds.values())
    missing = []

    def need(what, ok):
        if not ok:
            missing.append(what)
    need("degrees 4, 6, 8, 12, 16, 18", {4, 6, 8, 12, 16, 18} <= {d["degree"] for d in D})
    need("pieces < R at every degree of the form != 2^j + 1", all(d["pieces"] < d["R"] for d in D if d["degree"] in (4, 6, 8, 12, 16, 18)))
    need("R = 32", any(d["R"] == 32 for d in D))
    need("16 permutation sets at degree 3 (P = 16)", any(d["perm_sets"] == 16 and d["degree"] == 3 and d["perm_columns"] == 16 for d in D))
    need("16 permutation sets at degree 4 (P = 32)", any(d["perm_sets"] == 16 and d["degree"] == 4 and d["perm_columns"] == 32 for d in D))
    need("permutation sets 6..15", any(6 <= d["perm_sets"] < 16 for d in D) or any(d["perm_sets"] == 16 for d in D))
    need("blinding factors 6 and 8", {6, 8} <= {d["blinding_factors"] for d in D})
    need("advice rotations -3..+3", any(set(range(-3, 4)) <= set(d["advice_rotations"]) for d in D))
    need("fixed rotations +-2", any({-2, 2} <= set(d["fixed_rotations"]) for d in D))
    need("no instance column", any(d["instance_columns"] == 0 for d in D))
    need("three instance columns, one at rotation +-1, one not equality-enabled",
         any(d["instance_columns"] == 3 and {-1, 1} <= set(d["instance_rotations"]) and d["instance_eq"] < 3 for d in D))
    need("instance_len == usable", any(d["instance_full"] for d in D))
    need("four lookups", any(d["lookups"] >= 4 for d in D))
    need("a lookup of four expression pairs", any(max(d["lookup_pairs"] or [0]) >= 4 for d in D))
    need("a table expression of degree 2", any(max(d["table_degrees"] or [0]) >= 2 for d in D))
    need("lookup inputs on every usable row", any(d["full_row_lookup"] for d in D))
    need("no gates", any(d["gates"] == 0 for d in D))
    need("no permutation and no lookup", any(d["perm_sets"] + d["lookups"] == 0 for d in D))
    need("mixed-degree constraints at R >= 4 (degree split)", any(d["R"] >= 4 and d["low_constraints"] >= 8 and d["high_constraints"] >= 1 for d in D))
    need("every shape at the smallest k except one at k >= 10", all(d["k"] == d["k_min"] for n, d in ds.items() if n != "k10") and ds["k10"]["k"] >= 10)
    assert not missing, "BOUNDARY no longer covers: %s" % "; ".join(missing)
