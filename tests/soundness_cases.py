"""Inputs a prover or verifier must not be fooled by (helper module of the soundness tests, not a conftest).

`violations(kd, make, wseed)` breaks exactly one constraint of a circuits_random shape: a gate output on the first and
last enabled row of every gate, a gate input read at a negative and at a positive rotation, an advice copy inside one
permutation set, a copy that crosses a boundary between sets, an instance copy (a false statement: the instance value
alone changes), a copy to the constants column and to a fixed cell, and one input of every lookup that is not in its
table.  Each case is checked with `cr.satisfied`, which must name that failure and no earlier one.

`mutants(kd, proof, other)` rewrites one element of a proof: every point slot gets its negation, the identity, x + q
(the same point, non-canonical), "negative zero", the smallest x off the curve and the slot of `other`; every scalar
slot gets v + 1, v + p (the same value, non-canonical), 32 bytes of 0xFF and the slot of `other`; the whole proof is cut
or extended by one and by 32 bytes.  Every mutant must be rejected."""
import random

from oracle import verifier_py as vp
from taiga_b200 import circuits_random as cr
from taiga_b200.circuit import ADVICE, DELTA, EX_ADD, EX_ADVICE, EX_FIXED, EX_MUL, EX_NEG, EX_SCALE, FIXED, INSTANCE, P, ROOT, Column

Q = vp.Q
ENCODING_KINDS = ("identity", "x+q", "negative-zero", "off-curve", "v+p", "ff", "cut1", "cut32", "add1", "add32")
VALUE_KINDS = ("negated", "other", "v+1")


# ---------------------------------------------------------------- violating witnesses
def _leaves(cs, node, op, out):
    """(column index, rotation) of every query of kind `op` under `node`."""
    o, a, b = cs.nodes[node]
    if o == op:
        out.add((cs.advice_queries, cs.fixed_queries)[op - EX_ADVICE][a])
    if o in (EX_NEG, EX_ADD, EX_MUL, EX_SCALE):
        _leaves(cs, a, op, out)
    if o in (EX_ADD, EX_MUL):
        _leaves(cs, b, op, out)
    return out


def _enabled_rows(kd, fixed_col):
    return [r for r in range(kd.n) if any(kd.fixed[fixed_col, r])]


def _gates(kd):
    """[(name, selector rows, out column, advice reads of F)] of a circuits_random gate sel * (F - out)."""
    cs = kd.cs
    gates = []
    for name, polys in cs.gates:
        op, sel, body = cs.nodes[polys[0].node]
        assert op == EX_MUL and cs.nodes[sel][0] == EX_FIXED
        _, f, neg_out = cs.nodes[body]
        assert cs.nodes[neg_out][0] == EX_NEG
        out = cs.advice_queries[cs.nodes[cs.nodes[neg_out][1]][1]][0]
        gates.append((name, _enabled_rows(kd, cs.fixed_queries[cs.nodes[sel][1]][0]), out, sorted(_leaves(cs, f, EX_ADVICE, set()))))
    return gates


def _cycles(kd):
    """next cell of every cell of the permutation, cells as (perm column position, row)."""
    omega = pow(ROOT, 1 << (32 - kd.k), P)
    where, d = {}, 1
    for i in range(len(kd.cs.perm_columns)):
        o = d
        for j in range(kd.n):
            where[o] = (i, j)
            o = o * omega % P
        d = d * DELTA % P
    return {(i, j): where[int.from_bytes(kd.sigma[i, j].tobytes(), "little")] for i in range(len(kd.cs.perm_columns)) for j in range(kd.n)}


def _bump(asg, col, row):
    if col.kind == INSTANCE:
        asg.instance[col.index][row] = (asg.instance[col.index][row] + 1) % P
    else:
        asg.advice[col.index][row] = (asg.advice[col.index].get(row, 0) + 1) % P
    return asg


def violations(kd, make, wseed):
    """[(label, Assignment)]: each assignment is make(wseed) with one constraint broken (see the module docstring)."""
    cs, rs = kd.cs, kd.random_shape
    base = make(wseed)
    assert cr.satisfied(kd, base) is None, "%s: the honest witness does not satisfy the circuit" % kd.name
    windows_end = (2 * rs["m"] + 1) * (len(rs["gates"]) + len(rs["lookups"])) * rs["gate_rows"]
    cases = []    # (label, cell to bump, expected prefix of cr.satisfied's message)

    for g, (name, rows, out, reads) in enumerate(_gates(kd)):
        for which, row in (("first", rows[0]), ("last", rows[-1]))[:len(set((rows[0], rows[-1])))]:
            cases.append(("gate%d-out-%s" % (g, which), (Column(ADVICE, out), row), "gate %s poly 0 is not zero on row %d" % (name, row)))
    for sign in (-1, 1):    # every advice read at a rotation of this sign, in gate order: the first one that changes F is kept
        cases.append([("gate%d-read-rot%+d" % (g, x), (Column(ADVICE, c), rows[0] + x), "gate %s poly 0 is not zero on row %d" % (name, rows[0]))
                      for g, (name, rows, _, reads) in enumerate(_gates(kd)) for c, x in reads if x * sign > 0])

    if cs.perm_columns:
        nxt = _cycles(kd)
        prv = {b: a for a, b in nxt.items()}
        chunk = kd.degree - 2
        cols = cs.perm_columns
        found = {}
        for i, col in enumerate(cols):
            if col.kind == FIXED:
                continue
            for j in range(windows_end, rs["usable"]):
                if nxt[(i, j)] == (i, j) or (col.kind == INSTANCE and j >= len(base.instance[col.index])):
                    continue
                cyc, c = [(i, j)], nxt[(i, j)]
                while c != (i, j):
                    cyc.append(c)
                    c = nxt[c]
                fixed_cols = {cols[a] for a, _ in cyc if cols[a].kind == FIXED}
                if col.kind == INSTANCE:
                    kind = "instance-copy"
                elif cs.constants_column in fixed_cols:
                    kind = "constant-copy"
                elif fixed_cols:
                    kind = "fixed-copy"
                elif i // chunk == prv[(i, j)][0] // chunk == nxt[(i, j)][0] // chunk:
                    kind = "copy-in-set"
                elif prv[(i, j)][0] // chunk != i // chunk:
                    kind = "copy-across-sets"
                else:
                    continue
                # across sets: the longest cycle (the group through every witness column spans all sets)
                if kind not in found or (kind == "copy-across-sets" and len(cyc) > found[kind][1]):
                    found[kind] = ((col, j), len(cyc))
        for kind in ("copy-in-set", "copy-across-sets", "instance-copy", "constant-copy", "fixed-copy"):
            if kind in found:
                (col, j), _ = found[kind]
                cases.append((kind, (col, j), "copy"))

    for l, lk in enumerate(cs.lookups):
        inp = lk[0][0].node
        (c, x), = _leaves(cs, inp, EX_ADVICE, set())
        sel = _leaves(cs, inp, EX_FIXED, set())
        row = _enabled_rows(kd, next(iter(sel))[0])[0] if sel else rs["usable"] - 1    # the full-row lookup holds on every row
        cases.append(("lookup%d" % l, (Column(ADVICE, c), row + x), "lookup %d: input on row %d is not in the table" % (l, row)))

    def apply(label, col, row):
        asg = make(wseed)
        if label.startswith("lookup"):   # a value no table row holds (random: every table value is random or zero)
            asg.advice[col.index][row] = random.Random(repr((kd.name, wseed, label))).randrange(1, P)
        else:
            _bump(asg, col, row)
        return asg, cr.satisfied(kd, asg)

    out = []
    for case in cases:
        if isinstance(case, list):   # alternatives: a read can sit in a product whose other factor is zero on that row
            for label, (col, row), want in case:
                asg, why = apply(label, col, row)
                if why is not None:
                    break
            else:
                continue
        else:
            label, (col, row), want = case
            asg, why = apply(label, col, row)
        assert why and why.startswith(want), "%s %s: satisfied() reports %r, not %r" % (kd.name, label, why, want)
        if want == "copy":
            assert "(%r, %d)" % (col, row) in why, "%s %s: satisfied() reports another copy: %r" % (kd.name, label, why)
        out.append((label, asg))
    return out


# ---------------------------------------------------------------- proof mutants
def _off_curve_x():
    x = 1
    while pow(x ** 3 + 5, (Q - 1) // 2, Q) == 1:
        x += 1
    return x


OFF_CURVE_X = _off_curve_x()


def slots(kd):
    """[(section, element, offset, 'point' | 'scalar')] of every 32-byte element of a proof of kd."""
    out = []
    for name, a, b in cr.proof_sections(kd):
        cnt = (b - a) // 32
        for e in range(cnt):
            if name == "evaluations" or (name == "multiopen" and e >= 1) or (name == "IPA" and e >= cnt - 2):
                kind = "scalar"
            else:
                kind = "point"
            out.append((name, e, a + 32 * e, kind))
    return out


def mutants(kd, proof, other):
    """[(label, section, kind, bytes)]; kind is one of ENCODING_KINDS or VALUE_KINDS."""
    assert len(proof) == len(other) == kd.proof_size()
    out = []
    for name, e, off, what in slots(kd):
        v = int.from_bytes(proof[off:off + 32], "little")
        subs = []
        if what == "point":
            sign, x = v >> 255, v & ((1 << 255) - 1)
            subs.append(("negated", v ^ (1 << 255)))
            subs.append(("identity", 0))
            if x + Q < 1 << 255:
                subs.append(("x+q", (x + Q) | sign << 255))
            subs.append(("negative-zero", 1 << 255))
            subs.append(("off-curve", OFF_CURVE_X | sign << 255))
        else:
            subs.append(("v+1", (v + 1) % P))
            subs.append(("v+p", v + P))
            subs.append(("ff", (1 << 256) - 1))
        subs.append(("other", int.from_bytes(other[off:off + 32], "little")))
        for kind, nv in subs:
            m = proof[:off] + nv.to_bytes(32, "little") + proof[off + 32:]
            if m != proof:
                out.append(("%s[%d] %s" % (name, e, kind), name, kind, m))
    out += [("cut 1 byte", "length", "cut1", proof[:-1]), ("cut 32 bytes", "length", "cut32", proof[:-32]),
            ("1 zero byte appended", "length", "add1", proof + bytes(1)), ("32 zero bytes appended", "length", "add32", proof + bytes(32))]
    return out


def check_point_mutants(kd, proof):
    """The point encodings decode as intended: the negation, the identity, and Reject for the non-canonical ones."""
    for name, e, off, what in slots(kd):
        if what != "point":
            continue
        enc = proof[off:off + 32]
        v = int.from_bytes(enc, "little")
        pt = vp._to_affine(vp.decompress(enc))
        assert vp._to_affine(vp.decompress((v ^ (1 << 255)).to_bytes(32, "little"))) == (pt[0], (Q - pt[1]) % Q)
        assert vp.decompress(bytes(32))[2] == 0
        x, sign = v & ((1 << 255) - 1), v >> 255
        bad = [(1 << 255), OFF_CURVE_X | sign << 255] + ([(x + Q) | sign << 255] if x + Q < 1 << 255 else [])
        for b in bad:
            try:
                vp.decompress(b.to_bytes(32, "little"))
            except vp.Reject:
                continue
            raise AssertionError("%s[%d]: %064x decodes" % (name, e, b))
