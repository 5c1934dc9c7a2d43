"""CPU: the compiled gate and lookup programs (taiga_b200/csrc/gates.cuh - the compiler, the plan and the interpreter loop that
the quotient kernel and the verifier run) checked against a big-integer evaluation of the expression DAG, on every circuit
shape the repository builds, and the descriptor checks of circuit load, each on a minimally corrupted descriptor."""
import ctypes
import os
import random
import subprocess

import pytest

from conftest import ROOT
from taiga_b200 import circuits_mini as cm, circuits_random as cr, circuits_taiga as ct
from taiga_b200.circuit import (Assignment, CircuitKeyData, ConstraintSystem, EX_ADD, EX_ADVICE, EX_CONST, EX_FIXED, EX_INSTANCE, EX_MUL, EX_NEG, EX_SCALE, FIXED, P, TbColumn,
                                TbCsDesc, TbExprNode, TbLookup, TbQuery)

Q_ADD, Q_SUB, Q_FOLD_Y, Q_GBEGIN, Q_GFOLD, Q_GEND = 2, 3, 5, 10, 11, 12   # gates.cuh QOp


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("shim") / "host_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "host_shim.cpp")])
    return ctypes.CDLL(so)


def _corpus():
    out = [("standard_plonk", cm.standard_plonk()[0]), ("standard_plonk_no_lookups", cm.standard_plonk(n_lookups=0)[0]),
           ("standard_plonk_wide", cm.standard_plonk(wide=True)[0])]
    out += [(name, cr.boundary(name)[0]) for name, _ in cr.BOUNDARY]
    out += [("seed%d" % s, cr.random_shape(s)[0]) for s in range(30)]
    out += [("compliance_shape", ct.build(True, k=15)[0]), ("vp_shape", ct.build(False, k=11)[0])]   # the smallest k their rows allow
    return out


@pytest.fixture(scope="module")
def corpus():
    return _corpus()


def _plan(shim, desc, R, split):
    err = ctypes.create_string_buffer(512)
    ok = shim.hs_gate_plan(ctypes.byref(desc), R, int(split), err, 512)
    return ok, err.value.decode()


def _programs(shim, which):
    """[(code [(op, dst, akind, a, bkind, b)], nregs, last)] of plan list `which`"""
    out = []
    for p in range(shim.hs_gate_program(which, -1, None, 0, None)):
        meta = (ctypes.c_int * 2)()
        n = shim.hs_gate_program(which, p, None, 0, meta)
        words = (ctypes.c_uint32 * (4 * max(1, n)))()
        shim.hs_gate_program(which, p, words, n, meta)
        code = [(w & 0xff, (w >> 8) & 0xff, (w >> 16) & 0xff, a, w >> 24, b) for w, a, b in zip(words[0::4], words[1::4], words[2::4])][:n]
        out.append((code, meta[0], meta[1]))
    return out


def _positions(code, last):
    """the constraint indices a gate program folds, in order, read back from its fold instructions and gaps"""
    pos, group, end = [], None, None
    for op, _, _, _, _, gap in code:
        if op == Q_FOLD_Y:
            end = 0 if end is None else end + gap
            pos.append(end)
        elif op == Q_GBEGIN:
            assert gap == 0
            group = [0]
        elif op == Q_GFOLD:
            assert gap >= 1
            group.append(group[-1] + gap)
        elif op == Q_GEND:
            end = group[-1] if end is None else end + gap
            pos += [end - (group[-1] - g) for g in group]
            group = None
    assert group is None
    return [p - (pos[-1] - last) for p in pos] if pos else []


def _values(kd, rnd):
    cs = kd.cs
    return {kind: [rnd.randrange(P) for _ in qs] for kind, qs in ((EX_ADVICE, cs.advice_queries), (EX_FIXED, cs.fixed_queries),
                                                                  (EX_INSTANCE, cs.instance_queries))}


def _eval_nodes(cs, leaves):
    val = []
    for op, a, b in cs.nodes:
        if op == EX_CONST:
            v = cs.constants[a]
        elif op in (EX_ADVICE, EX_FIXED, EX_INSTANCE):
            v = leaves[op][a]
        elif op == EX_NEG:
            v = -val[a]
        elif op == EX_ADD:
            v = val[a] + val[b]
        elif op == EX_MUL:
            v = val[a] * val[b]
        else:
            assert op == EX_SCALE
            v = val[a] * cs.constants[b]
        val.append(v % P)
    return val


def _fe_array(vals):
    return (ctypes.c_uint8 * (32 * max(1, len(vals))))(*b"".join(v.to_bytes(32, "little") for v in vals) or bytes(32))


def _R(kd):
    return cr.describe(kd)["R"]


def test_gate_programs_match_the_expressions(shim, corpus):
    rnd = random.Random(11)
    seen = dict(group=0, sub=0, double=0, gap=0)
    for name, kd in corpus:
        cs, desc, R = kd.cs, kd.desc, _R(kd)
        roots = [p.node for _, polys in cs.gates for p in polys]
        J, L = len(roots), len(cs.lookups)
        deg = (ctypes.c_int * max(1, J))()
        shim.hs_constraint_degrees(ctypes.byref(desc), deg)
        assert list(deg[:J]) == [cr._expr_degree(cs, r) for r in roots], name
        for split in (False, True):
            ok, err = _plan(shim, desc, R, split)
            assert ok, (name, err)
            is_split = bool(shim.hs_gate_split())
            nsets = -(-len(cs.perm_columns) // (kd.degree - 2))
            assert shim.hs_gate_t_pl() == (2 * nsets + 1 if nsets else 0) + 5 * L   # permutation and lookup terms after the gates
            assert is_split <= split
            for big in (0, 1):
                hi, lo = _programs(shim, big), _programs(shim, 2 + big)
                assert len(hi) <= (8, 4)[big] and len(lo) <= (8, 4)[big] and bool(lo) == is_split, name
                # structure: the parts hold every constraint once, in order, split by degree
                hpos = [j for code, _, last in hi for j in _positions(code, last)]
                lpos = [j for code, _, last in lo for j in _positions(code, last)]
                assert all(1 <= nregs <= 48 for _, nregs, _ in hi + lo)
                if is_split:
                    assert lpos == [j for j in range(J) if deg[j] <= R // 2] and hpos == [j for j in range(J) if deg[j] > R // 2], name
                else:
                    assert hpos == list(range(J)), name
                # values: the parts combined as the quotient and the verifier combine them, and the lookups
                leaves = _values(kd, rnd)
                y, theta = rnd.randrange(P), rnd.randrange(P)
                gate = (ctypes.c_uint8 * 32)()
                lk = (ctypes.c_uint8 * (64 * max(1, L)))()
                assert shim.hs_gate_eval(ctypes.byref(desc), big, _fe_array(leaves[EX_ADVICE]), _fe_array(leaves[EX_FIXED]),
                                         _fe_array(leaves[EX_INSTANCE]), _fe_array([y]), _fe_array([theta]), gate, lk) == 0
                val = _eval_nodes(cs, leaves)
                want = 0
                for r in roots:
                    want = (want * y + val[r]) % P
                assert int.from_bytes(bytes(gate), "little") == want, (name, split, big)
                got = bytes(lk)
                for l, pairs in enumerate(cs.lookups):
                    a = t = 0
                    for i, tb in pairs:
                        a, t = (a * theta + val[i.node]) % P, (t * theta + val[tb.node]) % P
                    assert int.from_bytes(got[64 * l:64 * l + 32], "little") == a, (name, l)
                    assert int.from_bytes(got[64 * l + 32:64 * l + 64], "little") == t, (name, l)
                for code, _, _ in hi + lo + _programs(shim, 4):
                    for op, _, ak, a, bk, b in code:
                        seen["group"] += op == Q_GBEGIN
                        seen["sub"] += op == Q_SUB
                        seen["double"] += op == Q_ADD and (ak, a) == (bk, b)
                        seen["gap"] += op in (Q_FOLD_Y, Q_GFOLD, Q_GEND) and b > 1
    # every rewrite of the compiler ran somewhere in the corpus: selector groups, a - b, 2 x = x + x, folds over gaps
    assert all(seen.values()), seen


# ---------------------------------------------------------------- descriptor checks
def _copy(arr, n, ctype):
    return (ctype * max(1, n))(*[ctype.from_buffer_copy(arr[i]) if hasattr(ctype, "_fields_") else arr[i] for i in range(n)])


def _corrupted(kd, edit):
    """a deep copy of kd's descriptor (the arrays edit may touch are copies), changed by edit(desc, keep)"""
    d = TbCsDesc.from_buffer_copy(kd.desc)
    keep = []
    for name, count, ctype in (("advice_queries", "num_advice_queries", TbQuery), ("fixed_queries", "num_fixed_queries", TbQuery),
                               ("instance_queries", "num_instance_queries", TbQuery), ("perm_columns", "num_perm_columns", TbColumn),
                               ("nodes", "num_nodes", TbExprNode), ("constraint_roots", "num_constraints", ctypes.c_uint32),
                               ("lookups", "num_lookups", TbLookup)):
        arr = _copy(getattr(d, name), getattr(d, count), ctype)
        keep.append(arr)
        setattr(d, name, ctypes.cast(arr, type(getattr(d, name))))
    for l in range(d.num_lookups):
        lk = d.lookups[l]
        ins, tabs = _copy(lk.input_roots, lk.num_exprs, ctypes.c_uint32), _copy(lk.table_roots, lk.num_exprs, ctypes.c_uint32)
        keep += [ins, tabs]
        d.lookups[l] = TbLookup(lk.num_exprs, ctypes.cast(ins, ctypes.POINTER(ctypes.c_uint32)), ctypes.cast(tabs, ctypes.POINTER(ctypes.c_uint32)))
    edit(d)
    d._keep = keep
    return d


def _first(cs, *ops):
    return next(i for i, nd in enumerate(cs.nodes) if nd[0] in ops)


def _set_node(i, **kw):
    def edit(d):
        nd = d.nodes[i]
        d.nodes[i] = TbExprNode(kw.get("op", nd.op), kw.get("a", nd.a), kw.get("b", nd.b))
    return edit


def _set(arr, i, field, value):
    def edit(d):
        setattr(getattr(d, arr)[i], field, value)
    return edit


def _scaled():
    """a one-gate circuit with a SCALE node (a constant factor) and an instance query"""
    cs = ConstraintSystem()
    a, q, inst = cs.advice_column(), cs.selector(), cs.instance_column()
    cs.create_gate("scaled", [cs.query(q) * (cs.query(a) * 3 + cs.query(a, 1) - cs.query(inst))])
    return CircuitKeyData(cs, 4, Assignment(cs, 4))


def test_descriptor_checks(shim):
    kd, _ = cm.standard_plonk()
    kd_scale = _scaled()
    cs = kd.cs
    fixed_perm = next(c for c, col in enumerate(cs.perm_columns) if col.kind == FIXED)
    cases = [
        (kd, lambda d: setattr(d, "cs_degree", 2), "unsupported constraint system shape"),
        (kd, lambda d: setattr(d, "num_perm_columns", 16 * (d.cs_degree - 2) + 1), "unsupported constraint system shape"),
        (kd, lambda d: setattr(d, "blinding_factors", 0), "unsupported constraint system shape"),
        (kd, lambda d: setattr(d.lookups[0], "num_exprs", 0), "a lookup needs at least one expression pair"),
        (kd, _set("advice_queries", 0, "column", cs.num_advice), "advice query column out of range"),
        (kd, _set("fixed_queries", 0, "column", cs.num_fixed), "fixed query column out of range"),
        (kd, _set("instance_queries", 0, "column", cs.num_instance), "instance query column out of range"),
        (kd, _set_node(0, op=EX_SCALE + 1), "bad expression node"),
        (kd, _set_node(_first(cs, EX_CONST), a=len(cs.constants)), "expression constant index out of range"),
        (kd, _set_node(_first(cs, EX_ADVICE), a=len(cs.advice_queries)), "expression advice query index out of range"),
        (kd, _set_node(_first(cs, EX_FIXED), a=len(cs.fixed_queries)), "expression fixed query index out of range"),
        (kd_scale, _set_node(_first(kd_scale.cs, EX_INSTANCE), a=len(kd_scale.cs.instance_queries)), "expression instance query index out of range"),
        (kd, _set_node(_first(cs, EX_NEG), a=_first(cs, EX_NEG)), "expression nodes must be in topological order"),
        (kd, _set_node(_first(cs, EX_ADD), b=_first(cs, EX_ADD)), "expression nodes must be in topological order"),
        (kd, _set_node(_first(cs, EX_MUL), a=len(cs.nodes)), "expression nodes must be in topological order"),
        (kd_scale, _set_node(_first(kd_scale.cs, EX_SCALE), b=len(kd_scale.cs.constants)), "bad SCALE node"),
        (kd_scale, _set_node(_first(kd_scale.cs, EX_SCALE), a=_first(kd_scale.cs, EX_SCALE)), "bad SCALE node"),
        (kd, lambda d: d.constraint_roots.__setitem__(0, d.num_nodes), "constraint root out of range"),
        (kd, lambda d: d.lookups[1].input_roots.__setitem__(0, d.num_nodes), "lookup input root out of range"),
        (kd, lambda d: d.lookups[1].table_roots.__setitem__(0, d.num_nodes), "lookup table root out of range"),
        (kd, _set("perm_columns", 0, "kind", 3), "permutation column kind out of range"),
        (kd, _set("perm_columns", 0, "index", cs.num_advice), "permutation column index out of range"),
        (kd, _set("perm_columns", fixed_perm, "index", cs.num_fixed), "permutation column index out of range"),
    ]
    for base, _, _ in cases:
        assert _plan(shim, base.desc, _R(base), True) == (1, "")
    for i, (base, edit, msg) in enumerate(cases):
        ok, err = _plan(shim, _corrupted(base, edit), _R(base), True)
        assert not ok and err.startswith(msg + " ("), (i, msg, err)
    assert _plan(shim, kd.desc, _R(kd), True) == _plan(shim, kd_scale.desc, _R(kd_scale), True) == (1, "")   # the copies were changed, not these
