"""Random and boundary PLONKish constraint systems, satisfiable by construction.

`random_shape(seed, **overrides)` draws every structural knob of a constraint system from `seed` (any knob can be pinned)
and returns `(kd, make)` like `circuits_mini.standard_plonk`; `make(wseed)` synthesizes a satisfying witness.  The
shapes reach the parts of the prover the Taiga circuits do not: degrees whose quotient has fewer pieces than the extended
domain has sub-cosets, up to 16 permutation sets, more than five blinding factors, rotations beyond +-1, zero or several
instance columns, wide lookups and table expressions of degree 2, circuits without gates or without any argument.

Layout of a witness (every enabled row is the centre of its own window of 2 m + 1 rows, m = the largest |rotation|):
  * gate windows: each gate is `sel * (F(queries) - out)`; F never reads the `out` column, every other advice cell of
    the window is random and `out` is computed from F;
  * lookup windows: the queried input cells hold one row of the fixed table (which has an all-zero row and duplicates);
  * copy rows: each copy group is one row whose equality-enabled cells share one value, taken from a gate output, a
    constant, a fixed cell or the witness seed; groups are chained across permutation sets.
`satisfied(kd, asg)` checks an assignment without knowing this layout: every gate on every usable row, every lookup,
every cycle of the permutation the key was built with."""
import random

from .circuit import ADVICE, DELTA, EX_ADD, EX_ADVICE, EX_CONST, EX_FIXED, EX_INSTANCE, EX_MUL, EX_NEG, FIXED, INSTANCE, P, ROOT, \
    Assignment, CircuitKeyData, ConstraintSystem

KNOBS = ("k", "n_advice", "n_fixed", "n_instance", "adv_rots", "fix_rots", "inst_rots", "queries_per_column", "gates", "gate_rows",
         "lin_terms", "eq_advice", "eq_fixed", "eq_instance", "constants", "lookups", "full_row_lookup", "table_rows", "instance_full")


def _draw(r):
    """The random distribution of every knob (all kept small enough for k <= 8 and a CPU oracle run well under a second)."""
    rots = [0, -1, 1] + r.sample([-3, -2, 2, 3], r.randrange(0, 3))
    n_advice = r.randrange(1, 7)
    return dict(
        k=None,
        n_advice=n_advice,
        n_fixed=r.randrange(1, 3),
        n_instance=r.choice([0, 1, 1, 2, 3]),
        adv_rots=tuple(sorted(set(rots))),
        fix_rots=tuple(sorted({0} | set(r.sample([-2, -1, 1, 2], r.randrange(0, 3))))),
        inst_rots=tuple(sorted({0} | set(r.sample([-1, 1], r.randrange(0, 2))))),
        queries_per_column=r.randrange(1, 6),
        gates=tuple(r.choice([2, 2, 3, 3, 4, 5, 6, 7, 8, 9, 10, 12, 16]) for _ in range(r.randrange(0, 4))),
        gate_rows=r.randrange(1, 3),
        lin_terms=r.randrange(0, 3),
        eq_advice=r.randrange(0, n_advice + 1),
        eq_fixed=r.randrange(0, 2),
        eq_instance=r.randrange(0, 3),
        constants=r.random() < 0.5,
        lookups=tuple((r.randrange(1, 4), r.randrange(2, 4), r.randrange(1, 3)) for _ in range(r.randrange(0, 4))),
        full_row_lookup=r.random() < 0.3,
        table_rows=r.randrange(3, 12),
        instance_full=r.random() < 0.2,
    )


def random_shape(seed, **overrides):
    """-> (CircuitKeyData, make).  Knobs (see KNOBS): k (None = the smallest k the layout fits), column counts, the rotation
    set per column kind, queries_per_column (the most rotations one advice column is queried at: blinding factors
    max(3, q) + 2), gates (the degree of each gate, >= 2) and gate_rows (enabled rows per gate), lin_terms (extra linear
    terms of each F), eq_* (equality-enabled columns per kind) and constants (a constants column), lookups
    ((pairs, input degree >= 2, table degree 1 or 2) each), full_row_lookup (one more lookup of degree-1 inputs that holds
    on every usable row), table_rows, instance_full (instance column 0 has instance_len == usable)."""
    unknown = set(overrides) - set(KNOBS)
    assert not unknown, "unknown knobs %s" % sorted(unknown)
    r = random.Random(("shape", seed).__repr__())
    kn = _draw(r)
    kn.update(overrides)
    kn["n_instance"] = max(kn["n_instance"], 1 if kn["instance_full"] else 0)
    kn["eq_instance"] = min(kn["eq_instance"], kn["n_instance"])
    kn["eq_advice"] = min(kn["eq_advice"], kn["n_advice"])
    kn["eq_fixed"] = min(kn["eq_fixed"], kn["n_fixed"])
    assert kn["n_advice"] >= 1 and kn["n_fixed"] >= 1 and all(d >= 2 for d in kn["gates"]) and 0 in kn["adv_rots"]
    assert all(p >= 1 and 2 <= di and 1 <= dt <= 2 for p, di, dt in kn["lookups"])

    cs = ConstraintSystem()
    adv = [cs.advice_column() for _ in range(kn["n_advice"])]
    data = [cs.fixed_column() for _ in range(kn["n_fixed"])]
    inst = [cs.instance_column() for _ in range(kn["n_instance"])]
    sels = [cs.selector() for _ in kn["gates"]]
    lsels = [cs.selector() for _ in kn["lookups"]]
    n_pairs = max([p for p, _, _ in kn["lookups"]] + [1 if kn["full_row_lookup"] else 0])
    tabs = [cs.fixed_column() for _ in range(n_pairs)]
    tsel = cs.selector() if any(dt == 2 for _, _, dt in kn["lookups"]) else None
    full = [cs.advice_column() for _ in range(min(2, n_pairs) if kn["full_row_lookup"] else 0)]   # dedicated: a table row on every usable row
    consts = cs.fixed_column() if kn["constants"] else None

    # advice queries: the rotation set fills the columns in order, at most queries_per_column per column, so the first column
    # pins the blinding factors; rotations left over when every column is full are not queried
    q = max(1, kn["queries_per_column"])
    adv_rot = {c: [0] for c in adv}
    for x in kn["adv_rots"]:
        if x:
            c = next((c for c in adv if len(adv_rot[c]) < q), None)
            if c is not None:
                adv_rot[c].append(x)
    for c in adv:
        for x in adv_rot[c]:
            cs.query(c, x)
    for c in full:
        cs.query(c, 0)
    for c in data:
        for x in kn["fix_rots"]:
            cs.query(c, x)
    for t in tabs:
        cs.query(t, 0)
    inst_rot = {c: (kn["inst_rots"] if i == 0 else (0,)) for i, c in enumerate(inst)}
    for c in inst:
        for x in inst_rot[c]:
            cs.query(c, x)
    m = max([1] + [abs(x) for _, x in cs.advice_queries + cs.fixed_queries + cs.instance_queries])

    # equality: shuffled so that every permutation set mixes column kinds
    eq_cols = adv[:kn["eq_advice"]] + data[:kn["eq_fixed"]] + inst[:kn["eq_instance"]]
    r.shuffle(eq_cols)
    for c in eq_cols:
        cs.enable_equality(c)
    if consts is not None:
        cs.enable_constant(consts)

    # gates: sel * (c0 * prod(deg - 1 reads) + sum(c_i * read_i) + c - out)
    reads_all = [(c, x) for c in adv for x in adv_rot[c]] + [(c, x) for c in data for x in kn["fix_rots"]] + [(t, 0) for t in tabs] + \
                [(c, x) for c in inst for x in inst_rot[c]] + [(c, 0) for c in full]
    eq_adv = [c for c in adv if c in cs.perm_columns]
    gates = []
    for g, deg in enumerate(kn["gates"]):
        out = r.choice(eq_adv or adv)
        pool = [rd for rd in reads_all if rd[0] != out]
        terms = [(r.randrange(1, P), [r.choice(pool) for _ in range(deg - 1)])]
        terms += [(r.randrange(1, P), [r.choice(pool)]) for _ in range(kn["lin_terms"])]
        terms.append((r.randrange(P), []))
        e = None
        for coef, reads in terms:
            t = cs.constant(coef)
            for c, x in reads:
                t = t * cs.query(c, x)
            e = t if e is None else e + t
        cs.create_gate("g%d_deg%d" % (g, deg), [cs.query(sels[g]) * (e - cs.query(out))])
        gates.append((sels[g], out, terms))

    # lookups: input j = sel^(din - 1) * advice(col_j, rot_j) at distinct cells; table j = tabs[j] or tsel * tabs[j]
    lk_cells = [(c, x) for c in adv for x in adv_rot[c]]
    lookups = []
    for l, (p, din, dt) in enumerate(kn["lookups"]):
        cells = r.sample(lk_cells, min(p, len(lk_cells)))   # distinct input cells, so any table row can be looked up
        S = cs.query(lsels[l])
        pairs = []
        for j, (c, x) in enumerate(cells):
            inp = cs.query(c, x)
            for _ in range(din - 1):
                inp = S * inp
            tab = cs.query(tabs[j]) if dt == 1 else cs.query(tsel) * cs.query(tabs[j])
            pairs.append((inp, tab))
        cs.lookup(pairs)
        lookups.append((lsels[l], cells))
    if full:
        cs.lookup([(cs.query(c), cs.query(tabs[j])) for j, c in enumerate(full)])

    # copy groups: one row each; the first member is the source of the value
    groups = []
    eq_wit = [c for c in cs.perm_columns if c.kind != FIXED]
    eq_fix = [c for c in data if c in cs.perm_columns]
    outs = [(g, out) for g, (_, out, _) in enumerate(gates) if out in cs.perm_columns]
    if eq_wit:
        n_groups = max(2, len(cs.perm_columns) // 3)
        for i in range(n_groups):
            kinds = ["free"] + (["out"] if outs else []) + (["const"] if consts is not None else []) + (["fixed"] if eq_fix else [])
            src = kinds[i % len(kinds)]
            if i == 0:    # one cycle through every witness-side column: it spans every permutation set
                members = list(eq_wit)
            else:
                members = r.sample(eq_wit, r.randrange(1, min(4, len(eq_wit)) + 1))
            groups.append((src, (outs[i % len(outs)][0] if src == "out" else r.choice(eq_fix) if src == "fixed" else None), members))
    elif consts is not None or eq_fix:
        groups.append(("fixed-only", None, []))

    # rows: windows (gates, then lookups), then the copy rows
    spacing = 2 * m + 1
    gate_rows = [[m + spacing * (g * kn["gate_rows"] + i) for i in range(kn["gate_rows"])] for g in range(len(gates))]
    base = len(gates) * kn["gate_rows"]
    lk_rows = [[m + spacing * (base + l * kn["gate_rows"] + i) for i in range(kn["gate_rows"])] for l in range(len(lookups))]
    windows_end = spacing * (base + len(lookups) * kn["gate_rows"])
    copy_rows = [windows_end + i for i in range(len(groups))]
    table_rows = max(2, kn["table_rows"])
    rows_needed = max(windows_end + len(groups), table_rows, len(groups) + 1, 1)
    bf = cs.blinding_factors()
    k_min = 1
    while (1 << k_min) - (bf + 1) < rows_needed or (1 << k_min) < cs.minimum_rows():
        k_min += 1
    k = kn["k"] if kn["k"] is not None else k_min
    assert k >= k_min, "k=%d is below the smallest k (%d) this shape fits" % (k, k_min)
    n = 1 << k
    usable = n - (bf + 1)

    fr = random.Random(("fixed", seed).__repr__())
    table = [tuple(0 for _ in tabs)]
    for t in range(1, table_rows):
        table.append(table[fr.randrange(1, t)] if t >= 3 and fr.random() < 0.3 else tuple(fr.randrange(P) for _ in tabs))
    data_vals = [[fr.randrange(P) for _ in range(usable)] for _ in data]
    const_vals = [fr.randrange(1, P) for _ in groups]
    inst_len = [usable if (i == 0 and kn["instance_full"]) else min(usable, windows_end + len(groups) + 1 + i) for i in range(len(inst))]

    def make(wseed=1):
        w = random.Random(("witness", seed, wseed).__repr__())
        asg = Assignment(cs, k)
        for rows, (s, _, _) in zip(gate_rows, gates):
            for row in rows:
                asg.enable(s, row)
        for rows, (s, _) in zip(lk_rows, lookups):
            for row in rows:
                asg.enable(s, row)
        for t, tup in enumerate(table):
            for j, v in enumerate(tup):
                asg.assign(tabs[j], t, v)
            if tsel is not None:
                asg.enable(tsel, t)
        for c, vals in zip(data, data_vals):
            for row, v in enumerate(vals):
                asg.assign(c, row, v)
        for row in range(usable):   # the full-row lookup: every usable row holds one table row
            tup = table[w.randrange(len(table))]
            for j, c in enumerate(full):
                asg.assign(c, row, tup[j])
        for row in range(windows_end):
            for c in adv:
                asg.assign(c, row, w.randrange(P))
        ivals = [[w.randrange(P) for _ in range(ln)] for ln in inst_len]
        for rows, (_, cells) in zip(lk_rows, lookups):
            for row in rows:
                tup = table[w.randrange(len(table))]
                for j, (c, x) in enumerate(cells):
                    asg.assign(c, row + x, tup[j])

        def cell(c, row):
            if c.kind == INSTANCE:
                return ivals[c.index][row] if row < len(ivals[c.index]) else 0
            return asg.value((c, row))
        out_val = {}
        for g, ((_, out, terms), rows) in enumerate(zip(gates, gate_rows)):
            for row in rows:
                v = 0
                for coef, reads in terms:
                    t = coef
                    for c, x in reads:
                        t = t * cell(c, row + x) % P
                    v += t
                asg.assign(out, row, v)
            out_val[g] = (out, rows[0])
        for (src, arg, members), row, kc in zip(groups, copy_rows, const_vals):
            if src == "fixed-only":   # no witness column takes part in the permutation: tie a constant to a fixed cell at least
                if consts is not None:
                    asg.constant_cell(kc)
                continue
            if src == "out":
                out, orow = out_val[arg]
                v, first = asg.value((out, orow)), (out, orow)
            elif src == "const":
                v = kc
                first = asg.constant_cell(kc)
            elif src == "fixed":
                v, first = data_vals[arg.index][row], (arg, row)
            else:
                v, first = w.randrange(P), None
            prev = first
            for c in members:
                if c.kind == INSTANCE:
                    ivals[c.index][row] = v
                else:
                    asg.assign(c, row, v)
                if prev is not None:
                    asg.copy(prev, (c, row))
                prev = (c, row)
        for c, vals in zip(inst, ivals):
            asg.set_instance(c, vals)
        return asg

    kd = CircuitKeyData(cs, k, make(1), name="random_%s" % (seed,))
    kd.random_shape = dict(kn, k=k, k_min=k_min, rows_needed=rows_needed, instance_len=inst_len, usable=usable, m=m)
    return kd, make


# ---------------------------------------------------------------- the plain-Python mock prover
def _fixed_value(kd, col, row):
    return int.from_bytes(kd.fixed[col, row].tobytes(), "little")


def satisfied(kd, asg, blinding_seed=0):
    """halo2 MockProver restated: None if `asg` satisfies kd's constraint system, else a message naming the first failure.
    Fixed values and the permutation are the key's (kd.fixed, kd.sigma), advice and instance values the assignment's.
    Advice cells of the blinding rows hold random values, so a gate that reads one on an enabled row fails."""
    return next(failures(kd, asg, blinding_seed), None)


def failures(kd, asg, blinding_seed=0):
    """Every failure of `asg`, as satisfied's messages, in the order tb_check_batch reports them: gates by (row, constraint),
    then lookups by (lookup, row), then copies by (permutation column, row).  An instance column longer than the usable rows
    is reported alone, and a sigma value that is no cell ends the list."""
    cs, n = kd.cs, kd.n
    usable = n - (cs.blinding_factors() + 1)
    br = random.Random(blinding_seed)
    advice = [[asg.advice[c].get(row, 0) if row < usable else br.randrange(P) for row in range(n)] for c in range(cs.num_advice)]
    fixed = [[_fixed_value(kd, c, row) for row in range(n)] for c in range(cs.num_fixed)]
    instance = [[col[row] if row < len(col) else 0 for row in range(n)] for col in asg.instance]
    for c, col in enumerate(asg.instance):
        if len(col) > usable:
            yield "instance column %d has %d values, more than the %d usable rows" % (c, len(col), usable)
            return

    def evaluate(node, row, memo):
        if node in memo:
            return memo[node]
        op, a, b = cs.nodes[node]
        if op == EX_CONST:
            v = cs.constants[a]
        elif op in (EX_ADVICE, EX_FIXED, EX_INSTANCE):
            col, rot = (cs.advice_queries, cs.fixed_queries, cs.instance_queries)[op - EX_ADVICE][a]
            v = (advice, fixed, instance)[op - EX_ADVICE][col][(row + rot) % n]
        elif op == EX_NEG:
            v = -evaluate(a, row, memo)
        elif op == EX_ADD:
            v = evaluate(a, row, memo) + evaluate(b, row, memo)
        elif op == EX_MUL:
            v = evaluate(a, row, memo) * evaluate(b, row, memo)
        else:
            v = evaluate(a, row, memo) * cs.constants[b]
        memo[node] = v % P
        return memo[node]

    for row in range(usable):
        memo = {}
        for name, polys in cs.gates:
            for i, p in enumerate(polys):
                if evaluate(p.node, row, memo):
                    yield "gate %s poly %d is not zero on row %d" % (name, i, row)
    for l, lk in enumerate(cs.lookups):
        table = set()
        rows = []
        for row in range(usable):
            memo = {}
            table.add(tuple(evaluate(t.node, row, memo) for _, t in lk))
            rows.append(tuple(evaluate(i.node, row, memo) for i, _ in lk))
        for row, tup in enumerate(rows):
            if tup not in table:
                yield "lookup %d: input on row %d is not in the table" % (l, row)
    # the permutation the key commits to: sigma[i][j] = delta^i' omega^j' names the next cell of (i, j)'s cycle
    cols = cs.perm_columns
    omega = pow(ROOT, 1 << (32 - kd.k), P)
    where = {}
    d = 1
    for i in range(len(cols)):
        o = d
        for j in range(n):
            where[o] = (i, j)
            o = o * omega % P
        d = d * DELTA % P
    grid = {ADVICE: advice, FIXED: fixed, INSTANCE: instance}
    for i, c in enumerate(cols):
        for j in range(usable):
            s = int.from_bytes(kd.sigma[i, j].tobytes(), "little")
            if s not in where:
                yield "sigma of column %d row %d is not a cell" % (i, j)
                return
            pi, pj = where[s]
            if grid[c.kind][c.index][j] != grid[cols[pi].kind][cols[pi].index][pj]:
                yield "copy (%r, %d) -> (%r, %d) joins different values" % (c, j, cols[pi], pj)


# ---------------------------------------------------------------- shape summary
def _expr_degree(cs, node):
    op, a, b = cs.nodes[node]
    if op == EX_CONST:
        return 0
    if op in (EX_ADVICE, EX_FIXED, EX_INSTANCE):
        return 1
    if op == EX_MUL:
        return _expr_degree(cs, a) + _expr_degree(cs, b)
    if op == EX_ADD:
        return max(_expr_degree(cs, a), _expr_degree(cs, b))
    return _expr_degree(cs, a)


def describe(kd):
    """The structural parameters the prover's code paths depend on (dict; "id" is a compact one-line form)."""
    cs = kd.cs
    deg = kd.degree
    pieces = deg - 1
    ext_k = kd.k
    while (1 << ext_k) < kd.n * pieces:
        ext_k += 1
    R = 1 << (ext_k - kd.k)
    P_ = len(cs.perm_columns)
    nsets = -(-P_ // (deg - 2)) if P_ else 0
    cdeg = [_expr_degree(cs, p.node) for _, polys in cs.gates for p in polys]
    rs = getattr(kd, "random_shape", {})
    d = dict(
        k=kd.k, k_min=rs.get("k_min"), degree=deg, pieces=pieces, R=R, blinding_factors=kd.blinding_factors,
        perm_columns=P_, perm_sets=nsets, lookups=len(cs.lookups), lookup_pairs=[len(lk) for lk in cs.lookups],
        input_degrees=[max(_expr_degree(cs, i.node) for i, _ in lk) for lk in cs.lookups],
        table_degrees=[max(_expr_degree(cs, t.node) for _, t in lk) for lk in cs.lookups],
        instance_columns=cs.num_instance, instance_rotations=sorted({x for _, x in cs.instance_queries}),
        instance_eq=sum(c.kind == INSTANCE for c in cs.perm_columns),
        advice_rotations=sorted({x for _, x in cs.advice_queries}), fixed_rotations=sorted({x for _, x in cs.fixed_queries}),
        gates=len(cs.gates), constraint_degrees=sorted(cdeg),
        low_constraints=sum(1 for x in cdeg if R >= 4 and x <= R // 2), high_constraints=sum(1 for x in cdeg if not (R >= 4 and x <= R // 2)),
        instance_full=bool(rs.get("instance_full")), full_row_lookup=bool(rs.get("full_row_lookup")),
    )
    d["id"] = "k%d-deg%d-R%d-bf%d-P%d-sets%d-L%s-inst%d@%s-rot%s..%s-g%d" % (
        kd.k, deg, R, kd.blinding_factors, P_, nsets, "x".join(map(str, d["lookup_pairs"])) or "0", cs.num_instance,
        ",".join(map(str, d["instance_rotations"])) or "-", min(d["advice_rotations"]), max(d["advice_rotations"]), len(cs.gates))
    return d


# ---------------------------------------------------------------- proof layout (for naming the first differing byte)
def proof_sections(kd):
    """[(name, start, end)] byte ranges of a proof of kd, in transcript order."""
    cs = kd.cs
    P_ = len(cs.perm_columns)
    nsets = -(-P_ // (kd.degree - 2)) if P_ else 0
    L = len(cs.lookups)
    nev = len(cs.instance_queries) + len(cs.advice_queries) + len(cs.fixed_queries) + 1 + P_ + max(0, 3 * nsets - 1) + 5 * L
    parts = [("advice commitments", cs.num_advice), ("lookup permuted commitments", 2 * L), ("permutation Z commitments", nsets),
             ("lookup Z commitments", L), ("random commitment", 1), ("h commitments", kd.degree - 1), ("evaluations", nev),
             ("multiopen", 1 + kd.num_point_sets()), ("IPA", 1 + 2 * kd.k + 2)]
    out, pos = [], 0
    for name, cnt in parts:
        out.append((name, pos, pos + 32 * cnt))
        pos += 32 * cnt
    return out


def section_of(kd, offset):
    for name, a, b in proof_sections(kd):
        if a <= offset < b:
            return "%s (element %d of the section)" % (name, (offset - a) // 32)
    return "beyond the proof"


# ---------------------------------------------------------------- pinned boundary shapes
_FULL_ROTS = (-3, -2, -1, 0, 1, 2, 3)
BOUNDARY = [
    ("deg4", dict(gates=(4, 3, 2), lookups=(), eq_advice=2, n_advice=3)),
    ("deg6_lookup", dict(gates=(6,), lookups=((2, 2, 1),), n_advice=3, eq_advice=2)),
    ("deg8", dict(gates=(8, 2), lookups=((1, 2, 1),), n_advice=4, eq_advice=3, n_instance=1, eq_instance=1)),
    ("deg12", dict(gates=(12,), lookups=(), n_advice=3, eq_advice=1)),
    ("deg16", dict(gates=(16, 5), lookups=((1, 2, 2),), n_advice=4, eq_advice=2)),
    ("deg18_R32", dict(gates=(18,), lookups=(), n_advice=2, eq_advice=1, n_instance=1, eq_instance=1)),
    ("sets16_deg3", dict(gates=(3, 2), lookups=(), full_row_lookup=False, n_advice=12, eq_advice=12, n_fixed=2, eq_fixed=1, n_instance=2,
                         eq_instance=2, constants=True)),
    ("sets16_deg4", dict(gates=(4, 3), lookups=(), n_advice=28, eq_advice=28, n_fixed=2, eq_fixed=2, n_instance=1, eq_instance=1,
                         constants=True, queries_per_column=2)),
    ("no_perm_no_lookup", dict(gates=(3, 5), lookups=(), full_row_lookup=False, eq_advice=0, eq_fixed=0, eq_instance=0, constants=False,
                               n_instance=1)),
    ("no_gates", dict(gates=(), lookups=((2, 2, 1), (1, 3, 2)), full_row_lookup=True, n_advice=3, eq_advice=3, constants=True,
                      n_instance=1, eq_instance=1)),
    ("no_instance", dict(gates=(5, 3), n_instance=0, instance_full=False, lookups=((1, 2, 1),), eq_advice=2, n_advice=3, constants=True)),
    ("three_instance", dict(gates=(4, 3, 2), n_instance=3, eq_instance=2, inst_rots=(-1, 0, 1), n_advice=3, eq_advice=2,
                            lookups=())),
    ("rotations_3", dict(gates=(5, 4, 3), adv_rots=_FULL_ROTS, fix_rots=(-2, 0, 2), queries_per_column=3, n_advice=4, eq_advice=2,
                         lookups=((2, 2, 1),))),
    ("bf6", dict(gates=(4, 3), adv_rots=(-2, -1, 0, 1, 2), queries_per_column=4, n_advice=2, eq_advice=2, lookups=())),
    ("bf8", dict(gates=(5, 3), adv_rots=_FULL_ROTS, queries_per_column=6, n_advice=2, eq_advice=1, lookups=((1, 2, 1),))),
    ("lookups4_wide", dict(gates=(3,), lookups=((4, 2, 1), (1, 2, 2), (2, 3, 1), (3, 2, 2)), n_advice=5, eq_advice=2)),
    ("split_mixed_degrees", dict(gates=(8, 7) + (2, 3, 4, 2, 3, 4, 2, 3, 4, 4, 3, 2), lin_terms=2, lookups=((1, 2, 1),), n_advice=4, eq_advice=2)),
    ("k10", dict(k=10, gates=(6, 3), lookups=((2, 2, 2),), full_row_lookup=True, n_advice=3, eq_advice=2, n_instance=1, eq_instance=1)),
    ("instance_full_every_row_lookup", dict(gates=(4,), instance_full=True, n_instance=2, eq_instance=1, full_row_lookup=True,
                                            lookups=((1, 2, 1),), n_advice=3, eq_advice=2)),
]


def boundary(name):
    """(kd, make) of the pinned shape `name` (its seed only fills in the values the pin leaves open)."""
    for i, (nm, kn) in enumerate(BOUNDARY):
        if nm == name:
            return random_shape(1000 + i, **kn)
    raise KeyError(name)
