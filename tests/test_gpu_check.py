"""GPU: the batched witness check (tb_check_batch, ProvingKey.check_batch) against circuits_random.failures, the prover and
the verifier.

* Honest witnesses pass on the mini circuits, every boundary shape, random shapes and both Taiga shapes at k = 15, at batch
  sizes 1, 7, 8, 9 and 64 (B >= 8 selects the other gate part set).
* Every soundness_cases violation is named: in batches of 2 and 9 next to honest witnesses at moving positions, the first
  record renders as cr.satisfied's message, the records are the first items of cr.failures, the counts its totals, and
  each slot's result equals the result of that witness checked alone.
* A reported gate or copy failure <=> the device verifier rejects the witness's proof; a reported lookup failure <=>
  prove_batch refuses that slot and lookup.
* Truncation, blinding rows, seeds, refusals, concurrent contexts, proofs after checks and the exact launch count."""
import re
import threading

import numpy as np
import pytest

import soundness_cases as sc
from taiga_b200 import circuits_mini as cm
from taiga_b200 import circuits_random as cr
from taiga_b200 import circuits_taiga as ct
from taiga_b200 import lib
from taiga_b200.circuit import ADVICE, P

from test_gpu_verifier_soundness import PROVE_SHAPES, stack
from test_verifier_soundness import SEED, mutant_shape

pytestmark = pytest.mark.gpu

CHECK_SEED = bytes((11 * j + 3) & 0xFF for j in range(32))
MINI = {"plonk_k6_l2": lambda: cm.standard_plonk(k=6, n_lookups=2), "plonk_k6_l0": lambda: cm.standard_plonk(k=6, n_lookups=0),
        "plonk_k7_wide": lambda: cm.standard_plonk(k=7, n_lookups=2, wide=True)}
RANDOM_SEEDS = list(range(30))


@pytest.fixture(scope="module")
def keys(gpu_ctx, oracle_cpu):
    """shape id -> (kd, make, oracle key, device key); one device SRS per k."""
    srs_cache, cache = {}, {}

    def get(name):
        if name not in cache:
            if name in MINI:
                kd, make = MINI[name]()
            elif isinstance(name, int):
                kd, make = cr.random_shape(name)
            else:
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


def expected(kd, asg, max_failures):
    """(counts, first max_failures messages) of cr.failures."""
    msgs = list(cr.failures(kd, asg))
    gate_rows = {int(re.search(r"on row (\d+)$", m).group(1)) for m in msgs if m.startswith("gate ")}
    counts = (len(gate_rows), sum(m.startswith("lookup ") for m in msgs), sum(m.startswith("copy ") for m in msgs))
    return counts, msgs[:max_failures]


def check(pk, kd, asgs, max_failures=16, seed=CHECK_SEED, ctx=None):
    adv, inst, lens = stack(kd, asgs)
    res = pk.check_batch(adv, inst, lens, seed, max_failures=max_failures, ctx=ctx)
    return [(cnt, [lib.render_failure(kd, f) for f in fails], fails) for cnt, fails in res]


# ---------------------------------------------------------------- 1. honest witnesses pass
HONEST = list(MINI) + [name for name, _ in cr.BOUNDARY] + RANDOM_SEEDS


@pytest.mark.parametrize("name", HONEST, ids=[str(x) for x in HONEST])
def test_honest_witnesses_pass(keys, name):
    kd, make, _, pk = keys(name)
    for B in (1, 7, 8, 9):
        res = check(pk, kd, [make(500 + b) for b in range(B)])
        assert all(cnt == (0, 0, 0) and not msgs for cnt, msgs, _ in res), (name, B, res)
    asgs = [make(600 + b % 3) for b in range(64)]
    assert all(cnt == (0, 0, 0) for cnt, _, _ in check(pk, kd, asgs, max_failures=0)), (name, 64)


# ---------------------------------------------------------------- 2. every violation is named
VIOLATION_SHAPES = PROVE_SHAPES + ["no_gates"]


@pytest.mark.parametrize("B", [2, 9])
@pytest.mark.parametrize("name", VIOLATION_SHAPES)
def test_every_violation_is_named(keys, name, B):
    kd, make, _, pk = keys(name)
    bad = sc.violations(kd, make, 5)
    assert bad, name
    slots = []
    for c, i in enumerate(range(0, len(bad), B - 1)):
        batch = bad[i:i + B - 1]
        batch.insert(c % (len(batch) + 1), ("honest", make(100 + c)))
        batch += [("honest", make(200 + c * B + j)) for j in range(B - len(batch))]
        slots += batch
    M = 8
    for first in range(0, len(slots), B):
        batch = slots[first:first + B]
        res = check(pk, kd, [a for _, a in batch], max_failures=M)
        for (label, asg), (cnt, msgs, fails) in zip(batch, res):
            want_cnt, want_msgs = expected(kd, asg, M)
            if label == "honest":
                assert cnt == (0, 0, 0) and not msgs, (name, label, cnt, msgs)
                continue
            assert msgs[0] == cr.satisfied(kd, asg), (name, B, label, msgs[0])
            assert (cnt, msgs) == (want_cnt, want_msgs), (name, B, label)
            alone = check(pk, kd, [asg], max_failures=M)[0]
            assert (alone[0], alone[2]) == (cnt, fails), (name, B, label)


# ---------------------------------------------------------------- 3. agreement with the prover and the verifier
@pytest.mark.parametrize("name", PROVE_SHAPES)
def test_agrees_with_prover_and_verifier(keys, name):
    kd, make, _, pk = keys(name)
    cases = sc.violations(kd, make, 5) + [("honest", make(700)), ("honest", make(701))]
    for label, asg in cases:
        (cnt, msgs, fails), = check(pk, kd, [asg])
        adv, inst, lens = stack(kd, [asg])
        if cnt[1]:
            with pytest.raises(lib.ConstraintSystemFailure) as e:
                pk.prove_batch(adv, inst, lens, SEED)
            first_lookup = next(f.index for f in fails if f.kind == lib.TB_FAIL_LOOKUP)
            assert "proof 0 of the batch" in str(e.value) and "lookup %d " % first_lookup in str(e.value), (name, label, str(e.value))
            continue
        proof = pk.prove_batch(adv, inst, lens, SEED)[0]
        assert pk.verify_batch(inst, lens, [proof]) == [cnt == (0, 0, 0)], (name, label, cnt)


# ---------------------------------------------------------------- 4. truncation, counts, blinding rows, seeds
def random_witness(kd, make, seed):
    """make(seed) with every advice cell of the usable rows replaced by a random value."""
    asg = make(seed)
    r = np.random.default_rng(seed)
    usable = kd.n - (kd.cs.blinding_factors() + 1)
    for c in range(kd.cs.num_advice):
        for row in range(usable):
            asg.advice[c][row] = int(r.integers(0, 1 << 62))
    return asg


@pytest.mark.parametrize("M", [0, 1, 1000])
def test_random_witness_counts_and_truncation(keys, M):
    kd, make, _, pk = keys("rotations_3")
    asg = random_witness(kd, make, 3)
    (cnt, msgs, _), = check(pk, kd, [asg], max_failures=M)
    want_cnt, want_msgs = expected(kd, asg, M)
    assert cnt == want_cnt and msgs == want_msgs
    assert all(c > 0 for c in cnt)


def test_blinding_rows_and_seed_change_nothing(keys):
    kd, make, _, pk = keys("lookups4_wide")
    asg = random_witness(kd, make, 4)
    adv, inst, lens = stack(kd, [asg, make(5)])
    a = pk.check_batch(adv, inst, lens, CHECK_SEED, max_failures=50)
    usable = kd.n - (kd.cs.blinding_factors() + 1)
    adv2 = adv.copy()
    adv2[:, :, usable:, :] = np.random.default_rng(1).integers(0, 256, adv2[:, :, usable:, :].shape, dtype=np.uint8) & 0x1F
    assert pk.check_batch(adv2, inst, lens, CHECK_SEED, max_failures=50) == a
    assert pk.check_batch(adv, inst, lens, bytes(32), max_failures=50) == a
    assert a[1] == ((0, 0, 0), [])


# ---------------------------------------------------------------- 5. the Taiga shapes at k = 15
@pytest.fixture(scope="module")
def taiga(gpu_srs):
    out = {}
    for compliance in (True, False):
        kd, make = ct.build(compliance)
        out[compliance] = (kd, make, gpu_srs.load_circuit(kd))
    yield out
    for _, _, pk in out.values():
        pk.close()


def _copied_advice_cell(kd):
    """(column, row) of an advice cell of the usable rows that is copied to another cell."""
    cols = kd.cs.perm_columns
    usable = kd.n - (kd.cs.blinding_factors() + 1)
    for (i, j), nxt in sorted(sc._cycles(kd).items()):
        if cols[i].kind == ADVICE and nxt != (i, j) and j < usable:
            return cols[i].index, j
    raise AssertionError("no copied advice cell")


@pytest.mark.parametrize("compliance", [True, False], ids=["compliance", "vp"])
def test_taiga_k15(taiga, compliance):
    kd, make, pk = taiga[compliance]
    adv, inst, lens = stack(kd, [make(3)])
    for B in (1, 7, 8, 9, 64):
        res = pk.check_batch(np.repeat(adv, B, axis=0), np.repeat(inst, B, axis=0), lens, CHECK_SEED)
        assert all(cnt == (0, 0, 0) and not fails for cnt, fails in res), B
    col, row = _copied_advice_cell(kd)
    bad = make(3)
    bad.advice[col][row] = (bad.advice[col].get(row, 0) + 1) % P
    (cnt, msgs, _), = check(pk, kd, [bad])
    assert cnt != (0, 0, 0) and msgs[0] == cr.satisfied(kd, bad)


# ---------------------------------------------------------------- 6. edges
def test_refusals_leave_the_context_usable(gpu_ctx, oracle_cpu, keys):
    kd, make, okey, pk = keys("three_instance")
    asg = make(8)
    adv, inst, lens = stack(kd, [asg])
    long_lens = lens.copy()
    long_lens[0] = kd.n
    with pytest.raises(lib.TaigaB200Error, match="InstanceTooLarge") as e:
        pk.check_batch(adv, np.zeros((1, int(long_lens.sum()), 32), np.uint8), long_lens, CHECK_SEED)
    assert e.value.status == lib.TB_ERR_INVALID
    bad_kd, _ = mutant_shape("three_instance")
    bad_kd.sigma = bad_kd.sigma.copy()
    bad_kd.sigma[0, 3] = 0
    bad_kd.sigma[0, 3, 0] = 2
    bad_pk = pk.srs.load_circuit(bad_kd)
    with pytest.raises(lib.TaigaB200Error, match="not a cell") as e:
        bad_pk.check_batch(adv, inst, lens, CHECK_SEED)
    assert e.value.status == lib.TB_ERR_INVALID
    bad_pk.close()
    assert check(pk, kd, [asg])[0][0] == (0, 0, 0)
    proof = pk.prove_batch(adv, inst, lens, SEED)[0]
    assert proof == okey.prove(adv[0], inst[0], lens, SEED)


def test_two_contexts_share_one_key(keys):
    kd, make, okey, pk = keys("sets16_deg3")
    bad = [a for _, a in sc.violations(kd, make, 5)][:4] + [make(9)]
    want = check(pk, kd, bad)
    ctxs = [lib.Context(0), lib.Context(0)]
    got, errors = {}, []

    def run(i):
        try:
            for _ in range(3):
                got.setdefault(i, []).append(check(pk, kd, bad, ctx=ctxs[i]))
        except BaseException as ex:
            errors.append(ex)
    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors
    assert all(r == want for i in range(2) for r in got[i])
    for c in ctxs:
        c.close()


def test_prove_after_check_matches_the_oracle(keys):
    kd, make, okey, pk = keys("plonk_k6_l2")
    asgs = [make(10 + b) for b in range(3)]
    check(pk, kd, asgs)
    adv, inst, lens = stack(kd, asgs)
    proofs = pk.prove_batch(adv, inst, lens, SEED)
    for b in range(3):
        assert proofs[b] == okey.prove(adv[b], inst[b], lens, SEED, proof_index=b)


# ---------------------------------------------------------------- 7. launch count
def sort_launches(n):
    """lookup.cu sort_keys: one local pass, then per merge size above the tile its global steps and one local pass."""
    tile = min(n, 2048)
    count, k = 1, tile * 2
    while k <= n:
        count += (k.bit_length() - tile.bit_length()) + 1
        k *= 2
    return count


@pytest.mark.parametrize("name,B,M", [("plonk_k6_l2", 3, 16), ("split_mixed_degrees", 9, 4), ("no_gates", 2, 0)])
def test_launch_count(keys, monkeypatch, capfd, name, B, M):
    """upload (instance and advice conversions, one PRF fill per advice column), theta, y, powers of y; the gate parts
    (one launch per part set); lookups: compression, 2 key conversions, sort, search; copies: 1; report, listed rows (when
    there are constraints and records), assembly."""
    kd, make, _, pk = keys(name)
    cs = kd.cs
    adv, inst, lens = stack(kd, [make(20 + b) for b in range(B)])
    pk.check_batch(adv, inst, lens, CHECK_SEED, max_failures=M)   # first check builds the key's check tables
    J = sum(len(p) for _, p in cs.gates)
    monkeypatch.setenv("TB_DEBUG", "1")
    capfd.readouterr()
    pk.srs.load_circuit(kd).close()
    split = "split on" in capfd.readouterr().err
    monkeypatch.delenv("TB_DEBUG")
    want = (1 if cs.num_instance else 0) + 1 + cs.num_advice + 3
    want += (1 + (1 if split else 0)) if J else 0
    want += (4 + sort_launches(kd.n)) if cs.lookups else 0
    want += 1 if cs.perm_columns else 0
    want += 1 + (1 if J and M else 0) + 1
    before = pk.ctx.launch_count
    pk.check_batch(adv, inst, lens, CHECK_SEED, max_failures=M)
    assert pk.ctx.launch_count - before == want
