"""Every long-lived device allocation of libtaiga_b200 is held by one owner type, `DevMem` in common.cuh, and the context's
stream and events are created and destroyed only by `Ctx` and tb_ctx_create, so that each is freed exactly once, on error
paths too.

The CPU tests check the sources.  The GPU tests check that keys, SRSs and contexts can be created and released in any
order the API allows: a key proves on a second context after the one that loaded it is closed, a refused circuit leaves
its context usable, and repeated set-up and tear-down gives the same proof every time."""
import pytest

from taiga_b200 import circuits_mini as cm
from taiga_b200 import lib
from taiga_b200.circuit import Assignment, CircuitKeyData, ConstraintSystem
from test_launch_sites import sites, sources


def span(file, signature):
    """(file, start, end) of the brace-delimited body that follows `signature` in `file`."""
    text = sources()[file]
    start = text.index("{", text.index(signature))
    depth = 0
    for i in range(start, len(text)):
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        if depth == 0:
            return file, start, i + 1
    raise AssertionError("unbalanced body after " + signature)


def outside(found, *spans):
    """the matches of `found` that lie in none of `spans`"""
    return [(f, at) for f, at in found if not any(f == sf and lo <= at < hi for sf, lo, hi in spans)]


def test_synchronous_allocation_only_in_owner():
    found = sites(r"\bcuda(Malloc|Free)\(")
    assert found and outside(found, span("common.cuh", "struct DevMem {")) == []


def test_stream_ordered_allocation_only_in_context():
    found = sites(r"\bcuda(MallocAsync|FreeAsync)\(")
    assert found and outside(found, span("common.cuh", "T* alloc(size_t count)"), span("common.cuh", "void free(void* p)")) == []


def test_streams_and_events_only_in_context():
    found = sites(r"\bcuda(EventCreate|EventDestroy|StreamCreate\w*|StreamDestroy)\(")
    assert found and outside(found, span("common.cuh", "struct Ctx {"), span("capi.cu", "tb_status tb_ctx_create(")) == []


# ---------------------------------------------------------------- GPU
SEED = bytes(range(32))


@pytest.fixture(scope="module")
def plonk6(oracle_cpu):
    """k = 6 circuit with lookups and copy constraints, its SRS, one witness and the oracle's proof of it."""
    kd, make = cm.standard_plonk(k=6, n_lookups=2)
    srs = oracle_cpu.synthetic_srs(6)
    adv, inst, lens = kd.witness_arrays(make(9))
    want = oracle_cpu.OracleKey(kd, srs).prove(adv, inst, lens, SEED)
    return kd, srs, adv, inst, lens, want


def load_srs(ctx, srs):
    return ctx.load_srs(6, srs["g"], srs["g_lagrange"], srs["w"], srs["u"])


@pytest.mark.gpu
def test_key_proves_after_its_loading_context_is_closed(plonk6):
    kd, srs, adv, inst, lens, want = plonk6
    a, b = lib.Context(0), lib.Context(0)
    gsrs = load_srs(a, srs)
    pk = gsrs.load_circuit(kd)
    before = pk.prove_batch_raw(adv[None], 1, inst[None], lens, SEED, ctx=b)[0]
    assert before == want
    a.close()
    after = pk.prove_batch_raw(adv[None], 1, inst[None], lens, SEED, ctx=b)[0]
    assert after == before
    assert pk.verify_batch(inst[None], lens, [after], ctx=b) == [True]
    pk.close()
    gsrs.close()
    b.close()


def too_many_temporaries(k=6, terms=64):
    """One gate A*3 + (A*4 + (A*5 + ...)): evaluated right to left, each level keeps its left term live, so the expression
    needs about `terms` temporaries, more than the 48 the quotient interpreter holds."""
    cs = ConstraintSystem()
    A = cs.query(cs.advice_column())
    acc = A * (terms + 2)
    for i in reversed(range(terms - 1)):
        acc = A * (i + 3) + acc
    cs.create_gate("deep", [acc])
    return CircuitKeyData(cs, k, Assignment(cs, k), name="too_many_temporaries")


@pytest.mark.gpu
def test_refused_circuit_leaves_context_usable(plonk6):
    kd, srs, adv, inst, lens, want = plonk6
    ctx = lib.Context(0)
    gsrs = load_srs(ctx, srs)
    with pytest.raises(lib.TaigaB200Error, match="too many live temporaries") as e:
        gsrs.load_circuit(too_many_temporaries())
    assert e.value.status == lib.TB_ERR_INVALID
    pk = gsrs.load_circuit(kd)
    proof = pk.prove_batch(adv[None], inst[None], lens, SEED)[0]
    assert proof == want
    assert pk.verify_batch(inst[None], lens, [proof]) == [True]
    pk.close()
    gsrs.close()
    ctx.close()


@pytest.mark.gpu
def test_repeated_setup_and_teardown(plonk6):
    kd, srs, adv, inst, lens, want = plonk6
    for _ in range(10):
        ctx = lib.Context(0)
        gsrs = load_srs(ctx, srs)
        pk = gsrs.load_circuit(kd)
        proof = pk.prove_batch(adv[None], inst[None], lens, SEED)[0]
        assert proof == want
        assert pk.verify_batch(inst[None], lens, [proof]) == [True]
        pk.close()
        gsrs.close()
        ctx.close()
