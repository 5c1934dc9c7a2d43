"""GPU: proving into device memory (tb_dev_prove_batch, ProvingKey.prove_batch_dev, ProverService.build_ptx_batch_dev).

* Byte parity: every record equals tb_prove_batch's for the same seed and proof index, with every status TB_PROVED: the mini
  circuits, random and boundary shapes, both Taiga shapes in calls of 1, 64 and 65, a first_proof_index other than 0, and
  advice given as views of a larger device buffer.  The k = 15 keys are freed after their test, with their workspaces for
  batches of 64 and 65.
* Records at strides of proof_len + 1 and + 3 in a sentinel-filled tensor: the bytes outside the records keep the sentinel.
* Lookup failures: a witness that breaks lookup l, first, in the middle or last among honest witnesses, gets status 1 + l and
  a zero record, and every other record is the honest one; a witness that breaks two lookups reports the lower; tb_prove_batch
  on the same batch still raises ConstraintSystemFailure.
* The call returns while the stream is still busy, proves what torch's stream wrote just before it, and two calls on one
  context, or on two threads' own contexts, are both correct.
* Refusals return TB_ERR_INVALID, launch nothing and leave the outputs as they were.
* A device call launches the host call's kernels plus one.
* Round trip into the device verifier and the device batch verifier; ProverService.build_ptx_batch_dev for 1 and 64
  partial transactions gives build_ptx_batch's bytes, and verify_ptx_batch accepts the tensors."""
import ctypes
import threading

import numpy as np
import pytest
import torch

import soundness_cases as sc
from taiga_b200 import circuits_mini as cm
from taiga_b200 import circuits_random as cr
from taiga_b200 import circuits_taiga as ct
from taiga_b200 import lib, ptx

from test_gpu_batch_verify import MINI, RANDOM, SEEDS, srs_for  # noqa: F401
from test_gpu_verifier_soundness import keys, stack  # noqa: F401
from test_verifier_soundness import SEED

pytestmark = pytest.mark.gpu
SENTINEL = 0xA7


def d_adv(adv):
    return torch.from_numpy(np.ascontiguousarray(adv, dtype=np.uint8)).cuda()


def d_inst(inst, B):
    return torch.from_numpy(np.ascontiguousarray(inst, dtype=np.uint8).reshape(B, -1).copy()).cuda()


def dev_prove(pk, adv, inst, lens, seed=SEED, first=0, pad=0, ctx=None):
    """(records as byte strings, statuses, the whole [B, proof_len + pad] output tensor on the host) of one device call;
    `adv` a numpy array or a CUDA tensor"""
    ctx = ctx or pk.ctx
    B = adv.shape[0]
    a = adv if isinstance(adv, torch.Tensor) else d_adv(adv)
    buf = torch.full((B, pk.proof_len + pad), SENTINEL, dtype=torch.uint8, device="cuda")
    status = torch.full((B,), 0x55, dtype=torch.int32, device="cuda")
    pk.prove_batch_dev(a, d_inst(inst, B), lens, seed, buf[:, :pk.proof_len], status, first_proof_index=first, ctx=ctx)
    ctx.sync()
    host = buf.cpu().numpy()
    return [host[b, :pk.proof_len].tobytes() for b in range(B)], status.cpu().tolist(), host


def same(pk, adv, inst, lens, first=0):
    want = pk.prove_batch(adv, inst, lens, SEED, first_proof_index=first)
    got, status, _ = dev_prove(pk, adv, inst, lens, first=first)
    assert status == [lib.TB_PROVED] * len(want)
    assert got == want
    return want


# ---------------------------------------------------------------- byte parity
@pytest.mark.parametrize("k,wide,nl", MINI)
def test_mini_circuits(srs_for, k, wide, nl):
    kd, make = cm.standard_plonk(k=k, wide=wide, n_lookups=nl)
    _, gsrs = srs_for(k)
    pk = gsrs.load_circuit(kd)
    adv, inst, lens = stack(kd, [make(400 + b) for b in range(3)])
    same(pk, adv, inst, lens)
    same(pk, adv, inst, lens, first=7)
    pk.close()


@pytest.mark.parametrize("which", RANDOM, ids=["%s-%s" % w for w in RANDOM])
def test_random_and_boundary_shapes(srs_for, which):
    kind, v = which
    kd, make = cr.boundary(v) if kind == "boundary" else cr.random_shape(v)
    _, gsrs = srs_for(kd.k)
    pk = gsrs.load_circuit(kd)
    adv, inst, lens = stack(kd, [make(11 + b) for b in range(2)])
    same(pk, adv, inst, lens, first=3)
    pk.close()


@pytest.mark.parametrize("compliance", [True, False], ids=["compliance", "vp"])
def test_taiga_shapes(gpu_srs, compliance):
    """calls of 1, 64 and 65 proofs; then witnesses 3..9 at proof indices 3..9, their advice a view of a larger device buffer.
    The key, and with it the workspaces of these batch sizes, is freed at the end."""
    kd, make = ct.build(compliance)
    pk = gpu_srs.load_circuit(kd)
    wit = [kd.witness_arrays(make(40 + w)) for w in range(4)]
    host_adv = np.stack([wit[b % 4][0] for b in range(65)])
    inst = np.stack([wit[b % 4][1] for b in range(65)])
    lens = wit[0][2]
    proofs = pk.prove_batch(host_adv, inst, lens, SEED)
    adv = d_adv(host_adv)
    for B in (1, 64, 65):
        got, status, _ = dev_prove(pk, adv[:B], inst[:B], lens)
        assert status == [0] * B and got == proofs[:B], B
    big = torch.zeros((70,) + tuple(adv.shape[1:]), dtype=torch.uint8, device="cuda")
    big[2:67] = adv
    got, status, _ = dev_prove(pk, big[5:12], inst[3:10], lens, first=3)
    assert status == [0] * 7 and got == proofs[3:10]
    del adv, big
    torch.cuda.synchronize()
    pk.close()


# ---------------------------------------------------------------- strides
@pytest.fixture(scope="module")
def small(srs_for):
    """the k = 6 standard PLONK shape: (pk, 16 witnesses, their instances, lens, tb_prove_batch's proofs)"""
    kd, make = cm.standard_plonk(k=6, n_lookups=2)
    _, gsrs = srs_for(6)
    pk = gsrs.load_circuit(kd)
    adv, inst, lens = stack(kd, [make(400 + b) for b in range(16)])
    proofs = pk.prove_batch(adv, inst, lens, SEED)
    yield pk, adv, inst, lens, proofs
    pk.close()


@pytest.mark.parametrize("pad", [1, 3])
def test_odd_strides_leave_the_bytes_between_records(small, pad):
    pk, adv, inst, lens, proofs = small
    L = pk.proof_len
    got, status, host = dev_prove(pk, adv, inst, lens, pad=pad)
    assert status == [0] * 16 and got == proofs
    assert (host[:, L:] == SENTINEL).all()


# ---------------------------------------------------------------- lookup failures
_BROKEN = {}


def _lookup_breaker(kd, make, lookups):
    """advice [na, n, 32] of make(5) with the input of each lookup in `lookups` taken out of its table"""
    if kd.name not in _BROKEN:
        _BROKEN[kd.name] = (kd.witness_arrays(make(5))[0],
                            {int(label[len("lookup"):]): kd.witness_arrays(a)[0] for label, a in sc.violations(kd, make, 5) if label.startswith("lookup")})
    base, found = _BROKEN[kd.name]
    out = base.copy()
    for l in lookups:
        bad = found[l]
        mask = bad != base
        assert mask.any(), l
        out[mask] = bad[mask]
    return out


@pytest.mark.parametrize("name", ["lookups4_wide", "no_gates"])
def test_lookup_failures_among_honest_witnesses(keys, name):
    kd, make, okey, pk = keys(name)
    L = len(kd.cs.lookups)
    B = 5
    adv, inst, lens = stack(kd, [make(200 + b) for b in range(B)])
    honest = pk.prove_batch(adv, inst, lens, SEED, first_proof_index=10)
    cases = [((l,), pos) for l in range(L) for pos in (0, B // 2, B - 1)]
    cases.append(((L - 1, 0), 1) if L > 1 else ((0,), 1))
    for broken, pos in cases:
        bad = adv.copy()
        bad[pos] = _lookup_breaker(kd, make, broken)
        got, status, _ = dev_prove(pk, bad, inst, lens, first=10)
        assert status == [1 + min(broken) if b == pos else lib.TB_PROVED for b in range(B)], (broken, pos, status)
        assert got[pos] == bytes(pk.proof_len), (broken, pos)
        assert [g for b, g in enumerate(got) if b != pos] == [h for b, h in enumerate(honest) if b != pos], (broken, pos)
        with pytest.raises(lib.ConstraintSystemFailure):
            pk.prove_batch(bad, inst, lens, SEED, first_proof_index=10)


# ---------------------------------------------------------------- asynchrony
def test_returns_before_the_stream_has_run_the_call(small):
    pk, adv, inst, lens, proofs = small
    ctx = pk.ctx
    dev_prove(pk, adv[:4], inst[:4], lens)   # the workspace of this batch size exists: nothing left to set up
    a, i = d_adv(adv[:4]), d_inst(inst[:4], 4)
    out = torch.zeros((4, pk.proof_len), dtype=torch.uint8, device="cuda")
    status = torch.full((4,), 0x55, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    stream = torch.cuda.ExternalStream(ctx.stream)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(2_000_000_000)   # about a second
        pk.prove_batch_dev(a, i, lens, SEED, out, status)
        assert not stream.query()
    ctx.sync()
    assert status.cpu().tolist() == [0] * 4
    assert [bytes(r) for r in out.cpu().numpy()] == proofs[:4]


def test_reads_the_advice_torch_wrote_just_before(small):
    pk, adv, inst, lens, proofs = small
    real = d_adv(adv[:4])
    a = torch.zeros_like(real)
    torch.cuda.synchronize()
    torch.cuda._sleep(500_000_000)   # on torch's stream: the copy below lands well after the call has returned
    a.copy_(real)
    got, status, _ = dev_prove(pk, a, inst[:4], lens)
    assert status == [0] * 4 and got == proofs[:4]


def test_two_calls_on_one_context_without_a_wait(small):
    pk, adv, inst, lens, proofs = small
    other_seed = SEEDS[1]
    want2 = pk.prove_batch(adv[:8], inst[:8], lens, other_seed)
    a, i = d_adv(adv[:8]), d_inst(inst[:8], 8)
    outs = [torch.zeros((8, pk.proof_len), dtype=torch.uint8, device="cuda") for _ in range(2)]
    sts = [torch.full((8,), 0x55, dtype=torch.int32, device="cuda") for _ in range(2)]
    pk.prove_batch_dev(a, i, lens, SEED, outs[0], sts[0])
    pk.prove_batch_dev(a, i, lens, other_seed, outs[1], sts[1])
    pk.ctx.sync()
    assert sts[0].cpu().tolist() == [0] * 8 and sts[1].cpu().tolist() == [0] * 8
    assert [bytes(r) for r in outs[0].cpu().numpy()] == proofs[:8]
    assert [bytes(r) for r in outs[1].cpu().numpy()] == want2


def test_two_threads_on_their_own_contexts(small):
    pk, adv, inst, lens, proofs = small
    results, errors = {}, []

    def work(t):
        try:
            ctx = lib.Context(0)
            for _ in range(3):
                got, status, _ = dev_prove(pk, adv, inst, lens, ctx=ctx)
                results.setdefault(t, []).append((got, status))
            ctx.close()
        except Exception as e:   # reported below
            errors.append(e)
    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert len(results) == 2 and all(r == (proofs, [0] * 16) for rs in results.values() for r in rs)


# ---------------------------------------------------------------- refusals and launch counts
def test_refusals_launch_nothing_and_leave_the_outputs(small):
    pk, adv, inst, lens, proofs = small
    ctx = pk.ctx
    so = ctx._lib
    L = pk.proof_len
    a, i = d_adv(adv[:4]), d_inst(inst[:4], 4)
    out = torch.full((4, L), SENTINEL, dtype=torch.uint8, device="cuda")
    status = torch.full((8,), 0x55, dtype=torch.int32, device="cuda")
    ln = np.ascontiguousarray(lens, dtype=np.uint32)
    too_long = ln.copy()
    too_long[0] = (1 << 6) + 5
    seed = np.frombuffer(SEED, np.uint8).copy()
    host_out = np.full((4, L), SENTINEL, np.uint8)
    host_status = np.full(4, 0x55, np.uint32)
    host_adv = np.ascontiguousarray(adv[:4])
    P, I, O, S, SD = a.data_ptr(), i.data_ptr(), out.data_ptr(), status.data_ptr(), seed.ctypes.data
    cases = [(pk._h, 0, P, I, ln, SD, O, L, S),
             (pk._h, 65535, P, I, ln, SD, O, L, S),        # more than one call's grid allows
             (pk._h, 4, P, I, ln, SD, O, L - 1, S),        # stride below proof_len
             (pk._h, 4, P, I, too_long, SD, O, L, S),      # InstanceTooLarge
             (pk._h, 4, P, None, ln, SD, O, L, S),         # the circuit has instance columns
             (pk._h, 4, P, I, None, SD, O, L, S),
             (pk._h, 4, None, I, ln, SD, O, L, S),
             (pk._h, 4, P, I, ln, None, O, L, S),
             (pk._h, 4, P, I, ln, SD, None, L, S),
             (pk._h, 4, P, I, ln, SD, O, L, None),
             (None, 4, P, I, ln, SD, O, L, S),
             (pk._h, 4, P, I, ln, SD, host_out.ctypes.data, L, S),        # host memory as d_proofs_out
             (pk._h, 4, host_adv.ctypes.data, I, ln, SD, O, L, S),        # host memory as d_advice
             (pk._h, 4, P, I, ln, SD, O, L, host_status.ctypes.data)]     # host memory as d_status_out
    torch.cuda.synchronize()
    for c, (h, B, pa, pi, lens_, sd, po, stride, ps) in enumerate(cases):
        before = ctx.launch_count
        st = so.tb_dev_prove_batch(ctx._h, h, B, ctypes.c_void_p(pa), ctypes.c_void_p(pi), lib._ptr(lens_), ctypes.c_void_p(sd), 0,
                                   ctypes.c_void_p(po), stride, ctypes.c_void_p(ps))
        assert st == lib.TB_ERR_INVALID, (c, st)
        assert ctx.launch_count == before, c
    ctx.sync()
    assert (out.cpu().numpy() == SENTINEL).all() and status.cpu().tolist() == [0x55] * 8
    assert (host_out == SENTINEL).all() and (host_status == 0x55).all()


def test_a_device_call_launches_the_host_calls_kernels_plus_one(small):
    pk, adv, inst, lens, proofs = small
    ctx = pk.ctx
    pk.prove_batch(adv[:8], inst[:8], lens, SEED)
    dev_prove(pk, adv[:8], inst[:8], lens)
    before = ctx.launch_count
    pk.prove_batch(adv[:8], inst[:8], lens, SEED)
    host = ctx.launch_count - before
    a, i = d_adv(adv[:8]), d_inst(inst[:8], 8)
    out = torch.zeros((8, pk.proof_len), dtype=torch.uint8, device="cuda")
    status = torch.zeros(8, dtype=torch.int32, device="cuda")
    before = ctx.launch_count
    pk.prove_batch_dev(a, i, lens, SEED, out, status)
    assert ctx.launch_count - before == host + 1
    ctx.sync()


# ---------------------------------------------------------------- into the verifiers
def test_round_trip_into_the_device_verifiers(keys):
    kd, make, okey, pk = keys("lookups4_wide")
    vk = pk.verifying_key()
    B = 6
    adv, inst, lens = stack(kd, [make(300 + b) for b in range(B)])
    for bad_at in (None, 4):
        a = adv.copy()
        if bad_at is not None:
            a[bad_at] = _lookup_breaker(kd, make, (1,))
        proofs = torch.zeros((B, pk.proof_len), dtype=torch.uint8, device="cuda")
        status = torch.zeros(B, dtype=torch.int32, device="cuda")
        di = d_inst(inst, B)
        pk.prove_batch_dev(d_adv(a), di, lens, SEED, proofs, status)
        ok = torch.zeros(B, dtype=torch.uint8, device="cuda")
        vk.verify_batch_dev(di, lens, proofs, ok)
        bv = lib.BatchVerifier(pk.srs, SEEDS[2])
        bv.add(vk, di, lens, proofs)
        verdict = bv.finalize()
        bv.close()
        assert status.cpu().tolist() == [2 if b == bad_at else 0 for b in range(B)]
        assert ok.cpu().tolist() == [0 if b == bad_at else 1 for b in range(B)]
        assert verdict is (bad_at is None)
    vk.close()


@pytest.fixture(scope="module")
def service(srs_fixture):
    svc = ptx.ProverService(0, srs_fixture, c_workers=2, v_workers=2)
    base = svc.synthesize_ptx(2, wseed=9)
    yield svc, base


@pytest.mark.parametrize("n_ptx", [1, 64])
def test_service_builds_on_the_device(service, n_ptx):
    svc, base = service
    reps = (n_ptx + 1) // 2
    wit = {"c_inst": np.concatenate([base["c_inst"]] * reps)[:2 * n_ptx], "c_len": base["c_len"],
           "v_inst": np.concatenate([base["v_inst"]] * reps)[:4 * n_ptx], "v_len": base["v_len"]}
    c_adv = d_adv(base["c_adv"]).repeat(reps, 1, 1, 1)[:2 * n_ptx]
    v_adv = d_adv(base["v_adv"]).repeat(reps, 1, 1, 1)[:4 * n_ptx]
    seed = bytes(range(60, 92))
    nw = 2 if n_ptx == 1 else 1   # a 64-ptx step as bench.py runs it: one worker per circuit (a batch of 64 fills the GPU)
    pc, pv = svc.build_ptx_batch(wit, seed, c_adv, v_adv, workers_per_circuit=nw)
    dc, dv, sc_, sv = svc.build_ptx_batch_dev(wit, seed, c_adv, v_adv, workers_per_circuit=nw)
    assert sc_.cpu().tolist() == [0] * len(pc) and sv.cpu().tolist() == [0] * len(pv)
    assert [bytes(r) for r in dc.cpu().numpy()] == pc and [bytes(r) for r in dv.cpu().numpy()] == pv
    assert svc.verify_ptx_batch(dc, dv, wit, bytes(range(32))) == (True, [True] * n_ptx)
    # another split (one worker per circuit, calls of at most 16 proofs): the same proofs
    dc2, dv2, _, _ = svc.build_ptx_batch_dev(wit, seed, c_adv, v_adv, max_batch=16, workers_per_circuit=1)
    assert torch.equal(dc2, dc) and torch.equal(dv2, dv)
