"""GPU: verification of proofs held in device memory (tb_dev_verify_batch_vk, tb_dev_batch_verifier_add), with the
transcripts replayed on the device.

* Every verdict equals tb_verify_batch_vk's on host copies of the same bytes: honest proofs of the mini circuits, random
  and boundary shapes, both Taiga shapes in calls of 1, 64 and 65 and the golden proofs; every soundness mutant and proof of
  a false statement at moving positions among honest proofs; a non-canonical instance value; a wrong proof_len (all 0);
  rows one byte longer than the proof (an odd stride).
* Refusals return TB_ERR_INVALID, launch nothing and leave d_ok_out as it was.
* The call returns before the stream has run it, and reads its inputs in stream order.
* The batch verifier with device adds, alone and mixed with host adds; a cancelling pair split across a host and a device
  add; 4160 proofs; refused device adds; one batch fed by two contexts; two threads verifying on their own contexts."""
import ctypes
import os
import threading

import numpy as np
import pytest
import torch

import soundness_cases as sc
from conftest import GOLDEN
from taiga_b200 import circuits_mini as cm
from taiga_b200 import circuits_random as cr
from taiga_b200 import lib

from test_gpu_batch_verify import MINI, PLACEMENTS, RANDOM, SEEDS, _honest, keys, shift_f, small, srs_for, taiga  # noqa: F401
from test_gpu_verifier_soundness import PROVE_SHAPES, stack
from test_verifier_soundness import MUTANT_SHAPES, SEED

pytestmark = pytest.mark.gpu
P = cr.P


def d_proofs(proofs, pad=0):
    """the proofs on the device, one per row of a [B, L + pad] tensor, as a [B, L] view (row stride L + pad)"""
    L = len(proofs[0])
    t = torch.zeros((len(proofs), L + pad), dtype=torch.uint8)
    t[:, :L] = torch.from_numpy(np.frombuffer(b"".join(proofs), np.uint8).reshape(len(proofs), L).copy())
    return t.cuda()[:, :L]


def d_inst(inst, B):
    return torch.from_numpy(np.ascontiguousarray(inst, dtype=np.uint8).reshape(B, -1).copy()).cuda()


def dev_verify(vk, inst, lens, proofs, pad=0, proof_len=None, ctx=None):
    ctx = ctx or vk.ctx
    ok = torch.full((len(proofs),), 0xAB, dtype=torch.uint8, device="cuda")
    vk.verify_batch_dev(d_inst(inst, len(proofs)), lens, d_proofs(proofs, pad), ok, ctx=ctx, proof_len=proof_len)
    ctx.sync()
    return [bool(v) for v in ok.cpu().tolist()]


def same(vk, inst, lens, proofs):
    want = vk.verify_batch(inst, lens, proofs)
    assert dev_verify(vk, inst, lens, proofs) == want
    return want


def run_mixed(srs, seed, adds):
    """finalize() after adds (vk, instance, lens, proofs, on_device)"""
    bv = lib.BatchVerifier(srs, seed)
    try:
        for vk, inst, lens, proofs, on_dev in adds:
            if on_dev:
                bv.add(vk, d_inst(inst, len(proofs)), lens, d_proofs(proofs))
            else:
                bv.add(vk, inst, lens, proofs)
        return bv.finalize()
    finally:
        bv.close()


# ---------------------------------------------------------------- per-proof verdicts
@pytest.mark.parametrize("k,wide,nl", MINI)
def test_mini_circuits(srs_for, k, wide, nl):
    kd, make = cm.standard_plonk(k=k, wide=wide, n_lookups=nl)
    _, gsrs = srs_for(k)
    pk = gsrs.load_circuit(kd)
    vk = pk.verifying_key()
    proofs, inst, lens = _honest(kd, make, pk, 3)
    assert same(vk, inst, lens, proofs) == [True] * 3
    bad = bytearray(proofs[1])
    bad[len(bad) // 2] ^= 1
    assert same(vk, inst, lens, [proofs[0], bytes(bad), proofs[2]]) == [True, False, True]
    if (k, wide, nl) == (6, False, 2):
        _, inst1, lens1 = kd.witness_arrays(make(100))
        golden = open(os.path.join(GOLDEN, "proof_k6_plonk.bin"), "rb").read()
        assert same(vk, inst1[None], lens1, [golden]) == [True]
    vk.close()
    pk.close()


@pytest.mark.parametrize("which", RANDOM, ids=["%s-%s" % w for w in RANDOM])
def test_random_and_boundary_shapes(srs_for, which):
    kind, v = which
    kd, make = cr.boundary(v) if kind == "boundary" else cr.random_shape(v)
    _, gsrs = srs_for(kd.k)
    pk = gsrs.load_circuit(kd)
    vk = pk.verifying_key()
    proofs, inst, lens = _honest(kd, make, pk, 2, w0=11)
    assert same(vk, inst, lens, proofs) == [True, True]
    vk.close()
    pk.close()


def test_taiga_shapes_in_calls_of_1_64_65(taiga):
    for compliance in (True, False):
        kd, pk, vk, proofs, inst, lens, golden, golden_inst = taiga[compliance]
        for B in (1, 64, 65):
            assert dev_verify(vk, inst[:B], lens, proofs[:B]) == [True] * B
        assert same(vk, golden_inst, lens, [golden]) == [True]


@pytest.mark.parametrize("name", MUTANT_SHAPES)
def test_every_mutant_among_honest_proofs(keys, name):
    kd, make, gsrs, pk, vk = keys(name)
    proofs, inst, lens = _honest(kd, make, pk, 4)
    muts = [m for _, _, _, m in sc.mutants(kd, proofs[0], proofs[1]) if len(m) == len(proofs[0])]
    for i, m in enumerate(muts):
        at = i % 4
        row = list(proofs[1:])
        row.insert(at, m)
        rinst = np.stack([inst[j] for j in (1, 2, 3)][:at] + [inst[0]] + [inst[j] for j in (1, 2, 3)][at:])
        got = dev_verify(vk, rinst, lens, row)
        assert got == [j != at for j in range(4)], "%s mutant %d at %d: %r" % (name, i, at, got)
    assert dev_verify(vk, inst, lens, proofs) == [True] * 4


@pytest.mark.parametrize("name", PROVE_SHAPES)
def test_false_statements_among_honest_proofs(keys, name):
    kd, make, gsrs, pk, vk = keys(name)
    bad = [a for label, a in sc.violations(kd, make, 5) if not label.startswith("lookup")]
    adv, inst, lens = stack(kd, [make(100 + i) for i in range(3)] + bad)
    proofs = pk.prove_batch(adv, inst, lens, SEED)
    for i in range(len(bad)):
        at = i % 4
        order = [0, 1, 2]
        order.insert(at, 3 + i)
        assert same(vk, inst[order], lens, [proofs[j] for j in order]) == [j != at for j in range(4)]


def test_noncanonical_instance_wrong_length_and_odd_stride(small):
    gsrs, pk, vk, proofs, inst, lens = small
    assert lens[0] >= 1
    bad = np.array(inst[:3], dtype=np.uint8).reshape(3, -1)
    v = int.from_bytes(bad[1, :32].tobytes(), "little") + P   # the same value + p: not canonical
    assert v < 1 << 256
    bad[1, :32] = np.frombuffer(v.to_bytes(32, "little"), np.uint8)
    assert same(vk, bad, lens, proofs[:3]) == [True, False, True]
    assert dev_verify(vk, inst[:5], lens, proofs[:5], proof_len=len(proofs[0]) - 32) == [False] * 5
    assert dev_verify(vk, inst[:5], lens, proofs[:5], pad=1) == [True] * 5
    assert dev_verify(vk, inst[:5], lens, proofs[:5], pad=7) == [True] * 5


def test_refusals_launch_nothing_and_leave_the_verdicts(small):
    gsrs, pk, vk, proofs, inst, lens = small
    ctx = vk.ctx
    so = ctx._lib
    dp, di = d_proofs(proofs[:4]), d_inst(inst[:4], 4)
    L = len(proofs[0])
    ok = torch.full((8,), 0xAB, dtype=torch.uint8, device="cuda")
    lens_ok = np.ascontiguousarray(lens, dtype=np.uint32)
    too_long = lens_ok.copy()
    too_long[0] = (1 << 6) + 5
    host = np.frombuffer(b"".join(proofs[:4]), np.uint8).copy()
    cases = [(4097, di.data_ptr(), lens_ok, dp.data_ptr(), L, L, ok.data_ptr()),
             (0, di.data_ptr(), lens_ok, dp.data_ptr(), L, L, ok.data_ptr()),
             (4, di.data_ptr(), lens_ok, dp.data_ptr(), L - 1, L, ok.data_ptr()),
             (4, di.data_ptr(), too_long, dp.data_ptr(), L, L, ok.data_ptr()),
             (4, di.data_ptr(), lens_ok, None, L, L, ok.data_ptr()),
             (4, di.data_ptr(), lens_ok, host.ctypes.data, L, L, ok.data_ptr())]
    torch.cuda.synchronize()
    for i, (B, pi, ln, pp, stride, plen, po) in enumerate(cases):
        before = ctx.launch_count
        st = so.tb_dev_verify_batch_vk(ctx._h, vk._h, B, ctypes.c_void_p(pi), lib._ptr(ln), ctypes.c_void_p(pp), stride, plen, ctypes.c_void_p(po))
        assert st == lib.TB_ERR_INVALID, (i, st)
        assert ctx.launch_count == before, i
    ctx.sync()
    assert ok.cpu().tolist() == [0xAB] * 8


def test_returns_before_the_stream_and_reads_in_stream_order(small):
    gsrs, pk, vk, proofs, inst, lens = small
    ctx = vk.ctx
    honest = d_proofs(proofs[:16])
    target = d_proofs([bytes(b ^ 0x55 for b in p) for p in proofs[:16]])
    di = d_inst(inst[:16], 16)
    ok = torch.zeros(16, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    stream = torch.cuda.ExternalStream(ctx.stream)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(2_000_000_000)   # about a second
        target.copy_(honest)
        vk.verify_batch_dev(di, lens, target, ok)
        assert not stream.query()
    ctx.sync()
    assert ok.cpu().tolist() == [1] * 16


# ---------------------------------------------------------------- batch verifier
def test_device_adds_and_mixed_adds(small, taiga, gpu_srs):
    gsrs, pk, vk, proofs, inst, lens = small
    assert run_mixed(gsrs, SEEDS[0], [(vk, inst[:20], lens, proofs[:20], True), (vk, inst[20:], lens, proofs[20:], True)])
    assert run_mixed(gsrs, SEEDS[1], [(vk, inst[:20], lens, proofs[:20], False), (vk, inst[20:40], lens, proofs[20:40], True),
                                      (vk, inst[40:], lens, proofs[40:], False)])
    bad = bytearray(proofs[30])
    bad[200] ^= 1
    mixed = proofs[:30] + [bytes(bad)] + proofs[31:]
    for on_dev in (True, False):
        assert not run_mixed(gsrs, SEEDS[0], [(vk, inst[:20], lens, mixed[:20], not on_dev), (vk, inst[20:], lens, mixed[20:], on_dev)])
    c, v = taiga[True], taiga[False]
    assert run_mixed(gpu_srs, SEEDS[2], [(c[2], c[4], c[5], c[3], True), (v[2], v[4][:64], v[5], v[3][:64], False), (v[2], v[4][64:], v[5], v[3][64:], True)])


@pytest.mark.parametrize("seed", SEEDS, ids=["seed%d" % i for i in range(len(SEEDS))])
def test_cancelling_pair_across_host_and_device_adds(small, seed):
    gsrs, pk, vk, proofs, inst, lens = small
    up, down = shift_f(proofs[1], 1), shift_f(proofs[3], -1)
    assert dev_verify(vk, inst[:4], lens, [proofs[0], up, proofs[2], down]) == [True, False, True, False]
    assert not run_mixed(gsrs, seed, [(vk, inst[:2], lens, [proofs[0], up], False), (vk, inst[2:4], lens, [proofs[2], down], True)])
    assert not run_mixed(gsrs, seed, [(vk, inst[:2], lens, [proofs[0], up], True), (vk, inst[2:4], lens, [proofs[2], down], False)])


def test_4160_proofs_through_device_adds(small):
    gsrs, pk, vk, proofs, inst, lens = small
    allp = [proofs[i % 64] for i in range(4160)]
    alli = np.stack([inst[i % 64] for i in range(4160)])
    assert run_mixed(gsrs, SEEDS[0], [(vk, alli[:4096], lens, allp[:4096], True), (vk, alli[4096:], lens, allp[4096:], True)])
    bad = bytearray(allp[4100])
    bad[100] ^= 1
    allp[4100] = bytes(bad)
    assert not run_mixed(gsrs, SEEDS[0], [(vk, alli[:4096], lens, allp[:4096], True), (vk, alli[4096:], lens, allp[4096:], True)])


def test_refused_device_adds_leave_the_batch(small, srs_for):
    gsrs, pk, vk, proofs, inst, lens = small
    _, other = srs_for(7)
    kd7, _ = cm.standard_plonk(k=7, wide=True, n_lookups=1)
    pk7 = other.load_circuit(kd7)
    vk7 = pk7.verifying_key()
    ctx = gsrs.ctx
    bv = lib.BatchVerifier(gsrs, SEEDS[0])
    dp, di = d_proofs(proofs[:4]), d_inst(inst[:4], 4)
    L = len(proofs[0])
    ln = np.ascontiguousarray(lens, dtype=np.uint32)
    for h, B, stride in ((vk._h, 4097, L), (vk._h, 4, L - 1), (vk7._h, 4, L)):
        before = ctx.launch_count
        st = ctx._lib.tb_dev_batch_verifier_add(ctx._h, bv._h, h, B, ctypes.c_void_p(di.data_ptr()), lib._ptr(ln), ctypes.c_void_p(dp.data_ptr()), stride, L)
        assert st == lib.TB_ERR_INVALID and ctx.launch_count == before
    bv.add(vk, di, lens, dp)
    assert bv.finalize()
    st = ctx._lib.tb_dev_batch_verifier_add(ctx._h, bv._h, vk._h, 4, ctypes.c_void_p(di.data_ptr()), lib._ptr(ln), ctypes.c_void_p(dp.data_ptr()), L, L)
    assert st == lib.TB_ERR_INVALID
    bv.close()
    vk7.close()
    pk7.close()


def test_one_batch_fed_by_two_contexts(small):
    gsrs, pk, vk, proofs, inst, lens = small
    other = lib.Context(0)
    for bad_at in (None, 40):
        ps = list(proofs)
        if bad_at is not None:
            b = bytearray(ps[bad_at])
            b[64] ^= 1
            ps[bad_at] = bytes(b)
        bv = lib.BatchVerifier(gsrs, SEEDS[1])
        bv.add(vk, d_inst(inst[:32], 32), lens, d_proofs(ps[:32]))
        bv.add(vk, d_inst(inst[32:], 32), lens, d_proofs(ps[32:]), ctx=other)
        assert bv.finalize() is (bad_at is None)
        bv.close()
    other.close()


def test_concurrent_contexts(small):
    gsrs, pk, vk, proofs, inst, lens = small
    bad = bytearray(proofs[5])
    bad[300] ^= 1
    ps = proofs[:5] + [bytes(bad)] + proofs[6:32]
    want = [i != 5 for i in range(32)]
    results, errors = {}, []

    def work(t):
        try:
            ctx = lib.Context(0)
            for _ in range(3):
                results.setdefault(t, []).append(dev_verify(vk, inst[:32], lens, ps, ctx=ctx))
            ctx.close()
        except Exception as e:   # reported below
            errors.append(e)
    threads = [threading.Thread(target=work, args=(t,)) for t in range(2)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    assert all(r == want for rs in results.values() for r in rs) and len(results) == 2
