"""GPU parity at the batch sizes the metric is quoted on (BASELINE configs[2]: 64 partial transactions per GPU).

  * a k = 15 batch that crosses the `max_batch = 64` chunk boundary of ProverService (ptx.py), proved through the
    threaded multi-worker path bench.py times: sampled proofs must equal the CPU oracle's byte for byte (the oracle
    needs seconds per proof, so only a sample is re-proved), the rest must equal a second GPU run with another chunking,
    and every proof must be accepted by the device verifier;
  * the batched MSM path (msm_batch.cu: counting sort in shared memory + batch-affine rounds) against the latency path
    for skewed scalar distributions, at the sizes where the prover uses it.
The reference builds these proofs one by one (shielded_ptx.rs:107-125); the batch is this framework's unit of work."""
import os

import numpy as np
import pytest

from taiga_b200 import circuits_taiga as ct
from taiga_b200 import lib, ptx

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def service(srs_fixture):
    return ptx.ProverService(0, srs_fixture, c_workers=2, v_workers=2)


def test_batch_of_65_across_chunk_boundary_threaded(service, oracle_cpu, srs_fixture):
    svc = service
    n_c, n_v = 66, 70     # > max_batch = 64 with two workers each: chunks of 33 / 35; with max_batch = 16 many chunks
    base = svc.synthesize_ptx(2, wseed=7)   # 4 Compliance + 8 VP distinct witnesses, tiled (distinct proof indices => distinct proofs)
    wit = {"c_adv": np.concatenate([base["c_adv"]] * 17)[:n_c], "c_inst": np.concatenate([base["c_inst"]] * 17)[:n_c], "c_len": base["c_len"],
           "v_adv": np.concatenate([base["v_adv"]] * 9)[:n_v], "v_inst": np.concatenate([base["v_inst"]] * 9)[:n_v], "v_len": base["v_len"]}
    seed = bytes(range(50, 82))
    pc, pv = svc.build_ptx_batch(wit, seed)                       # threaded, 2 workers per circuit, one call per worker
    pc2, pv2 = svc.build_ptx_batch(wit, seed, max_batch=16)       # same proofs through many small chunks
    assert pc == pc2 and pv == pv2, "proof bytes depend on how the batch was chunked"
    assert len(set(pc)) == n_c and len(set(pv)) == n_v
    # every proof under the device verifier
    assert all(svc.pk_c.verify_batch(wit["c_inst"], wit["c_len"], pc))
    assert all(svc.pk_v.verify_batch(wit["v_inst"], wit["v_len"], pv, ctx=svc.v_workers[0][0]))
    # sampled proofs byte-identical to the CPU oracle (first / chunk boundary / last)
    okc, okv = oracle_cpu.OracleKey(svc.kd_c, srs_fixture), oracle_cpu.OracleKey(svc.kd_v, srs_fixture)
    for i in (0, 33, n_c - 1):
        assert pc[i] == okc.prove(wit["c_adv"][i], wit["c_inst"][i], wit["c_len"], seed, proof_index=i), "Compliance proof %d differs from the oracle" % i
    for i in (34, n_v - 1):
        assert pv[i] == okv.prove(wit["v_adv"][i], wit["v_inst"][i], wit["v_len"], seed, proof_index=(1 << 20) + i), "VP proof %d differs from the oracle" % i


def test_one_call_batch_64_matches_single_proofs(service):
    """tb_prove_batch with n_proofs = 64 in ONE call (the largest chunk ProverService issues) == 64 calls with n_proofs = 1."""
    svc = service
    base = svc.synthesize_ptx(1, wseed=3)
    adv = np.concatenate([base["v_adv"]] * 16)
    inst = np.concatenate([base["v_inst"]] * 16)
    seed = bytes(range(7, 39))
    ctx, pk = svc.v_workers[0]
    batch = pk.prove_batch_raw(adv, 64, inst, base["v_len"], seed, 500, ctx=ctx)
    for i in (0, 1, 31, 63):
        one = pk.prove_batch_raw(adv[i:i + 1], 1, inst[i:i + 1], base["v_len"], seed, 500 + i, ctx=ctx)
        assert one[0] == batch[i]


@pytest.mark.parametrize("kind", ["uniform", "ones", "bits", "witness", "same"])
def test_batched_msm_path_equals_latency_path(gpu_ctx, gpu_srs, oracle_cpu, srs_fixture, kind, monkeypatch):
    n, K = 1 << 15, 5
    rng = np.random.default_rng(11)
    s = rng.integers(0, 256, size=(K, n, 32), dtype=np.uint8)
    s[:, :, 31] &= 0x3F
    if kind == "ones":
        s[:] = 0; s[:, :, 0] = 1
    elif kind == "bits":
        s[:] = 0; s[:, :, 0] = rng.integers(0, 2, size=(K, n), dtype=np.uint8)
    elif kind == "witness":   # SURVEY 8d: 30 % zero, 30 % one, 20 % < 2^8, 8 % < 2^32, 12 % uniform
        u = rng.random((K, n))
        s[u < 0.3] = 0
        o = (u >= 0.3) & (u < 0.6); s[o] = 0; s[o, 0] = 1
        s[(u >= 0.6) & (u < 0.8), 1:] = 0
        s[(u >= 0.8) & (u < 0.88), 4:] = 0
    elif kind == "same":
        s[:] = s[:, :1, :]
    bl = rng.integers(0, 256, size=(K, 32), dtype=np.uint8); bl[:, 31] &= 0x3F
    monkeypatch.setenv("TB_MSM_BA_MIN_TERMS", str(1 << 30))
    a = gpu_srs.commit(s, bl, lagrange=True, batch=K)
    monkeypatch.setenv("TB_MSM_BA_MIN_TERMS", "0")
    b = gpu_srs.commit(s, bl, lagrange=True, batch=K)
    monkeypatch.setenv("TB_MSM_BA_ROUNDS", "4")      # leftovers go through the finishing kernel
    c = gpu_srs.commit(s, bl, lagrange=True, batch=K)
    assert a.tobytes() == b.tobytes() == c.tobytes()
    if kind in ("uniform", "witness"):   # ... and the oracle (Params::commit_lagrange = MSM + blind * w)
        want = oracle_cpu.msm(oracle_cpu.VESTA, np.concatenate([s[0], bl[0][None]]), np.concatenate([srs_fixture["g_lagrange"], srs_fixture["w"][None]]))
        assert want.tobytes() == a[0].tobytes()


def test_tuning_knobs_do_not_change_results(gpu_ctx, oracle_cpu, monkeypatch):
    """A mis-set TB_* environment variable on a user's box may cost speed, never correctness."""
    from taiga_b200 import circuits_mini as cm
    kd, make = cm.standard_plonk(k=9, wide=True, n_lookups=2)
    srs = oracle_cpu.synthetic_srs(9, seed=9)
    gsrs = gpu_ctx.load_srs(9, srs["g"], srs["g_lagrange"], srs["w"], srs["u"])
    pk = gsrs.load_circuit(kd)
    wit = [kd.witness_arrays(make(300 + b)) for b in range(3)]
    adv, inst, lens = np.stack([w[0] for w in wit]), np.stack([w[1] for w in wit]), wit[0][2]
    seed = bytes(range(32))
    ref = pk.prove_batch(adv, inst, lens, seed)
    for knobs in ({"TB_MSM_BA_MIN_TERMS": "0"}, {"TB_MSM_BA_MIN_TERMS": "0", "TB_MSM_BA_ROUNDS": "2", "TB_MSM_BA_CHUNK": "3"}):
        for k_, v_ in knobs.items():
            monkeypatch.setenv(k_, v_)
        assert pk.prove_batch(adv, inst, lens, seed) == ref, knobs
        for k_ in knobs:
            monkeypatch.delenv(k_)


def test_cpp_host_mirror_proves_and_verifies_on_the_gpu(tmp_path):
    """include/taiga_b200.hpp + examples/prove_cpp.cpp (the C++ mirror of Proof::create / Proof::verify, proof.rs:25-54) on real
    hardware: builds with the host compiler, creates a proof through the C ABI, verifies it and rejects a wrong instance."""
    import subprocess
    from conftest import ROOT
    exe = str(tmp_path / "prove_cpp")
    libdir = os.path.dirname(lib.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "prove_cpp.cpp"),
                        "-L", libdir, "-ltaiga_b200", "-Wl,-rpath," + libdir, "-o", exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "created and verified" in r.stdout and "wrong instance rejected" in r.stdout
