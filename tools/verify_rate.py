"""Verification rate of one 64-ptx step: the 128 Compliance and 256 VP proofs of 64 partial transactions, verified from their
verifying keys (tb_verify_batch_vk), one batch per circuit.

Reports, fastest of --repeats calls:
  * wall time and proofs/s of tb_verify_batch_vk and of tb_verify_batch (the proving-key path, same code);
  * the split of a vk call: device point decoding (decompress_kernel, CUDA events), device MSMs (the instance commitments,
    the per-proof variable-base MSM and the fixed-base g term), and the rest of the wall time: the host replay, the copies
    and the few small kernels outside the profiler's categories (the calls synchronise between phases, so host and device
    time do not overlap);
  * the batch verifier (tb_batch_verifier): the same 384 proofs in one batch, both circuits, one finalize, with the same
    split into device MSMs and the rest;
  * the device path (tb_dev_verify_batch_vk, and the batch verifier with device adds): proofs and instances already in device
    memory, transcripts replayed on the device; wall time, and the device time of replay_kernel and of decompress_kernel
    from torch.profiler (one profiled call);
  * the old path, which decoded every point on the host: the same points through the host build of the same decoder
    (tests/host_shim.cpp, g++ -O2, one thread), and the wall time that path would take (vk wall - device decode + host decode).

  python tools/verify_rate.py [--repeats 5] [--tree path/to/other/checkout]

--tree measures tb_verify_batch only, with the `taiga_b200` package (and its built library) of another checkout, e.g. the
previous commit's, for a before / after comparison on the same machine.  Prints one JSON line at the end."""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_PTX = 64
COMPLIANCE_PER_PTX, VP_PER_PTX = 2, 4
WITNESSES = 4     # distinct witnesses per circuit, tiled: every proof still differs (its proof index sets its blinding)


def load_srs(ctx):
    raw = np.fromfile(os.path.join(ROOT, "tests", "golden", "srs_k15_affine.bin"), dtype=np.uint8).reshape(-1, 64)
    n = 1 << 15
    return ctx.load_srs(15, raw[:n], raw[n:2 * n], raw[2 * n], raw[2 * n + 1])


def make_proofs(pk, kd, make, count, index0, seed):
    wit = [kd.witness_arrays(make(7 + w)) for w in range(WITNESSES)]
    lens = wit[0][2]
    proofs, chunk = [], 32
    for lo in range(0, count, chunk):
        hi = min(count, lo + chunk)
        adv = np.stack([wit[i % WITNESSES][0] for i in range(lo, hi)])
        inst = np.stack([wit[i % WITNESSES][1] for i in range(lo, hi)])
        proofs += pk.prove_batch(adv, inst, lens, seed, first_proof_index=index0 + lo)
    inst = np.stack([wit[i % WITNESSES][1] for i in range(count)])
    return proofs, inst, lens


def best(fn, repeats):
    out = None
    for _ in range(repeats):
        t = time.perf_counter()
        r = fn()
        dt = time.perf_counter() - t
        out = dt if out is None else min(out, dt)
        assert all(all(v) for v in r), "a proof was rejected"
    return out


def host_decode_seconds(points):
    """the host build of transcript.cuh's decompress_point over `points` (32-byte encodings), one thread"""
    with tempfile.TemporaryDirectory() as d:
        so = os.path.join(d, "host_shim.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "host_shim.cpp")])
        shim = ctypes.CDLL(so)
        buf = np.frombuffer(b"".join(points), np.uint8)
        xy = (ctypes.c_uint8 * 64)()
        base = buf.ctypes.data
        t = time.perf_counter()
        for i in range(len(points)):
            assert shim.hs_decompress(ctypes.c_void_p(base + 32 * i), xy) == 1
        return time.perf_counter() - t


def point_chunks(kd, proofs):
    """the 32-byte encoding of every point of every proof"""
    import soundness_cases as sc   # tests/ is on the path: the slot layout of a proof
    offs = [off for _, _, off, what in sc.slots(kd) if what == "point"]
    return [p[o:o + 32] for p in proofs for o in offs]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--tree", default=None, help="another checkout with a built library: time its tb_verify_batch only")
    args = ap.parse_args()
    if args.tree:
        sys.path.insert(0, os.path.abspath(args.tree))
    from taiga_b200 import lib
    from taiga_b200 import circuits_taiga as ct
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    ctx = lib.Context(0)
    srs = load_srs(ctx)
    seed = bytes(range(32))
    circuits = []
    for compliance, count, index0 in ((True, COMPLIANCE_PER_PTX * N_PTX, 0), (False, VP_PER_PTX * N_PTX, 1 << 20)):
        kd, make = ct.build(compliance)
        pk = srs.load_circuit(kd)
        proofs, inst, lens = make_proofs(pk, kd, make, count, index0, seed)
        circuits.append((kd, pk, proofs, inst, lens))
    n_proofs = sum(len(c[2]) for c in circuits)
    pk_s = best(lambda: [pk.verify_batch(inst, lens, proofs) for _, pk, proofs, inst, lens in circuits], args.repeats)
    res = {"proofs": n_proofs, "gpu": _gpu_name(), "power_limit": _power_limit(), "pk_seconds": round(pk_s, 4), "pk_proofs_per_s": round(n_proofs / pk_s, 1)}
    if args.tree:
        res["lib"] = lib.LIB_PATH
        print(json.dumps(res))
        return
    vks = [pk.verifying_key() for _, pk, _, _, _ in circuits]
    vk_s = best(lambda: [vk.verify_batch(c[3], c[4], c[2]) for vk, c in zip(vks, circuits)], args.repeats)
    ctx.prof_enable(True)
    for vk, c in zip(vks, circuits):
        vk.verify_batch(c[3], c[4], c[2])
    prof = ctx.prof_read()
    ctx.prof_enable(False)
    decode_ms = prof["transcript"][0]
    msm_ms = sum(prof[k][0] for k in ("msm_sort", "msm_accum", "msm_reduce"))
    device_ms = decode_ms + msm_ms
    points = [p for kd, _, proofs, _, _ in circuits for p in point_chunks(kd, proofs)]
    host_dec = host_decode_seconds(points)
    old_s = vk_s - decode_ms / 1e3 + host_dec
    res.update({"vk_seconds": round(vk_s, 4), "vk_proofs_per_s": round(n_proofs / vk_s, 1),
                "device_decode_ms": round(decode_ms, 3), "device_msm_ms": round(msm_ms, 2), "host_replay_and_copies_ms": round(vk_s * 1e3 - device_ms, 1),
                "points": len(points),
                "host_decode_ms": round(host_dec * 1e3, 1), "host_decode_us_per_point": round(host_dec * 1e6 / len(points), 2),
                "host_decode_path_seconds": round(old_s, 4), "host_decode_path_proofs_per_s": round(n_proofs / old_s, 1)})
    print("tb_verify_batch_vk: %d proofs in %.1f ms (%.0f proofs/s); device decode %.2f ms, device MSMs %.1f ms, host replay and copies %.0f ms"
          % (n_proofs, vk_s * 1e3, n_proofs / vk_s, decode_ms, msm_ms, vk_s * 1e3 - device_ms))
    print("host decoding of the same %d points: %.1f ms (%.1f us/point): that path would take %.1f ms (%.0f proofs/s)"
          % (len(points), host_dec * 1e3, host_dec * 1e6 / len(points), old_s * 1e3, n_proofs / old_s))
    # the batch verifier: one batch of both circuits, one finalize
    def batch():
        bv = lib.BatchVerifier(srs, bytes(range(7, 39)))
        for vk, c in zip(vks, circuits):
            bv.add(vk, c[3], c[4], c[2])
        ok = bv.finalize()
        bv.close()
        return [[ok]]
    bv_s = best(batch, args.repeats)
    ctx.prof_enable(True)
    batch()
    prof = ctx.prof_read()
    ctx.prof_enable(False)
    bv_msm_ms = sum(prof[k][0] for k in ("msm_sort", "msm_accum", "msm_reduce"))
    bv_other_ms = prof["transcript"][0] + prof["ipa_fold"][0]
    res.update({"batch_seconds": round(bv_s, 4), "batch_proofs_per_s": round(n_proofs / bv_s, 1), "batch_device_msm_ms": round(bv_msm_ms, 2),
                "batch_device_decode_weights_g_ms": round(bv_other_ms, 3), "batch_host_replay_and_copies_ms": round(bv_s * 1e3 - bv_msm_ms - bv_other_ms, 1)})
    print("tb_batch_verifier:  %d proofs in %.1f ms (%.0f proofs/s); device MSMs %.1f ms, device decode + weights + g-term %.2f ms, host replay and copies %.0f ms"
          % (n_proofs, bv_s * 1e3, n_proofs / bv_s, bv_msm_ms, bv_other_ms, bv_s * 1e3 - bv_msm_ms - bv_other_ms))
    res.update(device_path(ctx, srs, vks, circuits, args.repeats, n_proofs))
    print("measured on: %s, power limit %s" % (res["gpu"], res["power_limit"]))
    print(json.dumps(res))
    for vk in vks:
        vk.close()


def device_path(ctx, srs, vks, circuits, repeats, n_proofs):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from taiga_b200 import lib
    on_dev = [(vk, torch.from_numpy(np.frombuffer(b"".join(c[2]), np.uint8).reshape(len(c[2]), -1).copy()).cuda(),
               torch.from_numpy(np.ascontiguousarray(c[3], dtype=np.uint8).reshape(len(c[2]), -1).copy()).cuda(), c[4]) for vk, c in zip(vks, circuits)]
    oks = [torch.zeros(p.shape[0], dtype=torch.uint8, device="cuda") for _, p, _, _ in on_dev]
    torch.cuda.synchronize()

    def per_proof():
        for (vk, p, i, lens), ok in zip(on_dev, oks):
            vk.verify_batch_dev(i, lens, p, ok)
        ctx.sync()
        return [[bool(o.all())] for o in oks]

    def batch():
        bv = lib.BatchVerifier(srs, bytes(range(7, 39)))
        for vk, p, i, lens in on_dev:
            bv.add(vk, i, lens, p)
        ok = bv.finalize()
        bv.close()
        return [[ok]]
    out = {}
    for name, fn in (("dev_vk", per_proof), ("dev_batch", batch)):
        s = best(fn, repeats)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
        kern = {}
        for e in prof.key_averages():
            for k in ("replay_kernel", "decompress_kernel"):
                if k in e.key:
                    kern[k] = kern.get(k, 0.0) + e.device_time_total / 1e3
        out.update({name + "_seconds": round(s, 4), name + "_proofs_per_s": round(n_proofs / s, 1),
                    name + "_replay_kernel_ms": round(kern.get("replay_kernel", 0.0), 2), name + "_decompress_ms": round(kern.get("decompress_kernel", 0.0), 3)})
        print("%-19s %d proofs in %.1f ms (%.0f proofs/s); replay_kernel %.2f ms, decompress_kernel %.3f ms of device time"
              % (name + ":", n_proofs, s * 1e3, n_proofs / s, kern.get("replay_kernel", 0.0), kern.get("decompress_kernel", 0.0)))
    return out


def _gpu_name():
    try:
        import torch
        return torch.cuda.get_device_name(0)
    except Exception:
        return "?"


def _power_limit():
    """the enforced power limit of GPU 0, as nvidia-smi reports it (a read-only query)"""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "?"
    except Exception:
        return "?"


if __name__ == "__main__":
    main()
