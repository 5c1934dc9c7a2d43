"""Proving into device memory against proving into host memory, on partial-transaction steps whose advice is already resident
as device tensors (2 Compliance + 4 VP proofs per partial transaction; the witnesses of 2 synthesized partial transactions,
tiled: every proof still differs, its proof index sets its blinding).

Reports, each the fastest of --repeats steps, the two paths alternating:
  1. a 64-ptx step: ProverService.build_ptx_batch (one host thread per (context, key) pair, proofs downloaded to host memory,
     one worker per circuit as bench.py runs a batch) against build_ptx_batch_dev (every call enqueued from the calling thread,
     proofs and statuses left in device memory, one torch.cuda.synchronize() at the end);
  2. the host cost of the device path: the time until build_ptx_batch_dev returns (the enqueue), and the process CPU time
     per step of both paths;
  3. the same for 1-ptx steps, two (context, key) pairs per circuit: four host threads against one;
  4. prove, then verify on the device: build_ptx_batch_dev of a 64-ptx step (one worker per circuit) into one BatchVerifier
     with device adds and a single finalize; wall time and verdict.

  python tools/prove_rate.py [--repeats 5]

Prints the GPU's name, power limit and SM clock with the numbers, and one JSON line at the end."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def load_srs_arrays():
    raw = np.fromfile(os.path.join(ROOT, "tests", "golden", "srs_k15_affine.bin"), dtype=np.uint8).reshape(-1, 64)
    n = 1 << 15
    return {"k": 15, "g": raw[:n], "g_lagrange": raw[n:2 * n], "w": raw[2 * n], "u": raw[2 * n + 1]}


def step_inputs(base, n_ptx, dev):
    """(witness dictionary, Compliance advice, VP advice) of n_ptx partial transactions: base's tiled, advice on the device"""
    import torch
    reps = (n_ptx + 1) // 2
    wit = {"c_inst": np.concatenate([base["c_inst"]] * reps)[:2 * n_ptx], "c_len": base["c_len"],
           "v_inst": np.concatenate([base["v_inst"]] * reps)[:4 * n_ptx], "v_len": base["v_len"]}
    c = torch.from_numpy(np.ascontiguousarray(base["c_adv"])).to(dev).repeat(reps, 1, 1, 1)[:2 * n_ptx].contiguous()
    v = torch.from_numpy(np.ascontiguousarray(base["v_adv"])).to(dev).repeat(reps, 1, 1, 1)[:4 * n_ptx].contiguous()
    return wit, c, v


def compare(svc, wit, c, v, nw, repeats):
    """fastest wall, enqueue and process CPU times (seconds) of both paths, alternating; checks that they give the same proofs"""
    import torch
    seed = bytes(range(32))
    best = {}

    def keep(name, value):
        best[name] = value if name not in best else min(best[name], value)
    ref = None
    for r in range(repeats + 1):   # the first round warms both paths up (workspaces, tables) and is not kept
        torch.cuda.synchronize()
        t, p = time.perf_counter(), time.process_time()
        pc, pv = svc.build_ptx_batch(wit, seed, c, v, workers_per_circuit=nw)
        host = (time.perf_counter() - t, time.process_time() - p)
        torch.cuda.synchronize()
        t, p = time.perf_counter(), time.process_time()
        dc, dv, sc, sv = svc.build_ptx_batch_dev(wit, seed, c, v, workers_per_circuit=nw)
        enq = time.perf_counter() - t
        torch.cuda.synchronize()
        dev = (time.perf_counter() - t, time.process_time() - p)
        if ref is None:
            ref = (pc, pv)
            assert [bytes(x) for x in dc.cpu().numpy()] == pc and [bytes(x) for x in dv.cpu().numpy()] == pv, "device proofs differ"
            assert not sc.any() and not sv.any(), "a status is not TB_PROVED"
            continue
        keep("host_s", host[0])
        keep("host_cpu_s", host[1])
        keep("dev_s", dev[0])
        keep("dev_cpu_s", dev[1])
        keep("dev_enqueue_s", enq)
    return best


def prove_then_verify(svc, wit, c, v, repeats):
    import torch
    from taiga_b200 import lib
    vk_c, vk_v = svc.verifying_keys()
    dev = c.device
    ci = torch.from_numpy(np.ascontiguousarray(wit["c_inst"], dtype=np.uint8).reshape(len(wit["c_inst"]), -1)).to(dev)
    vi = torch.from_numpy(np.ascontiguousarray(wit["v_inst"], dtype=np.uint8).reshape(len(wit["v_inst"]), -1)).to(dev)
    best, verdict = None, None
    for r in range(repeats + 1):
        torch.cuda.synchronize()
        t = time.perf_counter()
        dc, dv, sc, sv = svc.build_ptx_batch_dev(wit, bytes(range(32)), c, v, workers_per_circuit=1)
        bv = lib.BatchVerifier(svc.srs, bytes(range(7, 39)))
        bv.add(vk_c, ci, wit["c_len"], dc)
        bv.add(vk_v, vi, wit["v_len"], dv)
        ok = bv.finalize()
        s = time.perf_counter() - t
        bv.close()
        verdict = ok if verdict is None else verdict and ok
        if r:
            best = s if best is None else min(best, s)
    return best, verdict


def measure(svc, repeats):
    """(64-ptx comparison, 1-ptx comparison, prove-then-verify seconds, verdict).  The device tensors live in this function
    only: torch frees a tensor used on a worker's stream with an event on that stream, so they must go before the service's
    contexts do."""
    import torch
    base = svc.synthesize_ptx(2, wseed=5)
    dev = torch.device("cuda", 0)
    wit64, c64, v64 = step_inputs(base, 64, dev)
    b64 = compare(svc, wit64, c64, v64, 1, repeats)
    pv_s, verdict = prove_then_verify(svc, wit64, c64, v64, repeats)
    wit1, c1, v1 = step_inputs(base, 1, dev)
    b1 = compare(svc, wit1, c1, v1, 2, repeats)
    torch.cuda.synchronize()
    return b64, b1, pv_s, verdict


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    from taiga_b200 import ptx
    svc = ptx.ProverService(0, load_srs_arrays(), c_workers=2, v_workers=2)
    res = {"gpu": _query("name"), "power_limit": _query("power.limit"), "sm_clock": _query("clocks.sm"), "sm_clock_max": _query("clocks.max.sm")}
    b64, b1, pv_s, verdict = measure(svc, args.repeats)
    for name, b in (("ptx64", b64), ("ptx1", b1)):
        for k_, v_ in b.items():
            res["%s_%s" % (name, k_.replace("_s", "_ms"))] = round(v_ * 1e3, 2)
    res.update({"ptx64_prove_verify_ms": round(pv_s * 1e3, 2), "ptx64_prove_verify_verdict": bool(verdict), "sm_clock_after": _query("clocks.sm")})
    print("64-ptx step: threads + host proofs %.1f ms (CPU %.0f ms); one thread + device proofs %.1f ms (enqueue %.1f ms, CPU %.0f ms)"
          % (b64["host_s"] * 1e3, b64["host_cpu_s"] * 1e3, b64["dev_s"] * 1e3, b64["dev_enqueue_s"] * 1e3, b64["dev_cpu_s"] * 1e3))
    print("1-ptx step:  4 threads + host proofs %.2f ms (CPU %.1f ms); one thread + device proofs %.2f ms (enqueue %.2f ms, CPU %.1f ms)"
          % (b1["host_s"] * 1e3, b1["host_cpu_s"] * 1e3, b1["dev_s"] * 1e3, b1["dev_enqueue_s"] * 1e3, b1["dev_cpu_s"] * 1e3))
    print("64-ptx step proved on the device, then one device batch verification: %.1f ms, verdict %s" % (pv_s * 1e3, verdict))
    print("measured on: %s, power limit %s, SM clock %s (max %s)" % (res["gpu"], res["power_limit"], res["sm_clock"], res["sm_clock_max"]))
    print(json.dumps(res))


def _query(field):
    """one field of GPU 0 as nvidia-smi reports it (a read-only query)"""
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + field, "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "?"
    except Exception:
        return "?"


if __name__ == "__main__":
    main()
