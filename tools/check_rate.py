"""Witness-check rate of one 64-ptx step: the 128 Compliance and 256 VP witnesses of 64 partial transactions checked with
tb_check_batch (MockProver::run(15, ..).verify() on the device), one call per circuit.

Prints, fastest of --repeats steps: wall time and witnesses/s, the per-category device time of one step (prof_read), the card,
its power limit and SM clock read in the same run, and the host comparison: circuits_random.satisfied (the pure-Python
restatement of MockProver, one host core) timed on one witness per circuit (--no-host skips it; about 15 s per witness).
The Rust MockProver is not available here, so its time is "not measured".  Prints one JSON line at the end.

  python tools/check_rate.py [--repeats 5] [--no-host]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_PTX = 64
COMPLIANCE_PER_PTX, VP_PER_PTX = 2, 4
WITNESSES = 4     # distinct witnesses per circuit, tiled


def load_srs(ctx):
    raw = np.fromfile(os.path.join(ROOT, "tests", "golden", "srs_k15_affine.bin"), dtype=np.uint8).reshape(-1, 64)
    n = 1 << 15
    return ctx.load_srs(15, raw[:n], raw[n:2 * n], raw[2 * n], raw[2 * n + 1])


def card():
    """(name, power limit, SM clock) as nvidia-smi reports them now (read only)."""
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [x.strip() for x in q.split(",")]
        return {"gpu": name, "power_limit": power, "sm_clock": sm, "sm_clock_max": sm_max}
    except Exception as ex:
        return {"gpu": "?", "error": str(ex)}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--no-host", action="store_true", help="skip timing circuits_random.satisfied")
    args = ap.parse_args()
    from taiga_b200 import circuits_random as cr
    from taiga_b200 import circuits_taiga as ct
    from taiga_b200 import lib
    ctx = lib.Context(0)
    srs = load_srs(ctx)
    seed = bytes(range(32))
    circuits = []
    for compliance, count in ((True, COMPLIANCE_PER_PTX * N_PTX), (False, VP_PER_PTX * N_PTX)):
        kd, make = ct.build(compliance)
        pk = srs.load_circuit(kd)
        asgs = [make(7 + w) for w in range(WITNESSES)]
        wit = [kd.witness_arrays(a) for a in asgs]
        adv = np.stack([wit[i % WITNESSES][0] for i in range(count)])
        inst = np.stack([wit[i % WITNESSES][1] for i in range(count)])
        circuits.append((kd, pk, adv, inst, wit[0][2], asgs[0]))

    def step():
        return [pk.check_batch(adv, inst, lens, seed) for _, pk, adv, inst, lens, _ in circuits]
    for res in step():   # first call: builds each key's check tables
        assert all(cnt == (0, 0, 0) for cnt, _ in res), "an honest witness failed the check"
    best = None
    for _ in range(args.repeats):
        t = time.perf_counter()
        step()
        dt = time.perf_counter() - t
        best = dt if best is None else min(best, dt)
    ctx.prof_enable(True)
    step()
    prof = ctx.prof_read()
    ctx.prof_enable(False)
    n = sum(len(c[3]) for c in circuits)
    out = {"witnesses": n, "seconds": round(best, 4), "witnesses_per_s": round(n / best, 1),
           "device_ms": {k: round(v[0], 3) for k, v in prof.items() if v[1]}}
    out.update(card())
    print("tb_check_batch: %d witnesses (128 Compliance + 256 VP, k = 15) in %.1f ms: %.0f witnesses/s" % (n, best * 1e3, n / best))
    print("device time of one step by category (ms):", out["device_ms"])
    print("card: %s, power limit %s, SM clock %s (max %s)" % (out.get("gpu"), out.get("power_limit"), out.get("sm_clock"), out.get("sm_clock_max")))
    if not args.no_host:
        host = {}
        for kd, _, _, _, _, asg in circuits:
            t = time.perf_counter()
            assert cr.satisfied(kd, asg) is None
            host[kd.name] = round(time.perf_counter() - t, 2)
        out["python_satisfied_seconds_per_witness"] = host
        print("circuits_random.satisfied (the Python restatement of MockProver, one host core), seconds per witness:", host)
    out["rust_mockprover"] = "not measured"
    print("Rust MockProver: not measured")
    print(json.dumps(out))


if __name__ == "__main__":
    main()
