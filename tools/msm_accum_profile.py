"""Per-kernel profile of the batch-affine accumulate path of the batched MSM (csrc/msm_batch.cu).

Times every kernel of `msm_accum` -- count, forward / inversion / backward of each round, finish -- with torch.profiler
(CUPTI device timestamps) over repeated commitments, for three chunk shapes the benchmark runs at k = 15:

  dense    K = 132 uniform scalars (h pieces, q', s)
  witness  K = 132 advice-like scalars (bench.witness_like)
  ipa      K = 128 IPA-round vectors: 64 proofs x (cL, cR), each half zero in blocks of m / 2 (ipa_round_scalars_kernel)

For each kernel it prints the pairs processed (counted on the host from the signed 13-bit digits, exactly as the sort kernel
forms the buckets), the Montgomery products, the bytes moved under the traffic model below, int_util (products x 247 SASS /
(time x SMs x 64 lanes x clock), as bench.py) and GB/s.  Run on the GPU:  python tools/msm_accum_profile.py

Traffic model (bytes per output item q of a round; "pair" = q has two inputs, "single" = it has one; a point is 64 B, a
coordinate 32 B; every item writes meta 4 B and a prefix product 32 B in fwd, and its result 64 B in bwd):
  fwd  round 0: entries 4 B per input, table x 2 x 32 B per pair, writes 8 B of table indices per item
       round r >= 1: x 2 x 32 B per pair
  bwd  round 0: meta 4 B + table indices 8 B per item, 2 x 64 B table points + prefix product 32 B per pair, 64 B per single
       round r >= 1: meta 4 B per item, 2 x 64 B points + prefix product 32 B per pair, 64 B per single
  both: 16 KB of round-0 counts per CTA (L2 resident) and the CTA's product tree (16 KB) are counted as well.
With 64-B point records (x and y together) and the classification repeated in bwd, round-0 fwd wrote no table indices and
round-0 bwd read 4 B of entries per input instead: within 8 B per item of the same totals.

The shapes are one chunk each only if K <= TB_MSM_BA_CHUNK (default: the GPU's SM count; 132 on an H100 SXM); on a GPU with
fewer SMs set TB_MSM_BA_CHUNK=132, or the pass count of the trace does not match and the tool stops.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N15 = 1 << 15
C, NB, W = 13, 1 << 12, 20
THREADS = 256
SASS_PER_MODMUL, INT_LANES_PER_SM = 247, 64


def witness_like(rng, n):
    """bench.witness_like: 30 % zero, 30 % one, 20 % < 2^8, 8 % < 2^32, 12 % uniform."""
    s = rng.integers(0, 256, size=(n, 32), dtype=np.uint8)
    s[:, 31] &= 0x3F
    u = rng.random(n)
    s[u < 0.3] = 0
    o = (u >= 0.3) & (u < 0.6)
    s[o] = 0
    s[o, 0] = 1
    s[(u >= 0.6) & (u < 0.8), 1:] = 0
    s[(u >= 0.8) & (u < 0.88), 4:] = 0
    return s


def shapes(rng, ipa_m):
    K = 132
    dense = rng.integers(0, 256, size=(K, N15, 32), dtype=np.uint8)
    dense[:, :, 31] &= 0x3F
    wit = np.stack([witness_like(rng, N15) for _ in range(K)])
    # one IPA round: cL[t] = p'[half + i] s[t] if i < half else 0, cR the other half (i = t mod m, half = m / 2)
    B = 64
    v = rng.integers(0, 256, size=(B, 2, N15, 32), dtype=np.uint8)
    v[..., 31] &= 0x3F
    low = (np.arange(N15) % ipa_m) < ipa_m // 2
    v[:, 0, ~low] = 0
    v[:, 1, low] = 0
    return [("dense", dense, True), ("witness", wit, True), ("ipa", v.reshape(2 * B, N15, 32), False)]


def bucket_counts(s):
    """[K, NB] entries per bucket: the signed c-bit digits of msm_sort_kernel (digit v > 2^(c-1) becomes 2^c - v, carry 1)."""
    K = s.shape[0]
    limbs = s.reshape(K * N15, 32).view("<u8").astype(np.uint64)   # 4 x 64-bit limbs, little endian
    carry = np.zeros(K * N15, np.uint64)
    counts = np.zeros(K * NB, np.int64)
    mask, half = np.uint64((1 << C) - 1), np.uint64(1 << (C - 1))
    kid = np.repeat(np.arange(K, dtype=np.int64) * NB, N15)
    for w in range(W):
        bit = w * C
        li, off = bit // 64, bit % 64
        v = limbs[:, li] >> np.uint64(off)
        if off > 64 - C and li + 1 < 4:
            v |= limbs[:, li + 1] << np.uint64(64 - off)
        v = (v & mask) + carry
        neg = v > half
        v = np.where(neg, np.uint64(1 << C) - v, v)
        carry = neg.astype(np.uint64)
        nz = v != 0
        counts += np.bincount(kid[nz] + (v[nz] - 1).astype(np.int64), minlength=K * NB)
    return counts.reshape(K, NB)


def model(counts, R, M):
    """per kernel: (name, pairs, items written, products, bytes)"""
    rows = []
    ctas = lambda n_out: np.ceil(n_out / (M * THREADS)).sum()   # CTAs that do work (the others leave at once)
    for r in range(R):
        a = (counts + (1 << r) - 1) >> r            # items per bucket entering round r
        n_out = ((a + 1) >> 1).sum(axis=1)           # items leaving, per MSM
        pairs = int((a >> 1).sum())
        items = int(n_out.sum())
        single = items - pairs
        nc = ctas(n_out)
        fixed = nc * (NB * 4 + 2 * THREADS * 32)     # counts + tree
        if r == 0:
            fb = pairs * (8 + 64) + single * 4 + items * (36 + 8) + fixed
            bb = items * (4 + 8) + pairs * (128 + 32) + single * 64 + items * 64 + fixed
        else:
            fb = pairs * 64 + items * 36 + fixed
            bb = items * 4 + pairs * (128 + 32) + single * 64 + items * 64 + fixed
        rows.append(("fwd r%d" % r, pairs, items, pairs + 255 * nc, fb))
        rows.append(("inv r%d" % r, 0, 0, 0, nc * 64))
        rows.append(("bwd r%d" % r, pairs, items, 5 * pairs + 510 * nc, bb))
    a = (counts + (1 << R) - 1) >> R
    left = int(a.sum())
    rows.append(("finish", 0, left, 10 * (left - int((a > 0).sum())), left * 64 + counts.size * 128))
    return rows


def kernel_times(ctx, srs, s, lagrange, reps):
    """{(kind, round): mean ms} over `reps` commitments, kernels in launch order of each call"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    bl = np.zeros((s.shape[0], 32), np.uint8)
    srs.commit(s, bl, lagrange=lagrange, batch=s.shape[0])   # warm: module load, pool
    ctx.sync()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            srs.commit(s, bl, lagrange=lagrange, batch=s.shape[0])
        ctx.sync()
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))["traceEvents"]
    ks = sorted((e for e in ev if e.get("cat") == "kernel" and "msm_ba_" in e.get("name", "")), key=lambda e: e["ts"])
    acc, rnd = {}, {}
    calls = 0
    for e in ks:
        n = e["name"]
        if "msm_ba_count_kernel" in n:
            key = ("count", 0); calls += 1; rnd = {"fwd": -1, "inv": -1, "bwd": -1}
        elif "msm_ba_finish_kernel" in n:
            key = ("finish", 0)
        else:
            kind = "fwd" if "msm_ba_fwd_kernel" in n else "inv" if "msm_ba_inv_kernel" in n else "bwd"
            rnd[kind] += 1
            key = (kind, rnd[kind])
        acc[key] = acc.get(key, 0.0) + e["dur"] * 1e-3
    if calls != reps:
        raise RuntimeError("expected %d accumulate passes in the trace, found %d (is the batched path on, K <= TB_MSM_BA_CHUNK?)" % (reps, calls))
    return {k: v / reps for k, v in acc.items()}


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        f = [x.strip() for x in out.strip().split(",")]
        return {"name": f[0], "power_limit_w": float(f[1]), "sm_max_mhz": float(f[2]), "sm_mhz_now": float(f[3])}
    except Exception as ex:   # nvidia-smi missing: the numbers still stand, without their hardware label
        return {"name": "unknown (%r)" % (ex,), "power_limit_w": None, "sm_max_mhz": None}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--ipa-m", type=int, default=1 << 8, help="IPA round block length m (n >> j)")
    ap.add_argument("--json", metavar="FILE", help="also write the table as JSON")
    args = ap.parse_args()
    import torch
    from taiga_b200 import lib
    os.environ["TB_MSM_BA_MIN_TERMS"] = "0"
    R = int(os.environ.get("TB_MSM_BA_ROUNDS", 10))
    M = 32   # pairs per thread (msm_batch.cu BA_M)
    raw = np.fromfile(os.path.join(ROOT, "tests", "golden", "srs_k15_affine.bin"), dtype=np.uint8).reshape(-1, 64)
    ctx = lib.Context(0)
    srs = ctx.load_srs(15, raw[:N15], raw[N15:2 * N15], raw[2 * N15], raw[2 * N15 + 1])
    info = gpu_info()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    clk = (info.get("sm_max_mhz") or 1980) * 1e6
    int_peak = sms * INT_LANES_PER_SM * clk
    print("GPU %s, power limit %s W, %d SMs, int_util at the max SM clock %.0f MHz; M=%d pairs per thread, R=%d" % (
        info["name"], info.get("power_limit_w"), sms, clk / 1e6, M, R), flush=True)
    rng = np.random.default_rng(7)
    report = {"gpu": info, "sms": sms, "shapes": {}}
    for name, s, lagrange in shapes(rng, args.ipa_m):
        counts = bucket_counts(s)
        t = kernel_times(ctx, srs, s, lagrange, args.reps)
        rows = model(counts, R, M)
        print("\n== %s: K = %d, %d bucket entries, %.1f additions per entry" % (name, s.shape[0], int(counts.sum()), sum(r[1] for r in rows if r[0].startswith("bwd")) / max(1, counts.sum())))
        print("%-10s %9s %12s %12s %10s %9s %8s %8s" % ("kernel", "ms", "pairs", "products", "MB", "GB/s", "int_util", "share"))
        total = sum(t.values())
        out = []
        def line(label, ms, pairs, prods, byts):
            gbs = byts / (ms * 1e-3) / 1e9 if ms > 0 else 0.0
            iu = prods * SASS_PER_MODMUL / (ms * 1e-3) / int_peak if ms > 0 else 0.0
            print("%-10s %9.3f %12d %12d %10.1f %9.0f %8.3f %7.1f%%" % (label, ms, pairs, prods, byts / 1e6, gbs, iu, 100 * ms / total))
            out.append({"kernel": label, "ms": ms, "pairs": pairs, "products": prods, "bytes": byts, "gbs": gbs, "int_util": iu})
        line("count", t.get(("count", 0), 0.0), 0, 0, counts.size * 4 * (R + 1))
        sums = {"fwd": [0.0, 0, 0, 0], "inv": [0.0, 0, 0, 0], "bwd": [0.0, 0, 0, 0]}
        for label, pairs, items, prods, byts in rows:
            kind, _, rr = label.partition(" ")
            ms = t.get(("finish", 0), 0.0) if kind == "finish" else t.get((kind, int(rr[1:])), 0.0)
            line(label, ms, pairs, int(prods), byts)
            if kind in sums:
                for i, v in enumerate((ms, pairs, int(prods), byts)):
                    sums[kind][i] += v
        for kind, (ms, pairs, prods, byts) in sums.items():
            line("all " + kind, ms, pairs, prods, byts)
        print("%-10s %9.3f" % ("total", total))
        report["shapes"][name] = out
    if args.json:
        with open(args.json, "w") as f:
            json.dump(report, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
