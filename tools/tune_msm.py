"""Timing of the batched commitment path for several knob settings (K = 704 dense MSMs of 2^15 terms)."""
import os, sys, json
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from taiga_b200 import lib
N15 = 1 << 15
raw = np.fromfile(os.path.join(ROOT, "tests", "golden", "srs_k15_affine.bin"), dtype=np.uint8).reshape(-1, 64)
ctx = lib.Context(0)
srs = ctx.load_srs(15, raw[:N15], raw[N15:2 * N15], raw[2 * N15], raw[2 * N15 + 1])
rng = np.random.default_rng(1)
K = 704
s = rng.integers(0, 256, size=(K, N15, 32), dtype=np.uint8); s[:, :, 31] &= 0x3F
bl = np.zeros((K, 32), np.uint8)
os.environ["TB_MSM_BA_MIN_TERMS"] = "0"
ref = None
CONFIGS = None
for cfg in CONFIGS or [{}, {"TB_MSM_BA_ROUNDS": "8"}, {"TB_MSM_BA_ROUNDS": "9"}, {"TB_MSM_BA_CHUNK": "704"}, {}]:
    os.environ.update(cfg)
    out = srs.commit(s, bl, lagrange=True, batch=K)
    ctx.prof_enable(True)
    out = srs.commit(s, bl, lagrange=True, batch=K)
    p = ctx.prof_read(); ctx.prof_enable(False)
    if ref is None: ref = out.tobytes()
    print("%-50s sort %.2f accum %.2f reduce %.2f same=%s" % (json.dumps(cfg), p["msm_sort"][0], p["msm_accum"][0], p["msm_reduce"][0], out.tobytes() == ref), flush=True)
    for k in cfg: os.environ.pop(k)
