"""Every kernel of libtaiga_b200 is launched through one helper, `launch_cluster` in common.cuh (`launch` forwards to it),
which checks the launch and counts it in `Ctx::launches`, the number tb_ctx_launch_count reports.

The CPU tests check the sources: no other launch site and no other code that changes the count.  The GPU tests pin the
exact count of call sequences whose launches follow from the host code."""
import os
import re

import numpy as np
import pytest

from oracle import pasta as o
from taiga_b200 import lib

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "taiga_b200", "csrc")


def sources():
    """{file name: text} of every CUDA source and header of the library."""
    out = {}
    for name in sorted(os.listdir(CSRC)):
        if name.endswith((".cu", ".cuh")):
            with open(os.path.join(CSRC, name)) as f:
                out[name] = f.read()
    return out


def helper_span(text):
    """(start, end) of the body of launch_cluster in common.cuh."""
    start = text.index("{", text.index("void launch_cluster("))
    depth = 0
    for i in range(start, len(text)):
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        if depth == 0:
            return start, i + 1
    raise AssertionError("unbalanced launch_cluster body")


def sites(pattern):
    """[(file, offset)] of every match of `pattern` in the library's sources."""
    return [(name, m.start()) for name, text in sources().items() for m in re.finditer(pattern, text)]


def in_helper(found):
    lo, hi = helper_span(sources()["common.cuh"])
    return len(found) == 1 and found[0][0] == "common.cuh" and lo <= found[0][1] < hi


def test_no_triple_chevron_launch():
    assert sites(r"<<<") == []


def test_launch_kernel_ex_only_in_helper():
    found = sites(r"\bcudaLaunchKernelEx\b")
    assert in_helper(found), found


def test_launch_count_changed_only_in_helper():
    # an assignment or increment of `launches`, other than the member's initialiser in Ctx
    found = sites(r"(?<!uint64_t )\blaunches\s*(\+\+|--|[-+*/]?=(?!=))|(\+\+|--)\s*[\w.>-]*\blaunches\b")
    assert in_helper(found), found


# ---------------------------------------------------------------- GPU: exact counts
def launches(ctx, fn):
    before = ctx.launch_count
    fn()
    return ctx.launch_count - before


def field_elements(n, seed):
    """n random canonical field elements (below 2^254, so below both Pasta moduli), 32 bytes little endian each."""
    x = np.random.default_rng(seed).integers(0, 256, size=(n, 32), dtype=np.uint8)
    x[:, 31] &= 0x3F
    return x


def scan_launches(n):
    """poly.cu exclusive_scan_u32: one block pass, then a scan of the block sums and an add pass while they exceed a block."""
    nblocks = (n + 2047) // 2048
    return 1 if nblocks == 1 else 2 + scan_launches(nblocks)


@pytest.mark.gpu
@pytest.mark.parametrize("logn,passes", [(8, 1), (12, 2), (19, 3)])
def test_ntt_launch_count(gpu_ctx, logn, passes):
    """Context.ntt: to Montgomery form, one launch per NTT pass, back from Montgomery form."""
    x = field_elements(1 << logn, logn)
    assert launches(gpu_ctx, lambda: gpu_ctx.ntt(lib.TB_FP, x)) == 1 + passes + 1


@pytest.mark.gpu
@pytest.mark.parametrize("n,heavy", [(64, 0), (1 << 14, 1)])
def test_msm_latency_path_launch_count(gpu_ctx, n, heavy):
    """Context.msm (variable base, so always the latency path of msm.cu) with the default window c:
    2 conversions of the inputs, digits count, scan, digits scatter, units, scan, accumulate, combine_sub, combine,
    combine_heavy (when a bucket may hold more than MSM_HEAVY_UNITS units), segsum, window, horner, to affine, 1 conversion
    of the output.  n = 64: c = 4, 64 windows x 8 buckets; n = 2^14: c = 10, 26 windows x 512 buckets, up to 53 248 units."""
    c = max(4, n.bit_length() - 1 - 4)
    nb_total = ((256 + c - 1) // c) << (c - 1)
    G = o.VESTA_GEN
    pts = np.tile(np.frombuffer(G[0].to_bytes(32, "little") + G[1].to_bytes(32, "little"), np.uint8), (n, 1))
    s = field_elements(n, n)
    want = 2 + 1 + scan_launches(nb_total) + 1 + 1 + scan_launches(nb_total) + 3 + heavy + 3 + 1 + 1
    assert launches(gpu_ctx, lambda: gpu_ctx.msm(lib.TB_VESTA, s, pts)) == want


@pytest.mark.gpu
def test_batched_commit_launch_count(gpu_srs, monkeypatch):
    """Srs.commit of K = 7 vectors on the batched path of msm_batch.cu, one round, chunks of 3 MSMs (3, 3 and 1):
    3 conversions (scalars, blinds, result) + chunks x (sort + count + 3 x rounds + finish) + linesum + weighted."""
    monkeypatch.setenv("TB_MSM_BA_MIN_TERMS", "0")
    monkeypatch.setenv("TB_MSM_BA_ROUNDS", "1")
    monkeypatch.setenv("TB_MSM_BA_CHUNK", "3")
    K, n = 7, gpu_srs.n
    s = field_elements(K * n, 7)
    blinds = field_elements(K, 8)
    chunks, rounds = 3, 1
    want = 3 + chunks * (1 + 1 + 3 * rounds + 1) + 2
    assert launches(gpu_srs.ctx, lambda: gpu_srs.commit(s, blinds, lagrange=True, batch=K)) == want
