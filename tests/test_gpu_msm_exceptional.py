"""MSM on exceptional inputs -- doublings, cancellations, identities and digits on the signed-recoding boundary -- on
every path of `msm_run`, against a discrete-log reference that shares no code with the CUDA kernels or the C++ oracle.

Every base has a known discrete log, B_i = [a_i]G, so MSM(s, B) + blind * w = [(sum_i s_i a_i + blind a_w) mod r]G with r
the group order (p for Vesta, q for Pallas): one exact integer sum and one scalar multiple, milliseconds even at n = 2^17.
Random SRS points never coincide or cancel inside a bucket; these base families do on purpose:

  ones             a_i = 1: with equal scalars every pair of every batch-affine round is a doubling
  plus_minus       a_i = +1, -1, +1, ...: pairs cancel, and the rounds after the first see identity items
  small            a_i = (i mod 7) - 3: identities, duplicates and negations mixed
  cross_window     a_i from {1, 2^c, 2^2c, -2^c}: the fixed-base table entry 2^(cw) B_i of one window equals another base in
                   a lower window, so the shared buckets of a fixed-base MSM hold equal and opposite points
  mostly_identity  ~90 % of the bases are (0, 0), the rest from a small set with negations

and the scalar families (the K vectors of one batched call) put every c-bit digit on the boundary of the signed recoding
(2^(c-1), and 2^(c-1) + 1 with a carry through every window), use p - 1 and p - 2, cancel in pairs, or are all equal.

The GPU tests run Srs.commit at k = 6, 8, 11, 15, 17 on the latency path and on the batch-affine path of msm_batch.cu under
its round / chunk settings, and Context.msm on both curves for n = 1 ... 2^16 and window_bits 0, 2 ... 20.  Each asserts
through the library's kernel-group profiler that its MSMs ran the path it is meant to test.
"""
import random

import numpy as np
import pytest

from oracle import pasta as o
from taiga_b200 import lib

CURVES = {lib.TB_VESTA: (o.VESTA, o.VESTA_GEN), lib.TB_PALLAS: (o.PALLAS, o.PALLAS_GEN)}
BASE_FAMILIES = ("ones", "plus_minus", "small", "cross_window", "mostly_identity")
SCALAR_FAMILIES = ("ones", "same", "pairs", "digits_half", "digits_half_plus1", "minus1", "minus1_minus2", "one_term", "uniform",
                   "witness", "zeros")
KNOBS = ("TB_MSM_BA_MIN_TERMS", "TB_MSM_BA_ROUNDS", "TB_MSM_BA_CHUNK")


# ---------------------------------------------------------------- reference
def _add(m, a, b):
    """Affine addition on y^2 = x^3 + 5 over F_m (None = identity), as pasta.Curve.add with a faster inverse."""
    if a is None:
        return b
    if b is None:
        return a
    (x1, y1), (x2, y2) = a, b
    if x1 == x2:
        if (y1 + y2) % m == 0:
            return None
        lam = 3 * x1 * x1 * pow(2 * y1, -1, m) % m
    else:
        lam = (y2 - y1) * pow(x2 - x1, -1, m) % m
    x3 = (lam * lam - x1 - x2) % m
    return x3, (lam * (x1 - x3) - y1) % m


def mul_g(curve, e):
    """[e]G on `curve` (TB_VESTA / TB_PALLAS) for any integer e, reduced mod the group order."""
    cv, pt = CURVES[curve]
    e %= cv.fs
    acc = None
    while e:
        if e & 1:
            acc = _add(cv.fb, acc, pt)
        pt = _add(cv.fb, pt, pt)
        e >>= 1
    return acc


def point_bytes(pt):
    """64-byte affine encoding of the ABI: x || y little endian, the identity as 64 zero bytes."""
    return bytes(64) if pt is None else pt[0].to_bytes(32, "little") + pt[1].to_bytes(32, "little")


def scalar_bytes(xs):
    return np.frombuffer(b"".join(x.to_bytes(32, "little") for x in xs), np.uint8).reshape(-1, 32)


def base_points(curve, logs):
    """[a_i]G for every log: each distinct multiple is computed once and tiled."""
    distinct = sorted(set(logs))
    table = np.frombuffer(b"".join(point_bytes(mul_g(curve, a)) for a in distinct), np.uint8).reshape(-1, 64)
    pos = {a: i for i, a in enumerate(distinct)}
    return table[np.fromiter((pos[a] for a in logs), np.int64, len(logs))]


def reference(curve, scalars, logs, extra=0):
    """Encoded [(sum_i s_i a_i + extra) mod r]G: the MSM over bases with discrete logs `logs`, plus `extra` in the exponent."""
    return point_bytes(mul_g(curve, sum(s * a for s, a in zip(scalars, logs)) + extra))


def base_logs(family, n, c, seed):
    """Discrete logs a_i of the bases of `family` (c: the window the cross-window family is aimed at)."""
    rnd = random.Random(seed)
    if family == "ones":
        return [1] * n
    if family == "plus_minus":
        return [1 - 2 * (i & 1) for i in range(n)]
    if family == "small":
        return [i % 7 - 3 for i in range(n)]
    if family == "cross_window":
        pal = [1, 1 << c, 1 << (2 * c), -(1 << c)]
        return [rnd.choice(pal) for _ in range(n)]
    if family == "mostly_identity":
        big = rnd.getrandbits(250)
        pal = [1, -1, 2, big, -big, big + 1]
        return [0 if rnd.random() < 0.9 else rnd.choice(pal) for _ in range(n)]
    raise ValueError(family)


# log of the blinding base w per base family: w = G collides with the `ones` bases, w = -G cancels against `plus_minus`
W_LOG = {"ones": 1, "plus_minus": -1, "small": 1, "cross_window": 1, "mostly_identity": 0}


def digit_scalar(c, d):
    """The scalar whose c-bit windows below bit 254 all hold d (so it is < 2^254 < p, q)."""
    s, w = 0, 0
    while c * (w + 1) <= 254:
        s |= d << (c * w)
        w += 1
    return s


def signed_digits(s, c):
    """The signed c-bit recoding of the MSM kernels: a digit above 2^(c-1) becomes digit - 2^c with a carry of 1."""
    out, carry = [], 0
    for w in range((256 + c - 1) // c):
        v = ((s >> (c * w)) & ((1 << c) - 1)) + carry
        carry = int(v > 1 << (c - 1))
        out.append(v - (carry << c))
    return out


def scalar_vectors(n, m, c, seed):
    """{family: n scalars mod m}; c is the window of the MSM the digit families are aimed at."""
    rnd = random.Random(seed)
    half = 1 << (c - 1)
    pair = [rnd.randrange(1, m) for _ in range((n + 1) // 2)]
    one = [0] * n
    one[rnd.randrange(n)] = rnd.randrange(1, m)

    def witness():   # SURVEY 8d: 30 % zero, 30 % one, 20 % < 2^8, 8 % < 2^32, 12 % uniform
        u = rnd.random()
        return 0 if u < .3 else 1 if u < .6 else rnd.randrange(256) if u < .8 else rnd.randrange(1 << 32) if u < .88 else rnd.randrange(m)

    vec = {
        "ones": [1] * n,
        "same": [rnd.randrange(1, m)] * n,
        "pairs": [pair[i >> 1] if i % 2 == 0 else m - pair[i >> 1] for i in range(n)],   # s, p - s: cancels on equal bases
        "digits_half": [digit_scalar(c, half)] * n,
        "digits_half_plus1": [digit_scalar(c, half + 1)] * n,
        "minus1": [m - 1] * n,
        "minus1_minus2": [m - 1 - (i & 1) for i in range(n)],
        "one_term": one,
        "uniform": [rnd.randrange(m) for _ in range(n)],
        "witness": [witness() for _ in range(n)],
        "zeros": [0] * n,
    }
    assert tuple(vec) == SCALAR_FAMILIES
    return vec


def blinds_for(m, seed):
    """The blind of every scalar family: zero where the commitment should be the identity (pairs over `ones`, zeros)."""
    rnd = random.Random(seed)
    b = {"ones": 1, "same": rnd.randrange(m), "pairs": 0, "digits_half": m - 1, "digits_half_plus1": rnd.randrange(m), "minus1": m - 1,
         "minus1_minus2": 1, "one_term": 0, "uniform": rnd.randrange(m), "witness": 0, "zeros": 0}
    return [b[f] for f in SCALAR_FAMILIES]


def default_window(n):
    """msm.cu msm_default_window: the variable-base window for window_bits = 0."""
    return min(16, max(4, n.bit_length() - 1 - 4))


def srs_window(k):
    """srs.cuh: the fixed-base window of an SRS of 2^k points."""
    return min(13, max(4, k - 2))


# ---------------------------------------------------------------- the reference against both oracles (CPU)
@pytest.mark.parametrize("curve", [lib.TB_VESTA, lib.TB_PALLAS])
@pytest.mark.parametrize("family", BASE_FAMILIES)
def test_reference_matches_oracles(oracle_cpu, curve, family):
    """The discrete-log reference equals oracle_cpu.msm for every base and scalar family, blinding term and identities
    included, and pasta.Curve.msm on a few terms of each scalar family (spread over the base families: it is slow)."""
    cv, G = CURVES[curve]
    m = cv.fs
    for n, c in ((64, 6), (5, 4)):
        logs = base_logs(family, n, c, seed=n) + [W_LOG[family]]   # the last term is blind * w
        pts = base_points(curve, logs)
        blinds = blinds_for(m, seed=n)
        for fi, (name, s) in enumerate(scalar_vectors(n, m, c, seed=n).items()):
            s = s + [blinds[fi]]
            want = reference(curve, s, logs)
            assert oracle_cpu.msm(curve, scalar_bytes(s), pts).tobytes() == want, (name, n)
            if n == 5 and fi % len(BASE_FAMILIES) == BASE_FAMILIES.index(family):   # pasta's own points and MSM
                assert point_bytes(cv.msm(s, [cv.mul(a, G) for a in logs])) == want, (name, n)
    assert reference(curve, [1, m - 1], [1, 1]) == bytes(64)
    assert point_bytes(mul_g(curve, -1)) == point_bytes(cv.neg(G))


@pytest.mark.parametrize("c", [2, 3, 4, 6, 9, 13, 16, 17, 20])
def test_digit_families_sit_on_the_recoding_boundary(c):
    """digits_half gives the digit 2^(c-1) (not negated) in every window below bit 254; digits_half_plus1 gives a negated digit
    and a carry in every such window, the carry landing in the window above."""
    half, top = 1 << (c - 1), 254 // c   # windows 0 .. top - 1 are set
    for d, want in ((half, [half] * top), (half + 1, [-(half - 1)] + [-(half - 2)] * (top - 1) + [1])):
        s = digit_scalar(c, d)
        dig = signed_digits(s, c)
        assert sum(v << (c * w) for w, v in enumerate(dig)) == s < 1 << 254
        assert dig[:len(want)] == want and not any(dig[len(want):]), (c, d)


# ---------------------------------------------------------------- GPU: which path ran
# The library's CUDA-event profiler records one kernel group per phase of an MSM: the latency path (msm.cu) records sort,
# accumulate (msm_accum_kernel) and two reduce groups (bucket combine, weighted sum) per MSM call; the batched path
# (msm_batch.cu) records sort and accumulate (the msm_ba_* rounds) once per chunk and one reduce group per call.
def msm_groups(ctx, fn):
    """(fn(), {category: kernel groups}) over the MSM categories of the context's profiler."""
    ctx.prof_enable(True)
    try:
        out = fn()
        groups = {k: v[1] for k, v in ctx.prof_read().items() if k.startswith("msm_")}
    finally:
        ctx.prof_enable(False)
    return out, groups


def assert_latency_path(groups, calls):
    assert groups == {"msm_sort": calls, "msm_accum": calls, "msm_reduce": 2 * calls}, "expected the latency path: %s" % groups


def assert_batched_path(groups, calls, chunks):
    assert groups == {"msm_sort": calls * chunks, "msm_accum": calls * chunks, "msm_reduce": calls}, "expected the batched path: %s" % groups


def assert_results(got, want, names, what):
    bad = [names[j] for j in range(len(want)) if got[j].tobytes() != want[j]]
    assert not bad, "%s: wrong MSM for the scalar families %s" % (what, bad)


# ---------------------------------------------------------------- GPU: fixed base (Srs.commit)
FIXED_PATHS = {
    "latency": {"TB_MSM_BA_MIN_TERMS": str(1 << 30)},
    "batched": {"TB_MSM_BA_MIN_TERMS": "0"},                              # default rounds (10)
    "rounds1": {"TB_MSM_BA_MIN_TERMS": "0", "TB_MSM_BA_ROUNDS": "1"},     # the finish kernel folds what one round leaves
    "rounds3": {"TB_MSM_BA_MIN_TERMS": "0", "TB_MSM_BA_ROUNDS": "3"},
    "chunk3": {"TB_MSM_BA_MIN_TERMS": "0", "TB_MSM_BA_CHUNK": "3"},       # with K = 7: chunks of 3, 3 and 1 MSMs
}
# c = 4 at k = 6 has no batched path (it needs c >= 6); k = 8 is its smallest window and the generic sort kernel, k = 15 the c = 13
# sort kernel, k = 17 several TMA tiles and many CTAs per round.  Consecutive cases share their SRS.
FIXED_CASES = [(k, fam, path) for k in (6, 8, 11, 15, 17) for fam in BASE_FAMILIES for path in (("latency",) if k == 6 else FIXED_PATHS)]


class FixedBase:
    """The SRS of one (k, base family) at a time -- g with logs a_i, g_lagrange with the logs rotated by one, w = [W_LOG]G --
    with the scalar vectors of k (converted once) and the expected commitments."""

    def __init__(self, ctx):
        self.ctx, self.key, self.srs, self.kvec = ctx, None, None, None

    def get(self, k, family):
        if self.key == (k, family):
            return self
        self.close()
        n, c, m = 1 << k, srs_window(k), o.P
        if self.kvec != k:
            vec = scalar_vectors(n, m, c, seed=1000 + k)
            self.names, self.ints = list(vec), list(vec.values())
            self.scalars = np.stack([scalar_bytes(v) for v in self.ints])
            self.blind_ints = blinds_for(m, seed=k)
            self.blinds = scalar_bytes(self.blind_ints)
            self.kvec = k
        logs = base_logs(family, n, c, seed=k)
        logs_l = logs[1:] + logs[:1]
        wl = W_LOG[family]
        self.srs = self.ctx.load_srs(k, base_points(lib.TB_VESTA, logs), base_points(lib.TB_VESTA, logs_l), base_points(lib.TB_VESTA, [wl]),
                                     base_points(lib.TB_VESTA, [5]))
        self.want_l = [reference(lib.TB_VESTA, s, logs_l, b * wl) for s, b in zip(self.ints, self.blind_ints)]
        self.want_g = [reference(lib.TB_VESTA, s, logs) for s in self.ints]
        self.key = (k, family)
        return self

    def close(self):
        if self.srs is not None:
            self.srs.close()
        self.srs, self.key = None, None


@pytest.fixture(scope="module")
def fixed_base(gpu_ctx):
    fb = FixedBase(gpu_ctx)
    yield fb
    fb.close()


@pytest.mark.gpu
@pytest.mark.parametrize("k,family,path", FIXED_CASES)
def test_srs_commit_exceptional(gpu_ctx, fixed_base, k, family, path, monkeypatch):
    """Srs.commit of every scalar family, lagrange with blinds and plain with blinds=None, equals the discrete-log reference."""
    fb = fixed_base.get(k, family)
    for var in KNOBS:
        monkeypatch.delenv(var, raising=False)
    for var, v in FIXED_PATHS[path].items():
        monkeypatch.setenv(var, v)
    sel = list(range(7 if path == "chunk3" else len(fb.names)))
    if path == "rounds1" and k >= 15:
        # one round leaves half of every bucket to one finish-kernel thread: the digit families put all n * W digits in one or
        # two buckets (~10^6 serial additions at k = 17), so at this size they run on the other paths only
        sel = [j for j in sel if not fb.names[j].startswith("digits")]
    names, K = [fb.names[j] for j in sel], len(sel)
    s = np.ascontiguousarray(fb.scalars[sel])

    def run():
        return (fb.srs.commit(s, fb.blinds[sel], lagrange=True, batch=K), fb.srs.commit(s, None, lagrange=False, batch=K))

    (got_l, got_g), groups = msm_groups(gpu_ctx, run)
    assert_results(got_l, [fb.want_l[j] for j in sel], names, "commit_lagrange with blinds")
    assert_results(got_g, [fb.want_g[j] for j in sel], names, "commit without blinds")
    if path == "latency":
        assert_latency_path(groups, 2)
    else:
        assert_batched_path(groups, 2, -(-K // int(FIXED_PATHS[path].get("TB_MSM_BA_CHUNK", K))))


@pytest.mark.gpu
def test_batched_window_grows_on_one_context(monkeypatch):
    """The sort kernel of the batched path needs more shared memory at a wider window.  A context that committed at c = 6 commits
    at c = 13, and still does after a second context of the device committed at c = 6."""
    monkeypatch.setenv("TB_MSM_BA_MIN_TERMS", "0")
    for var in ("TB_MSM_BA_ROUNDS", "TB_MSM_BA_CHUNK"):
        monkeypatch.delenv(var, raising=False)
    case = {}
    for k in (8, 15):
        logs = base_logs("small", 1 << k, srs_window(k), seed=k)
        vec = scalar_vectors(1 << k, o.P, srs_window(k), seed=k)
        vec = {f: vec[f] for f in ("uniform", "pairs")}
        case[k] = (base_points(lib.TB_VESTA, logs), np.stack([scalar_bytes(v) for v in vec.values()]), list(vec),
                   [reference(lib.TB_VESTA, v, logs) for v in vec.values()])
    w = base_points(lib.TB_VESTA, [1])[0]
    a, b = lib.Context(0), lib.Context(0)
    try:
        for ctx, k in ((a, 8), (a, 15), (b, 8), (a, 15)):
            pts, s, names, want = case[k]
            srs = ctx.load_srs(k, pts, pts, w, w)
            assert_results(srs.commit(s, None, batch=len(names)), want, names, "k = %d after smaller windows" % k)
            srs.close()
    finally:
        a.close()
        b.close()


# ---------------------------------------------------------------- GPU: variable base (Context.msm)
# (n, window_bits, base family); window_bits 0 is the default window of n.  Every window meets `small` or `mostly_identity`.
VAR_CASES = [(1, 0, "ones"), (1, 2, "small"), (2, 20, "plus_minus"), (2, 17, "ones"),
             (9, 0, "small"), (9, 3, "mostly_identity"), (9, 20, "small"),
             (1000, 0, "cross_window"), (1000, 2, "small"), (1000, 5, "plus_minus"), (1000, 8, "mostly_identity"), (1000, 13, "small"),
             (1000, 16, "small"), (1000, 17, "mostly_identity"),
             (1 << 16, 0, "small"), (1 << 16, 3, "ones"), (1 << 16, 5, "mostly_identity"), (1 << 16, 8, "small"), (1 << 16, 13, "cross_window"),
             (1 << 16, 16, "plus_minus")]
WIDE_WINDOW_FAMILIES = ("ones", "pairs", "digits_half_plus1")   # at c = 20 the buckets take 0.9 GB per MSM


def var_case(curve, n, window, family):
    cv, _ = CURVES[curve]
    c = window or default_window(n)
    seed = n * 64 + window + 17 * curve
    logs = base_logs(family, n, c, seed)
    vec = scalar_vectors(n, cv.fs, c, seed)
    if c == 20:
        vec = {f: vec[f] for f in WIDE_WINDOW_FAMILIES}
    s = np.stack([scalar_bytes(v) for v in vec.values()])
    return base_points(curve, logs), s, list(vec), [reference(curve, v, logs) for v in vec.values()]


@pytest.mark.gpu
@pytest.mark.parametrize("curve", [lib.TB_VESTA, lib.TB_PALLAS])
@pytest.mark.parametrize("n,window,family", VAR_CASES)
def test_msm_exceptional(gpu_ctx, curve, n, window, family):
    """Context.msm of every scalar family in one batched call equals the discrete-log reference."""
    pts, s, names, want = var_case(curve, n, window, family)
    got, groups = msm_groups(gpu_ctx, lambda: gpu_ctx.msm(curve, s, pts, batch=len(names), window_bits=window))
    assert_results(got, want, names, "tb_msm n=%d window_bits=%d" % (n, window))
    assert_latency_path(groups, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("window", [1, 21])
def test_msm_refuses_window(gpu_ctx, window):
    """window_bits outside 2..20 is refused with TB_ERR_INVALID, and the context computes a correct MSM afterwards."""
    pts, s, names, want = var_case(lib.TB_PALLAS, 9, 0, "small")
    with pytest.raises(lib.TaigaB200Error) as e:
        gpu_ctx.msm(lib.TB_PALLAS, s, pts, batch=len(names), window_bits=window)
    assert e.value.status == lib.TB_ERR_INVALID, str(e.value)
    assert_results(gpu_ctx.msm(lib.TB_PALLAS, s, pts, batch=len(names)), want, names, "tb_msm after a refused window")
