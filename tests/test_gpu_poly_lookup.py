"""The prover's polynomial and lookup kernels (polyops.cu, lookup.cu), each called on its own through the test probe
libtaiga_b200_probe.so and compared, canonical byte for canonical byte, with a Python big-integer reference written from
the operation's definition.

A whole proof only says which proof section holds the first differing byte.  These tests name the kernel, the size, the
batch item and the first differing index, and they run every launch shape of every driver:

  poly_kate_div    n = 2 ... 2^15: one CTA with fewer than 512 threads, one CTA with 1, 2 or 4 coefficients a thread, and the
                   8-CTA cluster with 1, 2, 4 or 8; n = 2^16 is refused before anything is launched
  poly_eval        n = 2 ... 2^16: idle threads below 256 coefficients, then n / 256 coefficients a thread
  batch_inverse    counts around the 16-element chunk, zeros inside chunks
  prefix_product   n = 2 ... 2^16, T = min(n, 512) threads
  lookup_keys, sort_keys, lookup_arrange
                   n = 2^3 ... 2^16 (the local bitonic network up to 2048 keys, global steps above), usable = n - bf - 1 for
                   bf in {1, 5, 8}; the arrangement is checked against a restatement of halo2's permute_expression_pair

and the small drivers (inner product, powers, fma / scale / copy / add_at, the scalar interpreter).  The CPU tests check that
the probe loads and exports its entry points, and that the references themselves satisfy the identities they stand for.
"""
import collections
import ctypes
import os
import random

import numpy as np
import pytest

from oracle import pasta as o
from taiga_b200 import lib

P = o.P
PROBE_PATH = os.path.join(os.path.dirname(lib.LIB_PATH), "libtaiga_b200_probe.so")
_vp, _i, _ll, _sz = ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_size_t
# every entry point of the probe (taiga_b200/csrc/probe/tb_probe.cu) the tests bind: argument types after the tb_ctx*
PROBE_SIGS = {
    "tbp_poly_fma": [_vp, _ll, _vp, _ll, _vp, _ll, _i, _i],
    "tbp_poly_scale": [_vp, _ll, _vp, _ll, _vp, _ll, _i, _i],
    "tbp_poly_copy": [_vp, _ll, _vp, _ll, _i, _i],
    "tbp_poly_add_at": [_vp, _ll, _i, _vp, _ll, _i, _i],
    "tbp_poly_eval": [_vp, _i, _vp, _ll, _vp, _ll, _i, _i],
    "tbp_poly_kate_div": [_vp, _ll, _vp, _ll, _vp, _ll, _i, _i],
    "tbp_batch_inverse": [_vp, _sz],
    "tbp_prefix_product": [_vp, _vp, _i, _i],
    "tbp_inner_product": [_vp, _ll, _vp, _ll, _vp, _ll, _i, _i],
    "tbp_powers": [_vp, _ll, _vp, _ll, _i, _i],
    "tbp_scalar_program": [_vp, _ll, _vp, _i, _vp, _i],
    "tbp_lookup_keys": [_vp, _vp, _i, _i, _i],
    "tbp_sort_keys": [_vp, _i, _i],
    "tbp_lookup_arrange": [_vp, _vp, _vp, _vp, _i, _i, _i, _vp],
}
# prover.cuh: struct EvalItem { const Fp* base; long long bstride; int point; int pad; }, struct ScalarInstr { uint16_t op, dst, a, b; uint32_t imm; }
EVAL_ITEM = np.dtype([("base", "<u8"), ("bstride", "<i8"), ("point", "<i4"), ("pad", "<i4")])
SCALAR_INSTR = np.dtype([("op", "<u2"), ("dst", "<u2"), ("a", "<u2"), ("b", "<u2"), ("imm", "<u4")])
S_MUL, S_ADD, S_SUB, S_INV, S_COPY, S_POW2K, S_CONST, S_NEG, S_FMA, S_POWI = range(10)
SENTINEL_KEY = (1 << 256) - 1   # lookup_keys' key of a row >= usable
KD_MAX_N = 1 << 15              # prover.cuh: the longest polynomial poly_kate_div divides
GARBAGE = 7                     # fills every output region a driver must not write


def load_probe():
    lib.load()
    so = ctypes.CDLL(PROBE_PATH)
    for name, args in PROBE_SIGS.items():
        fn = getattr(so, name)
        fn.restype, fn.argtypes = _i, [_vp] + args
    return so


# ---------------------------------------------------------------- references (Python integers mod p)
def kate_ref(a, z):
    """halo2 kate_division, resized to n: q_{n-1} = 0 and q_j = a_{j+1} + z q_{j+1}."""
    n = len(a)
    q = [0] * n
    for j in range(n - 2, -1, -1):
        q[j] = (a[j + 1] + z * q[j + 1]) % P
    return q


def horner(a, x):
    acc = 0
    for c in reversed(a):
        acc = (acc * x + c) % P
    return acc


def kate_identity_holds(a, q, z):
    """q(X) (X - z) + a(z) == a(X), with q of degree below n - 1."""
    n = len(a)
    if q[n - 1] != 0:
        return False
    prod = [(horner(a, z) - z * q[0]) % P] + [(q[j - 1] - z * q[j]) % P for j in range(1, n)]
    return prod == a


def permute_expression_pair(inputs, table):
    """halo2 lookup::prover::permute_expression_pair over the usable rows: (A', S'), or None where halo2 returns
    Error::ConstraintSystemFailure.  A' is the sorted inputs; the first row of each run of A' takes one copy of its value
    from a BTreeMap of table counts; the leftover table values, in ascending order, go to the repeated rows popped from
    the back of their list."""
    a = sorted(inputs)
    left = collections.Counter(table)
    s, repeated = [None] * len(a), []
    for i, v in enumerate(a):
        if i == 0 or v != a[i - 1]:
            if left[v] == 0:
                return None
            left[v] -= 1
            s[i] = v
        else:
            repeated.append(i)
    for v in sorted(left):
        for _ in range(left[v]):
            s[repeated.pop()] = v
    return a, s


def arrangement_holds(inputs, table, a, s):
    """The lookup argument's conditions on (A', S'): A' is the sorted inputs, S' a permutation of the table,
    A'[0] = S'[0], and every A'[i] equals S'[i] or A'[i - 1]."""
    return (a == sorted(inputs) and sorted(s) == sorted(table) and a[0] == s[0]
            and all(a[i] == s[i] or a[i] == a[i - 1] for i in range(1, len(a))))


def run_scalar_program(v, prog, consts):
    """prover.cuh's ScalarOp semantics on one proof's variables."""
    v = list(v)
    for op, dst, a, b, imm in prog:
        if op == S_MUL:
            r = v[a] * v[b]
        elif op == S_ADD:
            r = v[a] + v[b]
        elif op == S_SUB:
            r = v[a] - v[b]
        elif op == S_INV:
            r = pow(v[a], -1, P)
        elif op == S_COPY:
            r = v[a]
        elif op == S_POW2K:
            r = pow(v[a], 1 << imm, P)
        elif op == S_CONST:
            r = consts[imm]
        elif op == S_NEG:
            r = -v[a]
        elif op == S_FMA:
            r = v[dst] * v[a] + v[b]
        elif op == S_POWI:
            r = pow(v[a], imm, P)
        v[dst] = r % P
    return v


LOOKUP_FAMILIES = ("all_equal", "all_distinct", "table_repeats", "heavy_repetition", "top_limb", "bottom_limb", "extremes")


def lookup_family(name, u, rnd):
    """(inputs, table) of u usable rows, every input in the table."""
    rand = lambda: rnd.randrange(P)   # noqa: E731
    if name == "all_equal":
        table = [rand() for _ in range(u)]
        return [rnd.choice(table)] * u, table
    if name == "all_distinct":
        table = [rand() for _ in range(u)]
        inputs = table[:]
        rnd.shuffle(inputs)
        return inputs, table
    if name == "table_repeats":
        pal = [rand() for _ in range(max(1, u // 4))]
        table = [rnd.choice(pal) for _ in range(u)]
        return [rnd.choice(table) for _ in range(u)], table
    if name == "heavy_repetition":
        table = [rand() for _ in range(u)]
        small = table[:3]
        return [rnd.choice(small) for _ in range(u)], table
    if name == "top_limb":   # equal below bit 224
        base = rnd.getrandbits(224)
        table = [base + (t << 224) for t in rnd.sample(range(1 << 29), u)]
        return [rnd.choice(table[:max(1, u // 8)]) for _ in range(u)], table
    if name == "bottom_limb":   # equal above bit 32
        base = rnd.randrange(P >> 33) << 32
        table = [base + t for t in rnd.sample(range(1 << 32), u)]
        return [rnd.choice(table[:max(1, u // 8)]) for _ in range(u)], table
    if name == "extremes":
        pal = [0, P - 1, 1, P - 2]
        table = (pal + [rand() for _ in range(u)])[:u]
        return [rnd.choice(table[:4]) for _ in range(u)], table
    raise ValueError(name)


# ---------------------------------------------------------------- CPU: the probe and the references
def test_probe_loads_without_a_device_and_exports_every_wrapper():
    assert os.path.exists(PROBE_PATH), "libtaiga_b200_probe.so must be built in-tree (see __graft_entry__.build)"
    so = load_probe()
    for name in PROBE_SIGS:
        assert hasattr(so, name), name
    # not public ABI: the header and the ctypes binding of the library know nothing of it
    assert not any(name.startswith("tbp_") for name in lib.exported_symbols())
    # every wrapper refuses a null context without touching a device
    assert so.tbp_batch_inverse(None, None, 0) == lib.TB_ERR_INVALID
    assert so.tbp_sort_keys(None, None, 8, 1) == lib.TB_ERR_INVALID


def test_permute_expression_pair_worked_example():
    # repeated rows 1, 3, 4 take the leftovers 3, 4, 5: the smallest goes to the last repeated row
    assert permute_expression_pair([2, 1, 2, 1, 2], [5, 4, 3, 2, 1]) == ([1, 1, 2, 2, 2], [1, 5, 2, 4, 3])
    assert permute_expression_pair([1, 6], [1, 2]) is None


@pytest.mark.parametrize("u", [1, 2, 6, 57, 1000])
def test_permute_reference_satisfies_the_lookup_conditions(u):
    rnd = random.Random(u)
    for name in LOOKUP_FAMILIES:
        inputs, table = lookup_family(name, u, rnd)
        a, s = permute_expression_pair(inputs, table)
        assert arrangement_holds(inputs, table, a, s), (name, u)
    inputs, table = lookup_family("table_repeats", max(u, 2), rnd)
    inputs[-1] = (max(table) + 1) % P
    assert permute_expression_pair(inputs, table) is None


@pytest.mark.parametrize("logn", [1, 2, 5, 9, 12])
def test_kate_reference_satisfies_the_division_identity(logn):
    rnd = random.Random(logn)
    n = 1 << logn
    for z in (0, 1, P - 1, pow(o.ROOT_P, 1 << (32 - logn), P), rnd.randrange(P)):
        a = [rnd.randrange(P) for _ in range(n)]
        q = kate_ref(a, z)
        assert kate_identity_holds(a, q, z)
        assert not kate_identity_holds(a, q[:1] + [(q[1] + 1) % P] + q[2:] if n > 2 else [(q[0] + 1) % P] + q[1:], z)


# ---------------------------------------------------------------- GPU
def ints_to_np(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), np.uint8)


def np_to_ints(a):
    raw = a.tobytes()
    return [int.from_bytes(raw[i:i + 32], "little") for i in range(0, len(raw), 32)]


class Probe:
    """The probe bound to one context, with device buffers as flat uint8 torch tensors of 32-byte elements."""

    def __init__(self, ctx):
        import torch
        self.torch, self.ctx, self.so = torch, ctx, load_probe()

    def status(self, name, *args):
        self.torch.cuda.synchronize()   # torch's copies into the buffers are done before the context's stream reads them
        return getattr(self.so, name)(self.ctx._h, *args)

    def run(self, name, *args):
        st = self.status(name, *args)
        if st != lib.TB_OK:
            raise lib.TaigaB200Error(st, self.ctx._lib.tb_last_error(self.ctx._h).decode(errors="replace"))
        self.ctx.sync()

    def put(self, vals, mont=True):
        """device copy of field elements (Montgomery form unless mont=False)"""
        t = self.torch.from_numpy(ints_to_np(vals).copy()).cuda()
        self.torch.cuda.synchronize()
        if mont:
            self.ctx.dev_to_mont(lib.TB_FP, t, len(vals))
            self.ctx.sync()
        return t

    def raw(self, arr):
        t = self.torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(-1).copy()).cuda()
        self.torch.cuda.synchronize()
        return t

    def get(self, t, mont=True):
        self.ctx.sync()
        c = t.clone()
        self.torch.cuda.synchronize()
        if mont:
            self.ctx.dev_from_mont(lib.TB_FP, c, c.numel() // 32)
            self.ctx.sync()
        return np_to_ints(c.cpu().numpy())


def addr(t, elem=0):
    return t.data_ptr() + 32 * elem


def expect(what, got, want):
    """fail naming `what` (kernel, size, batch item) and the first differing index"""
    if got != want:
        if len(got) != len(want):
            pytest.fail("%s: %d values, want %d" % (what, len(got), len(want)))
        i = next(i for i in range(len(want)) if got[i] != want[i])
        pytest.fail("%s: first difference at index %d of %d: got %#x, want %#x" % (what, i, len(want), got[i], want[i]))


@pytest.fixture(scope="module")
def probe(gpu_ctx):
    return Probe(gpu_ctx)


def poly_family(name, n, rnd):
    if name == "zero":
        return [0] * n
    if name == "leading":
        return [0] * (n - 1) + [rnd.randrange(1, P)]
    return [rnd.randrange(P) for _ in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("logn", range(1, 16))
def test_kate_division(probe, logn):
    """B = 5 divisions, z = 0, 1, p - 1, a root of unity and a random z, read with the prover's strides: the inputs are the
    middle of three polynomials per proof (the nps * n stride of the q polynomials), z is one slot of NV per proof."""
    rnd = random.Random(1000 + logn)
    n, B, NV, nps = 1 << logn, 5, 7, 3
    zs = [0, 1, P - 1, pow(o.ROOT_P, rnd.randrange(1, 1 << 32), P), rnd.randrange(P)]
    for fam in ("zero", "leading", "random"):
        polys = [poly_family(fam, n, rnd) for _ in range(B)]
        src = [rnd.randrange(P) for _ in range(B * nps * n)]
        for b in range(B):
            src[(b * nps + 1) * n:(b * nps + 2) * n] = polys[b]
        zvec = [rnd.randrange(P) for _ in range(B * NV)]
        for b in range(B):
            zvec[b * NV + 3] = zs[b]
        d_in, d_z, d_out = probe.put(src), probe.put(zvec), probe.put([GARBAGE] * (B * 2 * n))
        probe.run("tbp_poly_kate_div", addr(d_out), 2 * n, addr(d_in, n), nps * n, addr(d_z, 3), NV, n, B)
        out = probe.get(d_out)
        for b in range(B):
            what = "poly_kate_div n=%d %s input, item %d (z=%#x)" % (n, fam, b, zs[b])
            q = out[2 * b * n:(2 * b + 1) * n]
            expect(what, q, kate_ref(polys[b], zs[b]))
            assert kate_identity_holds(polys[b], q, zs[b]), what
            expect(what + ", past the item", out[(2 * b + 1) * n:(2 * b + 2) * n], [GARBAGE] * n)
        assert probe.get(d_in) == src, "poly_kate_div n=%d wrote its input" % n


@pytest.mark.gpu
def test_kate_division_refuses_more_than_one_cluster(probe, gpu_ctx):
    n = 2 * KD_MAX_N
    d = probe.put([1] * n)
    z = probe.put([3])
    before = gpu_ctx.launch_count
    assert probe.status("tbp_poly_kate_div", addr(d), n, addr(d), n, addr(z), 1, n, 1) == lib.TB_ERR_INVALID
    assert "too long for one cluster" in gpu_ctx._lib.tb_last_error(gpu_ctx._h).decode()
    assert gpu_ctx.launch_count == before, "the refused division launched a kernel"


@pytest.mark.gpu
@pytest.mark.parametrize("logn", range(1, 17))
def test_poly_eval(probe, logn):
    """Four items in one launch over B = 3 proofs: a shared polynomial (bstride 0, like fixed and sigma columns), per-proof
    polynomials with strides 2n and n, and the shared one again at another point.  Points: 0, 1, p - 1 and a random x,
    rotated over the proofs, in slots of NV per proof; evaluations at a stride of nitems + 1."""
    rnd = random.Random(2000 + logn)
    n, B, NV = 1 << logn, 3, 6
    shared = [rnd.randrange(P) for _ in range(n)]
    shared[n - 1] = P - 1
    wide = [rnd.randrange(P) for _ in range(B * 2 * n)]
    tight = [rnd.randrange(P) for _ in range(B * n)]
    xs = [0, 1, P - 1, rnd.randrange(P)]
    pts = [0] * (B * NV)
    for b in range(B):
        for s in range(4):
            pts[b * NV + 1 + s] = xs[(s + b) % 4]
    d_shared, d_wide, d_tight, d_pts = probe.put(shared), probe.put(wide), probe.put(tight), probe.put(pts)
    items = np.zeros(4, EVAL_ITEM)
    items[0] = (addr(d_shared), 0, 1, 0)
    items[1] = (addr(d_wide, n // 2), 2 * n, 2, 0)
    items[2] = (addr(d_tight), n, 3, 0)
    items[3] = (addr(d_shared), 0, 4, 0)
    d_items = probe.raw(items)
    ev_stride = 5
    d_ev = probe.put([GARBAGE] * (B * ev_stride))
    probe.run("tbp_poly_eval", addr(d_items), 4, addr(d_pts), NV, addr(d_ev), ev_stride, n, B)
    ev = probe.get(d_ev)
    off = n // 2
    for b in range(B):
        polys = [shared, wide[b * 2 * n + off:b * 2 * n + off + n], tight[b * n:(b + 1) * n], shared]
        want = [horner(polys[t], pts[b * NV + 1 + t]) for t in range(4)] + [GARBAGE]
        expect("poly_eval n=%d proof %d (items 0..3, then the gap)" % (n, b), ev[b * ev_stride:(b + 1) * ev_stride], want)


@pytest.mark.gpu
@pytest.mark.parametrize("count", [1, 15, 16, 17, 33, 3 * (1 << 15) + 7])
def test_batch_inverse(probe, count):
    """Zeros between nonzero values (0 -> 0, and the rest of the chunk unharmed), a whole chunk of zeros, 1, p - 1 and random
    values; the 16 elements past `count` are not written."""
    rnd = random.Random(3000 + count)
    vals = [rnd.randrange(1, P) for _ in range(count)]
    for i in range(0, count, 3):
        vals[i] = 0
    for i, v in zip(range(1, count, 7), [1, P - 1] * count):
        vals[i] = v
    if count >= 64:
        vals[32:48] = [0] * 16
    d = probe.put(vals + [GARBAGE] * 16)
    probe.run("tbp_batch_inverse", addr(d), count)
    got = probe.get(d)
    want = [pow(v, -1, P) if v else 0 for v in vals] + [GARBAGE] * 16
    expect("batch_inverse count=%d" % count, got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("logn", range(1, 17))
def test_prefix_product(probe, logn):
    """Three vectors: random, one with a zero in the middle, one of 1 and p - 1; out[0] = 1 (the exclusive product)."""
    rnd = random.Random(4000 + logn)
    n, count = 1 << logn, 3
    vecs = [[rnd.randrange(P) for _ in range(n)] for _ in range(2)] + [[rnd.choice((1, P - 1)) for _ in range(n)]]
    vecs[1][n // 2] = 0
    d_in, d_out = probe.put(sum(vecs, [])), probe.put([GARBAGE] * (count * n))
    probe.run("tbp_prefix_product", addr(d_out), addr(d_in), n, count)
    out = probe.get(d_out)
    for c, v in enumerate(vecs):
        want, acc = [], 1
        for x in v:
            want.append(acc)
            acc = acc * x % P
        expect("prefix_product n=%d vector %d" % (n, c), out[c * n:(c + 1) * n], want)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 2, 15, 16, 17, 255, 256, 257, 1 << 15])
def test_inner_product_and_powers(probe, n):
    """B = 4 proofs with x = 0 (0^0 = 1), 1, p - 1 and a random x in slots of NV; the inner product reads a at stride 2n
    (the IPA's halves) and b at stride n."""
    rnd = random.Random(5000 + n)
    B, NV = 4, 5
    xs = [0, 1, P - 1, rnd.randrange(P)]
    xv = [rnd.randrange(P) for _ in range(B * NV)]
    for b in range(B):
        xv[b * NV + 2] = xs[b]
    d_x = probe.put(xv)
    d_pw = probe.put([GARBAGE] * (B * (n + 1)))
    probe.run("tbp_powers", addr(d_pw), n + 1, addr(d_x, 2), NV, n, B)
    pw = probe.get(d_pw)
    for b in range(B):
        want = [pow(xs[b], i, P) for i in range(n)] + [GARBAGE]
        expect("powers n=%d proof %d (x=%#x)" % (n, b, xs[b]), pw[b * (n + 1):(b + 1) * (n + 1)], want)

    a = [rnd.randrange(P) for _ in range(B * 2 * n)]
    bv = [rnd.randrange(P) for _ in range(B * n)]
    d_a, d_b, d_out = probe.put(a), probe.put(bv), probe.put([GARBAGE] * (B * NV))
    probe.run("tbp_inner_product", addr(d_out, 1), NV, addr(d_a), 2 * n, addr(d_b), n, n, B)
    out = probe.get(d_out)
    for b in range(B):
        want = sum(x * y for x, y in zip(a[b * 2 * n:b * 2 * n + n], bv[b * n:(b + 1) * n])) % P
        expect("inner_product n=%d proof %d" % (n, b), out[b * NV:(b + 1) * NV], [GARBAGE, want] + [GARBAGE] * (NV - 2))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 255, 256, 257, 4096])
def test_fma_scale_copy_add_at(probe, n):
    """B = 3 proofs at a stride of n + 3, scalars in slots of NV; inputs shared (stride 0) and per proof; add_at with
    sign +1 and -1.  Elements between the items are not written."""
    rnd = random.Random(6000 + n)
    B, NV, S = 3, 4, n + 3
    sv = [rnd.randrange(P) for _ in range(B * NV)]
    sv[0 * NV + 1], sv[1 * NV + 1] = 0, P - 1
    base = [rnd.randrange(P) for _ in range(B * S)]
    per = [rnd.randrange(P) for _ in range(B * S)]
    shared = [rnd.randrange(P) for _ in range(n)]
    d_s, d_per, d_shared = probe.put(sv), probe.put(per), probe.put(shared)
    s = [sv[b * NV + 1] for b in range(B)]

    def check(what, got, f):
        want = list(base)
        for b in range(B):
            for i in range(n):
                want[b * S + i] = f(b, i)
        for b in range(B):
            expect("%s n=%d proof %d" % (what, n, b), got[b * S:(b + 1) * S], want[b * S:(b + 1) * S])

    for in_stride, src in ((S, per), (0, None)):
        inp = (lambda b, i: per[b * S + i]) if src else (lambda b, i: shared[i])
        d_in = d_per if src else d_shared
        tag = "stride %d" % in_stride
        d_out = probe.put(base)
        probe.run("tbp_poly_fma", addr(d_out), S, addr(d_s, 1), NV, addr(d_in), in_stride, n, B)
        check("poly_fma " + tag, probe.get(d_out), lambda b, i: (base[b * S + i] * s[b] + inp(b, i)) % P)
        d_out = probe.put(base)
        probe.run("tbp_poly_scale", addr(d_out), S, addr(d_s, 1), NV, addr(d_in), in_stride, n, B)
        check("poly_scale " + tag, probe.get(d_out), lambda b, i: inp(b, i) * s[b] % P)
        d_out = probe.put(base)
        probe.run("tbp_poly_copy", addr(d_out), S, addr(d_in), in_stride, n, B)
        check("poly_copy " + tag, probe.get(d_out), inp)

    for sign in (1, -1):
        idx = n - 1
        d_out = probe.put(base)
        probe.run("tbp_poly_add_at", addr(d_out), S, idx, addr(d_s, 1), NV, sign, B)
        got = probe.get(d_out)
        want = list(base)
        for b in range(B):
            want[b * S + idx] = (base[b * S + idx] + sign * s[b]) % P
        expect("poly_add_at n=%d sign %d" % (n, sign), got, want)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [1, 37])
def test_scalar_program(probe, B):
    """Every opcode, with S_POW2K by 0 and 3, S_POWI by 0, 1, 5 and 2^32 - 1, S_FMA with its destination as a and as b,
    S_NEG of zero, in-place squaring; B = 37 leaves a partial warp.  No division by zero (halo2 would panic there)."""
    rnd = random.Random(7000 + B)
    NV = 16
    consts = [5, P - 1, 0, rnd.randrange(P)]
    prog = [
        (S_MUL, 8, 0, 1, 0), (S_ADD, 9, 1, 2, 0), (S_SUB, 10, 2, 0, 0), (S_SUB, 11, 3, 3, 0), (S_INV, 12, 0, 0, 0),
        (S_COPY, 13, 4, 0, 0), (S_POW2K, 14, 0, 0, 0), (S_POW2K, 15, 1, 0, 3), (S_CONST, 5, 0, 0, 1), (S_CONST, 6, 0, 0, 3),
        (S_NEG, 7, 11, 0, 0), (S_NEG, 3, 2, 0, 0), (S_FMA, 8, 9, 10, 0), (S_FMA, 9, 9, 12, 0), (S_FMA, 10, 0, 10, 0),
        (S_POWI, 13, 0, 0, 0), (S_POWI, 14, 1, 0, 1), (S_POWI, 15, 2, 0, 5), (S_POWI, 4, 0, 0, 0xFFFFFFFF), (S_MUL, 2, 2, 2, 0),
        (S_INV, 0, 5, 0, 0), (S_ADD, 1, 1, 1, 0),
    ]
    vars_ = [rnd.randrange(1, P) for _ in range(B * NV)]
    for b in range(B):
        vars_[b * NV + 2] = (0, 1, P - 1)[b % 3] if b % 4 == 3 else vars_[b * NV + 2]
    d_vars, d_consts = probe.put(vars_), probe.put(consts)
    d_prog = probe.raw(np.array(prog, SCALAR_INSTR))
    probe.run("tbp_scalar_program", addr(d_vars), NV, addr(d_prog), len(prog), addr(d_consts), B)
    got = probe.get(d_vars)
    for b in range(B):
        want = run_scalar_program(vars_[b * NV:(b + 1) * NV], prog, consts)
        expect("scalar_program proof %d of %d" % (b, B), got[b * NV:(b + 1) * NV], want)


def run_lookup(probe, inputs, tables, n, usable, rnd):
    """lookup_keys, sort_keys and lookup_arrange as the prover runs them, over len(inputs) arrays: the usable rows hold
    each array's values, the rows past them random values the keys must turn into sentinels.
    Returns (sorted input keys, arranged table, error flags), all canonical."""
    arrays = len(inputs)
    pad = lambda v: list(v) + [rnd.randrange(P) for _ in range(n - usable)]   # noqa: E731
    d_a, d_t = probe.put(sum((pad(v) for v in inputs), [])), probe.put(sum((pad(v) for v in tables), []))
    d_ka, d_kt, d_left = probe.put([0] * (arrays * n), mont=False), probe.put([0] * (arrays * n), mont=False), probe.put([0] * (arrays * n), mont=False)
    d_s = probe.put([GARBAGE] * (arrays * n), mont=False)
    d_err = probe.raw(np.zeros(arrays, np.uint32))
    probe.run("tbp_lookup_keys", addr(d_ka), addr(d_a), n, usable, arrays)
    probe.run("tbp_lookup_keys", addr(d_kt), addr(d_t), n, usable, arrays)
    probe.run("tbp_sort_keys", addr(d_ka), n, arrays)
    probe.run("tbp_sort_keys", addr(d_kt), n, arrays)
    probe.run("tbp_lookup_arrange", addr(d_ka), addr(d_kt), addr(d_left), addr(d_s), n, usable, arrays, addr(d_err))
    ka, kt, s = probe.get(d_ka, mont=False), probe.get(d_kt, mont=False), probe.get(d_s, mont=False)
    err = d_err.cpu().numpy().view(np.uint32).tolist()
    return ka, kt, s, err


@pytest.mark.gpu
@pytest.mark.parametrize("logn,bf", [(k, bf) for k in range(3, 17) for bf in (1, 5, 8) if (1 << k) > bf + 2])
def test_lookup_arrangement(probe, logn, bf):
    """Every value family as one array of a single launch; A' and S' equal permute_expression_pair's bit for bit, the rows
    past `usable` sort to the end as sentinels, and no error flag is set."""
    rnd = random.Random(8000 + 31 * logn + bf)
    n = 1 << logn
    usable = n - bf - 1
    fams = [lookup_family(f, usable, rnd) for f in LOOKUP_FAMILIES]
    ka, kt, s, err = run_lookup(probe, [f[0] for f in fams], [f[1] for f in fams], n, usable, rnd)
    for i, (name, (inputs, table)) in enumerate(zip(LOOKUP_FAMILIES, fams)):
        what = "n=%d usable=%d array %d (%s)" % (n, usable, i, name)
        a_ref, s_ref = permute_expression_pair(inputs, table)
        expect("lookup_keys + sort_keys (inputs) " + what, ka[i * n:(i + 1) * n], a_ref + [SENTINEL_KEY] * (n - usable))
        expect("lookup_keys + sort_keys (table) " + what, kt[i * n:(i + 1) * n], sorted(table) + [SENTINEL_KEY] * (n - usable))
        expect("lookup_arrange " + what, s[i * n:i * n + usable], s_ref)
        assert err[i] == 0, "lookup_arrange %s: error flag set on a valid lookup" % what
    # the arrangement writes no row past the usable ones
    assert all(s[i * n + r] == GARBAGE for i in range(len(fams)) for r in range(usable, n)), "lookup_arrange wrote past usable"


@pytest.mark.gpu
@pytest.mark.parametrize("logn,bad", [(4, 0), (10, 2), (12, 3)])
def test_lookup_error_flag_names_the_failing_array(probe, logn, bad):
    """Four arrays, one of which has an input missing from its table: only its flag is set, the others stay exact."""
    rnd = random.Random(9000 + logn)
    n, bf = 1 << logn, 5
    usable = n - bf - 1
    fams = [lookup_family(f, usable, rnd) for f in ("table_repeats", "heavy_repetition", "all_distinct", "bottom_limb")]
    inputs = [list(f[0]) for f in fams]
    tables = [f[1] for f in fams]
    present = set(tables[bad])
    missing = next(v for v in range(1, P) if v not in present)
    inputs[bad][rnd.randrange(usable)] = missing
    ka, kt, s, err = run_lookup(probe, inputs, tables, n, usable, rnd)
    assert err == [1 if i == bad else 0 for i in range(4)], "lookup_arrange n=%d: error flags %s, array %d is the failing one" % (n, err, bad)
    for i in range(4):
        if i == bad:
            assert permute_expression_pair(inputs[i], tables[i]) is None
            continue
        a_ref, s_ref = permute_expression_pair(inputs[i], tables[i])
        expect("lookup_keys + sort_keys n=%d array %d next to a failing one" % (n, i), ka[i * n:i * n + usable], a_ref)
        expect("lookup_arrange n=%d array %d next to a failing one" % (n, i), s[i * n:i * n + usable], s_ref)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2048, 4096, 1 << 16])
def test_sort_keys(probe, n):
    """Three arrays: runs of a few values whose boundaries straddle the 2048-key tiles, distinct keys in descending order,
    and random keys with duplicates and sentinels (sort_keys compares raw 256-bit keys)."""
    rnd = random.Random(10000 + n)
    few = [rnd.randrange(P) for _ in range(5)]
    runs = []
    while len(runs) < n:
        runs += [rnd.choice(few)] * rnd.randrange(1, 3000)
    desc = sorted((rnd.randrange(P) for _ in range(n)), reverse=True)
    mixed = [rnd.choice((SENTINEL_KEY, 0, rnd.randrange(P), few[0])) for _ in range(n)]
    keys = [runs[:n], desc, mixed]
    d = probe.put(sum(keys, []), mont=False)
    probe.run("tbp_sort_keys", addr(d), n, 3)
    got = probe.get(d, mont=False)
    for i, k in enumerate(keys):
        expect("sort_keys n=%d array %d" % (n, i), got[i * n:(i + 1) * n], sorted(k))
