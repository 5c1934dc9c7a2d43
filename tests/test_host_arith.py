"""CPU: the product's own field/curve and transcript source (taiga_b200/csrc/field.cuh, curve.cuh, transcript.cuh - the
code the kernels and the verifier compile) instantiated for the host and checked against the Python big-int oracle, hashlib
and the independent Python verifier."""
import ctypes
import hashlib
import os
import random
import subprocess

import pytest

from conftest import ROOT
from oracle import pasta as o


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("shim") / "host_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "host_shim.cpp")])
    return ctypes.CDLL(so)


def _b32(x):
    return (ctypes.c_uint8 * 32).from_buffer_copy(int(x).to_bytes(32, "little"))


def _b64(p):
    return (ctypes.c_uint8 * 64).from_buffer_copy(bytes(64) if p is None else int(p[0]).to_bytes(32, "little") + int(p[1]).to_bytes(32, "little"))


def test_field(shim):
    rnd = random.Random(5)

    def fo(f, op, a, b=0):
        out = (ctypes.c_uint8 * 32)()
        shim.hs_field(f, op, _b32(a), _b32(b), out)
        return int.from_bytes(bytes(out), "little")

    for f, m in [(0, o.P), (1, o.Q)]:
        edge = [0, 1, m - 1, m - 2, (1 << 256) % m, 2 ** 32 - 1, 2 ** 32, (1 << 255) % m, m >> 1]
        vals = edge + [rnd.randrange(m) for _ in range(200)]
        for a in vals:
            for b in rnd.sample(vals, 4) + edge[:4]:
                assert fo(f, 0, a, b) == (a + b) % m and fo(f, 1, a, b) == (a - b) % m and fo(f, 2, a, b) == a * b % m
            assert fo(f, 4, a) == (-a) % m and fo(f, 5, a) == a * a % m
        # inversion (divsteps, field.cuh::inv): every edge value, small values, powers of two and many random ones
        for a in vals + list(range(2, 40)) + [1 << i for i in range(1, 254, 7)] + [m - (1 << i) for i in range(1, 250, 11)] + [rnd.randrange(m) for _ in range(3000)]:
            assert fo(f, 3, a) == pow(a, m - 2, m), hex(a)


def test_curve(shim):
    rnd = random.Random(6)

    def po(c, op, a, b):
        out = (ctypes.c_uint8 * 64)()
        shim.hs_point(c, op, _b64(a), b if isinstance(b, ctypes.Array) else _b64(b), out)
        r = bytes(out)
        x, y = int.from_bytes(r[:32], "little"), int.from_bytes(r[32:], "little")
        return None if x == 0 and y == 0 else (x, y)

    for c, cv, G in [(0, o.VESTA, o.VESTA_GEN), (1, o.PALLAS, o.PALLAS_GEN)]:
        A, B = cv.mul(12345, G), cv.mul(99999, G)
        assert po(c, 0, A, B) == cv.add(A, B) and po(c, 0, A, A) == cv.add(A, A) and po(c, 0, A, cv.neg(A)) is None
        assert po(c, 0, A, None) == A and po(c, 0, None, B) == B
        assert po(c, 2, A, None) == cv.add(A, A) and po(c, 4, A, None) == cv.add(A, A)
        assert po(c, 3, A, B) == cv.add(cv.mul(2, A), cv.mul(3, B)) and po(c, 3, A, A) == cv.mul(5, A)
        for k in [0, 1, 2, 15, 16, cv.fs - 1, rnd.randrange(cv.fs)]:
            assert po(c, 1, A, _b32(k)) == cv.mul(k, A)


# ---------------------------------------------------------------- transcript.cuh: BLAKE2b, transcript, PRF, encodings
def _buf(b):
    return (ctypes.c_uint8 * max(1, len(b))).from_buffer_copy(bytes(b) or b"\0")


def _out(shim_fn, *args, n=32):
    out = (ctypes.c_uint8 * n)()
    shim_fn(*args, out)
    return bytes(out)


def _points(rnd, count):
    """count consecutive multiples of the Vesta generator from a random start, and their negations"""
    pts = [o.VESTA.mul(rnd.randrange(1, o.P), o.VESTA_GEN)]
    while len(pts) < count:
        pts.append(o.VESTA.add(pts[-1], o.VESTA_GEN))
    return pts + [o.VESTA.neg(p) for p in pts]


def test_blake2b_matches_hashlib(shim):
    rnd = random.Random(7)
    for person in (b"Halo2-Transcript", b"TaigaB200-Blind\0"):
        for n in (0, 1, 127, 128, 129, 255, 256, 257, 1000):
            data = bytes(rnd.randrange(256) for _ in range(n))
            ref = hashlib.blake2b(data, digest_size=64, person=person).digest()
            chunkings = [[n]]
            for _ in range(4):   # random cuts, empty pieces included
                cuts = sorted(rnd.randrange(n + 1) for _ in range(rnd.randrange(1, 6)))
                chunkings.append([b - a for a, b in zip([0] + cuts, cuts + [n])])
            for ch in chunkings:
                got = _out(shim.hs_blake2b, person, _buf(data), (ctypes.c_int * len(ch))(*ch), len(ch), n=64)
                assert got == ref, (person, n, ch)


def test_transcript_matches_oracle(shim):
    """Random interleavings of points, scalars and squeezes; every script squeezes once with exactly a multiple of 128
    bytes absorbed, where the last full block must stay buffered and be compressed as the final one."""
    rnd = random.Random(8)
    pts = _points(rnd, 16)
    boundary_squeezes = 0
    for _ in range(12):
        vk = rnd.randrange(o.P)
        ref = o.Transcript()
        ref.common_scalar(vk)
        ops, data, want = [], b"", []
        absorbed = 33
        pad_at = rnd.randrange(40)
        for i in range(40):
            kinds = [rnd.choice("PSZ")]
            if i == pad_at:   # a squeeze absorbs one byte: squeeze up to the next block boundary
                kinds = ["Z"] * (-absorbed % 128 or 128)
            for kind in kinds:
                if kind == "P":
                    p = rnd.choice(pts)
                    ref.common_point(p)
                    data += o.to_bytes(p[0]) + o.to_bytes(p[1])
                    absorbed += 65
                elif kind == "S":
                    s = rnd.randrange(o.P)
                    ref.common_scalar(s)
                    data += o.to_bytes(s)
                    absorbed += 33
                else:
                    want.append(ref.squeeze())
                    absorbed += 1
                    boundary_squeezes += absorbed % 128 == 0
                ops.append(kind)
        out = (ctypes.c_uint8 * (32 * len(want)))()
        assert shim.hs_transcript(_b32(vk), "".join(ops).encode(), len(ops), _buf(data), out) == -1
        assert [int.from_bytes(bytes(out)[32 * i:32 * i + 32], "little") for i in range(len(want))] == want
    assert boundary_squeezes >= 12
    # the identity is refused, as halo2's common_point refuses it
    with pytest.raises(ValueError):
        o.Transcript().common_point(None)
    assert shim.hs_transcript(_b32(0), b"SP", 2, _buf(bytes(96)), (ctypes.c_uint8 * 32)()) == 1


def test_prf_matches_hashlib(shim):
    seed = bytes(range(32))
    for proof, tag, idx in ((0, 1, 0), (5, 11, 32767), (1 << 20, 18, 14), (2 ** 32 - 1, 18, 2 ** 15 - 1)):
        m = seed + proof.to_bytes(4, "little") + tag.to_bytes(4, "little") + idx.to_bytes(4, "little") + bytes(4)
        ref = int.from_bytes(hashlib.blake2b(m, digest_size=64, person=b"TaigaB200-Blind\0").digest(), "little") % o.P
        assert int.from_bytes(_out(shim.hs_prf, _buf(seed), proof, tag, idx), "little") == ref


def test_point_and_scalar_encodings(shim):
    from oracle import verifier_py as vp
    from taiga_b200 import circuits_mini as cm
    import soundness_cases as sc

    def dec(enc):
        xy = (ctypes.c_uint8 * 64)()
        if not shim.hs_decompress(_buf(enc), xy):
            return "reject"
        r = bytes(xy)
        x, y = int.from_bytes(r[:32], "little"), int.from_bytes(r[32:], "little")
        return None if x == 0 and y == 0 else (x, y)

    def ref_dec(enc):
        try:
            p = vp.decompress(enc)
        except vp.Reject:
            return "reject"
        return None if p[2] == 0 else vp._to_affine(p)

    for p in _points(random.Random(9), 32) + [None]:
        assert _out(shim.hs_compress, _b64(p)) == o.VESTA.compress(p)
    kd, _ = cm.standard_plonk(k=6, wide=False, n_lookups=2)
    proof = open(os.path.join(ROOT, "tests", "golden", "proof_k6_plonk.bin"), "rb").read()
    slots = sc.slots(kd)
    assert len(proof) == slots[-1][2] + 32
    n_points = 0
    for name, e, off, kind in slots:
        v = int.from_bytes(proof[off:off + 32], "little")
        if kind == "point":
            n_points += 1
            x, sign = v & ((1 << 255) - 1), v >> 255
            for enc in (v, v ^ (1 << 255)):
                b = enc.to_bytes(32, "little")
                assert dec(b) == ref_dec(b) != "reject", (name, e)
            bad = [1 << 255, sc.OFF_CURVE_X | sign << 255, (1 << 256) - 1] + ([(x + vp.Q) | sign << 255] if x + vp.Q < 1 << 255 else [])
            for enc in bad:
                b = enc.to_bytes(32, "little")
                assert dec(b) == ref_dec(b) == "reject", (name, e, hex(enc))
        else:
            for enc, ok in ((v, True), (v + o.P, False), ((1 << 256) - 1, False)):
                out = (ctypes.c_uint8 * 32)()
                assert shim.hs_scalar(_buf(enc.to_bytes(32, "little")), out) == ok, (name, e, hex(enc))
                assert not ok or int.from_bytes(bytes(out), "little") == v
    assert n_points > 20
    assert dec(bytes(32)) is None and ref_dec(bytes(32)) is None


# ---------------------------------------------------------------- argument.cuh: permutation and lookup terms
def _fes(vals):
    return _buf(b"".join(o.to_bytes(v) for v in vals))


def _ints(vals):
    return (ctypes.c_int * max(1, len(vals)))(*vals)


def _perm_case(rnd, chunk, ncols, per_kind=3):
    """random permutation columns of every kind (each kind appears once there are 3 columns), values and sigmas"""
    kinds = [c % 3 for c in range(ncols)]
    rnd.shuffle(kinds)
    cols = [(k, rnd.randrange(per_kind)) for k in kinds]
    vals = [[rnd.randrange(o.P) for _ in range(per_kind)] for _ in range(3)]
    sig = [rnd.randrange(o.P) for _ in range(ncols)]
    return cols, vals, sig


def _ref_arg_terms(cols, vals, sig, pz, lk, x, beta, gamma, l_0, l_last, active, chunk):
    """oracle/verifier_py.py's permutation and lookup terms, from the same evaluations (pz[s] = z_s at x, wx, w^-(bf+1) x;
    lk[l] = Z(x), Z(wx), A'(x), A'(w^-1 x), S'(x) and the compressed input and table)"""
    P, DELTA, nsets = o.P, o.DELTA_P, len(pz)
    terms = []
    if nsets:
        terms.append(l_0 * (1 - pz[0][0]) % P)
        zl = pz[-1][0]
        terms.append(l_last * (zl * zl - zl) % P)
        for s in range(1, nsets):
            terms.append(l_0 * (pz[s][0] - pz[s - 1][2]) % P)
        for s in range(nsets):
            left, right = pz[s][1], pz[s][0]
            cur = beta * x % P * pow(DELTA, s * chunk, P) % P
            for ci, (kind, idx) in enumerate(cols[s * chunk:(s + 1) * chunk]):
                v = vals[kind][idx]
                left = left * (v + beta * sig[s * chunk + ci] + gamma) % P
                right = right * (v + cur + gamma) % P
                cur = cur * DELTA % P
            terms.append((left - right) * active % P)
    for z, zn, ap, apm, sp, a_c, t_c in lk:
        terms.append(l_0 * (1 - z) % P)
        terms.append(l_last * (z * z - z) % P)
        terms.append((zn * (ap + beta) % P * (sp + gamma) - z * (a_c + beta) % P * (t_c + gamma)) * active % P)
        terms.append(l_0 * (ap - sp) % P)
        terms.append((ap - sp) * (ap - apm) % P * active % P)
    return terms


# (chunk, columns): no permutation; one full set; one set partly filled; 4 sets, the last partly filled; 3 sets, the last
# partly filled; 16 sets of one column (the most a circuit may have)
_PERM_SHAPES = [(2, 0), (3, 3), (4, 2), (2, 7), (5, 13), (1, 16)]


def test_perm_set_products_match_big_int(shim):
    rnd = random.Random(10)
    P, k = o.P, 10
    for chunk, ncols in _PERM_SHAPES[1:]:
        cols, vals, sig = _perm_case(rnd, chunk, ncols)
        for s in range((ncols + chunk - 1) // chunk):
            beta, gamma, row = rnd.randrange(P), rnd.randrange(P), rnd.randrange(1 << k)
            cd = beta * pow(o.DELTA_P, s * chunk, P) % P * pow(o.omega(k), row, P) % P   # beta delta^(s chunk) X, X = omega^row
            out = (ctypes.c_uint8 * 64)()
            shim.hs_perm_set(_ints([c[0] for c in cols]), _ints([c[1] for c in cols]), _fes(vals[0]), _fes(vals[1]), _fes(vals[2]), _fes(sig), s, chunk, ncols,
                             _b32(beta), _b32(gamma), _b32(o.DELTA_P), _b32(cd), out)
            with_sigma = with_id = 1
            cur = cd
            for c in range(s * chunk, min((s + 1) * chunk, ncols)):
                v = vals[cols[c][0]][cols[c][1]]
                with_sigma = with_sigma * (v + beta * sig[c] + gamma) % P
                with_id = with_id * (v + cur + gamma) % P
                cur = cur * o.DELTA_P % P
            r = bytes(out)
            assert (int.from_bytes(r[:32], "little"), int.from_bytes(r[32:], "little")) == (with_sigma, with_id), (chunk, ncols, s)


def test_arg_fold_matches_big_int(shim):
    rnd = random.Random(11)
    P = o.P
    for chunk, ncols in _PERM_SHAPES:
        nsets = (ncols + chunk - 1) // chunk
        for L in (0, 1, 2):
            for _ in range(3):
                cols, vals, sig = _perm_case(rnd, chunk, ncols)
                pz = [[rnd.randrange(P) for _ in range(3)] for _ in range(nsets)]
                lk = [[rnd.randrange(P) for _ in range(7)] for _ in range(L)]
                acc, x, y, beta, gamma, l_0, l_last, active = (rnd.randrange(P) for _ in range(8))
                out = (ctypes.c_uint8 * 32)()
                shim.hs_arg_fold(_fes([acc, x, y, beta, gamma, l_0, l_last, active]), _b32(o.DELTA_P), _ints([c[0] for c in cols]), _ints([c[1] for c in cols]),
                                 _fes(vals[0]), _fes(vals[1]), _fes(vals[2]), _fes(sig), _fes([v for z in pz for v in z]), nsets, chunk, ncols, L,
                                 _fes([v for e in lk for v in e]), out)
                terms = _ref_arg_terms(cols, vals, sig, pz, lk, x, beta, gamma, l_0, l_last, active, chunk)
                want = acc
                for t in terms:
                    want = (want * y + t) % P
                assert int.from_bytes(bytes(out), "little") == want, (chunk, ncols, L)
                assert shim.hs_arg_terms(nsets, L) == len(terms)
