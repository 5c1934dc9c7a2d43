"""CPU: the verifying-key path without a device.

* The new entry points (tb_vk_load, tb_verify_batch_vk, tb_decompress) are reached through a context, which fails with
  TB_ERR_CUDA and a typed error when no device is present; the C++ example, which now verifies through a VerifyingKey,
  builds and reports the missing device as a BackendFailure.
* A verifying key holds the circuit's shape and its commitments only: no device allocation and no per-row table.
* The point decoder the device kernel compiles (transcript.cuh decompress_point), built for the host, matches verifier_py
  on every 32-byte chunk of both k = 15 golden proofs and on the non-canonical encodings the soundness tests use."""
import ctypes
import os
import re
import subprocess

import pytest

from conftest import GOLDEN, ROOT
from oracle import verifier_py as vp
from taiga_b200 import lib

import soundness_cases as sc

CSRC = os.path.join(ROOT, "taiga_b200", "csrc")


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def test_new_entry_points_fail_loudly_without_gpu():
    so = lib.load()
    # a null context or key is refused without touching a device
    assert so.tb_vk_load(None, None, None, None, None, None) == lib.TB_ERR_INVALID
    assert so.tb_verify_batch_vk(None, None, 1, None, None, None, 0, 0, None) == lib.TB_ERR_INVALID
    assert so.tb_decompress(None, 1, None, None, None) == lib.TB_ERR_INVALID
    assert so.tb_vk_proof_len(None) == 0
    so.tb_vk_free(None)
    if not _no_gpu():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    with pytest.raises(lib.TaigaB200Error) as e:
        lib.Context(0)
    assert e.value.status == lib.TB_ERR_CUDA


def test_cpp_example_verifies_through_a_verifying_key(tmp_path):
    src = open(os.path.join(ROOT, "examples", "prove_cpp.cpp")).read()
    assert re.search(r"VerifyingKey vk\(params, cs, ", src) and "proof.verify(vk, params, instance)" in src
    exe = str(tmp_path / "prove_cpp")
    libdir = os.path.dirname(lib.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), os.path.join(ROOT, "examples", "prove_cpp.cpp"),
                        "-L", libdir, "-ltaiga_b200", "-Wl,-rpath," + libdir, "-o", exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    if not _no_gpu():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "BackendFailure" in r.stderr and "status 2" in r.stderr, r.stdout + r.stderr


def _struct_body(text, name):
    start = text.index("{", text.index("struct %s " % name))
    depth = 0
    for i in range(start, len(text)):
        depth += {"{": 1, "}": -1}.get(text[i], 0)
        if depth == 0:
            return text[start:i + 1]
    raise AssertionError("unbalanced struct " + name)


def test_verifying_key_holds_no_device_memory_and_no_row_table():
    text = open(os.path.join(CSRC, "circuit.cuh")).read()
    shape, vk = _struct_body(text, "Shape"), _struct_body(text, "VerifyingKey")
    for body in (shape, vk):
        assert not re.search(r"\bDev(Mem|Buf)\b|\bint2\b", body), body
        # the per-row tables of the proving key: column values, coefficients, cosets, Lagrange and coset-factor tables
        assert not re.search(r"\b(fixed|sig)_(vals|polys|cosets)\b|\bl0\b|\bl_last\b|\bl_blind\b|\bcoset_pre\b|\bwr_inv\b", body), body
    assert re.search(r"\bShape shape;", vk) and re.search(r"std::vector<Aff<Fq>> fixed, sigma;", vk)
    # the proving key is the shape plus its device tables, and the verifier reads a shape, never a proving key
    assert "struct Circuit : Shape {" in text
    ver = open(os.path.join(CSRC, "verifier.cu")).read()
    body = ver[ver.index("static void verify_batch("):ver.index("static const Circuit& pk_commitments(")]
    assert "const Shape& C" in body and "Circuit" not in body


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("shim") / "host_shim.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(ROOT, "tests", "host_shim.cpp")])
    return ctypes.CDLL(so)


def host_decode(shim, enc):
    xy = (ctypes.c_uint8 * 64)()
    if not shim.hs_decompress((ctypes.c_uint8 * 32).from_buffer_copy(enc), xy):
        return "reject"
    r = bytes(xy)
    x, y = int.from_bytes(r[:32], "little"), int.from_bytes(r[32:], "little")
    return None if x == 0 and y == 0 else (x, y)


def ref_decode(enc):
    try:
        p = vp.decompress(enc)
    except vp.Reject:
        return "reject"
    return None if p[2] == 0 else vp._to_affine(p)


def encodings_of(chunk):
    """a 32-byte chunk, its sign-flipped twin, its x + q alias when it fits, negative zero and an x off the curve"""
    v = int.from_bytes(chunk, "little")
    x, sign = v & ((1 << 255) - 1), v >> 255
    out = [v, v ^ (1 << 255), 1 << 255, sc.OFF_CURVE_X | sign << 255]
    if x + vp.Q < 1 << 255:
        out.append((x + vp.Q) | sign << 255)
    return [e.to_bytes(32, "little") for e in out]


@pytest.mark.parametrize("name", ["proof_k15_compliance_shape.bin", "proof_k15_vp_shape.bin"])
def test_host_decoder_matches_verifier_py_on_golden_proofs(shim, name):
    proof = open(os.path.join(GOLDEN, name), "rb").read()
    assert len(proof) % 32 == 0
    seen = {"point": 0, "reject": 0, "identity": 0}
    for off in range(0, len(proof), 32):
        for enc in encodings_of(proof[off:off + 32]):
            got, want = host_decode(shim, enc), ref_decode(enc)
            assert got == want, "%s byte %d: %s decodes to %r, verifier_py to %r" % (name, off, enc.hex(), got, want)
            seen["reject" if want == "reject" else "identity" if want is None else "point"] += 1
    assert seen["point"] > 100 and seen["reject"] > 100, seen
    assert host_decode(shim, bytes(32)) is None and ref_decode(bytes(32)) is None
