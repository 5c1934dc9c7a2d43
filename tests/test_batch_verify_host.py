"""CPU: the batch verifier (tb_batch_verifier) without a device.

* The four entry points are declared in the header with the signatures lib._SIGS binds, the header states the soundness
  condition of the seed, and the weight's PRF tag differs from every other tag of the library.
* A null context or batch is refused without touching a device; freeing a null batch is a no-op.
* A C++ program that uses the header's BatchVerifier compiles with plain g++, links against the in-tree library, and
  reports the missing device as a typed BackendFailure.
* The source checks of the launch helper and of device ownership hold for the new code (it launches through `launch` and
  keeps its device state in DevMem)."""
import os
import re
import subprocess

import pytest

import test_device_ownership as own
import test_launch_sites as ls
from conftest import ROOT
from taiga_b200 import lib

NEW = ["tb_batch_verifier_create", "tb_batch_verifier_add", "tb_batch_verifier_finalize", "tb_batch_verifier_free"]


def _header():
    return open(os.path.join(ROOT, "include", "taiga_b200.h")).read()


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def test_declarations_match_the_binding():
    hdr = re.sub(r"/\*.*?\*/", "", _header(), flags=re.S)
    for name in NEW:
        m = re.search(r"\b(tb_status|void)\s+%s\s*\(([^;]*)\);" % name, hdr)
        assert m, name
        params = [p for p in m.group(2).replace("\n", " ").split(",") if p.strip()]
        res, args = lib._SIGS[name]
        assert (m.group(1) == "void") == (res is None), name
        assert len(params) == len(args), (name, params, args)
    # the same argument list as tb_verify_batch_vk after the batch handle
    assert lib._SIGS["tb_batch_verifier_add"][1][2:] == lib._SIGS["tb_verify_batch_vk"][1][1:-1]


def test_header_states_the_seed_condition_and_the_verdict():
    text = " ".join(_header().split())
    assert "unpredictable to whoever made the proofs" in text
    assert "at most 1/p" in text and "fresh seed per batch" in text
    assert "every proof added since create would be accepted by tb_verify_batch_vk" in text
    assert "An empty batch gives 1" in text


def test_weight_tag_is_distinct():
    text = open(os.path.join(ROOT, "taiga_b200", "csrc", "prover.cuh")).read()
    body = re.search(r"enum RndTag \{(.*?)\};", text, re.S).group(1)
    body = re.sub(r"//[^\n]*", "", body)
    values, nxt = {}, 0
    for item in (s.strip() for s in body.split(",")):
        if not item:
            continue
        name, _, val = item.partition("=")
        nxt = int(val) if val.strip() else nxt
        values[name.strip()] = nxt
        nxt += 1
    assert "R_BATCH_WEIGHT" in values
    assert len(set(values.values())) == len(values), values


def test_null_arguments_are_refused_without_a_device():
    so = lib.load()
    assert so.tb_batch_verifier_create(None, None, None, None) == lib.TB_ERR_INVALID
    assert so.tb_batch_verifier_add(None, None, None, 1, None, None, None, 0, 0) == lib.TB_ERR_INVALID
    assert so.tb_batch_verifier_finalize(None, None, None) == lib.TB_ERR_INVALID
    so.tb_batch_verifier_free(None)


CPP = r"""
#include <cstdio>
#include "taiga_b200.hpp"
using namespace taiga_b200;
int main() {
  try {
    Context ctx(0);
    std::vector<uint8_t> g(64 * 2, 0);
    Params params(ctx, 1, g.data(), g.data(), PointBytes{}, PointBytes{});
    BatchVerifier bv(params, std::array<uint8_t, 32>{});
    ConstraintSystem cs;
    VerifyingKey vk(params, cs, {}, {});
    bv.add_proof(vk, {}, Proof(std::vector<uint8_t>(32)));
    bv.add_proofs(vk, {Proof(std::vector<uint8_t>(32))}, {{}});
    std::printf("verdict %d\n", bv.finalize() ? 1 : 0);
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "%s (status %d): %s\n", e.kind(), e.status(), e.what());
    return 1;
  }
}
"""


def test_cpp_batch_verifier_builds_and_fails_loudly_without_gpu(tmp_path):
    src = tmp_path / "batch.cpp"
    src.write_text(CPP)
    exe = str(tmp_path / "batch")
    libdir = os.path.dirname(lib.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-L", libdir, "-ltaiga_b200", "-Wl,-rpath," + libdir, "-o", exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    if not _no_gpu():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "BackendFailure" in r.stderr and "status 2" in r.stderr, r.stdout + r.stderr


def test_new_code_passes_the_source_checks():
    assert "batch_g_scalars_kernel" in ls.sources()["verifier.cu"]
    ls.test_no_triple_chevron_launch()
    ls.test_launch_kernel_ex_only_in_helper()
    ls.test_launch_count_changed_only_in_helper()
    own.test_synchronous_allocation_only_in_owner()
    own.test_stream_ordered_allocation_only_in_context()
    own.test_streams_and_events_only_in_context()
    body = own.span("verifier.cu", "struct BatchVerifier {")
    text = ls.sources()["verifier.cu"][body[1]:body[2]]
    assert "DevMem<Fp> g;" in text and "DevMem<Xyzz<Fq>> acc;" in text and "DevBuf" not in text
