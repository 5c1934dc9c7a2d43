"""CPU: verification over device memory (tb_dev_verify_batch_vk, tb_dev_batch_verifier_add) without a device.

* The two entry points are declared in the header with the signatures lib._SIGS binds, and take the arguments of their host
  versions.
* A null context is refused without touching a device.
* A C++ program that uses the header's device-pointer overloads compiles with g++ -Wall -Werror and reports the missing
  device as a typed BackendFailure.
* The shared replay (replay.cuh) compiles with plain g++, as the other shared headers do, and the new code passes the
  launch and ownership source checks."""
import os
import re
import subprocess

import pytest

import test_device_ownership as own
import test_launch_sites as ls
from conftest import ROOT
from taiga_b200 import lib

NEW = {"tb_dev_verify_batch_vk": "tb_verify_batch_vk", "tb_dev_batch_verifier_add": "tb_batch_verifier_add"}


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def test_declarations_match_the_binding_and_the_host_versions():
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "taiga_b200.h")).read(), flags=re.S)
    for name, host in NEW.items():
        m = re.search(r"\btb_status\s+%s\s*\(([^;]*)\);" % name, hdr)
        assert m, name
        params = [p for p in m.group(1).replace("\n", " ").split(",") if p.strip()]
        assert len(params) == len(lib._SIGS[name][1]), (name, params)
        assert lib._SIGS[name] == lib._SIGS[host], name


def test_null_arguments_are_refused_without_a_device():
    so = lib.load()
    assert so.tb_dev_verify_batch_vk(None, None, 1, None, None, None, 0, 0, None) == lib.TB_ERR_INVALID
    assert so.tb_dev_batch_verifier_add(None, None, None, 1, None, None, None, 0, 0) == lib.TB_ERR_INVALID


CPP = r"""
#include <cstdio>
#include "taiga_b200.hpp"
using namespace taiga_b200;
int main() {
  try {
    Context ctx(0);
    std::vector<uint8_t> g(64 * 2, 0);
    Params params(ctx, 1, g.data(), g.data(), PointBytes{}, PointBytes{});
    ConstraintSystem cs;
    VerifyingKey vk(params, cs, {}, {});
    vk.verify_batch_device(1, nullptr, {}, nullptr, 32, nullptr);
    BatchVerifier bv(params, std::array<uint8_t, 32>{});
    bv.add_proofs_device(vk, 1, nullptr, {}, nullptr, 32);
    std::printf("verdict %d\n", bv.finalize() ? 1 : 0);
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "%s (status %d): %s\n", e.kind(), e.status(), e.what());
    return 1;
  }
}
"""


def test_cpp_device_overloads_build_and_fail_loudly_without_gpu(tmp_path):
    src = tmp_path / "dev.cpp"
    src.write_text(CPP)
    exe = str(tmp_path / "dev")
    libdir = os.path.dirname(lib.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-L", libdir, "-ltaiga_b200", "-Wl,-rpath," + libdir, "-o", exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    if not _no_gpu():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "BackendFailure" in r.stderr and "status 2" in r.stderr, r.stdout + r.stderr


def test_replay_header_compiles_with_plain_gxx(tmp_path):
    src = tmp_path / "replay_host.cpp"
    src.write_text('#include "%s"\nint main() { tb::ReplayShape s{}; (void)s; return 0; }\n'
                   % os.path.join(ROOT, "taiga_b200", "csrc", "replay.cuh"))
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-c", str(src), "-o", str(tmp_path / "replay_host.o")],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr


def test_new_code_passes_the_source_checks():
    text = ls.sources()["verifier.cu"]
    assert "replay_kernel" in text and "replay_proof(" in text
    # one replay: the host loop and the kernel both call replay_proof, and the old host-only replay is gone
    assert text.count("replay_proof(") == 2 and "VTranscript" not in text and "EvalView" not in text
    assert "std::map" not in ls.sources()["replay.cuh"]
    ls.test_no_triple_chevron_launch()
    ls.test_launch_kernel_ex_only_in_helper()
    ls.test_launch_count_changed_only_in_helper()
    own.test_synchronous_allocation_only_in_owner()
    own.test_stream_ordered_allocation_only_in_context()
    own.test_streams_and_events_only_in_context()
    body = own.span("verifier.cu", "struct BatchVerifier {")
    bv = text[body[1]:body[2]]
    assert "DevMem<Fp> g;" in bv and "DevMem<Xyzz<Fq>> acc;" in bv and "DevMem<uint8_t> alive;" in bv and "DevBuf" not in bv
