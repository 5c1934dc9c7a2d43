"""CPU: proving into device memory (tb_dev_prove_batch) without a device.

* The entry point is declared in the header with the signature lib._SIGS binds, and takes every argument of
  tb_prove_batch with the same type (a byte pointer there is a void pointer here), then d_status_out.
* A null context is refused without touching a device.
* A C++ program that uses Proof::create_batch_device compiles with g++ -Wall -Werror and reports the missing device as a
  typed BackendFailure.
* prove_emit_kernel passes the launch and ownership source checks, require_device_memory exists once for the prover and
  the verifier, and prover.cu cross-compiles for sm_90a with no spill in prove_emit_kernel."""
import os
import re
import shutil
import subprocess

import pytest

import test_device_ownership as own
import test_launch_sites as ls
from conftest import ROOT
from taiga_b200 import lib

CSRC = os.path.join(ROOT, "taiga_b200", "csrc")


def _no_gpu():
    import torch
    return not torch.cuda.is_available()


def _params(name):
    """[(type, name)] of the declaration of `name` in the header"""
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "taiga_b200.h")).read(), flags=re.S)
    m = re.search(r"\btb_status\s+%s\s*\(([^;]*)\);" % name, hdr)
    assert m, name
    out = []
    for p in m.group(1).replace("\n", " ").split(","):
        p = " ".join(p.replace("*", " * ").split())
        t, n = p.rsplit(" ", 1)
        n = n.split("[")[0]
        out.append((t.replace(" *", "*"), n))
    return out


def test_declaration_matches_the_binding_and_the_host_version():
    dev, host = _params("tb_dev_prove_batch"), _params("tb_prove_batch")
    assert len(dev) == len(lib._SIGS["tb_dev_prove_batch"][1]) == len(host) + 1
    assert lib._SIGS["tb_dev_prove_batch"][0] == lib._SIGS["tb_prove_batch"][0]
    assert lib._SIGS["tb_dev_prove_batch"][1][:len(host)] == lib._SIGS["tb_prove_batch"][1]
    by_name = dict((n, t) for t, n in dev)
    for t, n in host:
        got = by_name.get(n, by_name.get("d_" + n))
        assert got is not None, n
        assert got == t.replace("uint8_t*", "void*") or got == t, (n, t, got)
    assert dev[-1] == ("uint32_t*", "d_status_out")
    assert (lib.TB_PROVED, lib.TB_PROVE_INTERNAL) == (0, 0xFFFFFFFF)


def test_null_arguments_are_refused_without_a_device():
    so = lib.load()
    assert so.tb_dev_prove_batch(None, None, 1, None, None, None, None, 0, None, 0, None) == lib.TB_ERR_INVALID


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
    ProvingKey pk(params, cs, nullptr, nullptr);
    Proof::create_batch_device(pk, params, 1, nullptr, nullptr, {}, std::array<uint8_t, 32>{}, 0, nullptr, pk.proof_len(), nullptr);
    std::printf("enqueued\n");
    return 0;
  } catch (const Error& e) {
    std::fprintf(stderr, "%s (status %d): %s\n", e.kind(), e.status(), e.what());
    return 1;
  }
}
"""


def test_cpp_create_batch_device_builds_and_fails_loudly_without_gpu(tmp_path):
    src = tmp_path / "dev_prove.cpp"
    src.write_text(CPP)
    exe = str(tmp_path / "dev_prove")
    libdir = os.path.dirname(lib.LIB_PATH)
    r = subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src),
                        "-L", libdir, "-ltaiga_b200", "-Wl,-rpath," + libdir, "-o", exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
    if not _no_gpu():
        pytest.skip("GPU present: the no-device path cannot be exercised")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert r.returncode == 1 and "BackendFailure" in r.stderr and "status 2" in r.stderr, r.stdout + r.stderr


def test_new_code_passes_the_source_checks():
    src = ls.sources()
    prover = src["prover.cu"]
    assert "__global__ void prove_emit_kernel(" in prover
    assert len(re.findall(r"\blaunch\(ctx, prove_emit_kernel,", prover)) == 1
    # one copy of the device-memory check, shared by the prover and the verifier
    defs = [(f, m.start()) for f, t in src.items() for m in re.finditer(r"\bvoid require_device_memory\(", t)]
    assert [f for f, _ in defs] == ["common.cuh"], defs
    assert "require_device_memory(ctx->c, {d_advice, d_proofs_out, d_status_out" in prover
    ls.test_no_triple_chevron_launch()
    ls.test_launch_kernel_ex_only_in_helper()
    ls.test_launch_count_changed_only_in_helper()
    own.test_synchronous_allocation_only_in_owner()
    own.test_stream_ordered_allocation_only_in_context()
    own.test_streams_and_events_only_in_context()
    # the workspace's mark of its last device call: kept with the workspace, checked before one is released
    ws = src["circuit.cuh"]
    assert "Ctx::Event idle;" in ws and "idle.done()" in ws and "idle.wait()" in ws


def test_prover_cross_compiles_without_spills_in_the_emit_kernel(tmp_path):
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    if not os.path.exists(nvcc) and not shutil.which("nvcc"):
        pytest.skip("no CUDA toolkit")
    nvcc = nvcc if os.path.exists(nvcc) else shutil.which("nvcc")
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                        "--expt-relaxed-constexpr", "-Xptxas", "-v", "-c", os.path.join(CSRC, "prover.cu"), "-o", str(tmp_path / "prover.o")],
                       capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stderr[-4000:]
    log = r.stderr + r.stdout
    at = log.index("Function properties for _ZN2tb17prove_emit_kernel")
    m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log[at:])
    assert m and m.groups() == ("0", "0", "0"), log[at:at + 300]
