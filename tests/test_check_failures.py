"""CPU: circuits_random.failures, the list of every failure in the order tb_check_batch reports them, starts with what
circuits_random.satisfied names, on honest witnesses and on every soundness_cases violation; the C++ header's check_batch
compiles."""
import os
import subprocess

import pytest

import soundness_cases as sc
from conftest import ROOT
from taiga_b200 import circuits_mini as cm
from taiga_b200 import circuits_random as cr

SHAPES = [("boundary", name) for name, _ in cr.BOUNDARY] + [("seed", s) for s in range(30)]


def _shape(kind, arg):
    return cr.boundary(arg) if kind == "boundary" else cr.random_shape(arg)


@pytest.mark.parametrize("kind,arg", SHAPES, ids=["%s-%s" % s for s in SHAPES])
def test_first_failure_is_satisfied(kind, arg):
    kd, make = _shape(kind, arg)
    assert next(cr.failures(kd, make(3)), None) is None
    cases = sc.violations(kd, make, 5)
    assert cases
    for label, asg in cases:
        assert next(cr.failures(kd, asg), None) == cr.satisfied(kd, asg), label


@pytest.mark.parametrize("lookups,wide", [(2, False), (0, False), (2, True)])
def test_mini_circuits_have_no_failures(lookups, wide):
    kd, make = cm.standard_plonk(k=7 if wide else 6, n_lookups=lookups, wide=wide)
    assert list(cr.failures(kd, make(4))) == []


def test_failures_lists_every_broken_cell():
    """Two broken gate outputs and a broken lookup: all of them are listed, gates before lookups."""
    kd, make = cr.boundary("deg6_lookup")
    bad = [asg for label, asg in sc.violations(kd, make, 5) if label in ("gate0-out-first", "lookup0")]
    asg = bad[0]
    lk = bad[1]
    for c, col in enumerate(lk.advice):
        for row, v in col.items():
            if make(5).advice[c].get(row) != v:
                asg.advice[c][row] = v
    got = list(cr.failures(kd, asg))
    assert got[0] == cr.satisfied(kd, asg) and got[0].startswith("gate ")
    assert any(m.startswith("lookup 0: ") for m in got)
    kinds = [m.split()[0] for m in got]
    assert kinds == sorted(kinds, key=["gate", "lookup", "copy"].index)


def test_cpp_check_batch_compiles(tmp_path):
    src = tmp_path / "check.cpp"
    src.write_text('#include "taiga_b200.hpp"\n'
                   'int main() {\n'
                   '  using namespace taiga_b200;\n'
                   '  auto fn = &Proof::check_batch;\n'
                   '  CheckResult r; VerifyFailure f{VerifyFailure::Gate, 0, 0, 0, 0}; r.failures.push_back(f);\n'
                   '  return (fn != nullptr && !r.passed()) ? 0 : 1;\n'
                   '}\n')
    r = subprocess.run(["g++", "-std=c++17", "-Wall", "-Werror", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr
