"""CPU checks of the step-control feature: the oracle drivers of tests/test_gpu_step_control.py reach every loop of the line search on its
scenes with every energy comparison decided by a clear margin, and the ctypes mirrors of the new C structs match the compiler's layout."""
import ctypes as C
import os
import subprocess

import pytest

import test_gpu_step_control as T
from ipc_b200 import lib as L

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_oracle_line_search_reaches_every_loop():
    seen = [0, 0, 0, 0]
    rebuilt = friction = False
    for name, make in T.SCENES.items():
        sc = make()
        T.orc_lag(sc)
        r = T.oracle_line_search(sc, 1.0)
        assert r["status"] == 0 and not r["stopped"] and r["alpha"] > 0.0, name
        assert min(r["margins"]) > T.MARGIN, (name, r["margins"])  # no decision can flip on a summation-order difference
        seen = [a + b for a, b in zip(seen, r["counts"])]
        rebuilt |= r["rebuilt"]
        friction |= sc.fric is not None and len(sc.lag[0]) > 0
    assert all(seen) and rebuilt and friction, (seen, rebuilt, friction)


def test_oracle_line_search_refusals():
    sc = T.scene_intersection()
    assert T.oracle_line_search(sc, 0.0)["status"] == L.ERR_LINE_SEARCH
    sc.m.V[sc.m.nV // 2:, 2] -= 0.4  # the entry state intersects: no step helps
    r = T.oracle_line_search(sc, 1.0)
    assert r["status"] == L.ERR_LINE_SEARCH and r["alpha"] == 0.0


def test_ctypes_structs_match_the_header(tmp_path):
    src = tmp_path / "layout.cpp"
    fields = {"ipcgpu_line_search_terms": [f[0] for f in L.LineSearchTerms._fields_], "ipcgpu_step_control": [f[0] for f in L.StepControl._fields_]}
    lines = ['#include "ipcgpu.h"', "#include <cstddef>", "#include <cstdio>", "int main() {"]
    for s, fs in fields.items():
        lines.append(f'std::printf("%zu\\n", sizeof({s}));')
        lines += [f'std::printf("%zu\\n", offsetof({s}, {f}));' for f in fs]
    lines.append("return 0; }")
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    try:
        subprocess.check_call(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)])
    except FileNotFoundError:
        pytest.skip("no C++ compiler")
    got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
    want = []
    for cls in (L.LineSearchTerms, L.StepControl):
        want.append(C.sizeof(cls))
        want += [getattr(cls, f[0]).offset for f in cls._fields_]
    assert got == want


def test_new_symbols_exported():
    lib = L.load()
    for n in ("ipcgpu_ccd_cfl_ti", "ipcgpu_line_search", "ipcgpu_step_control_info"):
        assert hasattr(lib, n) and n in L.SIGNATURES
