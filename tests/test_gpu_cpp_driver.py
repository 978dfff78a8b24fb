"""A C++ program (tests/cpp/abi_driver.cpp), not Python, drives the C ABI end to end -- the position the reference-side adapters are in.
The test writes a scene file, builds and runs the driver, and compares what it wrote back with the oracle."""
import os
import subprocess

import numpy as np
import pytest

import oracle as orc
from gpu_common import rel, scalar_bits
from ipc_b200 import scenes
from stagecheck import contact_pattern_pairs

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "abi_driver.cpp")


def build_driver(tmp):
    exe = os.path.join(tmp, "abi_driver")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-Wextra", "-I", os.path.join(ROOT, "include"), SRC, "-L", os.path.join(ROOT, "ipc_b200"), "-lipcgpu",
                           "-Wl,-rpath," + os.path.join(ROOT, "ipc_b200"), "-o", exe])
    return exe


def test_header_is_plain_c_and_driver_links(tmp_path):
    """CPU-side: include/ipcgpu.h compiles as C99 (a cgo / JNI / ctypes binder can consume it) and the C++ driver links against the library"""
    c = tmp_path / "hdr.c"
    c.write_text('#include "ipcgpu.h"\nint main(void) { ipcgpu_iteration it; (void)it; return IPCGPU_OK; }\n')
    subprocess.check_call(["gcc", "-std=c99", "-Wall", "-Wextra", "-pedantic", "-fsyntax-only", "-I", os.path.join(ROOT, "include"), str(c)])
    assert os.path.exists(build_driver(str(tmp_path)))


@pytest.mark.gpu
def test_cpp_driver_matches_oracle(tmp_path):
    m, info = scenes.ball_pile(4, res=8, seed=5, height=4)
    dHat, p, kappa, dt2, tol = info["dHat"], info["p"], 1e8, 0.025 ** 2, 1e-6
    h = m.avgEdgeLen / 3
    s, o = orc.Surf(m), orc.Elastic(m)
    mm, pa, pe, cand = s.constraint_set(dHat, nthreads=8)
    ia, ja = m.csr_pattern(1, extra_pairs=contact_pattern_pairs(m, mm, pa, pe))
    scene, out = str(tmp_path / "scene.bin"), str(tmp_path / "out.bin")
    with open(scene, "wb") as f:
        f.write(np.array([m.nV, m.nT, len(m.SVI), len(m.SFEdges), len(m.SF), ja.size, m.energy, 0], dtype=np.int32).tobytes())
        f.write(np.array([dHat, kappa, dt2, h, tol, 0.0]).tobytes())
        for arr, dt in ((m.V_rest_soa, np.float64), (m.V_soa, np.float64), (p, np.float64), (m.T_soa, np.int32), (m.restTriInv, np.float64), (m.vol, np.float64),
                        (m.mu, np.float64), (m.lam, np.float64), (m.mass, np.float64), (m.SVI, np.int32), (m.SFEdges, np.int32), (m.SF_soa, np.int32),
                        (ia, np.int32), (ja, np.int32)):
            f.write(np.ascontiguousarray(arr, dtype=dt).tobytes())
    exe = build_driver(str(tmp_path))
    r = subprocess.run([exe, scene, out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "abi_driver ok" in r.stdout, r.stdout + r.stderr
    raw = open(out, "rb").read()
    ints = np.frombuffer(raw, dtype=np.int32, count=8)
    dbl = np.frombuffer(raw, dtype=np.float64, count=12, offset=32)
    off = 32 + 96
    g = np.frombuffer(raw, dtype=np.float64, count=3 * m.nV, offset=off); off += 24 * m.nV
    a = np.frombuffer(raw, dtype=np.float64, count=ja.size, offset=off); off += 8 * ja.size
    g2 = np.frombuffer(raw, dtype=np.float64, count=3 * m.nV, offset=off); off += 24 * m.nV
    a2 = np.frombuffer(raw, dtype=np.float64, count=ja.size, offset=off)
    # oracle
    E_el, E_b = o.energy(dt2)[0], s.barrier_energy(mm, pa, pe, dHat, kappa)[0]
    g_ref = s.barrier_gradient(mm, pa, pe, dHat, kappa, g=o.gradient(dt2, 1))
    a_ref = o.hessian_csr(dt2, ia, ja, 1, 1, 1)
    a_ref[np.asarray(ia[:-1], dtype=np.int64) - 1] += np.repeat(m.mass, 3)
    a_ref = s.barrier_hessian_csr(mm, pa, pe, dHat, kappa, ia, ja, 1, 1, a=a_ref)
    evf, eee = orc.ti_error(s.V, m.nV, None)
    al0, _ = o.inversion_step(p, 0.2, 1.0)
    al1, _ = orc.ccd_partial(s, p, cand, tol, evf, eee, al0, 8)
    gr, ag = orc.grid_swept(s, p, al1, h)
    al2, _, npairs = orc.ccd_full(s, p, gr, ag, tol, evf, eee, ag, 8)
    assert tuple(ints[:3]) == (len(mm), len(pa), len(cand)) and ints[3] == npairs == ints[7]
    assert ints[4] == 0 and ints[5] == 1 and ints[6] == 0  # no inverted tet, intersection free, status OK
    assert abs(dbl[0] - E_el) <= 1e-10 * abs(E_el) and abs(dbl[1] - E_b) <= 1e-10 * abs(E_b)
    assert abs(dbl[5] - E_el) <= 1e-10 * abs(E_el) and abs(dbl[6] - E_b) <= 1e-10 * abs(E_b)
    assert abs(dbl[2] - al0) <= 1e-9 * al0 and scalar_bits(dbl[3]) == scalar_bits(al1) and scalar_bits(dbl[4]) == scalar_bits(al2)
    assert scalar_bits(dbl[8]) == scalar_bits(al1) and scalar_bits(dbl[9]) == scalar_bits(al2) and scalar_bits(dbl[10]) == scalar_bits(al2)
    for gg, aa in ((g, a), (g2, a2)):
        assert rel(gg, g_ref) <= 1e-10 and rel(aa, a_ref) <= 1e-9
