"""The Tight-Inclusion narrow phase where its searches degenerate: tests/golden/ccd_regimes_golden.npz (tests/golden/gen_ccd_regimes_golden.py)
holds a soup of point-triangle and edge-edge stencils -- generic hits, impacts on a triangle's boundary, coplanar and grazing motion, exactly
and nearly parallel edges, degenerate primitives, zero relative motion, sizes 1e-4 .. 1e2, initial distances 0 and 1e-12 .. 1e-9, and
searches whose levels outgrow 184 and 4,096 boxes or end at the library's max_itr -- with mpmath references of the first time the exact
distance reaches a level.

Every search here uses the pair's own numerical error filter, err = ti_error of its four vertices at t = 0 and t = 1.

Bars, on every pair that finishes (CPU: the oracle; GPU: the device, which must also equal the oracle bit for bit).  Each coordinate of
F(t, u, v) is multilinear, so a box's co-domain (the hull of its 8 corner values) contains F on the whole box.
  conservative  a reported impact is no later than any time where the exact distance is <= the ms the search ended with (the ms = 0
                retry: 0), the witness of the reference: F there lies within ms of the origin in every coordinate, so every box holding
                that (t, u, v) contains the origin, and the search can only leave through a box that starts no later
  real miss     no impact at all: the distance stays above the pair's first ms on [0, max_t], by the same argument
  tight         a terminal exit (K1, K2, TOI_SKIP) returns t_lo of a box that contains the origin within err + ms and whose co-domain is
                at most `tolerance` wide per coordinate (conditions 1-3 of the library: width_tolerances bounds the variation of F over a
                box within the per-axis widths by tolerance), so at its corner (t_lo, u_lo, v_lo) every coordinate of F is within
                err_c + ms + tolerance of 0: the distance there is <= L = sqrt(3) (ms + max err + tolerance), plus the rounding of the
                corner evaluation (64 eps max|x|).  So toi >= the first time the distance reaches L (x 0.8 after the retry).
Pairs whose library-semantics search does not end within TRIP_CAP no_zero_toi trips and BOX_CAP boxes are a property of the library
(err of a pair that moves far is large enough to contain the origin at t = 0 for every t_max); they are listed in EXCLUDED and never run
on the device.
"""
import importlib.util
import os

import numpy as np
import pytest

import oracle as orc
from gpu_common import load_scene, own_context, scalar_bits
from ipc_b200 import mesh as M

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "ccd_regimes_golden.npz")
TOL = 1e-6
TRIP_CAP, BOX_CAP = 300, 1 << 23
# the library does not finish these within the caps: fast generic pairs (toi 1e-9, 3e-7, 1e-8, moved 1e3 .. 1e6 times their size) and
# initial distances 1e-12
EXCLUDED = {0, 1, 9, 48, 49}
# exits and no_zero_toi branches no finishing pair of the fixture takes (DESIGN §4)
UNCOVERED_EXITS = {"k2", "skip", "depth60"}
OLD_LEVEL_CAP = 4096  # the device's per-warp level buffers, which used to end a search that outgrew them


def gold():
    return dict(np.load(GOLD))


def soup_mesh(z):
    m = M.Mesh(z["V_rest"], z["T"])
    m.mu[:] = 0.0
    m.lam[:] = 0.0
    m.V = z["V"].copy()
    return m


def candidates(m, z):
    """per pair: (candidate as the narrow phase reads it, the four vertex ids in its order)"""
    sf = {frozenset(int(v) for v in f): i for i, f in enumerate(m.SF)}
    se = {frozenset(int(v) for v in e): i for i, e in enumerate(m.SFEdges)}
    sv = {int(v): i for i, v in enumerate(m.SVI)}
    out = []
    for k, kind in enumerate(z["kind"]):
        b = 4 * k
        if kind == 0:
            f = sf[frozenset((b + 1, b + 2, b + 3))]
            out.append(((-sv[b] - 1, f), [b] + [int(v) for v in m.SF[f]]))
        else:
            e1, e2 = se[frozenset((b, b + 1))], se[frozenset((b + 2, b + 3))]
            out.append(((e1, e2), [int(v) for v in m.SFEdges[e1]] + [int(v) for v in m.SFEdges[e2]]))
    return out


def pair_inputs(z, vs, kind):
    x0 = z["V"][vs]
    x1 = x0 + z["p"][vs]  # fl(x0 + p), as the narrow phase forms it
    evf, eee = orc.ti_error(np.ascontiguousarray(x0.T).ravel(), 4, z["p"][vs].ravel())
    return x0, x1, (evf if kind == 0 else eee)


def traces(z, m, level_cap=0):
    """{(k, max_t index): (r, toi, trace, err)} for every pair, library semantics unless level_cap > 0"""
    out = {}
    for k, (cand, vs) in enumerate(candidates(m, z)):
        kind = int(z["kind"][k])
        x0, x1, err = pair_inputs(z, vs, kind)
        for q, mt in enumerate(z["max_t"]):
            r, toi, tr = orc.ti_trace("vf" if kind == 0 else "ee", x0, x1, err, TOL, float(mt), TRIP_CAP, BOX_CAP, level_cap)
            out[(k, q)] = (r, toi, tr, err)
    return out


_cache = {}


def fixture_traces():
    if "t" not in _cache:
        z = gold()
        m = soup_mesh(z)
        _cache["t"] = (z, m, traces(z, m))
    return _cache["t"]


def gen_module():
    spec = importlib.util.spec_from_file_location("gen_ccd_regimes_golden", os.path.join(HERE, "golden", "gen_ccd_regimes_golden.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_generator_reproduces_the_inputs():
    """the stored inputs are what the generator builds, bit for bit (the mpmath references take minutes and are not recomputed here)"""
    g = gen_module()
    z = gold()
    V, Vr, P, T, kind, fam = g.soup(g.cases())
    for name, a in (("V", V), ("V_rest", Vr), ("p", P), ("T", T), ("kind", kind), ("family", fam)):
        assert np.array_equal(a, z[name]), name
    assert list(z["families"]) == list(g.FAMILIES) and np.array_equal(z["max_t"], np.array(g.MAX_T))


def test_excluded_pairs_are_the_ones_the_library_does_not_finish():
    z, m, tr = fixture_traces()
    unfinished = {k for (k, q), (r, toi, t, err) in tr.items() if t["unfinished"]}
    assert unfinished == EXCLUDED
    for (k, q), (r, toi, t, err) in tr.items():
        if k not in EXCLUDED:
            assert t["boxes"] <= BOX_CAP and sum(t["trips"]) <= TRIP_CAP


_refs = {}


def ref(z, m, k):
    """the pair's exact reference (gen_ccd_regimes_golden.Ref) in the vertex order the narrow phase reads"""
    if k not in _refs:
        cand, vs = candidates(m, z)[k]
        x0, x1, err = pair_inputs(z, vs, int(z["kind"][k]))
        _refs[k] = (gen_module().Ref(int(z["kind"][k]), x0, x1), np.abs(np.concatenate([x0, x1])).max())
    return _refs[k]


def check_bars(z, m, k, q, r, toi, t, err):
    """the bars of the module docstring for one result; returns which were asserted"""
    mt = float(z["max_t"][q])
    rf, xmax = ref(z, m, k)
    if r == -1:
        assert float(z["d0"][k]) == 0.0  # the zero-distance flag: the step becomes 0
        return set()
    if r == 0:
        ms0 = min(0.2 * float(z["d0"][k]), 1e-6)
        assert rf.dmin(mt) > ms0, (k, q)
        return {"miss"}
    done = set()
    assert 0.0 <= toi <= mt
    wit = rf.first(t["ms"])[1]
    if wit != float("inf"):
        assert toi <= wit, (k, q, toi, float(wit))
        done.add("conservative")
    if t["last_exit"] in ("k1", "k2", "skip"):
        L = np.sqrt(3.0) * (t["ms"] + float(np.max(err)) + t["tolerance"]) + 64 * np.finfo(float).eps * xmax
        t_lo = float(rf.first(L)[0])
        assert toi >= (0.8 if t["retry"] else 1.0) * t_lo, (k, q, toi, t_lo)
        done.add("tight")
    return done


def test_oracle_meets_the_bars():
    z, m, tr = fixture_traces()
    count = {}
    for (k, q), (r, toi, t, err) in tr.items():
        if k not in EXCLUDED:
            for b in check_bars(z, m, k, q, r, toi, t, err):
                count[b] = count.get(b, 0) + 1
    assert count["conservative"] >= 40 and count["tight"] >= 30 and count["miss"] >= 40, count


def test_every_search_shape_is_covered():
    z, m, tr = fixture_traces()
    live = [t for (k, q), (r, toi, t, err) in tr.items() if k not in EXCLUDED and r >= 0]
    exits = {e for t in live for e, n in t["exits"].items() if n}
    assert exits == {"exhausted", "k1", "max_itr"} and not exits & UNCOVERED_EXITS
    widths = [t["width"] for t in live]
    assert any(8 < w <= 184 for w in widths) and any(184 < w <= 4096 for w in widths) and any(w > 4096 for w in widths)
    # the tolerance branch of no_zero_toi; the t_max and ms branches are only taken by the excluded pairs
    assert any(t["trips"][2] for t in live) and not any(t["trips"][0] or t["trips"][1] for t in live)
    assert any(t["retry"] for t in live)  # the ms = 0 retry (with a hit)
    fams = {str(z["families"][z["family"][k]]) for (k, q) in tr if k not in EXCLUDED}
    assert fams == set(str(f) for f in z["families"])


def test_old_level_cap_rule_spins_where_the_library_stops():
    """The parallel-edge pair (two edges 1e-3 apart closing at 2e-3 per unit step): the library ends at max_itr with toi 0.46875, one level
    about 2^17 boxes wide.  Ending a search with the level's estimate when a level outgrows 4,096 boxes returns toi = 0 before the first
    box is split in t, and the no_zero_toi loop then shrinks t_max without end -- what the device did before it continued such searches in
    an overflow arena."""
    z, m, tr = fixture_traces()
    k = next(k for k in range(len(z["kind"])) if str(z["families"][z["family"][k]]) == "parallel")
    r, toi, t, err = tr[(k, 0)]
    assert r == 1 and toi == 0.46875 and t["last_exit"] == "max_itr" and t["width"] > OLD_LEVEL_CAP and t["early_outs"] == 1
    cand, vs = candidates(m, z)[k]
    x0, x1, err = pair_inputs(z, vs, 1)
    r2, toi2, t2 = orc.ti_trace("ee", x0, x1, err, TOL, 1.0, 200, BOX_CAP, OLD_LEVEL_CAP)
    assert t2["unfinished"] and t2["exits"]["level_cap"] == 201 and t2["trips"] == [200, 0, 0] and t2["t_max"] < 1e-8


# ---- GPU ------------------------------------------------------------------------------------------------------------------------------------
def expected(r, toi, mt):
    return 0.0 if r < 0 else (toi if r == 1 else mt)


def bounded(tr, keys):
    """the pairs a launch may hold: every one ends within the caps under the library's semantics, which the device implements"""
    for key in keys:
        t = tr[key][2]
        assert not t["unfinished"] and t["boxes"] <= BOX_CAP and sum(t["trips"]) <= TRIP_CAP, key


@pytest.fixture
def own_ctx():
    """a context of its own: the early-outs these searches take add to the warning count that the next fetch_iteration of the same
    context reports, and the other tests' contexts must not see them"""
    with own_context() as ctx:
        yield ctx


@pytest.mark.gpu
def test_each_pair_alone_matches_the_oracle(own_ctx):
    ctx = own_ctx
    z, m, tr = fixture_traces()
    load_scene(ctx, m)
    p = z["p"].ravel()
    mm0, pe0 = np.empty((0, 4), dtype=np.int32), np.empty((0, 2), dtype=np.int32)
    cands = candidates(m, z)
    run = [k for k in range(len(cands)) if k not in EXCLUDED]
    bounded(tr, [(k, q) for k in run for q in range(len(z["max_t"]))])
    s = orc.Surf(m)
    bad = []
    try:
        for k in run:
            cand = np.array([cands[k][0]], dtype=np.int32)
            ctx.set_constraint_set(mm0, mm0, pe0, cand)
            for q, mt in enumerate(z["max_t"]):
                r, toi, t, err = tr[(k, q)]
                want = expected(r, toi, float(mt))
                a_ref, _ = orc.ccd_partial(s, p, cand, TOL, err, err, float(mt))
                assert scalar_bits(a_ref) == scalar_bits(want), (k, q)  # the traced pair is the pair the narrow phase reads
                for budget in (-1, 0, 1 << 40):
                    ctx.ccd_debug_thread_budget(budget)
                    a = ctx.ccd_partial(p, TOL, err, err, float(mt))
                    warn = ctx.ccd_stats()[2]
                    if scalar_bits(a) != scalar_bits(want) or warn != t["early_outs"]:
                        bad.append((k, q, budget, a, want, warn, t["early_outs"]))
    finally:
        ctx.ccd_debug_thread_budget(-1)
    assert not bad, bad


@pytest.mark.gpu
def test_whole_soup_in_one_call(own_ctx):
    """all pairs in one candidate list with one err: the minimum over the pairs, twice, at each budget"""
    ctx = own_ctx
    z, m, tr = fixture_traces()
    load_scene(ctx, m)
    p = z["p"].ravel()
    cands = candidates(m, z)
    err = np.full(3, 1e-13)
    keep, best = [], {}
    for k in range(len(cands)):
        if k in EXCLUDED:
            continue
        x0, x1, _ = pair_inputs(z, cands[k][1], int(z["kind"][k]))
        res = [orc.ti_trace("vf" if z["kind"][k] == 0 else "ee", x0, x1, err, TOL, float(mt), TRIP_CAP, BOX_CAP) for mt in z["max_t"]]
        if any(t["unfinished"] for r, toi, t in res):
            continue  # checked on the CPU: never launched
        keep.append(k)
        for q, (r, toi, t) in enumerate(res):
            best[q] = min(best.get(q, float(z["max_t"][q])), expected(r, toi, float(z["max_t"][q])))
    assert len(keep) >= 40
    cand = np.array([cands[k][0] for k in keep], dtype=np.int32)
    mm0, pe0 = np.empty((0, 4), dtype=np.int32), np.empty((0, 2), dtype=np.int32)
    ctx.set_constraint_set(mm0, mm0, pe0, cand)
    s = orc.Surf(m)
    try:
        for q, mt in enumerate(z["max_t"]):
            a_ref, _ = orc.ccd_partial(s, p, cand, TOL, err, err, float(mt), nthreads=8)
            assert scalar_bits(a_ref) == scalar_bits(best[q])
            for budget in (-1, 0, 1 << 40):
                ctx.ccd_debug_thread_budget(budget)
                for _ in range(2):
                    assert scalar_bits(ctx.ccd_partial(p, TOL, err, err, float(mt))) == scalar_bits(a_ref), (q, budget)
    finally:
        ctx.ccd_debug_thread_budget(-1)
