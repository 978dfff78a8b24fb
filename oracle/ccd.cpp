/*
 * ccd.cpp -- CPU ORACLE (test infrastructure only; see oracle.h header).
 *
 * (1) The reference's swept spatial-hash geometry (src/Utils/SpatialHash.hpp:589-640, :841-845) and the CCD drivers
 *     SelfCollisionHandler::largestFeasibleStepSize_TightInclusion (src/CollisionObject/SelfCollisionHandler.cpp:690-866)
 *     and largestFeasibleStepSize_CCD_TightInclusion (:1370-1630), with the canonical semantics of SURVEY 8(a) row 10:
 *     every pair uses max_t = alpha on entry, the result is the minimum over pairs (the reference's shared stepSize is racy).
 * (2) Tight-Inclusion itself.  *** PARITY UNPINNED ***: the arithmetic lives in the un-vendored dependency
 *     CCD-Wrapper@23907da -> Continuous-Collision-Detection/Tight-Inclusion (inclusion_ccd::vertexFaceCCD_double /
 *     edgeEdgeCCD_double, CCD_TYPE=1, no_zero_toi=true), which is not under /root/reference and has no golden vectors in
 *     the reference's tests.  It is restated here from the published algorithm (Wang, Ferguson, Schneider, Jiang, Attene,
 *     Panozzo, "A Large-Scale Benchmark and an Inclusion-Based Algorithm for CCD", TOG 2021) and the call sites:
 *       - co-domain box of F(t,u,v) from its 8 corner values per coordinate, dyadic parameter boxes,
 *       - inclusion test against the [-(err+ms), +(err+ms)]^3 box, numerical error filter err = c * max(1,|x|max)^3,
 *       - per-parameter width tolerances tolerance / (3 * max displacement), breadth-first level order with earliest-t
 *         first, the three stopping conditions, the max_itr cut-off, the TOI_SKIP pruning, the no_zero_toi refinement.
 *     One deliberate specification choice: within a level, boxes are visited in ascending (t_lo, u_lo, v_lo) order.  The
 *     library's priority queue leaves ties between equal t_lo unspecified; a total order makes the result reproducible
 *     and is what the CUDA kernel implements, so "bit-exact" means GPU == this file.
 * All box arithmetic is written so that CPU (-ffp-contract=off) and GPU (explicit round-to-nearest mul/add) agree bitwise.
 */
#include "oracle.h"
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <limits>
#include <atomic>
#include <cstdlib>
#include <vector>

namespace {

struct Dy { /* interval [n/2^k, (n+1)/2^k] */
    uint64_t n;
    int k;
};
struct Box3 {
    Dy t, u, v;
};
inline double lo_of(Dy a) { return (double)a.n * std::ldexp(1.0, -a.k); }
inline double hi_of(Dy a) { return (double)(a.n + 1) * std::ldexp(1.0, -a.k); }
inline double width_of(Dy a) { return std::ldexp(1.0, -a.k); }
/* lo(a) + lo(b) <= 1 exactly (sum_no_larger_1) */
inline bool sum_le_1(Dy a, Dy b)
{
    int k = std::max(a.k, b.k);
    unsigned __int128 s = ((unsigned __int128)a.n << (k - a.k)) + ((unsigned __int128)b.n << (k - b.k));
    return s <= ((unsigned __int128)1 << k);
}

/* F at the 8 corners of a box, one coordinate.  x0/x1: 4 vertices (12 doubles) at t=0 / t=1.
 * VF: vertices (p, t0, t1, t2): F = p(t) - (t0(t) + u (t1(t)-t0(t)) + v (t2(t)-t0(t)))
 * EE: vertices (a0, a1, b0, b1): F = (a0(t) + u (a1(t)-a0(t))) - (b0(t) + v (b1(t)-b0(t))) */
inline void corner_values(bool vf, const double* x0, const double* x1, int c, const Box3& b, double out[8])
{
    const double tv[2] = { lo_of(b.t), hi_of(b.t) }, uv[2] = { lo_of(b.u), hi_of(b.u) }, vv[2] = { lo_of(b.v), hi_of(b.v) };
    int q = 0;
    for (int i = 0; i < 2; ++i) {
        double p[4];
        for (int k = 0; k < 4; ++k) p[k] = (x1[3 * k + c] - x0[3 * k + c]) * tv[i] + x0[3 * k + c];
        for (int j = 0; j < 2; ++j)
            for (int l = 0; l < 2; ++l) {
                if (vf) {
                    double pt = ((p[2] - p[1]) * uv[j] + (p[3] - p[1]) * vv[l]) + p[1];
                    out[q++] = p[0] - pt;
                }
                else {
                    double pa = (p[1] - p[0]) * uv[j] + p[0];
                    double pb = (p[3] - p[2]) * vv[l] + p[2];
                    out[q++] = pa - pb;
                }
            }
    }
}

/* Origin_in_function_bounding_box_double_vector_return_tolerance */
inline bool origin_in_box(bool vf, const double* x0, const double* x1, const Box3& b, const double err[3], double ms, bool& box_in, double true_tol[3])
{
    box_in = true;
    for (int c = 0; c < 3; ++c) {
        double v[8];
        corner_values(vf, x0, x1, c, b, v);
        double mn = v[0], mx = v[0];
        for (int q = 1; q < 8; ++q) { mn = std::min(mn, v[q]); mx = std::max(mx, v[q]); }
        true_tol[c] = mx - mn;
        const double eps = err[c] + ms;
        if (mn > eps || mx < -eps) return false;
        if (!(mn >= -eps && mx <= eps)) box_in = false;
    }
    return true;
}

inline double linf3(const double* a, const double* b) { return std::max(std::max(std::fabs(a[0] - b[0]), std::fabs(a[1] - b[1])), std::fabs(a[2] - b[2])); }

/* compute_face_vertex_tolerance_3d_new / compute_edge_edge_tolerance_new */
void width_tolerances(bool vf, const double* x0, const double* x1, double tolerance, double tol[3])
{
    double ps[4][3], pe[4][3]; /* p000, p001, p011, p010 */
    for (int side = 0; side < 2; ++side) {
        const double* x = side ? x1 : x0;
        double(*p)[3] = side ? pe : ps;
        for (int c = 0; c < 3; ++c) {
            if (vf) {
                p[0][c] = x[c] - x[3 + c];                           /* v - f0 */
                p[1][c] = x[c] - x[9 + c];                           /* v - f2 */
                p[2][c] = x[c] - (x[6 + c] + x[9 + c] - x[3 + c]);   /* v - (f1+f2-f0) */
                p[3][c] = x[c] - x[6 + c];                           /* v - f1 */
            }
            else {
                p[0][c] = x[c] - x[6 + c];     /* a0 - b0 */
                p[1][c] = x[c] - x[9 + c];     /* a0 - b1 */
                p[2][c] = x[3 + c] - x[9 + c]; /* a1 - b1 */
                p[3][c] = x[3 + c] - x[6 + c]; /* a1 - b0 */
            }
        }
    }
    double dl = 0, e0 = 0, e1 = 0;
    for (int q = 0; q < 4; ++q) dl = std::max(dl, linf3(pe[q], ps[q]));
    /* u direction: p000->p010, p001->p011 (both times) ; v direction: p000->p001, p010->p011 */
    e0 = std::max(std::max(linf3(ps[3], ps[0]), linf3(pe[3], pe[0])), std::max(linf3(pe[2], pe[1]), linf3(ps[2], ps[1])));
    e1 = std::max(std::max(linf3(ps[1], ps[0]), linf3(pe[1], pe[0])), std::max(linf3(pe[2], pe[3]), linf3(ps[2], ps[3])));
    tol[0] = tolerance / (3.0 * dl);
    tol[1] = tolerance / (3.0 * e0);
    tol[2] = tolerance / (3.0 * e1);
}

/* diagnostics for sizing the GPU passes (not part of the algorithm): histograms over root-finder calls of the boxes evaluated,
 * the widest level and the number of levels, in powers of two */
static std::atomic<long long> g_ti_hist[3][24];
struct TiStat {
    long long boxes = 0, width = 0, levels = 0;
    static int bin(long long v) { int b = 0; while (v > 1 && b < 23) { v >>= 1; ++b; } return b; }
    ~TiStat()
    {
        g_ti_hist[0][bin(boxes)].fetch_add(1, std::memory_order_relaxed);
        g_ti_hist[1][bin(width)].fetch_add(1, std::memory_order_relaxed);
        g_ti_hist[2][bin(levels)].fetch_add(1, std::memory_order_relaxed);
    }
};
extern "C" void orc_ti_stats(long long* out72, int reset)
{
    for (int a = 0; a < 3; ++a)
        for (int b = 0; b < 24; ++b) {
            out72[a * 24 + b] = g_ti_hist[a][b].load();
            if (reset) g_ti_hist[a][b].store(0);
        }
}

/* The library pops boxes of one level in ascending t_lo and leaves the order of boxes with EQUAL t_lo to its heap (unspecified).  The oracle
 * (and the GPU) fix it to ascending (u_lo, v_lo).  orc_ti_debug_tie_order(1) reverses that choice -- the opposite admissible order -- so that
 * tests can measure whether a result depends on it (tests/test_oracle_ccd.py::test_tie_order_of_equal_times_does_not_change_the_results). */
static std::atomic<int> g_tie_reversed{ 0 };
extern "C" void orc_ti_debug_tie_order(int reversed) { g_tie_reversed.store(reversed ? 1 : 0); }

/* orc_ti_debug_level_cap(n), n > 0: emulates a root finder whose level buffers hold n boxes and which, when the next level would outgrow
 * them, returns the per-level estimate of the current level (the estimate of the max_itr exit).  The CUDA narrow phase did this with
 * n = 4096 before it continued such searches in an overflow arena; 0 (the default) is the library, which has no such cap.  Kept so that
 * tests can show what that rule does to a search (tests/test_ccd_regimes.py). */
static std::atomic<long long> g_level_cap{ 0 };
extern "C" void orc_ti_debug_level_cap(long long n) { g_level_cap.store(n > 0 ? n : 0); }

/* How a search went (orc_ti_trace).  Exits of the root finder: */
enum TiExit { EXIT_EXHAUSTED = 0, EXIT_K1 = 1, EXIT_K2 = 2, EXIT_SKIP = 3, EXIT_MAX_ITR = 4, EXIT_DEPTH = 5, EXIT_LEVEL_CAP = 6, EXIT_UNFINISHED = 7 };
struct TiTrace {
    long long trip_cap, box_cap;   /* limits: no_zero_toi trips per ti_ccd call, boxes per trace */
    long long exits[8];            /* root-finder calls per exit */
    int last_exit;
    long long levels, width, boxes;
    long long trips[3];            /* no_zero_toi trips: t_max *= 0.9, ms *= 0.5, tolerance *= 0.1 */
    double ms, tolerance, t_max;   /* of the last root-finder call */
    int retry;                     /* pair_ccd ran its ms = 0 retry */
    int unfinished;
};
static thread_local TiTrace* g_trace = nullptr;

/* interval_root_finder_double_horizontal_tree with the canonical in-level order */
bool root_finder(bool vf, const double* x0, const double* x1, const double tol[3], double co_tol, double max_t, const double err[3], double ms,
    int max_itr, double& toi, double& out_tol)
{
    const bool check_t = (max_t != 1.0);
    std::vector<Box3> level(1), next;
    level[0] = { { 0, 0 }, { 0, 0 }, { 0, 0 } };
    double toi_skip = std::numeric_limits<double>::infinity();
    bool use_skip = false;
    long long refine = 0;
    double temp_toi = std::numeric_limits<double>::infinity(), temp_out_tol = co_tol;
    out_tol = co_tol;
    toi = std::numeric_limits<double>::infinity();
    bool overflow = false;
    int why = EXIT_MAX_ITR;
    TiTrace* tr = g_trace;
    const long long level_cap = g_level_cap.load(std::memory_order_relaxed);
    auto exit_as = [tr](int e) { if (tr) { tr->exits[e]++; tr->last_exit = e; } };
    TiStat stat;
    /* diagnostics only (sizing the GPU passes, never set by tests): ORC_TI_DIAG_PRUNE=<t> skips boxes that start at or after max(t, 1e-6), the
     * GPU's pruning rule against the running minimum in the limit of an instantly known final step */
    static const double diag_prune = [] { const char* e = std::getenv("ORC_TI_DIAG_PRUNE"); return e ? std::atof(e) : -1.0; }();
    while (!level.empty() && !overflow) {
        ++stat.levels;
        stat.width = std::max<long long>(stat.width, (long long)level.size());
        if (tr) {
            ++tr->levels;
            tr->width = std::max<long long>(tr->width, (long long)level.size());
        }
        const bool rev = g_tie_reversed.load(std::memory_order_relaxed) != 0;
        std::sort(level.begin(), level.end(), [rev](const Box3& a, const Box3& b) {
            double ta = lo_of(a.t), tb = lo_of(b.t);
            if (ta != tb) return ta < tb;
            double ua = lo_of(a.u), ub = lo_of(b.u);
            if (ua != ub) return rev ? ua > ub : ua < ub;
            return rev ? lo_of(a.v) > lo_of(b.v) : lo_of(a.v) < lo_of(b.v);
        });
        bool this_level_less_tol = true, find_level_root = false, origin_seen = false;
        next.clear();
        for (const Box3& cur : level) {
            const double t_lo = lo_of(cur.t);
            if (!(t_lo < toi_skip)) continue;
            if (diag_prune >= 0.0 && !(t_lo < std::max(diag_prune, 1e-6))) continue;
            ++refine;
            ++stat.boxes;
            if (tr && ++tr->boxes > tr->box_cap) {
                tr->unfinished = 1;
                exit_as(EXIT_UNFINISHED);
                toi = 0.0;
                return true;
            }
            bool box_in;
            double true_tol[3];
            if (!origin_in_box(vf, x0, x1, cur, err, ms, box_in, true_tol)) continue;
            const bool first_origin = !origin_seen;
            origin_seen = true;
            const double w[3] = { width_of(cur.t), width_of(cur.u), width_of(cur.v) };
            const bool tol_cond = true_tol[0] <= co_tol && true_tol[1] <= co_tol && true_tol[2] <= co_tol;
            const bool cond1 = w[0] <= tol[0] && w[1] <= tol[1] && w[2] <= tol[2];
            const bool cond2 = box_in && this_level_less_tol;
            if (!tol_cond) this_level_less_tol = false;
            const bool cond3 = this_level_less_tol;
            if (cond1 || cond2 || cond3) {
                exit_as(first_origin ? EXIT_K1 : EXIT_K2);
                toi = t_lo;
                return true;
            }
            if (max_itr > 0) {
                if (!find_level_root) {
                    temp_toi = t_lo;
                    temp_out_tol = std::max(std::max(std::max(true_tol[0], true_tol[1]), true_tol[2]), co_tol);
                    find_level_root = true;
                }
                if (refine > max_itr) {
                    overflow = true;
                    break;
                }
            }
            if (tol_cond || box_in) {
                if (t_lo < toi_skip) toi_skip = t_lo;
                use_skip = true;
                continue;
            }
            /* split the checked dimension with the largest width/tol ratio (ties: lowest index) */
            int split = -1;
            double best = -1.0;
            for (int i = 0; i < 3; ++i)
                if (w[i] > tol[i]) {
                    double r = w[i] / tol[i];
                    if (r > best) { best = r; split = i; }
                }
            Dy Box3::*mem = (split == 0) ? &Box3::t : (split == 1 ? &Box3::u : &Box3::v);
            const Dy parent = cur.*mem;
            if (parent.k >= 60) { /* bisection overflow */
                overflow = true;
                why = EXIT_DEPTH;
                break;
            }
            const Dy h1 = { parent.n * 2, parent.k + 1 }, h2 = { parent.n * 2 + 1, parent.k + 1 };
            for (int half = 0; half < 2; ++half) {
                const Dy h = half ? h2 : h1;
                bool keep = true;
                if (split == 0) { if (check_t) keep = !(hi_of(h) < 0.0 || lo_of(h) > max_t); }
                else if (vf) keep = (split == 1) ? sum_le_1(h, cur.v) : sum_le_1(h, cur.u);
                if (keep) {
                    Box3 c = cur;
                    c.*mem = h;
                    next.push_back(c);
                }
            }
        }
        if (!overflow && level_cap > 0 && (long long)next.size() > level_cap) {
            overflow = true;
            why = EXIT_LEVEL_CAP;
        }
        level.swap(next);
    }
    if (overflow) {
        exit_as(why);
        toi = temp_toi;
        out_tol = temp_out_tol;
        return true;
    }
    if (use_skip) {
        exit_as(EXIT_SKIP);
        toi = toi_skip;
        return true;
    }
    exit_as(EXIT_EXHAUSTED);
    return false;
}

/* vertexFaceCCD_double / edgeEdgeCCD_double with the no_zero_toi loop */
bool ti_ccd(bool vf, const double* x0, const double* x1, const double err[3], double ms, double tolerance, double t_max, int max_itr, bool no_zero_toi,
    double& toi, double& out_tol)
{
    double tolerance_in = tolerance, ms_in = ms;
    bool is_impacting = false, tmp = false;
    unsigned iter = 0;
    do {
        double tol[3];
        width_tolerances(vf, x0, x1, tolerance_in, tol);
        tmp = root_finder(vf, x0, x1, tol, tolerance_in, t_max, err, ms_in, max_itr, toi, out_tol);
        if (g_trace) {
            g_trace->ms = ms_in;
            g_trace->tolerance = tolerance_in;
            g_trace->t_max = t_max;
            if (g_trace->unfinished) break;
        }
        if (iter == 0) is_impacting = tmp;
        else toi = tmp ? toi : t_max;
        if (tmp && toi == 0 && no_zero_toi) {
            if (g_trace && g_trace->trips[0] + g_trace->trips[1] + g_trace->trips[2] >= g_trace->trip_cap) {
                g_trace->unfinished = 1;
                break;
            }
            const int branch = out_tol > tolerance_in ? 0 : (10 * tolerance_in < ms_in ? 1 : 2);
            if (branch == 0) t_max *= 0.9;
            else if (branch == 1) ms_in *= 0.5;
            else tolerance_in *= 0.1;
            if (g_trace) ++g_trace->trips[branch];
        }
        ++iter;
    } while (no_zero_toi && iter < 0x7fffffffu && tmp && toi == 0);
    return is_impacting;
}

inline void vert_of(const orc_surf* s, int v, double* out)
{
    out[0] = s->V[v];
    out[1] = s->V[(size_t)s->nV + v];
    out[2] = s->V[(size_t)2 * s->nV + v];
}
inline bool is_dbc(const orc_surf* s, int v) { return s->dbc && s->dbc[v] != 0; }
inline int codim(const orc_surf* s, int v) { return s->vCoDim ? s->vCoDim[v] : 3; }

int pair_ccd_x(bool vf, const double* x0, const double* x1, double tol, const double err[3], double max_t, double* toi_out);

/* one candidate: SelfCollisionHandler.cpp:725-790 (EE) / :795-861 (PT). returns -1 when d==0 (stepSize := 0) */
int pair_ccd(bool vf, const int v[4], const orc_surf* s, const double* p, double tol, const double err[3], double max_t, double* toi_out)
{
    double x0[12], x1[12];
    for (int k = 0; k < 4; ++k) {
        vert_of(s, v[k], x0 + 3 * k);
        for (int c = 0; c < 3; ++c) x1[3 * k + c] = x0[3 * k + c] + p[3 * (size_t)v[k] + c];
    }
    return pair_ccd_x(vf, x0, x1, tol, err, max_t, toi_out);
}

/* the same from the pair's coordinates (x1 = x0 + p already formed) */
int pair_ccd_x(bool vf, const double* x0, const double* x1, double tol, const double err[3], double max_t, double* toi_out)
{
    double d;
    if (vf) orc_point_tri_d(x0, &d);
    else orc_edge_edge_d(x0, &d);
    d = std::sqrt(d);
    if (d == 0) return -1;
    double toi, out_tol;
    bool hit = ti_ccd(vf, x0, x1, err, std::min(0.2 * d, 1e-6), tol, max_t, 1000000, true, toi, out_tol);
    if (hit && toi < 1e-6 && !(g_trace && g_trace->unfinished)) {
        if (g_trace) g_trace->retry = 1;
        hit = ti_ccd(vf, x0, x1, err, 0.0, tol, max_t, 1000000, true, toi, out_tol);
        if (hit) toi *= 0.8;
    }
    if (hit) {
        *toi_out = toi;
        return 1;
    }
    return 0;
}

} // namespace

extern "C" {

int orc_ti_vf(const double* x0, const double* x1, const double err[3], double ms, double tol, double max_t, int max_itr, int no_zero_toi, double* toi, double* out_tol)
{
    return ti_ccd(true, x0, x1, err, ms, tol, max_t, max_itr, no_zero_toi != 0, *toi, *out_tol) ? 1 : 0;
}
int orc_ti_ee(const double* x0, const double* x1, const double err[3], double ms, double tol, double max_t, int max_itr, int no_zero_toi, double* toi, double* out_tol)
{
    return ti_ccd(false, x0, x1, err, ms, tol, max_t, max_itr, no_zero_toi != 0, *toi, *out_tol) ? 1 : 0;
}

/* One pair as the narrow phase runs it (pair_ccd: ms = min(0.2 d, 1e-6), max_itr = 1e6, no_zero_toi, the ms = 0 retry), traced.
 * vf = 1: point-triangle (p, t0, t1, t2), 0: edge-edge (a0, a1, b0, b1); x1 = x0 + p as the caller formed it.  The search gives up once
 * a ti_ccd call takes trip_cap no_zero_toi trips or the pair evaluates box_cap boxes (out_i[9] = 1, "did not finish").
 * Returns what pair_ccd returns: -1 zero initial distance, 0 no impact, 1 impact (*toi set).
 * out_i[0..7]: root-finder calls per exit (exhausted, terminal K1, terminal K2, TOI_SKIP, max_itr, depth 60, level cap, unfinished);
 * out_i[8]: exit of the last call; [9] unfinished; [10] retry ran; [11] levels; [12] widest level; [13] boxes evaluated;
 * [14..16] no_zero_toi trips taking t_max *= 0.9, ms *= 0.5, tolerance *= 0.1.
 * out_d[0..2]: ms, tolerance and t_max of the last root-finder call. */
int orc_ti_trace(int vf, const double* x0, const double* x1, const double err[3], double tol, double max_t, long long trip_cap, long long box_cap, double* toi,
    long long* out_i, double* out_d)
{
    TiTrace tr{};
    tr.trip_cap = trip_cap;
    tr.box_cap = box_cap;
    tr.last_exit = -1;
    g_trace = &tr;
    *toi = std::numeric_limits<double>::quiet_NaN();
    const int r = pair_ccd_x(vf != 0, x0, x1, tol, err, max_t, toi);
    g_trace = nullptr;
    for (int e = 0; e < 8; ++e) out_i[e] = tr.exits[e];
    out_i[8] = tr.last_exit;
    out_i[9] = tr.unfinished;
    out_i[10] = tr.retry;
    out_i[11] = tr.levels;
    out_i[12] = tr.width;
    out_i[13] = tr.boxes;
    for (int b = 0; b < 3; ++b) out_i[14 + b] = tr.trips[b];
    out_d[0] = tr.ms;
    out_d[1] = tr.tolerance;
    out_d[2] = tr.t_max;
    return r;
}

/* CCDUtils.cpp:21-87: world bbox of V (and V+p), inflated to centre +- 10*radius*(1,1,1)/sqrt(3), then
 * Tight-Inclusion get_numerical_error(bbox corners, check_vf, using_minimum_separation = true) */
void orc_ti_error(const double* V, int nV, const double* p, double err_vf[3], double err_ee[3])
{
    double lo[3] = { 1e300, 1e300, 1e300 }, hi[3] = { -1e300, -1e300, -1e300 };
    for (int v = 0; v < nV; ++v)
        for (int c = 0; c < 3; ++c) {
            double x = V[(size_t)c * nV + v];
            lo[c] = std::min(lo[c], x); hi[c] = std::max(hi[c], x);
            if (p) {
                double y = x + p[3 * (size_t)v + c];
                lo[c] = std::min(lo[c], y); hi[c] = std::max(hi[c], y);
            }
        }
    double center[3], r2 = 0;
    for (int c = 0; c < 3; ++c) { center[c] = 0.5 * (lo[c] + hi[c]); r2 += (hi[c] - lo[c]) * (hi[c] - lo[c]); }
    double radius = 0.5 * std::sqrt(r2);
    double mx[3];
    for (int c = 0; c < 3; ++c) {
        double a = center[c] - 10.0 * radius / std::sqrt(3.0), b = center[c] + 10.0 * radius / std::sqrt(3.0);
        mx[c] = std::max(std::fabs(a), std::fabs(b));
        mx[c] = std::max(mx[c], 1.0);
    }
    const double eefilter = 7.105427357601002e-15, vffilter = 7.549516567451064e-15; /* with minimum separation */
    for (int c = 0; c < 3; ++c) {
        err_ee[c] = mx[c] * mx[c] * mx[c] * eefilter;
        err_vf[c] = mx[c] * mx[c] * mx[c] * vffilter;
    }
}

/* SpatialHash.hpp:589-640: swept grid geometry; alpha is divided by spanSize when spanSize > 1 */
void orc_grid_swept(const orc_surf* s, const double* p, double* alpha, double h, orc_grid* g)
{
    double pSize = 0;
    for (int i = 0; i < s->nSV; ++i) {
        int v = s->SVI[i];
        pSize += std::abs(p[3 * (size_t)v]);     /* three separate accumulations, in this order (SpatialHash.hpp:605-611): the sum is order-sensitive */
        pSize += std::abs(p[3 * (size_t)v + 1]);
        pSize += std::abs(p[3 * (size_t)v + 2]);
    }
    pSize /= (double)(s->nSV * 3);
    const double span = *alpha * pSize / h;
    if (span > 1) *alpha /= span;
    double lo[3] = { 1e300, 1e300, 1e300 }, hi[3] = { -1e300, -1e300, -1e300 };
    for (int v = 0; v < s->nV; ++v)
        for (int c = 0; c < 3; ++c) {
            double x = s->V[(size_t)c * s->nV + v];
            lo[c] = std::min(lo[c], x); hi[c] = std::max(hi[c], x);
        }
    for (int i = 0; i < s->nSV; ++i) {
        int v = s->SVI[i];
        for (int c = 0; c < 3; ++c) {
            double x = s->V[(size_t)c * s->nV + v] + *alpha * p[3 * (size_t)v + c];
            lo[c] = std::min(lo[c], x); hi[c] = std::max(hi[c], x);
        }
    }
    g->inv_h = 1.0 / h;
    double rmax = 0;
    bool bad = false;
    for (int c = 0; c < 3; ++c) {
        g->lo[c] = lo[c];
        g->count[c] = (int)std::ceil((hi[c] - lo[c]) * g->inv_h);
        rmax = std::max(rmax, hi[c] - lo[c]);
        if (g->count[c] <= 0) bad = true;
    }
    if (bad) {
        g->inv_h = 1.0 / (rmax * 1.01);
        g->count[0] = g->count[1] = g->count[2] = 1;
    }
}
void orc_grid_static(const orc_surf* s, double h, orc_grid* g)
{
    double a = 0.0;
    std::vector<double> zero((size_t)3 * s->nV, 0.0);
    orc_grid_swept(s, zero.data(), &a, h, g);
}

int orc_ccd_partial(const orc_surf* s, const double* p, const int* cand, int nCand, double tol, const double err_vf[3], const double err_ee[3], double* alpha, int nthreads)
{
    const double max_t = *alpha;
    double best = *alpha;
    int zero = 0;
#pragma omp parallel for num_threads(nthreads > 0 ? nthreads : 1) schedule(dynamic, 8) reduction(min : best) reduction(max : zero)
    for (int c = 0; c < nCand; ++c) {
        int v[4];
        bool vf = cand[2 * c] < 0;
        if (vf) {
            int svI = -cand[2 * c] - 1, sfI = cand[2 * c + 1];
            v[0] = s->SVI[svI]; v[1] = s->SF[sfI]; v[2] = s->SF[(size_t)s->nSF + sfI]; v[3] = s->SF[(size_t)2 * s->nSF + sfI];
        }
        else {
            v[0] = s->SE[2 * cand[2 * c]]; v[1] = s->SE[2 * cand[2 * c] + 1]; v[2] = s->SE[2 * cand[2 * c + 1]]; v[3] = s->SE[2 * cand[2 * c + 1] + 1];
        }
        double toi;
        int r = pair_ccd(vf, v, s, p, tol, vf ? err_vf : err_ee, max_t, &toi);
        if (r < 0) zero = 1;
        else if (r > 0 && toi < best) best = toi;
    }
    *alpha = zero ? 0.0 : best;
    return zero;
}

int orc_ccd_full(const orc_surf* s, const double* p, const orc_grid* g, double alpha_grid, double tol, const double err_vf[3], const double err_ee[3], double* alpha,
    long long* nPairs, int nthreads)
{
    /* per surface vertex: voxel index range of {x, x + alpha_grid p}  (SpatialHash.hpp:642-662) */
    std::vector<int> vmin((size_t)3 * s->nV, 0), vmax((size_t)3 * s->nV, 0);
    for (int i = 0; i < s->nSV; ++i) {
        int v = s->SVI[i];
        for (int c = 0; c < 3; ++c) {
            double x = s->V[(size_t)c * s->nV + v];
            double xt = x + alpha_grid * p[3 * (size_t)v + c];
            int a = (int)std::floor((x - g->lo[c]) * g->inv_h), b = (int)std::floor((xt - g->lo[c]) * g->inv_h);
            vmin[3 * (size_t)v + c] = std::min(a, b);
            vmax[3 * (size_t)v + c] = std::max(a, b);
        }
    }
    auto prim_range = [&](const int* vs, int n, int lo[3], int hi[3]) {
        for (int c = 0; c < 3; ++c) {
            lo[c] = vmin[3 * (size_t)vs[0] + c]; hi[c] = vmax[3 * (size_t)vs[0] + c];
            for (int k = 1; k < n; ++k) { lo[c] = std::min(lo[c], vmin[3 * (size_t)vs[k] + c]); hi[c] = std::max(hi[c], vmax[3 * (size_t)vs[k] + c]); }
        }
    };
    const double max_t = *alpha;
    double best = *alpha;
    int zero = 0;
    long long pairs = 0;
    std::vector<int> tlo((size_t)3 * s->nSF), thi((size_t)3 * s->nSF), elo((size_t)3 * s->nSE), ehi((size_t)3 * s->nSE);
    for (int f = 0; f < s->nSF; ++f) {
        int vs[3] = { s->SF[f], s->SF[(size_t)s->nSF + f], s->SF[(size_t)2 * s->nSF + f] };
        prim_range(vs, 3, &tlo[3 * (size_t)f], &thi[3 * (size_t)f]);
    }
    for (int e = 0; e < s->nSE; ++e) {
        int vs[2] = { s->SE[2 * e], s->SE[2 * e + 1] };
        prim_range(vs, 2, &elo[3 * (size_t)e], &ehi[3 * (size_t)e]);
    }
#pragma omp parallel for num_threads(nthreads > 0 ? nthreads : 1) schedule(dynamic, 8) reduction(min : best) reduction(max : zero) reduction(+ : pairs)
    for (int svI = 0; svI < s->nSV; ++svI) { /* :1385-1489 */
        int vI = s->SVI[svI];
        const int* plo = &vmin[3 * (size_t)vI];
        const int* phi = &vmax[3 * (size_t)vI];
        for (int f = 0; f < s->nSF; ++f) {
            const int* lo = &tlo[3 * (size_t)f];
            const int* hi = &thi[3 * (size_t)f];
            if (lo[0] > phi[0] || hi[0] < plo[0] || lo[1] > phi[1] || hi[1] < plo[1] || lo[2] > phi[2] || hi[2] < plo[2]) continue;
            int v[4] = { vI, s->SF[f], s->SF[(size_t)s->nSF + f], s->SF[(size_t)2 * s->nSF + f] };
            if (vI == v[1] || vI == v[2] || vI == v[3]) continue;
            if ((codim(s, vI) < 3 && codim(s, v[1]) < 3) || (is_dbc(s, vI) && is_dbc(s, v[1]) && is_dbc(s, v[2]) && is_dbc(s, v[3]))) continue;
            ++pairs;
            double toi;
            int r = pair_ccd(true, v, s, p, tol, err_vf, max_t, &toi);
            if (r < 0) zero = 1;
            else if (r > 0 && toi < best) best = toi;
        }
    }
#pragma omp parallel for num_threads(nthreads > 0 ? nthreads : 1) schedule(dynamic, 8) reduction(min : best) reduction(max : zero) reduction(+ : pairs)
    for (int eI = 0; eI < s->nSE; ++eI) { /* :1498-1614 + SpatialHash.hpp:803-832 */
        const int a0 = s->SE[2 * eI], a1 = s->SE[2 * eI + 1];
        double bi_lo[3], bi_hi[3];
        for (int c = 0; c < 3; ++c) {
            double x0 = s->V[(size_t)c * s->nV + a0], x1 = s->V[(size_t)c * s->nV + a1];
            double y0 = x0 + max_t * p[3 * (size_t)a0 + c], y1 = x1 + max_t * p[3 * (size_t)a1 + c];
            bi_hi[c] = std::max(std::max(x0, y0), std::max(x1, y1));
            bi_lo[c] = std::min(std::min(x0, y0), std::min(x1, y1));
        }
        for (int eJ = eI + 1; eJ < s->nSE; ++eJ) {
            const int* lo = &elo[3 * (size_t)eJ];
            const int* hi = &ehi[3 * (size_t)eJ];
            const int* qlo = &elo[3 * (size_t)eI];
            const int* qhi = &ehi[3 * (size_t)eI];
            if (lo[0] > qhi[0] || hi[0] < qlo[0] || lo[1] > qhi[1] || hi[1] < qlo[1] || lo[2] > qhi[2] || hi[2] < qlo[2]) continue;
            const int b0 = s->SE[2 * eJ], b1 = s->SE[2 * eJ + 1];
            bool sep = false;
            for (int c = 0; c < 3; ++c) {
                double x0 = s->V[(size_t)c * s->nV + b0], x1 = s->V[(size_t)c * s->nV + b1];
                double y0 = x0 + max_t * p[3 * (size_t)b0 + c], y1 = x1 + max_t * p[3 * (size_t)b1 + c];
                double jh = std::max(std::max(x0, y0), std::max(x1, y1)), jl = std::min(std::min(x0, y0), std::min(x1, y1));
                if (jl - bi_hi[c] > 0.0 || bi_lo[c] - jh > 0.0) sep = true;
            }
            if (sep) continue;
            if (a0 == b0 || a0 == b1 || a1 == b0 || a1 == b1) continue;
            if ((codim(s, a0) < 3 && codim(s, b0) < 3) || (is_dbc(s, a0) && is_dbc(s, a1) && is_dbc(s, b0) && is_dbc(s, b1))) continue;
            ++pairs;
            int v[4] = { a0, a1, b0, b1 };
            double toi;
            int r = pair_ccd(false, v, s, p, tol, err_ee, max_t, &toi);
            if (r < 0) zero = 1;
            else if (r > 0 && toi < best) best = toi;
        }
    }
    if (nPairs) *nPairs = pairs;
    *alpha = zero ? 0.0 : best;
    return zero;
}

} // extern "C"
