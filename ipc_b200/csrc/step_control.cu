// step_control.cu -- the data-dependent decisions of a Newton iteration on the device (sm_90a): the CFL branch of the step bound
// (Optimizer.cpp:1947-2027, CFL_FOR_CCD == 2) and the loop conditions of Optimizer::lineSearch (Optimizer.cpp:2662-2916, armijoParam = 0,
// lowerBound = 0), and the entry of a warm start (Optimizer::initX, Optimizer.cpp:1120-1215), whose two loops are the line search's first two.
//   *** compiled with --fmad=false (NOFMA_FILES): |p| = sqrt((x*x + y*y) + z*z) rounds like the CPU oracle ***
//
// Every decision is one single-thread kernel that reads IterState (energies, safeguard counts, flags), computes the next step in place
// (IterState::step_ord) and writes the decision word IterState::ls_cond.  Outside a capture the host reads that word; inside one the kernel
// also hands it to the conditional graph node that runs the loop body (cudaGraphSetConditional).  abi.h holds the two drivers (cond_node).
// The Krylov loops of the linear solves (kSolveStart, kSolveBurst) are decided here too: their residual test is the host loop's, so
// the iterations and the bits do not depend on which driver runs them.
#include "common.cuh"
#include "kernels.h"
#include "../../include/ipcgpu.h"
#include <algorithm>

namespace ipcgpu {

// max_i |p_{SVI[i]}| over the mesh's surface vertices (the obstacle tail excluded); the maximum is exact, so the order does not matter
__global__ void __launch_bounds__(256) k_cfl_pmax(int nSV, const int* __restrict__ SVI, int nVdof, const double* __restrict__ dir, unsigned long long* __restrict__ out)
{
    double m = 0.0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nSV; i += gridDim.x * blockDim.x) {
        const int v = SVI[i];
        if (v >= nVdof) continue;
        const double x = dir[3 * (size_t)v], y = dir[3 * (size_t)v + 1], z = dir[3 * (size_t)v + 2];
        m = fmax(m, sqrt((x * x + y * y) + z * z));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0 && m > 0.0) atomicMax(out, dbl_to_ord(m)); // (non-negative doubles order like their bit patterns)
}

DEV void fail(IterState* st, int code)
{
    if (st->sc_status == 0) st->sc_status = code;
}
// a loop condition of the line search: while the safeguard count `bad` is positive, halve the step (the loop ends at 0 with an error)
DEV int halve_while(IterState* st, bool bad, int counter)
{
    if (!bad) return 0;
    const double alpha = ord_to_dbl(st->step_ord);
    if (alpha == 0.0) { // the entry state itself fails the check: the reference would spin forever here
        fail(st, IPCGPU_ERR_LINE_SEARCH);
        return 0;
    }
    st->step_ord = dbl_to_ord(alpha / 2.0);
    ++st->ls_count[counter];
    return 1;
}
// E = ((E_el + E_in) + E_b) + E_f, the accumulation order of Optimizer::computeEnergyVal (Optimizer.cpp:3199-3378); with half-spaces
// ((E_el + E_in) + (E_b + E_plane_b)) + E_plane_f + E_f: both barrier parts are one kappa bVals.sum() (:3352), plane friction comes first (:3355-3377).
// The Neumann forces come right after the inertia term (:3241-3250), damping (:3381-3400) and the Dirichlet penalty (:3402-3404) last:
// ((((((E_el + E_in) + E_nbc) + E_b) + E_plane_f) + E_f) + E_damp) + E_dbc.  A term that is not set adds nothing (not even a 0).
DEV double energy_sum(const IterState* st, int terms)
{
    double e = st->energy[kEnergyElastic];
    if (terms & kTermInertia) e += st->energy[kEnergyInertia];
    if (terms & kTermNeumann) e += st->energy[kEnergyNeumann];
    e += (terms & kTermHalfSpace) ? st->energy[kEnergyBarrier] + st->energy[kEnergyPlaneBarrier] : st->energy[kEnergyBarrier];
    if (terms & kTermHalfSpaceFriction) e += st->energy[kEnergyPlaneFriction];
    if (terms & kTermFriction) e += st->energy[kEnergyFriction];
    if (terms & kTermDamping) e += st->energy[kEnergyDamping];
    if (terms & kTermDirichlet) e += st->energy[kEnergyDirichlet];
    return e;
}
// the intersection safeguard: surface triangles crossed by an edge, and with half-spaces the vertices with d <= 0 (isIntersected, :2627-2642)
DEV bool intersected(const IterState* st, int terms) { return st->checks[1] > 0 || ((terms & kTermHalfSpace) && st->hs_crossings > 0); }

// the solve fails: the status its result reports and the flag the fetch reports (a line search refuses to start while it is raised)
DEV void solve_fail(IterState* st)
{
    st->sv_run = 0;
    st->sv_status = IPCGPU_ERR_SOLVE;
    st->flags[FLAG_SOLVE] = 1;
}

__global__ void k_step_decide(IterState* st, int op, double a, int b, cudaGraphConditionalHandle h, const double* __restrict__ aux)
{
    if (threadIdx.x != 0) return;
    int cond = 0;
    const bool ok = st->sc_status == 0;
    switch (op) {
    case kCflBranch: { // :1951-1956, :1962, :2017-2024;  a = dHat, b = (k == 0)
        const double pMax = ord_to_dbl(st->sc_pmax_ord), alpha = ord_to_dbl(st->step_ord);
        const double cfl = sqrt(a) / (pMax * 2.0); // pMax == 0: inf, as in the reference
        st->sc_alpha_cfl = cfl;
        cond = (b && alpha > cfl) || alpha > 2.0 * cfl;
        st->sc_full_ccd = cond;
        if (!cond) {
            const double r = cfl < alpha ? cfl : alpha; // std::min(alpha, alpha_CFL)
            st->step_ord = dbl_to_ord(r);
            st->alpha_stage[2] = st->alpha_stage[3] = r;
            if (r == 0.0) fail(st, IPCGPU_ERR_LINE_SEARCH); // :2031-2033 exit(-1)
        }
        break;
    }
    case kCflClamp: { // :2009-2012, after the full CCD
        double alpha = ord_to_dbl(st->step_ord);
        if (alpha < st->sc_alpha_cfl) alpha = st->sc_alpha_cfl;
        st->step_ord = dbl_to_ord(alpha);
        if (alpha == 0.0) fail(st, IPCGPU_ERR_LINE_SEARCH);
        break;
    }
    case kLsEntry: { // a line search starts: its counters are per call
        for (int k = 0; k < 4; ++k) st->ls_count[k] = 0;
        st->ls_stopped = st->ls_rebuilt = st->ls_post_ran = 0;
        st->sc_status = 0;
        st->ls_E0 = st->ls_Et = 0.0;
        const double alpha = ord_to_dbl(st->step_ord);
        st->ls_LF = alpha;
        cond = alpha > 0.0;
        if (!cond) st->sc_status = IPCGPU_ERR_LINE_SEARCH;
        if (st->flags[FLAG_SOLVE]) { // the direction is that of a failed solve: V stays V0
            cond = 0;
            st->sc_status = IPCGPU_ERR_SOLVE;
        }
        break;
    }
    case kLsStart: // :2681 E0 = E(V) with the sets held on entry;  b = energy terms
        st->ls_E0 = energy_sum(st, b);
        if (st->flags[FLAG_NONPOSITIVE_DISTANCE]) fail(st, IPCGPU_ERR_NONPOSITIVE_DISTANCE);
        break;
    case kLsInversion: // :2710-2715
        cond = ok && halve_while(st, st->checks[0] > 0, 0);
        break;
    case kLsIntersection: // :2720-2733; the loop's exit is LFStepSize (:2750);  b = energy terms
        cond = ok && halve_while(st, intersected(st, b), 1);
        if (!cond) st->ls_LF = ord_to_dbl(st->step_ord);
        break;
    case kLsArmijo: { // :2744, :2761-2797 with c1m = 0 and lowerBound = 0;  b = energy terms
        st->ls_Et = energy_sum(st, b);
        if (st->flags[FLAG_NONPOSITIVE_DISTANCE]) fail(st, IPCGPU_ERR_NONPOSITIVE_DISTANCE); // :3296-3306
        const double alpha = ord_to_dbl(st->step_ord);
        if (st->sc_status == 0 && st->ls_Et > st->ls_E0 && alpha > 0.0) {
            st->step_ord = dbl_to_ord(alpha / 2.0);
            ++st->ls_count[2];
            if (alpha / 2.0 == 0.0) st->ls_stopped = 1; // (V and E_t stay those of the last trial)
            else cond = 1;
        }
        break;
    }
    case kLsPostCheck: // :2799
        cond = ok && ord_to_dbl(st->step_ord) < st->ls_LF;
        break;
    case kLsPostLoop: // :2801-2807;  b = energy terms
        cond = ok && halve_while(st, intersected(st, b), 3);
        if (cond) st->ls_post_ran = 1;
        break;
    case kLsRebuild: // :2808-2810
        cond = ok && st->ls_post_ran;
        st->ls_rebuilt = cond;
        break;
    case kWsEntry: // initX (:1123): a warm start begins at stepSize = a (1.0; 0.0 for option 0).  Its counters are per call, as a line
                   // search's are, but a step bound of 0 is not an error here ("CCD gives 0 in initX()" is only logged, :1186-1188): the loops
                   // then run at step 0 and only a failing entry state ends the call with IPCGPU_ERR_LINE_SEARCH (halve_while).
        for (int k = 0; k < 4; ++k) st->ls_count[k] = 0;
        st->ls_stopped = st->ls_rebuilt = st->ls_post_ran = 0;
        st->sc_status = 0;
        st->ls_E0 = st->ls_Et = 0.0;
        st->step_ord = dbl_to_ord(a);
        st->ls_LF = a;
        st->alpha_stage[0] = a; // the step the inversion filter starts from (it lowers it on Neo-Hookean meshes; no filter otherwise)
        break;
    case kSolveStart: // after the solver's set-up;  a = rel_tol, b = max_iter, aux = the solver's scalars ([4] |b|^2, [6] a pivot <= 0)
        st->sv_iters = 0;
        st->sv_status = 0;
        st->sv_max_iter = b;
        st->sv_tol = a;
        st->sv_bb = st->sv_rr = aux[4];
        st->sv_xmax_ord = 0;
        st->sv_run = aux[4] > 0.0;
        if (aux[6] != 0.0) solve_fail(st);
        break;
    case kSolveBurst: // before a burst of b iterations, and after each: stop on a non-finite residual, on convergence (checked after a burst
                      // only) or when the burst would pass max_iter.  Evaluated twice at one count (end of a loop, entry of the next), it
                      // decides the same.
        if (st->sv_run && st->sv_iters > 0) {
            const double rr = st->sv_rr;
            if (!(rr == rr)) solve_fail(st);
            else if (sqrt(rr) <= st->sv_tol * sqrt(st->sv_bb)) st->sv_run = 0;
        }
        cond = st->sv_run && st->sv_iters + b <= st->sv_max_iter;
        break;
    case kAmgRound: // before each pass of aggregation rounds: the first pass of a coarsened level, then while a row is undecided.  A pass
                    // beyond amg_limit (the level's rows: every round decides a row) stops the loop and raises amg_stuck
        cond = st->amg_limit > 0 && (st->amg_round == 0 || st->amg_undecided > 0);
        if (cond && st->amg_round > st->amg_limit) {
            cond = 0;
            st->amg_stuck = 1;
        }
        if (cond) {
            ++st->amg_round;
            st->amg_undecided = 0;
        }
        break;
    }
    st->ls_cond = cond;
    if (h) cudaGraphSetConditional(h, (unsigned)cond);
}

void cfl_pmax(int nSV, const int* SVI, int nVdof, const double* dir, IterState* st_dev, cudaStream_t st)
{
    zero_words(&st_dev->sc_pmax_ord, 2, st);
    if (nSV > 0) k_cfl_pmax<<<std::min((nSV + 255) / 256, kSMs * 4), 256, 0, st>>>(nSV, SVI, nVdof, dir, &st_dev->sc_pmax_ord);
}

void step_decide(IterState* st_dev, int op, double a, int b, unsigned long long handle, cudaStream_t st, const double* aux)
{
    k_step_decide<<<1, 32, 0, st>>>(st_dev, op, a, b, (cudaGraphConditionalHandle)handle, aux);
}

} // namespace ipcgpu
