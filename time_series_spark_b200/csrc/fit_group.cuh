// Grouped-lanes Prophet MAP fit for sm_90a: G lanes per series, 32 / G series per warp.
//
// Same per-series algorithm as fit_kernel.cuh (prep done by prep_kernel; Stan L-BFGS restated from
// bfgs.hpp / bfgs_linesearch.hpp / lbfgs_update.hpp; objective of python/stan/unix/prophet.stan, reached
// from reference src/jobs/prophet_modeler.py:65-66), for the class that carries the headline workload:
// regular time grid whose step divides the day into GPT_MIN..GPT steps, weekly + daily seasonality
// ("day table", variant 3).  Why a second kernel:
// with one warp per series much of the warp time went into the ~2.5 k-instruction per-evaluation serial
// code (line search, L-BFGS update, trend adjoints) whose operands are 42-element vectors and 26 trend
// segments -- most lanes idle or redundant, instruction fetch the top stall, and phase-aligning the warps of
// an SM did not help.  Here one pass through that code serves 32 / G series:
//   * every lane owns T / G contiguous points of ITS series; the point loop is the same instruction
//     stream for all lanes, so the groups of a warp stay converged through an evaluation;
//   * vectors live G-strided (element q on lane q mod G), trend segments blocked (32 / G per lane), and
//     reductions / scans are log2(G) shuffle steps within the group, under the full warp mask;
//   * the groups of a warp run the optimiser's state machine in lockstep at evaluation granularity:
//     [fetch + stage a series if idle] -> evaluate -> line-search step -> (accepted: update) -> new search / trial point;
//     the whole warp runs every routine of a round, and a group whose action differs (or an idle one) computes on its
//     own slot's state and stores nothing.
// Data layout per series slot: global workspace: y_scaled in steps of U points per lane (U = 2; 4 was measured and lost),
// step m of lane l at ((m G + l) U) doubles (a lane's cp.async is 16 B, a group's G lanes read 8 U G contiguous bytes), and the
// L-BFGS history Y[5], S[5] (read once per iteration); shared memory (GState): optimiser state, the six
// working vectors, segment arrays, the seasonal table s_p / R_p.
// Arithmetic differences from fit_kernel.cuh's day-table variant (parity is to the oracle, 1e-10 / 1e-8):
//   * t_i = i h (h = step / span) instead of a stored (ds_i - start) / span -- one rounding apart;
//   * logistic trend: e_i = exp(-k_j (t_i - m_j)) advanced by e_i = e_{i-1} q_j, q_j = exp(-k_j h), within
//     a lane's chunk (the exponent is continuous across changepoints by construction of the offsets m_j, so
//     only the ratio changes there); one true exp per lane per evaluation.  Evaluations whose exponent
//     leaves +-600 anywhere (wild line-search trials) take the direct-exp path.
#pragma once
#include <type_traits>

#include "fit_kernel.cuh"

namespace pb200 {
namespace grp {

constexpr int GK = 14, GKW = 6, GKD = 8; // weekly 3 + daily 4 harmonics
// SEAS = false: the class without any seasonality (regular grid, span under two days: reference config #4's short series) --
// the same state machine with no table, no weekly recurrences and the single all-zero feature column fbprophet keeps
template <bool SEAS> constexpr int gkx() { return SEAS ? GK : 1; }

constexpr int ST_IDLE = 0, ST_FIRST = 1, ST_SEARCH = 2, ST_OBJ = 3;

// SEAS = false (the class without seasonality) drops the table and shortens the vectors: 3.7 instead of 5.8 KB per series,
// the difference between 9 and 14 resident warps per SM (that class's time falls as they rise)
template <int G, bool SEAS>
struct GState {
    static constexpr int PPAD = SEAS ? GPPAD : GPPAD_PLAIN;
    static constexpr int PT = SEAS ? GPT : 2;        // (without a table: the scratch of the pass's two totals)
    static constexpr int TOTSS = SEAS ? GK : 1;      // where the pass leaves the residual sum of squares: stab[TOTSS]
    LSState ls;
    double cap_s, sigma, hstep, zmax;
    int T, S, ncp, chunk, tabP, tabPL, series, state, exprec, st0, i1max, pad_;
    double kc[GSEG], mc[GSEG], tc[GSEG], qs[GSEG], bndU[GSEG], bndV[GSEG];
    int bidx[GSEG];
    alignas(16) double bcoef[SEAS ? 16 : 2];
    double hrho[8];
    alignas(16) double rotw[2];          // (sin, cos) of one grid step's advance of the weekly angle
    alignas(16) double rotd[2];          // ... of the daily angle
    alignas(16) double stab[PT];         // s_p: daily part of X beta at table phase p
    alignas(16) double rtab[PT];         // R_p: residual bins; stab / rtab double as the reduction scratch
    alignas(16) double vec[6][PPAD];     // x g p x_trial g_trial p_prev (roles in ls.ix ...)
};

// per-lane constants of a lane's chunk of ITS series, kept in registers between evaluations (g_fetch leaves them in
// vec[1..5], which nothing reads before the first evaluation has written them)
struct LanePhase {
    double2 wph;        // weekly (sin, cos) two points before the lane's first point
    double2 wend;       // weekly (sin, cos) at the lane's second last point (padded to whole two-point steps)
    double2 dph;        // daily (sin, cos) at the lane's first table phase
    int j0;             // trend segment of the point before the lane's chunk
};

#ifndef PB200_GRP_RING
// stages of g_point_pass's cp.async ring for G = 8 (a power of two; loads run stages - 1 two-point steps ahead).  The slots of
// 8 resident CTAs per SM are more than an H100's L2 holds, so part of the y stream comes from HBM, whose round trip one step
// of lead does not cover: with 2 stages a fifth of the warp cycles went into cp.async.wait_group.  4 and 8 stages measured
// the same; 4 add 1 KB per CTA
#define PB200_GRP_RING 4
#endif
// (G = 16 runs 16 CTAs per SM: two more stages would cost one of them)
__host__ __device__ constexpr int grp_ring(int G) { return G == 8 ? PB200_GRP_RING : 2; }
static_assert(PB200_GRP_RING >= 2 && (PB200_GRP_RING & (PB200_GRP_RING - 1)) == 0, "ring stages: a power of two");

template <int G, bool SEAS>
inline size_t group_smem_bytes() {
    return (size_t)(32 / G) * ((sizeof(GState<G, SEAS>) + 15) & ~(size_t)15) + (size_t)grp_ring(G) * (grp_u(G) / 2) * 32 * 16   // + cp.async ring
           + sizeof(FitOptsDev)                                                                                  // + the options
           + (size_t)(32 / G) * sizeof(SeriesPrior);                                                             // + gprior
}
// global workspace per series slot (doubles): y pairs, then history Y[5], S[5]
__host__ __device__ inline size_t group_plane_doubles(int tmax, int G) {
    const int cmax = (tmax + G - 1) / G + GCHUNK_SLACK, U = grp_u(G);
    return (size_t)((cmax + U - 1) / U) * G * U + 8;
}
constexpr int GHIST = 2 * HMAX * GPPAD;

template <int G, bool SEAS>
__device__ __forceinline__ GState<G, SEAS>& gstate(int gi) {
    return *reinterpret_cast<GState<G, SEAS>*>(pb200_smem + (size_t)gi * ((sizeof(GState<G, SEAS>) + 15) & ~(size_t)15));
}
template <int G, bool SEAS>
__device__ __forceinline__ double2* gring() {
    return reinterpret_cast<double2*>(pb200_smem + (size_t)(32 / G) * ((sizeof(GState<G, SEAS>) + 15) & ~(size_t)15));
}
// the fit options, copied out of the kernel parameters once per warp (the optimiser's routines take them by reference;
// a reference into the parameter bank would force a local-memory copy that misses L1 on every use)
template <int G, bool SEAS>
__device__ __forceinline__ FitOptsDev& gopts() {
    return *reinterpret_cast<FitOptsDev*>(reinterpret_cast<unsigned char*>(gring<G, SEAS>()) + (size_t)grp_ring(G) * (grp_u(G) / 2) * 32 * 16);
}
// the prior scales of group gi's series (inv_seas2 = 1 without seasonality), behind the options rather than in GState: a
// longer GState moves every group's state to other shared-memory banks, which measured 4 % slower at G = 8
template <int G, bool SEAS>
__device__ __forceinline__ SeriesPrior& gprior(int gi) {
    return reinterpret_cast<SeriesPrior*>(&gopts<G, SEAS>() + 1)[gi];
}

// ---- L2 priority of the workspace slots (per-access cache hints only: nothing is set aside in L2 for the device) ----
// The first FitArgs::l2_keep slots (y plane and L-BFGS history) are evict_last; the host sizes their number to a share of the
// device's L2.  The other slots, and the series' inputs (read once), are evict_first.  Before a warp exits it returns its
// slots' lines to normal priority (grp_l2_release).
__device__ __forceinline__ unsigned long long l2_policy_evict_last() {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
__device__ __forceinline__ unsigned long long l2_policy_evict_normal() {
    unsigned long long pol;
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(pol));
    return pol;
}
// the policy of one class of accesses from the warp's L2 flags (bits L2F_*); created where it is used, so that no 64-bit
// policy register lives across the kernel's loop
constexpr int L2F_KEEP = 1, L2F_REST_FIRST = 2;
__device__ __forceinline__ unsigned long long l2_policy(const int l2f) {
    if (l2f & L2F_KEEP) return l2_policy_evict_last();
    return (l2f & L2F_REST_FIRST) ? l2_policy_evict_first() : l2_policy_evict_normal();
}
__device__ __forceinline__ void cp_async16_sa(const unsigned smem_addr, const void* gsrc, const unsigned long long pol) {
    asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" ::"r"(smem_addr), "l"(__cvta_generic_to_global(gsrc)),
                 "l"(pol) : "memory");
}
__device__ __forceinline__ void st_hint(double* p, const double v, const unsigned long long pol) {
    asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(__cvta_generic_to_global(p)), "d"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ void stcg_hint(double* p, const double v, const unsigned long long pol) {
    asm volatile("st.global.cg.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(__cvta_generic_to_global(p)), "d"(v), "l"(pol) : "memory");
}
__device__ __forceinline__ double ldcg_hint(const double* p, const unsigned long long pol) {
    double v;
    asm("ld.global.cg.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(__cvta_generic_to_global(p)), "l"(pol));
    return v;
}
__device__ __forceinline__ double load_y_hint(const void* y, const int dtype, const long long i, const unsigned long long pol) {
    if (dtype == PB200_Y_I32) {
        int v;
        asm("ld.global.nc.L2::cache_hint.s32 %0, [%1], %2;" : "=r"(v) : "l"(__cvta_generic_to_global((const int*)y + i)), "l"(pol));
        return (double)v;
    }
    if (dtype == PB200_Y_F32) {
        float v;
        asm("ld.global.nc.L2::cache_hint.f32 %0, [%1], %2;" : "=f"(v) : "l"(__cvta_generic_to_global((const float*)y + i)), "l"(pol));
        return (double)v;
    }
    double v;
    asm("ld.global.nc.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(__cvta_generic_to_global((const double*)y + i)), "l"(pol));
    return v;
}
// normal L2 priority again for the 128 B lines of [p, p + n doubles), lines split over the G lanes of the group
template <int G>
__device__ __forceinline__ void grp_l2_release(const double* p, const size_t n, const int gl) {
    const size_t b0 = (size_t)__cvta_generic_to_global(p) & ~(size_t)127, b1 = (size_t)__cvta_generic_to_global(p + n);
#pragma unroll 1
    for (size_t b = b0 + (size_t)gl * 128; b < b1; b += (size_t)G * 128)
        asm volatile("applypriority.global.L2::evict_normal [%0], 128;" ::"l"(b) : "memory");
}

// ---- warp-cycle accounting of the kernel's phases (dev builds with -DPB200_PHASE_CLOCKS only; read out through
// pb200_dev_phase_clocks, printed by tools/prof_phases.py).  Without the flag the macros expand to nothing ----
enum PhaseClock {
    PC_TOTAL, PC_FETCH, PC_SETUP, PC_PASS, PC_FINAL, PC_LS_STEP, PC_POST, PC_LS_BEGIN, PC_WRITE,   // exclusive, sum ~ PC_TOTAL
    PC_PASS_WAIT,      // inside PC_PASS: cp.async.wait_group of the y ring
    PC_POST_HIST,      // inside PC_POST: waiting for the history loads at their first use
    PC_DRAIN,          // inside PC_TOTAL: rounds after the queue ran dry with fewer than 32 / G active groups
    PC_PASS_LOOP,      // inside PC_PASS: g_point_pass's two step loops; the rest of the pass is the table and the reductions
    PC_ROUNDS,         // (a count, not cycles) evaluation rounds
    PC_WARPS,          // (a count) warps = CTAs of the launches
    PC_PASS_STEPS,     // (a count) steps run by the step loops
    PC_POST_CALLS,     // (a count) rounds in which the warp runs g_post_accept (PC_POST's cycles per call)
    PC_ACCEPTS,        // (a count) accepted line searches, over the groups
    PC_N
};
#ifdef PB200_PHASE_CLOCKS
__device__ unsigned long long g_phase_cycles[PC_N];
#define PB200_PCLK_DECL(v) long long v = 0
#define PB200_PCLK_NOW(v) v = clock64()
// time `stmt` into the accumulator `acc`
#define PB200_PCLK_SPAN(acc, stmt) { const long long t0_ = clock64(); stmt; acc += clock64() - t0_; }
// add (now - mark) to phase ph from lane `lane` == 0 and move the mark
#define PB200_PCLK_MARK(ph, mark, lane) { const long long t_ = clock64(); if ((lane) == 0) atomicAdd(&g_phase_cycles[ph], (unsigned long long)(t_ - mark)); mark = t_; }
#define PB200_PCLK_ADD(ph, v, cond) { if (cond) atomicAdd(&g_phase_cycles[ph], (unsigned long long)(v)); }
#else
#define PB200_PCLK_DECL(v)
#define PB200_PCLK_NOW(v)
#define PB200_PCLK_SPAN(acc, stmt) { stmt; }
#define PB200_PCLK_MARK(ph, mark, lane)
#define PB200_PCLK_ADD(ph, v, cond)
#endif

// ---- group collectives (lanes of one series).  The whole warp calls them: every shuffle runs under the full mask, with
// offsets below G (xor) or width G (scans), so that each group sees only its own lanes.  A group's lane mask is a run-time
// value, and a shuffle under it would first compile to a convergence test and a collective fallback ----
template <int G>
__device__ __forceinline__ double gsum(double v) {
#pragma unroll
    for (int o = G / 2; o >= 1; o >>= 1) v += __shfl_xor_sync(FULL, v, o);
    return v;
}
template <int G>
__device__ __forceinline__ double gmax(double v) {
#pragma unroll
    for (int o = G / 2; o >= 1; o >>= 1) v = fmax(v, __shfl_xor_sync(FULL, v, o));
    return v;
}
// sum of v over the lower lanes of the group (exclusive prefix); *tot = the group total
template <int G>
__device__ __forceinline__ double gscan_excl(double v, const int gl, double* tot) {
    double inc = v;
#pragma unroll
    for (int o = 1; o < G; o <<= 1) {
        const double a = __shfl_up_sync(FULL, inc, o, G);
        if (gl >= o) inc += a;
    }
    if (tot) *tot = __shfl_sync(FULL, inc, G - 1, G);
    return inc - v;
}
// sum of v over the HIGHER lanes of the group
template <int G>
__device__ __forceinline__ double gscan_excl_rev(double v, const int gl) {
    double inc = v;
#pragma unroll
    for (int o = 1; o < G; o <<= 1) {
        const double a = __shfl_down_sync(FULL, inc, o, G);
        if (gl + o < G) inc += a;
    }
    return inc - v;
}
template <int G, int PPAD>
__device__ __forceinline__ double gvdot(const double* a, const double* b, const int P, const int gl) {
    double s = 0.0;
#pragma unroll
    for (int u = 0; u < (PPAD + G - 1) / G; ++u) {
        const int q = gl + u * G;
        if (q < P) s = fma(a[q], b[q], s);
    }
    return gsum<G>(s);
}

// ---------------------------------------------------------------------------------------
// evaluation, part 1: trend segments of theta (rate, offset, per-step exp ratio), sigma, beta.  The whole warp calls it;
// an idle group (`active` false) computes on its own slot's state and stores nothing
// ---------------------------------------------------------------------------------------
template <int G, bool LOGI, bool SEAS>
__device__ __noinline__ void g_eval_setup(GState<G, SEAS>& s, const double* xv, const int gl, const bool active) {
    constexpr int NS = GSEG / G;
    const int S = s.S, jb = gl * NS;
    const double k = xv[0], m = xv[1];
    double d[NS], pre[NS], kcl[NS + 1], tcl[NS];
    double run = 0.0, rune = 0.0, pree[NS];
#pragma unroll
    for (int u = 0; u < NS; ++u) {
        const int j = jb + u;
        d[u] = j < S ? xv[2 + j] : 0.0;
        tcl[u] = j < S ? s.tc[j] : 0.0;
        pre[u] = run;
        run += d[u];
        if constexpr (!LOGI) { pree[u] = rune; rune = fma(-tcl[u], d[u], rune); }
    }
    const double ex = gscan_excl<G>(run, gl, nullptr);
#pragma unroll
    for (int u = 0; u < NS; ++u) kcl[u] = k + (ex + pre[u]);
    kcl[NS] = __shfl_down_sync(FULL, kcl[0], 1, G);               // first rate of the next lane's block
    if (active && gl == 0) s.sigma = exp_fastpath(xv[2 + S]);
    double mcl[NS + 1];
    if constexpr (LOGI) {
        // logistic_gamma: m_{j+1} = rho_j m_j + (1 - rho_j) t_change_j, rho_j = k_j / k_{j+1}
        double ra[NS], rb[NS], A = 1.0, B = 0.0;
#pragma unroll
        for (int u = 0; u < NS; ++u) {
            const int j = jb + u;
            const double rho = j < S ? div_const(kcl[u], kcl[u + 1], rcp_any(kcl[u + 1])) : 1.0;
            ra[u] = rho;
            rb[u] = j < S ? (1.0 - rho) * tcl[u] : 0.0;
            B = fma(ra[u], B, rb[u]);
            A = ra[u] * A;
        }
        double Ai = A, Bi = B;                                     // inclusive scan of the block maps
#pragma unroll
        for (int o = 1; o < G; o <<= 1) {
            const double Ap = __shfl_up_sync(FULL, Ai, o, G);
            const double Bp = __shfl_up_sync(FULL, Bi, o, G);
            if (gl >= o) { Bi = fma(Ai, Bp, Bi); Ai = Ai * Ap; }
        }
        double Ae = __shfl_up_sync(FULL, Ai, 1, G), Be = __shfl_up_sync(FULL, Bi, 1, G);
        if (gl == 0) { Ae = 1.0; Be = 0.0; }
        mcl[0] = fma(Ae, m, Be);
#pragma unroll
        for (int u = 0; u < NS; ++u) mcl[u + 1] = fma(ra[u], mcl[u], rb[u]);
        const double h = s.hstep;
        double zm = 0.0;
#pragma unroll
        for (int u = 0; u < NS; ++u) {
            const int j = jb + u;
            if (j <= S) {
                if (active) {
                    s.kc[j] = kcl[u];
                    s.mc[j] = mcl[u];
                    s.qs[j] = exp_fastpath(-(kcl[u] * h));
                }
                // the exponent k_j (t - m_j) is piecewise linear in t: its extremes sit at the segment ends
                const double tl = j == 0 ? -h : s.tc[j - 1];
                const double tr = j == S ? 1.0 : tcl[u];
                const double z0 = kcl[u] * (tl - mcl[u]), z1 = kcl[u] * (tr - mcl[u]);
                zm = fmax(zm, fmax(fabs(z0), fabs(z1)));
                if (!(fabs(z0) < 600.0) || !(fabs(z1) < 600.0)) zm = 1e300;   // NaN too
            }
        }
        zm = gmax<G>(zm);
        if (active && gl == 0) s.exprec = zm < 600.0 ? 1 : 0;
    } else {
        const double exe = gscan_excl<G>(rune, gl, nullptr);
#pragma unroll
        for (int u = 0; u < NS; ++u) {
            const int j = jb + u;
            if (active && j <= S) { s.kc[j] = kcl[u]; s.mc[j] = m + (exe + pree[u]); }
        }
        if (active && gl == 0) s.exprec = 0;
    }
#pragma unroll
    for (int u = 0; u < (gkx<SEAS>() + G - 1) / G; ++u) {
        const int q = gl + u * G;
        if (active && q < gkx<SEAS>()) s.bcoef[q] = xv[3 + S + q];
    }
    __syncwarp();
}

// features of table phase p from the (sin, cos) of the daily angle
__device__ __forceinline__ void day_features(const double2 w, double* X) { harmonics<4>(w, X); }

// one point: everything between the loads and the accumulations
template <bool LOGI, bool MULT>
struct GPoint {
    double r, cb, dz, tm;
    // dot: the seasonal term X beta of the point (table entry + weekly part; 1 + X beta in multiplicative mode)
    __device__ __forceinline__ void run(const double y, const double t, const double dot, const double e, const double kcj,
                                        const double mcj, const double cap, const bool valid) {
        double g, sig = 0.0;
        if constexpr (LOGI) {
            tm = t - mcj;
            sig = rcp_fastpath(1.0 + e);
            g = cap * sig;
        } else {
            tm = t;
            g = fma(kcj, t, mcj);
        }
        // multiplicative mode: the table entry already holds 1 + (daily part), so dot = 1 + X beta
        double opm, yhat;
        if constexpr (MULT) { opm = dot; yhat = g * opm; }
        else { opm = 1.0; yhat = g + dot; }
        r = valid ? y - yhat : 0.0;
        cb = MULT ? r * g : r;
        if constexpr (LOGI) {
            // d/dz of the trend term: r opm g (1 - sig) = (cb opm)(1 - sig) in multiplicative mode
            const double qg = MULT ? cb * opm : r * g;
            dz = qg * (1.0 - sig);
        } else {
            dz = MULT ? r * opm : r;
        }
        // A point past the lane's own (only the checked tail steps have them; `valid` is a constant true elsewhere) runs on
        // at virtual t > 1 when a longer series shares the warp, where the exp-ratio recurrence is unchecked: e = inf gives
        // sig = NaN, and 0 * NaN would poison the sums.  Its contributions are zeros by definition
        if (!valid) { cb = 0.0; dz = 0.0; }
    }
};

// ---------------------------------------------------------------------------------------
// evaluation, part 2: the pass over the points (all lanes of the warp, every active group)
// ---------------------------------------------------------------------------------------
template <int G, bool LOGI, bool MULT, bool SEAS, int U>
__device__ __noinline__ void g_point_pass(GState<G, SEAS>& s, const double* plane, const bool active, const int gl, const int lane,
                                          const LanePhase lp, const int l2f) {
    static_assert(U == 2 || U == 4, "points per lane per step");
    const int P = active ? s.tabP : GState<G, SEAS>::PT, PL = active ? s.tabPL : 0;     // (an idle group's lanes only keep step)
    const double2 rct = *reinterpret_cast<const double2*>(s.rotd);
    const double2 w0 = lp.dph;
    // ---- seasonal table of this evaluation; residual bins cleared ----
    if (SEAS && active) {
        double2 w = w0;
        int p = gl * PL;
#pragma unroll 2
        for (int q = 0; q < PL; ++q, ++p) {
            if (p < P) {
                double X[GKD];
                day_features(w, X);
                double d0 = 0.0, d1 = 0.0;
#pragma unroll
                for (int k = 0; k < GKD; k += 2) {
                    const double2 b = *reinterpret_cast<const double2*>(&s.bcoef[GKW + k]);
                    d0 = fma(b.x, X[k], d0);
                    d1 = fma(b.y, X[k + 1], d1);
                }
                s.stab[p] = (MULT ? 1.0 : 0.0) + (d0 + d1);       // multiplicative: 1 + seasonal sum, see GPoint::run
                s.rtab[p] = 0.0;
            }
            const double sn = fma(w.x, rct.y, w.y * rct.x);
            const double cn = fma(w.y, rct.y, -(w.x * rct.x));
            w = make_double2(sn, cn);
        }
    }
    __syncwarp();
    const int chunk = s.chunk, T = s.T, S = s.S;
    const int i0 = active ? (gl * chunk < T ? gl * chunk : T) : 0;
    const int i1 = active ? (i0 + chunk < T ? i0 + chunk : T) : 0;
    const int npts = i1 - i0;
    int j = active ? lp.j0 : 0;                        // trend segment of the point before the chunk
    const int j0 = j;
    double gacc[GK];
    if constexpr (SEAS) {
#pragma unroll
        for (int q = 0; q < GK; ++q) gacc[q] = 0.0;
    }
    double ss = 0.0, locU = 0.0, locV = 0.0;
    int nb = (active && j < S) ? s.bidx[j] : 0x7fffffff;
    double kcj = s.kc[j], mcj = s.mc[j];
    const double cap = s.cap_s, h = s.hstep;
    const bool erec = LOGI && s.exprec != 0;
    double qj = LOGI ? s.qs[j] : 0.0;
    double e = 0.0;
    if constexpr (LOGI) {
        if (erec) e = exp_fastpath(-(kcj * (((double)(i0 - 1)) * h - mcj)));     // at the virtual point before the chunk
    }
    // uniform trip counts over the warp (the lanes stay in step for the bin updates): nstep steps in all, the first
    // nfull of them complete for every lane that has points -- those run without per-point validity tests
    int nstep = active ? (chunk + U - 1) / U : 0;
    int nfull = active ? npts / U : 0x7fffffff;
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        nstep = max(nstep, __shfl_xor_sync(FULL, nstep, o));
        nfull = min(nfull, __shfl_xor_sync(FULL, nfull, o));
    }
    nfull = min(nfull, nstep);
    // cp.async ring: NR stages of U points per lane (stage st, half q: row (st (U / 2) + q) of 32 double2); step m's loads are
    // issued D = NR - 1 steps ahead, one commit group per step.  The 32-bit shared-window address is taken once: inside the
    // loop the generic-to-shared conversion cost an S2R per step
    constexpr int NR = grp_ring(G), D = NR - 1;
    const unsigned long long pol_y = l2_policy(l2f);
    double2* const ring = gring<G, SEAS>() + lane;
    const unsigned ring_sa = (unsigned)__cvta_generic_to_shared(ring);
    constexpr unsigned STAGE_B = (U / 2) * 32 * 16;
    const double2* gsrc = reinterpret_cast<const double2*>(plane) + gl * (U / 2);   // step m of this lane: gsrc[m G (U / 2) + q]
#pragma unroll
    for (int d = 0; d < D; ++d) {
        if (d * U < npts) {
#pragma unroll
            for (int q = 0; q < U / 2; ++q) cp_async16_sa(ring_sa + d * STAGE_B + q * 512, gsrc + d * G * (U / 2) + q, pol_y);
        }
        cp_async_commit();
    }
    const double2* gnext = gsrc + D * G * (U / 2);
    PB200_PCLK_DECL(wait_cyc);
    int pb = (SEAS && P > 0) ? i0 % P : 0;
    // The weekly part of the seasonal term and of the beta gradient WITHOUT the six weekly features per point.  Every
    // harmonic h of the weekly angle obeys the three-term recurrence y(i + 1) = c_h y(i) - y(i - 1), c_h = 2 cos(h delta),
    // for its sine, its cosine and therefore for u_h(i) = beta_sh sin + beta_ch cos:
    //   * the seasonal term: u_h advanced IN PLACE on its values at the previous two points (one DFMA per harmonic and
    //     point; after a two-point step the pair again holds the last two points in order);
    //   * the gradient sum_i c_i y(i): Clenshaw's recurrence on the reversed sequence, B_i = c_h B_{i-1} + c_i - B_{i-2}
    //     (two operations per harmonic and point, serving sine AND cosine), closed after the lane's last point with
    //     sum = y(n-1) (B_{n-1} - c_h B_{n-2}) + y(n-2) B_{n-2}.
    // 12 FP64 operations per point instead of 19 (features by recurrence 6 + dot 7 + gradient 6), 25 (rotation).
    // Rounding: recurrences grow errors like n eps / sin(h delta), delta = 2 pi / 672: ~1e-12 of the term over a
    // 180-point chunk (measured against 40-digit arithmetic: 6e-13 for h = 1) -- inside the 1e-10 objective and 1e-8
    // gradient tolerances, and every evaluation restarts from the lane's exact start / end phases.
    static_assert(U == 2, "the in-place three-term recurrences are written for two points per step");
    constexpr int NH = GKW / 2;
    double uw[NH][2], Bw[NH][2], cw[NH];
    const int nown = active ? 2 * ((npts + 1) >> 1) : 0;       // this lane's own points (padded to whole steps)
    if constexpr (SEAS) {
        const double2 rcw = *reinterpret_cast<const double2*>(s.rotw);
        double Xr[GKW], X0[GKW], X1[GKW];
        harmonics<3>(rcw, Xr);                              // cos(h delta) at the odd positions
        double2 w = lp.wph;                                 // weekly angle at point i0 - 2
        harmonics<3>(w, X0);
        w = make_double2(fma(w.x, rcw.y, w.y * rcw.x), fma(w.y, rcw.y, -(w.x * rcw.x)));
        harmonics<3>(w, X1);                                // ... and at i0 - 1
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) {
            cw[hh] = 2.0 * Xr[2 * hh + 1];
            const double bs = s.bcoef[2 * hh], bc = s.bcoef[2 * hh + 1];
            uw[hh][0] = fma(bs, X0[2 * hh], bc * X0[2 * hh + 1]);
            uw[hh][1] = fma(bs, X1[2 * hh], bc * X1[2 * hh + 1]);
            Bw[hh][0] = 0.0;
            Bw[hh][1] = 0.0;
        }
    }
    double tt[U];                                       // t of the step's points, advanced by U h per step
#pragma unroll
    for (int u = 0; u < U; ++u) tt[u] = (double)(i0 + u) * h;
    const double hU = (double)U * h;
    // direct_tag false: every lane of the warp is on the exp-ratio recurrence (erec), so the step leaves out the test
    auto step = [&](const int m, auto checked_tag, auto direct_tag) {
        constexpr bool CHECK = decltype(checked_tag)::value;
        constexpr bool DIRECT = decltype(direct_tag)::value;
        const int n = U * m;
        double2* const cur = ring + (m & (NR - 1)) * (U / 2) * 32;
        const unsigned fill_sa = ring_sa + ((m + D) & (NR - 1)) * STAGE_B;
        if (n + D * U < npts) {
#pragma unroll
            for (int q = 0; q < U / 2; ++q) cp_async16_sa(fill_sa + q * 512, gnext + q, pol_y);
        }
        cp_async_commit();
        gnext += G * (U / 2);
        PB200_PCLK_SPAN(wait_cyc, cp_async_wait<D>());
        double yv[U];
        bool val[U];
        [[maybe_unused]] int pu[U];
        [[maybe_unused]] double sp[U], Rv[U];
        int jlo[U + 1];                                    // (jlo[0] is not used)
        double ee[U], kcu[U], mcu[U];
#pragma unroll
        for (int q = 0; q < U / 2; ++q) {
            const double2 v = cur[q * 32];
            yv[2 * q] = v.x;
            yv[2 * q + 1] = v.y;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            val[u] = CHECK ? n + u < npts : true;
            if constexpr (SEAS) {
                pu[u] = pb;
                pb = (pb + 1 == P) ? 0 : pb + 1;
                sp[u] = s.stab[pu[u]];
                Rv[u] = s.rtab[pu[u]];
            }
        }
        // exp ratio recurrence: the step INTO a point uses the rate of the segment the previous point is in; then the
        // changepoints AT the point switch rate, offset and ratio.  Nearly all steps hold no changepoint of this lane:
        // one test, and one divergent region for the steps that do.  The boundaries AT the step's first point get the
        // lane's sums before the step right there; those at later points are recorded after the step's arithmetic, when
        // the contributions of the step's earlier points are known
        if (nb >= i0 + n + U) {
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if constexpr (LOGI) { e = e * qj; ee[u] = e; }
                else ee[u] = 0.0;
                kcu[u] = kcj;
                mcu[u] = mcj;
                jlo[u + 1] = j;
            }
        } else {
#pragma unroll
            for (int u = 0; u < U; ++u) {
                if constexpr (LOGI) { e = e * qj; ee[u] = e; }
                else ee[u] = 0.0;
                const int iu = i0 + n + u;
                const int j_before = j;
                while (val[u] && iu == nb) {
                    ++j;
                    kcj = s.kc[j];
                    mcj = s.mc[j];
                    if constexpr (LOGI) qj = s.qs[j];
                    nb = j < S ? s.bidx[j] : 0x7fffffff;
                }
                if (u == 0) {
#pragma unroll 1
                    for (int jj = j_before; jj < j; ++jj) {
                        s.bndU[jj] = locU;
                        s.bndV[jj] = locV;
                    }
                }
                kcu[u] = kcj;
                mcu[u] = mcj;
                jlo[u + 1] = j;
            }
        }
        if constexpr (LOGI) {
            if (DIRECT && !erec) {                             // exponent out of the recurrence's range: direct exp
#pragma unroll
                for (int u = 0; u < U; ++u) ee[u] = exp_fastpath(-(kcu[u] * (tt[u] - mcu[u])));
            }
        }
        GPoint<LOGI, (MULT && SEAS)> pt[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            double dot = 0.0;                                  // no seasonality: additive with a zero seasonal term
            if constexpr (SEAS) {
#pragma unroll
                for (int hh = 0; hh < NH; ++hh) uw[hh][u] = fma(cw[hh], uw[hh][u ^ 1], -uw[hh][u]);
                dot = sp[u] + ((uw[0][u] + uw[1][u]) + uw[2][u]);
            }
            pt[u].run(yv[u], tt[u], dot, ee[u], kcu[u], mcu[u], cap, val[u]);
            // (beyond the lane's own points c_i = 0 and B must stand still: only the checked tail steps can get there)
            if (SEAS && (!CHECK || n + u < nown)) {
#pragma unroll
                for (int hh = 0; hh < NH; ++hh) Bw[hh][u] = fma(cw[hh], Bw[hh][u ^ 1], pt[u].cb) - Bw[hh][u];
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) tt[u] += hU;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            ss = fma(pt[u].r, pt[u].r, ss);
            if constexpr (SEAS) {
                if (val[u]) s.rtab[pu[u]] = Rv[u] + pt[u].cb;  // R_p += c_i (bins of a step are pairwise distinct)
            }
        }
        double preU[U + 1], preV[U + 1];
        preU[0] = locU;
        preV[0] = locV;
#pragma unroll
        for (int u = 0; u < U; ++u) {
            preU[u + 1] = fma(pt[u].dz, pt[u].tm, preU[u]);
            preV[u + 1] = preV[u] + pt[u].dz;
        }
        locU = preU[U];
        locV = preV[U];
        if (jlo[U] != jlo[1]) {                                  // changepoints at point u > 0: sums over the points before it
#pragma unroll
            for (int u = 1; u < U; ++u) {
#pragma unroll 1
                for (int jj = jlo[u]; jj < jlo[u + 1]; ++jj) {
                    s.bndU[jj] = preU[u];
                    s.bndV[jj] = preV[u];
                }
            }
        }
        if constexpr (SEAS) __syncwarp();                      // (the bins: all lanes of the warp step together)
    };
    PB200_PCLK_DECL(loop_t0);
    PB200_PCLK_NOW(loop_t0);
    int m = 0;
    if (LOGI && __all_sync(FULL, erec)) {              // (warp-uniform: the steps stay in lockstep for the bins)
#pragma unroll 1
        for (; m < nfull; ++m) step(m, std::false_type{}, std::false_type{});
    } else {
#pragma unroll 1
        for (; m < nfull; ++m) step(m, std::false_type{}, std::true_type{});
    }
#pragma unroll 1
    for (; m < nstep; ++m) step(m, std::true_type{}, std::true_type{});
    PB200_PCLK_ADD(PC_PASS_LOOP, clock64() - loop_t0, lane == 0);
    PB200_PCLK_ADD(PC_PASS_STEPS, nstep, lane == 0);
    PB200_PCLK_ADD(PC_PASS_WAIT, wait_cyc, lane == 0);
    if constexpr (SEAS) {   // weekly beta gradient: close the Clenshaw sums with the features of the lane's last two (padded) points
        const double2 rcw = *reinterpret_cast<const double2*>(s.rotw);
        double Y2[GKW], Y1[GKW];
        double2 w = lp.wend;                                // weekly angle at point i0 + nown - 2
        harmonics<3>(w, Y2);
        w = make_double2(fma(w.x, rcw.y, w.y * rcw.x), fma(w.y, rcw.y, -(w.x * rcw.x)));
        harmonics<3>(w, Y1);                                // ... at i0 + nown - 1
#pragma unroll
        for (int hh = 0; hh < NH; ++hh) {
            const double B1 = Bw[hh][1], B2 = Bw[hh][0];    // B at the last and the second last point
            const double D = fma(-cw[hh], B2, B1);
            gacc[2 * hh] = fma(Y1[2 * hh], D, Y2[2 * hh] * B2);
            gacc[2 * hh + 1] = fma(Y1[2 * hh + 1], D, Y2[2 * hh + 1] * B2);
        }
    }
    // ---- table features' beta gradient from the residual bins ----
    if (SEAS && active) {
        double2 w = w0;
        int p = gl * PL;
#pragma unroll 2
        for (int q = 0; q < PL; ++q, ++p) {
            if (p < P) {
                double X[GKD];
                day_features(w, X);
                const double R = s.rtab[p];
#pragma unroll
                for (int k = 0; k < GKD; ++k) gacc[GKW + k] = fma(R, X[k], gacc[GKW + k]);
            }
            const double sn = fma(w.x, rct.y, w.y * rct.x);
            const double cn = fma(w.y, rct.y, -(w.x * rct.x));
            w = make_double2(sn, cn);
        }
    }
    // boundaries recorded by this lane get the sums of the lanes before it; totals to slot S
    double totU, totV;
    const double exU = gscan_excl<G>(locU, gl, &totU), exV = gscan_excl<G>(locV, gl, &totV);
    if (active) {
#pragma unroll 1
        for (int q = j0; q < j; ++q) {
            s.bndU[q] += exU;
            s.bndV[q] += exV;
        }
        if (gl == 0) { s.bndU[S] = totU; s.bndV[S] = totV; }
    }
    __syncwarp();
    if constexpr (!SEAS) {
        // only the residual sum of squares to total; the zero column's gradient sum is zero
        ss = gsum<G>(ss);
        double* scr = s.stab;                                   // (stab and rtab are contiguous: value v at scr[v])
        if (active && gl == 0) { scr[0] = 0.0; scr[GState<G, SEAS>::TOTSS] = ss; }
        __syncwarp();
        return;
    }
    // ---- group totals of (gacc[0..13], ss): transposed through the (now dead) table storage ----
    {
        double* scr = s.stab;                                   // stab and rtab are contiguous: 2 GPT doubles
        static_assert(!SEAS || 15 * 8 <= 2 * GState<G, SEAS>::PT, "reduction scratch");
        // fold the group's upper blocks of eight lanes onto the lowest block, top block first (fixed order)
#pragma unroll
        for (int blk = G / 8 - 1; blk >= 1; --blk) {
            if (gl >= 8 * blk && gl < 8 * blk + 8) {
#pragma unroll
                for (int v = 0; v < GK; ++v) scr[v * 8 + (gl - 8 * blk)] = gacc[v];
                scr[GK * 8 + (gl - 8 * blk)] = ss;
            }
            __syncwarp();
            if (gl >= 8 * blk - 8 && gl < 8 * blk) {
#pragma unroll
                for (int v = 0; v < GK; ++v) gacc[v] += scr[v * 8 + (gl - (8 * blk - 8))];
                ss += scr[GK * 8 + (gl - (8 * blk - 8))];
            }
            __syncwarp();
        }
        if (gl < 8) {
#pragma unroll
            for (int v = 0; v < GK; ++v) scr[v * 8 + gl] = gacc[v];
            scr[GK * 8 + gl] = ss;
        }
        __syncwarp();
        // lane v (< 15; v and v + 8 when G == 8) adds up the eight partials of value v
        double t0 = 0.0, t1 = 0.0;
        if (gl < 15) {
            const int v = gl;
            if (G >= 16 || v < 8) {
#pragma unroll
                for (int q = 0; q < 8; ++q) t0 += scr[v * 8 + q];
            }
            if (G == 8 && v + 8 < 15) {
#pragma unroll
                for (int q = 0; q < 8; ++q) t1 += scr[(v + 8) * 8 + q];
            }
        }
        __syncwarp();
        // totals: value v in scr[v] (v = 0..14)
        if (active) {
            if (G >= 16) { if (gl < 15) scr[gl] = t0; }
            else { scr[gl] = t0; if (gl + 8 < 15) scr[gl + 8] = t1; }
        }
        __syncwarp();
    }
}

// ---------------------------------------------------------------------------------------
// evaluation, part 3: objective value and gradient from the pass's sums; returns err (group-uniform).  The whole warp calls
// it; an idle group (`active` false) computes on its own slot's state and stores nothing.  `gm`: the group's lane mask
// ---------------------------------------------------------------------------------------
template <int G, bool LOGI, bool SEAS>
__device__ __noinline__ int g_eval_finalize(GState<G, SEAS>& s, const double* xv, double* gv, const int gl, const unsigned gm,
                                            const bool active, double* f_out) {
    constexpr int NS = GSEG / G;
    const int S = s.S, T = s.T, jb = gl * NS;
    const SeriesPrior& pr = gprior<G, SEAS>((threadIdx.x & 31) / G);
    const double tau = pr.tau, rtau = pr.rtau, inv_seas2 = pr.inv_seas2;
    const double* tot = s.stab;                     // value v of the pass: tot[v], v < 14 beta sums, tot[14] = ss
    const double ss = tot[GState<G, SEAS>::TOTSS];
    const double sigma = s.sigma;
    const double inv_s2 = rcp_any(sigma * sigma);
    const double scale = -inv_s2;
    const double k = xv[0], m = xv[1], u_ = xv[2 + S];
    const double totU = s.bndU[S], totV = s.bndV[S];
    int bad = 0;
    double kb_part = 0.0, ad_part = 0.0;
    double gm_ = 0.0;
    if constexpr (LOGI) {
        // per-segment sums dU_j, dV_j from the boundary prefixes; adjoints of rate and offset
        double PU[NS + 1], PV[NS + 1], kcl[NS + 1], mcl[NS], rhl[NS], tcl[NS], Gkc[NS], Gmc[NS];
        {
            const int jm = jb - 1;
            PU[0] = jm < 0 ? 0.0 : (jm <= S ? s.bndU[jm] : totU);
            PV[0] = jm < 0 ? 0.0 : (jm <= S ? s.bndV[jm] : totV);
        }
#pragma unroll
        for (int u = 0; u < NS; ++u) {
            const int j = jb + u;
            PU[u + 1] = j <= S ? s.bndU[j] : totU;
            PV[u + 1] = j <= S ? s.bndV[j] : totV;
            kcl[u] = j <= S ? s.kc[j] : 1.0;
            mcl[u] = j <= S ? s.mc[j] : 0.0;
            rhl[u] = 1.0;                                   // rho_j = k_j / k_{j+1}: recomputed below (same expression as g_eval_setup)
            tcl[u] = j < S ? s.tc[j] : 0.0;
            Gkc[u] = j <= S ? scale * (PU[u + 1] - PU[u]) : 0.0;
            Gmc[u] = j <= S ? scale * (-kcl[u]) * (PV[u + 1] - PV[u]) : 0.0;
        }
        kcl[NS] = __shfl_down_sync(FULL, kcl[0], 1, G);
        if (jb + NS > S) kcl[NS] = 1.0;
#pragma unroll
        for (int u = 0; u < NS; ++u)
            if (jb + u < S) rhl[u] = div_const(kcl[u], kcl[u + 1], rcp_any(kcl[u + 1]));
        // abar_S = Gmc_S, abar_j = Gmc_j + rho_j abar_{j+1}: reverse scan of the affine maps x -> a x + b
        // (a, b) = (rho_j, Gmc_j) for j < S, (0, Gmc_S) at j = S, identity above
        double ma[NS], mb[NS], A = 1.0, B = 0.0;
#pragma unroll
        for (int u = NS - 1; u >= 0; --u) {
            const int j = jb + u;
            ma[u] = j < S ? rhl[u] : (j == S ? 0.0 : 1.0);
            mb[u] = j <= S ? Gmc[u] : 0.0;
            // block map = map_first o ... o map_last: compose towards lower u
            B = fma(ma[u], B, mb[u]);
            A = ma[u] * A;
        }
        double Ai = A, Bi = B;
#pragma unroll
        for (int o = 1; o < G; o <<= 1) {
            const double An = __shfl_down_sync(FULL, Ai, o, G);
            const double Bn = __shfl_down_sync(FULL, Bi, o, G);
            if (gl + o < G) { Bi = fma(Ai, Bn, Bi); Ai = Ai * An; }
        }
        // value entering this block from above = (inclusive map of the next lane)(0)
        double xin = __shfl_down_sync(FULL, Bi, 1, G);
        if (gl == G - 1) xin = 0.0;
        double ab[NS + 1];
        ab[NS] = xin;
#pragma unroll
        for (int u = NS - 1; u >= 0; --u) ab[u] = fma(ma[u], ab[u + 1], mb[u]);
        // rate adjoints: kbar_j = Gkc_j + rb_j / k_{j+1} - (rb_{j-1} rho_{j-1}) / k_j,  rb_j = abar_{j+1} (m_j - t_change_j)
        double t2[NS], kbar[NS];
#pragma unroll
        for (int u = 0; u < NS; ++u) {
            const int j = jb + u;
            const double rb = j < S ? ab[u + 1] * (mcl[u] - tcl[u]) : 0.0;
            const double rk = rcp_any(kcl[u + 1]);
            const double t1 = j < S ? div_const(rb, kcl[u + 1], rk) : 0.0;
            t2[u] = j < S ? div_const(-(rb * rhl[u]), kcl[u + 1], rk) : 0.0;
            kbar[u] = j <= S ? Gkc[u] + t1 : 0.0;
        }
        double t2prev = __shfl_up_sync(FULL, t2[NS - 1], 1, G);
        if (gl == 0) t2prev = 0.0;
#pragma unroll
        for (int u = 0; u < NS; ++u) {
            const int j = jb + u;
            if (j <= S) kbar[u] += u == 0 ? t2prev : t2[u - 1];
        }
        // gd_s = sum_{j > s} kbar_j  (reverse inclusive scan, shifted by one)
        double suf[NS + 1], run = 0.0;
#pragma unroll
        for (int u = NS - 1; u >= 0; --u) { run += kbar[u]; suf[u] = run; }
        const double above = gscan_excl_rev<G>(run, gl);
        suf[NS] = 0.0;
#pragma unroll
        for (int u = 0; u < NS; ++u) {
            const int j = jb + u;            // delta index j: gradient = sum over segments > j
            if (j < S) {
                const double d = xv[2 + j];
                const double sg = d > 0.0 ? 1.0 : (d < 0.0 ? -1.0 : 0.0);
                const double gd = (above + suf[u + 1]) + div_const(sg, tau, rtau);
                if (active) gv[2 + j] = gd;
                if (!isfinite(gd)) bad = 1;
                ad_part += fabs(d);
            }
        }
        kb_part = run;
        gm_ = __shfl_sync(FULL, ab[0], 0, G) + div_const(m, 25.0, 0.04);
    } else {
#pragma unroll
        for (int u = 0; u < NS; ++u) {
            const int j = jb + u;
            if (j < S) {
                const double d = xv[2 + j];
                const double sg = d > 0.0 ? 1.0 : (d < 0.0 ? -1.0 : 0.0);
                const double gd = scale * ((totU - s.bndU[j]) - s.tc[j] * (totV - s.bndV[j])) + div_const(sg, tau, rtau);
                if (active) gv[2 + j] = gd;
                if (!isfinite(gd)) bad = 1;
                ad_part += fabs(d);
            }
        }
        gm_ = scale * totV + div_const(m, 25.0, 0.04);
    }
    // beta gradient and prior
    double pb = 0.0;
#pragma unroll
    for (int u = 0; u < (gkx<SEAS>() + G - 1) / G; ++u) {
        const int q = gl + u * G;
        if (q < gkx<SEAS>()) {
            const double b = xv[3 + S + q];
            const double gb = scale * tot[q] + b * inv_seas2;
            if (active) gv[3 + S + q] = gb;
            pb += 0.5 * b * b * inv_seas2;
            if (!isfinite(gb)) bad = 1;
        }
    }
    const double kb_sum = gsum<G>(kb_part), pb_sum = gsum<G>(pb), ad = gsum<G>(ad_part);
    const double k25 = div_const(k, 25.0, 0.04);
    const double gk = LOGI ? kb_sum + k25 : scale * totU + k25;
    const double gu = -ss * inv_s2 + (double)T + 4.0 * sigma * sigma;
    const double f = 0.5 * ss * inv_s2 + (double)T * u_ + div_const(k * k, 50.0, 0.02) + div_const(m * m, 50.0, 0.02) +
                     div_const(ad, tau, rtau) + 2.0 * sigma * sigma + pb_sum;
    if (gl == 0) {
        if (active) { gv[0] = gk; gv[1] = gm_; gv[2 + S] = gu; }
        if (!isfinite(gk) || !isfinite(gm_) || !isfinite(gu)) bad = 1;
    }
    if (!isfinite(f) || !(sigma > 0.0) || !isfinite(sigma)) bad = 1;
    bad = (__ballot_sync(FULL, bad) & gm) != 0;
    if (active && gl == 0) *f_out = f;             // (nothing here reads it: the caller's __syncwarp publishes it)
    return bad;
}

// ---------------------------------------------------------------------------------------
// Stan's L-BFGS over the group's LSState (see fit_kernel.cuh for the routine-by-routine mapping).  The whole warp calls
// each routine once per round, and a group's action is a register value: every group computes the routine's dot products
// under the full mask, and only the groups whose action uses one keep it.  A routine reads the LSState scalars once, and
// lane 0 stores the new ones once, behind one __syncwarp (the lanes of its group have read the old ones by then)
// ---------------------------------------------------------------------------------------
// actions besides fit_kernel.cuh's ACT_EVAL / ACT_ACCEPT / ACT_FAIL: none (idle, or done this round), and the three ways
// into a new line search: the first iteration, the retry from a reset Hessian after a failed search, the next iteration
// after an accepted one
constexpr int ACT_NONE = -1, ACT_BEGIN_FIRST = ACT_FAIL + 1, ACT_BEGIN_RETRY = ACT_FAIL + 2, ACT_BEGIN_NEXT = ACT_FAIL + 3;

// WolfeLineSearch / WolfLSZoom after the evaluation at the trial point.  Groups that are not in a line search (`search`
// false) return ACT_NONE.  ACT_EVAL: alpha is the step of the next trial point, which g_ls_begin forms.  (Returned by value:
// an out-pointer to the caller's register would put it on the stack)
struct LsStep {
    int act;
    double alpha;
};
template <int G, bool SEAS>
__device__ __noinline__ LsStep g_ls_step(GState<G, SEAS>& s, const int gl, const bool search, const int P, const int err) {
    LSState& ls = s.ls;
    const double c1 = 1e-4, c2 = 0.9, min_range = 1e-16;
    const int maxLSIts = 20, maxLSRestarts = 10;
    // the directional derivative at the trial point (the groups with err, or not searching, discard it)
    const double newDFp = gvdot<G, GState<G, SEAS>::PPAD>(s.vec[ls.igt], s.vec[ls.ip], P, gl);
    const double fk = ls.fk, ft = ls.ft, dfp = ls.dfp;
    const double c1dfp = c1 * dfp, c2dfp = c2 * dfp;
    double alpha = ls.alpha, alpha0 = ls.alpha0, prevF = ls.prevF, prevDFp = ls.prevDFp;
    double alo = ls.alo, aloF = ls.aloF, aloD = ls.aloD, ahi = ls.ahi, ahiF = ls.ahiF, ahiD = ls.ahiD;
    int itNum = ls.itNum, nits = ls.nits, lsRestarts = ls.lsRestarts, phase = ls.phase;
    // Stan's decisions on the local copies; every ACT_EVAL leaves the new state in them
    auto decide = [&]() -> int {
        if (phase == PH_LS) {
            // ---------------- WolfeLineSearch ----------------
            if (err) {
                if (lsRestarts >= maxLSRestarts) return ACT_FAIL;
                alpha = 0.5 * (alpha0 + alpha);
                lsRestarts += 1;
                return ACT_EVAL;
            }
            if (ft > fk + alpha * c1dfp || (ft >= prevF && nits > 0)) {
                alo = alpha0; aloF = prevF; aloD = prevDFp;
                ahi = alpha; ahiF = ft; ahiD = newDFp;
            } else if (fabs(newDFp) <= -c2dfp) {
                return ACT_ACCEPT;
            } else if (newDFp >= 0) {
                alo = alpha; aloF = ft; aloD = newDFp;
                ahi = alpha0; ahiF = prevF; ahiD = prevDFp;
            } else {
                if (nits + 1 >= maxLSIts) return ACT_FAIL;
                const double a10 = alpha * 10.0;
                alpha0 = alpha; prevF = ft; prevDFp = newDFp; alpha = a10; nits += 1;
                lsRestarts = 0;
                return ACT_EVAL;
            }
            itNum = 0;
        } else {
            // ---------------- WolfLSZoom: result of the evaluation at alpha ----------------
            if (err) {
                const double lo = fmin(alo, ahi);
                alpha = 0.5 * (alpha + lo);
                if (fabs(lo - alpha) < min_range) return ACT_FAIL;
                return ACT_EVAL;
            }
            if (ft > (fk + alpha * c1dfp) || ft >= aloF) {
                ahi = alpha; ahiF = ft; ahiD = newDFp;
            } else {
                if (fabs(newDFp) <= -c2dfp) return ACT_ACCEPT;
                if (newDFp * (ahi - alo) >= 0) { ahi = alo; ahiF = aloF; ahiD = aloD; }
                alo = alpha; aloF = ft; aloD = newDFp;
            }
        }
        // ---------------- WolfLSZoom: next trial step ----------------
        ++itNum;
        if (fabs(alo - ahi) < min_range) return ACT_FAIL;
        {
            // [guard, not in Stan] bracket = two adjacent doubles wider than min_range (see fit_kernel.cuh)
            const double mid = 0.5 * (alo + ahi);
            if (mid == alo || mid == ahi) return ACT_FAIL;
        }
        if (itNum % 5 == 0) {
            alpha = 0.5 * (alo + ahi);
        } else {
            const double d1 = aloD + ahiD - fdiv(3 * (aloF - ahiF), alo - ahi);
            double d2 = sqrt(d1 * d1 - aloD * ahiD);
            if (ahi < alo) d2 = -d2;
            alpha = ahi - fdiv((ahi - alo) * (ahiD + d2 - d1), ahiD - aloD + 2 * d2);
            const double lo = fmin(alo, ahi), hi = fmax(alo, ahi);
            if (!isfinite(alpha) || alpha < lo + 0.01 * fabs(alo - ahi) || alpha > hi - 0.01 * fabs(alo - ahi))
                alpha = 0.5 * (alo + ahi);
        }
        phase = PH_ZOOM;
        return ACT_EVAL;
    };
    const int act = search ? decide() : ACT_NONE;
    __syncwarp();
    if (act == ACT_EVAL && gl == 0) {          // (fields a branch leaves alone are stored back unchanged)
        ls.alpha = alpha; ls.alpha0 = alpha0; ls.prevF = prevF; ls.prevDFp = prevDFp;
        ls.alo = alo; ls.aloF = aloF; ls.aloD = aloD; ls.ahi = ahi; ls.ahiF = ahiF; ls.ahiD = ahiD;
        ls.itNum = itNum; ls.nits = nits; ls.lsRestarts = lsRestarts; ls.phase = phase;
    }
    return {act, alpha};
}

// A new line search for the groups that start one (act ACT_BEGIN_*): the direction is -g after a reset Hessian, and the
// initial step comes from Stan's cubic interpolation over the previous iteration.  Then the trial point x + alpha p of
// every group that evaluates one next: those groups and the ACT_EVAL ones (alpha = talpha)
template <int G, bool SEAS>
__device__ __noinline__ void g_ls_begin(GState<G, SEAS>& s, const int gl, const int P, const double init_alpha, const int act,
                                        const double talpha) {
    constexpr int NV = (GState<G, SEAS>::PPAD + G - 1) / G;
    LSState& ls = s.ls;
    const double minAlpha = 1e-12;
    const bool begin = act >= ACT_BEGIN_FIRST, trial = begin || act == ACT_EVAL;
    const int iters = act == ACT_BEGIN_FIRST ? 1 : (act == ACT_BEGIN_NEXT ? ls.iters + 1 : ls.iters);
    const int resetB = act == ACT_BEGIN_FIRST ? 1 : (act == ACT_BEGIN_RETRY ? 2 : (act == ACT_BEGIN_NEXT ? 0 : ls.resetB));
    const double fk = ls.fk;
    const double* x = s.vec[ls.ix];
    const double* g = s.vec[ls.ig];
    double* p = s.vec[ls.ip];
    double* xt = s.vec[ls.ixt];
    const bool neg = begin && resetB != 0;                 // the direction starts over at -g
    double pv[NV], l = 0.0;
#pragma unroll
    for (int u = 0; u < NV; ++u) {
        const int q = gl + u * G;
        pv[u] = 0.0;
        if (q < P) {
            pv[u] = neg ? -g[q] : p[q];
            l = fma(g[q], pv[u], l);
        }
    }
    const double dfp = gsum<G>(l);
    const double dprev = gvdot<G, GState<G, SEAS>::PPAD>(s.vec[ls.igt], s.vec[ls.ipp], P, gl);
    double alpha = talpha;
    if (begin) {
        if (iters > 1 && resetB != 2) alpha = fmin(1.0, 1.01 * cubic_interp(dprev, ls.alphak_1, fk - ls.fk_1, dfp, minAlpha, 1.0));
        else alpha = init_alpha;
    }
#pragma unroll
    for (int u = 0; u < NV; ++u) {
        const int q = gl + u * G;
        if (trial && q < P) {
            if (neg) p[q] = pv[u];
            xt[q] = x[q] + alpha * pv[u];
        }
    }
    __syncwarp();
    if (begin && gl == 0) {
        ls.dfp = dfp; ls.alpha = alpha; ls.alpha0 = minAlpha; ls.prevF = fk; ls.prevDFp = dfp;
        ls.nits = 0; ls.lsRestarts = 0; ls.phase = PH_LS; ls.iters = iters; ls.resetB = resetB;
        if (act == ACT_BEGIN_FIRST) s.state = ST_SEARCH;
    }
}

// the rest of BFGSMinimizer::step after an accepted line search; history Y[5], S[5] in global memory `hist`.
// The whole warp calls it, `acc` set in the groups whose line search was accepted: with every lane present the group
// reductions shuffle under the full mask (a group's lane mask is not known at compile time, and a shuffle under it first
// has to test which lanes take part).  The other groups run on zeros from their own slot and store nothing
template <int G, bool SEAS>
__device__ __noinline__ int g_post_accept(GState<G, SEAS>& s, double* hist, const int gl, const bool acc, const int P_,
                                          const FitOptsDev& o, double* trace, const int trace_cap, const int l2f) {
    constexpr int NV = (GState<G, SEAS>::PPAD + G - 1) / G;
    LSState& ls = s.ls;
    double* HY = hist;
    double* HS = hist + HMAX * GPPAD;
    const int P = acc ? P_ : 0;
    const int ix = acc ? ls.ixt : 0, ixt = acc ? ls.ix : 0, ig = acc ? ls.igt : 0, igt = acc ? ls.ig : 0;
    const int ip = acc ? ls.ipp : 0, ipp = acc ? ls.ip : 0;
    const double* x = s.vec[ix];
    const double* xt = s.vec[ixt];
    const double* g = s.vec[ig];
    const double* gt = s.vec[igt];
    double* p = s.vec[ip];
    double* pp = s.vec[ipp];
    const double fk_1 = ls.fk, fk = ls.ft, alpha = ls.alpha;
    const int resetB = acc ? ls.resetB : 0, H = o.history;
    int hn = acc ? ls.hn : 0, hhead = acc ? ls.hhead : 0;
    if (acc && trace && gl == 0 && ls.iters <= trace_cap) {
        double* tr = trace + (size_t)(ls.iters - 1) * 4;
        tr[0] = (double)ls.iters; tr[1] = fk; tr[2] = alpha; tr[3] = (double)ls.nevals;
    }
    // ---- LBFGSUpdate::update ----
    if (resetB) { hn = 0; hhead = 0; }
    int slot;
    if (hn < H) { slot = hhead + hn; if (slot >= H) slot -= H; ++hn; }
    else { slot = hhead; hhead = hhead + 1 == H ? 0 : hhead + 1; }
    // The new pair is position hn - 1 of the recursion order, whether the history is filling or full: it stays in registers
    // of its own (sn, yn, and 1 / s.y in rn).  The ho = hn - 1 older pairs, position h at slot (hhead + h) mod H, are loaded
    // up front (one L2 round trip) with their 1 / s.y
    const int ho = hn - 1;
    const unsigned long long pol_h = l2_policy(l2f);
    double hy[HMAX - 1][NV], hs[HMAX - 1][NV], hr[HMAX - 1];
#pragma unroll
    for (int h = 0; h < HMAX - 1; ++h) {
        int sl = hhead + h;
        if (sl >= H) sl -= H;
        const double* const hyp = HY + (sl * GPPAD + gl);         // (element u of the lane: a constant offset u G)
        const double* const hsp = HS + (sl * GPPAD + gl);
        hr[h] = h < ho ? s.hrho[sl] : 0.0;
#pragma unroll
        for (int u = 0; u < NV; ++u) {
            const int q = gl + u * G;
            const bool ld = h < ho && q < P;
            hy[h][u] = ld ? ldcg_hint(hyp + u * G, pol_h) : 0.0;
            hs[h][u] = ld ? ldcg_hint(hsp + u * G, pol_h) : 0.0;
        }
    }
    double nrm0 = 0.0, nrm1 = 0.0, nrm2 = 0.0, nrm3 = 0.0;   // s.y, y.y, s.s, g.g
    double gq[NV], sn[NV], yn[NV];
    double* const hyn = HY + (slot * GPPAD + gl);
    double* const hsn = HS + (slot * GPPAD + gl);
#pragma unroll
    for (int u = 0; u < NV; ++u) {
        const int q = gl + u * G;
        double sv = 0.0, yv = 0.0;
        gq[u] = 0.0;
        if (q < P) {
            sv = x[q] - xt[q];
            yv = g[q] - gt[q];
            gq[u] = g[q];
            stcg_hint(hsn + u * G, sv, pol_h);                  // (P = 0 outside the accepted groups)
            stcg_hint(hyn + u * G, yv, pol_h);
        }
        sn[u] = sv;
        yn[u] = yv;
        nrm0 = fma(sv, yv, nrm0); nrm1 = fma(yv, yv, nrm1);
        nrm2 = fma(sv, sv, nrm2); nrm3 = fma(gq[u], gq[u], nrm3);
    }
    const double skyk = gsum<G>(nrm0), ykyk = gsum<G>(nrm1);
    const double stepNorm = sqrt(gsum<G>(nrm2));
    const double gradNorm = sqrt(gsum<G>(nrm3));
    double alphak_1;
    if (resetB) {
        const double B0 = fdiv(ykyk, skyk), rB0 = rcp_any(B0);
#pragma unroll
        for (int u = 0; u < NV; ++u) {
            const int q = gl + u * G;
            if (q < P) pp[q] = div_const(pp[q], B0, rB0);
        }
        alphak_1 = alpha * B0;
    } else {
        alphak_1 = alpha;
    }
    const double gammak = fdiv(skyk, ykyk);
    const double rn = rcp_any(skyk);
    if (acc && gl == 0) s.hrho[slot] = rn;                          // (read by the calls that follow, after their own syncs)
#ifdef PB200_PHASE_CLOCKS
    {   // the history loads' exposed round trip: wait for all of them here, where the recursion first needs them
        const long long t0 = clock64();
        double chk = 0.0;
#pragma unroll
        for (int h = 0; h < HMAX - 1; ++h)
#pragma unroll
            for (int u = 0; u < NV; ++u) chk += hy[h][u] + hs[h][u];
        if (__double_as_longlong(chk) == 0x7ff8dead00000000ll) s.hrho[7] = chk;     // (never true: makes the wait real)
        PB200_PCLK_ADD(PC_POST_HIST, clock64() - t0, (threadIdx.x & 31) == __ffs(__activemask()) - 1);
    }
#endif
    // ---- LBFGSUpdate::search_direction (two-loop recursion): newest pair first in the first loop, last in the second ----
    double pv[NV], hal[HMAX - 1];
#pragma unroll
    for (int u = 0; u < NV; ++u) pv[u] = -gq[u];
    double aln;
    {
        double l = 0.0;
#pragma unroll
        for (int u = 0; u < NV; ++u) l = fma(sn[u], pv[u], l);
        aln = rn * gsum<G>(l);
#pragma unroll
        for (int u = 0; u < NV; ++u) pv[u] -= aln * yn[u];
    }
#pragma unroll
    for (int h = HMAX - 2; h >= 0; --h) {       // (positions h >= ho: every lane shuffles, nothing is kept)
        double l = 0.0;
#pragma unroll
        for (int u = 0; u < NV; ++u) l = fma(hs[h][u], pv[u], l);
        const double al = hr[h] * gsum<G>(l);
        const bool on = h < ho;
#pragma unroll
        for (int u = 0; u < NV; ++u) pv[u] = on ? pv[u] - al * hy[h][u] : pv[u];
        hal[h] = on ? al : 0.0;
    }
#pragma unroll
    for (int u = 0; u < NV; ++u) pv[u] *= gammak;
#pragma unroll
    for (int h = 0; h < HMAX - 1; ++h) {
        double l = 0.0;
#pragma unroll
        for (int u = 0; u < NV; ++u) l = fma(hy[h][u], pv[u], l);
        const double be = hr[h] * gsum<G>(l);
        const double cf = hal[h] - be;
        const bool on = h < ho;
#pragma unroll
        for (int u = 0; u < NV; ++u) pv[u] = on ? pv[u] + cf * hs[h][u] : pv[u];
    }
    {
        double l = 0.0;
#pragma unroll
        for (int u = 0; u < NV; ++u) l = fma(yn[u], pv[u], l);
        const double be = rn * gsum<G>(l);
        const double cf = aln - be;
#pragma unroll
        for (int u = 0; u < NV; ++u) pv[u] += cf * sn[u];
    }
    double gpl = 0.0;
#pragma unroll
    for (int u = 0; u < NV; ++u) {
        const int q = gl + u * G;
        if (q < P) p[q] = pv[u];
        gpl = fma(gq[u], pv[u], gpl);
    }
    const double gp = gsum<G>(gpl);
    // ---- convergence tests ----
    const double df = fabs(fk_1 - fk);
    int status = PB200_ST_SUCCESS;
    if (df < o.tol_obj) status = PB200_ST_ABSF;
    else if (df < o.tol_rel_obj_eps * fmax(fabs(fk_1), fmax(fabs(fk), 1.0))) status = PB200_ST_RELF;
    else if (gradNorm < o.tol_grad) status = PB200_ST_ABSGRAD;
    else if (fabs(gp) < o.tol_rel_grad_eps * fmax(fabs(fk), 1.0)) status = PB200_ST_RELGRAD;
    else if (stepNorm < o.tol_param) status = PB200_ST_ABSX;
    else if (ls.iters >= o.max_iter) status = PB200_ST_MAXIT;
    __syncwarp();
    if (acc && gl == 0) {
        ls.ix = ix; ls.ixt = ixt; ls.ig = ig; ls.igt = igt; ls.ip = ip; ls.ipp = ipp;
        ls.fk_1 = fk_1; ls.fk = fk; ls.alphak_1 = alphak_1; ls.hn = hn; ls.hhead = hhead;
        ls.status = status;
    }
    __syncwarp();
    return status;
}

// ---------------------------------------------------------------------------------------
// fetch the next series of the queue into this group's slot: stage y, phases, changepoints, initial point
// returns false when the queue is exhausted
// ---------------------------------------------------------------------------------------
template <int G, bool LOGI, bool SEAS>
__device__ __noinline__ bool g_fetch(GState<G, SEAS>& s, const FitArgs& a, double* plane, const int gl, const unsigned gm,
                                     const int l2f) {
    const unsigned long long pol_y = l2_policy(l2f), pol_in = l2_policy(l2f & L2F_REST_FIRST);
    if (gl == 0) {
        const int pos = atomicAdd(a.q_head, 1);
        s.series = pos < *a.q_count ? a.q_items[pos] : -1;
    }
    __syncwarp(gm);
    const int sidx = s.series;
    if (sidx < 0) return false;
    const int* mi = a.meta_i32 + (size_t)sidx * 8;
    const long long* ml = a.meta_i64 + (size_t)sidx * 2;
    const double* mf = a.meta_f64 + (size_t)sidx * 4;
    const int T = mi[0], S = mi[1], ncp = mi[2], st0 = mi[4], i1max = mi[7];
    const long long start = ml[0], tscale = ml[1];
    const double y_scale = mf[0], fl = mf[1], capv = mf[2];
    const long long off = a.offsets[sidx];
    const long long step = a.ds[off + 1] - a.ds[off];
    const int tabP = SEAS ? (int)((86400LL * 1000000000LL) / step) : 0;
    const int chunk = SEAS ? grp_chunk(T, tabP, G, grp_u(G)) : grp_chunk_plain(T, G);
    const double dts = (double)tscale;
    const double cap_s = LOGI ? (capv - fl) / y_scale : 0.0;
    const int PL = (tabP + G - 1) / G;
    __syncwarp(gm);
    if (gl == 0) {
        s.T = T; s.S = S; s.ncp = ncp; s.chunk = chunk; s.tabP = tabP; s.tabPL = PL;
        s.cap_s = cap_s; s.hstep = (double)step / dts; s.st0 = st0; s.i1max = i1max; s.exprec = 0;
        SeriesPrior& pr = gprior<G, SEAS>((threadIdx.x & 31) / G);
        pr = series_prior(a.prior, a.o, sidx);
        // (the all-zero column of the class without seasonality has prior scale 1: fbprophet's make_all_seasonality_features)
        if constexpr (!SEAS) pr.inv_seas2 = 1.0;
        if constexpr (SEAS) {
            const double dt_d = (1e-9 * (double)step) / 86400.0;
            double s_, c_;
            sincos(TWO_PI_FL * dt_d / 7.0, &s_, &c_);
            s.rotw[0] = s_; s.rotw[1] = c_;
            sincos(TWO_PI_FL * dt_d / 1.0, &s_, &c_);
            s.rotd[0] = s_; s.rotd[1] = c_;
        }
        LSState& ls = s.ls;
        ls.ix = 0; ls.ig = 1; ls.ip = 2; ls.ixt = 3; ls.igt = 4; ls.ipp = 5;
        ls.iters = 0; ls.nevals = 0; ls.resetB = 1; ls.hn = 0; ls.hhead = 0;
        ls.fk = NAN; ls.fk_1 = 0.0; ls.ft = 0.0; ls.alphak_1 = 0.0; ls.alpha = 0.0;
        ls.alo = ls.aloF = ls.aloD = ls.ahi = ls.ahiF = ls.ahiD = 0.0; ls.itNum = 0;
        ls.status = st0;
    }
    // ---- stage y (the only HBM read of the series) as point pairs; lane l owns points [l chunk, (l + 1) chunk).  The stores
    // set the slot's L2 priority at first touch ----
#pragma unroll 1
    for (int i = gl; i < T; i += G) {
        const double yv = load_y_hint(a.y, a.y_dtype, off + i, pol_in);
        constexpr int U = grp_u(G);
        const int own = i / chunk, n = i - own * chunk;
        st_hint(&plane[((size_t)(n / U) * G + own) * U + (n % U)], (yv - fl) / y_scale, pol_y);
    }
    // ---- per-lane start phases: weekly angle at the lane's first point, daily angle at its first table phase ----
    if constexpr (SEAS) {
        const long long d0 = a.ds[off];
        const int i0 = gl * chunk;
        const double tw = (1e-9 * (double)(d0 + (long long)(i0 - 2) * step)) / 86400.0;     // two points before the chunk
        double s_, c_;
        sincos(TWO_PI_FL * tw / 7.0, &s_, &c_);
        reinterpret_cast<double2*>(&s.vec[1][0])[gl] = make_double2(s_, c_);    // LanePhase hand-over through the vectors that are dead until the first evaluation, see the kernel
        const double td = (1e-9 * (double)(d0 + (long long)(gl * PL) * step)) / 86400.0;
        sincos(TWO_PI_FL * td / 1.0, &s_, &c_);
        reinterpret_cast<double2*>(&s.vec[1][0])[G + gl] = make_double2(s_, c_);
        const int i1 = i0 + chunk < T ? i0 + chunk : T, np_ = i1 > i0 ? i1 - i0 : 0;
        const double te = (1e-9 * (double)(d0 + (long long)(i0 + 2 * ((np_ + 1) >> 1) - 2) * step)) / 86400.0;
        sincos(TWO_PI_FL * te / 7.0, &s_, &c_);
        reinterpret_cast<double2*>(&s.vec[1][0])[2 * G + gl] = make_double2(s_, c_);
    }
    // ---- changepoints (Prophet.set_changepoints) and segment boundaries ----
#pragma unroll 1
    for (int q = gl; q < GSEG; q += G) {
        if (q < S) {
            double tcv;
            int b;
            if (ncp > 0) {
                const int hist = (int)floor((double)T * a.o.changepoint_range);
                const double stp = (double)(hist - 1) / (double)ncp;
                const int idx = q == ncp - 1 ? hist - 1 : (int)rint((double)(q + 1) * stp);
                tcv = (double)(a.ds[off + idx] - start) / dts;
                b = idx;                                     // regular grid: timestamps strictly increase
            } else {
                tcv = 0.0;
                b = 0;
            }
            s.tc[q] = tcv;
            s.bidx[q] = b;
            a.tchange[(size_t)sidx * a.smax + q] = tcv;
        } else {
            s.bidx[q] = 0x7fffffff;
        }
    }
#pragma unroll 1
    for (int q = S + gl; q < a.smax; q += G) a.tchange[(size_t)sidx * a.smax + q] = 0.0;
    __syncwarp(gm);
    {
        const int i0 = gl * chunk < T ? gl * chunk : T;
        int j0 = 0;
#pragma unroll 1
        for (int q = 0; q < S; ++q) j0 += s.bidx[q] < i0 ? 1 : 0;
        reinterpret_cast<int*>(&s.vec[1][0] + (SEAS ? 6 * G : 0))[gl] = j0;
    }
    // ---- initial point: Prophet.{linear,logistic}_growth_init + stan_init ----
    {
        const int P = S + gkx<SEAS>() + 3;
        const double y0 = (load_y(a.y, a.y_dtype, off) - fl) / y_scale;
        const double y1 = (load_y(a.y, a.y_dtype, off + i1max) - fl) / y_scale;
        const double t1v = (double)(a.ds[off + i1max] - start) / dts;
        double k0, m0;
        if constexpr (LOGI) {
            const double C0 = cap_s;
            const double yy0 = fmax(0.01 * C0, fmin(0.99 * C0, y0));
            const double yy1 = fmax(0.01 * C0, fmin(0.99 * C0, y1));
            double r0 = C0 / yy0;
            const double r1 = C0 / yy1;
            if (fabs(r0 - r1) <= 0.01) r0 = 1.05 * r0;
            const double L0 = log(r0 - 1.0), L1 = log(r1 - 1.0);
            m0 = L0 * t1v / (L0 - L1);
            k0 = (L0 - L1) / t1v;
        } else {
            k0 = (y1 - y0) / t1v;
            m0 = y0 - k0 * 0.0;
        }
        double* x = s.vec[0];
        const double* th = a.theta_in ? a.theta_in + (size_t)sidx * a.pstride : nullptr;
        if (th && !a.grad_out && !(th[0] == th[0])) th = nullptr;     // warm start: this series starts cold
#pragma unroll 1
        for (int q = gl; q < P; q += G) x[q] = th ? th[q] : (q == 0 ? k0 : (q == 1 ? m0 : 0.0));
    }
    __threadfence_block();
    __syncwarp(gm);
    return true;
}

// write the model record of the group's series (Stan's unconstrained optimum -> k, m, sigma_obs, delta, beta)
template <int G, bool SEAS>
__device__ __noinline__ void g_write_record(GState<G, SEAS>& s, const FitArgs& a, const int status, const int gl, const unsigned gm) {
    const int sidx = s.series, S = s.S, ncp = s.ncp;
    const double* x = s.vec[s.ls.ix];
    double* pr = a.params + (size_t)sidx * a.pstride;
    double kf = x[0];
    const double mfv = x[1];
    double sg = exp(x[2 + S]);
    if (status == PB200_ST_CONST_LINEAR) sg = 1e-9;
    if (ncp == 0) kf = kf + x[2];
#pragma unroll 1
    for (int q = gl; q < a.pstride; q += G) {
        double v = 0.0;
        if (q == 0) v = kf;
        else if (q == 1) v = mfv;
        else if (q == 2) v = sg;
        else if (q < 3 + a.smax) {
            const int c = q - 3;
            v = (c < S && ncp > 0) ? x[2 + c] : 0.0;
        } else {
            const int b = q - 3 - a.smax;
            v = b < gkx<SEAS>() ? x[3 + S + b] : 0.0;
        }
        pr[q] = v;
    }
    if (a.grad_out) {
        const double* g = s.vec[s.ls.ig];
        double* go = a.grad_out + (size_t)sidx * a.pstride;
        const int P = S + gkx<SEAS>() + 3;
#pragma unroll 1
        for (int q = gl; q < a.pstride; q += G) go[q] = q < P ? g[q] : 0.0;
    }
    if (gl == 0) {
        int* mi = a.meta_i32 + (size_t)sidx * 8;
        double* mf = a.meta_f64 + (size_t)sidx * 4;
        mi[4] = status; mi[5] = s.ls.iters; mi[6] = s.ls.nevals;
        mf[3] = s.ls.fk;
        if (status == PB200_ST_LSFAIL && a.nq_items) {          // fbprophet's Newton retry picks it up (newton_kernel)
            const int pos = atomicAdd(a.nq_count, 1);
            a.nq_items[pos] = sidx;
        }
    }
    __syncwarp(gm);
}

// ---------------------------------------------------------------------------------------
// the kernel: one warp per CTA, 32 / G series in flight per warp, persistent over the class's work queue
// ---------------------------------------------------------------------------------------
template <int G, bool LOGI, bool MULT, bool SEAS>
#ifndef PB200_GRP_BLOCKS
// resident one-warp CTAs per SM the G = 8 register budget is set for.  8 -> 242 registers on sm_90a; 9 -> spills in
// g_post_accept, which measured slower.  On an H100 a 50k x 1440 step takes 35 % less time with 8 CTAs per SM than with 4
// (DESIGN §3)
#define PB200_GRP_BLOCKS 8
#endif
#ifndef PB200_GRP_PLAIN_BLOCKS
// ... and for the class without seasonality, whose time DOES fall as resident warps rise (500k short series at
// 4 to 8 CTAs per SM): short point loops, the latency of the serial code dominates
#define PB200_GRP_PLAIN_BLOCKS 14
#endif
__global__ void __launch_bounds__(32, G != 8 ? 16 : (SEAS ? PB200_GRP_BLOCKS : PB200_GRP_PLAIN_BLOCKS)) fit_group_kernel(const __grid_constant__ FitArgs a) {
    // (__grid_constant__: g_fetch and g_write_record take `a` by reference without a copy of it in local memory)
    static_assert(G == 8 || G == 16, "lanes per series");
    static_assert(SEAS || !MULT, "without seasonality the additive form is the model");
    static_assert((SEAS ? 6 * G * 8 : 0) + G * 4 <= 5 * GState<G, SEAS>::PPAD * 8, "LanePhase hand-over through vec[1..5]");
    constexpr int NSER = 32 / G;
    const int lane = threadIdx.x & 31, gi = lane / G, gl = lane % G;
    const unsigned gm = ((1u << G) - 1u) << (gi * G);
    GState<G, SEAS>& s = gstate<G, SEAS>(gi);
    const size_t slot = (size_t)blockIdx.x * NSER + gi;
    double* const plane = reinterpret_cast<double*>(a.planes) + slot * (size_t)a.nseas_stride;
    double* const hist = plane + (a.nseas_stride - GHIST);
    double* const trace_base = a.trace;
    {   // every group's state starts zeroed: the idle groups run the round's routines on it (no trend segments, every vector
        // role on vec[0]: in bounds), and store nothing
        constexpr int NZ = (int)(NSER * ((sizeof(GState<G, SEAS>) + 15) & ~(size_t)15) / 16);
        double2* const z = reinterpret_cast<double2*>(pb200_smem);
#pragma unroll 1
        for (int i = lane; i < NZ; i += 32) z[i] = make_double2(0.0, 0.0);
    }
    __syncwarp();
    // (an idle group's prior scales: the options', so that its unstored evaluations stay finite as before any fetch)
    if (gl == 0) { s.state = ST_IDLE; s.series = -1; gprior<G, SEAS>(gi) = {a.o.tau, a.o.rtau, SEAS ? a.o.inv_seas2 : 1.0}; }
    if (lane == 0) gopts<G, SEAS>() = a.o;
    __syncwarp();
    const FitOptsDev& opt = gopts<G, SEAS>();
    const double init_alpha = a.o.init_alpha;
    const int trace_cap = a.trace_cap;
    // L2 priority of this slot's y plane and history, and of the series' inputs (see l2_policy_evict_last)
    const int l2f = (slot < (size_t)a.l2_keep ? L2F_KEEP : 0) | (a.l2_rest_first ? L2F_REST_FIRST : 0);
    bool exhausted = false;
    LanePhase lp;
    lp.wph = lp.dph = lp.wend = make_double2(0.0, 1.0);
    lp.j0 = 0;
    PB200_PCLK_DECL(t_k0);
    PB200_PCLK_DECL(t_mark);
    PB200_PCLK_NOW(t_k0);
    for (;;) {
        PB200_PCLK_DECL(t_r0);
        PB200_PCLK_NOW(t_r0);
        PB200_PCLK_NOW(t_mark);
        // ---- idle groups take the next series of the queue ----
        if (s.state == ST_IDLE && !exhausted) {
            if (g_fetch<G, LOGI, SEAS>(s, a, plane, gl, gm, l2f)) {
                if constexpr (SEAS) {
                    lp.wph = reinterpret_cast<const double2*>(&s.vec[1][0])[gl];
                    lp.dph = reinterpret_cast<const double2*>(&s.vec[1][0])[G + gl];
                    lp.wend = reinterpret_cast<const double2*>(&s.vec[1][0])[2 * G + gl];
                }
                lp.j0 = reinterpret_cast<const int*>(&s.vec[1][0] + (SEAS ? 6 * G : 0))[gl];
                int st = ST_FIRST;
                if (a.grad_out) st = ST_OBJ;
                else if (s.st0 == PB200_ST_CONST_LINEAR) {
                    g_write_record<G, SEAS>(s, a, PB200_ST_CONST_LINEAR, gl, gm);
                    st = ST_IDLE;
                }
                __syncwarp(gm);
                if (gl == 0) s.state = st;
                __syncwarp(gm);
            } else {
                exhausted = true;
            }
        }
        __syncwarp();
        PB200_PCLK_MARK(PC_FETCH, t_mark, lane);
        const int state = s.state;
        const bool active = state != ST_IDLE;
        if (!__any_sync(FULL, active)) {
            if (__all_sync(FULL, exhausted)) break;
            continue;
        }
        PB200_PCLK_ADD(PC_ROUNDS, 1, lane == 0);
        // ---- one objective + gradient evaluation per active group.  The whole warp runs every routine of the round: the
        // idle groups compute on their own slot's state and store nothing ----
        const bool first = state == ST_FIRST || state == ST_OBJ;
        const int ixv = first ? s.ls.ix : s.ls.ixt, igv = first ? s.ls.ig : s.ls.igt;
        const int P = s.S + gkx<SEAS>() + 3;
        g_eval_setup<G, LOGI, SEAS>(s, s.vec[ixv], gl, active);
        if (active && gl == 0) s.ls.nevals += 1;
        __syncwarp();
        PB200_PCLK_MARK(PC_SETUP, t_mark, lane);
        g_point_pass<G, LOGI, MULT, SEAS, grp_u(G)>(s, plane, active, gl, lane, lp, l2f);
        __syncwarp();
        PB200_PCLK_MARK(PC_PASS, t_mark, lane);
        const int err = g_eval_finalize<G, LOGI, SEAS>(s, s.vec[ixv], s.vec[igv], gl, gm, active, first ? &s.ls.fk : &s.ls.ft);
        __syncwarp();
        PB200_PCLK_MARK(PC_FINAL, t_mark, lane);
        // ---- the optimiser's reaction (BFGSMinimizer::step split at its evaluations); `act` carries each group's action
        // from one routine to the next ----
        const LsStep lss = g_ls_step<G, SEAS>(s, gl, state == ST_SEARCH, P, err);
        int act = lss.act, status = PB200_ST_SUCCESS;
        bool done = false;
        if (state == ST_OBJ || (state == ST_FIRST && err)) {
            status = err ? PB200_ST_INIT_ERROR : PB200_ST_SUCCESS;
            done = true;
        } else if (state == ST_FIRST) {
            act = ACT_BEGIN_FIRST;
        } else if (act == ACT_FAIL) {
            // line search failed: retry once from a reset Hessian, else give up (PyStan raises; fbprophet retries with Newton)
            if (s.ls.resetB) { status = PB200_ST_LSFAIL; done = true; act = ACT_NONE; }
            else act = ACT_BEGIN_RETRY;
        }
        __syncwarp();
        PB200_PCLK_MARK(PC_LS_STEP, t_mark, lane);
#ifdef PB200_PHASE_CLOCKS
        {
            const unsigned acc = __ballot_sync(FULL, act == ACT_ACCEPT);
            PB200_PCLK_ADD(PC_POST_CALLS, 1, acc != 0 && lane == 0);
            PB200_PCLK_ADD(PC_ACCEPTS, 1, act == ACT_ACCEPT && gl == 0);
        }
#endif
        if (__any_sync(FULL, act == ACT_ACCEPT)) {
            const bool acc = act == ACT_ACCEPT;
            double* tr = (trace_base && acc) ? trace_base + (size_t)s.series * trace_cap * 4 : nullptr;
            const int st = g_post_accept<G, SEAS>(s, hist, gl, acc, P, opt, tr, trace_cap, l2f);
            if (acc) {
                status = st;
                if (status != PB200_ST_SUCCESS) done = true;
                else act = ACT_BEGIN_NEXT;
            }
        }
        __syncwarp();
        PB200_PCLK_MARK(PC_POST, t_mark, lane);
        g_ls_begin<G, SEAS>(s, gl, P, init_alpha, act, lss.alpha);
        __syncwarp();
        PB200_PCLK_MARK(PC_LS_BEGIN, t_mark, lane);
        if (done) {
            g_write_record<G, SEAS>(s, a, status, gl, gm);
            if (gl == 0) s.state = ST_IDLE;
        }
        __syncwarp();
        PB200_PCLK_MARK(PC_WRITE, t_mark, lane);
#ifdef PB200_PHASE_CLOCKS
        if (__any_sync(FULL, exhausted) && __popc(__ballot_sync(FULL, active)) < 32) PB200_PCLK_ADD(PC_DRAIN, t_mark - t_r0, lane == 0);
#endif
    }
    PB200_PCLK_ADD(PC_TOTAL, clock64() - t_k0, lane == 0);
    PB200_PCLK_ADD(PC_WARPS, 1, lane == 0);
    // the workspace is dead: its lines go back to normal priority, so that nothing stays pinned in L2 after the kernel
    if (l2f & L2F_KEEP) grp_l2_release<G>(plane, (size_t)a.nseas_stride, gl);
}

}  // namespace grp
}  // namespace pb200
