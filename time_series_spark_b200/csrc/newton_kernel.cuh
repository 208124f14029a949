// Newton retry for the series whose L-BFGS ended in a line-search failure.
//
// fbprophet 0.5 Prophet.fit (reached from reference src/jobs/prophet_modeler.py:65-66):
//     try:    params = model.optimizing(dat, init=stan_init, iter=1e4, **kwargs)
//     except RuntimeError:
//             params = model.optimizing(dat, init=stan_init, iter=1e4, algorithm='Newton', **kwargs)
// so a series is only dropped (prophet_modeler.py:81-85) if the Newton run raises as well.  Restated from
// stan/services/optimize/newton.hpp, stan/optimization/newton.hpp (newton_step,
// make_negative_definite_and_solve) and stan/model/grad_hess_log_prob.hpp -- see oracle/prophet_oracle.py
// (stan_newton, _grad_hess) for the statement-by-statement version and the one recalled detail that is unsure.
//
// This is the cold path (about one series in 10^5 on ragged short series, none on the headline workload), so
// the code favours being obviously the same computation as the oracle's over speed: one CTA of NW_WARPS warps
// per failed series; an objective + gradient evaluation is a one-warp routine (points split over the lanes in
// contiguous chunks, Fourier features from one sincos per seasonality per point, trend recurrences and their
// adjoints run sequentially by lane 0 exactly like oracle/prophet_oracle.c::po_eval); the 4 P perturbed
// gradients of the finite-difference Hessian are spread over the warps (warp w owns whole rows d = w, w + NW,
// ... so every sum has a fixed order); the eigen-decomposition is cyclic Jacobi by warp 0.
#pragma once
#include "fit_kernel.cuh"
#include "regressors.cuh"

namespace pb200 {
namespace nw {

constexpr int NW_WARPS = 16;
constexpr int NW_PMAX = SEAS_PMAX;   // S + K + 3 <= 96: a seasonality table's limit (default models: 30 + 34 + 3 = 67)
constexpr int NW_SEG = 32;

struct NewtonArgs {
    const long long* ds;
    const void* y;
    int y_dtype;
    const long long* offsets;
    const int* nq_items;
    const int* nq_count;
    int* nq_head;
    double* params;
    double* tchange;
    int* meta_i32;
    const long long* meta_i64;
    double* meta_f64;
    int smax, kmax, pstride;
    const double* prior;     // per-series prior scales (FitArgs::prior); null: o's
    const double* x0;        // warm start points (PrepArgs::warm_x, k = NaN: cold); null: every series from stan_init
    FitOptsDev o;
    SeasTab tab;             // the models' seasonality table (n = 0: the compiled-in orders); mask = the table mask
    // the models' regressors (DESIGN §19; reg.R = 0: none): their columns follow the active seasonal ones, standardised
    // with the fit's reg_scale
    RegSpec reg;
    const double* reg_x;     // [R][n_rows]
    const double* reg_scale; // [n_series][R][2]
    long long n_rows;
};

struct WarpScratch {     // per warp
    double kc[NW_SEG], mc[NW_SEG], rho[NW_SEG], U[NW_SEG], V[NW_SEG];
    double x[NW_PMAX], g[NW_PMAX];
    double f;
    int err, pad_;
};

struct Series {          // per CTA
    int T, S, K, ncp, mask, logistic, mult, P;
    long long off, start, span;
    double y_scale, fl, cap_s, tau, rtau_unused, inv_seas2;
    double tc[NW_SEG];
    int bidx[NW_SEG];
    double x[NW_PMAX], g0[NW_PMAX], u[NW_PMAX], w[NW_PMAX], xn[NW_PMAX];
    double f, f0, f1, last;
    int it, nev, status, moved, stop, err;
    double isig[SEAS_KMAX];      // a table model's 1 / prior_scale^2 per packed column
    double rsc[2 * REG_MAX];     // the series' (mu, std) per regressor
};

inline size_t newton_smem_bytes(int P) {
    return sizeof(Series) + sizeof(WarpScratch) * NW_WARPS + (size_t)2 * P * P * 8 + 64;
}

// objective + gradient at ws.x -> ws.g, ws.f, ws.err (Stan ModelAdaptor error convention: nonzero = reject)
__device__ __noinline__ void nw_eval(const NewtonArgs& a, const Series& sr, WarpScratch& ws, const int lane) {
    const int R = a.reg.R;
    const int S = sr.S, T = sr.T, Kreal = (sr.mask || R) ? sr.K : 0;
    const double* th = ws.x;
    int bad = 0;
    for (int q = lane; q < sr.P; q += 32) if (!isfinite(th[q])) bad = 1;
    bad = __any_sync(FULL, bad);
    const double k = th[0], m = th[1], u_ = th[2 + S];
    const double sigma = exp(u_);
    if (!(sigma > 0.0) || !isfinite(sigma)) bad = 1;
    if (bad) { if (lane == 0) { ws.err = 1; ws.f = NAN; } __syncwarp(); return; }
    if (lane == 0) {
        double cum = 0.0;
        ws.kc[0] = k;
        for (int s = 0; s < S; ++s) { cum += th[2 + s]; ws.kc[s + 1] = k + cum; }
        ws.mc[0] = m;
        if (sr.logistic) {
            for (int s = 0; s < S; ++s) {
                ws.rho[s] = ws.kc[s] / ws.kc[s + 1];
                ws.mc[s + 1] = ws.mc[s] + (sr.tc[s] - ws.mc[s]) * (1.0 - ws.rho[s]);
            }
        } else {
            double c2 = 0.0;
            for (int s = 0; s < S; ++s) { c2 += -sr.tc[s] * th[2 + s]; ws.mc[s + 1] = m + c2; }
        }
    }
    __syncwarp();
    const int chunk = (T + 31) / 32;
    const int i0 = min(lane * chunk, T), i1 = min(i0 + chunk, T);
    int j = 0;
    for (int s = 0; s < S; ++s) j += sr.bidx[s] < i0 ? 1 : 0;
    const int j0 = j;
    const bool tab = a.tab.n > 0 || R > 0;
    double gb[SEAS_KMAX];      // fixed layout: yearly 0..19, weekly 20..25, daily 26..33; a table model: its packed columns
#pragma unroll
    for (int q = 0; q < SEAS_KMAX; ++q) gb[q] = 0.0;
    double ss = 0.0, locU = 0.0, locV = 0.0;
    const double dspan = (double)sr.span;
    const double* beta = th + 3 + S;
    const int bw = (sr.mask & 1) ? 20 : 0, bd = bw + ((sr.mask & 2) ? 6 : 0);    // packed column of the weekly / daily block
    int nonfinite = 0;
    for (int i = i0; i < i1; ++i) {
        while (j < S && i >= sr.bidx[j]) { ws.U[j] = locU; ws.V[j] = locV; ++j; }
        const long long d = a.ds[sr.off + i];
        const double t = (double)(d - sr.start) / dspan;
        const double yv = (load_y(a.y, a.y_dtype, sr.off + i) - sr.fl) / sr.y_scale;
        double Xy[20], Xw[6], Xd[8], Xt[SEAS_KMAX];
        double dot = 0.0;
        const double tau_d = (1e-9 * (double)d) / 86400.0;
        if (tab) {
            // the active entries in column order: one sincos per seasonality, harmonics by the three-term recurrence
            int col = 0;
            for (int e = 0; e < a.tab.n; ++e) {
                if (!((sr.mask >> e) & 1)) continue;
                double s_, c_;
                sincos(TWO_PI_FL * tau_d / a.tab.period[e], &s_, &c_);
                const double c2 = c_ + c_;
                double sp = 0.0, cp = 1.0, sn = s_, cn = c_;
                for (int h = 0; h < a.tab.order[e]; ++h, col += 2) {
                    Xt[col] = sn;
                    Xt[col + 1] = cn;
                    const double s2 = fma(c2, sn, -sp), cc = fma(c2, cn, -cp);
                    sp = sn; cp = cn; sn = s2; cn = cc;
                }
            }
            for (int r = 0; r < R; ++r)
                Xt[col + r] = reg_value(a.reg_x[(size_t)r * a.n_rows + sr.off + i], sr.rsc[2 * r], sr.rsc[2 * r + 1]);
            for (int q = 0; q < Kreal; ++q) dot = fma(Xt[q], beta[q], dot);
        }
        if (!tab && (sr.mask & 1)) {
            double s_, c_;
            sincos(TWO_PI_FL * tau_d / 365.25, &s_, &c_);
            harmonics<10>(make_double2(s_, c_), Xy);
#pragma unroll
            for (int q = 0; q < 20; ++q) dot = fma(Xy[q], beta[q], dot);
        }
        if (!tab && (sr.mask & 2)) {
            double s_, c_;
            sincos(TWO_PI_FL * tau_d / 7.0, &s_, &c_);
            harmonics<3>(make_double2(s_, c_), Xw);
#pragma unroll
            for (int q = 0; q < 6; ++q) dot = fma(Xw[q], beta[bw + q], dot);
        }
        if (!tab && (sr.mask & 4)) {
            double s_, c_;
            sincos(TWO_PI_FL * tau_d / 1.0, &s_, &c_);
            harmonics<4>(make_double2(s_, c_), Xd);
#pragma unroll
            for (int q = 0; q < 8; ++q) dot = fma(Xd[q], beta[bd + q], dot);
        }
        const double tm = t - ws.mc[j];
        double gtr, sig = 0.0;
        if (sr.logistic) { sig = 1.0 / (1.0 + exp(-(ws.kc[j] * tm))); gtr = sr.cap_s * sig; }
        else gtr = ws.kc[j] * t + ws.mc[j];
        const double opm = sr.mult ? 1.0 + dot : 1.0;
        const double yhat = sr.mult ? gtr * opm : gtr + dot;
        if (!isfinite(yhat)) nonfinite = 1;
        const double r = yv - yhat;
        ss = fma(r, r, ss);
        const double cb = sr.mult ? r * gtr : r;
        if (tab) {
            for (int q = 0; q < Kreal; ++q) gb[q] = fma(cb, Xt[q], gb[q]);
        } else if (sr.mask & 1) {
#pragma unroll
            for (int q = 0; q < 20; ++q) gb[q] = fma(cb, Xy[q], gb[q]);
        }
        if (!tab && (sr.mask & 2)) {
#pragma unroll
            for (int q = 0; q < 6; ++q) gb[20 + q] = fma(cb, Xw[q], gb[20 + q]);
        }
        if (!tab && (sr.mask & 4)) {
#pragma unroll
            for (int q = 0; q < 8; ++q) gb[26 + q] = fma(cb, Xd[q], gb[26 + q]);
        }
        const double qv = r * opm;
        if (sr.logistic) { const double dz = qv * gtr * (1.0 - sig); locU = fma(dz, tm, locU); locV += dz; }
        else { locU = fma(qv, t, locU); locV += qv; }
    }
    // prefix sums at the segment boundaries: ws.U[s] = sum over the points before boundary s; slot S = total
    double incU = locU, incV = locV;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double au = __shfl_up_sync(FULL, incU, o), av = __shfl_up_sync(FULL, incV, o);
        if (lane >= o) { incU += au; incV += av; }
    }
    const double exU = incU - locU, exV = incV - locV;
    for (int s = j0; s < j; ++s) { ws.U[s] += exU; ws.V[s] += exV; }
    // boundaries beyond the last point owned by anybody cannot occur (changepoints lie in the first 80 % of the history)
    if (lane == 31) { ws.U[S] = incU; ws.V[S] = incV; }
    ss = wsum(ss);
    if (tab) {
        for (int q = 0; q < Kreal; ++q) gb[q] = wsum(gb[q]);
    } else if (Kreal) {
#pragma unroll
        for (int q = 0; q < 34; ++q) gb[q] = wsum(gb[q]);
    }
    nonfinite = __any_sync(FULL, nonfinite);
    __syncwarp();
    const double inv_s2 = 1.0 / (sigma * sigma), scale = -inv_s2;
    double* g = ws.g;
    if (lane == 0) {
        double gk, gm;
        double ad = 0.0;
        if (sr.logistic) {
            double kbar[NW_SEG + 1], gmc[NW_SEG + 1], rbar[NW_SEG];
            double pu = 0.0, pv = 0.0;
            for (int q = 0; q <= S; ++q) {
                const double du = ws.U[q] - pu, dv = ws.V[q] - pv;
                pu = ws.U[q]; pv = ws.V[q];
                kbar[q] = scale * du;
                gmc[q] = scale * (-ws.kc[q]) * dv;
            }
            double abar = gmc[S];
            for (int s = S - 1; s >= 0; --s) { rbar[s] = abar * (ws.mc[s] - sr.tc[s]); abar = gmc[s] + ws.rho[s] * abar; }
            for (int s = 0; s < S; ++s) { kbar[s] += rbar[s] / ws.kc[s + 1]; kbar[s + 1] += -(rbar[s] * ws.rho[s]) / ws.kc[s + 1]; }
            double tot = 0.0;
            for (int q = S; q >= 0; --q) { tot += kbar[q]; if (q >= 1) g[2 + q - 1] = tot; }
            gk = tot + k / 25.0;
            gm = abar + m / 25.0;
        } else {
            const double totU = ws.U[S], totV = ws.V[S];
            for (int s = 0; s < S; ++s) g[2 + s] = scale * ((totU - ws.U[s]) - sr.tc[s] * (totV - ws.V[s]));
            gk = scale * totU + k / 25.0;
            gm = scale * totV + m / 25.0;
        }
        for (int s = 0; s < S; ++s) {
            const double d = th[2 + s];
            ad += fabs(d);
            g[2 + s] += (d > 0 ? 1.0 : (d < 0 ? -1.0 : 0.0)) / sr.tau;
        }
        g[0] = gk; g[1] = gm;
        g[2 + S] = -ss * inv_s2 + (double)T + 4.0 * sigma * sigma;
        ws.f = 0.5 * ss * inv_s2 + (double)T * u_ + k * k / 50.0 + m * m / 50.0 + ad / sr.tau + 2.0 * sigma * sigma;
    }
    __syncwarp();
    // beta block (lane 0; fixed accumulator layout -> packed columns)
    if (lane == 0) {
        const double isg = Kreal ? sr.inv_seas2 : 1.0;
        double pb = 0.0;
        if (!Kreal) {
            const double b = beta[0];
            g[3 + S] = b * isg;
            pb = 0.5 * b * b * isg;
        } else if (tab) {
            for (int c = 0; c < Kreal; ++c) {
                const double b = beta[c];
                g[3 + S + c] = scale * gb[c] + b * sr.isig[c];
                pb += 0.5 * b * b * sr.isig[c];
            }
        } else {
#pragma unroll
            for (int q = 0; q < 34; ++q) {
                const bool on = q < 20 ? (sr.mask & 1) != 0 : (q < 26 ? (sr.mask & 2) != 0 : (sr.mask & 4) != 0);
                if (on) {
                    const int c = q < 20 ? q : (q < 26 ? bw + q - 20 : bd + q - 26);
                    const double b = beta[c];
                    g[3 + S + c] = scale * gb[q] + b * isg;
                    pb += 0.5 * b * b * isg;
                }
            }
        }
        ws.f += pb;
    }
    __syncwarp();
    int e = nonfinite ? 1 : 0;
    for (int q = lane; q < sr.P; q += 32) if (!isfinite(g[q])) e = e ? e : 3;
    e = __reduce_max_sync(FULL, e);
    if (lane == 0) {
        if (!e && !isfinite(ws.f)) e = 2;
        ws.err = e;
    }
    __syncwarp();
}

// cyclic Jacobi on the symmetric n x n matrix A (row-major, destroyed: eigenvalues on the diagonal),
// eigenvectors in the columns of V; one warp
__device__ __noinline__ void nw_jacobi(double* A, double* V, const int n, const int lane) {
    for (int q = lane; q < n * n; q += 32) V[q] = (q / n == q % n) ? 1.0 : 0.0;
    __syncwarp();
    for (int sweep = 0; sweep < 60; ++sweep) {
        double off = 0.0, diag = 0.0;
        for (int q = lane; q < n * n; q += 32) {
            const int i = q / n, j = q % n;
            const double v = A[q];
            if (i == j) diag = fma(v, v, diag);
            else if (j > i) off = fma(v, v, off);
        }
        off = wsum(off);
        diag = wsum(diag);
        if (off <= 1e-30 * diag || off == 0.0) break;
        for (int p = 0; p < n - 1; ++p)
            for (int q = p + 1; q < n; ++q) {
                const double apq = A[p * n + q];
                if (apq == 0.0) continue;                    // uniform: all lanes read the same element
                const double theta = (A[q * n + q] - A[p * n + p]) / (2.0 * apq);
                const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
                const double c = 1.0 / sqrt(t * t + 1.0), s_ = t * c;
                __syncwarp();
                for (int k = lane; k < n; k += 32) {          // columns p, q of A and V
                    const double akp = A[k * n + p], akq = A[k * n + q];
                    A[k * n + p] = c * akp - s_ * akq; A[k * n + q] = s_ * akp + c * akq;
                    const double vkp = V[k * n + p], vkq = V[k * n + q];
                    V[k * n + p] = c * vkp - s_ * vkq; V[k * n + q] = s_ * vkp + c * vkq;
                }
                __syncwarp();
                for (int k = lane; k < n; k += 32) {          // rows p, q of A
                    const double apk = A[p * n + k], aqk = A[q * n + k];
                    A[p * n + k] = c * apk - s_ * aqk; A[q * n + k] = s_ * apk + c * aqk;
                }
                __syncwarp();
            }
    }
    __syncwarp();
}

__global__ void __launch_bounds__(32 * NW_WARPS, 1) newton_kernel(const NewtonArgs a) {
    extern __shared__ __align__(16) unsigned char nw_smem[];
    Series& sr = *reinterpret_cast<Series*>(nw_smem);
    WarpScratch* wsa = reinterpret_cast<WarpScratch*>(nw_smem + ((sizeof(Series) + 15) & ~(size_t)15));
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    WarpScratch& ws = wsa[warp];
    double* const Hm = reinterpret_cast<double*>(wsa + NW_WARPS);
    __shared__ int s_item;
    for (;;) {
        if (tid == 0) {
            const int pos = atomicAdd(a.nq_head, 1);
            s_item = pos < *a.nq_count ? a.nq_items[pos] : -1;
        }
        __syncthreads();
        const int sidx = s_item;
        if (sidx < 0) break;
        int* mi = a.meta_i32 + (size_t)sidx * 8;
        double* mf = a.meta_f64 + (size_t)sidx * 4;
        // ---- the series (meta written by prep_kernel, changepoint times by the fit kernel) ----
        if (tid == 0) {
            sr.T = mi[0]; sr.S = mi[1]; sr.ncp = mi[2]; sr.mask = mi[3];
            sr.K = sr.mask ? ((sr.mask & 1) ? 20 : 0) + ((sr.mask & 2) ? 6 : 0) + ((sr.mask & 4) ? 8 : 0) : 1;
            if (a.tab.n > 0 || a.reg.R > 0) {
                const int K = tab_k(a.tab, sr.mask) + a.reg.R;
                sr.K = K > 0 ? K : 1;
                int c = 0;
                for (int e = 0; e < a.tab.n; ++e)
                    if ((sr.mask >> e) & 1)
                        for (int q = 0; q < 2 * a.tab.order[e]; ++q) sr.isig[c++] = a.tab.inv_sig2[e];
                for (int r = 0; r < a.reg.R; ++r) {
                    sr.isig[c++] = a.reg.inv_sig2[r];
                    sr.rsc[2 * r] = a.reg_scale[((size_t)sidx * a.reg.R + r) * 2];
                    sr.rsc[2 * r + 1] = a.reg_scale[((size_t)sidx * a.reg.R + r) * 2 + 1];
                }
            }
            sr.P = sr.S + sr.K + 3;
            sr.logistic = a.o.growth == PB200_GROWTH_LOGISTIC;
            sr.mult = a.o.mult;
            sr.off = a.offsets[sidx];
            sr.start = a.meta_i64[(size_t)sidx * 2];
            sr.span = a.meta_i64[(size_t)sidx * 2 + 1];
            sr.y_scale = mf[0]; sr.fl = mf[1];
            sr.cap_s = sr.logistic ? (mf[2] - mf[1]) / mf[0] : 0.0;
            const SeriesPrior pr = series_prior(a.prior, a.o, sidx);
            sr.tau = pr.tau; sr.inv_seas2 = pr.inv_seas2;
            sr.it = 0; sr.nev = 0; sr.status = PB200_ST_NEWTON; sr.stop = 0;
        }
        __syncthreads();
        const int T = sr.T, S = sr.S, P = sr.P;
        double* const Vm = Hm + P * P;
        if (tid < NW_SEG) {
            if (tid < S) {                                   // Prophet.set_changepoints, as in the fit kernels
                double tcv = 0.0;
                int b = 0;
                if (sr.ncp > 0) {
                    const int hist = (int)floor((double)T * a.o.changepoint_range);
                    const double stp = (double)(hist - 1) / (double)sr.ncp;
                    const int idx = tid == sr.ncp - 1 ? hist - 1 : (int)rint((double)(tid + 1) * stp);
                    const double dts = (double)sr.span;
                    tcv = (double)(a.ds[sr.off + idx] - sr.start) / dts;
                    b = idx;
                    while (b > 0 && (double)(a.ds[sr.off + b - 1] - sr.start) / dts >= tcv) --b;
                }
                sr.tc[tid] = tcv;
                sr.bidx[tid] = b;
                a.tchange[(size_t)sidx * a.smax + tid] = tcv;
            } else {
                sr.bidx[tid] = 0x7fffffff;
                sr.tc[tid] = 0.0;
            }
        }
        // ---- initial point: the same stan_init (or warm start point) the L-BFGS run started from ----
        if (tid == 0) {
            const double* w = a.x0 ? a.x0 + (size_t)sidx * a.pstride : nullptr;
            if (w && !(w[0] == w[0])) w = nullptr;
            const int i1max = mi[7];
            const double y0 = (load_y(a.y, a.y_dtype, sr.off) - sr.fl) / sr.y_scale;
            const double y1 = (load_y(a.y, a.y_dtype, sr.off + i1max) - sr.fl) / sr.y_scale;
            const double t1v = (double)(a.ds[sr.off + i1max] - sr.start) / (double)sr.span;
            double k0, m0;
            if (sr.logistic) {
                const double C0 = sr.cap_s;
                const double yy0 = fmax(0.01 * C0, fmin(0.99 * C0, y0)), yy1 = fmax(0.01 * C0, fmin(0.99 * C0, y1));
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
            for (int q = 0; q < P; ++q) sr.x[q] = w ? w[q] : (q == 0 ? k0 : (q == 1 ? m0 : 0.0));
        }
        __syncthreads();
        // services::optimize::newton: lp at the initial point (an error there is caught: lp = -inf)
        if (warp == 0) {
            for (int q = lane; q < P; q += 32) ws.x[q] = sr.x[q];
            __syncwarp();
            nw_eval(a, sr, ws, lane);
            if (lane == 0) { sr.f = ws.err ? INFINITY : ws.f; sr.nev = 1; }
        }
        __syncthreads();
        const double eps = 1e-3, half_inv_eps = 0.5 / eps;
        for (int it = 1; it <= a.o.max_iter; ++it) {
            // ---- grad_hess_log_prob: gradient at x, Hessian rows from 4-point central differences of gradients ----
            if (tid == 0) sr.err = 0;
            __syncthreads();
            if (warp == 0) {
                for (int q = lane; q < P; q += 32) ws.x[q] = sr.x[q];
                __syncwarp();
                nw_eval(a, sr, ws, lane);
                for (int q = lane; q < P; q += 32) sr.g0[q] = ws.g[q];
                if (lane == 0) { sr.f0 = ws.f; if (ws.err) sr.err = 1; }
            }
            for (int d = warp; d < P; d += NW_WARPS) {
                double* const Rd = Vm + d * P;                     // row d of R (staged in V's storage), this warp's own
                for (int q = lane; q < P; q += 32) Rd[q] = 0.0;
                int e = 0;
                for (int i = 0; i < 4; ++i) {
                    const double pert = i == 0 ? -2 * eps : (i == 1 ? -eps : (i == 2 ? eps : 2 * eps));
                    const double coef = i == 0 ? 1.0 / 12.0 : (i == 1 ? -2.0 / 3.0 : (i == 2 ? 2.0 / 3.0 : -1.0 / 12.0));
                    for (int q = lane; q < P; q += 32) ws.x[q] = sr.x[q] + (q == d ? pert : 0.0);
                    __syncwarp();
                    nw_eval(a, sr, ws, lane);
                    if (ws.err) e = 1;
                    for (int q = lane; q < P; q += 32) Rd[q] += half_inv_eps * coef * ws.g[q];
                    __syncwarp();
                }
                if (e && lane == 0) atomicExch(&sr.err, 1);
            }
            __syncthreads();
            if (sr.err) {                                          // Stan throws: PyStan raises again, the series is dropped
                if (tid == 0) { sr.status = PB200_ST_LSFAIL; sr.it = it; sr.nev += 1 + 4 * P; }
                __syncthreads();
                break;
            }
            for (int q = tid; q < P * P; q += blockDim.x) Hm[q] = Vm[q] + Vm[(q % P) * P + q / P];   // H = R + R'
            __syncthreads();
            // ---- make_negative_definite_and_solve (for f = -lp): u = V diag(1 / |lambda|) V' g ----
            if (warp == 0) nw_jacobi(Hm, Vm, P, lane);
            __syncthreads();
            for (int j = tid; j < P; j += blockDim.x) {
                double s_ = 0.0;
                for (int k = 0; k < P; ++k) s_ += Vm[k * P + j] * sr.g0[k];
                sr.w[j] = s_ / fabs(Hm[j * P + j]);
            }
            __syncthreads();
            for (int k = tid; k < P; k += blockDim.x) {
                double s_ = 0.0;
                for (int j = 0; j < P; ++j) s_ += Vm[k * P + j] * sr.w[j];
                sr.u[k] = s_;
            }
            __syncthreads();
            // ---- newton_step's step halving: accept the first step that does not increase f ----
            if (warp == 0) {
                double step = 2.0;
                int moved = 0, nls = 0;
                const double f0 = sr.f0;
                for (;;) {
                    step *= 0.5;
                    if (step < 1e-50) break;
                    for (int q = lane; q < P; q += 32) { const double v = sr.x[q] - step * sr.u[q]; sr.xn[q] = v; ws.x[q] = v; }
                    __syncwarp();
                    nw_eval(a, sr, ws, lane);
                    ++nls;
                    if (ws.err || !(ws.f <= f0)) continue;
                    moved = 1;
                    break;
                }
                const double last = sr.f;
                double f;
                if (moved) {
                    for (int q = lane; q < P; q += 32) sr.x[q] = sr.xn[q];
                    f = ws.f;
                } else {
                    f = f0;
                }
                __syncwarp();
                if (lane == 0) {
                    sr.f = f; sr.it = it; sr.nev += 1 + 4 * P + nls;
                    sr.stop = (it > 1 && fabs(f - last) < 1e-8) ? 1 : 0;
                }
            }
            __syncthreads();
            if (sr.stop) break;
        }
        __syncthreads();
        // ---- model record ----
        if (sr.status == PB200_ST_NEWTON) {
            double* pr = a.params + (size_t)sidx * a.pstride;
            const double* x = sr.x;
            for (int q = tid; q < a.pstride; q += blockDim.x) {
                double v = 0.0;
                if (q == 0) v = sr.ncp == 0 ? x[0] + x[2] : x[0];
                else if (q == 1) v = x[1];
                else if (q == 2) v = exp(x[2 + S]);
                else if (q < 3 + a.smax) {
                    const int c = q - 3;
                    v = (c < S && sr.ncp > 0) ? x[2 + c] : 0.0;
                } else {
                    // only fbprophet's zero column (no seasonality and no regressor) is recorded as 0: a history without
                    // seasonality still has its R regressor betas in columns 0 .. R - 1
                    const int b = q - 3 - a.smax;
                    v = ((sr.mask || a.reg.R) && b < sr.K) ? x[3 + S + b] : 0.0;
                }
                pr[q] = v;
            }
        }
        if (tid == 0) {
            mi[4] = sr.status; mi[5] += sr.it; mi[6] += sr.nev;
            if (sr.status == PB200_ST_NEWTON) mf[3] = sr.f;
        }
        __syncthreads();
    }
}

}  // namespace nw
}  // namespace pb200
