// Fit class of the models with a seasonality table (DESIGN §18): custom seasonalities and non-default Fourier orders.
// One warp per series, persistent over its own work queue, on any grid (regular, irregular, duplicate timestamps).
// The orders are run-time values, so the Fourier columns are regenerated per point by the three-term recurrence from one
// stored base (sin, cos) per active seasonality, in loops that are not unrolled over harmonics, and each lane's share
// of the beta gradient accumulates in shared memory instead of registers.
//
// The trend and sigma terms, Stan's L-BFGS (line search, update, stop rules) and the trajectory hook are the routines of
// fit_kernel.cuh, called as they are: eval_setup / eval_finalize see a model without Fourier columns (K = 0) at a
// shadow of the point whose beta is zero, and this file adds the beta terms with a prior scale per column.
// The REG instances (DESIGN §19) add the model's extra regressors as R more columns after the seasonal ones.
#include <type_traits>

#include "fit_kernel.cuh"
#include "launch.h"
#include "seas_table.cuh"

namespace pb200 {

constexpr int GS_STRIDE = 33;    // lane stride of the per-lane gradient rows: conflict-free row and column walks

// behind the sixteen optimiser vectors of the shared memory layout
struct TabExt {
    double xs[SEAS_PMAX + 4];            // shadow of the evaluated point: k, m, delta, log sigma, then a zero beta
    double beta[SEAS_KMAX];
    double isig2[SEAS_KMAX];             // 1 / prior_scale^2 of each column
    double gs[SEAS_KMAX * GS_STRIDE];    // per-lane partial beta gradient, column c of lane l at c * 33 + l
    double period[SEAS_TMAX];            // active entries of this series, in column order
    int order[SEAS_TMAX];
    int ne, K;
};

__host__ __device__ inline size_t fit_table_smem_bytes(int ppad) {
    return ((sizeof(Smem<1>) + 15) & ~(size_t)15) + (size_t)(6 + 2 * HMAX) * ppad * 8 + sizeof(TabExt);
}

__device__ __forceinline__ TabExt& tab_ext() { return *reinterpret_cast<TabExt*>(smem_ring<1>(smem_hdr<1>().ppad)); }

// behind TabExt in the instances with regressors (DESIGN §19).  Their columns follow the seasonal ones in TabExt's beta,
// isig2 and gs (K_seas + R <= SEAS_KMAX); their standardised values are staged as ceil(R / 2) double2 planes after the
// series' active seasonal planes, regressor r in component r & 1 of plane r >> 1
struct RegExt {
    int R;
};
static_assert(sizeof(TabExt) % 8 == 0, "RegExt follows TabExt");

__device__ __forceinline__ RegExt& reg_ext() { return *reinterpret_cast<RegExt*>(&tab_ext() + 1); }

// regressor r of the point at pt (its double2 of plane 0), in a slice whose active seasonal planes are ne
template <class D2>
__device__ __forceinline__ auto& reg_at(D2* pt, const int ne, const int Tp, const int r) {
    using D = std::conditional_t<std::is_const_v<D2>, const double, double>;
    return reinterpret_cast<D*>(pt + (size_t)(ne + 1 + (r >> 1)) * Tp)[r & 1];
}

// objective + gradient pass over lane's points [i0, i1): the trend partial sums as point_pass, the Fourier columns of
// every active seasonality twice per point (for the dot product, then for the gradient once the residual is known)
template <bool LOGI, bool REG>
PB200_EVAL_FN void table_point_pass(const int lane, const int i0, const int i1, const int j0) {
    Smem<1>& sm = smem_hdr<1>();
    TabExt& ex = tab_ext();
    const int K = ex.K, ne = ex.ne, S = sm.S, nact = sm.nact, Tp = sm.Tp;
    double* gs = ex.gs + lane;
#pragma unroll 1
    for (int c = 0; c < K; ++c) gs[c * GS_STRIDE] = 0.0;
    double ss = 0.0, locU = 0.0, locV = 0.0;
    int j = j0;
    int nb = j < S ? sm.bidx[j] : 0x7fffffff;
    double kcj = sm.kc[j], mcj = sm.mc[j];
    const double cap = sm.cap_s;
    const double mfl = sm.mult != 0 ? 1.0 : 0.0, afl = 1.0 - mfl;
    const double2* src = sm.TY + lane;
#pragma unroll 1
    for (int n = 0; n < i1 - i0; ++n) {
        const int i = i0 + n;
        const double2* pt = src + (size_t)n * nact;
        const double2 ty = pt[0];
        while (i == nb) {
            sm.bndU[j] = locU;
            sm.bndV[j] = locV;
            ++j;
            kcj = sm.kc[j];
            mcj = sm.mc[j];
            nb = j < S ? sm.bidx[j] : 0x7fffffff;
        }
        double dot = 0.0;
        {
            int col = 0;
#pragma unroll 1
            for (int e = 0; e < ne; ++e) {
                const double2 b = pt[(size_t)(e + 1) * Tp];
                const double c2 = b.y + b.y;
                double sp = 0.0, cp = 1.0, sn = b.x, cn = b.y;
#pragma unroll 1
                for (int h = 0; h < ex.order[e]; ++h, col += 2) {
                    dot = fma(ex.beta[col], sn, dot);
                    dot = fma(ex.beta[col + 1], cn, dot);
                    const double s2 = fma(c2, sn, -sp), cc = fma(c2, cn, -cp);
                    sp = sn; cp = cn; sn = s2; cn = cc;
                }
            }
            if constexpr (REG) {
                const int R = reg_ext().R;
#pragma unroll 1
                for (int r = 0; r < R; ++r) dot = fma(ex.beta[col + r], reg_at(pt, ne, Tp, r), dot);
            }
        }
        double g, sig = 0.0;
        const double tm = ty.x - mcj;
        if constexpr (LOGI) {
            sig = rcp_fastpath(1.0 + exp_fastpath(-(kcj * tm)));
            g = cap * sig;
        } else {
            g = fma(kcj, ty.x, mcj);
        }
        const double opm = fma(mfl, dot, 1.0);
        const double yhat = fma(g, opm, afl * dot);
        const double r = ty.y - yhat;
        ss = fma(r, r, ss);
        {
            const double cb = r * fma(mfl, g, afl);
            int col = 0;
#pragma unroll 1
            for (int e = 0; e < ne; ++e) {
                const double2 b = pt[(size_t)(e + 1) * Tp];
                const double c2 = b.y + b.y;
                double sp = 0.0, cp = 1.0, sn = b.x, cn = b.y;
#pragma unroll 1
                for (int h = 0; h < ex.order[e]; ++h, col += 2) {
                    gs[col * GS_STRIDE] = fma(cb, sn, gs[col * GS_STRIDE]);
                    gs[(col + 1) * GS_STRIDE] = fma(cb, cn, gs[(col + 1) * GS_STRIDE]);
                    const double s2 = fma(c2, sn, -sp), cc = fma(c2, cn, -cp);
                    sp = sn; cp = cn; sn = s2; cn = cc;
                }
            }
            if constexpr (REG) {
                const int R = reg_ext().R;
#pragma unroll 1
                for (int r = 0; r < R; ++r) gs[(col + r) * GS_STRIDE] = fma(cb, reg_at(pt, ne, Tp, r), gs[(col + r) * GS_STRIDE]);
            }
        }
        const double qv = r * opm;
        if constexpr (LOGI) {
            const double dz = qv * g * (1.0 - sig);
            locU = fma(dz, tm, locU);
            locV += dz;
        } else {
            locU = fma(qv, ty.x, locU);
            locV += qv;
        }
    }
    // warp inclusive scan of (locU, locV): the boundaries this lane recorded get the exclusive prefix of the lanes before it
    double incU = locU, incV = locV;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const double a = __shfl_up_sync(FULL, incU, o);
        const double b = __shfl_up_sync(FULL, incV, o);
        if (lane >= o) { incU += a; incV += b; }
    }
    double exU = __shfl_up_sync(FULL, incU, 1), exV = __shfl_up_sync(FULL, incV, 1);
    if (lane == 0) { exU = 0.0; exV = 0.0; }
#pragma unroll 1
    for (int s = j0; s < j; ++s) {
        sm.bndU[s] += exU;
        sm.bndV[s] += exV;
    }
    if (lane == 31) {
        sm.wtot[0][0] = incU;
        sm.wtot[0][1] = incV;
    }
    ss = wsum(ss);
    if (lane == 0) sm.red[0][0] = ss;    // what eval_finalize reads as the residual sum of squares of a K = 0 model
    __syncwarp();
}

// one objective + gradient evaluation at vector xv -> gv, f -> *f_out; returns err (uniform)
template <bool LOGI, bool REG>
__device__ __forceinline__ int table_eval(const double* xv, double* gv, double* f_out, const int lane, const int i0,
                                          const int i1, const int j0) {
    Smem<1>& sm = smem_hdr<1>();
    TabExt& ex = tab_ext();
    const int S = sm.S, K = ex.K, KE = K > 0 ? K : 1;
#pragma unroll 1
    for (int q = lane; q < 4 + S; q += 32) ex.xs[q] = q < 3 + S ? xv[q] : 0.0;
#pragma unroll 1
    for (int q = lane; q < K; q += 32) ex.beta[q] = xv[3 + S + q];
    __syncwarp();
    eval_setup<1, LOGI>(ex.xs, lane, 0);
    if (lane == 0) sm.ls.nevals += 1;
    table_point_pass<LOGI, REG>(lane, i0, i1, j0);
    double f0;
    int bad = eval_finalize<1, LOGI>(ex.xs, gv, lane, 0, &f0);
    // the beta terms: gradient scale * X'c + beta / sigma_c^2, prior sum of beta^2 / (2 sigma_c^2)
    const double scale = -rcp_any(sm.sigma * sm.sigma);
    double pb = 0.0;
    int badb = 0;
#pragma unroll 1
    for (int q = lane; q < KE; q += 32) {
        double raw = 0.0;
        if (q < K) {
            const double* row = ex.gs + q * GS_STRIDE;
#pragma unroll 1
            for (int l = 0; l < 32; ++l) raw += row[l];
        }
        const double b = xv[3 + S + q], is2 = ex.isig2[q];
        const double gb = scale * raw + b * is2;
        gv[3 + S + q] = gb;
        pb += 0.5 * b * b * is2;
        if (!isfinite(gb)) badb = 1;
    }
    pb = wsum(pb);
    const double f = f0 + pb;
    bad = bad | __any_sync(FULL, badb) | !isfinite(f);
    __syncwarp();
    *f_out = f;
    return bad;
}

template <bool REG>
using TableFitArgsT = std::conditional_t<REG, RegTableFitArgs, TableFitArgs>;

// REG: the model's regressors (RegTableFitArgs) as R more columns; <LOGI, false> is the table class without them
template <bool LOGI, bool REG>
__global__ void __launch_bounds__(32) fit_table_kernel(const TableFitArgsT<REG> a) {
    const int lane = threadIdx.x;
    Smem<1>& sm = smem_hdr<1>();
    TabExt& ex = *reinterpret_cast<TabExt*>(smem_ring<1>(a.ppad));
    double2* const TYp = a.planes + (size_t)blockIdx.x * a.nseas_stride;
    if (lane == 0) {
        sm.TY = TYp;
        sm.Tp = a.Tp;
        sm.ppad = a.ppad;
        sm.mult = a.o.mult;
    }
    for (;;) {
        if (lane == 0) {
            const int pos = atomicAdd(a.q_head, 1);
            sm.series = pos < *a.q_count ? a.q_items[pos] : -1;
        }
        __syncwarp();
        const int sidx = sm.series;
        if (sidx < 0) break;
        int* mi = a.meta_i32 + (size_t)sidx * 8;
        const long long* ml = a.meta_i64 + (size_t)sidx * 2;
        double* mf = a.meta_f64 + (size_t)sidx * 4;
        const int T = mi[0], S = mi[1], ncp = mi[2], mask = mi[3], st0 = mi[4], i1max = mi[7];
        const long long start = ml[0], tscale = ml[1];
        const double y_scale = mf[0], fl = mf[1], capv = mf[2];
        const long long off = a.offsets[sidx];
        const int chunk = (T + 31) / 32;
        const int nact = (T + chunk - 1) / chunk;
        const double cap_s = LOGI ? (capv - fl) / y_scale : 0.0;
        int Kc = tab_k(a.tab, mask);
        if constexpr (REG) Kc += a.spec.R;
        const int K = Kc, KE = K > 0 ? K : 1;
        if (lane == 0) {
            sm.T = T; sm.S = S; sm.chunk = chunk; sm.nact = nact;
            sm.cap_s = cap_s;
            sm.prior = series_prior(nullptr, a.o, sidx);
            sm.trace = a.trace ? a.trace + (size_t)sidx * a.trace_cap * 4 : nullptr;
            sm.trace_cap = a.trace_cap;
            int ne = 0, col = 0;
            for (int e = 0; e < a.tab.n; ++e) {
                if (!((mask >> e) & 1)) continue;
                ex.period[ne] = a.tab.period[e];
                ex.order[ne] = a.tab.order[e];
                for (int q = 0; q < 2 * a.tab.order[e]; ++q) ex.isig2[col++] = a.tab.inv_sig2[e];
                ++ne;
            }
            if constexpr (REG) {
                for (int r = 0; r < a.spec.R; ++r) ex.isig2[col++] = a.spec.inv_sig2[r];
                reg_ext().R = a.spec.R;
            }
            if (K == 0) ex.isig2[0] = 1.0;      // fbprophet's zero column has prior scale 1
            ex.ne = ne;
            ex.K = K;
        }
        __syncwarp();
        const int P = S + KE + 3;
        const double dts = (double)tscale;

        // ---- stage the series into this CTA's workspace slice: (t, y) and the base (sin, cos) of each active seasonality ----
        for (int i = lane; i < T; i += 32) {
            const long long d = a.ds[off + i];
            const double yv = load_y(a.y, a.y_dtype, off + i);
            const int own = i / chunk, n = i - own * chunk;
            const int ph = n * nact + own;
            TYp[ph] = make_double2((double)(d - start) / dts, (yv - fl) / y_scale);
            const double tau_d = (1e-9 * (double)d) / 86400.0;
            for (int e = 0; e < ex.ne; ++e) {
                double s_, c_;
                sincos(TWO_PI_FL * tau_d / ex.period[e], &s_, &c_);
                TYp[(size_t)(e + 1) * a.Tp + ph] = make_double2(s_, c_);
            }
            if constexpr (REG) {
                const double* sc = a.reg_scale + (size_t)sidx * a.spec.R * 2;
                for (int r = 0; r < a.spec.R; ++r)
                    reg_at(TYp + ph, ex.ne, a.Tp, r) = reg_value(a.reg[(size_t)r * a.n_rows + off + i], sc[2 * r], sc[2 * r + 1]);
            }
        }
        // ---- changepoints (Prophet.set_changepoints) and segment boundaries ----
        if (lane < S) {
            double tcv;
            int b;
            if (ncp > 0) {
                const int hist = (int)floor((double)T * a.o.changepoint_range);
                const double step = (double)(hist - 1) / (double)ncp;
                const int idx = lane == ncp - 1 ? hist - 1 : (int)rint((double)(lane + 1) * step);
                tcv = (double)(a.ds[off + idx] - start) / dts;
                b = idx;
                while (b > 0 && (double)(a.ds[off + b - 1] - start) / dts >= tcv) --b;
            } else {
                tcv = 0.0;
                b = 0;
            }
            sm.tc[lane] = tcv;
            sm.bidx[lane] = b;
            sm.bown[lane] = 0;
            a.tchange[(size_t)sidx * a.smax + lane] = tcv;
        }
#pragma unroll 1
        for (int s = S + lane; s < a.smax; s += 32) a.tchange[(size_t)sidx * a.smax + s] = 0.0;
        __threadfence_block();
        __syncwarp();
        const int i0 = lane * chunk < T ? lane * chunk : T;
        const int i1 = i0 + chunk < T ? i0 + chunk : T;
        int j0 = 0;
#pragma unroll 1
        for (int s = 0; s < S; ++s) j0 += sm.bidx[s] < i0 ? 1 : 0;

        LSState& ls = sm.ls;
        if (lane == 0) {
            ls.ix = 0; ls.ig = 1; ls.ip = 2; ls.ixt = 3; ls.igt = 4; ls.ipp = 5;
            ls.iters = 0; ls.nevals = 0; ls.resetB = 1; ls.hn = 0; ls.hhead = 0;
            ls.fk = NAN; ls.fk_1 = 0.0; ls.ft = 0.0; ls.alphak_1 = 0.0; ls.alpha = 0.0;
            ls.alo = ls.aloF = ls.aloD = ls.ahi = ls.ahiF = ls.ahiD = 0.0; ls.itNum = 0;
            ls.status = st0;
        }
        __syncwarp();
        double* x = vecp<1>(0);
        double* g = vecp<1>(1);
        // ---- initial point: Prophet.{linear,logistic}_growth_init + stan_init ----
        {
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
            const double* th = a.theta_in ? a.theta_in + (size_t)sidx * a.pstride : nullptr;
#pragma unroll 1
            for (int q = lane; q < P; q += 32) x[q] = th ? th[q] : (q == 0 ? k0 : (q == 1 ? m0 : 0.0));
            __syncwarp();
        }
        int status = st0;
        if (a.grad_out) {
            const int err = table_eval<LOGI, REG>(vecp<1>(0), vecp<1>(1), &ls.fk, lane, i0, i1, j0);
            status = err ? PB200_ST_INIT_ERROR : PB200_ST_SUCCESS;
            double* go = a.grad_out + (size_t)sidx * a.pstride;
#pragma unroll 1
            for (int q = lane; q < a.pstride; q += 32) go[q] = q < P ? g[q] : 0.0;
        } else if (status != PB200_ST_CONST_LINEAR) {
            // ======== stan::optimization::BFGSMinimizer<..., LBFGSUpdate>, as fit_kernel ========
            int err = table_eval<LOGI, REG>(vecp<1>(0), vecp<1>(1), &ls.fk, lane, i0, i1, j0);
            if (err) {
                status = PB200_ST_INIT_ERROR;
            } else {
                status = PB200_ST_SUCCESS;
                if (lane == 0) { ls.iters = 1; ls.resetB = 1; }
                __syncwarp();
                ls_begin<1>(lane, P, a.o.init_alpha);
                for (;;) {
                    err = table_eval<LOGI, REG>(vecp<1>(ls.ixt), vecp<1>(ls.igt), &ls.ft, lane, i0, i1, j0);
                    const int act = ls_step<1>(lane, P, err);
                    if (act == ACT_EVAL) continue;
                    if (act == ACT_FAIL) {
                        if (ls.resetB) { status = PB200_ST_LSFAIL; break; }
                        __syncwarp();
                        if (lane == 0) ls.resetB = 2;
                        __syncwarp();
                        ls_begin<1>(lane, P, a.o.init_alpha);
                        continue;
                    }
                    status = post_accept<1, true>(lane, P, a.o);
                    if (status != PB200_ST_SUCCESS) break;
                    if (lane == 0) { ls.iters += 1; ls.resetB = 0; }
                    __syncwarp();
                    ls_begin<1>(lane, P, a.o.init_alpha);
                }
            }
        }
        __syncwarp();
        x = vecp<1>(ls.ix);
        const int iters = ls.iters, nevals = ls.nevals;
        const double fk = ls.fk;
        // ---- the model record: params row k, m, sigma_obs, delta[smax], beta[kmax] (active columns packed from 0) ----
        {
            double* pr = a.params + (size_t)sidx * a.pstride;
            double kf = x[0];
            const double mfv = x[1];
            double sg = exp(x[2 + S]);
            if (status == PB200_ST_CONST_LINEAR) sg = 1e-9;
            if (ncp == 0) kf = kf + x[2];
#pragma unroll 1
            for (int q = lane; q < a.pstride; q += 32) {
                double v = 0.0;
                if (q == 0) v = kf;
                else if (q == 1) v = mfv;
                else if (q == 2) v = sg;
                else if (q < 3 + a.smax) {
                    const int s = q - 3;
                    v = (s < S && ncp > 0) ? x[2 + s] : 0.0;
                } else {
                    const int b = q - 3 - a.smax;
                    v = b < K ? x[3 + S + b] : 0.0;
                }
                pr[q] = v;
            }
            if (lane == 0) {
                mi[4] = status; mi[5] = iters; mi[6] = nevals;
                mf[3] = fk;
                if (status == PB200_ST_LSFAIL && a.nq_items) {      // fbprophet's Newton retry picks it up (newton_kernel)
                    const int pos = atomicAdd(a.nq_count, 1);
                    a.nq_items[pos] = sidx;
                }
            }
        }
        __syncwarp();
    }
}

template <bool REG>
static cudaError_t launch_table_inst(int logi, const TableFitArgsT<REG>& a, int grid, size_t smem, cudaStream_t st, int* occ) {
    auto kern = logi ? fit_table_kernel<true, REG> : fit_table_kernel<false, REG>;
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    if (occ) return cudaOccupancyMaxActiveBlocksPerMultiprocessor(occ, kern, 32, smem);
    kern<<<grid, 32, smem, st>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_fit_table(int logi, const TableFitArgs& a, int grid, size_t smem, cudaStream_t st, int* occ) {
    return launch_table_inst<false>(logi, a, grid, smem, st, occ);
}

cudaError_t launch_fit_table_reg(int logi, const RegTableFitArgs& a, int grid, size_t smem, cudaStream_t st, int* occ) {
    return launch_table_inst<true>(logi, a, grid, smem, st, occ);
}

size_t fit_table_smem(int ppad) { return fit_table_smem_bytes(ppad); }
size_t fit_table_reg_smem(int ppad) { return fit_table_smem_bytes(ppad) + sizeof(RegExt); }

}  // namespace pb200
