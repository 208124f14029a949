// C ABI of libprophet_b200.so (see include/prophet_b200.h).  Host-side orchestration only:
// length classes, work queues, launches, staging copies.  All arithmetic is in the kernels.
#define PB200_WITH_PREP 1
#include "fit_kernel.cuh"
#include "launch.h"
#include "predict_kernel.cuh"
#include "mc_kernel.cuh"
#include "newton_kernel.cuh"
#include "csv_kernel.cuh"
#include "cv_kernel.cuh"
#include "insample_kernel.cuh"
#include "reg_scale_kernel.cuh"
#include "join_kernel.cuh"
#include "../../include/prophet_b200_window_quantiles.h"

#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

namespace {

thread_local std::string g_err;

int fail(int code, const char* what, cudaError_t e = cudaSuccess) {
    char buf[512];
    if (e != cudaSuccess) snprintf(buf, sizeof buf, "%s: %s", what, cudaGetErrorString(e));
    else snprintf(buf, sizeof buf, "%s", what);
    g_err = buf;
    return code;
}

#define CK(call)                                                      \
    do {                                                              \
        cudaError_t e_ = (call);                                      \
        if (e_ != cudaSuccess) return fail(PB200_E_CUDA, #call, e_);  \
    } while (0)

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = n + n / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
};

struct HostBuf {   // pinned
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
        size_t want = n + n / 8 + 256;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() {
        if (p) cudaFreeHost(p);
        p = nullptr;
        cap = 0;
    }
};

constexpr int NLC = 2;
const int LC_NT[NLC] = {32, 128};

// the work queues' expected-cost key is points x (1 + QKEY_CV_WEIGHT x cv), cv the coefficient of variation of y: a noisier
// series takes more evaluations (DESIGN §3)
constexpr double QKEY_CV_WEIGHT = 2.0;

int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return v && *v ? atoi(v) : dflt;
}

// the arrays the *_host entry points stage on the device (Staging), one growth-only buffer per role: repeated identical
// calls allocate nothing after the first
enum StageRole {
    ST_DS, ST_Y, ST_REG, ST_REGSC, ST_CAP, ST_PRIOR, ST_IPARAMS, ST_IMETA, ST_WARM, ST_THETA, ST_GRAD, ST_TRACE,   // fit inputs
    ST_PARAMS, ST_TCHANGE, ST_MI32, ST_MI64, ST_MF64,   // the model records
    ST_FUT, ST_FLOOR,                                   // predict inputs (ST_FUT: the predicted rows' ds)
    ST_YHAT, ST_LO, ST_HI, ST_YINT, ST_COMP, ST_TLO, ST_THI, ST_SUMS, ST_QUANT,   // predict outputs
    N_STAGE
};

}  // namespace

struct pb200_ctx {
    int device = 0;
    int sms = 0;
    cudaStream_t stream = nullptr;  // the stream of every call
    int64_t launches = 0;
    // fit workspace
    cudaEvent_t ctl_ev = nullptr;   // recorded after the H2D copies out of h_ctl
    bool ctl_pending = false;
    DevBuf d_offsets, d_order, d_lenclass, d_qitems, d_qctl;   // control workspace (device)
    DevBuf d_qkey, d_qhist;         // counting sort of the work queues by expected cost (prep_kernel, queue_*_kernel)
    DevBuf d_nq;                    // [0] count, [1] head, [2..] series whose L-BFGS failed its line search (Newton retry queue)
    DevBuf d_planes;                // fit kernels' per-series workspace (one slice per resident CTA / series slot)
    HostBuf h_ctl;                  // pinned staging for offsets / order / lenclass
    DevBuf d_vcount;                // series of the last fit call per kernel variant x seasonality class
    DevBuf d_warm_x;                // warm start points of pb200_fit_warm_* (prep_kernel -> fit kernels, Newton retry)
    DevBuf d_regbad;                // regressor fits: series with a non-finite regressor value (reg_scale_kernel -> prep_kernel)
    DevBuf d_hoff;                  // device copy of pb200_predict_history_*'s frame offsets
    DevBuf stage[N_STAGE];          // the *_host entry points' arrays, by StageRole
    int lc0_max = 1 << 30; // PB200_LC0_MAX: longest series on one warp per series, longer ones get four (unset: no limit)
    bool lc_auto = true;   // false when PB200_LC0_MAX pins the CTA width
    bool tab_on = true;    // PB200_NO_TAB=1 disables the seasonal-table variants (A/B runs)
    int grp_g = -1;        // lanes per series of the grouped day-table kernel (fit_group.cuh); PB200_GROUP=0|8|16 pins it
                           // (0 = point_pass_tab), unset = by batch size: 8 from grp_min series on, 16 below
    int plain_grp = 0;     // PB200_PLAIN_GROUP=1: the class WITHOUT seasonality (regular grid; reference config #4) on the grouped kernel
                           // too.  Off: it beat one warp per series only at the largest batches measured (500k short series) --
                           // its rounds are longer, and small batches are latency bound
    int grp_min = 16384;   // PB200_GROUP_MIN: smallest batch that gets 8 lanes per series; smaller ones get 16 (a warp with 4
                           // series drains longer once the queue is empty).  H100 (400 W), 1440-point series, ms per step at 12 500 / 50 000
                           // series: G = 8: 156 / 529, G = 16: 147 / 526 (the same within the run-to-run spread of ~5 %) -- measured
                           // before the 4-stage G = 8 ring and the workspace's L2 hints, which brought G = 8 at 50 000 to 454 ms and
                           // G = 16 at 12 500 to 143 ms (DESIGN §3, §5)
    size_t l2_bytes = 0;   // the device's L2
    int l2_keep_pct = 65;  // PB200_L2_KEEP_PCT: share of the L2 the grouped kernel's workspace slots may hold at evict_last priority
                           // (< 0: no cache hints -- A/B runs).  40 to 85 measured the same on an H100
    int grid_max = 0;      // PB200_FIT_GRID_MAX (tests): at most this many CTAs per fit launch (grouped and one-series kernels) and per
                           // Newton launch; unset or <= 0: no cap.  The workspace is sized from the capped grid; the kernel variant, G and
                           // the evict_last slot count are chosen as without it.  With a small cap every slot fits many series in turn
                           // (a series' result must not depend on which slot or launch geometry it gets)
};

namespace {

using pb200::FitArgs;
using pb200::FitOptsDev;
using pb200::NQ;

typedef cudaError_t (*launch_fn)(int, int, int, const FitArgs&, int, size_t, cudaStream_t, int*);
const launch_fn LAUNCH[8] = {pb200::launch_fit_mask0, pb200::launch_fit_mask1, pb200::launch_fit_mask2,
                             pb200::launch_fit_mask3, pb200::launch_fit_mask4, pb200::launch_fit_mask5,
                             pb200::launch_fit_mask6, pb200::launch_fit_mask7};

int opts_table(const pb200_options* o, pb200::SeasTab* t);
int opts_reg(const pb200_options* o, pb200::RegSpec* r);

// options of version 2 and 3 carry a seasonality table (version 3 also the regressors)
bool has_table(const pb200_options* o) {
    return o->abi_version == PB200_ABI_VERSION_TABLE || o->abi_version == PB200_ABI_VERSION_REGRESSORS;
}

// regs: the caller is a regressor entry point (pb200_*_regressors_*) or pb200_get_layout.  Every other entry point refuses
// options with regressors: it has nowhere to receive their values
int check_opts(const pb200_options* o, bool regs = false) {
    if (!o) return fail(PB200_E_ARG, "options is null");
    if (o->abi_version != PB200_ABI_VERSION && !has_table(o)) return fail(PB200_E_ARG, "options.abi_version mismatch");
    if (o->growth != PB200_GROWTH_LINEAR && o->growth != PB200_GROWTH_LOGISTIC) return fail(PB200_E_ARG, "growth");
    if (o->n_changepoints < 0 || o->n_changepoints > 30) return fail(PB200_E_UNSUPPORTED, "n_changepoints must be in [0, 30]");
    if (o->history_size < 1 || o->history_size > pb200::HMAX) return fail(PB200_E_UNSUPPORTED, "history_size must be in [1, 5]");
    if (!(o->changepoint_range > 0.0 && o->changepoint_range <= 1.0)) return fail(PB200_E_ARG, "changepoint_range");
    if (!(o->changepoint_prior_scale > 0.0) || !(o->seasonality_prior_scale > 0.0)) return fail(PB200_E_ARG, "prior scales");
    for (int v : {o->yearly, o->weekly, o->daily})   // at version 2 the orders are v2's *_order
        if (v != PB200_SEAS_AUTO && v != 0 && v != 1) return fail(PB200_E_UNSUPPORTED, "seasonality switch must be AUTO, 0 or 1");
    if (o->max_iter < 1) return fail(PB200_E_ARG, "max_iter");
    if (o->algorithm < PB200_ALG_LBFGS_NEWTON || o->algorithm > PB200_ALG_NEWTON) return fail(PB200_E_ARG, "algorithm");
    pb200::RegSpec r;
    int rc = opts_reg(o, &r);
    if (rc) return rc;
    if (r.R > 0 && !regs)
        return fail(PB200_E_UNSUPPORTED, "options with regressors (n_regressors > 0) are taken only by pb200_fit_regressors_*, "
                                         "pb200_objective_regressors_host and pb200_predict_regressors_*");
    pb200::SeasTab t;
    return opts_table(o, &t);
}

// The regressors of *o (DESIGN §19), checked: r->R = 0 below version 3
int opts_reg(const pb200_options* o, pb200::RegSpec* r) {
    r->R = 0;
    if (o->abi_version != PB200_ABI_VERSION_REGRESSORS) return PB200_OK;
    const pb200_options_v3* v = reinterpret_cast<const pb200_options_v3*>(o);
    char msg[200];
    const int n = v->n_regressors;
    if (n < 0 || n > PB200_MAX_REGRESSORS) {
        snprintf(msg, sizeof msg, "n_regressors must be in [0, %d] (got %d)", PB200_MAX_REGRESSORS, n);
        return fail(PB200_E_UNSUPPORTED, msg);
    }
    if (n == 0) return PB200_OK;
    if (!v->regressors) return fail(PB200_E_ARG, "regressors is null");
    if (!(v->holidays_prior_scale > 0.0 && v->holidays_prior_scale < INFINITY))
        return fail(PB200_E_ARG, "holidays_prior_scale must be finite and > 0");
    for (int i = 0; i < n; ++i) {
        const pb200_regressor& e = v->regressors[i];
        const size_t len = strnlen(e.name, sizeof e.name);
        if (len == 0 || len == sizeof e.name) return fail(PB200_E_ARG, "regressor name must be 1 to 15 bytes, NUL-terminated");
        for (int j = 0; j < i; ++j)
            if (strncmp(e.name, v->regressors[j].name, sizeof e.name) == 0) {
                snprintf(msg, sizeof msg, "regressor '%s' is added twice", e.name);
                return fail(PB200_E_ARG, msg);
            }
        bool seas_name = strcmp(e.name, "yearly") == 0 || strcmp(e.name, "weekly") == 0 || strcmp(e.name, "daily") == 0;
        for (int j = 0; j < v->v2.n_seasonalities && v->v2.seasonalities; ++j)
            seas_name = seas_name || strncmp(e.name, v->v2.seasonalities[j].name, sizeof e.name) == 0;
        if (seas_name) {
            snprintf(msg, sizeof msg, "regressor '%s' has a seasonality's name", e.name);
            return fail(PB200_E_ARG, msg);
        }
        if (!(e.prior_scale >= 0.0 && e.prior_scale < INFINITY)) {
            snprintf(msg, sizeof msg, "regressor '%s': prior_scale must be > 0 (got %g)", e.name, e.prior_scale);
            return fail(PB200_E_ARG, msg);
        }
        if (e.standardize != PB200_STD_AUTO && e.standardize != 0 && e.standardize != 1) {
            snprintf(msg, sizeof msg, "regressor '%s': standardize must be AUTO, 0 or 1", e.name);
            return fail(PB200_E_ARG, msg);
        }
        const double ps = e.prior_scale > 0.0 ? e.prior_scale : v->holidays_prior_scale;
        r->standardize[i] = e.standardize;
        r->inv_sig2[i] = 1.0 / (ps * ps);
    }
    r->R = n;
    return PB200_OK;
}

// The seasonality table of *o, normalised to fbprophet's column order (custom entries as added, then yearly, weekly,
// daily) and checked against the limits.  t->n = 0 for a v1 model and for a v2 one that restates the defaults.
//
// Options of version 3 with regressors are table models even when the table restates the defaults; their limits count
// the R regressor columns with the seasonal ones.
int opts_table(const pb200_options* o, pb200::SeasTab* t) {
    t->n = 0;
    if (!has_table(o)) return PB200_OK;
    const pb200_options_v2* v = reinterpret_cast<const pb200_options_v2*>(o);
    const int R = o->abi_version == PB200_ABI_VERSION_REGRESSORS
                      ? std::max(0, reinterpret_cast<const pb200_options_v3*>(o)->n_regressors) : 0;
    char msg[160];
    const int ns = v->n_seasonalities;
    if (ns < 0 || ns > PB200_MAX_SEASONALITIES) {
        snprintf(msg, sizeof msg, "n_seasonalities must be in [0, %d] (got %d)", PB200_MAX_SEASONALITIES, ns);
        return fail(PB200_E_UNSUPPORTED, msg);
    }
    if (ns > 0 && !v->seasonalities) return fail(PB200_E_ARG, "seasonalities is null");
    static const char* const BNAME[3] = {"yearly", "weekly", "daily"};
    const int dflt[3] = {10, 3, 4}, ord[3] = {v->yearly_order, v->weekly_order, v->daily_order};
    const int sw[3] = {o->yearly, o->weekly, o->daily};
    bool replaced[3] = {false, false, false};
    for (int b = 0; b < 3; ++b)
        if (ord[b] < 0) {
            snprintf(msg, sizeof msg, "%s_order must be >= 0 (got %d)", BNAME[b], ord[b]);
            return fail(PB200_E_ARG, msg);
        }
    for (int i = 0; i < ns; ++i) {
        const pb200_seasonality& e = v->seasonalities[i];
        const size_t len = strnlen(e.name, sizeof e.name);
        if (len == 0 || len == sizeof e.name) return fail(PB200_E_ARG, "seasonality name must be 1 to 15 bytes, NUL-terminated");
        for (int j = 0; j < i; ++j)
            if (strncmp(e.name, v->seasonalities[j].name, sizeof e.name) == 0) {
                snprintf(msg, sizeof msg, "seasonality '%s' is added twice", e.name);
                return fail(PB200_E_ARG, msg);
            }
        if (!(e.period > 0.0 && e.period < INFINITY)) {
            snprintf(msg, sizeof msg, "seasonality '%s': period must be finite and > 0 (got %g)", e.name, e.period);
            return fail(PB200_E_ARG, msg);
        }
        if (e.fourier_order <= 0) {
            snprintf(msg, sizeof msg, "seasonality '%s': fourier_order must be > 0 (got %d)", e.name, e.fourier_order);
            return fail(PB200_E_ARG, msg);
        }
        if (!(e.prior_scale >= 0.0 && e.prior_scale < INFINITY)) {
            snprintf(msg, sizeof msg, "seasonality '%s': prior_scale must be > 0 (got %g)", e.name, e.prior_scale);
            return fail(PB200_E_ARG, msg);
        }
        for (int b = 0; b < 3; ++b)
            if (strcmp(e.name, BNAME[b]) == 0) {
                if (sw[b] != PB200_SEAS_AUTO) {
                    snprintf(msg, sizeof msg, "custom seasonality '%s' replaces the built-in only when its switch is AUTO", e.name);
                    return fail(PB200_E_UNSUPPORTED, msg);
                }
                replaced[b] = true;
            }
    }
    bool restates = ns == 0 && R == 0;
    for (int b = 0; b < 3; ++b) restates = restates && (ord[b] == 0 || ord[b] == dflt[b] || sw[b] == 0);
    if (restates) return PB200_OK;
    int n = 0;
    double ps[PB200_MAX_SEASONALITIES + 3];
    int order[PB200_MAX_SEASONALITIES + 3], kind[PB200_MAX_SEASONALITIES + 3];
    double period[PB200_MAX_SEASONALITIES + 3];
    for (int i = 0; i < ns; ++i) {
        const pb200_seasonality& e = v->seasonalities[i];
        period[n] = e.period; order[n] = e.fourier_order; kind[n] = 0;
        ps[n++] = e.prior_scale > 0.0 ? e.prior_scale : o->seasonality_prior_scale;
    }
    const double bper[3] = {365.25, 7.0, 1.0};
    for (int b = 0; b < 3; ++b) {
        if (sw[b] == 0 || replaced[b]) continue;
        period[n] = bper[b]; order[n] = ord[b] > 0 ? ord[b] : dflt[b]; kind[n] = 1 << b;
        ps[n++] = o->seasonality_prior_scale;
    }
    if (n > PB200_MAX_SEASONALITIES) {
        snprintf(msg, sizeof msg, "the model has %d seasonalities; at most %d", n, PB200_MAX_SEASONALITIES);
        return fail(PB200_E_UNSUPPORTED, msg);
    }
    int K = 0;
    for (int i = 0; i < n; ++i) K += 2 * order[i];
    if (K > pb200::SEAS_KMAX) {
        snprintf(msg, sizeof msg, "the seasonalities have K = %d Fourier columns; at most %d", K, pb200::SEAS_KMAX);
        return fail(PB200_E_UNSUPPORTED, msg);
    }
    if (R > 0 && K + R > pb200::SEAS_KMAX) {
        snprintf(msg, sizeof msg, "the seasonalities' K = %d columns and the %d regressors make %d; at most %d", K, R, K + R,
                 pb200::SEAS_KMAX);
        return fail(PB200_E_UNSUPPORTED, msg);
    }
    K += R;
    const int P = 3 + (o->n_changepoints > 0 ? o->n_changepoints : 1) + K;
    if (P > pb200::SEAS_PMAX) {
        snprintf(msg, sizeof msg, R > 0 ? "the model has P = 3 + S + K + R = %d parameters; at most %d"
                                        : "the model has P = 3 + S + K = %d parameters; at most %d", P, pb200::SEAS_PMAX);
        return fail(PB200_E_UNSUPPORTED, msg);
    }
    t->n = n;
    int extra = 0;
    for (int i = 0; i < n; ++i) {
        t->period[i] = period[i];
        t->order[i] = order[i];
        t->kind[i] = kind[i];
        t->inv_sig2[i] = 1.0 / (ps[i] * ps[i]);
        int pl = -1;
        for (int b = 0; b < 3; ++b)
            if (kind[i] == 1 << b || (i < ns && strcmp(v->seasonalities[i].name, BNAME[b]) == 0)) pl = PB200_COMP_YEARLY + b;
        t->plane[i] = pl >= 0 ? pl : PB200_N_COMPONENTS + extra++;
    }
    t->nplanes = PB200_N_COMPONENTS + extra;
    return PB200_OK;
}

// the MC interval options, checked before anything is copied or launched: the kernel turns interval_width into ranks of the
// sorted draws, so a width outside [0, 1] (or NaN) would index outside a point's row of draws
int check_mc_opts(const pb200_options* o) {
    if (o->uncertainty_samples < 2 || o->uncertainty_samples > pb200::MC_NP)
        return fail(PB200_E_UNSUPPORTED, "uncertainty_samples must be in [2, 1024]");
    if (!(o->interval_width >= 0.0 && o->interval_width <= 1.0)) return fail(PB200_E_ARG, "interval_width must be in [0, 1]");
    return PB200_OK;
}

FitOptsDev to_dev(const pb200_options* o) {
    FitOptsDev d;
    const double eps = 2.220446049250313e-16;
    d.growth = o->growth;
    d.mult = o->multiplicative ? 1 : 0;
    d.n_changepoints = o->n_changepoints;
    d.max_iter = o->max_iter;
    d.history = o->history_size;
    d.yearly = o->yearly;
    d.weekly = o->weekly;
    d.daily = o->daily;
    d.changepoint_range = o->changepoint_range;
    d.tau = o->changepoint_prior_scale;
    d.seas_prior = o->seasonality_prior_scale;
    d.rtau = 1.0 / o->changepoint_prior_scale;
    d.inv_seas2 = 1.0 / (o->seasonality_prior_scale * o->seasonality_prior_scale);
    d.init_alpha = o->init_alpha;
    d.tol_obj = o->tol_obj;
    d.tol_rel_obj_eps = o->tol_rel_obj * eps;
    d.tol_grad = o->tol_grad;
    d.tol_rel_grad_eps = o->tol_rel_grad * eps;
    d.tol_param = o->tol_param;
    return d;
}

int mask_nseas(int m) { return pb200::stored_planes((m & 1) ? 10 : 0, (m & 2) ? 3 : 0, (m & 4) ? 4 : 0); }   // stored planes
int mask_k(int m) { return ((m & 1) ? 20 : 0) + ((m & 2) ? 6 : 0) + ((m & 4) ? 8 : 0); }

size_t y_elem(int dt) { return dt == PB200_Y_F64 ? 8 : 4; }

// The staging of one *_host call on the context's stream.  in() copies a host array into its role's buffer; out() makes
// room for an output (zeroed on the device when asked) and records its copy back; finish() enqueues the recorded copies
// and synchronises once.  A null host array stages nothing and gives a null device pointer, a count of 0 copies nothing.
// The first CUDA error is kept and every later step skips: status() reports it before the device body runs.
struct Staging {
    struct Copy { void* h; const void* d; size_t bytes; };
    pb200_ctx* c;
    cudaError_t err;
    std::vector<Copy> outs;

    explicit Staging(pb200_ctx* ctx) : c(ctx), err(cudaSetDevice(ctx->device)) {}
    void* reserve(StageRole role, size_t bytes) {
        if (err == cudaSuccess) err = c->stage[role].reserve(bytes);
        return err == cudaSuccess ? c->stage[role].p : nullptr;
    }
    template <class T> T* in(StageRole role, const T* h, size_t n) {
        if (!h) return nullptr;
        T* d = (T*)reserve(role, n * sizeof(T));
        if (n && err == cudaSuccess) err = cudaMemcpyAsync(d, h, n * sizeof(T), cudaMemcpyHostToDevice, c->stream);
        return d;
    }
    template <class T> T* out(StageRole role, T* h, size_t n, bool zero = false) {
        if (!h) return nullptr;
        T* d = (T*)reserve(role, n * sizeof(T));
        if (zero && n && err == cudaSuccess) err = cudaMemsetAsync(d, 0, n * sizeof(T), c->stream);
        later(h, d, n);
        return d;
    }
    template <class T> void later(T* h, const T* d, size_t n) {
        if (n) outs.push_back({h, d, n * sizeof(T)});
    }
    int status() const { return err == cudaSuccess ? PB200_OK : fail(PB200_E_CUDA, "staging of the host arrays", err); }
    int finish() {
        for (const Copy& o : outs)
            if (err == cudaSuccess) err = cudaMemcpyAsync(o.h, o.d, o.bytes, cudaMemcpyDeviceToHost, c->stream);
        if (err == cudaSuccess) err = cudaStreamSynchronize(c->stream);
        return status();
    }
};

// One fit request (fit_impl): device arrays, or host arrays in fit_host / objective_host.  The leading members are the
// arguments every fit entry point takes, in their order; the others are optional.  offsets is always a host array.
struct FitCall {
    const pb200_options* opts;
    const int64_t* ds;
    const void* y;
    int32_t y_dtype;
    const int64_t* offsets;
    int64_t n_series;
    double floor, cap_multiplier;
    const double* cap;
    double* params;
    double* tchange;
    int32_t* meta_i32;
    int64_t* meta_i64;
    double* meta_f64;
    const double* prior = nullptr;         // per-series prior scales [n_series][2]; null: the options'
    const double* init_params = nullptr;   // warm start: the previous models (pb200_fit_warm_*), their meta and codes
    const int32_t* init_meta = nullptr;
    int32_t* warm = nullptr;
    const double* theta = nullptr;         // an objective evaluation: -log p and its gradient at theta, no fit
    double* grad = nullptr;
    double* trace = nullptr;               // trace_cap trajectory rows per series
    int32_t trace_cap = 0;
    bool regs = false;                     // a regressor entry point: the options may carry regressors
    const double* reg = nullptr;           // their values [R][rows] and (mu, std) [n_series][R][2]
    double* reg_scale = nullptr;
    const double* reg_scale_copy = nullptr;   // pb200_fit_regressors_copy_device's scales
};

}  // namespace

extern "C" {

PB200_API void pb200_default_options(pb200_options* o) {
    if (!o) return;
    memset(o, 0, sizeof *o);
    o->abi_version = PB200_ABI_VERSION;
    o->growth = PB200_GROWTH_LOGISTIC;       // prophet_modeler.py:65
    o->multiplicative = 1;                   // prophet_modeler.py:65
    o->n_changepoints = 25;
    o->changepoint_range = 0.8;
    o->changepoint_prior_scale = 0.05;
    o->seasonality_prior_scale = 10.0;
    o->yearly = o->weekly = o->daily = PB200_SEAS_AUTO;
    o->max_iter = 10000;
    o->history_size = 5;
    o->init_alpha = 1e-3;
    o->tol_obj = 1e-12;
    o->tol_rel_obj = 1e4;
    o->tol_grad = 1e-8;
    o->tol_rel_grad = 1e7;
    o->tol_param = 1e-8;
    o->interval_width = 0.8;
    o->uncertainty_samples = 1000;
}

PB200_API int pb200_get_layout(const pb200_options* o, pb200_layout* out) {
    int rc = check_opts(o, true);
    if (rc) return rc;
    if (!out) return fail(PB200_E_ARG, "layout is null");
    out->smax = o->n_changepoints > 0 ? o->n_changepoints : 1;
    int k = 0;
    if (o->yearly != 0) k += 20;
    if (o->weekly != 0) k += 6;
    if (o->daily != 0) k += 8;
    pb200::SeasTab t;
    opts_table(o, &t);
    pb200::RegSpec r;
    opts_reg(o, &r);
    if (t.n > 0 || r.R > 0) k = pb200::tab_k(t, (1 << t.n) - 1) + r.R;
    out->kmax = k > 0 ? k : 1;
    out->pstride = 3 + out->smax + out->kmax;
    out->meta_i32_stride = 8;
    out->meta_i64_stride = 2;
    out->meta_f64_stride = 4;
    return PB200_OK;
}

PB200_API const char* pb200_last_error(void) { return g_err.c_str(); }

PB200_API pb200_ctx* pb200_create(int device) {
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        fail(PB200_E_CUDA, "no CUDA device (this library has no CPU path)", e);
        return nullptr;
    }
    if (device < 0 || device >= n) {
        fail(PB200_E_ARG, "device index out of range");
        return nullptr;
    }
    if (cudaSetDevice(device) != cudaSuccess) {
        fail(PB200_E_CUDA, "cudaSetDevice");
        return nullptr;
    }
    pb200_ctx* c = new pb200_ctx();
    c->device = device;
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    c->sms = prop.multiProcessorCount;
    c->l2_bytes = (size_t)prop.l2CacheSize;
    if (prop.major != 9 || prop.minor != 0) {
        fail(PB200_E_CUDA, "device is not sm_90 (this library is compiled for sm_90a only)");
        delete c;
        return nullptr;
    }
    if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&c->ctl_ev, cudaEventDisableTiming) != cudaSuccess) {
        fail(PB200_E_CUDA, "cudaStreamCreate / cudaEventCreate");
        if (c->stream) cudaStreamDestroy(c->stream);
        delete c;
        return nullptr;
    }
    c->lc0_max = env_int("PB200_LC0_MAX", 1 << 30);
    c->lc_auto = !getenv("PB200_LC0_MAX");
    c->tab_on = env_int("PB200_NO_TAB", 0) == 0;
    c->grp_g = env_int("PB200_GROUP", -1);
    if (c->grp_g != -1 && c->grp_g != 8 && c->grp_g != 16) c->grp_g = 0;
    c->grp_min = env_int("PB200_GROUP_MIN", 16384);
    c->plain_grp = env_int("PB200_PLAIN_GROUP", 0) != 0;
    c->l2_keep_pct = std::min(100, env_int("PB200_L2_KEEP_PCT", 65));
    c->grid_max = std::max(0, env_int("PB200_FIT_GRID_MAX", 0));
    return c;
}

PB200_API void pb200_destroy(pb200_ctx* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);
    for (DevBuf* b : {&c->d_offsets, &c->d_order, &c->d_lenclass, &c->d_qitems, &c->d_qctl, &c->d_qkey, &c->d_qhist,
                      &c->d_nq, &c->d_planes, &c->d_vcount, &c->d_warm_x, &c->d_regbad, &c->d_hoff})
        b->release();
    for (DevBuf& b : c->stage) b.release();
    c->h_ctl.release();
    cudaEventDestroy(c->ctl_ev);
    cudaStreamDestroy(c->stream);
    delete c;
}

PB200_API void* pb200_stream(pb200_ctx* c) { return c ? (void*)c->stream : nullptr; }
PB200_API int64_t pb200_launch_count(pb200_ctx* c) { return c ? c->launches : 0; }

PB200_API int32_t pb200_tab_chunk(int32_t T, int32_t P) {
    if (T < 1 || P < 2) return -1;
    return pb200::tab_chunk(T, P);
}

PB200_API int pb200_last_fit_variant_counts(pb200_ctx* c, int32_t* h_counts) {
    if (!c || !h_counts) return fail(PB200_E_ARG, "null argument");
    static_assert(PB200_N_VARIANT_COUNTS == NQ, "variant count layout");
    for (int i = 0; i < NQ; ++i) h_counts[i] = 0;
    if (!c->d_vcount.p) return PB200_OK;      // no fit yet
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    CK(cudaMemcpy(h_counts, c->d_vcount.p, NQ * 4, cudaMemcpyDeviceToHost));
    return PB200_OK;
}

PB200_API int32_t pb200_component_count(const pb200_options* o) {
    int rc = check_opts(o);
    if (rc) return rc;
    pb200::SeasTab t;
    opts_table(o, &t);
    return t.n > 0 ? t.nplanes : PB200_N_COMPONENTS;
}

PB200_API int pb200_last_fit_table_count(pb200_ctx* c, int64_t* h_count) {
    if (!c || !h_count) return fail(PB200_E_ARG, "null argument");
    *h_count = 0;
    if (!c->d_vcount.p) return PB200_OK;      // no fit yet
    int32_t n = 0;
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    CK(cudaMemcpy(&n, (const int32_t*)c->d_vcount.p + NQ, 4, cudaMemcpyDeviceToHost));
    *h_count = n;
    return PB200_OK;
}

PB200_API int pb200_synchronize(pb200_ctx* c) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    CK(cudaSetDevice(c->device));
    CK(cudaStreamSynchronize(c->stream));
    return PB200_OK;
}

}  // extern "C"

// newton_kernel over the queue {count, head, items...} at d_nq (16-warp CTAs with up to ~113 KB of shared memory, at P = 67)
// (f's series, offsets and queue as fit_impl staged them; x0: the warm start points, or null)
static int launch_newton(pb200_ctx* c, const FitCall& f, const double* x0) {
    static_assert(pb200::SEAS_PMAX <= pb200::nw::NW_PMAX, "newton_kernel holds every P check_opts admits");
    pb200_layout L;
    pb200_get_layout(f.opts, &L);
    if (f.opts->algorithm == PB200_ALG_LBFGS) return PB200_OK;
    int* nq = (int*)c->d_nq.p;
    pb200::nw::NewtonArgs na;
    na.ds = (const long long*)f.ds;
    na.y = f.y;
    na.y_dtype = f.y_dtype;
    na.offsets = (const long long*)c->d_offsets.p;
    na.nq_count = nq;
    na.nq_head = nq + 1;
    na.nq_items = nq + 2;
    na.params = f.params;
    na.tchange = f.tchange;
    na.meta_i32 = f.meta_i32;
    na.meta_i64 = (const long long*)f.meta_i64;
    na.meta_f64 = f.meta_f64;
    na.smax = L.smax;
    na.kmax = L.kmax;
    na.pstride = L.pstride;
    na.prior = f.prior;
    na.x0 = x0;
    na.o = to_dev(f.opts);
    opts_table(f.opts, &na.tab);
    opts_reg(f.opts, &na.reg);
    na.reg_x = f.reg;
    na.reg_scale = f.reg_scale;
    na.n_rows = f.offsets[f.n_series];
    const size_t nsm = pb200::nw::newton_smem_bytes(L.pstride);
    CK(cudaFuncSetAttribute(pb200::nw::newton_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)nsm));
    int ngrid = (int)std::min<int64_t>(f.n_series, f.opts->algorithm == PB200_ALG_NEWTON ? (int64_t)c->sms * 2 : (int64_t)c->sms);
    if (c->grid_max > 0) ngrid = std::min(ngrid, c->grid_max);
    pb200::nw::newton_kernel<<<ngrid, 32 * pb200::nw::NW_WARPS, nsm, c->stream>>>(na);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

// every fit call: zeroes the variant counters, then queues, fit kernels and (unless this is an objective evaluation,
// f.grad set) the Newton retry on the context's stream
static int fit_impl(pb200_ctx* c, const FitCall& f) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    CK(cudaSetDevice(c->device));
    CK(c->d_vcount.reserve((NQ + 1) * 4));     // [NQ]: the table class
    CK(cudaMemsetAsync(c->d_vcount.p, 0, (NQ + 1) * 4, c->stream));
    int rc = check_opts(f.opts, f.regs);
    if (rc) return rc;
    pb200::SeasTab tab;
    opts_table(f.opts, &tab);
    pb200::RegSpec reg;
    opts_reg(f.opts, &reg);
    const bool tabcls = tab.n > 0 || reg.R > 0;     // the table class (fit_table.cu)
    if (tabcls) {
        if (f.prior) return fail(PB200_E_UNSUPPORTED, "per-series prior scales are not supported with a seasonality table");
        if (f.init_params) return fail(PB200_E_UNSUPPORTED, "warm start is not supported with a seasonality table");
    }
    const int NQT = NLC * NQ + 1;    // the work queues: (length class, variant, mask), then the table class
    if (f.n_series < 0 || f.n_series > (1LL << 30)) return fail(PB200_E_ARG, "n_series");
    if (f.n_series == 0) return PB200_OK;
    if (!f.ds || !f.y || !f.offsets || !f.params || !f.tchange || !f.meta_i32 || !f.meta_i64 || !f.meta_f64)
        return fail(PB200_E_ARG, "null pointer");
    if (f.y_dtype < 0 || f.y_dtype > 2) return fail(PB200_E_ARG, "y_dtype");
    if (f.init_params && !f.init_meta) return fail(PB200_E_ARG, "d_init_meta_i32 is null");
    if (reg.R > 0 && (!f.reg || !f.reg_scale)) return fail(PB200_E_ARG, "null pointer (regressors / reg_scale)");
    pb200_layout L;
    pb200_get_layout(f.opts, &L);
    const int N = (int)f.n_series;
    const double* warm_x = nullptr;     // the start points prep_kernel writes for the fit kernels and the Newton retry
    if (f.init_params) {
        CK(c->d_warm_x.reserve((size_t)N * L.pstride * 8));
        warm_x = (const double*)c->d_warm_x.p;
    }

    // ---- host: length classes and longest-first order (counting sort on T) ----
    size_t ctl_bytes = (size_t)(N + 1) * 8 + (size_t)N * 4 * 2;
    if (c->ctl_pending) {   // the pinned staging of the previous call must have been consumed
        CK(cudaEventSynchronize(c->ctl_ev));
        c->ctl_pending = false;
    }
    CK(c->h_ctl.reserve(ctl_bytes));
    int64_t* ho = (int64_t*)c->h_ctl.p;
    int* horder = (int*)(ho + N + 1);
    int* hlc = horder + N;
    memcpy(ho, f.offsets, (size_t)(N + 1) * 8);
    int lc_n[NLC] = {0, 0}, lc_tmax[NLC] = {0, 0};
    int64_t tmax_all = 0;
    for (int i = 0; i < N; ++i) {
        const int64_t T = ho[i + 1] - ho[i];
        if (T < 0) return fail(PB200_E_ARG, "offsets not monotone");
        if (T > tmax_all) tmax_all = T;
    }
    if (tmax_all > (1 << 24)) return fail(PB200_E_UNSUPPORTED, "series longer than 2^24 rows");
    {
        std::vector<int> cnt((size_t)tmax_all + 2, 0);
        for (int i = 0; i < N; ++i) cnt[(size_t)(ho[i + 1] - ho[i])]++;
        // descending T: position of length t = number of series with length > t
        std::vector<int> posv((size_t)tmax_all + 2, 0);
        int acc = 0;
        for (int64_t t = tmax_all; t >= 0; --t) { posv[(size_t)t] = acc; acc += cnt[(size_t)t]; }
        for (int i = 0; i < N; ++i) {
            const int T = (int)(ho[i + 1] - ho[i]);
            horder[posv[(size_t)T]++] = i;
            // CTA width: one warp per series fills the chip once there are >= ~8 series per SM; a small
            // batch of long series gets 4 warps per series instead (same kernels, NT = 128)
            const int lc = (T > c->lc0_max || (c->lc_auto && N < c->sms * 8 && T >= 256)) ? 1 : 0;
            hlc[i] = lc;
            lc_n[lc]++;
            if (T > lc_tmax[lc]) lc_tmax[lc] = T;
        }
    }
    // ---- device control buffers ----
    CK(c->d_offsets.reserve((size_t)(N + 1) * 8));
    CK(c->d_order.reserve((size_t)N * 4));
    CK(c->d_lenclass.reserve((size_t)N * 4));
    CK(c->d_qitems.reserve((size_t)NQT * N * 4));
    CK(c->d_qctl.reserve((size_t)NQT * 2 * 4));
    CK(c->d_qkey.reserve((size_t)N * 4));
    CK(c->d_qhist.reserve((size_t)NQT * pb200::QBINS * 4));
    CK(cudaMemsetAsync(c->d_qkey.p, 0xff, (size_t)N * 4, c->stream));
    CK(cudaMemsetAsync(c->d_qhist.p, 0, (size_t)NQT * pb200::QBINS * 4, c->stream));
    CK(c->d_nq.reserve((size_t)(N + 2) * 4));             // count, head, items[N]
    int* nq = (int*)c->d_nq.p;
    CK(cudaMemsetAsync(nq, 0, 8, c->stream));
    CK(cudaMemcpyAsync(c->d_offsets.p, ho, (size_t)(N + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemcpyAsync(c->d_order.p, horder, (size_t)N * 4, cudaMemcpyHostToDevice, c->stream));
    CK(cudaMemcpyAsync(c->d_lenclass.p, hlc, (size_t)N * 4, cudaMemcpyHostToDevice, c->stream));
    CK(cudaEventRecord(c->ctl_ev, c->stream));
    c->ctl_pending = true;
    CK(cudaMemsetAsync(c->d_qctl.p, 0, (size_t)NQT * 2 * 4, c->stream));
    CK(cudaMemsetAsync(f.params, 0, (size_t)N * L.pstride * 8, c->stream));
    CK(cudaMemsetAsync(f.tchange, 0, (size_t)N * L.smax * 8, c->stream));
    int* q_count = (int*)c->d_qctl.p;
    int* q_head = q_count + NQT;
    const int64_t n_rows = ho[N];
    // ---- the regressors' standardisation, which prep_kernel's status and every evaluation read ----
    if (reg.R > 0) {
        CK(c->d_regbad.reserve((size_t)N));
        pb200::RegScaleArgs ra;
        ra.reg = f.reg;
        ra.n_rows = n_rows;
        ra.offsets = (const long long*)c->d_offsets.p;
        ra.n_series = N;
        ra.spec = reg;
        ra.reg_scale = f.reg_scale;
        ra.bad = (unsigned char*)c->d_regbad.p;
        ra.scale_copy = f.reg_scale_copy;
        pb200::reg_scale_kernel<<<std::min((N + 7) / 8, c->sms * 8), 256, 0, c->stream>>>(ra);
        CK(cudaGetLastError());
        c->launches++;
    }

    const FitOptsDev od = to_dev(f.opts);
    // lanes per series of the grouped day-table kernel
    const int grp_g = !c->tab_on ? 0 : (c->grp_g >= 0 ? c->grp_g : (N >= c->grp_min ? 8 : 16));
    // ---- prep kernel ----
    {
        pb200::PrepArgs pa;
        pa.ds = (const long long*)f.ds;
        pa.y = f.y;
        pa.y_dtype = f.y_dtype;
        pa.offsets = (const long long*)c->d_offsets.p;
        pa.order = (const int*)c->d_order.p;
        pa.cap = f.cap;
        pa.floor = f.floor;
        pa.cap_multiplier = f.cap_multiplier;
        pa.n_series = N;
        pa.meta_i32 = f.meta_i32;
        pa.meta_i64 = (long long*)f.meta_i64;
        pa.meta_f64 = f.meta_f64;
        pa.lenclass = (const int*)c->d_lenclass.p;
        pa.q_items = (int*)c->d_qitems.p;
        pa.q_count = q_count;
        pa.o = od;
        pa.tab_lc_mask = 0;
        for (int lc = 0; lc < NLC; ++lc)
            if (c->tab_on && LC_NT[lc] == 32) pa.tab_lc_mask |= 1 << lc;
        pa.grp_g = grp_g;
        pa.grp_plain = (c->plain_grp && grp_g > 0) ? 1 : 0;
        pa.cv_weight = QKEY_CV_WEIGHT;
        pa.newton_only = (f.opts->algorithm == PB200_ALG_NEWTON && !f.grad) ? 1 : 0;
        pa.nq_count = nq;
        pa.nq_items = nq + 2;
        pa.vcount = (int*)c->d_vcount.p;
        pa.qkey = (int*)c->d_qkey.p;
        pa.qhist = (int*)c->d_qhist.p;
        pa.prior = f.prior;
        pa.init_params = f.init_params;
        pa.init_meta = f.init_meta;
        pa.warm_x = (double*)warm_x;
        pa.warm = f.warm;
        pa.smax = L.smax;
        pa.pstride = L.pstride;
        pa.tab = tab;
        pa.tab_queue = NLC * NQ;
        pa.reg_bad = reg.R > 0 ? (const unsigned char*)c->d_regbad.p : nullptr;
        const int warps_per_block = 8;
        int grid = (N + warps_per_block - 1) / warps_per_block;
        grid = std::min(grid, c->sms * 8);
        pb200::prep_kernel<<<grid, warps_per_block * 32, 0, c->stream>>>(pa);
        CK(cudaGetLastError());
        pb200::queue_scan_kernel<<<(NQT + 127) / 128, 128, 0, c->stream>>>((int*)c->d_qhist.p, NQT);
        CK(cudaGetLastError());
        pb200::queue_scatter_kernel<<<std::min((N + 255) / 256, c->sms * 8), 256, 0, c->stream>>>(
            (const int*)c->d_qkey.p, (int*)c->d_qhist.p, (int*)c->d_qitems.p, N);
        CK(cudaGetLastError());
        c->launches += 3;
    }
    // ---- fit kernels: one persistent launch per (length class, seasonality class) ----
    // pass 1: launch geometry and the planes workspace (one slice per resident CTA)
    struct Geo { int grid, Tp, ppad; size_t smem, slice, off; bool on, grouped; };
    Geo geo[NLC][NQ];       // [length class][variant * 8 + seasonality class]
    size_t planes_bytes = 0;
    auto cap_grid = [&](int64_t grid) { return (int)(c->grid_max > 0 ? std::min<int64_t>(grid, c->grid_max) : grid); };
    for (int lc = 0; lc < NLC; ++lc)
        for (int rm = 0; rm < NQ; ++rm) {
            const int mask = rm & 7, reg = rm >> 3;
            Geo& g = geo[lc][rm];
            g.on = false;
            g.grouped = false;
            if (lc_n[lc] == 0 || tabcls) continue;
            const bool plain_grp = reg == 3 && mask == 0 && grp_g > 0 && c->plain_grp;   // grouped kernel's class without seasonality
            if (reg && mask == 0 && !plain_grp) continue;                // no Fourier features: nothing to regenerate
            if (reg >= 2 && ((mask != 6 && !plain_grp) || LC_NT[lc] != 32 || !c->tab_on)) continue;   // seasonal-table variants
            auto impossible = [&](int bit, int sw) { return (sw == 0 && (mask & bit)) || (sw == 1 && !(mask & bit)); };
            if (impossible(1, f.opts->yearly) || impossible(2, f.opts->weekly) || impossible(4, f.opts->daily)) continue;
            const int NT = LC_NT[lc];
            const int chunk = std::max((lc_tmax[lc] + NT - 1) / NT, 1);
            g.Tp = ((lc_tmax[lc] + chunk + pb200::TAB_CHUNK_SLACK + 1 + 7) / 8) * 8;   // the table variants may widen a chunk
            const int K = mask_k(mask);
            g.ppad = ((L.smax + (K > 0 ? K : 1) + 3) + 1) & ~1;
            const int nst = reg ? 0 : mask_nseas(mask);                    // stored feature planes
            const int nsa = (mask & 1) + ((mask >> 1) & 1) + ((mask >> 2) & 1);   // active seasonalities
            g.smem = pb200::fit_smem_bytes(NT, 1 + nst, g.ppad, reg == 1 ? nsa : (reg == 2 ? 1 : (reg == 3 ? 2 : 0)),
                                           reg == 2 ? pb200::PTAB_WEEK_MAX : (reg == 3 ? pb200::PTAB_DAY_MAX : 0));
            int occ = 0;
            FitArgs dummy{};
            g.slice = (size_t)(1 + nst) * g.Tp;                   // double2 elements
            g.off = planes_bytes;
            if (reg == 3 && grp_g > 0) {
                // grouped day-table kernel: one warp per CTA, 32 / grp_g series per warp, one workspace slot per series
                const int nser = 32 / grp_g;
                CK(pb200::launch_fit_group(grp_g, f.opts->growth, f.opts->multiplicative ? 1 : 0, mask != 0, dummy, 0, c->stream, &occ));
                if (occ < 1) return fail(PB200_E_UNSUPPORTED, "grouped fit kernel does not fit on an SM");
                g.grouped = true;
                g.slice = pb200::fit_group_plane_doubles(lc_tmax[lc], grp_g);           // doubles per slot
                g.grid = cap_grid(std::min<int64_t>(((int64_t)lc_n[lc] + nser - 1) / nser, (int64_t)c->sms * occ));
                planes_bytes += (size_t)g.grid * nser * g.slice * 8;
                g.on = true;
                continue;
            }
            CK(LAUNCH[mask](NT, f.opts->growth, reg, dummy, 0, g.smem, c->stream, &occ));
            if (occ < 1) return fail(PB200_E_UNSUPPORTED, "fit kernel does not fit on an SM");
            g.grid = cap_grid(std::min<int64_t>((int64_t)lc_n[lc], (int64_t)c->sms * occ));
            planes_bytes += (size_t)g.grid * g.slice * 16;
            g.on = true;
        }
    // the table class: one warp per series, (t, y) and one base (sin, cos) plane per table entry in each slice, then
    // ceil(R / 2) planes of the standardised regressors
    int tab_grid = 0, tab_Tp = 0, tab_ppad = 0, tab_planes = 0;
    size_t tab_smem = 0, tab_off = 0;
    if (tabcls) {
        tab_Tp = (int)(((tmax_all + (tmax_all + 31) / 32 + 7) / 8) * 8);
        tab_ppad = (L.pstride + 1) & ~1;
        tab_planes = 1 + tab.n + (reg.R + 1) / 2;
        tab_smem = reg.R > 0 ? pb200::fit_table_reg_smem(tab_ppad) : pb200::fit_table_smem(tab_ppad);
        int occ = 0;
        if (reg.R > 0) {
            pb200::RegTableFitArgs dummy{};
            CK(pb200::launch_fit_table_reg(f.opts->growth, dummy, 0, tab_smem, c->stream, &occ));
        } else {
            pb200::TableFitArgs dummy{};
            CK(pb200::launch_fit_table(f.opts->growth, dummy, 0, tab_smem, c->stream, &occ));
        }
        if (occ < 1) return fail(PB200_E_UNSUPPORTED, "table fit kernel does not fit on an SM");
        tab_grid = cap_grid(std::min<int64_t>((int64_t)N, (int64_t)c->sms * occ));
        tab_off = planes_bytes;
        planes_bytes += (size_t)tab_grid * tab_planes * tab_Tp * 16;
    }
    CK(c->d_planes.reserve(planes_bytes));
    // the arguments every fit launch shares; each launch adds its queue, workspace and geometry.  The table class has no
    // warm start and no per-series prior scales (refused above), so it gets theta and a null prior from here too
    FitArgs base{};
    base.ds = (const long long*)f.ds;
    base.y = f.y;
    base.y_dtype = f.y_dtype;
    base.offsets = (const long long*)c->d_offsets.p;
    base.params = f.params;
    base.tchange = f.tchange;
    base.meta_i32 = f.meta_i32;
    base.meta_i64 = (long long*)f.meta_i64;
    base.meta_f64 = f.meta_f64;
    base.smax = L.smax;
    base.kmax = L.kmax;
    base.pstride = L.pstride;
    base.theta_in = f.theta ? f.theta : warm_x;
    base.grad_out = f.grad;
    base.trace = f.trace;
    base.trace_cap = f.trace_cap;
    base.nq_count = nq;
    base.nq_items = f.opts->algorithm == PB200_ALG_LBFGS_NEWTON ? nq + 2 : nullptr;
    base.o = od;
    base.prior = f.prior;
    base.l2_keep = base.l2_rest_first = 0;
    if (tabcls) {
        pb200::TableFitArgs fa;
        static_cast<FitArgs&>(fa) = base;
        const int q = NLC * NQ;
        fa.q_items = (const int*)c->d_qitems.p + (size_t)q * N;
        fa.q_count = q_count + q;
        fa.q_head = q_head + q;
        fa.Tp = tab_Tp;
        fa.ppad = tab_ppad;
        fa.planes = (double2*)((char*)c->d_planes.p + tab_off);
        fa.nseas_stride = tab_planes * tab_Tp;
        fa.tab = tab;
        if (reg.R > 0) {
            pb200::RegTableFitArgs ra;
            static_cast<pb200::TableFitArgs&>(ra) = fa;
            ra.reg = f.reg;
            ra.reg_scale = f.reg_scale;
            ra.n_rows = n_rows;
            ra.spec = reg;
            CK(pb200::launch_fit_table_reg(f.opts->growth, ra, tab_grid, tab_smem, c->stream, nullptr));
        } else {
            CK(pb200::launch_fit_table(f.opts->growth, fa, tab_grid, tab_smem, c->stream, nullptr));
        }
        c->launches++;
    }
    for (int lc = 0; lc < NLC && !tabcls; ++lc) {
        if (lc_n[lc] == 0) continue;
        const int NT = LC_NT[lc];
        for (int rm = 0; rm < NQ; ++rm) {
            const int mask = rm & 7, reg = rm >> 3;
            const Geo& g = geo[lc][rm];
            if (!g.on) continue;
            FitArgs fa = base;
            const int q = lc * NQ + rm;
            fa.q_items = (const int*)c->d_qitems.p + (size_t)q * N;
            fa.q_count = q_count + q;
            fa.q_head = q_head + q;
            fa.Tp = g.Tp;
            fa.ppad = g.ppad;
            fa.planes = (double2*)((char*)c->d_planes.p + g.off);
            fa.nseas_stride = (int)g.slice;
            if (g.grouped && c->l2_keep_pct >= 0) {
                // the slots' y planes are read once per evaluation round, cyclically: an LRU-like L2 smaller than all of them
                // would miss on nearly every line.  A fixed subset that fits stays resident (evict_last); the rest streams
                // from HBM (evict_first, so that it does not push the subset out) behind the point pass's cp.async ring
                const int64_t nslots = (int64_t)g.grid * (32 / grp_g);
                fa.l2_keep = (int)std::min<int64_t>(nslots, (int64_t)(c->l2_bytes / 100) * c->l2_keep_pct / ((int64_t)g.slice * 8));
                fa.l2_rest_first = 1;
            }
            if (g.grouped) {
                CK(pb200::launch_fit_group(grp_g, f.opts->growth, f.opts->multiplicative ? 1 : 0, mask != 0, fa, g.grid, c->stream, nullptr));
            } else {
                CK(LAUNCH[mask](NT, f.opts->growth, reg, fa, g.grid, g.smem, c->stream, nullptr));
            }
            c->launches++;
        }
    }
    // ---- fbprophet's Newton retry over the series whose L-BFGS failed its line search (normally an empty queue) ----
    if (!f.grad) return launch_newton(c, f, warm_x);
    return PB200_OK;
}

// argument checks of the *_host fit entry points (outs: the caller's own pointers are all set); n_series == 0 passes
static int check_host_fit(pb200_ctx* c, const FitCall& h, bool outs) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    int rc = check_opts(h.opts, h.regs);
    if (rc) return rc;
    if (h.n_series <= 0) return h.n_series == 0 ? PB200_OK : fail(PB200_E_ARG, "n_series");
    if (!h.ds || !h.y || !h.offsets || !outs) return fail(PB200_E_ARG, "null pointer");
    if (h.y_dtype < 0 || h.y_dtype > 2) return fail(PB200_E_ARG, "y_dtype");
    return PB200_OK;
}

// ... and their common staging of d's series (host arrays in, device arrays after): ds and y in, with R regressors their
// values in and their (mu, std) out
static void stage_series(Staging& s, FitCall& d, int R) {
    const size_t N = (size_t)d.n_series, rows = (size_t)d.offsets[d.n_series];
    d.ds = s.in(ST_DS, d.ds, rows);
    d.y = s.in(ST_Y, (const char*)d.y, rows * y_elem(d.y_dtype));
    d.reg = s.in(ST_REG, R > 0 ? d.reg : nullptr, (size_t)R * rows);
    d.reg_scale = s.out(ST_REGSC, R > 0 ? d.reg_scale : nullptr, N * R * 2);
}

// pb200_fit_host, pb200_fit_trace_host, pb200_fit_warm_host and pb200_fit_regressors_host (h: host arrays; traced:
// h.trace_cap trajectory rows per series into h.trace): copy in, fit, copy out
static int fit_host(pb200_ctx* c, const FitCall& h, bool traced) {
    int rc = check_host_fit(c, h, h.params && h.tchange && h.meta_i32 && h.meta_i64 && h.meta_f64 && (h.trace || !traced));
    if (rc || h.n_series == 0) return rc;
    if (h.init_params && !h.init_meta) return fail(PB200_E_ARG, "h_init_meta_i32 is null");
    if (traced && (h.trace_cap < 1 || (int64_t)h.trace_cap * h.n_series > (1LL << 26))) return fail(PB200_E_ARG, "trace_cap");
    pb200::RegSpec reg;
    opts_reg(h.opts, &reg);
    if (reg.R > 0 && (!h.reg || !h.reg_scale)) return fail(PB200_E_ARG, "null pointer (regressors / reg_scale)");
    pb200_layout L;
    pb200_get_layout(h.opts, &L);
    const size_t N = (size_t)h.n_series;
    Staging s(c);
    FitCall d = h;
    stage_series(s, d, reg.R);
    d.cap = s.in(ST_CAP, h.cap, N);
    d.prior = s.in(ST_PRIOR, h.prior, N * 2);
    d.init_params = s.in(ST_IPARAMS, h.init_params, N * L.pstride);
    d.init_meta = s.in(ST_IMETA, h.init_params ? h.init_meta : nullptr, N * 8);
    d.warm = s.out(ST_WARM, h.init_params ? h.warm : nullptr, N);
    d.trace = s.out(ST_TRACE, traced ? h.trace : nullptr, N * (size_t)h.trace_cap * 4, true);
    d.params = s.out(ST_PARAMS, h.params, N * L.pstride);
    d.tchange = s.out(ST_TCHANGE, h.tchange, N * L.smax);
    d.meta_i32 = s.out(ST_MI32, h.meta_i32, N * 8);
    d.meta_i64 = s.out(ST_MI64, h.meta_i64, N * 2);
    d.meta_f64 = s.out(ST_MF64, h.meta_f64, N * 4);
    if ((rc = s.status()) || (rc = fit_impl(c, d))) return rc;
    return s.finish();
}

// pb200_objective_host and pb200_objective_regressors_host (h: host arrays; the objective goes to h_f): -log p and its
// gradient at h.theta
static int objective_host(pb200_ctx* c, const FitCall& h, double* h_f) {
    int rc = check_host_fit(c, h, h.theta && h_f && h.grad && h.meta_i32);
    if (rc || h.n_series == 0) return rc;
    pb200::RegSpec reg;
    opts_reg(h.opts, &reg);
    if (reg.R > 0 && (!h.reg || !h.reg_scale)) return fail(PB200_E_ARG, "null pointer (regressors / reg_scale)");
    pb200_layout L;
    pb200_get_layout(h.opts, &L);
    const size_t N = (size_t)h.n_series;
    std::vector<double> mf(N * 4);
    Staging s(c);
    FitCall d = h;
    stage_series(s, d, reg.R);
    d.theta = s.in(ST_THETA, h.theta, N * L.pstride);
    d.grad = s.out(ST_GRAD, h.grad, N * L.pstride, true);
    d.params = (double*)s.reserve(ST_PARAMS, N * L.pstride * 8);
    d.tchange = (double*)s.reserve(ST_TCHANGE, N * L.smax * 8);
    d.meta_i32 = s.out(ST_MI32, h.meta_i32, N * 8);
    d.meta_i64 = (int64_t*)s.reserve(ST_MI64, N * 2 * 8);
    d.meta_f64 = s.out(ST_MF64, mf.data(), N * 4);
    if ((rc = s.status()) || (rc = fit_impl(c, d)) || (rc = s.finish())) return rc;
    for (size_t i = 0; i < N; ++i) h_f[i] = mf[i * 4 + 3];
    return PB200_OK;
}

extern "C" {

PB200_API int pb200_fit_prior_device(pb200_ctx* c, const pb200_options* opts, const int64_t* d_ds, const void* d_y,
                                     int32_t y_dtype, const int64_t* h_offsets, int64_t n_series, double floor,
                                     double cap_multiplier, const double* d_cap, const double* d_prior, double* d_params,
                                     double* d_tchange, int32_t* d_meta_i32, int64_t* d_meta_i64, double* d_meta_f64) {
    FitCall f = {opts, d_ds, d_y, y_dtype, h_offsets, n_series, floor, cap_multiplier, d_cap, d_params, d_tchange,
                 d_meta_i32, d_meta_i64, d_meta_f64};
    f.prior = d_prior;
    return fit_impl(c, f);
}

PB200_API int pb200_fit_warm_device(pb200_ctx* c, const pb200_options* opts, const int64_t* d_ds, const void* d_y,
                                    int32_t y_dtype, const int64_t* h_offsets, int64_t n_series, double floor,
                                    double cap_multiplier, const double* d_cap, const double* d_prior,
                                    const double* d_init_params, const int32_t* d_init_meta_i32, double* d_params,
                                    double* d_tchange, int32_t* d_meta_i32, int64_t* d_meta_i64, double* d_meta_f64,
                                    int32_t* d_warm) {
    FitCall f = {opts, d_ds, d_y, y_dtype, h_offsets, n_series, floor, cap_multiplier, d_cap, d_params, d_tchange,
                 d_meta_i32, d_meta_i64, d_meta_f64};
    f.prior = d_prior;
    f.init_params = d_init_params;
    f.init_meta = d_init_meta_i32;
    f.warm = d_init_params ? d_warm : nullptr;
    return fit_impl(c, f);
}

PB200_API int pb200_fit_warm_host(pb200_ctx* c, const pb200_options* opts, const int64_t* h_ds, const void* h_y,
                                  int32_t y_dtype, const int64_t* h_offsets, int64_t n_series, double floor,
                                  double cap_multiplier, const double* h_cap, const double* h_prior,
                                  const double* h_init_params, const int32_t* h_init_meta_i32, double* h_params,
                                  double* h_tchange, int32_t* h_meta_i32, int64_t* h_meta_i64, double* h_meta_f64,
                                  int32_t* h_warm, double* h_trace, int32_t trace_cap) {
    FitCall h = {opts, h_ds, h_y, y_dtype, h_offsets, n_series, floor, cap_multiplier, h_cap, h_params, h_tchange,
                 h_meta_i32, h_meta_i64, h_meta_f64};
    h.prior = h_prior;
    h.init_params = h_init_params;
    h.init_meta = h_init_meta_i32;
    h.warm = h_warm;
    h.trace = h_trace;
    h.trace_cap = trace_cap;
    return fit_host(c, h, h_trace != nullptr);
}

PB200_API int pb200_fit_device(pb200_ctx* c, const pb200_options* opts, const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                     const int64_t* h_offsets, int64_t n_series, double floor, double cap_multiplier,
                     const double* d_cap, double* d_params, double* d_tchange, int32_t* d_meta_i32,
                     int64_t* d_meta_i64, double* d_meta_f64) {
    const FitCall f = {opts, d_ds, d_y, y_dtype, h_offsets, n_series, floor, cap_multiplier, d_cap, d_params, d_tchange,
                       d_meta_i32, d_meta_i64, d_meta_f64};
    return fit_impl(c, f);
}

PB200_API int pb200_objective_host(pb200_ctx* c, const pb200_options* opts, const int64_t* h_ds, const void* h_y,
                                   int32_t y_dtype, const int64_t* h_offsets, int64_t n_series, double floor,
                                   double cap_multiplier, const double* h_theta, double* h_f, double* h_grad,
                                   int32_t* h_meta_i32) {
    FitCall h = {opts, h_ds, h_y, y_dtype, h_offsets, n_series, floor, cap_multiplier};
    h.theta = h_theta;
    h.grad = h_grad;
    h.meta_i32 = h_meta_i32;
    return objective_host(c, h, h_f);
}

PB200_API int pb200_objective_regressors_host(pb200_ctx* c, const pb200_options* opts, const int64_t* h_ds, const void* h_y,
                                              int32_t y_dtype, const int64_t* h_offsets, int64_t n_series, double floor,
                                              double cap_multiplier, const double* h_reg, double* h_reg_scale,
                                              const double* h_theta, double* h_f, double* h_grad, int32_t* h_meta_i32) {
    FitCall h = {opts, h_ds, h_y, y_dtype, h_offsets, n_series, floor, cap_multiplier};
    h.regs = true;
    h.reg = h_reg;
    h.reg_scale = h_reg_scale;
    h.theta = h_theta;
    h.grad = h_grad;
    h.meta_i32 = h_meta_i32;
    return objective_host(c, h, h_f);
}

PB200_API int pb200_fit_regressors_device(pb200_ctx* c, const pb200_options* opts, const int64_t* d_ds, const void* d_y,
                                          int32_t y_dtype, const int64_t* h_offsets, int64_t n_series, double floor,
                                          double cap_multiplier, const double* d_cap, const double* d_reg, double* d_reg_scale,
                                          double* d_params, double* d_tchange, int32_t* d_meta_i32, int64_t* d_meta_i64,
                                          double* d_meta_f64) {
    FitCall f = {opts, d_ds, d_y, y_dtype, h_offsets, n_series, floor, cap_multiplier, d_cap, d_params, d_tchange,
                 d_meta_i32, d_meta_i64, d_meta_f64};
    f.regs = true;
    f.reg = d_reg;
    f.reg_scale = d_reg_scale;
    return fit_impl(c, f);
}

PB200_API int pb200_fit_regressors_copy_device(pb200_ctx* c, const pb200_options* opts, const int64_t* d_ds,
                                               const void* d_y, int32_t y_dtype, const int64_t* h_offsets,
                                               int64_t n_series, double floor, double cap_multiplier, const double* d_cap,
                                               const double* d_reg, const double* d_reg_scale_copy, double* d_reg_scale,
                                               double* d_params, double* d_tchange, int32_t* d_meta_i32,
                                               int64_t* d_meta_i64, double* d_meta_f64) {
    if (!d_reg_scale_copy && n_series > 0) return fail(PB200_E_ARG, "null pointer (reg_scale_copy)");
    FitCall f = {opts, d_ds, d_y, y_dtype, h_offsets, n_series, floor, cap_multiplier, d_cap, d_params, d_tchange,
                 d_meta_i32, d_meta_i64, d_meta_f64};
    f.regs = true;
    f.reg = d_reg;
    f.reg_scale = d_reg_scale;
    f.reg_scale_copy = d_reg_scale_copy;
    return fit_impl(c, f);
}

PB200_API int pb200_regressor_scales_device(pb200_ctx* c, const pb200_options* opts, const double* d_reg,
                                            const int64_t* h_offsets, int64_t n_series, double* d_reg_scale,
                                            uint8_t* d_bad) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    int rc = check_opts(opts, true);
    if (rc) return rc;
    pb200::RegSpec reg;
    opts_reg(opts, &reg);
    if (reg.R < 1) return fail(PB200_E_ARG, "options without regressors");
    if (n_series < 0 || n_series > (1LL << 30)) return fail(PB200_E_ARG, "n_series");
    if (n_series == 0) return PB200_OK;
    if (!d_reg || !h_offsets || !d_reg_scale || !d_bad) return fail(PB200_E_ARG, "null pointer");
    for (int64_t i = 0; i < n_series; ++i)
        if (h_offsets[i + 1] < h_offsets[i] || h_offsets[0] != 0) return fail(PB200_E_ARG, "offsets");
    CK(cudaSetDevice(c->device));
    CK(c->d_offsets.reserve((size_t)(n_series + 1) * 8));
    CK(cudaMemcpyAsync(c->d_offsets.p, h_offsets, (size_t)(n_series + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    pb200::RegScaleArgs ra;
    ra.reg = d_reg;
    ra.n_rows = h_offsets[n_series];
    ra.offsets = (const long long*)c->d_offsets.p;
    ra.n_series = (int)n_series;
    ra.spec = reg;
    ra.reg_scale = d_reg_scale;
    ra.bad = d_bad;
    ra.scale_copy = nullptr;
    const int N = (int)n_series;
    pb200::reg_scale_kernel<<<std::min((N + 7) / 8, c->sms * 8), 256, 0, c->stream>>>(ra);
    CK(cudaGetLastError());
    c->launches++;
    CK(cudaStreamSynchronize(c->stream));      // the offsets' staging buffer is the context's
    return PB200_OK;
}

PB200_API int pb200_cv_gather_regressors_device(pb200_ctx* c, const double* d_reg, int64_t n_rows, int32_t n_regressors,
                                                const double* d_reg_scale_full, const int64_t* d_offsets,
                                                const int32_t* d_pair_series, const int64_t* d_hist_end,
                                                const int64_t* d_win_end, const int64_t* d_pairs, int64_t n,
                                                const int64_t* d_fit_off, int32_t hmax, double* d_reg_fit,
                                                double* d_reg_future) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n < 0 || hmax < 1 || n_rows < 0) return fail(PB200_E_ARG, "sizes");
    if (n_regressors < 1 || n_regressors > PB200_MAX_REGRESSORS) return fail(PB200_E_ARG, "n_regressors");
    if (n == 0) return PB200_OK;
    if (!d_reg || !d_reg_scale_full || !d_offsets || !d_pair_series || !d_hist_end || !d_win_end || !d_pairs ||
        !d_fit_off || !d_reg_fit || !d_reg_future)
        return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    pb200::CvRegGatherArgs a;
    a.reg = d_reg;
    a.n_rows = n_rows;
    a.R = n_regressors;
    a.scale_full = d_reg_scale_full;
    a.offsets = (const long long*)d_offsets;
    a.pair_series = d_pair_series;
    a.hist_end = (const long long*)d_hist_end;
    a.win_end = (const long long*)d_win_end;
    a.pairs = (const long long*)d_pairs;
    a.n = n;
    a.fit_off = (const long long*)d_fit_off;
    a.hmax = hmax;
    a.reg_fit = d_reg_fit;
    a.reg_fut = d_reg_future;
    const int grid = (int)std::min<int64_t>(n, (int64_t)c->sms * 32);
    pb200::cv_gather_regressors_kernel<<<grid, 256, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

PB200_API int pb200_fit_regressors_host(pb200_ctx* c, const pb200_options* opts, const int64_t* h_ds, const void* h_y,
                                        int32_t y_dtype, const int64_t* h_offsets, int64_t n_series, double floor,
                                        double cap_multiplier, const double* h_cap, const double* h_reg, double* h_reg_scale,
                                        double* h_params, double* h_tchange, int32_t* h_meta_i32, int64_t* h_meta_i64,
                                        double* h_meta_f64, double* h_trace, int32_t trace_cap) {
    FitCall h = {opts, h_ds, h_y, y_dtype, h_offsets, n_series, floor, cap_multiplier, h_cap, h_params, h_tchange,
                 h_meta_i32, h_meta_i64, h_meta_f64};
    h.regs = true;
    h.reg = h_reg;
    h.reg_scale = h_reg_scale;
    h.trace = h_trace;
    h.trace_cap = trace_cap;
    return fit_host(c, h, h_trace != nullptr && trace_cap > 0);
}

PB200_API int pb200_fit_host(pb200_ctx* c, const pb200_options* opts, const int64_t* h_ds, const void* h_y, int32_t y_dtype,
                   const int64_t* h_offsets, int64_t n_series, double floor, double cap_multiplier, const double* h_cap,
                   double* h_params, double* h_tchange, int32_t* h_meta_i32, int64_t* h_meta_i64, double* h_meta_f64) {
    const FitCall h = {opts, h_ds, h_y, y_dtype, h_offsets, n_series, floor, cap_multiplier, h_cap, h_params, h_tchange,
                       h_meta_i32, h_meta_i64, h_meta_f64};
    return fit_host(c, h, false);
}

PB200_API int pb200_fit_trace_host(pb200_ctx* c, const pb200_options* opts, const int64_t* h_ds, const void* h_y, int32_t y_dtype,
                         const int64_t* h_offsets, int64_t n_series, double floor, double cap_multiplier, double* h_params,
                         double* h_tchange, int32_t* h_meta_i32, int64_t* h_meta_i64, double* h_meta_f64, double* h_trace,
                         int32_t trace_cap) {
    FitCall h = {opts, h_ds, h_y, y_dtype, h_offsets, n_series, floor, cap_multiplier};
    h.params = h_params;
    h.tchange = h_tchange;
    h.meta_i32 = h_meta_i32;
    h.meta_i64 = h_meta_i64;
    h.meta_f64 = h_meta_f64;
    h.trace = h_trace;
    h.trace_cap = trace_cap;
    return fit_host(c, h, true);
}

PB200_API int pb200_make_future_device(pb200_ctx* c, const int64_t* d_last_ds, int64_t n_models, int32_t horizon, int64_t freq_ns,
                             int64_t* d_future_ds) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n_models < 0 || horizon < 0) return fail(PB200_E_ARG, "sizes");
    if (n_models == 0 || horizon == 0) return PB200_OK;
    if (!d_last_ds || !d_future_ds) return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    const int64_t n = n_models * horizon;
    const int grid = (int)std::min<int64_t>((n + 255) / 256, (int64_t)c->sms * 16);
    pb200::make_future_kernel<<<grid, 256, 0, c->stream>>>((const long long*)d_last_ds, n_models, horizon, freq_ns,
                                                           (long long*)d_future_ds);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

namespace {

// the component arguments of pb200_predict_components_*: the planes are required, the trend bounds come in pairs and
// ride on the yhat intervals
int check_comp_args(const pb200_options* o, const void* comp, const void* lo, const void* hi, const void* tlo,
                    const void* thi) {
    if (!comp) return fail(PB200_E_ARG, "null pointer (components)");
    if (!tlo != !thi) return fail(PB200_E_ARG, "trend_lower and trend_upper go together");
    if (tlo && !(lo && hi && o->uncertainty_samples > 0))
        return fail(PB200_E_ARG, "trend bounds need the yhat intervals (yhat_lower / yhat_upper, uncertainty_samples > 0)");
    return PB200_OK;
}

struct QuantOut;

// the window arguments of pb200_predict_sums_*: the rule, the slots per model and the seven outputs (device pointers in
// predict_device, host pointers in predict_host)
struct SumOut {
    int64_t width_ns, origin_ns;
    int32_t wmax;
    int32_t* n_windows;
    int64_t* win_start;
    int32_t* win_points;
    double* yhat_sum;
    int64_t* quantity_sum;
    double* sum_lower;
    double* sum_upper;
    // pb200_predict_sums_anchored_device: an origin and a frame length per model, in place of origin_ns and the horizon
    const int64_t* origins = nullptr;
    const int32_t* frame_len = nullptr;
    // pb200_predict_period_sums_*: the calendar periods of (months, month_shift), in place of width_ns / origin_ns
    int32_t months = 0, month_shift = 0;
    // pb200_predict_*sums*_quantiles_*: the levels and their planes [n_q][n_models * wmax] (DESIGN §21)
    const QuantOut* quant = nullptr;
};

// checked before anything is copied or launched
int check_sum_args(const pb200_options* o, const SumOut& s) {
    const int rc = check_mc_opts(o);
    if (rc) return rc;
    if (s.months != 0) {
        if (!(s.months == 1 || s.months == 3 || s.months == 12) || s.month_shift < 0 || s.month_shift >= s.months)
            return fail(PB200_E_ARG, "months must be 1, 3 or 12 and month_shift in [0, months)");
    } else if (s.width_ns <= 0) {
        return fail(PB200_E_ARG, "width_ns must be > 0");
    }
    if (s.wmax <= 0) return fail(PB200_E_ARG, "wmax must be > 0");
    if (!s.n_windows || !s.win_start || !s.win_points || !s.yhat_sum || !s.quantity_sum || !s.sum_lower || !s.sum_upper)
        return fail(PB200_E_ARG, "null pointer (window outputs)");
    return PB200_OK;
}

// the level arguments of pb200_predict_quantiles_*: n_q percentiles (a host array) and the planes (device pointer in
// predict_device, host pointer in predict_host)
struct QuantOut {
    int32_t n_q;
    const double* percentiles;
    double* planes;
};

// checked before anything is copied or launched
int check_quant_args(const pb200_options* o, const QuantOut& q) {
    const int rc = check_mc_opts(o);
    if (rc) return rc;
    if (q.n_q < 1 || q.n_q > pb200::MC_QMAX) return fail(PB200_E_ARG, "n_q must be in [1, 32]");
    if (!q.percentiles || !q.planes) return fail(PB200_E_ARG, "null pointer (percentiles / quantiles)");
    for (int i = 0; i < q.n_q; ++i)
        if (!(q.percentiles[i] >= 0.0 && q.percentiles[i] <= 100.0)) return fail(PB200_E_ARG, "percentiles must be in [0, 100]");
    return PB200_OK;
}

// One predict request: device arrays in predict_device / predict_history_device, host arrays in predict_host /
// pb200_predict_history_host.  The leading members are the arguments every predict entry point takes, in their order;
// the others are optional
struct PredictCall {
    const pb200_options* opts;
    const double* params;
    const double* tchange;
    const int32_t* meta_i32;
    const int64_t* meta_i64;
    const double* meta_f64;
    int64_t n_models;
    const int64_t* future_ds;
    int32_t horizon;
    const double* floor;
    const double* cap;
    uint64_t seed;
    double* yhat;
    double* yhat_lower;
    double* yhat_upper;
    int32_t* yhat_int;
    double* comp = nullptr;          // the component planes and the trend bounds (pb200_predict_components_*)
    double* tlo = nullptr;
    double* thi = nullptr;
    const SumOut* sums = nullptr;    // window totals (pb200_predict_sums_*, pb200_predict_period_sums_*)
    const QuantOut* quant = nullptr;
    bool regs = false;               // a regressor entry point: the options may carry regressors
    const double* future_reg = nullptr;
    const double* reg_scale = nullptr;
    const int64_t* offsets = nullptr;   // pb200_predict_history_*: model i's rows of future_ds (a host array)
};

// the arguments every predict_kernel and mc_kernel instance takes
void predict_args(pb200::PredictArgs& a, const PredictCall& p) {
    pb200_layout L;
    pb200_get_layout(p.opts, &L);
    opts_table(p.opts, &a.tab);
    a.params = p.params;
    a.tchange = p.tchange;
    a.meta_i32 = p.meta_i32;
    a.meta_i64 = (const long long*)p.meta_i64;
    a.meta_f64 = p.meta_f64;
    a.future_ds = (const long long*)p.future_ds;
    a.floor = p.floor;
    a.cap = p.cap;
    a.n_models = (int)p.n_models;
    a.horizon = p.horizon;
    a.smax = L.smax;
    a.kmax = L.kmax;
    a.pstride = L.pstride;
    a.growth = p.opts->growth;
    a.mult = p.opts->multiplicative ? 1 : 0;
    a.yhat = p.yhat;
    a.trend = p.comp;
    a.yhat_int = p.yhat_int;
}

// pb200_predict_device; p.comp != null: the components instance of predict_kernel, p.tlo / p.thi != null: the
// trend-bounds instance of mc_kernel; p.sums != null: mc_sum_kernel after them (it also runs on an empty frame, where
// every model has no window), its per-model instance when sums->origins != null, its calendar instance when
// sums->months != 0; p.quant != null: mc_kernel also writes the quantile planes, from the same selection as the bounds
int predict_device(pb200_ctx* c, const PredictCall& p) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    int rc = check_opts(p.opts, p.regs);
    if (rc) return rc;
    if (p.n_models < 0 || p.horizon < 0 || p.n_models > (1LL << 30)) return fail(PB200_E_ARG, "sizes");
    if (p.sums && (rc = check_sum_args(p.opts, *p.sums))) return rc;
    if (p.sums && p.sums->quant && (rc = check_quant_args(p.opts, *p.sums->quant))) return rc;
    if (p.quant && (rc = check_quant_args(p.opts, *p.quant))) return rc;
    if (p.n_models == 0 || (p.horizon == 0 && !p.sums)) return PB200_OK;
    if (!p.params || !p.tchange || !p.meta_i32 || !p.meta_i64 || !p.meta_f64 || !p.floor || !p.cap ||
        (p.horizon > 0 && (!p.future_ds || !p.yhat || !p.yhat_int)))
        return fail(PB200_E_ARG, "null pointer");
    const bool mc = p.horizon > 0 && p.yhat_lower && p.yhat_upper && p.opts->uncertainty_samples > 0;
    if (mc && (rc = check_mc_opts(p.opts))) return rc;
    pb200::RegSpec reg;
    opts_reg(p.opts, &reg);
    if (reg.R > 0 && p.horizon > 0 && (!p.future_reg || !p.reg_scale)) return fail(PB200_E_ARG, "null pointer (regressors / reg_scale)");
    pb200::PredictArgs a;
    predict_args(a, p);
    CK(cudaSetDevice(c->device));
    if (reg.R > 0) {
        // the regressor instances: yhat and its interval (every other output is refused for these options by check_opts)
        pb200::RegPredictArgs ra;
        static_cast<pb200::PredictArgs&>(ra) = a;
        ra.reg.future_reg = p.future_reg;
        ra.reg.reg_scale = p.reg_scale;
        ra.reg.R = reg.R;
        if (p.horizon == 0) return PB200_OK;
        dim3 grid((unsigned)p.n_models, (unsigned)std::min((p.horizon + 1023) / 1024, 64));
        pb200::predict_kernel<false, false, true><<<grid, 256, 0, c->stream>>>(ra);
        CK(cudaGetLastError());
        c->launches++;
        if (mc) {
            rc = pb200::launch_mc_reg(c->stream, c->sms, a, ra.reg, p.opts->uncertainty_samples, p.opts->interval_width, p.seed,
                                      p.yhat_lower, p.yhat_upper);
            if (rc == -1) return fail(PB200_E_ARG, "uncertainty_samples / interval_width out of range");
            if (rc) return fail(PB200_E_CUDA, "mc kernel launch", cudaGetLastError());
            c->launches++;
        }
        return PB200_OK;
    }
    if (p.horizon > 0) {
        // one CTA per (model, 1024 future points): the per-model prologue (parameters, the serial gamma recurrence) is paid
        // once for config #5's 672 periods instead of three times
        dim3 grid((unsigned)p.n_models, (unsigned)std::min((p.horizon + 1023) / 1024, 64));
        if (p.comp) pb200::predict_kernel<true><<<grid, 256, 0, c->stream>>>(a);
        else pb200::predict_kernel<false><<<grid, 256, 0, c->stream>>>(a);
        CK(cudaGetLastError());
        c->launches++;
    }
    if (mc || (p.quant && p.horizon > 0)) {
        rc = pb200::launch_mc(c->stream, c->sms, a, p.opts->uncertainty_samples, p.opts->interval_width, p.seed,
                              mc ? p.yhat_lower : nullptr, mc ? p.yhat_upper : nullptr, p.tlo, p.thi, p.quant ? p.quant->n_q : 0,
                              p.quant ? p.quant->percentiles : nullptr, p.quant ? p.quant->planes : nullptr);
        if (rc == -1) return fail(PB200_E_ARG, "uncertainty_samples / interval_width / n_q out of range");
        if (rc) return fail(PB200_E_CUDA, "mc kernel launch", cudaGetLastError());
        c->launches++;
    }
    if (const SumOut* sums = p.sums) {
        pb200::McSumArgs s;
        s.mc.lower = sums->sum_lower;
        s.mc.upper = sums->sum_upper;
        s.width_ns = sums->width_ns;
        s.origin_ns = sums->origin_ns;
        s.wmax = sums->wmax;
        s.n_windows = sums->n_windows;
        s.win_start = (long long*)sums->win_start;
        s.win_points = sums->win_points;
        s.yhat_sum = sums->yhat_sum;
        s.quantity_sum = (long long*)sums->quantity_sum;
        s.origins = (const long long*)sums->origins;
        s.frame_len = sums->frame_len;
        const QuantOut* q = sums->quant;
        rc = pb200::launch_mc_sum(c->stream, c->sms, a, p.opts->uncertainty_samples, p.opts->interval_width, p.seed, s,
                                  sums->months, sums->month_shift, q ? q->n_q : 0, q ? q->percentiles : nullptr,
                                  q ? q->planes : nullptr);
        if (rc == -1) return fail(PB200_E_ARG, q ? "uncertainty_samples / interval_width / n_q out of range"
                                                 : "uncertainty_samples / interval_width out of range");
        if (rc) return fail(PB200_E_CUDA, "mc sum kernel launch", cudaGetLastError());
        c->launches++;
    }
    return PB200_OK;
}

// pb200_predict_host and the other fixed-frame *_host predict calls (h: host arrays): copy in, predict, copy out
int predict_host(pb200_ctx* c, const PredictCall& h) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    int rc = check_opts(h.opts, h.regs);
    if (rc) return rc;
    if (h.quant && (rc = check_quant_args(h.opts, *h.quant))) return rc;
    if (h.sums) {
        if (h.n_models < 0 || h.horizon < 0) return fail(PB200_E_ARG, "sizes");
        if ((rc = check_sum_args(h.opts, *h.sums))) return rc;
        if (h.sums->quant && (rc = check_quant_args(h.opts, *h.sums->quant))) return rc;
        if (h.n_models == 0) return PB200_OK;
    } else if (h.n_models <= 0 || h.horizon <= 0) {
        return (h.n_models == 0 || h.horizon == 0) ? PB200_OK : fail(PB200_E_ARG, "sizes");
    }
    if (!h.params || !h.tchange || !h.meta_i32 || !h.meta_i64 || !h.meta_f64 || !h.floor || !h.cap ||
        (h.horizon > 0 && (!h.future_ds || !h.yhat || !h.yhat_int)))
        return fail(PB200_E_ARG, "null pointer");
    const bool mc = h.horizon > 0 && h.yhat_lower && h.yhat_upper && h.opts->uncertainty_samples > 0;
    if (mc && (rc = check_mc_opts(h.opts))) return rc;
    pb200::RegSpec reg;
    opts_reg(h.opts, &reg);
    if (reg.R > 0 && (!h.future_reg || !h.reg_scale)) return fail(PB200_E_ARG, "null pointer (regressors / reg_scale)");
    pb200_layout L;
    pb200_get_layout(h.opts, &L);
    const size_t N = (size_t)h.n_models, NH = N * (size_t)h.horizon;
    Staging s(c);
    PredictCall d = h;
    d.params = s.in(ST_PARAMS, h.params, N * L.pstride);
    d.tchange = s.in(ST_TCHANGE, h.tchange, N * L.smax);
    d.meta_i32 = s.in(ST_MI32, h.meta_i32, N * 8);
    d.meta_i64 = s.in(ST_MI64, h.meta_i64, N * 2);
    d.meta_f64 = s.in(ST_MF64, h.meta_f64, N * 4);
    d.future_ds = s.in(ST_FUT, h.future_ds, NH);
    d.floor = s.in(ST_FLOOR, h.floor, N);
    d.cap = s.in(ST_CAP, h.cap, N);
    d.future_reg = s.in(ST_REG, reg.R > 0 ? h.future_reg : nullptr, NH * reg.R);
    d.reg_scale = s.in(ST_REGSC, reg.R > 0 ? h.reg_scale : nullptr, N * reg.R * 2);
    d.yhat = s.out(ST_YHAT, h.yhat, NH);
    d.yhat_int = s.out(ST_YINT, h.yhat_int, NH);
    d.yhat_lower = s.out(ST_LO, mc ? h.yhat_lower : nullptr, NH);
    d.yhat_upper = s.out(ST_HI, mc ? h.yhat_upper : nullptr, NH);
    d.comp = s.out(ST_COMP, h.comp, NH * pb200_component_count(h.opts));
    d.tlo = s.out(ST_TLO, h.tlo, NH);
    d.thi = s.out(ST_THI, h.thi, NH);
    QuantOut dquant;
    if (h.quant) {
        dquant = *h.quant;
        dquant.planes = s.out(ST_QUANT, h.quant->planes, NH * h.quant->n_q);
        d.quant = &dquant;
    }
    SumOut dsum;
    QuantOut dsq;
    if (const SumOut* hs = h.sums) {
        // on the device: five 8-byte arrays [N * wmax], the n_q planes [n_q][N * wmax] of the levels, then win_points
        // [N * wmax] and n_windows [N]
        const size_t NW = N * (size_t)hs->wmax, nq = hs->quant ? (size_t)hs->quant->n_q : 0;
        char* next = (char*)s.reserve(ST_SUMS, NW * (44 + 8 * nq) + N * 4);
        if ((rc = s.status())) return rc;
        auto carve = [&](auto* h, size_t n) {   // the next n elements of the buffer, copied back to h
            auto* dp = (decltype(h))next;
            next += n * sizeof *h;
            s.later(h, dp, n);
            return dp;
        };
        dsum = *hs;
        dsum.win_start = carve(hs->win_start, NW);
        dsum.quantity_sum = carve(hs->quantity_sum, NW);
        dsum.yhat_sum = carve(hs->yhat_sum, NW);
        dsum.sum_lower = carve(hs->sum_lower, NW);
        dsum.sum_upper = carve(hs->sum_upper, NW);
        if (hs->quant) {
            dsq = *hs->quant;
            dsq.planes = carve(hs->quant->planes, NW * nq);
            dsum.quant = &dsq;
        }
        dsum.win_points = carve(hs->win_points, NW);
        dsum.n_windows = carve(hs->n_windows, N);
        d.sums = &dsum;
    }
    if ((rc = s.status()) || (rc = predict_device(c, d))) return rc;
    return s.finish();
}

}  // namespace

PB200_API int pb200_predict_device(pb200_ctx* c, const pb200_options* opts, const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64, const double* d_meta_f64,
                         int64_t n_models, const int64_t* d_future_ds, int32_t horizon, const double* d_floor,
                         const double* d_cap, uint64_t seed, double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int) {
    const PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                           horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    return predict_device(c, p);
}

PB200_API int pb200_predict_host(pb200_ctx* c, const pb200_options* opts, const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64, const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon, const double* h_floor, const double* h_cap,
                       uint64_t seed, double* h_yhat, double* h_yhat_lower, double* h_yhat_upper, int32_t* h_yhat_int) {
    const PredictCall p = {opts, h_params, h_tchange, h_meta_i32, h_meta_i64, h_meta_f64, n_models, h_future_ds,
                           horizon, h_floor, h_cap, seed, h_yhat, h_yhat_lower, h_yhat_upper, h_yhat_int};
    return predict_host(c, p);
}

PB200_API int pb200_predict_regressors_device(pb200_ctx* c, const pb200_options* opts, const double* d_params,
                         const double* d_tchange, const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models, const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed, const double* d_future_reg,
                         const double* d_reg_scale, double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int) {
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                     horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    p.regs = true;
    p.future_reg = d_future_reg;
    p.reg_scale = d_reg_scale;
    return predict_device(c, p);
}

PB200_API int pb200_predict_regressors_host(pb200_ctx* c, const pb200_options* opts, const double* h_params,
                       const double* h_tchange, const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models, const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed, const double* h_future_reg,
                       const double* h_reg_scale, double* h_yhat, double* h_yhat_lower, double* h_yhat_upper,
                       int32_t* h_yhat_int) {
    PredictCall p = {opts, h_params, h_tchange, h_meta_i32, h_meta_i64, h_meta_f64, n_models, h_future_ds,
                     horizon, h_floor, h_cap, seed, h_yhat, h_yhat_lower, h_yhat_upper, h_yhat_int};
    p.regs = true;
    p.future_reg = h_future_reg;
    p.reg_scale = h_reg_scale;
    return predict_host(c, p);
}

PB200_API int pb200_predict_components_device(pb200_ctx* c, const pb200_options* opts, const double* d_params,
                         const double* d_tchange, const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models, const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed, double* d_yhat, double* d_yhat_lower,
                         double* d_yhat_upper, int32_t* d_yhat_int, double* d_components, double* d_trend_lower,
                         double* d_trend_upper) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    int rc = check_opts(opts);
    if (rc) return rc;
    if ((rc = check_comp_args(opts, d_components, d_yhat_lower, d_yhat_upper, d_trend_lower, d_trend_upper))) return rc;
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                     horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    p.comp = d_components;
    p.tlo = d_trend_lower;
    p.thi = d_trend_upper;
    return predict_device(c, p);
}

PB200_API int pb200_predict_components_host(pb200_ctx* c, const pb200_options* opts, const double* h_params,
                       const double* h_tchange, const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models, const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed, double* h_yhat, double* h_yhat_lower,
                       double* h_yhat_upper, int32_t* h_yhat_int, double* h_components, double* h_trend_lower,
                       double* h_trend_upper) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    int rc = check_opts(opts);
    if (rc) return rc;
    if ((rc = check_comp_args(opts, h_components, h_yhat_lower, h_yhat_upper, h_trend_lower, h_trend_upper))) return rc;
    PredictCall p = {opts, h_params, h_tchange, h_meta_i32, h_meta_i64, h_meta_f64, n_models, h_future_ds,
                     horizon, h_floor, h_cap, seed, h_yhat, h_yhat_lower, h_yhat_upper, h_yhat_int};
    p.comp = h_components;
    p.tlo = h_trend_lower;
    p.thi = h_trend_upper;
    return predict_host(c, p);
}

PB200_API int pb200_predict_sums_device(pb200_ctx* c, const pb200_options* opts, const double* d_params, const double* d_tchange,
                         const int32_t* d_meta_i32, const int64_t* d_meta_i64, const double* d_meta_f64,
                         int64_t n_models, const int64_t* d_future_ds, int32_t horizon, const double* d_floor,
                         const double* d_cap, uint64_t seed, double* d_yhat, double* d_yhat_lower, double* d_yhat_upper,
                         int32_t* d_yhat_int, int64_t width_ns, int64_t origin_ns, int32_t wmax, int32_t* d_n_windows,
                         int64_t* d_win_start, int32_t* d_win_points, double* d_yhat_sum, int64_t* d_quantity_sum,
                         double* d_sum_lower, double* d_sum_upper) {
    const SumOut s = {width_ns, origin_ns, wmax, d_n_windows, d_win_start, d_win_points, d_yhat_sum, d_quantity_sum,
                      d_sum_lower, d_sum_upper};
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                     horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    p.sums = &s;
    return predict_device(c, p);
}

PB200_API int pb200_predict_sums_anchored_device(pb200_ctx* c, const pb200_options* opts, const double* d_params,
                         const double* d_tchange, const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models, const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed, double* d_yhat, double* d_yhat_lower,
                         double* d_yhat_upper, int32_t* d_yhat_int, int64_t width_ns, const int64_t* d_origin_ns,
                         const int32_t* d_frame_len, int32_t wmax, int32_t* d_n_windows, int64_t* d_win_start,
                         int32_t* d_win_points, double* d_yhat_sum, int64_t* d_quantity_sum, double* d_sum_lower,
                         double* d_sum_upper) {
    if (n_models > 0 && (!d_origin_ns || !d_frame_len)) return fail(PB200_E_ARG, "null pointer (origins / frame lengths)");
    SumOut s = {width_ns, 0, wmax, d_n_windows, d_win_start, d_win_points, d_yhat_sum, d_quantity_sum, d_sum_lower,
                d_sum_upper};
    s.origins = d_origin_ns;
    s.frame_len = d_frame_len;
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                     horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    p.sums = &s;
    return predict_device(c, p);
}

PB200_API int pb200_predict_sums_host(pb200_ctx* c, const pb200_options* opts, const double* h_params, const double* h_tchange,
                       const int32_t* h_meta_i32, const int64_t* h_meta_i64, const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon, const double* h_floor, const double* h_cap,
                       uint64_t seed, double* h_yhat, double* h_yhat_lower, double* h_yhat_upper, int32_t* h_yhat_int,
                       int64_t width_ns, int64_t origin_ns, int32_t wmax, int32_t* h_n_windows, int64_t* h_win_start,
                       int32_t* h_win_points, double* h_yhat_sum, int64_t* h_quantity_sum, double* h_sum_lower,
                       double* h_sum_upper) {
    const SumOut s = {width_ns, origin_ns, wmax, h_n_windows, h_win_start, h_win_points, h_yhat_sum, h_quantity_sum,
                      h_sum_lower, h_sum_upper};
    PredictCall p = {opts, h_params, h_tchange, h_meta_i32, h_meta_i64, h_meta_f64, n_models, h_future_ds,
                     horizon, h_floor, h_cap, seed, h_yhat, h_yhat_lower, h_yhat_upper, h_yhat_int};
    p.sums = &s;
    return predict_host(c, p);
}

PB200_API int pb200_predict_period_sums_device(pb200_ctx* c, const pb200_options* opts, const double* d_params,
                         const double* d_tchange, const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models, const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed, double* d_yhat, double* d_yhat_lower,
                         double* d_yhat_upper, int32_t* d_yhat_int, int32_t months, int32_t month_shift, int32_t wmax,
                         int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points, double* d_yhat_sum,
                         int64_t* d_quantity_sum, double* d_sum_lower, double* d_sum_upper) {
    SumOut s = {0, 0, wmax, d_n_windows, d_win_start, d_win_points, d_yhat_sum, d_quantity_sum, d_sum_lower, d_sum_upper};
    s.months = months;
    s.month_shift = month_shift;
    if (months == 0) return fail(PB200_E_ARG, "months must be 1, 3 or 12 and month_shift in [0, months)");
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                     horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    p.sums = &s;
    return predict_device(c, p);
}

PB200_API int pb200_predict_period_sums_host(pb200_ctx* c, const pb200_options* opts, const double* h_params,
                       const double* h_tchange, const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models, const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed, double* h_yhat, double* h_yhat_lower,
                       double* h_yhat_upper, int32_t* h_yhat_int, int32_t months, int32_t month_shift, int32_t wmax,
                       int32_t* h_n_windows, int64_t* h_win_start, int32_t* h_win_points, double* h_yhat_sum,
                       int64_t* h_quantity_sum, double* h_sum_lower, double* h_sum_upper) {
    SumOut s = {0, 0, wmax, h_n_windows, h_win_start, h_win_points, h_yhat_sum, h_quantity_sum, h_sum_lower, h_sum_upper};
    s.months = months;
    s.month_shift = month_shift;
    if (months == 0) return fail(PB200_E_ARG, "months must be 1, 3 or 12 and month_shift in [0, months)");
    PredictCall p = {opts, h_params, h_tchange, h_meta_i32, h_meta_i64, h_meta_f64, n_models, h_future_ds,
                     horizon, h_floor, h_cap, seed, h_yhat, h_yhat_lower, h_yhat_upper, h_yhat_int};
    p.sums = &s;
    return predict_host(c, p);
}

PB200_API int pb200_period_host(const int64_t* ds, int64_t n, int32_t months, int32_t month_shift, int64_t* period,
                                int64_t* start) {
    if (!(months == 1 || months == 3 || months == 12) || month_shift < 0 || month_shift >= months)
        return fail(PB200_E_ARG, "months must be 1, 3 or 12 and month_shift in [0, months)");
    if (n < 0) return fail(PB200_E_ARG, "sizes");
    if (n > 0 && (!ds || !period || !start)) return fail(PB200_E_ARG, "null pointer");
    for (int64_t i = 0; i < n; ++i) {
        period[i] = pb200::period_of(ds[i], months, month_shift);
        start[i] = pb200::period_start(period[i], months, month_shift);
    }
    return PB200_OK;
}

PB200_API int pb200_predict_quantiles_device(pb200_ctx* c, const pb200_options* opts, const double* d_params,
                         const double* d_tchange, const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models, const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed, double* d_yhat, double* d_yhat_lower,
                         double* d_yhat_upper, int32_t* d_yhat_int, int32_t n_q, const double* h_percentiles,
                         double* d_quantiles) {
    const QuantOut q = {n_q, h_percentiles, d_quantiles};
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                     horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    p.quant = &q;
    return predict_device(c, p);
}

PB200_API int pb200_predict_quantiles_host(pb200_ctx* c, const pb200_options* opts, const double* h_params,
                       const double* h_tchange, const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models, const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed, double* h_yhat, double* h_yhat_lower,
                       double* h_yhat_upper, int32_t* h_yhat_int, int32_t n_q, const double* h_percentiles,
                       double* h_quantiles) {
    const QuantOut q = {n_q, h_percentiles, h_quantiles};
    PredictCall p = {opts, h_params, h_tchange, h_meta_i32, h_meta_i64, h_meta_f64, n_models, h_future_ds,
                     horizon, h_floor, h_cap, seed, h_yhat, h_yhat_lower, h_yhat_upper, h_yhat_int};
    p.quant = &q;
    return predict_host(c, p);
}

// ---- quantiles of the window totals (DESIGN §21): the sums entry points plus n_q levels and their planes ----
PB200_API int pb200_predict_sums_quantiles_device(pb200_ctx* c, const pb200_options* opts, const double* d_params,
                         const double* d_tchange, const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                         const double* d_meta_f64, int64_t n_models, const int64_t* d_future_ds, int32_t horizon,
                         const double* d_floor, const double* d_cap, uint64_t seed, double* d_yhat, double* d_yhat_lower,
                         double* d_yhat_upper, int32_t* d_yhat_int, int64_t width_ns, int64_t origin_ns, int32_t wmax,
                         int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points, double* d_yhat_sum,
                         int64_t* d_quantity_sum, double* d_sum_lower, double* d_sum_upper, int32_t n_q,
                         const double* h_percentiles, double* d_sum_quantiles) {
    const QuantOut q = {n_q, h_percentiles, d_sum_quantiles};
    SumOut s = {width_ns, origin_ns, wmax, d_n_windows, d_win_start, d_win_points, d_yhat_sum, d_quantity_sum,
                d_sum_lower, d_sum_upper};
    s.quant = &q;
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                     horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    p.sums = &s;
    return predict_device(c, p);
}

PB200_API int pb200_predict_sums_quantiles_host(pb200_ctx* c, const pb200_options* opts, const double* h_params,
                       const double* h_tchange, const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                       const double* h_meta_f64, int64_t n_models, const int64_t* h_future_ds, int32_t horizon,
                       const double* h_floor, const double* h_cap, uint64_t seed, double* h_yhat, double* h_yhat_lower,
                       double* h_yhat_upper, int32_t* h_yhat_int, int64_t width_ns, int64_t origin_ns, int32_t wmax,
                       int32_t* h_n_windows, int64_t* h_win_start, int32_t* h_win_points, double* h_yhat_sum,
                       int64_t* h_quantity_sum, double* h_sum_lower, double* h_sum_upper, int32_t n_q,
                       const double* h_percentiles, double* h_sum_quantiles) {
    const QuantOut q = {n_q, h_percentiles, h_sum_quantiles};
    SumOut s = {width_ns, origin_ns, wmax, h_n_windows, h_win_start, h_win_points, h_yhat_sum, h_quantity_sum,
                h_sum_lower, h_sum_upper};
    s.quant = &q;
    PredictCall p = {opts, h_params, h_tchange, h_meta_i32, h_meta_i64, h_meta_f64, n_models, h_future_ds,
                     horizon, h_floor, h_cap, seed, h_yhat, h_yhat_lower, h_yhat_upper, h_yhat_int};
    p.sums = &s;
    return predict_host(c, p);
}

PB200_API int pb200_predict_sums_anchored_quantiles_device(pb200_ctx* c, const pb200_options* opts,
                         const double* d_params, const double* d_tchange, const int32_t* d_meta_i32,
                         const int64_t* d_meta_i64, const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon, const double* d_floor, const double* d_cap,
                         uint64_t seed, double* d_yhat, double* d_yhat_lower, double* d_yhat_upper, int32_t* d_yhat_int,
                         int64_t width_ns, const int64_t* d_origin_ns, const int32_t* d_frame_len, int32_t wmax,
                         int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points, double* d_yhat_sum,
                         int64_t* d_quantity_sum, double* d_sum_lower, double* d_sum_upper, int32_t n_q,
                         const double* h_percentiles, double* d_sum_quantiles) {
    if (n_models > 0 && (!d_origin_ns || !d_frame_len)) return fail(PB200_E_ARG, "null pointer (origins / frame lengths)");
    const QuantOut q = {n_q, h_percentiles, d_sum_quantiles};
    SumOut s = {width_ns, 0, wmax, d_n_windows, d_win_start, d_win_points, d_yhat_sum, d_quantity_sum, d_sum_lower,
                d_sum_upper};
    s.origins = d_origin_ns;
    s.frame_len = d_frame_len;
    s.quant = &q;
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                     horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    p.sums = &s;
    return predict_device(c, p);
}

PB200_API int pb200_predict_period_sums_quantiles_device(pb200_ctx* c, const pb200_options* opts,
                         const double* d_params, const double* d_tchange, const int32_t* d_meta_i32,
                         const int64_t* d_meta_i64, const double* d_meta_f64, int64_t n_models,
                         const int64_t* d_future_ds, int32_t horizon, const double* d_floor, const double* d_cap,
                         uint64_t seed, double* d_yhat, double* d_yhat_lower, double* d_yhat_upper, int32_t* d_yhat_int,
                         int32_t months, int32_t month_shift, int32_t wmax, int32_t* d_n_windows, int64_t* d_win_start,
                         int32_t* d_win_points, double* d_yhat_sum, int64_t* d_quantity_sum, double* d_sum_lower,
                         double* d_sum_upper, int32_t n_q, const double* h_percentiles, double* d_sum_quantiles) {
    if (months == 0) return fail(PB200_E_ARG, "months must be 1, 3 or 12 and month_shift in [0, months)");
    const QuantOut q = {n_q, h_percentiles, d_sum_quantiles};
    SumOut s = {0, 0, wmax, d_n_windows, d_win_start, d_win_points, d_yhat_sum, d_quantity_sum, d_sum_lower, d_sum_upper};
    s.months = months;
    s.month_shift = month_shift;
    s.quant = &q;
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_future_ds,
                     horizon, d_floor, d_cap, seed, d_yhat, d_yhat_lower, d_yhat_upper, d_yhat_int};
    p.sums = &s;
    return predict_device(c, p);
}

PB200_API int pb200_predict_period_sums_quantiles_host(pb200_ctx* c, const pb200_options* opts,
                       const double* h_params, const double* h_tchange, const int32_t* h_meta_i32,
                       const int64_t* h_meta_i64, const double* h_meta_f64, int64_t n_models,
                       const int64_t* h_future_ds, int32_t horizon, const double* h_floor, const double* h_cap,
                       uint64_t seed, double* h_yhat, double* h_yhat_lower, double* h_yhat_upper, int32_t* h_yhat_int,
                       int32_t months, int32_t month_shift, int32_t wmax, int32_t* h_n_windows, int64_t* h_win_start,
                       int32_t* h_win_points, double* h_yhat_sum, int64_t* h_quantity_sum, double* h_sum_lower,
                       double* h_sum_upper, int32_t n_q, const double* h_percentiles, double* h_sum_quantiles) {
    if (months == 0) return fail(PB200_E_ARG, "months must be 1, 3 or 12 and month_shift in [0, months)");
    const QuantOut q = {n_q, h_percentiles, h_sum_quantiles};
    SumOut s = {0, 0, wmax, h_n_windows, h_win_start, h_win_points, h_yhat_sum, h_quantity_sum, h_sum_lower, h_sum_upper};
    s.months = months;
    s.month_shift = month_shift;
    s.quant = &q;
    PredictCall p = {opts, h_params, h_tchange, h_meta_i32, h_meta_i64, h_meta_f64, n_models, h_future_ds,
                     horizon, h_floor, h_cap, seed, h_yhat, h_yhat_lower, h_yhat_upper, h_yhat_int};
    p.sums = &s;
    return predict_host(c, p);
}

// ---- forecast CSV rows formatted on the device (csv_kernel.cuh) ----
static int csv_args(pb200::csv::CsvArgs& a, const int32_t* sid, const int32_t* did, const int64_t* ds, const int32_t* qty, int64_t n,
                    const char* created, int32_t created_len) {
    if (created_len < 0 || created_len > pb200::csv::MAX_CREATED) return fail(PB200_E_ARG, "created_timestamp longer than 64 bytes");
    if (created_len && !created) return fail(PB200_E_ARG, "null pointer");
    a.sid = sid; a.did = did; a.ds_ns = (const long long*)ds; a.qty = qty; a.n = n; a.created_len = created_len;
    memset(a.created, 0, sizeof(a.created));
    if (created_len) memcpy(a.created, created, (size_t)created_len);
    a.row_len = nullptr; a.row_off = nullptr; a.out = nullptr;
    return PB200_OK;
}

PB200_API int pb200_forecast_csv_lengths_device(pb200_ctx* c, const int32_t* d_series_id, const int32_t* d_dim_id,
                                                const int32_t* d_quantity, int64_t n_rows, int32_t created_len,
                                                int64_t* d_row_len) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n_rows < 0) return fail(PB200_E_ARG, "sizes");
    if (n_rows == 0) return PB200_OK;
    if (!d_series_id || !d_dim_id || !d_quantity || !d_row_len) return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    pb200::csv::CsvArgs a;
    char pad[pb200::csv::MAX_CREATED] = {0};
    int rc = csv_args(a, d_series_id, d_dim_id, nullptr, d_quantity, n_rows, pad, created_len);
    if (rc) return rc;
    a.row_len = (long long*)d_row_len;
    const int grid = (int)std::min<int64_t>((n_rows + 255) / 256, (int64_t)c->sms * 16);
    pb200::csv::csv_lengths_kernel<<<grid, 256, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

PB200_API int pb200_forecast_csv_rows_device(pb200_ctx* c, const int32_t* d_series_id, const int32_t* d_dim_id,
                                             const int64_t* d_ds_ns, const int32_t* d_quantity, int64_t n_rows,
                                             const char* h_created, int32_t created_len, const int64_t* d_row_off,
                                             uint8_t* d_out) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n_rows < 0) return fail(PB200_E_ARG, "sizes");
    if (n_rows == 0) return PB200_OK;
    if (!d_series_id || !d_dim_id || !d_ds_ns || !d_quantity || !d_row_off || !d_out) return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    pb200::csv::CsvArgs a;
    int rc = csv_args(a, d_series_id, d_dim_id, d_ds_ns, d_quantity, n_rows, h_created, created_len);
    if (rc) return rc;
    a.row_off = (const long long*)d_row_off;
    a.out = d_out;
    const int64_t warps = (n_rows + 31) / 32;
    const int grid = (int)std::min<int64_t>((warps + 3) / 4, (int64_t)c->sms * 8);
    pb200::csv::csv_rows_kernel<<<grid, 128, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

PB200_API int32_t pb200_forecast_csv_row_host(int32_t series_id, int32_t dim_id, int64_t ds_ns, int32_t quantity,
                                              const char* created, int32_t created_len, char* out) {
    if (created_len < 0 || created_len > pb200::csv::MAX_CREATED || !out || (created_len && !created)) return -1;
    char* e = pb200::csv::put_row(out, series_id, dim_id, ds_ns, quantity, created, created_len);
    const int n = (int)(e - out);
    return n == pb200::csv::row_len(series_id, dim_id, quantity, created_len) ? n : -1;
}

// ---- backtest: cutoff plan, truncated-history gather, performance metrics (cv_kernel.cuh) ----
static int cv_plan_args(pb200::cv::PlanArgs& a, const pb200_options* opts, const int64_t* d_ds, const int64_t* d_offsets,
                        int64_t n_series, int64_t horizon_ns, int64_t period_ns, int64_t initial_ns) {
    int rc = check_opts(opts);
    if (rc) return rc;
    if (n_series < 0) return fail(PB200_E_ARG, "n_series");
    if (horizon_ns <= 0 || period_ns <= 0 || initial_ns <= 0) return fail(PB200_E_ARG, "horizon, period and initial must be > 0");
    if (n_series && (!d_ds || !d_offsets)) return fail(PB200_E_ARG, "null pointer");
    memset(&a, 0, sizeof a);
    a.ds = (const long long*)d_ds;
    a.offsets = (const long long*)d_offsets;
    a.n_series = n_series;
    a.horizon = horizon_ns;
    a.period = period_ns;
    a.initial = initial_ns;
    a.yearly = opts->yearly;
    a.weekly = opts->weekly;
    a.daily = opts->daily;
    return PB200_OK;
}

static int cv_plan_launch(pb200_ctx* c, const pb200::cv::PlanArgs& a) {
    const int64_t warps = a.n_series;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((warps + 7) / 8, (int64_t)c->sms * 16));
    pb200::cv::cv_plan_kernel<<<grid, 256, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

PB200_API int pb200_cv_plan_counts_device(pb200_ctx* c, const pb200_options* opts, const int64_t* d_ds, const int64_t* d_offsets,
                                          int64_t n_series, int64_t horizon_ns, int64_t period_ns, int64_t initial_ns,
                                          int32_t* d_n_cutoffs, int32_t* d_mask, int32_t* d_err) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    pb200::cv::PlanArgs a;
    int rc = cv_plan_args(a, opts, d_ds, d_offsets, n_series, horizon_ns, period_ns, initial_ns);
    if (rc) return rc;
    if (n_series == 0) return PB200_OK;
    if (!d_n_cutoffs || !d_mask || !d_err) return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    a.n_cut = d_n_cutoffs;
    a.mask = d_mask;
    a.err = d_err;
    return cv_plan_launch(c, a);
}

PB200_API int pb200_cv_plan_device(pb200_ctx* c, const pb200_options* opts, const int64_t* d_ds, const int64_t* d_offsets,
                                   int64_t n_series, int64_t horizon_ns, int64_t period_ns, int64_t initial_ns,
                                   const int64_t* d_pair_off, int32_t* d_err, int32_t* d_pair_series, int64_t* d_cutoff,
                                   int64_t* d_hist_end, int64_t* d_win_end) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    pb200::cv::PlanArgs a;
    int rc = cv_plan_args(a, opts, d_ds, d_offsets, n_series, horizon_ns, period_ns, initial_ns);
    if (rc) return rc;
    if (n_series == 0) return PB200_OK;
    if (!d_pair_off || !d_err || !d_pair_series || !d_cutoff || !d_hist_end || !d_win_end) return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    a.pair_off = (const long long*)d_pair_off;
    a.err = d_err;
    a.pair_series = d_pair_series;
    a.cutoff = (long long*)d_cutoff;
    a.hist_end = (long long*)d_hist_end;
    a.win_end = (long long*)d_win_end;
    return cv_plan_launch(c, a);
}

PB200_API int pb200_cv_gather_device(pb200_ctx* c, const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                                     const int64_t* d_offsets, const int32_t* d_pair_series, const int64_t* d_hist_end,
                                     const int64_t* d_win_end, const int64_t* d_pairs, int64_t n, const int64_t* d_fit_off,
                                     int32_t hmax, int64_t* d_ds_out, void* d_y_out, int64_t* d_future_ds) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n < 0 || hmax < 1) return fail(PB200_E_ARG, "sizes");
    if (y_dtype < 0 || y_dtype > 2) return fail(PB200_E_ARG, "y_dtype");
    if (n == 0) return PB200_OK;
    if (!d_ds || !d_y || !d_offsets || !d_pair_series || !d_hist_end || !d_win_end || !d_pairs || !d_fit_off || !d_ds_out ||
        !d_y_out || !d_future_ds)
        return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    pb200::cv::GatherArgs a;
    a.ds = (const long long*)d_ds;
    a.y = d_y;
    a.y_dtype = y_dtype;
    a.offsets = (const long long*)d_offsets;
    a.pair_series = d_pair_series;
    a.hist_end = (const long long*)d_hist_end;
    a.win_end = (const long long*)d_win_end;
    a.pairs = (const long long*)d_pairs;
    a.n = n;
    a.fit_off = (const long long*)d_fit_off;
    a.hmax = hmax;
    a.ds_out = (long long*)d_ds_out;
    a.y_out = d_y_out;
    a.fut = (long long*)d_future_ds;
    const int grid = (int)std::min<int64_t>(n, (int64_t)c->sms * 32);
    pb200::cv::cv_gather_kernel<<<grid, 256, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

PB200_API int pb200_cv_metrics_device(pb200_ctx* c, const int64_t* d_horizon, const double* d_y, const double* d_yhat,
                                      const double* d_yhat_lower, const double* d_yhat_upper, const int64_t* d_order,
                                      const int64_t* d_srow_off, int64_t n_series, double rolling_window, int64_t* d_out_horizon,
                                      int64_t* d_scratch, double* d_mse, double* d_rmse, double* d_mae, double* d_mape,
                                      double* d_coverage, int32_t* d_valid) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n_series < 0) return fail(PB200_E_ARG, "n_series");
    if (!(rolling_window >= 0.0 && rolling_window <= 1.0)) return fail(PB200_E_ARG, "rolling_window must be in [0, 1]");
    if (!d_yhat_lower != !d_yhat_upper) return fail(PB200_E_ARG, "yhat_lower and yhat_upper go together");
    if (n_series == 0) return PB200_OK;
    if (!d_horizon || !d_y || !d_yhat || !d_order || !d_srow_off || !d_out_horizon || !d_scratch || !d_mse || !d_rmse ||
        !d_mae || !d_mape || !d_coverage || !d_valid)
        return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    pb200::cv::MetricsArgs a;
    a.horizon = (const long long*)d_horizon;
    a.y = d_y;
    a.yhat = d_yhat;
    a.lo = d_yhat_lower;
    a.hi = d_yhat_upper;
    a.order = (const long long*)d_order;
    a.srow_off = (const long long*)d_srow_off;
    a.n_series = n_series;
    a.rolling_window = rolling_window;
    a.out_h = (long long*)d_out_horizon;
    a.out_n = (long long*)d_scratch;
    a.out_mse = d_mse;
    a.out_rmse = d_rmse;
    a.out_mae = d_mae;
    a.out_mape = d_mape;
    a.out_cov = d_coverage;
    a.out_valid = d_valid;
    const int grid = (int)std::min<int64_t>((n_series + 127) / 128, (int64_t)c->sms * 16);
    pb200::cv::cv_metrics_kernel<<<grid, 128, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

PB200_API int pb200_cv_quantile_metrics_device(pb200_ctx* c, const int64_t* d_horizon, const double* d_y,
                                               const double* d_yq, int64_t n_rows, int32_t n_q, const double* h_levels,
                                               const int64_t* d_order, const int64_t* d_srow_off, int64_t n_series,
                                               double rolling_window, int64_t* d_out_horizon, int64_t* d_scratch,
                                               double* d_pinball, double* d_share_below, int32_t* d_valid) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n_series < 0 || n_rows < 0) return fail(PB200_E_ARG, "sizes");
    if (!(rolling_window >= 0.0 && rolling_window <= 1.0)) return fail(PB200_E_ARG, "rolling_window must be in [0, 1]");
    if (n_q < 1 || n_q > pb200::cv::CV_QMAX) return fail(PB200_E_ARG, "n_q must be in [1, 32]");
    if (!h_levels) return fail(PB200_E_ARG, "null pointer (levels)");
    pb200::cv::QuantMetricsArgs a;
    for (int q = 0; q < n_q; ++q) {
        if (!(h_levels[q] >= 0.0 && h_levels[q] <= 1.0)) return fail(PB200_E_ARG, "levels must be in [0, 1]");
        a.level[q] = h_levels[q];
    }
    if (n_series == 0) return PB200_OK;
    if (!d_horizon || !d_y || !d_yq || !d_order || !d_srow_off || !d_out_horizon || !d_scratch || !d_pinball ||
        !d_share_below || !d_valid)
        return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    a.horizon = (const long long*)d_horizon;
    a.y = d_y;
    a.yq = d_yq;
    a.n_rows = n_rows;
    a.nq = n_q;
    a.order = (const long long*)d_order;
    a.srow_off = (const long long*)d_srow_off;
    a.n_series = n_series;
    a.rolling_window = rolling_window;
    a.out_h = (long long*)d_out_horizon;
    a.out_n = (long long*)d_scratch;
    a.out_pinball = d_pinball;
    a.out_below = d_share_below;
    a.out_valid = d_valid;
    const int grid = (int)std::min<int64_t>((n_series + 127) / 128, (int64_t)c->sms * 16);
    pb200::cv::cv_quantile_metrics_kernel<<<grid, 128, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

PB200_API int pb200_cv_windows_device(pb200_ctx* c, const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                                      const int64_t* d_cutoff, const int64_t* d_hist_end, const int64_t* d_win_end,
                                      const int64_t* d_pairs, int64_t n, const double* d_yhat, int32_t hmax, int64_t width_ns,
                                      int32_t wmax, int32_t* d_n_windows, int64_t* d_win_start, int32_t* d_win_points,
                                      double* d_y_sum, double* d_yhat_sum) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n < 0 || hmax < 1 || wmax < 1) return fail(PB200_E_ARG, "sizes");
    if (width_ns <= 0) return fail(PB200_E_ARG, "width_ns must be > 0");
    if (y_dtype < 0 || y_dtype > 2) return fail(PB200_E_ARG, "y_dtype");
    if (n == 0) return PB200_OK;
    if (!d_ds || !d_y || !d_cutoff || !d_hist_end || !d_win_end || !d_pairs || !d_yhat || !d_n_windows || !d_win_start ||
        !d_win_points || !d_y_sum || !d_yhat_sum)
        return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    pb200::cv::WindowArgs a;
    a.ds = (const long long*)d_ds;
    a.y = d_y;
    a.y_dtype = y_dtype;
    a.cutoff = (const long long*)d_cutoff;
    a.hist_end = (const long long*)d_hist_end;
    a.win_end = (const long long*)d_win_end;
    a.pairs = (const long long*)d_pairs;
    a.n = n;
    a.yhat = d_yhat;
    a.hmax = hmax;
    a.width = width_ns;
    a.wmax = wmax;
    a.n_windows = d_n_windows;
    a.win_start = (long long*)d_win_start;
    a.points = d_win_points;
    a.y_sum = d_y_sum;
    a.yhat_sum = d_yhat_sum;
    const int grid = (int)std::min<int64_t>((n + 7) / 8, (int64_t)c->sms * 4);   // 8 warps per CTA, one per entry
    pb200::cv::cv_window_kernel<<<grid, 256, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

}  // extern "C"

// ---- in-sample predict over ragged frames, outlier flags and the kept rows (DESIGN §16) ----
namespace {

// pb200_predict_history_device: pb200_predict_device's checks, then the ragged instances of predict_kernel and mc_kernel
// over model i's rows [p.offsets[i], p.offsets[i + 1]) of p.future_ds (the history's ds; p.horizon is 0); the offsets
// are copied to the device here
int predict_history_device(pb200_ctx* c, const PredictCall& p) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    int rc = check_opts(p.opts);
    if (rc) return rc;
    const int64_t n_models = p.n_models;
    if (n_models < 0 || n_models > (1LL << 30)) return fail(PB200_E_ARG, "sizes");
    if (n_models == 0) return PB200_OK;
    if (!p.offsets) return fail(PB200_E_ARG, "null pointer (offsets)");
    if (p.offsets[0] < 0) return fail(PB200_E_ARG, "offsets[0] < 0");
    int64_t tmax = 0;
    for (int64_t i = 0; i < n_models; ++i) {
        const int64_t T = p.offsets[i + 1] - p.offsets[i];
        if (T < 0) return fail(PB200_E_ARG, "offsets not monotone");
        if (T > INT32_MAX) return fail(PB200_E_UNSUPPORTED, "a frame longer than 2^31 - 1 rows");
        tmax = std::max(tmax, T);
    }
    if (tmax == 0) return PB200_OK;
    if (!p.params || !p.tchange || !p.meta_i32 || !p.meta_i64 || !p.meta_f64 || !p.floor || !p.cap || !p.future_ds || !p.yhat)
        return fail(PB200_E_ARG, "null pointer");
    const bool mc = p.yhat_lower && p.yhat_upper && p.opts->uncertainty_samples > 0;
    if (mc && (rc = check_mc_opts(p.opts))) return rc;
    CK(cudaSetDevice(c->device));
    const size_t N = (size_t)n_models;
    CK(c->d_hoff.reserve((N + 1) * 8));
    CK(cudaMemcpyAsync(c->d_hoff.p, p.offsets, (N + 1) * 8, cudaMemcpyHostToDevice, c->stream));
    pb200::RaggedPredictArgs a;
    predict_args(a, p);
    a.offsets = (const long long*)c->d_hoff.p;
    // the fixed frame's geometry over the longest frame: CTAs past a shorter model's rows leave at once
    dim3 grid((unsigned)n_models, (unsigned)std::min<int64_t>((tmax + 1023) / 1024, 64));
    pb200::predict_kernel<false, true><<<grid, 256, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    if (mc) {
        rc = pb200::launch_mc_ragged(c->stream, c->sms, a, a.offsets, p.opts->uncertainty_samples, p.opts->interval_width,
                                     p.seed, p.yhat_lower, p.yhat_upper);
        if (rc == -1) return fail(PB200_E_ARG, "uncertainty_samples / interval_width out of range");
        if (rc) return fail(PB200_E_CUDA, "mc kernel launch", cudaGetLastError());
        c->launches++;
    }
    return PB200_OK;
}

}  // namespace

extern "C" {

PB200_API int pb200_predict_history_device(pb200_ctx* c, const pb200_options* opts, const double* d_params,
                                           const double* d_tchange, const int32_t* d_meta_i32, const int64_t* d_meta_i64,
                                           const double* d_meta_f64, int64_t n_models, const int64_t* d_ds,
                                           const int64_t* h_offsets, const double* d_floor, const double* d_cap,
                                           uint64_t seed, double* d_yhat, double* d_yhat_lower, double* d_yhat_upper) {
    PredictCall p = {opts, d_params, d_tchange, d_meta_i32, d_meta_i64, d_meta_f64, n_models, d_ds, 0, d_floor, d_cap,
                     seed, d_yhat, d_yhat_lower, d_yhat_upper};
    p.offsets = h_offsets;
    return predict_history_device(c, p);
}

PB200_API int pb200_predict_history_host(pb200_ctx* c, const pb200_options* opts, const double* h_params,
                                         const double* h_tchange, const int32_t* h_meta_i32, const int64_t* h_meta_i64,
                                         const double* h_meta_f64, int64_t n_models, const int64_t* h_ds,
                                         const int64_t* h_offsets, const double* h_floor, const double* h_cap,
                                         uint64_t seed, double* h_yhat, double* h_yhat_lower, double* h_yhat_upper) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    int rc = check_opts(opts);
    if (rc) return rc;
    if (n_models < 0 || n_models > (1LL << 30)) return fail(PB200_E_ARG, "sizes");
    if (n_models == 0) return PB200_OK;
    if (!h_offsets) return fail(PB200_E_ARG, "null pointer (offsets)");
    const int64_t rows = h_offsets[n_models];
    if (rows < 0) return fail(PB200_E_ARG, "offsets");
    if (!h_params || !h_tchange || !h_meta_i32 || !h_meta_i64 || !h_meta_f64 || !h_floor || !h_cap ||
        (rows > 0 && (!h_ds || !h_yhat)))
        return fail(PB200_E_ARG, "null pointer");
    const bool mc = h_yhat_lower && h_yhat_upper && opts->uncertainty_samples > 0;
    if (mc && (rc = check_mc_opts(opts))) return rc;
    pb200_layout L;
    pb200_get_layout(opts, &L);
    const size_t N = (size_t)n_models, R = (size_t)rows;
    Staging s(c);
    PredictCall d = {opts};
    d.params = s.in(ST_PARAMS, h_params, N * L.pstride);
    d.tchange = s.in(ST_TCHANGE, h_tchange, N * L.smax);
    d.meta_i32 = s.in(ST_MI32, h_meta_i32, N * 8);
    d.meta_i64 = s.in(ST_MI64, h_meta_i64, N * 2);
    d.meta_f64 = s.in(ST_MF64, h_meta_f64, N * 4);
    d.n_models = n_models;
    d.future_ds = s.in(ST_FUT, h_ds, R);
    d.offsets = h_offsets;
    d.floor = s.in(ST_FLOOR, h_floor, N);
    d.cap = s.in(ST_CAP, h_cap, N);
    d.seed = seed;
    d.yhat = s.out(ST_YHAT, h_yhat, R);
    d.yhat_lower = s.out(ST_LO, mc ? h_yhat_lower : nullptr, R);
    d.yhat_upper = s.out(ST_HI, mc ? h_yhat_upper : nullptr, R);
    if ((rc = s.status()) || (rc = predict_history_device(c, d))) return rc;
    return s.finish();
}

static int outlier_grid(const pb200_ctx* c, int64_t n_series) {   // one warp per series, 8 per CTA
    return (int)std::max<int64_t>(1, std::min<int64_t>((n_series + pb200::insample::WARPS - 1) / pb200::insample::WARPS,
                                                       (int64_t)c->sms * 16));
}

PB200_API int pb200_outlier_counts_device(pb200_ctx* c, const void* d_y, int32_t y_dtype, const int64_t* d_offsets,
                                          int64_t n_series, const double* d_lower, const double* d_upper, uint8_t* d_flag,
                                          int32_t* d_kept) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n_series < 0) return fail(PB200_E_ARG, "n_series");
    if (y_dtype < 0 || y_dtype > 2) return fail(PB200_E_ARG, "y_dtype");
    if (n_series == 0) return PB200_OK;
    if (!d_y || !d_offsets || !d_lower || !d_upper || !d_flag || !d_kept) return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    pb200::insample::FlagArgs a;
    a.y = d_y;
    a.y_dtype = y_dtype;
    a.offsets = (const long long*)d_offsets;
    a.n_series = n_series;
    a.lower = d_lower;
    a.upper = d_upper;
    a.flag = d_flag;
    a.kept = d_kept;
    pb200::insample::outlier_counts_kernel<<<outlier_grid(c, n_series), pb200::insample::THREADS, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

PB200_API int pb200_outlier_compact_device(pb200_ctx* c, const int64_t* d_ds, const void* d_y, int32_t y_dtype,
                                           const int64_t* d_offsets, int64_t n_series, const uint8_t* d_flag,
                                           const int64_t* d_kept_off, int64_t* d_ds_out, void* d_y_out) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n_series < 0) return fail(PB200_E_ARG, "n_series");
    if (y_dtype < 0 || y_dtype > 2) return fail(PB200_E_ARG, "y_dtype");
    if (n_series == 0) return PB200_OK;
    if (!d_ds || !d_y || !d_offsets || !d_flag || !d_kept_off || !d_ds_out || !d_y_out) return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    pb200::insample::CompactArgs a;
    a.ds = (const long long*)d_ds;
    a.y = d_y;
    a.y_dtype = y_dtype;
    a.offsets = (const long long*)d_offsets;
    a.n_series = n_series;
    a.flag = d_flag;
    a.kept_off = (const long long*)d_kept_off;
    a.ds_out = (long long*)d_ds_out;
    a.y_out = d_y_out;
    pb200::insample::outlier_compact_kernel<<<outlier_grid(c, n_series), pb200::insample::THREADS, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

PB200_API int pb200_join_future_regressors_device(pb200_ctx* c, const int64_t* d_tab_ds, const int64_t* d_tab_offsets,
                                                  const double* d_tab_reg, int64_t n_rows, int32_t n_regressors,
                                                  const int64_t* d_model_group, const int64_t* d_future_ds,
                                                  int64_t n_models, int32_t horizon, double* d_future_reg,
                                                  int32_t* d_missing, int64_t* d_first_missing) {
    if (!c) return fail(PB200_E_ARG, "ctx is null");
    if (n_rows < 0 || n_models < 0 || horizon < 0) return fail(PB200_E_ARG, "sizes");
    if (n_regressors < 1 || n_regressors > PB200_MAX_REGRESSORS) return fail(PB200_E_ARG, "n_regressors");
    if (n_models == 0) return PB200_OK;
    if (!d_tab_offsets || !d_model_group || !d_missing || !d_first_missing || (n_rows > 0 && (!d_tab_ds || !d_tab_reg)) ||
        (horizon > 0 && (!d_future_ds || !d_future_reg)))
        return fail(PB200_E_ARG, "null pointer");
    CK(cudaSetDevice(c->device));
    pb200::join::JoinArgs a;
    a.tab_ds = (const long long*)d_tab_ds;
    a.tab_offsets = (const long long*)d_tab_offsets;
    a.tab_reg = d_tab_reg;
    a.rows = n_rows;
    a.R = n_regressors;
    a.model_group = (const long long*)d_model_group;
    a.future_ds = (const long long*)d_future_ds;
    a.n_models = n_models;
    a.horizon = horizon;
    a.future_reg = d_future_reg;
    a.missing = d_missing;
    a.first_missing = (long long*)d_first_missing;
    const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((n_models + pb200::join::WARPS - 1) / pb200::join::WARPS,
                                                                 (int64_t)c->sms * 16));
    pb200::join::join_future_regressors_kernel<<<grid, pb200::join::THREADS, 0, c->stream>>>(a);
    CK(cudaGetLastError());
    c->launches++;
    return PB200_OK;
}

}  // extern "C"
