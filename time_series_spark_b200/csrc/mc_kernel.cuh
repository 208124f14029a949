// Monte-Carlo predictive intervals (yhat_lower / yhat_upper) for sm_90a.
// Restates fbprophet 0.5 Prophet.predict_uncertainty -> sample_posterior_predictive ->
// sample_model -> sample_predictive_trend (reached from reference
// src/jobs/prophet_scorer.py:70 and discarded at :86): per draw, new changepoints from a
// Poisson process with rate S on (1, Tmax], slope changes ~ Laplace(0, mean|delta| + 1e-8),
// piecewise trend, observation noise N(0, sigma_obs) * y_scale, then the
// 100(1-w)/2 and 100(1+w)/2 percentiles (numpy linear interpolation) over the draws.
//
// fbprophet draws n ~ Poisson(S (Tmax-1)) then n sorted uniforms; this kernel generates the
// SAME process by exponential inter-arrival gaps (rate S), which needs O(1) state per draw
// and no sort of changepoints.  The reference uses the unseeded global numpy RNG, so only
// the distribution -- not the stream -- can be matched; here the stream is counter-based
// Philox4x32-10, keyed by the seed and a hash of the model's own record (model_key) and counted by draw:
// a model's intervals are a function of the model and the seed, whatever else is in the batch and on
// whichever shard it runs.  oracle/mc_stream.py restates the stream and the sampler in numpy.
//
// One CTA per model; thread j owns draws j and j + 512; the draws of a tile of 16 future
// points are staged in shared memory ([16][1024] fp64) and each warp sorts one row's order
// statistics (256-bin histogram + exact selection inside the bin; bitonic sort as fallback).  Requires future timestamps ascending
// within a model (make_future_dataframe's output is).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include <algorithm>

#include "calendar.cuh"
#include "predict_kernel.cuh"

namespace pb200 {

constexpr int MC_TILE = 16;
constexpr int MC_THREADS = 512;
constexpr int MC_NP = 1024;   // padded draws per point

struct Philox {
    uint32_t k0, k1;
    __device__ __forceinline__ void gen(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t* out) const {
        uint32_t a0 = k0, a1 = k1;
#pragma unroll
        for (int r = 0; r < 10; ++r) {
            const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
            const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
            const uint32_t n0 = hi1 ^ c1 ^ a0, n1 = lo1, n2 = hi0 ^ c3 ^ a1, n3 = lo0;
            c0 = n0; c1 = n1; c2 = n2; c3 = n3;
            a0 += 0x9E3779B9u;
            a1 += 0xBB67AE85u;
        }
        out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
    }
};

// uniform in (0, 1) with 53 random bits
__device__ __forceinline__ double u01(uint32_t a, uint32_t b) {
    const uint64_t v = ((uint64_t)a << 32 | b) >> 11;
    return ((double)v + 0.5) * (1.0 / 9007199254740992.0);
}

struct DrawState {
    double k, m;          // current rate / offset of the piecewise trend
    double next_cp;       // time of the next simulated changepoint (inf if none)
    int s_hist;           // fitted changepoints already applied
    uint32_t cp_ctr;      // counter of the changepoint stream
};

constexpr int MC_QMAX = 32;                // quantile levels per call (DESIGN §15)
constexpr int MC_QLEV = MC_QMAX + 2;       // with the two interval bounds
constexpr int MC_QRANK = 2 * MC_QLEV;      // distinct order statistics read (each level reads i and min(i + 1, n - 1))

// The percentiles a row's selection writes, as order statistics of the sorted draws s: level l is
// s[rank[ia[l]]] + (s[rank[ib[l]]] - s[rank[ia[l]]]) * frac[l].  Levels [0, nq) are the quantile planes, then (when
// requested) the lower and the upper interval bound.  mc_args fills it.
struct McLevels {
    int nlev, nq;                // nlev = nq + 2 with the bounds
    int nrank;                   // distinct order statistics, ascending
    int rank[MC_QRANK];
    unsigned char ia[MC_QLEV], ib[MC_QLEV];
    double frac[MC_QLEV];
};

struct McArgs {
    PredictArgs p;
    int n_samples;
    McLevels lv;
    uint64_t seed;
    double* lower;
    double* upper;
    double* tlower;       // trend bounds: written by mc_kernel<LOGI, true> only
    double* tupper;
    double* planes;       // [nq][n_models * horizon]: the quantile planes (mc_kernel<LOGI, false> only)
};

// mc_kernel's ragged instance (pb200_predict_history_*): model i's frame is rows [offsets[i], offsets[i + 1]) of
// p.future_ds and of lower / upper.  Derived, as RaggedPredictArgs, so that McArgs and the fixed-frame instances keep
// their layout and code.
struct RaggedMcArgs : McArgs {
    const long long* offsets;   // [n_models + 1]
};
// mc_kernel's instance with regressors (pb200_predict_regressors_*, DESIGN §19).  Derived, as RaggedMcArgs
struct RegMcArgs : McArgs {
    RegFrame reg;
};
template <bool RAGGED, bool REGR = false>
using McArgsT = std::conditional_t<RAGGED, RaggedMcArgs, std::conditional_t<REGR, RegMcArgs, McArgs>>;

__device__ __forceinline__ uint64_t splitmix64(uint64_t z) {
    z += 0x9E3779B97F4A7C15ull;
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

// Philox key of one model, a function of the seed and the model's own record only -- not of its index in the batch -- so
// that a model gets the same intervals in any batch, on any shard.  Words of the record, in order: params[0, pstride),
// tchange[0, smax), start_ns, t_scale_ns and the bits of y_scale, floor, cap.  Word i contributes
// splitmix64(w_i ^ splitmix64(i)); the contributions are XORed (lane l of warp 0 takes words l, l + 32, ...) and the key is
// splitmix64(xor ^ splitmix64(seed)): k0 its low, k1 its high 32 bits.  oracle/mc_stream.py restates it.
__device__ __forceinline__ uint64_t model_key(const McArgs& a, const int model, const int lane) {
    const PredictArgs& p = a.p;
    const int nw = p.pstride + p.smax + 5;
    uint64_t h = 0;
    for (int i = lane; i < nw; i += 32) {
        uint64_t w;
        if (i < p.pstride) {
            w = (uint64_t)__double_as_longlong(p.params[(size_t)model * p.pstride + i]);
        } else if (i < p.pstride + p.smax) {
            w = (uint64_t)__double_as_longlong(p.tchange[(size_t)model * p.smax + (i - p.pstride)]);
        } else {
            const int j = i - p.pstride - p.smax;
            if (j < 2) w = (uint64_t)p.meta_i64[(size_t)model * 2 + j];
            else if (j == 2) w = (uint64_t)__double_as_longlong(p.meta_f64[(size_t)model * 4]);
            else w = (uint64_t)__double_as_longlong(j == 3 ? p.floor[model] : p.cap[model]);
        }
        h ^= splitmix64(w ^ splitmix64((uint64_t)i));
    }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) h ^= __shfl_xor_sync(0xffffffffu, h, o);
    return splitmix64(h ^ splitmix64(a.seed));
}

template <bool LOGI>
__device__ __forceinline__ void advance(DrawState& d, const ModelSm& ms, const double t, const Philox& ph,
                                        const uint32_t draw, const double rate) {
    // fitted changepoints (identical for every draw)
    while (d.s_hist < ms.S && t >= ms.tc[d.s_hist]) {
        const double dl = ms.delta[d.s_hist];
        d.k += dl;
        d.m += ms.gamma[d.s_hist];
        ++d.s_hist;
    }
    // simulated changepoints
    while (t >= d.next_cp) {
        uint32_t r[4];
        ph.gen(draw, d.cp_ctr, 1u, 0u, r);
        ++d.cp_ctr;
        const double ul = u01(r[0], r[1]) - 0.5;
        const double dl = -ms.lam * (ul < 0 ? -1.0 : 1.0) * log(1.0 - 2.0 * fabs(ul));   // Laplace(0, lam)
        const double kn = d.k + dl;
        if (LOGI) d.m += (d.next_cp - d.m) * (1.0 - d.k / kn);
        else d.m += -d.next_cp * dl;
        d.k = kn;
        d.next_cp += -log(u01(r[2], r[3])) / rate;
    }
}

constexpr int MC_CAND = 64;    // candidates kept per histogram bin before falling back to a full sort

// The order statistics lv.rank[0, nrank) of one row of n values into sel[0, nrank).  One 256-bin histogram, then one
// candidate gather per distinct bin that holds a target rank: every target rank in that bin is selected from the one
// candidate set.  Returns 1; 2 for a constant row (sel[0] is then every level's value); 0 when such a bin holds more
// than MC_CAND values -- unless TIES and they are all equal: then every target rank in the bin is that value (exact).
// Trend draws need it: before a draw's first simulated changepoint its trend is the fitted one, so at early horizons
// most draws of a point are exactly equal.  0 also when a value compares with nothing (NaN).  On 0 the caller sorts.
// hist and tb / trb (per target: its bin, its rank inside the bin) are the warp's scratch.
template <bool TIES>
__device__ __forceinline__ int select_ranks(const double* row, const int n, const McLevels& lv, int* hist, int* tb, int* trb,
                                            double* cand, int* cnt, const int lane, double* sel) {
    double mn = INFINITY, mx = -INFINITY;
    for (int e = lane; e < n; e += 32) { const double v = row[e]; mn = fmin(mn, v); mx = fmax(mx, v); }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (!(mx > mn) || !isfinite(mx - mn)) {
        if (mx == mn) {
            if (lane == 0) sel[0] = mn;
            __syncwarp();
            return 2;
        }
        return 0;
    }
    const double scale = 256.0 / (mx - mn);
    for (int q = 0; q < 8; ++q) hist[lane * 8 + q] = 0;
    __syncwarp();
    for (int e = lane; e < n; e += 32) atomicAdd(&hist[min(255, (int)((row[e] - mn) * scale))], 1);
    __syncwarp();
    int lsum = 0;
    for (int q = 0; q < 8; ++q) lsum += hist[lane * 8 + q];
    int inc = lsum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, inc, o);
        if (lane >= o) inc += t;
    }
    // the histogram becomes the first rank of each bin; a target's bin is the last one starting at or before it
    int cum = inc - lsum;
    for (int q = 0; q < 8; ++q) { const int c = hist[lane * 8 + q]; hist[lane * 8 + q] = cum; cum += c; }
    __syncwarp();
    for (int t = lane; t < lv.nrank; t += 32) {
        const int k = lv.rank[t];
        int lo = 0, hi = 255;
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (hist[mid] <= k) lo = mid; else hi = mid - 1;
        }
        tb[t] = lo;
        trb[t] = k - hist[lo];
    }
    __syncwarp();
    for (int t0 = 0; t0 < lv.nrank;) {
        const int b = tb[t0];
        int t1 = t0 + 1;
        while (t1 < lv.nrank && tb[t1] == b) ++t1;
        if (lane == 0) *cnt = 0;
        __syncwarp();
        double bmn = INFINITY, bmx = -INFINITY;
        for (int e = lane; e < n; e += 32) {
            const double v = row[e];
            if (min(255, (int)((v - mn) * scale)) == b) {
                const int pos = atomicAdd(cnt, 1);
                if (pos < MC_CAND) cand[pos] = v;
                if (TIES) { bmn = fmin(bmn, v); bmx = fmax(bmx, v); }
            }
        }
        __syncwarp();
        const int m = *cnt;
        if (m > MC_CAND) {
            if (!TIES) return 0;
#pragma unroll
            for (int o = 16; o >= 1; o >>= 1) {
                bmn = fmin(bmn, __shfl_xor_sync(0xffffffffu, bmn, o));
                bmx = fmax(bmx, __shfl_xor_sync(0xffffffffu, bmx, o));
            }
            if (bmn != bmx) return 0;
            for (int t = t0 + lane; t < t1; t += 32) sel[t] = bmn;
        } else {
            // the candidate with exactly r candidates ordered before it is the bin's r-th smallest
            int found = 0;
            for (int i = lane; i < m; i += 32) {
                const double vi = cand[i];
                int r = 0;
                for (int j = 0; j < m; ++j) {
                    const double vj = cand[j];
                    r += (vj < vi || (vj == vi && j < i)) ? 1 : 0;
                }
                for (int t = t0; t < t1; ++t)
                    if (trb[t] == r) { sel[t] = vi; ++found; }
            }
            if (__reduce_add_sync(0xffffffffu, found) != t1 - t0) return 0;
        }
        __syncwarp();
        t0 = t1;
    }
    return 1;
}

// ascending bitonic sort of one row's MC_NP slots by one warp
__device__ __forceinline__ void sort_row(double* row, const int lane) {
    for (int k = 2; k <= MC_NP; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int e = lane; e < MC_NP / 2; e += 32) {
                const int i = ((e & ~(j - 1)) << 1) | (e & (j - 1));
                const int l = i | j;
                const bool up = (i & k) == 0;
                const double x = row[i], y = row[l];
                const bool sw = up ? (x > y) : (x < y);
                if (sw) { row[i] = y; row[l] = x; }
            }
            __syncwarp();
        }
    }
}

// Per-warp scratch of the selection, carved from the dynamic shared memory after the [MC_TILE][MC_NP] rows.
struct SelScratch {
    double* cand;    // [MC_CAND]
    int* hist;       // [256]
    int* cnt;
    double* sel;     // [MC_QRANK]
    int* tb;         // [MC_QRANK]
    int* trb;        // [MC_QRANK]
};

constexpr int MC_WARPS = MC_THREADS / 32;
constexpr size_t MC_SMEM = (size_t)MC_TILE * MC_NP * 8 + (size_t)MC_WARPS * (MC_CAND * 8 + MC_QRANK * 16 + 256 * 4 + 4) + 16;

__device__ __forceinline__ SelScratch sel_scratch(unsigned char* smem, const int warp) {
    double* rows_end = (double*)smem + MC_TILE * MC_NP;
    double* cand = rows_end;                                       // [MC_WARPS][MC_CAND]
    double* sel = cand + MC_WARPS * MC_CAND;                       // [MC_WARPS][MC_QRANK]
    int* hist = (int*)(sel + MC_WARPS * MC_QRANK);                 // [MC_WARPS][256]
    int* tb = hist + MC_WARPS * 256;                               // [MC_WARPS][MC_QRANK]
    int* trb = tb + MC_WARPS * MC_QRANK;
    int* cnt = trb + MC_WARPS * MC_QRANK;                          // [MC_WARPS]
    return {cand + warp * MC_CAND, hist + warp * 256, cnt + warp, sel + warp * MC_QRANK, tb + warp * MC_QRANK,
            trb + warp * MC_QRANK};
}

// Every level of lv over one row of n draws (numpy's linear-interpolation percentiles): select_ranks, or -- when a
// histogram bin is too crowded for it -- a full bitonic sort of the row (all MC_NP slots: the padding draws hold
// INFINITY and sort to the end).  put(l, v) receives level l's value; the warp's lanes take levels l, l + 32, ...
template <bool TIES, class Put>
__device__ __forceinline__ void row_levels(double* row, const int n, const McLevels& lv, const SelScratch& w, const int lane,
                                           Put&& put) {
    const int got = select_ranks<TIES>(row, n, lv, w.hist, w.tb, w.trb, w.cand, w.cnt, lane, w.sel);
    if (got == 0) {
        sort_row(row, lane);
        for (int t = lane; t < lv.nrank; t += 32) w.sel[t] = row[lv.rank[t]];
        __syncwarp();
    }
    for (int l = lane; l < lv.nlev; l += 32) {
        const double v0 = w.sel[lv.ia[l]], v1 = w.sel[lv.ib[l]];
        put(l, got == 2 ? w.sel[0] : v0 + (v1 - v0) * lv.frac[l]);
    }
    __syncwarp();
}

// model i's frame: its first row and its points, model * H and H of a fixed frame of H points (RAGGED: the rows
// [offsets[i], offsets[i + 1]))
template <bool RAGGED>
__device__ __forceinline__ size_t frame_base(const McArgsT<RAGGED>& a, const int model, const int H) {
    if constexpr (RAGGED) return (size_t)a.offsets[model];
    else return (size_t)model * H;
}
template <bool RAGGED>
__device__ __forceinline__ int frame_len(const McArgsT<RAGGED>& a, const int model, const int H) {
    if constexpr (RAGGED) return (int)(a.offsets[model + 1] - a.offsets[model]);
    else return H;
}

// What a CTA does for a model before its first point: Tmax = max t over the whole frame, the model's Philox key, and
// the state of this thread's two draws (tid and tid + MC_THREADS) with the time of their first simulated changepoint.
// red_t [MC_THREADS / 32] and key_sm are shared scratch; every thread of the CTA calls it.
template <bool RAGGED = false>
__device__ __forceinline__ void start_draws(const McArgsT<RAGGED>& a, const ModelSm& ms, const int model, const int tid,
                                            double* red_t, uint64_t* key_sm, Philox& ph, DrawState* d, bool* live) {
    const int lane = tid & 31, warp = tid >> 5;
    const size_t base = frame_base<RAGGED>(a, model, a.p.horizon);
    const int H = frame_len<RAGGED>(a, model, a.p.horizon);
    double tm = -INFINITY;
    for (int h = tid; h < H; h += MC_THREADS) tm = fmax(tm, (double)(a.p.future_ds[base + h] - ms.start) / ms.t_scale);
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) tm = fmax(tm, __shfl_xor_sync(0xffffffffu, tm, o));
    if (lane == 0) red_t[warp] = tm;
    if (warp == 0) {
        const uint64_t key = model_key(a, model, lane);
        if (lane == 0) *key_sm = key;
    }
    __syncthreads();
    tm = red_t[0];
    for (int w = 1; w < MC_THREADS / 32; ++w) tm = fmax(tm, red_t[w]);
    const double rate = (double)ms.S;
    ph.k0 = (uint32_t)*key_sm;
    ph.k1 = (uint32_t)(*key_sm >> 32);
#pragma unroll
    for (int q = 0; q < 2; ++q) {
        const uint32_t draw = tid + q * MC_THREADS;
        live[q] = (int)draw < a.n_samples;
        d[q].k = ms.k; d[q].m = ms.m; d[q].s_hist = 0; d[q].cp_ctr = 0; d[q].next_cp = INFINITY;
        if (live[q] && tm > 1.0) {
            uint32_t r[4];
            ph.gen(draw, 0xffffffffu, 1u, 0u, r);
            d[q].next_cp = 1.0 - log(u01(r[0], r[1])) / rate;
        }
    }
}

// the two standard normals of one draw for the points 2 * pair and 2 * pair + 1 of the frame (Box-Muller: two per Philox call)
__device__ __forceinline__ void noise_pair(const Philox& ph, const uint32_t draw, const uint32_t pair, double* z) {
    uint32_t r[4];
    ph.gen(draw, pair, 0u, 0u, r);
    const double rad = sqrt(-2.0 * log(u01(r[0], r[1])));
    double sn, cs;
    sincospi(2.0 * u01(r[2], r[3]), &sn, &cs);
    z[0] = rad * cs;
    z[1] = rad * sn;
}

// one draw's yhat at the next point of the frame (time t, seasonal term sd, standard normal z): advances the draw's trend
// state to t; tr gets the noise-free trend.  rate = S, nscale = sigma_obs * y_scale
template <bool LOGI>
__device__ __forceinline__ double draw_point(DrawState& d, const ModelSm& ms, const double t, const double sd, const double z,
                                             const Philox& ph, const uint32_t draw, const double rate, const double nscale,
                                             const int mult, double& tr) {
    advance<LOGI>(d, ms, t, ph, draw, rate);
    if (LOGI) tr = ms.cap_s / (1.0 + exp(-d.k * (t - d.m)));
    else tr = d.k * t + d.m;
    tr = tr * ms.y_scale + ms.floor;
    return (mult ? tr * (1.0 + sd) : tr + sd * ms.y_scale) + nscale * z;
}

// TREND: also the bounds of the noise-free trend draws.  The tile is then TILE = 8 points: rows [0, 8) hold the yhat
// draws and rows [8, 16) the trend draws of the same points, in the same 128 KB, and warp w still selects row w.  The
// yhat draws are the same numbers (the noise counters go by pairs of points and 8 is even; the trend state advances per
// draw across tiles; Tmax is over the whole frame), so are their bounds.
// RAGGED: model i's frame is its own rows [offsets[i], offsets[i + 1]) (RaggedMcArgs), walked as a frame of that length:
// the same Tmax, key and counters as a fixed frame holding those rows first, so the same draws at those points.
// REGR: the models' regressors (RegMcArgs) added to the seasonal term of every draw, as predict_kernel adds them to yhat.
template <bool LOGI, bool TREND, bool RAGGED = false, bool REGR = false>
__global__ void __launch_bounds__(MC_THREADS, 1) mc_kernel(const McArgsT<RAGGED, REGR> a) {
    static_assert(!REGR || (!TREND && !RAGGED), "the regressor instance is the fixed-frame interval");
    constexpr int TILE = TREND ? MC_TILE / 2 : MC_TILE;
    extern __shared__ __align__(16) unsigned char mc_smem[];
    double* rows = (double*)mc_smem;                       // [MC_TILE][MC_NP]
    const SelScratch sw = sel_scratch(mc_smem, threadIdx.x >> 5);
    __shared__ ModelSm ms;
    __shared__ double seas[MC_TILE], tt[MC_TILE];
    __shared__ double red_t[MC_THREADS / 32];
    __shared__ uint64_t key_sm;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int H = a.p.horizon;
    const size_t NH = (size_t)a.p.n_models * H;
    const McLevels& lv = a.lv;
    // level l of point i: a quantile plane, or (the last two levels) the yhat bounds -- the trend bounds for trend rows
    auto out = [&](const int l, const size_t i, const bool trend) -> double& {
        if (l < lv.nq) return a.planes[(size_t)l * NH + i];
        if (TREND && trend) return l == lv.nq ? a.tlower[i] : a.tupper[i];
        return l == lv.nq ? a.lower[i] : a.upper[i];
    };
    for (int model = blockIdx.x; model < a.p.n_models; model += gridDim.x) {
        __syncthreads();
        load_model(ms, a.p, model, tid, MC_THREADS);
        const size_t base = frame_base<RAGGED>(a, model, H);
        const int HM = frame_len<RAGGED>(a, model, H);     // the model's points
        bool failed = ms.status < 0;
        if constexpr (REGR) failed = !reg_finite(a.reg, NH, model, H, tid, MC_THREADS) || failed;
        if (failed) {
            for (int l = 0; l < lv.nlev; ++l)
                for (int h = tid; h < HM; h += MC_THREADS) {
                    out(l, base + h, false) = NAN;
                    if (TREND) out(l, base + h, true) = NAN;
                }
            continue;
        }
        Philox ph;
        DrawState d[2];
        bool live[2];
        start_draws<RAGGED>(a, ms, model, tid, red_t, &key_sm, ph, d, live);
        const double rate = (double)ms.S, nscale = ms.sigma * ms.y_scale;
        for (int h0 = 0; h0 < HM; h0 += TILE) {
            const int np = min(TILE, HM - h0);
            if (tid < np) {
                const long long dsv = a.p.future_ds[base + h0 + tid];
                tt[tid] = (double)(dsv - ms.start) / ms.t_scale;
                double sv = ms.K > 0 ? seasonal_term(ms, dsv) : 0.0;
                if constexpr (REGR) sv += reg_term(a.reg, NH, ms, model, base + h0 + tid);
                seas[tid] = sv;
            }
            __syncthreads();
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const uint32_t draw = tid + q * MC_THREADS;
                if (!live[q]) {
                    for (int p = 0; p < np; ++p) {
                        rows[p * MC_NP + draw] = INFINITY;
                        if (TREND) rows[(TILE + p) * MC_NP + draw] = INFINITY;
                    }
                    continue;
                }
                for (int p = 0; p < np; p += 2) {
                    double z[2];
                    noise_pair(ph, draw, (uint32_t)((h0 + p) >> 1), z);
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        if (p + e >= np) break;
                        double tr;
                        const double yh = draw_point<LOGI>(d[q], ms, tt[p + e], seas[p + e], z[e], ph, draw, rate, nscale, a.p.mult, tr);
                        rows[(p + e) * MC_NP + draw] = yh;
                        if (TREND) rows[(TILE + p + e) * MC_NP + draw] = tr;
                    }
                }
            }
            __syncthreads();
            // ---- percentiles: warp w selects the order statistics of row w (point pt of the tile) ----
            const int pt = TREND ? (warp & (TILE - 1)) : warp;
            if (pt < np)
                row_levels<TREND>(rows + warp * MC_NP, a.n_samples, lv, sw, lane, [&](const int l, const double v) {
                    out(l, base + h0 + pt, TREND && warp >= TILE) = v;
                });
            __syncthreads();
        }
    }
}

// ---- window sums (DESIGN §13): fbprophet's predictive_samples summed per window, percentiles over the sums ----
struct McSumArgs {
    McArgs mc;                    // lower / upper: the window bounds [n_models * wmax]; tlower / tupper unused
    long long width_ns, origin_ns;
    int wmax;
    int* n_windows;               // [n_models]
    long long* win_start;         // [n_models * wmax] from here on
    int* win_points;
    double* yhat_sum;
    long long* quantity_sum;
    // mc_sum_kernel<LOGI, true> only (DESIGN §14): a window origin and a frame length per model, in place of origin_ns and
    // the horizon; the points past frame_len (the backtest frame's padding) are not walked
    const long long* origins;     // [n_models]
    const int* frame_len;         // [n_models]
};

// mc_sum_kernel's calendar instance (DESIGN §17): the windows are the calendar periods of the rule (months, month_shift)
// (calendar.cuh) in place of floor((ds - origin_ns) / width_ns).  Derived, as RaggedMcArgs, so that McSumArgs and the
// fixed-width instances keep their layout and code.
struct PeriodSumArgs : McSumArgs {
    int months, month_shift;
};
template <bool CAL>
using McSumArgsT = std::conditional_t<CAL, PeriodSumArgs, McSumArgs>;

constexpr int MC_SUM_TILE = 512;  // points whose t, seasonal term, window and predict outputs are staged at once (even: noise pairs)

// mathematical floor((ds - origin) / width), width > 0
__device__ __forceinline__ long long window_of(const long long ds, const long long origin, const long long width) {
    const long long a = ds - origin;
    const long long q = a / width;
    return (a % width != 0 && a < 0) ? q - 1 : q;
}

// The draws of mc_kernel (same key, counters, Tmax, trend state: the same numbers), but instead of selecting per point each
// thread keeps the running sum of its two draws over the points of the current window -- plain fp64 adds in frame order --
// and stores them into row (window mod 16) of the staging area when the window index of the next point differs.  After 16
// closed windows, and at the frame's end, warp r selects the percentiles of row r.  Thread 0 sums yhat / yhat_int of
// predict_kernel's output over the same windows, in the same order.  Windows at or past wmax are counted and not written.
// PER_MODEL: model i's windows are taken from origins[i] over its first frame_len[i] points only.  Tmax, the key and the
// counters stay those of the whole frame, so the draws at the walked points are unchanged (the backtest pads a frame by
// repeating its last timestamp, which leaves Tmax as it is).
// CAL: the windows are the calendar periods of a.months / a.month_shift (PeriodSumArgs), each starting at its period start;
// the draws, the sums and the selection are those of the fixed-width instance.
// QUANT (DESIGN §21): the same selection also writes levels [0, mc.lv.nq) of each window's sums to the planes
// mc.planes [nq][n_models * wmax] (the slot layout of lower / upper); the bounds are levels nq and nq + 1.
template <bool LOGI, bool PER_MODEL, bool CAL = false, bool QUANT = false>
__global__ void __launch_bounds__(MC_THREADS, 1) mc_sum_kernel(const McSumArgsT<CAL> a) {
    extern __shared__ __align__(16) unsigned char mc_smem[];
    double* rows = (double*)mc_smem;                       // [MC_TILE][MC_NP], as mc_kernel
    const SelScratch sw = sel_scratch(mc_smem, threadIdx.x >> 5);
    __shared__ ModelSm ms;
    __shared__ double seas[MC_SUM_TILE], tt[MC_SUM_TILE], yh_t[MC_SUM_TILE];
    __shared__ long long win[MC_SUM_TILE];
    __shared__ int yi_t[MC_SUM_TILE];
    __shared__ double red_t[MC_THREADS / 32];
    __shared__ uint64_t key_sm;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const McArgs& mc = a.mc;
    const int H = mc.p.horizon;
    for (int model = blockIdx.x; model < mc.p.n_models; model += gridDim.x) {
        __syncthreads();
        load_model(ms, mc.p, model, tid, MC_THREADS);
        const size_t base = (size_t)model * H, wbase = (size_t)model * a.wmax;
        int nw = 0;                                        // closed windows (the same in every thread)
        if (ms.status >= 0) {
            Philox ph;
            DrawState d[2];
            bool live[2];
            start_draws(mc, ms, model, tid, red_t, &key_sm, ph, d, live);
            const double rate = (double)ms.S, nscale = ms.sigma * ms.y_scale;
            double s[2] = {0.0, 0.0}, ys = 0.0;            // ys, qs: thread 0's sums of the point forecast
            long long qs = 0, cur_w = 0;
            int pts = 0;                                   // points of the open window (0: none open)
            // rows [0, n) hold the draws' sums of windows [nw - n, nw): warp r selects row r
            auto select_rows = [&](const int n) {
                __syncthreads();
                const int wi = nw - n + warp;
                if (warp < n && wi < a.wmax)
                    row_levels<false>(rows + warp * MC_NP, mc.n_samples, mc.lv, sw, lane, [&](const int l, const double v) {
                        if constexpr (QUANT) {
                            if (l < mc.lv.nq) mc.planes[(size_t)l * mc.p.n_models * a.wmax + wbase + wi] = v;
                            else (l == mc.lv.nq ? mc.lower : mc.upper)[wbase + wi] = v;
                        } else {
                            (l == 0 ? mc.lower : mc.upper)[wbase + wi] = v;
                        }
                    });
                __syncthreads();
            };
            auto close_window = [&]() {
                const int r = nw & (MC_TILE - 1);
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    rows[r * MC_NP + tid + q * MC_THREADS] = live[q] ? s[q] : INFINITY;
                    s[q] = 0.0;
                }
                if (tid == 0 && nw < a.wmax) {
                    if constexpr (CAL) a.win_start[wbase + nw] = period_start(cur_w, a.months, a.month_shift);
                    else a.win_start[wbase + nw] = (PER_MODEL ? a.origins[model] : a.origin_ns) + cur_w * a.width_ns;
                    a.win_points[wbase + nw] = pts;
                    a.yhat_sum[wbase + nw] = ys;
                    a.quantity_sum[wbase + nw] = qs;
                }
                ys = 0.0; qs = 0; pts = 0;
                if ((++nw & (MC_TILE - 1)) == 0) select_rows(MC_TILE);
            };
            const int HW = PER_MODEL ? min(a.frame_len[model], H) : H;   // points walked
            for (int h0 = 0; h0 < HW; h0 += MC_SUM_TILE) {
                const int np = min(MC_SUM_TILE, HW - h0);
                __syncthreads();                           // the previous tile has been walked
                if (tid < np) {
                    const long long dsv = mc.p.future_ds[base + h0 + tid];
                    tt[tid] = (double)(dsv - ms.start) / ms.t_scale;
                    seas[tid] = ms.K > 0 ? seasonal_term(ms, dsv) : 0.0;
                    if constexpr (CAL) win[tid] = period_of(dsv, a.months, a.month_shift);
                    else win[tid] = window_of(dsv, PER_MODEL ? a.origins[model] : a.origin_ns, a.width_ns);
                    yh_t[tid] = mc.p.yhat[base + h0 + tid];
                    yi_t[tid] = mc.p.yhat_int[base + h0 + tid];
                }
                __syncthreads();
                for (int p = 0; p < np; p += 2) {
                    double z[2][2];
#pragma unroll
                    for (int q = 0; q < 2; ++q)
                        if (live[q]) noise_pair(ph, tid + q * MC_THREADS, (uint32_t)((h0 + p) >> 1), z[q]);
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        if (p + e >= np) break;
                        const long long wv = win[p + e];
                        if (pts > 0 && wv != cur_w) close_window();
                        cur_w = wv;
                        ++pts;
#pragma unroll
                        for (int q = 0; q < 2; ++q) {
                            if (!live[q]) continue;
                            double tr;
                            const double yh = draw_point<LOGI>(d[q], ms, tt[p + e], seas[p + e], z[q][e], ph,
                                                               tid + q * MC_THREADS, rate, nscale, mc.p.mult, tr);
                            s[q] = __dadd_rn(s[q], yh);    // never contracted into the draw's last multiply-add
                        }
                        if (tid == 0) { ys = __dadd_rn(ys, yh_t[p + e]); qs += yi_t[p + e]; }
                    }
                }
            }
            if (pts > 0) close_window();
            if (nw & (MC_TILE - 1)) select_rows(nw & (MC_TILE - 1));
        }
        if (tid == 0) a.n_windows[model] = nw;
        for (int w = min(nw, a.wmax) + tid; w < a.wmax; w += MC_THREADS) {
            a.win_start[wbase + w] = INT64_MIN;
            a.win_points[wbase + w] = 0;
            a.yhat_sum[wbase + w] = NAN;
            a.quantity_sum[wbase + w] = INT64_MIN;
            mc.lower[wbase + w] = NAN;
            mc.upper[wbase + w] = NAN;
            if constexpr (QUANT)
                for (int l = 0; l < mc.lv.nq; ++l) mc.planes[(size_t)l * mc.p.n_models * a.wmax + wbase + w] = NAN;
        }
    }
}

template <bool LOGI, bool TREND, bool RAGGED = false, bool REGR = false>
cudaError_t launch_mc_inst(cudaStream_t st, int grid, size_t smem, const McArgsT<RAGGED, REGR>& a) {
    const cudaError_t e = cudaFuncSetAttribute(mc_kernel<LOGI, TREND, RAGGED, REGR>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    mc_kernel<LOGI, TREND, RAGGED, REGR><<<grid, MC_THREADS, smem, st>>>(a);
    return cudaGetLastError();
}

template <bool LOGI, bool PER_MODEL, bool CAL = false, bool QUANT = false>
cudaError_t launch_mc_sum_inst(cudaStream_t st, int grid, const McSumArgsT<CAL>& a) {
    const cudaError_t e = cudaFuncSetAttribute(mc_sum_kernel<LOGI, PER_MODEL, CAL, QUANT>,
                                               cudaFuncAttributeMaxDynamicSharedMemorySize, (int)MC_SMEM);
    if (e != cudaSuccess) return e;
    mc_sum_kernel<LOGI, PER_MODEL, CAL, QUANT><<<grid, MC_THREADS, MC_SMEM, st>>>(a);
    return cudaGetLastError();
}

// the instance of mc_sum_kernel for the growth, the window rule and the levels (nq > 0: QUANT)
template <bool QUANT>
cudaError_t launch_mc_sum_rule(cudaStream_t st, int grid, bool logi, bool per_model, const McSumArgs& s, int months,
                               int month_shift) {
    if (months > 0) {
        PeriodSumArgs c;
        static_cast<McSumArgs&>(c) = s;
        c.months = months;
        c.month_shift = month_shift;
        return logi ? launch_mc_sum_inst<true, false, true, QUANT>(st, grid, c)
                    : launch_mc_sum_inst<false, false, true, QUANT>(st, grid, c);
    }
    return logi ? (per_model ? launch_mc_sum_inst<true, true, false, QUANT>(st, grid, s)
                             : launch_mc_sum_inst<true, false, false, QUANT>(st, grid, s))
                : (per_model ? launch_mc_sum_inst<false, true, false, QUANT>(st, grid, s)
                             : launch_mc_sum_inst<false, false, false, QUANT>(st, grid, s));
}

// the sample count, the levels (McLevels: the nq percentiles pct[0, nq), each in [0, 100], then with `bounds` the
// interval's 100 (1 -+ width) / 2), the seed.  A level's rank and fraction are x = p / 100.0 * (n_samples - 1),
// i = floor(x), f = x - floor(x), so a plane at a bound's percentile is that bound.  False: sample count, interval width
// or level count out of range
inline bool mc_args(McArgs& a, const PredictArgs& p, int n_samples, double width, uint64_t seed, bool bounds = true,
                    int nq = 0, const double* pct = nullptr) {
    if (n_samples < 2 || n_samples > MC_NP || !(width >= 0.0 && width <= 1.0) || nq < 0 || nq > MC_QMAX) return false;
    a.p = p;
    a.n_samples = n_samples;
    McLevels& lv = a.lv;
    lv.nq = nq;
    lv.nlev = nq + (bounds ? 2 : 0);
    const double lower_p = 100.0 * (1.0 - width) / 2.0, upper_p = 100.0 * (1.0 + width) / 2.0;
    int r0[MC_QLEV], r1[MC_QLEV];
    for (int l = 0; l < lv.nlev; ++l) {
        const double pl = l < nq ? pct[l] : (l == nq ? lower_p : upper_p);
        const double x = pl / 100.0 * (n_samples - 1);
        r0[l] = (int)floor(x);
        r1[l] = r0[l] + 1 < n_samples - 1 ? r0[l] + 1 : n_samples - 1;
        lv.frac[l] = x - floor(x);
    }
    int rk[MC_QRANK];
    int nr = 0;
    for (int l = 0; l < lv.nlev; ++l) { rk[nr++] = r0[l]; rk[nr++] = r1[l]; }
    std::sort(rk, rk + nr);
    lv.nrank = (int)(std::unique(rk, rk + nr) - rk);
    for (int t = 0; t < MC_QRANK; ++t) lv.rank[t] = t < lv.nrank ? rk[t] : 0;
    for (int l = 0; l < MC_QLEV; ++l) {
        lv.ia[l] = l < lv.nlev ? (unsigned char)(std::lower_bound(rk, rk + lv.nrank, r0[l]) - rk) : 0;
        lv.ib[l] = l < lv.nlev ? (unsigned char)(std::lower_bound(rk, rk + lv.nrank, r1[l]) - rk) : 0;
        if (l >= lv.nlev) lv.frac[l] = 0.0;
    }
    a.seed = seed;
    a.lower = a.upper = a.tlower = a.tupper = a.planes = nullptr;
    return true;
}

// returns 0 ok, -1 sample count, interval width or level count out of range, 1 CUDA error.  lower / upper: the bounds, or
// both null; tlower / tupper: trend bounds (with the bounds), or both null; nq > 0: the quantile planes at the percentiles
// pct [nq] (not with the trend bounds)
inline int launch_mc(cudaStream_t st, int sms, const PredictArgs& p, int n_samples, double width, uint64_t seed,
                     double* lower, double* upper, double* tlower = nullptr, double* tupper = nullptr, int nq = 0,
                     const double* pct = nullptr, double* planes = nullptr) {
    McArgs a;
    const bool bounds = lower && upper;
    if ((!bounds && nq == 0) || (tlower && (!bounds || nq > 0))) return -1;
    if (!mc_args(a, p, n_samples, width, seed, bounds, nq, pct)) return -1;
    a.lower = lower;
    a.upper = upper;
    a.tlower = tlower;
    a.tupper = tupper;
    a.planes = planes;
    const bool trend = tlower && tupper;
    const int grid = p.n_models < sms ? p.n_models : sms;
    const bool logi = p.growth == PB200_GROWTH_LOGISTIC;
    const cudaError_t e = logi ? (trend ? launch_mc_inst<true, true>(st, grid, MC_SMEM, a) : launch_mc_inst<true, false>(st, grid, MC_SMEM, a))
                               : (trend ? launch_mc_inst<false, true>(st, grid, MC_SMEM, a) : launch_mc_inst<false, false>(st, grid, MC_SMEM, a));
    return e == cudaSuccess ? 0 : 1;
}

// the bounds of mc_kernel's ragged instance over model i's rows [offsets[i], offsets[i + 1]) of p.future_ds (device
// array [n_models + 1]).  Returns as launch_mc
inline int launch_mc_ragged(cudaStream_t st, int sms, const PredictArgs& p, const long long* offsets, int n_samples,
                            double width, uint64_t seed, double* lower, double* upper) {
    RaggedMcArgs a;
    if (!mc_args(a, p, n_samples, width, seed)) return -1;
    a.lower = lower;
    a.upper = upper;
    a.offsets = offsets;
    const int grid = p.n_models < sms ? p.n_models : sms;
    const cudaError_t e = p.growth == PB200_GROWTH_LOGISTIC ? launch_mc_inst<true, false, true>(st, grid, MC_SMEM, a)
                                                            : launch_mc_inst<false, false, true>(st, grid, MC_SMEM, a);
    return e == cudaSuccess ? 0 : 1;
}

// the bounds of mc_kernel's instance with regressors over p's fixed frame.  Returns as launch_mc
inline int launch_mc_reg(cudaStream_t st, int sms, const PredictArgs& p, const RegFrame& reg, int n_samples, double width,
                         uint64_t seed, double* lower, double* upper) {
    RegMcArgs a;
    if (!mc_args(a, p, n_samples, width, seed)) return -1;
    a.lower = lower;
    a.upper = upper;
    a.reg = reg;
    const int grid = p.n_models < sms ? p.n_models : sms;
    const cudaError_t e = p.growth == PB200_GROWTH_LOGISTIC ? launch_mc_inst<true, false, false, true>(st, grid, MC_SMEM, a)
                                                            : launch_mc_inst<false, false, false, true>(st, grid, MC_SMEM, a);
    return e == cudaSuccess ? 0 : 1;
}

// mc_sum_kernel over the frame of p, whose yhat / yhat_int predict_kernel has written on the same stream; s.mc is filled
// here but for its lower / upper (the window bounds).  s.origins != null: the per-model instance (s.frame_len as well);
// months > 0: the calendar instance over the periods of (months, month_shift), whose width_ns / origin_ns are unused.
// nq > 0: the QUANT instance, which also writes the window quantiles at the percentiles pct [nq] to planes
// [nq][n_models * wmax].  Returns as launch_mc
inline int launch_mc_sum(cudaStream_t st, int sms, const PredictArgs& p, int n_samples, double width, uint64_t seed,
                         McSumArgs& s, int months = 0, int month_shift = 0, int nq = 0, const double* pct = nullptr,
                         double* planes = nullptr) {
    double* const lo = s.mc.lower;
    double* const hi = s.mc.upper;
    if ((nq > 0) != (planes != nullptr)) return -1;
    if (!mc_args(s.mc, p, n_samples, width, seed, true, nq, pct)) return -1;
    s.mc.lower = lo;
    s.mc.upper = hi;
    s.mc.planes = planes;
    const int grid = p.n_models < sms ? p.n_models : sms;
    const bool logi = p.growth == PB200_GROWTH_LOGISTIC, per_model = s.origins != nullptr;
    const cudaError_t e = nq > 0 ? launch_mc_sum_rule<true>(st, grid, logi, per_model, s, months, month_shift)
                                 : launch_mc_sum_rule<false>(st, grid, logi, per_model, s, months, month_shift);
    return e == cudaSuccess ? 0 : 1;
}

}  // namespace pb200
