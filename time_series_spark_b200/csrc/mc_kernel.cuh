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
// Philox4x32-10 keyed by (seed, model, draw), reproducible and shard-independent.
//
// One CTA per model; thread j owns draws j and j + 512; the draws of a tile of 16 future
// points are staged in shared memory ([16][1024] fp64) and each warp sorts one row's order
// statistics (256-bin histogram + exact selection inside the bin; bitonic sort as fallback).  Requires future timestamps ascending
// within a model (make_future_dataframe's output is).
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

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

struct McArgs {
    PredictArgs p;
    int n_samples;
    int lo_i, hi_i;
    double lo_f, hi_f;
    uint64_t seed;
    double* lower;
    double* upper;
};

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

// k-th smallest of the n values of `row` (k 0-based) by a 256-bin histogram + exact selection inside
// the bin that holds rank k.  Returns false if that bin holds more than MC_CAND values.
__device__ __forceinline__ bool kth_smallest(const double* row, const int n, const int k, const double mn,
                                             const double scale, const int* hist, const int base, const int lsum,
                                             double* cand, int* cnt, const int lane, double& out) {
    // which lane's 8 bins contain rank k, and which bin
    int b = -1, rb = 0;
    if (k >= base && k < base + lsum) {
        int cum = base;
        for (int q = 0; q < 8; ++q) {
            const int c = hist[lane * 8 + q];
            if (k < cum + c) { b = lane * 8 + q; rb = k - cum; break; }
            cum += c;
        }
    }
    const unsigned who = __ballot_sync(0xffffffffu, b >= 0);
    const int src = __ffs(who) - 1;
    b = __shfl_sync(0xffffffffu, b, src);
    rb = __shfl_sync(0xffffffffu, rb, src);
    if (lane == 0) *cnt = 0;
    __syncwarp();
    for (int e = lane; e < n; e += 32) {
        const double v = row[e];
        const int bb = min(255, (int)((v - mn) * scale));
        if (bb == b) {
            const int pos = atomicAdd(cnt, 1);
            if (pos < MC_CAND) cand[pos] = v;
        }
    }
    __syncwarp();
    const int m = *cnt;
    if (m > MC_CAND) return false;
    // exact selection: the candidate with exactly rb candidates ordered before it
    double found = 0.0;
    int have = 0;
    for (int i = lane; i < m; i += 32) {
        const double vi = cand[i];
        int r = 0;
        for (int j = 0; j < m; ++j) {
            const double vj = cand[j];
            r += (vj < vi || (vj == vi && j < i)) ? 1 : 0;
        }
        if (r == rb) { found = vi; have = 1; }
    }
    const unsigned w2 = __ballot_sync(0xffffffffu, have);
    out = __shfl_sync(0xffffffffu, found, __ffs(w2) - 1);
    __syncwarp();
    return w2 != 0;
}

// numpy percentile (linear interpolation) at the two interval bounds from the draws of one point
__device__ __forceinline__ bool select_quantiles(const double* row, const int n, const int lo_i, const double lo_f,
                                                 const int hi_i, const double hi_f, int* hist, double* cand, int* cnt,
                                                 const int lane, double& lo_v, double& hi_v) {
    double mn = INFINITY, mx = -INFINITY;
    for (int e = lane; e < n; e += 32) { const double v = row[e]; mn = fmin(mn, v); mx = fmax(mx, v); }
#pragma unroll
    for (int o = 16; o >= 1; o >>= 1) {
        mn = fmin(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if (!(mx > mn) || !isfinite(mx - mn)) {
        if (mx == mn) { lo_v = hi_v = mn; return true; }
        return false;
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
    const int base = inc - lsum;
    double v[4];
    const int ranks[4] = {lo_i, min(lo_i + 1, n - 1), hi_i, min(hi_i + 1, n - 1)};
    for (int q = 0; q < 4; ++q) {
        if (q > 0 && ranks[q] == ranks[q - 1]) { v[q] = v[q - 1]; continue; }
        if (!kth_smallest(row, n, ranks[q], mn, scale, hist, base, lsum, cand, cnt, lane, v[q])) return false;
    }
    lo_v = v[0] + (v[1] - v[0]) * lo_f;
    hi_v = v[2] + (v[3] - v[2]) * hi_f;
    return true;
}

template <bool LOGI>
__global__ void __launch_bounds__(MC_THREADS, 1) mc_kernel(const McArgs a) {
    extern __shared__ __align__(16) unsigned char mc_smem[];
    double* rows = (double*)mc_smem;                       // [MC_TILE][MC_NP]
    double* cand = rows + MC_TILE * MC_NP;                 // [MC_THREADS/32][MC_CAND]
    int* hist = (int*)(cand + (MC_THREADS / 32) * MC_CAND);   // [MC_THREADS/32][256]
    int* cnt = hist + (MC_THREADS / 32) * 256;             // [MC_THREADS/32]
    __shared__ ModelSm ms;
    __shared__ double seas[MC_TILE], tt[MC_TILE];
    __shared__ double red_t[MC_THREADS / 32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int H = a.p.horizon;
    for (int model = blockIdx.x; model < a.p.n_models; model += gridDim.x) {
        __syncthreads();
        load_model(ms, a.p, model, tid, MC_THREADS);
        const size_t base = (size_t)model * H;
        if (ms.status < 0) {
            for (int h = tid; h < H; h += MC_THREADS) { a.lower[base + h] = NAN; a.upper[base + h] = NAN; }
            continue;
        }
        // Tmax = max t over the frame
        double tm = -INFINITY;
        for (int h = tid; h < H; h += MC_THREADS) tm = fmax(tm, (double)(a.p.future_ds[base + h] - ms.start) / ms.t_scale);
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) tm = fmax(tm, __shfl_xor_sync(0xffffffffu, tm, o));
        if (lane == 0) red_t[warp] = tm;
        __syncthreads();
        tm = red_t[0];
        for (int w = 1; w < MC_THREADS / 32; ++w) tm = fmax(tm, red_t[w]);
        const double rate = (double)ms.S;
        Philox ph;
        ph.k0 = (uint32_t)a.seed ^ (uint32_t)model * 0x9E3779B1u;
        ph.k1 = (uint32_t)(a.seed >> 32) ^ 0x85EBCA6Bu ^ (uint32_t)((uint64_t)model >> 7);
        DrawState d[2];
        bool live[2];
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
        const double nscale = ms.sigma * ms.y_scale;
        for (int h0 = 0; h0 < H; h0 += MC_TILE) {
            const int np = min(MC_TILE, H - h0);
            if (tid < np) {
                const long long dsv = a.p.future_ds[base + h0 + tid];
                tt[tid] = (double)(dsv - ms.start) / ms.t_scale;
                seas[tid] = ms.K > 0 ? seasonal_term(ms, dsv) : 0.0;
            }
            __syncthreads();
#pragma unroll
            for (int q = 0; q < 2; ++q) {
                const uint32_t draw = tid + q * MC_THREADS;
                if (!live[q]) {
                    for (int p = 0; p < np; ++p) rows[p * MC_NP + draw] = INFINITY;
                    continue;
                }
                for (int p = 0; p < np; p += 2) {
                    uint32_t r[4];
                    ph.gen(draw, (uint32_t)((h0 + p) >> 1), 0u, 0u, r);
                    // Box-Muller: two normals per Philox call
                    const double rad = sqrt(-2.0 * log(u01(r[0], r[1])));
                    double sn, cs;
                    sincospi(2.0 * u01(r[2], r[3]), &sn, &cs);
                    const double z[2] = {rad * cs, rad * sn};
#pragma unroll
                    for (int e = 0; e < 2; ++e) {
                        if (p + e >= np) break;
                        const double t = tt[p + e];
                        advance<LOGI>(d[q], ms, t, ph, draw, rate);
                        double tr;
                        if (LOGI) tr = ms.cap_s / (1.0 + exp(-d[q].k * (t - d[q].m)));
                        else tr = d[q].k * t + d[q].m;
                        tr = tr * ms.y_scale + ms.floor;
                        const double sd = seas[p + e];
                        const double yh = (a.p.mult ? tr * (1.0 + sd) : tr + sd * ms.y_scale) + nscale * z[e];
                        rows[(p + e) * MC_NP + draw] = yh;
                    }
                }
            }
            __syncthreads();
            // ---- percentiles: warp w selects the order statistics of row w ----
            if (warp < np) {
                double* row = rows + warp * MC_NP;
                double lo_v, hi_v;
                if (!select_quantiles(row, a.n_samples, a.lo_i, a.lo_f, a.hi_i, a.hi_f, hist + warp * 256,
                                      cand + warp * MC_CAND, cnt + warp, lane, lo_v, hi_v)) {
                    // fallback (a histogram bin too crowded): full bitonic sort of the row
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
                    const double l0 = row[a.lo_i], l1 = row[min(a.lo_i + 1, a.n_samples - 1)];
                    const double u0 = row[a.hi_i], u1 = row[min(a.hi_i + 1, a.n_samples - 1)];
                    lo_v = l0 + (l1 - l0) * a.lo_f;
                    hi_v = u0 + (u1 - u0) * a.hi_f;
                }
                if (lane == 0) {
                    a.lower[base + h0 + warp] = lo_v;
                    a.upper[base + h0 + warp] = hi_v;
                }
            }
            __syncthreads();
        }
    }
}

// returns 0 ok, -1 unsupported sample count, 1 CUDA error
inline int launch_mc(cudaStream_t st, int sms, const PredictArgs& p, int n_samples, double width, uint64_t seed,
                     double* lower, double* upper) {
    if (n_samples < 2 || n_samples > MC_NP) return -1;
    McArgs a;
    a.p = p;
    a.n_samples = n_samples;
    const double lower_p = 100.0 * (1.0 - width) / 2.0, upper_p = 100.0 * (1.0 + width) / 2.0;
    const double li = lower_p / 100.0 * (n_samples - 1), ui = upper_p / 100.0 * (n_samples - 1);
    a.lo_i = (int)floor(li); a.lo_f = li - floor(li);
    a.hi_i = (int)floor(ui); a.hi_f = ui - floor(ui);
    a.seed = seed;
    a.lower = lower;
    a.upper = upper;
    const size_t smem = (size_t)MC_TILE * MC_NP * 8 + (size_t)(MC_THREADS / 32) * (MC_CAND * 8 + 256 * 4 + 4) + 16;
    const int grid = p.n_models < sms ? p.n_models : sms;
    cudaError_t e;
    if (p.growth == PB200_GROWTH_LOGISTIC) {
        e = cudaFuncSetAttribute(mc_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return 1;
        mc_kernel<true><<<grid, MC_THREADS, smem, st>>>(a);
    } else {
        e = cudaFuncSetAttribute(mc_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return 1;
        mc_kernel<false><<<grid, MC_THREADS, smem, st>>>(a);
    }
    return cudaGetLastError() == cudaSuccess ? 0 : 1;
}

}  // namespace pb200
