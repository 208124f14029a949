// Proleptic Gregorian civil-date arithmetic over the whole int64-ns range (1677-09-21 .. 2262-04-11), and the calendar
// periods of DESIGN §17: the period of ds under a rule (months, shift) is floor((mi + shift) / months), mi the months of
// ds's civil date since 1970-01, and period p starts at 00:00 on day 1 of month p * months - shift.  Every function is
// __host__ __device__ so that the CPU tests run the very code the kernels run (pb200_period_host).  civil_from_days /
// days_from_civil are Howard Hinnant's algorithms, with the era floored so that negative day counts work too.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pb200 {

constexpr int64_t NS_PER_DAY = 86400LL * 1000000000LL;

// mathematical floor(a / b), b > 0
__host__ __device__ __forceinline__ int64_t floor_div(const int64_t a, const int64_t b) {
    const int64_t q = a / b;
    return (a % b != 0 && a < 0) ? q - 1 : q;
}

// civil date of a day count since 1970-01-01
__host__ __device__ __forceinline__ void civil_from_days(int64_t z, int& y, int& m, int& d) {
    z += 719468;
    const int64_t era = (z >= 0 ? z : z - 146096) / 146097;
    const unsigned doe = (unsigned)(z - era * 146097);
    const unsigned yoe = (doe - doe / 1460 + doe / 36524 - doe / 146096) / 365;
    const unsigned doy = doe - (365 * yoe + yoe / 4 - yoe / 100);
    const unsigned mp = (5 * doy + 2) / 153;
    d = (int)(doy - (153 * mp + 2) / 5 + 1);
    m = (int)(mp < 10 ? mp + 3 : mp - 9);
    y = (int)(yoe + era * 400) + (m <= 2 ? 1 : 0);
}

// day count since 1970-01-01 of the civil date y-m-d
__host__ __device__ __forceinline__ int64_t days_from_civil(int64_t y, const int m, const int d) {
    y -= m <= 2 ? 1 : 0;
    const int64_t era = (y >= 0 ? y : y - 399) / 400;
    const unsigned yoe = (unsigned)(y - era * 400);
    const unsigned doy = (153 * (unsigned)(m > 2 ? m - 3 : m + 9) + 2) / 5 + (unsigned)d - 1;
    const unsigned doe = yoe * 365 + yoe / 4 - yoe / 100 + doy;
    return era * 146097 + (int64_t)doe - 719468;
}

// the period of ds (ns since 1970-01-01, naive) under the rule (months, shift), months in {1, 3, 12}, 0 <= shift < months
__host__ __device__ __forceinline__ int64_t period_of(const int64_t ds, const int months, const int shift) {
    int y, m, d;
    civil_from_days(floor_div(ds, NS_PER_DAY), y, m, d);
    const int64_t mi = 12 * (int64_t)(y - 1970) + (m - 1);
    return floor_div(mi + shift, months);
}

// the start (ns) of period p under the rule (months, shift).  The product is taken mod 2^64: a start before the int64-ns
// minimum (Y-JAN's period of 1678-01 starts in 1677-02) wraps to a value above every ds of its period, which is how the
// callers recognise it
__host__ __device__ __forceinline__ int64_t period_start(const int64_t p, const int months, const int shift) {
    const int64_t mi = p * months - shift;
    const int64_t yi = floor_div(mi, 12);
    const int64_t days = days_from_civil(1970 + yi, (int)(mi - 12 * yi) + 1, 1);
    return (int64_t)((uint64_t)days * (uint64_t)NS_PER_DAY);
}

}  // namespace pb200
