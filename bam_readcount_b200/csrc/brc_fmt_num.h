// brc_fmt_num.h — exact, printf-free number formatting for the text emitter.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

namespace brc {

inline void put_u(std::string &o, uint64_t x) {
    char t[24]; int n = 0;
    do { t[n++] = (char)('0' + x % 10); x /= 10; } while (x);
    while (n) o += t[--n];
}

// Compiled by nvcc for the device (the site filter's entry bounds, brc_device.cuh) and by the host compiler for the emitter.
#ifdef __CUDACC__
#define BRC_NUM_HD __host__ __device__
#else
#define BRC_NUM_HD
#endif

// The hundredths printf("%.2f", (double)x) prints for |x| (what `std::fixed << std::setprecision(2) << float` prints,
// R:src/lib/bamrc/BasicStat.cpp:115-141): the binary value times 100 rounded half-to-even in integer arithmetic, so 0.125
// gives 12 and 0.375 gives 38.  Exact for |x| < 2^54; larger values, infinities and NaN give UINT64_MAX.
BRC_NUM_HD inline uint64_t f2_hundredths(float x) {
    uint32_t b; std::memcpy(&b, &x, 4);
    const uint32_t ex = (b >> 23) & 0xFF, mant = b & 0x7FFFFF;
    if (ex >= 150 + 31) return ~0ull;
    const uint64_t m = ex ? (uint64_t)(mant | 0x800000u) : (uint64_t)mant;
    const int e = (ex ? (int)ex : 1) - 150;          // |x| = m * 2^e
    const uint64_t x100 = m * 100u;
    if (e >= 0) return x100 << e;
    const int sh = -e;
    if (sh >= 64) return 0;
    uint64_t q = x100 >> sh;
    const uint64_t r = x100 & ((1ull << sh) - 1), half = 1ull << (sh - 1);
    if (r > half || (r == half && (q & 1))) ++q;
    return q;
}

// printf("%.2f", (double)x) for a float32, printf-free
inline void put_f2(std::string &o, float x) {
    uint32_t b; std::memcpy(&b, &x, 4);
    if (((b >> 23) & 0xFF) >= 150 + 31) {   // NaN / inf / >= 2^54: let libc do it
        char t[96]; int n = std::snprintf(t, sizeof t, "%.2f", (double)x); o.append(t, (size_t)n); return;
    }
    const uint64_t q = f2_hundredths(x);
    if (b >> 31) o += '-';
    put_u(o, q / 100);
    o += '.';
    const unsigned f = (unsigned)(q % 100);
    o += (char)('0' + f / 10); o += (char)('0' + f % 10);
}

}  // namespace brc
