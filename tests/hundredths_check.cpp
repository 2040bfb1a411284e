// brc::f2_hundredths (the digits put_f2 prints, and the value the site filter's entry bounds compare) against printf("%.2f"):
// every quotient (float)a / (float)b with a < 2^16, b <= 2048, 10^7 random finite float32 bit patterns below 2^40 in
// magnitude, and binary ties.  Compiled and run by tests/test_site_filter_bounds.py.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <thread>
#include <vector>
#include "../bam_readcount_b200/csrc/brc_fmt_num.h"

static bool same(float f) {
    char t[96];
    std::snprintf(t, sizeof t, "%.2f", (double)f);
    const char *p = t[0] == '-' ? t + 1 : t;
    uint64_t want = 0;
    for (; *p; ++p) if (*p != '.') want = want * 10 + (uint64_t)(*p - '0');
    return brc::f2_hundredths(f) == want;
}

int main() {
    const int nt = std::max(1u, std::thread::hardware_concurrency());
    std::vector<long> bad((size_t)nt, 0), n((size_t)nt, 0);
    std::vector<std::thread> th;
    for (int t = 0; t < nt; ++t)
        th.emplace_back([&, t] {
            for (uint32_t b = 1 + (uint32_t)t; b <= 2048; b += (uint32_t)nt)
                for (uint32_t a = 0; a < (1u << 16); ++a) {
                    const float q = (float)a / (float)b;
                    ++n[(size_t)t];
                    if (!same(q)) { if (bad[(size_t)t]++ < 3) std::printf("MISMATCH %u/%u = %a\n", a, b, (double)q); }
                }
            std::mt19937 rng(1234u + (uint32_t)t);
            for (long i = 0; i < 10000000 / nt + 1; ++i) {
                uint32_t bits = rng() & 0x7FFFFFFFu;
                if (((bits >> 23) & 0xFF) >= 127 + 40) bits = (bits & 0x807FFFFFu) | ((uint32_t)((bits >> 23) % (127 + 40)) << 23);
                bits |= rng() & 0x80000000u;
                float f; std::memcpy(&f, &bits, 4);
                ++n[(size_t)t];
                if (!same(f)) { if (bad[(size_t)t]++ < 3) std::printf("MISMATCH bits %08x\n", bits); }
            }
        });
    for (auto &x : th) x.join();
    long tb = 0, tn = 0;
    for (int t = 0; t < nt; ++t) { tb += bad[(size_t)t]; tn += n[(size_t)t]; }
    const struct { float f; uint64_t h; } ties[] = {{0.125f, 12}, {0.375f, 38}, {0.625f, 62}, {0.875f, 88}, {2.5f / 8.0f * 8.0f, 250},
                                                   {1.0f / 8.0f + 1.0f, 112}, {0.005f, 0}, {0.015f, 1}, {0.0f, 0}};
    for (auto &c : ties) { ++tn; if (brc::f2_hundredths(c.f) != c.h || !same(c.f)) { ++tb; std::printf("TIE %a\n", (double)c.f); } }
    std::printf("checked %ld values, %ld mismatches\n", tn, tb);
    return tb ? 1 : 0;
}
