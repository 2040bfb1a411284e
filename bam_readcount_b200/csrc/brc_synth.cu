// brc_synth.cu — counter-based generator of the synthetic BASELINE workloads (include/brc_synth.h): libbrc_synth.so.
//
// One source for the device kernels and the host implementation: every value is an integer function of
// (seed, contig | site, block, read), so a window generated in HBM on the GPU box and the same window generated on
// the host (for the oracle / the reference binary) are byte-identical.  Workload infrastructure — the engine
// (libbrc_engine.so) never links this.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/brc_synth.h"
#include "brc_seq.cuh"

#define HD __host__ __device__ __forceinline__

namespace {

constexpr int RL = BRC_SYNTH_READ_LEN, SB = (BRC_SYNTH_READ_LEN + 1) / 2, BR = BRC_SYNTH_BLOCK_READS, BBP = BRC_SYNTH_BLOCK_BP;
constexpr int32_t TAG_ABSENT = INT32_MIN;

HD int64_t imin64(int64_t a, int64_t b) { return a < b ? a : b; }
HD uint64_t mix64(uint64_t x) {
    x ^= x >> 30; x *= 0xbf58476d1ce4e5b9ULL;
    x ^= x >> 27; x *= 0x94d049bb133111ebULL;
    x ^= x >> 31;
    return x;
}
HD uint64_t read_key(uint64_t seed, uint64_t unit, uint64_t blk, uint64_t j) {
    return mix64(mix64(seed + 0x9E3779B97F4A7C15ULL * (unit + 1)) ^ (blk * 0xD1B54A32D192ED03ULL + j * 0x8CB92BA72F3D8DD7ULL + 0x632BE59BD9B4E019ULL));
}
HD uint64_t sub_stream(uint64_t rk, uint64_t s) { return mix64(rk + (s + 1) * 0xA24BAED4963EE407ULL); }
HD uint64_t ref_word(uint64_t seed, uint64_t contig, uint64_t w) {   // 32 bases, 2 bits each
    return mix64(mix64((seed ^ 0x5EEDBA5E5EEDBA5EULL) + contig * 0x9E3779B97F4A7C15ULL) ^ (w * 0xC2B2AE3D27D4EB4FULL + 0x165667B19E3779F9ULL));
}
HD uint32_t ref_base(uint64_t seed, uint64_t contig, int64_t p) { return (uint32_t)(ref_word(seed, contig, (uint64_t)p >> 5) >> (2 * (p & 31))) & 3u; }

struct Hdr {
    uint64_t rk;
    int32_t kind;       // 0: 150M, 1: 70M2I78M, 2: 60M3D90M, 3: 10S140M
    int32_t reverse, mapq, tail, n_subs;
    uint32_t off;       // WGS: start offset inside the block
};
HD Hdr make_hdr(uint64_t seed, uint64_t unit, uint64_t blk, uint64_t j) {
    Hdr h;
    h.rk = read_key(seed, unit, blk, j);
    const uint64_t h0 = sub_stream(h.rk, 0), h1 = sub_stream(h.rk, 1);
    h.off = (uint32_t)(h0 & 0xFFFFFFFFu) % (uint32_t)BBP;
    const uint32_t kk = (uint32_t)(h0 >> 32) & 0xFFFFu;
    h.kind = kk < 58982u ? 0 : (kk < 60948u ? 1 : (kk < 62914u ? 2 : 3));
    h.reverse = (int32_t)((h0 >> 48) & 1u);
    const uint32_t mi = (uint32_t)((h0 >> 49) & 0x7FFFu) % 6u;
    h.mapq = mi < 3u ? 60 : (mi == 3u ? 40 : (mi == 4u ? 20 : 0));
    h.tail = (!h.reverse && (uint32_t)(h1 & 0xFFFFu) < 13107u) ? 1 + (int32_t)(((uint32_t)(h1 >> 16) & 0xFFFFu) % 19u) : 0;
    const uint32_t u = (uint32_t)(h1 >> 32) & 0xFFFFu;   // Binomial(150, 0.005) by inverse CDF
    h.n_subs = u < 30898u ? 0 : (u < 54188u ? 1 : (u < 62908u ? 2 : (u < 65069u ? 3 : (u < 65469u ? 4 : (u < 65527u ? 5 : 6)))));
    return h;
}
HD int n_cigar_of(int kind) { return kind == 0 ? 1 : (kind == 3 ? 2 : 3); }
HD int span_of(int kind) { return kind == 0 ? 150 : (kind == 1 ? 148 : (kind == 2 ? 153 : 140)); }
HD void cigar_of(int kind, uint32_t *c) {
    if (kind == 0) { c[0] = (150u << 4) | 0u; }
    else if (kind == 1) { c[0] = (70u << 4) | 0u; c[1] = (2u << 4) | 1u; c[2] = (78u << 4) | 0u; }
    else if (kind == 2) { c[0] = (60u << 4) | 0u; c[1] = (3u << 4) | 2u; c[2] = (90u << 4) | 0u; }
    else { c[0] = (10u << 4) | 4u; c[1] = (140u << 4) | 0u; }
}
// query position -> reference offset from the read start, or -1 for inserted / clipped bases
HD int ref_off(int kind, int q) {
    if (kind == 0) return q;
    if (kind == 1) return q < 70 ? q : (q < 72 ? -1 : q - 2);
    if (kind == 2) return q < 60 ? q : q + 3;
    return q < 10 ? -1 : q - 10;
}

// bases (4-bit packed, 75 bytes) and qualities (150 bytes) of one read; returns NM.
// Everything stays in registers (no indexed local arrays): quality values come out of a packed constant, the <= 6 substitution
// positions live in one 64-bit word and are patched into the finished row.
HD int32_t make_body(uint64_t seed, uint64_t contig, const Hdr &h, int64_t start, uint8_t *seq, uint8_t *qual) {
    const uint64_t hb = sub_stream(h.rk, 4);
    uint64_t rw = 0; int64_t rw_idx = -1;
    const uint64_t qtab = 0x020C191E252525ULL;                     // {37,37,37,30,25,12,2}, 8 bits each
    uint64_t hq = 0; uint32_t hi_nib = 0;
    const int tail_from = RL - h.tail;
    for (int q = 0; q < RL; ++q) {
        if ((q & 7) == 0) hq = sub_stream(h.rk, 8 + (uint64_t)(q >> 3));
        const uint32_t qb = (uint32_t)(hq >> (8 * (q & 7))) & 0xFFu;
        qual[q] = q >= tail_from ? (uint8_t)2 : (uint8_t)(qtab >> (8 * ((qb * 7u) >> 8)));
        const int ro = ref_off(h.kind, q);
        uint32_t base;
        if (ro >= 0) {
            const int64_t p = start + ro;
            if ((p >> 5) != rw_idx) { rw_idx = p >> 5; rw = ref_word(seed, contig, (uint64_t)rw_idx); }
            base = (uint32_t)(rw >> (2 * (p & 31))) & 3u;
        } else base = (uint32_t)(hb >> (2 * (q & 31))) & 3u;
        const uint32_t nib = 1u << base;
        if (q & 1) seq[q >> 1] = (uint8_t)((hi_nib << 4) | nib); else hi_nib = nib;
    }
    if (RL & 1) seq[RL >> 1] = (uint8_t)(hi_nib << 4);
    // substitutions: distinct positions (first occurrence wins), only on bases that came from the reference
    int32_t nm = h.kind == 1 ? 2 : (h.kind == 2 ? 3 : 0);
    if (h.n_subs > 0) {
        const uint64_t h2 = sub_stream(h.rk, 2), h3 = sub_stream(h.rk, 3);
        uint64_t seen = ~0ull;                                      // up to 6 positions, 8 bits each (0xFF = none)
        for (int t = 0; t < 6; ++t) {
            if (t >= h.n_subs) break;
            const uint64_t src = t < 3 ? h2 >> (20 * t) : h3 >> (20 * (t - 3));
            const uint32_t p = (uint32_t)(src & 0xFFFFu) % (uint32_t)RL;
            const uint32_t sft = 1u + ((uint32_t)((src >> 16) & 0xFu) % 3u);
            bool dup = false;
            for (int k = 0; k < 6; ++k) dup = dup || ((uint32_t)(seen >> (8 * k)) & 0xFFu) == p;
            if (dup) continue;
            seen = (seen << 8) | p;
            if (ref_off(h.kind, (int)p) < 0) continue;
            const uint32_t byte = seq[p >> 1];
            const uint32_t nib = (p & 1u) ? (byte & 15u) : (byte >> 4);
            const uint32_t code = nib == 1u ? 0u : (nib == 2u ? 1u : (nib == 4u ? 2u : 3u));
            const uint32_t nn = 1u << ((code + sft) & 3u);
            seq[p >> 1] = (uint8_t)((p & 1u) ? ((byte & 0xF0u) | nn) : ((byte & 0x0Fu) | (nn << 4)));
            ++nm;
        }
    }
    return nm;
}

// identity of read r (file order) of CTA-block b of the window: WGS needs the block's sorted order (key array)
struct Slot { Hdr h; int64_t start; uint64_t unit, blk, j; int32_t lib, region; bool valid; };

HD int64_t wgs_start(const brc_synth_spec &S, int64_t block, uint32_t off) {
    int64_t s = block * BBP + off;
    const int64_t last = S.contig_len - BRC_SYNTH_MAX_SPAN;
    return s > last ? (last > 0 ? last : 0) : s;
}
HD Slot deep_slot(const brc_synth_spec &S, int64_t site_lo, int64_t idx, int64_t n_reads) {
    Slot s; s.valid = idx < n_reads;
    const int64_t k = idx / S.depth, i = idx - k * S.depth;
    s.unit = 0; s.blk = (uint64_t)(site_lo + k); s.j = (uint64_t)i;
    s.h = make_hdr(S.seed, 0, s.blk, s.j);
    const int64_t p = 500 + (site_lo + k) * (int64_t)S.site_stride;
    s.start = p - 139 + (i * 140) / S.depth;
    s.lib = (int32_t)(i % S.n_libs); s.region = (int32_t)k;
    return s;
}

// ------------------------------------------------------------------------------------------------
// device
// ------------------------------------------------------------------------------------------------
struct DevArgs { brc_synth_spec S; int32_t contig; int64_t blk_lo, n_reads; brc_synth_out O; unsigned long long *blk_cig; };

static_assert(RL % 2 == 0 && RL % 8 != 0 && BR == 256, "the fill writes whole quality groups and bytes of two bases");
constexpr int NG = (RL + 7) / 8;   // quality groups of 8 per read: one sub_stream word each, the fill's unit of work
constexpr int NWIN = 48;           // reference words staged per CTA: a WGS block's reads touch at most 45 (1280 + 152 bp)

// ascending sort of 256 unique keys, one per thread (key of thread t on return = rank t).  Strides below 32 exchange by
// shuffle; the six larger ones go through `xs` (256 words).
__device__ uint32_t bitonic256(uint32_t key, uint32_t *xs, int t) {
    for (int size = 2; size <= BR; size <<= 1)
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            uint32_t other;
            if (stride >= 32) { __syncthreads(); xs[t] = key; __syncthreads(); other = xs[t ^ stride]; }
            else other = __shfl_xor_sync(0xffffffffu, key, stride);
            key = (((t & stride) == 0) == ((t & size) == 0)) ? min(key, other) : max(key, other);
        }
    return key;
}

// exclusive prefix sum over the CTA (256 threads); `ws` holds 8 warp totals
__device__ uint32_t cta_exclusive_scan(uint32_t v, uint32_t *ws, int t) {
    uint32_t x = v;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if ((t & 31) >= o) x += y; }
    if ((t & 31) == 31) ws[t >> 5] = x;
    __syncthreads();
    for (int w = 0; w < (t >> 5); ++w) x += ws[w];
    return x - v;
}

// the substitutions make_body applies, as a list: entry k (bits 10k..10k+9) = position | shift << 8, the count in bits 60..63.
// Same draw and the same rule: distinct positions, first occurrence wins, and a position is remembered before the check that it
// came from the reference.  Returns NM.
__device__ int32_t sub_list(const Hdr &h, uint64_t &list) {
    int32_t nm = h.kind == 1 ? 2 : (h.kind == 2 ? 3 : 0);
    uint64_t l = 0; int n = 0;
    if (h.n_subs > 0) {
        const uint64_t h2 = sub_stream(h.rk, 2), h3 = sub_stream(h.rk, 3);
        uint64_t seen = ~0ull;
        for (int t = 0; t < 6; ++t) {
            if (t >= h.n_subs) break;
            const uint64_t src = t < 3 ? h2 >> (20 * t) : h3 >> (20 * (t - 3));
            const uint32_t p = (uint32_t)(src & 0xFFFFu) % (uint32_t)RL;
            const uint32_t sft = 1u + ((uint32_t)((src >> 16) & 0xFu) % 3u);
            bool dup = false;
            for (int k = 0; k < 6; ++k) dup = dup || ((uint32_t)(seen >> (8 * k)) & 0xFFu) == p;
            if (dup) continue;
            seen = (seen << 8) | p;
            if (ref_off(h.kind, (int)p) < 0) continue;
            l |= (uint64_t)(p | (sft << 8)) << (10 * n);
            ++n; ++nm;
        }
    }
    list = l | ((uint64_t)n << 60);
    return nm;
}

// 4 quality bytes from 4 bytes b of a quality word: {37,37,37,30,25,12,2}[(b * 7) >> 8], two bytes per 16-bit lane, one byte permute
__device__ __forceinline__ uint32_t qual4(uint32_t w) {
    const uint32_t e = (((w & 0x00FF00FFu) * 7u) >> 8) & 0x00070007u, o = ((((w >> 8) & 0x00FF00FFu) * 7u) >> 8) & 0x00070007u;
    return __byte_perm(0x1E252525u, 0x00020C19u, (e | (e >> 8) | (o << 4) | (o >> 4)) & 0x7777u);
}

// 4 packed sequence bytes from 8 base codes (2 bits each, base k at bits 2k): byte j = (1 << b[2j]) << 4 | 1 << b[2j+1]
__device__ __forceinline__ uint32_t seq4(uint32_t c) {
    uint32_t x = (c | (c << 8)) & 0x00FF00FFu;
    x = (x | (x << 4)) & 0x0F0F0F0Fu;
    x = (x | (x << 2)) & 0x33333333u;                       // base k in bits 4k, 4k+1
    const uint32_t b0 = x & 0x11111111u, b1 = (x >> 1) & 0x11111111u;
    const uint32_t nib = (~(b0 | b1) & 0x11111111u) | ((b0 & ~b1) << 1) | ((b1 & ~b0) << 2) | ((b0 & b1) << 3);
    return ((nib & 0x0F0F0F0Fu) << 4) | ((nib >> 4) & 0x0F0F0F0Fu);
}

// quality group g (query positions 8g .. 8g+7) of a read: 8 quality bytes (little-endian) and 8 base codes (2 bits each), before
// the substitutions.  The values make_body computes, position for position.
__device__ __forceinline__ void fill_group(const Hdr &h, int64_t start, int g, const uint64_t *win, int64_t w_lo,
                                           uint64_t seed, uint64_t unit, uint64_t &qual8, uint32_t &codes) {
    const int q0 = 8 * g;
    const uint64_t hq = sub_stream(h.rk, 8 + (uint64_t)g);
    uint64_t qv = (uint64_t)qual4((uint32_t)hq) | (uint64_t)qual4((uint32_t)(hq >> 32)) << 32;
    const int tail_from = RL - h.tail - q0;              // bytes k >= tail_from are the Q2 tail
    if (tail_from < 8) {
        const uint64_t m = tail_from <= 0 ? ~0ull : ~0ull << (8 * tail_from);
        qv = (qv & ~m) | (0x0202020202020202ull & m);
    }
    qual8 = qv;
    // the group's reference bases lie within 11 bp from its first one (a 3 bp deletion at most): 32 bases from there
    const int ro0 = max(ref_off(h.kind, q0), 0);
    const int64_t p0 = start + ro0, w0 = p0 >> 5;
    auto word = [&](int64_t w) { const int64_t k = w - w_lo; return (uint64_t)k < (uint64_t)NWIN ? win[k] : ref_word(seed, unit, (uint64_t)w); };
    const int s = 2 * (int)(p0 & 31);
    const uint64_t wa = word(w0);
    const uint64_t bases = s ? (wa >> s) | (word(w0 + 1) << (64 - s)) : wa;
    uint32_t c = (uint32_t)bases & 0xFFFFu;                // the group's bases are the 8 from its first one ...
    const bool clipped = (h.kind == 1 && g == 8) || (h.kind == 3 && g <= 1);
    if (clipped || (h.kind == 2 && g == 7)) {               // ... unless it holds an insertion, the clip or the deletion
        const uint64_t hb = clipped ? sub_stream(h.rk, 4) : 0;
        c = 0;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const int q = q0 + k, ro = ref_off(h.kind, q);
            const uint32_t b = ro >= 0 ? (uint32_t)(bases >> (2 * (ro - ro0))) & 3u : (uint32_t)(hb >> (2 * (q & 31))) & 3u;
            c |= b << (2 * k);
        }
    }
    codes = c;
}

__global__ void __launch_bounds__(BR) synth_count_kernel(DevArgs A) {
    __shared__ uint32_t red[BR / 32];
    const int t = threadIdx.x;
    int c = 0;
    if (A.S.mode == BRC_SYNTH_DEEP) { const Slot s = deep_slot(A.S, A.blk_lo, (int64_t)blockIdx.x * BR + t, A.n_reads); c = s.valid ? n_cigar_of(s.h.kind) : 0; }
    else c = n_cigar_of(make_hdr(A.S.seed, (uint64_t)A.contig, (uint64_t)(A.blk_lo + blockIdx.x), (uint64_t)t).kind);   // the block's total is order-free
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if ((t & 31) == 0) red[t >> 5] = (uint32_t)c;
    __syncthreads();
    if (t == 0) { uint32_t tot = 0; for (int w = 0; w < BR / 32; ++w) tot += red[w]; A.blk_cig[blockIdx.x] = tot; }
}

__global__ void __launch_bounds__(1024) synth_scan_kernel(unsigned long long *v, int64_t n) {   // exclusive scan, one CTA; v[n] = total
    __shared__ unsigned long long ws[32];
    const int t = threadIdx.x;
    const int64_t per = (n + 1023) / 1024, lo = imin64(n, per * t), hi = imin64(n, lo + per);
    unsigned long long s = 0;
    for (int64_t i = lo; i < hi; ++i) s += v[i];
    unsigned long long x = s;                            // CTA-inclusive scan of the 1024 partial sums
    for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o); if ((t & 31) >= o) x += y; }
    if ((t & 31) == 31) ws[t >> 5] = x;
    __syncthreads();
    if (t < 32) {
        unsigned long long w = ws[t];
        for (int o = 1; o < 32; o <<= 1) { const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o); if (t >= o) w += y; }
        ws[t] = w;
    }
    __syncthreads();
    unsigned long long acc = x - s + ((t >> 5) ? ws[(t >> 5) - 1] : 0ull);
    if (t == 1023) v[n] = acc + s;
    for (int64_t i = lo; i < hi; ++i) { const unsigned long long y = v[i]; v[i] = acc; acc += y; }
}

// One CTA = one block of 256 reads.  Each read's header is hashed once and kept in shared memory for the sort; after it, thread t
// owns row t: its metadata, its substitution list and its 19 quality groups, the header, start and list held in registers and the
// reference bases taken from words staged once per CTA.  The substitutions are patched into the row once, after its groups.  The
// rows are staged in shared memory and leave with 16-byte stores.
__global__ void __launch_bounds__(BR) synth_fill_kernel(DevArgs A) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t *seq_s = smem, *qual_s = smem + BR * SB;                                          // 19200 + 38400 bytes
    Hdr *hs = reinterpret_cast<Hdr *>(smem + BR * (SB + RL));                                 // headers by j (the sort's lookup)
    uint64_t *win = reinterpret_cast<uint64_t *>(hs + BR);                                    // NWIN reference words from w_lo
    uint32_t *xs = reinterpret_cast<uint32_t *>(win + NWIN);                                  // sort exchange / scan totals
    __shared__ int64_t w_lo_s;
    const int t = threadIdx.x;
    const int64_t b = blockIdx.x, i = b * BR + t;
    const bool deep = A.S.mode == BRC_SYNTH_DEEP;
    const uint64_t seed = A.S.seed, unit = deep ? 0 : (uint64_t)A.contig;
    const int64_t block = A.blk_lo + b;
    Slot s;
    if (deep) {
        s = deep_slot(A.S, A.blk_lo, i, A.n_reads);
        if (t == 0) w_lo_s = s.start >> 5;                            // the CTA's first read starts leftmost
        __syncthreads();
    } else {
        if (t < NWIN) win[t] = ref_word(seed, unit, (uint64_t)((block * BBP >> 5) + t));   // every start is >= block * BBP
        const Hdr h = make_hdr(seed, unit, (uint64_t)block, (uint64_t)t);
        hs[t] = h;
        const uint32_t key = bitonic256(((uint32_t)(wgs_start(A.S, block, h.off) - block * BBP + BRC_SYNTH_MAX_SPAN) << 8) | (uint32_t)t, xs, t);
        __syncthreads();
        s.valid = true; s.unit = unit; s.blk = (uint64_t)block; s.j = key & 255u;     // (start, j): unique, so any sort gives this order
        s.h = hs[s.j];
        s.start = wgs_start(A.S, block, s.h.off);
        s.lib = (int32_t)((block * BR + t) % A.S.n_libs); s.region = 0;
    }
    const int64_t w_lo = deep ? w_lo_s : block * BBP >> 5;
    if (deep && t < NWIN) win[t] = ref_word(seed, unit, (uint64_t)(w_lo + t));
    // block-exclusive scan of the CIGAR op counts
    const int nc = s.valid ? n_cigar_of(s.h.kind) : 0;
    const unsigned long long coff = A.blk_cig[b] + cta_exclusive_scan((uint32_t)nc, xs, t);   // its barrier: every header read by j
    const brc_synth_out &O = A.O;
    uint64_t subs = 0;
    if (s.valid) {
        const int32_t nm = sub_list(s.h, subs);
        if (O.tid) O.tid[i] = A.contig;
        O.pos[i] = (int32_t)s.start; O.flag[i] = (uint16_t)(s.h.reverse ? 16 : 0); O.mapq[i] = (uint8_t)s.h.mapq; O.lib[i] = (uint16_t)s.lib;
        O.l_qseq[i] = RL; O.nm[i] = nm; O.sm[i] = TAG_ABSENT;
        O.cigar_off[i] = coff; O.seq_off[i] = (uint64_t)i * SB; O.qual_off[i] = (uint64_t)i * RL;
        uint32_t c[3]; cigar_of(s.h.kind, c);
        for (int k = 0; k < nc; ++k) O.cigar[coff + k] = c[k];
        if (O.region_of_read) O.region_of_read[i] = s.region;
        if (i == A.n_reads - 1) { O.cigar_off[i + 1] = coff + nc; O.seq_off[i + 1] = (uint64_t)(i + 1) * SB; O.qual_off[i + 1] = (uint64_t)(i + 1) * RL; }
    }
    // bases and qualities: thread t builds row t (its own read) group by group, then patches in the read's substitutions
    const int rows = (int)imin64(BR, A.n_reads - b * BR);
    if (t < rows) {
        uint16_t *qd = reinterpret_cast<uint16_t *>(qual_s + t * RL);                          // rows and groups start at even bytes
        uint8_t *sd = seq_s + t * SB;
#pragma unroll 2
        for (int g = 0; g < NG; ++g) {
            uint64_t qv; uint32_t codes;
            fill_group(s.h, s.start, g, win, w_lo, seed, unit, qv, codes);
            const int nq = g == NG - 1 ? RL - 8 * (NG - 1) : 8;
            const uint32_t sq = seq4(codes);
            for (int k = 0; k < nq / 2; ++k) {
                qd[4 * g + k] = (uint16_t)(qv >> (16 * k));
                sd[4 * g + k] = (uint8_t)(sq >> (8 * k));
            }
        }
        // distinct positions: each substitution shifts the base the group left there
        for (int k = 0; k < (int)(subs >> 60); ++k) {
            const uint32_t e = (uint32_t)(subs >> (10 * k)), p = e & 0xFFu;
            const uint32_t byte = sd[p >> 1], sh = (p & 1u) ? 0u : 4u;
            const uint32_t code = __ffs((byte >> sh) & 15u) - 1;
            sd[p >> 1] = (uint8_t)((byte & ~(15u << sh)) | (1u << ((code + ((e >> 8) & 3u)) & 3u)) << sh);
        }
    }
    __syncthreads();
    // coalesced copy of the staged rows (the CTA's rows are contiguous in the pools; 256 rows start 16-byte aligned)
    {
        const int64_t nb = rows * SB; uint8_t *dst = O.seq + b * BR * SB;
        for (int64_t k = t; k < nb / 16; k += BR) reinterpret_cast<int4 *>(dst)[k] = reinterpret_cast<const int4 *>(seq_s)[k];
        for (int64_t k = (nb / 16) * 16 + t; k < nb; k += BR) dst[k] = seq_s[k];
    }
    {
        const int64_t nb = rows * RL; uint8_t *dst = O.qual + b * BR * RL;
        for (int64_t k = t; k < nb / 16; k += BR) reinterpret_cast<int4 *>(dst)[k] = reinterpret_cast<const int4 *>(qual_s)[k];
        for (int64_t k = (nb / 16) * 16 + t; k < nb; k += BR) dst[k] = qual_s[k];
    }
}

__global__ void synth_ref_kernel(brc_synth_spec S, int32_t contig, int64_t beg, int64_t len, char *out) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < len) out[i] = "ACGT"[ref_base(S.seed, (uint64_t)contig, beg + i)];
}

// Checksum of a byte string = sum over its 16-byte groups g of (lo64 ^ rotl(hi64, 29) + 1) * (2 g + 1)  (mod 2^64; a short last
// group is zero-padded).  One 16-byte load and a handful of integer instructions per group: the emitter stand-in has to read
// every received byte, not to compete with the pileup kernel for issue slots (the round-2 word-wise mix64 cost rank 0 ~16 % of a
// pileup launch per round at 4 GPUs).  Position-weighted, so a misplaced or truncated message changes it.
__device__ __forceinline__ unsigned long long cs_term(unsigned long long lo, unsigned long long hi, int64_t g) {
    return ((lo ^ ((hi << 29) | (hi >> 35))) + 1ull) * (2ull * (unsigned long long)g + 1ull);
}
__global__ void checksum_kernel(const uint32_t *w, int64_t n_words, int aligned16, unsigned long long *acc) {
    unsigned long long s = 0;
    const int64_t n_groups = (n_words + 3) / 4, n_full = n_words / 4;
    const int64_t t0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, step = (int64_t)gridDim.x * blockDim.x;
    if (aligned16) {
        const uint4 *v = reinterpret_cast<const uint4 *>(w);
        for (int64_t g = t0; g < n_full; g += step) {
            const uint4 x = v[g];
            s += cs_term((unsigned long long)x.x | ((unsigned long long)x.y << 32), (unsigned long long)x.z | ((unsigned long long)x.w << 32), g);
        }
    } else {
        for (int64_t g = t0; g < n_full; g += step)
            s += cs_term((unsigned long long)w[4 * g] | ((unsigned long long)w[4 * g + 1] << 32),
                         (unsigned long long)w[4 * g + 2] | ((unsigned long long)w[4 * g + 3] << 32), g);
    }
    if (t0 == 0 && n_groups > n_full) {          // zero-padded last group
        uint32_t x[4] = {0u, 0u, 0u, 0u};
        for (int64_t k = 4 * n_full; k < n_words; ++k) x[k - 4 * n_full] = w[k];
        s += cs_term((unsigned long long)x[0] | ((unsigned long long)x[1] << 32), (unsigned long long)x[2] | ((unsigned long long)x[3] << 32), n_full);
    }
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    __shared__ unsigned long long red[32];
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long tot = 0; for (int k = 0; k < (int)(blockDim.x >> 5); ++k) tot += red[k]; atomicAdd(acc, tot); }
}

int check_spec(const brc_synth_spec *S, int32_t contig, int64_t lo, int64_t hi) {
    if (!S || lo < 0 || hi < lo || S->n_libs <= 0) return BRC_E_INVALID;
    if (S->mode == BRC_SYNTH_WGS) { if (S->contig_len < BBP || S->contig_len % BBP || hi > S->contig_len / BBP || contig < 0) return BRC_E_INVALID; }
    else if (S->mode == BRC_SYNTH_DEEP) { if (S->depth <= 0 || S->site_stride < 300) return BRC_E_INVALID; }
    else return BRC_E_INVALID;
    return BRC_OK;
}

}  // namespace

extern "C" {

int64_t brc_synth_window_reads(const brc_synth_spec *S, int64_t lo, int64_t hi) {
    if (!S || hi < lo) return 0;
    return S->mode == BRC_SYNTH_DEEP ? (hi - lo) * (int64_t)S->depth : (hi - lo) * BR;
}

int brc_synth_ref_host(const brc_synth_spec *S, int32_t contig, int64_t beg, int64_t len, char *out) {
    if (!S || !out || beg < 0 || len < 0) return BRC_E_INVALID;
    unsigned hw = std::thread::hardware_concurrency();
    const int nt = (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)(hw ? hw : 1), (int64_t)32, len / 1000000 + 1}));
    auto work = [&](int t) {
        const int64_t a = len * t / nt, b = len * (t + 1) / nt;
        for (int64_t i = a; i < b; ++i) out[i] = "ACGT"[ref_base(S->seed, (uint64_t)contig, beg + i)];
    };
    std::vector<std::thread> th;
    for (int t = 1; t < nt; ++t) th.emplace_back(work, t);
    work(0);
    for (auto &x : th) x.join();
    return BRC_OK;
}

int brc_synth_ref_device(const brc_synth_spec *S, int32_t contig, int64_t beg, int64_t len, char *out_dev, void *stream) {
    if (!S || !out_dev || beg < 0 || len < 0) return BRC_E_INVALID;
    if (len == 0) return BRC_OK;
    synth_ref_kernel<<<(unsigned)((len + 255) / 256), 256, 0, (cudaStream_t)stream>>>(*S, contig, beg, len, out_dev);
    return cudaGetLastError() == cudaSuccess ? BRC_OK : BRC_E_CUDA;
}

int brc_synth_fill_host(const brc_synth_spec *S, int32_t contig, int64_t lo, int64_t hi, const brc_synth_out *O, int n_threads) {
    int rc = check_spec(S, contig, lo, hi);
    if (rc != BRC_OK || !O) return rc != BRC_OK ? rc : BRC_E_INVALID;
    const int64_t n = brc_synth_window_reads(S, lo, hi);
    if (O->n_reads != n) return BRC_E_INVALID;
    const int64_t nblk = (n + BR - 1) / BR;
    std::vector<uint64_t> blk_cig((size_t)nblk + 1, 0);
    const int nt = (int)std::max<int64_t>(1, std::min<int64_t>(n_threads > 0 ? n_threads : 1, nblk));
    const uint64_t unit = S->mode == BRC_SYNTH_DEEP ? 0 : (uint64_t)contig;
    // the slots of CTA-block b, file order
    auto block_slots = [&](int64_t b, Slot *sl) {
        if (S->mode == BRC_SYNTH_DEEP) { for (int t = 0; t < BR; ++t) sl[t] = deep_slot(*S, lo, b * BR + t, n); return; }
        const int64_t block = lo + b;
        uint32_t keys[BR];
        for (int t = 0; t < BR; ++t) {
            const Hdr h = make_hdr(S->seed, unit, (uint64_t)block, (uint64_t)t);
            keys[t] = ((uint32_t)(wgs_start(*S, block, h.off) - block * BBP + BRC_SYNTH_MAX_SPAN) << 8) | (uint32_t)t;
        }
        std::sort(keys, keys + BR);
        for (int t = 0; t < BR; ++t) {
            Slot &s = sl[t]; s.valid = true; s.unit = unit; s.blk = (uint64_t)block; s.j = keys[t] & 255u;
            s.h = make_hdr(S->seed, unit, s.blk, s.j); s.start = wgs_start(*S, block, s.h.off);
            s.lib = (int32_t)((block * BR + t) % S->n_libs); s.region = 0;
        }
    };
    auto run = [&](int pass) {
        auto work = [&](int w) {
            std::vector<Slot> sl(BR);
            for (int64_t b = nblk * w / nt; b < nblk * (w + 1) / nt; ++b) {
                block_slots(b, sl.data());
                uint64_t coff = blk_cig[(size_t)b];
                uint64_t cnt = 0;
                for (int t = 0; t < BR; ++t) {
                    const Slot &s = sl[t];
                    if (!s.valid) continue;
                    const int nc = n_cigar_of(s.h.kind);
                    if (pass == 0) { cnt += (uint64_t)nc; continue; }
                    const int64_t i = b * BR + t;
                    const int32_t nm = make_body(S->seed, unit, s.h, s.start, O->seq + i * SB, O->qual + i * RL);
                    if (O->tid) O->tid[i] = contig;
                    O->pos[i] = (int32_t)s.start; O->flag[i] = (uint16_t)(s.h.reverse ? 16 : 0); O->mapq[i] = (uint8_t)s.h.mapq; O->lib[i] = (uint16_t)s.lib;
                    O->l_qseq[i] = RL; O->nm[i] = nm; O->sm[i] = TAG_ABSENT;
                    O->cigar_off[i] = coff; O->seq_off[i] = (uint64_t)i * SB; O->qual_off[i] = (uint64_t)i * RL;
                    uint32_t c[3]; cigar_of(s.h.kind, c);
                    for (int k = 0; k < nc; ++k) O->cigar[coff + k] = c[k];
                    coff += (uint64_t)nc;
                    if (O->region_of_read) O->region_of_read[i] = s.region;
                    if (i == n - 1) { O->cigar_off[n] = coff; O->seq_off[n] = (uint64_t)n * SB; O->qual_off[n] = (uint64_t)n * RL; }
                }
                if (pass == 0) blk_cig[(size_t)b] = cnt;
            }
        };
        std::vector<std::thread> th;
        for (int w = 1; w < nt; ++w) th.emplace_back(work, w);
        work(0);
        for (auto &x : th) x.join();
    };
    run(0);
    { uint64_t acc = 0; for (int64_t b = 0; b < nblk; ++b) { const uint64_t x = blk_cig[(size_t)b]; blk_cig[(size_t)b] = acc; acc += x; } blk_cig[(size_t)nblk] = acc; }
    if (n == 0) { O->cigar_off[0] = 0; O->seq_off[0] = 0; O->qual_off[0] = 0; return BRC_OK; }
    run(1);
    return BRC_OK;
}

int brc_synth_fill_device(const brc_synth_spec *S, int32_t contig, int64_t lo, int64_t hi, const brc_synth_out *O, void *scratch_dev, void *stream) {
    int rc = check_spec(S, contig, lo, hi);
    if (rc != BRC_OK || !O || !scratch_dev) return rc != BRC_OK ? rc : BRC_E_INVALID;
    const int64_t n = brc_synth_window_reads(S, lo, hi);
    if (O->n_reads != n) return BRC_E_INVALID;
    if (n == 0) return BRC_OK;
    const int64_t nblk = (n + BR - 1) / BR;
    const int smem = BR * (SB + RL) + BR * (int)sizeof(Hdr) + NWIN * (int)sizeof(uint64_t) + BR * 4;
    if (cudaFuncSetAttribute(synth_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess) return BRC_E_CUDA;
    DevArgs A; A.S = *S; A.contig = contig; A.blk_lo = lo; A.n_reads = n; A.O = *O; A.blk_cig = reinterpret_cast<unsigned long long *>(scratch_dev);
    cudaStream_t s = (cudaStream_t)stream;
    synth_count_kernel<<<(unsigned)nblk, BR, 0, s>>>(A);
    synth_scan_kernel<<<1, 1024, 0, s>>>(A.blk_cig, nblk);
    synth_fill_kernel<<<(unsigned)nblk, BR, smem, s>>>(A);
    return cudaGetLastError() == cudaSuccess ? BRC_OK : BRC_E_CUDA;
}

// SAM text of a window (header + records; RG:Z:rg<lib>, LB:lib<lib>) for `samtools view -b`: the same bytes the host fill
// produces, so the reference binary / the CLI read exactly the window the device path computes.
int brc_synth_write_sam(const brc_synth_spec *S, int32_t contig, int64_t lo, int64_t hi, const char *path, const char *contig_name,
                        int64_t declared_len, int n_threads) {
    if (!S || !path || !contig_name) return BRC_E_INVALID;
    const int64_t n = brc_synth_window_reads(S, lo, hi);
    std::vector<int32_t> pos((size_t)n), l_qseq((size_t)n), nm((size_t)n), sm((size_t)n);
    std::vector<uint16_t> flag((size_t)n), lib((size_t)n);
    std::vector<uint8_t> mapq((size_t)n), seq((size_t)n * SB + 64), qual((size_t)n * RL + 64);
    std::vector<uint64_t> co((size_t)n + 1), so((size_t)n + 1), qo((size_t)n + 1);
    std::vector<uint32_t> cig((size_t)n * 3 + 16);
    brc_synth_out O{};
    O.n_reads = n; O.tid = nullptr; O.pos = pos.data(); O.flag = flag.data(); O.mapq = mapq.data(); O.lib = lib.data(); O.l_qseq = l_qseq.data();
    O.nm = nm.data(); O.sm = sm.data(); O.cigar_off = co.data(); O.cigar = cig.data(); O.seq_off = so.data(); O.seq = seq.data();
    O.qual_off = qo.data(); O.qual = qual.data(); O.region_of_read = nullptr;
    int rc = brc_synth_fill_host(S, contig, lo, hi, &O, n_threads);
    if (rc != BRC_OK) return rc;
    FILE *fh = std::fopen(path, "w");
    if (!fh) return BRC_E_INVALID;
    std::fprintf(fh, "@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:%s\tLN:%lld\n", contig_name, (long long)declared_len);
    for (int i = 0; i < S->n_libs; ++i) std::fprintf(fh, "@RG\tID:rg%d\tSM:s\tLB:lib%d\n", i, i);
    const char *ops = "MIDNSHP=XB";
    std::string line;
    char tmp[64];
    const int64_t base_index = S->mode == BRC_SYNTH_DEEP ? lo * (int64_t)S->depth : lo * BR;
    for (int64_t i = 0; i < n; ++i) {
        line.clear();
        std::snprintf(tmp, sizeof tmp, "r%lld\t%u\t", (long long)(base_index + i), (unsigned)flag[(size_t)i]); line += tmp;
        line += contig_name;
        std::snprintf(tmp, sizeof tmp, "\t%d\t%u\t", pos[(size_t)i] + 1, (unsigned)mapq[(size_t)i]); line += tmp;
        for (uint64_t k = co[(size_t)i]; k < co[(size_t)i + 1]; ++k) { std::snprintf(tmp, sizeof tmp, "%u%c", cig[k] >> 4, ops[cig[k] & 15]); line += tmp; }
        line += "\t*\t0\t0\t";
        const uint8_t *sq = seq.data() + so[(size_t)i];
        for (int q = 0; q < RL; ++q) line += brc::seq_nt16_str[brc::seq_nib(sq, 0, q)];
        line += '\t';
        const uint8_t *ql = qual.data() + qo[(size_t)i];
        for (int q = 0; q < RL; ++q) line += (char)(ql[q] + 33);
        std::snprintf(tmp, sizeof tmp, "\tNM:i:%d\tRG:Z:rg%u\n", nm[(size_t)i], (unsigned)lib[(size_t)i]); line += tmp;
        std::fwrite(line.data(), 1, line.size(), fh);
    }
    std::fclose(fh);
    return BRC_OK;
}

int brc_synth_checksum_device(const void *buf_dev, int64_t n_bytes, unsigned long long *acc_dev, void *stream) {
    if (!buf_dev || !acc_dev || n_bytes < 0 || (n_bytes & 3)) return BRC_E_INVALID;
    if (n_bytes == 0) return BRC_OK;
    const int64_t n = n_bytes / 4;
    const unsigned grid = (unsigned)std::min<int64_t>(132 * 2, (n / 4 + 255) / 256 + 1);       // 2 CTAs per SM: a reader, not a tenant
    checksum_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const uint32_t *>(buf_dev), n, ((uintptr_t)buf_dev & 15) == 0 ? 1 : 0, acc_dev);
    return cudaGetLastError() == cudaSuccess ? BRC_OK : BRC_E_CUDA;
}

}  // extern "C"
