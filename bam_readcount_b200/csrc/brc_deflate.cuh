// brc_deflate.cuh — the serial pieces of the BGZF encoder (brc_deflate.cu), host+device code, as brc_bgzf.cuh is for the
// decoder: the Huffman code-length builder with its 15-bit limit, canonical codes, the dynamic-header writer (code lengths
// run-length coded as RFC 1951 §3.2.7), the fixed and stored encodings, DEFLATE's length/distance symbols, CRC32 and its
// combine, and the BGZF member framing htslib writes.  The kernel runs them on one thread of a CTA (or, for the bit sink,
// on every thread); tests/deflate_check.cpp runs the same code on the CPU against zlib.
//
// No piece keeps an array of its own on the stack: every table lives in a caller-supplied scratch area, which is shared
// memory in the kernel (so the kernel has no stack frame).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define BRC_DHD __host__ __device__ __forceinline__
#else
#define BRC_DHD inline
#endif

namespace brc {
namespace deflate {

constexpr int BLOCK = 65280;           // input bytes per BGZF member (htslib's BGZF_BLOCK_SIZE, the cut bgzip makes)
constexpr int MAX_MEMBER = 65536;      // a member's largest size
constexpr int HDR = 18, TRAILER = 8;   // gzip header with the BC subfield; CRC32 + ISIZE
constexpr int LCODES = 286, DCODES = 30, BLCODES = 19, MAXBITS = 15, MAXBLBITS = 7;
constexpr int MIN_MATCH = 3, MAX_MATCH = 258, WINDOW = 32768;
enum Mode { STORED = 0, FIXED = 1, DYNAMIC = 2 };

// The 28-byte empty member that ends every BGZF file.
// (A fixed-Huffman block holding only the end-of-block code, CRC32 0, ISIZE 0.)
BRC_DHD uint8_t eof_byte(int i) {
    const uint64_t w = i < 8 ? 0x00000000004088b1full : i < 16 ? 0x000243420006ff00ull : i < 24 ? 0x000000000003001bull : 0;
    return (uint8_t)(w >> (8 * (i & 7)));
}

BRC_DHD int ilog2(uint32_t x) {
#if defined(__CUDA_ARCH__)
    return 31 - __clz(x);
#else
    return 31 - __builtin_clz(x);
#endif
}
BRC_DHD uint32_t rev(uint32_t v, int n) {
#if defined(__CUDA_ARCH__)
    return __brev(v) >> (32 - n);
#else
    uint32_t r = 0;
    for (int i = 0; i < n; ++i) { r = (r << 1) | (v & 1u); v >>= 1; }
    return r;
#endif
}

// ---- LSB-first bit sink over zero-initialised 32-bit words; every word is OR-ed in (atomically on the device), so many
// writers may fill one buffer, each at its own bit offset, and a word shared by two of them takes both halves.
struct Sink { uint32_t *w; uint64_t wi; uint64_t acc; int cnt; };
BRC_DHD void or_word(uint32_t *p, uint32_t v) {
    if (!v) return;
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
}
BRC_DHD void sink_init(Sink &s, uint32_t *w, uint64_t bitpos) { s.w = w; s.wi = bitpos >> 5; s.cnt = (int)(bitpos & 31); s.acc = 0; }
BRC_DHD uint64_t sink_pos(const Sink &s) { return (s.wi << 5) + (uint64_t)s.cnt; }
BRC_DHD void sink_put(Sink &s, uint32_t v, int n) {          // n <= 32; v has no bits at or above n
    s.acc |= (uint64_t)v << s.cnt;
    s.cnt += n;
    if (s.cnt >= 32) { or_word(s.w + s.wi, (uint32_t)s.acc); ++s.wi; s.acc >>= 32; s.cnt -= 32; }
}
BRC_DHD void sink_flush(Sink &s) { if (s.cnt > 0) or_word(s.w + s.wi, (uint32_t)s.acc); }
BRC_DHD void sink_align(Sink &s) { const int pad = (8 - (s.cnt & 7)) & 7; if (pad) sink_put(s, 0, pad); }

// ---- DEFLATE symbols of a match (RFC 1951 §3.2.5) ----
BRC_DHD int len_sym(int len, int &ebits, int &eval) {        // 3 <= len <= 258
    if (len == MAX_MATCH) { ebits = 0; eval = 0; return 285; }
    const int x = len - 3;
    if (x < 8) { ebits = 0; eval = 0; return 257 + x; }
    const int e = ilog2((uint32_t)x) - 2;
    ebits = e; eval = x & ((1 << e) - 1);
    return 257 + 4 * (e + 1) + ((x >> e) - 4);
}
BRC_DHD int dist_sym(int dist, int &ebits, int &eval) {      // 1 <= dist <= 32768
    const int y = dist - 1;
    if (y < 4) { ebits = 0; eval = 0; return y; }
    const int e = ilog2((uint32_t)y) - 1;
    ebits = e; eval = y & ((1 << e) - 1);
    return 2 * (e + 1) + ((y >> e) - 2);
}
BRC_DHD int len_extra(int sym) { return (sym < 265 || sym == 285) ? 0 : (sym - 261) / 4; }   // extra bits of a length symbol
BRC_DHD int dist_extra(int sym) { return sym < 4 ? 0 : sym / 2 - 1; }

// ---- Huffman code lengths ----
// Scratch of the code-length builder: sort keys, their in-place tree, and the count of codes per length.
struct LenWork { uint32_t key[LCODES]; uint32_t a[LCODES]; uint32_t blc[MAXBITS + 1]; };

// Minimum-redundancy code lengths of A[0..m), sorted ascending, computed in place (Moffat and Katajainen, 1995).
BRC_DHD void min_redundancy(uint32_t *A, int m) {
    A[0] += A[1];
    int root = 0, leaf = 2;
    for (int next = 1; next < m - 1; ++next) {
        if (leaf >= m || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = (uint32_t)next; }
        else A[next] = A[leaf++];
        if (leaf >= m || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = (uint32_t)next; }
        else A[next] += A[leaf++];
    }
    A[m - 2] = 0;
    for (int next = m - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
    int avail = 1, used = 0, depth = 0, root2 = m - 2, next = m - 1;
    while (avail > 0) {
        while (root2 >= 0 && (int)A[root2] == depth) { ++used; --root2; }
        while (avail > used) { A[next--] = (uint32_t)depth; --avail; }
        avail = 2 * used; ++depth; used = 0;
    }
}

// Code lengths of n (<= 286) symbols of frequencies freq, none longer than maxbits.  No symbol used: all 0.  One: length 1.
// Two or more: a complete code (Kraft sum exactly 1).  Ties are broken by symbol number, so the result depends on freq alone.
BRC_DHD void build_lengths(const uint32_t *freq, int n, int maxbits, uint8_t *len, LenWork &W) {
    int m = 0;
    for (int s = 0; s < n; ++s) { len[s] = 0; if (freq[s]) W.key[m++] = freq[s] << 9 | (uint32_t)s; }
    if (m == 0) return;
    if (m == 1) { len[W.key[0] & 511u] = 1; return; }
    int gap = 1;
    while (gap < m / 3) gap = 3 * gap + 1;
    for (; gap > 0; gap /= 3)                                // shell sort, ascending (frequency, symbol)
        for (int i = gap; i < m; ++i) {
            const uint32_t v = W.key[i];
            int j = i;
            for (; j >= gap && W.key[j - gap] > v; j -= gap) W.key[j] = W.key[j - gap];
            W.key[j] = v;
        }
    for (int i = 0; i < m; ++i) W.a[i] = W.key[i] >> 9;
    min_redundancy(W.a, m);
    for (int b = 0; b <= maxbits; ++b) W.blc[b] = 0;
    for (int i = 0; i < m; ++i) W.blc[W.a[i] < (uint32_t)maxbits ? W.a[i] : (uint32_t)maxbits]++;
    // codes folded into maxbits over-fill the code space: move leaves down one level until the Kraft sum is 1 again
    uint32_t total = 0;
    for (int b = maxbits; b > 0; --b) total += W.blc[b] << (maxbits - b);
    while (total != (1u << maxbits)) {
        W.blc[maxbits]--;
        for (int b = maxbits - 1; b > 0; --b)
            if (W.blc[b]) { W.blc[b]--; W.blc[b + 1] += 2; break; }
        --total;
    }
    // the longest codes go to the least frequent symbols
    int j = 0;
    for (int b = maxbits; b > 0; --b)
        for (uint32_t k = 0; k < W.blc[b]; ++k) len[W.key[j++] & 511u] = (uint8_t)b;
}

// Canonical codes (RFC 1951 §3.2.2), bit-reversed for LSB-first output.  next: MAXBITS + 1 words of scratch.
BRC_DHD void canonical(const uint8_t *len, int n, uint16_t *code, uint32_t *next) {
    for (int b = 0; b <= MAXBITS; ++b) next[b] = 0;
    for (int s = 0; s < n; ++s) if (len[s]) next[len[s]]++;
    uint32_t c = 0, prev = 0;
    for (int b = 1; b <= MAXBITS; ++b) { const uint32_t cnt = next[b]; c = (c + prev) << 1; next[b] = c; prev = cnt; }
    for (int s = 0; s < n; ++s) code[s] = len[s] ? (uint16_t)rev(next[len[s]]++, len[s]) : 0;
}

// The codes a block is written with: literal/length and distance.
struct Codes { uint16_t lcode[288]; uint8_t llen[288]; uint16_t dcode[32]; uint8_t dlen[32]; };

BRC_DHD void fixed_codes(Codes &C, uint32_t *next) {
    for (int s = 0; s < 288; ++s) C.llen[s] = s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8;
    for (int s = 0; s < 32; ++s) C.dlen[s] = 5;
    canonical(C.llen, 288, C.lcode, next);
    canonical(C.dlen, 32, C.dcode, next);
}

// ---- dynamic header (RFC 1951 §3.2.7) ----
// The order the code-length code lengths are sent in (16 17 18 0 8 7 9 6 10 5 11 4 12 3 13 2 14 1 15), five bits per entry
BRC_DHD int cl_order(int i) { return (int)((i < 12 ? 0x022caa324e804a30ull >> (5 * i) : 0x3c2e1346cull >> (5 * (i - 12))) & 31u); }

struct DynHeader {
    uint8_t sym[LCODES + DCODES], ext[LCODES + DCODES];     // the run-length coded code lengths
    uint8_t cl_len[BLCODES]; uint16_t cl_code[BLCODES];
    uint32_t cl_freq[BLCODES];
    int n, hlit, hdist, hclen;
    uint32_t bits;                                          // HLIT .. the last code length, without the 3 block-type bits
};

// The header of the code C.llen[0..286) / C.dlen[0..30): its run-length code, its code-length code and its size in bits.
// The lengths form one sequence, so a run may cross from the literal/length lengths into the distance lengths.
BRC_DHD void dyn_header(const Codes &C, DynHeader &H, LenWork &W) {
    int hlit = LCODES; while (hlit > 257 && C.llen[hlit - 1] == 0) --hlit;
    int hdist = DCODES; while (hdist > 1 && C.dlen[hdist - 1] == 0) --hdist;
    H.hlit = hlit; H.hdist = hdist;
    const int total = hlit + hdist;
    auto at = [&](int i) -> int { return i < hlit ? C.llen[i] : C.dlen[i - hlit]; };
    int n = 0;
    for (int i = 0; i < total;) {
        const int v = at(i);
        int run = 1;
        while (i + run < total && at(i + run) == v) ++run;
        i += run;
        if (v == 0) {
            while (run >= 11) { const int r = run < 138 ? run : 138; H.sym[n] = 18; H.ext[n++] = (uint8_t)(r - 11); run -= r; }
            if (run >= 3) { H.sym[n] = 17; H.ext[n++] = (uint8_t)(run - 3); run = 0; }
        } else {
            H.sym[n] = (uint8_t)v; H.ext[n++] = 0; --run;
            while (run >= 3) { const int r = run < 6 ? run : 6; H.sym[n] = 16; H.ext[n++] = (uint8_t)(r - 3); run -= r; }
        }
        while (run-- > 0) { H.sym[n] = (uint8_t)v; H.ext[n++] = 0; }
    }
    H.n = n;
    for (int s = 0; s < BLCODES; ++s) H.cl_freq[s] = 0;
    for (int k = 0; k < n; ++k) H.cl_freq[H.sym[k]]++;
    build_lengths(H.cl_freq, BLCODES, MAXBLBITS, H.cl_len, W);
    int used = 0, one = 0;
    for (int s = 0; s < BLCODES; ++s) if (H.cl_len[s]) { ++used; one = s; }
    if (used == 1) H.cl_len[one == 0 ? 1 : 0] = 1;          // zlib refuses an incomplete code-length code: complete it
    canonical(H.cl_len, BLCODES, H.cl_code, W.blc);
    int hclen = BLCODES; while (hclen > 4 && H.cl_len[cl_order(hclen - 1)] == 0) --hclen;
    H.hclen = hclen;
    uint32_t bits = 5 + 5 + 4 + 3 * (uint32_t)hclen;
    for (int k = 0; k < n; ++k) bits += H.cl_len[H.sym[k]] + (H.sym[k] == 16 ? 2 : H.sym[k] == 17 ? 3 : H.sym[k] == 18 ? 7 : 0);
    H.bits = bits;
}

BRC_DHD void put_dyn_header(Sink &s, const DynHeader &H) {
    sink_put(s, (uint32_t)(H.hlit - 257), 5);
    sink_put(s, (uint32_t)(H.hdist - 1), 5);
    sink_put(s, (uint32_t)(H.hclen - 4), 4);
    for (int i = 0; i < H.hclen; ++i) sink_put(s, H.cl_len[cl_order(i)], 3);
    for (int k = 0; k < H.n; ++k) {
        const int y = H.sym[k];
        sink_put(s, H.cl_code[y], H.cl_len[y]);
        if (y >= 16) sink_put(s, H.ext[k], y == 16 ? 2 : y == 17 ? 3 : 7);
    }
}

// Bits of the payload under code C, from the symbol histogram (literal/length lf[286] with EOB, distance df[30]).
BRC_DHD uint64_t payload_bits(const Codes &C, const uint32_t *lf, const uint32_t *df) {
    uint64_t b = 0;
    for (int s = 0; s < LCODES; ++s) b += (uint64_t)lf[s] * (uint32_t)(C.llen[s] + (s > 256 ? len_extra(s) : 0));
    for (int s = 0; s < DCODES; ++s) b += (uint64_t)df[s] * (uint32_t)(C.dlen[s] + dist_extra(s));
    return b;
}

BRC_DHD uint32_t literal_bits(const Codes &C, int byte) { return C.llen[byte]; }
BRC_DHD uint32_t match_bits(const Codes &C, int len, int dist) {
    int le, lv, de, dv;
    const int ls = len_sym(len, le, lv), ds = dist_sym(dist, de, dv);
    return (uint32_t)(C.llen[ls] + le + C.dlen[ds] + de);
}
BRC_DHD void put_literal(Sink &s, const Codes &C, int byte) { sink_put(s, C.lcode[byte], C.llen[byte]); }
BRC_DHD void put_match(Sink &s, const Codes &C, int len, int dist) {
    int le, lv, de, dv;
    const int ls = len_sym(len, le, lv), ds = dist_sym(dist, de, dv);
    sink_put(s, C.lcode[ls], C.llen[ls]);
    if (le) sink_put(s, (uint32_t)lv, le);
    sink_put(s, C.dcode[ds], C.dlen[ds]);
    if (de) sink_put(s, (uint32_t)dv, de);
}
BRC_DHD void put_eob(Sink &s, const Codes &C) { sink_put(s, C.lcode[256], C.llen[256]); }

// A stored block (BFINAL set) of n <= 65535 bytes: 3 header bits, padding to the byte, LEN, NLEN.  Returns nothing: the
// n bytes follow at the next byte.
BRC_DHD void put_stored_header(Sink &s, int n) {
    sink_put(s, 1, 3);
    sink_align(s);
    sink_put(s, (uint32_t)n, 16);
    sink_put(s, (uint32_t)(~n & 0xffff), 16);
}
constexpr int STORED_OVERHEAD = 5;

// ---- CRC32 (the gzip polynomial, reflected) ----
BRC_DHD uint32_t crc_table_entry(uint32_t i) {
    uint32_t c = i;
    for (int k = 0; k < 8; ++k) c = (c & 1u) ? (c >> 1) ^ 0xEDB88320u : c >> 1;
    return c;
}
BRC_DHD uint32_t crc_update(const uint32_t *T, uint32_t crc, const uint8_t *p, int64_t n) {
    crc = ~crc;
    for (int64_t i = 0; i < n; ++i) crc = T[(crc ^ p[i]) & 255u] ^ (crc >> 8);
    return ~crc;
}
// a * b modulo the CRC polynomial, both in the reflected representation (bit 31 is x^0)
BRC_DHD uint32_t gf2_mul(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (uint32_t m = 1u << 31; m; m >>= 1) {
        if (a & m) p ^= b;
        b = (b & 1u) ? (b >> 1) ^ 0xEDB88320u : b >> 1;
    }
    return p;
}
// crc * x^(8 n): the CRC of a message moved n zero bytes further from the end.  The factors x^(8 * 2^k) are formed by
// squaring as the bits of n are taken, so any n costs at most 2 * 64 products.
BRC_DHD uint32_t crc_shift(uint32_t crc, uint64_t n) {
    uint32_t f = 1u << 23;                                   // x^8
    while (n) {
        if (n & 1u) crc = gf2_mul(crc, f);
        f = gf2_mul(f, f);
        n >>= 1;
    }
    return crc;
}
// CRC32 of A followed by B from CRC32(A), CRC32(B) and |B|.  CRC32(A B C ...) is the XOR of every part's CRC shifted by
// the bytes after it, which is how the kernel combines its per-thread segments.
BRC_DHD uint32_t crc_combine(uint32_t crc_a, uint32_t crc_b, uint64_t len_b) { return crc_shift(crc_a, len_b) ^ crc_b; }

// ---- BGZF member (htslib's layout): gzip header with FEXTRA and the BC subfield holding BSIZE = member length - 1;
// the raw DEFLATE stream; CRC32 and ISIZE.
BRC_DHD void put_member_header(Sink &s, uint32_t member_len) {
    const uint32_t bsize = member_len - 1;
    sink_put(s, 0x04088b1fu, 32);                            // ID1 ID2 CM=8 FLG=FEXTRA
    sink_put(s, 0, 32);                                      // MTIME
    sink_put(s, 0xff00u, 16);                                // XFL=0 OS=255
    sink_put(s, 6, 16);                                      // XLEN
    sink_put(s, 0x00024342u, 32);                            // 'B' 'C' SLEN=2
    sink_put(s, bsize, 16);
}
BRC_DHD void put_member_trailer(Sink &s, uint32_t crc, uint32_t isize) { sink_put(s, crc, 32); sink_put(s, isize, 32); }

}  // namespace deflate
}  // namespace brc
