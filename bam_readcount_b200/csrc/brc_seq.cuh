// brc_seq.cuh — htslib's base-code and CIGAR rules: one definition for the kernels, the engine host, the text emitter and
// brc-readcount.  Plain C++ under g++ (brc-readcount, tests/seq_check.cpp), __host__ __device__ under nvcc.
//
//   seq_nt16_table   V:htslib-1.10/hts.c:73-91: ASCII -> 4-bit code (an index into seq_nt16_str), either case; the digits
//                    '0'..'3' are 1/2/4/8 as in htslib 1.10; 15 (N) for anything else
//   canonical16      bam_nt16_canonical_table (R:bamreadcount.cpp:36-39): 4-bit code -> index into "=ACGTN"
//   cigar_span       bam_cigar2rlen (V:htslib-1.10/sam.c:497-505): the reference length of a CIGAR (M, D, N, = and X)
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define BRC_SEQ_HD __host__ __device__ __forceinline__
#else
#define BRC_SEQ_HD inline
#endif

namespace brc {

// The initializer of seq_nt16_table and of the device's __constant__ copy (brc_kernels.cu c_nt16).
#define BRC_SEQ_NT16_TABLE { \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
     1,  2,  4,  8, 15, 15, 15, 15, 15, 15, 15, 15, 15,  0, 15, 15, \
    15,  1, 14,  2, 13, 15, 15,  4, 11, 15, 15, 12, 15,  3, 15, 15, \
    15, 15,  5,  6,  8, 15,  7,  9, 15, 10, 15, 15, 15, 15, 15, 15, \
    15,  1, 14,  2, 13, 15, 15,  4, 11, 15, 15, 12, 15,  3, 15, 15, \
    15, 15,  5,  6,  8, 15,  7,  9, 15, 10, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, \
    15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15, 15 }
constexpr uint8_t seq_nt16_table[256] = BRC_SEQ_NT16_TABLE;
constexpr char seq_nt16_str[] = "=ACMGRSVTWYHKDBN";
constexpr char canonical_nt[] = "=ACGTN";

BRC_SEQ_HD uint32_t canonical16(uint32_t nib) {
    // packed 16 x 4-bit LUT: {0,1,2,5,3,5,5,5,4,5,5,5,5,5,5,5}
    return (0x5555555455535210ull >> (nib * 4)) & 0xFu;
}
// 4-bit code of read base i of the packed bases starting at seq[off] (BAM packing: first base in the high nibble)
BRC_SEQ_HD uint32_t seq_nib(const uint8_t *seq, uint64_t off, int i) {
    uint32_t b = seq[off + (uint32_t)(i >> 1)];
    return (i & 1) ? (b & 0xFu) : (b >> 4);
}

// CIGAR op codes (BAM_C*): M 0, I 1, D 2, N 3, S 4, H 5, P 6, = 7, X 8
BRC_SEQ_HD bool cigar_consumes_ref(uint32_t op) { return op == 0 || op == 2 || op == 3 || op == 7 || op == 8; }   // M D N = X
BRC_SEQ_HD bool cigar_is_match(uint32_t op) { return op == 0 || op == 7 || op == 8; }                               // M = X

// The reference length of n CIGAR words, and n_indel plus the number of their I and D ops (a caller that sums the I/D ops of
// many reads passes its running total, which then stays in a register across its loop).  bam_endpos is pos + rlen, or pos + 1
// for a read without CIGAR or an unmapped one: each caller applies that rule itself.
struct CigarSpan { int64_t rlen, n_indel; };
BRC_SEQ_HD CigarSpan cigar_span(const uint32_t *cig, uint64_t n, int64_t n_indel = 0) {
    CigarSpan s{0, n_indel};
    for (uint64_t k = 0; k < n; ++k) {
        const uint32_t op = cig[k] & 0xFu;
        if (cigar_consumes_ref(op)) s.rlen += cig[k] >> 4;
        if (op == 1 || op == 2) ++s.n_indel;
    }
    return s;
}

}  // namespace brc
