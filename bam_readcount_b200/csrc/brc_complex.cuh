// brc_complex.cuh — the flank walk of a complex-record query (brc_set_complex_queries, DESIGN.md §12 "MNP and complex
// records"), shared by the device kernel of brc_complex.cu and its host twin.
//
// A read spans a record whose span is reference positions [p, p + n) when both flanks, p - 1 and p + n, are aligned to read
// bases by a match-type op (M, = or X).  Its allele string is then the read bases strictly between the two flank query
// positions: inserted bases anywhere between them included, deleted and skipped reference positions contributing nothing.  A
// flank in a deletion or a skip, or outside the aligned ops (in a soft clip, before the read's start or past its end), means
// the read does not span.  On the host the same function compiles with g++, so the walk the kernel runs is tested on the CPU
// against the Python rule (tests/complex_check.cpp).
#pragma once
#include <cstdint>

#include "brc_seq.cuh"

namespace brc {

struct Flanks { int32_t ql, qr; };     // query positions of the left and right flank; ql = -1: the read does not span

// cig: the read's n_cigar BAM CIGAR words (op in bits [0:4), length in [4:32)); pos: its leftmost reference position;
// left = p - 1, right = p + n (left < right).
BRC_SEQ_HD Flanks resolve_flanks(const uint32_t *cig, uint32_t n_cigar, int64_t pos, int64_t left, int64_t right) {
    Flanks f{-1, -1};
    int64_t rp = pos;
    int64_t qp = 0;
    int32_t ql = -1;
    for (uint32_t k = 0; k < n_cigar; ++k) {
        const uint32_t c = cig[k], op = c & 0xFu;
        const int64_t len = (int64_t)(c >> 4);
        if (cigar_is_match(op)) {                           // M = X: reference and query advance together
            if (ql < 0 && left >= rp && left < rp + len) ql = (int32_t)(qp + (left - rp));
            if (right >= rp && right < rp + len) {
                if (ql >= 0) { f.ql = ql; f.qr = (int32_t)(qp + (right - rp)); }
                return f;
            }
            rp += len; qp += len;
        } else if (op == 1u || op == 4u) {                   // I S: query only
            qp += len;
        } else if (op == 2u || op == 3u) {                   // D N: reference only
            if (ql < 0 && left >= rp && left < rp + len) return f;      // the left flank is not aligned to a read base
            if (right >= rp && right < rp + len) return f;
            rp += len;
        }                                                    // H P B: neither
        if (rp > right) return f;
    }
    return f;
}

}  // namespace brc
