// seq_check.cpp — the base-code and CIGAR rules of brc_seq.cuh against the oracle's own C definitions (oracle/brc_oracle.c,
// whose helpers are static, so it is compiled into this program).
//   seq_check tables   seq_nt16_table for all 256 bytes, canonical16 and canonical_nt for all 16 codes, seq_nib at both nibble
//                      phases: one line "ok <checks>", or one line per mismatch and exit status 1
//   seq_check span     each line of STDIN is "flag pos n_cigar w1 .. wn" (BAM CIGAR words); each line of STDOUT the oracle's
//                      read_endpos, bam_endpos from cigar_span (pos + 1 for an unmapped read or one without CIGAR), and
//                      cigar_span's I/D op count.  tests/test_seq_rules.py runs both.
#include <cstdio>
#include <cstring>
#include <vector>

#include "brc_seq.cuh"
#include "../oracle/brc_oracle.c"

static int tables() {
    int checks = 0, bad = 0;
    for (int c = 0; c < 256; ++c, ++checks)
        if (brc::seq_nt16_table[c] != seq_nt16((unsigned char)c)) { std::printf("seq_nt16_table[%d] = %d, oracle %d\n", c, brc::seq_nt16_table[c], seq_nt16((unsigned char)c)); ++bad; }
    for (uint32_t nib = 0; nib < 16; ++nib, checks += 3) {
        if (brc::canonical16(nib) != canonical16[nib]) { std::printf("canonical16(%u) = %u, oracle %d\n", nib, brc::canonical16(nib), canonical16[nib]); ++bad; }
        if (brc::canonical_nt[brc::canonical16(nib)] != canonical_nt[canonical16[nib]]) { std::printf("canonical_nt of %u\n", nib); ++bad; }
        if (brc::seq_nt16_table[(unsigned char)brc::seq_nt16_str[nib]] != nib) { std::printf("seq_nt16_str[%u] = %c\n", nib, brc::seq_nt16_str[nib]); ++bad; }
    }
    if (std::strcmp(brc::canonical_nt, canonical_nt) != 0) { std::printf("canonical_nt \"%s\", oracle \"%s\"\n", brc::canonical_nt, canonical_nt); ++bad; }
    for (int b = 0; b < 256; ++b) {
        const uint8_t packed[2] = {(uint8_t)b, (uint8_t)(255 - b)};
        for (int i = 0; i < 4; ++i, ++checks)
            if (brc::seq_nib(packed, 0, i) != (uint32_t)seqi(packed, i)) { std::printf("seq_nib byte %d base %d\n", b, i); ++bad; }
    }
    if (bad) return 1;
    std::printf("ok %d\n", checks);
    return 0;
}

static int spans() {
    int flag; int pos; unsigned n;
    while (std::scanf("%d %d %u", &flag, &pos, &n) == 3) {
        std::vector<uint32_t> cig(n + 1);
        for (unsigned k = 0; k < n; ++k) if (std::scanf("%u", &cig[k]) != 1) return 1;
        const uint16_t fl = (uint16_t)flag;
        const uint64_t off[2] = {0, n};
        orc_reads R;
        std::memset(&R, 0, sizeof R);
        R.n_reads = 1; R.pos = &pos; R.flag = &fl; R.cigar_off = off; R.cigar = cig.data();
        const brc::CigarSpan s = brc::cigar_span(cig.data(), n);
        const long long end = !(fl & 4) && n > 0 ? (long long)pos + s.rlen : (long long)pos + 1;
        std::printf("%lld %lld %lld\n", (long long)read_endpos(&R, 0), end, (long long)s.n_indel);
    }
    return 0;
}

int main(int argc, char **argv) {
    if (argc == 2 && std::strcmp(argv[1], "tables") == 0) return tables();
    if (argc == 2 && std::strcmp(argv[1], "span") == 0) return spans();
    std::fprintf(stderr, "usage: seq_check tables|span\n");
    return 2;
}
