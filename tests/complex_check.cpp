// complex_check.cpp — the flank walk of the complex-record kernel (brc_complex.cuh resolve_flanks), compiled for the CPU.
// Each line of STDIN is "pos left right n_cigar w1 .. wn" (BAM CIGAR words); each line of STDOUT the two flank query positions,
// or "-1 -1" when the read does not span.  tests/test_vcf_complex_cli.py compares it with tests/complex_rule.py's resolve.
#include <cstdio>
#include <vector>

#include "brc_complex.cuh"

int main() {
    long long pos, left, right; unsigned n;
    while (std::scanf("%lld %lld %lld %u", &pos, &left, &right, &n) == 4) {
        std::vector<uint32_t> cig(n);
        for (unsigned k = 0; k < n; ++k) if (std::scanf("%u", &cig[k]) != 1) return 1;
        const brc::Flanks f = brc::resolve_flanks(cig.data(), n, pos, left, right);
        std::printf("%d %d\n", f.ql, f.ql < 0 ? -1 : f.qr);
    }
    return 0;
}
