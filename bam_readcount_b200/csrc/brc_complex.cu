// brc_complex.cu — complex-record queries on the device (brc_set_complex_queries, DESIGN.md §12 "MNP and complex records").
//
// Runs on the launch stream after the allele kernels, over what K0 left in HBM: the read descriptors and the per-tile read
// ranges.  One warp per query, one lane per read: the candidates are the reads of the K0 tile range of the tile holding the
// span's first base (a read spanning both flanks covers it), taken 32 at a time.  A lane drops its read when it is FM_DEAD,
// does not reach both flanks, or has a base of quality below -b between them; otherwise its allele string S (the read bases
// between the flanks, brc_complex.cuh) is compared with the query's alleles, lengths first.  The totals per allele and strand
// are ballots and popcounts: no atomics, and the answers are written once, by the lane that owns each allele.
#include "brc_complex.cuh"
#include "brc_device.cuh"

namespace brc {
namespace {

constexpr int COMPLEX_CTA = 256;       // 8 queries per CTA

__global__ void __launch_bounds__(COMPLEX_CTA) complex_query_kernel(ComplexParams P) {
    const int lane = threadIdx.x & 31;
    const int64_t qi = (int64_t)blockIdx.x * (COMPLEX_CTA / 32) + (threadIdx.x >> 5);
    if (qi >= P.n_q) return;                                       // uniform per warp
    const ComplexQuery Q = P.q[qi];
    const int64_t left = (int64_t)Q.pos - 1, right = (int64_t)Q.pos + Q.ref_len;
    const int64_t lo = Q.tile >= 0 ? (int64_t)P.tile_lo[Q.tile] : 0, hi = Q.tile >= 0 ? (int64_t)P.tile_hi[Q.tile] : 0;
    uint32_t depth = 0;
    // alleles in groups of 32: lane j keeps the totals of allele g0 + j (a record with more than 32 alleles walks its reads again)
    for (int g0 = 0; g0 < Q.n_alleles; g0 += 32) {
        const int ng = min(32, Q.n_alleles - g0);
        uint32_t cnt = 0, plus = 0;
        for (int64_t base = lo; base < hi; base += 32) {
            const int64_t r = base + lane;
            bool counted = false, fwd = false;
            int32_t ql = -1, len = 0;
            uint64_t soff = 0;
            if (r < hi) {
                const ReadDesc &d = P.desc[r];
                const uint32_t fm = d.fm;
                if (!(fm & FM_DEAD) && (int64_t)d.pos <= left && (int64_t)d.end > right) {
                    if (fm & FM_SIMPLE) { ql = (int32_t)(left - d.pos) + (int32_t)d.cig; len = Q.ref_len; }   // d.cig: qoff
                    else {
                        const Flanks f = resolve_flanks(P.cigar + P.cigar_off[r], d.n_cigar, d.pos, left, right);
                        ql = f.ql; len = f.qr - f.ql - 1;
                    }
                }
                if (ql >= 0) {
                    counted = true;
                    const uint8_t *qual = P.qual + P.qual_off[r] + ql + 1;
                    for (int k = 0; k < len && counted; ++k) counted = (int)qual[k] >= P.min_bq;
                    fwd = !(fm & 16u);
                    soff = P.seq_off[r];
                }
            }
            const unsigned m_dp = __ballot_sync(0xffffffffu, counted), m_fwd = __ballot_sync(0xffffffffu, counted && fwd);
            depth += (uint32_t)__popc(m_dp);
            if (!m_dp) continue;
            for (int j = 0; j < ng; ++j) {
                const brc_complex_allele A = P.alleles[Q.allele0 + g0 + j];
                bool same = counted && len == A.len;
                for (int k = 0; same && k < len; ++k) same = canonical16(seq_nib(P.seq, soff, ql + 1 + k)) == P.bases[A.bases_off + k];
                const unsigned m = __ballot_sync(0xffffffffu, same);
                if (lane == j) { cnt += (uint32_t)__popc(m); plus += (uint32_t)__popc(m & m_fwd); }
            }
        }
        if (lane < ng) P.counts[Q.allele0 + g0 + lane] = brc_complex_count{cnt, plus};
        if (g0 + 32 < Q.n_alleles) depth = 0;                      // the next group counts the same reads again
    }
    if (lane == 0) P.depth[qi] = depth;
}

}  // namespace

cudaError_t launch_complex(const ComplexParams &P, cudaStream_t st) {
    const int64_t per = COMPLEX_CTA / 32;
    const unsigned g = (unsigned)((P.n_q + per - 1) / per);
    if (g) complex_query_kernel<<<g, COMPLEX_CTA, 0, st>>>(P);
    return cudaGetLastError();
}

}  // namespace brc
