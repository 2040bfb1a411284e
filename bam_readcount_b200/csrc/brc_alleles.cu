// brc_alleles.cu — allele queries on the device (brc_set_allele_queries, DESIGN.md §12).
//
// Runs on the launch stream after the pileup kernels, over the packed records they left in HBM, and answers each query with
// the 13 accumulators of one entry of one printed line, the line's depth and whether the line is printed:
//   allele_record_kernel  one thread per secondary-pool record: the depth terms of the pool (pool_depth_term), then the queries
//                         whose entry the record is (binary search of its slot among the queries sorted by `match`): base
//                         classes and escaped primaries by class, deletions by length, insertions by length and bases
//   allele_query_kernel   one thread per query: the line and its depth (site_line), the primary held in the packed words, and
//                         all zeros for a site that prints no line
#include "brc_device.cuh"

namespace brc {
namespace {

constexpr int ALLELE_CTA = 256;

// the record's inserted bases (read bases qpos+1 .. qpos+len, as the text prints them) equal the query's
__device__ __forceinline__ bool same_insertion(const AlleleParams &P, const SecRec &rec, const AlleleQuery &Q) {
    const uint64_t off = P.seq_off[rec.read];
    const int len = (int)(rec.kind_len >> 8);
    for (int k = 1; k <= len; ++k)
        if (canonical16(seq_nib(P.seq, off, rec.qpos + k)) != P.bases[Q.bases_off + k - 1]) return false;
    return true;
}

__global__ void __launch_bounds__(ALLELE_CTA) allele_record_kernel(AlleleParams P) {
    const int64_t j = (int64_t)blockIdx.x * ALLELE_CTA + threadIdx.x;
    const int64_t n_rec = (int64_t)*P.sec_count < P.sec_cap ? (int64_t)*P.sec_count : P.sec_cap;
    if (j >= n_rec) return;
    const SecRec &rec = P.sec[j];
    pool_depth_term(P.words, P.n_rows, P.n_slots, rec, P.dsum, P.esc_np);
    const uint32_t kind = rec.kind_len & 0xFFu;
    // the key the record answers: an escaped primary is its base class (none when the site has no passing base)
    const uint32_t key = kind >= KIND_WIDE ? kind - KIND_WIDE : rec.kind_len;
    if (kind >= KIND_WIDE && key >= 6u) return;
    int64_t lo = 0, hi = P.n_q;
    while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (P.q[m].match < rec.slot) lo = m + 1; else hi = m; }
    for (; lo < P.n_q && P.q[lo].match == rec.slot; ++lo) {
        const AlleleQuery &Q = P.q[lo];
        if (Q.kind_len != key || (kind == (uint32_t)KIND_INS && !same_insertion(P, rec, Q))) continue;
        brc_allele_answer &A = P.ans[Q.out];
        for (int k = 0; k < N_STATS; ++k) A.stats[k] = rec.stats[k];
    }
}

__global__ void __launch_bounds__(ALLELE_CTA) allele_query_kernel(AlleleParams P) {
    const int64_t i = (int64_t)blockIdx.x * ALLELE_CTA + threadIdx.x;
    if (i >= P.n_q) return;
    const AlleleQuery Q = P.q[i];
    brc_allele_answer &A = P.ans[Q.out];
    const SiteLine L = Q.site == NO_SLOT ? SiteLine{0, false, false, false}
                                         : site_line(P.words, P.n_rows, P.n_slots, Q.site, Q.left != 0u, P.dsum, P.esc_np);
    if (!L.live) {                           // no line, so no entry: whatever the record pass found does not print
        for (int k = 0; k < N_STATS; ++k) A.stats[k] = 0u;
        A.depth = 0u; A.line = 0u;
        return;
    }
    A.depth = (uint32_t)L.depth; A.line = 1u;
    const uint32_t kind = Q.kind_len & 0xFFu;
    const int64_t NS = P.n_slots, s = Q.site;
    const uint32_t w1 = P.words[NS + s];
    if (kind >= 6u || (w1 & 7u) != kind) return;   // not the primary held in the words (pool records came from the record pass)
    unpack_primary(P.words, NS, s, A.stats);   // one library row: RS = NS
}

}  // namespace

cudaError_t launch_alleles(const AlleleParams &P, cudaStream_t st) {
    const unsigned gp = (unsigned)((P.sec_cap + ALLELE_CTA - 1) / ALLELE_CTA), gq = (unsigned)((P.n_q + ALLELE_CTA - 1) / ALLELE_CTA);
    if (gp) allele_record_kernel<<<gp, ALLELE_CTA, 0, st>>>(P);
    if (gq) allele_query_kernel<<<gq, ALLELE_CTA, 0, st>>>(P);
    return cudaGetLastError();
}

}  // namespace brc
