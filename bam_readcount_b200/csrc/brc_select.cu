// brc_select.cu — the alternative-allele site filter on the device (brc_set_site_filter, DESIGN.md §10).
//
// Runs on the launch stream after the pileup kernels, over the packed records they left in HBM, and leaves behind only what
// the text emitter needs for the lines that pass the filter:
//   sel_pool_kernel    one thread per secondary-pool record: largest alternative count per site, the depth and largest count a
//                      site's deletions add to the next site's line, the npass of escaped primaries
//   sel_site_kernel    one thread per site: depth, largest alternative count, the rule; keep bits
//   sel_flag_kernel    one thread per site: the emit byte (1 passes; 2 keep-all range, or the last live site of an argv region
//                      that a library row covers); shipped = emit byte set, or the left neighbour of a site with one (the
//                      emitter replays its deletion pushes, so the line and its depth are whole)
//   scan (brc_scan.cuh, three kernels): compact index of every shipped site
//   sel_gather_sites_kernel / sel_gather_sec_kernel: the shipped sites' ids, emit bytes, packed words and pool records, the
//                      records' slot rewritten to row * n_sel + compact index
#include <algorithm>

#include "brc_device.cuh"
#include "brc_scan.cuh"

namespace brc {
namespace {

constexpr int SEL_CTA = 256;
constexpr int SEL_LAST_ROWS = 32;    // library rows whose last live site sel_site_kernel collects in shared memory first
static_assert(SELECT_SCAN_CTA == scan::SCAN_CTA, "partial sums are sized by SELECT_SCAN_CTA");

__device__ __forceinline__ int64_t region_of(const SelectParams &P, int64_t s) {   // last region with slot_base <= s
    int64_t lo = 0, hi = P.n_regions;
    while (hi - lo > 1) { const int64_t m = (lo + hi) >> 1; if (P.regions[m].slot_base <= s) lo = m; else hi = m; }
    return lo;
}

// seq_nt16 code of the reference at `pos`; 15 (N) outside the window or when the emitter has no characters for the contig: the
// code of the reference column the text prints
__device__ __forceinline__ uint32_t ref_code(const SelectParams &P, const SelRegion &R, int64_t pos) {
    if (!R.ref_on_host) return 15u;
    const RefWin w = P.refs[R.tid_slot];
    const int64_t i = pos - w.win_beg;
    if (i < 0 || i >= w.win_len || pos >= w.chrom_len) return 15u;
    const uint32_t b = (uint8_t)w.seq[i >> 1];
    return (i & 1) ? (b & 15u) : (b >> 4);
}

__device__ __forceinline__ uint64_t umax(uint64_t a, uint64_t b) { return a > b ? a : b; }

__device__ __forceinline__ bool row_covers(const SelectParams &P, int64_t idx) {
    const int64_t RS = (int64_t)P.n_rows * P.n_slots;
    return (P.words[RS + idx] & 7u) == PB_ESCAPE || (P.words[idx] & 0xFFu) != 0u;
}

__device__ __forceinline__ bool abandoned(const SelectParams &P, int64_t s) {
    const int64_t RS = (int64_t)P.n_rows * P.n_slots;
    bool ab = false;
    for (int r = 0; r < P.n_rows; ++r) ab |= (P.words[RS + (int64_t)r * P.n_slots + s] & 8u) != 0u;
    return ab;
}

__global__ void __launch_bounds__(SEL_CTA) sel_pool_kernel(SelectParams P) {
    const int64_t j = (int64_t)blockIdx.x * SEL_CTA + threadIdx.x;
    const int64_t n_rec = (int64_t)*P.sec_count < P.sec_cap ? (int64_t)*P.sec_count : P.sec_cap;
    if (j >= n_rec) return;
    const SecRec &rec = P.sec[j];
    const int64_t slot = rec.slot, r = slot / P.n_slots, s = slot - r * P.n_slots;
    const uint32_t kind = rec.kind_len & 0xFFu, cnt = rec.stats[0];
    if (kind == (uint32_t)KIND_DEL) {
        // pushed here, printed in the same row's block of the next site when that row spans it (same region: sel_site_kernel)
        if (s + 1 < P.n_slots && row_covers(P, r * P.n_slots + s + 1)) { atomicAdd(&P.dsum[s], cnt); atomicMax(&P.dbest[s], cnt); }
        return;
    }
    if (kind == (uint32_t)KIND_INS) { atomicMax(&P.best[s], cnt); return; }
    const uint32_t bc = kind >= KIND_WIDE ? kind - KIND_WIDE : kind;
    if (kind >= KIND_WIDE) atomicAdd(&P.esc_np[s], (uint32_t)rec.qpos);
    if (bc >= 1u && bc <= 4u && cnt > 0u) {
        const SelRegion R = P.regions[region_of(P, s)];
        if (base_is_alt(bc, ref_code(P, R, R.first_pos + (s - R.slot_base)))) atomicMax(&P.best[s], cnt);
    }
}

__global__ void __launch_bounds__(SEL_CTA) sel_site_kernel(SelectParams P) {
    __shared__ int64_t s_g0;
    __shared__ unsigned int s_last[SEL_LAST_ROWS];
    const int64_t s = (int64_t)blockIdx.x * SEL_CTA + threadIdx.x;
    const bool in = s < P.n_slots;
    const int64_t g = in ? region_of(P, s) : -1;
    if (threadIdx.x == 0) s_g0 = g;
    if (threadIdx.x < SEL_LAST_ROWS) s_last[threadIdx.x] = 0u;
    __syncthreads();
    bool ab = false, live = false;
    if (in) {
        const SelRegion R = P.regions[g];
        const int64_t o = s - R.slot_base, pos = R.first_pos + o;
        const int64_t NS = P.n_slots, RS = (int64_t)P.n_rows * NS;
        const uint32_t rc = ref_code(P, R, pos);
        bool covered = false;
        uint64_t depth = P.esc_np[s], best = P.best[s];
        for (int r = 0; r < P.n_rows; ++r) {
            const uint32_t w0 = P.words[(int64_t)r * NS + s], w1 = P.words[RS + (int64_t)r * NS + s], pc = w1 & 7u;
            ab |= (w1 & 8u) != 0u;
            if (pc == PB_ESCAPE) { covered = true; continue; }      // full-width primary: a pool record
            covered |= (w0 & 0xFFu) != 0u;
            depth += (w0 >> 8) & 0xFFu;
            if (base_is_alt(pc, rc)) best = umax(best, (w0 >> 16) & 0xFFu);
        }
        if (o > 0 && !abandoned(P, s - 1)) { depth += P.dsum[s - 1]; best = umax(best, P.dbest[s - 1]); }
        live = covered && !ab;
        uint8_t k = 0;
        if (live) {
            k = 4;
            if (pos >= R.beg && pos < R.end && site_passes(best, depth, P.min_alt_count, P.min_alt_fraction)) k |= 1;
            if (o < R.keep_all_n) k |= 2;
            // argv region: per library row, the last live site the row covers.  The emitter drops a row's queued deletions only
            // at a line where the row has reads; shipping that site makes the queue a region hands on the unfiltered one.
            if (R.argv)
                for (int r = 0; r < P.n_rows; ++r) {
                    const int64_t idx = (int64_t)r * NS + s;
                    if ((P.words[RS + idx] & 7u) != PB_ESCAPE && (P.words[idx] & 0xFFu) == 0u) continue;
                    if (g == s_g0 && r < SEL_LAST_ROWS) atomicMax(&s_last[r], (unsigned int)(o + 1));
                    else atomicMax(&P.reg_last[g * P.n_rows + r], (uint32_t)(o + 1));
                }
        }
        P.keep[s] = k;
    }
    const unsigned nab = __popc(__ballot_sync(0xffffffffu, ab));
    if ((threadIdx.x & 31) == 0 && nab) atomicAdd(&P.counters[1], (unsigned long long)nab);
    __syncthreads();
    if (threadIdx.x < SEL_LAST_ROWS && threadIdx.x < P.n_rows && s_last[threadIdx.x])
        atomicMax(&P.reg_last[s_g0 * P.n_rows + threadIdx.x], s_last[threadIdx.x]);
}

// emit byte of site s (offset o in region g): 1 the line passes; 2 the emitter forms the line and decides (keep-all range, or
// the last live site of an argv region that some library row covers); 0 none
__device__ __forceinline__ uint8_t emit_byte(const SelectParams &P, int64_t g, const SelRegion &R, int64_t o, int64_t s) {
    const uint8_t k = P.keep[s];
    if (k & 1) return 1;
    if (!(k & 4)) return 0;
    if (k & 2) return 2;
    if (R.argv)
        for (int r = 0; r < P.n_rows; ++r)
            if (P.reg_last[g * P.n_rows + r] == (uint32_t)(o + 1)) return 2;
    return 0;
}

__global__ void __launch_bounds__(SEL_CTA) sel_flag_kernel(SelectParams P) {
    const int64_t s = (int64_t)blockIdx.x * SEL_CTA + threadIdx.x;
    if (s >= P.n_slots) return;
    const int64_t g = region_of(P, s);
    const SelRegion R = P.regions[g];
    const int64_t o = s - R.slot_base;
    const uint8_t em = emit_byte(P, g, R, o, s);
    const bool context = (P.keep[s] & 4) && o + 1 < R.n_slots && emit_byte(P, g, R, o + 1, s + 1) != 0;
    P.emit[s] = em;
    P.ship[s] = (em || context) ? 1u : 0u;
}

__global__ void __launch_bounds__(SEL_CTA) sel_gather_sites_kernel(SelectParams P) {
    const int64_t s = (int64_t)blockIdx.x * SEL_CTA + threadIdx.x;
    if (s >= P.n_slots || !P.ship[s]) return;
    const int64_t NS = P.n_slots, n = (int64_t)P.idx[NS], i = (int64_t)P.idx[s];
    P.c_site[i] = (uint32_t)s;
    P.c_emit[i] = P.emit[s];
    for (int w = 0; w < N_WORDS; ++w)
        for (int r = 0; r < P.n_rows; ++r)
            P.c_words[((int64_t)w * P.n_rows + r) * n + i] = P.words[((int64_t)w * P.n_rows + r) * NS + s];
}

__global__ void __launch_bounds__(SEL_CTA) sel_gather_sec_kernel(SelectParams P) {
    const int64_t j = (int64_t)blockIdx.x * SEL_CTA + threadIdx.x;
    const int64_t n_rec = (int64_t)*P.sec_count < P.sec_cap ? (int64_t)*P.sec_count : P.sec_cap;
    if (j >= n_rec) return;
    SecRec rec = P.sec[j];
    const int64_t NS = P.n_slots, r = (int64_t)rec.slot / NS, s = (int64_t)rec.slot - r * NS;
    if (!P.ship[s]) return;
    const unsigned long long k = atomicAdd(&P.counters[0], 1ull);
    rec.slot = (uint32_t)(r * (int64_t)P.idx[NS] + (int64_t)P.idx[s]);
    rec.next = -1;
    P.c_sec[k] = rec;
}

}  // namespace

cudaError_t launch_select(const SelectParams &P, cudaStream_t st) {
    const int64_t NS = P.n_slots;
    if (NS <= 0) return cudaGetLastError();
    const unsigned gs = (unsigned)((NS + SEL_CTA - 1) / SEL_CTA), gp = (unsigned)std::max<int64_t>(1, (P.sec_cap + SEL_CTA - 1) / SEL_CTA);
    sel_pool_kernel<<<gp, SEL_CTA, 0, st>>>(P);
    sel_site_kernel<<<gs, SEL_CTA, 0, st>>>(P);
    sel_flag_kernel<<<gs, SEL_CTA, 0, st>>>(P);
    scan::scan_partial_kernel<<<dim3((unsigned)P.nb, 1), scan::SCAN_CTA, 0, st>>>(P.ship, NS, P.partial, P.nb);
    scan::scan_top_kernel<<<1, 1024, 0, st>>>(P.partial, P.nb);
    scan::scan_apply_kernel<<<dim3((unsigned)P.nb, 1), scan::SCAN_CTA, 0, st>>>(P.ship, NS, P.partial, P.nb, P.idx, nullptr, nullptr);
    sel_gather_sites_kernel<<<gs, SEL_CTA, 0, st>>>(P);
    sel_gather_sec_kernel<<<gp, SEL_CTA, 0, st>>>(P);
    return cudaGetLastError();
}

}  // namespace brc
