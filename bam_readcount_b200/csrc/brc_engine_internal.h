// brc_engine_internal.h — host-side engine state shared by brc_engine.cu and brc_format.cpp.
#pragma once
#include <algorithm>
#include <cstdint>
#include <deque>
#include <queue>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/brc_engine.h"
#include "brc_device.cuh"
#include "brc_reads.h"

namespace brc {

struct DevBuf {   // grow-only device allocation
    void *p = nullptr; size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) { cudaFree(p); p = nullptr; cap = 0; }
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};
struct PinBuf {   // grow-only pinned host allocation
    void *p = nullptr; size_t cap = 0;
    cudaError_t reserve(size_t bytes) {
        if (bytes <= cap) return cudaSuccess;
        if (p) { cudaFreeHost(p); p = nullptr; cap = 0; }
        size_t want = bytes + bytes / 8 + 256;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
    template <class T> T *as() const { return reinterpret_cast<T *>(p); }
};

struct HostRef {
    int32_t tid = -1;
    std::string name;
    int64_t chrom_len = 0, win_beg = 0, win_len = 0;
    std::string seq;       // host copy (deletion alleles, reference base column)
    DevBuf dev;            // device copy
};

struct HostReads : ReadArrays {   // staging SoA of admitted reads, all regions, file order, and the region of each
    std::vector<int32_t> region;
    void clear() { ReadArrays::clear(); region.clear(); }
};

// pileup-buffer admission state of the open region (bam_plp_push, V:htslib-1.10/sam.c:4484-4531)
struct Admission {
    int32_t it_tid = 0; int64_t it_pos = 0;        // iterator position (calloc'd to 0, V:sam.c:4154)
    int32_t max_tid = -1; int64_t max_pos = -1;
    std::priority_queue<int64_t, std::vector<int64_t>, std::greater<int64_t>> live_ends;
    void reset() { it_tid = 0; it_pos = 0; max_tid = -1; max_pos = -1; live_ends = decltype(live_ends)(); }
};

// IndelQueue state of the text emitter (R:src/lib/bamrc/IndelQueue.cpp:3-15): per library row, the deletions waiting for the
// line of the site after their anchor.  The argv-region loop of the reference never clears it (R:bamreadcount.cpp:650-656).
struct QEnt { int32_t tid; int64_t pos; uint32_t st[BRC_N_STATS]; std::string allele; };
struct EmitState {
    std::vector<std::deque<QEnt>> q;
    std::vector<char> q_exists;
    EmitState() {}
    explicit EmitState(int rows) : q((size_t)rows), q_exists((size_t)rows, 0) {}
    void clear() { for (auto &d : q) d.clear(); std::fill(q_exists.begin(), q_exists.end(), 0); }
    bool pending() const { for (auto &d : q) if (!d.empty()) return true; return false; }
};

}  // namespace brc

struct brc_engine {
    brc_config cfg{};
    int n_rows = 1;
    cudaStream_t stream = nullptr;
    cudaStream_t s_in = nullptr, s_out = nullptr, s_sec = nullptr;   // copy streams of the pipelined push path (reads in, words out, pool records out)
    std::vector<cudaEvent_t> pipe_ev;
    int64_t h2d_bytes_last = 0;      // bytes the last push path actually sent over PCIe (after the elision below)
    int skip_h2d = 0;                // borrowed batch: bit0 seq_off, bit1 qual_off arithmetic; bit2 l_qseq, bit3 sm constant -> rebuilt on the device
    cudaEvent_t ev[7] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};   // see brc_last_stage_ms
    std::string err;

    std::vector<brc::HostRef> refs;
    brc::DevBuf d_refs;              // RefWin table

    // push path.  `reads` = engine-owned staging copy; `borrowed` = zero-copy view of the caller's batch
    // (one fully-admitted brc_push_reads per brc_reset): H2D copies then run straight from the caller's buffers.
    brc::HostReads reads;
    bool is_borrowed = false;
    brc_read_batch borrowed{};
    int64_t n_host_reads() const { return is_borrowed ? borrowed.n_reads : reads.n(); }
    brc_read_batch host_batch() const { return is_borrowed ? borrowed : reads.batch(); }
    std::vector<brc_region> regions;
    bool region_open = false;
    brc::Admission adm;
    int64_t open_max_end = 0;
    int64_t n_indel_ops = 0;

    // geometry (push path or plan_device)
    std::vector<brc::TileInfo> tiles;
    std::vector<int32_t> deep_tiles;   // tiles of <= DEEP_MAX_SITES sites in regions with many reads: candidates of the deep-site kernel
    int32_t deep_min_reads = 2048;     // a candidate tile with at least this many reads in its window takes the deep-site kernel
    std::vector<brc::RegionDev> regions_dev;
    int64_t n_slots = 0;
    int64_t sec_cap = 0;
    bool planned = false;

    // device buffers
    brc::DevBuf d_in[14];            // uploaded read arrays (push path)
    brc::DevBuf d_desc, d_tiles, d_tile_lo, d_tile_hi, d_regions, d_deep_tiles;
    brc::DevBuf d_words;             // packed per-site records [N_WORDS][rows*slots]
    brc::DevBuf d_sec, d_sec_count, d_warn;   // secondary pool (SecRec[sec_cap]) + its counter
    brc::ReadsDev dev_reads{};       // what the kernels read (push path: d_in; device path: caller's pointers)

    // host results: the PACKED records as they come off the device (pinned) ...
    brc::PinBuf h_words, h_sec, h_misc;
    int64_t h_n_sec = 0;
    // The last run: the kind of results its launch produces (BRC_RESULTS_*, fixed where its kernels are queued) and whether they
    // have reached the host.  filter_on and queries_on below are requests for the next run.
    struct LastRun { int kind = BRC_RESULTS_NONE; bool on_host = false; } last;
    int results_kind() const { return last.on_host ? last.kind : BRC_RESULTS_NONE; }   // the kind the host holds (brc_last_results_kind)
    // ... and the full-width view brc_get_results / the text emitter read, expanded from them on first use (ensure_wide)
    struct Wide {
        std::vector<uint32_t> ncover, npass, pstats, sec_stats;
        std::vector<uint8_t> flags, pbase, sec_kind;
        std::vector<int32_t> sec_head, sec_next, sec_len, sec_qpos;
        std::vector<int64_t> sec_read;
        int64_t n_sec = 0;           // records that are keys (escaped primaries are folded into the slot arrays)
        bool valid = false;
    } wide;
    int64_t warn_counts[4] = {0, 0, 0, 0};

    // text of the last brc_format_* call, so the usual size-query + fill pair formats only once
    std::vector<std::string> fmt_parts; int64_t fmt_key[3] = {-2, -2, -2}; bool fmt_valid = false;

    // f-2: a batch inflated + framed on the device from BGZF blocks (brc_bgzf.cu)
    struct Decoded {
        brc::DevBuf comp, btab, u, meta, scratch, count, partial, arr[12], cigar, seq, qual, ins_idx, ins_out;
        brc_read_batch batch{};          // device pointers into the buffers above
        int64_t n_reads = 0, max_end = 0, n_cigar = 0, n_seq = 0, n_qual = 0, h2d_bytes = 0;
        int kernels = 0;
        bool valid = false;              // a decoded batch is resident
        bool pushed = false;             // ... and it is the open / only region's read stream (brc_push_bam_span)
        cudaStream_t stream = nullptr;   // the stream the decode kernels ran on
        std::vector<std::vector<uint8_t>> host;   // brc_fetch_decoded_batch
        // packed bases of the reads that carry an insertion allele (the text emitter prints them), fetched after the kernels
        std::vector<int64_t> ins_reads; std::vector<uint64_t> ins_off; std::vector<uint8_t> ins_pool;
    } dec;
    // packed bases of read `r` of the pushed stream, wherever they live on the host (staging copy, borrowed batch, or the
    // sparse copy of a device-decoded batch); nullptr when unknown
    const uint8_t *host_read_seq(int64_t r) const {
        if (dec.pushed) {
            const auto it = std::lower_bound(dec.ins_reads.begin(), dec.ins_reads.end(), r);
            if (it == dec.ins_reads.end() || *it != r) return nullptr;
            return dec.ins_pool.data() + dec.ins_off[(size_t)(it - dec.ins_reads.begin())];
        }
        const brc_read_batch b = host_batch();
        return b.seq + b.seq_off[(size_t)r];
    }

    // deletion queue carried from one formatting pass to the next (brc_set_queue_carry): lets a caller flush argv regions
    // batch by batch and still reproduce the reference's never-cleared queue
    bool carry_on = false;
    brc::EmitState carry;

    // alternative-allele site filter (brc_set_site_filter, brc_select.cu).  With it set, the kernels' records are compacted on
    // the device to the sites that print a passing line plus their context, and only those cross PCIe.
    bool filter_on = false;
    brc_site_filter filter{};
    brc_entry_bounds bounds{};                 // brc_set_site_filter_bounds; no bit set: none
    std::vector<brc::SelRegion> sel_regions;   // the selection's region table of the current batch
    brc::DevBuf d_sel, d_sel_regions;          // scratch + compact outputs; region table
    brc::SelectParams sel_params{};            // the last selection ran on these buffers
    brc_site_filter sel_filter{};              // the filter and entry bounds the selection ran with
    brc_entry_bounds sel_bounds{};
    // SELECTED host results: n_sel shipped sites (ids ascending, emit bytes in h_sel), their words in h_words as
    // [N_WORDS][rows*n_sel], their pool records in h_sec with slot = row * n_sel + compact index
    int64_t n_sel = 0, sel_abandoned = 0;
    brc::PinBuf h_sel;
    const uint32_t *sel_site() const { return h_sel.as<uint32_t>(); }
    const uint8_t *sel_emit() const { return reinterpret_cast<const uint8_t *>(h_sel.as<uint32_t>() + n_sel); }
    bool selected() const { return last.kind == BRC_RESULTS_SELECTED; }   // the last run is SELECTED: n_sel columns
    int64_t result_cols() const { return selected() ? n_sel : n_slots; }   // columns of the host word / wide arrays

    // allele queries (brc_set_allele_queries, brc_alleles.cu).  With them set, the kernels' records stay on the device and only
    // the answers cross PCIe; there is no dense view.
    bool queries_on = false;
    std::vector<brc::AlleleQuery> aq;          // sorted by match slot
    std::vector<uint8_t> aq_bases;             // insertion bases as indices into "=ACGTN"
    brc::DevBuf d_aq;                          // queries, bases, scratch, answers
    brc::AlleleParams aq_params{};             // the last allele kernels ran on these buffers
    brc::PinBuf h_ans;                         // ANSWERS host results (no records on the host)

    // complex-record queries (brc_set_complex_queries, brc_complex.cu): the same lifecycle and results kind as the allele
    // queries; both may be set for one batch, and the complex kernel runs after the allele kernels.
    bool complex_on = false;
    std::vector<brc_complex_query> cq;         // as the caller gave them
    std::vector<brc_complex_allele> ca;        // bases_off rebased into cq_bases
    std::vector<uint8_t> cq_bases;             // allele bases as indices into "=ACGTN"
    brc::DevBuf d_cq;                          // queries, alleles, bases, answers
    brc::ComplexParams cq_params{};            // the last complex kernel ran on these buffers (n_q = 0: it did not run)
    brc::PinBuf h_cans;                        // its answers on the host: depth[n_q], then counts[n_alleles] at cans_counts
    size_t cans_counts = 0;
    bool answers_on() const { return queries_on || complex_on; }   // the next run produces BRC_RESULTS_ANSWERS

    int launch_count = 0;
};

namespace brc {
int set_error(brc_engine *e, int status, const std::string &msg);
int set_cuda_error(brc_engine *e, cudaError_t ce, const char *what);
const HostRef *find_ref(const brc_engine *e, int32_t tid);
// The guard of every result view: BRC_OK when the host holds results of a kind in `kinds` (a mask of 1 << BRC_RESULTS_*);
// otherwise BRC_E_INVALID, with a message naming `who` and the getter that serves what the host holds.
int check_view(brc_engine *e, const char *who, unsigned kinds);
int fetch_insertion_reads(brc_engine *e, cudaStream_t s);   // brc_bgzf.cu
void ensure_wide(brc_engine *e);   // expand the packed host records into e->wide (multi-threaded; no-op when already done)
}  // namespace brc
