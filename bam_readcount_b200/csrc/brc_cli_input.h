// brc_cli_input.h — the input side of brc-readcount: a small BGZF/BAM/BAI/FASTA reader written against the SAM specification
// (zlib for inflate), the record decoder, the merged site-list fetch, the compressed-span builder, the parallel window decoder
// and the CRAM reader.  The per-record code (Bgzf::read, read_record, rec_endpos, rec_lib, RegionFetcher::fetch) is inline
// here, so that the loops that call it in other units can inline it.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/brc_engine.h"
#include "brc_aux.cuh"
#include "brc_reads.h"
#include "brc_seq.cuh"

namespace brc::cli {

// ------------------------------------------------------------------------------------------
// BGZF (SAM spec §4.1): random access by virtual offset (coffset<<16 | uoffset)
// ------------------------------------------------------------------------------------------
struct Bgzf {
    FILE *fp = nullptr;
    std::vector<uint8_t> block;
    uint64_t block_coff = 0;     // compressed offset of the current block
    uint64_t next_coff = 0;      // compressed offset of the next block
    size_t upos = 0;             // position inside `block`
    bool eof = false;
    bool error = false;          // a block failed to inflate / a header is malformed / the file ends inside a block: not a clean EOF
    // read-ahead: a span of consecutive blocks is read with one fread and inflated by several threads
    struct Ahead { uint64_t coff, next; std::vector<uint8_t> data; bool ok; };
    std::vector<Ahead> ahead; size_t ahead_pos = 0;
    std::vector<uint8_t> raw;
    int max_threads = 16;
    size_t span_blocks = 64;

    bool open(const std::string &path) { fp = std::fopen(path.c_str(), "rb"); return fp != nullptr; }
    // a reader owned by ONE decode thread of ParallelFetcher: inflates inline, short read-ahead spans
    bool open_worker(const std::string &path) { max_threads = 1; span_blocks = 16; return open(path); }
    ~Bgzf() { if (fp) std::fclose(fp); }

    static bool inflate_block(const uint8_t *src, size_t clen, std::vector<uint8_t> &dst, uint32_t isize);
    // parse one block header at h; returns total block size (0 on error / truncated)
    static size_t block_size(const uint8_t *h, size_t avail, size_t &hdr_len);
    bool fill_ahead(uint64_t coff);
    bool load_block(uint64_t coff);
    bool seek(uint64_t voff);
    uint64_t tell() const { return (block_coff << 16) + (uint64_t)upos; }   // upos may equal a full 64 KiB block
    // read exactly n bytes (spanning blocks); false at EOF
    bool read(void *dst, size_t n) {
        uint8_t *d = (uint8_t *)dst;
        while (n) {
            if (upos >= block.size()) {
                if (!load_block(next_coff)) return false;
                if (block.empty()) { if (eof) return false; continue; }
            }
            const size_t k = std::min(n, block.size() - upos);
            std::memcpy(d, block.data() + upos, k);
            d += k; upos += k; n -= k;
        }
        return true;
    }
};

// ------------------------------------------------------------------------------------------
// BAM header + BAI index (SAM spec §4.2, §5.2)
// ------------------------------------------------------------------------------------------
struct BamFile {
    Bgzf bz;
    std::string text;
    std::vector<std::string> names;
    std::vector<int32_t> lens;
    std::map<std::string, int> tid_of;
    uint64_t first_rec = 0;
    // BAI
    struct RefIdx { std::vector<uint64_t> linear; uint64_t min_chunk = ~0ull; std::map<uint32_t, std::vector<std::pair<uint64_t, uint64_t>>> bins; };
    std::vector<RefIdx> idx;
    bool have_idx = false;

    bool open(const std::string &path);
    bool load_index(const std::string &bam_path);
    // smallest virtual offset of a record that can overlap position `beg` on `tid` (linear index, 16 kb windows)
    bool query_offset(int tid, int64_t beg, uint64_t &voff) const;
};

// ------------------------------------------------------------------------------------------
// Records
// ------------------------------------------------------------------------------------------
struct Rec {   // one decoded alignment (the bam1_t fields the path reads)
    int32_t tid, pos, l_qseq, nm, sm; uint16_t flag; uint8_t mapq; uint32_t n_cigar;
    int64_t endpos;              // bam_endpos, filled by RegionFetcher
    std::vector<uint8_t> data;   // whole record body
    const uint32_t *cigar; const uint8_t *seq, *qual; std::string rg; bool has_rg;
};

inline bool read_record(Bgzf &bz, Rec &r) {
    int32_t bs;
    if (!bz.read(&bs, 4)) return false;                                   // EOF (clean unless bz.error)
    if (bs < 32) { bz.error = true; return false; }                       // not a BAM record
    r.data.resize((size_t)bs);
    if (!bz.read(r.data.data(), (size_t)bs)) { bz.error = true; return false; }   // file ends inside a record
    const uint8_t *d = r.data.data();
    int32_t refid, pos, l_seq; uint8_t l_rn, mapq; uint16_t n_cig, flag;
    std::memcpy(&refid, d, 4); std::memcpy(&pos, d + 4, 4); l_rn = d[8]; mapq = d[9];
    std::memcpy(&n_cig, d + 12, 2); std::memcpy(&flag, d + 14, 2); std::memcpy(&l_seq, d + 16, 4);
    r.tid = refid; r.pos = pos; r.mapq = mapq; r.flag = flag; r.l_qseq = l_seq;
    size_t o = 32 + l_rn + 4 * (size_t)n_cig;
    r.seq = d + o; o += ((size_t)l_seq + 1) / 2;
    r.qual = d + o; o += (size_t)l_seq;
    const brc::aux::RecAux ax = brc::aux::scan(d, bs, (int64_t)o, 32 + l_rn, n_cig);     // NM, SM, RG, CG (brc_aux.cuh)
    r.cigar = (const uint32_t *)(d + ax.cig_o); r.n_cigar = ax.n_cigar;
    r.nm = ax.nm; r.sm = ax.sm;
    r.has_rg = ax.rg_o >= 0;
    if (r.has_rg) r.rg.assign((const char *)d + ax.rg_o, (size_t)ax.rg_len);
    return true;
}

inline int64_t rec_endpos(const Rec &r) {   // bam_endpos
    if (!(r.flag & 4) && r.n_cigar > 0) return r.pos + brc::cigar_span(r.cigar, r.n_cigar).rlen;
    return (int64_t)r.pos + 1;
}

using RgLib = std::unordered_map<std::string, uint16_t>;   // @RG ID -> library rank

// the library the engine counts a record under: 0 without -p; under -p the rank of its read group's LB, or BRC_LIB_NONE
// where bam_get_library finds none (no RG tag, or an ID without an LB in the header)
inline uint16_t rec_lib(const Rec &r, const RgLib &rg_lib, bool per_lib) {
    if (!per_lib) return 0;
    if (r.has_rg) { auto it = rg_lib.find(r.rg); if (it != rg_lib.end()) return it->second; }
    return (uint16_t)BRC_LIB_NONE;
}

// A record that can warn (Warner::candidate, brc_cli_warn.h): what the per-read warning replay needs of it
struct WarnCand { int32_t pos; int64_t endpos; uint16_t flag; uint8_t mapq; bool no_nm, no_sm, no_lib; std::vector<uint32_t> cigar; std::vector<uint8_t> qual; std::string qname; };

// ------------------------------------------------------------------------------------------
// SURVEY.md §8 f-2: the compressed bytes + index entry points covering samfetch(tid, fbeg, fend), for brc_push_bam_span — the
// records are inflated and framed on the device, only compressed bytes cross PCIe.  The BAI's chunk begins and linear-index
// offsets are starts of real records: each starts an independent framing chain.
// ------------------------------------------------------------------------------------------
struct SpanBuilder {
    std::vector<uint8_t> comp; std::vector<uint64_t> entries; int64_t end_voff = -1;
    bool build(BamFile &bam, int tid, int64_t fbeg, int64_t fend);
};

// ------------------------------------------------------------------------------------------
// samfetch(in, idx, tid, fbeg, fend) for a run of regions (SURVEY.md §8 f-3).  The reference re-seeks through the index and
// re-decodes up to a 16 kb linear-index window of records for every line of a site list; here consecutive regions on one
// contig with ascending starts share ONE forward pass over the file: records still overlapping a later region wait in a
// small window, everything else streams straight to the caller.  Each region still receives exactly the records samfetch
// yields (tid, endpos > fbeg, pos < fend) in file order.  `next_fbeg` (start of the following region, or INT64_MAX) only
// bounds what is retained; a caller that then asks for something else simply falls back to an index seek.
// ------------------------------------------------------------------------------------------
struct RegionFetcher {
    BamFile &bam;
    std::deque<Rec> win;          // decoded records that may overlap a later region, file order
    std::vector<Rec> spare;       // recycled records (keeps their heap buffers)
    bool active = false, stream_done = false;
    int cur_tid = -1;
    int64_t last_fbeg = -1, keep_floor = -1, last_pos = -1;
    uint64_t n_seeks = 0, n_decoded = 0;

    explicit RegionFetcher(BamFile &b) : bam(b) {}

    Rec take() { if (spare.empty()) return Rec(); Rec r = std::move(spare.back()); spare.pop_back(); return r; }
    void give(Rec &&r) { if (spare.size() < 4096) spare.push_back(std::move(r)); }

    template <class Emit> void fetch(int tid, int64_t fbeg, int64_t fend, int64_t next_fbeg, Emit &&emit) {
        uint64_t voff;
        if (!bam.query_offset(tid, fbeg, voff)) return;
        const bool cont = active && tid == cur_tid && fbeg >= last_fbeg && fbeg >= keep_floor && voff <= bam.bz.tell();
        if (!cont) {
            while (!win.empty()) { give(std::move(win.back())); win.pop_back(); }
            stream_done = false; last_pos = -1; ++n_seeks;
            if (!bam.bz.seek(voff)) { active = false; return; }
            active = true; cur_tid = tid;
        }
        last_fbeg = fbeg; keep_floor = next_fbeg >= fbeg ? next_fbeg : fbeg;      // an unsorted successor seeks anyway
        for (const Rec &r : win) { if (r.pos >= fend) break; if (r.endpos > fbeg) emit(r); }
        while (!stream_done && last_pos < fend) {
            Rec r = take();
            if (!read_record(bam.bz, r) || r.tid != tid) { stream_done = true; give(std::move(r)); break; }
            ++n_decoded;
            r.endpos = rec_endpos(r); last_pos = r.pos;
            if (r.pos < fend && r.endpos > fbeg) emit(r);
            if (r.pos >= fend || r.endpos > keep_floor) win.push_back(std::move(r)); else give(std::move(r));
        }
        // drop what no later region (start >= keep_floor) can overlap; order of the rest is kept
        size_t w = 0;
        for (size_t i = 0; i < win.size(); ++i) {
            if (win[i].endpos > keep_floor) { if (w != i) std::swap(win[w], win[i]); ++w; }
        }
        while (win.size() > w) { give(std::move(win.back())); win.pop_back(); }
    }
};

// ------------------------------------------------------------------------------------------
// CRAM (or any htslib-readable alignment file) through htslib: header, index, and samfetch()'s iterator per region.
// Records are re-laid-out as the Rec the BAM reader produces, so everything downstream is shared.  In a host built without
// htslib (no BRC_WITH_HTSLIB), open() fails.
// ------------------------------------------------------------------------------------------
struct HtsSource {
    uint64_t n_seeks = 0, n_decoded = 0; bool error = false;
    HtsSource();
    ~HtsSource();
    HtsSource(const HtsSource &) = delete; HtsSource &operator=(const HtsSource &) = delete;
    static bool available();    // this host was built with htslib
    bool open(const std::string &path, const std::string &fasta, BamFile &meta);
    bool load_index(const std::string &path);
    void fetch(int tid, int64_t fbeg, int64_t fend, const std::function<void(const Rec &)> &emit);
private:
    struct Files;               // htslib's handles
    std::unique_ptr<Files> f;
};

// ------------------------------------------------------------------------------------------
// Parallel decode of one big fetch (a window of a cut region): the position range is cut at 16 kb linear-index boundaries
// into one sub-range per thread; every thread has its own BGZF reader, seeks through the index and keeps the records whose
// START lies in its sub-range (the first thread also keeps the earlier records that reach into the fetch), so the slices
// concatenated in thread order are exactly samfetch's records in file order.  Each slice is decoded straight into the
// struct-of-arrays layout of brc_read_batch; the slices are then copied (in parallel) into ONE page-locked batch that
// brc_push_reads borrows, so the engine's pipelined upload runs out of it with no further host copy.
// Unmapped records are dropped here (the pileup buffer refuses them, V:htslib-1.10/sam.c:4488-4490).
// ------------------------------------------------------------------------------------------
struct Slice {
    ReadArrays reads;
    std::vector<WarnCand> cands; bool cand_overflow = false, error = false; uint64_t n_decoded = 0;
    void clear() { reads.clear(); cands.clear(); cand_overflow = false; error = false; n_decoded = 0; }
};

struct PinnedBuf {   // grow-only host buffer: page-locked through the engine when there is one (brc_host_alloc), plain otherwise
    void *p = nullptr; size_t cap = 0; bool pinned = false;
    bool reserve(size_t bytes, bool want_pinned);
    void release();
    ~PinnedBuf() { release(); }
    PinnedBuf() = default; PinnedBuf(const PinnedBuf &) = delete; PinnedBuf &operator=(const PinnedBuf &) = delete;
};

struct WindowJob {   // one decoded window: the slices and their concatenation, a batch whose arrays are carved from `block`
    std::vector<Slice> slices;
    PinnedBuf block;
    brc_read_batch batch{};
    uint64_t n_decoded = 0; bool error = false, cand_overflow = false;
    int tid = -1; int64_t fbeg = 0, fend = 0;
    std::string timing;           // BRC_CLI_TIMING line, printed to the sample's stream by the thread that takes the job
};

struct ParallelFetcher {
    const BamFile &bam; const RgLib &rg_lib; std::string path; int n_threads; bool per_lib, want_pinned;
    std::vector<std::unique_ptr<Bgzf>> readers;
    static constexpr size_t MAX_CANDS = 65536;

    ParallelFetcher(const BamFile &b, const RgLib &rl, const std::string &p, bool pl, bool pin);
    static bool eligible(int64_t fbeg, int64_t fend) { return fend - fbeg >= (int64_t(1) << 18); }   // >= 16 linear-index windows
    // records of contig `tid` with lo <= pos < hi (first slice: also pos < lo with endpos > fbeg), in file order
    void decode_slice(Bgzf &bz, int tid, int64_t lo, int64_t hi, bool first, int64_t fbeg, bool collect, Slice &out) const;
    // decode [fbeg, fend) of `tid` into job.slices and job.batch; false when a reader could not be opened
    bool run(int tid, int64_t fbeg, int64_t fend, bool collect, WindowJob &job);
};

// ------------------------------------------------------------------------------------------
// FASTA + .fai (fai_fetch of a whole chromosome, R:...:87)
// ------------------------------------------------------------------------------------------
struct Fasta {
    std::string path;
    struct Ent { int64_t len, off, lb, lw; };
    std::map<std::string, Ent> ents;
    bool open(const std::string &p);
    bool fetch(const std::string &name, std::string &out) const;
};

// samtools region string "name[:beg[-end]]" as bam_parse_region handles it (brc_cli_input.cpp)
int parse_region(const BamFile &bam, const std::string &s, int &tid, int &beg, int &end);

}  // namespace brc::cli
