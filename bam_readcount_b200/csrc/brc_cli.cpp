// brc_cli.cpp — `brc-readcount`: the C++ host.  Same command line and STDOUT as bam-readcount
// (R:src/exe/bam-readcount/bamreadcount.cpp:421-670), with the pileup hot path routed through
// libbrc_engine.so (include/brc_engine.h).  File decode stays on the host, as the north star says:
// a small BGZF/BAM/BAI/FASTA reader written against the SAM specification (zlib for inflate);
// htslib is not needed for BAM.  CRAM input (R:test-data/cram_site_test.sh, BASELINE config 2b) is decoded through htslib when the
// host is built with -DBRC_WITH_HTSLIB against a libhts.a (tools/build_htslib.sh builds the copy vendored with the reference,
// htslib 1.10); without it a .cram argument is refused with a message.
//
// Mirrors, region by region, the reference's two loops:
//   -l site list : R:...:574-608  (d.beg=beg-1, d.end=end, queues cleared per region)
//   argv regions : R:...:641-657  (bam_parse_region; a bare contig name keeps the previous beg/end, A.6)
// With --bam-list the same per-sample run is repeated over a list of inputs in one process (DESIGN.md §11); --vcf-samples
// does the same for the sample columns of one VCF (DESIGN.md §12).
#include <algorithm>
#include <cctype>
#include <cerrno>
#include <cstdarg>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <getopt.h>
#include <deque>
#include <fcntl.h>
#include <filesystem>
#include <map>
#include <set>
#include <sstream>
#include <string>
#include <vector>
#include <zlib.h>
#include <chrono>
#include <future>
#include <memory>
#include <thread>
#include <unordered_map>
#include <unistd.h>

#include "../../include/brc_engine.h"
#include "brc_aux.cuh"
#ifdef BRC_WITH_HTSLIB
#include <functional>
#include <htslib/sam.h>
#include <htslib/hts.h>
#endif

namespace {

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
    int n_threads = 8;
    size_t span_blocks = 64;

    bool open(const std::string &path) {
        fp = std::fopen(path.c_str(), "rb");
        unsigned hw = std::thread::hardware_concurrency();
        n_threads = (int)std::max(1u, std::min(hw ? hw : 1u, 16u));
        return fp != nullptr;
    }
    // a reader owned by ONE decode thread of ParallelFetcher: inflates inline, short read-ahead spans
    bool open_worker(const std::string &path) { fp = std::fopen(path.c_str(), "rb"); n_threads = 1; span_blocks = 16; return fp != nullptr; }
    ~Bgzf() { if (fp) std::fclose(fp); }

    static bool inflate_block(const uint8_t *src, size_t clen, std::vector<uint8_t> &dst, uint32_t isize) {
        dst.resize(isize);
        if (!isize) return true;
        z_stream zs{};
        if (inflateInit2(&zs, -15) != Z_OK) return false;
        zs.next_in = const_cast<uint8_t *>(src); zs.avail_in = (uInt)clen; zs.next_out = dst.data(); zs.avail_out = isize;
        const int rc = inflate(&zs, Z_FINISH);
        inflateEnd(&zs);
        return rc == Z_STREAM_END;
    }
    // parse one block header at raw[o..]; returns total block size (0 on error / truncated)
    static size_t block_size(const uint8_t *h, size_t avail, size_t &hdr_len) {
        if (avail < 18 || h[0] != 31 || h[1] != 139 || h[2] != 8 || !(h[3] & 4)) return 0;
        const size_t xlen = (size_t)(h[10] | (h[11] << 8));
        if (avail < 12 + xlen) return 0;
        int bsize = -1;
        for (size_t i = 0; i + 4 <= xlen;) {
            const size_t sl = (size_t)(h[12 + i + 2] | (h[12 + i + 3] << 8));
            if (h[12 + i] == 'B' && h[12 + i + 1] == 'C' && sl == 2) bsize = h[12 + i + 4] | (h[12 + i + 5] << 8);
            i += 4 + sl;
        }
        if (bsize < 0) return 0;
        hdr_len = 12 + xlen;
        return (size_t)bsize + 1;
    }
    bool fill_ahead(uint64_t coff) {
        ahead.clear(); ahead_pos = 0;
        if (fseeko(fp, (off_t)coff, SEEK_SET) != 0) return false;
        raw.resize(span_blocks * 65536 + 65536);
        const size_t got = std::fread(raw.data(), 1, raw.size(), fp);
        if (got == 0) { eof = true; return false; }                      // clean end of file at a block boundary
        if (got < 18) { eof = true; error = true; return false; }        // a fragment of a block header
        struct Job { size_t off, hdr, total; };
        std::vector<Job> jobs;
        for (size_t o = 0; o < got && jobs.size() < span_blocks;) {
            size_t hdr = 0; const size_t tot = block_size(raw.data() + o, got - o, hdr);
            if (!tot || o + tot > got) break;
            jobs.push_back({o, hdr, tot}); o += tot;
        }
        if (jobs.empty()) { error = true; return false; }                // bytes are there but no whole, well-formed block
        ahead.resize(jobs.size());
        auto work = [&](size_t t) {
            for (size_t j = t; j < jobs.size(); j += (size_t)n_threads) {
                const Job &jb = jobs[j];
                const uint8_t *b = raw.data() + jb.off;
                const size_t clen = jb.total - jb.hdr - 8;
                const uint8_t *tail = b + jb.total - 4;
                const uint32_t isize = tail[0] | (tail[1] << 8) | (tail[2] << 16) | ((uint32_t)tail[3] << 24);
                ahead[j].coff = coff + jb.off; ahead[j].next = coff + jb.off + jb.total;
                ahead[j].ok = inflate_block(b + jb.hdr, clen, ahead[j].data, isize);
            }
        };
        std::vector<std::thread> th;
        const int nt = (int)std::min<size_t>((size_t)n_threads, jobs.size());
        for (int t = 1; t < nt; ++t) th.emplace_back(work, (size_t)t);
        work(0);
        for (auto &x : th) x.join();
        return true;
    }
    bool load_block(uint64_t coff) {
        if (!(ahead_pos < ahead.size() && ahead[ahead_pos].coff == coff)) {
            // look inside the current span first (seeks within it), else read a new span
            bool found = false;
            for (size_t j = 0; j < ahead.size(); ++j) if (ahead[j].coff == coff && !ahead[j].data.empty()) { ahead_pos = j; found = true; break; }
            if (!found && !fill_ahead(coff)) { block.clear(); upos = 0; return false; }
        }
        Ahead &a = ahead[ahead_pos];
        if (!a.ok) { error = true; return false; }
        block = a.data;                 // keep the span entry intact: sorted site lists revisit blocks
        block_coff = a.coff; next_coff = a.next; upos = 0; eof = false;
        ++ahead_pos;
        return true;
    }
    bool seek(uint64_t voff) {
        // sorted site lists keep landing in the block that is already inflated
        if (!((voff >> 16) == block_coff && !block.empty() && !eof) && !load_block(voff >> 16)) return false;
        upos = (size_t)(voff & 0xFFFF);
        return true;
    }
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

    bool open(const std::string &path) {
        if (!bz.open(path) || !bz.load_block(0)) return false;
        char magic[4]; int32_t l_text, n_ref;
        if (!bz.read(magic, 4) || std::memcmp(magic, "BAM\1", 4) != 0) return false;
        if (!bz.read(&l_text, 4)) return false;
        text.resize((size_t)l_text);
        if (l_text && !bz.read(&text[0], (size_t)l_text)) return false;
        text = text.c_str();
        if (!bz.read(&n_ref, 4)) return false;
        for (int i = 0; i < n_ref; ++i) {
            int32_t ln, sl;
            if (!bz.read(&ln, 4)) return false;
            std::string nm((size_t)ln, 0);
            if (!bz.read(&nm[0], (size_t)ln) || !bz.read(&sl, 4)) return false;
            nm = nm.c_str();
            tid_of[nm] = i; names.push_back(nm); lens.push_back(sl);
        }
        first_rec = bz.tell();
        return true;
    }
    bool load_index(const std::string &bam_path) {
        std::string p = bam_path + ".bai";
        FILE *f = std::fopen(p.c_str(), "rb");
        if (!f && bam_path.size() > 4) { p = bam_path.substr(0, bam_path.size() - 4) + ".bai"; f = std::fopen(p.c_str(), "rb"); }
        if (!f) return false;
        auto rd = [&](void *d, size_t n) { return std::fread(d, 1, n, f) == n; };
        char magic[4]; int32_t n_ref;
        bool ok = rd(magic, 4) && std::memcmp(magic, "BAI\1", 4) == 0 && rd(&n_ref, 4);
        idx.assign((size_t)std::max(n_ref, 0), RefIdx());
        for (int r = 0; ok && r < n_ref; ++r) {
            int32_t n_bin; ok = rd(&n_bin, 4);
            for (int b = 0; ok && b < n_bin; ++b) {
                uint32_t bin; int32_t n_chunk; ok = rd(&bin, 4) && rd(&n_chunk, 4);
                for (int c = 0; ok && c < n_chunk; ++c) {
                    uint64_t cb, ce; ok = rd(&cb, 8) && rd(&ce, 8);
                    if (ok && bin != 37450) { idx[(size_t)r].min_chunk = std::min(idx[(size_t)r].min_chunk, cb); idx[(size_t)r].bins[bin].push_back({cb, ce}); }
                }
            }
            int32_t n_intv; ok = ok && rd(&n_intv, 4);
            if (ok) { idx[(size_t)r].linear.resize((size_t)n_intv); ok = n_intv == 0 || rd(idx[(size_t)r].linear.data(), 8 * (size_t)n_intv); }
        }
        std::fclose(f);
        have_idx = ok;
        return ok;
    }
    // smallest virtual offset of a record that can overlap position `beg` on `tid` (linear index, 16 kb windows)
    bool query_offset(int tid, int64_t beg, uint64_t &voff) const {
        if (tid < 0 || tid >= (int)idx.size()) return false;
        const RefIdx &ri = idx[(size_t)tid];
        if (ri.min_chunk == ~0ull) return false;                      // no alignments on this reference
        int64_t w = beg >> 14;
        voff = ri.min_chunk;
        if (!ri.linear.empty()) {
            if (w >= (int64_t)ri.linear.size()) w = (int64_t)ri.linear.size() - 1;
            for (; w >= 0; --w) if (ri.linear[(size_t)w] != 0) { voff = std::max(voff, ri.linear[(size_t)w]); break; }
        }
        return true;
    }
};

struct Rec {   // one decoded alignment (the bam1_t fields the path reads)
    int32_t tid, pos, l_qseq, nm, sm; uint16_t flag; uint8_t mapq; uint32_t n_cigar;
    int64_t endpos;              // bam_endpos, filled by RegionFetcher
    std::vector<uint8_t> data;   // whole record body
    const uint32_t *cigar; const uint8_t *seq, *qual; std::string rg; bool has_rg;
};

bool read_record(Bgzf &bz, Rec &r) {
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

int64_t rec_endpos(const Rec &r) {   // bam_endpos
    if (!(r.flag & 4) && r.n_cigar > 0) {
        int64_t l = 0;
        for (uint32_t k = 0; k < r.n_cigar; ++k) { uint32_t op = r.cigar[k] & 0xF; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) l += r.cigar[k] >> 4; }
        return r.pos + l;
    }
    return (int64_t)r.pos + 1;
}

using RgLib = std::unordered_map<std::string, uint16_t>;   // @RG ID -> library rank

// the library the engine counts a record under: 0 without -p; under -p the rank of its read group's LB, or BRC_LIB_NONE
// where bam_get_library finds none (no RG tag, or an ID without an LB in the header)
uint16_t rec_lib(const Rec &r, const RgLib &rg_lib, bool per_lib) {
    if (!per_lib) return 0;
    if (r.has_rg) { auto it = rg_lib.find(r.rg); if (it != rg_lib.end()) return it->second; }
    return (uint16_t)BRC_LIB_NONE;
}

// ------------------------------------------------------------------------------------------
// SURVEY.md §8 f-2: the compressed bytes + index entry points covering samfetch(tid, fbeg, fend), for brc_push_bam_span — the
// records are inflated and framed on the device, only compressed bytes cross PCIe.  The BAI's chunk begins and linear-index
// offsets are starts of real records: each starts an independent framing chain.
// ------------------------------------------------------------------------------------------
struct SpanBuilder {
    std::vector<uint8_t> comp; std::vector<uint64_t> entries; int64_t end_voff = -1;
    bool build(BamFile &bam, int tid, int64_t fbeg, int64_t fend) {
        if (tid < 0 || tid >= (int)bam.idx.size()) return false;
        const BamFile::RefIdx &ri = bam.idx[(size_t)tid];
        uint64_t min_lin = 0;
        if (!ri.linear.empty()) { int64_t w = std::min<int64_t>(fbeg >> 14, (int64_t)ri.linear.size() - 1); min_lin = ri.linear[(size_t)w]; }
        uint64_t v0 = ~0ull, v1 = 0; std::vector<uint64_t> cand;
        const int64_t b = std::max<int64_t>(fbeg, 0), e = std::max<int64_t>(fend, b + 1) - 1;
        auto visit = [&](uint32_t bin) {
            auto it = ri.bins.find(bin);
            if (it == ri.bins.end()) return;
            for (const auto &c : it->second) if (c.second > min_lin) { const uint64_t cb = std::max(c.first, min_lin); v0 = std::min(v0, cb); v1 = std::max(v1, c.second); cand.push_back(cb); }
        };
        visit(0);
        const int sh[5] = {26, 23, 20, 17, 14}; const uint32_t of[5] = {1, 9, 73, 585, 4681};
        for (int l = 0; l < 5; ++l) for (int64_t k = b >> sh[l]; k <= (e >> sh[l]); ++k) visit(of[l] + (uint32_t)k);
        if (v0 == ~0ull || v1 <= v0) return false;
        for (int64_t w = std::min<int64_t>(b >> 14, (int64_t)ri.linear.size()); w < std::min<int64_t>((e >> 14) + 2, (int64_t)ri.linear.size()); ++w) cand.push_back(ri.linear[(size_t)w]);
        const uint64_t c0 = v0 >> 16, c1 = v1 >> 16;
        comp.resize((size_t)(c1 - c0) + 65536 + 32);
        if (fseeko(bam.bz.fp, (off_t)c0, SEEK_SET) != 0) return false;
        const size_t got = std::fread(comp.data(), 1, comp.size(), bam.bz.fp);
        std::vector<uint64_t> starts; size_t o = 0;
        while (o + 18 <= got) {
            size_t hdr = 0; const size_t tot = Bgzf::block_size(comp.data() + o, got - o, hdr);
            if (!tot || o + tot > got) break;
            starts.push_back(c0 + o); o += tot;
            if (starts.back() >= c1) break;
        }
        if (starts.empty()) return false;
        comp.resize(o);
        auto rel = [&](uint64_t v, uint64_t &out) { const uint64_t co = v >> 16; if (!std::binary_search(starts.begin(), starts.end(), co)) return false; out = ((co - c0) << 16) | (v & 0xFFFF); return true; };
        std::sort(cand.begin(), cand.end()); cand.erase(std::unique(cand.begin(), cand.end()), cand.end());
        entries.clear();
        for (uint64_t v : cand) { uint64_t r; if (v >= v0 && v < v1 && rel(v, r)) entries.push_back(r); }
        uint64_t r1; end_voff = rel(v1, r1) ? (int64_t)r1 : -1;
        bam.bz.block.clear(); bam.bz.ahead.clear(); bam.bz.ahead_pos = 0; bam.bz.eof = false;     // the reader's position is stale now
        return !entries.empty();
    }
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

#ifdef BRC_WITH_HTSLIB
// ------------------------------------------------------------------------------------------
// CRAM (or any htslib-readable alignment file) through htslib: header, index, and samfetch()'s iterator per region.
// Records are re-laid-out as the Rec the BAM reader produces, so everything downstream is shared.
// ------------------------------------------------------------------------------------------
struct HtsSource {
    samFile *fp = nullptr; bam_hdr_t *hdr = nullptr; hts_idx_t *idx = nullptr; bam1_t *b = nullptr;
    uint64_t n_seeks = 0, n_decoded = 0; bool error = false;
    ~HtsSource() { if (b) bam_destroy1(b); if (idx) hts_idx_destroy(idx); if (hdr) bam_hdr_destroy(hdr); if (fp) sam_close(fp); }
    bool open(const std::string &path, const std::string &fasta, BamFile &meta) {
        fp = sam_open(path.c_str(), "r");
        if (!fp) return false;
        if (!fasta.empty() && hts_set_fai_filename(fp, (fasta + ".fai").c_str()) != 0) return false;   // R:bamreadcount.cpp:503-523
        hdr = sam_hdr_read(fp);
        if (!hdr) return false;
        meta.text.assign(hdr->text ? hdr->text : "", hdr->text ? hdr->l_text : 0);
        for (int i = 0; i < hdr->n_targets; ++i) { meta.names.push_back(hdr->target_name[i]); meta.lens.push_back((int32_t)hdr->target_len[i]); meta.tid_of[hdr->target_name[i]] = i; }
        b = bam_init1();
        return true;
    }
    bool load_index(const std::string &path) { idx = sam_index_load(fp, path.c_str()); return idx != nullptr; }
    void fetch(int tid, int64_t fbeg, int64_t fend, const std::function<void(const Rec &)> &emit) {
        hts_itr_t *it = sam_itr_queryi(idx, tid, fbeg, fend);
        if (!it) return;
        ++n_seeks;
        Rec r; int ret;
        while ((ret = sam_itr_next(fp, it, b)) >= 0) {
            ++n_decoded;
            const bam1_core_t &c = b->core;
            r.tid = c.tid; r.pos = (int32_t)c.pos; r.l_qseq = c.l_qseq; r.flag = c.flag; r.mapq = c.qual; r.n_cigar = c.n_cigar;
            r.data.assign(32, 0); r.data.insert(r.data.end(), b->data, b->data + b->l_data);      // qname at +32, as in a BAM record body
            const uint8_t *d = r.data.data() + 32;
            r.cigar = (const uint32_t *)(d + c.l_qname); r.seq = d + c.l_qname + 4 * (size_t)c.n_cigar; r.qual = r.seq + ((size_t)c.l_qseq + 1) / 2;
            uint8_t *p;
            r.nm = (p = bam_aux_get(b, "NM")) ? (int32_t)bam_aux2i(p) : BRC_TAG_ABSENT;
            r.sm = (p = bam_aux_get(b, "SM")) ? (int32_t)bam_aux2i(p) : BRC_TAG_ABSENT;
            r.has_rg = (p = bam_aux_get(b, "RG")) != nullptr;                                        // bam_get_library: the first RG, any type
            if (r.has_rg) r.rg.assign((const char *)(p + 1), strnlen((const char *)(p + 1), (size_t)(b->data + b->l_data - (p + 1))));
            r.endpos = rec_endpos(r);
            emit(r);
        }
        if (ret < -1) error = true;
        hts_itr_destroy(it);
    }
};
#endif

// ------------------------------------------------------------------------------------------
// Per-read warning lines (R:src/lib/bamrc/ReadWarnings.hpp:12-50; call sites R:BasicStat.cpp:85,100 and R:bamreadcount.cpp:282).
// The engine returns per-type event COUNTS; the text names reads, in the order the reference meets the events: region by
// region, site by site, spanning reads in file order, and inside one event process_read's own order (SM before NM; an
// indel event calls process_read for the indel key and again for the base key).  The host replays exactly that walk over the
// reads that can warn at all (no NM tag, proper pair without SM tag, no library under -p) until every type has used up its
// -w budget, then stops collecting.  With -w -1 the reference prints one line per offending EVENT without bound; this host
// prints the first 1000 per type and then the engine's exact total (the one documented STDERR difference).
// ------------------------------------------------------------------------------------------
struct Warner {
    enum { SM = 0, NM = 1, ZM = 2, LIB = 3, NT = 4 };
    struct Cand { int32_t pos; int64_t endpos; uint16_t flag; uint8_t mapq; bool no_nm, no_sm, no_lib; std::vector<uint32_t> cigar; std::vector<uint8_t> qual; std::string qname; };
    struct Reg { int tid, beg, end; bool skip_halo; size_t c0, c1; };
    long long max_per_type; bool unlimited; int min_mapq, min_bq; bool per_lib, ic;
    long long counts[NT] = {0, 0, 0, 0};
    std::vector<Cand> cands; std::vector<Reg> regs;
    FILE *err = stderr;           // the sample's message stream
    Warner(long long mw, int q, int b, bool p, bool i) : max_per_type(mw < 0 ? 1000 : mw), unlimited(mw < 0), min_mapq(q), min_bq(b), per_lib(p), ic(i) {}
    bool budget_left() const { return counts[SM] < max_per_type || counts[NM] < max_per_type || (per_lib && counts[LIB] < max_per_type); }
    bool collecting() const { return max_per_type > 0 && budget_left(); }
    void begin_region(int tid, int beg, int end, bool skip_halo) { regs.push_back({tid, beg, end, skip_halo, cands.size(), cands.size()}); }
    // a record that can warn at all (no NM tag, proper pair without SM tag, or `lib` == BRC_LIB_NONE) becomes `c`
    static bool candidate(const Rec &r, uint16_t lib, Cand &c) {
        const bool no_nm = r.nm == BRC_TAG_ABSENT, no_sm = (r.flag & 2) && r.sm == BRC_TAG_ABSENT, no_lib = lib == (uint16_t)BRC_LIB_NONE;
        if (!no_nm && !no_sm && !no_lib) return false;
        c.pos = r.pos; c.endpos = rec_endpos(r); c.flag = r.flag; c.mapq = r.mapq; c.no_nm = no_nm; c.no_sm = no_sm; c.no_lib = no_lib;
        c.cigar.assign(r.cigar, r.cigar + r.n_cigar); c.qual.assign(r.qual, r.qual + r.l_qseq);
        c.qname = (const char *)(r.data.data() + 32);
        return true;
    }
    // a record of the record stream, in file order
    void consider(const Rec &r, uint16_t lib) {
        if (!collecting() || (r.flag & 4) || regs.empty()) return;
        Cand c;
        if (!candidate(r, lib, c)) return;
        cands.push_back(std::move(c)); regs.back().c1 = cands.size();
    }
    // candidates collected by a parallel decode (ParallelFetcher), already in file order
    void take(std::vector<Cand> &more) {
        if (!collecting() || regs.empty()) { more.clear(); return; }
        for (Cand &c : more) cands.push_back(std::move(c));
        more.clear(); regs.back().c1 = cands.size();
    }
    void emit(int type, const std::string &qname) {
        static const char *msg[NT] = {"Couldn't find single-end mapping quality. Check to see if the SM tag is in BAM.",
                                      "Couldn't find number of mismatches. Check to see if the NM tag is in BAM.",
                                      "Couldn't find the generated tag.",
                                      "Library unavailable. Check to make sure the LB tag is present in the @RG entries of the header."};
        ++counts[type];
        if (counts[type] > max_per_type) return;
        std::fprintf(err, "WARNING: In read %s: %s\n", qname.c_str(), msg[type]);
        if (!unlimited && counts[type] == max_per_type) std::fprintf(err, "The previous warning has been emitted %lld times and will be disabled.\n", counts[type]);
    }
    // stateless resolve_cigar2 (V:htslib-1.10/sam.c:3964-4041): qpos / is_del / indel of `site` in a read
    static bool resolve(const Cand &c, int64_t site, int &qpos, int &indel) {
        int64_t x = c.pos; int y = 0; size_t k = 0; uint32_t op = 0; int len = 0; const size_t n = c.cigar.size();
        auto refop = [](uint32_t o) { return o == 0 || o == 2 || o == 3 || o == 7 || o == 8; };
        auto matchop = [](uint32_t o) { return o == 0 || o == 7 || o == 8; };
        for (; k < n; ++k) {
            op = c.cigar[k] & 0xF; len = (int)(c.cigar[k] >> 4);
            if (refop(op)) { if (site < x + len) break; x += len; if (matchop(op)) y += len; }
            else if (op == 1 || op == 4) y += len;
        }
        indel = 0;
        if (k >= n) return false;
        const bool is_del = !matchop(op);
        qpos = is_del ? y : y + (int)(site - x);
        if (x + len - 1 == site && k + 1 < n) {
            const uint32_t op2 = c.cigar[k + 1] & 0xF; const int l2 = (int)(c.cigar[k + 1] >> 4);
            if (op2 == 2) indel = -l2;
            else if (op2 == 1) indel = l2;
            else if (op2 == 6) { int l3 = 0; for (size_t m = k + 2; m < n; ++m) { const uint32_t o3 = c.cigar[m] & 0xF; if (o3 == 1) l3 += (int)(c.cigar[m] >> 4); else if (refop(o3)) break; } if (l3 > 0) indel = l3; }
        }
        return !is_del;
    }
    void replay() {
        for (const Reg &g : regs) {
            if (!budget_left()) break;
            if (g.c0 == g.c1) continue;
            const int64_t first = g.skip_halo ? g.beg : std::max(g.beg - 1, 0);
            size_t lo = g.c0;
            for (int64_t p = std::max<int64_t>(first, cands[g.c0].pos); p < g.end && budget_left(); ++p) {
                while (lo < g.c1 && cands[lo].endpos <= p) ++lo;          // leading reads that ended (later ones are re-checked below)
                if (lo >= g.c1) break;
                if (cands[lo].pos > p) { p = cands[lo].pos - 1; continue; }
                for (size_t i = lo; i < g.c1 && cands[i].pos <= p; ++i) {
                    const Cand &c = cands[i];
                    if (c.endpos <= p) continue;
                    if (c.no_lib) { emit(LIB, c.qname); break; }            // pileup_func returns: nothing after it at this site (R:...:281-284)
                    int qpos = 0, indel = 0;
                    if (!resolve(c, p, qpos, indel)) continue;               // is_del
                    if ((int)c.mapq < min_mapq || qpos >= (int)c.qual.size() || (int)c.qual[(size_t)qpos] < min_bq || (c.flag & (4 | 256 | 512 | 1024))) continue;
                    const int calls = (indel != 0 ? 1 : 0) + ((indel < 1 || !ic) ? 1 : 0);
                    for (int k = 0; k < calls; ++k) { if (c.no_sm) emit(SM, c.qname); if (c.no_nm) emit(NM, c.qname); }
                }
            }
        }
        cands.clear(); regs.clear();
    }
    void finish(const int64_t engine_counts[4]) const {
        if (!unlimited) return;
        static const char *nm[NT] = {"SM tag missing", "NM tag missing", "generated tag missing", "library unavailable"};
        for (int t = 0; t < NT; ++t) if (engine_counts[t] > max_per_type) std::fprintf(err, "WARNING: %s: %lld events in total (only the first %lld are listed)\n", nm[t], (long long)engine_counts[t], max_per_type);
    }
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
    std::vector<int32_t> pos, l_qseq, nm, sm; std::vector<uint16_t> flag, lib; std::vector<uint8_t> mapq;
    std::vector<uint64_t> cigar_off, seq_off, qual_off; std::vector<uint32_t> cigar; std::vector<uint8_t> seq, qual;
    std::vector<Warner::Cand> cands; bool cand_overflow = false, error = false; uint64_t n_decoded = 0;
    void clear() {
        pos.clear(); l_qseq.clear(); nm.clear(); sm.clear(); flag.clear(); lib.clear(); mapq.clear();
        cigar_off.assign(1, 0); seq_off.assign(1, 0); qual_off.assign(1, 0); cigar.clear(); seq.clear(); qual.clear();
        cands.clear(); cand_overflow = false; error = false; n_decoded = 0;
    }
    size_t n() const { return pos.size(); }
    void append(const Rec &r, uint16_t l) {
        pos.push_back(r.pos); flag.push_back(r.flag); mapq.push_back(r.mapq); lib.push_back(l); l_qseq.push_back(r.l_qseq);
        nm.push_back(r.nm); sm.push_back(r.sm);
        cigar.insert(cigar.end(), r.cigar, r.cigar + r.n_cigar); cigar_off.push_back(cigar.size());
        seq.insert(seq.end(), r.seq, r.seq + ((size_t)r.l_qseq + 1) / 2); seq_off.push_back(seq.size());
        qual.insert(qual.end(), r.qual, r.qual + r.l_qseq); qual_off.push_back(qual.size());
    }
};

struct PinnedBuf {   // grow-only host buffer: page-locked through the engine when there is one (brc_host_alloc), plain otherwise
    void *p = nullptr; size_t cap = 0; bool pinned = false;
    bool reserve(size_t bytes, bool want_pinned) {
        if (bytes <= cap) return true;
        release();
        const size_t want = bytes + bytes / 8 + 4096;
        if (want_pinned && brc_host_alloc(want, &p) == BRC_OK && p) { pinned = true; cap = want; return true; }
        p = std::malloc(want); pinned = false; cap = p ? want : 0;
        return p != nullptr;
    }
    void release() { if (p) { if (pinned) brc_host_free(p); else std::free(p); } p = nullptr; cap = 0; }
    ~PinnedBuf() { release(); }
    PinnedBuf() = default; PinnedBuf(const PinnedBuf &) = delete; PinnedBuf &operator=(const PinnedBuf &) = delete;
};

struct WindowJob {   // one decoded window: the slices and the concatenated batch
    std::vector<Slice> slices;
    PinnedBuf buf[13];
    brc_read_batch batch{};
    uint64_t n_decoded = 0; bool error = false, cand_overflow = false;
    int tid = -1; int64_t fbeg = 0, fend = 0;
    std::string timing;           // BRC_CLI_TIMING line, printed to the sample's stream by the thread that takes the job
};

struct ParallelFetcher {
    const BamFile &bam; const RgLib &rg_lib; std::string path; int n_threads; bool per_lib, want_pinned;
    std::vector<std::unique_ptr<Bgzf>> readers;
    static constexpr size_t MAX_CANDS = 65536;

    ParallelFetcher(const BamFile &b, const RgLib &rl, const std::string &p, bool pl, bool pin) : bam(b), rg_lib(rl), path(p), per_lib(pl), want_pinned(pin) {
        unsigned hw = std::thread::hardware_concurrency();
        n_threads = (int)std::max(1u, std::min(hw ? hw : 1u, 16u));
        if (const char *ov = std::getenv("BRC_CLI_DECODE_THREADS")) n_threads = std::max(1, std::atoi(ov));
    }
    static bool eligible(int64_t fbeg, int64_t fend) { return fend - fbeg >= (int64_t(1) << 18); }   // >= 16 linear-index windows

    // records of contig `tid` with lo <= pos < hi (first slice: also pos < lo with endpos > fbeg), in file order
    void decode_slice(Bgzf &bz, int tid, int64_t lo, int64_t hi, bool first, int64_t fbeg, bool collect, Slice &out) const {
        out.clear();
        uint64_t voff;
        if (!bam.query_offset(tid, lo, voff)) return;
        if (!bz.seek(voff)) { out.error = bz.error; return; }
        Rec r;
        for (;;) {
            if (!read_record(bz, r)) { out.error = bz.error; break; }
            if (r.tid != tid || r.pos >= hi) break;
            ++out.n_decoded;
            if (r.pos < lo) {
                if (!first) continue;
                r.endpos = rec_endpos(r);
                if (r.endpos <= fbeg) continue;
            }
            if (r.flag & 4) continue;
            const uint16_t lib = rec_lib(r, rg_lib, per_lib);
            if (collect && !out.cand_overflow) {
                Warner::Cand c;
                if (Warner::candidate(r, lib, c)) {
                    if (out.cands.size() >= MAX_CANDS) out.cand_overflow = true;
                    else out.cands.push_back(std::move(c));
                }
            }
            out.append(r, lib);
        }
    }

    // decode [fbeg, fend) of `tid` into job.slices and job.batch; false when a reader could not be opened
    bool run(int tid, int64_t fbeg, int64_t fend, bool collect, WindowJob &job) {
        job.tid = tid; job.fbeg = fbeg; job.fend = fend; job.error = false; job.cand_overflow = false; job.n_decoded = 0; job.timing.clear();
        const int64_t w0 = fbeg >> 14, w1 = (fend + 16383) >> 14;
        const int T = (int)std::max<int64_t>(1, std::min<int64_t>(n_threads, (w1 - w0) / 4));
        while ((int)readers.size() < T) { readers.emplace_back(new Bgzf()); if (!readers.back()->open_worker(path)) return false; }
        job.slices.resize((size_t)T);
        std::vector<int64_t> cut((size_t)T + 1);
        for (int t = 0; t <= T; ++t) cut[(size_t)t] = t == 0 ? fbeg : t == T ? fend : ((w0 + (w1 - w0) * t / T) << 14);
        auto work = [&](int t) { decode_slice(*readers[(size_t)t], tid, cut[(size_t)t], cut[(size_t)t + 1], t == 0, fbeg, collect, job.slices[(size_t)t]); };
        const bool timing = std::getenv("BRC_CLI_TIMING") != nullptr;
        auto clk = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
        const double t0 = clk();
        {
            std::vector<std::thread> th;
            for (int t = 1; t < T; ++t) th.emplace_back(work, t);
            work(0);
            for (auto &x : th) x.join();
        }
        const double t1 = clk();
        // ---- concatenate: prefix sums, then every thread copies its slice ----
        std::vector<size_t> rn((size_t)T + 1, 0), cn((size_t)T + 1, 0), sn((size_t)T + 1, 0), qn((size_t)T + 1, 0);
        for (int t = 0; t < T; ++t) {
            const Slice &sl = job.slices[(size_t)t];
            rn[(size_t)t + 1] = rn[(size_t)t] + sl.n(); cn[(size_t)t + 1] = cn[(size_t)t] + sl.cigar.size();
            sn[(size_t)t + 1] = sn[(size_t)t] + sl.seq.size(); qn[(size_t)t + 1] = qn[(size_t)t] + sl.qual.size();
            job.error = job.error || sl.error; job.cand_overflow = job.cand_overflow || sl.cand_overflow; job.n_decoded += sl.n_decoded;
        }
        const size_t n = rn[(size_t)T];
        const size_t bytes[13] = {n * 4, n * 2, n, n * 2, n * 4, n * 4, n * 4, (n + 1) * 8, cn[(size_t)T] * 4, (n + 1) * 8, sn[(size_t)T], (n + 1) * 8, qn[(size_t)T]};
        for (int k = 0; k < 13; ++k) if (!job.buf[k].reserve(bytes[k] + 64, want_pinned)) return false;
        int32_t *pos = (int32_t *)job.buf[0].p; uint16_t *flag = (uint16_t *)job.buf[1].p; uint8_t *mapq = (uint8_t *)job.buf[2].p; uint16_t *lib = (uint16_t *)job.buf[3].p;
        int32_t *lq = (int32_t *)job.buf[4].p, *nm = (int32_t *)job.buf[5].p, *sm = (int32_t *)job.buf[6].p;
        uint64_t *coff = (uint64_t *)job.buf[7].p; uint32_t *cig = (uint32_t *)job.buf[8].p; uint64_t *soff = (uint64_t *)job.buf[9].p; uint8_t *seq = (uint8_t *)job.buf[10].p;
        uint64_t *qoff = (uint64_t *)job.buf[11].p; uint8_t *qual = (uint8_t *)job.buf[12].p;
        auto copy = [&](int t) {
            const Slice &sl = job.slices[(size_t)t];
            const size_t r0 = rn[(size_t)t], m = sl.n();
            if (m) {
                std::memcpy(pos + r0, sl.pos.data(), m * 4); std::memcpy(flag + r0, sl.flag.data(), m * 2); std::memcpy(mapq + r0, sl.mapq.data(), m);
                std::memcpy(lib + r0, sl.lib.data(), m * 2); std::memcpy(lq + r0, sl.l_qseq.data(), m * 4); std::memcpy(nm + r0, sl.nm.data(), m * 4);
                std::memcpy(sm + r0, sl.sm.data(), m * 4);
                if (!sl.cigar.empty()) std::memcpy(cig + cn[(size_t)t], sl.cigar.data(), sl.cigar.size() * 4);
                if (!sl.seq.empty()) std::memcpy(seq + sn[(size_t)t], sl.seq.data(), sl.seq.size());
                if (!sl.qual.empty()) std::memcpy(qual + qn[(size_t)t], sl.qual.data(), sl.qual.size());
                for (size_t i = 0; i < m; ++i) { coff[r0 + i] = cn[(size_t)t] + sl.cigar_off[i]; soff[r0 + i] = sn[(size_t)t] + sl.seq_off[i]; qoff[r0 + i] = qn[(size_t)t] + sl.qual_off[i]; }
            }
            if (t == T - 1) { coff[n] = cn[(size_t)T]; soff[n] = sn[(size_t)T]; qoff[n] = qn[(size_t)T]; }
        };
        {
            std::vector<std::thread> th;
            for (int t = 1; t < T; ++t) th.emplace_back(copy, t);
            copy(0);
            for (auto &x : th) x.join();
        }
        if (timing) {
            char line[256];
            std::snprintf(line, sizeof line, "[brc timing] window %d:%lld-%lld: %d threads decode %.3fs, concatenate %.3fs (%zu reads)\n", tid, (long long)fbeg, (long long)fend, T, t1 - t0, clk() - t1, n);
            job.timing = line;
        }
        brc_read_batch &b = job.batch;
        b = brc_read_batch{};
        b.n_reads = (int64_t)n; b.tid = nullptr; b.pos = pos; b.flag = flag; b.mapq = mapq; b.lib = lib; b.l_qseq = lq; b.nm = nm; b.sm = sm;
        b.cigar_off = coff; b.cigar = cig; b.seq_off = soff; b.seq = seq; b.qual_off = qoff; b.qual = qual;
        return true;
    }
};

// ------------------------------------------------------------------------------------------
// FASTA + .fai (fai_fetch of a whole chromosome, R:...:87)
// ------------------------------------------------------------------------------------------
struct Fasta {
    std::string path;
    struct Ent { int64_t len, off, lb, lw; };
    std::map<std::string, Ent> ents;
    bool open(const std::string &p) {
        path = p;
        std::ifstream f(p + ".fai");
        if (!f) return false;
        std::string line;
        while (std::getline(f, line)) { std::istringstream ss(line); std::string n; Ent e; if (ss >> n >> e.len >> e.off >> e.lb >> e.lw) ents[n] = e; }
        return true;
    }
    bool fetch(const std::string &name, std::string &out) const {
        auto it = ents.find(name);
        if (it == ents.end()) return false;
        const Ent &e = it->second;
        FILE *f = std::fopen(path.c_str(), "rb");
        if (!f) return false;
        const int64_t n_lines = (e.len + e.lb - 1) / e.lb;
        std::vector<char> raw((size_t)(n_lines * e.lw + 8));
        fseeko(f, (off_t)e.off, SEEK_SET);
        const size_t got = std::fread(raw.data(), 1, raw.size(), f);
        std::fclose(f);
        out.clear(); out.reserve((size_t)e.len);
        for (size_t i = 0; i < got && (int64_t)out.size() < e.len; ++i) if (raw[i] != '\n' && raw[i] != '\r') out.push_back(raw[i]);
        return (int64_t)out.size() == e.len;
    }
};

void usage() {
    std::printf("Usage: bam-readcount [OPTIONS] bam_file|cram_file [region]\nGenerate metrics for bam_file at single nucleotide positions.\n"
                "Example: bam-readcount -f ref.fa some.bam|some.cram\n\nAvailable options:\n"
                "  -h [ --help ]                         produce this message\n"
                "  -v [ --version ]                      output the version number\n"
                "  -q [ --min-mapping-quality ] arg (=0) minimum mapping quality of reads used for counting.\n"
                "  -b [ --min-base-quality ] arg (=0)    minimum base quality at a position to use the read for counting.\n"
                "  -d [ --max-count ] arg (=10000000)    max depth to avoid excessive memory usage.\n"
                "  -l [ --site-list ] arg                file containing a list of regions to report readcounts within.\n"
                "  -f [ --reference-fasta ] arg          reference sequence in the fasta format.\n"
                "  -D [ --print-individual-mapq ] arg    report the mapping qualities as a comma separated list.\n"
                "  -p [ --per-library ]                  report results by library.\n"
                "  -w [ --max-warnings ] arg             maximum number of warnings of each type to emit. -1 gives an unlimited number.\n"
                "  -i [ --insertion-centric ]            generate indel centric readcounts. Reads containing insertions will not be\n"
                "                                        included in per-base counts\n"
                "  --shard RANK/COUNT                    (this host) compute only shard RANK of COUNT: the regions are cut into COUNT runs of\n"
                "                                        about equal BAI-estimated coverage, one process per GPU (BRC_DEVICE); outputs\n"
                "                                        concatenate in rank order\n"
                "  --min-alt-count N                     (this host) print only the sites where an alternative allele (a base other than\n"
                "                                        the reference base, an insertion or a deletion) has a count of at least N\n"
                "  --min-alt-fraction F                  (this host) ... and of at least F times the site's depth (0 <= F <= 1; without\n"
                "                                        --min-alt-count the count must be at least 1).  Printed lines are unchanged\n"
                "  --bam-list FILE                       (this host) run many samples in one process.  Each line of FILE is\n"
                "                                        INPUT<TAB>OUT or INPUT<TAB>OUT<TAB>ERR (ERR defaults to OUT.log); OUT and ERR get\n"
                "                                        exactly what `brc-readcount <options> INPUT <regions>` prints on STDOUT and\n"
                "                                        STDERR.  Every positional argument is a region; a failed sample does not stop\n"
                "                                        the others (exit status 1 at the end)\n"
                "  --vcf FILE                            (this host) write FILE (VCF, plain or bgzip) back to STDOUT with the read counts of\n"
                "                                        each record's REF and SNV / insertion / deletion ALT alleles as FORMAT fields BRC_DP,\n"
                "                                        BRC_AD, BRC_ADF, BRC_ADR and BRC_AF: the values the line of each record's site prints\n"
                "                                        (STDERR is that of -l over the records' sites).  Not with -l, regions, -p,\n"
                "                                        --min-alt-*, --shard or --bam-list\n"
                "  --vcf-sample NAME                     (this host) the sample column that takes the values (required with several; names\n"
                "                                        the column added to a sites-only VCF)\n"
                "  --vcf-samples FILE                    (this host) with --vcf and no positional argument: annotate several sample columns\n"
                "                                        in one process.  Each line of FILE is NAME<TAB>INPUT or NAME<TAB>INPUT<TAB>ERR;\n"
                "                                        NAME's column gets the values of `--vcf-sample NAME INPUT`, ERR (default: STDERR)\n"
                "                                        that run's STDERR.  A failed sample gets '.' and does not stop the others (exit\n"
                "                                        status 1 at the end)\n"
                "  --vcf-complex                         (this host) with --vcf: also count MNP and complex records (an A/C/G/T/N ALT\n"
                "                                        that no printed entry answers) by each read's bases between the two reference\n"
                "                                        bases flanking REF, matched exactly against REF and each ALT\n\n");
}

// samtools region string "name[:beg[-end]]" as bam_parse_region (V:bam_aux.c:65-75) handles it.  Returns 0 when beg and end were
// set; -1 when only the contig is known — a bare name, an open end ("chr:100", "chr:100-": the 64-bit end exceeds INT_MAX so the
// legacy wrapper bails out after setting the contig) or unparsable coordinates: the caller's beg/end keep their previous values
// (initially 0 .. 0x7fffffff; probe with the reference binary: "21:10405200" prints the whole contig, and as a second region it
// repeats the previous one, SURVEY.md A.6).  Thousands separators are accepted ("21:10,402,985-10,402,990").
int parse_region(const BamFile &bam, const std::string &s, int &tid, int &beg, int &end) {
    std::string name = s; tid = -1;
    const size_t colon = s.rfind(':');
    bool ranged = false;
    int64_t b = 0, e = 0;
    if (colon != std::string::npos && bam.tid_of.find(s) == bam.tid_of.end()) {
        std::string coords = s.substr(colon + 1); name = s.substr(0, colon);
        coords.erase(std::remove(coords.begin(), coords.end(), ','), coords.end());
        const char *c = coords.c_str();
        auto digits = [](const char *&q, int64_t &v) { const char *q0 = q; v = 0; while (*q >= '0' && *q <= '9') { v = v * 10 + (*q - '0'); ++q; } return q != q0; };
        if (*c == '-') { ++c; b = 1; ranged = digits(c, e); }                     // "chr:-end": from the first base
        else if (digits(c, b) && *c == '-') { ++c; ranged = digits(c, e); }       // "chr:beg-end"; "chr:beg" / "chr:beg-" stay open
        if (ranged) b = b > 0 ? b - 1 : 0;
    }
    auto it = bam.tid_of.find(name);
    if (it == bam.tid_of.end()) return -1;
    tid = it->second;
    if (!ranged) return -1;
    beg = (int)std::min<int64_t>(b, 0x7fffffff); end = (int)std::min<int64_t>(e, 0x7fffffff);
    return 0;
}

// ------------------------------------------------------------------------------------------
// One sample = what a run on one BAM/CRAM does.  The run is split in two so that a cohort (--bam-list) can open sample k+1
// on a worker thread while sample k computes:
//   open_sample : the input, its header, @RG/LB map, BAI/CRAI, the FASTA index, the region list and its windows, and the
//                 decode of the first window.  Its messages go to Sample::log (Messages).
//   run_sample  : the region loop on the engine handle for the sample's library count; text to a given fd, messages to
//                 stderr, which a cohort points at the sample's ERR file for the time of the sample (htslib writes there too).
// A run on one input calls the same two functions with STDOUT_FILENO and the process's stderr, so each sample of a cohort
// prints exactly the bytes its own run prints.
// ------------------------------------------------------------------------------------------
// ------------------------------------------------------------------------------------------
// --vcf FILE: the per-allele read counts of each VCF record, written back as FORMAT fields (DESIGN.md §12).  A record is
// counted when one of its ALT alleles is an SNV, an insertion after its anchor base or a deletion after it; its site is one
// line "CHROM L L" of a derived -l site list (L = POS, or POS + 1 for a deletion, whose entry prints on the line after the
// anchor), and its values are what that run prints on the line: the engine answers them (brc_set_allele_queries).
// With --vcf-complex a record with an A/C/G/T/N ALT that no entry answers (an MNP, a complex substitution, an indel without
// its anchor base) is counted by the complex rule instead: its site is the line "CHROM POS POS", and the engine matches each
// read's bases between the two flanks of REF against REF and its ALTs (brc_set_complex_queries).
// ------------------------------------------------------------------------------------------
const char kVcfFormat[] = ":BRC_DP:BRC_AD:BRC_ADF:BRC_ADR:BRC_AF";
const char kVcfHeader[] =
    "##FORMAT=<ID=BRC_DP,Number=1,Type=Integer,Description=\"brc-readcount depth of the site's line\">\n"
    "##FORMAT=<ID=BRC_AD,Number=R,Type=Integer,Description=\"brc-readcount count of the REF and each ALT allele\">\n"
    "##FORMAT=<ID=BRC_ADF,Number=R,Type=Integer,Description=\"brc-readcount plus-strand count of the REF and each ALT allele\">\n"
    "##FORMAT=<ID=BRC_ADR,Number=R,Type=Integer,Description=\"brc-readcount minus-strand count of the REF and each ALT allele\">\n"
    "##FORMAT=<ID=BRC_AF,Number=A,Type=Float,Description=\"brc-readcount BRC_AD of each ALT allele over BRC_DP\">\n";

struct VcfRecord {
    std::vector<std::string> cols;
    bool counted = false;
    int32_t line_pos = 0;                 // L: 1-based position of the derived site-list line
    uint32_t ref_kind = 0;                // the REF entry: a base class of "=ACGTN"
    std::vector<int64_t> alt_kind_len;    // per ALT: query kind | length << 8, or -1 when the ALT is not countable
    std::vector<std::string> alt_bases;   // per ALT: an insertion's bases; a complex record: the ALT as upper-case letters
    bool complex = false;                 // counted by the complex rule (--vcf-complex): alt_kind_len 0 for each A/C/G/T/N ALT
    std::string ref;                      // a complex record: REF as upper-case letters
    size_t n_queries = 0;                 // counted: the REF and each countable ALT
    size_t word_off = 0;                  // counted: where its answer words start in a sample's VcfAnswers
};
struct Vcf {
    std::string path;
    std::vector<std::string> header;      // every line before #CHROM
    std::string chrom_line;
    size_t n_cols = 0;
    // the samples that take values, in the order given: each an existing column (target_of_col), or, in a sites-only VCF, a
    // column added after an added FORMAT column
    std::vector<std::string> samples;
    std::vector<int> target_of_col;       // per column: the index in `samples` of the sample it holds, or -1
    std::vector<VcfRecord> rec;
    size_t n_words = 0;                   // answer words of one sample: 1 + 3 * n_queries per counted record
};

// One sample's answers.  For each counted record, at its word_off: the depth of the record's line (0 when it prints none), then
// count, plus and minus of the REF entry and of each countable ALT's entry.  A sample that failed has none.
struct VcfAnswers {
    std::vector<uint32_t> words;
    std::vector<uint8_t> answered;        // per record: its words are set (counted, and its contig is in the sample's input)
    bool failed = false;
    explicit VcfAnswers(const Vcf &v) : words(v.n_words), answered(v.rec.size()) {}
};

std::vector<std::string> split(const std::string &s, char c) {
    std::vector<std::string> out; size_t p = 0;
    for (size_t t; (t = s.find(c, p)) != std::string::npos; p = t + 1) out.push_back(s.substr(p, t - p));
    out.push_back(s.substr(p));
    return out;
}

// the whole file, plain or BGZF (bgzip); false with a message
bool read_vcf_bytes(const std::string &path, std::string &out, std::string &why) {
    FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) { why = "cannot open " + path + ": " + std::strerror(errno); return false; }
    uint8_t head[512]; const size_t got = std::fread(head, 1, sizeof head, f);
    if (got < 2 || head[0] != 31 || head[1] != 139) {
        out.assign((const char *)head, got);
        char buf[1 << 16];
        for (size_t n; (n = std::fread(buf, 1, sizeof buf, f)) > 0;) out.append(buf, n);
        const bool bad = std::ferror(f);
        std::fclose(f);
        if (bad) why = "cannot read " + path;
        return !bad;
    }
    std::fclose(f);
    size_t hdr = 0;
    if (!Bgzf::block_size(head, got, hdr)) { why = path + " is gzip-compressed but not BGZF: compress it with bgzip"; return false; }
    Bgzf bz;
    if (!bz.open(path)) { why = "cannot open " + path; return false; }
    for (uint64_t coff = 0; bz.load_block(coff); coff = bz.next_coff) out.append((const char *)bz.block.data(), bz.block.size());
    if (bz.error) { why = path + ": truncated or corrupt BGZF block"; return false; }
    return true;
}

// Parses the whole VCF, applies the allele rule and resolves the samples that take values: `samples` as named by option `opt`,
// or none given (the VCF's only sample column).  False with a message (nothing may have been written yet).
bool parse_vcf(const std::string &path, const std::vector<std::string> &samples, const char *opt, bool complex_on, Vcf &v,
               std::string &why) {
    std::string text;
    if (!read_vcf_bytes(path, text, why)) return false;
    v.path = path;
    auto up = [](std::string s) { for (char &c : s) c = (char)std::toupper((unsigned char)c); return s; };
    auto acgtn = [](const std::string &s, size_t from) {
        if (s.size() <= from) return false;
        for (size_t i = from; i < s.size(); ++i) if (!std::strchr("ACGTN", s[i]) || !s[i]) return false;
        return true;
    };
    auto kind_of = [](char c) { return (uint32_t)(std::strchr("=ACGTN", c) - "=ACGTN"); };
    bool in_header = true;
    size_t ln = 0;
    for (size_t p = 0; p < text.size();) {
        size_t e = text.find('\n', p);
        if (e == std::string::npos) e = text.size();
        std::string line = text.substr(p, e - p);
        p = e + 1; ++ln;
        const std::string at = path + ": line " + std::to_string(ln) + ": ";
        if (in_header && line.compare(0, 2, "##") == 0) {
            if (line.compare(0, 16, "##FORMAT=<ID=BRC") == 0 && line.size() > 16 && line[16] == '_') { why = at + "the header already declares a BRC_* FORMAT field"; return false; }
            v.header.push_back(line);
            continue;
        }
        if (in_header && line.compare(0, 6, "#CHROM") == 0) {
            v.chrom_line = line; v.n_cols = split(line, '\t').size(); in_header = false;
            if (v.n_cols < 8) { why = at + "the #CHROM line has fewer than 8 columns"; return false; }
            if (v.n_cols == 9) { why = at + "a FORMAT column without sample columns"; return false; }
            continue;
        }
        if (in_header) { why = at + "data before the #CHROM header line"; return false; }
        VcfRecord r;
        r.cols = split(line, '\t');
        if (r.cols.size() < 8) { why = at + "fewer than 8 columns"; return false; }
        if (r.cols.size() != v.n_cols) { why = at + std::to_string(r.cols.size()) + " columns, the #CHROM line has " + std::to_string(v.n_cols); return false; }
        const std::string &ps = r.cols[1];
        int64_t pos = 0;
        bool ok = !ps.empty() && ps.size() <= 10;
        for (char c : ps) ok = ok && c >= '0' && c <= '9';
        if (ok) pos = std::atoll(ps.c_str());
        if (!ok || pos < 1 || pos >= INT32_MAX) { why = at + "POS is not a positive integer below 2^31 - 1"; return false; }
        const std::string ref = up(r.cols[3]);
        const bool ref_ok = acgtn(ref, 0);
        std::vector<std::string> alts;
        for (const std::string &a0 : split(r.cols[4], ',')) {
            const std::string a = up(a0);
            alts.push_back(a);
            int64_t kl = -1; std::string bases;
            if (ref_ok && ref.size() == 1 && a.size() == 1 && acgtn(a, 0)) kl = kind_of(a[0]);
            else if (ref_ok && ref.size() == 1 && a.size() >= 2 && a[0] == ref[0] && acgtn(a, 1)) { kl = BRC_KIND_INS | (int64_t)(a.size() - 1) << 8; bases = a.substr(1); }
            else if (ref_ok && ref.size() >= 2 && a.size() == 1 && a[0] == ref[0]) kl = BRC_KIND_DEL | (int64_t)(ref.size() - 1) << 8;
            r.counted = r.counted || kl >= 0;
            r.complex = r.complex || (complex_on && pos >= 2 && ref_ok && kl < 0 && acgtn(a, 0));
            r.alt_kind_len.push_back(kl); r.alt_bases.push_back(bases);
        }
        if (r.complex) {      // the whole record by the complex rule: the REF and every A/C/G/T/N ALT
            r.counted = true; r.line_pos = (int32_t)pos; r.ref = ref;
            for (size_t i = 0; i < alts.size(); ++i) {
                r.alt_kind_len[i] = acgtn(alts[i], 0) ? 0 : -1;
                r.alt_bases[i] = r.alt_kind_len[i] >= 0 ? alts[i] : "";
            }
        }
        if (r.counted) {
            if (!r.complex) { r.line_pos = (int32_t)(ref.size() == 1 ? pos : pos + 1); r.ref_kind = kind_of(ref[ref.size() == 1 ? 0 : 1]); }
            r.n_queries = 1 + (size_t)std::count_if(r.alt_kind_len.begin(), r.alt_kind_len.end(), [](int64_t x) { return x >= 0; });
            r.word_off = v.n_words; v.n_words += 1 + 3 * r.n_queries;
        }
        v.rec.push_back(std::move(r));
    }
    if (in_header) { why = path + ": no #CHROM header line"; return false; }
    const std::vector<std::string> hc = split(v.chrom_line, '\t');
    v.target_of_col.assign(v.n_cols, -1);
    if (v.n_cols == 8) {
        if (samples.empty()) { why = path + " has no sample column: --vcf-sample NAME names the one added"; return false; }
        v.samples = samples;
        return true;
    }
    if (samples.empty()) {
        if (hc.size() > 10) { why = path + " has " + std::to_string(hc.size() - 9) + " sample columns: --vcf-sample NAME is required"; return false; }
        v.samples.assign(1, hc[9]); v.target_of_col[9] = 0;
        return true;
    }
    for (size_t t = 0; t < samples.size(); ++t) {
        int n_match = 0, col = -1;
        for (size_t c = 9; c < hc.size(); ++c) if (hc[c] == samples[t]) { ++n_match; col = (int)c; }
        if (n_match == 0) { why = std::string(opt) + " " + samples[t] + ": no such sample in " + path; return false; }
        if (n_match > 1) { why = std::string(opt) + " " + samples[t] + " is ambiguous: " + std::to_string(n_match) + " sample columns of " + path + " have that name"; return false; }
        v.target_of_col[(size_t)col] = (int)t;
    }
    v.samples = samples;
    return true;
}

bool write_all(int fd, const std::string &s) {
    for (size_t done = 0; done < s.size();) {
        const ssize_t w = ::write(fd, s.data() + done, s.size() - done);
        if (w < 0) { if (errno == EINTR) continue; return false; }
        done += (size_t)w;
    }
    return true;
}

// Record ri's five values in one sample from its answer words (REF first, then each countable ALT in order).  A record the
// sample did not answer, and every record of a failed sample, gets '.' in all five.
void vcf_values(const Vcf &v, size_t ri, const VcfAnswers &a, std::string &out) {
    if (a.failed || !a.answered[ri]) { out += ".:.:.:.:."; return; }
    const VcfRecord &r = v.rec[ri];
    const uint32_t *w = a.words.data() + r.word_off;
    const uint32_t dp = w[0];
    std::string ad, adf, adr, af;
    auto put = [&](const uint32_t *q) {
        ad += q ? std::to_string(q[0]) : "."; adf += q ? std::to_string(q[1]) : "."; adr += q ? std::to_string(q[2]) : ".";
    };
    put(w + 1);
    size_t k = 1;
    for (size_t i = 0; i < r.alt_kind_len.size(); ++i) {
        const uint32_t *q = r.alt_kind_len[i] >= 0 ? w + 1 + 3 * k++ : nullptr;
        ad += ','; adf += ','; adr += ',';
        put(q);
        if (i) af += ',';
        if (!q || dp == 0) { af += '.'; continue; }
        char b[64]; std::snprintf(b, sizeof b, "%.6g", (double)q[0] / (double)dp);
        af += b;
    }
    out += std::to_string(dp); out += ':'; out += ad; out += ':'; out += adf; out += ':'; out += adr; out += ':'; out += af;
}

// Record ri's line, appended to `out`: the values of sample t from ans[t] in that sample's column.
void vcf_line(const Vcf &v, size_t ri, const VcfAnswers *ans, std::string &out) {
    const VcfRecord &r = v.rec[ri];
    const size_t n = r.cols.size();
    for (size_t c = 0; c < n; ++c) {
        if (c) out += '\t';
        out += r.cols[c];
        if (c == 8) { out += kVcfFormat; continue; }
        const int t = v.target_of_col[c];
        if (t < 0) continue;
        const size_t keys = (size_t)std::count(r.cols[8].begin(), r.cols[8].end(), ':') + 1;
        for (size_t have = (size_t)std::count(r.cols[c].begin(), r.cols[c].end(), ':') + 1; have < keys; ++have) out += ":.";
        out += ':';
        vcf_values(v, ri, ans[t], out);
    }
    if (n == 8) {
        out += '\t'; out += kVcfFormat + 1;
        for (size_t t = 0; t < v.samples.size(); ++t) { out += '\t'; vcf_values(v, ri, ans[t], out); }
    }
    out += '\n';
}

std::string vcf_header(const Vcf &v) {
    std::string out;
    for (const std::string &h : v.header) { out += h; out += '\n'; }
    out += kVcfHeader;
    out += v.chrom_line;
    if (v.n_cols == 8) { out += "\tFORMAT"; for (const std::string &s : v.samples) { out += '\t'; out += s; } }
    out += '\n';
    return out;
}

// A batch's answers into sample `a`'s words: record ri's queries are ans[0 .. n_queries) (brc_get_allele_answers' order).
void vcf_store(const Vcf &v, size_t ri, const brc_allele_answer *ans, VcfAnswers &a) {
    const VcfRecord &r = v.rec[ri];
    uint32_t *w = a.words.data() + r.word_off;
    w[0] = ans[0].line ? ans[0].depth : 0;
    for (size_t k = 0; k < r.n_queries; ++k) {
        w[1 + 3 * k] = ans[k].stats[BRC_S_COUNT]; w[2 + 3 * k] = ans[k].stats[BRC_S_PLUS]; w[3 + 3 * k] = ans[k].stats[BRC_S_MINUS];
    }
    a.answered[ri] = 1;
}
// A complex record's answer (brc_get_complex_answers): the reads that count, then per allele (REF first) count, plus, minus.
void vcf_store_complex(const Vcf &v, size_t ri, uint32_t depth, const brc_complex_count *c, VcfAnswers &a) {
    const VcfRecord &r = v.rec[ri];
    uint32_t *w = a.words.data() + r.word_off;
    w[0] = depth;
    for (size_t k = 0; k < r.n_queries; ++k) { w[1 + 3 * k] = c[k].count; w[2 + 3 * k] = c[k].plus; w[3 + 3 * k] = c[k].count - c[k].plus; }
    a.answered[ri] = 1;
}

struct Options {   // everything on the command line except the inputs: the same for every sample
    int min_mapq = 0, min_bq = 0, max_cnt = 10000000; bool per_lib = false, ic = false; long long max_warn = -1;
    const Vcf *vcf = nullptr;     // --vcf: the parsed file
    bool vcf_samples = false;     // --vcf-samples: a sample only fills its answers; the VCF is written after the last sample
    bool vcf_complex = false;     // --vcf-complex: MNP and complex records are counted too (DESIGN.md §12)
    std::string fn_pos, fn_fa, dist_arg;
    std::vector<std::string> region_args;
    int shard_rank = 0, shard_count = 1;
    bool site_filter = false; brc_site_filter filter{};
    bool decode_only = false, device_decode = false, timing = false;
    bool dist_refused() const { return dist_arg == "1" || dist_arg == "true"; }
};

double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// The messages of open_sample.  A run on one input prints them as they come (`live` = stderr), between whatever the libraries
// it calls print themselves; a cohort opening the next sample under the current one holds them until that sample runs.
struct Messages {
    FILE *live = nullptr;
    std::string held;
    void say(const char *fmt, ...) __attribute__((format(printf, 2, 3))) {
        va_list ap;
        if (live) { va_start(ap, fmt); std::vfprintf(live, fmt, ap); va_end(ap); return; }
        va_start(ap, fmt); const int n = std::vsnprintf(nullptr, 0, fmt, ap); va_end(ap);
        if (n <= 0) return;
        std::string line((size_t)n + 1, '\0');
        va_start(ap, fmt); std::vsnprintf(&line[0], line.size(), fmt, ap); va_end(ap);
        line.pop_back();
        held += line;
    }
};

struct Region { int tid, beg, end; bool site_list; bool cont = false; };   // cont: a later window of a cut region (its halo site belongs to the window before)

// the end of region g's fetch, clamped to the contig's length (a region that starts beyond the contig keeps one base)
int64_t fetch_end(const BamFile &bam, const Region &g) {
    return std::min<int64_t>(g.end, std::max<int64_t>(bam.lens[(size_t)g.tid], (int64_t)g.beg + 1));
}

struct Sample {
    const Options &o;
    std::string path; bool is_cram = false;
    Messages log;                 // the run's STDERR up to its region loop (held when opened ahead of its turn)
    int status = 1;               // 0 once open_sample got to the end; otherwise the run exits 1 after printing `log`
    double t0 = 0;                // when opening began
    BamFile bam;
#ifdef BRC_WITH_HTSLIB
    HtsSource hts;
#endif
    Fasta fa; bool have_fa = false;
    RgLib rg_lib;
    std::vector<std::string> lib_names; std::vector<const char *> lib_ptrs;
    std::vector<Region> regions;
    std::vector<int64_t> vcf_region;   // --vcf: per record, the index of its site-list region (-1: not counted, or contig not in the BAM)
    Warner warner;
    // big fetches (windows of a cut region) of a BAM are decoded by several threads, one window ahead of the engine
    // (ParallelFetcher), unless the engine decodes the file itself (BRC_CLI_DEVICE_DECODE)
    ParallelFetcher pf;
    bool allow_parallel = false;
    WindowJob *jobs;              // the process's two window jobs (page-locked buffers), used by one sample at a time
    std::future<bool> ahead; size_t ahead_gi = (size_t)-1; int ahead_slot = 0;   // waited for when the sample goes
    bool par_decode_error = false; uint64_t par_decoded = 0, par_windows = 0;

    Sample(const Options &opt, const std::string &p, WindowJob *pool)
        : o(opt), path(p), warner(opt.max_warn, opt.min_mapq, opt.min_bq, opt.per_lib, opt.ic), pf(bam, rg_lib, p, opt.per_lib, !opt.decode_only), jobs(pool) {}
    Sample(const Sample &) = delete; Sample &operator=(const Sample &) = delete;

    void fetch_range(size_t gi, int64_t &fb, int64_t &fe) const {
        fb = std::max<int64_t>((int64_t)regions[gi].beg - 1, 0);
        fe = fetch_end(bam, regions[gi]);
    }
    bool par_ok(size_t gi) const {
        if (!allow_parallel || gi >= regions.size()) return false;
        int64_t fb, fe; fetch_range(gi, fb, fe);
        return ParallelFetcher::eligible(fb, fe);
    }
    std::future<bool> start_decode(size_t gi, int slot) {
        int64_t fb, fe; fetch_range(gi, fb, fe);
        const int tid = regions[gi].tid; const bool collect = warner.collecting();
        WindowJob *job = &jobs[slot]; ParallelFetcher *pfp = &pf;
        return std::async(std::launch::async, [pfp, job, tid, fb, fe, collect] { return pfp->run(tid, fb, fe, collect, *job); });
    }
    // the decoded window for region gi (prefetched or decoded now); nullptr = take the sequential path
    WindowJob *decoded_window(size_t gi) {
        int slot = 0; bool ok;
        if (ahead.valid() && ahead_gi == gi) { ok = ahead.get(); slot = ahead_slot; }
        else { if (ahead.valid()) ahead.get(); ok = start_decode(gi, 0).get(); }
        ahead_gi = (size_t)-1;
        WindowJob *job = &jobs[slot];
        if (!job->timing.empty()) { std::fputs(job->timing.c_str(), warner.err); job->timing.clear(); }
        if (ok && gi + 1 < regions.size() && par_ok(gi + 1)) { ahead_slot = slot ^ 1; ahead_gi = gi + 1; ahead = start_decode(gi + 1, ahead_slot); }
        if (!ok) return nullptr;
        if (job->cand_overflow && warner.collecting()) return nullptr;      // a BAM full of untagged reads: the per-read warning replay wants them all
        par_decode_error = par_decode_error || job->error; par_decoded += job->n_decoded; ++par_windows;
        return job;
    }
    bool uses_windows() const { for (size_t gi = 0; gi < regions.size(); ++gi) if (par_ok(gi)) return true; return false; }
    int64_t next_fbeg(size_t gi) const {   // start of the following fetch when it continues this one, else "keep nothing"
        if (gi + 1 >= regions.size() || regions[gi + 1].tid != regions[gi].tid) return INT64_MAX;
        return std::max<int64_t>((int64_t)regions[gi + 1].beg - 1, 0);
    }
};

bool is_cram_path(const std::string &p) { return p.size() > 5 && p.substr(p.size() - 5) == ".cram"; }

// `live`: print the messages as they come (else hold them in s.log).  `first_window`: start decoding the first window into
// `pool` (only when no other sample is using it).
std::unique_ptr<Sample> open_sample(const Options &o, const std::string &bam_path, double t0, FILE *live, WindowJob *pool, bool first_window) {
    std::unique_ptr<Sample> sp(new Sample(o, bam_path, pool));
    Sample &s = *sp; Messages &log = s.log; BamFile &bam = s.bam;
    s.t0 = t0; log.live = live;
    log.say("Minimum mapping quality is set to %d\n", o.min_mapq);
    if (o.dist_refused()) { log.say("Not currently supporting distributions\n"); return sp; }
    s.is_cram = is_cram_path(bam_path);
#ifdef BRC_WITH_HTSLIB
    if (s.is_cram) { if (!s.hts.open(bam_path, o.fn_fa, bam)) { log.say("Fail to open BAM file %s\n", bam_path.c_str()); return sp; } }
    else
#else
    if (s.is_cram) { log.say("CRAM input needs a host built with htslib (tools/build_htslib.sh, then python -m bam_readcount_b200.build); convert to BAM\n"); return sp; }
#endif
    if (!bam.open(bam_path)) { log.say("Fail to open BAM file %s\n", bam_path.c_str()); return sp; }
    s.have_fa = !o.fn_fa.empty() && s.fa.open(o.fn_fa);
    if (!o.fn_fa.empty() && !s.have_fa) { log.say("Fail to open reference file %s\n", o.fn_fa.c_str()); return sp; }

    // @RG ID -> rank of its LB: the first @RG line of an ID wins, libraries in std::set order (R:...:92-111, 526-529)
    std::set<std::string> libs; std::vector<std::pair<std::string, std::string>> id_lb;
    {
        std::istringstream ss(bam.text); std::string line;
        while (std::getline(ss, line)) {
            if (line.compare(0, 3, "@RG") != 0) continue;
            std::istringstream ls(line); std::string tok, id, lb; bool has_lb = false;
            while (std::getline(ls, tok, '\t')) { if (tok.compare(0, 3, "ID:") == 0) id = tok.substr(3); else if (tok.compare(0, 3, "LB:") == 0) { lb = tok.substr(3); has_lb = true; } }
            if (has_lb) { libs.insert(lb); if (!id.empty()) id_lb.emplace_back(id, lb); }
        }
    }
    for (const auto &l : libs) log.say("Expect library: %s in BAM\n", l.c_str());
    s.lib_names.assign(libs.begin(), libs.end());
    for (const auto &p : id_lb)
        s.rg_lib.emplace(p.first, (uint16_t)(std::lower_bound(s.lib_names.begin(), s.lib_names.end(), p.second) - s.lib_names.begin()));
    for (auto &n : s.lib_names) s.lib_ptrs.push_back(n.c_str());
    if (s.lib_ptrs.empty()) s.lib_ptrs.push_back("");

    if (o.fn_pos.empty() && o.region_args.empty() && !o.vcf) {
        log.say("Whole-file mode is not supported (the reference skips its per-read pre-processing there, R:...:624); give regions or -l\n");
        return sp;
    }
#ifdef BRC_WITH_HTSLIB
    if (s.is_cram) { if (!s.hts.load_index(bam_path)) { log.say("BAM indexing file is not available.\n"); return sp; } }
    else
#endif
    if (!bam.load_index(bam_path)) { log.say("BAM indexing file is not available.\n"); return sp; }
    if (!s.have_fa && !o.decode_only) { log.say("A reference FASTA (-f) is required in region / site-list mode\n"); return sp; }

    std::vector<Region> &regions = s.regions;
    // one line "name b e" of a site list: its region, or the -l loop's message when the BAM has no such contig
    auto site_line = [&](const std::string &name, int b, int e) {
        auto it = bam.tid_of.find(name);
        if (it == bam.tid_of.end()) { log.say("%s not found in bam file. Region %s %i %i skipped.\n", name.c_str(), name.c_str(), b, e); return false; }
        regions.push_back({it->second, b - 1, e, true});
        return true;
    };
    if (o.vcf) {          // the derived site list: one line per counted record, in file order
        for (const VcfRecord &r : o.vcf->rec)
            s.vcf_region.push_back(r.counted && site_line(r.cols[0], r.line_pos, r.line_pos) ? (int64_t)regions.size() - 1 : -1);
    } else if (!o.fn_pos.empty()) {
        std::ifstream fp(o.fn_pos);
        if (!fp) { log.say("Failed to open region list file: %s\n", o.fn_pos.c_str()); return sp; }
        std::string line;
        while (std::getline(fp, line)) {
            std::istringstream ss(line); std::string name; int b, e;
            if (!(ss >> name >> b >> e)) continue;
            site_line(name, b, e);
        }
    } else {
        int beg = 0, end = 0x7fffffff;
        for (const auto &rs : o.region_args) {
            int tid;
            parse_region(bam, rs, tid, beg, end);
            if (tid < 0) { log.say("Invalid region %s\n", rs.c_str()); return sp; }
            regions.push_back({tid, beg, end, false});
        }
    }

    // Long regions are cut into consecutive windows so host staging and result buffers stay bounded (a 250 Mb chromosome
    // at 30x would otherwise need tens of GB).  A window is just a region of the -l loop: it recomputes the site to its left
    // (the 1-site halo), so the concatenated output equals the unsplit region's.  Only the last window of an argv region keeps
    // argv semantics.  (With a tiny -d the max-count rule sees the window's own fetch order; SURVEY.md §8e.)
    s.allow_parallel = !s.is_cram && !o.device_decode;
    {
        // 2 Mb windows: each is decoded by all threads in ~40 ms one window ahead of the engine and needs 110 MB of page-locked memory
        // (8 Mb windows were 0.6 s slower on a 10 Mb BAM, r02t); the record-by-record paths (CRAM, device decode) keep 8 Mb
        int64_t W = std::getenv("BRC_CLI_WINDOW") ? std::atoll(std::getenv("BRC_CLI_WINDOW")) : (s.allow_parallel ? 2000000 : 8000000);
        if (o.shard_count > 1 && !std::getenv("BRC_CLI_WINDOW")) W = 1000000;      // finer units so the shards can balance
        std::vector<Region> cut;
        for (const Region &g : regions) {
            const int64_t e_eff = fetch_end(bam, g);
            if (e_eff - g.beg <= W) { cut.push_back(g); continue; }
            for (int64_t b = g.beg; b < e_eff; b += W) {
                const bool last = b + W >= e_eff;
                Region w{g.tid, (int)b, last ? g.end : (int)(b + W), last ? g.site_list : true};
                w.cont = b != g.beg;
                cut.push_back(w);
            }
        }
        regions.swap(cut);
    }

    // --shard RANK/COUNT: one process per GPU (SURVEY.md §8e).  The (windowed) regions are the units; each unit's weight is the
    // compressed-byte span the BAI linear index gives for it — the coverage estimate the index offers without touching the data
    // — and the units are cut into COUNT contiguous runs of about equal weight; this process computes run RANK.  Units are
    // independent (every window recomputes its left halo site), so the concatenation of the ranks' outputs in rank order is the
    // unsharded output; only the reference's never-cleared argv deletion queue does not cross a shard boundary.
    if (o.shard_count > 1) {
        const int shard_rank = o.shard_rank, shard_count = o.shard_count;
        std::vector<double> wgt(regions.size(), 1.0);
        for (size_t i = 0; i < regions.size(); ++i) {
            const Region &g = regions[i];
            const int64_t e_eff = fetch_end(bam, g);
            double w = (double)std::max<int64_t>(e_eff - g.beg, 1) * 0.05;                 // no index information: 0.05 bytes per base
            if (g.tid < (int)bam.idx.size() && !bam.idx[(size_t)g.tid].linear.empty()) {
                const auto &lin = bam.idx[(size_t)g.tid].linear;
                auto off_at = [&](int64_t p) { int64_t k = std::min<int64_t>(std::max<int64_t>(p >> 14, 0), (int64_t)lin.size() - 1); while (k > 0 && lin[(size_t)k] == 0) --k; return (double)(lin[(size_t)k] >> 16); };
                const double d = off_at(e_eff + 16384) - off_at(g.beg);
                if (d > 0) w = d * (double)(e_eff - g.beg) / (double)((((e_eff + 16384) >> 14) - (g.beg >> 14)) * 16384);
            }
            wgt[i] = w;
        }
        double tot = 0; for (double w : wgt) tot += w;
        std::vector<size_t> cutpt((size_t)shard_count + 1, regions.size()); cutpt[0] = 0;
        { double acc = 0; int r = 1; for (size_t i = 0; i < regions.size() && r < shard_count; ++i) { acc += wgt[i]; while (r < shard_count && acc >= tot * r / shard_count) cutpt[(size_t)r++] = i + 1; } }
        std::vector<Region> mine(regions.begin() + (long)cutpt[(size_t)shard_rank], regions.begin() + (long)cutpt[(size_t)shard_rank + 1]);
        if (o.timing) log.say("[brc shard] %d/%d: units %zu..%zu of %zu\n", shard_rank, shard_count, cutpt[(size_t)shard_rank], cutpt[(size_t)shard_rank + 1], regions.size());
        regions.swap(mine);
    }

    // decode under the CUDA start-up (first sample) or under the previous sample's compute (cohort)
    if (first_window && !regions.empty() && s.par_ok(0)) { s.ahead_slot = 0; s.ahead_gi = 0; s.ahead = s.start_decode(0, 0); }
    s.status = 0;
    return sp;
}

// ------------------------------------------------------------------------------------------
// The engine handles of a process.  One CUDA context, brought up once by a throw-away engine on a thread of its own while the
// first sample is opened.  A handle's library rows are fixed at brc_create, so under -p there is one handle per library count,
// kept and reused by the later samples with that count (brc_create allocates nothing on the device until first use); without
// -p every sample shares one handle.  Each handle remembers which contig it holds the reference of for every tid: tids are
// per-header, so the reference is uploaded again only when a sample's tid names another contig.
// ------------------------------------------------------------------------------------------
struct Engines {
    brc_config cfg{};
    std::thread warm; int warm_rc = BRC_OK;
    struct Handle { brc_engine *eng = nullptr; std::unordered_map<int, std::string> ref_name; };
    std::map<int32_t, Handle> handles;

    void start_warm() {
        brc_config w = cfg; w.per_lib = 0;
        warm = std::thread([this, w] { brc_engine *tmp = nullptr; warm_rc = brc_create(&w, &tmp); if (tmp) brc_destroy(tmp); });
    }
    // the handle for a sample with n_libs libraries; nullptr (message on err) when it cannot be created
    Handle *get(int32_t n_libs, const Options &o, FILE *err) {
        if (warm.joinable()) warm.join();
        const int32_t key = cfg.per_lib ? n_libs : 0;
        auto it = handles.find(key);
        if (it != handles.end()) return &it->second;
        brc_config c = cfg; c.n_libs = n_libs;
        brc_engine *eng = nullptr;
        const int rc = warm_rc != BRC_OK ? warm_rc : brc_create(&c, &eng);
        if (rc != BRC_OK) { std::fprintf(err, "brc_create: %s\n", brc_strerror(rc)); return nullptr; }
        if (o.site_filter && brc_set_site_filter(eng, &o.filter) != BRC_OK) { std::fprintf(err, "brc_set_site_filter: %s\n", brc_last_error(eng)); brc_destroy(eng); return nullptr; }
        Handle &h = handles[key]; h.eng = eng;
        return &h;
    }
    void destroy() { for (auto &kv : handles) brc_destroy(kv.second.eng); handles.clear(); }
    ~Engines() { if (warm.joinable()) warm.join(); }
};

// One sample's region loop (the two loops of the reference, R:...:574-608 and 641-657): text to out_fd, messages to err.
// With --vcf the answers go to `vcf_ans`, and a single-sample run streams the VCF to out_fd as its batches complete.
// Returns the exit status of the run on this input alone (0 or 1), or -1 when no engine could be created.
int run_sample(const Options &o, Engines &engines, Sample &s, int out_fd, FILE *err, double t_main0, VcfAnswers *vcf_ans) {
    std::fputs(s.log.held.c_str(), err);
    if (s.status != 0) return 1;
    s.warner.err = err;
    BamFile &bam = s.bam; const std::vector<Region> &regions = s.regions; Warner &warner = s.warner;
    const std::vector<const char *> &lib_ptrs = s.lib_ptrs;
    Engines::Handle *h = nullptr; brc_engine *eng = nullptr;
    if (!o.decode_only) {
        if (!(h = engines.get((int32_t)s.lib_names.size(), o, err))) return -1;
        eng = h->eng;
        // nothing left from an earlier sample: no pushed reads (a sample that failed mid-way) and no queued deletion
        // (switching the carry empties the queue); the argv loop's queue is then carried across this sample's flushes
        brc_reset(eng); brc_set_queue_carry(eng, 0); brc_set_queue_carry(eng, 1);
    }

    std::string chrom;
    double t_decode = 0, t_compute = 0, t_format = 0, t_ref = 0, t_results = 0, t_reset = 0, ms_alleles = 0, ms_complex = 0;
    // BRC_CLI_DEVICE_DECODE=1: BGZF inflate + BAM framing on the GPU (per-read warning lines need host-decoded reads: counts only)
    std::vector<const char *> rg_ids; std::vector<uint16_t> rg_libs;
    for (const auto &kv : s.rg_lib) { rg_ids.push_back(kv.first.c_str()); rg_libs.push_back(kv.second); }
    int64_t warn_total[4] = {0, 0, 0, 0};
    // --vcf: a single-sample run writes the records in file order, each once its region's batch is computed
    const Vcf *vcf = o.vcf;
    const bool vcf_stream = vcf && !o.vcf_samples && !o.decode_only;
    std::vector<int64_t> vcf_rec_of_region(regions.size(), -1);
    for (size_t k = 0; k < s.vcf_region.size(); ++k) if (s.vcf_region[k] >= 0) vcf_rec_of_region[(size_t)s.vcf_region[k]] = (int64_t)k;
    size_t vcf_next = 0;
    auto vcf_write = [&](int64_t regions_done) {     // every record not yet written whose region is done (or that has none)
        std::string out;
        for (; vcf_next < s.vcf_region.size() && s.vcf_region[vcf_next] < regions_done; ++vcf_next) vcf_line(*vcf, vcf_next, vcf_ans, out);
        return write_all(out_fd, out);
    };
    if (vcf_stream && !write_all(out_fd, vcf_header(*vcf))) { std::fprintf(err, "writing the VCF: %s\n", std::strerror(errno)); return 1; }
    int64_t batch_first = 0, batch_n = 0;            // the regions begun since the last brc_reset
    auto flush = [&]() -> int {
        int r;
        std::vector<brc_allele_query> q;
        std::string q_bases;
        std::vector<brc_complex_query> cq; std::vector<brc_complex_allele> ca; std::string c_bases;
        if (vcf) {            // the REF entry and every countable ALT of each record of the batch
            for (int64_t g = 0; g < batch_n; ++g) {
                const VcfRecord &rec = vcf->rec[(size_t)vcf_rec_of_region[(size_t)(batch_first + g)]];
                if (rec.complex) {      // the REF and every A/C/G/T/N ALT, matched against the reads' bases between the flanks
                    cq.push_back({g, rec.line_pos - 1, (int32_t)rec.ref.size(), (int32_t)rec.n_queries, 0});
                    ca.push_back({(int64_t)c_bases.size(), (int32_t)rec.ref.size(), 0}); c_bases += rec.ref;
                    for (size_t i = 0; i < rec.alt_kind_len.size(); ++i)
                        if (rec.alt_kind_len[i] >= 0) { ca.push_back({(int64_t)c_bases.size(), (int32_t)rec.alt_bases[i].size(), 0}); c_bases += rec.alt_bases[i]; }
                    continue;
                }
                q.push_back({g, rec.line_pos - 1, rec.ref_kind, 0});
                for (size_t i = 0; i < rec.alt_kind_len.size(); ++i)
                    if (rec.alt_kind_len[i] >= 0) { q.push_back({g, rec.line_pos - 1, (uint32_t)rec.alt_kind_len[i], (int64_t)q_bases.size()}); q_bases += rec.alt_bases[i]; }
            }
            if ((r = brc_set_allele_queries(eng, q.data(), (int64_t)q.size(), q_bases.data(), (int64_t)q_bases.size())) != BRC_OK) { std::fprintf(err, "brc_set_allele_queries: %s\n", brc_last_error(eng)); return r; }
            if (!cq.empty() && (r = brc_set_complex_queries(eng, cq.data(), (int64_t)cq.size(), ca.data(), (int64_t)ca.size(), c_bases.data(), (int64_t)c_bases.size())) != BRC_OK) { std::fprintf(err, "brc_set_complex_queries: %s\n", brc_last_error(eng)); return r; }
        }
        const double c0 = now();
        r = brc_compute(eng);
        t_compute += now() - c0;
        if (r != BRC_OK) { std::fprintf(err, "brc_compute: %s\n", brc_last_error(eng)); return r; }
        brc_results res{};
        const double g0 = now();
        if (vcf) {
            const brc_allele_answer *ans = nullptr; int64_t n_ans = 0;
            if ((r = brc_get_allele_answers(eng, &ans, &n_ans)) != BRC_OK || n_ans != (int64_t)q.size()) { std::fprintf(err, "brc_get_allele_answers: %s\n", brc_last_error(eng)); return r ? r : -1; }
            const uint32_t *c_depth = nullptr; const brc_complex_count *c_cnt = nullptr; int64_t n_c = 0, n_ca = 0;
            if (!cq.empty() && ((r = brc_get_complex_answers(eng, &c_depth, &c_cnt, &n_c, &n_ca)) != BRC_OK || n_c != (int64_t)cq.size() || n_ca != (int64_t)ca.size())) { std::fprintf(err, "brc_get_complex_answers: %s\n", brc_last_error(eng)); return r ? r : -1; }
            t_results += now() - g0;
            if (o.timing) { ms_alleles += brc_last_stage_ms(eng, 4); ms_complex += brc_last_stage_ms(eng, 5); }
            const double f0 = now();
            for (int64_t g = 0, k = 0, c = 0, a = 0; g < batch_n; ++g) {
                const size_t ri = (size_t)vcf_rec_of_region[(size_t)(batch_first + g)];
                const VcfRecord &rec = vcf->rec[ri];
                if (rec.complex) { vcf_store_complex(*vcf, ri, c_depth[c++], c_cnt + a, *vcf_ans); a += (int64_t)rec.n_queries; continue; }
                vcf_store(*vcf, ri, ans + k, *vcf_ans);
                k += (int64_t)rec.n_queries;
            }
            if (vcf_stream && !vcf_write(batch_first + batch_n)) { std::fprintf(err, "writing the VCF: %s\n", std::strerror(errno)); return -1; }
            t_format += now() - f0;
        } else {
            if (o.site_filter) {          // only the selected sites came back: no dense view, the region table is all the loop needs
                brc_selected_results sel{};
                if ((r = brc_get_selected_results(eng, &sel)) != BRC_OK) { std::fprintf(err, "brc_get_selected_results: %s\n", brc_last_error(eng)); return r; }
                res.n_regions = sel.n_regions; res.regions = sel.regions;
            } else if ((r = brc_get_results(eng, &res)) != BRC_OK) { std::fprintf(err, "brc_get_results: %s\n", brc_last_error(eng)); return r; }
            const double f0 = now();
            t_results += f0 - g0;
            const bool argv_chain = res.n_regions > 1 && !res.regions[0].site_list_mode;   // never-cleared deletion queue: one sequential pass
            int64_t total_slots = 0;
            for (int64_t g = 0; g < res.n_regions; ++g) total_slots += res.regions[g].n_slots;
            const bool many_small = res.n_regions > 1 && total_slots <= (int64_t(1) << 22);  // a site list: all regions in one formatting pass
            if (argv_chain || many_small) {
                if (brc_write_text(eng, -1, 0, -1, lib_ptrs.data(), out_fd) < 0) { std::fprintf(err, "format: %s\n", brc_last_error(eng)); return -1; }
            } else {
                const int64_t WIN = 1 << 21;   // stream big regions in 2M-site windows (each formatted by several threads)
                for (int64_t g = 0; g < res.n_regions; ++g)
                    for (int64_t first = 0; first < res.regions[g].n_slots; first += WIN)
                        if (brc_write_text(eng, g, first, WIN, lib_ptrs.data(), out_fd) < 0) { std::fprintf(err, "format: %s\n", brc_last_error(eng)); return -1; }
            }
            t_format += now() - f0;
        }
        batch_first += batch_n; batch_n = 0;
        { int64_t wc[4]; if (brc_get_warning_counts(eng, wc) == BRC_OK) for (int k = 0; k < 4; ++k) warn_total[k] += wc[k]; }
        warner.replay();
        const double r0 = now();
        const int rr = brc_reset(eng);
        t_reset += now() - r0;
        return rr;
    };
    int64_t pushed = 0;
    RegionFetcher fetcher(bam);
    const double t_loop0 = now();
    for (size_t gi = 0; gi < regions.size(); ++gi) {
        const Region &g = regions[gi];
        const double d0 = now();
        if (!o.decode_only) {
            const std::string &contig = bam.names[(size_t)g.tid];
            auto loaded = h->ref_name.find(g.tid);
            if (loaded == h->ref_name.end() || loaded->second != contig) {   // load_reference: whole chromosome
                h->ref_name.erase(g.tid);
                if (!s.fa.fetch(contig, chrom)) { std::fprintf(err, "Failed to fetch %s from %s\n", contig.c_str(), o.fn_fa.c_str()); return 1; }
                const int rc = brc_set_reference(eng, g.tid, contig.c_str(), (int64_t)chrom.size(), 0, chrom.data(), (int64_t)chrom.size());
                if (rc != BRC_OK) { std::fprintf(err, "brc_set_reference: %s\n", brc_last_error(eng)); return 1; }
                h->ref_name[g.tid] = contig;
                t_ref += now() - d0;
            }
        }
        const double d1 = now();
        // the source: a window decoded by ParallelFetcher, the compressed span (device decode), or the record stream.  A window
        // or a span is a batch of its own: whatever smaller regions are pending goes out first.
        const bool window = s.par_ok(gi), span = !window && o.device_decode && !s.is_cram;
        if ((window || span) && pushed > 0) { if (flush() != BRC_OK) return 1; pushed = 0; }
        WindowJob *job = window ? s.decoded_window(gi) : nullptr;      // nullptr: the record stream after all
        if (!o.decode_only) {
            brc_begin_region(eng, g.tid, g.beg, g.end, g.site_list ? 1 : 0);
            ++batch_n;
            warner.begin_region(g.tid, g.beg, g.end, g.cont);
        }
        // samfetch(in, idx, ref, d.beg-1, d.end): records with tid, endpos > max(beg-1,0), pos < end, in file order
        const int64_t fbeg = std::max<int64_t>((int64_t)g.beg - 1, 0), fend = g.end;
        int64_t n = 0, psum = 0, qsum = 0;                             // decode-only: what the region received
        if (job) {
            // ONE borrowed batch (the engine streams it to the GPU in chunks) while the next window is already being decoded
            const brc_read_batch &b = job->batch;
            if (o.decode_only) {
                n = b.n_reads;
                for (int64_t i = 0; i < b.n_reads; ++i) psum += b.pos[i];
                for (uint64_t k = b.qual_off[0]; k < b.qual_off[b.n_reads]; ++k) qsum += b.qual[k];
            } else {
                for (Slice &sl : job->slices) warner.take(sl.cands);
                if (b.n_reads > 0) {
                    const int prc = brc_push_reads(eng, &b);
                    if (prc != BRC_OK) { std::fprintf(err, "brc_push_reads: %s\n", brc_last_error(eng)); return 1; }
                }
            }
            fetcher.active = false;
        } else if (span) {
            // f-2: hand the engine the compressed span; it inflates, frames and computes on the device
            SpanBuilder sb;
            if (sb.build(bam, g.tid, fbeg, fend)) {
                brc_bam_span sp{}; sp.comp = sb.comp.data(); sp.comp_len = (int64_t)sb.comp.size(); sp.n_entry = (int64_t)sb.entries.size(); sp.entry = sb.entries.data();
                sp.end_voff = sb.end_voff; sp.tid = g.tid; sp.n_rg = (int32_t)rg_ids.size(); sp.rg_id = rg_ids.data(); sp.rg_lib = rg_libs.data();
                const int prc = brc_push_bam_span(eng, &sp);
                if (prc != BRC_OK) { std::fprintf(err, "brc_push_bam_span: %s\n", brc_last_error(eng)); return 1; }
            }
            fetcher.active = false;
        } else {
            auto stream = [&](auto &&sink) {
#ifdef BRC_WITH_HTSLIB
                if (s.is_cram) { s.hts.fetch(g.tid, fbeg, fend, sink); return; }
#endif
                fetcher.fetch(g.tid, fbeg, fend, s.next_fbeg(gi), sink);
            };
            int push_rc = BRC_OK;
            auto push = [&](const Rec &r) {
                const uint16_t lib = rec_lib(r, s.rg_lib, o.per_lib);
                warner.consider(r, lib);
                const int prc = brc_push_read(eng, r.tid, r.pos, r.flag, r.mapq, lib, r.l_qseq, r.nm, r.sm, r.n_cigar, r.cigar, r.seq, r.qual);
                if (prc != BRC_OK && push_rc == BRC_OK) push_rc = prc;
                ++pushed;
            };
            auto count = [&](const Rec &r) {
                if (r.flag & 4) return;
                int64_t q = 0;             // a local sum: the quality bytes may alias qsum, which would be stored once per byte
                for (int k = 0; k < r.l_qseq; ++k) q += r.qual[k];
                ++n; psum += r.pos; qsum += q;
            };
            if (o.decode_only) stream(count); else stream(push);
            if (push_rc != BRC_OK) { std::fprintf(err, "brc_push_read: %s\n", brc_last_error(eng)); return 1; }
        }
        if (o.decode_only) {
            dprintf(out_fd, "%d\t%d\t%d\t%lld\t%lld\t%lld\n", g.tid, g.beg, g.end, (long long)n, (long long)psum, (long long)qsum);
            continue;
        }
        brc_end_region(eng);
        t_decode += now() - d1;
        // a window's batch is borrowed until its text is out, and a span is one batch; record-stream regions go out in batches
        // at region boundaries (the deletion queue of the argv loop is carried by the engine, brc_set_queue_carry)
        if (job || span || gi + 1 == regions.size() || pushed > 1500000) { if (flush() != BRC_OK) return 1; pushed = 0; }
    }
    if (vcf_stream && !vcf_write(INT64_MAX)) { std::fprintf(err, "writing the VCF: %s\n", std::strerror(errno)); return 1; }
    warner.finish(warn_total);
#ifdef BRC_WITH_HTSLIB
    const bool decode_error = bam.bz.error || s.hts.error || s.par_decode_error;
#else
    const bool decode_error = bam.bz.error || s.par_decode_error;
#endif
    if (s.ahead.valid()) s.ahead.get();
    if (decode_error) std::fprintf(err, "[E::bgzf_read] %s: truncated or corrupt BGZF block / BAM record — the output above is incomplete\n", s.path.c_str());
    if (o.timing) std::fprintf(err, "[brc timing] index seeks %llu  records decoded %llu  (+ %llu records in %llu windows decoded by %d threads)\n", (unsigned long long)fetcher.n_seeks,
                               (unsigned long long)fetcher.n_decoded, (unsigned long long)s.par_decoded, (unsigned long long)s.par_windows, s.pf.n_threads);
    if (o.decode_only) return decode_error ? 1 : 0;
    if (o.timing) std::fprintf(err, "[brc timing] reference %.3fs  decode+push %.3fs  compute %.3fs  results %.3fs  format %.3fs  reset %.3fs  | region loop %.3fs, since main() %.3fs\n",
                               t_ref, t_decode, t_compute, t_results, t_format, t_reset, now() - t_loop0, now() - t_main0);
    if (o.timing) std::fprintf(err, "[brc timing] startup (CUDA context, header, index, first window) %.3fs\n", t_loop0 - s.t0);
    if (o.timing && vcf) std::fprintf(err, "[brc timing] allele kernels %.3f ms\n", ms_alleles);
    if (o.timing && o.vcf_complex) std::fprintf(err, "[brc timing] complex kernel %.3f ms\n", ms_complex);
    return decode_error ? 1 : 0;
}

// Everything is printed: leave without tearing down the CUDA context, the page-locked buffers and the thread pools one by
// one (a teardown that takes a noticeable part of a second) — the kernel reclaims them.  BRC_CLI_CLEAN_EXIT=1 tears down.
// A run that failed before it asked for an engine still waits for the CUDA start-up thread, as returning from main() would.
int leave(Engines &engines, std::unique_ptr<Sample> &last, int status) {
    if (engines.warm.joinable()) engines.warm.join();
    if (!std::getenv("BRC_CLI_CLEAN_EXIT")) {
        std::fflush(nullptr);
        _exit(status);
    }
    last.reset();
    engines.destroy();
    return status;
}

// The output files of one sample (OUT and ERR of a cohort sample, the ERR of a --vcf-samples sample).  Nothing is created or
// emptied until all are open: a sample that cannot have them all leaves no new file behind and no earlier file truncated.
bool open_outputs(const std::vector<const std::string *> &path, std::vector<int> &fd, std::string &why) {
    const size_t n = path.size();
    fd.assign(n, -1); std::vector<bool> made(n, false);
    auto undo = [&](size_t m) { for (size_t j = 0; j < m; ++j) { ::close(fd[j]); if (made[j]) ::unlink(path[j]->c_str()); } };
    for (size_t i = 0; i < n; ++i) {
        fd[i] = ::open(path[i]->c_str(), O_WRONLY | O_CREAT | O_EXCL | O_CLOEXEC, 0666);
        if (fd[i] >= 0) made[i] = true;
        else if (errno == EEXIST) fd[i] = ::open(path[i]->c_str(), O_WRONLY | O_CLOEXEC);
        if (fd[i] < 0) { why = "cannot open " + *path[i] + ": " + std::strerror(errno); undo(i); return false; }
    }
    for (size_t i = 0; i < n; ++i)
        if (::ftruncate(fd[i], 0) != 0) { why = "cannot truncate " + *path[i] + ": " + std::strerror(errno); undo(n); return false; }
    return true;
}

// The lines of a sample list (--bam-list, --vcf-samples): every non-empty line, a trailing '\r' dropped, split at tabs into 2 or 3
// non-empty fields (`shape` names them in the message), with its line number.  False with a message on stderr.
struct ListLine { int ln; std::vector<std::string> fld; };
bool read_list(const std::string &list_path, const char *shape, std::vector<ListLine> &out) {
    std::ifstream f(list_path);
    if (!f) { std::fprintf(stderr, "Failed to open sample list file: %s\n", list_path.c_str()); return false; }
    std::string line; int ln = 0;
    while (std::getline(f, line)) {
        ++ln;
        if (!line.empty() && line.back() == '\r') line.pop_back();
        if (line.empty()) continue;
        std::vector<std::string> fld = split(line, '\t');
        const bool empty_field = std::any_of(fld.begin(), fld.end(), [](const std::string &x) { return x.empty(); });
        if ((fld.size() != 2 && fld.size() != 3) || empty_field) {
            std::fprintf(stderr, "%s:%d: a sample line is %s\n", list_path.c_str(), ln, shape);
            return false;
        }
        out.push_back({ln, std::move(fld)});
    }
    if (out.empty()) { std::fprintf(stderr, "%s lists no sample\n", list_path.c_str()); return false; }
    return true;
}

// Adds an output path to `used` (absolute and normalised); false, with a message on stderr, when an earlier sample has it.
bool claim_output(std::set<std::string> &used, const std::string &list_path, int ln, const std::string &path) {
    std::error_code ec;
    std::filesystem::path abs = std::filesystem::absolute(path, ec);
    if (ec) abs = path;
    if (used.insert(abs.lexically_normal().string()).second) return true;
    std::fprintf(stderr, "%s:%d: %s is already the output of an earlier sample\n", list_path.c_str(), ln, path.c_str());
    return false;
}

// One input of a sample list and where its STDOUT and STDERR go: files, or the process's own when the path is empty.
struct ListSample { std::string in, out, err; };

// Runs the samples of a list in order, each exactly as a run on its input alone (DESIGN.md §11).  `vcf_ans` (--vcf-samples):
// sample k's answers go to vcf_ans[k], which is marked failed when the sample fails.  A sample whose own run would exit 1, or
// whose output files cannot be opened or written, gets one line on the process's STDERR and the list goes on.  Returns the number
// of failed samples, or -1 when no engine could be created: the remaining samples are not run.
//
// While a sample with an ERR file runs, file descriptor 2 is that file, so whatever a library prints there (htslib's CRAM and
// index messages) lands in that sample's ERR in the order its own run prints it.  The next sample is opened on a worker thread
// while the current one computes, holding its messages until its turn, unless it is a CRAM: htslib prints while it opens one, so
// a CRAM is opened at its turn.  Its first window is decoded ahead only when the current sample does not use the process's two
// window jobs, so page-locked window memory stays at two jobs, reused from sample to sample.
int run_list(const Options &o, Engines &engines, const std::vector<ListSample> &list, std::vector<VcfAnswers> *vcf_ans, double t_main0) {
    std::unique_ptr<WindowJob[]> pool(new WindowJob[2]);
    auto open_ahead = [&](size_t k, bool first_window) {
        return std::async(std::launch::async, open_sample, std::cref(o), list[k].in, now(), nullptr, pool.get(), first_window);
    };
    if (!o.decode_only && !o.dist_refused()) engines.start_warm();
    std::future<std::unique_ptr<Sample>> ahead;                          // sample k, opened ahead of its turn
    if (!is_cram_path(list[0].in)) ahead = open_ahead(0, true);          // under the CUDA start-up
    int n_failed = 0;
    for (size_t k = 0; k < list.size(); ++k) {
        const ListSample &e = list[k];
        const bool next_ahead = k + 1 < list.size() && !is_cram_path(list[k + 1].in);
        auto failed = [&](const char *fmt, const std::string &what) {
            ++n_failed;
            if (vcf_ans) (*vcf_ans)[k].failed = true;
            std::fprintf(stderr, fmt, k + 1, e.in.c_str(), what.c_str());
        };
        std::vector<const std::string *> paths; std::vector<int> fd; std::string why;
        if (!e.out.empty()) paths.push_back(&e.out);
        if (!e.err.empty()) paths.push_back(&e.err);
        if (!open_outputs(paths, fd, why)) {
            if (ahead.valid()) ahead.get();
            failed("sample %zu (%s) failed: %s\n", why);
            if (next_ahead) ahead = open_ahead(k + 1, true);
            continue;
        }
        const int out_fd = e.out.empty() ? STDOUT_FILENO : fd[0], err_fd = e.err.empty() ? -1 : fd.back();
        int saved_fd2 = -1;
        if (err_fd >= 0) { std::fflush(stderr); saved_fd2 = ::dup(2); ::dup2(err_fd, 2); }
        std::unique_ptr<Sample> cur = ahead.valid() ? ahead.get() : open_sample(o, e.in, now(), stderr, pool.get(), true);
        if (next_ahead) ahead = open_ahead(k + 1, !cur->uses_windows());
        const int rc = run_sample(o, engines, *cur, out_fd, stderr, t_main0, vcf_ans ? &(*vcf_ans)[k] : nullptr);
        cur.reset();                                                     // htslib's closing lines still go to this ERR
        if (err_fd >= 0) {
            if (std::fflush(stderr) != 0) why = e.err + ": " + std::strerror(errno);
            else if (std::ferror(stderr)) why = e.err + ": write error";
            std::clearerr(stderr);
            ::dup2(saved_fd2, 2);
            ::close(saved_fd2);
            if (::close(err_fd) != 0 && why.empty()) why = e.err + ": " + std::strerror(errno);
        }
        if (out_fd != STDOUT_FILENO && ::close(out_fd) != 0 && why.empty()) why = e.out + ": " + std::strerror(errno);
        const std::string see = e.err.empty() ? "the lines above" : e.err;
        if (rc < 0) {
            std::fprintf(stderr, "sample %zu (%s): no engine could be created (see %s); the remaining samples are not run\n", k + 1, e.in.c_str(), see.c_str());
            return -1;
        }
        if (!why.empty()) failed("sample %zu (%s) failed: writing %s\n", why);
        else if (rc != 0) failed("sample %zu (%s) failed: see %s\n", see);
    }
    return n_failed;
}

// --bam-list FILE: a cohort in one process.  Each non-empty line of FILE is INPUT<TAB>OUT[<TAB>ERR] (ERR defaults to OUT.log);
// OUT and ERR receive exactly what a run on INPUT alone with the same options and regions prints on STDOUT and STDERR.  A
// sample whose own run would exit 1 is reported on this process's STDERR and the batch goes on; the exit status is 1 when any
// sample failed.  The list is checked whole before any sample runs.
int run_cohort(const Options &o, Engines &engines, const std::string &list_path, double t_main0) {
    std::vector<ListLine> lines;
    if (!read_list(list_path, "INPUT<TAB>OUT or INPUT<TAB>OUT<TAB>ERR", lines)) return 1;
    std::vector<ListSample> list;
    std::set<std::string> outputs;
    for (const ListLine &l : lines) {
        ListSample e{l.fld[0], l.fld[1], l.fld.size() == 3 ? l.fld[2] : l.fld[1] + ".log"};
        if (!claim_output(outputs, list_path, l.ln, e.out) || !claim_output(outputs, list_path, l.ln, e.err)) return 1;
        list.push_back(std::move(e));
    }
    std::unique_ptr<Sample> none;
    const int n_failed = run_list(o, engines, list, nullptr, t_main0);
    if (n_failed < 0) return leave(engines, none, 1);
    if (o.timing) std::fprintf(stderr, "[brc timing] cohort: %zu samples (%d failed) in %.3fs since main()\n", list.size(), n_failed, now() - t_main0);
    return leave(engines, none, n_failed ? 1 : 0);
}

// --vcf FILE --vcf-samples LIST: each non-empty line of LIST is NAME<TAB>INPUT[<TAB>ERR].  Every sample runs as the list's
// next sample (run_list) and fills its answers; after the last one the VCF is written once, sample NAME's column holding what
// `--vcf FILE --vcf-sample NAME INPUT` writes there, or '.' in all five fields when the sample failed.  ERR (the process's
// STDERR without one) receives that run's STDERR.  Under BRC_CLI_DECODE_ONLY STDOUT is the samples' decode summaries in list
// order and no VCF is written, as a single-sample run writes none.
int run_vcf_samples(const Options &o, Engines &engines, const std::vector<ListSample> &list, double t_main0) {
    std::vector<VcfAnswers> ans(list.size(), VcfAnswers(*o.vcf));
    std::unique_ptr<Sample> none;
    const int n_failed = run_list(o, engines, list, &ans, t_main0);
    if (n_failed < 0) return leave(engines, none, 1);
    int status = n_failed ? 1 : 0;
    if (!o.decode_only) {
        std::string out = vcf_header(*o.vcf);
        bool ok = true;
        for (size_t ri = 0; ri < o.vcf->rec.size() && ok; ++ri) {
            vcf_line(*o.vcf, ri, ans.data(), out);
            if (out.size() >= (size_t(1) << 22)) { ok = write_all(STDOUT_FILENO, out); out.clear(); }
        }
        if (!ok || !write_all(STDOUT_FILENO, out)) { std::fprintf(stderr, "writing the VCF: %s\n", std::strerror(errno)); status = 1; }
    }
    if (o.timing) std::fprintf(stderr, "[brc timing] vcf-samples: %zu samples (%d failed) in %.3fs since main()\n", list.size(), n_failed, now() - t_main0);
    return leave(engines, none, status);
}

}  // namespace

int main(int argc, char **argv) {
    const double t_main0 = now();
    Options o;
    std::string bam_list, vcf_path, vcf_sample, vcf_samples; bool shard_given = false, vcf_sample_given = false;
    static option lo[] = {{"help", 0, 0, 'h'}, {"version", 0, 0, 'v'}, {"min-mapping-quality", 1, 0, 'q'}, {"min-base-quality", 1, 0, 'b'},
                          {"max-count", 1, 0, 'd'}, {"site-list", 1, 0, 'l'}, {"reference-fasta", 1, 0, 'f'}, {"print-individual-mapq", 1, 0, 'D'},
                          {"per-library", 0, 0, 'p'}, {"max-warnings", 1, 0, 'w'}, {"insertion-centric", 0, 0, 'i'}, {"shard", 1, 0, 1000},
                          {"min-alt-count", 1, 0, 1001}, {"min-alt-fraction", 1, 0, 1002}, {"bam-list", 1, 0, 1003},
                          {"vcf", 1, 0, 1004}, {"vcf-sample", 1, 0, 1005}, {"vcf-samples", 1, 0, 1006},
                          {"vcf-complex", 0, 0, 1007}, {0, 0, 0, 0}};
    long min_alt_count = 0; double min_alt_fraction = -1.0;       // site filter (brc_set_site_filter); off unless one is given
    bool help = false, version = false;
    for (int c; (c = getopt_long(argc, argv, "hvq:b:d:l:f:D:pw:i", lo, nullptr)) != -1;) {
        switch (c) {
        case 'h': help = true; break; case 'v': version = true; break;
        case 'q': o.min_mapq = std::atoi(optarg); break; case 'b': o.min_bq = std::atoi(optarg); break; case 'd': o.max_cnt = std::atoi(optarg); break;
        case 'l': o.fn_pos = optarg; break; case 'f': o.fn_fa = optarg; break; case 'D': o.dist_arg = optarg; break;
        case 'p': o.per_lib = true; break; case 'w': o.max_warn = std::atoll(optarg); break; case 'i': o.ic = true; break;
        case 1000: if (std::sscanf(optarg, "%d/%d", &o.shard_rank, &o.shard_count) != 2 || o.shard_count < 1 || o.shard_rank < 0 || o.shard_rank >= o.shard_count) { std::fprintf(stderr, "--shard wants RANK/COUNT with 0 <= RANK < COUNT\n"); return 1; }
                   shard_given = true; break;
        case 1001: {
            char *end = nullptr; errno = 0;
            min_alt_count = std::strtol(optarg, &end, 10);
            if (errno || end == optarg || *end || min_alt_count < 1 || min_alt_count > INT32_MAX) { std::fprintf(stderr, "--min-alt-count wants an integer N >= 1\n"); return 1; }
            break;
        }
        case 1002: {
            char *end = nullptr; errno = 0;
            min_alt_fraction = std::strtod(optarg, &end);
            if (errno || end == optarg || *end || !(min_alt_fraction >= 0.0 && min_alt_fraction <= 1.0)) { std::fprintf(stderr, "--min-alt-fraction wants a number F with 0 <= F <= 1\n"); return 1; }
            break;
        }
        case 1003: bam_list = optarg; break;
        case 1004: vcf_path = optarg; break;
        case 1005: vcf_sample = optarg; vcf_sample_given = true; break;
        case 1006: vcf_samples = optarg; break;
        case 1007: o.vcf_complex = true; break;
        default: usage(); return 1;
        }
    }
    o.site_filter = min_alt_count > 0 || min_alt_fraction >= 0.0;
    o.filter.min_alt_count = (int32_t)std::max<long>(min_alt_count, 1); o.filter.min_alt_fraction = std::max(min_alt_fraction, 0.0);
    if (version) { std::printf("bam-readcount version: b200 (engine ABI %d)\n", brc_abi_version()); return 1; }   // R:...:467-470 (exit 1)
    if (help || (optind >= argc && bam_list.empty() && vcf_samples.empty())) { usage(); return 1; }                 // R:...:472-475
    if (!bam_list.empty() && shard_given) { std::fprintf(stderr, "--bam-list and --shard cannot be combined: shard a cohort by splitting its list\n"); return 1; }
    Vcf vcf;
    if (vcf_sample_given && vcf_path.empty()) { std::fprintf(stderr, "--vcf-sample needs --vcf\n"); return 1; }
    if (o.vcf_complex && vcf_path.empty()) { std::fprintf(stderr, "--vcf-complex needs --vcf\n"); return 1; }
    if (!vcf_samples.empty()) {
        const char *why = vcf_path.empty() ? "--vcf-samples needs --vcf" : vcf_sample_given ? "--vcf-samples cannot be combined with --vcf-sample"
                        : optind < argc ? "--vcf-samples takes no positional argument: the inputs are in its list" : nullptr;
        if (why) { std::fprintf(stderr, "%s\n", why); return 1; }
    }
    std::vector<ListSample> vcf_list;     // --vcf-samples
    std::vector<std::string> vcf_names;
    if (!vcf_path.empty()) {
        const char *clash = !o.fn_pos.empty() ? "-l" : optind + 1 < argc ? "positional regions" : o.per_lib ? "-p" : o.site_filter ? "--min-alt-count/--min-alt-fraction"
                          : shard_given ? "--shard" : !bam_list.empty() ? "--bam-list" : nullptr;
        if (clash) { std::fprintf(stderr, "--vcf cannot be combined with %s\n", clash); return 1; }
        if (vcf_sample_given) vcf_names.push_back(vcf_sample);
        if (!vcf_samples.empty()) {
            std::vector<ListLine> lines;
            if (!read_list(vcf_samples, "NAME<TAB>INPUT or NAME<TAB>INPUT<TAB>ERR", lines)) return 1;
            std::set<std::string> names, errs;
            for (const ListLine &l : lines) {
                if (!names.insert(l.fld[0]).second) { std::fprintf(stderr, "%s:%d: sample %s is listed twice\n", vcf_samples.c_str(), l.ln, l.fld[0].c_str()); return 1; }
                if (l.fld.size() == 3 && !claim_output(errs, vcf_samples, l.ln, l.fld[2])) return 1;
                vcf_names.push_back(l.fld[0]);
                vcf_list.push_back({l.fld[1], "", l.fld.size() == 3 ? l.fld[2] : ""});
            }
        }
        std::string why;
        if (!parse_vcf(vcf_path, vcf_names, vcf_samples.empty() ? "--vcf-sample" : "--vcf-samples", o.vcf_complex, vcf, why)) { std::fprintf(stderr, "--vcf: %s\n", why.c_str()); return 1; }
        o.vcf = &vcf;
        o.vcf_samples = !vcf_samples.empty();
    }
    o.decode_only = std::getenv("BRC_CLI_DECODE_ONLY") != nullptr;   // test hook: exercise BGZF/BAI/region fetch without a GPU
    o.device_decode = std::getenv("BRC_CLI_DEVICE_DECODE") != nullptr && !o.decode_only;
    o.timing = std::getenv("BRC_CLI_TIMING") != nullptr;

    Engines engines;
    brc_config &cfg = engines.cfg;
    cfg.min_mapq = o.min_mapq; cfg.min_bq = o.min_bq; cfg.max_cnt = o.max_cnt; cfg.per_lib = o.per_lib; cfg.insertion_centric = o.ic;
    cfg.n_libs = 0; cfg.device = std::getenv("BRC_DEVICE") ? std::atoi(std::getenv("BRC_DEVICE")) : 0;
    if (!bam_list.empty()) {
        o.region_args.assign(argv + optind, argv + argc);          // every positional argument is a region of every sample
        return run_cohort(o, engines, bam_list, t_main0);
    }
    if (o.vcf_samples) return run_vcf_samples(o, engines, vcf_list, t_main0);
    const std::string bam_path = argv[optind];
    o.region_args.assign(argv + optind + 1, argv + argc);
    // CUDA context creation takes a second or two: do it while the BAM header, index and FASTA index are read
    if (!o.decode_only && !o.dist_refused()) engines.start_warm();
    std::unique_ptr<WindowJob[]> pool(new WindowJob[2]);
    std::unique_ptr<Sample> s = open_sample(o, bam_path, t_main0, stderr, pool.get(), true);
    std::vector<VcfAnswers> vcf_ans;
    if (o.vcf) vcf_ans.emplace_back(vcf);
    const int rc = run_sample(o, engines, *s, STDOUT_FILENO, stderr, t_main0, vcf_ans.data());
    return leave(engines, s, rc < 0 ? 1 : rc);
}
