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
// With --bam-list the same per-sample run is repeated over a list of inputs in one process (DESIGN.md §11).
#include <algorithm>
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
    bool active = false, stream_done = false, merge = true;
    int cur_tid = -1;
    int64_t last_fbeg = -1, keep_floor = -1, last_pos = -1;
    uint64_t n_seeks = 0, n_decoded = 0;

    explicit RegionFetcher(BamFile &b) : bam(b) { merge = std::getenv("BRC_CLI_NO_MERGE") == nullptr; }

    Rec take() { if (spare.empty()) return Rec(); Rec r = std::move(spare.back()); spare.pop_back(); return r; }
    void give(Rec &&r) { if (spare.size() < 4096) spare.push_back(std::move(r)); }

    template <class Emit> void fetch(int tid, int64_t fbeg, int64_t fend, int64_t next_fbeg, Emit &&emit) {
        uint64_t voff;
        if (!bam.query_offset(tid, fbeg, voff)) return;
        const bool cont = merge && active && tid == cur_tid && fbeg >= last_fbeg && fbeg >= keep_floor && voff <= bam.bz.tell();
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
    void consider(const Rec &r, bool no_lib) {
        if (!collecting() || (r.flag & 4) || regs.empty()) return;
        const bool no_nm = r.nm == BRC_TAG_ABSENT, no_sm = (r.flag & 2) && r.sm == BRC_TAG_ABSENT;
        if (!no_nm && !no_sm && !(per_lib && no_lib)) return;
        Cand c; c.pos = r.pos; c.endpos = r.endpos; c.flag = r.flag; c.mapq = r.mapq; c.no_nm = no_nm; c.no_sm = no_sm; c.no_lib = per_lib && no_lib;
        c.cigar.assign(r.cigar, r.cigar + r.n_cigar); c.qual.assign(r.qual, r.qual + r.l_qseq);
        c.qname = (const char *)(r.data.data() + 32);
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
    const BamFile &bam; std::string path; int n_threads; bool per_lib, want_pinned;
    std::unordered_map<std::string, uint16_t> rg_lib;      // @RG ID -> library rank
    std::vector<std::unique_ptr<Bgzf>> readers;
    static constexpr size_t MAX_CANDS = 65536;

    ParallelFetcher(const BamFile &b, const std::string &p, bool pl, bool pin) : bam(b), path(p), per_lib(pl), want_pinned(pin) {
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
            uint16_t lib = 0; bool no_lib = false;
            if (per_lib) {
                lib = (uint16_t)BRC_LIB_NONE;
                if (r.has_rg) { auto it = rg_lib.find(r.rg); if (it != rg_lib.end()) lib = it->second; }
                no_lib = lib == (uint16_t)BRC_LIB_NONE;
            }
            if (collect && !out.cand_overflow) {
                const bool no_nm = r.nm == BRC_TAG_ABSENT, no_sm = (r.flag & 2) && r.sm == BRC_TAG_ABSENT;
                if (no_nm || no_sm || no_lib) {
                    if (out.cands.size() >= MAX_CANDS) out.cand_overflow = true;
                    else {
                        Warner::Cand c; c.pos = r.pos; c.endpos = rec_endpos(r); c.flag = r.flag; c.mapq = r.mapq; c.no_nm = no_nm; c.no_sm = no_sm; c.no_lib = no_lib;
                        c.cigar.assign(r.cigar, r.cigar + r.n_cigar); c.qual.assign(r.qual, r.qual + r.l_qseq); c.qname = (const char *)(r.data.data() + 32);
                        out.cands.push_back(std::move(c));
                    }
                }
            }
            out.pos.push_back(r.pos); out.flag.push_back(r.flag); out.mapq.push_back(r.mapq); out.lib.push_back(lib); out.l_qseq.push_back(r.l_qseq);
            out.nm.push_back(r.nm); out.sm.push_back(r.sm);
            out.cigar.insert(out.cigar.end(), r.cigar, r.cigar + r.n_cigar); out.cigar_off.push_back(out.cigar.size());
            out.seq.insert(out.seq.end(), r.seq, r.seq + ((size_t)r.l_qseq + 1) / 2); out.seq_off.push_back(out.seq.size());
            out.qual.insert(out.qual.end(), r.qual, r.qual + r.l_qseq); out.qual_off.push_back(out.qual.size());
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
                "                                        the others (exit status 1 at the end)\n\n");
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
struct Options {   // everything on the command line except the inputs: the same for every sample
    int min_mapq = 0, min_bq = 0, max_cnt = 10000000; bool per_lib = false, ic = false; long long max_warn = -1;
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
    std::map<std::string, std::string> rg_lb;                   // @RG ID -> LB
    std::map<std::string, uint16_t> lib_rank;
    std::vector<std::string> lib_names; std::vector<const char *> lib_ptrs;
    std::vector<Region> regions;
    Warner warner;
    // big fetches (windows of a cut region) are decoded by several threads, one window ahead of the engine (ParallelFetcher)
    ParallelFetcher pf;
    bool allow_parallel = false;
    WindowJob *jobs;              // the process's two window jobs (page-locked buffers), used by one sample at a time
    std::future<bool> ahead; size_t ahead_gi = (size_t)-1; int ahead_slot = 0;   // waited for when the sample goes
    bool par_decode_error = false; uint64_t par_decoded = 0, par_windows = 0;

    Sample(const Options &opt, const std::string &p, WindowJob *pool)
        : o(opt), path(p), warner(opt.max_warn, opt.min_mapq, opt.min_bq, opt.per_lib, opt.ic), pf(bam, p, opt.per_lib, !opt.decode_only), jobs(pool) {}
    Sample(const Sample &) = delete; Sample &operator=(const Sample &) = delete;

    void fetch_range(size_t gi, int64_t &fb, int64_t &fe) const {
        const Region &g = regions[gi];
        const int64_t clen = bam.lens[(size_t)g.tid];
        fb = std::max<int64_t>((int64_t)g.beg - 1, 0);
        fe = std::min<int64_t>(g.end, std::max<int64_t>(clen, (int64_t)g.beg + 1));
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

    // @RG ID -> LB; libraries in std::set order (R:...:92-111, 526-529)
    std::set<std::string> libs;
    {
        std::istringstream ss(bam.text); std::string line;
        while (std::getline(ss, line)) {
            if (line.compare(0, 3, "@RG") != 0) continue;
            std::istringstream ls(line); std::string tok, id, lb; bool has_lb = false;
            while (std::getline(ls, tok, '\t')) { if (tok.compare(0, 3, "ID:") == 0) id = tok.substr(3); else if (tok.compare(0, 3, "LB:") == 0) { lb = tok.substr(3); has_lb = true; } }
            if (has_lb) { libs.insert(lb); if (!id.empty() && !s.rg_lb.count(id)) s.rg_lb[id] = lb; }
        }
    }
    for (const auto &l : libs) log.say("Expect library: %s in BAM\n", l.c_str());
    s.lib_names.assign(libs.begin(), libs.end());
    for (size_t i = 0; i < s.lib_names.size(); ++i) s.lib_rank[s.lib_names[i]] = (uint16_t)i;
    for (auto &n : s.lib_names) s.lib_ptrs.push_back(n.c_str());
    if (s.lib_ptrs.empty()) s.lib_ptrs.push_back("");

    if (o.fn_pos.empty() && o.region_args.empty()) {
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
    if (!o.fn_pos.empty()) {
        std::ifstream fp(o.fn_pos);
        if (!fp) { log.say("Failed to open region list file: %s\n", o.fn_pos.c_str()); return sp; }
        std::string line;
        while (std::getline(fp, line)) {
            std::istringstream ss(line); std::string name; int b, e;
            if (!(ss >> name >> b >> e)) continue;
            auto it = bam.tid_of.find(name);
            if (it == bam.tid_of.end()) { log.say("%s not found in bam file. Region %s %i %i skipped.\n", name.c_str(), name.c_str(), b, e); continue; }
            regions.push_back({it->second, b - 1, e, true});
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
    {
        // 2 Mb windows: each is decoded by all threads in ~40 ms one window ahead of the engine and needs 110 MB of page-locked memory
        // (8 Mb windows were 0.6 s slower on a 10 Mb BAM, r02t); the record-by-record paths (CRAM, BRC_CLI_SEQUENTIAL) keep 8 Mb
        const bool par_windows_ok = !s.is_cram && std::getenv("BRC_CLI_DEVICE_DECODE") == nullptr && std::getenv("BRC_CLI_SEQUENTIAL") == nullptr;
        int64_t W = std::getenv("BRC_CLI_WINDOW") ? std::atoll(std::getenv("BRC_CLI_WINDOW")) : (par_windows_ok ? 2000000 : 8000000);
        if (o.shard_count > 1 && !std::getenv("BRC_CLI_WINDOW")) W = 1000000;      // finer units so the shards can balance
        std::vector<Region> cut;
        for (const Region &g : regions) {
            const int64_t clen = bam.lens[(size_t)g.tid];
            const int64_t e_eff = std::min<int64_t>(g.end, std::max<int64_t>(clen, (int64_t)g.beg + 1));
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
            const int64_t clen = bam.lens[(size_t)g.tid];
            const int64_t e_eff = std::min<int64_t>(g.end, std::max<int64_t>(clen, (int64_t)g.beg + 1));
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

    for (const auto &kv : s.rg_lb) s.pf.rg_lib[kv.first] = s.lib_rank[kv.second];
    s.allow_parallel = !s.is_cram && !o.device_decode && std::getenv("BRC_CLI_SEQUENTIAL") == nullptr;
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
// Returns the exit status of the run on this input alone (0 or 1), or -1 when no engine could be created.
int run_sample(const Options &o, Engines &engines, Sample &s, int out_fd, FILE *err, double t_main0) {
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
    double t_decode = 0, t_compute = 0, t_format = 0, t_write = 0, t_ref = 0, t_results = 0, t_reset = 0;
    // BRC_CLI_DEVICE_DECODE=1: BGZF inflate + BAM framing on the GPU (per-read warning lines need host-decoded reads: counts only)
    std::vector<const char *> rg_ids; std::vector<uint16_t> rg_libs;
    for (const auto &kv : s.rg_lb) { rg_ids.push_back(kv.first.c_str()); rg_libs.push_back(s.lib_rank[kv.second]); }
    int64_t warn_total[4] = {0, 0, 0, 0};
    auto flush = [&]() -> int {
        const double c0 = now();
        int r = brc_compute(eng);
        t_compute += now() - c0;
        if (r != BRC_OK) { std::fprintf(err, "brc_compute: %s\n", brc_last_error(eng)); return r; }
        brc_results res{};
        const double g0 = now();
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
        if (o.decode_only) {
            const int64_t fbeg = std::max<int64_t>((int64_t)g.beg - 1, 0), fend = g.end;
            int64_t n = 0, psum = 0, qsum = 0;
            auto count = [&](const Rec &r) { if (r.flag & 4) return; ++n; psum += r.pos; for (int k = 0; k < r.l_qseq; ++k) qsum += r.qual[k]; };
            WindowJob *job = s.par_ok(gi) ? s.decoded_window(gi) : nullptr;
            if (job) {
                const brc_read_batch &b = job->batch;
                n = b.n_reads;
                for (int64_t i = 0; i < b.n_reads; ++i) psum += b.pos[i];
                for (uint64_t k = b.qual_off[0]; k < b.qual_off[b.n_reads]; ++k) qsum += b.qual[k];
                fetcher.active = false;
            } else
#ifdef BRC_WITH_HTSLIB
            if (s.is_cram) s.hts.fetch(g.tid, fbeg, fend, count); else
#endif
            fetcher.fetch(g.tid, fbeg, fend, s.next_fbeg(gi), count);
            dprintf(out_fd, "%d\t%d\t%d\t%lld\t%lld\t%lld\n", g.tid, g.beg, g.end, (long long)n, (long long)psum, (long long)qsum);
            continue;
        }
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
        const double d1 = now();
        if (s.par_ok(gi)) {
            // one window = one batch: whatever smaller regions are pending goes out first, then the window is pushed as ONE borrowed
            // batch (the engine streams it to the GPU in chunks) while the next window is already being decoded
            if (pushed > 0) { if (flush() != BRC_OK) return 1; pushed = 0; }
            if (WindowJob *job = s.decoded_window(gi)) {
                brc_begin_region(eng, g.tid, g.beg, g.end, g.site_list ? 1 : 0);
                warner.begin_region(g.tid, g.beg, g.end, g.cont);
                for (Slice &sl : job->slices) warner.take(sl.cands);
                if (job->batch.n_reads > 0) {
                    const int prc = brc_push_reads(eng, &job->batch);
                    if (prc != BRC_OK) { std::fprintf(err, "brc_push_reads: %s\n", brc_last_error(eng)); return 1; }
                }
                brc_end_region(eng);
                fetcher.active = false;
                t_decode += now() - d1;
                if (flush() != BRC_OK) return 1;     // the batch is borrowed until the text is out
                pushed = 0;
                continue;
            }
        }
        brc_begin_region(eng, g.tid, g.beg, g.end, g.site_list ? 1 : 0);
        warner.begin_region(g.tid, g.beg, g.end, g.cont);
        // samfetch(in, idx, ref, d.beg-1, d.end): records with tid, endpos > max(beg-1,0), pos < end, in file order
        const int64_t fbeg = std::max<int64_t>((int64_t)g.beg - 1, 0), fend = g.end;
        int push_rc = BRC_OK;
        if (o.device_decode && !s.is_cram) {
            // f-2: hand the engine the compressed span; it inflates, frames and computes on the device.  One span per batch.
            SpanBuilder sb;
            if (sb.build(bam, g.tid, fbeg, fend)) {
                brc_bam_span sp{}; sp.comp = sb.comp.data(); sp.comp_len = (int64_t)sb.comp.size(); sp.n_entry = (int64_t)sb.entries.size(); sp.entry = sb.entries.data();
                sp.end_voff = sb.end_voff; sp.tid = g.tid; sp.n_rg = (int32_t)rg_ids.size(); sp.rg_id = rg_ids.data(); sp.rg_lib = rg_libs.data();
                const int prc = brc_push_bam_span(eng, &sp);
                if (prc != BRC_OK) { std::fprintf(err, "brc_push_bam_span: %s\n", brc_last_error(eng)); return 1; }
            }
            fetcher.active = false;
            brc_end_region(eng);
            t_decode += now() - d1;
            if (flush() != BRC_OK) return 1;
            pushed = 0;
            continue;
        }
        auto push = [&](const Rec &r) {
            uint16_t lib = 0;
            if (o.per_lib) {
                lib = (uint16_t)BRC_LIB_NONE;
                if (r.has_rg) { auto it = s.rg_lb.find(r.rg); if (it != s.rg_lb.end()) lib = s.lib_rank[it->second]; }
            }
            warner.consider(r, lib == (uint16_t)BRC_LIB_NONE);
            const int prc = brc_push_read(eng, r.tid, r.pos, r.flag, r.mapq, lib, r.l_qseq, r.nm, r.sm, r.n_cigar, r.cigar, r.seq, r.qual);
            if (prc != BRC_OK && push_rc == BRC_OK) push_rc = prc;
            ++pushed;
        };
#ifdef BRC_WITH_HTSLIB
        if (s.is_cram) s.hts.fetch(g.tid, fbeg, fend, push); else
#endif
        fetcher.fetch(g.tid, fbeg, fend, s.next_fbeg(gi), push);
        if (push_rc != BRC_OK) { std::fprintf(err, "brc_push_read: %s\n", brc_last_error(eng)); return 1; }
        brc_end_region(eng);
        t_decode += now() - d1;
        // flush in batches at region boundaries; the deletion queue of the argv loop is carried by the engine (brc_set_queue_carry)
        if (gi + 1 == regions.size() || pushed > 1500000) { if (flush() != BRC_OK) return 1; pushed = 0; }
    }
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
    if (o.timing) std::fprintf(err, "[brc timing] reference %.3fs  decode+push %.3fs  compute %.3fs  results %.3fs  format %.3fs  reset %.3fs  write %.3fs  | region loop %.3fs, since main() %.3fs\n",
                               t_ref, t_decode, t_compute, t_results, t_format, t_reset, t_write, now() - t_loop0, now() - t_main0);
    if (o.timing) std::fprintf(err, "[brc timing] startup (CUDA context, header, index, first window) %.3fs\n", t_loop0 - s.t0);
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

// OUT and ERR of one cohort sample.  Nothing is created or emptied until both are open: a sample that cannot have both
// leaves no new file behind and no earlier file truncated.
bool open_outputs(const std::string &out, const std::string &err, int &out_fd, int &err_fd, std::string &why) {
    const std::string *path[2] = {&out, &err};
    int fd[2] = {-1, -1}; bool made[2] = {false, false};
    auto undo = [&](int n) { for (int j = 0; j < n; ++j) { ::close(fd[j]); if (made[j]) ::unlink(path[j]->c_str()); } };
    for (int i = 0; i < 2; ++i) {
        fd[i] = ::open(path[i]->c_str(), O_WRONLY | O_CREAT | O_EXCL | O_CLOEXEC, 0666);
        if (fd[i] >= 0) made[i] = true;
        else if (errno == EEXIST) fd[i] = ::open(path[i]->c_str(), O_WRONLY | O_CLOEXEC);
        if (fd[i] < 0) { why = "cannot open " + *path[i] + ": " + std::strerror(errno); undo(i); return false; }
    }
    for (int i = 0; i < 2; ++i)
        if (::ftruncate(fd[i], 0) != 0) { why = "cannot truncate " + *path[i] + ": " + std::strerror(errno); undo(2); return false; }
    out_fd = fd[0]; err_fd = fd[1];
    return true;
}

// --bam-list FILE: a cohort in one process.  Each non-empty line of FILE is INPUT<TAB>OUT[<TAB>ERR] (ERR defaults to OUT.log);
// OUT and ERR receive exactly what a run on INPUT alone with the same options and regions prints on STDOUT and STDERR.  A
// sample whose own run would exit 1 is reported on this process's STDERR and the batch goes on; the exit status is 1 when any
// sample failed.  The list is checked whole before any sample runs.
//
// While a sample runs, file descriptor 2 is its ERR file, so whatever a library prints there (htslib's CRAM and index messages)
// lands in that sample's ERR in the order its own run prints it.  The next sample is opened on a worker thread while the current
// one computes, holding its messages until its turn, unless it is a CRAM: htslib prints while it opens one, so a CRAM is opened
// at its turn.  Its first window is decoded ahead only when the current sample does not use the process's two window jobs, so
// page-locked window memory stays at two jobs, reused from sample to sample.
int run_cohort(const Options &o, Engines &engines, const std::string &list_path, double t_main0) {
    struct Entry { std::string in, out, err; };
    std::vector<Entry> list;
    {
        std::ifstream f(list_path);
        if (!f) { std::fprintf(stderr, "Failed to open sample list file: %s\n", list_path.c_str()); return 1; }
        std::set<std::string> outputs;
        std::string line; int ln = 0;
        while (std::getline(f, line)) {
            ++ln;
            if (!line.empty() && line.back() == '\r') line.pop_back();
            if (line.empty()) continue;
            std::vector<std::string> fld; size_t p = 0;
            for (size_t t; (t = line.find('\t', p)) != std::string::npos; p = t + 1) fld.push_back(line.substr(p, t - p));
            fld.push_back(line.substr(p));
            const bool empty_field = std::any_of(fld.begin(), fld.end(), [](const std::string &x) { return x.empty(); });
            if ((fld.size() != 2 && fld.size() != 3) || empty_field) {
                std::fprintf(stderr, "%s:%d: a sample line is INPUT<TAB>OUT or INPUT<TAB>OUT<TAB>ERR\n", list_path.c_str(), ln);
                return 1;
            }
            Entry e{fld[0], fld[1], fld.size() == 3 ? fld[2] : fld[1] + ".log"};
            for (const std::string *path : {&e.out, &e.err}) {
                std::error_code ec;
                std::filesystem::path abs = std::filesystem::absolute(*path, ec);
                if (ec) abs = *path;
                if (!outputs.insert(abs.lexically_normal().string()).second) {
                    std::fprintf(stderr, "%s:%d: %s is already the output of an earlier sample\n", list_path.c_str(), ln, path->c_str());
                    return 1;
                }
            }
            list.push_back(std::move(e));
        }
        if (list.empty()) { std::fprintf(stderr, "%s lists no sample\n", list_path.c_str()); return 1; }
    }
    std::unique_ptr<WindowJob[]> pool(new WindowJob[2]);
    auto open_ahead = [&](size_t k, bool first_window) {
        return std::async(std::launch::async, open_sample, std::cref(o), list[k].in, now(), nullptr, pool.get(), first_window);
    };
    if (!o.decode_only && !o.dist_refused()) engines.start_warm();
    std::future<std::unique_ptr<Sample>> ahead;                          // sample k, opened ahead of its turn
    if (!is_cram_path(list[0].in)) ahead = open_ahead(0, true);          // under the CUDA start-up
    std::unique_ptr<Sample> cur;
    int n_failed = 0;
    for (size_t k = 0; k < list.size(); ++k) {
        const Entry &e = list[k];
        const bool next_ahead = k + 1 < list.size() && !is_cram_path(list[k + 1].in);
        int out_fd = -1, err_fd = -1; std::string why;
        if (!open_outputs(e.out, e.err, out_fd, err_fd, why)) {
            if (ahead.valid()) ahead.get();
            std::fprintf(stderr, "sample %zu (%s) failed: %s\n", k + 1, e.in.c_str(), why.c_str());
            ++n_failed;
            if (next_ahead) ahead = open_ahead(k + 1, true);
            continue;
        }
        std::fflush(stderr);
        const int saved_fd2 = ::dup(2);
        ::dup2(err_fd, 2);
        cur = ahead.valid() ? ahead.get() : open_sample(o, e.in, now(), stderr, pool.get(), true);
        if (next_ahead) ahead = open_ahead(k + 1, !cur->uses_windows());
        const int rc = run_sample(o, engines, *cur, out_fd, stderr, t_main0);
        cur.reset();                                                     // htslib's closing lines still go to this ERR
        if (std::fflush(stderr) != 0) why = e.err + ": " + std::strerror(errno);
        else if (std::ferror(stderr)) why = e.err + ": write error";
        std::clearerr(stderr);
        ::dup2(saved_fd2, 2);
        ::close(saved_fd2);
        if (::close(err_fd) != 0 && why.empty()) why = e.err + ": " + std::strerror(errno);
        if (::close(out_fd) != 0 && why.empty()) why = e.out + ": " + std::strerror(errno);
        if (rc < 0) {
            std::fprintf(stderr, "sample %zu (%s): no engine could be created (see %s); the remaining samples are not run\n", k + 1, e.in.c_str(), e.err.c_str());
            return leave(engines, cur, 1);
        }
        if (rc != 0 || !why.empty()) {
            ++n_failed;
            if (!why.empty()) std::fprintf(stderr, "sample %zu (%s) failed: writing %s\n", k + 1, e.in.c_str(), why.c_str());
            else std::fprintf(stderr, "sample %zu (%s) failed: see %s\n", k + 1, e.in.c_str(), e.err.c_str());
        }
    }
    if (o.timing) std::fprintf(stderr, "[brc timing] cohort: %zu samples (%d failed) in %.3fs since main()\n", list.size(), n_failed, now() - t_main0);
    return leave(engines, cur, n_failed ? 1 : 0);
}

}  // namespace

int main(int argc, char **argv) {
    const double t_main0 = now();
    Options o;
    std::string bam_list; bool shard_given = false;
    static option lo[] = {{"help", 0, 0, 'h'}, {"version", 0, 0, 'v'}, {"min-mapping-quality", 1, 0, 'q'}, {"min-base-quality", 1, 0, 'b'},
                          {"max-count", 1, 0, 'd'}, {"site-list", 1, 0, 'l'}, {"reference-fasta", 1, 0, 'f'}, {"print-individual-mapq", 1, 0, 'D'},
                          {"per-library", 0, 0, 'p'}, {"max-warnings", 1, 0, 'w'}, {"insertion-centric", 0, 0, 'i'}, {"shard", 1, 0, 1000},
                          {"min-alt-count", 1, 0, 1001}, {"min-alt-fraction", 1, 0, 1002}, {"bam-list", 1, 0, 1003}, {0, 0, 0, 0}};
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
        default: usage(); return 1;
        }
    }
    o.site_filter = min_alt_count > 0 || min_alt_fraction >= 0.0;
    o.filter.min_alt_count = (int32_t)std::max<long>(min_alt_count, 1); o.filter.min_alt_fraction = std::max(min_alt_fraction, 0.0);
    if (version) { std::printf("bam-readcount version: b200 (engine ABI %d)\n", brc_abi_version()); return 1; }   // R:...:467-470 (exit 1)
    if (help || (optind >= argc && bam_list.empty())) { usage(); return 1; }                                        // R:...:472-475
    if (!bam_list.empty() && shard_given) { std::fprintf(stderr, "--bam-list and --shard cannot be combined: shard a cohort by splitting its list\n"); return 1; }
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
    const std::string bam_path = argv[optind];
    o.region_args.assign(argv + optind + 1, argv + argc);
    // CUDA context creation takes a second or two: do it while the BAM header, index and FASTA index are read
    if (!o.decode_only && !o.dist_refused()) engines.start_warm();
    std::unique_ptr<WindowJob[]> pool(new WindowJob[2]);
    std::unique_ptr<Sample> s = open_sample(o, bam_path, t_main0, stderr, pool.get(), true);
    const int rc = run_sample(o, engines, *s, STDOUT_FILENO, stderr, t_main0);
    return leave(engines, s, rc < 0 ? 1 : rc);
}
