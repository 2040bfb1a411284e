// brc_cli_input.cpp — the input side of brc-readcount (brc_cli_input.h).  CRAM input (R:test-data/cram_site_test.sh, BASELINE
// config 2b) is decoded through htslib when the host is built with -DBRC_WITH_HTSLIB against a libhts.a (tools/build_htslib.sh
// builds the copy vendored with the reference, htslib 1.10); without it HtsSource::open fails.
#include "brc_cli_input.h"

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <fstream>
#include <sstream>
#include <type_traits>
#include <zlib.h>

#include "brc_cli_warn.h"
#ifdef BRC_WITH_HTSLIB
#include <htslib/hts.h>
#include <htslib/sam.h>
#endif

namespace brc::cli {

// ------------------------------------------------------------------------------------------
// BGZF
// ------------------------------------------------------------------------------------------
bool Bgzf::inflate_block(const uint8_t *src, size_t clen, std::vector<uint8_t> &dst, uint32_t isize) {
    dst.resize(isize);
    if (!isize) return true;
    z_stream zs{};
    if (inflateInit2(&zs, -15) != Z_OK) return false;
    zs.next_in = const_cast<uint8_t *>(src); zs.avail_in = (uInt)clen; zs.next_out = dst.data(); zs.avail_out = isize;
    const int rc = inflate(&zs, Z_FINISH);
    inflateEnd(&zs);
    return rc == Z_STREAM_END;
}

size_t Bgzf::block_size(const uint8_t *h, size_t avail, size_t &hdr_len) {
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

bool Bgzf::fill_ahead(uint64_t coff) {
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
    const int nt = worker_count((int64_t)jobs.size() - 1, 1, max_threads);   // a thread per block, at most max_threads
    fan_out(nt, [&](int t) {
        for (size_t j = (size_t)t; j < jobs.size(); j += (size_t)nt) {
            const Job &jb = jobs[j];
            const uint8_t *b = raw.data() + jb.off;
            const size_t clen = jb.total - jb.hdr - 8;
            const uint8_t *tail = b + jb.total - 4;
            const uint32_t isize = tail[0] | (tail[1] << 8) | (tail[2] << 16) | ((uint32_t)tail[3] << 24);
            ahead[j].coff = coff + jb.off; ahead[j].next = coff + jb.off + jb.total;
            ahead[j].ok = inflate_block(b + jb.hdr, clen, ahead[j].data, isize);
        }
    });
    return true;
}

bool Bgzf::load_block(uint64_t coff) {
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

bool Bgzf::seek(uint64_t voff) {
    // sorted site lists keep landing in the block that is already inflated
    if (!((voff >> 16) == block_coff && !block.empty() && !eof) && !load_block(voff >> 16)) return false;
    upos = (size_t)(voff & 0xFFFF);
    return true;
}

// ------------------------------------------------------------------------------------------
// BAM header + BAI index
// ------------------------------------------------------------------------------------------
bool BamFile::open(const std::string &path) {
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

bool BamFile::load_index(const std::string &bam_path) {
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

bool BamFile::query_offset(int tid, int64_t beg, uint64_t &voff) const {
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

// ------------------------------------------------------------------------------------------
// The compressed span of a fetch (brc_push_bam_span)
// ------------------------------------------------------------------------------------------
bool SpanBuilder::build(BamFile &bam, int tid, int64_t fbeg, int64_t fend) {
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

// ------------------------------------------------------------------------------------------
// CRAM through htslib
// ------------------------------------------------------------------------------------------
#ifdef BRC_WITH_HTSLIB
struct HtsSource::Files {
    samFile *fp = nullptr; bam_hdr_t *hdr = nullptr; hts_idx_t *idx = nullptr; bam1_t *b = nullptr;
    ~Files() { if (b) bam_destroy1(b); if (idx) hts_idx_destroy(idx); if (hdr) bam_hdr_destroy(hdr); if (fp) sam_close(fp); }
};

bool HtsSource::available() { return true; }

bool HtsSource::open(const std::string &path, const std::string &fasta, BamFile &meta) {
    f.reset(new Files());
    f->fp = sam_open(path.c_str(), "r");
    if (!f->fp) return false;
    if (!fasta.empty() && hts_set_fai_filename(f->fp, (fasta + ".fai").c_str()) != 0) return false;   // R:bamreadcount.cpp:503-523
    bam_hdr_t *hdr = f->hdr = sam_hdr_read(f->fp);
    if (!hdr) return false;
    meta.text.assign(hdr->text ? hdr->text : "", hdr->text ? hdr->l_text : 0);
    for (int i = 0; i < hdr->n_targets; ++i) { meta.names.push_back(hdr->target_name[i]); meta.lens.push_back((int32_t)hdr->target_len[i]); meta.tid_of[hdr->target_name[i]] = i; }
    f->b = bam_init1();
    return true;
}

bool HtsSource::load_index(const std::string &path) { f->idx = sam_index_load(f->fp, path.c_str()); return f->idx != nullptr; }

void HtsSource::fetch(int tid, int64_t fbeg, int64_t fend, const std::function<void(const Rec &)> &emit) {
    hts_itr_t *it = sam_itr_queryi(f->idx, tid, fbeg, fend);
    if (!it) return;
    ++n_seeks;
    bam1_t *b = f->b;
    Rec r; int ret;
    while ((ret = sam_itr_next(f->fp, it, b)) >= 0) {
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
#else
struct HtsSource::Files {};
bool HtsSource::available() { return false; }
bool HtsSource::open(const std::string &, const std::string &, BamFile &) { return false; }
bool HtsSource::load_index(const std::string &) { return false; }
void HtsSource::fetch(int, int64_t, int64_t, const std::function<void(const Rec &)> &) {}
#endif
HtsSource::HtsSource() = default;
HtsSource::~HtsSource() = default;

// ------------------------------------------------------------------------------------------
// Parallel window decode
// ------------------------------------------------------------------------------------------
bool PinnedBuf::reserve(size_t bytes, bool want_pinned) {
    if (bytes <= cap) return true;
    release();
    const size_t want = bytes + bytes / 8 + 4096;
    if (want_pinned && brc_host_alloc(want, &p) == BRC_OK && p) { pinned = true; cap = want; return true; }
    p = std::malloc(want); pinned = false; cap = p ? want : 0;
    return p != nullptr;
}

void PinnedBuf::release() { if (p) { if (pinned) brc_host_free(p); else std::free(p); } p = nullptr; cap = 0; }

ParallelFetcher::ParallelFetcher(const BamFile &b, const RgLib &rl, const std::string &p, bool pl, bool pin)
    : bam(b), rg_lib(rl), path(p), per_lib(pl), want_pinned(pin) {
    n_threads = worker_count(INT32_MAX, 1, 16);          // the core count, at most 16
    if (const char *ov = std::getenv("BRC_CLI_DECODE_THREADS")) n_threads = std::max(1, std::atoi(ov));
}

void ParallelFetcher::decode_slice(Bgzf &bz, int tid, int64_t lo, int64_t hi, bool first, int64_t fbeg, bool collect, Slice &out) const {
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
            WarnCand c;
            if (Warner::candidate(r, lib, c)) {
                if (out.cands.size() >= MAX_CANDS) out.cand_overflow = true;
                else out.cands.push_back(std::move(c));
            }
        }
        out.reads.append(r.pos, r.flag, r.mapq, lib, r.l_qseq, r.nm, r.sm, r.n_cigar, r.cigar, r.seq, r.qual);
    }
}

bool ParallelFetcher::run(int tid, int64_t fbeg, int64_t fend, bool collect, WindowJob &job) {
    job.tid = tid; job.fbeg = fbeg; job.fend = fend; job.error = false; job.cand_overflow = false; job.n_decoded = 0; job.timing.clear();
    const int64_t w0 = fbeg >> 14, w1 = (fend + 16383) >> 14;
    const int T = (int)std::max<int64_t>(1, std::min<int64_t>(n_threads, (w1 - w0) / 4));
    while ((int)readers.size() < T) { readers.emplace_back(new Bgzf()); if (!readers.back()->open_worker(path)) return false; }
    job.slices.resize((size_t)T);
    std::vector<int64_t> cut((size_t)T + 1);
    for (int t = 0; t <= T; ++t) cut[(size_t)t] = t == 0 ? fbeg : t == T ? fend : ((w0 + (w1 - w0) * t / T) << 14);
    const bool timing = std::getenv("BRC_CLI_TIMING") != nullptr;
    auto clk = [] { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = clk();
    fan_out(T, [&](int t) { decode_slice(*readers[(size_t)t], tid, cut[(size_t)t], cut[(size_t)t + 1], t == 0, fbeg, collect, job.slices[(size_t)t]); });
    const double t1 = clk();
    for (const Slice &sl : job.slices) { job.error = job.error || sl.error; job.cand_overflow = job.cand_overflow || sl.cand_overflow; job.n_decoded += sl.n_decoded; }

    // ---- concatenate: the batch's columns are carved from one block, then every thread copies its slice ----
    // elements of a column in the slices before slice t (t = T: in all of them)
    auto before = [&](int t, auto col) { size_t k = 0; for (int s = 0; s < t; ++s) k += (job.slices[(size_t)s].reads.*col).size(); return k; };
    const size_t n = before(T, &ReadArrays::pos);
    brc_read_batch &b = job.batch;
    b = brc_read_batch{};
    b.n_reads = (int64_t)n;
    auto carve = [&](uintptr_t base) {    // points the batch's columns into a block at `base`; returns the bytes they take
        size_t used = 0;
        auto place = [&](auto field, size_t count) {
            used = (used + 63) & ~(size_t)63;
            b.*field = reinterpret_cast<std::remove_reference_t<decltype(b.*field)>>(base + used);
            used += count * sizeof(*(b.*field));
        };
        for_each_column([&](auto, auto field) { place(field, n); },
                        [&](auto, auto off_field, auto col, auto field) { place(off_field, n + 1); place(field, before(T, col)); });
        return used;
    };
    if (!job.block.reserve(carve(0) + 64, want_pinned)) return false;
    carve((uintptr_t)job.block.p);
    fan_out(T, [&](int t) {
        const ReadArrays &sl = job.slices[(size_t)t].reads;
        const size_t r0 = before(t, &ReadArrays::pos), m = (size_t)sl.n();
        auto dst = [](const auto *p) { return const_cast<std::remove_const_t<std::remove_reference_t<decltype(*p)>> *>(p); };   // the job's own block
        for_each_column(
            [&](auto col, auto field) { if (m) std::memcpy(dst(b.*field) + r0, (sl.*col).data(), m * sizeof((sl.*col)[0])); },
            [&](auto off, auto off_field, auto col, auto field) {
                const size_t p0 = before(t, col), k = (sl.*col).size();
                if (k) std::memcpy(dst(b.*field) + p0, (sl.*col).data(), k * sizeof((sl.*col)[0]));
                uint64_t *o = dst(b.*off_field);
                for (size_t i = 0; i < m; ++i) o[r0 + i] = p0 + (sl.*off)[i];
                if (t == T - 1) o[n] = p0 + k;
            });
    });
    if (timing) {
        char line[256];
        std::snprintf(line, sizeof line, "[brc timing] window %d:%lld-%lld: %d threads decode %.3fs, concatenate %.3fs (%zu reads)\n", tid, (long long)fbeg, (long long)fend, T, t1 - t0, clk() - t1, n);
        job.timing = line;
    }
    return true;
}

// ------------------------------------------------------------------------------------------
// FASTA
// ------------------------------------------------------------------------------------------
bool Fasta::open(const std::string &p) {
    path = p;
    std::ifstream f(p + ".fai");
    if (!f) return false;
    std::string line;
    while (std::getline(f, line)) { std::istringstream ss(line); std::string n; Ent e; if (ss >> n >> e.len >> e.off >> e.lb >> e.lw) ents[n] = e; }
    return true;
}

bool Fasta::fetch(const std::string &name, std::string &out) const {
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

}  // namespace brc::cli
