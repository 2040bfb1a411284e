// brc_engine.cu — host side of libbrc_engine.so: the C ABI of include/brc_engine.h.
//
// Mirrors the reference's region driver (R:src/exe/bam-readcount/bamreadcount.cpp:588-605,
// 644-656): begin_region ≙ d.beg/d.end + bam_plbuf_init, push_read ≙ fetch_func +
// bam_plbuf_push (admission rules of V:htslib-1.10/sam.c:4484-4531 evaluated here, on the
// host, in file order), end_region ≙ bam_plbuf_push(0).  All arithmetic of the hot path runs
// in the CUDA kernels of brc_kernels.cu; this file only batches, copies and launches.
#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>

#include "brc_engine_internal.h"

using namespace brc;

static_assert(sizeof(brc_sec_record) == sizeof(brc::SecRec), "public and device secondary records must match");
static_assert(BRC_N_WORDS == brc::N_WORDS && BRC_KIND_WIDE == brc::KIND_WIDE && BRC_PB_ESCAPE == brc::PB_ESCAPE, "packed-format constants");

namespace brc {
int set_error(brc_engine *e, int status, const std::string &msg) { if (e) e->err = msg; return status; }
int set_cuda_error(brc_engine *e, cudaError_t ce, const char *what) {
    if (e) e->err = std::string(what) + ": " + cudaGetErrorString(ce);
    return BRC_E_CUDA;
}
const HostRef *find_ref(const brc_engine *e, int32_t tid) {
    for (const auto &r : e->refs) if (r.tid == tid) return &r;
    return nullptr;
}
}  // namespace brc

#define CU(call, what) do { cudaError_t ce_ = (call); if (ce_ != cudaSuccess) return set_cuda_error(e, ce_, what); } while (0)

// bam_cigar2rlen: reference length of a CIGAR; with n_indel, also counts its I and D ops there
static inline int64_t cigar_rlen(const uint32_t *cig, uint64_t n, int64_t *n_indel = nullptr) {
    int64_t l = 0;
    for (uint64_t k = 0; k < n; ++k) {
        const uint32_t op = cig[k] & 0xF;
        if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) l += cig[k] >> 4;
        if (n_indel && (op == 1 || op == 2)) ++*n_indel;
    }
    return l;
}

// The kernels' view of a batch whose arrays are in device memory.
static ReadsDev reads_dev(const brc_read_batch &b) {
    ReadsDev R;
    R.n_reads = b.n_reads; R.pos = b.pos; R.flag = b.flag; R.mapq = b.mapq; R.lib = b.lib; R.l_qseq = b.l_qseq; R.nm = b.nm; R.sm = b.sm;
    R.cigar_off = b.cigar_off; R.cigar = b.cigar; R.seq_off = b.seq_off; R.seq = b.seq; R.qual_off = b.qual_off; R.qual = b.qual;
    return R;
}

// The read arrays uploaded into d_in[0..12] (brc_read_batch field order) as a device batch of n reads.
static brc_read_batch d_in_batch(const brc_engine *e, int64_t n) {
    brc_read_batch b{};
    b.n_reads = n; b.pos = e->d_in[0].as<int32_t>(); b.flag = e->d_in[1].as<uint16_t>(); b.mapq = e->d_in[2].as<uint8_t>();
    b.lib = e->d_in[3].as<uint16_t>(); b.l_qseq = e->d_in[4].as<int32_t>(); b.nm = e->d_in[5].as<int32_t>(); b.sm = e->d_in[6].as<int32_t>();
    b.cigar_off = e->d_in[7].as<uint64_t>(); b.cigar = e->d_in[8].as<uint32_t>(); b.seq_off = e->d_in[9].as<uint64_t>();
    b.seq = e->d_in[10].as<uint8_t>(); b.qual_off = e->d_in[11].as<uint64_t>(); b.qual = e->d_in[12].as<uint8_t>();
    return b;
}

// Installs the reference window of `tid` from win_len FASTA characters in device memory, asynchronously on `s`: finds or adds
// its HostRef, encodes the characters into the device copy (4-bit codes: K0 compares nibbles) and refreshes the device RefWin
// table.  `host_seq` is kept as the host copy (the text emitter's deletion alleles and reference column), or null for none.
static int install_ref(brc_engine *e, int32_t tid, const char *contig_name, int64_t chrom_len, int64_t win_beg, int64_t win_len,
                       const char *host_seq, const char *dev_ascii, cudaStream_t s) {
    HostRef *r = nullptr;
    for (auto &x : e->refs) if (x.tid == tid) r = &x;
    if (!r) { e->refs.emplace_back(); r = &e->refs.back(); }
    r->tid = tid; r->name = contig_name ? contig_name : ""; r->chrom_len = chrom_len; r->win_beg = win_beg; r->win_len = win_len;
    if (host_seq) r->seq.assign(host_seq, (size_t)win_len); else r->seq.clear();
    CU(r->dev.reserve((size_t)win_len / 2 + 32), "cudaMalloc(reference)");
    CU(cudaMemsetAsync(r->dev.p, 0xFF, (size_t)win_len / 2 + 32, s), "memset(reference)");
    CU(launch_ref_encode(dev_ascii, r->dev.as<uint8_t>(), win_len, s), "reference encode");
    std::vector<RefWin> tab(e->refs.size());
    for (size_t i = 0; i < e->refs.size(); ++i)
        tab[i] = RefWin{e->refs[i].dev.as<char>(), e->refs[i].chrom_len, e->refs[i].win_beg, e->refs[i].win_len};
    CU(e->d_refs.reserve(tab.size() * sizeof(RefWin)), "cudaMalloc(refs)");
    CU(cudaMemcpyAsync(e->d_refs.p, tab.data(), tab.size() * sizeof(RefWin), cudaMemcpyHostToDevice, s), "H2D refs");   // pageable source: staged before the call returns
    return BRC_OK;
}

extern "C" {

int brc_abi_version(void) { return BRC_ABI_VERSION; }

const char *brc_strerror(int s) {
    switch (s) {
    case BRC_OK: return "ok";
    case BRC_E_INVALID: return "invalid argument or call order";
    case BRC_E_NO_DEVICE: return "no usable CUDA device";
    case BRC_E_CUDA: return "CUDA failure";
    case BRC_E_NOMEM: return "out of memory";
    case BRC_E_UNSORTED: return "reads not sorted by position";
    case BRC_E_NO_REFERENCE: return "reference window missing or too small";
    case BRC_E_BAD_LIBRARY: return "library id out of range";
    case BRC_E_OVERFLOW: return "internal pool overflow";
    default: return "unknown status";
    }
}

const char *brc_last_error(const brc_engine *e) { return e ? e->err.c_str() : ""; }

static std::atomic<int> g_last_device{-1};      // device of the most recent brc_create: where brc_host_alloc page-locks

int brc_create(const brc_config *cfg, brc_engine **out) {
    if (!cfg || !out) return BRC_E_INVALID;
    *out = nullptr;
    if (cfg->per_lib && (cfg->n_libs < 0 || cfg->n_libs > 65534)) return BRC_E_INVALID;
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0) { cudaGetLastError(); return BRC_E_NO_DEVICE; }
    if (cfg->device < 0 || cfg->device >= n_dev) return BRC_E_NO_DEVICE;
    if (cudaSetDevice(cfg->device) != cudaSuccess) { cudaGetLastError(); return BRC_E_NO_DEVICE; }
    g_last_device.store(cfg->device, std::memory_order_relaxed);
    brc_engine *e = new (std::nothrow) brc_engine();
    if (!e) return BRC_E_NOMEM;
    e->cfg = *cfg;
    e->n_rows = cfg->per_lib ? std::max(1, cfg->n_libs) : 1;
    if (cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking) != cudaSuccess) { delete e; return BRC_E_CUDA; }
    for (auto &ev : e->ev) if (cudaEventCreate(&ev) != cudaSuccess) { delete e; return BRC_E_CUDA; }
    *out = e;
    return BRC_OK;
}

void brc_destroy(brc_engine *e) {
    if (!e) return;
    cudaSetDevice(e->cfg.device);
    cudaDeviceSynchronize();
    for (auto &r : e->refs) r.dev.release();
    DevBuf *bufs[] = {&e->d_refs, &e->d_desc, &e->d_tiles, &e->d_tile_lo, &e->d_tile_hi, &e->d_regions, &e->d_deep_tiles,
                      &e->d_words, &e->d_sec, &e->d_sec_count, &e->d_warn, &e->d_sel, &e->d_sel_regions};
    for (auto *b : bufs) b->release();
    for (auto &b : e->d_in) b.release();
    { brc_engine::Decoded &D = e->dec; DevBuf *db[] = {&D.comp, &D.btab, &D.u, &D.meta, &D.scratch, &D.count, &D.partial, &D.cigar, &D.seq, &D.qual, &D.ins_idx, &D.ins_out};
      for (auto *b : db) b->release(); for (auto &b : D.arr) b.release(); }
    PinBuf *pins[] = {&e->h_words, &e->h_sec, &e->h_misc, &e->h_sel};
    for (auto *b : pins) b->release();
    for (auto &ev : e->ev) if (ev) cudaEventDestroy(ev);
    for (auto &ev : e->pipe_ev) if (ev) cudaEventDestroy(ev);
    if (e->s_in) cudaStreamDestroy(e->s_in);
    if (e->s_out) cudaStreamDestroy(e->s_out);
    if (e->s_sec) cudaStreamDestroy(e->s_sec);
    if (e->stream) cudaStreamDestroy(e->stream);
    delete e;
}

int brc_set_reference(brc_engine *e, int32_t tid, const char *contig_name, int64_t chrom_len, int64_t win_beg,
                      const char *seq, int64_t win_len) {
    if (!e || !seq || win_len < 0 || win_beg < 0 || chrom_len < 0) return BRC_E_INVALID;
    cudaSetDevice(e->cfg.device);
    DevBuf ascii;   // the FASTA characters cross once; the device keeps only their 4-bit codes
    cudaError_t ce = ascii.reserve((size_t)win_len + 16);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(ascii.p, seq, (size_t)win_len, cudaMemcpyHostToDevice, e->stream);
    int rc = ce != cudaSuccess ? set_cuda_error(e, ce, "reference upload")
                               : install_ref(e, tid, contig_name, chrom_len, win_beg, win_len, seq, ascii.as<char>(), e->stream);
    if ((ce = cudaStreamSynchronize(e->stream)) != cudaSuccess && rc == BRC_OK) rc = set_cuda_error(e, ce, "reference upload/encode");
    ascii.release();
    return rc;
}

// Reference window already in DEVICE memory as ASCII (a generator or a device-side FASTA decoder wrote it): encoded on `stream`,
// no host copy is kept — brc_format_* (deletion alleles, reference column) then needs brc_set_reference for that contig.
int brc_set_reference_device(brc_engine *e, int32_t tid, const char *contig_name, int64_t chrom_len, int64_t win_beg,
                             const char *dev_ascii, int64_t win_len, void *stream) {
    if (!e || !dev_ascii || win_len < 0 || win_beg < 0 || chrom_len < 0) return BRC_E_INVALID;
    cudaSetDevice(e->cfg.device);
    return install_ref(e, tid, contig_name, chrom_len, win_beg, win_len, nullptr, dev_ascii, (cudaStream_t)stream);
}

int brc_reset(brc_engine *e) {
    if (!e) return BRC_E_INVALID;
    e->reads.clear(); e->is_borrowed = false; e->regions.clear(); e->region_open = false; e->adm.reset(); e->n_indel_ops = 0;
    e->results_valid = false; e->planned = false; e->tiles.clear(); e->regions_dev.clear(); e->n_slots = 0; e->wide.valid = false;
    e->sparse = false; e->sel_launched = false; e->n_sel = 0;
    e->dec.pushed = false; e->dec.ins_reads.clear(); e->dec.ins_off.clear(); e->dec.ins_pool.clear();
    for (auto &w : e->warn_counts) w = 0;
    return BRC_OK;
}

// A borrowed batch becomes an owned copy (bulk memcpy) as soon as anything else is pushed after it.
static void materialize_borrowed(brc_engine *e) {
    const brc_read_batch &B = e->borrowed;
    HostReads &H = e->reads;
    const size_t n = (size_t)B.n_reads;
    H.pos.assign(B.pos, B.pos + n); H.flag.assign(B.flag, B.flag + n); H.mapq.assign(B.mapq, B.mapq + n);
    if (B.lib) H.lib.assign(B.lib, B.lib + n); else H.lib.assign(n, 0);
    H.l_qseq.assign(B.l_qseq, B.l_qseq + n); H.nm.assign(B.nm, B.nm + n); H.sm.assign(B.sm, B.sm + n);
    H.region.assign(n, 0);
    // offsets are rebased to 0 (a borrowed batch may be a slice of larger pools)
    const uint64_t c0 = B.cigar_off[0], s0 = B.seq_off[0], q0 = B.qual_off[0];
    H.cigar_off.resize(n + 1); H.seq_off.resize(n + 1); H.qual_off.resize(n + 1);
    for (size_t i = 0; i <= n; ++i) { H.cigar_off[i] = B.cigar_off[i] - c0; H.seq_off[i] = B.seq_off[i] - s0; H.qual_off[i] = B.qual_off[i] - q0; }
    H.cigar.assign(B.cigar + c0, B.cigar + B.cigar_off[n]);
    H.seq.assign(B.seq + s0, B.seq + B.seq_off[n]);
    H.qual.assign(B.qual + q0, B.qual + B.qual_off[n]);
    e->is_borrowed = false;
    if (e->region_open && n) {   // more reads may follow in the same region: rebuild the pileup-buffer admission state
        Admission &A = e->adm;
        A.reset();
        A.max_tid = A.it_tid = e->regions.back().tid; A.max_pos = A.it_pos = H.pos[n - 1];
        for (size_t i = 0; i < n; ++i) {
            const uint64_t nc = H.cigar_off[i + 1] - H.cigar_off[i];
            const int64_t end = nc ? (int64_t)H.pos[i] + cigar_rlen(H.cigar.data() + H.cigar_off[i], nc) : (int64_t)H.pos[i] + 1;
            if (end >= A.it_pos) A.live_ends.push(end);
        }
    }
}

int brc_begin_region(brc_engine *e, int32_t tid, int32_t beg, int32_t end, int32_t site_list_mode) {
    if (!e || e->region_open) return set_error(e, BRC_E_INVALID, "begin_region: previous region still open");
    brc_region r{};
    r.tid = tid; r.beg = beg; r.end = end; r.site_list_mode = site_list_mode;
    if (e->is_borrowed) materialize_borrowed(e);   // more regions follow: fall back to the engine-owned staging copy
    r.read_lo = r.read_hi = e->reads.n();
    r.first_pos = beg - 1 > 0 ? beg - 1 : 0;
    r.slot_base = e->regions.empty() ? 0 : e->regions.back().slot_base + e->regions.back().n_slots;
    r.n_slots = 0;
    e->regions.push_back(r);
    e->region_open = true; e->adm.reset(); e->open_max_end = r.first_pos;
    e->results_valid = false; e->planned = false;
    return BRC_OK;
}

int brc_push_read(brc_engine *e, int32_t tid, int32_t pos, uint16_t flag, uint8_t mapq, uint16_t lib, int32_t l_qseq,
                  int32_t nm, int32_t sm, uint32_t n_cigar, const uint32_t *cigar, const uint8_t *seq,
                  const uint8_t *qual) {
    if (!e || !e->region_open) return set_error(e, BRC_E_INVALID, "push_read: no open region");
    if (e->is_borrowed) materialize_borrowed(e);
    if (l_qseq < 0 || (n_cigar && !cigar) || (l_qseq && (!seq || !qual))) return set_error(e, BRC_E_INVALID, "push_read: null data");
    brc_region &rg = e->regions.back();
    Admission &A = e->adm;
    // fetch_func runs for every yielded record but has no observable effect for records the
    // pileup buffer refuses; bam_plp_push (V:htslib-1.10/sam.c:4484-4531):
    if (tid < 0 || (flag & 4)) return BRC_OK;                                   // :4488-4490
    if (e->cfg.per_lib && lib != BRC_LIB_NONE && (int)lib >= e->n_rows) return set_error(e, BRC_E_BAD_LIBRARY, "push_read: library id >= n_libs");
    int64_t indel_ops = 0;
    const int64_t end = n_cigar > 0 ? (int64_t)pos + cigar_rlen(cigar, n_cigar, &indel_ops) : (int64_t)pos + 1;  // bam_endpos
    if (A.it_tid == tid && A.it_pos == pos) {                                   // :4491 maxcnt rule
        while (!A.live_ends.empty() && A.live_ends.top() < A.it_pos) A.live_ends.pop();   // retired while draining positions < it_pos
        if ((int64_t)A.live_ends.size() + 1 > (int64_t)e->cfg.max_cnt) return BRC_OK;
    }
    if (tid < A.max_tid || (tid == A.max_tid && pos < A.max_pos)) return set_error(e, BRC_E_UNSORTED, "push_read: reads out of order");
    A.max_tid = tid; A.max_pos = pos;
    const bool linked = end > A.it_pos || tid > A.it_tid;                       // :4513
    if (tid > A.it_tid) { A.live_ends = decltype(A.live_ends)(); }
    A.it_tid = tid; A.it_pos = pos;                                             // the drain leaves the iterator at max_pos
    if (!linked) return BRC_OK;
    A.live_ends.push(end);
    if (tid != rg.tid) return BRC_OK;   // another contig's read can never span a site of this region

    HostReads &H = e->reads;
    H.pos.push_back(pos); H.flag.push_back(flag); H.mapq.push_back(mapq); H.lib.push_back(lib); H.l_qseq.push_back(l_qseq);
    H.nm.push_back(nm); H.sm.push_back(sm); H.region.push_back((int32_t)(e->regions.size() - 1));
    H.cigar.insert(H.cigar.end(), cigar, cigar + n_cigar); H.cigar_off.push_back(H.cigar.size());
    const size_t sb = (size_t)(l_qseq + 1) / 2;
    H.seq.insert(H.seq.end(), seq, seq + sb); H.seq_off.push_back(H.seq.size());
    H.qual.insert(H.qual.end(), qual, qual + l_qseq); H.qual_off.push_back(H.qual.size());
    e->n_indel_ops += indel_ops;
    if (end > e->open_max_end) e->open_max_end = end;
    rg.read_hi = H.n();
    return BRC_OK;
}

// Parallel scan of a batch: are all reads admitted by the pileup buffer as they are (so the batch can be used in
// place), and what is the largest bam_endpos?  The -d rule cannot fire when the whole batch is smaller than max_cnt.
struct BatchScan {
    bool ok = true; int64_t max_end = 0; int64_t indel_ops = 0;
    // arrays the device can rebuild instead of receiving (fixed-length reads): offsets that are arithmetic, constant columns
    bool reg_seq = true, reg_qual = true, const_lq = true, const_sm = true;
};
static BatchScan scan_batch(const brc_read_batch *b, int32_t rtid, int per_lib, int n_rows) {
    const int64_t n = b->n_reads;
    const int nt = worker_count(n, 65536, 16);
    std::vector<BatchScan> part((size_t)nt);
    fan_out(nt, [&](int t) {
        const int64_t lo = n * t / nt, hi = n * (t + 1) / nt;
        BatchScan r;
        const uint64_t s0 = b->seq_off[0], q0 = b->qual_off[0];
        const uint64_t ks = n ? b->seq_off[1] - s0 : 0, kq = n ? b->qual_off[1] - q0 : 0;
        const int32_t lq0 = n ? b->l_qseq[0] : 0, sm0 = n ? b->sm[0] : 0;
        for (int64_t i = lo; i < hi && r.ok; ++i) {
            r.reg_seq = r.reg_seq && b->seq_off[i + 1] - s0 == (uint64_t)(i + 1) * ks;
            r.reg_qual = r.reg_qual && b->qual_off[i + 1] - q0 == (uint64_t)(i + 1) * kq;
            r.const_lq = r.const_lq && b->l_qseq[i] == lq0;
            r.const_sm = r.const_sm && b->sm[i] == sm0;
            if ((b->tid && b->tid[i] != rtid) || (b->flag[i] & 4)) { r.ok = false; break; }
            if (i > 0 && b->pos[i] < b->pos[i - 1]) { r.ok = false; break; }
            if (per_lib && b->lib && b->lib[i] != BRC_LIB_NONE && (int)b->lib[i] >= n_rows) { r.ok = false; break; }
            // cigar_rlen written out: calling it here made the C3 push path (e2e leg) about 2.5 ms per window slower
            // (22.7 -> 25.2 ms, H100 80GB HBM3 at 400 W), although its inner loop compiles the same
            const uint64_t c0 = b->cigar_off[i], c1 = b->cigar_off[i + 1];
            int64_t l = 0;
            for (uint64_t k = c0; k < c1; ++k) {
                const uint32_t op = b->cigar[k] & 0xF;
                if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) l += b->cigar[k] >> 4;
                if (op == 1 || op == 2) ++r.indel_ops;
            }
            const int64_t end = c1 > c0 ? (int64_t)b->pos[i] + l : (int64_t)b->pos[i] + 1;
            if (end <= (int64_t)b->pos[i] && i > 0 && b->pos[i] == b->pos[i - 1]) { r.ok = false; break; }  // zero-span read: exact linking rule lives in brc_push_read
            if (end > r.max_end) r.max_end = end;
        }
        part[(size_t)t] = r;
    });
    BatchScan out;
    for (auto &r : part) {
        out.ok = out.ok && r.ok; out.max_end = std::max(out.max_end, r.max_end); out.indel_ops += r.indel_ops;
        out.reg_seq = out.reg_seq && r.reg_seq; out.reg_qual = out.reg_qual && r.reg_qual; out.const_lq = out.const_lq && r.const_lq; out.const_sm = out.const_sm && r.const_sm;
    }
    return out;
}

int brc_push_reads(brc_engine *e, const brc_read_batch *b) {
    if (!e || !b) return BRC_E_INVALID;
    if (!e->region_open) return set_error(e, BRC_E_INVALID, "push_reads: no open region");
    if (e->is_borrowed) materialize_borrowed(e);
    brc_region &rg = e->regions.back();
    const int32_t rtid = rg.tid;
    // Fast path: the first batch after brc_reset, pushed into the only region, with every record admitted as is
    // (mapped, on the region's contig, sorted, and fewer records than -d so the max-count rule cannot fire):
    // keep a VIEW of the caller's arrays — brc_compute DMAs straight out of them (pin them for full PCIe speed).
    if (e->regions.size() == 1 && e->reads.n() == 0 && b->n_reads > 0 && b->n_reads < (int64_t)e->cfg.max_cnt &&
        b->n_reads < 0x7fffffffLL && e->adm.max_pos < 0) {
        const BatchScan sc = scan_batch(b, rtid, e->cfg.per_lib, e->n_rows);
        if (sc.ok) {
            e->skip_h2d = (sc.reg_seq ? 1 : 0) | (sc.reg_qual ? 2 : 0) | (sc.const_lq ? 4 : 0) | (sc.const_sm ? 8 : 0);
            if (std::getenv("BRC_NO_H2D_ELISION") || b->n_reads < 2) e->skip_h2d = 0;
            e->is_borrowed = true; e->borrowed = *b;
            e->n_indel_ops += sc.indel_ops;
            if (sc.max_end > e->open_max_end) e->open_max_end = sc.max_end;
            rg.read_hi = b->n_reads;
            return BRC_OK;
        }
    }
    for (int64_t i = 0; i < b->n_reads; ++i) {
        const uint64_t c0 = b->cigar_off[i], c1 = b->cigar_off[i + 1];
        int rc = brc_push_read(e, b->tid ? b->tid[i] : rtid, b->pos[i], b->flag[i], b->mapq[i], b->lib ? b->lib[i] : (uint16_t)0,
                               b->l_qseq[i], b->nm[i], b->sm[i], (uint32_t)(c1 - c0), b->cigar + c0, b->seq + b->seq_off[i],
                               b->qual + b->qual_off[i]);
        if (rc != BRC_OK) return rc;
    }
    return BRC_OK;
}

// f-2 region-loop form: the compressed span IS the region's read stream; decoded on the device right away (the count and the
// largest bam_endpos come back with one synchronisation), computed by brc_compute without the reads ever being on the host.
int brc_push_bam_span(brc_engine *e, const brc_bam_span *span) {
    if (!e || !span) return BRC_E_INVALID;
    if (!e->region_open) return set_error(e, BRC_E_INVALID, "push_bam_span: no open region");
    if (e->regions.size() != 1 || e->n_host_reads() != 0 || e->dec.pushed) return set_error(e, BRC_E_INVALID, "push_bam_span: must be the only data pushed since brc_reset (one region, one span)");
    brc_read_batch dev{};
    int rc = brc_decode_bam_span(e, span, &dev, e->stream);
    if (rc != BRC_OK) return rc;
    if (dev.n_reads >= (int64_t)e->cfg.max_cnt) return set_error(e, BRC_E_INVALID, "push_bam_span: -d is smaller than the region's read count; use brc_push_read (host admission)");
    brc_region &rg = e->regions.back();
    rg.read_lo = 0; rg.read_hi = dev.n_reads;
    if (e->dec.max_end > e->open_max_end) e->open_max_end = e->dec.max_end;
    e->dec.pushed = true;
    return BRC_OK;
}

int brc_end_region(brc_engine *e) {
    if (!e || !e->region_open) return set_error(e, BRC_E_INVALID, "end_region: no open region");
    brc_region &rg = e->regions.back();
    // sites are only ever produced where an admitted read spans them: clamp the dense slot range
    int64_t last = std::min<int64_t>(rg.end, e->open_max_end);
    rg.n_slots = (int32_t)std::max<int64_t>(0, last - rg.first_pos);
    e->region_open = false;
    return BRC_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// geometry + launches
// ---------------------------------------------------------------------------------------------
static int build_geometry(brc_engine *e, const brc_region *regs, int64_t n_regions) {
    e->tiles.clear(); e->regions_dev.clear(); e->deep_tiles.clear();
    if (const char *ov = std::getenv("BRC_DEEP_MIN_READS")) e->deep_min_reads = std::max(1, std::atoi(ov));   // test hook (0x7fffffff disables the deep-site kernel)
    int64_t n_slots = 0;
    for (int64_t g = 0; g < n_regions; ++g) {
        const brc_region &r = regs[g];
        int slot = -1;
        for (size_t i = 0; i < e->refs.size(); ++i) if (e->refs[i].tid == r.tid) slot = (int)i;
        if (slot < 0) return set_error(e, BRC_E_NO_REFERENCE, "no reference set for region contig (the reference binary dereferences NULL here)");
        RegionDev d{};
        d.tid_slot = slot; d.first_pos = r.first_pos; d.end = r.first_pos + r.n_slots; d.ref_len_check = r.site_list_mode;
        d.tile_base = (int64_t)e->tiles.size(); d.read_lo = r.read_lo; d.read_hi = r.read_hi;
        e->regions_dev.push_back(d);
        if (r.slot_base != n_slots) return set_error(e, BRC_E_INVALID, "regions: slot_base must be the running sum of n_slots");
        for (int32_t o = 0; o < r.n_slots; o += TILE) {
            const int32_t tn = std::min(TILE, r.n_slots - o);
            if (r.read_hi - r.read_lo >= e->deep_min_reads && deep_shape_ok(tn, e->n_rows)) e->deep_tiles.push_back((int32_t)e->tiles.size());
            e->tiles.push_back(TileInfo{r.first_pos + o, tn, r.slot_base + o});
        }
        n_slots += r.n_slots;
    }
    e->n_slots = n_slots;
    return BRC_OK;
}

static int alloc_outputs(brc_engine *e, int64_t n_reads_cap) {
    const int64_t rs = (int64_t)e->n_rows * e->n_slots;
    const int64_t rs1 = std::max<int64_t>(rs, 1);
    CU(e->d_desc.reserve((size_t)std::max<int64_t>(n_reads_cap, 1) * sizeof(ReadDesc)), "cudaMalloc(desc)");
    const size_t nt = std::max<size_t>(e->tiles.size(), 1);
    CU(e->d_tiles.reserve(nt * sizeof(TileInfo)), "cudaMalloc(tiles)");
    CU(e->d_tile_lo.reserve(nt * 4), "cudaMalloc(tile_lo)");
    CU(e->d_tile_hi.reserve(nt * 4), "cudaMalloc(tile_hi)");
    CU(e->d_regions.reserve(std::max<size_t>(e->regions_dev.size(), 1) * sizeof(RegionDev)), "cudaMalloc(regions)");
    CU(e->d_deep_tiles.reserve(std::max<size_t>(e->deep_tiles.size(), 1) * 4), "cudaMalloc(deep_tiles)");
    if (rs >= 0xFFFFFFFFll) return set_error(e, BRC_E_INVALID, "more than 2^32 (library, site) slots in one batch: window the region");
    CU(e->d_words.reserve(rs1 * 4 * N_WORDS), "cudaMalloc(words)");
    CU(e->d_sec_count.reserve(16), "cudaMalloc(sec_count)");
    CU(e->d_warn.reserve((WARN_WORDS + N_WORK_COUNTERS) * 8), "cudaMalloc(warn)");
    return BRC_OK;
}

static int alloc_sec(brc_engine *e, int64_t cap) {
    cap = std::max<int64_t>(cap, 1024);
    e->sec_cap = cap;
    CU(e->d_sec.reserve((size_t)cap * sizeof(SecRec)), "cudaMalloc(sec)");
    return BRC_OK;
}

static ResultsDev results_dev(brc_engine *e) {
    ResultsDev S{};
    S.n_rows = e->n_rows; S.n_slots = e->n_slots;
    S.words = e->d_words.as<uint32_t>();
    S.sec_cap = e->sec_cap; S.sec_count = e->d_sec_count.as<int32_t>(); S.sec = e->d_sec.as<SecRec>();
    S.warn = e->d_warn.as<unsigned long long>();
    return S;
}

static int upload_geometry(brc_engine *e, cudaStream_t s) {
    if (!e->tiles.empty())
        CU(cudaMemcpyAsync(e->d_tiles.p, e->tiles.data(), e->tiles.size() * sizeof(TileInfo), cudaMemcpyHostToDevice, s), "H2D tiles");
    if (!e->regions_dev.empty())
        CU(cudaMemcpyAsync(e->d_regions.p, e->regions_dev.data(), e->regions_dev.size() * sizeof(RegionDev), cudaMemcpyHostToDevice, s), "H2D regions");
    if (!e->deep_tiles.empty())
        CU(cudaMemcpyAsync(e->d_deep_tiles.p, e->deep_tiles.data(), e->deep_tiles.size() * 4, cudaMemcpyHostToDevice, s), "H2D deep tiles");
    return BRC_OK;
}

// ---------------------------------------------------------------------------------------------
// alternative-allele site filter: region table, launch, compact fetch (kernels in brc_select.cu)
// ---------------------------------------------------------------------------------------------
// Once per brc_compute / brc_run_device.  The emitter's deletion queue is never cleared between argv regions (R:...:650-656),
// so deletions of one region print in a later one that overlaps or abuts it, where the device cannot see them: the slots of a
// region up to the last position such a deletion can print at are shipped whole (keep_all_n), and the host rule decides.  Those
// positions are, per contig, the ends of the earlier argv regions of this batch and, with queue carry on, the positions of the
// entries the last formatting pass left in the carried queue.  A site-list region empties the queue at its end.
static void plan_selection(brc_engine *e) {
    e->sel_regions.clear();
    if (!e->filter_on) return;
    std::vector<std::pair<int32_t, int64_t>> hist;        // contig -> last position a queued deletion may print at
    auto at = [&](int32_t tid) { for (auto &x : hist) if (x.first == tid) return &x; hist.emplace_back(tid, (int64_t)-1); return &hist.back(); };
    if (e->carry_on)
        for (const auto &q : e->carry.q)
            for (const QEnt &x : q) { auto *h = at(x.tid); h->second = std::max<int64_t>(h->second, x.pos); }
    for (size_t g = 0; g < e->regions.size(); ++g) {
        const brc_region &r = e->regions[g];
        const HostRef *ref = find_ref(e, r.tid);
        SelRegion d{};
        d.slot_base = r.slot_base; d.n_slots = r.n_slots; d.first_pos = r.first_pos; d.beg = r.beg; d.end = r.end;
        d.argv = r.site_list_mode ? 0 : 1; d.tid_slot = e->regions_dev[g].tid_slot;
        d.ref_on_host = ref && !ref->seq.empty();
        auto *h = at(r.tid);
        d.keep_all_n = (int32_t)std::max<int64_t>(0, std::min<int64_t>(r.n_slots, h->second - r.first_pos + 1));
        e->sel_regions.push_back(d);
        if (r.site_list_mode) hist.clear();
        else h->second = std::max<int64_t>(h->second, r.end);
    }
}

// The selection kernels after the pileup kernels on stream s (ev[3] after them); no-op without a filter.
static int launch_selection(brc_engine *e, cudaStream_t s) {
    e->sel_launched = false;
    if (!e->filter_on) return BRC_OK;
    const int64_t NS = e->n_slots, rows = e->n_rows, R = (int64_t)e->sel_regions.size();
    const int64_t nb = std::max<int64_t>(1, (NS + SELECT_SCAN_CTA - 1) / SELECT_SCAN_CTA);
    size_t off = 0;
    auto take = [&](size_t bytes) { const size_t o = off; off = (off + bytes + 15) & ~(size_t)15; return o; };
    const size_t o_best = take((size_t)NS * 16), o_last = take((size_t)R * rows * 4), o_cnt = take(16), zero_end = off;
    const size_t o_keep = take((size_t)NS), o_emit = take((size_t)NS), o_ship = take((size_t)NS * 4), o_idx = take((size_t)(NS + 1) * 8);
    const size_t o_part = take((size_t)(nb + 1) * 8), o_site = take((size_t)NS * 4), o_cemit = take((size_t)NS);
    // The compact outputs are sized for the worst case (every site and record shipped), so the launches need no host round trip
    // for the count; this doubles the device result footprint of a filtered batch (about 43 B per site and row plus a second
    // pool).  Sizing them after the count is known would trade that memory for one synchronisation per batch.
    const size_t o_words = take((size_t)NS * rows * 4 * N_WORDS), o_sec = take((size_t)e->sec_cap * sizeof(SecRec));
    CU(e->d_sel.reserve(off), "cudaMalloc(selection)");
    CU(e->d_sel_regions.reserve((size_t)std::max<int64_t>(R, 1) * sizeof(SelRegion)), "cudaMalloc(selection regions)");
    if (R) CU(cudaMemcpyAsync(e->d_sel_regions.p, e->sel_regions.data(), (size_t)R * sizeof(SelRegion), cudaMemcpyHostToDevice, s), "H2D selection regions");
    char *b = e->d_sel.as<char>();
    CU(cudaMemsetAsync(b, 0, zero_end, s), "memset(selection)");
    SelectParams P{};
    P.words = e->d_words.as<uint32_t>(); P.n_rows = e->n_rows; P.n_slots = NS;
    P.sec = e->d_sec.as<SecRec>(); P.sec_count = e->d_sec_count.as<int32_t>(); P.sec_cap = e->sec_cap;
    P.regions = e->d_sel_regions.as<SelRegion>(); P.n_regions = R; P.refs = e->d_refs.as<RefWin>();
    P.min_alt_count = e->filter.min_alt_count; P.min_alt_fraction = e->filter.min_alt_fraction;
    P.best = reinterpret_cast<uint32_t *>(b + o_best); P.dsum = P.best + NS; P.dbest = P.dsum + NS; P.esc_np = P.dbest + NS;
    P.reg_last = reinterpret_cast<uint32_t *>(b + o_last); P.counters = reinterpret_cast<unsigned long long *>(b + o_cnt);
    P.keep = reinterpret_cast<uint8_t *>(b + o_keep); P.emit = reinterpret_cast<uint8_t *>(b + o_emit);
    P.ship = reinterpret_cast<uint32_t *>(b + o_ship); P.idx = reinterpret_cast<uint64_t *>(b + o_idx);
    P.partial = reinterpret_cast<unsigned long long *>(b + o_part); P.nb = nb;
    P.c_site = reinterpret_cast<uint32_t *>(b + o_site); P.c_emit = reinterpret_cast<uint8_t *>(b + o_cemit);
    P.c_words = reinterpret_cast<uint32_t *>(b + o_words); P.c_sec = reinterpret_cast<SecRec *>(b + o_sec);
    CU(launch_select(P, s), "launch selection");
    if (NS > 0) e->launch_count += SELECT_KERNELS;
    CU(cudaEventRecord(e->ev[3], s), "event");
    e->sel_params = P;
    e->sel_filter = e->filter;
    e->sel_launched = true;
    return BRC_OK;
}

// The compact selection to the host: the counts first, then exactly the shipped bytes.
static int fetch_selected(brc_engine *e, cudaStream_t s) {
    const SelectParams &P = e->sel_params;
    int32_t cnt = 0;
    CU(e->h_misc.reserve(64), "pin");
    uint64_t *hm = e->h_misc.as<uint64_t>();
    hm[0] = hm[1] = hm[2] = 0;
    CU(cudaMemcpyAsync(&cnt, e->d_sec_count.p, 4, cudaMemcpyDeviceToHost, s), "D2H sec_count");
    if (P.n_slots > 0) {
        CU(cudaMemcpyAsync(hm, P.idx + P.n_slots, 8, cudaMemcpyDeviceToHost, s), "D2H selected sites");
        CU(cudaMemcpyAsync(hm + 1, P.counters, 16, cudaMemcpyDeviceToHost, s), "D2H selection counters");
    }
    CU(cudaStreamSynchronize(s), "sync");
    if ((int64_t)cnt > e->sec_cap) return set_error(e, BRC_E_OVERFLOW, "secondary key pool overflow (re-plan with a larger n_sec_cap)");
    const int64_t n = (int64_t)hm[0], ns = (int64_t)hm[1];
    e->sel_abandoned = (int64_t)hm[2];
    const size_t wbytes = (size_t)n * e->n_rows * 4 * N_WORDS;
    CU(e->h_words.reserve(std::max<size_t>(wbytes, 4)), "pin"); CU(e->h_sec.reserve((size_t)std::max<int64_t>(ns, 1) * sizeof(SecRec)), "pin");
    CU(e->h_sel.reserve((size_t)std::max<int64_t>(n, 1) * 5), "pin");
    if (n) {
        CU(cudaMemcpyAsync(e->h_words.p, P.c_words, wbytes, cudaMemcpyDeviceToHost, s), "D2H selected words");
        CU(cudaMemcpyAsync(e->h_sel.p, P.c_site, (size_t)n * 4, cudaMemcpyDeviceToHost, s), "D2H selected site ids");
        CU(cudaMemcpyAsync(e->h_sel.as<uint32_t>() + n, P.c_emit, (size_t)n, cudaMemcpyDeviceToHost, s), "D2H selected emit bytes");
    }
    if (ns) CU(cudaMemcpyAsync(e->h_sec.p, P.c_sec, (size_t)ns * sizeof(SecRec), cudaMemcpyDeviceToHost, s), "D2H selected records");
    CU(cudaMemcpyAsync(hm + 4, e->d_warn.p, 16, cudaMemcpyDeviceToHost, s), "D2H warn");
    CU(cudaStreamSynchronize(s), "sync D2H");
    e->warn_counts[0] = (int64_t)hm[4]; e->warn_counts[1] = (int64_t)hm[5]; e->warn_counts[2] = 0;
    e->warn_counts[3] = -1;
    e->n_sel = n; e->h_n_sec = ns; e->sparse = true;
    e->results_valid = true; e->fmt_valid = false; e->wide.valid = false;
    return BRC_OK;
}

static void make_params(brc_engine *e, const int32_t *d_region_of_read, PrecomputeParams &P0, PileupParams &P1) {
    P0 = PrecomputeParams{};
    P0.reads = e->dev_reads; P0.regions = e->d_regions.as<RegionDev>(); P0.n_regions = (int64_t)e->regions_dev.size();
    P0.region_of_read = d_region_of_read; P0.refs = e->d_refs.as<RefWin>(); P0.desc = e->d_desc.as<ReadDesc>();
    P0.tile_lo = e->d_tile_lo.as<int32_t>(); P0.tile_hi = e->d_tile_hi.as<int32_t>();
    P0.read_begin = 0; P0.read_end = e->dev_reads.n_reads; P0.min_mapq = e->cfg.min_mapq;
    P1 = PileupParams{};
    P1.min_mapq = e->cfg.min_mapq; P1.min_bq = e->cfg.min_bq; P1.per_lib = e->cfg.per_lib; P1.insertion_centric = e->cfg.insertion_centric;
    P1.desc = e->d_desc.as<ReadDesc>(); P1.cigar_off = e->dev_reads.cigar_off; P1.cigar = e->dev_reads.cigar; P1.seq = e->dev_reads.seq; P1.qual = e->dev_reads.qual;
    P1.seq_off = e->dev_reads.seq_off; P1.qual_off = e->dev_reads.qual_off;
    P1.tiles = e->d_tiles.as<TileInfo>(); P1.tile_lo = P0.tile_lo; P1.tile_hi = P0.tile_hi; P1.n_tiles = (int64_t)e->tiles.size(); P1.tile_begin = 0; P1.tile_count = P1.n_tiles;
    P1.res = results_dev(e);
    P1.deep_tiles = e->deep_tiles.empty() ? nullptr : e->d_deep_tiles.as<int32_t>(); P1.n_deep = (int32_t)e->deep_tiles.size(); P1.deep_min_reads = e->deep_min_reads;
    P1.work_counter = P1.res.warn + WARN_WORDS;                 // launch k of a run takes dispenser k
}

// K(init) + K0 + K1 on stream s.  Returns BRC_E_OVERFLOW (after syncing) if the secondary pool was too small.
static int run_kernels(brc_engine *e, const int32_t *d_region_of_read, cudaStream_t s, bool check_overflow) {
    PrecomputeParams P0; PileupParams P1;
    make_params(e, d_region_of_read, P0, P1);

    e->launch_count = 0;
    CU(cudaEventRecord(e->ev[0], s), "event");
    CU(launch_init_tiles(P0.tile_lo, P0.tile_hi, P1.n_tiles, P1.res.sec_count, P1.res.warn, s), "launch init_tiles"); e->launch_count++;
    CU(launch_precompute(P0, s), "launch read_precompute"); if (P0.reads.n_reads) e->launch_count++;
    CU(cudaEventRecord(e->ev[1], s), "event");
    CU(launch_pileup(P1, s), "launch pileup"); if (P1.n_tiles) e->launch_count++;
    CU(launch_deep_sites(P1, s), "launch deep_sites"); if (P1.n_deep) e->launch_count++;
    CU(cudaEventRecord(e->ev[2], s), "event");
    const int rs = launch_selection(e, s);
    if (rs != BRC_OK) return rs;
    if (check_overflow) {
        int32_t cnt = 0;
        CU(cudaMemcpyAsync(&cnt, P1.res.sec_count, 4, cudaMemcpyDeviceToHost, s), "D2H sec_count");
        CU(cudaStreamSynchronize(s), "sync kernels");
        e->h_n_sec = cnt;
        if ((int64_t)cnt > e->sec_cap) return BRC_E_OVERFLOW;
    }
    return BRC_OK;
}

static int fetch_results(brc_engine *e, cudaStream_t s, bool slots_already_fetched = false, int64_t sec_done = 0) {
    if (e->sel_launched) return fetch_selected(e, s);
    const int64_t rs = (int64_t)e->n_rows * e->n_slots;
    int32_t cnt = 0;
    CU(cudaMemcpyAsync(&cnt, e->d_sec_count.p, 4, cudaMemcpyDeviceToHost, s), "D2H sec_count");
    CU(cudaStreamSynchronize(s), "sync");
    if ((int64_t)cnt > e->sec_cap) return set_error(e, BRC_E_OVERFLOW, "secondary key pool overflow (re-plan with a larger n_sec_cap)");
    e->h_n_sec = cnt;
    const int64_t rs1 = std::max<int64_t>(rs, 1), ns1 = std::max<int64_t>(cnt, 1);
    CU(e->h_words.reserve(rs1 * 4 * N_WORDS), "pin"); CU(e->h_sec.reserve((size_t)ns1 * sizeof(SecRec)), "pin");
    CU(e->h_misc.reserve(64), "pin");
    if (rs && !slots_already_fetched) CU(cudaMemcpyAsync(e->h_words.p, e->d_words.p, rs * 4 * N_WORDS, cudaMemcpyDeviceToHost, s), "D2H words");
    if (cnt > sec_done)      // records [0, sec_done) were copied while the kernels ran (compute_pipelined)
        CU(cudaMemcpyAsync((char *)e->h_sec.p + (size_t)sec_done * sizeof(SecRec), (char *)e->d_sec.p + (size_t)sec_done * sizeof(SecRec),
                           (size_t)(cnt - sec_done) * sizeof(SecRec), cudaMemcpyDeviceToHost, s), "D2H sec");
    CU(cudaMemcpyAsync(e->h_misc.p, e->d_warn.p, 16, cudaMemcpyDeviceToHost, s), "D2H warn");
    CU(cudaStreamSynchronize(s), "sync D2H");
    const unsigned long long *w = e->h_misc.as<unsigned long long>();
    e->warn_counts[0] = (int64_t)w[0]; e->warn_counts[1] = (int64_t)w[1]; e->warn_counts[2] = 0;
    e->warn_counts[3] = -1;          // LIBRARY_UNAVAILABLE: counted from the flag bits on demand (brc_get_warning_counts)
    e->sparse = false;
    e->results_valid = true; e->fmt_valid = false; e->wide.valid = false;
    return BRC_OK;
}

// The kernels on the batch e->dev_reads, then the results to the host.  The secondary pool starts at `cap` records and
// doubles while it overflows, for at most 8 runs.
static int compute_batch(brc_engine *e, int64_t cap, const int32_t *d_region_of_read, cudaStream_t s) {
    int rc = upload_geometry(e, s);
    if (rc != BRC_OK) return rc;
    for (int attempt = 0; attempt < 8; ++attempt) {
        rc = alloc_sec(e, cap);
        if (rc != BRC_OK) return rc;
        rc = run_kernels(e, d_region_of_read, s, true);
        if (rc != BRC_E_OVERFLOW) break;
        cap = std::max<int64_t>(cap * 2, e->h_n_sec + 1024);
    }
    if (rc != BRC_OK) return rc == BRC_E_OVERFLOW ? set_error(e, rc, "secondary key pool overflow") : rc;
    return fetch_results(e, s);
}

// ---------------------------------------------------------------------------------------------
// packed host records -> the full-width arrays of brc_results (include/brc_engine.h)
// ---------------------------------------------------------------------------------------------
namespace brc {
void ensure_wide(brc_engine *e) {
    brc_engine::Wide &W = e->wide;
    if (W.valid) return;
    const int64_t rs = (int64_t)e->n_rows * e->result_cols(), ns = e->h_n_sec;   // sparse results: the shipped sites' columns
    const uint32_t *words = e->h_words.as<uint32_t>();
    const SecRec *sec = e->h_sec.as<SecRec>();
    W.ncover.resize((size_t)rs); W.npass.resize((size_t)rs); W.flags.resize((size_t)rs); W.pbase.resize((size_t)rs);
    W.sec_head.resize((size_t)rs); W.pstats.resize((size_t)rs * N_STATS);
    const int nt = worker_count(rs, 262144, 16);
    fan_out(nt, [&](int t) {
        const int64_t lo = rs * t / nt, hi = rs * (t + 1) / nt;
        uint32_t *ps = W.pstats.data();
        for (int64_t i = lo; i < hi; ++i) {
            const uint32_t w0 = words[i], w1 = words[rs + i], w2 = words[2 * rs + i], w3 = words[3 * rs + i];
            const uint32_t count = (w0 >> 16) & 0xFFu, plus = w0 >> 24, pc = w1 & 7u;
            W.ncover[(size_t)i] = w0 & 0xFFu; W.npass[(size_t)i] = (w0 >> 8) & 0xFFu;
            W.flags[(size_t)i] = (uint8_t)((w1 >> 3) & 1u); W.pbase[(size_t)i] = (uint8_t)(pc < 6u ? pc : BRC_NO_BASE);
            W.sec_head[(size_t)i] = -1;
            ps[0 * rs + i] = count; ps[1 * rs + i] = w1 >> 16; ps[2 * rs + i] = w2 & 0xFFFFu; ps[3 * rs + i] = w2 >> 16;
            ps[4 * rs + i] = plus; ps[5 * rs + i] = count - plus; ps[6 * rs + i] = words[4 * rs + i]; ps[7 * rs + i] = words[5 * rs + i];
            ps[8 * rs + i] = w3 >> 16; ps[9 * rs + i] = (w1 >> 8) & 0xFFu; ps[10 * rs + i] = words[6 * rs + i]; ps[11 * rs + i] = w3 & 0xFFFFu;
            ps[12 * rs + i] = words[7 * rs + i];
        }
    });
    // secondary records: keys are chained per slot (order is immaterial to every consumer); escaped primaries fill their slot
    const size_t n1 = (size_t)std::max<int64_t>(ns, 1);
    W.sec_next.assign(n1, -1); W.sec_kind.assign(n1, 0); W.sec_len.assign(n1, 0); W.sec_read.assign(n1, 0); W.sec_qpos.assign(n1, 0);
    W.sec_stats.assign(n1 * N_STATS, 0u);
    for (int64_t j = 0; j < ns; ++j) {
        const SecRec &r = sec[j];
        const uint32_t kind = r.kind_len & 0xFFu, len = r.kind_len >> 8;
        const int64_t i = (int64_t)r.slot;
        if (i < 0 || i >= rs) continue;
        if (kind >= KIND_WIDE) {
            const uint32_t pc = kind - KIND_WIDE;
            W.ncover[(size_t)i] = len; W.npass[(size_t)i] = (uint32_t)r.qpos; W.flags[(size_t)i] = (uint8_t)(r.read & 1);
            W.pbase[(size_t)i] = (uint8_t)(pc < 6u ? pc : BRC_NO_BASE);
            for (int k = 0; k < N_STATS; ++k) W.pstats[(size_t)((int64_t)k * rs + i)] = r.stats[k];
            W.sec_kind[(size_t)j] = 0xFF;      // not a key
            continue;
        }
        W.sec_kind[(size_t)j] = (uint8_t)kind; W.sec_len[(size_t)j] = (int32_t)len; W.sec_read[(size_t)j] = r.read; W.sec_qpos[(size_t)j] = r.qpos;
        for (int k = 0; k < N_STATS; ++k) W.sec_stats[(size_t)((int64_t)k * (int64_t)n1 + j)] = r.stats[k];
        W.sec_next[(size_t)j] = W.sec_head[(size_t)i]; W.sec_head[(size_t)i] = (int32_t)j;
    }
    W.n_sec = ns;
    W.valid = true;
}
}  // namespace brc

// Push path, one borrowed region: stream the batch through the GPU in read-index chunks so that the H2D copy of
// chunk c+1, the kernels of chunk c and the D2H copy of the finished tiles of chunk c-1 overlap (PCIe is full
// duplex; three streams + events).  Reads are position-sorted, so every tile that ends at or before the first
// position of chunk c+1 is complete once chunk c is on the device.

// Device buffers + chunked H2D of the borrowed batch on s_in; records pipe_ev[2c] after chunk c.  The copies are issued here,
// from brc_compute, and not from brc_push_reads ahead of its admission scan: an upload started that early runs ahead alone and
// leaves the result download alone on the link at the end, where issued with the kernels both directions stream concurrently
// for the whole step.
static int issue_h2d_chunks(brc_engine *e, int &n_chunks) {
    const brc_read_batch &B = e->borrowed;
    const int64_t n = B.n_reads;
    if (!e->s_in) CU(cudaStreamCreateWithFlags(&e->s_in, cudaStreamNonBlocking), "stream");
    if (!e->s_out) CU(cudaStreamCreateWithFlags(&e->s_out, cudaStreamNonBlocking), "stream");
    const uint64_t n_cig = B.cigar_off[n], n_seq = B.seq_off[n], n_qual = B.qual_off[n];
    const size_t tot[13] = {(size_t)n * 4, (size_t)n * 2, (size_t)n, (size_t)n * 2, (size_t)n * 4, (size_t)n * 4, (size_t)n * 4,
                            (size_t)(n + 1) * 8, (size_t)n_cig * 4, (size_t)(n + 1) * 8, (size_t)n_seq, (size_t)(n + 1) * 8, (size_t)n_qual};
    for (int k = 0; k < 13; ++k) CU(e->d_in[k].reserve(tot[k] + 16), "cudaMalloc(reads)");
    size_t in_bytes = 0; for (int k = 0; k < 13; ++k) in_bytes += tot[k];
    n_chunks = (int)std::min<int64_t>(32, std::max<int64_t>(1, (int64_t)(in_bytes >> 26)));   // ~64 MiB of input per chunk
    n_chunks = (int)std::min<int64_t>(n_chunks, std::max<int64_t>(1, n / 4096));
    if (const char *ov = std::getenv("BRC_PIPE_CHUNKS")) n_chunks = (int)std::max<int64_t>(1, std::min<int64_t>(std::atoi(ov), std::max<int64_t>(1, n)));   // test hook
    while (e->pipe_ev.size() < (size_t)(3 * n_chunks + 2)) { cudaEvent_t ev; CU(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming), "event"); e->pipe_ev.push_back(ev); }
    // fixed-length reads: arithmetic offsets and constant columns are rebuilt on the device instead of crossing PCIe
    // (24 of the 277 bytes a 150 bp read costs: brc_push_reads' admission scan found them regular)
    const int skip = e->skip_h2d;
    if (skip & 1) CU(launch_fill_offsets(e->d_in[9].as<uint64_t>(), n + 1, B.seq_off[0], B.seq_off[1] - B.seq_off[0], e->s_in), "fill seq_off");
    if (skip & 2) CU(launch_fill_offsets(e->d_in[11].as<uint64_t>(), n + 1, B.qual_off[0], B.qual_off[1] - B.qual_off[0], e->s_in), "fill qual_off");
    if (skip & 4) CU(launch_fill_i32(e->d_in[4].as<int32_t>(), n, B.l_qseq[0], e->s_in), "fill l_qseq");
    if (skip & 8) CU(launch_fill_i32(e->d_in[6].as<int32_t>(), n, B.sm[0], e->s_in), "fill sm");
    if (!B.lib) CU(cudaMemsetAsync(e->d_in[3].p, 0, (size_t)n * 2, e->s_in), "memset lib");
    // Copy order: a small cudaMemcpyAsync costs a fixed slice of link time whatever its size, so the eleven small arrays are sent
    // WHOLE, once (<= 11 copies), and only the two big byte pools are cut into chunks that the kernels and the result copies follow.
    // All of it goes on s_in, so each chunk's event also follows the small arrays.
    e->h2d_bytes_last = 0;
    #define H2D(k, host, off, cnt, esz) if ((cnt) > 0) { e->h2d_bytes_last += (int64_t)(cnt) * (int64_t)(esz); CU(cudaMemcpyAsync((char *)e->d_in[k].p + (size_t)(off) * (esz), (const char *)(host) + (size_t)(off) * (esz), (size_t)(cnt) * (esz), cudaMemcpyHostToDevice, e->s_in), "H2D"); }
    H2D(0, B.pos, 0, n, 4); H2D(1, B.flag, 0, n, 2); H2D(2, B.mapq, 0, n, 1);
    if (B.lib) H2D(3, B.lib, 0, n, 2);
    if (!(skip & 4)) H2D(4, B.l_qseq, 0, n, 4);
    H2D(5, B.nm, 0, n, 4);
    if (!(skip & 8)) H2D(6, B.sm, 0, n, 4);
    H2D(7, B.cigar_off, 0, n + 1, 8); H2D(8, B.cigar, B.cigar_off[0], B.cigar_off[n] - B.cigar_off[0], 4);
    if (!(skip & 1)) H2D(9, B.seq_off, 0, n + 1, 8);
    if (!(skip & 2)) H2D(11, B.qual_off, 0, n + 1, 8);
    for (int c = 0; c < n_chunks; ++c) {
        const int64_t a = n * c / n_chunks, b = n * (c + 1) / n_chunks;
        H2D(12, B.qual, B.qual_off[a], B.qual_off[b] - B.qual_off[a], 1);
        H2D(10, B.seq, B.seq_off[a], B.seq_off[b] - B.seq_off[a], 1);
        CU(cudaEventRecord(e->pipe_ev[2 * c], e->s_in), "event");
    }
    #undef H2D
    return BRC_OK;
}

static int compute_pipelined(brc_engine *e) {
    const brc_read_batch &B = e->borrowed;
    const int64_t n = B.n_reads;
    const brc_region &rg = e->regions[0];
    const int64_t n_tiles = (int64_t)e->tiles.size();
    const int64_t rs = (int64_t)e->n_rows * e->n_slots;
    int n_chunks = 0;
    int rc = issue_h2d_chunks(e, n_chunks);
    if (rc != BRC_OK) return rc;
    e->dev_reads = reads_dev(d_in_batch(e, n));
    // host result buffers (with a site filter only the compacted selection comes back, after the kernels: fetch_selected)
    const bool sel = e->filter_on;
    const int64_t rs1 = std::max<int64_t>(rs, 1);
    if (!sel) CU(e->h_words.reserve(rs1 * 4 * N_WORDS), "pin");
    CU(e->h_sec.reserve((size_t)e->sec_cap * sizeof(SecRec)), "pin");          // pool records leave while the kernels run
    CU(e->h_misc.reserve(64 + 4 * 64), "pin");
    if (!e->s_sec) CU(cudaStreamCreateWithFlags(&e->s_sec, cudaStreamNonBlocking), "stream");
    int32_t *h_cnt = e->h_misc.as<int32_t>() + 16;                              // pool counter after each chunk's kernels
    std::vector<int> cnt_chunks;

    PrecomputeParams P0; PileupParams P1;
    make_params(e, nullptr, P0, P1);
    cudaStream_t sk = e->stream;
    e->launch_count = 0;
    CU(cudaEventRecord(e->ev[0], sk), "event");
    CU(launch_init_tiles(P0.tile_lo, P0.tile_hi, n_tiles, P1.res.sec_count, P1.res.warn, sk), "launch init_tiles"); e->launch_count++;
    int64_t tile_done = 0;
    int k1_launches = 0;
    for (int c = 0; c < n_chunks; ++c) {
        const int64_t a = n * c / n_chunks, b = n * (c + 1) / n_chunks;
        // ---- kernels: K0 on the chunk, K1 on the tiles it completes ----
        CU(cudaStreamWaitEvent(sk, e->pipe_ev[2 * c], 0), "wait");
        P0.read_begin = a; P0.read_end = b;
        CU(launch_precompute(P0, sk), "launch read_precompute"); e->launch_count++;
        int64_t tile_to = n_tiles;
        if (c + 1 < n_chunks) {
            const int64_t next_pos = B.pos[b];
            tile_to = next_pos <= rg.first_pos ? 0 : std::min<int64_t>(n_tiles, (next_pos - rg.first_pos) / TILE);
            tile_to = std::max(tile_to, tile_done);
        }
        if (tile_to > tile_done) {
            P1.tile_begin = tile_done; P1.tile_count = tile_to - tile_done;
            CU(launch_pileup(P1, sk), "launch pileup"); e->launch_count++;
            if (P1.work_counter) P1.work_counter = ++k1_launches < N_WORK_COUNTERS ? P1.work_counter + 1 : nullptr;   // next launch: next dispenser
            CU(launch_deep_sites(P1, sk), "launch deep_sites"); if (P1.n_deep) e->launch_count++;
            CU(cudaEventRecord(e->pipe_ev[2 * c + 1], sk), "event");
            if (!sel && c < 64) {   // snapshot of the pool counter: the records allocated so far are final (a tile is computed by exactly one launch)
                CU(cudaMemcpyAsync(h_cnt + c, P1.res.sec_count, 4, cudaMemcpyDeviceToHost, sk), "D2H pool counter");
                CU(cudaEventRecord(e->pipe_ev[2 * n_chunks + 2 + (int)cnt_chunks.size()], sk), "event");
                cnt_chunks.push_back(c);
            }
            // ---- D2H of the finished slots ----
            if (sel) { tile_done = tile_to; continue; }
            CU(cudaStreamWaitEvent(e->s_out, e->pipe_ev[2 * c + 1], 0), "wait");
            const int64_t s0 = e->tiles[(size_t)tile_done].slot0;
            const int64_t s1 = tile_to < n_tiles ? e->tiles[(size_t)tile_to].slot0 : e->n_slots;
            const size_t w = (size_t)(s1 - s0);
            const size_t pitch4 = (size_t)e->n_slots * 4;
            const int rows = e->n_rows;
            // the finished slots of all N_WORDS x rows word arrays: one plain copy per array (one strided 2-D copy for many library rows)
            if (rows * N_WORDS <= 64) {      // plain copies beat one strided 2-D copy (r02e: 17.0 vs 18.4 ms per window)
                for (int k = 0; k < rows * N_WORDS; ++k)
                    CU(cudaMemcpyAsync((char *)e->h_words.p + (size_t)k * pitch4 + s0 * 4, (char *)e->d_words.p + (size_t)k * pitch4 + s0 * 4, w * 4, cudaMemcpyDeviceToHost, e->s_out), "D2H");
            } else
            CU(cudaMemcpy2DAsync((char *)e->h_words.p + s0 * 4, pitch4, (char *)e->d_words.p + s0 * 4, pitch4, w * 4, (size_t)rows * N_WORDS, cudaMemcpyDeviceToHost, e->s_out), "D2H");
            tile_done = tile_to;
        }
    }
    CU(cudaEventRecord(e->ev[1], sk), "event");
    CU(cudaEventRecord(e->ev[2], sk), "event");
    rc = launch_selection(e, sk);
    if (rc != BRC_OK) return rc;
    // everything is queued: follow the kernels and ship the pool records each chunk finished (their own stream: the word copies
    // of later chunks are already queued on s_out)
    int64_t sec_done = 0;
    for (size_t k = 0; k + 1 < cnt_chunks.size(); ++k) {     // the last chunk's records go with fetch_results
        CU(cudaEventSynchronize(e->pipe_ev[2 * n_chunks + 2 + (int)k]), "sync pool counter");
        const int64_t cur = std::min<int64_t>(h_cnt[cnt_chunks[k]], e->sec_cap);
        if (cur > sec_done) {
            CU(cudaMemcpyAsync((char *)e->h_sec.p + (size_t)sec_done * sizeof(SecRec), (char *)e->d_sec.p + (size_t)sec_done * sizeof(SecRec),
                               (size_t)(cur - sec_done) * sizeof(SecRec), cudaMemcpyDeviceToHost, e->s_sec), "D2H sec (chunk)");
            sec_done = cur;
        }
    }
    CU(cudaStreamSynchronize(e->s_in), "sync H2D");
    CU(cudaStreamSynchronize(sk), "sync kernels");
    CU(cudaStreamSynchronize(e->s_out), "sync D2H");
    int32_t cnt = 0;
    CU(cudaMemcpy(&cnt, e->d_sec_count.p, 4, cudaMemcpyDeviceToHost), "D2H sec_count");
    e->h_n_sec = cnt;
    CU(cudaStreamSynchronize(e->s_sec), "sync D2H sec");
    if ((int64_t)cnt > e->sec_cap) return BRC_E_OVERFLOW;
    return fetch_results(e, sk, true, sec_done);
}

extern "C" {

int brc_compute(brc_engine *e) {
    if (!e || e->region_open) return set_error(e, BRC_E_INVALID, "compute: a region is still open");
    cudaSetDevice(e->cfg.device);
    int rc = build_geometry(e, e->regions.data(), (int64_t)e->regions.size());
    if (rc != BRC_OK) return rc;
    plan_selection(e);
    if (e->dec.pushed) {
        // f-2: the region's reads were inflated and framed on the device (brc_push_bam_span): kernels straight on that batch
        if (!e->dec.valid || e->regions.size() != 1) return set_error(e, BRC_E_INVALID, "compute: the device-decoded batch is gone");
        if (!find_ref(e, e->regions[0].tid)) return set_error(e, BRC_E_NO_REFERENCE, "no reference for contig");
        const brc_read_batch &b = e->dec.batch;
        rc = alloc_outputs(e, b.n_reads);
        if (rc != BRC_OK) return rc;
        e->dev_reads = reads_dev(b);
        rc = compute_batch(e, std::max<int64_t>(e->sec_cap, (int64_t)e->n_rows * e->n_slots / 6 + b.n_reads / 8 + 1024), nullptr, e->stream);
        if (rc != BRC_OK) return rc;
        return brc::fetch_insertion_reads(e, e->stream);
    }
    const bool bw = e->is_borrowed;
    brc_read_batch src = e->host_batch();
    const int64_t n = src.n_reads;
    // reference window must cover every read's span (K0 reads it; the emitter reads deletion alleles)
    for (const brc_region &r : e->regions) {
        const HostRef *hr = find_ref(e, r.tid);
        if (!hr) return set_error(e, BRC_E_NO_REFERENCE, "no reference for contig");
        if (r.read_hi > r.read_lo) {
            int64_t lo = src.pos[(size_t)r.read_lo], hi = (int64_t)r.first_pos + r.n_slots;
            lo = std::max<int64_t>(0, std::min<int64_t>(lo, r.first_pos));
            hi = std::min(hi, hr->chrom_len);
            if (lo < hr->win_beg || hi > hr->win_beg + hr->win_len)
                return set_error(e, BRC_E_NO_REFERENCE, "reference window does not cover the region's reads");
        }
    }
    rc = alloc_outputs(e, n);
    if (rc != BRC_OK) return rc;
    cudaStream_t s = e->stream;
    const int64_t cap = std::max<int64_t>(e->sec_cap, (int64_t)e->n_rows * e->n_slots / 8 + 2 * e->n_indel_ops + 1024);
    if (bw && e->regions.size() == 1 && n > 0 && !e->tiles.empty()) {
        rc = upload_geometry(e, s);
        if (rc != BRC_OK) return rc;
        rc = alloc_sec(e, cap);
        if (rc != BRC_OK) return rc;
        rc = compute_pipelined(e);
        if (rc != BRC_OK && e->s_in) cudaStreamSynchronize(e->s_in);   // on an error return too, no copy from the caller's buffers outlives this call
        if (rc != BRC_E_OVERFLOW) return rc;
        // pool too small: fall through to the plain path, which grows the pool
    }
    // H2D of the read arrays (borrowed batches: straight from the caller's buffers)
    std::vector<uint16_t> zero_lib;      // a borrowed batch may come without library ids
    if (!src.lib) { zero_lib.assign((size_t)n, 0); src.lib = zero_lib.data(); }
    const void *host[14] = {src.pos, src.flag, src.mapq, src.lib, src.l_qseq, src.nm, src.sm, src.cigar_off, src.cigar, src.seq_off,
                            src.seq, src.qual_off, src.qual, bw ? nullptr : e->reads.region.data()};
    const size_t bytes[14] = {(size_t)n * 4, (size_t)n * 2, (size_t)n, (size_t)n * 2, (size_t)n * 4, (size_t)n * 4, (size_t)n * 4,
                              (size_t)(n + 1) * 8, (size_t)src.cigar_off[n] * 4, (size_t)(n + 1) * 8, (size_t)src.seq_off[n],
                              (size_t)(n + 1) * 8, (size_t)src.qual_off[n], bw ? (size_t)0 : (size_t)n * 4};
    e->h2d_bytes_last = 0;
    for (int k = 0; k < 14; ++k) {
        CU(e->d_in[k].reserve(bytes[k] + 16), "cudaMalloc(reads)");
        e->h2d_bytes_last += (int64_t)bytes[k];
        if (bytes[k]) CU(cudaMemcpyAsync(e->d_in[k].p, host[k], bytes[k], cudaMemcpyHostToDevice, s), "H2D reads");
    }
    e->dev_reads = reads_dev(d_in_batch(e, n));
    return compute_batch(e, cap, e->regions.size() > 1 ? e->d_in[13].as<int32_t>() : nullptr, s);
}

int brc_get_results(brc_engine *e, brc_results *out) {
    if (!e || !out) return BRC_E_INVALID;
    if (!e->results_valid) return set_error(e, BRC_E_INVALID, "get_results: no results (call brc_compute)");
    if (e->sparse) return set_error(e, BRC_E_INVALID, "get_results: a site filter is set, there is no dense view (brc_get_selected_results)");
    brc::ensure_wide(e);
    const brc_engine::Wide &W = e->wide;
    out->n_regions = (int64_t)e->regions.size(); out->regions = e->regions.data(); out->n_rows = e->n_rows; out->n_slots = e->n_slots;
    out->ncover = W.ncover.data(); out->npass = W.npass.data(); out->flags = W.flags.data();
    out->pbase = W.pbase.data(); out->sec_head = W.sec_head.data(); out->pstats = W.pstats.data();
    out->n_sec = W.n_sec; out->sec_next = W.sec_next.data(); out->sec_kind = W.sec_kind.data();
    out->sec_len = W.sec_len.data(); out->sec_read = W.sec_read.data(); out->sec_qpos = W.sec_qpos.data();
    out->sec_stats = W.sec_stats.data();
    return BRC_OK;
}

int brc_get_packed_results(brc_engine *e, brc_packed_results *out) {
    if (!e || !out) return BRC_E_INVALID;
    if (!e->results_valid) return set_error(e, BRC_E_INVALID, "get_packed_results: no results (call brc_compute)");
    if (e->sparse) return set_error(e, BRC_E_INVALID, "get_packed_results: a site filter is set, there is no dense view (brc_get_selected_results)");
    out->n_regions = (int64_t)e->regions.size(); out->regions = e->regions.data(); out->n_rows = e->n_rows; out->n_slots = e->n_slots;
    out->words = e->h_words.as<uint32_t>(); out->n_sec = e->h_n_sec; out->sec = e->h_sec.as<brc_sec_record>(); out->sec_count = nullptr;
    return BRC_OK;
}

int brc_get_warning_counts(brc_engine *e, int64_t out[4]) {
    if (!e || !out) return BRC_E_INVALID;
    if (e->results_valid && e->warn_counts[3] < 0) {
        // LIBRARY_UNAVAILABLE fires once per abandoned site callback (R:bamreadcount.cpp:281-284)
        int64_t lu = 0;
        if (e->cfg.per_lib && e->sparse) lu = e->sel_abandoned;   // counted by the selection's site pass
        else if (e->cfg.per_lib) {
            const uint32_t *w1 = e->h_words.as<uint32_t>() + (int64_t)e->n_rows * e->n_slots;
            for (int64_t sidx = 0; sidx < e->n_slots; ++sidx) {
                bool ab = false;
                for (int r = 0; r < e->n_rows && !ab; ++r) ab = (w1[(int64_t)r * e->n_slots + sidx] & 8u) != 0;
                lu += ab;
            }
        }
        e->warn_counts[3] = lu;
    }
    for (int k = 0; k < 4; ++k) out[k] = e->warn_counts[k] < 0 ? 0 : e->warn_counts[k];
    return BRC_OK;
}

int brc_plan_device(brc_engine *e, const brc_region *regions, int64_t n_regions, int64_t n_reads_cap, int64_t n_sec_cap) {
    if (!e || !regions || n_regions <= 0) return BRC_E_INVALID;
    cudaSetDevice(e->cfg.device);
    e->regions.assign(regions, regions + n_regions);
    e->region_open = false; e->results_valid = false;
    int rc = build_geometry(e, e->regions.data(), n_regions);
    if (rc != BRC_OK) return rc;
    rc = alloc_outputs(e, n_reads_cap);
    if (rc != BRC_OK) return rc;
    rc = alloc_sec(e, n_sec_cap > 0 ? n_sec_cap : (int64_t)e->n_rows * e->n_slots / 4 + 4096);
    if (rc != BRC_OK) return rc;
    rc = upload_geometry(e, e->stream);
    if (rc != BRC_OK) return rc;
    CU(cudaStreamSynchronize(e->stream), "sync plan");
    e->planned = true;
    return BRC_OK;
}

int brc_run_device(brc_engine *e, const brc_read_batch *b, const int32_t *dev_region_of_read, void *stream) {
    if (!e || !b) return BRC_E_INVALID;
    if (!e->planned) return set_error(e, BRC_E_INVALID, "run_device: call brc_plan_device first");
    if (e->regions.size() > 1 && !dev_region_of_read) return set_error(e, BRC_E_INVALID, "run_device: region_of_read required for >1 region");
    cudaSetDevice(e->cfg.device);
    e->dev_reads = reads_dev(*b);
    if ((size_t)std::max<int64_t>(b->n_reads, 1) * sizeof(ReadDesc) > e->d_desc.cap) return set_error(e, BRC_E_INVALID, "run_device: batch larger than planned n_reads_cap");
    e->results_valid = false;
    plan_selection(e);
    return run_kernels(e, dev_region_of_read, (cudaStream_t)stream, false);
}

int brc_device_packed_results(brc_engine *e, brc_packed_results *out) {
    if (!e || !out || !e->planned) return BRC_E_INVALID;
    out->n_regions = (int64_t)e->regions.size(); out->regions = e->regions.data(); out->n_rows = e->n_rows; out->n_slots = e->n_slots;
    out->words = e->d_words.as<uint32_t>(); out->n_sec = e->sec_cap; out->sec = e->d_sec.as<brc_sec_record>();
    out->sec_count = e->d_sec_count.as<int32_t>();
    return BRC_OK;
}

int brc_fetch_device_results(brc_engine *e, void *stream) {
    if (!e || !e->planned) return BRC_E_INVALID;
    cudaSetDevice(e->cfg.device);
    return fetch_results(e, (cudaStream_t)stream);
}

int brc_last_launch_count(const brc_engine *e) { return e ? e->launch_count : 0; }

int brc_set_site_filter(brc_engine *e, const brc_site_filter *f) {
    if (!e) return BRC_E_INVALID;
    if (!f) { e->filter_on = false; e->filter = brc_site_filter{}; return BRC_OK; }
    if (f->min_alt_count < 1 || f->reserved != 0 || !(f->min_alt_fraction >= 0.0 && f->min_alt_fraction <= 1.0))
        return set_error(e, BRC_E_INVALID, "set_site_filter: min_alt_count must be >= 1 and min_alt_fraction in [0, 1]");
    e->filter = *f; e->filter_on = true;
    return BRC_OK;
}

int brc_get_selected_results(brc_engine *e, brc_selected_results *out) {
    if (!e || !out) return BRC_E_INVALID;
    if (!e->results_valid) return set_error(e, BRC_E_INVALID, "get_selected_results: no results (call brc_compute)");
    if (!e->sparse) return set_error(e, BRC_E_INVALID, "get_selected_results: the last run had no site filter (brc_get_packed_results)");
    out->n_regions = (int64_t)e->regions.size(); out->regions = e->regions.data(); out->n_rows = e->n_rows; out->n_slots = e->n_slots;
    out->n_sites = e->n_sel; out->site = e->sel_site(); out->emit = e->sel_emit(); out->words = e->h_words.as<uint32_t>();
    out->n_sec = e->h_n_sec; out->sec = e->h_sec.as<brc_sec_record>();
    return BRC_OK;
}

int64_t brc_selftest_fastmath(brc_engine *e, int32_t max_b) {
    if (!e || max_b < 1) return BRC_E_INVALID;
    cudaSetDevice(e->cfg.device);
    unsigned long long *d_bad = nullptr, h_bad = 0;
    CU(cudaMalloc(&d_bad, 8), "cudaMalloc");
    cudaMemsetAsync(d_bad, 0, 8, e->stream);
    cudaError_t ce = launch_fastmath_selftest(max_b, d_bad, e->stream);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync(&h_bad, d_bad, 8, cudaMemcpyDeviceToHost, e->stream);
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(e->stream);
    cudaFree(d_bad);
    if (ce != cudaSuccess) return set_cuda_error(e, ce, "fastmath selftest");
    return (int64_t)h_bad;
}
int brc_host_alloc(size_t bytes, void **out) {
    if (!out) return BRC_E_INVALID;
    *out = nullptr;
    const int dev = g_last_device.load(std::memory_order_relaxed);          // a caller thread that never touched CUDA sits on device 0
    if (dev >= 0 && cudaSetDevice(dev) != cudaSuccess) { cudaGetLastError(); return BRC_E_NO_DEVICE; }
    if (cudaHostAlloc(out, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); *out = nullptr; return BRC_E_NO_DEVICE; }
    return BRC_OK;
}

void brc_host_free(void *p) { if (p) { cudaFreeHost(p); cudaGetLastError(); } }

int64_t brc_last_h2d_bytes(const brc_engine *e) { return e ? e->h2d_bytes_last : 0; }

float brc_last_stage_ms(const brc_engine *e, int stage) {
    if (!e || stage < 0 || stage > 3 || (stage == 3 && !e->sel_launched)) return 0.0f;
    // events were recorded on the launching stream around K0, K1 and the selection; wait for the last one
    if (cudaEventSynchronize(e->ev[stage == 3 ? 3 : 2]) != cudaSuccess) { cudaGetLastError(); return 0.0f; }
    float ms = 0.0f;
    const int a = stage == 2 ? 0 : stage, b = stage == 2 ? 2 : (stage == 3 ? 3 : stage + 1);
    if (stage == 3 && cudaEventElapsedTime(&ms, e->ev[2], e->ev[3]) != cudaSuccess) { cudaGetLastError(); return 0.0f; }
    if (stage != 3 && cudaEventElapsedTime(&ms, e->ev[a], e->ev[b]) != cudaSuccess) { cudaGetLastError(); return 0.0f; }
    return ms;
}

}  // extern "C"
