// brc_bgzf.cu — SURVEY.md §8 f-2: BGZF inflate + BAM record framing on the device.
//
//   bgzf_inflate_kernel   ≙ bgzf_read_block / inflate_block     V:htslib-1.10/bgzf.c:897, :697   (one warp per BGZF block)
//   bam_frame_kernel      ≙ the block_size walk of bam_read1     V:htslib-1.10/sam.c:598-612      (one thread per index entry point)
//   bam_extract_kernel    ≙ bam_read1's field decode + the aux lookups fetch_func/process_read do  V:...sam.c:613-659,
//                           R:src/lib/bamrc/BasicStat.cpp:79,94, V:bam.c:77-101 (RG -> library); the aux and CG rules: brc_aux.cuh
//   scan / copy kernels   : pool offsets (exclusive scans) and the CIGAR / base / quality bytes into the engine's SoA batch
//
// The caller hands the COMPRESSED bytes of a run of whole BGZF blocks plus the record starts the index knows (BAI linear index
// and bin chunks are virtual offsets of real record starts): each such entry starts an independent chain of block_size hops, so
// framing parallelises without guessing record boundaries.  What comes out is the brc_read_batch the kernels of
// brc_kernels.cu consume, resident in HBM — only compressed bytes cross PCIe.
#include <algorithm>
#include <cstring>
#include <vector>

#include "brc_aux.cuh"
#include "brc_bgzf.cuh"
#include "brc_engine_internal.h"
#include "brc_scan.cuh"

using namespace brc;

namespace {

struct BlockEnt { uint64_t cdata_off; uint32_t clen, isize; uint64_t uoff; };
struct RgEnt { uint64_t hash; uint16_t lib, len; char id[44]; };

__host__ __device__ inline uint64_t fnv1a(const char *s, int n) { uint64_t h = 1469598103934665603ull; for (int i = 0; i < n; ++i) { h ^= (uint8_t)s[i]; h *= 1099511628211ull; } return h; }

constexpr int INFL_WARPS = 8;

__global__ void __launch_bounds__(INFL_WARPS * 32) bgzf_inflate_kernel(const uint8_t *comp, const BlockEnt *blocks, int64_t n_blocks, uint8_t *U, int32_t *status) {
    __shared__ inflate::Tables tabs[INFL_WARPS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int64_t b = (int64_t)blockIdx.x * INFL_WARPS + warp;
    if (b >= n_blocks) return;
    // the DEFLATE symbol stream is serial: all 32 lanes run the decoder in lockstep (the cost of one), lane 0 writes tables and
    // literals, the warp copies matches together; block-level parallelism fills the GPU
    const BlockEnt e = blocks[b];
    const int rc = e.isize ? inflate::inflate_block(inflate::Lanes{lane, 32}, comp + e.cdata_off, e.clen, U + e.uoff, e.isize, tabs[warp]) : 0;
    if (rc != 0 && lane == 0) atomicMin(status, rc);
}

__device__ __forceinline__ uint32_t ld_u32(const uint8_t *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
__device__ __forceinline__ uint32_t ld_u16(const uint8_t *p) { return p[0] | (p[1] << 8); }

// chain i walks records from entry[i] up to entry[i+1] (or u_end); scratch[base[i] + k] = offset of its k-th record
__global__ void bam_frame_kernel(const uint8_t *U, int64_t u_end, const int64_t *entry, const int64_t *base, int64_t n_entry, int64_t *scratch, int32_t *count, int32_t *status) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n_entry) return;
    int64_t off = entry[i];
    const int64_t stop = i + 1 < n_entry ? entry[i + 1] : u_end;
    const int64_t cap = base[i + 1] - base[i];
    int64_t k = 0;
    while (off < stop) {
        if (off + 4 > u_end) break;                              // a record cut by the end of the span
        const int64_t bs = (int64_t)(int32_t)ld_u32(U + off);
        if (bs < 32 || off + 4 + bs > u_end) { if (bs < 32) atomicMin(status, -30); break; }
        if (k >= cap) { atomicMin(status, -31); break; }
        scratch[base[i] + k] = off;
        ++k; off += 4 + bs;
    }
    if (off > stop && i + 1 < n_entry) atomicMin(status, -32);   // the chain jumped over the next entry: the entries are not record starts
    count[i] = (int32_t)k;
}

struct ExtractArgs {
    const uint8_t *U; const int64_t *scratch; const int64_t *base; const int64_t *prefix; int64_t n_entry; int64_t n_reads;
    int32_t tid; const RgEnt *rg; int32_t n_rg;
    int32_t *pos; uint16_t *flag; uint8_t *mapq; uint16_t *lib; int32_t *l_qseq, *nm, *sm;
    int64_t *src_off;             // [2][n_reads]: offset in U of the CIGAR (the field, or a CG array), of the packed bases
    uint32_t *sz;                 // [3][n_reads]: n_cigar, seq bytes, qual bytes
    unsigned long long *max_end;
};

__global__ void bam_extract_kernel(ExtractArgs A) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= A.n_reads) return;
    // chain of record i: the last c with prefix[c] <= i
    int64_t lo = 0, hi = A.n_entry;
    while (hi - lo > 1) { const int64_t m = (lo + hi) >> 1; if (A.prefix[m] <= i) lo = m; else hi = m; }
    const int64_t off = A.scratch[A.base[lo] + (i - A.prefix[lo])];
    const uint8_t *d = A.U + off + 4;
    const int32_t bs = (int32_t)ld_u32(A.U + off);
    const int32_t refid = (int32_t)ld_u32(d), pos = (int32_t)ld_u32(d + 4);
    const uint32_t l_rn = d[8], mapq = d[9], n_cig = ld_u16(d + 12);
    uint32_t flag = ld_u16(d + 14);
    const int32_t l_seq = (int32_t)ld_u32(d + 16);
    const int64_t seq_o = 32 + (int64_t)l_rn + 4 * (int64_t)n_cig;
    const aux::RecAux ax = aux::scan(d, bs, seq_o + ((int64_t)l_seq + 1) / 2 + l_seq, 32 + l_rn, n_cig);   // NM, SM, RG, CG (brc_aux.cuh)
    uint32_t lib = BRC_LIB_NONE;
    if (ax.rg_o >= 0) {
        const int n = (int)ax.rg_len;
        const uint64_t h = fnv1a((const char *)d + ax.rg_o, n);
        for (int r = 0; r < A.n_rg; ++r) {
            if (A.rg[r].hash != h || A.rg[r].len != n) continue;
            bool same = true;
            for (int q = 0; q < n && q < 44 && same; ++q) same = A.rg[r].id[q] == (char)d[ax.rg_o + q];
            if (same) { lib = A.rg[r].lib; break; }
        }
    }
    if (refid != A.tid) flag |= 4u;                              // another contig's record inside the span: never admitted (bam_plp_push skips FUNMAP)
    A.pos[i] = pos; A.flag[i] = (uint16_t)flag; A.mapq[i] = (uint8_t)mapq; A.lib[i] = (uint16_t)lib; A.l_qseq[i] = l_seq; A.nm[i] = ax.nm; A.sm[i] = ax.sm;
    A.src_off[i] = off + 4 + ax.cig_o; A.src_off[A.n_reads + i] = off + 4 + seq_o;
    const uint32_t n_cigar = ax.n_cigar;
    A.sz[i] = n_cigar; A.sz[A.n_reads + i] = (uint32_t)((l_seq + 1) / 2); A.sz[2 * A.n_reads + i] = (uint32_t)l_seq;
    if (!(flag & 4u)) {
        int64_t rl = 0;
        for (uint32_t k = 0; k < n_cigar; ++k) { const uint32_t c = ld_u32(d + ax.cig_o + 4 * k), op = c & 15u; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rl += c >> 4; }
        const unsigned long long end = (unsigned long long)((int64_t)pos + (n_cigar ? rl : 1));
        atomicMax(A.max_end, end);
    }
}

// pool offsets: the three exclusive scans (u32 sizes -> u64 offsets) of brc_scan.cuh

// one warp per record: CIGAR ops, packed bases, qualities from the inflated bytes into the pools
__global__ void bam_copy_kernel(const uint8_t *U, const int64_t *src_off, const uint32_t *sz, int64_t n, const uint64_t *cig_off, const uint64_t *seq_off, const uint64_t *qual_off,
                                uint32_t *cigar, uint8_t *seq, uint8_t *qual) {
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= n) return;
    const uint8_t *cs = U + src_off[i];
    const uint32_t nc = sz[i], ns = sz[n + i], nq = sz[2 * n + i];
    uint32_t *c = cigar + cig_off[i];
    for (uint32_t k = lane; k < nc; k += 32) c[k] = ld_u32(cs + 4 * k);
    const uint8_t *ss = U + src_off[n + i]; uint8_t *sd = seq + seq_off[i];
    for (uint32_t k = lane; k < ns; k += 32) sd[k] = ss[k];
    const uint8_t *qs = ss + ns; uint8_t *qd = qual + qual_off[i];
    for (uint32_t k = lane; k < nq; k += 32) qd[k] = qs[k];
}

// packed bases of selected reads (those carrying an insertion allele): sizes, then bytes
__global__ void read_sizes_kernel(const uint64_t *seq_off, const int64_t *idx, int64_t m, uint32_t *sz) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < m) sz[i] = (uint32_t)(seq_off[idx[i] + 1] - seq_off[idx[i]]);
}
__global__ void read_gather_kernel(const uint8_t *seq, const uint64_t *seq_off, const int64_t *idx, const uint64_t *out_off, int64_t m, uint8_t *out) {
    const int64_t i = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (i >= m) return;
    const uint8_t *s = seq + seq_off[idx[i]];
    const uint32_t n = (uint32_t)(seq_off[idx[i] + 1] - seq_off[idx[i]]);
    uint8_t *d = out + out_off[i];
    for (uint32_t k = lane; k < n; k += 32) d[k] = s[k];
}

#define CUB(call, what) do { cudaError_t ce_ = (call); if (ce_ != cudaSuccess) return set_cuda_error(e, ce_, what); } while (0)

}  // namespace

namespace brc {
// after the kernels of a device-decoded batch: bring back the packed bases of the reads that secondary records name as
// insertion alleles (R:bamreadcount.cpp:324-330 prints them) — a few percent of the reads, the only read bytes the host needs
int fetch_insertion_reads(brc_engine *e, cudaStream_t s) {
    brc_engine::Decoded &D = e->dec;
    D.ins_reads.clear(); D.ins_off.clear(); D.ins_pool.clear();
    const SecRec *sec = e->h_sec.as<SecRec>();
    for (int64_t j = 0; j < e->h_n_sec; ++j) if ((sec[j].kind_len & 0xFFu) == (uint32_t)KIND_INS) D.ins_reads.push_back(sec[j].read);
    std::sort(D.ins_reads.begin(), D.ins_reads.end());
    D.ins_reads.erase(std::unique(D.ins_reads.begin(), D.ins_reads.end()), D.ins_reads.end());
    const int64_t m = (int64_t)D.ins_reads.size();
    if (m == 0) return BRC_OK;
    CUB(D.ins_idx.reserve((size_t)m * (8 + 8 + 4) + 64), "cudaMalloc(insertion reads)");
    int64_t *d_idx = D.ins_idx.as<int64_t>(); uint64_t *d_off = reinterpret_cast<uint64_t *>(d_idx + m); uint32_t *d_sz = reinterpret_cast<uint32_t *>(d_off + m);
    CUB(cudaMemcpyAsync(d_idx, D.ins_reads.data(), (size_t)m * 8, cudaMemcpyHostToDevice, s), "H2D insertion reads");
    read_sizes_kernel<<<(unsigned)((m + 255) / 256), 256, 0, s>>>(D.batch.seq_off, d_idx, m, d_sz);
    std::vector<uint32_t> sz((size_t)m);
    CUB(cudaMemcpyAsync(sz.data(), d_sz, (size_t)m * 4, cudaMemcpyDeviceToHost, s), "D2H sizes");
    CUB(cudaStreamSynchronize(s), "sync");
    D.ins_off.resize((size_t)m + 1); D.ins_off[0] = 0;
    for (int64_t i = 0; i < m; ++i) D.ins_off[(size_t)i + 1] = D.ins_off[(size_t)i] + sz[(size_t)i];
    D.ins_pool.resize((size_t)D.ins_off.back() + 8);
    CUB(D.ins_out.reserve((size_t)D.ins_off.back() + 64), "cudaMalloc(insertion bases)");
    CUB(cudaMemcpyAsync(d_off, D.ins_off.data(), (size_t)m * 8, cudaMemcpyHostToDevice, s), "H2D offsets");
    read_gather_kernel<<<(unsigned)((m * 32 + 255) / 256), 256, 0, s>>>(D.batch.seq, D.batch.seq_off, d_idx, d_off, m, D.ins_out.as<uint8_t>());
    CUB(cudaMemcpyAsync(D.ins_pool.data(), D.ins_out.p, (size_t)D.ins_off.back(), cudaMemcpyDeviceToHost, s), "D2H insertion bases");
    CUB(cudaStreamSynchronize(s), "sync");
    return BRC_OK;
}
}  // namespace brc

extern "C" {

int brc_decode_bam_span(brc_engine *e, const brc_bam_span *sp, brc_read_batch *out, void *stream) {
    if (!e || !sp || !out || !sp->comp || sp->comp_len <= 0 || sp->n_entry <= 0 || !sp->entry) return BRC_E_INVALID;
    cudaSetDevice(e->cfg.device);
    cudaStream_t s = stream ? (cudaStream_t)stream : e->stream;
    brc_engine::Decoded &D = e->dec;
    D.valid = false;
    // ---- 1. BGZF block table (SAM spec §4.1): header fields are tiny, the host walks them ----
    std::vector<BlockEnt> blocks; std::vector<uint64_t> bstart;
    uint64_t uoff = 0;
    for (int64_t o = 0; o + 18 <= sp->comp_len;) {
        const uint8_t *h = sp->comp + o;
        if (h[0] != 31 || h[1] != 139 || h[2] != 8 || !(h[3] & 4)) return set_error(e, BRC_E_INVALID, "decode_bam_span: not a BGZF block header");
        const size_t xlen = (size_t)(h[10] | (h[11] << 8));
        if (o + 12 + (int64_t)xlen > sp->comp_len) return set_error(e, BRC_E_INVALID, "decode_bam_span: truncated BGZF header");
        int bsize = -1;
        for (size_t i = 0; i + 4 <= xlen;) { const size_t sl = (size_t)(h[12 + i + 2] | (h[12 + i + 3] << 8)); if (h[12 + i] == 'B' && h[12 + i + 1] == 'C' && sl == 2) bsize = h[12 + i + 4] | (h[12 + i + 5] << 8); i += 4 + sl; }
        if (bsize < 0 || o + bsize + 1 > sp->comp_len || (size_t)bsize + 1 < 12 + xlen + 8) return set_error(e, BRC_E_INVALID, "decode_bam_span: truncated BGZF block");
        const uint8_t *tail = h + bsize + 1 - 4;
        const uint32_t isize = tail[0] | (tail[1] << 8) | (tail[2] << 16) | ((uint32_t)tail[3] << 24);
        if (isize > 65536) return set_error(e, BRC_E_INVALID, "decode_bam_span: BGZF block larger than 64 KiB");
        blocks.push_back(BlockEnt{(uint64_t)o + 12 + xlen, (uint32_t)(bsize + 1 - (12 + xlen) - 8), isize, uoff});
        bstart.push_back((uint64_t)o);
        uoff += isize; o += bsize + 1;
    }
    if (blocks.empty()) return set_error(e, BRC_E_INVALID, "decode_bam_span: no whole BGZF block");
    const int64_t nblk = (int64_t)blocks.size(), u_len = (int64_t)uoff;
    auto to_u = [&](uint64_t v, int64_t &u) {      // (block offset in comp) << 16 | offset in the block's data -> offset in the inflated span
        const uint64_t co = v >> 16; const auto it = std::lower_bound(bstart.begin(), bstart.end(), co);
        if (it == bstart.end() || *it != co) return false;
        const BlockEnt &b = blocks[(size_t)(it - bstart.begin())];
        if ((v & 0xFFFF) > b.isize) return false;
        u = (int64_t)(b.uoff + (v & 0xFFFF)); return true;
    };
    std::vector<int64_t> entry((size_t)sp->n_entry), base((size_t)sp->n_entry + 1, 0);
    for (int64_t i = 0; i < sp->n_entry; ++i) {
        if (!to_u(sp->entry[i], entry[(size_t)i]) || (i && entry[(size_t)i] <= entry[(size_t)i - 1])) return set_error(e, BRC_E_INVALID, "decode_bam_span: entries must be ascending record starts inside the span");
    }
    int64_t u_end = u_len;
    if (sp->end_voff >= 0 && !to_u((uint64_t)sp->end_voff, u_end)) return set_error(e, BRC_E_INVALID, "decode_bam_span: end offset not inside the span");
    for (int64_t i = 0; i < sp->n_entry; ++i) {
        const int64_t stop = i + 1 < sp->n_entry ? entry[(size_t)i + 1] : u_end;
        base[(size_t)i + 1] = base[(size_t)i] + std::max<int64_t>(stop - entry[(size_t)i], 0) / 36 + 1;     // a record is at least 36 bytes
    }
    // ---- 2. device buffers ----
    std::vector<RgEnt> rgs((size_t)std::max(sp->n_rg, 0));
    for (int r = 0; r < sp->n_rg; ++r) {
        RgEnt &g = rgs[(size_t)r]; std::memset(&g, 0, sizeof g);
        const char *id = sp->rg_id[r]; const int n = (int)std::strlen(id);
        g.hash = fnv1a(id, n); g.len = (uint16_t)n; g.lib = sp->rg_lib[r]; std::memcpy(g.id, id, (size_t)std::min(n, 44));
    }
    CUB(D.comp.reserve((size_t)sp->comp_len + 64), "cudaMalloc(comp)");
    CUB(D.btab.reserve((size_t)nblk * sizeof(BlockEnt)), "cudaMalloc(block table)");
    CUB(D.u.reserve((size_t)u_len + 64), "cudaMalloc(inflated)");
    CUB(D.meta.reserve((size_t)(sp->n_entry + 1) * 8 * 3 + 64 + rgs.size() * sizeof(RgEnt)), "cudaMalloc(entries)");
    CUB(D.scratch.reserve((size_t)base.back() * 8 + 8), "cudaMalloc(frame scratch)");
    CUB(D.count.reserve((size_t)sp->n_entry * 4 + 64), "cudaMalloc(counts)");
    int64_t *d_entry = D.meta.as<int64_t>(), *d_base = d_entry + sp->n_entry + 1, *d_prefix = d_base + sp->n_entry + 1;
    RgEnt *d_rg = reinterpret_cast<RgEnt *>(d_prefix + sp->n_entry + 1);
    int32_t *d_status = D.count.as<int32_t>() + sp->n_entry;                  // [0] status, [2..3] max_end (u64)
    unsigned long long *d_maxend = reinterpret_cast<unsigned long long *>(D.count.as<int32_t>() + ((sp->n_entry + 2 + 1) & ~1ll));
    CUB(cudaMemcpyAsync(D.comp.p, sp->comp, (size_t)sp->comp_len, cudaMemcpyHostToDevice, s), "H2D compressed span");
    CUB(cudaMemcpyAsync(D.btab.p, blocks.data(), blocks.size() * sizeof(BlockEnt), cudaMemcpyHostToDevice, s), "H2D block table");
    CUB(cudaMemcpyAsync(d_entry, entry.data(), entry.size() * 8, cudaMemcpyHostToDevice, s), "H2D entries");
    CUB(cudaMemcpyAsync(d_base, base.data(), base.size() * 8, cudaMemcpyHostToDevice, s), "H2D chain bases");
    if (!rgs.empty()) CUB(cudaMemcpyAsync(d_rg, rgs.data(), rgs.size() * sizeof(RgEnt), cudaMemcpyHostToDevice, s), "H2D read groups");
    CUB(cudaMemsetAsync(D.count.p, 0, (size_t)sp->n_entry * 4 + 64, s), "memset");
    // ---- 3. inflate, frame ----
    bgzf_inflate_kernel<<<(unsigned)((nblk + INFL_WARPS - 1) / INFL_WARPS), INFL_WARPS * 32, 0, s>>>(D.comp.as<uint8_t>(), D.btab.as<BlockEnt>(), nblk, D.u.as<uint8_t>(), d_status);
    bam_frame_kernel<<<(unsigned)((sp->n_entry + 127) / 128), 128, 0, s>>>(D.u.as<uint8_t>(), u_end, d_entry, d_base, sp->n_entry, D.scratch.as<int64_t>(), D.count.as<int32_t>(), d_status);
    CUB(cudaGetLastError(), "launch inflate/frame");
    std::vector<int32_t> cnt((size_t)sp->n_entry + 1);
    CUB(cudaMemcpyAsync(cnt.data(), D.count.p, (size_t)(sp->n_entry + 1) * 4, cudaMemcpyDeviceToHost, s), "D2H counts");
    CUB(cudaStreamSynchronize(s), "sync framing");
    if (cnt[(size_t)sp->n_entry] != 0) return set_error(e, BRC_E_INVALID, "decode_bam_span: corrupt DEFLATE stream or BAM framing (device status " + std::to_string(cnt[(size_t)sp->n_entry]) + ")");
    std::vector<int64_t> prefix((size_t)sp->n_entry + 1, 0);
    for (int64_t i = 0; i < sp->n_entry; ++i) prefix[(size_t)i + 1] = prefix[(size_t)i] + cnt[(size_t)i];
    const int64_t n = prefix.back();
    if (n >= 0x7fffffffLL) return set_error(e, BRC_E_INVALID, "decode_bam_span: too many records in one span");
    CUB(cudaMemcpyAsync(d_prefix, prefix.data(), prefix.size() * 8, cudaMemcpyHostToDevice, s), "H2D prefix");
    // ---- 4. fields, offsets, pools ----
    const size_t n1 = (size_t)std::max<int64_t>(n, 1);
    const size_t per[9] = {n1 * 4, n1 * 2, n1, n1 * 2, n1 * 4, n1 * 4, n1 * 4, n1 * 16, n1 * 12};   // pos flag mapq lib l_qseq nm sm src_off sizes
    for (int k = 0; k < 9; ++k) CUB(D.arr[k].reserve(per[k] + 64), "cudaMalloc(decoded fields)");
    for (int k = 9; k < 12; ++k) CUB(D.arr[k].reserve((n1 + 1) * 8 + 64), "cudaMalloc(decoded offsets)");
    const int64_t nb = (n + scan::SCAN_CTA - 1) / scan::SCAN_CTA;
    CUB(D.partial.reserve((size_t)(nb + 1) * 8 * 3 + 64), "cudaMalloc(scan partials)");
    ExtractArgs A{};
    A.U = D.u.as<uint8_t>(); A.scratch = D.scratch.as<int64_t>(); A.base = d_base; A.prefix = d_prefix; A.n_entry = sp->n_entry; A.n_reads = n;
    A.tid = sp->tid; A.rg = d_rg; A.n_rg = sp->n_rg;
    A.pos = D.arr[0].as<int32_t>(); A.flag = D.arr[1].as<uint16_t>(); A.mapq = D.arr[2].as<uint8_t>(); A.lib = D.arr[3].as<uint16_t>();
    A.l_qseq = D.arr[4].as<int32_t>(); A.nm = D.arr[5].as<int32_t>(); A.sm = D.arr[6].as<int32_t>(); A.src_off = D.arr[7].as<int64_t>(); A.sz = D.arr[8].as<uint32_t>();
    A.max_end = d_maxend;
    uint64_t *cig_off = D.arr[9].as<uint64_t>(), *seq_off = D.arr[10].as<uint64_t>(), *qual_off = D.arr[11].as<uint64_t>();
    unsigned long long tot[3] = {0, 0, 0};
    if (n > 0) {
        bam_extract_kernel<<<(unsigned)((n + 127) / 128), 128, 0, s>>>(A);
        scan::scan_partial_kernel<<<dim3((unsigned)nb, 3), scan::SCAN_CTA, 0, s>>>(A.sz, n, D.partial.as<unsigned long long>(), nb);
        scan::scan_top_kernel<<<3, 1024, 0, s>>>(D.partial.as<unsigned long long>(), nb);
        scan::scan_apply_kernel<<<dim3((unsigned)nb, 3), scan::SCAN_CTA, 0, s>>>(A.sz, n, D.partial.as<unsigned long long>(), nb, cig_off, seq_off, qual_off);
        CUB(cudaGetLastError(), "launch extract/scan");
        for (int k = 0; k < 3; ++k) CUB(cudaMemcpyAsync(&tot[k], D.partial.as<unsigned long long>() + (size_t)k * (nb + 1) + nb, 8, cudaMemcpyDeviceToHost, s), "D2H totals");
    } else {
        CUB(cudaMemsetAsync(cig_off, 0, 8, s), "memset"); CUB(cudaMemsetAsync(seq_off, 0, 8, s), "memset"); CUB(cudaMemsetAsync(qual_off, 0, 8, s), "memset");
    }
    unsigned long long max_end = 0;
    CUB(cudaMemcpyAsync(&max_end, d_maxend, 8, cudaMemcpyDeviceToHost, s), "D2H max_end");
    CUB(cudaStreamSynchronize(s), "sync extract");
    CUB(D.cigar.reserve((size_t)tot[0] * 4 + 64), "cudaMalloc(cigar pool)");
    CUB(D.seq.reserve((size_t)tot[1] + 64), "cudaMalloc(seq pool)");
    CUB(D.qual.reserve((size_t)tot[2] + 64), "cudaMalloc(qual pool)");
    if (n > 0) {
        bam_copy_kernel<<<(unsigned)((n * 32 + 255) / 256), 256, 0, s>>>(D.u.as<uint8_t>(), A.src_off, A.sz, n, cig_off, seq_off, qual_off, D.cigar.as<uint32_t>(), D.seq.as<uint8_t>(), D.qual.as<uint8_t>());
        CUB(cudaGetLastError(), "launch copy");
    }
    D.n_reads = n; D.max_end = (int64_t)max_end; D.n_cigar = (int64_t)tot[0]; D.n_seq = (int64_t)tot[1]; D.n_qual = (int64_t)tot[2];
    D.h2d_bytes = sp->comp_len; D.kernels = n > 0 ? 7 : 2; D.valid = true; D.stream = s;
    std::memset(out, 0, sizeof *out);
    out->n_reads = n; out->tid = nullptr; out->pos = A.pos; out->flag = A.flag; out->mapq = A.mapq; out->lib = A.lib; out->l_qseq = A.l_qseq; out->nm = A.nm; out->sm = A.sm;
    out->cigar_off = cig_off; out->cigar = D.cigar.as<uint32_t>(); out->seq_off = seq_off; out->seq = D.seq.as<uint8_t>(); out->qual_off = qual_off; out->qual = D.qual.as<uint8_t>();
    D.batch = *out;
    return BRC_OK;
}

// test / debug: the decoded batch copied to host memory the engine owns (valid until the next decode)
int brc_fetch_decoded_batch(brc_engine *e, brc_read_batch *host_out) {
    if (!e || !host_out || !e->dec.valid) return BRC_E_INVALID;
    cudaSetDevice(e->cfg.device);
    brc_engine::Decoded &D = e->dec;
    CUB(cudaStreamSynchronize(D.stream), "sync decode");     // the copy kernel may still run: cudaMemcpy does not wait for a non-blocking stream
    const size_t n = (size_t)D.n_reads;
    const size_t bytes[12] = {n * 4, n * 2, n, n * 2, n * 4, n * 4, n * 4, (n + 1) * 8, (size_t)D.n_cigar * 4, (n + 1) * 8, (size_t)D.n_seq, (n + 1) * 8};
    const void *src[13] = {D.batch.pos, D.batch.flag, D.batch.mapq, D.batch.lib, D.batch.l_qseq, D.batch.nm, D.batch.sm, D.batch.cigar_off, D.batch.cigar,
                           D.batch.seq_off, D.batch.seq, D.batch.qual_off, D.batch.qual};
    D.host.resize(13);
    for (int k = 0; k < 13; ++k) {
        const size_t b = k < 12 ? bytes[k] : (size_t)D.n_qual;
        D.host[(size_t)k].resize(b + 8);
        if (b) CUB(cudaMemcpy(D.host[(size_t)k].data(), src[k], b, cudaMemcpyDeviceToHost), "D2H decoded batch");
    }
    host_out->n_reads = D.n_reads; host_out->tid = nullptr;
    host_out->pos = (const int32_t *)D.host[0].data(); host_out->flag = (const uint16_t *)D.host[1].data(); host_out->mapq = D.host[2].data();
    host_out->lib = (const uint16_t *)D.host[3].data(); host_out->l_qseq = (const int32_t *)D.host[4].data(); host_out->nm = (const int32_t *)D.host[5].data();
    host_out->sm = (const int32_t *)D.host[6].data(); host_out->cigar_off = (const uint64_t *)D.host[7].data(); host_out->cigar = (const uint32_t *)D.host[8].data();
    host_out->seq_off = (const uint64_t *)D.host[9].data(); host_out->seq = D.host[10].data(); host_out->qual_off = (const uint64_t *)D.host[11].data(); host_out->qual = D.host[12].data();
    return BRC_OK;
}

}  // extern "C"
