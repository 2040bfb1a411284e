// brc_kernels.cu — hand-written sm_90a (H100) kernels of the pileup-readcount hot path.
//
//   K0  read_precompute_kernel  ≙ fetch_func           R:src/exe/bam-readcount/bamreadcount.cpp:114-253
//                                 + bam_plp_push admit  V:htslib-1.10/sam.c:4484-4531 (FUNMAP / tid<0)
//                                 + bam_endpos          V:htslib-1.10/sam.c:507-513
//   K1  pileup_kernel           ≙ bam_plp64_next        V:htslib-1.10/sam.c:4416-4466   (which reads span a site)
//                                 + resolve_cigar2      V:htslib-1.10/sam.c:3964-4041   (qpos / is_del / indel)
//                                 + pileup_func         R:...bamreadcount.cpp:265-346   (filters, classification)
//                                 + BasicStat::process_read  R:src/lib/bamrc/BasicStat.cpp:28-107
//
// Formulation (DESIGN.md §2): site-centric gather.  One thread owns one (site, library-row);
// it walks the reads overlapping its warp's 32 sites IN FILE ORDER and accumulates the 13
// statistics of the site's primary allele in registers.  File order per key is exactly the
// reference's accumulation order, so the four float32 sums (and the one double-rounded add)
// are bit-identical to the CPU reference at any depth (SURVEY.md §7 hard part 1) — no
// event tuples are ever written to HBM.  The site's second base class is accumulated in shared
// memory; rarer keys (a third base class, indel alleles) go to an L2-resident record pool owned
// by the same thread.
//
// Data movement: both kernels stage their read bytes with bulk TMA copies (cp.async.bulk ->
// UBLKCP) that complete on mbarriers; K1 is persistent and warp-specialised (one producer warp
// feeding a 2-stage shared-memory ring, eight consumer warps).
//
// Float arithmetic uses explicit round-to-nearest intrinsics and the library is built with
// --fmad=false: results must match the reference's x86-64 SSE arithmetic bit for bit.  The two
// shortcuts of the hot loop (reciprocal division for small integers, float<->double by bit
// casts) are exact and checked against the IEEE intrinsics by brc_selftest_fastmath.
#include <algorithm>
#include <atomic>
#include <mutex>
#include <cstdlib>

#include "brc_device.cuh"

namespace brc {

// seq_nt16_table (V:htslib-1.10/hts.c:73-91): ASCII -> 4-bit IUPAC code, 15 for anything else
__constant__ uint8_t c_nt16[256];
// bam_nt16_canonical_table (R:bamreadcount.cpp:36-39): nibble -> index into "=ACGTN"
__device__ __forceinline__ uint32_t canonical16(uint32_t nib) {
    // packed 16 x 4-bit LUT: {0,1,2,5,3,5,5,5,4,5,5,5,5,5,5,5}
    return (0x5555555455535210ull >> (nib * 4)) & 0xFu;
}

// one-time, per-device set-up (constant table, opt-in shared-memory sizes, SM count) shared by every engine handle of the
// process: callers may drive several handles from several host threads, so it is serialised and published with atomics
static std::mutex g_init_mu;
static uint8_t h_nt16[256];
static bool h_nt16_ready = false;          // guarded by g_init_mu
static void build_nt16() {
    for (int i = 0; i < 256; ++i) h_nt16[i] = 15;
    const char *s = "=ACMGRSVTWYHKDBN";
    for (int i = 0; i < 16; ++i) {
        h_nt16[(unsigned char)s[i]] = (uint8_t)i;
        if (s[i] >= 'A' && s[i] <= 'Z') h_nt16[(unsigned char)(s[i] + 32)] = (uint8_t)i;
    }
    h_nt16['0'] = 1; h_nt16['1'] = 2; h_nt16['2'] = 4; h_nt16['3'] = 8;
    h_nt16_ready = true;
}

__device__ __forceinline__ bool is_refop(uint32_t op) { return op == 0 || op == 2 || op == 3 || op == 7 || op == 8; }
__device__ __forceinline__ bool is_matchop(uint32_t op) { return op == 0 || op == 7 || op == 8; }
__device__ __forceinline__ uint32_t seq_nib(const uint8_t *seq, uint64_t off, int i) {
    uint32_t b = seq[off + (uint32_t)(i >> 1)];
    return (i & 1) ? (b & 0xFu) : (b >> 4);
}

// ---------------------------------------------------------------------------------------------
// init: tile read ranges + counters
// ---------------------------------------------------------------------------------------------
__global__ void init_tiles_kernel(int32_t *tile_lo, int32_t *tile_hi, int64_t n_tiles, int32_t *sec_count,
                                  unsigned long long *warn) {
    int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n_tiles) { tile_lo[i] = 0x7fffffff; tile_hi[i] = 0; }
    if (i == 0) { *sec_count = 0; warn[0] = 0; warn[1] = 0; }
    if (i < N_WORK_COUNTERS) warn[WARN_WORDS + i] = 0ull;   // tile dispensers of this run's pileup launches
}

cudaError_t launch_init_tiles(int32_t *tile_lo, int32_t *tile_hi, int64_t n_tiles, int32_t *sec_count,
                              unsigned long long *warn, cudaStream_t s) {
    int64_t n = n_tiles > 1 ? n_tiles : 1;
    init_tiles_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(tile_lo, tile_hi, n_tiles, sec_count, warn);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// reference window: ASCII -> 4-bit codes, once per brc_set_reference (part of load_reference, not of a step)
// ---------------------------------------------------------------------------------------------
__global__ void ref_encode_kernel(const char *ascii, uint8_t *packed, int64_t n) {
    // two bases per byte, first base in the high nibble (the BAM sequence packing), so K0 can XOR 8 bases at a time
    int64_t b = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (2 * b >= n) return;
    const uint32_t hi = c_nt16[(unsigned char)ascii[2 * b]];
    const uint32_t lo = (2 * b + 1 < n) ? c_nt16[(unsigned char)ascii[2 * b + 1]] : 15u;
    packed[b] = (uint8_t)((hi << 4) | lo);
}

static cudaError_t ensure_tables() {
    static std::atomic<bool> uploaded[64];
    int dev = 0; cudaGetDevice(&dev);
    if (dev < 64 && uploaded[dev].load(std::memory_order_acquire)) return cudaSuccess;
    std::lock_guard<std::mutex> lk(g_init_mu);
    if (!h_nt16_ready) build_nt16();
    if (dev >= 64 || !uploaded[dev].load(std::memory_order_relaxed)) {
        cudaError_t e = cudaMemcpyToSymbol(c_nt16, h_nt16, 256);
        if (e != cudaSuccess) return e;
        if (dev < 64) uploaded[dev].store(true, std::memory_order_release);
    }
    return cudaSuccess;
}

cudaError_t launch_ref_encode(const char *d_ascii, uint8_t *d_code, int64_t n, cudaStream_t s) {
    cudaError_t e = ensure_tables();
    if (e != cudaSuccess || n == 0) return e;
    const int64_t nb = (n + 1) / 2;
    ref_encode_kernel<<<(unsigned)((nb + 255) / 256), 256, 0, s>>>(d_ascii, d_code, n);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// columns of a batch of fixed-length reads the device rebuilds instead of receiving over PCIe (brc_engine.cu, push path)
// ---------------------------------------------------------------------------------------------
__global__ void fill_offsets_kernel(uint64_t *off, int64_t n, uint64_t base, uint64_t stride) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) off[i] = base + (uint64_t)i * stride;
}
__global__ void fill_i32_kernel(int32_t *dst, int64_t n, int32_t v) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < n) dst[i] = v;
}
cudaError_t launch_fill_offsets(uint64_t *off, int64_t n, uint64_t base, uint64_t stride, cudaStream_t s) {
    if (n > 0) fill_offsets_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(off, n, base, stride);
    return cudaGetLastError();
}
cudaError_t launch_fill_i32(int32_t *dst, int64_t n, int32_t v, cudaStream_t s) {
    if (n > 0) fill_i32_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(dst, n, v);
    return cudaGetLastError();
}

// --- mbarrier / bulk-TMA primitives (PTX; SASS: SYNCS.*, UBLKCP) ---
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(phase) : "memory");
}
// producer-side wait: long suspend-time hint so the idle producer lane does not burn issue slots
// consumer-side wait: probe, then back off with nanosleep so a waiting warp does not steal issue slots from the
// warps that share its scheduler (a bare try_wait loop re-issues every ~20 cycles)
template <uint32_t SLEEP_NS>
__device__ __forceinline__ void mbar_wait_hint(uint64_t *bar, uint32_t phase) {
    const uint32_t addr = smem_u32(bar);
    for (;;) {
        uint32_t ok;
        asm volatile(
            "{\n"
            ".reg .pred p;\n"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
            "selp.u32 %0, 1, 0, p;\n"
            "}\n" : "=r"(ok) : "r"(addr), "r"(phase) : "memory");
        if (ok) return;
        __nanosleep(SLEEP_NS);
    }
}
__device__ __forceinline__ void mbar_wait_relaxed(uint64_t *bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAITR_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
        "@p bra DONER_%=;\n"
        "bra WAITR_%=;\n"
        "DONER_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(phase), "r"(20000u) : "memory");
}
// global -> shared bulk copy through the TMA unit; completes on `bar` with `bytes` transaction bytes.
// dst/src 16-byte aligned, bytes a multiple of 16.
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}

// ---------------------------------------------------------------------------------------------
// K0: per-read precompute.  One CTA = K0_READS consecutive reads; their packed bases and
// qualities (two contiguous byte ranges of the pools) are staged in shared memory by bulk TMA,
// then one thread walks one read.  Reference codes come straight from global memory: reads are
// position-sorted, so a warp's 32 walks touch one or two 128-byte lines per step.
// ---------------------------------------------------------------------------------------------
// 8 consecutive 4-bit symbols starting at symbol index t of a packed array (first symbol in the high nibble of a
// byte), returned big-endian: symbol t in bits 31:28.  Reads up to 8 bytes from the aligned word holding byte t/2.
__device__ __forceinline__ uint32_t nib8(const uint8_t *base, int64_t t) {
    const uint8_t *p = base + (t >> 1);
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(p) & 3u);
    const uint32_t *w = reinterpret_cast<const uint32_t *>(p - sh);
    const uint32_t w0 = w[0], w1 = w[1];
    const uint32_t sel = (sh + 3u) | ((sh + 2u) << 4) | ((sh + 1u) << 8) | (sh << 12);
    uint32_t x = __byte_perm(w0, w1, sel);                       // bytes p[0..3], p[0] in the most significant byte
    if (t & 1) x = (x << 4) | ((__byte_perm(w0, w1, sh + 4u) >> 4) & 0xFu);
    return x;
}
// same, from shared memory with 32-bit addressing (addr = byte address of symbol 0)
__device__ __forceinline__ uint32_t nib8_smem(uint32_t addr, int t) {
    const uint32_t a = addr + (uint32_t)(t >> 1);
    const uint32_t sh = a & 3u, aw = a - sh;
    uint32_t w0, w1;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w0) : "r"(aw));
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(w1) : "r"(aw + 4u));
    const uint32_t sel = (sh + 3u) | ((sh + 2u) << 4) | ((sh + 1u) << 8) | (sh << 12);
    uint32_t x = __byte_perm(w0, w1, sel);
    if (t & 1) x = (x << 4) | ((__byte_perm(w0, w1, sh + 4u) >> 4) & 0xFu);
    return x;
}
__device__ __forceinline__ uint32_t lds_u8_k0(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint32_t nib_nonzero(uint32_t v) { return (v | (v >> 1) | (v >> 2) | (v >> 3)) & 0x11111111u; }

constexpr int K0_READS = 128;
constexpr int K0_SEQ_CAP = K0_READS * 80 + 32;
constexpr int K0_QUAL_CAP = K0_READS * 160 + 32;
constexpr int K0_REF_CAP = 4096;      // staged packed reference codes (8192 bases): the block's reads are position-sorted
struct __align__(128) K0Smem {
    uint8_t seq[K0_SEQ_CAP];
    uint8_t qual[K0_QUAL_CAP];
    uint8_t ref[K0_REF_CAP + 16];
    uint64_t bar;
};

__global__ void __launch_bounds__(K0_READS) read_precompute_kernel(PrecomputeParams P) {
    __shared__ K0Smem ks;
    const ReadsDev &R = P.reads;
    const int64_t r0 = P.read_begin + blockIdx.x * (int64_t)K0_READS;
    const int64_t r1 = min(r0 + (int64_t)K0_READS, P.read_end);
    const int64_t i = r0 + threadIdx.x;

    // stage the block's byte ranges (uniform decision)
    const uint64_t qa = R.qual_off[r0] & ~15ull, qb = (R.qual_off[r1] + 15ull) & ~15ull;
    const uint64_t sa = R.seq_off[r0] & ~15ull, sb = (R.seq_off[r1] + 15ull) & ~15ull;
    const bool staged = (qb - qa) <= (uint64_t)K0_QUAL_CAP && (sb - sa) <= (uint64_t)K0_SEQ_CAP;
    // single-region batches: the block's reads are position-sorted on one contig, so the reference codes they
    // touch are one short window — stage it too (reads reaching past it fall back to global loads per op)
    int64_t ra = 0, rb = 0;   // staged byte range of the packed reference, [ra, rb)
    if (staged && P.n_regions == 1) {
        const RefWin rw0 = P.refs[P.regions[0].tid_slot];
        const int64_t p_first = (int64_t)R.pos[r0] - rw0.win_beg, p_last = (int64_t)R.pos[r1 - 1] - rw0.win_beg;
        const int64_t nbytes = (rw0.win_len + 1) / 2 + 16;            // allocation is padded by >= 16 bytes of 'N'
        ra = (p_first > 0 ? p_first >> 1 : 0) & ~15ll;
        rb = min((((p_last + 1024) >> 1) + 31) & ~15ll, nbytes & ~15ll);
        if (rb <= ra || rb - ra > K0_REF_CAP) { ra = rb = 0; }
    }
    if (staged) {
        if (threadIdx.x == 0) {
            mbar_init(&ks.bar, 1);
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            mbar_expect_tx(&ks.bar, (uint32_t)(qb - qa) + (uint32_t)(sb - sa) + (uint32_t)(rb - ra));
            tma_bulk_g2s(ks.qual, R.qual + qa, (uint32_t)(qb - qa), &ks.bar);
            tma_bulk_g2s(ks.seq, R.seq + sa, (uint32_t)(sb - sa), &ks.bar);
            if (rb > ra) tma_bulk_g2s(ks.ref, reinterpret_cast<const uint8_t *>(P.refs[P.regions[0].tid_slot].seq) + ra, (uint32_t)(rb - ra), &ks.bar);
        }
        __syncthreads();   // barrier initialised before anyone waits on it
    }
    const bool live = i < r1;
    // per-read scalars: coalesced global loads, overlapped with the bulk copies
    int32_t pos = 0, l_qseq = 0, nm = 0, smtag = 0; uint32_t flag = 0, mapq = 0, lib = 0, n_cigar = 0;
    uint64_t coff = 0, soff = 0, qoffb = 0;
    RegionDev rg{}; RefWin rw{};
    if (live) {
        const int32_t g = P.region_of_read ? P.region_of_read[i] : 0;
        rg = P.regions[g]; rw = P.refs[rg.tid_slot];
        pos = R.pos[i]; flag = R.flag[i]; mapq = R.mapq[i]; l_qseq = R.l_qseq[i]; nm = R.nm[i]; smtag = R.sm[i];
        lib = R.lib ? (uint32_t)R.lib[i] : 0u;
        coff = R.cigar_off[i]; n_cigar = (uint32_t)(R.cigar_off[i + 1] - coff);
        soff = R.seq_off[i]; qoffb = R.qual_off[i];
    }
    if (staged) mbar_wait(&ks.bar, 0);
    const unsigned live_mask = __ballot_sync(0xffffffffu, live);
    if (!live) return;
    const uint32_t *cig = R.cigar + coff;
    // generic pointers: shared memory when staged, the global pools otherwise (reads too long for the stage)
    const uint8_t *seq = staged ? (ks.seq + (soff - sa)) : (R.seq + soff);
    const uint8_t *qual = staged ? (ks.qual + (qoffb - qa)) : (R.qual + qoffb);
    const uint32_t seq_sa = smem_u32(ks.seq) + (uint32_t)(soff - sa), qual_sa = smem_u32(ks.qual) + (uint32_t)(qoffb - qa);   // staged: 32-bit shared addresses
    const uint32_t ref_sa = smem_u32(ks.ref) - (uint32_t)ra;
    const uint8_t *refc = reinterpret_cast<const uint8_t *>(rw.seq);   // packed 4-bit codes (launch_ref_encode)

    // --- fetch_func CIGAR/reference walk (R:...:133-199) + bam_cigar2rlen + SIMPLE detection ---
    // Flattened into ONE loop whose iterations are either "fetch the next CIGAR op" or "compare 8 bases of the
    // current M op", so the 32 reads of a warp stay converged whatever their CIGAR shapes are.
    uint32_t sum_mmq = 0;
    int left_clip = 0, clipped_length = l_qseq, right_clip = l_qseq;
    int last_mm_pos = -1, last_mm_qual = 0;
    int64_t reference_position = pos;
    int read_position = 0;
    bool walking = true;            // false after the reference's `break` out of the op loop
    int64_t rlen = 0;               // reference span (all ref-consuming ops, incl. = and X)
    int n_refops = 0, qoff = 0;
    bool simple = true, seen_ref = false;
    uint32_t k = 0;
    bool in_m = false, hit_nul = false;
    int j = 0, jend = 0, m_len = 0;
    int64_t wrel = 0;
    bool ref_staged = false;
    for (;;) {
        if (!in_m) {
            if (k >= n_cigar) break;
            const uint32_t c = cig[k];
            const int op_length = (int)(c >> 4);
            const uint32_t op = c & 0xFu;
            if (is_refop(op)) { rlen += op_length; n_refops++; seen_ref = true; if (!is_matchop(op)) simple = false; }
            else if (op == 1 || op == 6) simple = false;
            else if (op == 4 && !seen_ref) qoff += op_length;
            if (walking) {
                if (op == 0) {
                    // positions whose reference base exists: [0, jn); at refpos == chrom_len the reference string's NUL stops the walk
                    int jn = op_length;
                    hit_nul = false;
                    if (reference_position + op_length > rw.chrom_len) {
                        if (rg.ref_len_check && reference_position > rw.chrom_len) jn = 0;   // -l mode: every position is skipped (R:...:144-148)
                        else { const int64_t room = rw.chrom_len - reference_position; jn = room > 0 ? (int)room : 0; hit_nul = true; }
                    }
                    // positions outside the supplied reference window count as 'N' (no mismatch): clip to the window
                    wrel = reference_position - rw.win_beg;
                    j = wrel < 0 ? (int)min((int64_t)jn, -wrel) : 0;
                    jend = (int)max((int64_t)j, min((int64_t)jn, rw.win_len - wrel));
                    // reference codes of this op: the staged window when it holds all of them (nib8 may read 8 bytes on)
                    ref_staged = rb > ra && ((wrel + j) >> 1) >= ra && ((wrel + jend) >> 1) + 8 < rb;
                    m_len = op_length; in_m = true;
                } else if (op == 2 || op == 3) reference_position += op_length;
                else if (op == 1) read_position += op_length;
                else if (op == 4) {
                    read_position += op_length; clipped_length -= op_length;
                    if (k == 0) left_clip += op_length; else right_clip -= op_length;
                }
            }
            ++k;
            continue;
        }
        if (j < jend) {
            // 8 bases per step: XOR of the packed read nibbles with the packed reference codes
            const uint32_t X = staged ? nib8_smem(seq_sa, read_position + j) : nib8(seq, read_position + j);
            const uint32_t Y = ref_staged ? nib8_smem(ref_sa, (int)(wrel + j)) : nib8(refc, wrel + j);
            const uint32_t x = X ^ Y;
            if (x != 0u) {
                const int nv = jend - j;
                const uint32_t keep = nv >= 8 ? 0xFFFFFFFFu : ~(0xFFFFFFFFu >> (4 * nv));
                // mismatch iff read != ref && ref != 15 && read != 0   (R:...:152)
                uint32_t m = nib_nonzero(x) & ~((Y & (Y >> 1) & (Y >> 2) & (Y >> 3)) & 0x11111111u) & nib_nonzero(X) & keep;
                while (m) {
                    const int k8 = __clz(m) >> 2;          // flag of symbol i sits at bit 28-4i
                    m &= ~(0x10000000u >> (4 * k8));
                    const int cur = read_position + j + k8;
                    const int q = staged ? (int)lds_u8_k0(qual_sa + (uint32_t)cur) : (int)qual[cur];
                    if (last_mm_pos != -1) {
                        if (last_mm_pos + 1 != cur) { sum_mmq += (uint32_t)last_mm_qual; last_mm_qual = q; }
                        else if (last_mm_qual < q) last_mm_qual = q;
                        last_mm_pos = cur;
                    } else { last_mm_pos = cur; last_mm_qual = q; }
                }
            }
            j += 8;
            continue;
        }
        // M op finished.  Site-list mode skips positions beyond chrom_len (R:...:144-148) but position == chrom_len still reads the NUL.
        if (hit_nul) walking = false;
        else { reference_position += m_len; read_position += m_len; }
        in_m = false;
    }
    sum_mmq += (uint32_t)last_mm_qual;
    if (n_refops != 1) simple = false;

    // --- Q2 run / effective 3' end (R:...:202-238) ---
    int tpi, q2_pos = -1, kk, inc;
    const bool reverse = (flag & 16u) != 0;
    if (reverse) { kk = tpi = 0; inc = 1; if (tpi < left_clip) tpi = left_clip; }
    else { kk = tpi = l_qseq - 1; inc = -1; if (tpi > right_clip) tpi = right_clip; }
    while (kk >= 0 && kk < l_qseq) {
        if ((staged ? lds_u8_k0(qual_sa + (uint32_t)kk) : (uint32_t)qual[kk]) != 2u) { q2_pos = kk - 1; break; }
        kk += inc;
    }
    if (reverse) { if (tpi < q2_pos) tpi = q2_pos; }
    else { if (tpi > q2_pos && q2_pos != -1) tpi = q2_pos; }

    // --- admission (bam_plp_push) and span (bam_endpos) ---
    const bool unmapped = (flag & 4u) != 0;
    int64_t end = (!unmapped && n_cigar > 0) ? (int64_t)pos + rlen : (int64_t)pos + 1;
    if (unmapped) end = pos;      // never admitted to the pileup: covers nothing

    ReadDesc d;
    d.pos = pos; d.end = (int32_t)end; d.fl = (float)l_qseq;
    uint32_t fm = (flag & 0xFFFFu) | (mapq << 16);
    if (simple) fm |= FM_SIMPLE;
    const int32_t sm = smtag;
    if (nm == INT32_MIN) fm |= FM_NM_ABSENT;
    int32_t se;
    if (flag & 2u) { if (sm != INT32_MIN) se = sm; else { se = 0; fm |= FM_SM_MISSING; } }
    else se = (int32_t)mapq;
    const bool fast = l_qseq >= 1 && l_qseq <= FASTDIV_MAX && clipped_length >= 1 && clipped_length <= FASTDIV_MAX;
    if (fast) fm |= FM_FASTDIV;
    if (simple && fast && !(fm & (FM_NM_ABSENT | FM_SM_MISSING))) fm |= FM_HOT;
    if ((int)mapq < P.min_mapq || (flag & FLAG_FILTER)) fm |= FM_DEAD;
    d.fm = fm;
    d.mmq = (int32_t)sum_mmq; d.clen = clipped_length; d.lclip = left_clip; d.tpi = tpi;
    d.q2 = q2_pos;
    d.nmfrac = (nm == INT32_MIN) ? 0.0f : __fdiv_rn((float)nm, (float)clipped_length);
    d.se = se;
    d.lib_nc = lib | ((n_cigar > 0xFFFFu ? 0xFFFFu : n_cigar) << 16);
    d.qual32 = (uint32_t)qoffb; d.seq32 = (uint32_t)soff;
    d.cig = simple ? (uint32_t)qoff : (uint32_t)coff; d.n_cigar = n_cigar;
    d.rcp_l = fast ? __frcp_rn((float)l_qseq) : 0.0f;
    d.rcp_clen = fast ? __frcp_rn((float)clipped_length) : 0.0f;
    d.fclen = (float)clipped_length; d.inc = 1u | ((flag & 16u) ? 0u : 256u) | (q2_pos > -1 ? 65536u : 0u);
    // 5 x 16-byte stores
    int4 *dst = reinterpret_cast<int4 *>(P.desc + i);
    const int4 *src = reinterpret_cast<const int4 *>(&d);
#pragma unroll
    for (int q = 0; q < 5; ++q) dst[q] = src[q];

    // --- which tiles of this read's region does it overlap?  (first/last read per tile) ---
    // Lanes of a warp hold consecutive reads, so a tile's smallest read index comes from the lowest lane touching
    // it and the largest from the highest: a lane skips the atomic when its neighbour covers the same tile
    // (32x fewer same-address atomics on deep sites).
    int64_t a = pos > rg.first_pos ? pos : rg.first_pos;
    int64_t b = end < rg.end ? end : rg.end;
    const bool has = b > a;
    const int64_t t0 = has ? rg.tile_base + (a - rg.first_pos) / TILE : 1;
    const int64_t t1 = has ? rg.tile_base + (b - 1 - rg.first_pos) / TILE : 0;    // empty range when !has
    const int lane = threadIdx.x & 31;
    const int64_t p0 = __shfl_up_sync(live_mask, t0, 1), p1 = __shfl_up_sync(live_mask, t1, 1);
    const int64_t n0 = __shfl_down_sync(live_mask, t0, 1), n1 = __shfl_down_sync(live_mask, t1, 1);
    const bool has_prev = lane > 0, has_next = lane < 31 && ((live_mask >> (lane + 1)) & 1u);
    const int32_t idx = (int32_t)i;
    for (int64_t t = t0; t <= t1; ++t) {
        if (!(has_prev && p0 <= t && t <= p1)) atomicMin(P.tile_lo + t, idx);
        if (!(has_next && n0 <= t && t <= n1)) atomicMax(P.tile_hi + t, idx + 1);
    }
}

cudaError_t launch_precompute(const PrecomputeParams &p, cudaStream_t s) {
    cudaError_t e = ensure_tables();
    if (e != cudaSuccess) return e;
    const int64_t n = p.read_end - p.read_begin;
    if (n <= 0) return cudaSuccess;
    read_precompute_kernel<<<(unsigned)((n + K0_READS - 1) / K0_READS), K0_READS, 0, s>>>(p);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// K1: site-centric pileup + ordered accumulation.
//
// Persistent, warp-specialised CTAs (DESIGN.md §4.2): warp 8 is the PRODUCER — it walks this CTA's
// tiles, cuts each tile's position-sorted read range into chunks and streams every chunk
// (descriptors + quality bytes + packed bases) into a 2-stage shared-memory ring with bulk-TMA copies
// that complete on an mbarrier; warps 0-7 are CONSUMERS — thread = site, each warp walks the staged
// reads in file order and accumulates in registers.  full/empty mbarriers are the only
// synchronisation, so chunk i+1 is in flight while chunk i is being consumed.
// ---------------------------------------------------------------------------------------------
#ifdef BRC_K1_PROFILE
__device__ unsigned long long g_k1prof[8];   // [0] consumer wait, [1] consumer busy, [2] producer wait-empty, [3] producer issue, [4] items
#endif
constexpr int N_CONSUMER_WARPS = TILE / 32;
constexpr int K1_THREADS = TILE + 32;
constexpr int NSTAGE = 2;
#ifndef BRC_K1_CTAS_PER_SM
#define BRC_K1_CTAS_PER_SM 3
#endif

struct Acc {  // 13 accumulators in registers (print order BRC_S_*); minus strand = count - plus
    uint32_t count, mapq, baseq, se, plus;
    float nmf;
    uint32_t mmqs, nq2;
    float q2d;
    uint32_t clip;
    float d3p;
    double posd;  // sum_event_location, always holding a float32-representable value
};

// RN_f32(x) as a double, for finite |x| in the float32 normal range, without F2F conversions:
// adding and subtracting C = 2^(e+29) (e = exponent of x) rounds x to 24 significant bits, ties to even.
__device__ __forceinline__ double round_to_f32_precision(double x) {
    const int hi = __double2hiint(x);
    const double c = __hiloint2double((hi & (int)0xfff00000) + (29 << 20), 0);   // copysign(2^(e+29), x)
    return __dsub_rn(__dadd_rn(x, c), c);
}
// exact float32 -> float64 for finite, non-denormal f >= 0 (and +0) by bit manipulation
__device__ __forceinline__ double f32_to_f64_nonneg(float f) {
    const uint32_t b = __float_as_uint(f);
    const uint32_t hi = b == 0u ? 0u : (b >> 3) + (896u << 20);
    return __hiloint2double((int)hi, (int)(b << 29));
}
// RN(a / b) for small non-negative integer-valued a and positive integer-valued b <= FASTDIV_MAX with rcp = RN(1/b):
// one Newton step on the product (Markstein); verified exhaustively against __fdiv_rn by the GPU tests.
__device__ __forceinline__ float div_small(float a, float b, float rcp) {
    const float q0 = __fmul_rn(a, rcp);
    const float r = __fmaf_rn(-b, q0, a);
    return __fmaf_rn(r, rcp, q0);
}

// One (site, read) event's contributions — the body of BasicStat::process_read (R:BasicStat.cpp:28-107).
struct Terms { float q2term, d3pterm, posf; double posterm; };   // posterm == 1.0 - (double)posf
__device__ __forceinline__ Terms event_terms(bool fast, int qpos, int q2pos, int tpi, int lclip, int clen, float fl, float fclen,
                                             float rcp_l, float rcp_c) {
    Terms t;
    const float a_3p = (float)abs(qpos - tpi);
    if (fast) {
        t.d3pterm = div_small(a_3p, fl, rcp_l);
        // the Q2 term is only accumulated when the read has a Q2 position, and for most forward reads that position IS
        // the effective 3' end (R:...:229-238): both tests are uniform across the warp (one read per iteration)
        t.q2term = (q2pos < 0 || q2pos == tpi) ? t.d3pterm : div_small((float)abs(qpos - q2pos), fl, rcp_l);
        // |(qpos-lclip) - clen/2| / (clen/2)  ==  |2(qpos-lclip) - clen| / clen   (numerator and denominator exact)
        const float f = div_small((float)abs(2 * (qpos - lclip) - clen), fclen, rcp_c);
        t.posf = f;
        t.posterm = __dsub_rn(1.0, f32_to_f64_nonneg(f));
    } else {
        t.q2term = __fdiv_rn((float)abs(qpos - q2pos), fl);
        t.d3pterm = __fdiv_rn(a_3p, fl);
        const float rc = __fmul_rn(fclen, 0.5f);
        const float f = __fdiv_rn(fabsf(__fsub_rn((float)(qpos - lclip), rc)), rc);
        t.posf = f;
        t.posterm = __dsub_rn(1.0, (double)f);
    }
    return t;
}

// stateless resolve_cigar2.  Returns {qpos, indel, is_del}.
__device__ __noinline__ int3 resolve_general(const uint32_t *cig, uint32_t n_cigar, int32_t pos, int32_t site) {
    int64_t x = pos; int y = 0; uint32_t k = 0; uint32_t op = 0; int len = 0;
    for (; k < n_cigar; ++k) {
        const uint32_t c = cig[k]; op = c & 0xFu; len = (int)(c >> 4);
        if (is_refop(op)) {
            if ((int64_t)site < x + len) break;
            x += len; if (is_matchop(op)) y += len;
        } else if (op == 1 || op == 4) y += len;
    }
    int3 out = make_int3(0, 0, 0);
    if (k >= n_cigar) { out.z = 1; return out; }  // cannot happen for pos <= site < end
    if (is_matchop(op)) out.x = y + (int)(site - x); else { out.z = 1; out.x = y; }
    if (x + len - 1 == site && k + 1 < n_cigar) {
        const uint32_t c2 = cig[k + 1]; const uint32_t op2 = c2 & 0xFu; const int l2 = (int)(c2 >> 4);
        if (op2 == 2) out.y = -l2;
        else if (op2 == 1) out.y = l2;
        else if (op2 == 6 && k + 2 < n_cigar) {
            int l3 = 0;
            for (uint32_t m = k + 2; m < n_cigar; ++m) {
                const uint32_t c3 = cig[m]; const uint32_t op3 = c3 & 0xFu;
                if (op3 == 1) l3 += (int)(c3 >> 4);
                else if (op3 == 2 || op3 == 0 || op3 == 3 || op3 == 7 || op3 == 8) break;
            }
            if (l3 > 0) out.y = l3;
        }
    }
    return out;
}

// Rare keys (indel alleles, a third base class at a site): find-or-append a record in the thread's private
// chain in the L2-resident pool and accumulate there.  Recomputes the event from the global descriptor so
// the hot loop carries no state for it.  Returns the new chain head.
//
// What the rare path reads, passed BY VALUE: a reference to the kernel's parameter block would make every kernel that
// calls these out-of-line functions copy the whole block to local memory and read its fields back from there, the hot
// loop's base-quality threshold included.
struct RareCtx {
    const ReadDesc *desc;
    const uint8_t *seq;
    const uint64_t *seq_off;
    SecRec *sec;
    int32_t *sec_count;
    int64_t sec_cap;
};
__device__ __forceinline__ RareCtx rare_ctx(const PileupParams &P) {
    return RareCtx{P.desc, P.seq, P.seq_off, P.res.sec, P.res.sec_count, P.res.sec_cap};
}
__device__ __forceinline__ bool same_insertion(const RareCtx &C, int32_t read_a, int qpos_a, int32_t read_b, int qpos_b, int len) {
    // same inserted bases?  compare canonicalised read bases (R:bamreadcount.cpp:324-330)
    const uint64_t oa = C.seq_off[read_a], ob = C.seq_off[read_b];
    bool same = true;
    for (int k = 1; k <= len && same; ++k)
        same = canonical16(seq_nib(C.seq, oa, qpos_a + k)) == canonical16(seq_nib(C.seq, ob, qpos_b + k));
    return same;
}
__device__ __forceinline__ void sec_init(SecRec &r, uint32_t slot, int32_t next, uint32_t kind, uint32_t len, int32_t read, int32_t qpos) {
    r.slot = slot; r.next = next; r.kind_len = kind | (len << 8); r.read = read; r.qpos = qpos;
#pragma unroll
    for (int k = 0; k < N_STATS; ++k) r.stats[k] = 0u;
}
// one event of BasicStat::process_read into a pool record (slow, exact IEEE path)
__device__ __forceinline__ void sec_accumulate(const ReadDesc *desc, SecRec &r, int32_t read, int qpos, uint32_t bq, bool is_indel) {
    const ReadDesc d = desc[read];
    const Terms t = event_terms(false, qpos, d.q2, d.tpi, d.lclip, d.clen, d.fl, d.fclen, 0.f, 0.f);
    uint32_t v[N_STATS];
#pragma unroll
    for (int k = 0; k < N_STATS; ++k) v[k] = r.stats[k];
    v[0] += 1u;
    v[1] += (d.fm >> 16) & 0xFFu;
    if (!is_indel) v[2] += bq;
    v[3] += (uint32_t)d.se;
    if (d.fm & 16u) v[5] += 1u; else v[4] += 1u;
    v[6] = __float_as_uint(__double2float_rn(__dadd_rn((double)__uint_as_float(v[6]), t.posterm)));
    v[7] = __float_as_uint(__fadd_rn(__uint_as_float(v[7]), d.nmfrac));
    v[8] += (uint32_t)d.mmq;
    if (d.q2 > -1) { v[9] += 1u; v[10] = __float_as_uint(__fadd_rn(__uint_as_float(v[10]), t.q2term)); }
    v[11] += (uint32_t)d.clen;
    v[12] = __float_as_uint(__fadd_rn(__uint_as_float(v[12]), t.d3pterm));
#pragma unroll
    for (int k = 0; k < N_STATS; ++k) r.stats[k] = v[k];
}
// find-or-append of the allele's record in the chain starting at `head`; returns the record index (>= sec_cap on overflow:
// the host sees sec_count > cap and retries with a larger pool)
__device__ __noinline__ int32_t rare_find_or_append(const RareCtx C, int32_t &head, uint32_t slot, int kind, int len, int32_t read, int qpos) {
    const uint32_t want = (uint32_t)kind | ((uint32_t)len << 8);
    int32_t j = head;
    while (j >= 0) {
        const SecRec &r = C.sec[j];
        if (r.kind_len == want && (kind != KIND_INS || same_insertion(C, read, qpos, r.read, r.qpos, len))) break;
        j = r.next;
    }
    if (j < 0) {
        j = atomicAdd(C.sec_count, 1);
        if ((int64_t)j >= C.sec_cap) return j;
        sec_init(C.sec[j], slot, head, (uint32_t)kind, (uint32_t)len, read, qpos);
        head = j;
    }
    return j;
}
__device__ __noinline__ int32_t rare_event(const RareCtx C, int32_t head, uint32_t slot, int kind, int len, int32_t read, int qpos,
                                           uint32_t bq, bool is_indel) {
    const int32_t j = rare_find_or_append(C, head, slot, kind, len, read, qpos);
    if ((int64_t)j < C.sec_cap) sec_accumulate(C.desc, C.sec[j], read, qpos, bq, is_indel);
    return head;
}

struct __align__(16) ChunkInfo {
    int32_t work;        // work item (row * n_tiles + tile), -1 = no more work
    int32_t r0, r1;      // reads [r0, r1) staged in this slot
    uint32_t qbase32, sbase32;
    uint32_t flags;      // bit0 staged (qual/seq in smem), bit1 first chunk of the tile, bit2 last chunk of the tile, bit3 narrow -p tile,
                         // bit4 CIGAR ops staged (cbase32 = index of the first staged op)
    int32_t pos0, n;     // TileInfo
    int64_t slot0;
    uint32_t row, cbase32;
};
struct __align__(128) StageBuf {
    int4 desc[(STAGE_READS + 2) * 5];   // + the sentinel the producer writes behind the chunk's last descriptor, + the record the
                                        // consumers load (and never use) as the sentinel's pair partner
    uint8_t qual[STAGE_QUAL];
    uint8_t seq[STAGE_SEQ];
    uint32_t cigar[STAGE_CIGAR];
};
struct __align__(128) PileupSmem {
    StageBuf st[NSTAGE];
    uint32_t sacc[N_STATS][TILE];   // second base class of each site (stat-major: conflict-free)
    uint32_t warn[2][TILE];         // per-thread warning counters (NM missing, SM missing): off the register file
    ChunkInfo info[NSTAGE];
    uint64_t full[NSTAGE], empty[NSTAGE];
};

__device__ __forceinline__ uint32_t lds_u8(uint32_t addr) {
    uint32_t v;
    asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

// per-thread (= per-site) state of a consumer, all in registers
struct SiteState {
    Acc acc;
    uint32_t ncover, npass, flags, pbase, sbase;
    int32_t sec_head;
    bool warp_done;
    int32_t site;      // -1 for lanes beyond the tile's last site (never covered: positions are >= 0)
    int32_t wfirst;    // first site of this warp; the warp's window is [wfirst, wfirst+31]
    uint32_t row;      // library row this thread accumulates
};
template <bool PER_LIB>
__device__ __forceinline__ void site_reset(SiteState &S, const ChunkInfo &ci, int tid, int n_rows) {
    Acc &a = S.acc;
    a.count = a.mapq = a.baseq = a.se = a.plus = a.mmqs = a.nq2 = a.clip = 0;
    a.nmf = a.q2d = a.d3p = 0.0f; a.posd = 0.0;
    S.ncover = S.npass = 0; if (PER_LIB) S.flags = 0; S.pbase = S.sbase = NO_BASE; S.sec_head = -1;
    if (PER_LIB && (ci.flags & 8u)) {   // narrow tile: warp = library row, lane = site
        const int lane = tid & 31;
        S.row = ci.row + (uint32_t)(tid >> 5);
        const bool ok = S.row < (uint32_t)n_rows && lane < ci.n;
        S.site = ok ? ci.pos0 + lane : -1;
        S.wfirst = ci.pos0;
        S.warp_done = S.row >= (uint32_t)n_rows;
    } else {
        S.row = PER_LIB ? ci.row : 0u;
        S.site = tid < ci.n ? ci.pos0 + tid : -1;
        S.wfirst = ci.pos0 + (tid & ~31);
        S.warp_done = (tid & ~31) >= ci.n;
    }
}

// shared-memory loads by 32-bit address: the hot loop walks the staged descriptors with one 32-bit register instead of a
// generic 64-bit pointer plus its shared-window twin (ncu r02a: three loop values were spilled to local memory)
__device__ __forceinline__ int2 lds64(uint32_t a) { int2 v; asm volatile("ld.shared.v2.u32 {%0,%1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a)); return v; }
__device__ __forceinline__ int4 lds128(uint32_t a) { int4 v; asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a)); return v; }
// row * n_slots + slot of the site this thread owns
template <bool PER_LIB>
__device__ __forceinline__ uint32_t slot_index(const PileupParams &P, const ChunkInfo &ci, const SiteState &S) {
    return (uint32_t)((PER_LIB ? (int64_t)S.row * P.res.n_slots : 0) + ci.slot0 + (S.site - ci.pos0));
}
constexpr uint32_t DSZ = (uint32_t)sizeof(ReadDesc);

// A passing event whose base is not the site's primary class: the site's second base class accumulates in shared memory,
// a third one in the record pool.  `da` = the read's staged descriptor, `read` its index.
template <bool PER_LIB>
__device__ __forceinline__ void off_primary_event(const PileupParams &P, uint32_t (*sacc)[TILE], const ChunkInfo &ci, SiteState &S, int tid,
                                                  uint32_t da, int32_t read, bool fast, uint32_t fm, int qpos, uint32_t bq, uint32_t base) {
    if (S.sbase != NO_BASE && base != S.sbase) {   // third base class at this site: rare
        S.sec_head = rare_event(rare_ctx(P), S.sec_head, slot_index<PER_LIB>(P, ci, S), (int)base, 0, read, qpos, bq, false);
        return;
    }
    const int4 q1 = lds128(da + 16u);                            // mmq,clen,lclip,tpi
    const int4 q2 = lds128(da + 32u);                            // q2,nmfrac,se,fl
    const int4 q4 = lds128(da + 64u);                            // rcp_l, rcp_clen, fclen
    const Terms t = event_terms(fast, qpos, q2.x, q1.w, q1.z, q1.y, __int_as_float(q2.w), __int_as_float(q4.z),
                                __int_as_float(q4.x), __int_as_float(q4.y));
    const uint32_t plus = (fm & 16u) ? 0u : 1u;
    if (S.sbase == NO_BASE) {
        S.sbase = base;
#pragma unroll
        for (int k = 0; k < N_STATS; ++k) sacc[k][tid] = 0u;
    }
    sacc[0][tid] += 1u; sacc[1][tid] += (fm >> 16) & 0xFFu; sacc[2][tid] += bq; sacc[3][tid] += (uint32_t)q2.z;
    sacc[4][tid] += plus; sacc[5][tid] += 1u - plus;
    sacc[6][tid] = __float_as_uint(__double2float_rn(__dadd_rn((double)__uint_as_float(sacc[6][tid]), t.posterm)));
    sacc[7][tid] = __float_as_uint(__fadd_rn(__uint_as_float(sacc[7][tid]), __int_as_float(q2.y)));
    sacc[8][tid] += (uint32_t)q1.x;
    if (q2.x > -1) { sacc[9][tid] += 1u; sacc[10][tid] = __float_as_uint(__fadd_rn(__uint_as_float(sacc[10][tid]), t.q2term)); }
    sacc[11][tid] += (uint32_t)q1.y;
    sacc[12][tid] = __float_as_uint(__fadd_rn(__uint_as_float(sacc[12][tid]), t.d3pterm));
}

// Two consecutive staged FM_HOT reads A (descriptor at `da`) and B (at da + DSZ) in one body without branches: every lane
// computes both events (a lane off a read loads a valid byte of it and drops the result) and applies them as predicated
// updates, A before B, so each accumulator still sees file order.  Only the rare event that is not the site's primary class
// (a second or third base class, ~0.5 % of events) branches, again A before B.  -p: neither read is library-less, so the
// site's library-less flag cannot change here; a lane whose flag is already set takes neither read.
template <bool PER_LIB>
__device__ __forceinline__ void hot_pair(const PileupParams &P, uint32_t (*sacc)[TILE], const ChunkInfo &ci, SiteState &S, int tid,
                                         uint32_t da, uint32_t desc_s, uint32_t qual_s, uint32_t seq_s,
                                         int2 pe_a, uint32_t fm_a, uint32_t lib_a, int2 pe_b, uint32_t fm_b, uint32_t lib_b,
                                         uint32_t &pk3, uint32_t &pkmb) {
    const uint32_t db = da + DSZ;
    const int4 q3a = lds128(da + 48u), q3b = lds128(db + 48u);    // qual32,seq32,qoff,n_cigar
    bool cov_a = S.site >= pe_a.x && S.site < pe_a.y;
    bool cov_b = S.site >= pe_b.x && S.site < pe_b.y;
    if (PER_LIB) {
        const bool open = !(S.flags & 1u);
        cov_a = cov_a && open && (lib_a & 0xFFFFu) == S.row;
        cov_b = cov_b && open && (lib_b & 0xFFFFu) == S.row;
    }
    pk3 += ((uint32_t)cov_a + (uint32_t)cov_b) << 24;
    const int qpos_a = cov_a ? S.site - pe_a.x + q3a.z : 0;        // FM_HOT reads have l_qseq >= 1: byte 0 exists
    const int qpos_b = cov_b ? S.site - pe_b.x + q3b.z : 0;
    const uint32_t bq_a = lds_u8(qual_s + (uint32_t)q3a.x + (uint32_t)qpos_a);
    const uint32_t bq_b = lds_u8(qual_s + (uint32_t)q3b.x + (uint32_t)qpos_b);
    const uint32_t byte_a = lds_u8(seq_s + (uint32_t)q3a.y + ((uint32_t)qpos_a >> 1));
    const uint32_t byte_b = lds_u8(seq_s + (uint32_t)q3b.y + ((uint32_t)qpos_b >> 1));
    const bool pass_a = cov_a && !(fm_a & FM_DEAD) && (int)bq_a >= P.min_bq;
    const bool pass_b = cov_b && !(fm_b & FM_DEAD) && (int)bq_b >= P.min_bq;
    S.npass += (uint32_t)pass_a + (uint32_t)pass_b;
    const uint32_t base_a = canonical16((byte_a >> ((~qpos_a & 1) << 2)) & 0xFu);
    const uint32_t base_b = canonical16((byte_b >> ((~qpos_b & 1) << 2)) & 0xFu);
    if (pass_a && S.pbase == NO_BASE) S.pbase = base_a;
    const bool prim_a = pass_a && base_a == S.pbase;
    if (pass_b && S.pbase == NO_BASE) S.pbase = base_b;
    const bool prim_b = pass_b && base_b == S.pbase;

    const int4 q1a = lds128(da + 16u), q1b = lds128(db + 16u);    // mmq,clen,lclip,tpi
    const int4 q2a = lds128(da + 32u), q2b = lds128(db + 32u);    // q2,nmfrac,se,fl
    const int4 q4a = lds128(da + 64u), q4b = lds128(db + 64u);    // rcp_l, rcp_clen, fclen, inc
    const float fl_a = __int_as_float(q2a.w), rcp_la = __int_as_float(q4a.x);
    const float fl_b = __int_as_float(q2b.w), rcp_lb = __int_as_float(q4b.x);
    const float d3_a = div_small((float)abs(qpos_a - q1a.w), fl_a, rcp_la);
    const float d3_b = div_small((float)abs(qpos_b - q1b.w), fl_b, rcp_lb);
    const float f_a = div_small((float)abs(2 * (qpos_a - q1a.z) - q1a.y), __int_as_float(q4a.z), __int_as_float(q4a.y));
    const float f_b = div_small((float)abs(2 * (qpos_b - q1b.z) - q1b.y), __int_as_float(q4b.z), __int_as_float(q4b.y));
    // the Q2 term only counts when the read has a Q2 position, which for most forward reads IS the effective 3' end
    const float q2t_a = q2a.x == q1a.w ? d3_a : div_small((float)abs(qpos_a - q2a.x), fl_a, rcp_la);
    const float q2t_b = q2b.x == q1b.w ? d3_b : div_small((float)abs(qpos_b - q2b.x), fl_b, rcp_lb);
    const bool q2_a = prim_a && (q4a.w & 0x10000), q2_b = prim_b && (q4b.w & 0x10000);

    // integer sums: adding 0 for a dropped event is exact
    pk3 += (prim_a ? (uint32_t)q4a.w : 0u) + (prim_b ? (uint32_t)q4b.w : 0u);
    pkmb += (prim_a ? (fm_a & 0x00FF0000u) + bq_a : 0u) + (prim_b ? (fm_b & 0x00FF0000u) + bq_b : 0u);
    Acc &a = S.acc;
    a.mmqs += (prim_a ? (uint32_t)q1a.x : 0u) + (prim_b ? (uint32_t)q1b.x : 0u);
    a.clip += (prim_a ? (uint32_t)q1a.y : 0u) + (prim_b ? (uint32_t)q1b.y : 0u);
    a.se += (prim_a ? (uint32_t)q2a.z : 0u) + (prim_b ? (uint32_t)q2b.z : 0u);
    // float sums: a dropped event keeps the old value (never "+ 0"), A's add before B's
    a.q2d = q2_a ? __fadd_rn(a.q2d, q2t_a) : a.q2d;
    a.q2d = q2_b ? __fadd_rn(a.q2d, q2t_b) : a.q2d;
    a.d3p = prim_a ? __fadd_rn(a.d3p, d3_a) : a.d3p;
    a.d3p = prim_b ? __fadd_rn(a.d3p, d3_b) : a.d3p;
    a.posd = prim_a ? round_to_f32_precision(__dadd_rn(a.posd, __dsub_rn(1.0, f32_to_f64_nonneg(f_a)))) : a.posd;
    a.posd = prim_b ? round_to_f32_precision(__dadd_rn(a.posd, __dsub_rn(1.0, f32_to_f64_nonneg(f_b)))) : a.posd;
    a.nmf = prim_a ? __fadd_rn(a.nmf, __int_as_float(q2a.y)) : a.nmf;
    a.nmf = prim_b ? __fadd_rn(a.nmf, __int_as_float(q2b.y)) : a.nmf;

    const bool off_a = pass_a && !prim_a, off_b = pass_b && !prim_b;
    if (off_a || off_b) {
        const int32_t read_a = ci.r0 + (int)((da - desc_s) / DSZ);
        if (off_a) off_primary_event<PER_LIB>(P, sacc, ci, S, tid, da, read_a, true, fm_a, qpos_a, bq_a, base_a);
        if (off_b) off_primary_event<PER_LIB>(P, sacc, ci, S, tid, db, read_a + 1, true, fm_b, qpos_b, bq_b, base_b);
    }
}

// The hot loop: one warp walks the chunk's reads in file order; lane = site.
//
// K0 has already classified every read (uniform per iteration): FM_DEAD reads only count as spanning reads; FM_HOT reads
// (one match-type CIGAR op, lengths <= FASTDIV_MAX, no missing tag) take a straight-line path whose event is the site's
// primary base class in ~99 % of the cases; everything else takes the general path.  Two consecutive FM_HOT reads of a
// staged chunk take hot_pair instead.  The primary class's small integer sums and the coverage count are kept PACKED for
// the duration of a chunk (<= STAGE_READS reads: four 8-bit counters in one word, two 16-bit sums in another) and flushed
// into the full-width accumulators at the end of the chunk.
template <bool PER_LIB, bool STAGED>
__device__ __forceinline__ void process_chunk(const PileupParams &P, const StageBuf &sb, uint32_t (*sacc)[TILE], uint32_t (*warn)[TILE],
                                              const ChunkInfo &ci, SiteState &S, int tid) {
    const uint32_t desc_s = smem_u32(sb.desc);                // descriptor j of the chunk sits at desc_s + 80 j
    uint32_t da = desc_s;
    const uint32_t qual_s = smem_u32(sb.qual) - ci.qbase32;   // staged bytes are addressed with the reads' low-32 pool offsets
    const uint32_t seq_s = smem_u32(sb.seq) - ci.sbase32;
    const int32_t wfirst = S.wfirst;
    {   // vectorised skip of the leading reads that end before this warp's first site (32 reads per ballot):
        // keeps the 8 warps of a tile in step — the last warp would otherwise walk ~45 dead reads one by one
        const int n_in = ci.r1 - ci.r0, lane = tid & 31;
        int start = 0;
        for (; start < n_in; start += 32) {
            const int j = start + lane;
            const int endj = j < n_in ? sb.desc[j * 5].y : 0x7fffffff;
            const unsigned m = __ballot_sync(0xffffffffu, endj > wfirst);
            if (m) { start += __ffs(m) - 1; break; }
        }
        if (start >= n_in) return;
        da += (uint32_t)start * (uint32_t)sizeof(ReadDesc);
    }
    uint32_t pk3 = 0u, pkmb = 0u;                                 // count | plus << 8 | nq2 << 16 | ncover << 24 ;  baseq | mapq << 16
    // no loop bound: the producer wrote a sentinel descriptor (pos = INT_MAX, fm = 0) behind the chunk's last read
    for (;; da += DSZ) {
        const int2 pe = lds64(da);                                // pos, end
        const int2 fl2 = lds64(da + 8u);                          // fm, lib_nc
        // the next read's: when `pe` is the sentinel this is the spare record behind it in desc[], loaded and never used
        const int2 pe_b = lds64(da + DSZ), fl_b = lds64(da + DSZ + 8u);
        if (pe.x - wfirst > 31) { if (pe.x != 0x7fffffff) S.warp_done = true; break; }   // reads are position-sorted within a region; INT_MAX = end of chunk
        if (STAGED) {
            // Two FM_HOT reads (A = this one, B = the next) in one predicated body; the test is uniform across the warp.  -p: a
            // read without a library (which stops the site's accumulation) is never part of a pair.  B is never the sentinel.
            bool pair = ((uint32_t)fl2.x & (uint32_t)fl_b.x & FM_HOT) != 0u;
            if (PER_LIB) pair = pair && ((uint32_t)fl2.y & 0xFFFFu) != LIB_NONE && ((uint32_t)fl_b.y & 0xFFFFu) != LIB_NONE;
            if (pair) {
                const bool b_in = pe_b.x - wfirst <= 31;          // B beyond the warp's window: it covers no lane and ends the walk
                hot_pair<PER_LIB>(P, sacc, ci, S, tid, da, desc_s, qual_s, seq_s, pe, (uint32_t)fl2.x, (uint32_t)fl2.y,
                                  b_in ? pe_b : make_int2(0x7fffffff, 0), (uint32_t)fl_b.x, (uint32_t)fl_b.y, pk3, pkmb);
                if (!b_in) { S.warp_done = true; break; }
                da += DSZ;
                continue;
            }
        }
        if (pe.y <= wfirst) continue;
        const bool cover = S.site >= pe.x && S.site < pe.y;
        if (PER_LIB) {
            const uint32_t lib = (uint32_t)fl2.y & 0xFFFFu;
            if (lib == LIB_NONE) { if (cover) S.flags |= 1u; continue; }
            if (lib != S.row) continue;
            // -p: pileup_func returns at the first read without a library (R:...:281-284); nothing after
            // it in pileup (= file) order is processed or warned about at this site
            if (S.flags & 1u) continue;
        }
        if (!cover) continue;
        pk3 += 1u << 24;                                          // ncover
        const uint32_t fm = (uint32_t)fl2.x;
        const int4 q3 = lds128(da + 48u);                        // qual32,seq32,cig,n_cigar
        int qpos, indel = 0;
        uint32_t bq, base;
        if (fm & FM_HOT) {
            // ---- straight-line path: filters decided by K0, single match op, exact reciprocal divisions ----
            if (fm & FM_DEAD) continue;
            qpos = S.site - pe.x + q3.z;
            if (STAGED) bq = lds_u8(qual_s + (uint32_t)q3.x + (uint32_t)qpos);
            else bq = P.qual[P.qual_off[ci.r0 + (int)((da - desc_s) / (uint32_t)sizeof(ReadDesc))] + (uint32_t)qpos];
            if ((int)bq < P.min_bq) continue;
            S.npass++;
            uint32_t byte;
            if (STAGED) byte = lds_u8(seq_s + (uint32_t)q3.y + ((uint32_t)qpos >> 1));
            else byte = P.seq[P.seq_off[ci.r0 + (int)((da - desc_s) / (uint32_t)sizeof(ReadDesc))] + ((uint32_t)qpos >> 1)];
            base = canonical16((byte >> ((~qpos & 1) << 2)) & 0xFu);
            if (S.pbase == NO_BASE) S.pbase = base;
            if (base == S.pbase) {
                const int4 q1 = lds128(da + 16u);                // mmq,clen,lclip,tpi
                const int4 q2 = lds128(da + 32u);                // q2,nmfrac,se,fl
                const int4 q4 = lds128(da + 64u);                // rcp_l, rcp_clen, fclen, inc
                const float fl = __int_as_float(q2.w), rcp_l = __int_as_float(q4.x);
                const float d3 = div_small((float)abs(qpos - q1.w), fl, rcp_l);
                const float f = div_small((float)abs(2 * (qpos - q1.z) - q1.y), __int_as_float(q4.z), __int_as_float(q4.y));
                Acc &a = S.acc;
                pk3 += (uint32_t)q4.w;
                pkmb += (fm & 0x00FF0000u) + bq;
                a.mmqs += (uint32_t)q1.x; a.clip += (uint32_t)q1.y; a.se += (uint32_t)q2.z;
                if (q4.w & 0x10000) {                            // the read has a Q2 position (usually == the effective 3' end, R:...:229-238)
                    const float q2t = q2.x == q1.w ? d3 : div_small((float)abs(qpos - q2.x), fl, rcp_l);
                    a.q2d = __fadd_rn(a.q2d, q2t);
                }
                a.d3p = __fadd_rn(a.d3p, d3);
                a.posd = round_to_f32_precision(__dadd_rn(a.posd, __dsub_rn(1.0, f32_to_f64_nonneg(f))));
                a.nmf = __fadd_rn(a.nmf, __int_as_float(q2.y));
                continue;
            }
        } else {
            // ---- general path ----
            if (fm & FM_SIMPLE) qpos = S.site - pe.x + q3.z;
            else {
                // staged ops are indexed with the reads' pool op indices; their address derives from desc_s, which the loop
                // keeps anyway (not from the ring slot's index, which would be reloaded from local memory)
                const uint32_t *cig_base = (ci.flags & 16u)
                    ? static_cast<const uint32_t *>(__cvta_shared_to_generic(desc_s + (uint32_t)offsetof(StageBuf, cigar))) - ci.cbase32 : P.cigar;
                const int3 rr = resolve_general(cig_base + (uint32_t)q3.z, (uint32_t)q3.w, pe.x, S.site);
                if (rr.z) continue;                              // is_del
                qpos = rr.x; indel = rr.y;
            }
            if (fm & FM_DEAD) continue;                          // mapq / flag filter (R:...:288-310)
            if (STAGED) bq = lds_u8(qual_s + (uint32_t)q3.x + (uint32_t)qpos);
            else bq = P.qual[P.qual_off[ci.r0 + (int)((da - desc_s) / (uint32_t)sizeof(ReadDesc))] + (uint32_t)qpos];
            if ((int)bq < P.min_bq) continue;
            S.npass++;
            const bool warns = (fm & (FM_NM_ABSENT | FM_SM_MISSING)) != 0;   // a tag the reference warns about is missing
            if (indel != 0) {
                const int32_t r = ci.r0 + (int)((da - desc_s) / (uint32_t)sizeof(ReadDesc));
                S.sec_head = rare_event(rare_ctx(P), S.sec_head, slot_index<PER_LIB>(P, ci, S), indel > 0 ? KIND_INS : KIND_DEL, indel > 0 ? indel : -indel, r, qpos, bq, true);
                if (warns) { warn[0][tid] += (fm >> 25) & 1u; warn[1][tid] += (fm >> 26) & 1u; }
                if (indel > 0 && P.insertion_centric) continue;
            }
            if (warns) { warn[0][tid] += (fm >> 25) & 1u; warn[1][tid] += (fm >> 26) & 1u; }
            uint32_t byte;
            if (STAGED) byte = lds_u8(seq_s + (uint32_t)q3.y + ((uint32_t)qpos >> 1));
            else byte = P.seq[P.seq_off[ci.r0 + (int)((da - desc_s) / (uint32_t)sizeof(ReadDesc))] + ((uint32_t)qpos >> 1)];
            base = canonical16((byte >> ((~qpos & 1) << 2)) & 0xFu);
            if (S.pbase == NO_BASE) S.pbase = base;
        }
        // ---- an event that is not (hot, primary): full-width accumulation ----
        if (base != S.pbase) {
            off_primary_event<PER_LIB>(P, sacc, ci, S, tid, da, ci.r0 + (int)((da - desc_s) / DSZ), (fm & FM_FASTDIV) != 0, fm, qpos, bq, base);
            continue;
        }
        const int4 q1 = lds128(da + 16u);                        // mmq,clen,lclip,tpi
        const int4 q2 = lds128(da + 32u);                        // q2,nmfrac,se,fl
        const int4 q4 = lds128(da + 64u);                        // rcp_l, rcp_clen, fclen
        const Terms t = event_terms((fm & FM_FASTDIV) != 0, qpos, q2.x, q1.w, q1.z, q1.y, __int_as_float(q2.w), __int_as_float(q4.z),
                                    __int_as_float(q4.x), __int_as_float(q4.y));
        Acc &a = S.acc;
        pk3 += (uint32_t)q4.w;                                   // count, plus, nq2: the packed counters, as on the hot path
        pkmb += (fm & 0x00FF0000u) + bq;
        a.mmqs += (uint32_t)q1.x;
        if (q2.x > -1) a.q2d = __fadd_rn(a.q2d, t.q2term);
        a.d3p = __fadd_rn(a.d3p, t.d3pterm);
        a.clip += (uint32_t)q1.y;
        a.posd = round_to_f32_precision(__dadd_rn(a.posd, t.posterm));
        a.se += (uint32_t)q2.z;
        a.nmf = __fadd_rn(a.nmf, __int_as_float(q2.y));
    }
    // flush the chunk's packed counters of the primary class
    S.acc.count += pk3 & 0xFFu; S.acc.plus += (pk3 >> 8) & 0xFFu; S.acc.nq2 += (pk3 >> 16) & 0xFFu; S.ncover += pk3 >> 24;
    S.acc.baseq += pkmb & 0xFFFFu; S.acc.mapq += pkmb >> 16;
}

// Packs one site's header + primary accumulators into the 8-word narrow record, or escapes it to a full-width pool record
// (brc_device.cuh).  `st` = the 13 accumulators in print order.  Returns false when the pool overflowed (host retries).
__device__ __forceinline__ void emit_packed(const ResultsDev &R, int64_t idx, uint32_t ncover, uint32_t npass, uint32_t flags, uint32_t pbase,
                                            int32_t sec_head, const uint32_t (&st)[N_STATS]) {
    const uint32_t pcode = pbase < 6u ? pbase : PB_NONE;
    const bool narrow = ncover <= 255u && st[1] <= 0xFFFFu && st[2] <= 0xFFFFu && st[3] <= 0xFFFFu && st[11] <= 0xFFFFu && st[8] <= 0xFFFFu;
    uint32_t w[N_WORDS];
    if (narrow) {
        w[0] = ncover | (npass << 8) | (st[0] << 16) | (st[4] << 24);
        w[1] = pcode | ((flags & 1u) << 3) | (sec_head >= 0 ? 16u : 0u) | (st[9] << 8) | (st[1] << 16);
        w[2] = st[2] | (st[3] << 16);
        w[3] = st[11] | (st[8] << 16);
        w[4] = st[6]; w[5] = st[7]; w[6] = st[10]; w[7] = st[12];
    } else {
        const int32_t j = atomicAdd(R.sec_count, 1);
        if ((int64_t)j < R.sec_cap) {
            SecRec &r = R.sec[j];
            r.slot = (uint32_t)idx; r.next = sec_head; r.kind_len = (KIND_WIDE + pcode) | (ncover << 8); r.read = (int32_t)flags; r.qpos = (int32_t)npass;
#pragma unroll
            for (int k = 0; k < N_STATS; ++k) r.stats[k] = st[k];
        }
        w[0] = 0u; w[1] = PB_ESCAPE | ((flags & 1u) << 3) | 16u; w[2] = w[3] = w[4] = w[5] = w[6] = w[7] = 0u;
    }
    const int64_t stride = (int64_t)R.n_rows * R.n_slots;
    uint32_t *dst = R.words + idx;
#pragma unroll
    for (int k = 0; k < N_WORDS; ++k) dst[k * stride] = w[k];     // each a fully-coalesced 128-byte line per warp
}

// last chunk of a tile: write the site's packed record (coalesced SoA stores)
template <bool PER_LIB>
__device__ __forceinline__ void site_emit(const PileupParams &P, uint32_t (*sacc)[TILE], const ChunkInfo &ci, SiteState &S, int tid) {
    if (S.site < 0) return;
    const ResultsDev &R = P.res;
    int32_t sec_head = S.sec_head;
    const int64_t idx = (PER_LIB ? (int64_t)S.row * R.n_slots : 0) + ci.slot0 + (S.site - ci.pos0);
    if (S.sbase != NO_BASE) {   // move the second base class into the record pool
        const int32_t j = atomicAdd(R.sec_count, 1);
        if ((int64_t)j < R.sec_cap) {
            SecRec &r = R.sec[j];
            r.slot = (uint32_t)idx; r.next = sec_head; r.kind_len = S.sbase; r.read = 0; r.qpos = 0;
#pragma unroll
            for (int k = 0; k < N_STATS; ++k) r.stats[k] = sacc[k][tid];
            sec_head = j;
        }
    }
    const Acc &a = S.acc;
    const uint32_t st[N_STATS] = {a.count, a.mapq, a.baseq, a.se, a.plus, a.count - a.plus, __float_as_uint(__double2float_rn(a.posd)),
                                  __float_as_uint(a.nmf), a.mmqs, a.nq2, __float_as_uint(a.q2d), a.clip, __float_as_uint(a.d3p)};
    emit_packed(R, idx, S.ncover, S.npass, PER_LIB ? S.flags : 0u, S.pbase, sec_head, st);
}

template <bool PER_LIB>
__global__ void __launch_bounds__(K1_THREADS, BRC_K1_CTAS_PER_SM) pileup_kernel(PileupParams P) {
    extern __shared__ __align__(128) uint8_t smem_raw[];
    PileupSmem &sm = *reinterpret_cast<PileupSmem *>(smem_raw);
    const int tid = threadIdx.x;
    const int warp = tid >> 5, lane = tid & 31;
    const int64_t n_work = P.tile_count * (int64_t)P.res.n_rows;

    if (tid == 0) {
        for (int s = 0; s < NSTAGE; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], N_CONSUMER_WARPS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp == N_CONSUMER_WARPS) {
        // =========================== PRODUCER ===========================
        if (lane != 0) return;
        uint32_t item = 0;
        // Tiles are handed out by an atomic dispenser (zeroed by init_tiles_kernel), not by a fixed stride: SMs that also host
        // another stream's CTAs (the NCCL send/recv kernels of the ordered-emit gather, a neighbouring window's K0) run their tiles
        // slower, and with a fixed stride the slowest SM set the launch time (r02m8: 2.8 -> 4.2 ms per window at 4 GPUs).  The
        // producer runs up to NSTAGE chunks ahead of the consumers, which hides the atomic's round trip.
        int64_t w_static = blockIdx.x;
        for (;; w_static += gridDim.x) {
            const int64_t w = P.work_counter ? (int64_t)atomicAdd(P.work_counter, 1ull) : w_static;
            const bool done = w >= n_work;
            int32_t lo = 0, hi = 0; TileInfo ti{0, 0, 0}; uint32_t row = 0;
            bool narrow = false;
            if (!done) {
                const int64_t tile = P.tile_begin + w % P.tile_count; row = (uint32_t)(w / P.tile_count);
                ti = P.tiles[tile]; lo = P.tile_lo[tile]; hi = P.tile_hi[tile];
                if (lo >= hi) { lo = 0; hi = 0; }
                // -p on a tile of <= 32 sites (site lists, deep panels): the 8 consumer warps take 8 LIBRARIES of the
                // same sites instead of 8 site ranges, so one staged chunk serves 8 rows
                narrow = PER_LIB && ti.n <= 32;
                // deep narrow tiles (a single site under thousands of reads) belong to deep_site_kernel
                if (P.n_deep > 0 && deep_shape_ok(ti.n, P.res.n_rows) && hi - lo >= P.deep_min_reads) continue;
                if (narrow && (row % N_CONSUMER_WARPS) != 0) continue;
            }
            int32_t r0 = lo;
            bool first = true;
            do {
                const int s = item % NSTAGE; const uint32_t ph = (item / NSTAGE) & 1u;
#ifdef BRC_K1_PROFILE
                const long long tp0 = clock64();
#endif
                mbar_wait_relaxed(&sm.empty[s], ph ^ 1u);  // consumers released this slot
#ifdef BRC_K1_PROFILE
                const long long tp1 = clock64();
#endif
                ChunkInfo ci{};
                ci.work = done ? -1 : (int32_t)w;
                ci.pos0 = ti.pos0; ci.n = ti.n; ci.slot0 = ti.slot0; ci.row = row;
                uint32_t bytes = 0;
                int32_t r1 = r0;
                if (r0 < hi) {
                    r1 = min(r0 + STAGE_READS, hi);
                    uint64_t qa, qb, sa, sb; bool staged;
                    for (;;) {   // as many reads as fit the stage: shrink proportionally to the overshoot
                        qa = P.qual_off[r0] & ~15ull; qb = (P.qual_off[r1] + 15ull) & ~15ull;
                        sa = P.seq_off[r0] & ~15ull;  sb = (P.seq_off[r1] + 15ull) & ~15ull;
                        staged = (qb - qa) <= (uint64_t)STAGE_QUAL && (sb - sa) <= (uint64_t)STAGE_SEQ;
                        if (staged || r1 - r0 == 1) break;
                        const double fq = (double)(STAGE_QUAL - 32) / (double)(qb - qa), fs = (double)(STAGE_SEQ - 32) / (double)(sb - sa);
                        const int32_t n2 = (int32_t)((double)(r1 - r0) * (fq < fs ? fq : fs));
                        r1 = r0 + max(1, min(n2, r1 - r0 - 1));
                    }
                    const uint32_t db = (uint32_t)(r1 - r0) * (uint32_t)sizeof(ReadDesc);
                    const uint32_t qbytes = staged ? (uint32_t)(qb - qa) : 0u, sbytes = staged ? (uint32_t)(sb - sa) : 0u;
                    // the chunk's CIGAR ops (contiguous in the pool), 16-byte aligned window of u32 ops
                    const uint64_t ca = P.cigar_off[r0] & ~3ull, cb = (P.cigar_off[r1] + 3ull) & ~3ull;
                    const uint32_t cbytes = (cb - ca) <= (uint64_t)STAGE_CIGAR ? (uint32_t)(cb - ca) * 4u : 0u;
                    bytes = db + qbytes + sbytes + cbytes;
                    ci.qbase32 = (uint32_t)qa; ci.sbase32 = (uint32_t)sa; ci.cbase32 = (uint32_t)ca;
                    ci.flags = (staged ? 1u : 0u) | (cbytes ? 16u : 0u);
                    ci.r0 = r0; ci.r1 = r1;
                    ci.flags |= (first ? 2u : 0u) | (r1 >= hi ? 4u : 0u) | (narrow ? 8u : 0u);
                    sm.info[s] = ci;
                    sm.st[s].desc[(r1 - r0) * 5] = make_int4(0x7fffffff, 0x7fffffff, 0, 0);   // sentinel (pos, end): released to the consumers by the arrive below
                    mbar_expect_tx(&sm.full[s], bytes);
                    tma_bulk_g2s(sm.st[s].desc, P.desc + r0, db, &sm.full[s]);
                    if (qbytes) tma_bulk_g2s(sm.st[s].qual, P.qual + qa, qbytes, &sm.full[s]);
                    if (sbytes) tma_bulk_g2s(sm.st[s].seq, P.seq + sa, sbytes, &sm.full[s]);
                    if (cbytes) tma_bulk_g2s(sm.st[s].cigar, P.cigar + ca, cbytes, &sm.full[s]);
                } else {   // tile without reads, or the terminator
                    ci.r0 = ci.r1 = 0; ci.flags = 2u | 4u | (narrow ? 8u : 0u);
                    sm.info[s] = ci;
                    mbar_arrive(&sm.full[s]);
                }
#ifdef BRC_K1_PROFILE
                atomicAdd(&g_k1prof[2], (unsigned long long)(tp1 - tp0)); atomicAdd(&g_k1prof[3], (unsigned long long)(clock64() - tp1)); atomicAdd(&g_k1prof[4], 1ull);
#endif
                item++; first = false; r0 = r1;
            } while (r0 < hi);
            if (done) break;
        }
        return;
    }

    // =========================== CONSUMERS ===========================
    SiteState S0;
    sm.warn[0][tid] = 0u; sm.warn[1][tid] = 0u;   // only this thread touches its two slots
    for (uint32_t item = 0;; ++item) {
        const int s = item % NSTAGE; const uint32_t ph = (item / NSTAGE) & 1u;
#ifdef BRC_K1_PROFILE
        const long long tc0 = clock64();
#endif
        mbar_wait_hint<200>(&sm.full[s], ph);        // ncu r02a: this poll loop is 8 % of the issued instructions but 2 % of the stall samples
#ifdef BRC_K1_PROFILE
        const long long tc1 = clock64();
#endif
        const ChunkInfo &ci = sm.info[s];   // stays valid until this warp arrives on empty[s]
        if (ci.work < 0) break;
        if (ci.flags & 2u) site_reset<PER_LIB>(S0, ci, tid, P.res.n_rows);   // first chunk of a tile
        if (!S0.warp_done) {
            if (ci.flags & 1u) process_chunk<PER_LIB, true>(P, sm.st[s], sm.sacc, sm.warn, ci, S0, tid);
            else process_chunk<PER_LIB, false>(P, sm.st[s], sm.sacc, sm.warn, ci, S0, tid);
        }
        if (ci.flags & 4u) site_emit<PER_LIB>(P, sm.sacc, ci, S0, tid);   // last chunk of the tile
        __syncwarp();
#ifdef BRC_K1_PROFILE
        if (lane == 0) { atomicAdd(&g_k1prof[0], (unsigned long long)(tc1 - tc0)); atomicAdd(&g_k1prof[1], (unsigned long long)(clock64() - tc1)); }
#endif
        if (lane == 0) mbar_arrive(&sm.empty[s]);   // this warp is done with the slot
    }
    // warning counters: warp-reduce then one atomic per warp
    uint32_t warn_nm = sm.warn[0][tid], warn_sm = sm.warn[1][tid];
    for (int o = 16; o; o >>= 1) { warn_sm += __shfl_xor_sync(0xffffffffu, warn_sm, o); warn_nm += __shfl_xor_sync(0xffffffffu, warn_nm, o); }
    if (lane == 0) {
        if (warn_sm) atomicAdd(P.res.warn + 0, (unsigned long long)warn_sm);
        if (warn_nm) atomicAdd(P.res.warn + 1, (unsigned long long)warn_nm);
    }
}

static std::atomic<int> g_sm_count[64];
#ifdef BRC_K1_PROFILE
extern "C" __attribute__((visibility("default"))) void brc_debug_k1prof(unsigned long long *out, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out, g_k1prof, sizeof(g_k1prof));
    if (reset) { unsigned long long z[8] = {0}; cudaMemcpyToSymbol(g_k1prof, z, sizeof(z)); }
}
#endif
cudaError_t launch_pileup(const PileupParams &p, cudaStream_t s) {
    if (p.tile_count <= 0) return cudaSuccess;
    int dev = 0; cudaGetDevice(&dev);
    int sms = dev < 64 ? g_sm_count[dev].load(std::memory_order_acquire) : 0;
    if (sms == 0) {
        std::lock_guard<std::mutex> lk(g_init_mu);
        cudaError_t e1 = cudaFuncSetAttribute(pileup_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PileupSmem));
        cudaError_t e2 = cudaFuncSetAttribute(pileup_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(PileupSmem));
        if (e1 != cudaSuccess) return e1;
        if (e2 != cudaSuccess) return e2;
        if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) { cudaGetLastError(); sms = 132; }
        if (dev < 64) g_sm_count[dev].store(sms, std::memory_order_release);
    }
    const int64_t n_work = p.tile_count * (int64_t)p.res.n_rows;
    // persistent CTAs, 3 per SM.  A multi-GPU caller whose NCCL send/recv kernels must run NEXT to this kernel (the ordered-emit
    // gather, bam_readcount_b200/stream.py) leaves a few CTA slots free with BRC_K1_RESERVE_CTAS: a grid that fills every slot
    // makes the collective wait for the tail of each launch (r02m2: 2-GPU step 483 ms against 348 ms of compute)
    static const int reserve = std::getenv("BRC_K1_RESERVE_CTAS") ? std::max(0, std::atoi(std::getenv("BRC_K1_RESERVE_CTAS"))) : 0;
    const int64_t slots = std::max<int64_t>((int64_t)sms * BRC_K1_CTAS_PER_SM - reserve, sms);
    const unsigned grid = (unsigned)std::min<int64_t>(n_work, slots);
    const size_t smem = sizeof(PileupSmem);
    if (p.per_lib) pileup_kernel<true><<<grid, K1_THREADS, smem, s>>>(p);
    else pileup_kernel<false><<<grid, K1_THREADS, smem, s>>>(p);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// K1-deep: one CTA per DEEP tile — a tile of <= DEEP_MAX_SITES sites (a site-list line: the site and its left neighbour)
// whose read window holds thousands of reads (amplicon / panel depth).  pileup_kernel would walk those reads one by one in
// a single lane per (site, library); here the per-event work is done read-parallel and only the accumulation is ordered:
//   phase 1  thread = read (256 per block, file order): coverage, resolve_cigar2, filters, base class, the 13 terms of
//            BasicStat::process_read; passing events are written to shared memory, stably partitioned by (site, library)
//            (warp match + per-warp counts), so each group's events stay in file order;
//   phase 2  thread = (site, library, statistic): walks its group's events in order and adds its one term to a register —
//            the same sequence of float32 / double-rounded additions as the reference, so results stay bit-identical.
//            The first passing base class is the primary allele (registers -> pstats).  The other base classes accumulate
//            the same way in shared-memory cells (so a site whose first read carries a sequencing error costs the same),
//            and become pool records at the end; indel alleles are handed, in order, to rare_event by the group's
//            statistic-0 thread.
// Integer statistics go through the same ordered loop: it keeps one code path and costs one predicated add.
// ---------------------------------------------------------------------------------------------
#ifdef BRC_DEEP_PROFILE
__device__ unsigned long long g_deepprof[8];
#endif
constexpr int DEEP_EVENTS = DEEP_THREADS * DEEP_MAX_SITES;
constexpr int DEEP_GROUPS = 17;                              // largest n_sites * n_rows deep_shape_ok admits
constexpr int DEEP_WARPS = DEEP_THREADS / 32;
constexpr int DEEP_ICACHE = 8;
constexpr int DEEP_PAD = 136;                                // bank-skew slack of the event arrays: 0 + 1 + ... + 16 slots
struct __align__(16) DeepStage {                             // one block of reads, fetched with cp.async a block ahead
    ReadDesc desc[DEEP_THREADS];
    uint64_t qoff[DEEP_THREADS], soff[DEEP_THREADS];
};
struct __align__(16) DeepSmem {
    DeepStage stage[2];
    uint32_t term[N_STATS][DEEP_EVENTS + DEEP_PAD + 1];   // odd row length: the owners of a group read one column of different rows -> different banks
    uint32_t meta[DEEP_EVENTS + DEEP_PAD];                // base class [0:3) | bit3 has indel | bit4 has base part | bq << 8
    int32_t eread[DEEP_EVENTS + DEEP_PAD];                // read index
    int32_t eqpos[DEEP_EVENTS + DEEP_PAD];
    int32_t eindel[DEEP_EVENTS + DEEP_PAD];
    uint32_t wcnt[DEEP_WARPS][DEEP_GROUPS + 1];   // phase 1: events of group g in warp w -> exclusive offset inside the group
    uint32_t gcnt[DEEP_GROUPS + 1], gbase[DEEP_GROUPS + 1];
    uint32_t ncover[DEEP_GROUPS + 1], npass[DEEP_GROUPS + 1];
    int32_t first_libless[DEEP_MAX_SITES];        // -p: first covering read without a library (nothing after it counts)
    int32_t recj[DEEP_GROUPS + 1];                // emit: pool record of the class being written
    uint32_t ikey[DEEP_GROUPS + 1][DEEP_ICACHE];  // indel alleles of a group already in the pool: packed (kind, length, inserted bases)
    int32_t irec[DEEP_GROUPS + 1][DEEP_ICACHE];   //   -> pool record
    uint32_t icount[DEEP_GROUPS + 1];
    unsigned long long other[6][DEEP_THREADS];    // accumulators of the non-primary base classes, one cell per owner thread
};

__device__ __forceinline__ void cp_async16(void *dst, const void *src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8(void *dst, const void *src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

// one indel event of a group (called by the group's read_count owner, in file order)
__device__ __forceinline__ void deep_indel_event(const PileupParams &P, DeepSmem &sm, int og, uint32_t slot, int32_t &sec_head, int indel, int32_t read, int qpos, uint32_t bq) {
    const int kind = indel > 0 ? KIND_INS : KIND_DEL, len = indel > 0 ? indel : -indel;
    const bool cacheable = len <= 127 && (kind == KIND_DEL || len <= 8);
    uint32_t key = 0u;
    if (cacheable) {
        key = (kind == KIND_INS ? 0x80000000u : 0u) | ((uint32_t)len << 24);
        if (kind == KIND_INS) {
            const uint64_t oa = P.seq_off[read];
            for (int k = 1; k <= len; ++k) key |= canonical16(seq_nib(P.seq, oa, qpos + k)) << (3 * (k - 1));   // the allele string (R:...:324-330)
        }
    }
    int32_t j = -1;
    const uint32_t nc = sm.icount[og];
    if (cacheable) for (uint32_t e = 0; e < nc; ++e) if (sm.ikey[og][e] == key) j = sm.irec[og][e];
    if (j < 0) {
        j = rare_find_or_append(rare_ctx(P), sec_head, slot, kind, len, read, qpos);
        if (cacheable && (int64_t)j < P.res.sec_cap && nc < (uint32_t)DEEP_ICACHE) { sm.ikey[og][nc] = key; sm.irec[og][nc] = j; sm.icount[og] = nc + 1u; }
    }
    if ((int64_t)j < P.res.sec_cap) sec_accumulate(P.desc, P.res.sec[j], read, qpos, bq, true);
}

// this thread's read of the block starting at `blk` -> its own slots of stage st (no other thread touches them)
__device__ __forceinline__ void deep_fetch(const PileupParams &P, DeepStage &st, int32_t r, int32_t hi, int tid) {
    if (r < hi) {
        const char *src = reinterpret_cast<const char *>(P.desc + r);
        char *dst = reinterpret_cast<char *>(&st.desc[tid]);
#pragma unroll
        for (int k = 0; k < (int)sizeof(ReadDesc); k += 16) cp_async16(dst + k, src + k);
        cp_async8(&st.qoff[tid], P.qual_off + r);
        cp_async8(&st.soff[tid], P.seq_off + r);
    }
    cp_async_commit();
}

template <bool PER_LIB>
__global__ void __launch_bounds__(DEEP_THREADS, 2) deep_site_kernel(PileupParams P) {
    extern __shared__ __align__(128) uint8_t deep_smem_raw[];
    DeepSmem &sm = *reinterpret_cast<DeepSmem *>(deep_smem_raw);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int32_t tile = P.deep_tiles[blockIdx.x];
    if (tile < P.tile_begin || tile >= P.tile_begin + P.tile_count) return;
    const TileInfo ti = P.tiles[tile];
    int32_t lo = P.tile_lo[tile], hi = P.tile_hi[tile];
    if (lo >= hi) { lo = 0; hi = 0; }
    // this CTA's library rows [row0, row0 + n_rows): n_rows <= DEEP_ROWS, all of them in all-library mode (one row)
    const int row0 = (int)blockIdx.y * DEEP_ROWS;
    const int n_rows = min(DEEP_ROWS, P.res.n_rows - row0);
    if (!deep_shape_ok(ti.n, P.res.n_rows) || hi - lo < P.deep_min_reads) return;   // pileup_kernel computes it (same predicate)
    const int G = ti.n * n_rows;

    deep_fetch(P, sm.stage[0], lo + tid, hi, tid);
    for (int i = tid; i <= DEEP_GROUPS; i += DEEP_THREADS) { sm.ncover[i] = 0u; sm.npass[i] = 0u; sm.icount[i] = 0u; }
    if (tid < DEEP_MAX_SITES) sm.first_libless[tid] = 0x7fffffff;
#pragma unroll
    for (int c = 0; c < 6; ++c) sm.other[c][tid] = 0ull;

    // phase-2 owner state: thread -> (statistic oj, group og = site * n_rows + row); kinds start on warp boundaries
    bool owner = false; int og = 0, oj = 0, kind = 0;   // kind 0 integer, 1 float, 2 double-rounded
    {
        const int fb = deep_flt_base(G), db = deep_dbl_base(G);
        if (tid < 9 * G) { const int k = tid / G; og = tid - k * G; oj = k < 6 ? k : (k == 6 ? 8 : (k == 7 ? 9 : 11)); kind = 0; owner = true; }
        else if (tid >= fb && tid < fb + 3 * G) { const int k = (tid - fb) / G; og = tid - fb - k * G; oj = k == 0 ? 7 : (k == 1 ? 10 : 12); kind = 1; owner = true; }
        else if (tid >= db && tid < db + G) { og = tid - db; oj = 6; kind = 2; owner = true; }
    }
    uint32_t acc_u = 0u; float acc_f = 0.0f; double acc_d = 0.0;
    uint32_t pbase = NO_BASE; int32_t sec_head = -1;
    const uint32_t oslot = owner ? (uint32_t)((int64_t)(row0 + og % n_rows) * P.res.n_slots + ti.slot0 + og / n_rows) : 0u;   // row * n_slots + slot of the owner's group
    uint32_t warn_nm = 0u, warn_sm = 0u;
#ifdef BRC_DEEP_PROFILE
    long long prof[6] = {0, 0, 0, 0, 0, 0};
#endif
    __syncthreads();

    int stg = 0;
    for (int32_t blk = lo; blk < hi; blk += DEEP_THREADS, stg ^= 1) {
        const int32_t r = blk + tid;
        const bool valid = r < hi;
#ifdef BRC_DEEP_PROFILE
        const long long tq0 = clock64();
#endif
        cp_async_wait_all();                                       // this thread's slots of stage[stg] have landed
        ReadDesc d; uint64_t qoff = 0, soff = 0;
        d.pos = 0; d.end = 0; d.fm = 0u; d.lib_nc = 0u;
        if (valid) { d = sm.stage[stg].desc[tid]; qoff = sm.stage[stg].qoff[tid]; soff = sm.stage[stg].soff[tid]; }
        deep_fetch(P, sm.stage[stg ^ 1], r + DEEP_THREADS, hi, tid);   // next block: in flight during this whole iteration
        // ---- phase 1a: coverage; -p: the first covering read without a library ----
        const uint32_t fm = d.fm, lib = d.lib_nc & 0xFFFFu;
        bool cover[DEEP_MAX_SITES];
#pragma unroll
        for (int sg = 0; sg < DEEP_MAX_SITES; ++sg) {
            const int32_t site = ti.pos0 + sg;
            cover[sg] = valid && sg < ti.n && site >= d.pos && site < d.end;
            if (PER_LIB && cover[sg] && lib == LIB_NONE) atomicMin(&sm.first_libless[sg], r);
        }
        for (int i = tid; i < DEEP_WARPS * (DEEP_GROUPS + 1); i += DEEP_THREADS) (&sm.wcnt[0][0])[i] = 0u;
        __syncthreads();
#ifdef BRC_DEEP_PROFILE
        const long long tq1 = clock64();
#endif
        // ---- phase 1b: the events of this read.  Stage i: coverage / library / resolve_cigar2 for both sites ----
        bool has[DEEP_MAX_SITES]; int grp[DEEP_MAX_SITES], eq[DEEP_MAX_SITES], ei[DEEP_MAX_SITES], gcov[DEEP_MAX_SITES];
        const uint32_t mapq = (fm >> 16) & 0xFFu;
#pragma unroll
        for (int sg = 0; sg < DEEP_MAX_SITES; ++sg) {
            has[sg] = false; grp[sg] = 0; eq[sg] = 0; ei[sg] = 0; gcov[sg] = -1;
            if (!cover[sg]) continue;
            uint32_t row = 0u;
            if (PER_LIB) {
                if (lib == LIB_NONE || lib < (uint32_t)row0 || lib >= (uint32_t)(row0 + n_rows)) continue;   // another CTA's library
                if (r > sm.first_libless[sg]) continue;          // pileup_func returned early at this site (R:...:281-284)
                row = lib - (uint32_t)row0;
            }
            grp[sg] = sg * n_rows + (int)row;
            gcov[sg] = grp[sg];                                  // counts as a covering read of (site, row)
            const int32_t site = ti.pos0 + sg;
            if (fm & FM_SIMPLE) eq[sg] = site - d.pos + (int)d.cig;
            else {
                const int3 rr = resolve_general(P.cigar + d.cig, d.n_cigar, d.pos, site);
                if (rr.z) continue;
                eq[sg] = rr.x; ei[sg] = rr.y;
            }
            has[sg] = (int)mapq >= P.min_mapq && !(fm & FLAG_FILTER);
        }
        // stage ii: the quality and base bytes of both sites, all loads in flight together
        uint32_t bqv[DEEP_MAX_SITES], bytev[DEEP_MAX_SITES];
#pragma unroll
        for (int sg = 0; sg < DEEP_MAX_SITES; ++sg) {
            bqv[sg] = 0u; bytev[sg] = 0u;
            if (has[sg]) { bqv[sg] = P.qual[qoff + (uint32_t)eq[sg]]; bytev[sg] = P.seq[soff + ((uint32_t)eq[sg] >> 1)]; }
        }
        // stage iii: base-quality filter, base class, the 13 terms
        uint32_t w[DEEP_MAX_SITES][N_STATS], emeta[DEEP_MAX_SITES];
#pragma unroll
        for (int sg = 0; sg < DEEP_MAX_SITES; ++sg) {
            emeta[sg] = 0u;
            if (!has[sg]) continue;
            const uint32_t bq = bqv[sg];
            if ((int)bq < P.min_bq) { has[sg] = false; continue; }
            const int qpos = eq[sg], indel = ei[sg];
            const bool base_part = !(indel > 0 && P.insertion_centric);
            const uint32_t nw = (indel != 0 ? 1u : 0u) + (base_part ? 1u : 0u);   // process_read calls that warn
            warn_nm += nw * ((fm >> 25) & 1u); warn_sm += nw * ((fm >> 26) & 1u);
            const uint32_t base = canonical16((bytev[sg] >> ((~qpos & 1) << 2)) & 0xFu);
            const Terms t = event_terms((fm & FM_FASTDIV) != 0, qpos, d.q2, d.tpi, d.lclip, d.clen, d.fl, d.fclen, d.rcp_l, d.rcp_clen);
            const uint32_t plus = (fm & 16u) ? 0u : 1u;
            const bool has_q2 = d.q2 > -1;
            w[sg][0] = 1u; w[sg][1] = mapq; w[sg][2] = bq; w[sg][3] = (uint32_t)d.se; w[sg][4] = plus; w[sg][5] = 1u - plus;
            w[sg][6] = __float_as_uint(t.posf); w[sg][7] = __float_as_uint(d.nmfrac); w[sg][8] = (uint32_t)d.mmq;
            w[sg][9] = has_q2 ? 1u : 0u; w[sg][10] = has_q2 ? __float_as_uint(t.q2term) : 0u;   // + 0.0f leaves the sum unchanged
            w[sg][11] = (uint32_t)d.clen; w[sg][12] = __float_as_uint(t.d3pterm);
            emeta[sg] = base | (indel != 0 ? 8u : 0u) | (base_part ? 16u : 0u) | (bq << 8);
        }
#ifdef BRC_DEEP_PROFILE
        const long long tq2 = clock64();
#endif
        // stable partition by group: one match per site on the covering reads' group; the passing events of a group are the
        // matched lanes that also passed, so rank and count come from the same mask
        int rank[DEEP_MAX_SITES];
#pragma unroll
        for (int sg = 0; sg < DEEP_MAX_SITES; ++sg) {
            const unsigned mc = __match_any_sync(0xffffffffu, gcov[sg] >= 0 ? gcov[sg] : -1 - lane);
            const unsigned mp_ = mc & __ballot_sync(0xffffffffu, has[sg]);
            const unsigned lt = (1u << lane) - 1u;
            rank[sg] = __popc(mp_ & lt);
            if (gcov[sg] >= 0 && (mc & lt) == 0u) atomicAdd(&sm.ncover[gcov[sg]], (uint32_t)__popc(mc));   // leader of the covering group
            if (has[sg] && rank[sg] == 0) { sm.wcnt[warp][grp[sg]] = (uint32_t)__popc(mp_); atomicAdd(&sm.npass[grp[sg]], (uint32_t)__popc(mp_)); }
        }
        __syncthreads();
        if (warp == 0) {
            uint32_t tot = 0u;
            if (lane < G) for (int wv = 0; wv < DEEP_WARPS; ++wv) { const uint32_t c = sm.wcnt[wv][lane]; sm.wcnt[wv][lane] = tot; tot += c; }
            // group bases: consecutive segments, each start nudged (by < 32 slots) onto a bank no earlier group starts on.
            // Owners of different groups read their i-th events together; equal-sized groups (a panel with evenly mixed
            // libraries) would otherwise all start on multiples of 32 — a G-way conflict on every LDS of the ordered pass.
            uint32_t cur = 0u, used = 0u, mybase = 0u;
            for (int g = 0; g < G; ++g) {
                const uint32_t tg = __shfl_sync(0xffffffffu, tot, g);
                const uint32_t rot = cur & 31u;
                const uint32_t taken = rot ? ((used >> rot) | (used << (32u - rot))) : used;   // bit p <=> bank (cur + p) % 32 is taken
                const uint32_t base = cur + (uint32_t)__ffs((int)~taken) - 1u;                  // <= 17 groups: a free bank exists
                used |= 1u << (base & 31u);
                if (lane == g) mybase = base;
                cur = base + tg;
            }
            if (lane < G) { sm.gcnt[lane] = tot; sm.gbase[lane] = mybase; }
        }
        __syncthreads();
#pragma unroll
        for (int sg = 0; sg < DEEP_MAX_SITES; ++sg) {
            if (!has[sg]) continue;
            const uint32_t slot = sm.gbase[grp[sg]] + sm.wcnt[warp][grp[sg]] + (uint32_t)rank[sg];
#pragma unroll
            for (int k = 0; k < N_STATS; ++k) sm.term[k][slot] = w[sg][k];
            sm.meta[slot] = emeta[sg]; sm.eread[slot] = r; sm.eqpos[slot] = eq[sg]; sm.eindel[slot] = ei[sg];
        }
        __syncthreads();
#ifdef BRC_DEEP_PROFILE
        const long long tq3 = clock64();
        prof[0] += tq1 - tq0; prof[1] += tq2 - tq1; prof[2] += tq3 - tq2; prof[3] += 1;
#endif
        // ---- phase 2: ordered accumulation (one loop per kind of statistic; a warp holds one kind) ----
        if (owner) {
            const uint32_t b0 = sm.gbase[og], n = sm.gcnt[og];
            const uint32_t *mp = sm.meta + b0, *xp = sm.term[oj] + b0;
            uint32_t i = 0;
            if (pbase == NO_BASE) {            // the first base event of the group fixes the primary class
                for (; i < n; ++i) { const uint32_t m = mp[i]; if (m & 16u) { pbase = m & 7u; break; } }
            }
            const uint32_t want = 16u | pbase;  // (m & 0x17) == want  <=>  base event of the primary class
            const bool is0 = oj == 0;
            // indel-only events before the first base event (insertion-centric): still the read_count owner's to replay
            if (is0) for (uint32_t k = 0; k < i; ++k) { const uint32_t m = mp[k]; if (m & 8u) deep_indel_event(P, sm, og, oslot, sec_head, sm.eindel[b0 + k], sm.eread[b0 + k], sm.eqpos[b0 + k], m >> 8); }
            // 32 events at a time, branch-free: a non-primary event adds 0 (exact: the sums are non-negative) and sets a bit;
            // the few marked events are then replayed in order — other base classes into their shared-memory cells, indel
            // alleles (separate keys, so their order relative to base events is immaterial) into the record pool
            for (uint32_t c0 = i; c0 < n; c0 += 32u) {
                const uint32_t cn = min(32u, n - c0);
                const uint32_t *mq = mp + c0, *xq = xp + c0;
                uint32_t nm = 0u, im = 0u;
                if (kind == 0) {
                    uint32_t a = acc_u;
#pragma unroll 4
                    for (uint32_t q = 0; q < cn; ++q) { const uint32_t m = mq[q], x = xq[q]; const bool take = (m & 0x17u) == want; a += take ? x : 0u; nm |= ((take ? 0u : m) >> 4 & 1u) << q; im |= (m >> 3 & 1u) << q; }
                    acc_u = a;
                } else if (kind == 1) {
                    float a = acc_f;
#pragma unroll 4
                    for (uint32_t q = 0; q < cn; ++q) { const uint32_t m = mq[q], x = xq[q]; const bool take = (m & 0x17u) == want; a = __fadd_rn(a, take ? __uint_as_float(x) : 0.0f); nm |= ((take ? 0u : m) >> 4 & 1u) << q; }
                    acc_f = a;
                } else {
                    double a = acc_d;
#pragma unroll 2
                    for (uint32_t q = 0; q < cn; ++q) {
                        const uint32_t m = mq[q], x = xq[q]; const bool take = (m & 0x17u) == want;
                        const double t = take ? __dsub_rn(1.0, (double)__uint_as_float(x)) : 0.0;     // off the carried chain
                        a = round_to_f32_precision(__dadd_rn(a, t)); nm |= ((take ? 0u : m) >> 4 & 1u) << q;
                    }
                    acc_d = a;
                }
                if (is0) while (im) {
                    const uint32_t q = (uint32_t)__ffs(im) - 1u; im &= im - 1u;
                    const uint32_t slot = b0 + c0 + q;
                    deep_indel_event(P, sm, og, oslot, sec_head, sm.eindel[slot], sm.eread[slot], sm.eqpos[slot], mq[q] >> 8);
                }
                while (nm) {
                    const uint32_t q = (uint32_t)__ffs(nm) - 1u; nm &= nm - 1u;
                    const uint32_t m = mq[q], x = xq[q];
                    unsigned long long &cell = sm.other[m & 7u][tid];
                    if (kind == 0) cell = (unsigned long long)((uint32_t)cell + x);
                    else if (kind == 1) cell = (unsigned long long)__float_as_uint(__fadd_rn(__uint_as_float((uint32_t)cell), __uint_as_float(x)));
                    else cell = (unsigned long long)__double_as_longlong(round_to_f32_precision(__dadd_rn(__longlong_as_double((long long)cell), __dsub_rn(1.0, (double)__uint_as_float(x)))));
                }
            }
        }
#ifdef BRC_DEEP_PROFILE
        const long long tq4 = clock64();
#endif
        __syncthreads();
#ifdef BRC_DEEP_PROFILE
        prof[4] += tq4 - tq3; prof[5] += clock64() - tq4;
#endif
    }
    cp_async_wait_all();

    // ---- emit: non-primary base classes become pool records (what site_emit does with its second class) ----
    for (int c = 0; c < 6; ++c) {
        const bool present = owner && (uint32_t)c != pbase && (uint32_t)sm.other[c][og] != 0u;   // thread og owns read_count of group og
        if (present && oj == 0) {
            const ResultsDev &R = P.res;
            const int32_t j = atomicAdd(R.sec_count, 1);
            if ((int64_t)j < R.sec_cap) {
                SecRec &r = R.sec[j];
                r.slot = oslot; r.next = sec_head; r.kind_len = (uint32_t)c; r.read = 0; r.qpos = 0;
                sec_head = j;
            }
            sm.recj[og] = j;
        }
        __syncthreads();
        if (present) {
            const int32_t j = sm.recj[og];
            if ((int64_t)j < P.res.sec_cap) {
                const unsigned long long cell = sm.other[c][tid];
                P.res.sec[j].stats[oj] = kind == 2 ? __float_as_uint(__double2float_rn(__longlong_as_double((long long)cell))) : (uint32_t)cell;
            }
        }
        __syncthreads();
    }
    // ---- emit: the packed record site_emit writes; the 13 owners of a group hand their sums to its read_count owner ----
    uint32_t *scr = sm.meta;                                   // free after the last block: [group][16] scratch
    if (owner) scr[og * 16 + oj] = kind == 2 ? __float_as_uint(__double2float_rn(acc_d)) : (kind == 1 ? __float_as_uint(acc_f) : acc_u);
    __syncthreads();
    if (owner && oj == 0) {
        const int sg = og / n_rows;
        uint32_t st[N_STATS];
#pragma unroll
        for (int k = 0; k < N_STATS; ++k) st[k] = scr[og * 16 + k];
        emit_packed(P.res, (int64_t)oslot, sm.ncover[og], sm.npass[og], (PER_LIB && sm.first_libless[sg] != 0x7fffffff) ? 1u : 0u, pbase, sec_head, st);
    }
    for (int o = 16; o; o >>= 1) { warn_sm += __shfl_xor_sync(0xffffffffu, warn_sm, o); warn_nm += __shfl_xor_sync(0xffffffffu, warn_nm, o); }
    if (lane == 0) {
        if (warn_sm) atomicAdd(P.res.warn + 0, (unsigned long long)warn_sm);
        if (warn_nm) atomicAdd(P.res.warn + 1, (unsigned long long)warn_nm);
    }
#ifdef BRC_DEEP_PROFILE
    if (tid == 0) for (int k = 0; k < 6; ++k) atomicAdd(&g_deepprof[k], (unsigned long long)prof[k]);
#endif
}

#ifdef BRC_DEEP_PROFILE
// cycles of thread 0 summed over CTAs: [0] phase 1a + barrier, [1] phase 1b, [2] partition + scatter, [3] blocks, [4] phase 2 (thread 0), [5] wait for the slowest owner
extern "C" __attribute__((visibility("default"))) void brc_debug_deepprof(unsigned long long *out, int reset) {
    cudaDeviceSynchronize();
    cudaMemcpyFromSymbol(out, g_deepprof, sizeof(g_deepprof));
    if (reset) { unsigned long long z[8] = {0}; cudaMemcpyToSymbol(g_deepprof, z, sizeof(z)); }
}
#endif

cudaError_t launch_deep_sites(const PileupParams &p, cudaStream_t s) {
    if (p.n_deep <= 0 || p.tile_count <= 0) return cudaSuccess;
    static std::atomic<bool> attr_set[64];
    int dev = 0; cudaGetDevice(&dev);
    if (dev >= 64 || !attr_set[dev].load(std::memory_order_acquire)) {
        std::lock_guard<std::mutex> lk(g_init_mu);
        cudaError_t e1 = cudaFuncSetAttribute(deep_site_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DeepSmem));
        cudaError_t e2 = cudaFuncSetAttribute(deep_site_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(DeepSmem));
        if (e1 != cudaSuccess) return e1;
        if (e2 != cudaSuccess) return e2;
        if (dev < 64) attr_set[dev].store(true, std::memory_order_release);
    }
    const dim3 grid((unsigned)p.n_deep, (unsigned)((p.res.n_rows + DEEP_ROWS - 1) / DEEP_ROWS));   // y: batches of DEEP_ROWS libraries
    if (p.per_lib) deep_site_kernel<true><<<grid, DEEP_THREADS, sizeof(DeepSmem), s>>>(p);
    else deep_site_kernel<false><<<grid, DEEP_THREADS, sizeof(DeepSmem), s>>>(p);
    return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// self-test: div_small / round_to_f32_precision / f32_to_f64_nonneg against the IEEE intrinsics
// ---------------------------------------------------------------------------------------------
__global__ void fastmath_selftest_kernel(int max_b, unsigned long long *bad) {
    const int b = blockIdx.x + 1;
    if (b > max_b) return;
    const float fb = (float)b, rcp = __frcp_rn(fb);
    unsigned long long nbad = 0;
    // every numerator the hot path can form for any divisor: |2 (qpos - left_clip) - clipped_length| reaches 2 (l_qseq - 1) when a
    // soft clip after a hard clip counts as a right clip (5H100S10M: 190..208 over 10)
    for (int a = threadIdx.x; a <= 2 * FASTDIV_MAX + 2; a += blockDim.x) {
        const float fa = (float)a;
        const float want = __fdiv_rn(fa, fb), got = div_small(fa, fb, rcp);
        if (__float_as_uint(want) != __float_as_uint(got)) nbad++;
        // 1 - f in double, added to a float-valued running sum, rounded back to float
        const double t_want = __dsub_rn(1.0, (double)want), t_got = __dsub_rn(1.0, f32_to_f64_nonneg(want));
        if (__double_as_longlong(t_want) != __double_as_longlong(t_got)) nbad++;
        for (int k = 0; k < 4; ++k) {
            const float s = __fmul_rn((float)(a * 7 + k * 131 + b), k == 3 ? -0.37f : 0.618034f);
            const double x = __dadd_rn((double)s, t_want);
            const float r_want = __double2float_rn(x);
            const double r_got = round_to_f32_precision(x);
            if ((double)r_want != r_got) nbad++;
        }
    }
    if (nbad) atomicAdd(bad, nbad);
}

cudaError_t launch_fastmath_selftest(int max_b, unsigned long long *d_bad, cudaStream_t s) {
    fastmath_selftest_kernel<<<max_b, 128, 0, s>>>(max_b, d_bad);
    return cudaGetLastError();
}

}  // namespace brc
