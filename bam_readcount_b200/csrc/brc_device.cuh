// brc_device.cuh — device-side data layout shared by the kernels and the host engine.
//
// HBM layout (all SoA unless noted; DESIGN.md §3):
//   reads   : pos/flag/mapq/lib/l_qseq/nm/sm arrays + cigar/seq/qual byte pools with offsets
//             (exactly the brc_read_batch of include/brc_engine.h, device pointers)
//   desc    : ReadDesc[n_reads]  (AoS, 80 B, 16-B aligned) written by K0, read by K1 —
//             the packed replacement of the reference's "Zm" string tag (R:auxfields.hpp:6-35)
//   tiles   : TileInfo[n_tiles]  one per TILE consecutive computed sites of a region
//   tile_lo / tile_hi : int32[n_tiles]  first / one-past-last read overlapping the tile (K0 atomics)
//   results : per (row, slot) header + 13 primary accumulators, secondary key records
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace brc {

constexpr int TILE = 256;            // sites per CTA of the pileup kernel (threads = sites)
constexpr int N_STATS = 13;
constexpr uint32_t LIB_NONE = 0xFFFFu;
constexpr int KIND_INS = 6, KIND_DEL = 7;
constexpr uint8_t NO_BASE = 255;

// flag bits the reference filters on (R:bamreadcount.cpp:295-310)
constexpr uint32_t FLAG_FILTER = 4u | 256u | 512u | 1024u;

// ReadDesc.fm layout: flag[0:16) | mapq[16:24) | bits below
constexpr uint32_t FM_SIMPLE = 1u << 24;     // CIGAR has exactly one ref-consuming op, of match type, and no I/D/N/P
constexpr uint32_t FM_NM_ABSENT = 1u << 25;  // NM tag missing -> NM_TAG_MISSING warning per process_read
constexpr uint32_t FM_SM_MISSING = 1u << 26; // proper pair without SM tag -> SM_TAG_MISSING warning per process_read
constexpr uint32_t FM_FASTDIV = 1u << 27;    // 1 <= l_qseq, clipped_length <= FASTDIV_MAX: reciprocal division is exact (tests)
constexpr uint32_t FM_HOT = 1u << 28;        // SIMPLE && FASTDIV && no missing-tag warnings: the hot loop's straight-line path
constexpr uint32_t FM_DEAD = 1u << 29;       // fails -q or the flag filter (R:bamreadcount.cpp:288-310): only counts as a spanning read
constexpr int FASTDIV_MAX = 2048;

struct __align__(16) ReadDesc {
    // q0
    int32_t pos;        // leftmost reference position
    int32_t end;        // bam_endpos (== pos for reads the pileup buffer never admits)
    uint32_t fm;        // flag | mapq<<16 | FM_* bits
    uint32_t lib_nc;    // lib[0:16) | min(n_cigar,0xFFFF)<<16
    // q1 : four of the five values of fetch_func (R:bamreadcount.cpp:248-253)
    int32_t mmq;        // sum_of_mismatch_qualities
    int32_t clen;       // clipped_length
    int32_t lclip;      // left_clip
    int32_t tpi;        // three_prime_index
    // q2
    int32_t q2;         // q2_pos
    float nmfrac;       // (float)NM / (float)clipped_length   (R:BasicStat.cpp:97), +0 if NM absent
    int32_t se;         // contribution to sum_single_ended_map_qualities (R:BasicStat.cpp:78-91)
    float fl;           // (float)l_qseq
    // q3
    uint32_t qual32;    // low 32 bits of the read's byte offset in the qual pool
    uint32_t seq32;     // low 32 bits of the read's byte offset in the seq pool
    uint32_t cig;       // SIMPLE: qoff (qpos = site - pos + qoff); else index of the first CIGAR op
    uint32_t n_cigar;
    // q4
    float rcp_l;        // RN(1 / (float)l_qseq)         (FM_FASTDIV only)
    float rcp_clen;     // RN(1 / (float)clipped_length) (FM_FASTDIV only)
    float fclen;        // (float)clipped_length
    uint32_t inc;       // per-event increments of the packed chunk counters: 1 | plus << 8 | (q2 > -1) << 16
};
static_assert(sizeof(ReadDesc) == 80, "ReadDesc must be 80 bytes");

// K1 shared-memory staging: capacity of ONE slot of the 2-stage TMA ring
#ifndef BRC_STAGE_READS
#define BRC_STAGE_READS 96
#endif
constexpr int STAGE_READS = BRC_STAGE_READS;                 // descriptors per chunk
constexpr int STAGE_QUAL = STAGE_READS * 152 + 32;          // staged quality bytes per chunk (incl. 16-B alignment slack both ends)
constexpr int STAGE_SEQ = STAGE_READS * 76 + 32;            // staged packed-base bytes per chunk
constexpr int STAGE_CIGAR = STAGE_READS * 2;                // staged CIGAR ops per chunk (u32); chunks with more fall back to global loads

struct TileInfo {
    int32_t pos0;       // absolute position of the tile's first site
    int32_t n;          // sites in this tile (<= TILE)
    int64_t slot0;      // result slot of the first site
};

struct RegionDev {
    int32_t tid_slot;   // index into RefWin table
    int32_t first_pos;  // max(beg-1, 0)
    int32_t end;        // exclusive
    int32_t ref_len_check; // site-list mode (R:bamreadcount.cpp:144-148)
    int64_t tile_base;  // first tile of the region
    int64_t read_lo, read_hi;
};

struct RefWin {
    const char *seq;    // device pointer to PACKED 4-bit reference codes (seq_nt16_table of the FASTA characters, two per
                        // byte, first in the high nibble); symbol 0 = position win_beg; 16 readable bytes of padding
    int64_t chrom_len;
    int64_t win_beg;
    int64_t win_len;
};

struct ReadsDev {
    int64_t n_reads;
    const int32_t *pos;
    const uint16_t *flag;
    const uint8_t *mapq;
    const uint16_t *lib;      // may be null
    const int32_t *l_qseq;
    const int32_t *nm;
    const int32_t *sm;
    const uint64_t *cigar_off;
    const uint32_t *cigar;
    const uint64_t *seq_off;
    const uint8_t *seq;
    const uint64_t *qual_off;
    const uint8_t *qual;
};

// Packed per-site record (include/brc_engine.h "packed results"): 8 x u32 words per (row, slot), stored SoA as
// words[w][row * n_slots + slot].  A site whose counters do not fit the narrow fields (depth > 255, 16-bit sums
// overflowing) is ESCAPED: its words carry only the flags and its full-width record lives in the secondary pool.
//   W0  ncover[0:8) | npass[8:16) | count[16:24) | plus[24:32)
//   W1  pbase code [0:3) (0..5 = "=ACGTN", 6 = none, 7 = escaped) | libless flag bit 3 | has-secondary bit 4 |
//       nq2 [8:16) | sum mapq [16:32)
//   W2  sum baseq [0:16) | sum SE-mapq [16:32)
//   W3  sum clipped length [0:16) | sum mismatch qualities [16:32)
//   W4..W7  float32 bits: sum_event_location, sum_number_of_mismatches, sum_q2_distance, sum_3p_distance
constexpr int N_WORDS = 8;
constexpr uint32_t PB_NONE = 6u, PB_ESCAPE = 7u;
constexpr uint32_t KIND_WIDE = 8u;    // secondary-pool record holding an escaped site's primary: kind = 8 + pbase code (0..6)

// Secondary-pool record (72 B, AoS): other base classes, indel alleles and escaped primaries of one (row, slot).
struct SecRec {
    uint32_t slot;       // row * n_slots + slot
    int32_t next;        // previous record of the same (row, slot) or -1 (device-internal chain)
    uint32_t kind_len;   // kind [0:8) | length [8:32): indel length; escaped primary: ncover
    int32_t read;        // representative read carrying the inserted bases; escaped primary: flags
    int32_t qpos;        // its qpos; escaped primary: npass
    uint32_t stats[N_STATS];
};
static_assert(sizeof(SecRec) == 72, "SecRec must be 72 bytes");

struct ResultsDev {
    int32_t n_rows;
    int64_t n_slots;
    uint32_t *words;      // [N_WORDS][rows*slots]
    // secondary key pool
    int64_t sec_cap;
    int32_t *sec_count;   // device counter (may exceed cap -> overflow)
    SecRec *sec;
    unsigned long long *warn; // [0]=SM missing events, [1]=NM missing events
};

struct PileupParams {
    int32_t min_mapq, min_bq, per_lib, insertion_centric;
    const ReadDesc *desc;
    const uint64_t *cigar_off; // [n_reads+1]
    const uint32_t *cigar;
    const uint8_t *seq;       // 16-byte aligned, >= 16 readable bytes past the last read
    const uint8_t *qual;      // 16-byte aligned, >= 16 readable bytes past the last read
    const uint64_t *seq_off;  // [n_reads+1]
    const uint64_t *qual_off; // [n_reads+1]
    const TileInfo *tiles;
    const int32_t *tile_lo;
    const int32_t *tile_hi;
    int64_t n_tiles;       // tiles of the whole plan
    int64_t tile_begin;    // this launch covers tiles [tile_begin, tile_begin + tile_count)
    int64_t tile_count;
    ResultsDev res;
    // deep-site kernel (brc_kernels.cu): candidate tiles (<= DEEP_MAX_SITES sites); a candidate whose read window holds at
    // least deep_min_reads reads is computed by deep_site_kernel and skipped by pileup_kernel
    const int32_t *deep_tiles;
    int32_t n_deep;
    int32_t deep_min_reads;
    // tile dispenser of THIS launch (ResultsDev::warn + WARN_WORDS + k, zeroed by init_tiles_kernel); nullptr = fixed stride
    unsigned long long *work_counter;
};
constexpr int WARN_WORDS = 4;          // ResultsDev::warn: [0] SM missing, [1] NM missing, [2..3] spare
constexpr int N_WORK_COUNTERS = 64;    // followed by one tile dispenser per pileup launch of a run

constexpr int DEEP_MAX_SITES = 2;
constexpr int DEEP_THREADS = 256;
// one owner thread per (site, library row, statistic) must fit one CTA: a CTA takes the tile's sites x up to DEEP_ROWS library
// rows; a -p tile with more libraries is spread over ceil(n_rows / DEEP_ROWS) CTAs (grid.y), each streaming the tile's reads and
// keeping the events of its own rows
// (integer, float and double statistics start on warp boundaries so a warp runs one kind of loop: 9G | 3G | G threads)
constexpr int DEEP_ROWS = 8;
__host__ __device__ inline int deep_flt_base(int G) { return (9 * G + 31) & ~31; }
__host__ __device__ inline int deep_dbl_base(int G) { return (deep_flt_base(G) + 3 * G + 31) & ~31; }
__host__ __device__ inline bool deep_shape_ok(int n_sites, int n_rows) {
    const int G = n_sites * (n_rows < DEEP_ROWS ? n_rows : DEEP_ROWS);
    return n_sites <= DEEP_MAX_SITES && G >= 1 && deep_dbl_base(G) + G <= DEEP_THREADS;
}

struct PrecomputeParams {
    ReadsDev reads;
    const RegionDev *regions;
    int64_t n_regions;
    const int32_t *region_of_read;  // null when n_regions == 1
    const RefWin *refs;
    ReadDesc *desc;
    int32_t *tile_lo;
    int32_t *tile_hi;
    int64_t read_begin;    // this launch covers reads [read_begin, read_end)
    int64_t read_end;
    int32_t min_mapq;      // -q: reads below it (or failing the flag filter) are marked FM_DEAD
};

// ---- alternative-allele site filter (brc_select.cu on the device, the text emitter on the host; DESIGN.md §10) ----
// A base class 1..4 ("ACGT") is an alternative allele unless the reference base encodes exactly that one base (seq_nt16 codes
// 1/2/4/8); a reference N, IUPAC code or missing character makes every base alternative.
__host__ __device__ inline bool base_is_alt(uint32_t base_class, uint32_t ref_code) {
    return base_class >= 1u && base_class <= 4u && (1u << (base_class - 1u)) != ref_code;
}
// The rule for one printed line: its largest alternative-allele count against min_alt_count and min_alt_fraction * depth (IEEE
// double; depth = the line's 4th column).  The one predicate both the device selection and the host emitter evaluate.
__host__ __device__ inline bool site_passes(uint64_t best_alt, uint64_t depth, int32_t min_alt_count, double min_alt_fraction) {
    return best_alt >= (uint64_t)min_alt_count && (double)best_alt >= min_alt_fraction * (double)depth;
}

struct SelRegion {         // one region as the selection kernels see it
    int64_t slot_base;
    int32_t n_slots;
    int32_t first_pos;
    int32_t beg, end;      // printed positions [beg, end)
    int32_t keep_all_n;    // slots [0, keep_all_n) are shipped whenever they print a line (deletions carried in from other regions)
    int32_t argv;          // argv region: the last live site of every library row is shipped too (the deletion queue it leaves)
    int32_t tid_slot;      // index into the RefWin table
    int32_t ref_on_host;   // 0: the emitter has no reference characters for this contig and prints N, so every base is alternative
};

struct SelectParams {
    const uint32_t *words;  // [N_WORDS][rows*slots]
    int32_t n_rows;
    int64_t n_slots;
    const SecRec *sec;
    const int32_t *sec_count;
    int64_t sec_cap;
    const SelRegion *regions;
    int64_t n_regions;
    const RefWin *refs;
    int32_t min_alt_count;
    double min_alt_fraction;
    // per-site scratch, [n_slots] each (best .. esc_np and reg_last, counters zeroed before the pool pass)
    uint32_t *best;         // largest alternative count of the site's pool records
    uint32_t *dsum;         // deletion counts anchored here that print at the next site (extra depth there)
    uint32_t *dbest;        // largest such deletion count
    uint32_t *esc_np;       // npass of the site's escaped primaries
    uint32_t *reg_last;     // [n_regions][n_rows] 1 + offset of the last live site of an argv region that the row covers
    unsigned long long *counters;   // [0] pool records shipped, [1] abandoned sites (-p, a read without library)
    uint8_t *keep;          // bit0 rule holds, bit1 keep-all range, bit2 live (a line is formed at the site)
    uint8_t *emit;          // emit byte of the shipped site
    uint32_t *ship;         // 1 = shipped (scan input)
    unsigned long long *partial;
    int64_t nb;
    uint64_t *idx;          // [n_slots+1] compact index of each shipped site; idx[n_slots] = shipped sites
    // compact outputs
    uint32_t *c_site;
    uint8_t *c_emit;
    uint32_t *c_words;      // [N_WORDS][rows*n_sel]
    SecRec *c_sec;
};

// launch wrappers (brc_kernels.cu)
cudaError_t launch_init_tiles(int32_t *tile_lo, int32_t *tile_hi, int64_t n_tiles, int32_t *sec_count,
                              unsigned long long *warn, cudaStream_t s);
cudaError_t launch_precompute(const PrecomputeParams &p, cudaStream_t s);
cudaError_t launch_ref_encode(const char *d_ascii, uint8_t *d_code, int64_t n, cudaStream_t s);
cudaError_t launch_pileup(const PileupParams &p, cudaStream_t s);
cudaError_t launch_deep_sites(const PileupParams &p, cudaStream_t s);   // no-op when p.n_deep == 0
cudaError_t launch_fill_offsets(uint64_t *off, int64_t n, uint64_t base, uint64_t stride, cudaStream_t s);   // off[i] = base + i * stride
cudaError_t launch_fill_i32(int32_t *dst, int64_t n, int32_t v, cudaStream_t s);
cudaError_t launch_fastmath_selftest(int max_b, unsigned long long *d_bad, cudaStream_t s);
// brc_select.cu: pool pass, site pass, ship flags, scan, compaction of sites and pool records (SELECT_KERNELS launches)
constexpr int SELECT_KERNELS = 8;
constexpr int SELECT_SCAN_CTA = 256;   // sites per scan partial (SelectParams::nb = ceil(n_slots / SELECT_SCAN_CTA))
cudaError_t launch_select(const SelectParams &p, cudaStream_t s);

}  // namespace brc
