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

#include "../../include/brc_engine.h"
#include "brc_fmt_num.h"
#include "brc_seq.cuh"

namespace brc {

constexpr int TILE = 256;            // sites per CTA of the pileup kernel (threads = sites)
constexpr int N_STATS = BRC_N_STATS; // a 13-vector of statistics is indexed by the BRC_S_* names (print order)
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
// Exact quotient tables of the FM_FASTDIV event terms (brc_kernels.cu, one copy per device).  Row d (1 <= d <= FASTDIV_MAX) holds,
// at column QTAB_MID + j for -QTAB_MID <= j < QTAB_MID:
//   Q[d][QTAB_MID + j] = RN(|j| / d)                          (float)
//   P[d][QTAB_MID + j] = 1 - (double)RN(|2 j - d| / d)        (double, exact)
// so an event reads d3p at j = qpos - three_prime_index and the Q2 term at j = qpos - q2_pos in row l_qseq, and 1 - posf at
// j = qpos - left_clip in row clipped_length: the read's row and offset are folded into one base index, the event adds qpos.
// Every such j lies in (-QTAB_MID, QTAB_MID) since 0 <= qpos, left_clip, three_prime_index < l_qseq <= FASTDIV_MAX, except the
// Q2 column of a read without a Q2 position (q2_pos = -1), whose value is never used and whose j = l_qseq can reach QTAB_MID:
// row QTAB_ROWS - 1 is there to keep that load inside the allocation.  The row of l_qseq is found from ReadDesc::fl without a
// conversion: the bits of fl + 2^23 are 0x4B000000 + l_qseq, and shifted left by QTAB_SHIFT only l_qseq << QTAB_SHIFT remains.
constexpr int QTAB_SHIFT = 12;
constexpr int QTAB_MID = FASTDIV_MAX;
constexpr int QTAB_ROWS = FASTDIV_MAX + 2;
constexpr int64_t QTAB_ENTRIES = (int64_t)QTAB_ROWS << QTAB_SHIFT;
static_assert(2 * QTAB_MID == 1 << QTAB_SHIFT, "a quotient-table row spans j in [-QTAB_MID, QTAB_MID)");

struct __align__(16) ReadDesc {
    // q0
    int32_t pos;        // leftmost reference position
    int32_t end;        // bam_endpos clamped to INT32_MAX (== pos for reads the pileup buffer never admits)
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
    uint32_t cig;       // SIMPLE: qoff (qpos = site - pos + qoff); else low 32 bits of the index of the first CIGAR op
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
    // tile dispenser of THIS launch (ResultsDev::warn + WARN_WORDS + k, zeroed by init_tiles_kernel)
    unsigned long long *work_counter;
    // the device's quotient tables (QTAB_* above), filled in by launch_pileup for the kernels that read them (brc_kernels.cu USE_QTAB)
    const float *qtab_q;
    const double *qtab_p;
};
constexpr int WARN_WORDS = 4;          // ResultsDev::warn: [0] SM missing, [1] NM missing, [2..3] spare; followed by one tile
                                       // dispenser per pileup launch of a run

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

// Entry bounds (brc_set_site_filter_bounds): the entry that makes a line pass must satisfy every bound that is set, on its fields
// as the line prints them, in hundredths.  Evaluated by the device selection (pool records and the packed primaries) and by the
// host emitter (lines it forms itself), like site_passes.
using EntryBounds = brc_entry_bounds;
constexpr uint32_t BOUNDS_MASK = (1u << N_STATS) - 1u;

// The float32 quotient put_stat (brc_format.cpp) prints for a sum over a count.  Both evaluators round it once to nearest:
// __fdiv_rn is the IEEE division on the device whatever -prec-div says, the library is built with --fmad=false so nothing is
// contracted around it, and the host's `/` on floats is the IEEE division.  The u32 sums are converted to float with
// round-to-nearest on both sides too (__uint2float_rn, the host conversion).
__host__ __device__ inline float stat_u2f(uint32_t v) {
#ifdef __CUDA_ARCH__
    return __uint2float_rn(v);
#else
    return (float)v;
#endif
}
__host__ __device__ inline float stat_bits(uint32_t v) { float f; std::memcpy(&f, &v, 4); return f; }
__host__ __device__ inline float stat_quot(float num, uint32_t den) {
#ifdef __CUDA_ARCH__
    return __fdiv_rn(num, __uint2float_rn(den));
#else
    return num / (float)den;
#endif
}
// a printed average in hundredths (put_f2's digits, signed); no average of the engine's sums reaches 2^54, which saturates
__host__ __device__ inline int64_t printed_hundredths(float q) {
    const uint64_t h = f2_hundredths(q);
    if (h > (uint64_t)INT64_MAX) return INT64_MAX;
    return q < 0.0f ? -(int64_t)h : (int64_t)h;
}
// Field k (BRC_S_*) of an entry as put_stat prints it, in hundredths.
__host__ __device__ inline int64_t entry_field(const uint32_t v[N_STATS], int k, bool is_indel) {
    const uint32_t n = v[BRC_S_COUNT];
    if (n == 0) return 0;                                     // the all-zero entry
    switch (k) {
    case BRC_S_COUNT: case BRC_S_PLUS: case BRC_S_MINUS: case BRC_S_NQ2: return (int64_t)v[k] * 100;
    case BRC_S_BASEQ: return is_indel ? 0 : printed_hundredths(stat_quot(stat_u2f(v[k]), n));
    case BRC_S_MAPQ: case BRC_S_SE_MAPQ: case BRC_S_MMQS: case BRC_S_CLIP_LEN: return printed_hundredths(stat_quot(stat_u2f(v[k]), n));
    case BRC_S_Q2_DIST: return v[BRC_S_NQ2] ? printed_hundredths(stat_quot(stat_bits(v[k]), v[BRC_S_NQ2])) : 0;
    default: return printed_hundredths(stat_quot(stat_bits(v[k]), n));   // POS_FRAC, NM_FRAC, 3P_DIST: float sums
    }
}
// Every bound that is set holds on the entry; only the fields with a bound are evaluated.
__host__ __device__ inline bool entry_within(const uint32_t v[N_STATS], bool is_indel, const EntryBounds &B) {
    const uint32_t set = B.lo_set | B.hi_set;
    if (!set) return true;
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int k = 0; k < N_STATS; ++k) {
        if (!((set >> k) & 1u)) continue;
        const int64_t x = entry_field(v, k, is_indel);
        if ((((B.lo_set >> k) & 1u) && x < B.lo[k]) || (((B.hi_set >> k) & 1u) && x > B.hi[k])) return false;
    }
    return true;
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
    EntryBounds bounds;     // no bit set: no bounds
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

// ---- the line a site forms (brc_format.cpp format_site), as the packed records hold it ----
// One definition for the site selection (brc_select.cu), the allele queries (brc_alleles.cu) and the engine host (ensure_wide,
// brc_get_warning_counts).
// Row r spans site s (column idx = r * n_slots + s): an escaped primary, or ncover > 0.  RS = n_rows * n_slots.
__host__ __device__ __forceinline__ bool row_covers(const uint32_t *words, int64_t RS, int64_t idx) {
    return (words[RS + idx] & 7u) == PB_ESCAPE || (words[idx] & 0xFFu) != 0u;
}
// The 13 accumulators of the primary held in the packed words of column idx (word w at words[w * RS + idx]; layout above).
__host__ __device__ __forceinline__ void unpack_primary(const uint32_t *words, int64_t RS, int64_t idx, uint32_t v[N_STATS]) {
    uint32_t w[N_WORDS];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int k = 0; k < N_WORDS; ++k) w[k] = words[k * RS + idx];
    const uint32_t count = (w[0] >> 16) & 0xFFu, plus = w[0] >> 24;
    v[BRC_S_COUNT] = count; v[BRC_S_MAPQ] = w[1] >> 16; v[BRC_S_BASEQ] = w[2] & 0xFFFFu; v[BRC_S_SE_MAPQ] = w[2] >> 16;
    v[BRC_S_PLUS] = plus; v[BRC_S_MINUS] = count - plus; v[BRC_S_POS_FRAC] = w[4]; v[BRC_S_NM_FRAC] = w[5];
    v[BRC_S_MMQS] = w[3] >> 16; v[BRC_S_NQ2] = (w[1] >> 8) & 0xFFu; v[BRC_S_Q2_DIST] = w[6]; v[BRC_S_CLIP_LEN] = w[3] & 0xFFFFu;
    v[BRC_S_3P_DIST] = w[7];
}
// Some row has a read without library at site s: -p abandons the site (no line, and its deletions are never queued).
__host__ __device__ __forceinline__ bool site_abandoned(const uint32_t *words, int n_rows, int64_t NS, int64_t s) {
    const int64_t RS = (int64_t)n_rows * NS;
    bool ab = false;
    for (int r = 0; r < n_rows; ++r) ab |= (words[RS + (int64_t)r * NS + s] & 8u) != 0u;
    return ab;
}
#ifdef __CUDACC__   // device atomics: not for the host-only translation units
// Pool pass, one secondary-pool record: what it adds to the depth of a line.  An escaped primary adds its npass to esc_np[s];
// a deletion adds its count to dsum[s] (extra depth of the next site's line) when the same row spans the next site, where the
// row's block prints it.  Returns true for such a deletion.  dsum and esc_np are [n_slots], zeroed before the pass.
__device__ __forceinline__ bool pool_depth_term(const uint32_t *words, int n_rows, int64_t NS, const SecRec &rec, uint32_t *dsum,
                                                uint32_t *esc_np) {
    const int64_t r = (int64_t)rec.slot / NS, s = (int64_t)rec.slot - r * NS;
    const uint32_t kind = rec.kind_len & 0xFFu;
    if (kind >= KIND_WIDE) { atomicAdd(&esc_np[s], (uint32_t)rec.qpos); return false; }
    if (kind != (uint32_t)KIND_DEL || s + 1 >= NS || !row_covers(words, (int64_t)n_rows * NS, r * NS + s + 1)) return false;
    atomicAdd(&dsum[s], rec.stats[BRC_S_COUNT]);
    return true;
}
// Site pass, after the pool pass: does site s form a line (a row spans it and no row abandons it), and its depth (the line's
// 4th column): Σ npass + the escaped primaries' npass + the deletions anchored at the left neighbour, when that neighbour is in
// the same region (`left_in_region`) and formed a line of its own.  `left` reports that last condition.
struct SiteLine { uint64_t depth; bool live, abandoned, left; };
__device__ __forceinline__ SiteLine site_line(const uint32_t *words, int n_rows, int64_t NS, int64_t s, bool left_in_region,
                                              const uint32_t *dsum, const uint32_t *esc_np) {
    const int64_t RS = (int64_t)n_rows * NS;
    SiteLine L{esc_np[s], false, false, false};
    bool covered = false;
    for (int r = 0; r < n_rows; ++r) {
        const uint32_t w0 = words[(int64_t)r * NS + s], w1 = words[RS + (int64_t)r * NS + s];
        L.abandoned |= (w1 & 8u) != 0u;
        if ((w1 & 7u) == PB_ESCAPE) { covered = true; continue; }      // full-width primary: a pool record (esc_np)
        covered |= (w0 & 0xFFu) != 0u;
        L.depth += (w0 >> 8) & 0xFFu;
    }
    L.left = left_in_region && !site_abandoned(words, n_rows, NS, s - 1);
    if (L.left) L.depth += dsum[s - 1];
    L.live = covered && !L.abandoned;
    return L;
}

#endif

// ---- allele queries (brc_alleles.cu; brc_set_allele_queries, DESIGN.md §12) ----
constexpr uint32_t NO_SLOT = 0xFFFFFFFFu;
struct AlleleQuery {      // one query as the kernels see it; the host sorts them by `match`
    uint32_t match;       // slot whose pool records hold the entry: the site's own, or its left neighbour's for a deletion;
                          // NO_SLOT when no record can (a deletion whose anchor lies outside the region, a site without a slot)
    uint32_t kind_len;    // as brc_allele_query (base classes with length 0)
    uint32_t site;        // slot of the queried site; NO_SLOT when the region computed none for it (no read reaches it)
    uint32_t left;        // 1: the left neighbour is in the same region
    int64_t bases_off;    // insertion: offset of its bases in AlleleParams::bases (indices into "=ACGTN")
    int64_t out;          // index of its answer (the caller's order)
};
static_assert(sizeof(AlleleQuery) == 32, "AlleleQuery is 32 bytes");
static_assert(sizeof(brc_allele_answer) == 64, "brc_allele_answer is 64 bytes");

struct AlleleParams {
    const uint32_t *words;  // [N_WORDS][rows*slots]
    int32_t n_rows;
    int64_t n_slots;
    const SecRec *sec;
    const int32_t *sec_count;
    int64_t sec_cap;
    const uint64_t *seq_off;  // the device batch: packed bases of a record's representative read (insertion alleles)
    const uint8_t *seq;
    const AlleleQuery *q;
    int64_t n_q;
    const uint8_t *bases;
    uint32_t *dsum, *esc_np;  // [n_slots] each, zeroed before the record pass
    brc_allele_answer *ans;   // [n_q], zeroed before the record pass
};

// ---- complex-record queries (brc_complex.cu; brc_set_complex_queries, DESIGN.md §12) ----
struct ComplexQuery {     // one query as the kernel sees it, resolved against the batch's geometry when it is launched
    int64_t tile;         // the tile holding `pos`; -1 when no read can span (no slot there, or the right flank past the contig)
    int32_t pos;          // first span base
    int32_t ref_len;
    int64_t allele0;      // its alleles are ComplexParams::alleles[allele0, allele0 + n_alleles), its answers the same counts
    int32_t n_alleles;
    int32_t reserved;
};
static_assert(sizeof(ComplexQuery) == 32, "ComplexQuery is 32 bytes");

struct ComplexParams {
    const ReadDesc *desc;
    const int32_t *tile_lo, *tile_hi;
    const uint64_t *cigar_off; const uint32_t *cigar;
    const uint64_t *seq_off; const uint8_t *seq;
    const uint64_t *qual_off; const uint8_t *qual;
    int32_t min_bq;
    const ComplexQuery *q;
    int64_t n_q;
    const brc_complex_allele *alleles;   // bases_off indexes `bases`
    int64_t n_alleles;
    const uint8_t *bases;                // allele bases as indices into "=ACGTN"
    uint32_t *depth;                     // [n_q]
    brc_complex_count *counts;           // [n_alleles]
};

// launch wrappers (brc_kernels.cu)
cudaError_t launch_init_tiles(int32_t *tile_lo, int32_t *tile_hi, int64_t n_tiles, int32_t *sec_count,
                              unsigned long long *warn, int n_dispensers, cudaStream_t s);
cudaError_t launch_precompute(const PrecomputeParams &p, cudaStream_t s);
cudaError_t launch_ref_encode(const char *d_ascii, uint8_t *d_code, int64_t n, cudaStream_t s);
cudaError_t launch_pileup(const PileupParams &p, cudaStream_t s);
cudaError_t launch_deep_sites(const PileupParams &p, cudaStream_t s);   // no-op when p.n_deep == 0
cudaError_t launch_fill_offsets(uint64_t *off, int64_t n, uint64_t base, uint64_t stride, cudaStream_t s);   // off[i] = base + i * stride
cudaError_t launch_fill_i32(int32_t *dst, int64_t n, int32_t v, cudaStream_t s);
cudaError_t launch_fastmath_selftest(int max_b, unsigned long long *d_bad, cudaStream_t s);
// the current device's quotient tables (QTAB_*), built on first use
cudaError_t quotient_tables(const float **q, const double **p);
// brc_select.cu: pool pass, site pass, ship flags, scan, compaction of sites and pool records (SELECT_KERNELS launches)
constexpr int SELECT_KERNELS = 8;
constexpr int SELECT_SCAN_CTA = 256;   // sites per scan partial (SelectParams::nb = ceil(n_slots / SELECT_SCAN_CTA))
cudaError_t launch_select(const SelectParams &p, cudaStream_t s);
// brc_alleles.cu: record pass, query pass (ALLELE_KERNELS launches; the scratch and answers are zeroed by the caller)
constexpr int ALLELE_KERNELS = 2;
cudaError_t launch_alleles(const AlleleParams &p, cudaStream_t s);
// brc_complex.cu: one warp per complex query (COMPLEX_KERNELS launch)
constexpr int COMPLEX_KERNELS = 1;
cudaError_t launch_complex(const ComplexParams &p, cudaStream_t s);

}  // namespace brc
