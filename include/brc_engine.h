/*
 * brc_engine.h — C ABI of the H100-native pileup-readcount engine (libbrc_engine.so).
 *
 * Drop-in boundary for ONE path of genome/bam-readcount: the two htslib callbacks its
 * region loops register (SURVEY.md §8b):
 *
 *   typedef int (*bam_fetch_f)(const bam1_t *b, void *data);                 V:bam.h:452
 *       fetch_func()      R:src/exe/bam-readcount/bamreadcount.cpp:114-261
 *   typedef int (*bam_pileup_f)(uint32_t tid, uint32_t pos, int n,
 *                               const bam_pileup1_t *pl, void *data);        V:bam.h:388
 *       pileup_func()     R:src/exe/bam-readcount/bamreadcount.cpp:265-419
 *
 * plus the per-region driver around them (bam_plbuf_init / samfetch / bam_plbuf_push(0) /
 * bam_plbuf_destroy, R:bamreadcount.cpp:591-605 and :650-656).  Mapping:
 *
 *   reference call (file:line)                               engine entry point
 *   -------------------------------------------------------  ---------------------------
 *   pileup_data_t d{} + flags          R:...:430-465          brc_create(&cfg,&e)
 *   load_reference()/fai_fetch         R:...:83-90            brc_set_reference()
 *   d.beg/d.end + bam_plbuf_init +
 *     bam_plp_set_maxcnt               R:...:588-592,644-651  brc_begin_region()
 *   fetch_func(b) + bam_plbuf_push(b)  R:...:114-261,259      brc_push_read() / brc_push_reads()
 *   bam_plbuf_push(0,buf)+destroy      R:...:603-604,655-656  brc_end_region()
 *   every pileup_func() invocation     R:...:265-419          brc_compute() -> brc_get_results()
 *   operator<<(BasicStat) + cout line  R:BasicStat.cpp:110-159,
 *                                      R:...:351-416          brc_format_text()
 *   ReadWarnings counters              R:ReadWarnings.hpp     brc_get_warning_counts()
 *
 * Plain pointers and sizes only; no C++ or torch types cross this boundary; nothing throws.
 * All functions return 0 (BRC_OK) or a negative brc_status.  One caller thread per handle
 * (the reference's callbacks are not re-entrant either, SURVEY.md §8b "Threading"); different
 * handles are independent and may be driven from different threads at the same time (their
 * streams, device buffers and pinned host buffers are their own; the process-wide per-device
 * set-up is serialised inside the library).
 * The library REQUIRES a CUDA device: there is no CPU fallback (brc_create fails with
 * BRC_E_NO_DEVICE when none is usable).
 */
#ifndef BRC_ENGINE_H
#define BRC_ENGINE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define BRC_ABI_VERSION 2

#if defined(__GNUC__)
#define BRC_API __attribute__((visibility("default")))
#else
#define BRC_API
#endif

typedef enum {
    BRC_OK = 0,
    BRC_E_INVALID = -1,       /* bad argument / call order */
    BRC_E_NO_DEVICE = -2,     /* no usable CUDA device */
    BRC_E_CUDA = -3,          /* CUDA runtime failure (brc_last_error has the text) */
    BRC_E_NOMEM = -4,
    BRC_E_UNSORTED = -5,      /* reads of a region not sorted by position (htslib: "Pileup aborts", V:htslib-1.10/sam.c:4502-4511) */
    BRC_E_NO_REFERENCE = -6,  /* reference window does not cover the region (the reference binary would SIGSEGV, SURVEY.md A.6) */
    BRC_E_BAD_LIBRARY = -7,   /* library id >= n_libs */
    BRC_E_OVERFLOW = -8,      /* internal pool overflow that retry could not resolve */
    BRC_E_IO = -9             /* write() to an output failed (errno holds its reason when a brc_bgzf_* call returns it) */
} brc_status;

#define BRC_TAG_ABSENT INT32_MIN  /* NM:i / SM:i tag not present on the read */
#define BRC_LIB_NONE 0xFFFFu      /* read has no RG, or its @RG has no LB (bam_get_library()==NULL, V:bam.c:77-101) */

/* allele kinds of a result key */
#define BRC_KIND_INS 6            /* kinds 0..5 index "=ACGTN" (R:bamreadcount.cpp:34) */
#define BRC_KIND_DEL 7
#define BRC_NO_BASE 255

/* the 13 accumulators of BasicStat (R:src/lib/bamrc/BasicStat.hpp:12-24), in print order */
enum {
    BRC_S_COUNT = 0,      /* read_count                      u32 */
    BRC_S_MAPQ = 1,       /* sum_map_qualities               u32 */
    BRC_S_BASEQ = 2,      /* sum_base_qualities              u32 (not accumulated for indel keys) */
    BRC_S_SE_MAPQ = 3,    /* sum_single_ended_map_qualities  u32 */
    BRC_S_PLUS = 4,       /* num_plus_strand                 u32 */
    BRC_S_MINUS = 5,      /* num_minus_strand                u32 */
    BRC_S_POS_FRAC = 6,   /* sum_event_location              f32 bits */
    BRC_S_NM_FRAC = 7,    /* sum_number_of_mismatches        f32 bits */
    BRC_S_MMQS = 8,       /* sum_of_mismatch_qualities       u32 */
    BRC_S_NQ2 = 9,        /* num_q2_reads                    u32 */
    BRC_S_Q2_DIST = 10,   /* sum_q2_distance                 f32 bits */
    BRC_S_CLIP_LEN = 11,  /* sum_of_clipped_lengths          u32 */
    BRC_S_3P_DIST = 12,   /* sum_3p_distance                 f32 bits */
    BRC_N_STATS = 13
};

typedef struct brc_engine brc_engine;

/* pileup_data_t's option fields (R:bamreadcount.cpp:55-71, flags :438-446) */
typedef struct {
    int32_t min_mapq;           /* -q */
    int32_t min_bq;             /* -b */
    int32_t max_cnt;            /* -d  (bam_plp_set_maxcnt) */
    int32_t per_lib;            /* -p */
    int32_t insertion_centric;  /* -i */
    int32_t n_libs;             /* number of distinct LB names; ids are ranks in byte-lexicographic (std::map) order */
    int32_t device;             /* CUDA device ordinal */
    int32_t reserved;
} brc_config;

/* Struct-of-arrays batch of decoded reads in file order == the bam1_t fields the path reads
 * (SURVEY.md §8a row a1).  Host pointers for brc_push_reads, device pointers for brc_run_device. */
typedef struct {
    int64_t n_reads;
    const int32_t *tid;         /* may be NULL (= region tid) ; reads with tid<0 are not admitted (V:sam.c:4488) */
    const int32_t *pos;         /* bam1_core_t.pos, 0-based */
    const uint16_t *flag;       /* bam1_core_t.flag */
    const uint8_t *mapq;        /* bam1_core_t.qual */
    const uint16_t *lib;        /* library id or BRC_LIB_NONE; may be NULL when !per_lib */
    const int32_t *l_qseq;      /* bam1_core_t.l_qseq */
    const int32_t *nm;          /* bam_aux2i(NM) or BRC_TAG_ABSENT */
    const int32_t *sm;          /* bam_aux2i(SM) or BRC_TAG_ABSENT */
    const uint64_t *cigar_off;  /* [n_reads+1] offsets into cigar */
    const uint32_t *cigar;      /* bam1_cigar(b): len<<4|op */
    const uint64_t *seq_off;    /* [n_reads+1] byte offsets into seq */
    const uint8_t *seq;         /* bam1_seq(b): 4-bit packed, (l_qseq+1)/2 bytes per read.  Device batches: pool base
                                 * 16-byte aligned with >= 16 readable bytes after the last read (bulk-TMA staging) */
    const uint64_t *qual_off;   /* [n_reads+1] byte offsets into qual */
    const uint8_t *qual;        /* bam1_qual(b); device batches: same alignment/padding rule as seq */
} brc_read_batch;

/* One region of the reference's loops: compute sites [beg-1, end), print [beg, end). */
typedef struct {
    int32_t tid;
    int32_t beg;                /* d.beg : 0-based first printed site */
    int32_t end;                /* d.end : exclusive */
    int32_t site_list_mode;     /* 1: -l loop (ref_len check R:...:144-148, queues cleared per region :605); 0: argv regions */
    int64_t read_lo, read_hi;   /* this region's reads inside the pushed stream */
    int64_t slot_base;          /* first result slot; slot = slot_base + (pos - (beg-1 clamped to >=0)) */
    int32_t first_pos;          /* max(beg-1,0) */
    int32_t n_slots;            /* end - first_pos */
} brc_region;

/* Result arrays (engine-owned, valid until the next brc_compute/brc_reset/brc_destroy).
 * Dense "slots": one per computed site per library row (row 0 = "all" when !per_lib);
 * index = row * n_slots + slot.  Every slot carries its PRIMARY key (the first passing base
 * class seen at the site) inline; further keys (other bases, indel alleles) are chained
 * through `sec_*` records starting at sec_head. */
typedef struct {
    int64_t n_regions;
    const brc_region *regions;
    int32_t n_rows;
    int64_t n_slots;
    const uint32_t *ncover;     /* reads spanning the site (before any filter) == pileup n for that library */
    const uint32_t *npass;      /* events passing mapq/baseq/flag filters (this row's share of mapq_n, R:...:312) */
    const uint8_t *flags;       /* bit0: a read without library spans the site (-p abandons it, R:...:281-284) */
    const uint8_t *pbase;       /* primary base class 0..5 or BRC_NO_BASE */
    const int32_t *sec_head;    /* first secondary record or -1 */
    const uint32_t *pstats;     /* [BRC_N_STATS][n_rows*n_slots] primary accumulators (floats as IEEE bits) */
    int64_t n_sec;
    const int32_t *sec_next;    /* next record of the same (row,slot) or -1 */
    const uint8_t *sec_kind;    /* 0..5 base class, BRC_KIND_INS, BRC_KIND_DEL */
    const int32_t *sec_len;     /* indel length (0 for bases) */
    const int64_t *sec_read;    /* representative read (index into the pushed stream) carrying the insertion bases */
    const int32_t *sec_qpos;    /* its qpos: inserted bases are read bases qpos+1 .. qpos+len */
    const uint32_t *sec_stats;  /* [BRC_N_STATS][n_sec] */
} brc_results;

/* PACKED results: what the kernels write and what crosses PCIe / NVLink (32 B per site instead of 66 B).
 * Per (row, slot) eight u32 words, stored struct-of-arrays as words[w][row * n_slots + slot]:
 *   W0  ncover[0:8) | npass[8:16) | count[16:24) | plus[24:32)                 (minus = count - plus)
 *   W1  primary base code [0:3): 0..5 = "=ACGTN", 6 = none, 7 = ESCAPED | bit 3: flags bit0 (read without library) |
 *       bit 4: the site has records in the secondary pool | nq2 [8:16) | sum_map_qualities [16:32)
 *   W2  sum_base_qualities [0:16) | sum_single_ended_map_qualities [16:32)
 *   W3  sum_of_clipped_lengths [0:16) | sum_of_mismatch_qualities [16:32)
 *   W4..W7  IEEE float32 bits of sum_event_location, sum_number_of_mismatches, sum_q2_distance, sum_3p_distance
 * A site whose counters do not fit (more than 255 spanning reads, a 16-bit sum overflowing) is ESCAPED: its words carry
 * only the flag bits and its full-width primary is a secondary-pool record of kind BRC_KIND_WIDE + base code.
 * Secondary-pool records (other base classes, indel alleles, escaped primaries), 72 bytes each, any order: */
#define BRC_N_WORDS 8
#define BRC_PB_NONE 6
#define BRC_PB_ESCAPE 7
#define BRC_KIND_WIDE 8           /* kinds 8..14: escaped primary with base code kind-8; then length = ncover, read = flags, qpos = npass */
typedef struct {
    uint32_t slot;                /* row * n_slots + slot */
    int32_t next;                 /* device-internal chain link (ignore) */
    uint32_t kind_len;            /* kind in bits [0:8), indel length in bits [8:32) */
    int32_t read;                 /* representative read (index into the pushed stream) carrying the insertion bases */
    int32_t qpos;                 /* its qpos: inserted bases are read bases qpos+1 .. qpos+len */
    uint32_t stats[BRC_N_STATS];
} brc_sec_record;
typedef struct {
    int64_t n_regions;
    const brc_region *regions;
    int32_t n_rows;
    int64_t n_slots;
    const uint32_t *words;        /* [BRC_N_WORDS][n_rows*n_slots] */
    int64_t n_sec;                /* host view: records in use; device view: pool capacity */
    const brc_sec_record *sec;
    const int32_t *sec_count;     /* device view only: the pool's live counter (device pointer); NULL in the host view */
} brc_packed_results;

/* ---- lifecycle ------------------------------------------------------------------------- */
BRC_API int brc_abi_version(void);
BRC_API int brc_create(const brc_config *cfg, brc_engine **out);
BRC_API void brc_destroy(brc_engine *e);
BRC_API const char *brc_last_error(const brc_engine *e);   /* text of the last failure on this handle ("" if none) */
BRC_API const char *brc_strerror(int status);

/* ---- reference window (load_reference, R:bamreadcount.cpp:83-90) ------------------------
 * seq[0] is position win_beg of contig tid; chrom_len is the full contig length (d.len).
 * The window must cover every base the region's reads and deletion alleles touch. */
BRC_API int brc_set_reference(brc_engine *e, int32_t tid, const char *contig_name, int64_t chrom_len, int64_t win_beg,
                      const char *seq, int64_t win_len);

/* Same, from a window that already sits in DEVICE memory as ASCII (a generator or a device-side decoder wrote it): the
 * encode kernel is enqueued on `stream` (a cudaStream_t), nothing is synchronised and no host copy is kept — the text
 * emitter (brc_format_*) refuses regions of that contig until brc_set_reference supplies the characters. */
BRC_API int brc_set_reference_device(brc_engine *e, int32_t tid, const char *contig_name, int64_t chrom_len, int64_t win_beg,
                             const char *dev_ascii, int64_t win_len, void *stream);

/* ---- region loop ----------------------------------------------------------------------- */
BRC_API int brc_reset(brc_engine *e);                      /* drop all pushed regions/reads and results */
BRC_API int brc_begin_region(brc_engine *e, int32_t tid, int32_t beg, int32_t end, int32_t site_list_mode);
/* one record, in file order: fetch_func(b) + bam_plbuf_push(b).  lib: id or BRC_LIB_NONE. */
BRC_API int brc_push_read(brc_engine *e, int32_t tid, int32_t pos, uint16_t flag, uint8_t mapq, uint16_t lib, int32_t l_qseq,
                  int32_t nm, int32_t sm, uint32_t n_cigar, const uint32_t *cigar, const uint8_t *seq,
                  const uint8_t *qual);
/* Bulk form of brc_push_read.  When the batch is the only data pushed since brc_reset and every record is admitted
 * as is (mapped, on the region's contig, position-sorted, fewer records than max_cnt), the engine BORROWS the arrays
 * instead of copying them: they must stay valid and unmodified until brc_compute returns, and brc_compute DMAs
 * straight out of them (page-lock them for full PCIe bandwidth).  Otherwise records are copied one by one. */
BRC_API int brc_push_reads(brc_engine *e, const brc_read_batch *batch);
BRC_API int brc_end_region(brc_engine *e);

/* ---- f-2: BAM records straight from the file's BGZF blocks, inflated and framed ON THE DEVICE -------------------------
 * (V:htslib-1.10/bgzf.c:697,897 inflate_block / bgzf_read_block; V:htslib-1.10/sam.c:598-659 bam_read1.)  Only the COMPRESSED
 * bytes cross PCIe.  `comp` holds consecutive whole BGZF blocks; `entry` lists record starts the index knows inside them
 * (BAI linear-index / bin-chunk virtual offsets are starts of real records), each encoded as
 * (byte offset of its block inside comp) << 16 | offset inside that block's inflated data, ascending, entry[0] = the first
 * record wanted.  Every entry starts an independent chain of block_size hops, so framing needs no guessing.  Records whose
 * refID differs from `tid` are kept but never admitted.  Read groups: rg_id[i] -> rg_lib[i] (library rank or BRC_LIB_NONE).
 * The -d max-count rule is not evaluated on this path (use brc_push_read when -d is smaller than the region's read count). */
typedef struct {
    const uint8_t *comp;
    int64_t comp_len;
    int64_t n_entry;
    const uint64_t *entry;
    int64_t end_voff;             /* records starting at or after it are not decoded (same encoding); < 0: to the end of the span */
    int32_t tid;
    int32_t n_rg;
    const char *const *rg_id;
    const uint16_t *rg_lib;
} brc_bam_span;
/* decode only: the batch (DEVICE pointers, engine-owned until the next decode) a caller can hand to brc_run_device */
BRC_API int brc_decode_bam_span(brc_engine *e, const brc_bam_span *span, brc_read_batch *dev_batch_out, void *stream);
/* region loop form: the span is the open region's read stream (instead of brc_push_read(s)); brc_compute then runs on it */
BRC_API int brc_push_bam_span(brc_engine *e, const brc_bam_span *span);
/* test / debug: the decoded batch copied to engine-owned HOST memory */
BRC_API int brc_fetch_decoded_batch(brc_engine *e, brc_read_batch *host_out);

/* Runs the GPU path over everything pushed since brc_reset: H2D, per-read precompute kernel,
 * pileup/accumulate kernel, D2H.  Reads not admitted by the pileup buffer (tid<0, FUNMAP,
 * the -d rule of V:htslib-1.10/sam.c:4491) are dropped on the host while batching. */
BRC_API int brc_compute(brc_engine *e);
BRC_API int brc_get_results(brc_engine *e, brc_results *out);      /* full-width view, expanded from the packed records on first use */
BRC_API int brc_get_packed_results(brc_engine *e, brc_packed_results *out);   /* the records as they came off the device (pinned host memory) */
/* counts of the reference's per-event warnings: [0]=SM_TAG_MISSING [1]=NM_TAG_MISSING
 * [2]=Zm_TAG_MISSING (always 0) [3]=LIBRARY_UNAVAILABLE (R:src/lib/bamrc/ReadWarnings.hpp:12-18) */
BRC_API int brc_get_warning_counts(brc_engine *e, int64_t out[4]);

/* Text of the reference's STDOUT for region `region_index` (all regions if -1), formatted
 * exactly as R:bamreadcount.cpp:351-416 + R:BasicStat.cpp:110-159.  lib_names: n_libs strings.
 * Returns the number of bytes required (excluding NUL); writes at most cap-1 bytes + NUL. */
BRC_API int64_t brc_format_text(brc_engine *e, int64_t region_index, const char *const *lib_names, char *buf, int64_t cap);

/* The deletion queue of the reference's argv-region loop is never cleared between regions (R:bamreadcount.cpp:650-656; its -l
 * loop clears it per line, :605).  By default every brc_format_* / brc_write_text call starts with an empty queue, so all argv
 * regions of a run must be formatted in one call.  With carry ON the queue left by one formatting pass (all regions, or the
 * windows of one region in order) is the starting queue of the next — across brc_reset / brc_compute — so a caller can flush
 * argv regions batch by batch.  Switching it (on or off) empties the queue. */
BRC_API int brc_set_queue_carry(brc_engine *e, int on);

/* Same, for a window of one region's sites: slot offsets [first, first+count) inside region `region_index` (site
 * first_pos+first onwards).  Lets a caller stream the text of a large region piecewise; the window's first site
 * re-derives its deletion columns from the site to its left.  Formatting runs on several host threads. */
BRC_API int64_t brc_format_window(brc_engine *e, int64_t region_index, int64_t first, int64_t count, const char *const *lib_names,
                                  char *buf, int64_t cap);

/* Same text written straight to a file descriptor (no intermediate copy).  region_index < 0: every region (first/count
 * ignored); otherwise the window [first, first+count) of that region (count < 0: to its end).  Returns bytes written. */
BRC_API int64_t brc_write_text(brc_engine *e, int64_t region_index, int64_t first, int64_t count, const char *const *lib_names, int fd);

/* ---- alternative-allele site filter ----------------------------------------------------------
 * Prints only the lines a user would keep when looking for non-reference alleles: a line is printed iff one of its allele
 * entries (any library block with -p) is an ALTERNATIVE allele whose count c satisfies c >= min_alt_count and
 * c >= min_alt_fraction * depth (IEEE double; depth = the line's 4th column).  Alternative alleles: every insertion (+...)
 * and deletion (-...) entry printed on the line, and an A/C/G/T entry whose seq_nt16 code differs from the reference base's
 * (a reference N, IUPAC code or missing character makes all four alternative; case is ignored).  "=" and "N" never are.
 * The reference base is the one the text prints: for a contig set only with brc_set_reference_device that is N.
 * Every printed line is byte-identical to the line the unfiltered run prints for that site; the filter only removes lines.
 *
 * The sites are selected on the device right after the pileup kernels (brc_compute, brc_run_device) and only the selected
 * sites' records are copied to the host.  While a filter is set there is no dense view: brc_get_results and
 * brc_get_packed_results return BRC_E_INVALID; brc_get_selected_results is the sparse view. */
typedef struct {
    int32_t min_alt_count;        /* >= 1 */
    int32_t reserved;             /* 0 */
    double min_alt_fraction;      /* in [0, 1] */
} brc_site_filter;
/* f == NULL turns the filter off (the unfiltered path, exactly as without this call); takes effect at the next brc_compute /
 * brc_run_device.  Out-of-range values: BRC_E_INVALID. */
BRC_API int brc_set_site_filter(brc_engine *e, const brc_site_filter *f);
/* Bounds on an alternative allele's statistics, for filters in the style of false-positive filters (one-strand alleles,
 * read-end alleles, low base quality ...).  With bounds, the entry that makes a line pass must also satisfy every bound that
 * is set: lo[k] <= value (bit k of lo_set) and value <= hi[k] (bit k of hi_set), k = BRC_S_*.  The value is the field as the
 * line prints it, in hundredths: an integer field (count, strand counts, Q2 reads) times 100; an average the two decimals the
 * line prints (so avg_basequality of an indel entry is 0, as is the Q2 distance of an entry without Q2 reads).  A deletion is
 * judged on the line where it prints (p+1). */
typedef struct {
    uint32_t lo_set, hi_set;      /* bit k: lo[k] / hi[k] is a bound; bits 13..31 are 0 */
    int64_t lo[BRC_N_STATS];      /* hundredths, >= 0 */
    int64_t hi[BRC_N_STATS];      /* hundredths, >= 0, and >= lo[k] when both are set */
} brc_entry_bounds;
/* brc_set_site_filter with bounds.  b == NULL is exactly brc_set_site_filter(e, f); f == NULL with bounds, a mask bit past
 * bit 12, a negative bound or lo > hi on one field: BRC_E_INVALID.  brc_set_site_filter clears the bounds. */
BRC_API int brc_set_site_filter_bounds(brc_engine *e, const brc_site_filter *f, const brc_entry_bounds *b);
/* Sparse host view of a filtered run: the shipped sites (global slot ids, ascending) with their emit byte
 *   1: the line passes the filter   2: shipped for the deletion queue (a range whose lines may carry deletions queued by an
 *      earlier region, or the last site of an argv region that forms a line and that a library row covers); the emitter forms
 *      the line and evaluates the rule on it   0: context only (the left neighbour of a site with emit byte 1 or 2: its
 *      deletions print on that line)
 * their packed words [BRC_N_WORDS][n_rows * n_sites] (the packed layout with n_sites columns) and their secondary-pool
 * records, whose slot is row * n_sites + index into site[]. */
typedef struct {
    int64_t n_regions;
    const brc_region *regions;
    int32_t n_rows;
    int64_t n_slots;              /* dense slots of the batch (site[] indexes them) */
    int64_t n_sites;
    const uint32_t *site;
    const uint8_t *emit;
    const uint32_t *words;
    int64_t n_sec;
    const brc_sec_record *sec;
} brc_selected_results;
BRC_API int brc_get_selected_results(brc_engine *e, brc_selected_results *out);

/* ---- allele queries ---------------------------------------------------------------------------
 * "The read counts of THESE alleles at THESE sites" (a VCF's REF and ALT alleles, DESIGN.md §12), answered on the device from
 * the packed records the kernels left in HBM: only the answers (64 B each), the warning words and the pool counter cross PCIe.
 *
 * One query names an entry of one printed line:
 *   region     index of the region in brc_begin_region order since brc_reset (or in the brc_plan_device table)
 *   pos        0-based site of that region that the text would print (beg <= pos < end)
 *   kind_len   kind in bits [0:8): 0..5 a base entry of "=ACGTN" (length 0), BRC_KIND_INS or BRC_KIND_DEL with the indel
 *              length (>= 1) in bits [8:32)
 *   bases_off  BRC_KIND_INS: offset of its `length` upper-case A/C/G/T/N characters in the `bases` buffer (the "+..." entry's
 *              characters: read bases as the text prints them, IUPAC codes read as N); ignored otherwise
 * Its answer:
 *   stats      the entry's 13 accumulators (floats as IEEE bits), exactly what brc_get_results holds for that key; all zeros
 *              when the line has no such entry
 *   depth      the line's 4th column;  line  1 when the site prints a line (0: no read spans it; stats and depth are 0)
 * A deletion entry prints on the line after its anchor: a BRC_KIND_DEL query at `pos` is answered from the deletion of that
 * length anchored at pos - 1, when the anchor lies in the same region (the -l loop's view; at most one deletion of a length
 * starts at one anchor, so the length names it).
 *
 * Queries belong to the current batch: set them after the last brc_end_region (or brc_plan_device) and before brc_compute /
 * brc_run_device; brc_reset, brc_begin_region and brc_plan_device drop them.  While they are set there is no dense view:
 * brc_get_results, brc_get_packed_results and brc_format_* return BRC_E_INVALID.  brc_run_device leaves the answers on the
 * device and brc_fetch_device_results copies them.  BRC_E_INVALID: per_lib (more than one library row), a site filter set, a
 * region or position out of range, an unknown kind, insertion bases that are not A/C/G/T/N or lie outside `bases`. */
typedef struct {
    int64_t region;
    int32_t pos;
    uint32_t kind_len;
    int64_t bases_off;
} brc_allele_query;
typedef struct {
    uint32_t stats[BRC_N_STATS];
    uint32_t depth;
    uint32_t line;
    uint32_t reserved;            /* 0 */
} brc_allele_answer;              /* 64 B */
BRC_API int brc_set_allele_queries(brc_engine *e, const brc_allele_query *q, int64_t n, const char *bases, int64_t n_bases);
/* the answers of the last run, in query order (engine-owned, valid until the next run or brc_reset) */
BRC_API int brc_get_allele_answers(brc_engine *e, const brc_allele_answer **out, int64_t *n);

/* ---- complex-record queries (DESIGN.md §12 "MNP and complex records") ----------------------
 * A query counts the reads of one record whose span is reference positions [pos, pos + ref_len) by their bases between the
 * two flanks pos - 1 and pos + ref_len:
 *   region     as brc_allele_query;  pos  0-based first span base, a site of that region (beg <= pos < end), >= 1
 *   ref_len    >= 1;  n_alleles  >= 1: its alleles are the next n_alleles entries of `a`, in query order
 * An allele is >= 1 upper-case A/C/G/T/N characters at bases[bases_off .. bases_off + len).
 * A read counts when it is not dropped by -q or the flag filter, both flanks are aligned to read bases by M, = or X ops, and
 * every read base strictly between them (inserted bases included) has quality >= -b.  Its string S is those bases, IUPAC
 * codes read as N.  Answers: depth[i] = the reads that count for query i; counts[j] = those whose S equals allele j exactly,
 * and how many of them are on the forward strand.  A right flank past the contig's end gives 0.  -i has no effect.
 * Same lifecycle as the allele queries, and both may be set for one batch (each is answered as it would be alone); the
 * results are BRC_RESULTS_ANSWERS.  BRC_E_INVALID: per_lib, a site filter set, a region or position out of range, pos < 1,
 * ref_len < 1, n_alleles < 1, allele counts that do not add up to n_alleles, allele bases that are not A/C/G/T/N or lie
 * outside `bases`. */
typedef struct { int64_t region; int32_t pos; int32_t ref_len; int32_t n_alleles; int32_t reserved; } brc_complex_query;
typedef struct { int64_t bases_off; int32_t len; int32_t reserved; } brc_complex_allele;
BRC_API int brc_set_complex_queries(brc_engine *e, const brc_complex_query *q, int64_t n, const brc_complex_allele *a,
                                    int64_t n_alleles, const char *bases, int64_t n_bases);
typedef struct { uint32_t count, plus; } brc_complex_count;        /* minus = count - plus */
/* the answers of the last run: depth[n] in query order, counts[n_alleles] in allele order (engine-owned, valid until the next
 * run or brc_reset) */
BRC_API int brc_get_complex_answers(brc_engine *e, const uint32_t **depth, const brc_complex_count **counts, int64_t *n,
                                    int64_t *n_alleles);

/* ---- device-resident path (bench "value": inputs already in HBM) -------------------------
 * brc_plan_device: fix the region geometry (host array of n_regions regions with read_lo/hi,
 * slot_base, first_pos, n_slots filled) and size the outputs.  brc_run_device: launch the
 * kernels on `stream` (a cudaStream_t) over a batch whose pointers are DEVICE pointers and the
 * reference window set by brc_set_reference; results stay on the device.  brc_device_packed_results
 * returns DEVICE pointers to the packed records (what a multi-GPU run sends over NCCL for the ordered
 * emit).  brc_fetch_device_results copies them to the host arrays brc_get_results /
 * brc_get_packed_results expose. */
BRC_API int brc_plan_device(brc_engine *e, const brc_region *regions, int64_t n_regions, int64_t n_reads_cap,
                    int64_t n_sec_cap);
BRC_API int brc_run_device(brc_engine *e, const brc_read_batch *dev_batch, const int32_t *dev_region_of_read, void *stream);
BRC_API int brc_device_packed_results(brc_engine *e, brc_packed_results *out);
BRC_API int brc_fetch_device_results(brc_engine *e, void *stream);
/* Self-test of the kernels' exact-arithmetic shortcuts (reciprocal division, float<->double bit casts, the quotient tables)
 * against the IEEE intrinsics for every divisor 1..max_b; returns the number of mismatches (0 = ok). */
BRC_API int64_t brc_selftest_fastmath(brc_engine *e, int32_t max_b);
/* Rows d_lo..d_hi (1 <= d_lo <= d_hi <= 2048) of the device's quotient tables, which the pileup kernels read in place of divisions
 * (brc_device.cuh QTAB_*): 4096 entries per row, entry c of row d being, with j = c - 2048,
 *   q: RN((float)|j| / (float)d)    p: 1.0 - (double)RN((float)|2 j - d| / (float)d).
 * Copies (d_hi - d_lo + 1) * 4096 floats to `q` and as many doubles to `p`; returns that count or a negative status. */
BRC_API int64_t brc_get_quotient_rows(brc_engine *e, int32_t d_lo, int32_t d_hi, float *q, double *p);
/* The packed reference window of contig `tid` as the kernels read it: seq_nt16 codes, two per byte, first base in the high
 * nibble, then 0xFF padding (win_len / 2 + 32 bytes in all).  Waits for the device, copies min(cap, that size) bytes to `out`
 * and returns the full size, or a negative status (BRC_E_NO_REFERENCE when the contig has none). */
BRC_API int64_t brc_get_reference_codes(brc_engine *e, int32_t tid, uint8_t *out, int64_t cap);
/* The per-read work of the last brc_run_device/brc_compute as the pileup kernels read it (debug view): the read descriptors K0
 * wrote (80 bytes each, brc_device.cuh ReadDesc) and the first / one-past-last read index of every tile.  Waits for the device,
 * copies min(desc_cap, n_reads) descriptors to `desc` and min(tile_cap, n_tiles) entries to `tile_lo` / `tile_hi`, stores n_tiles
 * in *n_tiles and returns n_reads, or a negative status (BRC_E_INVALID before any run). */
BRC_API int64_t brc_get_read_descriptors(brc_engine *e, void *desc, int64_t desc_cap, int32_t *tile_lo, int32_t *tile_hi, int64_t tile_cap,
                                         int64_t *n_tiles);
/* kernels launched by the last brc_run_device/brc_compute (for bench.py's gpu_launches) */
/* Page-locked host memory for batches handed to brc_push_reads (a borrowed batch is DMA'd straight out of the caller's arrays:
 * from pageable memory the copies are staged and synchronous).  cudaHostAlloc / cudaFreeHost behind plain pointers, so that a host
 * written against this header does not need the CUDA runtime.  BRC_E_NO_DEVICE without a usable device. */
BRC_API int brc_host_alloc(size_t bytes, void **out);
BRC_API void brc_host_free(void *p);

BRC_API int brc_last_launch_count(const brc_engine *e);
/* which view the host holds of the last run: BRC_RESULTS_DENSE (brc_get_results, brc_get_packed_results), BRC_RESULTS_SELECTED
 * (brc_get_selected_results: a site filter was set when it was launched), BRC_RESULTS_ANSWERS (brc_get_allele_answers and
 * brc_get_complex_answers: allele or complex queries were set), or BRC_RESULTS_NONE (nothing fetched since the last brc_reset,
 * brc_begin_region, brc_plan_device or brc_run_device; brc_set_allele_queries and brc_set_complex_queries drop earlier
 * answers) */
enum { BRC_RESULTS_NONE = 0, BRC_RESULTS_DENSE = 1, BRC_RESULTS_SELECTED = 2, BRC_RESULTS_ANSWERS = 3 };
BRC_API int brc_last_results_kind(const brc_engine *e);
/* bytes the last brc_compute() of pushed host reads copied host->device (regular offset arrays and constant columns of
 * fixed-length reads are rebuilt on the device and do not count) */
BRC_API int64_t brc_last_h2d_bytes(const brc_engine *e);
/* elapsed GPU milliseconds of the named stage of the last run, measured with CUDA events on the
 * launching stream: 0 = per-read precompute kernel, 1 = pileup kernel, 2 = whole device step (without the selection),
 * 3 = site selection + compaction (0 when no filter was set), 4 = allele queries (0 when none were set), 5 = the complex-record
 * kernel, without the upload of its queries (0 when none were set) */
BRC_API float brc_last_stage_ms(const brc_engine *e, int stage);

/* ---- BGZF output, compressed on the device (DESIGN.md §13) ----------------------------------
 * A writer turns the bytes given to brc_bgzf_write into a BGZF file on `fd` as htslib writes one: members of 65280 input bytes
 * (the last one shorter), each the smallest of a dynamic-Huffman, fixed-Huffman or stored DEFLATE stream, then the 28-byte
 * empty EOF member.  The bytes written depend only on the byte stream, not on how it was split into calls.  No engine handle:
 * the writer uses the device current at brc_bgzf_open (brc_set_device chooses it) on its own stream; each call makes that device
 * current and restores the caller's.  It stages the stream in page-locked memory and compresses a chunk of members on the
 * device while the caller produces the next one; members reach `fd` in order.
 * A failed write() (EPIPE, ENOSPC, ...) or CUDA failure is returned by the next call and by brc_bgzf_close.  Not thread-safe. */
typedef struct brc_bgzf_writer brc_bgzf_writer;
/* makes `device` current on the calling thread (cudaSetDevice), so that a host built without the CUDA runtime opens its writer
 * on the device its engines use (brc_config.device); BRC_E_NO_DEVICE when that is not a usable device */
BRC_API int brc_set_device(int device);
BRC_API int brc_bgzf_open(int fd, brc_bgzf_writer **out);           /* BRC_E_NO_DEVICE without a usable device */
BRC_API int brc_bgzf_write(brc_bgzf_writer *w, const void *buf, size_t n);   /* BRC_E_IO: errno is set to the write's */
/* flush, the EOF member, free (fd stays open); the first failure seen, if any (BRC_E_IO: errno is set to the write's) */
BRC_API int brc_bgzf_close(brc_bgzf_writer *w);
/* bytes taken, compressed bytes written, and GPU milliseconds of the chunks' kernels (CUDA events), so far */
BRC_API int brc_bgzf_stats(const brc_bgzf_writer *w, int64_t *bytes_in, int64_t *bytes_out, double *kernel_ms);
/* brc_write_text's text handed to a BGZF writer instead of a file descriptor (the formatted parts go straight into its staging).
 * Returns the bytes of text, or a negative status (the writer's, when it failed). */
BRC_API int64_t brc_write_text_bgzf(brc_engine *e, int64_t region_index, int64_t first, int64_t count, const char *const *lib_names,
                                    brc_bgzf_writer *w);

#ifdef __cplusplus
}
#endif
#endif /* BRC_ENGINE_H */
