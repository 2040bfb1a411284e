/*
 * brc_oracle.c — TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * A plain-C, single-threaded CPU restatement of bam-readcount's per-position pileup
 * hot path, used only as the checker for the CUDA engine (tests/, __graft_entry__.smoke(),
 * bench.py's cpu_baseline leg).  The product (bam_readcount_b200/) never links, imports
 * or executes this file.
 *
 * Parity status: PINNED.  tests/test_oracle_golden.py checks this restatement byte-for-byte
 * against the reference's four golden files (test-data/expected_*) and, where oracle/_ref
 * (the unmodified reference binary built by oracle/build_ref.sh) is present, against the
 * reference binary on synthetic BAMs with deletions / -q / -b / -d / -p / -i.
 *
 * It deliberately follows the reference's control flow (a live-read list advanced position
 * by position, an incremental CIGAR cursor, a per-library deletion FIFO), i.e. it is NOT
 * the stateless site-centric formulation the GPU kernels use.  Each function cites the
 * reference lines it restates:
 *   R: = /root/reference/...                       (first-party bam-readcount, c7c76e6)
 *   V: = vendor/samtools-1.10.tar.bz2 : samtools-1.10/...   (htslib 1.10 pileup engine)
 */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>

#define ORC_TAG_ABSENT INT32_MIN
#define ORC_LIB_NONE 0xFFFFu

/* ---- inputs (flat, caller-owned) ------------------------------------------------------ */
typedef struct {
    int64_t n_reads;
    const int32_t *tid;        /* per read */
    const int32_t *pos;        /* 0-based leftmost */
    const uint16_t *flag;
    const uint8_t *mapq;
    const uint16_t *lib;       /* dense library id in byte-lexicographic LB order, ORC_LIB_NONE = no RG/LB */
    const int32_t *l_qseq;
    const int32_t *nm;         /* NM:i value or ORC_TAG_ABSENT */
    const int32_t *sm;         /* SM:i value or ORC_TAG_ABSENT */
    const uint64_t *cigar_off; /* n_reads+1 offsets into cigar[] (uint32 BAM encoding len<<4|op) */
    const uint32_t *cigar;
    const uint64_t *seq_off;   /* n_reads+1 byte offsets into seq[] (BAM 4-bit packing, (l+1)/2 bytes per read) */
    const uint8_t *seq;
    const uint64_t *qual_off;  /* n_reads+1 byte offsets into qual[] */
    const uint8_t *qual;
} orc_reads;

typedef struct {
    int32_t min_mapq, min_bq, max_cnt, per_lib, insertion_centric, n_libs;
    const char *const *lib_names; /* n_libs names (for text) */
} orc_config;

typedef struct {
    int32_t tid;
    const char *name;     /* contig name for text output */
    int64_t chrom_len;    /* d.len */
    int64_t win_beg;      /* seq[0] is reference position win_beg */
    int64_t win_len;
    const char *seq;      /* raw FASTA characters (case preserved) */
} orc_ref;

/* ---- growable text buffer --------------------------------------------------------------- */
typedef struct { char *s; size_t n, cap; } orc_buf;
static void buf_put(orc_buf *b, const char *p, size_t n) {
    if (b->n + n + 1 > b->cap) {
        size_t c = b->cap ? b->cap * 2 : 4096;
        while (c < b->n + n + 1) c *= 2;
        b->s = (char *)realloc(b->s, c); b->cap = c;
    }
    memcpy(b->s + b->n, p, n); b->n += n; b->s[b->n] = 0;
}
static void buf_puts(orc_buf *b, const char *p) { buf_put(b, p, strlen(p)); }
static void buf_printf(orc_buf *b, const char *fmt, double v) { char t[64]; int n = snprintf(t, sizeof t, fmt, v); buf_put(b, t, (size_t)n); }
static void buf_u(orc_buf *b, unsigned long long v) { char t[32]; int n = snprintf(t, sizeof t, "%llu", v); buf_put(b, t, (size_t)n); }
static void buf_i(orc_buf *b, long long v) { char t[32]; int n = snprintf(t, sizeof t, "%lld", v); buf_put(b, t, (size_t)n); }

/* ---- BasicStat  (R:src/lib/bamrc/BasicStat.hpp:12-27) ----------------------------------- */
typedef struct {
    uint32_t read_count, sum_map_qualities, sum_single_ended_map_qualities, num_plus_strand, num_minus_strand;
    float sum_event_location, sum_q2_distance;
    uint32_t num_q2_reads;
    float sum_number_of_mismatches;
    uint32_t sum_of_mismatch_qualities, sum_of_clipped_lengths;
    float sum_3p_distance;
    uint32_t sum_base_qualities;
    int is_indel;
} orc_stat;

/* per-read values of fetch_func (R:src/lib/bamrc/auxfields.hpp:6-11) */
typedef struct { int32_t mmq, clipped_length, left_clip, three_prime_index, q2_pos; } orc_zm;

/* htslib tables (V:htslib-1.10/hts.c:73-91 seq_nt16_table; R:bamreadcount.cpp:34-39) */
static uint8_t nt16_of_ascii(unsigned char c) {
    switch (c) {
    case '=': return 0;
    case 'A': case 'a': return 1;  case 'C': case 'c': return 2;  case 'M': case 'm': return 3;
    case 'G': case 'g': return 4;  case 'R': case 'r': return 5;  case 'S': case 's': return 6;
    case 'V': case 'v': return 7;  case 'T': case 't': return 8;  case 'W': case 'w': return 9;
    case 'Y': case 'y': return 10; case 'H': case 'h': return 11; case 'K': case 'k': return 12;
    case 'D': case 'd': return 13; case 'B': case 'b': return 14;
    default: return 15;
    }
}
/* htslib's table also maps the digits '0'..'3' to 1,2,4,8 (V:htslib-1.10/hts.c:77) */
static uint8_t seq_nt16(unsigned char c) {
    if (c == '0') return 1; if (c == '1') return 2; if (c == '2') return 4; if (c == '3') return 8;
    return nt16_of_ascii(c);
}
static const uint8_t canonical16[16] = {0, 1, 2, 5, 3, 5, 5, 5, 4, 5, 5, 5, 5, 5, 5, 5};
static const char canonical_nt[] = "=ACGTN";

static inline int seqi(const uint8_t *s, int64_t i) { return (s[i >> 1] >> ((~i & 1) << 2)) & 0xf; }

static inline char ref_at(const orc_ref *r, int64_t p) {
    /* the reference holds the whole chromosome as a NUL-terminated string; p == len reads the NUL */
    if (p < 0 || p >= r->chrom_len) return 0;
    if (p < r->win_beg || p >= r->win_beg + r->win_len) return 'N'; /* outside the supplied window: caller's contract violation */
    return r->seq[p - r->win_beg];
}

/* ---- fetch_func: per-read values (R:src/exe/bam-readcount/bamreadcount.cpp:114-253) ----- */
static orc_zm fetch_values(const orc_reads *R, int64_t i, const orc_ref *ref, int ref_len_check) {
    const uint32_t *cig = R->cigar + R->cigar_off[i];
    int n_cigar = (int)(R->cigar_off[i + 1] - R->cigar_off[i]);
    const uint8_t *seq = R->seq + R->seq_off[i];
    const uint8_t *qual = R->qual + R->qual_off[i];
    int l_qseq = R->l_qseq[i];
    uint32_t sum_mmq = 0;
    int left_clip = 0, clipped_length = l_qseq, right_clip = l_qseq;
    int last_mm_pos = -1, last_mm_qual = 0;
    int64_t reference_position = R->pos[i];
    int read_position = 0;
    for (int k = 0; k < n_cigar; ++k) {
        int op_length = (int)(cig[k] >> 4), op = (int)(cig[k] & 0xf);
        if (op == 0) { /* BAM_CMATCH only; '=' and 'X' fall through untouched (R:...:138) */
            int j;
            for (j = 0; j < op_length; j++) {
                int cur = read_position + j;
                int read_base = seqi(seq, cur);
                int64_t refpos = reference_position + j;
                if (ref_len_check && refpos > ref->chrom_len) continue;   /* R:...:144-148 (site-list mode only) */
                char rc = ref_at(ref, refpos);
                int ref_base = seq_nt16((unsigned char)rc);
                if (rc == 0) break;                                        /* R:...:151 */
                if (read_base != ref_base && ref_base != 15 && read_base != 0) {
                    int q = qual[cur];
                    if (last_mm_pos != -1) {
                        if (last_mm_pos + 1 != cur) { sum_mmq += (uint32_t)last_mm_qual; last_mm_qual = q; last_mm_pos = cur; }
                        else { if (last_mm_qual < q) last_mm_qual = q; last_mm_pos = cur; }
                    } else { last_mm_pos = cur; last_mm_qual = q; }
                }
            }
            if (j < op_length) break;                                      /* R:...:175 */
            reference_position += op_length; read_position += op_length;
        } else if (op == 2 || op == 3) { reference_position += op_length;  /* D, N */
        } else if (op == 1) { read_position += op_length;                  /* I */
        } else if (op == 4) {                                              /* S */
            read_position += op_length; clipped_length -= op_length;
            if (k == 0) left_clip += op_length; else right_clip -= op_length;
        }
    }
    sum_mmq += (uint32_t)last_mm_qual;                                     /* R:...:199 */
    int tpi, q2_pos = -1, kk, inc;
    int reverse = R->flag[i] & 16;
    if (reverse) { kk = tpi = 0; inc = 1; if (tpi < left_clip) tpi = left_clip; }
    else { kk = tpi = l_qseq - 1; inc = -1; if (tpi > right_clip) tpi = right_clip; }
    while (q2_pos < 0 && kk >= 0 && kk < l_qseq) {                         /* R:...:222-228 */
        if (qual[kk] != 2) { q2_pos = kk - 1; break; }
        kk += inc;
    }
    if (reverse) { if (tpi < q2_pos) tpi = q2_pos; }
    else { if (tpi > q2_pos && q2_pos != -1) tpi = q2_pos; }
    orc_zm z; z.mmq = (int32_t)sum_mmq; z.clipped_length = clipped_length; z.left_clip = left_clip;
    z.three_prime_index = tpi; z.q2_pos = q2_pos;
    return z;
}

/* bam_endpos / bam_cigar2rlen (V:htslib-1.10/sam.c:497-513) */
static int64_t read_endpos(const orc_reads *R, int64_t i) {
    const uint32_t *cig = R->cigar + R->cigar_off[i];
    int n_cigar = (int)(R->cigar_off[i + 1] - R->cigar_off[i]);
    if (!(R->flag[i] & 4) && n_cigar > 0) {
        int64_t l = 0;
        for (int k = 0; k < n_cigar; ++k) { int op = cig[k] & 0xf; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) l += cig[k] >> 4; }
        return R->pos[i] + l;
    }
    return (int64_t)R->pos[i] + 1;
}

/* fetch_values and read_endpos of reads [lo, hi), one reference (tests: the read descriptors of the engine's K0).
 * out_zm: 5 int32 per read in orc_zm order; out_end: one int64 per read. */
void orc_read_values(const orc_ref *ref, const orc_reads *R, int64_t lo, int64_t hi, int ref_len_check, int32_t *out_zm,
                     int64_t *out_end) {
    for (int64_t i = lo; i < hi; ++i) {
        orc_zm z = fetch_values(R, i, ref, ref_len_check);
        memcpy(out_zm + 5 * (i - lo), &z, sizeof z);
        out_end[i - lo] = read_endpos(R, i);
    }
}

/* ---- live list node + incremental CIGAR cursor (V:htslib-1.10/sam.c:3904-3918) ---------- */
typedef struct { int64_t read; int64_t beg, end; int k, y; int64_t x; orc_zm zm; } orc_node;
typedef struct { int qpos, indel, is_del, is_refskip; } orc_plp;

static int is_refop(int op) { return op == 0 || op == 2 || op == 3 || op == 7 || op == 8; }
static int is_matchop(int op) { return op == 0 || op == 7 || op == 8; }

/* resolve_cigar2 (V:htslib-1.10/sam.c:3964-4041) */
static void resolve_cigar(const orc_reads *R, orc_node *nd, int64_t pos, orc_plp *p) {
    const uint32_t *cigar = R->cigar + R->cigar_off[nd->read];
    int n_cigar = (int)(R->cigar_off[nd->read + 1] - R->cigar_off[nd->read]);
    int k;
    if (nd->k == -1) {
        p->qpos = 0;
        if (n_cigar == 1) {
            if (is_matchop(cigar[0] & 0xf)) { nd->k = 0; nd->x = R->pos[nd->read]; nd->y = 0; }
        } else {
            nd->x = R->pos[nd->read]; nd->y = 0;
            for (k = 0; k < n_cigar; ++k) {
                int op = cigar[k] & 0xf, l = (int)(cigar[k] >> 4);
                if (is_refop(op)) break;
                else if (op == 1 || op == 4) nd->y += l;
            }
            nd->k = k;
        }
    } else {
        int op, l = (int)(cigar[nd->k] >> 4);
        if (pos - nd->x >= l) {
            op = cigar[nd->k + 1] & 0xf;
            if (is_refop(op)) {
                if (is_matchop(cigar[nd->k] & 0xf)) nd->y += l;
                nd->x += l; ++nd->k;
            } else {
                if (is_matchop(cigar[nd->k] & 0xf)) nd->y += l;
                nd->x += l;
                for (k = nd->k + 1; k < n_cigar; ++k) {
                    op = cigar[k] & 0xf; l = (int)(cigar[k] >> 4);
                    if (is_refop(op)) break;
                    else if (op == 1 || op == 4) nd->y += l;
                }
                nd->k = k;
            }
        }
    }
    {
        int op = cigar[nd->k] & 0xf, l = (int)(cigar[nd->k] >> 4);
        p->is_del = p->indel = p->is_refskip = 0;
        if (nd->x + l - 1 == pos && nd->k + 1 < n_cigar) {
            int op2 = cigar[nd->k + 1] & 0xf, l2 = (int)(cigar[nd->k + 1] >> 4);
            if (op2 == 2) p->indel = -l2;
            else if (op2 == 1) p->indel = l2;
            else if (op2 == 6 && nd->k + 2 < n_cigar) {
                int l3 = 0;
                for (k = nd->k + 2; k < n_cigar; ++k) {
                    op2 = cigar[k] & 0xf; l2 = (int)(cigar[k] >> 4);
                    if (op2 == 1) l3 += l2;
                    else if (op2 == 2 || op2 == 0 || op2 == 3 || op2 == 7 || op2 == 8) break;
                }
                if (l3 > 0) p->indel = l3;
            }
        }
        if (is_matchop(op)) p->qpos = nd->y + (int)(pos - nd->x);
        else if (op == 2 || op == 3) { p->is_del = 1; p->qpos = nd->y; p->is_refskip = (op == 3); }
    }
}

/* ---- BasicStat::process_read (R:src/lib/bamrc/BasicStat.cpp:28-107) --------------------- */
typedef struct { int64_t sm_missing, nm_missing, lib_unavailable; } orc_warn;

static void process_read(orc_stat *s, const orc_reads *R, const orc_node *nd, const orc_plp *p, orc_warn *w) {
    int64_t i = nd->read;
    int l_qseq = R->l_qseq[i];
    s->read_count++;
    s->sum_map_qualities += R->mapq[i];
    if (R->flag[i] & 16) s->num_minus_strand++; else s->num_plus_strand++;
    const orc_zm *z = &nd->zm;
    s->sum_of_mismatch_qualities += (uint32_t)z->mmq;
    if (z->q2_pos > -1) {
        s->sum_q2_distance += (float)abs(p->qpos - z->q2_pos) / (float)l_qseq;
        s->num_q2_reads++;
    }
    s->sum_3p_distance += (float)abs(p->qpos - z->three_prime_index) / (float)l_qseq;
    s->sum_of_clipped_lengths += (uint32_t)z->clipped_length;
    float read_center = (float)((float)z->clipped_length / 2.0);
    /* float += double expression: the add happens in double, then rounds to float */
    s->sum_event_location = (float)((double)s->sum_event_location +
                                    (1.0 - (double)(fabsf((float)(p->qpos - z->left_clip) - read_center) / read_center)));
    if (R->flag[i] & 2) {
        if (R->sm[i] != ORC_TAG_ABSENT) s->sum_single_ended_map_qualities += (uint32_t)R->sm[i];
        else w->sm_missing++;
    } else s->sum_single_ended_map_qualities += R->mapq[i];
    if (R->nm[i] != ORC_TAG_ABSENT) s->sum_number_of_mismatches += (float)R->nm[i] / (float)z->clipped_length;
    else w->nm_missing++;
    if (!s->is_indel) s->sum_base_qualities += (R->qual + R->qual_off[i])[p->qpos];
}

/* operator<<(BasicStat) (R:src/lib/bamrc/BasicStat.cpp:110-159) */
static void print_stat(orc_buf *b, const orc_stat *s) {
    buf_u(b, s->read_count); buf_puts(b, ":");
    if (s->read_count > 0) {
        float rc = (float)s->read_count;
        buf_printf(b, "%.2f:", (double)((float)s->sum_map_qualities / rc));
        if (s->is_indel) buf_puts(b, "0.00:"); else buf_printf(b, "%.2f:", (double)((float)s->sum_base_qualities / rc));
        buf_printf(b, "%.2f:", (double)((float)s->sum_single_ended_map_qualities / rc));
        buf_u(b, s->num_plus_strand); buf_puts(b, ":"); buf_u(b, s->num_minus_strand); buf_puts(b, ":");
        buf_printf(b, "%.2f:", (double)(s->sum_event_location / rc));
        buf_printf(b, "%.2f:", (double)(s->sum_number_of_mismatches / rc));
        buf_printf(b, "%.2f:", (double)((float)s->sum_of_mismatch_qualities / rc));
        buf_u(b, s->num_q2_reads); buf_puts(b, ":");
        if (s->num_q2_reads > 0) buf_printf(b, "%.2f:", (double)(s->sum_q2_distance / (float)s->num_q2_reads));
        else buf_puts(b, "0.00:");
        buf_printf(b, "%.2f:", (double)((float)s->sum_of_clipped_lengths / rc));
        buf_printf(b, "%.2f", (double)(s->sum_3p_distance / rc));
    } else buf_puts(b, "0.00:0.00:0.00:0:0:0.00:0.00:0.00:0:0.00:0.00:0.00");
}

/* raw accumulator dump: exact comparison against the GPU engine's binary results */
static uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
static void dump_stat(orc_buf *b, const orc_stat *s) {
    char t[256];
    int n = snprintf(t, sizeof t, "%u %u %u %u %u %u %08x %08x %u %u %08x %u %08x",
                     s->read_count, s->sum_map_qualities, s->sum_base_qualities, s->sum_single_ended_map_qualities,
                     s->num_plus_strand, s->num_minus_strand, fbits(s->sum_event_location), fbits(s->sum_number_of_mismatches),
                     s->sum_of_mismatch_qualities, s->num_q2_reads, fbits(s->sum_q2_distance), s->sum_of_clipped_lengths,
                     fbits(s->sum_3p_distance));
    buf_put(b, t, (size_t)n);
}

/* ---- per-site containers (R:bamreadcount.cpp:46-50 LibraryCounts) ----------------------- */
typedef struct { char *allele; int len; orc_stat st; } orc_indel;
typedef struct { int present; int64_t ncover; orc_stat base[6]; orc_indel *indel; int n_indel, cap_indel; } orc_libcounts;

static int allele_cmp(const char *a, int la, const char *b, int lb) { /* std::string operator< */
    int m = la < lb ? la : lb; int c = memcmp(a, b, (size_t)m);
    if (c) return c; return la - lb;
}
static orc_stat *indel_slot(orc_libcounts *lc, const char *allele, int len) {
    for (int i = 0; i < lc->n_indel; ++i)
        if (lc->indel[i].len == len && memcmp(lc->indel[i].allele, allele, (size_t)len) == 0) return &lc->indel[i].st;
    if (lc->n_indel == lc->cap_indel) { lc->cap_indel = lc->cap_indel ? lc->cap_indel * 2 : 4; lc->indel = (orc_indel *)realloc(lc->indel, sizeof(orc_indel) * (size_t)lc->cap_indel); }
    orc_indel *e = &lc->indel[lc->n_indel++];
    e->allele = (char *)malloc((size_t)len + 1); memcpy(e->allele, allele, (size_t)len); e->allele[len] = 0; e->len = len;
    memset(&e->st, 0, sizeof e->st);
    return &e->st;
}
static int indel_order(const void *a, const void *b) {
    const orc_indel *x = (const orc_indel *)a, *y = (const orc_indel *)b;
    return allele_cmp(x->allele, x->len, y->allele, y->len);
}

/* ---- IndelQueue (R:src/lib/bamrc/IndelQueue.cpp:3-15, IndelQueueEntry.hpp:8-15) ---------- */
typedef struct { uint32_t tid, pos; orc_stat st; char *allele; int len; } orc_qent;
typedef struct { orc_qent *e; int head, n, cap; } orc_queue;
typedef struct {
    orc_queue *q;   /* one per library row (row 0 = "all" when !per_lib) */
    int *q_exists;  /* indel_queue_map has an entry for this library (R:...:394 creates it on first push) */
    int n_rows;
    orc_buf text;   /* reference STDOUT text */
    orc_buf dump;   /* raw accumulators of every computed site */
    orc_warn warn;
    int64_t n_lines;
} orc_ctx;

orc_ctx *orc_ctx_new(int n_rows) {
    orc_ctx *c = (orc_ctx *)calloc(1, sizeof *c);
    c->n_rows = n_rows < 1 ? 1 : n_rows;
    c->q = (orc_queue *)calloc((size_t)c->n_rows, sizeof(orc_queue));
    c->q_exists = (int *)calloc((size_t)c->n_rows, sizeof(int));
    return c;
}
/* d.indel_queue_map.clear() (R:bamreadcount.cpp:605) — the site-list loop calls this per region, the argv loop never */
void orc_ctx_clear_queues(orc_ctx *c) {
    for (int r = 0; r < c->n_rows; ++r) {
        orc_queue *q = &c->q[r];
        for (int i = q->head; i < q->head + q->n; ++i) free(q->e[i].allele);
        q->head = q->n = 0; c->q_exists[r] = 0;
    }
}
void orc_ctx_free(orc_ctx *c) {
    orc_ctx_clear_queues(c);
    for (int r = 0; r < c->n_rows; ++r) free(c->q[r].e);
    free(c->q); free(c->q_exists); free(c->text.s); free(c->dump.s); free(c);
}
const char *orc_ctx_text(orc_ctx *c) { return c->text.s ? c->text.s : ""; }
const char *orc_ctx_dump(orc_ctx *c) { return c->dump.s ? c->dump.s : ""; }
int64_t orc_ctx_text_len(orc_ctx *c) { return (int64_t)c->text.n; }
int64_t orc_ctx_dump_len(orc_ctx *c) { return (int64_t)c->dump.n; }
void orc_ctx_reset_output(orc_ctx *c) { c->text.n = 0; c->dump.n = 0; if (c->text.s) c->text.s[0] = 0; if (c->dump.s) c->dump.s[0] = 0; }
void orc_ctx_warnings(orc_ctx *c, int64_t *out3) { out3[0] = c->warn.sm_missing; out3[1] = c->warn.nm_missing; out3[2] = c->warn.lib_unavailable; }
int64_t orc_ctx_lines(orc_ctx *c) { return c->n_lines; }

static void queue_push(orc_queue *q, uint32_t tid, uint32_t pos, const orc_stat *st, const char *allele, int len) {
    if (q->head + q->n == q->cap) {
        if (q->head > 0) { memmove(q->e, q->e + q->head, sizeof(orc_qent) * (size_t)q->n); q->head = 0; }
        else { q->cap = q->cap ? q->cap * 2 : 8; q->e = (orc_qent *)realloc(q->e, sizeof(orc_qent) * (size_t)q->cap); }
    }
    orc_qent *e = &q->e[q->head + q->n++];
    e->tid = tid; e->pos = pos; e->st = *st; e->len = len;
    e->allele = (char *)malloc((size_t)len + 1); memcpy(e->allele, allele, (size_t)len); e->allele[len] = 0;
}
static int queue_process(orc_queue *q, uint32_t tid, uint32_t pos, orc_buf *rec, orc_buf *dump, int row) {
    int extra = 0;
    while (q->n && ((q->e[q->head].tid == tid && q->e[q->head].pos < pos) || q->e[q->head].tid != tid)) { free(q->e[q->head].allele); q->head++; q->n--; }
    while (q->n && q->e[q->head].tid == tid && q->e[q->head].pos == pos) {
        orc_qent *e = &q->e[q->head];
        buf_puts(rec, "\t"); buf_put(rec, e->allele, (size_t)e->len); buf_puts(rec, ":"); print_stat(rec, &e->st);
        if (dump) { buf_puts(dump, "Q "); buf_i(dump, row); buf_puts(dump, " "); buf_put(dump, e->allele, (size_t)e->len); buf_puts(dump, " "); dump_stat(dump, &e->st); buf_puts(dump, "\n"); }
        extra += (int)e->st.read_count;
        free(e->allele); q->head++; q->n--;
    }
    if (q->n == 0) q->head = 0;
    return extra;
}

/* ---- pileup_func (R:src/exe/bam-readcount/bamreadcount.cpp:265-419) --------------------- */
static void pileup_site(orc_ctx *C, const orc_config *cfg, const orc_ref *ref, const orc_reads *R,
                        int32_t tid, int64_t pos, int n, orc_node **nodes, const orc_plp *pl,
                        int64_t beg, int64_t end) {
    if (!(pos >= beg - 1 && pos < end)) return;                            /* R:...:269 */
    int n_rows = C->n_rows;
    orc_libcounts *lc = (orc_libcounts *)calloc((size_t)n_rows, sizeof *lc);
    int mapq_n = 0, abandoned = 0;
    for (int i = 0; i < n && !abandoned; ++i) {
        const orc_node *nd = nodes[i]; const orc_plp *p = &pl[i]; int64_t r = nd->read;
        int row = 0;
        if (cfg->per_lib) {
            if (R->lib[r] == ORC_LIB_NONE || R->lib[r] >= (unsigned)n_rows) { C->warn.lib_unavailable++; abandoned = 1; break; } /* R:...:281-284 */
            row = R->lib[r];
        }
        orc_libcounts *cur = &lc[row]; cur->present = 1; cur->ncover++;     /* R:...:286 */
        const uint8_t *qual = R->qual + R->qual_off[r]; const uint8_t *seq = R->seq + R->seq_off[r];
        if (!p->is_del && R->mapq[r] >= cfg->min_mapq && qual[p->qpos] >= cfg->min_bq) {
            if (R->flag[r] & (4 | 256 | 512 | 1024)) continue;               /* R:...:295-310 */
            mapq_n++;
            if (p->indel != 0) {                                           /* R:...:315-342 (ref is always loaded here) */
                int len = p->indel > 0 ? p->indel : -p->indel;
                char *allele = (char *)malloc((size_t)len + 2);
                if (p->indel > 0) {
                    allele[0] = '+';
                    for (int k = 0; k < len; ++k) allele[1 + k] = canonical_nt[canonical16[seqi(seq, p->qpos + 1 + k)]];
                } else {
                    allele[0] = '-';
                    for (int k = 0; k < len; ++k) { char c = ref_at(ref, pos + k + 1); allele[1 + k] = c ? c : 'N'; }
                }
                orc_stat *st = indel_slot(cur, allele, len + 1);
                st->is_indel = 1; process_read(st, R, nd, p, &C->warn);
                free(allele);
            }
            if (p->indel < 1 || !cfg->insertion_centric) {                  /* R:...:343-346 */
                int c = canonical16[seqi(seq, p->qpos)];
                process_read(&cur->base[c], R, nd, p, &C->warn);
            }
        }
    }
    if (!abandoned) {
        orc_buf rec = {0, 0, 0};
        int extra_depth = 0;
        /* raw dump header for this computed site */
        buf_puts(&C->dump, "S "); buf_i(&C->dump, tid); buf_puts(&C->dump, " "); buf_i(&C->dump, pos); buf_puts(&C->dump, " "); buf_i(&C->dump, n);
        buf_puts(&C->dump, " "); buf_i(&C->dump, mapq_n); buf_puts(&C->dump, "\n");
        for (int row = 0; row < n_rows; ++row) {                           /* std::map order == library id order */
            orc_libcounts *cur = &lc[row];
            if (!cur->present) continue;
            buf_puts(&C->dump, "L "); buf_i(&C->dump, row); buf_puts(&C->dump, " "); buf_i(&C->dump, cur->ncover); buf_puts(&C->dump, "\n");
            if (cfg->per_lib) { buf_puts(&rec, "\t"); buf_puts(&rec, cfg->lib_names[row]); buf_puts(&rec, "\t{"); }
            for (int j = 0; j < 6; ++j) {
                char t[3] = {'\t', canonical_nt[j], ':'}; buf_put(&rec, t, 3); print_stat(&rec, &cur->base[j]);
                if (cur->base[j].read_count) { buf_puts(&C->dump, "K "); buf_i(&C->dump, row); char a[3] = {' ', canonical_nt[j], ' '}; buf_put(&C->dump, a, 3); dump_stat(&C->dump, &cur->base[j]); buf_puts(&C->dump, "\n"); }
            }
            if (cur->n_indel > 1) qsort(cur->indel, (size_t)cur->n_indel, sizeof(orc_indel), indel_order);
            for (int k = 0; k < cur->n_indel; ++k) {
                orc_indel *e = &cur->indel[k];
                buf_puts(&C->dump, "K "); buf_i(&C->dump, row); buf_puts(&C->dump, " "); buf_put(&C->dump, e->allele, (size_t)e->len); buf_puts(&C->dump, " "); dump_stat(&C->dump, &e->st); buf_puts(&C->dump, "\n");
                if (e->allele[0] == '-') { queue_push(&C->q[row], (uint32_t)tid, (uint32_t)(pos + 1), &e->st, e->allele, e->len); C->q_exists[row] = 1; }
                else { buf_puts(&rec, "\t"); buf_put(&rec, e->allele, (size_t)e->len); buf_puts(&rec, ":"); print_stat(&rec, &e->st); }
            }
            if (C->q_exists[row]) extra_depth += queue_process(&C->q[row], (uint32_t)tid, (uint32_t)pos, &rec, &C->dump, row);
            if (cfg->per_lib) buf_puts(&rec, "\t}");
        }
        if (pos >= beg && pos < end) {                                     /* R:...:414-416 */
            char rb = (pos < ref->chrom_len) ? ref_at(ref, pos) : 'N';
            buf_puts(&C->text, ref->name); buf_puts(&C->text, "\t"); buf_i(&C->text, pos + 1); buf_puts(&C->text, "\t");
            buf_put(&C->text, &rb, 1); buf_puts(&C->text, "\t"); buf_i(&C->text, mapq_n + extra_depth);
            if (rec.s) buf_put(&C->text, rec.s, rec.n);
            buf_puts(&C->text, "\n");
            C->n_lines++;
        }
        buf_puts(&C->dump, "D "); buf_i(&C->dump, mapq_n + extra_depth); buf_puts(&C->dump, "\n");
        free(rec.s);
    } else {
        buf_puts(&C->dump, "A "); buf_i(&C->dump, tid); buf_puts(&C->dump, " "); buf_i(&C->dump, pos); buf_puts(&C->dump, "\n");
    }
    for (int row = 0; row < n_rows; ++row) { for (int k = 0; k < lc[row].n_indel; ++k) free(lc[row].indel[k].allele); free(lc[row].indel); }
    free(lc);
}

/* ---- one region: fetch_func + bam_plbuf_push per read, then the EOF flush ----------------
 * (R:bamreadcount.cpp:591-604 / 650-656; V:bam_plbuf.c:59-69; V:htslib-1.10/sam.c:4416-4531)
 * The caller supplies, in file order, the records the index iterator would yield for
 * [beg-1, end) (V:htslib-1.10/hts.c:3229-3236).  Returns the number of admitted reads.      */
int64_t orc_region(orc_ctx *C, const orc_config *cfg, const orc_ref *ref, const orc_reads *R,
                   int64_t read_lo, int64_t read_hi, int32_t tid, int64_t beg, int64_t end, int ref_len_check) {
    int64_t cap = read_hi - read_lo + 1, n_live = 0, admitted = 0;
    orc_node *pool = (orc_node *)malloc(sizeof(orc_node) * (size_t)cap);
    orc_node **live = (orc_node **)malloc(sizeof(orc_node *) * (size_t)cap);
    orc_node **plp_nodes = (orc_node **)malloc(sizeof(orc_node *) * (size_t)cap);
    orc_plp *plp = (orc_plp *)malloc(sizeof(orc_plp) * (size_t)cap);
    int64_t n_pool = 0;
    /* iterator state (V:htslib-1.10/sam.c:4230-4245 bam_plp_init: tid=pos=0, max_tid=max_pos=-1) */
    int32_t it_tid = 0, max_tid = -1; int64_t it_pos = 0, max_pos = -1; int is_eof = 0;
    for (int64_t i = read_lo; i <= read_hi; ++i) {
        int pushed_any = 0;
        if (i < read_hi) {
            orc_zm zm = fetch_values(R, i, ref, ref_len_check);             /* fetch_func runs for every yielded record */
            if (R->tid[i] < 0 || (R->flag[i] & 4)) continue;               /* V:sam.c:4488-4490 */
            /* mp->cnt counts live nodes plus the tail sentinel (V:sam.c:3941, 4491) */
            if (it_tid == R->tid[i] && it_pos == R->pos[i] && (n_live + 1) > (int64_t)cfg->max_cnt) continue;
            int64_t e = read_endpos(R, i);
            max_tid = R->tid[i]; max_pos = R->pos[i];
            if (e > it_pos || R->tid[i] > it_tid) {
                orc_node *nd = &pool[n_pool++];
                nd->read = i; nd->beg = R->pos[i]; nd->end = e; nd->k = -1; nd->y = 0; nd->x = 0; nd->zm = zm;
                live[n_live++] = nd; admitted++;
            }
            pushed_any = 1;
        } else { is_eof = 1; pushed_any = 1; }
        if (!pushed_any) continue;
        /* drain: bam_plp64_next loop (V:htslib-1.10/sam.c:4416-4466) */
        for (;;) {
            if (is_eof && n_live == 0) break;
            if (!(is_eof || max_tid > it_tid || (max_tid == it_tid && max_pos > it_pos))) break;
            int n_plp = 0; int64_t w = 0;
            for (int64_t j = 0; j < n_live; ++j) {
                orc_node *nd = live[j];
                int32_t ntid = R->tid[nd->read];
                if (ntid < it_tid || (ntid == it_tid && nd->end <= it_pos)) continue; /* retire */
                if (ntid == it_tid && nd->beg <= it_pos) { plp_nodes[n_plp] = nd; resolve_cigar(R, nd, it_pos, &plp[n_plp]); n_plp++; }
                live[w++] = nd;
            }
            n_live = w;
            int32_t cb_tid = it_tid; int64_t cb_pos = it_pos;
            if (n_live > 0) {
                int32_t htid = R->tid[live[0]->read];
                if (it_tid < htid) { it_tid = htid; it_pos = live[0]->beg; }
                else if (it_pos < live[0]->beg) it_pos = live[0]->beg;
                else ++it_pos;
            } else ++it_pos; /* head==tail: htslib compares against the stale sentinel; with sorted input this only advances */
            if (n_plp) pileup_site(C, cfg, ref, R, cb_tid, cb_pos, n_plp, plp_nodes, plp, beg, end);
            if (is_eof && n_live == 0) break;
        }
    }
    free(pool); free(live); free(plp_nodes); free(plp);
    return admitted;
}
