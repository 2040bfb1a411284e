// brc_aux.cuh — what a BAM record's aux fields say about NM, SM, RG and a long CIGAR: one rule set for every BAM decoder here
// (bam_extract_kernel of brc_bgzf.cu on the device, read_record of brc_cli.cpp on the host; bamio.read_bam restates it in Python).
//
// The rules are htslib 1.10's, which the reference binary reads records with:
//   bam_aux_get   walks the tags in order and returns the FIRST one named; the walk stops (every later tag is absent) at a value
//                 that cannot be skipped: an unknown type, a B array of unknown subtype, a fixed-size or B value cut by the end of
//                 the record.  Types and sizes: A c C 1, s S 2, i I f 4, d 8, Z H up to a NUL (or the record end), B subtype+count.
//                 A wanted tag whose own value cannot be skipped is absent too, and so is a wanted Z or H without its NUL.
//   bam_aux2i     c C s S i I give their value; any other type is still a PRESENT tag, worth 0 (V:htslib-1.10/sam.c:3662-3683).
//   bam_get_library  the first RG tag decides, whatever its type: the ID is the bytes from its value up to a NUL (V:bam.c:77-89).
//                 For Z and H that is the string; for another type it is the value's raw bytes, which in practice name no @RG.
//   bam_tag2cigar a record on a contig whose first CIGAR op is <l_qseq>S and whose first CG tag is B:I with a count in
//                 [n_cigar, 2^29) carries its real CIGAR in that array (samtools writes this for reads of more than 65535 ops).
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define BRC_AUX_HD __host__ __device__ __forceinline__
#else
#define BRC_AUX_HD inline
#endif

namespace brc {
namespace aux {

struct RecAux {
    int32_t nm, sm;              // bam_aux2i of the first NM / SM, or INT32_MIN (BRC_TAG_ABSENT) when absent
    int64_t rg_o, rg_len;        // ID bytes of the first RG tag (offset in the record body, length); rg_o < 0: no RG tag
    int64_t cig_o;               // offset of the real CIGAR in the record body (the CIGAR field, or the CG array)
    uint32_t n_cigar;            // its op count
};

BRC_AUX_HD uint32_t ld32(const uint8_t *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }

// bytes of one element of a fixed-size type; 0 = not a fixed-size type
BRC_AUX_HD int64_t fixed_size(uint8_t t) {
    switch (t) {
    case 'A': case 'c': case 'C': return 1;
    case 's': case 'S': return 2;
    case 'i': case 'I': case 'f': return 4;
    case 'd': return 8;
    default: return 0;
    }
}

// the offset just past the value whose type byte is at d[o] (o < end), or -1 when it cannot be skipped (skip_aux's NULL)
BRC_AUX_HD int64_t skip(const uint8_t *d, int64_t o, int64_t end) {
    const uint8_t t = d[o++];
    if (t == 'Z' || t == 'H') { while (o < end && d[o]) ++o; return o < end ? o + 1 : end; }
    if (t == 'B') {
        if (end - o < 5) return -1;
        const int64_t es = fixed_size(d[o]);
        const int64_t n = ld32(d + o + 1);
        o += 5;
        if (es == 0 || end - o < es * n) return -1;
        return o + es * n;
    }
    const int64_t sz = fixed_size(t);
    if (sz == 0 || end - o < sz) return -1;
    return o + sz;
}

// bam_aux2i of the value whose type byte is at d[o], as the int32_t the reference stores it in
BRC_AUX_HD int32_t to_int(const uint8_t *d, int64_t o) {
    const uint8_t *v = d + o + 1;
    switch (d[o]) {
    case 'c': return (int8_t)v[0];
    case 'C': return v[0];
    case 's': return (int16_t)(v[0] | (v[1] << 8));
    case 'S': return v[0] | (v[1] << 8);
    case 'i': case 'I': return (int32_t)ld32(v);
    default: return 0;
    }
}

// d: record body (after block_size), bs: its length; aux_o: where the tags start; cig_o / n_cigar: the CIGAR field
BRC_AUX_HD RecAux scan(const uint8_t *d, int64_t bs, int64_t aux_o, int64_t cig_o, uint32_t n_cigar) {
    RecAux r{INT32_MIN, INT32_MIN, -1, 0, cig_o, n_cigar};
    bool got_nm = false, got_sm = false, got_rg = false, got_cg = false;
    int64_t cg = -1;                                             // type byte of the first CG tag
    for (int64_t o = aux_o; bs - o >= 3;) {
        const uint8_t a = d[o], b = d[o + 1];
        o += 2;
        const int64_t e = skip(d, o, bs);
        const bool cut = e < 0 || ((d[o] == 'Z' || d[o] == 'H') && d[e - 1] != 0);    // a wanted Z/H needs its NUL
        if (a == 'N' && b == 'M' && !got_nm) { got_nm = true; if (!cut) r.nm = to_int(d, o); }
        else if (a == 'S' && b == 'M' && !got_sm) { got_sm = true; if (!cut) r.sm = to_int(d, o); }
        else if (a == 'R' && b == 'G' && !got_rg) {
            got_rg = true;
            if (!cut) { int64_t z = o + 1; while (z < bs && d[z]) ++z; r.rg_o = o + 1; r.rg_len = z - (o + 1); }
        } else if (a == 'C' && b == 'G' && !got_cg) { got_cg = true; if (!cut) cg = o; }
        if (e < 0) break;
        o = e;
    }
    const int32_t tid = (int32_t)ld32(d), pos = (int32_t)ld32(d + 4), l_qseq = (int32_t)ld32(d + 16);
    if (cg >= 0 && d[cg] == 'B' && d[cg + 1] == 'I' && n_cigar > 0 && tid >= 0 && pos >= 0) {   // a skippable B value has 5 more bytes
        const uint32_t c0 = ld32(d + cig_o), cnt = ld32(d + cg + 2);
        if ((c0 & 15u) == 4u && (c0 >> 4) == (uint32_t)l_qseq && cnt >= n_cigar && cnt < (1u << 29)) { r.cig_o = cg + 6; r.n_cigar = cnt; }
    }
    return r;
}

}  // namespace aux
}  // namespace brc
