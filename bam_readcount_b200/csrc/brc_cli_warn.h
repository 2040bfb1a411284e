// brc_cli_warn.h — brc-readcount's per-read warning lines.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "brc_cli_input.h"

namespace brc::cli {

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
    using Cand = WarnCand;
    struct Reg { int tid, beg, end; bool skip_halo; size_t c0, c1; };
    long long max_per_type; bool unlimited; int min_mapq, min_bq; bool per_lib, ic;
    long long counts[NT] = {0, 0, 0, 0};
    std::vector<Cand> cands; std::vector<Reg> regs;
    FILE *err = stderr;           // the sample's message stream
    Warner(long long mw, int q, int b, bool p, bool i) : max_per_type(mw < 0 ? 1000 : mw), unlimited(mw < 0), min_mapq(q), min_bq(b), per_lib(p), ic(i) {}
    bool budget_left() const { return counts[SM] < max_per_type || counts[NM] < max_per_type || (per_lib && counts[LIB] < max_per_type); }
    bool collecting() const { return max_per_type > 0 && budget_left(); }
    void begin_region(int tid, int beg, int end, bool skip_halo) { regs.push_back({tid, beg, end, skip_halo, cands.size(), cands.size()}); }
    // a record that can warn at all (no NM tag, proper pair without SM tag, or `lib` == BRC_LIB_NONE) becomes `c`
    static bool candidate(const Rec &r, uint16_t lib, Cand &c) {
        const bool no_nm = r.nm == BRC_TAG_ABSENT, no_sm = (r.flag & 2) && r.sm == BRC_TAG_ABSENT, no_lib = lib == (uint16_t)BRC_LIB_NONE;
        if (!no_nm && !no_sm && !no_lib) return false;
        c.pos = r.pos; c.endpos = rec_endpos(r); c.flag = r.flag; c.mapq = r.mapq; c.no_nm = no_nm; c.no_sm = no_sm; c.no_lib = no_lib;
        c.cigar.assign(r.cigar, r.cigar + r.n_cigar); c.qual.assign(r.qual, r.qual + r.l_qseq);
        c.qname = (const char *)(r.data.data() + 32);
        return true;
    }
    // a record of the record stream, in file order
    void consider(const Rec &r, uint16_t lib) {
        if (!collecting() || (r.flag & 4) || regs.empty()) return;
        Cand c;
        if (!candidate(r, lib, c)) return;
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
        for (; k < n; ++k) {
            op = c.cigar[k] & 0xF; len = (int)(c.cigar[k] >> 4);
            if (cigar_consumes_ref(op)) { if (site < x + len) break; x += len; if (cigar_is_match(op)) y += len; }
            else if (op == 1 || op == 4) y += len;
        }
        indel = 0;
        if (k >= n) return false;
        const bool is_del = !cigar_is_match(op);
        qpos = is_del ? y : y + (int)(site - x);
        if (x + len - 1 == site && k + 1 < n) {
            const uint32_t op2 = c.cigar[k + 1] & 0xF; const int l2 = (int)(c.cigar[k + 1] >> 4);
            if (op2 == 2) indel = -l2;
            else if (op2 == 1) indel = l2;
            else if (op2 == 6) { int l3 = 0; for (size_t m = k + 2; m < n; ++m) { const uint32_t o3 = c.cigar[m] & 0xF; if (o3 == 1) l3 += (int)(c.cigar[m] >> 4); else if (cigar_consumes_ref(o3)) break; } if (l3 > 0) indel = l3; }
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

}  // namespace brc::cli
