// brc_format.cpp — host text emitter: turns the engine's binary per-site records into the
// reference's STDOUT lines.
//
//   line assembly + deletion queue   R:src/exe/bam-readcount/bamreadcount.cpp:351-416
//   BasicStat printer                R:src/lib/bamrc/BasicStat.cpp:110-159
//   IndelQueue::process              R:src/lib/bamrc/IndelQueue.cpp:3-15
//
// Only formatting, ordering of allele strings and the p -> p+1 deletion shift live here; every
// number printed was accumulated on the GPU.  Averages are float32 divisions printed exactly like
// `std::fixed << setprecision(2)` == printf("%.2f", (double)f): `put_f2` rounds the exact binary value
// half-to-even in integer arithmetic (no printf in the hot path); a region is formatted by several
// threads over disjoint site ranges — the deletion shift only needs the site to the left, which each
// thread re-derives for its first site.
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <deque>
#include <string>
#include <vector>

#include <unistd.h>

#include "brc_engine_internal.h"
#include "brc_fmt_num.h"

namespace {

struct Stat { uint32_t v[BRC_N_STATS]; };
inline float f32(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }

using brc::put_u;
using brc::put_f2;

// operator<<(std::ostream&, const BasicStat&)
void put_stat(std::string &o, const Stat *s, bool is_indel) {
    if (!s || s->v[BRC_S_COUNT] == 0) { o += "0:0.00:0.00:0.00:0:0:0.00:0.00:0.00:0:0.00:0.00:0.00"; return; }
    const uint32_t *v = s->v;
    const float rc = (float)v[BRC_S_COUNT];
    put_u(o, v[BRC_S_COUNT]); o += ':';
    put_f2(o, (float)v[BRC_S_MAPQ] / rc); o += ':';
    if (is_indel) o += "0.00"; else put_f2(o, (float)v[BRC_S_BASEQ] / rc);
    o += ':';
    put_f2(o, (float)v[BRC_S_SE_MAPQ] / rc); o += ':';
    put_u(o, v[BRC_S_PLUS]); o += ':'; put_u(o, v[BRC_S_MINUS]); o += ':';
    put_f2(o, f32(v[BRC_S_POS_FRAC]) / rc); o += ':';
    put_f2(o, f32(v[BRC_S_NM_FRAC]) / rc); o += ':';
    put_f2(o, (float)v[BRC_S_MMQS] / rc); o += ':';
    put_u(o, v[BRC_S_NQ2]); o += ':';
    if (v[BRC_S_NQ2] > 0) put_f2(o, f32(v[BRC_S_Q2_DIST]) / (float)v[BRC_S_NQ2]); else o += "0.00";
    o += ':';
    put_f2(o, (float)v[BRC_S_CLIP_LEN] / rc); o += ':';
    put_f2(o, f32(v[BRC_S_3P_DIST]) / rc);
}

using brc::QEnt;
using brc::EmitState;
inline QEnt make_qent(int32_t tid, int64_t pos, const Stat &st, const std::string &allele) {
    QEnt q; q.tid = tid; q.pos = pos; std::memcpy(q.st, st.v, sizeof q.st); q.allele = allele; return q;
}
inline const Stat *qstat(const QEnt &q) { return reinterpret_cast<const Stat *>(q.st); }

const char kNt[] = "=ACGTN";
const uint8_t kCanon[16] = {0, 1, 2, 5, 3, 5, 5, 5, 4, 5, 5, 5, 5, 5, 5, 5};

struct View {   // raw result arrays of one engine
    const brc_engine *e; const brc_region *rg; const brc::HostRef *ref;
    int rows; int64_t NS, RS, SC;
    const uint32_t *ncover, *npass, *pstats, *sstats; const uint8_t *flags, *pbase, *skind;
    const int32_t *shead, *snext, *slen, *sqpos; const int64_t *sread;
    // site filter: the arrays hold only the shipped sites (column i = site csite[i], emit byte cemit[i]); null when dense
    const uint32_t *csite = nullptr; const uint8_t *cemit = nullptr; int64_t n_sel = 0;
    View(const brc_engine *en, int64_t g) : e(en), rg(&en->regions[(size_t)g]), ref(brc::find_ref(en, rg->tid)) {
        const brc_engine::Wide &W = e->wide;            // full-width view of the packed device records (brc::ensure_wide)
        rows = e->n_rows; NS = e->result_cols(); RS = (int64_t)rows * NS; SC = (int64_t)W.sec_next.size();
        if (e->sparse) { csite = e->sel_site(); cemit = e->sel_emit(); n_sel = e->n_sel; }
        ncover = W.ncover.data(); npass = W.npass.data(); pstats = W.pstats.data(); sstats = W.sec_stats.data();
        flags = W.flags.data(); pbase = W.pbase.data(); skind = W.sec_kind.data();
        shead = W.sec_head.data(); snext = W.sec_next.data(); slen = W.sec_len.data(); sqpos = W.sec_qpos.data();
        sread = W.sec_read.data();
    }
};

struct Indel { std::string allele; Stat st; };
struct Scratch { std::string rec; std::vector<Indel> indels; };

// seq_nt16 code of a reference character (1/2/4/8 for one base; 15 for N, IUPAC codes and anything else)
inline uint32_t nt16(char c) {
    switch (c) { case 'A': case 'a': return 1; case 'C': case 'c': return 2; case 'G': case 'g': return 4; case 'T': case 't': return 8; default: return 15; }
}

// One site: pileup_func's print section.  emit=false only replays the deletion pushes (used to seed a thread's first site).
// `slot` is the site's column in the result arrays (dense: rg.slot_base + s; sparse: its index among the shipped sites).  With
// a site filter the line is printed only when the filter's rule holds on it (brc::site_passes, the device selection's rule).
void format_site(const View &V, int32_t s, int64_t slot, const char *const *lib_names, EmitState &st, std::string &out, Scratch &W, bool emit) {
    const brc_region &rg = *V.rg;
    const int rows = V.rows; const int64_t NS = V.NS;
    const int64_t pos = (int64_t)rg.first_pos + s;
    uint64_t n_total = 0, mapq_n = 0; bool abandoned = false;
    for (int r = 0; r < rows; ++r) { n_total += V.ncover[r * NS + slot]; mapq_n += V.npass[r * NS + slot]; abandoned |= (V.flags[r * NS + slot] & 1) != 0; }
    if (n_total == 0 || abandoned) return;   // no callback / -p with a read lacking a library: `return 0` before anything is kept
    std::string &rec = W.rec; rec.clear();
    int64_t extra_depth = 0;
    char rb = 'N';
    if (emit && V.ref && pos < V.ref->chrom_len && pos >= V.ref->win_beg && pos < V.ref->win_beg + (int64_t)V.ref->seq.size()) rb = V.ref->seq[(size_t)(pos - V.ref->win_beg)];   // a device-only reference window (brc_set_reference_device) has no characters here
    const bool gate = emit && V.csite;
    const uint32_t rcode = gate ? nt16(rb) : 15u;
    uint64_t best_alt = 0;
    for (int r = 0; r < rows; ++r) {
        const int64_t idx = r * NS + slot;
        if (V.ncover[idx] == 0) continue;
        if (emit && V.e->cfg.per_lib) { rec += '\t'; rec += lib_names ? lib_names[r] : "?"; rec += "\t{"; }
        Stat base[6]; bool have[6] = {false, false, false, false, false, false};
        W.indels.clear();
        if (V.pbase[idx] < 6) { for (int k = 0; k < BRC_N_STATS; ++k) base[V.pbase[idx]].v[k] = V.pstats[(int64_t)k * V.RS + idx]; have[V.pbase[idx]] = true; }
        for (int32_t j = V.shead[idx]; j >= 0; j = V.snext[j]) {
            Stat t; for (int k = 0; k < BRC_N_STATS; ++k) t.v[k] = V.sstats[(int64_t)k * V.SC + j];
            if (V.skind[j] < 6) { base[V.skind[j]] = t; have[V.skind[j]] = true; continue; }
            Indel in; in.st = t;
            if (V.skind[j] == BRC_KIND_INS) {          // "+" + canonicalised read bases qpos+1..qpos+len  (R:...:324-330)
                in.allele = "+";
                const uint8_t *sq = V.e->host_read_seq(V.sread[j]);
                for (int k = 1; k <= V.slen[j]; ++k) { int i = V.sqpos[j] + k; uint8_t b = sq ? sq[i >> 1] : (uint8_t)0xFF; in.allele += kNt[kCanon[(i & 1) ? (b & 15) : (b >> 4)]]; }
            } else {                                   // "-" + raw reference characters pos+1..pos+len (R:...:331-339)
                in.allele = "-";
                for (int k = 1; k <= V.slen[j]; ++k) {
                    int64_t p = pos + k; char c = 'N';
                    if (V.ref && p >= V.ref->win_beg && p < V.ref->win_beg + (int64_t)V.ref->seq.size() && p < V.ref->chrom_len) c = V.ref->seq[(size_t)(p - V.ref->win_beg)];
                    in.allele += c;
                }
            }
            W.indels.push_back(std::move(in));
        }
        if (emit) for (int j = 0; j < 6; ++j) { rec += '\t'; rec += kNt[j]; rec += ':'; put_stat(rec, have[j] ? &base[j] : nullptr, false); }
        if (gate) for (int j = 1; j <= 4; ++j) if (have[j] && brc::base_is_alt((uint32_t)j, rcode)) best_alt = std::max<uint64_t>(best_alt, base[j].v[BRC_S_COUNT]);
        if (W.indels.size() > 1) std::sort(W.indels.begin(), W.indels.end(), [](const Indel &a, const Indel &b) { return a.allele < b.allele; });
        for (auto &in : W.indels) {
            if (in.allele[0] == '-') { st.q[(size_t)r].push_back(make_qent(rg.tid, pos + 1, in.st, in.allele)); st.q_exists[(size_t)r] = 1; }
            else if (emit) { rec += '\t'; rec += in.allele; rec += ':'; put_stat(rec, &in.st, true); best_alt = std::max<uint64_t>(best_alt, in.st.v[BRC_S_COUNT]); }
        }
        if (emit && st.q_exists[(size_t)r]) {          // IndelQueue::process(tid, pos, record)
            auto &q = st.q[(size_t)r];
            while (!q.empty() && ((q.front().tid == rg.tid && q.front().pos < pos) || q.front().tid != rg.tid)) q.pop_front();
            while (!q.empty() && q.front().tid == rg.tid && q.front().pos == pos) {
                rec += '\t'; rec += q.front().allele; rec += ':'; put_stat(rec, qstat(q.front()), true);
                extra_depth += q.front().st[BRC_S_COUNT];
                best_alt = std::max<uint64_t>(best_alt, q.front().st[BRC_S_COUNT]);
                q.pop_front();
            }
        }
        if (emit && V.e->cfg.per_lib) rec += "\t}";
    }
    if (emit && pos >= rg.beg && pos < rg.end &&
        (!gate || brc::site_passes(best_alt, mapq_n + (uint64_t)extra_depth, V.e->sel_filter.min_alt_count, V.e->sel_filter.min_alt_fraction))) {
        if (V.ref) out += V.ref->name; else out += '?';
        out += '\t'; put_u(out, (uint64_t)(pos + 1)); out += '\t'; out += rb; out += '\t';
        put_u(out, (uint64_t)((int64_t)mapq_n + extra_depth));
        out += rec; out += '\n';
    }
}

// sites [s0, s1) of region g, sequentially, with the caller's queue state; seed: first replay the deletion pushes of site s0-1.
// Sparse results walk the shipped sites of the range: emit byte 0 (context) only replays pushes, the others form their line.
void format_range(const View &V, int32_t s0, int32_t s1, const char *const *lib_names, EmitState &st, std::string &out, bool seed) {
    Scratch W;
    const int64_t base = V.rg->slot_base;
    if (!V.csite) {
        if (seed && s0 > 0) { std::string sink; format_site(V, s0 - 1, base + s0 - 1, lib_names, st, sink, W, false); }
        for (int32_t s = s0; s < s1; ++s) format_site(V, s, base + s, lib_names, st, out, W, true);
        return;
    }
    const uint32_t *c = V.csite, *ce = V.csite + V.n_sel;
    const int64_t from = base + s0 - (seed && s0 > 0 ? 1 : 0);
    for (const uint32_t *p = std::lower_bound(c, ce, (uint32_t)from); p < ce && (int64_t)*p < base + s1; ++p) {
        const int64_t i = p - c;
        const int32_t s = (int32_t)((int64_t)*p - base);
        format_site(V, s, i, lib_names, st, out, W, s >= s0 && V.cemit[i] != 0);
    }
}

// Formats sites [s0, s1) of region g.  The text is appended to `parts` as one string per worker thread (in site order), so
// nothing is concatenated or copied here.
void format_region(const brc_engine *e, int64_t g, int32_t s0, int32_t s1, const char *const *lib_names, EmitState &st,
                   std::vector<std::string> &parts_out, bool seed_from_left) {
    const View V(e, g);
    const brc_region &rg = *V.rg;
    s0 = std::max(s0, 0); s1 = std::min(s1, rg.n_slots);
    if (s1 <= s0) { if (rg.site_list_mode && s1 >= rg.n_slots) st.clear(); return; }
    const int32_t n = s1 - s0;
    int nt = brc::worker_count(n, 16384, 32);
    // The deletion queue carries state across sites.  Inside one region only the site to the left matters, so ranges can be
    // formatted independently — except in the argv loop with several regions, whose queue is never cleared (A.6): keep that sequential.
    if (!rg.site_list_mode && e->regions.size() > 1) nt = 1;
    if (st.pending()) nt = 1;      // entries carried in from an earlier region / batch may print anywhere in this range
    const size_t base = parts_out.size();
    parts_out.resize(base + (size_t)nt);
    if (nt <= 1) {
        parts_out[base].reserve((size_t)(V.csite ? 0 : n) * 96);
        format_range(V, s0, s1, lib_names, st, parts_out[base], seed_from_left);
    } else {
        std::vector<EmitState> states; states.reserve((size_t)nt);
        for (int t = 0; t < nt; ++t) states.emplace_back(e->n_rows);
        brc::fan_out(nt, [&](int t) {
            const int32_t a = s0 + (int32_t)((int64_t)n * t / nt), b = s0 + (int32_t)((int64_t)n * (t + 1) / nt);
            EmitState &ls = t == 0 ? st : states[(size_t)t];
            std::string &dst = parts_out[base + (size_t)t];
            if (!V.csite) dst.reserve((size_t)(b - a) * 420);
            format_range(V, a, b, lib_names, ls, dst, t > 0 || seed_from_left);
        });
        st.clear();
        for (size_t r = 0; r < st.q.size(); ++r) { st.q[r] = states[(size_t)nt - 1].q[r]; st.q_exists[r] = states[(size_t)nt - 1].q_exists[r]; }
    }
    if (rg.site_list_mode && s1 >= rg.n_slots) st.clear();                  // d.indel_queue_map.clear()  (R:...:605)
}

// Many regions of the -l loop (a site list is typically thousands of one-base lines): every region starts with an empty
// deletion queue (R:...:605), so whole regions are dealt to worker threads — one output string per thread, regions in order.
// Returns false (nothing done) when the batch is not of that shape.
bool format_many_site_list_regions(const brc_engine *e, const char *const *lib_names, std::vector<std::string> &parts_out) {
    const size_t nr = e->regions.size();
    if (nr < 2) return false;
    int64_t total = 0;
    for (const brc_region &rg : e->regions) { if (!rg.site_list_mode) return false; total += rg.n_slots; }
    const int nt = brc::worker_count(total, 16384, 32);
    std::vector<size_t> cut((size_t)nt + 1, nr);
    cut[0] = 0;
    { int64_t acc = 0; int t = 1; for (size_t g = 0; g < nr && t < nt; ++g) { acc += e->regions[g].n_slots; while (t < nt && acc >= total * t / nt) cut[(size_t)t++] = g + 1; } }
    const size_t base = parts_out.size();
    parts_out.resize(base + (size_t)nt);
    brc::fan_out(nt, [&](int t) {
        EmitState st(e->n_rows);
        std::string &dst = parts_out[base + (size_t)t];
        int64_t slots = 0;
        for (size_t g = cut[(size_t)t]; g < cut[(size_t)t + 1]; ++g) slots += e->regions[g].n_slots;
        if (!e->sparse) dst.reserve((size_t)slots * 200);
        for (size_t g = cut[(size_t)t]; g < cut[(size_t)t + 1]; ++g) {
            const View V(e, (int64_t)g);
            format_range(V, 0, V.rg->n_slots, lib_names, st, dst, false);
            st.clear();
        }
    });
    return true;
}

// the caller's usual pattern is a size query (buf == NULL) followed by the fill: format once, keep the parts
void ensure_formatted(brc_engine *e, int64_t k0, int64_t k1, int64_t k2, const char *const *lib_names) {
    if (e->fmt_valid && e->fmt_key[0] == k0 && e->fmt_key[1] == k1 && e->fmt_key[2] == k2) return;
    brc::ensure_wide(e);
    e->fmt_parts.clear();
    // deletion queue: fresh per call, or (brc_set_queue_carry) the one the previous formatting pass left behind
    const bool carry = e->carry_on && (k1 == -1 || k1 == 0);
    if (e->carry.q.size() != (size_t)e->n_rows) e->carry = EmitState(e->n_rows);
    EmitState local(e->n_rows);
    EmitState &st = carry ? e->carry : local;
    if (k1 == -1) {   // whole regions
        if (k0 < 0 && !format_many_site_list_regions(e, lib_names, e->fmt_parts))
            for (int64_t g = 0; g < (int64_t)e->regions.size(); ++g) format_region(e, g, 0, e->regions[(size_t)g].n_slots, lib_names, st, e->fmt_parts, false);
        if (k0 >= 0) format_region(e, k0, 0, e->regions[(size_t)k0].n_slots, lib_names, st, e->fmt_parts, false);
    } else {
        format_region(e, k0, (int32_t)k1, (int32_t)std::min<int64_t>(k1 + k2, 0x7fffffff), lib_names, st, e->fmt_parts, !carry);
        // a later window of a carried region: hand its final queue on when it reaches the region's end
        if (e->carry_on && !carry && k1 + k2 >= e->regions[(size_t)k0].n_slots) e->carry = local;
    }
    e->fmt_key[0] = k0; e->fmt_key[1] = k1; e->fmt_key[2] = k2; e->fmt_valid = true;
}
int64_t parts_size(const brc_engine *e) { int64_t n = 0; for (auto &p : e->fmt_parts) n += (int64_t)p.size(); return n; }
void release_parts(brc_engine *e) { e->fmt_valid = false; std::vector<std::string>().swap(e->fmt_parts); }

int64_t serve(brc_engine *e, int64_t k0, int64_t k1, int64_t k2, const char *const *lib_names, char *buf, int64_t cap) {
    ensure_formatted(e, k0, k1, k2, lib_names);
    const int64_t n = parts_size(e);
    if (buf && cap > 0) {
        // parallel copy of the parts into the caller's buffer (truncated at cap-1)
        std::vector<int64_t> off(e->fmt_parts.size() + 1, 0);
        for (size_t i = 0; i < e->fmt_parts.size(); ++i) off[i + 1] = off[i] + (int64_t)e->fmt_parts[i].size();
        const int64_t lim = std::min<int64_t>(n, cap - 1);
        brc::fan_out((int)e->fmt_parts.size(), [&](int i) {
            const int64_t a = off[(size_t)i], b = std::min(off[(size_t)i + 1], lim);
            if (b > a) std::memcpy(buf + a, e->fmt_parts[(size_t)i].data(), (size_t)(b - a));
        });
        buf[lim] = 0;
        release_parts(e);   // delivered
    }
    return n;
}

}  // namespace

extern "C" int brc_set_queue_carry(brc_engine *e, int on) {
    if (!e) return BRC_E_INVALID;
    e->carry_on = on != 0;
    e->carry = EmitState(e->n_rows);
    e->fmt_valid = false;
    return BRC_OK;
}

extern "C" int64_t brc_format_text(brc_engine *e, int64_t region_index, const char *const *lib_names, char *buf, int64_t cap) {
    if (!e) return BRC_E_INVALID;
    if (!e->results_valid) return brc::set_error(e, BRC_E_INVALID, "format_text: no results");
    if (e->n_host_reads() == 0 && e->h_n_sec > 0 && !e->dec.pushed) return brc::set_error(e, BRC_E_INVALID, "format_text: needs the pushed reads (push path only)");
    if (region_index >= (int64_t)e->regions.size()) return BRC_E_INVALID;
    return serve(e, region_index < 0 ? -1 : region_index, -1, -1, lib_names, buf, cap);
}

// A window of one region's sites (slot offsets [first, first+count) inside the region), for callers that stream the text
// of a large region piecewise.  The deletion columns of the window's first site are re-derived from the site to its left.
extern "C" int64_t brc_format_window(brc_engine *e, int64_t region_index, int64_t first, int64_t count, const char *const *lib_names,
                                     char *buf, int64_t cap) {
    if (!e || region_index < 0 || region_index >= (int64_t)e->regions.size() || first < 0 || count < 0) return BRC_E_INVALID;
    if (!e->results_valid) return brc::set_error(e, BRC_E_INVALID, "format_window: no results");
    return serve(e, region_index, first, count, lib_names, buf, cap);
}

// Same text straight to a file descriptor (no intermediate buffer): region_index < 0 = all regions (first/count ignored),
// otherwise the window [first, first+count) of that region (count < 0 = to the region's end).  Returns bytes written.
extern "C" int64_t brc_write_text(brc_engine *e, int64_t region_index, int64_t first, int64_t count, const char *const *lib_names, int fd) {
    if (!e || region_index >= (int64_t)e->regions.size() || first < 0) return BRC_E_INVALID;
    if (!e->results_valid) return brc::set_error(e, BRC_E_INVALID, "write_text: no results");
    if (region_index < 0) ensure_formatted(e, -1, -1, -1, lib_names);
    else ensure_formatted(e, region_index, first, count < 0 ? (int64_t)0x7fffffff : count, lib_names);
    int64_t total = 0;
    for (auto &p : e->fmt_parts) {
        size_t done = 0;
        while (done < p.size()) {
            const ssize_t w = ::write(fd, p.data() + done, p.size() - done);
            if (w < 0) { release_parts(e); return brc::set_error(e, BRC_E_INVALID, "write_text: write() failed"); }
            done += (size_t)w;
        }
        total += (int64_t)p.size();
    }
    release_parts(e);
    return total;
}
