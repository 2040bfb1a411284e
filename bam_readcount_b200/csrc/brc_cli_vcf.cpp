// brc_cli_vcf.cpp — `brc-readcount --vcf FILE` (brc_cli_vcf.h): parsing, the engine queries of a batch and their answers,
// and the VCF text.
#include "brc_cli_vcf.h"

#include <algorithm>
#include <cctype>
#include <cerrno>
#include <climits>
#include <cstring>
#include <unistd.h>

#include "brc_cli_input.h"

namespace brc::cli {

const char kVcfFormat[] = ":BRC_DP:BRC_AD:BRC_ADF:BRC_ADR:BRC_AF";
const char kVcfHeader[] =
    "##FORMAT=<ID=BRC_DP,Number=1,Type=Integer,Description=\"brc-readcount depth of the site's line\">\n"
    "##FORMAT=<ID=BRC_AD,Number=R,Type=Integer,Description=\"brc-readcount count of the REF and each ALT allele\">\n"
    "##FORMAT=<ID=BRC_ADF,Number=R,Type=Integer,Description=\"brc-readcount plus-strand count of the REF and each ALT allele\">\n"
    "##FORMAT=<ID=BRC_ADR,Number=R,Type=Integer,Description=\"brc-readcount minus-strand count of the REF and each ALT allele\">\n"
    "##FORMAT=<ID=BRC_AF,Number=A,Type=Float,Description=\"brc-readcount BRC_AD of each ALT allele over BRC_DP\">\n";

std::vector<std::string> split(const std::string &s, char c) {
    std::vector<std::string> out; size_t p = 0;
    for (size_t t; (t = s.find(c, p)) != std::string::npos; p = t + 1) out.push_back(s.substr(p, t - p));
    out.push_back(s.substr(p));
    return out;
}

// the whole file, plain or BGZF (bgzip); false with a message
bool read_vcf_bytes(const std::string &path, std::string &out, std::string &why) {
    FILE *f = std::fopen(path.c_str(), "rb");
    if (!f) { why = "cannot open " + path + ": " + std::strerror(errno); return false; }
    uint8_t head[512]; const size_t got = std::fread(head, 1, sizeof head, f);
    if (got < 2 || head[0] != 31 || head[1] != 139) {
        out.assign((const char *)head, got);
        char buf[1 << 16];
        for (size_t n; (n = std::fread(buf, 1, sizeof buf, f)) > 0;) out.append(buf, n);
        const bool bad = std::ferror(f);
        std::fclose(f);
        if (bad) why = "cannot read " + path;
        return !bad;
    }
    std::fclose(f);
    size_t hdr = 0;
    if (!Bgzf::block_size(head, got, hdr)) { why = path + " is gzip-compressed but not BGZF: compress it with bgzip"; return false; }
    Bgzf bz;
    if (!bz.open(path)) { why = "cannot open " + path; return false; }
    for (uint64_t coff = 0; bz.load_block(coff); coff = bz.next_coff) out.append((const char *)bz.block.data(), bz.block.size());
    if (bz.error) { why = path + ": truncated or corrupt BGZF block"; return false; }
    return true;
}

// Parses the whole VCF, applies the allele rule and resolves the samples that take values: `samples` as named by option `opt`,
// or none given (the VCF's only sample column).  False with a message (nothing may have been written yet).
bool parse_vcf(const std::string &path, const std::vector<std::string> &samples, const char *opt, bool complex_on, Vcf &v,
               std::string &why) {
    std::string text;
    if (!read_vcf_bytes(path, text, why)) return false;
    v.path = path;
    auto up = [](std::string s) { for (char &c : s) c = (char)std::toupper((unsigned char)c); return s; };
    auto acgtn = [](const std::string &s, size_t from) {
        if (s.size() <= from) return false;
        for (size_t i = from; i < s.size(); ++i) if (!std::strchr(canonical_nt + 1, s[i]) || !s[i]) return false;
        return true;
    };
    auto kind_of = [](char c) { return (uint32_t)(std::strchr(canonical_nt, c) - canonical_nt); };
    bool in_header = true;
    size_t ln = 0;
    for (size_t p = 0; p < text.size();) {
        size_t e = text.find('\n', p);
        if (e == std::string::npos) e = text.size();
        std::string line = text.substr(p, e - p);
        p = e + 1; ++ln;
        const std::string at = path + ": line " + std::to_string(ln) + ": ";
        if (in_header && line.compare(0, 2, "##") == 0) {
            if (line.compare(0, 16, "##FORMAT=<ID=BRC") == 0 && line.size() > 16 && line[16] == '_') { why = at + "the header already declares a BRC_* FORMAT field"; return false; }
            v.header.push_back(line);
            continue;
        }
        if (in_header && line.compare(0, 6, "#CHROM") == 0) {
            v.chrom_line = line; v.n_cols = split(line, '\t').size(); in_header = false;
            if (v.n_cols < 8) { why = at + "the #CHROM line has fewer than 8 columns"; return false; }
            if (v.n_cols == 9) { why = at + "a FORMAT column without sample columns"; return false; }
            continue;
        }
        if (in_header) { why = at + "data before the #CHROM header line"; return false; }
        VcfRecord r;
        r.cols = split(line, '\t');
        if (r.cols.size() < 8) { why = at + "fewer than 8 columns"; return false; }
        if (r.cols.size() != v.n_cols) { why = at + std::to_string(r.cols.size()) + " columns, the #CHROM line has " + std::to_string(v.n_cols); return false; }
        const std::string &ps = r.cols[1];
        int64_t pos = 0;
        bool ok = !ps.empty() && ps.size() <= 10;
        for (char c : ps) ok = ok && c >= '0' && c <= '9';
        if (ok) pos = std::atoll(ps.c_str());
        if (!ok || pos < 1 || pos >= INT32_MAX) { why = at + "POS is not a positive integer below 2^31 - 1"; return false; }
        const std::string ref = up(r.cols[3]);
        const bool ref_ok = acgtn(ref, 0);
        std::vector<std::string> alts;
        for (const std::string &a0 : split(r.cols[4], ',')) {
            const std::string a = up(a0);
            alts.push_back(a);
            int64_t kl = -1; std::string bases;
            if (ref_ok && ref.size() == 1 && a.size() == 1 && acgtn(a, 0)) kl = kind_of(a[0]);
            else if (ref_ok && ref.size() == 1 && a.size() >= 2 && a[0] == ref[0] && acgtn(a, 1)) { kl = BRC_KIND_INS | (int64_t)(a.size() - 1) << 8; bases = a.substr(1); }
            else if (ref_ok && ref.size() >= 2 && a.size() == 1 && a[0] == ref[0]) kl = BRC_KIND_DEL | (int64_t)(ref.size() - 1) << 8;
            r.counted = r.counted || kl >= 0;
            r.complex = r.complex || (complex_on && pos >= 2 && ref_ok && kl < 0 && acgtn(a, 0));
            r.alt_kind_len.push_back(kl); r.alt_bases.push_back(bases);
        }
        if (r.complex) {      // the whole record by the complex rule: the REF and every A/C/G/T/N ALT
            r.counted = true; r.line_pos = (int32_t)pos; r.ref = ref;
            for (size_t i = 0; i < alts.size(); ++i) {
                r.alt_kind_len[i] = acgtn(alts[i], 0) ? 0 : -1;
                r.alt_bases[i] = r.alt_kind_len[i] >= 0 ? alts[i] : "";
            }
        }
        if (r.counted) {
            if (!r.complex) { r.line_pos = (int32_t)(ref.size() == 1 ? pos : pos + 1); r.ref_kind = kind_of(ref[ref.size() == 1 ? 0 : 1]); }
            r.n_queries = 1 + (size_t)std::count_if(r.alt_kind_len.begin(), r.alt_kind_len.end(), [](int64_t x) { return x >= 0; });
            r.word_off = v.n_words; v.n_words += 1 + 3 * r.n_queries;
        }
        v.rec.push_back(std::move(r));
    }
    if (in_header) { why = path + ": no #CHROM header line"; return false; }
    const std::vector<std::string> hc = split(v.chrom_line, '\t');
    v.target_of_col.assign(v.n_cols, -1);
    if (v.n_cols == 8) {
        if (samples.empty()) { why = path + " has no sample column: --vcf-sample NAME names the one added"; return false; }
        v.samples = samples;
        return true;
    }
    if (samples.empty()) {
        if (hc.size() > 10) { why = path + " has " + std::to_string(hc.size() - 9) + " sample columns: --vcf-sample NAME is required"; return false; }
        v.samples.assign(1, hc[9]); v.target_of_col[9] = 0;
        return true;
    }
    for (size_t t = 0; t < samples.size(); ++t) {
        int n_match = 0, col = -1;
        for (size_t c = 9; c < hc.size(); ++c) if (hc[c] == samples[t]) { ++n_match; col = (int)c; }
        if (n_match == 0) { why = std::string(opt) + " " + samples[t] + ": no such sample in " + path; return false; }
        if (n_match > 1) { why = std::string(opt) + " " + samples[t] + " is ambiguous: " + std::to_string(n_match) + " sample columns of " + path + " have that name"; return false; }
        v.target_of_col[(size_t)col] = (int)t;
    }
    v.samples = samples;
    return true;
}

bool write_all(int fd, const std::string &s) {
    for (size_t done = 0; done < s.size();) {
        const ssize_t w = ::write(fd, s.data() + done, s.size() - done);
        if (w < 0) { if (errno == EINTR) continue; return false; }
        done += (size_t)w;
    }
    return true;
}

// Record ri's five values in one sample from its answer words (REF first, then each countable ALT in order).  A record the
// sample did not answer, and every record of a failed sample, gets '.' in all five.
void vcf_values(const Vcf &v, size_t ri, const VcfAnswers &a, std::string &out) {
    if (a.failed || !a.answered[ri]) { out += ".:.:.:.:."; return; }
    const VcfRecord &r = v.rec[ri];
    const uint32_t *w = a.words.data() + r.word_off;
    const uint32_t dp = w[0];
    std::string ad, adf, adr, af;
    auto put = [&](const uint32_t *q) {
        ad += q ? std::to_string(q[0]) : "."; adf += q ? std::to_string(q[1]) : "."; adr += q ? std::to_string(q[2]) : ".";
    };
    put(w + 1);
    size_t k = 1;
    for (size_t i = 0; i < r.alt_kind_len.size(); ++i) {
        const uint32_t *q = r.alt_kind_len[i] >= 0 ? w + 1 + 3 * k++ : nullptr;
        ad += ','; adf += ','; adr += ',';
        put(q);
        if (i) af += ',';
        if (!q || dp == 0) { af += '.'; continue; }
        char b[64]; std::snprintf(b, sizeof b, "%.6g", (double)q[0] / (double)dp);
        af += b;
    }
    out += std::to_string(dp); out += ':'; out += ad; out += ':'; out += adf; out += ':'; out += adr; out += ':'; out += af;
}

// Record ri's line, appended to `out`: the values of sample t from ans[t] in that sample's column.
void vcf_line(const Vcf &v, size_t ri, const VcfAnswers *ans, std::string &out) {
    const VcfRecord &r = v.rec[ri];
    const size_t n = r.cols.size();
    for (size_t c = 0; c < n; ++c) {
        if (c) out += '\t';
        out += r.cols[c];
        if (c == 8) { out += kVcfFormat; continue; }
        const int t = v.target_of_col[c];
        if (t < 0) continue;
        const size_t keys = (size_t)std::count(r.cols[8].begin(), r.cols[8].end(), ':') + 1;
        for (size_t have = (size_t)std::count(r.cols[c].begin(), r.cols[c].end(), ':') + 1; have < keys; ++have) out += ":.";
        out += ':';
        vcf_values(v, ri, ans[t], out);
    }
    if (n == 8) {
        out += '\t'; out += kVcfFormat + 1;
        for (size_t t = 0; t < v.samples.size(); ++t) { out += '\t'; vcf_values(v, ri, ans[t], out); }
    }
    out += '\n';
}

std::string vcf_header(const Vcf &v) {
    std::string out;
    for (const std::string &h : v.header) { out += h; out += '\n'; }
    out += kVcfHeader;
    out += v.chrom_line;
    if (v.n_cols == 8) { out += "\tFORMAT"; for (const std::string &s : v.samples) { out += '\t'; out += s; } }
    out += '\n';
    return out;
}

// Record ri's answer into a's words: the depth of its line, then (count, plus, minus) of each of its queries, REF first, as
// triple(k, out) writes them for query k.
template <class Triple> void vcf_store(const Vcf &v, size_t ri, uint32_t depth, const Triple &triple, VcfAnswers &a) {
    const VcfRecord &r = v.rec[ri];
    uint32_t *w = a.words.data() + r.word_off;
    w[0] = depth;
    for (size_t k = 0; k < r.n_queries; ++k) triple(k, w + 1 + 3 * k);
    a.answered[ri] = 1;
}

int vcf_set_queries(brc_engine *eng, const Vcf &v, const int64_t *recs, int64_t n, FILE *err) {
    std::vector<brc_allele_query> q; std::string q_bases;
    std::vector<brc_complex_query> cq; std::vector<brc_complex_allele> ca; std::string c_bases;
    for (int64_t g = 0; g < n; ++g) {
        const VcfRecord &rec = v.rec[(size_t)recs[g]];
        if (rec.complex) {      // the REF and every A/C/G/T/N ALT, matched against the reads' bases between the flanks
            cq.push_back({g, rec.line_pos - 1, (int32_t)rec.ref.size(), (int32_t)rec.n_queries, 0});
            ca.push_back({(int64_t)c_bases.size(), (int32_t)rec.ref.size(), 0}); c_bases += rec.ref;
            for (size_t i = 0; i < rec.alt_kind_len.size(); ++i)
                if (rec.alt_kind_len[i] >= 0) { ca.push_back({(int64_t)c_bases.size(), (int32_t)rec.alt_bases[i].size(), 0}); c_bases += rec.alt_bases[i]; }
            continue;
        }
        q.push_back({g, rec.line_pos - 1, rec.ref_kind, 0});
        for (size_t i = 0; i < rec.alt_kind_len.size(); ++i)
            if (rec.alt_kind_len[i] >= 0) { q.push_back({g, rec.line_pos - 1, (uint32_t)rec.alt_kind_len[i], (int64_t)q_bases.size()}); q_bases += rec.alt_bases[i]; }
    }
    int r;
    if ((r = brc_set_allele_queries(eng, q.data(), (int64_t)q.size(), q_bases.data(), (int64_t)q_bases.size())) != BRC_OK) { std::fprintf(err, "brc_set_allele_queries: %s\n", brc_last_error(eng)); return r; }
    if (!cq.empty() && (r = brc_set_complex_queries(eng, cq.data(), (int64_t)cq.size(), ca.data(), (int64_t)ca.size(), c_bases.data(), (int64_t)c_bases.size())) != BRC_OK) { std::fprintf(err, "brc_set_complex_queries: %s\n", brc_last_error(eng)); return r; }
    return BRC_OK;
}

int vcf_get_answers(brc_engine *eng, const Vcf &v, const int64_t *recs, int64_t n, VcfAnswers &a, FILE *err) {
    int64_t n_q = 0, n_cq = 0, n_cqa = 0;       // the queries vcf_set_queries set: allele queries, complex queries and their alleles
    for (int64_t g = 0; g < n; ++g) {
        const VcfRecord &rec = v.rec[(size_t)recs[g]];
        if (rec.complex) { ++n_cq; n_cqa += (int64_t)rec.n_queries; } else n_q += (int64_t)rec.n_queries;
    }
    int r;
    const brc_allele_answer *ans = nullptr; int64_t n_ans = 0;
    if ((r = brc_get_allele_answers(eng, &ans, &n_ans)) != BRC_OK || n_ans != n_q) { std::fprintf(err, "brc_get_allele_answers: %s\n", brc_last_error(eng)); return r ? r : -1; }
    const uint32_t *c_depth = nullptr; const brc_complex_count *c_cnt = nullptr; int64_t n_c = 0, n_ca = 0;
    if (n_cq && ((r = brc_get_complex_answers(eng, &c_depth, &c_cnt, &n_c, &n_ca)) != BRC_OK || n_c != n_cq || n_ca != n_cqa)) { std::fprintf(err, "brc_get_complex_answers: %s\n", brc_last_error(eng)); return r ? r : -1; }
    for (int64_t g = 0; g < n; ++g) {
        const size_t ri = (size_t)recs[g];
        if (v.rec[ri].complex) {
            vcf_store(v, ri, *c_depth++, [c = c_cnt](size_t k, uint32_t *t) { t[0] = c[k].count; t[1] = c[k].plus; t[2] = c[k].count - c[k].plus; }, a);
            c_cnt += v.rec[ri].n_queries;
        } else {
            vcf_store(v, ri, ans[0].line ? ans[0].depth : 0, [q = ans](size_t k, uint32_t *t) { t[0] = q[k].stats[BRC_S_COUNT]; t[1] = q[k].stats[BRC_S_PLUS]; t[2] = q[k].stats[BRC_S_MINUS]; }, a);
            ans += v.rec[ri].n_queries;
        }
    }
    return BRC_OK;
}

}  // namespace brc::cli
