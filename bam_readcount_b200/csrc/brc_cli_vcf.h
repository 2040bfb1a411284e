// brc_cli_vcf.h — `brc-readcount --vcf FILE`: the per-allele read counts of each VCF record, written back as FORMAT fields
// (DESIGN.md §12).  A record is counted when one of its ALT alleles is an SNV, an insertion after its anchor base or a deletion
// after it; its site is one line "CHROM L L" of a derived -l site list (L = POS, or POS + 1 for a deletion, whose entry prints
// on the line after the anchor), and its values are what that run prints on the line: the engine answers them
// (brc_set_allele_queries).  With --vcf-complex a record with an A/C/G/T/N ALT that no entry answers (an MNP, a complex
// substitution, an indel without its anchor base) is counted by the complex rule instead: its site is the line "CHROM POS POS",
// and the engine matches each read's bases between the two flanks of REF against REF and its ALTs (brc_set_complex_queries).
#pragma once
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/brc_engine.h"

namespace brc::cli {

struct VcfRecord {
    std::vector<std::string> cols;
    bool counted = false;
    int32_t line_pos = 0;                 // L: 1-based position of the derived site-list line
    uint32_t ref_kind = 0;                // the REF entry: a base class of "=ACGTN"
    std::vector<int64_t> alt_kind_len;    // per ALT: query kind | length << 8, or -1 when the ALT is not countable
    std::vector<std::string> alt_bases;   // per ALT: an insertion's bases; a complex record: the ALT as upper-case letters
    bool complex = false;                 // counted by the complex rule (--vcf-complex): alt_kind_len 0 for each A/C/G/T/N ALT
    std::string ref;                      // a complex record: REF as upper-case letters
    size_t n_queries = 0;                 // counted: the REF and each countable ALT
    size_t word_off = 0;                  // counted: where its answer words start in a sample's VcfAnswers
};
struct Vcf {
    std::string path;
    std::vector<std::string> header;      // every line before #CHROM
    std::string chrom_line;
    size_t n_cols = 0;
    // the samples that take values, in the order given: each an existing column (target_of_col), or, in a sites-only VCF, a
    // column added after an added FORMAT column
    std::vector<std::string> samples;
    std::vector<int> target_of_col;       // per column: the index in `samples` of the sample it holds, or -1
    std::vector<VcfRecord> rec;
    size_t n_words = 0;                   // answer words of one sample: 1 + 3 * n_queries per counted record
};

// One sample's answers.  For each counted record, at its word_off: the depth of the record's line (0 when it prints none), then
// count, plus and minus of the REF entry and of each countable ALT's entry.  A sample that failed has none.
struct VcfAnswers {
    std::vector<uint32_t> words;
    std::vector<uint8_t> answered;        // per record: its words are set (counted, and its contig is in the sample's input)
    bool failed = false;
    explicit VcfAnswers(const Vcf &v) : words(v.n_words), answered(v.rec.size()) {}
};

std::vector<std::string> split(const std::string &s, char c);
bool write_all(int fd, const std::string &s);

// Parses the whole VCF, applies the allele rule and resolves the samples that take values: `samples` as named by option `opt`,
// or none given (the VCF's only sample column).  False with a message (nothing may have been written yet).
bool parse_vcf(const std::string &path, const std::vector<std::string> &samples, const char *opt, bool complex_on, Vcf &v,
               std::string &why);
std::string vcf_header(const Vcf &v);
// Record ri's line, appended to `out`: the values of sample t from ans[t] in that sample's column.
void vcf_line(const Vcf &v, size_t ri, const VcfAnswers *ans, std::string &out);

// A batch of n regions whose region g is the site of record recs[g].  vcf_set_queries sets the batch's queries on `eng`: the
// REF entry and every countable ALT of each ordinary record as allele queries, and each --vcf-complex record's REF and
// A/C/G/T/N ALTs as a complex query.  vcf_get_answers reads the answers of the computed batch into `a`.  Both return BRC_OK, or
// a failed status with a message on `err`.
int vcf_set_queries(brc_engine *eng, const Vcf &v, const int64_t *recs, int64_t n, FILE *err);
int vcf_get_answers(brc_engine *eng, const Vcf &v, const int64_t *recs, int64_t n, VcfAnswers &a, FILE *err);

}  // namespace brc::cli
