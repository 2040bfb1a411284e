// brc_cli.cpp — `brc-readcount`: the C++ host.  Same command line and STDOUT as bam-readcount
// (R:src/exe/bam-readcount/bamreadcount.cpp:421-670), with the pileup hot path routed through
// libbrc_engine.so (include/brc_engine.h).  File decode stays on the host, as the north star says: the input unit
// (brc_cli_input.h) reads BGZF, BAM, BAI and FASTA itself, and CRAM through htslib when the host is built with it.
// This unit holds the options, the samples and the region loop; --vcf is brc_cli_vcf.h, the per-read warnings brc_cli_warn.h.
//
// Mirrors, region by region, the reference's two loops:
//   -l site list : R:...:574-608  (d.beg=beg-1, d.end=end, queues cleared per region)
//   argv regions : R:...:641-657  (bam_parse_region; a bare contig name keeps the previous beg/end, A.6)
// With --bam-list the same per-sample run is repeated over a list of inputs in one process (DESIGN.md §11); --vcf-samples
// does the same for the sample columns of one VCF (DESIGN.md §12).
#include <algorithm>
#include <cerrno>
#include <cstdarg>
#include <climits>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <getopt.h>
#include <fcntl.h>
#include <filesystem>
#include <map>
#include <set>
#include <sstream>
#include <string>
#include <vector>
#include <chrono>
#include <future>
#include <memory>
#include <thread>
#include <unordered_map>
#include <unistd.h>

#include "../../include/brc_engine.h"
#include "brc_cli_input.h"
#include "brc_cli_vcf.h"
#include "brc_cli_warn.h"

namespace brc::cli {

void usage() {
    std::printf("Usage: bam-readcount [OPTIONS] bam_file|cram_file [region]\nGenerate metrics for bam_file at single nucleotide positions.\n"
                "Example: bam-readcount -f ref.fa some.bam|some.cram\n\nAvailable options:\n"
                "  -h [ --help ]                         produce this message\n"
                "  -v [ --version ]                      output the version number\n"
                "  -q [ --min-mapping-quality ] arg (=0) minimum mapping quality of reads used for counting.\n"
                "  -b [ --min-base-quality ] arg (=0)    minimum base quality at a position to use the read for counting.\n"
                "  -d [ --max-count ] arg (=10000000)    max depth to avoid excessive memory usage.\n"
                "  -l [ --site-list ] arg                file containing a list of regions to report readcounts within.\n"
                "  -f [ --reference-fasta ] arg          reference sequence in the fasta format.\n"
                "  -D [ --print-individual-mapq ] arg    report the mapping qualities as a comma separated list.\n"
                "  -p [ --per-library ]                  report results by library.\n"
                "  -w [ --max-warnings ] arg             maximum number of warnings of each type to emit. -1 gives an unlimited number.\n"
                "  -i [ --insertion-centric ]            generate indel centric readcounts. Reads containing insertions will not be\n"
                "                                        included in per-base counts\n"
                "  --shard RANK/COUNT                    (this host) compute only shard RANK of COUNT: the regions are cut into COUNT runs of\n"
                "                                        about equal BAI-estimated coverage, one process per GPU (BRC_DEVICE); outputs\n"
                "                                        concatenate in rank order\n"
                "  --min-alt-count N                     (this host) print only the sites where an alternative allele (a base other than\n"
                "                                        the reference base, an insertion or a deletion) has a count of at least N\n"
                "  --min-alt-fraction F                  (this host) ... and of at least F times the site's depth (0 <= F <= 1; without\n"
                "                                        --min-alt-count the count must be at least 1).  Printed lines are unchanged\n"
                "  --alt-min NAME=V                      (this host) ... and that allele's field NAME, as the line prints it, is at least V\n"
                "                                        (V: digits with at most two decimals; NAME: count, avg_mapping_quality,\n"
                "                                        avg_basequality, avg_se_mapping_quality, num_plus_strand, num_minus_strand,\n"
                "                                        avg_pos_as_fraction, avg_num_mismatches_as_fraction, avg_sum_mismatch_qualities,\n"
                "                                        num_q2_containing_reads, avg_distance_to_q2_start_in_q2_reads, avg_clipped_length,\n"
                "                                        avg_distance_to_effective_3p_end).  Repeatable; alone it means count >= 1\n"
                "  --alt-max NAME=V                      (this host) ... and at most V\n"
                "  --bam-list FILE                       (this host) run many samples in one process.  Each line of FILE is\n"
                "                                        INPUT<TAB>OUT or INPUT<TAB>OUT<TAB>ERR (ERR defaults to OUT.log); OUT and ERR get\n"
                "                                        exactly what `brc-readcount <options> INPUT <regions>` prints on STDOUT and\n"
                "                                        STDERR.  Every positional argument is a region; a failed sample does not stop\n"
                "                                        the others (exit status 1 at the end)\n"
                "  --vcf FILE                            (this host) write FILE (VCF, plain or bgzip) back to STDOUT with the read counts of\n"
                "                                        each record's REF and SNV / insertion / deletion ALT alleles as FORMAT fields BRC_DP,\n"
                "                                        BRC_AD, BRC_ADF, BRC_ADR and BRC_AF: the values the line of each record's site prints\n"
                "                                        (STDERR is that of -l over the records' sites).  Not with -l, regions, -p,\n"
                "                                        --min-alt-*, --alt-min/--alt-max, --shard or --bam-list\n"
                "  --vcf-sample NAME                     (this host) the sample column that takes the values (required with several; names\n"
                "                                        the column added to a sites-only VCF)\n"
                "  --vcf-samples FILE                    (this host) with --vcf and no positional argument: annotate several sample columns\n"
                "                                        in one process.  Each line of FILE is NAME<TAB>INPUT or NAME<TAB>INPUT<TAB>ERR;\n"
                "                                        NAME's column gets the values of `--vcf-sample NAME INPUT`, ERR (default: STDERR)\n"
                "                                        that run's STDERR.  A failed sample gets '.' and does not stop the others (exit\n"
                "                                        status 1 at the end)\n"
                "  --vcf-complex                         (this host) with --vcf: also count MNP and complex records (an A/C/G/T/N ALT\n"
                "                                        that no printed entry answers) by each read's bases between the two reference\n"
                "                                        bases flanking REF, matched exactly against REF and each ALT\n"
                "  --bgzf                                (this host) write STDOUT, the VCF and every --bam-list OUT file as BGZF (bgzip's\n"
                "                                        format, compressed on the GPU); STDERR and ERR files stay plain\n\n");
}

struct Options {   // everything on the command line except the inputs: the same for every sample
    int min_mapq = 0, min_bq = 0, max_cnt = 10000000; bool per_lib = false, ic = false; long long max_warn = -1;
    const Vcf *vcf = nullptr;     // --vcf: the parsed file
    bool vcf_samples = false;     // --vcf-samples: a sample only fills its answers; the VCF is written after the last sample
    bool vcf_complex = false;     // --vcf-complex: MNP and complex records are counted too (DESIGN.md §12)
    std::string fn_pos, fn_fa, dist_arg;
    std::vector<std::string> region_args;
    int shard_rank = 0, shard_count = 1;
    bool site_filter = false; brc_site_filter filter{};
    bool has_bounds = false; brc_entry_bounds bounds{};   // --alt-min / --alt-max (brc_set_site_filter_bounds)
    bool decode_only = false, device_decode = false, timing = false;
    bool bgzf = false;            // --bgzf: every output destination gets a BGZF writer (not under BRC_CLI_DECODE_ONLY: no device)
    int device = 0;               // BRC_DEVICE: the device of the engines and of the BGZF writers
    bool dist_refused() const { return dist_arg == "1" || dist_arg == "true"; }
};

// One output destination (STDOUT, a --bam-list OUT file): plain writes to fd, or with --bgzf a BGZF writer on fd.  Every write of
// text or VCF lines goes through here.
struct Out {
    int fd = STDOUT_FILENO;
    brc_bgzf_writer *bgzf = nullptr;
    bool failed = false;          // a BGZF write failed and the caller reported it
    // --bgzf: the writer is opened with the destination, on the engines' device; false with the reason in `why`
    bool open(const Options &o, int f, std::string &why) {
        fd = f;
        if (!o.bgzf || o.decode_only) return true;
        int rc = brc_set_device(o.device);
        if (rc == BRC_OK) rc = brc_bgzf_open(fd, &bgzf);
        if (rc != BRC_OK) why = std::string("--bgzf: ") + brc_strerror(rc);
        return rc == BRC_OK;
    }
    bool write(const std::string &s) {
        if (!bgzf) return write_all(fd, s);
        failed = failed || brc_bgzf_write(bgzf, s.data(), s.size()) != BRC_OK;
        return !failed;
    }
    int64_t text(brc_engine *eng, int64_t g, int64_t first, int64_t count, const char *const *libs) {
        if (!bgzf) return brc_write_text(eng, g, first, count, libs, fd);
        const int64_t n = brc_write_text_bgzf(eng, g, first, count, libs, bgzf);
        failed = failed || n < 0;
        return n;
    }
    // the rest of the BGZF stream and its EOF member; false (errno set when a write failed) on failure.  fd stays open.
    bool close() {
        if (!bgzf) return true;
        const int rc = brc_bgzf_close(bgzf);
        bgzf = nullptr;
        if (rc != BRC_OK && rc != BRC_E_IO) errno = EIO;
        return rc == BRC_OK;
    }
};

// the allele entry's 13 numbers by bam-readcount's column names, in print order (BRC_S_*)
const char *const kEntryFields[BRC_N_STATS] = {
    "count", "avg_mapping_quality", "avg_basequality", "avg_se_mapping_quality", "num_plus_strand", "num_minus_strand",
    "avg_pos_as_fraction", "avg_num_mismatches_as_fraction", "avg_sum_mismatch_qualities", "num_q2_containing_reads",
    "avg_distance_to_q2_start_in_q2_reads", "avg_clipped_length", "avg_distance_to_effective_3p_end"};

// --alt-min / --alt-max NAME=V: V is ^[0-9]+(\.[0-9]{1,2})?$, kept exactly as hundredths.  False (message on stderr) when malformed.
bool parse_bound(const char *opt, const char *arg, uint32_t &set, int64_t *val) {
    const char *eq = std::strchr(arg, '=');
    if (!eq) { std::fprintf(stderr, "%s wants NAME=V, got '%s'\n", opt, arg); return false; }
    const std::string name(arg, (size_t)(eq - arg));
    int k = 0;
    while (k < BRC_N_STATS && name != kEntryFields[k]) ++k;
    if (k == BRC_N_STATS) { std::fprintf(stderr, "%s: unknown field '%s' (NAME=V with NAME one of the allele entry's column names)\n", opt, name.c_str()); return false; }
    const char *v = eq + 1, *p = v;
    int64_t h = 0; int ip = 0, fp = -1;
    for (; *p >= '0' && *p <= '9'; ++p, ++ip) if (ip < 15) h = h * 10 + (*p - '0');
    if (*p == '.') for (fp = 0, ++p; *p >= '0' && *p <= '9'; ++p) { if (++fp <= 2) h = h * 10 + (*p - '0'); }
    if (ip == 0 || ip > 15 || *p || fp == 0 || fp > 2) { std::fprintf(stderr, "%s %s: V wants digits with at most two decimals\n", opt, name.c_str()); return false; }
    for (int f = fp < 0 ? 0 : fp; f < 2; ++f) h *= 10;
    if ((set >> k) & 1u) { std::fprintf(stderr, "%s %s is given twice\n", opt, name.c_str()); return false; }
    set |= 1u << k; val[k] = h;
    return true;
}

double now() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// The messages of open_sample.  A run on one input prints them as they come (`live` = stderr), between whatever the libraries
// it calls print themselves; a cohort opening the next sample under the current one holds them until that sample runs.
struct Messages {
    FILE *live = nullptr;
    std::string held;
    void say(const char *fmt, ...) __attribute__((format(printf, 2, 3))) {
        va_list ap;
        if (live) { va_start(ap, fmt); std::vfprintf(live, fmt, ap); va_end(ap); return; }
        va_start(ap, fmt); const int n = std::vsnprintf(nullptr, 0, fmt, ap); va_end(ap);
        if (n <= 0) return;
        std::string line((size_t)n + 1, '\0');
        va_start(ap, fmt); std::vsnprintf(&line[0], line.size(), fmt, ap); va_end(ap);
        line.pop_back();
        held += line;
    }
};

struct Region { int tid, beg, end; bool site_list; bool cont = false; };   // cont: a later window of a cut region (its halo site belongs to the window before)

// the end of region g's fetch, clamped to the contig's length (a region that starts beyond the contig keeps one base)
int64_t fetch_end(const BamFile &bam, const Region &g) {
    return std::min<int64_t>(g.end, std::max<int64_t>(bam.lens[(size_t)g.tid], (int64_t)g.beg + 1));
}

struct Sample {
    const Options &o;
    std::string path; bool is_cram = false;
    Messages log;                 // the run's STDERR up to its region loop (held when opened ahead of its turn)
    int status = 1;               // 0 once open_sample got to the end; otherwise the run exits 1 after printing `log`
    double t0 = 0;                // when opening began
    BamFile bam;
    HtsSource hts;                // a CRAM input
    Fasta fa; bool have_fa = false;
    RgLib rg_lib;
    std::vector<std::string> lib_names; std::vector<const char *> lib_ptrs;
    std::vector<Region> regions;
    std::vector<int64_t> vcf_region;   // --vcf: per record, the index of its site-list region (-1: not counted, or contig not in the BAM)
    Warner warner;
    // big fetches (windows of a cut region) of a BAM are decoded by several threads, one window ahead of the engine
    // (ParallelFetcher), unless the engine decodes the file itself (BRC_CLI_DEVICE_DECODE)
    ParallelFetcher pf;
    bool allow_parallel = false;
    WindowJob *jobs;              // the process's two window jobs (page-locked buffers), used by one sample at a time
    std::future<bool> ahead; size_t ahead_gi = (size_t)-1; int ahead_slot = 0;   // waited for when the sample goes
    bool par_decode_error = false; uint64_t par_decoded = 0, par_windows = 0;

    Sample(const Options &opt, const std::string &p, WindowJob *pool)
        : o(opt), path(p), warner(opt.max_warn, opt.min_mapq, opt.min_bq, opt.per_lib, opt.ic), pf(bam, rg_lib, p, opt.per_lib, !opt.decode_only), jobs(pool) {}
    Sample(const Sample &) = delete; Sample &operator=(const Sample &) = delete;

    void fetch_range(size_t gi, int64_t &fb, int64_t &fe) const {
        fb = std::max<int64_t>((int64_t)regions[gi].beg - 1, 0);
        fe = fetch_end(bam, regions[gi]);
    }
    bool par_ok(size_t gi) const {
        if (!allow_parallel || gi >= regions.size()) return false;
        int64_t fb, fe; fetch_range(gi, fb, fe);
        return ParallelFetcher::eligible(fb, fe);
    }
    std::future<bool> start_decode(size_t gi, int slot) {
        int64_t fb, fe; fetch_range(gi, fb, fe);
        const int tid = regions[gi].tid; const bool collect = warner.collecting();
        WindowJob *job = &jobs[slot]; ParallelFetcher *pfp = &pf;
        return std::async(std::launch::async, [pfp, job, tid, fb, fe, collect] { return pfp->run(tid, fb, fe, collect, *job); });
    }
    // the decoded window for region gi (prefetched or decoded now); nullptr = take the sequential path
    WindowJob *decoded_window(size_t gi) {
        int slot = 0; bool ok;
        if (ahead.valid() && ahead_gi == gi) { ok = ahead.get(); slot = ahead_slot; }
        else { if (ahead.valid()) ahead.get(); ok = start_decode(gi, 0).get(); }
        ahead_gi = (size_t)-1;
        WindowJob *job = &jobs[slot];
        if (!job->timing.empty()) { std::fputs(job->timing.c_str(), warner.err); job->timing.clear(); }
        if (ok && gi + 1 < regions.size() && par_ok(gi + 1)) { ahead_slot = slot ^ 1; ahead_gi = gi + 1; ahead = start_decode(gi + 1, ahead_slot); }
        if (!ok) return nullptr;
        if (job->cand_overflow && warner.collecting()) return nullptr;      // a BAM full of untagged reads: the per-read warning replay wants them all
        par_decode_error = par_decode_error || job->error; par_decoded += job->n_decoded; ++par_windows;
        return job;
    }
    bool uses_windows() const { for (size_t gi = 0; gi < regions.size(); ++gi) if (par_ok(gi)) return true; return false; }
    int64_t next_fbeg(size_t gi) const {   // start of the following fetch when it continues this one, else "keep nothing"
        if (gi + 1 >= regions.size() || regions[gi + 1].tid != regions[gi].tid) return INT64_MAX;
        return std::max<int64_t>((int64_t)regions[gi + 1].beg - 1, 0);
    }
};

bool is_cram_path(const std::string &p) { return p.size() > 5 && p.substr(p.size() - 5) == ".cram"; }

// @RG ID -> rank of its LB: the first @RG line of an ID wins, libraries in std::set order (R:...:92-111, 526-529)
void read_libraries(Sample &s) {
    std::set<std::string> libs; std::vector<std::pair<std::string, std::string>> id_lb;
    {
        std::istringstream ss(s.bam.text); std::string line;
        while (std::getline(ss, line)) {
            if (line.compare(0, 3, "@RG") != 0) continue;
            std::istringstream ls(line); std::string tok, id, lb; bool has_lb = false;
            while (std::getline(ls, tok, '\t')) { if (tok.compare(0, 3, "ID:") == 0) id = tok.substr(3); else if (tok.compare(0, 3, "LB:") == 0) { lb = tok.substr(3); has_lb = true; } }
            if (has_lb) { libs.insert(lb); if (!id.empty()) id_lb.emplace_back(id, lb); }
        }
    }
    for (const auto &l : libs) s.log.say("Expect library: %s in BAM\n", l.c_str());
    s.lib_names.assign(libs.begin(), libs.end());
    for (const auto &p : id_lb)
        s.rg_lib.emplace(p.first, (uint16_t)(std::lower_bound(s.lib_names.begin(), s.lib_names.end(), p.second) - s.lib_names.begin()));
    for (auto &n : s.lib_names) s.lib_ptrs.push_back(n.c_str());
    if (s.lib_ptrs.empty()) s.lib_ptrs.push_back("");
}

// The region list: the derived site list of --vcf, the -l site list or the argv regions.  False when the run stops.
bool read_regions(Sample &s) {
    const Options &o = s.o; const BamFile &bam = s.bam; Messages &log = s.log;
    std::vector<Region> &regions = s.regions;
    // one line "name b e" of a site list: its region, or the -l loop's message when the BAM has no such contig
    auto site_line = [&](const std::string &name, int b, int e) {
        auto it = bam.tid_of.find(name);
        if (it == bam.tid_of.end()) { log.say("%s not found in bam file. Region %s %i %i skipped.\n", name.c_str(), name.c_str(), b, e); return false; }
        regions.push_back({it->second, b - 1, e, true});
        return true;
    };
    if (o.vcf) {          // the derived site list: one line per counted record, in file order
        for (const VcfRecord &r : o.vcf->rec)
            s.vcf_region.push_back(r.counted && site_line(r.cols[0], r.line_pos, r.line_pos) ? (int64_t)regions.size() - 1 : -1);
    } else if (!o.fn_pos.empty()) {
        std::ifstream fp(o.fn_pos);
        if (!fp) { log.say("Failed to open region list file: %s\n", o.fn_pos.c_str()); return false; }
        std::string line;
        while (std::getline(fp, line)) {
            std::istringstream ss(line); std::string name; int b, e;
            if (!(ss >> name >> b >> e)) continue;
            site_line(name, b, e);
        }
    } else {
        int beg = 0, end = 0x7fffffff;
        for (const auto &rs : o.region_args) {
            int tid;
            parse_region(bam, rs, tid, beg, end);
            if (tid < 0) { log.say("Invalid region %s\n", rs.c_str()); return false; }
            regions.push_back({tid, beg, end, false});
        }
    }
    return true;
}

// Long regions are cut into consecutive windows so host staging and result buffers stay bounded (a 250 Mb chromosome
// at 30x would otherwise need tens of GB).  A window is just a region of the -l loop: it recomputes the site to its left
// (the 1-site halo), so the concatenated output equals the unsplit region's.  Only the last window of an argv region keeps
// argv semantics.  (With a tiny -d the max-count rule sees the window's own fetch order; SURVEY.md §8e.)
void cut_windows(Sample &s) {
    const Options &o = s.o; const BamFile &bam = s.bam; std::vector<Region> &regions = s.regions;
    // 2 Mb windows: each is decoded by all threads in ~40 ms one window ahead of the engine and needs 110 MB of page-locked memory
    // (8 Mb windows were 0.6 s slower on a 10 Mb BAM, r02t); the record-by-record paths (CRAM, device decode) keep 8 Mb
    int64_t W = std::getenv("BRC_CLI_WINDOW") ? std::atoll(std::getenv("BRC_CLI_WINDOW")) : (s.allow_parallel ? 2000000 : 8000000);
    if (o.shard_count > 1 && !std::getenv("BRC_CLI_WINDOW")) W = 1000000;      // finer units so the shards can balance
    std::vector<Region> cut;
    for (const Region &g : regions) {
        const int64_t e_eff = fetch_end(bam, g);
        if (e_eff - g.beg <= W) { cut.push_back(g); continue; }
        for (int64_t b = g.beg; b < e_eff; b += W) {
            const bool last = b + W >= e_eff;
            Region w{g.tid, (int)b, last ? g.end : (int)(b + W), last ? g.site_list : true};
            w.cont = b != g.beg;
            cut.push_back(w);
        }
    }
    regions.swap(cut);
}

// --shard RANK/COUNT: one process per GPU (SURVEY.md §8e).  The (windowed) regions are the units; each unit's weight is the
// compressed-byte span the BAI linear index gives for it — the coverage estimate the index offers without touching the data
// — and the units are cut into COUNT contiguous runs of about equal weight; this process computes run RANK.  Units are
// independent (every window recomputes its left halo site), so the concatenation of the ranks' outputs in rank order is the
// unsharded output; only the reference's never-cleared argv deletion queue does not cross a shard boundary.
void keep_shard(Sample &s) {
    const Options &o = s.o; const BamFile &bam = s.bam; std::vector<Region> &regions = s.regions;
    const int shard_rank = o.shard_rank, shard_count = o.shard_count;
    std::vector<double> wgt(regions.size(), 1.0);
    for (size_t i = 0; i < regions.size(); ++i) {
        const Region &g = regions[i];
        const int64_t e_eff = fetch_end(bam, g);
        double w = (double)std::max<int64_t>(e_eff - g.beg, 1) * 0.05;                 // no index information: 0.05 bytes per base
        if (g.tid < (int)bam.idx.size() && !bam.idx[(size_t)g.tid].linear.empty()) {
            const auto &lin = bam.idx[(size_t)g.tid].linear;
            auto off_at = [&](int64_t p) { int64_t k = std::min<int64_t>(std::max<int64_t>(p >> 14, 0), (int64_t)lin.size() - 1); while (k > 0 && lin[(size_t)k] == 0) --k; return (double)(lin[(size_t)k] >> 16); };
            const double d = off_at(e_eff + 16384) - off_at(g.beg);
            if (d > 0) w = d * (double)(e_eff - g.beg) / (double)((((e_eff + 16384) >> 14) - (g.beg >> 14)) * 16384);
        }
        wgt[i] = w;
    }
    double tot = 0; for (double w : wgt) tot += w;
    std::vector<size_t> cutpt((size_t)shard_count + 1, regions.size()); cutpt[0] = 0;
    { double acc = 0; int r = 1; for (size_t i = 0; i < regions.size() && r < shard_count; ++i) { acc += wgt[i]; while (r < shard_count && acc >= tot * r / shard_count) cutpt[(size_t)r++] = i + 1; } }
    std::vector<Region> mine(regions.begin() + (long)cutpt[(size_t)shard_rank], regions.begin() + (long)cutpt[(size_t)shard_rank + 1]);
    if (o.timing) s.log.say("[brc shard] %d/%d: units %zu..%zu of %zu\n", shard_rank, shard_count, cutpt[(size_t)shard_rank], cutpt[(size_t)shard_rank + 1], regions.size());
    regions.swap(mine);
}

// `live`: print the messages as they come (else hold them in s.log).  `first_window`: start decoding the first window into
// `pool` (only when no other sample is using it).
std::unique_ptr<Sample> open_sample(const Options &o, const std::string &bam_path, double t0, FILE *live, WindowJob *pool, bool first_window) {
    std::unique_ptr<Sample> sp(new Sample(o, bam_path, pool));
    Sample &s = *sp; Messages &log = s.log; BamFile &bam = s.bam;
    s.t0 = t0; log.live = live;
    log.say("Minimum mapping quality is set to %d\n", o.min_mapq);
    if (o.dist_refused()) { log.say("Not currently supporting distributions\n"); return sp; }
    s.is_cram = is_cram_path(bam_path);
    if (s.is_cram && !s.hts.open(bam_path, o.fn_fa, bam)) {
        if (HtsSource::available()) log.say("Fail to open BAM file %s\n", bam_path.c_str());
        else log.say("CRAM input needs a host built with htslib (tools/build_htslib.sh, then python -m bam_readcount_b200.build); convert to BAM\n");
        return sp;
    }
    if (!s.is_cram && !bam.open(bam_path)) { log.say("Fail to open BAM file %s\n", bam_path.c_str()); return sp; }
    s.have_fa = !o.fn_fa.empty() && s.fa.open(o.fn_fa);
    if (!o.fn_fa.empty() && !s.have_fa) { log.say("Fail to open reference file %s\n", o.fn_fa.c_str()); return sp; }
    read_libraries(s);

    if (o.fn_pos.empty() && o.region_args.empty() && !o.vcf) {
        log.say("Whole-file mode is not supported (the reference skips its per-read pre-processing there, R:...:624); give regions or -l\n");
        return sp;
    }
    if (!(s.is_cram ? s.hts.load_index(bam_path) : bam.load_index(bam_path))) { log.say("BAM indexing file is not available.\n"); return sp; }
    if (!s.have_fa && !o.decode_only) { log.say("A reference FASTA (-f) is required in region / site-list mode\n"); return sp; }
    if (!read_regions(s)) return sp;
    s.allow_parallel = !s.is_cram && !o.device_decode;
    cut_windows(s);
    if (o.shard_count > 1) keep_shard(s);

    // decode under the CUDA start-up (first sample) or under the previous sample's compute (cohort)
    if (first_window && !s.regions.empty() && s.par_ok(0)) { s.ahead_slot = 0; s.ahead_gi = 0; s.ahead = s.start_decode(0, 0); }
    s.status = 0;
    return sp;
}

// ------------------------------------------------------------------------------------------
// The engine handles of a process.  One CUDA context, brought up once by a throw-away engine on a thread of its own while the
// first sample is opened.  A handle's library rows are fixed at brc_create, so under -p there is one handle per library count,
// kept and reused by the later samples with that count (brc_create allocates nothing on the device until first use); without
// -p every sample shares one handle.  Each handle remembers which contig it holds the reference of for every tid: tids are
// per-header, so the reference is uploaded again only when a sample's tid names another contig.
// ------------------------------------------------------------------------------------------
struct Engines {
    brc_config cfg{};
    std::thread warm; int warm_rc = BRC_OK;
    struct Handle { brc_engine *eng = nullptr; std::unordered_map<int, std::string> ref_name; };
    std::map<int32_t, Handle> handles;

    void start_warm() {
        brc_config w = cfg; w.per_lib = 0;
        warm = std::thread([this, w] { brc_engine *tmp = nullptr; warm_rc = brc_create(&w, &tmp); if (tmp) brc_destroy(tmp); });
    }
    // the handle for a sample with n_libs libraries; nullptr (message on err) when it cannot be created
    Handle *get(int32_t n_libs, const Options &o, FILE *err) {
        if (warm.joinable()) warm.join();
        const int32_t key = cfg.per_lib ? n_libs : 0;
        auto it = handles.find(key);
        if (it != handles.end()) return &it->second;
        brc_config c = cfg; c.n_libs = n_libs;
        brc_engine *eng = nullptr;
        const int rc = warm_rc != BRC_OK ? warm_rc : brc_create(&c, &eng);
        if (rc != BRC_OK) { std::fprintf(err, "brc_create: %s\n", brc_strerror(rc)); return nullptr; }
        if (o.site_filter && brc_set_site_filter_bounds(eng, &o.filter, o.has_bounds ? &o.bounds : nullptr) != BRC_OK) {
            std::fprintf(err, "brc_set_site_filter: %s\n", brc_last_error(eng)); brc_destroy(eng); return nullptr;
        }
        Handle &h = handles[key]; h.eng = eng;
        return &h;
    }
    void destroy() { for (auto &kv : handles) brc_destroy(kv.second.eng); handles.clear(); }
    ~Engines() { if (warm.joinable()) warm.join(); }
};

// ------------------------------------------------------------------------------------------
// The region loop (the two loops of the reference, R:...:574-608 and 641-657).  For each region, its source into a sink: a
// window decoded by ParallelFetcher, the compressed span (BRC_CLI_DEVICE_DECODE), or the record stream.  A window or a span is
// a batch of its own.  The sink is an engine run (Run) or, under BRC_CLI_DECODE_ONLY, the decode summary.  False when the
// sink failed (it printed why).
// ------------------------------------------------------------------------------------------
template <class Sink> bool region_loop(Sample &s, RegionFetcher &fetcher, Sink &sink) {
    const std::vector<Region> &regions = s.regions;
    for (size_t gi = 0; gi < regions.size(); ++gi) {
        const Region &g = regions[gi];
        const bool window = s.par_ok(gi), span = !window && s.o.device_decode && !s.is_cram;
        if (!sink.begin(g, window || span)) return false;
        WindowJob *job = window ? s.decoded_window(gi) : nullptr;      // nullptr: the record stream after all
        // samfetch(in, idx, ref, d.beg-1, d.end): records with tid, endpos > max(beg-1,0), pos < end, in file order
        const int64_t fbeg = std::max<int64_t>((int64_t)g.beg - 1, 0), fend = g.end;
        auto read = [&](const Rec &r) { sink.read(r); };
        bool ok = true;
        if (job) ok = sink.window(*job);
        else if (span) ok = sink.span(g, fbeg, fend);
        else if (s.is_cram) s.hts.fetch(g.tid, fbeg, fend, read);
        else fetcher.fetch(g.tid, fbeg, fend, s.next_fbeg(gi), read);
        if (job || span) fetcher.active = false;
        if (!ok || !sink.end(job || span, gi + 1 == regions.size())) return false;
    }
    return true;
}

// BRC_CLI_DECODE_ONLY: no engine.  Each region prints what it received, "tid beg end reads sum(pos) sum(qual)", so that BGZF,
// the index and the region fetch can be checked without a GPU.
struct DecodeSummary {
    int out_fd;
    const Region *g = nullptr; int64_t n = 0, psum = 0, qsum = 0;
    bool begin(const Region &r, bool) { g = &r; n = psum = qsum = 0; return true; }
    bool window(const WindowJob &job) {
        const brc_read_batch &b = job.batch;
        n = b.n_reads;
        for (int64_t i = 0; i < b.n_reads; ++i) psum += b.pos[i];
        for (uint64_t k = b.qual_off[0]; k < b.qual_off[b.n_reads]; ++k) qsum += b.qual[k];
        return true;
    }
    bool span(const Region &, int64_t, int64_t) { return true; }   // device decode needs an engine: not taken here
    void read(const Rec &r) {
        if (r.flag & 4) return;
        int64_t q = 0;             // a local sum: the quality bytes may alias qsum, which would be stored once per byte
        for (int k = 0; k < r.l_qseq; ++k) q += r.qual[k];
        ++n; psum += r.pos; qsum += q;
    }
    bool end(bool, bool) {
        dprintf(out_fd, "%d\t%d\t%d\t%lld\t%lld\t%lld\n", g->tid, g->beg, g->end, (long long)n, (long long)psum, (long long)qsum);
        return true;
    }
};

// One sample's run on an engine handle, the sink of its region loop.  Regions are pushed as they come and computed in batches
// (flush): text to out, or, with --vcf, the answers to vcf_ans.  Messages go to err.
struct Run {
    const Options &o; Sample &s; Engines::Handle &h; brc_engine *eng; Out &out; FILE *err;
    const Vcf *vcf; VcfAnswers *vcf_ans;
    const bool vcf_stream;        // --vcf: a single-sample run writes the records in file order, each once its region's batch is computed
    std::vector<int64_t> vcf_rec_of_region; size_t vcf_next = 0;
    std::vector<const char *> rg_ids; std::vector<uint16_t> rg_libs;   // the read groups of brc_push_bam_span
    std::string chrom;
    int64_t batch_first = 0, batch_n = 0;            // the regions begun since the last brc_reset
    int64_t pushed = 0; int push_rc = BRC_OK;        // reads pushed one by one since then, and the first failure
    int64_t warn_total[4] = {0, 0, 0, 0};
    double t_decode = 0, t_compute = 0, t_format = 0, t_ref = 0, t_results = 0, t_reset = 0, ms_alleles = 0, ms_complex = 0, d1 = 0;

    Run(const Options &opt, Sample &smp, Engines::Handle &hd, Out &dst, FILE *e, VcfAnswers *ans)
        : o(opt), s(smp), h(hd), eng(hd.eng), out(dst), err(e), vcf(opt.vcf), vcf_ans(ans), vcf_stream(opt.vcf && !opt.vcf_samples),
          vcf_rec_of_region(smp.regions.size(), -1) {
        for (size_t k = 0; k < s.vcf_region.size(); ++k) if (s.vcf_region[k] >= 0) vcf_rec_of_region[(size_t)s.vcf_region[k]] = (int64_t)k;
        for (const auto &kv : s.rg_lib) { rg_ids.push_back(kv.first.c_str()); rg_libs.push_back(kv.second); }
    }
    bool fail(const char *what) { std::fprintf(err, "%s: %s\n", what, brc_last_error(eng)); return false; }

    // ---- the sink ----
    bool begin(const Region &g, bool own_batch) {
        if (!reference(g)) return false;
        d1 = now();
        if (own_batch && pushed > 0 && !flush()) return false;     // whatever smaller regions are pending goes out first
        brc_begin_region(eng, g.tid, g.beg, g.end, g.site_list ? 1 : 0);
        ++batch_n;
        s.warner.begin_region(g.tid, g.beg, g.end, g.cont);
        return true;
    }
    bool window(WindowJob &job) {
        // ONE borrowed batch (the engine streams it to the GPU in chunks) while the next window is already being decoded
        for (Slice &sl : job.slices) s.warner.take(sl.cands);
        if (job.batch.n_reads > 0 && brc_push_reads(eng, &job.batch) != BRC_OK) return fail("brc_push_reads");
        return true;
    }
    bool span(const Region &g, int64_t fbeg, int64_t fend) {
        // f-2: hand the engine the compressed span; it inflates, frames and computes on the device
        SpanBuilder sb;
        if (!sb.build(s.bam, g.tid, fbeg, fend)) return true;
        brc_bam_span sp{}; sp.comp = sb.comp.data(); sp.comp_len = (int64_t)sb.comp.size(); sp.n_entry = (int64_t)sb.entries.size(); sp.entry = sb.entries.data();
        sp.end_voff = sb.end_voff; sp.tid = g.tid; sp.n_rg = (int32_t)rg_ids.size(); sp.rg_id = rg_ids.data(); sp.rg_lib = rg_libs.data();
        if (brc_push_bam_span(eng, &sp) != BRC_OK) return fail("brc_push_bam_span");
        return true;
    }
    void read(const Rec &r) {
        const uint16_t lib = rec_lib(r, s.rg_lib, o.per_lib);
        s.warner.consider(r, lib);
        const int prc = brc_push_read(eng, r.tid, r.pos, r.flag, r.mapq, lib, r.l_qseq, r.nm, r.sm, r.n_cigar, r.cigar, r.seq, r.qual);
        if (prc != BRC_OK && push_rc == BRC_OK) push_rc = prc;
        ++pushed;
    }
    bool end(bool own_batch, bool last) {
        if (push_rc != BRC_OK) return fail("brc_push_read");
        brc_end_region(eng);
        t_decode += now() - d1;
        // a window's batch is borrowed until its text is out, and a span is one batch; record-stream regions go out in batches
        // at region boundaries (the deletion queue of the argv loop is carried by the engine, brc_set_queue_carry)
        return !(own_batch || last || pushed > 1500000) || flush();
    }

    // load_reference: the whole chromosome, unless the handle holds this contig for the tid already
    bool reference(const Region &g) {
        const double d0 = now();
        const std::string &contig = s.bam.names[(size_t)g.tid];
        auto loaded = h.ref_name.find(g.tid);
        if (loaded != h.ref_name.end() && loaded->second == contig) return true;
        h.ref_name.erase(g.tid);
        if (!s.fa.fetch(contig, chrom)) { std::fprintf(err, "Failed to fetch %s from %s\n", contig.c_str(), o.fn_fa.c_str()); return false; }
        if (brc_set_reference(eng, g.tid, contig.c_str(), (int64_t)chrom.size(), 0, chrom.data(), (int64_t)chrom.size()) != BRC_OK) return fail("brc_set_reference");
        h.ref_name[g.tid] = contig;
        t_ref += now() - d0;
        return true;
    }

    // ---- one batch: its queries (--vcf), compute, its results as text or answers, its warnings, reset ----
    bool flush() {
        if (vcf && vcf_set_queries(eng, *vcf, vcf_rec_of_region.data() + batch_first, batch_n, err) != BRC_OK) return false;
        const double c0 = now();
        const int rc = brc_compute(eng);
        t_compute += now() - c0;
        if (rc != BRC_OK) return fail("brc_compute");
        if (!(vcf ? answers() : text())) return false;
        batch_first += batch_n; batch_n = 0; pushed = 0;
        warnings();
        const double r0 = now();
        const int rr = brc_reset(eng);
        t_reset += now() - r0;
        return rr == BRC_OK;
    }
    bool text() {
        brc_results res{};
        const double g0 = now();
        if (o.site_filter) {          // only the selected sites came back: no dense view, the region table is all the loop needs
            brc_selected_results sel{};
            if (brc_get_selected_results(eng, &sel) != BRC_OK) return fail("brc_get_selected_results");
            res.n_regions = sel.n_regions; res.regions = sel.regions;
        } else if (brc_get_results(eng, &res) != BRC_OK) return fail("brc_get_results");
        const double f0 = now();
        t_results += f0 - g0;
        const char *const *libs = s.lib_ptrs.data();
        const bool argv_chain = res.n_regions > 1 && !res.regions[0].site_list_mode;   // never-cleared deletion queue: one sequential pass
        int64_t total_slots = 0;
        for (int64_t g = 0; g < res.n_regions; ++g) total_slots += res.regions[g].n_slots;
        const bool many_small = res.n_regions > 1 && total_slots <= (int64_t(1) << 22);  // a site list: all regions in one formatting pass
        if (argv_chain || many_small) {
            if (out.text(eng, -1, 0, -1, libs) < 0) return fail("format");
        } else {
            const int64_t WIN = 1 << 21;   // stream big regions in 2M-site windows (each formatted by several threads)
            for (int64_t g = 0; g < res.n_regions; ++g)
                for (int64_t first = 0; first < res.regions[g].n_slots; first += WIN)
                    if (out.text(eng, g, first, WIN, libs) < 0) return fail("format");
        }
        t_format += now() - f0;
        return true;
    }
    bool answers() {
        const double g0 = now();
        if (vcf_get_answers(eng, *vcf, vcf_rec_of_region.data() + batch_first, batch_n, *vcf_ans, err) != BRC_OK) return false;
        t_results += now() - g0;
        if (o.timing) { ms_alleles += brc_last_stage_ms(eng, 4); ms_complex += brc_last_stage_ms(eng, 5); }
        const double f0 = now();
        if (vcf_stream && !vcf_write(batch_first + batch_n)) return false;
        t_format += now() - f0;
        return true;
    }
    void warnings() {   // the batch's per-read warning lines, and the engine's event counts for the totals of -w -1
        int64_t wc[4];
        if (brc_get_warning_counts(eng, wc) == BRC_OK) for (int k = 0; k < 4; ++k) warn_total[k] += wc[k];
        s.warner.replay();
    }

    // every record not yet written whose region is done (or that has none)
    bool vcf_write(int64_t regions_done) {
        std::string out;
        for (; vcf_next < s.vcf_region.size() && s.vcf_region[vcf_next] < regions_done; ++vcf_next) vcf_line(*vcf, vcf_next, vcf_ans, out);
        return write_out(out);
    }
    bool write_out(const std::string &text) {
        if (out.write(text)) return true;
        std::fprintf(err, "writing the VCF: %s\n", std::strerror(errno));
        return false;
    }
};

// The end of a sample's decode: waits for a window decoded ahead, reports a decode error, and under BRC_CLI_TIMING the index
// seeks.  True when the input could not be decoded to its end.
bool decode_report(Sample &s, const RegionFetcher &fetcher, FILE *err) {
    const bool decode_error = s.bam.bz.error || s.hts.error || s.par_decode_error;
    if (s.ahead.valid()) s.ahead.get();
    if (decode_error) std::fprintf(err, "[E::bgzf_read] %s: truncated or corrupt BGZF block / BAM record — the output above is incomplete\n", s.path.c_str());
    if (s.o.timing) std::fprintf(err, "[brc timing] index seeks %llu  records decoded %llu  (+ %llu records in %llu windows decoded by %d threads)\n", (unsigned long long)fetcher.n_seeks,
                                 (unsigned long long)fetcher.n_decoded, (unsigned long long)s.par_decoded, (unsigned long long)s.par_windows, s.pf.n_threads);
    return decode_error;
}

// One sample's region loop: text to out, messages to err.  With --vcf the answers go to `vcf_ans`, and a single-sample run
// streams the VCF to out as its batches complete.  Returns the exit status of the run on this input alone (0 or 1), or -1
// when no engine could be created.
int run_sample(const Options &o, Engines &engines, Sample &s, Out &out, FILE *err, double t_main0, VcfAnswers *vcf_ans) {
    std::fputs(s.log.held.c_str(), err);
    if (s.status != 0) return 1;
    s.warner.err = err;
    RegionFetcher fetcher(s.bam);
    if (o.decode_only) {
        DecodeSummary summary{out.fd};
        region_loop(s, fetcher, summary);
        return decode_report(s, fetcher, err) ? 1 : 0;
    }
    Engines::Handle *h = engines.get((int32_t)s.lib_names.size(), o, err);
    if (!h) return -1;
    // nothing left from an earlier sample: no pushed reads (a sample that failed mid-way) and no queued deletion
    // (switching the carry empties the queue); the argv loop's queue is then carried across this sample's flushes
    brc_reset(h->eng); brc_set_queue_carry(h->eng, 0); brc_set_queue_carry(h->eng, 1);
    Run run(o, s, *h, out, err, vcf_ans);
    if (run.vcf_stream && !run.write_out(vcf_header(*o.vcf))) return 1;
    const double t_loop0 = now();
    if (!region_loop(s, fetcher, run)) return 1;
    if (run.vcf_stream && !run.vcf_write(INT64_MAX)) return 1;
    s.warner.finish(run.warn_total);
    const bool decode_error = decode_report(s, fetcher, err);
    if (o.timing) {
        std::fprintf(err, "[brc timing] reference %.3fs  decode+push %.3fs  compute %.3fs  results %.3fs  format %.3fs  reset %.3fs  | region loop %.3fs, since main() %.3fs\n",
                     run.t_ref, run.t_decode, run.t_compute, run.t_results, run.t_format, run.t_reset, now() - t_loop0, now() - t_main0);
        std::fprintf(err, "[brc timing] startup (CUDA context, header, index, first window) %.3fs\n", t_loop0 - s.t0);
        if (o.vcf) std::fprintf(err, "[brc timing] allele kernels %.3f ms\n", run.ms_alleles);
        if (o.vcf_complex) std::fprintf(err, "[brc timing] complex kernel %.3f ms\n", run.ms_complex);
    }
    return decode_error ? 1 : 0;
}

// Everything is printed: leave without tearing down the CUDA context, the page-locked buffers and the thread pools one by
// one (a teardown that takes a noticeable part of a second) — the kernel reclaims them.  BRC_CLI_CLEAN_EXIT=1 tears down.
// A run that failed before it asked for an engine still waits for the CUDA start-up thread, as returning from main() would.
int leave(Engines &engines, std::unique_ptr<Sample> &last, int status) {
    if (engines.warm.joinable()) engines.warm.join();
    if (!std::getenv("BRC_CLI_CLEAN_EXIT")) {
        std::fflush(nullptr);
        _exit(status);
    }
    last.reset();
    engines.destroy();
    return status;
}

// The output files of one sample (OUT and ERR of a cohort sample, the ERR of a --vcf-samples sample).  Nothing is created or
// emptied until all are open: a sample that cannot have them all leaves no new file behind and no earlier file truncated.
bool open_outputs(const std::vector<const std::string *> &path, std::vector<int> &fd, std::string &why) {
    const size_t n = path.size();
    fd.assign(n, -1); std::vector<bool> made(n, false);
    auto undo = [&](size_t m) { for (size_t j = 0; j < m; ++j) { ::close(fd[j]); if (made[j]) ::unlink(path[j]->c_str()); } };
    for (size_t i = 0; i < n; ++i) {
        fd[i] = ::open(path[i]->c_str(), O_WRONLY | O_CREAT | O_EXCL | O_CLOEXEC, 0666);
        if (fd[i] >= 0) made[i] = true;
        else if (errno == EEXIST) fd[i] = ::open(path[i]->c_str(), O_WRONLY | O_CLOEXEC);
        if (fd[i] < 0) { why = "cannot open " + *path[i] + ": " + std::strerror(errno); undo(i); return false; }
    }
    for (size_t i = 0; i < n; ++i)
        if (::ftruncate(fd[i], 0) != 0) { why = "cannot truncate " + *path[i] + ": " + std::strerror(errno); undo(n); return false; }
    return true;
}

// The lines of a sample list (--bam-list, --vcf-samples): every non-empty line, a trailing '\r' dropped, split at tabs into 2 or 3
// non-empty fields (`shape` names them in the message), with its line number.  False with a message on stderr.
struct ListLine { int ln; std::vector<std::string> fld; };
bool read_list(const std::string &list_path, const char *shape, std::vector<ListLine> &out) {
    std::ifstream f(list_path);
    if (!f) { std::fprintf(stderr, "Failed to open sample list file: %s\n", list_path.c_str()); return false; }
    std::string line; int ln = 0;
    while (std::getline(f, line)) {
        ++ln;
        if (!line.empty() && line.back() == '\r') line.pop_back();
        if (line.empty()) continue;
        std::vector<std::string> fld = split(line, '\t');
        const bool empty_field = std::any_of(fld.begin(), fld.end(), [](const std::string &x) { return x.empty(); });
        if ((fld.size() != 2 && fld.size() != 3) || empty_field) {
            std::fprintf(stderr, "%s:%d: a sample line is %s\n", list_path.c_str(), ln, shape);
            return false;
        }
        out.push_back({ln, std::move(fld)});
    }
    if (out.empty()) { std::fprintf(stderr, "%s lists no sample\n", list_path.c_str()); return false; }
    return true;
}

// Adds an output path to `used` (absolute and normalised); false, with a message on stderr, when an earlier sample has it.
bool claim_output(std::set<std::string> &used, const std::string &list_path, int ln, const std::string &path) {
    std::error_code ec;
    std::filesystem::path abs = std::filesystem::absolute(path, ec);
    if (ec) abs = path;
    if (used.insert(abs.lexically_normal().string()).second) return true;
    std::fprintf(stderr, "%s:%d: %s is already the output of an earlier sample\n", list_path.c_str(), ln, path.c_str());
    return false;
}

// One input of a sample list and where its STDOUT and STDERR go: files, or the process's own when the path is empty.
struct ListSample { std::string in, out, err; };

// Runs the samples of a list in order, each exactly as a run on its input alone (DESIGN.md §11).  `vcf_ans` (--vcf-samples):
// sample k's answers go to vcf_ans[k], which is marked failed when the sample fails.  A sample whose own run would exit 1, or
// whose output files cannot be opened or written, gets one line on the process's STDERR and the list goes on.  Returns the number
// of failed samples, or -1 when no engine could be created: the remaining samples are not run.
//
// While a sample with an ERR file runs, file descriptor 2 is that file, so whatever a library prints there (htslib's CRAM and
// index messages) lands in that sample's ERR in the order its own run prints it.  The next sample is opened on a worker thread
// while the current one computes, holding its messages until its turn, unless it is a CRAM: htslib prints while it opens one, so
// a CRAM is opened at its turn.  Its first window is decoded ahead only when the current sample does not use the process's two
// window jobs, so page-locked window memory stays at two jobs, reused from sample to sample.
int run_list(const Options &o, Engines &engines, const std::vector<ListSample> &list, std::vector<VcfAnswers> *vcf_ans, double t_main0) {
    std::unique_ptr<WindowJob[]> pool(new WindowJob[2]);
    auto open_ahead = [&](size_t k, bool first_window) {
        return std::async(std::launch::async, open_sample, std::cref(o), list[k].in, now(), nullptr, pool.get(), first_window);
    };
    if (!o.decode_only && !o.dist_refused()) engines.start_warm();
    std::future<std::unique_ptr<Sample>> ahead;                          // sample k, opened ahead of its turn
    if (!is_cram_path(list[0].in)) ahead = open_ahead(0, true);          // under the CUDA start-up
    int n_failed = 0;
    for (size_t k = 0; k < list.size(); ++k) {
        const ListSample &e = list[k];
        const bool next_ahead = k + 1 < list.size() && !is_cram_path(list[k + 1].in);
        auto failed = [&](const char *fmt, const std::string &what) {
            ++n_failed;
            if (vcf_ans) (*vcf_ans)[k].failed = true;
            std::fprintf(stderr, fmt, k + 1, e.in.c_str(), what.c_str());
        };
        std::vector<const std::string *> paths; std::vector<int> fd; std::string why;
        if (!e.out.empty()) paths.push_back(&e.out);
        if (!e.err.empty()) paths.push_back(&e.err);
        if (!open_outputs(paths, fd, why)) {
            if (ahead.valid()) ahead.get();
            failed("sample %zu (%s) failed: %s\n", why);
            if (next_ahead) ahead = open_ahead(k + 1, true);
            continue;
        }
        const int out_fd = e.out.empty() ? STDOUT_FILENO : fd[0], err_fd = e.err.empty() ? -1 : fd.back();
        Out out;                                                 // (--vcf-samples: the samples write no STDOUT)
        out.fd = out_fd;
        if (!e.out.empty() && !out.open(o, out_fd, why)) {
            for (int f : fd) ::close(f);
            if (ahead.valid()) ahead.get();
            failed("sample %zu (%s) failed: %s\n", why);
            if (next_ahead) ahead = open_ahead(k + 1, true);
            continue;
        }
        int saved_fd2 = -1;
        if (err_fd >= 0) { std::fflush(stderr); saved_fd2 = ::dup(2); ::dup2(err_fd, 2); }
        std::unique_ptr<Sample> cur = ahead.valid() ? ahead.get() : open_sample(o, e.in, now(), stderr, pool.get(), true);
        if (next_ahead) ahead = open_ahead(k + 1, !cur->uses_windows());
        const int rc = run_sample(o, engines, *cur, out, stderr, t_main0, vcf_ans ? &(*vcf_ans)[k] : nullptr);
        cur.reset();                                                     // htslib's closing lines still go to this ERR
        if (err_fd >= 0) {
            if (std::fflush(stderr) != 0) why = e.err + ": " + std::strerror(errno);
            else if (std::ferror(stderr)) why = e.err + ": write error";
            std::clearerr(stderr);
            ::dup2(saved_fd2, 2);
            ::close(saved_fd2);
            if (::close(err_fd) != 0 && why.empty()) why = e.err + ": " + std::strerror(errno);
        }
        if (!out.close() && why.empty()) why = e.out + ": " + std::strerror(errno);
        if (out_fd != STDOUT_FILENO && ::close(out_fd) != 0 && why.empty()) why = e.out + ": " + std::strerror(errno);
        const std::string see = e.err.empty() ? "the lines above" : e.err;
        if (rc < 0) {
            std::fprintf(stderr, "sample %zu (%s): no engine could be created (see %s); the remaining samples are not run\n", k + 1, e.in.c_str(), see.c_str());
            return -1;
        }
        if (!why.empty()) failed("sample %zu (%s) failed: writing %s\n", why);
        else if (rc != 0) failed("sample %zu (%s) failed: see %s\n", see);
    }
    return n_failed;
}

// --bam-list FILE: a cohort in one process.  Each non-empty line of FILE is INPUT<TAB>OUT[<TAB>ERR] (ERR defaults to OUT.log);
// OUT and ERR receive exactly what a run on INPUT alone with the same options and regions prints on STDOUT and STDERR.  A
// sample whose own run would exit 1 is reported on this process's STDERR and the batch goes on; the exit status is 1 when any
// sample failed.  The list is checked whole before any sample runs.
int run_cohort(const Options &o, Engines &engines, const std::string &list_path, double t_main0) {
    std::vector<ListLine> lines;
    if (!read_list(list_path, "INPUT<TAB>OUT or INPUT<TAB>OUT<TAB>ERR", lines)) return 1;
    std::vector<ListSample> list;
    std::set<std::string> outputs;
    for (const ListLine &l : lines) {
        ListSample e{l.fld[0], l.fld[1], l.fld.size() == 3 ? l.fld[2] : l.fld[1] + ".log"};
        if (!claim_output(outputs, list_path, l.ln, e.out) || !claim_output(outputs, list_path, l.ln, e.err)) return 1;
        list.push_back(std::move(e));
    }
    std::unique_ptr<Sample> none;
    const int n_failed = run_list(o, engines, list, nullptr, t_main0);
    if (n_failed < 0) return leave(engines, none, 1);
    if (o.timing) std::fprintf(stderr, "[brc timing] cohort: %zu samples (%d failed) in %.3fs since main()\n", list.size(), n_failed, now() - t_main0);
    return leave(engines, none, n_failed ? 1 : 0);
}

// --vcf FILE --vcf-samples LIST: each non-empty line of LIST is NAME<TAB>INPUT[<TAB>ERR].  Every sample runs as the list's
// next sample (run_list) and fills its answers; after the last one the VCF is written once, sample NAME's column holding what
// `--vcf FILE --vcf-sample NAME INPUT` writes there, or '.' in all five fields when the sample failed.  ERR (the process's
// STDERR without one) receives that run's STDERR.  Under BRC_CLI_DECODE_ONLY STDOUT is the samples' decode summaries in list
// order and no VCF is written, as a single-sample run writes none.
int run_vcf_samples(const Options &o, Engines &engines, const std::vector<ListSample> &list, double t_main0) {
    std::vector<VcfAnswers> ans(list.size(), VcfAnswers(*o.vcf));
    std::unique_ptr<Sample> none;
    const int n_failed = run_list(o, engines, list, &ans, t_main0);
    if (n_failed < 0) return leave(engines, none, 1);
    int status = n_failed ? 1 : 0;
    if (!o.decode_only) {
        Out dst; std::string why;
        if (!dst.open(o, STDOUT_FILENO, why)) { std::fprintf(stderr, "%s\n", why.c_str()); return leave(engines, none, 1); }
        std::string out = vcf_header(*o.vcf);
        bool ok = true;
        for (size_t ri = 0; ri < o.vcf->rec.size() && ok; ++ri) {
            vcf_line(*o.vcf, ri, ans.data(), out);
            if (out.size() >= (size_t(1) << 22)) { ok = dst.write(out); out.clear(); }
        }
        ok = ok && dst.write(out);
        if (!dst.close()) ok = false;
        if (!ok) { std::fprintf(stderr, "writing the VCF: %s\n", std::strerror(errno)); status = 1; }
    }
    if (o.timing) std::fprintf(stderr, "[brc timing] vcf-samples: %zu samples (%d failed) in %.3fs since main()\n", list.size(), n_failed, now() - t_main0);
    return leave(engines, none, status);
}

}  // namespace brc::cli

using namespace brc::cli;

int main(int argc, char **argv) {
    const double t_main0 = now();
    Options o;
    std::string bam_list, vcf_path, vcf_sample, vcf_samples; bool shard_given = false, vcf_sample_given = false;
    static option lo[] = {{"help", 0, 0, 'h'}, {"version", 0, 0, 'v'}, {"min-mapping-quality", 1, 0, 'q'}, {"min-base-quality", 1, 0, 'b'},
                          {"max-count", 1, 0, 'd'}, {"site-list", 1, 0, 'l'}, {"reference-fasta", 1, 0, 'f'}, {"print-individual-mapq", 1, 0, 'D'},
                          {"per-library", 0, 0, 'p'}, {"max-warnings", 1, 0, 'w'}, {"insertion-centric", 0, 0, 'i'}, {"shard", 1, 0, 1000},
                          {"min-alt-count", 1, 0, 1001}, {"min-alt-fraction", 1, 0, 1002}, {"bam-list", 1, 0, 1003},
                          {"vcf", 1, 0, 1004}, {"vcf-sample", 1, 0, 1005}, {"vcf-samples", 1, 0, 1006},
                          {"vcf-complex", 0, 0, 1007}, {"alt-min", 1, 0, 1008}, {"alt-max", 1, 0, 1009}, {"bgzf", 0, 0, 1010}, {0, 0, 0, 0}};
    long min_alt_count = 0; double min_alt_fraction = -1.0;       // site filter (brc_set_site_filter); off unless one is given
    bool help = false, version = false;
    for (int c; (c = getopt_long(argc, argv, "hvq:b:d:l:f:D:pw:i", lo, nullptr)) != -1;) {
        switch (c) {
        case 'h': help = true; break; case 'v': version = true; break;
        case 'q': o.min_mapq = std::atoi(optarg); break; case 'b': o.min_bq = std::atoi(optarg); break; case 'd': o.max_cnt = std::atoi(optarg); break;
        case 'l': o.fn_pos = optarg; break; case 'f': o.fn_fa = optarg; break; case 'D': o.dist_arg = optarg; break;
        case 'p': o.per_lib = true; break; case 'w': o.max_warn = std::atoll(optarg); break; case 'i': o.ic = true; break;
        case 1000: if (std::sscanf(optarg, "%d/%d", &o.shard_rank, &o.shard_count) != 2 || o.shard_count < 1 || o.shard_rank < 0 || o.shard_rank >= o.shard_count) { std::fprintf(stderr, "--shard wants RANK/COUNT with 0 <= RANK < COUNT\n"); return 1; }
                   shard_given = true; break;
        case 1001: {
            char *end = nullptr; errno = 0;
            min_alt_count = std::strtol(optarg, &end, 10);
            if (errno || end == optarg || *end || min_alt_count < 1 || min_alt_count > INT32_MAX) { std::fprintf(stderr, "--min-alt-count wants an integer N >= 1\n"); return 1; }
            break;
        }
        case 1002: {
            char *end = nullptr; errno = 0;
            min_alt_fraction = std::strtod(optarg, &end);
            if (errno || end == optarg || *end || !(min_alt_fraction >= 0.0 && min_alt_fraction <= 1.0)) { std::fprintf(stderr, "--min-alt-fraction wants a number F with 0 <= F <= 1\n"); return 1; }
            break;
        }
        case 1003: bam_list = optarg; break;
        case 1004: vcf_path = optarg; break;
        case 1005: vcf_sample = optarg; vcf_sample_given = true; break;
        case 1006: vcf_samples = optarg; break;
        case 1007: o.vcf_complex = true; break;
        case 1008: if (!parse_bound("--alt-min", optarg, o.bounds.lo_set, o.bounds.lo)) return 1; break;
        case 1009: if (!parse_bound("--alt-max", optarg, o.bounds.hi_set, o.bounds.hi)) return 1; break;
        case 1010: o.bgzf = true; break;
        default: usage(); return 1;
        }
    }
    for (int k = 0; k < BRC_N_STATS; ++k)
        if (((o.bounds.lo_set & o.bounds.hi_set) >> k & 1u) && o.bounds.lo[k] > o.bounds.hi[k]) {
            std::fprintf(stderr, "--alt-min %s is larger than --alt-max %s\n", kEntryFields[k], kEntryFields[k]); return 1;
        }
    o.has_bounds = (o.bounds.lo_set | o.bounds.hi_set) != 0;
    o.site_filter = min_alt_count > 0 || min_alt_fraction >= 0.0 || o.has_bounds;
    o.filter.min_alt_count = (int32_t)std::max<long>(min_alt_count, 1); o.filter.min_alt_fraction = std::max(min_alt_fraction, 0.0);
    if (version) { std::printf("bam-readcount version: b200 (engine ABI %d)\n", brc_abi_version()); return 1; }   // R:...:467-470 (exit 1)
    if (help || (optind >= argc && bam_list.empty() && vcf_samples.empty())) { usage(); return 1; }                 // R:...:472-475
    if (!bam_list.empty() && shard_given) { std::fprintf(stderr, "--bam-list and --shard cannot be combined: shard a cohort by splitting its list\n"); return 1; }
    Vcf vcf;
    if (vcf_sample_given && vcf_path.empty()) { std::fprintf(stderr, "--vcf-sample needs --vcf\n"); return 1; }
    if (o.vcf_complex && vcf_path.empty()) { std::fprintf(stderr, "--vcf-complex needs --vcf\n"); return 1; }
    if (!vcf_samples.empty()) {
        const char *why = vcf_path.empty() ? "--vcf-samples needs --vcf" : vcf_sample_given ? "--vcf-samples cannot be combined with --vcf-sample"
                        : optind < argc ? "--vcf-samples takes no positional argument: the inputs are in its list" : nullptr;
        if (why) { std::fprintf(stderr, "%s\n", why); return 1; }
    }
    std::vector<ListSample> vcf_list;     // --vcf-samples
    std::vector<std::string> vcf_names;
    if (!vcf_path.empty()) {
        const char *clash = !o.fn_pos.empty() ? "-l" : optind + 1 < argc ? "positional regions" : o.per_lib ? "-p" : o.has_bounds ? "--alt-min/--alt-max" : o.site_filter ? "--min-alt-count/--min-alt-fraction"
                          : shard_given ? "--shard" : !bam_list.empty() ? "--bam-list" : nullptr;
        if (clash) { std::fprintf(stderr, "--vcf cannot be combined with %s\n", clash); return 1; }
        if (vcf_sample_given) vcf_names.push_back(vcf_sample);
        if (!vcf_samples.empty()) {
            std::vector<ListLine> lines;
            if (!read_list(vcf_samples, "NAME<TAB>INPUT or NAME<TAB>INPUT<TAB>ERR", lines)) return 1;
            std::set<std::string> names, errs;
            for (const ListLine &l : lines) {
                if (!names.insert(l.fld[0]).second) { std::fprintf(stderr, "%s:%d: sample %s is listed twice\n", vcf_samples.c_str(), l.ln, l.fld[0].c_str()); return 1; }
                if (l.fld.size() == 3 && !claim_output(errs, vcf_samples, l.ln, l.fld[2])) return 1;
                vcf_names.push_back(l.fld[0]);
                vcf_list.push_back({l.fld[1], "", l.fld.size() == 3 ? l.fld[2] : ""});
            }
        }
        std::string why;
        if (!parse_vcf(vcf_path, vcf_names, vcf_samples.empty() ? "--vcf-sample" : "--vcf-samples", o.vcf_complex, vcf, why)) { std::fprintf(stderr, "--vcf: %s\n", why.c_str()); return 1; }
        o.vcf = &vcf;
        o.vcf_samples = !vcf_samples.empty();
    }
    o.decode_only = std::getenv("BRC_CLI_DECODE_ONLY") != nullptr;   // test hook: exercise BGZF/BAI/region fetch without a GPU
    o.device_decode = std::getenv("BRC_CLI_DEVICE_DECODE") != nullptr && !o.decode_only;
    o.timing = std::getenv("BRC_CLI_TIMING") != nullptr;
    o.device = std::getenv("BRC_DEVICE") ? std::atoi(std::getenv("BRC_DEVICE")) : 0;

    Engines engines;
    brc_config &cfg = engines.cfg;
    cfg.min_mapq = o.min_mapq; cfg.min_bq = o.min_bq; cfg.max_cnt = o.max_cnt; cfg.per_lib = o.per_lib; cfg.insertion_centric = o.ic;
    cfg.n_libs = 0; cfg.device = o.device;
    if (!bam_list.empty()) {
        o.region_args.assign(argv + optind, argv + argc);          // every positional argument is a region of every sample
        return run_cohort(o, engines, bam_list, t_main0);
    }
    if (o.vcf_samples) return run_vcf_samples(o, engines, vcf_list, t_main0);
    const std::string bam_path = argv[optind];
    o.region_args.assign(argv + optind + 1, argv + argc);
    // CUDA context creation takes a second or two: do it while the BAM header, index and FASTA index are read
    if (!o.decode_only && !o.dist_refused()) engines.start_warm();
    std::unique_ptr<WindowJob[]> pool(new WindowJob[2]);
    std::unique_ptr<Sample> s = open_sample(o, bam_path, t_main0, stderr, pool.get(), true);
    std::vector<VcfAnswers> vcf_ans;
    if (o.vcf) vcf_ans.emplace_back(vcf);
    Out out; std::string why;
    if (!out.open(o, STDOUT_FILENO, why)) { std::fprintf(stderr, "%s\n", why.c_str()); return leave(engines, s, 1); }
    int rc = run_sample(o, engines, *s, out, stderr, t_main0, vcf_ans.data());
    if (!out.close()) {                   // a failure a write already reported is not reported twice
        if (!out.failed) std::fprintf(stderr, "writing the output: %s\n", std::strerror(errno));
        rc = 1;
    }
    return leave(engines, s, rc < 0 ? 1 : rc);
}

