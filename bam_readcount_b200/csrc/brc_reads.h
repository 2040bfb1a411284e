// brc_reads.h — the read columns of a brc_read_batch and the worker-thread fan-out, shared by the engine and the C++ host.
// Free of CUDA, so that the host can include it.
#pragma once
#include <algorithm>
#include <cstdint>
#include <thread>
#include <vector>

#include "../../include/brc_engine.h"

namespace brc {

// The 13 columns of a brc_read_batch as growing arrays, reads in file order.  The CIGAR, sequence and quality pools are
// indexed by offsets that start at 0.
struct ReadArrays {
    std::vector<int32_t> pos, l_qseq, nm, sm;
    std::vector<uint16_t> flag, lib;
    std::vector<uint8_t> mapq;
    std::vector<uint64_t> cigar_off{0}, seq_off{0}, qual_off{0};
    std::vector<uint32_t> cigar;
    std::vector<uint8_t> seq, qual;

    int64_t n() const { return (int64_t)pos.size(); }
    void append(int32_t p, uint16_t fl, uint8_t mq, uint16_t lb, int32_t lq, int32_t nm_tag, int32_t sm_tag, uint32_t n_cigar,
                const uint32_t *cig, const uint8_t *sq, const uint8_t *ql) {
        pos.push_back(p); flag.push_back(fl); mapq.push_back(mq); lib.push_back(lb); l_qseq.push_back(lq);
        nm.push_back(nm_tag); sm.push_back(sm_tag);
        cigar.insert(cigar.end(), cig, cig + n_cigar); cigar_off.push_back(cigar.size());
        seq.insert(seq.end(), sq, sq + ((size_t)lq + 1) / 2); seq_off.push_back(seq.size());
        qual.insert(qual.end(), ql, ql + lq); qual_off.push_back(qual.size());
    }
    void clear() {
        pos.clear(); l_qseq.clear(); nm.clear(); sm.clear(); flag.clear(); lib.clear(); mapq.clear();
        cigar_off.assign(1, 0); seq_off.assign(1, 0); qual_off.assign(1, 0); cigar.clear(); seq.clear(); qual.clear();
    }
    brc_read_batch batch() const;   // a view of the arrays (tid NULL: every read is on its region's contig)
};

// The column layout of a batch, listed once: row(column, field) for each of the seven per-read columns, then
// pool(offsets, offsets field, pool, pool field) for the CIGAR, sequence and quality pools.  Both take member pointers, of
// ReadArrays and of brc_read_batch, in brc_read_batch order.
template <class Row, class Pool> void for_each_column(Row &&row, Pool &&pool) {
    row(&ReadArrays::pos, &brc_read_batch::pos); row(&ReadArrays::flag, &brc_read_batch::flag);
    row(&ReadArrays::mapq, &brc_read_batch::mapq); row(&ReadArrays::lib, &brc_read_batch::lib);
    row(&ReadArrays::l_qseq, &brc_read_batch::l_qseq); row(&ReadArrays::nm, &brc_read_batch::nm); row(&ReadArrays::sm, &brc_read_batch::sm);
    pool(&ReadArrays::cigar_off, &brc_read_batch::cigar_off, &ReadArrays::cigar, &brc_read_batch::cigar);
    pool(&ReadArrays::seq_off, &brc_read_batch::seq_off, &ReadArrays::seq, &brc_read_batch::seq);
    pool(&ReadArrays::qual_off, &brc_read_batch::qual_off, &ReadArrays::qual, &brc_read_batch::qual);
}

inline brc_read_batch ReadArrays::batch() const {
    brc_read_batch b{};
    b.n_reads = n();
    for_each_column([&](auto col, auto field) { b.*field = (this->*col).data(); },
                    [&](auto off, auto off_field, auto col, auto field) { b.*off_field = (this->*off).data(); b.*field = (this->*col).data(); });
    return b;
}

// Worker threads for n items: one more per `grain` items, at most `cap` and the core count.
inline int worker_count(int64_t n, int64_t grain, int cap) {
    const unsigned hw = std::thread::hardware_concurrency();
    return (int)std::max<int64_t>(1, std::min<int64_t>({(int64_t)(hw ? hw : 1), (int64_t)cap, n / grain + 1}));
}
// Runs work(t) for t in [0, nt): t >= 1 on threads of their own, t = 0 on the calling thread; returns when all are done.
template <class F> void fan_out(int nt, const F &work) {
    std::vector<std::thread> th;
    for (int t = 1; t < nt; ++t) th.emplace_back(work, t);
    if (nt > 0) work(0);
    for (auto &x : th) x.join();
}

}  // namespace brc
