"""GPU: the CUDA engine, called through the C ABI (libbrc_engine.so), against
  (1) the reference's golden files and the committed reference-binary outputs — text, byte-exact;
  (2) the CPU oracle on the same inputs — every raw accumulator of every computed site,
      bit-exact (integers AND the float32 sums: accumulation order is preserved);
  (3) the reference's warning counters.
"""
import numpy as np
import pytest

import cases
import golden_jobs

pytestmark = pytest.mark.gpu

JOBS = golden_jobs.jobs()
first_diff = cases.first_diff


@pytest.mark.parametrize("job", JOBS, ids=[j[0] for j in JOBS])
def test_engine_text_matches_reference_golden(job):
    _, getter, flags, site_list, golden = job
    case = getter()
    text = cases.run_engine(case, flags, site_list=site_list, dump=False).text
    want = cases.load_golden_text(golden)
    assert text == want, first_diff(text, want)


@pytest.mark.parametrize("job", JOBS, ids=[j[0] for j in JOBS])
def test_engine_accumulators_match_oracle_bit_exact(job):
    _, getter, flags, _, _ = job
    case = getter()
    # site-list semantics for both (fresh deletion queue per region) so the raw dumps are comparable
    cases.assert_same(cases.run_engine(case, flags, site_list=True), cases.run_oracle(case, flags, site_list=True),
                      fields=("dump", "warnings"))


@pytest.mark.parametrize("job", JOBS, ids=[j[0] for j in JOBS])
def test_deep_site_kernel_matches_oracle_bit_exact(job, monkeypatch):
    """Every tile of <= 2 sites forced through deep_site_kernel (read-parallel events, ordered accumulation) instead of
    pileup_kernel: same raw accumulators, warning counters and text.  (By default only tiles under >= 2048 reads take it:
    the deep-* jobs above already do.)"""
    monkeypatch.setenv("BRC_DEEP_MIN_READS", "1")
    _, getter, flags, site_list, golden = job
    case = getter()
    cases.assert_same(cases.run_engine(case, flags, site_list=True), cases.run_oracle(case, flags, site_list=True),
                      fields=("dump", "warnings"))
    text = cases.run_engine(case, flags, site_list=site_list, dump=False).text
    want = cases.load_golden_text(golden)
    assert text == want, first_diff(text, want)


def test_deep_site_kernel_is_what_runs_on_a_deep_panel(monkeypatch):
    """50 000x on one site, 8 libraries: identical results with the deep-site kernel (default) and with it disabled."""
    case = cases.deep_case(n_sites=2, depth=20000, seed=9)
    fl = dict(per_lib=True, max_cnt=100000000)
    r1 = cases.run_engine(case, fl, site_list=True)
    monkeypatch.setenv("BRC_DEEP_MIN_READS", "2147483647")
    r2 = cases.run_engine(case, fl, site_list=True)
    assert r1.dump == r2.dump and tuple(r1.warnings) == tuple(r2.warnings)
    assert r1.dump == cases.run_oracle(case, fl, site_list=True).dump


@pytest.mark.parametrize("n_libs", [12, 19])
def test_deep_site_kernel_with_more_than_eight_libraries(n_libs, monkeypatch):
    """-p panels with more libraries than one CTA's owner threads hold: the tile's libraries are spread over several CTAs
    (grid.y batches of 8), each streaming the tile's reads; identical to the oracle and to pileup_kernel."""
    case = cases.deep_case(n_sites=2, depth=3000, seed=13, n_libs=n_libs)
    fl = dict(per_lib=True, max_cnt=100000000, min_bq=10)
    want = cases.run_oracle(case, fl, site_list=True)
    cases.assert_same(cases.run_engine(case, fl, site_list=True), want, fields=("dump", "warnings"))
    monkeypatch.setenv("BRC_DEEP_MIN_READS", "2147483647")
    assert cases.run_engine(case, fl, site_list=True).dump == want.dump


def test_exact_arithmetic_shortcuts_match_ieee_intrinsics():
    """K1 replaces __fdiv_rn by a reciprocal + one FMA correction and float<->double conversions by bit
    casts for read lengths <= 2048; every (numerator, divisor) pair it can see must agree with IEEE."""
    from bam_readcount_b200.engine import Engine
    e = Engine()
    try:
        assert e.lib.brc_selftest_fastmath(e.h, 2048) == 0
    finally:
        e.close()


def test_sharded_engine_equals_unsharded():
    """Multi-GPU sharding rule (one engine per shard, contiguous site ranges, 1-site halo): the concatenation
    of the shards' output equals the unsharded output, deletions across the cut included."""
    from bam_readcount_b200 import shard
    from bam_readcount_b200.engine import Engine
    case = cases.synthetic_case(L=9000, depth=30, seed=21, regions=((0, 501, 8500),))
    name, clen, seq, wb = case["contigs"][0]
    flags = dict(per_lib=True, insertion_centric=True)

    def run(b, e):
        eng = Engine(lib_names=case["lib_names"], **flags)
        try:
            eng.set_reference(0, name, clen, seq, wb)
            eng.begin_region(0, b, e, True)
            eng.push_reads(case["batch"].select(shard.shard_read_indices(case["batch"], 0, b, e)))
            eng.end_region()
            eng.compute()
            return eng.format_text()
        finally:
            eng.close()
    whole = run(500, 8500)
    parts = "".join(run(b, e) for b, e in shard.plan_shards(case["batch"].pos, 500, 8500, 4))
    assert parts == whole
    assert len(whole.splitlines()) == 8000


def test_borrowed_and_copied_batches_agree():
    """brc_push_reads borrows a fully-admitted batch (zero-copy) and copies otherwise; both must give the same result."""
    case = cases.synthetic_case(L=6000, depth=30, seed=4, regions=((0, 1, 6000),))
    # two pushes into one region: the first is borrowed, then materialised when the second arrives
    outs = [cases.run_engine(case, dict(min_mapq=20), site_list=False, dump=False, push=push).text for push in ("one", "halves")]
    assert outs[0] == outs[1] and len(outs[0]) > 100000


def test_pipelined_push_path_many_chunks(monkeypatch):
    """The borrowed push path streams the batch in read-index chunks (H2D / kernels / D2H overlapped); force many
    tiny chunks and check every accumulator against the oracle."""
    monkeypatch.setenv("BRC_PIPE_CHUNKS", "7")
    case = cases.synthetic_case(L=20000, depth=30, seed=13, regions=((0, 1, 20000),), site_list=False)
    for flags in (dict(), dict(per_lib=True, insertion_centric=True, min_mapq=20, min_bq=20)):
        cases.assert_same(cases.run_engine(case, flags, site_list=True), cases.run_oracle(case, flags, site_list=True),
                          fields=("dump", "text"))


def _long_read_case(seed=77, L=120000):
    """Reads of 3-25 kb (beyond the reciprocal-division fast path at 2048 bp and beyond a K0/K1 shared-memory stage)."""
    import numpy as np
    from bam_readcount_b200 import synth
    from bam_readcount_b200.batch import BatchBuilder
    import edge_cases
    rng = np.random.default_rng(seed)
    ref = synth.synth_reference(L, seed)
    recs = []
    for i in range(60):
        lq = int(rng.choice([3000, 5000, 9000, 16000, 25000, 150]))
        p = int(rng.integers(10, L - 2 * lq - 100))
        ops, span = edge_cases._rand_cigar(rng, lq)
        seq = edge_cases._read_from_ref(rng, ref, p, ops, sub_rate=0.01)
        flag = 16 if rng.random() < 0.5 else 0
        recs.append(dict(tid=0, pos=p, flag=flag, mapq=int(rng.choice([60, 30, 0])), lib=int(rng.integers(0, 3)),
                         cigar="".join(f"{l}{o}" for l, o in ops), seq=seq, qual=edge_cases._quals(rng, lq, bool(flag)),
                         nm=int(rng.integers(0, 50)), sm=None, qname=f"L{i}"))
    recs.sort(key=lambda r: r["pos"])
    bb = BatchBuilder()
    for r in recs:
        bb.add_sam(**r)
    return dict(name="longreads", contigs=[("c", L, ref.tobytes(), 0)], batch=bb.build(), regions=[(0, 1, L)], site_list=True,
                lib_names=["lib0", "lib1", "lib2"])


def test_long_reads_exact_slow_paths():
    case = _long_read_case()
    for flags in (dict(), dict(per_lib=True, min_mapq=20, min_bq=20)):
        cases.assert_same(cases.run_engine(case, flags, site_list=True), cases.run_oracle(case, flags, site_list=True),
                          fields=("dump", "text"))


def test_two_contigs_and_empty_region_in_one_batch():
    """Several regions on two contigs (two reference windows, region_of_read path) plus a region without reads."""
    import numpy as np
    from bam_readcount_b200 import synth
    from bam_readcount_b200.batch import ReadBatch
    a = cases.synthetic_case(L=8000, depth=25, seed=51)
    b = cases.synthetic_case(L=9000, depth=35, seed=52)
    bb = b["batch"]
    bb = ReadBatch(**{**{k: getattr(bb, k) for k in ("pos", "flag", "mapq", "lib", "l_qseq", "nm", "sm", "cigar_off", "cigar", "seq_off",
                                                         "seq", "qual_off", "qual")}, "tid": np.full(bb.n_reads, 1, np.int32)})
    batch = ReadBatch.concat([a["batch"], bb])
    gap = synth.synth_reference(500, 3).tobytes()
    case = dict(name="twocontigs", contigs=[a["contigs"][0], ("chr2", 9000, b["contigs"][0][2], 0)], batch=batch,
                regions=[(0, 100, 3000), (0, 7990, 8000), (1, 1, 50), (1, 4000, 8999), (0, 3500, 3600)], site_list=True,
                lib_names=a["lib_names"])
    # make the tail of contig 1 read-free: region (0, 7990, 8000) has no reads (synth reads stop at L-153)
    for flags in (dict(insertion_centric=True), dict(per_lib=True)):
        cases.assert_same(cases.run_engine(case, flags, site_list=True), cases.run_oracle(case, flags, site_list=True),
                          fields=("dump", "text"))
    _ = gap


def test_empty_batches_and_reuse_of_one_handle():
    """compute() with nothing pushed, a region without reads, then real work on the same handle (buffers are reused)."""
    from bam_readcount_b200.engine import Engine
    case = cases.synthetic_case(L=5000, depth=20, seed=9, regions=((0, 1, 5000),))
    name, clen, seq, wb = case["contigs"][0]
    eng = Engine()
    try:
        eng.set_reference(0, name, clen, seq, wb)
        res = eng.compute()
        assert res.n_slots == 0 and eng.format_text() == ""
        eng.reset()
        eng.begin_region(0, 100, 200, True); eng.end_region()          # no reads pushed
        res = eng.compute()
        assert eng.format_text() == ""
        want, _, _ = cases.run_oracle(case, dict(), site_list=True)
        for _ in range(2):
            eng.reset()
            eng.begin_region(0, 0, 5000, True); eng.push_reads(case["batch"]); eng.end_region()
            eng.compute()
            assert eng.format_text() == want
    finally:
        eng.close()


def test_carried_deletion_queue_equals_one_batch():
    """brc_set_queue_carry: argv regions flushed one per brc_compute (what brc-readcount does to bound its memory) print exactly
    what the same regions print as ONE batch — the reference's never-cleared deletion queue (R:bamreadcount.cpp:650-656) travels
    with the engine — and exactly what the reference binary printed (golden edge_alleles_*)."""
    import edge_cases
    case = edge_cases.multi_allele_case()
    for fl_name, fl in case["flag_sets"].items():
        one = cases.run_engine(case, fl, site_list=False, dump=False).text
        # run_engine_per_region turns the carry off again at the end: a fresh queue per call
        assert "".join(r.text for r in cases.run_engine_per_region(case, fl, site_list=False)) == one, fl_name
        assert one == cases.load_golden_text(f"edge_alleles_{fl_name}.txt")


def test_two_handles_driven_from_two_threads():
    """bench.py's e2e caller keeps two engine handles in flight, one host thread each (brc_compute blocks): both must give what a
    lone handle gives — the per-device set-up they share (constant table, opt-in shared-memory sizes) is serialised."""
    import threading
    from bam_readcount_b200.engine import Engine
    jobs = []
    for seed, L in ((21, 9000), (22, 7000)):
        jobs.append((cases.synthetic_case(L=L, depth=30, seed=seed, regions=((0, 1, L),)), dict(min_mapq=20, min_bq=20), L))

    def run(i, reps, out):
        case, flags, L = jobs[i]
        name, clen, seq, wb = case["contigs"][0]
        eng = Engine(**flags)
        try:
            for rep in range(reps):                    # reuse of a handle while the other one is mid-compute
                eng.reset()
                eng.set_reference(0, name, clen, seq, wb)
                eng.begin_region(0, 0, L, False)
                eng.push_reads(case["batch"])
                eng.end_region()
                eng.compute()
                out.append(eng.format_text())
        finally:
            eng.close()

    alone = [[], []]
    for i in range(2):
        run(i, 1, alone[i])
    outs = [[], []]
    ths = [threading.Thread(target=run, args=(i, 3, outs[i])) for i in range(2)]
    for t in ths:
        t.start()
    for t in ths:
        t.join()
    for i in range(2):
        assert len(outs[i]) == 3 and len(alone[i][0]) > 100000
        for rep in range(3):
            assert outs[i][rep] == alone[i][0], (i, rep, first_diff(outs[i][rep], alone[i][0]))


def test_h2d_byte_report_counts_what_crossed_pcie(monkeypatch):
    """brc_last_h2d_bytes: regular offset arrays and constant columns of fixed-length reads are rebuilt on the device and are not
    counted; with the elision off every array of the batch is."""
    from bam_readcount_b200.engine import Engine
    case = cases.synthetic_case(L=8000, depth=30, seed=5, regions=((0, 1, 8000),))
    name, clen, seq, wb = case["contigs"][0]
    b = case["batch"]
    n = b.n_reads
    full = sum(int(np.asarray(a).nbytes) for a in (b.pos, b.flag, b.mapq, b.lib, b.l_qseq, b.nm, b.sm, b.cigar_off, b.cigar, b.seq_off, b.seq,
                                                    b.qual_off, b.qual) if a is not None)
    got = {}
    for mode in ("elide", "all"):
        if mode == "all":
            monkeypatch.setenv("BRC_NO_H2D_ELISION", "1")
        eng = Engine(min_mapq=20)
        try:
            eng.set_reference(0, name, clen, seq, wb)
            eng.begin_region(0, 0, 8000, False)
            eng.push_reads(b)
            eng.end_region()
            eng.compute()
            got[mode] = (eng.h2d_bytes(), eng.format_text())
        finally:
            eng.close()
    assert got["elide"][1] == got["all"][1]
    assert 0 < got["elide"][0] <= got["all"][0] <= full + 4 * n + 64
    assert got["all"][0] >= full - 16 * n - 64          # never less than the arrays that cannot be rebuilt
