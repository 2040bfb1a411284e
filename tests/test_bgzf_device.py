"""SURVEY.md §8 f-2: BGZF inflate + BAM framing on the device (bam_readcount_b200/csrc/brc_bgzf.cu).

CPU: the DEFLATE core the kernel runs (brc_bgzf.cuh, host+device code) against zlib on every block of the fixtures, and the BAI
span builder.  GPU: the device-decoded batch equals the host decoder's records field for field, and a region computed from the
compressed span equals the region computed from host-decoded reads (text and raw accumulators)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import cases
from bam_readcount_b200 import bamio
from cases import GOLDEN

def test_deflate_core_matches_zlib_on_every_block(tmp_path):
    """The exact DEFLATE code the kernel runs (host+device source), block by block against zlib: dynamic, fixed and stored blocks."""
    exe = cases.check_program("inflate_check", "-lz")
    files = [os.path.join(GOLDEN, "test.bam"), os.path.join(GOLDEN, "test_bad_rg.bam")]
    from oracle.oracle import REF_SAMTOOLS
    if os.path.exists(REF_SAMTOOLS):
        from bam_readcount_b200 import synth_cb
        sp = synth_cb.Spec(seed=2, contig_len=1280 * 200)
        info = synth_cb.write_sample_bam(sp, 0, 0, 120, str(tmp_path), REF_SAMTOOLS)
        files.append(info["bam"])
        for lv in ("-u", "-1"):                        # stored blocks / fast compression
            out = os.path.join(str(tmp_path), f"x{lv}.bam")
            subprocess.check_call([REF_SAMTOOLS, "view", lv, "-b", "-o", out, info["bam"]])
            files.append(out)
    nblk, bad = map(int, subprocess.check_output([exe] + files).split())
    assert bad == 0 and nblk >= 20


def test_bai_span_covers_the_fetch():
    bai = bamio.BaiIndex(os.path.join(GOLDEN, "test.bam.bai"))
    sp = bamio.bam_span(os.path.join(GOLDEN, "test.bam"), bai, 20, 10402984, 10405200)
    assert sp is not None and sp["entries"] == sorted(sp["entries"]) and len(sp["comp"]) > 1000
    assert bamio.bam_span(os.path.join(GOLDEN, "test.bam"), bai, 3, 100, 200) is None
    w = bai.window_weights(20, 700)
    assert w.sum() > 0 and w[:600].sum() == 0               # all the coverage sits around 10.4 Mb


def _records_of(batch, idx):
    b = batch.select(idx)
    return [(int(b.pos[i]), int(b.flag[i]), int(b.mapq[i]), int(b.l_qseq[i]), int(b.nm[i]), int(b.sm[i]), int(b.lib[i]),
             b.cigar[int(b.cigar_off[i]):int(b.cigar_off[i + 1])].tobytes(), b.seq[int(b.seq_off[i]):int(b.seq_off[i + 1])].tobytes(),
             b.qual[int(b.qual_off[i]):int(b.qual_off[i + 1])].tobytes()) for i in range(b.n_reads)]


@pytest.mark.gpu
def test_device_decoded_batch_equals_host_decoder():
    from bam_readcount_b200.engine import Engine
    jobs = [(os.path.join(GOLDEN, "test.bam"), 20, 10402000, 10406000), (os.path.join(GOLDEN, "test_bad_rg.bam"), 20, 10402984, 10402985)]
    from oracle.oracle import REF_SAMTOOLS
    tmp = tempfile.mkdtemp()
    if os.path.exists(REF_SAMTOOLS):
        from bam_readcount_b200 import synth_cb
        sp = synth_cb.Spec(seed=6, contig_len=1280 * 2000)
        info = synth_cb.write_sample_bam(sp, 0, 0, 1500, tmp, REF_SAMTOOLS)
        jobs += [(info["bam"], 0, 200_000, 1_500_000), (info["bam"], 0, 0, 50_000)]
    e = Engine(per_lib=True, lib_names=["a"] * 16)
    try:
        for path, tid, beg, end in jobs:
            hdr, host = bamio.read_bam(path)
            rg_lib = {rg: hdr.lib_of_rg(rg) for rg in hdr.rg_lb}
            bai = bamio.BaiIndex(path + ".bai")
            span = bamio.bam_span(path, bai, tid, beg, end, rg_lib)
            dev = e.decode_bam_span(span)
            want = _records_of(host, host.fetch(tid, beg, end))
            got = _records_of(dev, np.arange(dev.n_reads))
            # the span holds every record samfetch yields, in file order (plus neighbours the kernels ignore)
            pos = {r: i for i, r in enumerate(got)}
            assert all(r in pos for r in want), path
            idx = [pos[r] for r in want]
            assert idx == sorted(idx)
            assert len(span["entries"]) >= 1 and dev.n_reads >= len(want)
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [dict(), dict(per_lib=True, insertion_centric=True, min_mapq=10, min_bq=15)])
def test_region_from_compressed_span_equals_region_from_host_reads(flags):
    """brc_push_bam_span (inflate + framing + kernels, reads never on the host) == brc_push_reads of the host-decoded records."""
    samtools = cases.samtools()
    from bam_readcount_b200 import synth_cb
    tmp = tempfile.mkdtemp()
    sp = synth_cb.Spec(seed=12, contig_len=1280 * 600)
    info = synth_cb.write_sample_bam(sp, 0, 0, 600, tmp, samtools)
    hdr, host = bamio.read_bam(info["bam"])
    rg_lib = {rg: hdr.lib_of_rg(rg) for rg in hdr.rg_lb}
    beg, end = 100_000, 700_000
    case = dict(name="span", contigs=[("chr1", info["length"], sp.ref_host(0, 0, info["length"]), 0)], batch=host,
                regions=[(0, beg + 1, end)], site_list=False, lib_names=hdr.lib_names)

    def push_span(e, tid, beg, end, sub):
        e.push_bam_span(bamio.bam_span(info["bam"], bamio.BaiIndex(info["bam"] + ".bai"), 0, beg - 1, end, rg_lib))
    texts = [cases.run_engine(case, flags, dump=False, push=push).text for push in ("one", push_span)]
    assert texts[0] == texts[1] and len(texts[0].splitlines()) == end - beg


@pytest.mark.gpu
def test_cli_device_decode_matches_host_decode(tmp_path):
    """brc-readcount with BRC_CLI_DEVICE_DECODE=1 (compressed spans -> GPU inflate/framing) prints what the host-decode path prints."""
    samtools = cases.samtools()
    from bam_readcount_b200 import build, synth_cb
    exe = build.build_cli()
    sp = synth_cb.Spec(seed=21, contig_len=1280 * 500)
    info = synth_cb.write_sample_bam(sp, 0, 0, 500, str(tmp_path), samtools)
    for extra in ([], ["-p", "-q", "20", "-b", "20"]):
        args = [exe, "-w", "0"] + extra + ["-f", info["fasta"], info["bam"], "chr1:5001-600000"]
        env = dict(os.environ, BRC_CLI_WINDOW="150000")
        host = subprocess.run(args, capture_output=True, env=env)
        dev = subprocess.run(args, capture_output=True, env=dict(env, BRC_CLI_DEVICE_DECODE="1"))
        assert host.returncode == 0 and dev.returncode == 0, dev.stderr.decode()[-1500:]
        assert dev.stdout == host.stdout and len(host.stdout.splitlines()) == 595000
