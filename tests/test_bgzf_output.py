"""BGZF output compressed on the device (brc_deflate.cu, `brc-readcount --bgzf`).

CPU: the serial pieces the kernel runs (brc_deflate.cuh, through tests/deflate_check.cpp) against zlib and htslib's layout; the
writer refuses a machine without a device; the CLI accepts --bgzf under the decode-only hook.  GPU: the writer's files inflate
to their input and parse member by member, do not depend on how the input was split, compress about as well as zlib level 1;
every output of the CLI under --bgzf decompresses to the plain run's bytes."""
import gzip
import os
import random
import struct
import subprocess
import zlib

import pytest

import cases
import vcf_cases
from cases import GOLDEN

BLOCK = 0xff00
HEADER = b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00"
EOF = HEADER + b"\x1b\x00\x03\x00\x00\x00\x00\x00\x00\x00\x00\x00"


@pytest.fixture(scope="module")
def dc():
    return cases.check_program("deflate_check")


def members(data: bytes):
    """Every member of a BGZF file, checked: header bytes, BSIZE + 1 = its length <= 65536, ISIZE <= 65280 and CRC32 of the
    inflated bytes; the file ends with the EOF member.  Returns the inflated bytes of each member."""
    out, o = [], 0
    assert data.endswith(EOF)
    while o < len(data):
        assert data[o:o + 16] == HEADER, o
        size = struct.unpack_from("<H", data, o + 16)[0] + 1
        assert size <= 65536 and o + size <= len(data)
        crc, isize = struct.unpack_from("<II", data, o + size - 8)
        raw = zlib.decompress(data[o + 18:o + size - 8], -15)
        assert len(raw) == isize <= BLOCK and zlib.crc32(raw) == crc
        out.append(raw)
        o += size
    assert out[-1] == b""
    return out


# ---------------------------------------------------------------------------------------------------------------- CPU
def _lengths(dc, freqs, maxbits=15):
    return [int(x) for x in subprocess.check_output([dc, "lengths", str(maxbits)] + [str(f) for f in freqs]).split()]


def test_code_lengths_are_limited_and_complete(dc):
    rng = random.Random(5)
    fib = [1, 1]
    while len(fib) < 40:
        fib.append(fib[-1] + fib[-2])
    hists = [[0] * 286, [0] * 285 + [7], [3] + [0] * 284 + [9], [1] * 286, [100] * 286, fib[:25] + [0] * 261, fib[:30],
             [rng.choice([0, 0, 1, 2, 5, 1000, 60000]) for _ in range(286)]]
    hists += [[rng.randint(0, 2000) for _ in range(rng.choice([19, 30, 286]))] for _ in range(20)]
    for h in hists:
        for maxbits in (15, 7):
            if maxbits == 7 and len(h) > 128:
                continue
            ln = _lengths(dc, h, maxbits)
            used = [l for f, l in zip(h, ln) if f]
            assert all((l > 0) == (f > 0) for f, l in zip(h, ln)) and max(ln) <= maxbits
            kraft = sum(2.0 ** -l for l in used)
            assert kraft == (1.0 if len(used) >= 2 else 0.5 * len(used)), (h, ln)
    # a Fibonacci histogram needs lengths past 15 without the limit: the limit is what kept them at 15
    assert max(_lengths(dc, fib[:30])) == 15


def _tokens(rng, n, dist_max=32768, lits=b"ACGT\t\n:.0123456789"):
    data, toks = bytearray(), []
    while len(toks) < n:
        if data and rng.random() < 0.35:
            d = rng.randint(1, min(len(data), dist_max))
            ln = rng.choice([3, 4, 10, 11, 18, 19, 130, 227, 257, 258, rng.randint(3, 258)])
            for _ in range(ln):
                data.append(data[-d])
            toks.append(f"M {ln} {d}")
        else:
            b = rng.choice(lits)
            data.append(b)
            toks.append(f"L {b}")
    return "\n".join(toks), bytes(data)


def test_dynamic_fixed_and_stored_encoders_inflate_with_zlib(dc):
    rng = random.Random(9)
    streams = [_tokens(rng, 5), _tokens(rng, 3000), _tokens(random.Random(2), 400, lits=bytes(range(256))),
               ("L 65\n" + "\n".join(["M 258 1"] * 100), b"A" * (1 + 258 * 100)),
               ("\n".join(f"L {b}" for b in b"xyz") + "\n" + "\n".join(["L 7"] * 32765) + "\nM 258 32768", None),
               ("L 0", b"\x00"), ("\n".join(f"L {i}" for i in range(256)), bytes(range(256)))]
    for toks, want in streams:
        if want is None:        # the distance-32768 match copies the stream's first bytes
            head = b"xyz" + b"\x07" * 32765
            want = head + (head * 2)[:258]
        for mode in ("dynamic", "fixed"):
            raw = subprocess.check_output([dc, "encode", mode], input=toks.encode())
            assert zlib.decompress(raw, -15) == want, mode
    for n in (0, 1, 100, BLOCK):
        data = bytes(random.Random(n).getrandbits(8) for _ in range(n))
        raw = subprocess.check_output([dc, "encode", "stored"], input=data)
        assert len(raw) == n + 5 and zlib.decompress(raw, -15) == data


def test_crc_combine_equals_zlib_over_random_splits(dc):
    rng = random.Random(3)
    for n in (0, 1, 7, 1000, 65280):
        data = bytes(rng.getrandbits(8) for _ in range(n))
        for _ in range(4):
            cuts = sorted(rng.randint(0, n) for _ in range(rng.randint(0, 6)))
            cuts += [cuts[-1]] if cuts else []                      # a 0-length part
            got = subprocess.check_output([dc, "crc"] + [str(c) for c in cuts], input=data).strip().decode()
            assert int(got, 16) == zlib.crc32(data), (n, cuts)


def test_member_framing_is_htslibs_layout(dc):
    for n in (0, 1, 1000, BLOCK):
        data = bytes(random.Random(n).getrandbits(8) for _ in range(n))
        deflated = bytes([1]) + struct.pack("<HH", n, n ^ 0xffff) + data
        want = HEADER + struct.pack("<H", 18 + len(deflated) + 8 - 1) + deflated + struct.pack("<II", zlib.crc32(data), n)
        assert subprocess.check_output([dc, "member"], input=data) == want
    assert subprocess.check_output([dc, "eof"]) == EOF and len(EOF) == 28


def test_writer_needs_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from bam_readcount_b200 import engine
    with pytest.raises(engine.BrcError) as ei:
        engine.BgzfWriter(1)
    assert ei.value.status == -2   # BRC_E_NO_DEVICE


def test_cli_opens_its_writer_on_brc_device():
    """The writer goes to BRC_DEVICE, the engines' device: one that does not exist is refused before anything is written."""
    exe = cases.cli()
    p = subprocess.run([exe, "--bgzf", os.path.join(GOLDEN, "test.bam"), "21:10402985-10402990"], capture_output=True,
                       env=dict(os.environ, BRC_DEVICE="99"))
    assert p.returncode == 1 and p.stdout == b"" and b"--bgzf: no usable CUDA device" in p.stderr


def test_set_device_refuses_a_missing_device():
    from bam_readcount_b200 import engine
    lib = engine.load_library()
    assert lib.brc_set_device(99) == -2 and lib.brc_set_device(-1) == -2   # BRC_E_NO_DEVICE


def test_cli_accepts_bgzf_under_decode_only():
    exe = cases.cli()
    env = dict(os.environ, BRC_CLI_DECODE_ONLY="1")
    args = [os.path.join(GOLDEN, "test.bam"), "21:10402985-10402990"]
    plain = subprocess.run([exe] + args, capture_output=True, env=env)
    got = subprocess.run([exe, "--bgzf"] + args, capture_output=True, env=env)
    assert plain.returncode == got.returncode == 0
    assert got.stdout == plain.stdout and got.stderr == plain.stderr and plain.stdout.count(b"\n") == 1


# ---------------------------------------------------------------------------------------------------------------- GPU
def compress(chunks, tmp_path):
    from bam_readcount_b200.engine import BgzfWriter
    path = str(tmp_path / "out.gz")
    fd = os.open(path, os.O_WRONLY | os.O_CREAT | os.O_TRUNC, 0o644)
    try:
        with BgzfWriter(fd) as w:
            for c in chunks:
                w.write(c)
    finally:
        os.close(fd)
    with open(path, "rb") as fh:
        return fh.read()


def _texts():
    names = sorted(f[:-3] for f in os.listdir(GOLDEN) if f.endswith(".txt.gz"))
    return {n: cases.load_golden_text(n).encode("latin-1") for n in names}


def _crafted_inputs():
    rng = random.Random(11)
    far = bytes(rng.getrandbits(8) for _ in range(300))
    return {
        "empty": b"", "one": b"x",
        "65279": bytes(rng.getrandbits(8) for _ in range(65279)), "65280": b"ACGT\n" * 13056,
        "65281": (b"21\t10402985\tA\t30\t" * 4000)[:65281], "2x65280": bytes(range(256)) * 510,
        "random": bytes(rng.getrandbits(8) for _ in range(3 * BLOCK + 77)),
        "one byte repeated": b"\x00" * (2 * BLOCK + 5),
        "distance 32768": far + bytes(rng.getrandbits(8) for _ in range(32768 - 300)) + far,
        "distance 32769": far + bytes(rng.getrandbits(8) for _ in range(32769 - 300)) + far,
    }


@pytest.mark.gpu
def test_writer_on_the_device_set_before_it_opens(tmp_path):
    from bam_readcount_b200 import engine
    import torch
    lib = engine.load_library()
    n = torch.cuda.device_count()
    assert lib.brc_set_device(n) == -2
    for dev in range(min(n, 2)):
        assert lib.brc_set_device(dev) == 0
        assert gzip.decompress(compress([b"ACGT\n" * 70000], tmp_path)) == b"ACGT\n" * 70000


@pytest.mark.gpu
def test_writer_round_trip_and_member_layout(tmp_path):
    inputs = dict(_crafted_inputs())
    inputs.update(_texts())
    vcf = vcf_cases.vcf_text(vcf_cases.fixture_records()).encode()
    inputs["vcf fixture"] = vcf
    for name, data in inputs.items():
        out = compress([data], tmp_path)
        parts = members(out)
        assert b"".join(parts) == data and gzip.decompress(out) == data, name
        assert [len(p) for p in parts[:-1]] == [min(BLOCK, len(data) - i) for i in range(0, len(data), BLOCK)], name
        if name == "empty":
            assert out == EOF
        if name == "random":          # incompressible: every block is stored (BFINAL 1, BTYPE 00, LEN, NLEN, the bytes)
            o = 0
            for raw in parts[:-1]:
                size = struct.unpack_from("<H", out, o + 16)[0] + 1
                assert size == len(raw) + 31 and out[o + 18] == 1
                assert struct.unpack_from("<HH", out, o + 19) == (len(raw), len(raw) ^ 0xffff) and out[o + 23:o + 23 + len(raw)] == raw
                o += size


@pytest.mark.gpu
def test_writer_output_does_not_depend_on_the_write_calls(tmp_path):
    rng = random.Random(4)
    data = b"".join(list(_texts().values())[:3]) + _crafted_inputs()["random"]
    big = data * ((40 << 20) // len(data) + 1)          # about 40 MB: the writer's 16.7 MB chunks, and a part of one more
    whole = compress([big], tmp_path)
    assert gzip.decompress(whole) == big
    cuts, i = [], 0
    while i < len(big):
        k = rng.choice([1, 17, 4096, 65280, 65281, 1 << 20, 20 << 20])
        cuts.append(big[i:i + k]); i += k
    assert compress(cuts, tmp_path) == whole
    small = data[:200000]
    assert compress([small[j:j + 1] for j in range(len(small))], tmp_path) == compress([small], tmp_path)


@pytest.mark.gpu
def test_ratio_against_zlib_level_1_on_the_golden_texts(tmp_path):
    ours = theirs = 0
    for name, data in _texts().items():
        if not name.startswith("ref_syn") and not name.startswith("edge"):
            continue
        ours += len(compress([data], tmp_path)) - len(EOF)
        theirs += sum(len(zlib.compress(data[i:i + BLOCK], 1)) - 6 + 26 for i in range(0, len(data), BLOCK))
    print(f"device {ours} B, zlib -1 {theirs} B, ratio {ours / theirs:.3f}")
    assert ours <= 1.05 * theirs


# ---- the CLI ----
def _plain_and_bgzf(argv, env=None, rc=0):
    exe = cases.cli()
    plain = subprocess.run([exe] + argv, capture_output=True, env=env)
    got = subprocess.run([exe, "--bgzf"] + argv, capture_output=True, env=env)
    assert plain.returncode == rc and got.returncode == rc, got.stderr.decode()[-2000:]
    assert got.stderr == plain.stderr
    assert b"".join(members(got.stdout)) == plain.stdout
    return plain.stdout, got.stdout


@pytest.mark.gpu
def test_cli_bgzf_integration_lines_and_site_filter(tmp_path):
    ref = cases.write_testbam_fasta(str(tmp_path / "ref.fa"))
    sl = os.path.join(GOLDEN, "site_list")
    regions = ["21:10402985-10402985", "21:10405200-10405200"]
    runs = [["-l", sl], ["-p", "-l", sl], ["-i", "-l", sl], ["-i", "-p", "-l", sl]]
    for bam in ("test.bam", "test_bad_rg.bam"):
        runs.append([bam] + regions)
    runs.append(["--min-alt-count", "2", "--alt-min", "avg_basequality=20", "-l", sl])
    for r in runs:
        bam = r[0] if r[0].endswith(".bam") else "test.bam"
        opts = [a for a in r if not a.endswith(".bam") and a not in regions]
        plain, _ = _plain_and_bgzf(["-w", "1", "-f", ref] + opts + [os.path.join(GOLDEN, bam)] + [a for a in r if a in regions])
        assert plain.count(b"\n") >= 1


@pytest.mark.gpu
def test_cli_bgzf_vcf_plain_bgzip_complex_and_samples(tmp_path):
    fa = cases.write_testbam_fasta(str(tmp_path / "ref.fa"))
    text = vcf_cases.vcf_text(vcf_cases.fixture_records())
    plain_vcf, gz_vcf = str(tmp_path / "a.vcf"), str(tmp_path / "a.vcf.gz")
    open(plain_vcf, "w").write(text)
    vcf_cases.write_bgzf(gz_vcf, text.encode())
    bam = os.path.join(GOLDEN, "test.bam")
    for path in (plain_vcf, gz_vcf):
        for extra in ([], ["--vcf-complex"]):
            out, _ = _plain_and_bgzf(["-w", "1", "-f", fa, "--vcf", path] + extra + [bam])
            assert out.startswith(b"##fileformat")
    two = vcf_cases.vcf_text(vcf_cases.fixture_records(), samples=("S1", "S2"))
    vcf2 = str(tmp_path / "two.vcf")
    open(vcf2, "w").write(two)
    lst = tmp_path / "samples.txt"
    lst.write_text(f"S1\t{bam}\nS2\t{os.path.join(GOLDEN, 'test_bad_rg.bam')}\n")
    _plain_and_bgzf(["-w", "1", "-f", fa, "--vcf", vcf2, "--vcf-samples", str(lst)])


@pytest.mark.gpu
def test_cli_bgzf_bam_list_out_files(tmp_path):
    exe = cases.cli()
    ref = cases.write_testbam_fasta(str(tmp_path / "ref.fa"))
    bams = [os.path.join(GOLDEN, b) for b in ("test.bam", "test_bad_rg.bam", "test.bam")]
    regions = ["21:10402985-10402990", "21:10405200-10405210"]
    outs = {}
    for mode in ("plain", "bgzf"):
        lst = tmp_path / f"{mode}.list"
        lst.write_text("".join(f"{b}\t{tmp_path}/{mode}.{k}.out\n" for k, b in enumerate(bams)))
        p = subprocess.run([exe, "-w", "1", "-f", ref] + (["--bgzf"] if mode == "bgzf" else []) + ["--bam-list", str(lst)] + regions,
                           capture_output=True)
        assert p.returncode == 0, p.stderr.decode()[-2000:]
        outs[mode] = [(open(f"{tmp_path}/{mode}.{k}.out", "rb").read(), open(f"{tmp_path}/{mode}.{k}.out.log", "rb").read())
                      for k in range(len(bams))]
    for (po, pe), (go, ge) in zip(outs["plain"], outs["bgzf"]):
        assert b"".join(members(go)) == po and ge == pe and po.count(b"\n") >= 2


@pytest.mark.gpu
def test_cli_bgzf_shards_concatenate(tmp_path):
    from bam_readcount_b200 import synth_cb
    sp = synth_cb.Spec(seed=8, contig_len=1280 * 300)
    info = synth_cb.write_sample_bam(sp, 0, 0, 300, str(tmp_path), cases.samtools())
    env = dict(os.environ, BRC_CLI_WINDOW="50000")
    args = ["-w", "0", "-i", "-f", info["fasta"], info["bam"], "chr1:2001-380000"]
    plains, gzs = [], []
    for r in range(2):
        p, g = _plain_and_bgzf(["--shard", f"{r}/2"] + args, env=env)
        plains.append(p); gzs.append(g)
    assert gzip.decompress(gzs[0] + gzs[1]) == plains[0] + plains[1] and all(plains)


@pytest.mark.gpu
def test_cli_bgzf_to_a_full_device_fails():
    exe = cases.cli()
    args = ["-w", "1", os.path.join(GOLDEN, "test.bam"), "21:10402985-10402990"]
    for flags in ([], ["--bgzf"]):
        with open("/dev/full", "wb") as full:
            p = subprocess.run([exe] + flags + args, stdout=full, stderr=subprocess.PIPE)
        assert p.returncode == 1 and p.stderr.strip(), flags
