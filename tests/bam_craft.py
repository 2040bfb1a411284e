"""Hand-made BAM files for the record-decode tests, and an independent statement of how htslib 1.10 reads their records.

Writer: records with arbitrary aux bytes (any type, duplicate tags, a `d` value, tails cut by the end of the record, a CG:B:I
long-CIGAR pair), BGZF members cut where the caller says and compressed at the level / strategy the caller says.

Restatement (`Restated`): the per-read fields the reference binary sees, written from htslib's documented behaviour and kept
independent of bamio and of csrc/brc_aux.cuh:
  - bam_aux_get(tag): walk the tags from the start; return the first one named `tag`; give up (absent) as soon as a value cannot
    be skipped -- an unknown type, a B array of unknown subtype, a value running past the end of the record -- including the
    wanted tag's own value.  A wanted Z or H value that the record ends before its NUL is absent too.
  - bam_aux2i: integer types give their value (kept in an int32_t by the reference), any other type gives 0.
  - bam_get_library: the first RG tag's value bytes up to a NUL are the @RG ID, whatever the tag's type.
  - bam_tag2cigar: a placed record (tid >= 0, pos >= 0) whose first CIGAR op is <l_qseq>S and whose first CG tag is B:I with
    n_cigar <= count < 2^29 has that array as its CIGAR.
"""
from __future__ import annotations

import os
import struct
import subprocess
import zlib
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from bam_readcount_b200.batch import LIB_NONE, TAG_ABSENT, ReadBatch

OPS = "MIDNSHP=X"
NT16 = "=ACMGRSVTWYHKDBN"


# ------------------------------------------------------------------------------------------------
# aux values
# ------------------------------------------------------------------------------------------------
_FMT = {"A": "<c", "c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I", "f": "<f", "d": "<d"}


def tag(name: str, typ: str, value) -> bytes:
    """One aux field.  Z/H take a str (NUL added), B takes (subtype, list), the rest a number (A: a 1-char str)."""
    head = name.encode() + typ.encode()
    if typ in "ZH":
        return head + value.encode() + b"\0"
    if typ == "B":
        sub, vals = value
        return head + sub.encode() + struct.pack("<I", len(vals)) + b"".join(struct.pack(_FMT[sub], v) for v in vals)
    if typ == "A":
        return head + value.encode()
    return head + struct.pack(_FMT[typ], value)


def cigar_words(cig: Sequence[Tuple[str, int]]) -> List[int]:
    return [n << 4 | OPS.index(op) for op, n in cig]


def parse_cigar(s: str) -> List[Tuple[str, int]]:
    out, n = [], ""
    for ch in s:
        if ch.isdigit():
            n += ch
        else:
            out.append((ch, int(n)))
            n = ""
    return out


def ref_span(cig: Sequence[Tuple[str, int]]) -> int:
    return sum(n for op, n in cig if op in "MDN=X")


def reg2bin(beg: int, end: int) -> int:
    end -= 1
    for sh, off in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> sh == end >> sh:
            return off + (beg >> sh)
    return 0


def record(qname: str, tid: int, pos: int, cig: Sequence[Tuple[str, int]], seq: str, qual: Sequence[int], aux: bytes = b"",
           flag: int = 0, mapq: int = 60, cigar_field: Optional[Sequence[Tuple[str, int]]] = None) -> bytes:
    """One BAM record (block_size included).  `cig` is the alignment; `cigar_field`, when given, is what the CIGAR field holds
    instead (the <l_qseq>S<span>N placeholder of a CG-carried CIGAR)."""
    field = cigar_words(cigar_field if cigar_field is not None else cig)
    end = pos + max(ref_span(cig), 1)
    l = len(seq)
    packed = bytearray((l + 1) // 2)
    for i, ch in enumerate(seq):
        packed[i >> 1] |= NT16.index(ch) << (4 if i % 2 == 0 else 0)
    qn = qname.encode() + b"\0"
    body = struct.pack("<iiBBHHHiiii", tid, pos, len(qn), mapq, reg2bin(max(pos, 0), end), len(field), flag, l, -1, -1, 0)
    body += qn + b"".join(struct.pack("<I", w) for w in field) + bytes(packed) + bytes(qual) + aux
    return struct.pack("<i", len(body)) + body


def header_bytes(text: str, refs: Sequence[Tuple[str, int]]) -> bytes:
    t = text.encode()
    out = b"BAM\1" + struct.pack("<i", len(t)) + t + struct.pack("<i", len(refs))
    for name, ln in refs:
        n = name.encode() + b"\0"
        out += struct.pack("<i", len(n)) + n + struct.pack("<i", ln)
    return out


# ------------------------------------------------------------------------------------------------
# BGZF
# ------------------------------------------------------------------------------------------------
BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def bgzf_member(data: bytes, deflated: Optional[bytes] = None, level: int = 6, strategy: int = zlib.Z_DEFAULT_STRATEGY) -> bytes:
    """One BGZF member holding `data`: its raw-DEFLATE stream is `deflated` when given, else zlib's at level / strategy."""
    assert len(data) <= 65536
    if deflated is None:
        c = zlib.compressobj(level, zlib.DEFLATED, -15, 9, strategy)
        deflated = c.compress(data) + c.flush()
    assert zlib.decompress(deflated, -15) == data
    bsize = 18 + len(deflated) + 8
    assert bsize <= 65536, "member too large"
    hdr = bytes([31, 139, 8, 4, 0, 0, 0, 0, 0, 255]) + struct.pack("<H", 6) + b"BC" + struct.pack("<HH", 2, bsize - 1)
    return hdr + deflated + struct.pack("<II", zlib.crc32(data), len(data))


def chunks_default(data: bytes, size: int = 0xff00) -> List[bytes]:
    return [data[i:i + size] for i in range(0, len(data), size)]


def write_bam(path: str, text: str, refs: Sequence[Tuple[str, int]], records: Sequence[bytes], members=None, level: int = 6,
              strategy: int = zlib.Z_DEFAULT_STRATEGY, index: Optional[str] = None) -> str:
    """Header in its own member, then the records.  `members(data) -> [bytes | (bytes, deflated)]` decides where the record
    bytes are cut (default: 0xff00-byte pieces) and, per piece, optionally the DEFLATE stream.  `index`: samtools to index with."""
    data = b"".join(records)
    out = bgzf_member(header_bytes(text, refs), level=level)
    for m in (members or chunks_default)(data):
        raw, dfl = (m, None) if isinstance(m, (bytes, bytearray)) else m
        out += bgzf_member(bytes(raw), dfl, level, strategy)
    with open(path, "wb") as fh:
        fh.write(out + BGZF_EOF)
    if index:
        subprocess.check_call([index, "index", path])
    return path


# ------------------------------------------------------------------------------------------------
# the restatement of htslib's record reading
# ------------------------------------------------------------------------------------------------
_FIXED = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4, "d": 8}


def _value_end(rec: bytes, t: int) -> Optional[int]:
    """Where the value whose type byte is rec[t] ends, None when it cannot be skipped."""
    typ = chr(rec[t])
    v = t + 1
    if typ in ("Z", "H"):
        nul = rec.find(b"\0", v)
        return len(rec) if nul < 0 else nul + 1
    if typ == "B":
        if len(rec) - v < 5 or chr(rec[v]) not in _FIXED:
            return None
        n = int.from_bytes(rec[v + 1:v + 5], "little")
        stop = v + 5 + _FIXED[chr(rec[v])] * n
        return stop if stop <= len(rec) else None
    if typ not in _FIXED or v + _FIXED[typ] > len(rec):
        return None
    return v + _FIXED[typ]


def aux_get(rec: bytes, aux_start: int, name: bytes) -> Optional[int]:
    """bam_aux_get: offset of the type byte of the first tag `name`, or None."""
    p = aux_start
    while len(rec) - p >= 3:
        here = rec[p:p + 2]
        stop = _value_end(rec, p + 2)
        if here == name:
            if stop is None or (chr(rec[p + 2]) in "ZH" and rec[stop - 1] != 0):    # a Z/H value needs its NUL
                return None
            return p + 2
        if stop is None:
            return None
        p = stop
    return None


def aux2i(rec: bytes, t: int) -> int:
    """bam_aux2i as the reference stores it: in an int32_t."""
    typ = chr(rec[t])
    if typ not in "cCsSiI":
        return 0
    v = struct.unpack_from(_FMT[typ], rec, t + 1)[0]
    return (v + 2 ** 31) % 2 ** 32 - 2 ** 31


class Restated:
    """What the reference binary reads from a BAM file: header facts and one ReadBatch in file order."""

    def __init__(self, path: str):
        with open(path, "rb") as fh:
            raw = _gunzip_members(fh.read())
        assert raw[:4] == b"BAM\1"
        l_text = int.from_bytes(raw[4:8], "little")
        self.text = raw[8:8 + l_text].rstrip(b"\0").decode()
        o = 8 + l_text
        n_ref = int.from_bytes(raw[o:o + 4], "little"); o += 4
        self.refs = []
        for _ in range(n_ref):
            ln = int.from_bytes(raw[o:o + 4], "little"); o += 4
            self.refs.append((raw[o:o + ln - 1].decode(), int.from_bytes(raw[o + ln:o + ln + 4], "little"))); o += ln + 4
        # @RG ID -> LB (first line of an ID wins); libraries ranked in byte order
        self.rg_lb: Dict[bytes, Optional[bytes]] = {}
        for line in self.text.split("\n"):
            if line.startswith("@RG\t"):
                f = dict(x.split(":", 1) for x in line.split("\t")[1:] if ":" in x)
                self.rg_lb.setdefault(f["ID"].encode(), f["LB"].encode() if "LB" in f else None)
        self.lib_names = sorted({lb for lb in self.rg_lb.values() if lb is not None})
        rank = {lb: i for i, lb in enumerate(self.lib_names)}
        cols = {k: [] for k in ("tid", "pos", "flag", "mapq", "lib", "l_qseq", "nm", "sm")}
        cig, seq, qual, self.qnames = [], [], [], []
        while o + 4 <= len(raw):
            bs = int.from_bytes(raw[o:o + 4], "little")
            rec = raw[o + 4:o + 4 + bs]
            o += 4 + bs
            tid, pos, l_rn, mapq, _bin, n_cig, flag, l_seq = struct.unpack_from("<iiBBHHHi", rec, 0)
            c = 32 + l_rn
            words = list(struct.unpack_from(f"<{n_cig}I", rec, c))
            s0 = c + 4 * n_cig
            aux0 = s0 + (l_seq + 1) // 2 + l_seq
            cg = aux_get(rec, aux0, b"CG")
            if (cg is not None and n_cig > 0 and tid >= 0 and pos >= 0 and words[0] == (l_seq << 4 | 4)
                    and rec[cg:cg + 2] == b"BI"):
                cnt = int.from_bytes(rec[cg + 2:cg + 6], "little")
                if n_cig <= cnt < 1 << 29:
                    words = list(struct.unpack_from(f"<{cnt}I", rec, cg + 6))
            nm, sm, rg = aux_get(rec, aux0, b"NM"), aux_get(rec, aux0, b"SM"), aux_get(rec, aux0, b"RG")
            lib = LIB_NONE
            if rg is not None:
                nul = rec.find(b"\0", rg + 1)
                lb = self.rg_lb.get(rec[rg + 1:len(rec) if nul < 0 else nul])
                if lb is not None:
                    lib = rank[lb]
            for k, v in (("tid", tid), ("pos", pos), ("flag", flag), ("mapq", mapq), ("lib", lib), ("l_qseq", l_seq),
                         ("nm", TAG_ABSENT if nm is None else aux2i(rec, nm)), ("sm", TAG_ABSENT if sm is None else aux2i(rec, sm))):
                cols[k].append(int(v))
            cig.append(np.array(words, dtype=np.uint32))
            seq.append(np.frombuffer(rec[s0:s0 + (l_seq + 1) // 2], dtype=np.uint8))
            qual.append(np.frombuffer(rec[s0 + (l_seq + 1) // 2:aux0], dtype=np.uint8))
            self.qnames.append(rec[32:32 + l_rn - 1].decode())

        def offs(parts):
            return np.concatenate([[0], np.cumsum([len(x) for x in parts])]).astype(np.uint64)

        def cat(parts, dt):
            return np.concatenate(parts).astype(dt) if parts else np.zeros(0, dt)
        dts = dict(tid=np.int32, pos=np.int32, flag=np.uint16, mapq=np.uint8, lib=np.uint16, l_qseq=np.int32, nm=np.int32, sm=np.int32)
        self.batch = ReadBatch(**{k: np.array(v, dtype=dts[k]) for k, v in cols.items()},
                               cigar_off=offs(cig), cigar=cat(cig, np.uint32), seq_off=offs(seq), seq=cat(seq, np.uint8),
                               qual_off=offs(qual), qual=cat(qual, np.uint8), qname=list(self.qnames))

    @property
    def lib_name_strs(self) -> List[str]:
        return [x.decode() for x in self.lib_names]

    def rg_lib(self) -> Dict[str, int]:
        """@RG ID -> library rank (or LIB_NONE), as brc_push_bam_span takes it."""
        rank = {lb: i for i, lb in enumerate(self.lib_names)}
        return {k.decode(): (rank[v] if v is not None else int(LIB_NONE)) for k, v in self.rg_lb.items()}


def _gunzip_members(d: bytes) -> bytes:
    out, o = [], 0
    while o < len(d):
        z = zlib.decompressobj(31)
        out.append(z.decompress(d[o:]))
        o = len(d) - len(z.unused_data)
    return b"".join(out)


# ------------------------------------------------------------------------------------------------
# the crafted corpus: one small BAM per rule, each with its controls
# ------------------------------------------------------------------------------------------------
HEADER_RG = ("@RG\tID:g1\tSM:s\tLB:L1\n@RG\tID:g2\tSM:s\tLB:L2\n@RG\tID:AB12\tSM:s\tLB:L4\n"
             "@RG\tID:" + "long_read_group_identifier_" + "x" * 24 + "\tSM:s\tLB:L3\n")
LONG_RG = "long_read_group_identifier_" + "x" * 24          # 51 bytes: longer than the device's 44-byte ID copy
FLAG_SETS = {"default": [], "p": ["-p"], "i": ["-i"], "q20b20": ["-q", "20", "-b", "20"]}


def _ref(length: int, seed: int) -> str:
    rng = np.random.default_rng(seed)
    return "".join("ACGT"[i] for i in rng.integers(0, 4, length))


def _read_on(ref: str, pos: int, cig, rng) -> Tuple[str, List[int]]:
    """Read bases for `cig` at `pos` (one substitution in every aligned stretch) and qualities between 10 and 40."""
    s, r = [], pos
    for op, n in cig:
        if op in "M=X":
            part = list(ref[r:r + n])
            k = int(rng.integers(0, n))
            part[k] = "ACGT"[("ACGT".index(part[k]) + 1) % 4]
            s += part; r += n
        elif op in "IS":
            s += ["ACGT"[int(x)] for x in rng.integers(0, 4, n)]
        elif op in "DN":
            r += n
    return "".join(s), [int(x) for x in rng.integers(10, 41, len(s))]


def _cases(ref: str) -> Dict[str, List[dict]]:
    """name -> reads: dict(q=qname, pos, cig=str, aux=bytes, flag, mapq, field=placeholder-CIGAR-or-None)."""
    nm5, sm37, g1 = tag("NM", "i", 5), tag("SM", "i", 37), tag("RG", "Z", "g1")
    real = "10M2I15M3D13M"
    cgw = ("I", cigar_words(parse_cigar(real)))
    ph = [("S", 40), ("N", ref_span(parse_cigar(real)))]
    unknown = b"XUq" + b"\1\2\3\4"                                          # a tag of a type BAM does not define
    c = {
        # row 1: the real CIGAR of a long read lives in CG:B:I behind a <l_qseq>S<span>N placeholder
        "cg": [dict(q="cg_moved", cig=real, aux=nm5 + tag("CG", "B", cgw) + g1, field=ph),
               dict(q="cg_after_d", cig=real, aux=tag("XD", "d", 2.5) + tag("CG", "B", cgw) + nm5 + g1, field=ph),
               dict(q="cg_first_tag", cig=real, aux=tag("CG", "B", cgw) + sm37 + nm5, field=ph, flag=3),
               dict(q="cg_count_below_n_cigar", cig="40M", aux=nm5 + tag("CG", "B", ("I", cigar_words([("M", 40)]))) + g1,
                    field=[("S", 40), ("N", 40)]),
               dict(q="cg_signed_subtype", cig=real, aux=nm5 + tag("CG", "B", ("i", cgw[1])) + g1, field=ph),
               dict(q="cg_behind_cg_z", cig=real, aux=nm5 + tag("CG", "Z", "x") + tag("CG", "B", cgw) + g1, field=ph),
               dict(q="cg_clip_not_whole_read", cig="39S1M", aux=nm5 + tag("CG", "B", cgw) + g1)],
        # row 2: a `d` value is 8 bytes; the tags after it count
        "dtag": [dict(q="d_before_nm", aux=tag("XD", "d", 1.5) + nm5 + sm37 + tag("RG", "Z", "g2"), flag=3),
                 dict(q="two_d", aux=tag("XD", "d", -3.0) + tag("YD", "d", 1e300) + tag("NM", "C", 2) + g1),
                 dict(q="plain", aux=nm5 + sm37 + g1, flag=3)],
        # row 3: a non-integer NM / SM is present and worth 0; controls: every integer type
        "nmtype": [dict(q="nm_f", aux=tag("NM", "f", 3.0) + g1),
                   dict(q="nm_A", aux=tag("NM", "A", "7") + g1),
                   dict(q="nm_Z", aux=tag("NM", "Z", "4") + g1),
                   dict(q="nm_H", aux=tag("NM", "H", "1F") + g1),
                   dict(q="nm_d", aux=tag("NM", "d", 2.0) + g1),
                   dict(q="nm_B", aux=tag("NM", "B", ("c", [1, 2])) + g1),
                   dict(q="sm_f", aux=nm5 + tag("SM", "f", 20.0) + g1, flag=3),
                   dict(q="sm_Z", aux=nm5 + tag("SM", "Z", "20") + g1, flag=3),
                   dict(q="nm_f_then_i", aux=tag("NM", "f", 1.0) + tag("NM", "i", 9) + g1),
                   dict(q="nm_c", aux=tag("NM", "c", -3) + g1), dict(q="nm_C", aux=tag("NM", "C", 200) + g1),
                   dict(q="nm_s", aux=tag("NM", "s", -300) + g1), dict(q="nm_S", aux=tag("NM", "S", 60000) + g1),
                   dict(q="nm_i", aux=tag("NM", "i", -5) + g1), dict(q="nm_I", aux=tag("NM", "I", 3000000000) + g1),
                   dict(q="sm_S", aux=nm5 + tag("SM", "S", 65535) + g1, flag=3)],
        # row 4: the first RG decides whatever its type; H names an ID as Z does
        "rg": [dict(q="rg_H", aux=nm5 + tag("RG", "H", "AB12")),
               dict(q="rg_long_id", aux=nm5 + tag("RG", "Z", LONG_RG)),
               dict(q="rg_z_twice", aux=nm5 + tag("RG", "Z", "g2") + g1)],
        # ... so a non-string first RG leaves the read without a library (under -p the reference then prints nothing)
        "rg_nolib": [dict(q="rg_plain", aux=nm5 + g1),
                     dict(q="rg_i_then_z", aux=nm5 + tag("RG", "i", 7) + g1),
                     dict(q="rg_A_then_z", aux=nm5 + tag("RG", "A", "g") + g1),
                     dict(q="rg_Z_unknown_id", aux=nm5 + tag("RG", "Z", "nope")),
                     dict(q="rg_none", aux=nm5)],
        # row 5: a value cut by the record end, or a B array of unknown subtype before the tag, leaves the tag absent.  The
        # reference binary appends its own Zm tag to every read before it looks tags up, and on these reads that tag is lost
        # or swallowed, so only the decoded fields are compared here, never the reference's output (DESIGN.md §9).
        "trunc": [dict(q="unknown_before_nm", aux=unknown + nm5 + sm37 + g1, flag=3),
                  dict(q="b_unknown_subtype", aux=tag("XB", "B", ("C", [1, 2, 3]))[:3] + b"q" + struct.pack("<I", 1) + b"\0" * 8 + nm5 + sm37 + g1, flag=3),
                  dict(q="b_count_past_end", aux=b"XBBC" + struct.pack("<I", 1000) + b"\0" * 4 + nm5 + g1),
                  dict(q="z_without_nul_last", aux=nm5 + g1 + b"XZZabc"),
                  dict(q="nm_cut", aux=g1 + tag("NM", "i", 3)[:5]),
                  dict(q="rg_without_nul", aux=nm5 + b"RGZg1")],
    }
    out = {}
    for name, reads in c.items():
        out[name] = []
        for k, r in enumerate(reads):
            out[name].append(dict(dict(pos=100 + 9 * k, cig="40M", flag=0, mapq=60 if k % 3 else 15, field=None), **r))
    return out


def write_corpus(d: str, samtools: str) -> List[dict]:
    """Writes every crafted BAM (+ index) and its reference under d.  Returns [dict(name, bam, fasta, regions)]."""
    from bam_readcount_b200 import synth
    out = []
    ref = _ref(1200, 7)
    synth.write_fasta(os.path.join(d, "c.fa"), "c1", np.frombuffer(ref.encode(), dtype=np.uint8))
    text = "@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:c1\tLN:1200\n" + HEADER_RG
    for name, reads in _cases(ref).items():
        rng = np.random.default_rng(len(name))
        recs = []
        for r in reads:
            cig = parse_cigar(r["cig"])
            seq, qual = _read_on(ref, r["pos"], cig, rng)
            recs.append(record(r["q"], 0, r["pos"], cig, seq, qual, r["aux"], r["flag"], r["mapq"], r["field"]))
        bam = write_bam(os.path.join(d, name + ".bam"), text, [("c1", 1200)], recs, index=samtools)
        out.append(dict(name=name, bam=bam, fasta=os.path.join(d, "c.fa"), regions=["c1:90-260"], vs_reference=name != "trunc"))
        if name.startswith("rg"):               # the same reads as CRAM: brc-readcount reads those through htslib
            cram = os.path.join(d, name + ".cram")
            subprocess.check_call([samtools, "view", "-C", "-T", os.path.join(d, "c.fa"), "-o", cram, bam])
            subprocess.check_call([samtools, "index", cram])
            out.append(dict(out[-1], name=name + "_cram", bam=cram))
    out.append(long_cigar_bam(d, samtools))
    return out


def long_cigar_bam(d: str, samtools: str) -> dict:
    """A read of 65537 CIGAR ops among ordinary reads, written as SAM text and converted by samtools, which stores its CIGAR in
    CG:B:I (the only way BAM can hold more than 65535 ops)."""
    from bam_readcount_b200 import synth
    L = 66000
    ref = _ref(L, 11)
    synth.write_fasta(os.path.join(d, "long.fa"), "c1", np.frombuffer(ref.encode(), dtype=np.uint8))
    rng = np.random.default_rng(5)
    long_cig = [("M", 1), ("D", 1)] * 32768 + [("M", 10)]
    rows = []
    for q, pos, cig in [("before", 50, "40M"), ("long", 60, None), ("mid", 100, "20M2I20M"), ("near_end", 65500, "30M"),
                        ("after", 65560, "5M1D30M")]:
        c = long_cig if cig is None else parse_cigar(cig)
        seq, qual = _read_on(ref, pos, c, rng)
        cs = "".join(f"{n}{op}" for op, n in c)
        rows.append(f"{q}\t3\tc1\t{pos + 1}\t60\t{cs}\t=\t{pos + 1}\t0\t{seq}\t{''.join(chr(x + 33) for x in qual)}\tNM:i:2\tSM:i:30\tRG:Z:g1")
    sam = os.path.join(d, "long.sam")
    with open(sam, "w") as fh:
        fh.write(f"@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:c1\tLN:{L}\n" + HEADER_RG + "\n".join(rows) + "\n")
    bam = os.path.join(d, "long.bam")
    subprocess.check_call([samtools, "view", "-b", "-o", bam, sam])
    subprocess.check_call([samtools, "index", bam])
    return dict(name="long", bam=bam, fasta=os.path.join(d, "long.fa"), regions=["c1:40-400", "c1:65480-65620"], vs_reference=True)


# ------------------------------------------------------------------------------------------------
# BGZF members made by the DEFLATE encoder (deflate_craft.py), and framing
# ------------------------------------------------------------------------------------------------
def deflate_bam(d: str) -> Tuple[str, List[int]]:
    """A BAM whose middle read carries, as its qualities, the bytes of every crafted DEFLATE member, each stored in a BGZF member
    of its own with its crafted stream.  Returns (path, [start, end) of that read's bytes in the record stream + member ends)."""
    import deflate_craft
    members = deflate_craft.corpus_members()
    payload = b"".join(m[0] for m in members)
    rng = np.random.default_rng(3)
    small = [record(f"r{k}", 0, 10 + k, [("M", 30)], "ACGT" * 7 + "AC", [int(x) for x in rng.integers(0, 41, 30)],
                    tag("NM", "i", k) + tag("RG", "Z", "g1")) for k in range(2)]
    big = record("crafted", 0, 12, [("M", len(payload))], "A" * len(payload), list(payload), tag("NM", "i", 1) + tag("RG", "Z", "g2"))
    q0 = len(small[0]) + len(big) - len(tag("NM", "i", 1) + tag("RG", "Z", "g2")) - len(payload)     # first quality byte
    data = small[0] + big + small[1]
    pieces = chunks_default(data[:q0]) + [(m[0], m[1]) for m in members] + chunks_default(data[q0 + len(payload):])
    assert b"".join(p if isinstance(p, bytes) else p[0] for p in pieces) == data
    ends, o = [], 0
    for p in pieces:
        o += len(p if isinstance(p, bytes) else p[0])
        ends.append(o)
    text = "@HD\tVN:1.6\tSO:coordinate\n@SQ\tSN:c1\tLN:1000000\n" + HEADER_RG
    path = write_bam(os.path.join(d, "deflate.bam"), text, [("c1", 1000000)], [data], members=lambda _: pieces)
    return path, [len(small[0]), len(small[0]) + len(big)] + ends


def frame_bam(d: str) -> Tuple[str, List[int], List[int]]:
    """Fourteen reads on two contigs (reads 6 and 7 on the second) in three members: one cut inside read 2, one exactly at the
    start of read 8.  Returns (path, start of every read in the record stream, member ends)."""
    rng = np.random.default_rng(9)
    recs = []
    for k in range(14):
        tid = 1 if k in (6, 7) else 0
        seq = "".join("ACGT"[int(x)] for x in rng.integers(0, 4, 50 + 7 * k))
        recs.append(record(f"f{k}", tid, 100 + 5 * k, [("M", len(seq))], seq, [int(x) for x in rng.integers(0, 41, len(seq))],
                           tag("NM", "i", k) + tag("RG", "Z", "g1" if k % 2 else "g2")))
    starts = list(np.cumsum([0] + [len(r) for r in recs[:-1]]))
    data = b"".join(recs)
    cuts = [starts[2] + 17, starts[8], len(data)]
    pieces = [data[a:b] for a, b in zip([0] + cuts[:-1], cuts)]
    text = "@HD\tVN:1.6\n@SQ\tSN:c1\tLN:5000\n@SQ\tSN:c2\tLN:5000\n" + HEADER_RG
    path = write_bam(os.path.join(d, "frame.bam"), text, [("c1", 5000), ("c2", 5000)], [data], members=lambda _: pieces)
    return path, [int(x) for x in starts], cuts
