"""Host-side decode: BGZF/BAM records, SAM header @RG->LB map, FASTA (+.fai).

The north star leaves file decode on the host ("BAM/CRAM decode and BAI/CRAI region
iteration left on the host"); this module is the Python host's decoder feeding
``ReadBatch``.  It implements the published BAM container layout (SAM spec §4) directly —
no htslib.  Region selection mirrors the index iterator's overlap rule
(V:htslib-1.10/hts.c:3229-3236) with a linear scan; a BAI reader is not needed for parity.
CRAM is out of scope for this decoder (SURVEY.md §8f).
"""
from __future__ import annotations

import gzip
import struct
from typing import Dict, List, Optional, Tuple

import numpy as np

from .batch import LIB_NONE, TAG_ABSENT, ReadBatch


class BamHeader:
    def __init__(self, text: str, names: List[str], lengths: List[int]):
        self.text = text
        self.target_names = names
        self.target_lengths = lengths
        self.tid_of = {n: i for i, n in enumerate(names)}
        # @RG ID -> LB, like sam_hdr_find_tag_id(h,"RG","ID",rg,"LB") (V:bam.c:88)
        self.rg_lb: Dict[str, Optional[str]] = {}
        for line in text.split("\n"):
            if line.startswith("@RG"):
                tags = dict(f.split(":", 1) for f in line.split("\t")[1:] if ":" in f)
                if "ID" in tags and tags["ID"] not in self.rg_lb:
                    self.rg_lb[tags["ID"]] = tags.get("LB")
        # std::set<std::string> order == byte-lexicographic (R:bamreadcount.cpp:92-111)
        self.lib_names: List[str] = sorted({lb for lb in self.rg_lb.values() if lb is not None},
                                           key=lambda s: s.encode())
        self.lib_id = {lb: i for i, lb in enumerate(self.lib_names)}

    def lib_of_rg(self, rg: Optional[str]) -> int:
        if rg is None:
            return int(LIB_NONE)
        lb = self.rg_lb.get(rg)
        if lb is None:
            return int(LIB_NONE)
        return self.lib_id[lb]


_AUX_SIZE = {"A": 1, "c": 1, "C": 1, "s": 2, "S": 2, "i": 4, "I": 4, "f": 4, "d": 8}
_AUX_INT = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<i"}   # I: bam_aux2i kept in an int32_t, as the reference does


def _skip_aux(d: bytes, o: int, end: int) -> int:
    """Offset past the value whose type byte is at d[o], or -1 when it cannot be skipped (csrc/brc_aux.cuh: skip)."""
    t = chr(d[o]); o += 1
    if t in "ZH":
        j = d.find(b"\0", o, end)
        return end if j < 0 else j + 1
    if t == "B":
        if end - o < 5:
            return -1
        es = _AUX_SIZE.get(chr(d[o]), 0)
        n = struct.unpack_from("<I", d, o + 1)[0]
        o += 5
        return -1 if es == 0 or end - o < es * n else o + es * n
    sz = _AUX_SIZE.get(t, 0)
    return -1 if sz == 0 or end - o < sz else o + sz


def _scan_aux(d: bytes, aux_o: int, end: int):
    """(NM, SM, RG ID bytes, CG type offset) of the record body d[..end) whose tags start at aux_o, by the rules of
    csrc/brc_aux.cuh: the first tag of each name; the walk stops at a value that cannot be skipped; a non-integer NM/SM is
    present and worth 0; the first RG names the read group whatever its type."""
    nm = sm = rg = cg = None
    o = aux_o
    while end - o >= 3:
        tag = d[o:o + 2]; o += 2
        e = _skip_aux(d, o, end)
        if e >= 0 and chr(d[o]) in "ZH" and d[e - 1] != 0:
            e = -2                                           # a wanted Z/H without its NUL is absent; the walk ends here anyway
        if tag in (b"NM", b"SM") and (nm if tag == b"NM" else sm) is None:
            v = False
            if e >= 0:
                t = chr(d[o])
                v = struct.unpack_from(_AUX_INT[t], d, o + 1)[0] if t in _AUX_INT else 0
            if tag == b"NM":
                nm = v
            else:
                sm = v
        elif tag == b"RG" and rg is None:
            if e >= 0:
                z = d.find(b"\0", o + 1, end)
                rg = d[o + 1:end if z < 0 else z]
            else:
                rg = False
        elif tag == b"CG" and cg is None:
            cg = o if e >= 0 else False
        if e < 0:
            break
        o = e
    # False: the first tag of that name could not be read, so the read has none
    return tuple(None if x is False else x for x in (nm, sm, rg, cg))


def read_bam(path: str) -> Tuple[BamHeader, ReadBatch]:
    """Decode a whole BAM file (BGZF members are gzip members) into one ReadBatch, file order."""
    with open(path, "rb") as fh:
        raw = gzip.decompress(fh.read())
    assert raw[:4] == b"BAM\1", "not a BAM file"
    l_text = struct.unpack_from("<i", raw, 4)[0]
    text = raw[8:8 + l_text].split(b"\0")[0].decode()
    o = 8 + l_text
    n_ref = struct.unpack_from("<i", raw, o)[0]; o += 4
    names, lens = [], []
    for _ in range(n_ref):
        ln = struct.unpack_from("<i", raw, o)[0]; o += 4
        names.append(raw[o:o + ln - 1].decode()); o += ln
        lens.append(struct.unpack_from("<i", raw, o)[0]); o += 4
    hdr = BamHeader(text, names, lens)

    tid, pos, flag, mapq, lib, lq, nm, sm = [], [], [], [], [], [], [], []
    cig_parts, seq_parts, qual_parts, qnames = [], [], [], []
    n_raw = len(raw)
    while o + 4 <= n_raw:
        bs = struct.unpack_from("<i", raw, o)[0]; o += 4
        (refid, p, l_rn, mq, _bin, n_cig, fl, l_seq, _nref, _npos, _tlen) = struct.unpack_from("<iiBBHHHiiii", raw, o)
        q = o + 32
        qnames.append(raw[q:q + l_rn - 1].decode()); q += l_rn
        cig = np.frombuffer(raw, dtype="<u4", count=n_cig, offset=q); q += 4 * n_cig
        sq = np.frombuffer(raw, dtype=np.uint8, count=(l_seq + 1) // 2, offset=q); q += (l_seq + 1) // 2
        ql = np.frombuffer(raw, dtype=np.uint8, count=l_seq, offset=q); q += l_seq
        a_nm, a_sm, a_rg, a_cg = _scan_aux(raw, q, o + bs)
        # a long CIGAR kept in CG:B:I behind a <l_qseq>S placeholder (csrc/brc_aux.cuh: scan)
        if (a_cg is not None and raw[a_cg:a_cg + 2] == b"BI" and n_cig > 0 and refid >= 0 and p >= 0
                and int(cig[0]) == (l_seq << 4 | 4)):
            n_cg = struct.unpack_from("<I", raw, a_cg + 2)[0]
            if n_cig <= n_cg < 1 << 29:
                cig = np.frombuffer(raw, dtype="<u4", count=n_cg, offset=a_cg + 6)
        o += bs
        tid.append(refid); pos.append(p); flag.append(fl); mapq.append(mq); lq.append(l_seq)
        lib.append(hdr.lib_of_rg(None if a_rg is None else a_rg.decode("utf-8", "surrogateescape")))
        nm.append(int(TAG_ABSENT) if a_nm is None else a_nm)
        sm.append(int(TAG_ABSENT) if a_sm is None else a_sm)
        cig_parts.append(cig); seq_parts.append(sq); qual_parts.append(ql)
    n = len(pos)

    def offs(parts):
        off = np.zeros(n + 1, dtype=np.uint64)
        if n:
            off[1:] = np.cumsum([x.shape[0] for x in parts])
        return off

    def cat(parts, dt):
        return np.concatenate(parts).astype(dt) if n else np.zeros(0, dtype=dt)
    batch = ReadBatch(
        tid=np.array(tid, dtype=np.int32), pos=np.array(pos, dtype=np.int32), flag=np.array(flag, dtype=np.uint16),
        mapq=np.array(mapq, dtype=np.uint8), lib=np.array(lib, dtype=np.uint16), l_qseq=np.array(lq, dtype=np.int32),
        nm=np.array(nm, dtype=np.int32), sm=np.array(sm, dtype=np.int32),
        cigar_off=offs(cig_parts), cigar=cat(cig_parts, np.uint32), seq_off=offs(seq_parts), seq=cat(seq_parts, np.uint8),
        qual_off=offs(qual_parts), qual=cat(qual_parts, np.uint8), qname=qnames)
    return hdr, batch


class Fasta:
    """Indexed FASTA (.fai) reader; ``fetch`` returns raw characters, case preserved (fai_fetch)."""

    def __init__(self, path: str):
        self.path = path
        self.index: Dict[str, Tuple[int, int, int, int]] = {}
        with open(path + ".fai") as fh:
            for line in fh:
                f = line.rstrip("\n").split("\t")
                self.index[f[0]] = (int(f[1]), int(f[2]), int(f[3]), int(f[4]))

    def length(self, name: str) -> int:
        return self.index[name][0]

    def fetch(self, name: str, beg: int = 0, end: Optional[int] = None) -> bytes:
        ln, off, lb, lw = self.index[name]
        end = ln if end is None else min(end, ln)
        beg = max(0, beg)
        if end <= beg:
            return b""
        fo = off + (beg // lb) * lw + beg % lb
        fe = off + ((end - 1) // lb) * lw + (end - 1) % lb + 1
        with open(self.path, "rb") as fh:
            fh.seek(fo)
            raw = fh.read(fe - fo)
        return raw.replace(b"\n", b"").replace(b"\r", b"")


# ------------------------------------------------------------------------------------------------
# BAI (SAM spec §5.2) and BGZF spans for the device decoder (SURVEY.md §8 f-2, engine: brc_push_bam_span)
# ------------------------------------------------------------------------------------------------
class BaiIndex:
    """Bins, chunks and the 16 kb linear index of every reference: the virtual offsets in it are starts of real records."""

    def __init__(self, path: str):
        d = open(path, "rb").read()
        assert d[:4] == b"BAI\1", "not a BAI file"
        o = 4
        n_ref, = struct.unpack_from("<i", d, o); o += 4
        self.bins: List[Dict[int, List[Tuple[int, int]]]] = []
        self.linear: List[np.ndarray] = []
        for _ in range(n_ref):
            n_bin, = struct.unpack_from("<i", d, o); o += 4
            bins: Dict[int, List[Tuple[int, int]]] = {}
            for _ in range(n_bin):
                b, n_chunk = struct.unpack_from("<Ii", d, o); o += 8
                ch = [struct.unpack_from("<QQ", d, o + 16 * k) for k in range(n_chunk)]
                o += 16 * n_chunk
                if b != 37450:
                    bins[b] = ch
            n_intv, = struct.unpack_from("<i", d, o); o += 4
            self.linear.append(np.frombuffer(d, dtype="<u8", count=n_intv, offset=o).copy())
            o += 8 * n_intv
            self.bins.append(bins)

    @staticmethod
    def reg2bins(beg: int, end: int) -> List[int]:
        end -= 1
        out = [0]
        for shift, off in ((26, 1), (23, 9), (20, 73), (17, 585), (14, 4681)):
            out += list(range(off + (beg >> shift), off + (end >> shift) + 1))
        return out

    def window_weights(self, tid: int, n_windows: int) -> np.ndarray:
        """Compressed bytes per 16 kb window from the linear index: the coverage proxy shards are balanced by."""
        lin = self.linear[tid].astype(np.int64) >> 16
        w = np.zeros(n_windows, dtype=np.float64)
        if lin.size < 2:
            return w
        filled = lin.copy()
        for i in range(1, filled.size):
            if filled[i] == 0:
                filled[i] = filled[i - 1]
        d = np.diff(filled).clip(min=0)
        w[:min(n_windows, d.size)] = d[:n_windows]
        return w


def bam_span(bam_path: str, bai: BaiIndex, tid: int, beg: int, end: int, rg_lib: Optional[Dict[str, int]] = None) -> Optional[dict]:
    """The compressed bytes and index entry points that cover every record overlapping [beg, end) of `tid` — what
    samfetch(tid, beg, end) would read — for brc_push_bam_span.  None when the index has nothing there."""
    chunks = []
    min_lin = int(bai.linear[tid][min(beg >> 14, bai.linear[tid].size - 1)]) if bai.linear[tid].size else 0
    for b in BaiIndex.reg2bins(max(beg, 0), max(end, beg + 1)):
        for cb, ce in bai.bins[tid].get(b, ()):
            if ce > min_lin:
                chunks.append((max(cb, min_lin), ce))
    if not chunks:
        return None
    v0 = min(c[0] for c in chunks)
    v1 = max(c[1] for c in chunks)
    c0, c1 = v0 >> 16, v1 >> 16
    with open(bam_path, "rb") as fh:
        fh.seek(c0)
        head = fh.read(c1 - c0 + 65536 + 32)
    # whole blocks from c0 through the block that holds v1
    o, blocks = 0, []
    while o + 18 <= len(head):
        xlen = head[o + 10] | (head[o + 11] << 8)
        bsize, i = -1, 0
        while i + 4 <= xlen:
            sl = head[o + 12 + i + 2] | (head[o + 12 + i + 3] << 8)
            if head[o + 12 + i:o + 12 + i + 2] == b"BC":
                bsize = head[o + 12 + i + 4] | (head[o + 12 + i + 5] << 8)
            i += 4 + sl
        if bsize < 0 or o + bsize + 1 > len(head):
            break
        blocks.append(o)
        o += bsize + 1
        if c0 + blocks[-1] >= c1:
            break
    comp = head[:o]
    in_span = {c0 + b for b in blocks}
    # entry points: v0, the chunk starts and the linear-index offsets that fall inside the span
    cand = {v0}
    for cb, _ in chunks:
        cand.add(cb)
    lin = bai.linear[tid]
    for w in range(min(beg >> 14, lin.size), min((end >> 14) + 2, lin.size)):
        cand.add(int(lin[w]))
    for b in BaiIndex.reg2bins(max(beg, 0), max(end, beg + 1)):
        for cb, _ in bai.bins[tid].get(b, ()):
            cand.add(cb)
    entries = sorted(v for v in cand if v0 <= v < v1 and (v >> 16) in in_span)
    rel = lambda v: (((v >> 16) - c0) << 16) | (v & 0xFFFF)      # noqa: E731
    return dict(comp=comp, entries=[rel(v) for v in entries], end_voff=rel(v1) if (v1 >> 16) in in_span else -1, tid=tid,
                rg_lib=dict(rg_lib or {}))
