"""A small raw-DEFLATE (RFC 1951) encoder for tests: stored, fixed and dynamic blocks built from explicit tokens and explicit code
lengths, so a test can put exactly the constructs it names into a stream.  Every stream is checked against zlib
(wbits=-15) before it is used, and the encoder records which constructs it emitted (`Stream.seen`) so a test can assert that
its corpus covers them.

Tokens: an int 0..255 is a literal, a tuple (length, distance) a match."""
from __future__ import annotations

import zlib
from typing import Dict, List, Sequence, Set, Tuple, Union

Token = Union[int, Tuple[int, int]]

LEN_BASE = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
LEN_EXTRA = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
DIST_BASE = [1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145,
             8193, 12289, 16385, 24577]
DIST_EXTRA = [0, 0, 0, 0] + [e for e in range(1, 14) for _ in (0, 1)]
CL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
FIXED_LIT = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
FIXED_DIST = [5] * 30


def len_code(n: int) -> Tuple[int, int, int]:
    """(symbol 257.., extra bits, extra value) of a match length; 258 is symbol 285."""
    i = 28 if n == 258 else max(k for k in range(28) if LEN_BASE[k] <= n)
    return 257 + i, LEN_EXTRA[i], n - LEN_BASE[i]


def dist_code(d: int) -> Tuple[int, int, int]:
    i = max(k for k in range(30) if DIST_BASE[k] <= d)
    return i, DIST_EXTRA[i], d - DIST_BASE[i]


def canonical(lengths: Sequence[int]) -> List[int]:
    """Canonical Huffman codes (RFC 1951 §3.2.2) of the given code lengths."""
    bl = [0] * 16
    for l in lengths:
        if l:
            bl[l] += 1
    code, nxt = 0, [0] * 16
    for b in range(1, 16):
        code = (code + bl[b - 1]) << 1 if b > 1 else 0
        nxt[b] = code
    out = [0] * len(lengths)
    for s, l in enumerate(lengths):
        if l:
            out[s] = nxt[l]
            nxt[l] += 1
    return out


def chain_lengths(n: int, chain: Sequence[int], top: int = 15) -> List[int]:
    """A complete code over n symbols in which the symbols of `chain` get the lengths of a leaf split len(chain)-1 times (k+1,
    k+2, ..., top, top), the others a balanced code.  That puts codes of every length up to `top` on chosen symbols."""
    t = len(chain) - 1
    m = n - t                                   # balanced over m symbols, then one leaf of length top - t is split t times
    L = max(1, (m - 1).bit_length())
    n_short = (1 << L) - m                      # symbols of length L - 1
    lens = [L - 1] * n_short + [L] * (m - n_short)
    assert lens[-1] == top - t, (lens[-1], top, t)
    rest = [s for s in range(n) if s not in chain]
    out = [0] * n
    for s, l in zip(rest, lens[:-1]):
        out[s] = l
    for k, s in enumerate(chain):
        out[s] = min(top - t + 1 + k, top)
    return out


def balanced(symbols: Sequence[int], n: int) -> List[int]:
    m = len(symbols)
    L = max(1, (m - 1).bit_length())
    n_short = (1 << L) - m
    out = [0] * n
    for k, s in enumerate(symbols):
        out[s] = L - 1 if k < n_short else L
    return out


class Stream:
    def __init__(self):
        self.bits: List[int] = []
        self.out = bytearray()
        self.seen: Set[str] = set()
        self.blocks: List[str] = []
        self.matches: Set[Tuple[int, int]] = set()

    def put(self, v: int, n: int):                       # LSB first
        for i in range(n):
            self.bits.append((v >> i) & 1)

    def put_code(self, code: int, n: int):               # Huffman codes go MSB first
        for i in range(n - 1, -1, -1):
            self.bits.append((code >> i) & 1)

    def stored(self, data: bytes, last: bool = False):
        assert len(data) <= 65535
        if self.blocks and self.blocks[-1] == "fixed" and len(self.bits) % 8:
            self.seen.add("stored_after_fixed_mid_byte")
        self.put(int(last), 1); self.put(0, 2)
        while len(self.bits) % 8:
            self.bits.append(0)
        self.put(len(data), 16); self.put(len(data) ^ 0xFFFF, 16)
        for b in data:
            self.put(b, 8)
        self.out += data
        self.seen.add(f"stored_{len(data)}")
        self.blocks.append("stored")

    def fixed(self, tokens: Sequence[Token], last: bool = False):
        self.put(int(last), 1); self.put(1, 2)
        self._tokens(tokens, FIXED_LIT, FIXED_DIST, "fixed")
        for b in tokens:
            if isinstance(b, int):
                self.seen.add("fixed_lit_8bit" if b < 144 else "fixed_lit_9bit")
        if len(self.blocks) >= 2 and self.blocks[-2:] == ["fixed", "dynamic"]:
            self.seen.add("fixed_dynamic_fixed")
        self.blocks.append("fixed")

    def dynamic(self, tokens: Sequence[Token], lit: Sequence[int], dist: Sequence[int], last: bool = False, zero_run_16: bool = False):
        """lit / dist: the code lengths (len(lit) = HLIT + 257, len(dist) = HDIST + 1).  The code-length code is a fixed complete
        code over all 19 symbols; runs use 16/17/18 (zero runs as 0 + 16 when zero_run_16)."""
        nlen, ndist = len(lit), len(dist)
        seq = list(lit) + list(dist)
        rle: List[Tuple[int, int, int, int]] = []          # (symbol, extra bits, extra value, first index it covers)
        i = 0
        while i < len(seq):
            v, r = seq[i], 1
            while i + r < len(seq) and seq[i + r] == v:
                r += 1
            if v == 0 and r >= 11 and not zero_run_16:
                k = min(r, 138); rle.append((18, 7, k - 11, i)); i += k; continue
            if v == 0 and r >= 3 and not zero_run_16:
                k = min(r, 10); rle.append((17, 3, k - 3, i)); i += k; continue
            rle.append((v, 0, 0, i)); i += 1; r -= 1
            while r >= 3:
                k = min(r, 6)
                rle.append((16, 2, k - 3, i))
                if i < nlen <= i + k - 1:
                    self.seen.add("code16_across_lit_dist")
                i += k; r -= k
            # a remainder of 1-2 goes round the loop as literals
        cl_lens = [4 if s < 13 else 5 for s in range(19)]      # 13 x 4 bits + 6 x 5 bits: complete
        cl_codes = canonical(cl_lens)
        self.put(int(last), 1); self.put(2, 2)
        self.put(nlen - 257, 5); self.put(ndist - 1, 5); self.put(19 - 4, 4)
        for s in CL_ORDER:
            self.put(cl_lens[s], 3)
        for sym, eb, ev, _ in rle:
            self.put_code(cl_codes[sym], cl_lens[sym])
            if eb:
                self.put(ev, eb)
        if nlen == 286:
            self.seen.add("nlen_286")
        if ndist == 30:
            self.seen.add("ndist_30")
        if sum(1 for l in dist if l) == 1:
            self.seen.add("single_code_dist_tree")
        self._tokens(tokens, lit, dist, "dynamic")
        self.blocks.append("dynamic")

    def _tokens(self, tokens, lit, dist, kind):
        lc, dc = canonical(lit), canonical(dist)
        prev = None
        for t in tokens:
            if isinstance(t, int):
                assert lit[t], t
                self.put_code(lc[t], lit[t])
                if kind == "dynamic":
                    self.seen.add(f"lit_code_{lit[t]}bits")
                self.out.append(t)
            else:
                n, d = t
                o = len(self.out)
                assert 3 <= n <= 258 and 1 <= d <= o, t
                s, eb, ev = len_code(n)
                assert lit[s], s
                self.put_code(lc[s], lit[s]); self.put(ev, eb)
                ds, deb, dev = dist_code(d)
                assert dist[ds], ds
                self.put_code(dc[ds], dist[ds]); self.put(dev, deb)
                if kind == "dynamic":
                    self.seen.add(f"lit_code_{lit[s]}bits")
                    self.seen.add(f"dist_code_{dist[ds]}bits")
                for k in range(n):
                    self.out.append(self.out[o - d + k])
                self.matches.add((n, d))
                if d == 32768:
                    self.seen.add("dist_32768")
                if d == n:
                    self.seen.add("dist_eq_len")
                if d == n + 1:
                    self.seen.add("dist_eq_len_plus_1")
                if isinstance(prev, int) and d == 1:
                    self.seen.add("literal_then_dist_1")
                if isinstance(prev, tuple) and prev[2] <= o - d < o:     # reads bytes the previous match wrote
                    self.seen.add("match_reads_previous_match")
                prev = (n, d, o)
                continue
            prev = t
        self.put_code(lc[256], lit[256])

    def finish(self) -> bytes:
        bits = self.bits + [0] * (-len(self.bits) % 8)
        raw = bytes(sum(bits[i + k] << k for k in range(8)) for i in range(0, len(bits), 8))
        assert zlib.decompress(raw, -15) == bytes(self.out), "stream does not inflate under zlib to the intended bytes"
        return raw


def _rand(n: int, seed: int) -> bytes:
    import random
    r = random.Random(seed)
    return bytes(r.randrange(256) for _ in range(n))


STORED_MAX = 65480


def corpus_members() -> List[Tuple[bytes, bytes, Set[str], Set[Tuple[int, int]]]]:
    """The crafted members: [(inflated bytes, raw DEFLATE stream, constructs, (length, distance) matches)]."""
    out = []

    def done(s: Stream):
        out.append((bytes(s.out), s.finish(), set(s.seen), set(s.matches)))

    # 1. fixed (8- and 9-bit literals, ends mid-byte) -> stored 0 -> stored 1 -> fixed (literal + distance-1 match) ->
    #    dynamic -> fixed: the fixed tables are rebuilt after the dynamic block
    s = Stream()
    s.fixed([0x41, 0x90, 0xC8, 0xFF, 0x00, (258, 1), 0x7E])
    s.stored(b"")
    s.stored(b"\x5a")
    s.fixed([0x33, (10, 1), 0xA0, 0xA1])
    lit = balanced(list(range(258)), 260)
    s.dynamic([0x10, 0x20, 0x30, 0x40, (3, 4), (3, 4), 0xEE], lit, [0, 0, 0, 1], zero_run_16=True)   # single-code distance tree;
    s.fixed([0xF0, 0x0F, (5, 2)], last=True)                                                          # a 16 crosses lit/dist
    done(s)

    # 2. fixed: 32768 literals, a match at distance 32768, length 258 at every distance 1..33 and 64, dist = len,
    #    dist = len + 1, back-to-back matches where the second reads what the first wrote
    s = Stream()
    toks: List[Token] = list(_rand(32768, 1))
    toks.append((258, 32768))
    for d in list(range(1, 34)) + [64]:
        toks += [0x55, (258, d)]
    toks += [0x61, (10, 10), 0x62, (10, 11), (20, 5), (20, 15), (258, 40)]
    s.fixed(toks, last=True)
    done(s)

    # 3. dynamic, nlen = 286 and ndist = 30, codes of 10-15 bits on used literal / length and distance symbols
    s = Stream()
    lit = chain_lengths(286, [65, 66, 285, 67, 68, 69, 284])
    dist = chain_lengths(30, list(range(11)))
    toks = [65, 66, 67, 68, 69, 70, 71]
    for d in (1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 40):
        toks += [66, (258, d), 67, (250, d), 68]
    s.dynamic(toks, lit, dist, last=True)
    done(s)

    # 4. a member of 65536 bytes: a stored block as large as a BGZF member leaves room for (a 65535-byte one cannot fit the
    #    member's 64 KiB limit with its own header and trailer), then a fixed block of a literal and a match
    s = Stream()
    s.stored(_rand(STORED_MAX, 2))
    s.fixed([0x99, (65536 - STORED_MAX - 1, 1)], last=True)
    done(s)

    # 5. an empty member mid-span
    s = Stream()
    s.stored(b"", last=True)
    done(s)
    return out


REQUIRED = ({"stored_0", "stored_1", f"stored_{STORED_MAX}", "stored_after_fixed_mid_byte", "fixed_lit_8bit", "fixed_lit_9bit", "dist_32768",
             "fixed_dynamic_fixed", "single_code_dist_tree", "code16_across_lit_dist", "nlen_286", "ndist_30", "dist_eq_len",
             "dist_eq_len_plus_1", "literal_then_dist_1", "match_reads_previous_match"}
            | {f"lit_code_{b}bits" for b in range(11, 16)} | {f"dist_code_{b}bits" for b in range(10, 16)})
REQUIRED_MATCHES = {(258, d) for d in list(range(1, 34)) + [64]}


def audit(members) -> Dict[str, bool]:
    """Which required constructs the members hold (all must be True)."""
    seen = set().union(*(m[2] for m in members))
    matches = set().union(*(m[3] for m in members))
    res = {k: k in seen for k in sorted(REQUIRED)}
    res.update({f"len258_dist{d}": (258, d) in matches for _, d in sorted(REQUIRED_MATCHES)})
    res["member_isize_65536"] = any(len(m[0]) == 65536 for m in members)
    res["empty_member"] = any(len(m[0]) == 0 for m in members)
    return res
