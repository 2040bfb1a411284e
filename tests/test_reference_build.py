"""Reference preparation of the device path: the runners of one genome share each contig's generated characters
(stream.ContigReferences), and ref_encode_kernel packs them 16 bytes at a time with htslib's seq_nt16 rule."""
import numpy as np
import pytest

import boundary_cases as bc
import cases
from bam_readcount_b200 import stream as st
from bam_readcount_b200 import synth_cb


class _FakeReference:
    """Stands in for DeviceReference: records which streams were made to wait for it."""
    made = []

    def __init__(self, spec, contig, stream, device):
        self.contig, self.length, self.readers = contig, st.reference_length(spec), []
        self.ascii = self
        _FakeReference.made.append(self)

    def data_ptr(self):
        return id(self)

    def use_on(self, stream):
        self.readers.append(stream)


class _FakeEngine:
    def __init__(self):
        self.encoded = []            # (tid, ASCII pointer, stream) of every brc_set_reference_device

    def set_reference_device(self, tid, name, chrom_len, win_beg, ptr, win_len, stream_ptr):
        self.encoded.append((tid, ptr, stream_ptr))

    def close(self):
        pass


class _FakeStream:
    def __init__(self, i):
        self.cuda_stream = 1000 + i


def _runner(spec, i):
    r = object.__new__(st.WindowRunner)          # no engine handle or device buffers: only the reference bookkeeping runs
    r.spec, r.device, r.refs, r.cur_contig = spec, None, st.shared_references(spec, 0), -1
    r.stream, r.eng = _FakeStream(i), _FakeEngine()
    return r


def test_one_pass_generates_each_contig_once(monkeypatch):
    """bench.py's C4 loop (24 contigs x 10 windows dealt round-robin to three runners): 24 generations per pass, not 72; each
    handle still encodes every contig into its own window; no contig is dropped while a runner holds it."""
    made = []
    monkeypatch.setattr(_FakeReference, "made", made)
    monkeypatch.setattr(st, "DeviceReference", _FakeReference)
    spec = synth_cb.Spec(contig_len=1280 * 40, n_contigs=24)
    windows = st.wgs_windows(spec, 10)
    runners = [_runner(spec, i) for i in range(3)]
    refs = runners[0].refs
    assert all(r.refs is refs for r in runners) and st.shared_references(synth_cb.Spec(), 0) is not refs
    for _ in range(2):
        n_made, n_encoded = len(made), sum(len(r.eng.encoded) for r in runners)
        for k, w in enumerate(windows):
            run = runners[k % 3]
            run._ensure_reference(w.contig)
            live = refs.live()
            assert len(live) <= 2
            for r in runners:
                if r.cur_contig >= 0:
                    assert r.cur_contig in live, "a contig was dropped while a runner still holds it"
                    tid, ptr, sp = r.eng.encoded[-1]
                    ref = next(x for x in made if id(x) == ptr)
                    assert tid == ref.contig == r.cur_contig and r.stream in ref.readers and sp == r.stream.cuda_stream
        assert len(made) - n_made == 24
        assert sorted(x.contig for x in made[n_made:]) == list(range(24))
        assert sum(len(r.eng.encoded) for r in runners) - n_encoded == 72
    assert refs.generated == 48
    for r in runners:
        r.close()
    assert refs.live() == []


def test_runner_dropped_without_close_stops_holding_its_contig(monkeypatch):
    import gc
    monkeypatch.setattr(st, "DeviceReference", _FakeReference)
    spec = synth_cb.Spec(contig_len=1280 * 40, n_contigs=3)
    a, b = _runner(spec, 0), _runner(spec, 1)
    a._ensure_reference(0)
    b._ensure_reference(1)
    assert a.refs.live() == [0, 1]
    del b
    gc.collect()
    assert a.refs.live() == [0]
    a._ensure_reference(2)                      # the next move drops the buffer nobody holds
    assert a.refs.live() == [2] and sorted(a.refs._live) == [2]


def _nt16_pack(ascii: np.ndarray) -> np.ndarray:
    """htslib's seq_nt16 rule one character at a time, two codes per byte, then the 0xFF padding of the packed window."""
    table = np.full(256, 15, np.uint8)
    for i, c in enumerate(b"=ACMGRSVTWYHKDBN"):
        table[c] = i
        table[ord(chr(c).lower())] = i
    table[[ord("0"), ord("1"), ord("2"), ord("3")]] = [1, 2, 4, 8]
    n = len(ascii)
    codes = np.append(table[ascii], np.uint8(15)) if n % 2 else table[ascii]
    packed = (codes[0::2] << 4) | codes[1::2]
    return np.concatenate([packed, np.full(n // 2 + 32 - len(packed), 0xFF, np.uint8)])


_ODD = np.frombuffer(b"NnacgtRYKMSWBDHVrykmswbdhv=0123*.-" + bytes([1, 0x7F, 0x80, 0xFF]), np.uint8)


def _odd_reference_case(L, seed):
    """Reads from a clean ACGT contig, to and past its end; the reference the engine is given has 30 % of its bytes, its last
    three and every 16th replaced by IUPAC codes, lowercase, '=', digits and bytes htslib maps to N."""
    clean = bc._ref(seed, L)
    R = bc._Reads(clean, seed)
    for p in range(0, L, 3):
        R.add(min(p, L - 1), "50M", lib=p % 3, sub_rate=0.03)
    rng = np.random.default_rng(seed + 1)
    pick = rng.random(L) < 0.3
    pick[-3:] = True
    pick[::16] = True
    odd = clean.copy()
    odd[pick] = rng.choice(_ODD, size=int(pick.sum()))
    return bc._case(f"odd_ref_{L}", odd, R.build(), [(0, 1, L)]), odd


@pytest.mark.gpu
def test_reference_codes_equal_nt16_pack():
    """Byte for byte, padding included: every length 0-96 and 4093-4131 (every residue of the encode's 32-character group and
    of its 16-byte store), every byte value, from an aligned host upload and from device pointers at offsets 1-15."""
    import torch
    from bam_readcount_b200.engine import Engine
    rng = np.random.default_rng(77)
    e = Engine()
    try:
        tid = 0
        for L in list(range(0, 97)) + list(range(4093, 4132)):
            ascii = rng.integers(0, 256, L, dtype=np.uint8)
            ascii[::3] = rng.choice(_ODD, size=len(ascii[::3]))
            want = _nt16_pack(ascii)
            e.set_reference(tid, f"h{L}", L, ascii.tobytes(), 0)
            assert np.array_equal(e.reference_codes(tid), want), f"host upload, L={L}"
            off = 1 + L % 15
            buf = torch.zeros(L + 64, dtype=torch.uint8, device="cuda")
            buf[off:off + L].copy_(torch.from_numpy(ascii))
            torch.cuda.synchronize()
            e.set_reference_device(tid + 1, f"d{L}", L, 0, buf.data_ptr() + off, L, torch.cuda.current_stream().cuda_stream)
            assert np.array_equal(e.reference_codes(tid + 1), want), f"device pointer at offset {off}, L={L}"
            tid += 2
    finally:
        e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("L", range(600, 633))
def test_reference_encode_matches_nt16_rule(L):
    """Every length mod 32 (the encode's group), from a 16-byte aligned host upload and from a misaligned device pointer: the
    engine's mismatch statistics equal the oracle's, which reads the characters through seq_nt16 one at a time."""
    import torch
    from bam_readcount_b200.batch import ReadBatch
    from bam_readcount_b200.engine import Engine, admitted
    case, odd = _odd_reference_case(L, seed=900 + L)
    want = cases.run_oracle(case, {})
    cases.assert_same(cases.run_engine(case, {}), want, f"L={L} host reference")
    off = 1 + L % 15
    buf = torch.zeros(L + 64, dtype=torch.uint8, device="cuda")
    buf[off:off + L].copy_(torch.from_numpy(odd))
    torch.cuda.synchronize()
    e = Engine(lib_names=case["lib_names"])
    try:
        e.set_reference_device(0, "c", L, 0, buf.data_ptr() + off, L, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        pushed = cases.push_regions(e, case, case["site_list"])
        res = e.compute()
        reads = ReadBatch.concat([sub.select(admitted(sub, tid, 10_000_000)) for tid, sub in pushed])
        got = res.dump(reads, {0: (0, odd.tobytes())})
    finally:
        e.close()
    assert got == want.dump, f"L={L} device reference at offset {off}: " + cases.first_diff(got, want.dump)
