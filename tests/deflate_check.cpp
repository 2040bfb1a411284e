// The serial pieces of the device BGZF encoder (brc_deflate.cuh, host+device code), run on the CPU for tests/test_bgzf_output.py:
//   lengths MAXBITS F0 F1 ...        code lengths of the histogram, one line
//   encode dynamic|fixed|stored      stdin: tokens, one per line ("L byte" or "M length distance"), or the raw bytes for stored;
//                                    stdout: the raw DEFLATE stream (one final block) the kernel's code writes for them
//   crc CUT1 CUT2 ...                stdin: bytes; the CRC32 of the parts between the cuts, combined with crc_combine, in hex
//   member                           stdin: at most 65280 bytes; stdout: the BGZF member of a stored block holding them
//   eof                              stdout: the 28-byte EOF member
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include "brc_deflate.cuh"

using namespace brc::deflate;

static std::vector<uint8_t> read_stdin() {
    std::vector<uint8_t> d; uint8_t buf[65536]; size_t n;
    while ((n = fread(buf, 1, sizeof buf, stdin)) > 0) d.insert(d.end(), buf, buf + n);
    return d;
}
static void put_bytes(const std::vector<uint32_t> &w, uint64_t bits) { fwrite(w.data(), 1, (size_t)((bits + 7) / 8), stdout); }

int main(int argc, char **argv) {
    if (argc < 2) return 2;
    static LenWork W;
    const std::string cmd = argv[1];
    if (cmd == "lengths") {
        const int maxbits = atoi(argv[2]), n = argc - 3;
        std::vector<uint32_t> f(n); std::vector<uint8_t> len(n);
        for (int i = 0; i < n; ++i) f[i] = (uint32_t)strtoul(argv[3 + i], nullptr, 10);
        build_lengths(f.data(), n, maxbits, len.data(), W);
        for (int i = 0; i < n; ++i) printf("%d%c", len[i], i + 1 < n ? ' ' : '\n');
        return 0;
    }
    if (cmd == "encode") {
        const std::string mode = argv[2];
        std::vector<uint32_t> out(1 << 16, 0);
        Sink s; sink_init(s, out.data(), 0);
        if (mode == "stored") {
            const std::vector<uint8_t> d = read_stdin();
            put_stored_header(s, (int)d.size());
            for (uint8_t b : d) sink_put(s, b, 8);
            sink_flush(s);
            put_bytes(out, sink_pos(s));
            return 0;
        }
        std::vector<uint32_t> tok;                        // len << 16 | dist, or the literal byte with len 0
        char kind; int a, b = 0;
        while (scanf(" %c %d", &kind, &a) == 2) {
            if (kind == 'M') { if (scanf("%d", &b) != 1) return 2; tok.push_back((uint32_t)a << 16 | (uint32_t)b); }
            else tok.push_back((uint32_t)a);
        }
        static uint32_t lf[LCODES], df[DCODES];
        static Codes C; static DynHeader H;
        int e, v;
        for (uint32_t t : tok) {
            if (t >> 16) { lf[len_sym((int)(t >> 16), e, v)]++; df[dist_sym((int)(t & 0xffff), e, v)]++; }
            else lf[t]++;
        }
        lf[256]++;
        if (mode == "fixed") {
            fixed_codes(C, W.blc);
            sink_put(s, 3, 3);
        } else {
            build_lengths(lf, LCODES, MAXBITS, C.llen, W);
            build_lengths(df, DCODES, MAXBITS, C.dlen, W);
            canonical(C.llen, 288, C.lcode, W.blc);
            canonical(C.dlen, 32, C.dcode, W.blc);
            dyn_header(C, H, W);
            sink_put(s, 5, 3);
            put_dyn_header(s, H);
            if (sink_pos(s) != 3 + H.bits) { fprintf(stderr, "header size %llu, expected %u\n", (unsigned long long)sink_pos(s), 3 + H.bits); return 1; }
        }
        const uint64_t p0 = sink_pos(s);
        uint64_t want = 0;
        for (uint32_t t : tok) {
            if (t >> 16) { put_match(s, C, (int)(t >> 16), (int)(t & 0xffff)); want += match_bits(C, (int)(t >> 16), (int)(t & 0xffff)); }
            else { put_literal(s, C, (int)t); want += literal_bits(C, (int)t); }
        }
        put_eob(s, C);
        sink_flush(s);
        if (sink_pos(s) - p0 != payload_bits(C, lf, df) || sink_pos(s) - p0 != want + C.llen[256]) { fprintf(stderr, "payload size mismatch\n"); return 1; }
        put_bytes(out, sink_pos(s));
        return 0;
    }
    if (cmd == "crc") {
        const std::vector<uint8_t> d = read_stdin();
        static uint32_t T[256];
        for (uint32_t i = 0; i < 256; ++i) T[i] = crc_table_entry(i);
        std::vector<size_t> cut{0};
        for (int i = 2; i < argc; ++i) cut.push_back((size_t)strtoull(argv[i], nullptr, 10));
        cut.push_back(d.size());
        uint32_t crc = 0;
        for (size_t k = 0; k + 1 < cut.size(); ++k) {
            const uint32_t part = crc_update(T, 0, d.data() + cut[k], (int64_t)(cut[k + 1] - cut[k]));
            crc = k == 0 ? part : crc_combine(crc, part, cut[k + 1] - cut[k]);
        }
        printf("%08x\n", crc);
        return 0;
    }
    if (cmd == "member") {
        const std::vector<uint8_t> d = read_stdin();
        if (d.size() > (size_t)BLOCK) return 2;
        static uint32_t T[256];
        for (uint32_t i = 0; i < 256; ++i) T[i] = crc_table_entry(i);
        const uint32_t member = HDR + STORED_OVERHEAD + (uint32_t)d.size() + TRAILER;
        std::vector<uint32_t> out(1 << 15, 0);
        Sink s; sink_init(s, out.data(), 0);
        put_member_header(s, member);
        put_stored_header(s, (int)d.size());
        for (uint8_t b : d) sink_put(s, b, 8);
        put_member_trailer(s, crc_update(T, 0, d.data(), (int64_t)d.size()), (uint32_t)d.size());
        sink_flush(s);
        put_bytes(out, sink_pos(s));
        return 0;
    }
    if (cmd == "eof") {
        for (int i = 0; i < 28; ++i) putchar(eof_byte(i));
        return 0;
    }
    return 2;
}
