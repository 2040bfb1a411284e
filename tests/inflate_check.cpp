// The DEFLATE core of the device BGZF decoder (brc_bgzf.cuh, host+device code), one lane on the CPU, against zlib: every BGZF
// member of every file named on the command line is inflated by both and compared, and must be refused when cut in half.
// Prints "<members> <failures>"; exits 1 on any failure.
#include <cstdio>
#include <cstring>
#include <vector>
#include <zlib.h>
#include "brc_bgzf.cuh"
int main(int argc, char **argv) {
    int bad = 0, nblk = 0;
    for (int a = 1; a < argc; ++a) {
        FILE *f = fopen(argv[a], "rb"); std::vector<uint8_t> d; uint8_t buf[65536]; size_t n;
        while ((n = fread(buf, 1, sizeof buf, f)) > 0) d.insert(d.end(), buf, buf + n);
        fclose(f);
        size_t o = 0; static brc::inflate::Tables T;
        while (o + 18 <= d.size()) {
            const uint8_t *h = &d[o]; if (h[0] != 31 || h[1] != 139) break;
            size_t xlen = h[10] | (h[11] << 8); int bsize = -1;
            for (size_t i = 0; i + 4 <= xlen;) { size_t sl = h[12 + i + 2] | (h[12 + i + 3] << 8); if (h[12 + i] == 'B' && h[12 + i + 1] == 'C') bsize = h[12 + i + 4] | (h[12 + i + 5] << 8); i += 4 + sl; }
            size_t total = bsize + 1, hdr = 12 + xlen; const uint8_t *tail = h + total - 4;
            uint32_t isize = tail[0] | (tail[1] << 8) | (tail[2] << 16) | ((uint32_t)tail[3] << 24);
            std::vector<uint8_t> want(isize + 1), got(isize + 1);
            z_stream zs{}; inflateInit2(&zs, -15); zs.next_in = (Bytef *)h + hdr; zs.avail_in = total - hdr - 8; zs.next_out = want.data(); zs.avail_out = isize;
            int rc = inflate(&zs, Z_FINISH); inflateEnd(&zs);
            int r = brc::inflate::inflate_block(brc::inflate::Lanes{0, 1}, h + hdr, total - hdr - 8, got.data(), isize, T);
            if (r != 0 || memcmp(want.data(), got.data(), isize) || (isize && rc != Z_STREAM_END)) ++bad;
            // a truncated stream must be refused, not over-read
            if (isize > 100 && brc::inflate::inflate_block(brc::inflate::Lanes{0, 1}, h + hdr, (total - hdr - 8) / 2, got.data(), isize, T) == 0) ++bad;
            ++nblk; o += total;
        }
    }
    printf("%d %d\n", nblk, bad);
    return bad != 0;
}
