// brc_deflate.cu — BGZF output compressed on the device (brc_bgzf_open / brc_bgzf_write / brc_bgzf_close, DESIGN.md §13).
//
// The byte stream is cut into members of BLOCK (65280) input bytes, as bgzip cuts it; the writer stages up to CHUNK_BLOCKS
// of them in page-locked memory and hands them to the device in one launch.  One CTA encodes one block:
//   1. match finding: the block in shared memory; a 12-bit hash of the 4 bytes at each position; the candidates of a
//      position are the WAYS nearest earlier positions with its hash.  Positions are taken CTA at a time: a block-wide sort
//      of (hash, position) gives each position its earlier same-hash partners inside the round, and a WAYS-deep table per
//      hash the ones of earlier rounds.  The longest match (distance <= 32768, length <= 258; the nearer one on a tie)
//      is kept per position.
//   2. greedy parse, next(i) = i + max(1, len(i)): each thread walks its 256 positions from a guessed entry, then takes the
//      exit of the thread before it as its entry and walks again only where that entry is not on its own path — a few
//      rounds, and the parse is exactly the serial one.
//   3. histogram of the tokens; on one thread, 15-bit-limited code lengths, the dynamic header and the sizes of the
//      dynamic, fixed and stored encodings (brc_deflate.cuh); the smallest is written.
//   4. a block-wide exclusive scan of the threads' token bits gives each thread its bit offset; every thread writes its
//      tokens into the member's 64 KiB slot through the OR-ing bit sink.  CRC32: per thread over its segment, shifted by
//      the bytes after it and XOR-ed together.
// Then brc_scan.cuh's scan of the member sizes places the members back to back, and a copy kernel writes them straight into
// the page-locked output buffer, which the host writes to the file descriptor in chunk order.
//
// The bytes depend on the input stream alone: how it was split into writes, the chunking and the device play no part.
#include <algorithm>
#include <cerrno>
#include <cstdlib>
#include <cstring>
#include <new>
#include <unistd.h>
#include <cuda_runtime.h>
#include <cub/block/block_radix_sort.cuh>
#include <cub/block/block_scan.cuh>

#include "../../include/brc_engine.h"
#include "brc_deflate.cuh"
#include "brc_scan.cuh"

namespace brc {
namespace deflate {

constexpr int CTA = 256, SEG = 256;                    // thread t parses and encodes positions [SEG t, SEG t + SEG)
static_assert(CTA * SEG >= BLOCK, "the threads' segments cover a block");
constexpr int HASH_BITS = 12, HASH_SIZE = 1 << HASH_BITS, WAYS = 4;
constexpr uint32_t NO_HASH = HASH_SIZE;                // key of a position with fewer than 4 bytes left
constexpr uint16_t EMPTY = 0xffff;
constexpr int CHUNK_BLOCKS = 256;
constexpr int64_t CHUNK_BYTES = (int64_t)CHUNK_BLOCKS * BLOCK;
constexpr int SLOT_WORDS = MAX_MEMBER / 4;

using Sort = cub::BlockRadixSort<uint32_t, CTA, 1>;
using Scan = cub::BlockScan<uint32_t, CTA>;

struct Encode {                                        // the parse and encode phase, in the space the hash table had
    uint32_t vis[CTA * SEG / 32];                      // the positions the parse visits
    uint32_t lf[LCODES], df[DCODES];
    Codes C, F;                                        // dynamic and fixed
    DynHeader H;
    LenWork W;
};
struct Smem {
    uint32_t data[(BLOCK + 16) / 4];                   // the block, zero-padded
    union {
        uint16_t table[HASH_SIZE][WAYS];               // the WAYS latest positions of each hash, nearest first
        Encode e;
    } u;
    union { Sort::TempStorage sort; Scan::TempStorage scan; } cub;
    uint32_t keys[CTA], exitp[CTA], crc_t[256], red[CTA / 32];
    int mode; uint32_t start_bits, dbytes;
};

__device__ __forceinline__ uint32_t ld32(const uint32_t *d, int i) {   // the 4 bytes at byte i
    return __funnelshift_r(d[i >> 2], d[(i >> 2) + 1], (i & 3) * 8);
}
__device__ __forceinline__ int match_len(const uint32_t *d, int p, int c, int maxl) {
    int k = 0;
    while (k < maxl) {
        const uint32_t x = ld32(d, p + k) ^ ld32(d, c + k);
        if (x) { k += (__ffs((int)x) - 1) >> 3; break; }
        k += 4;
    }
    return min(k, maxl);
}
__device__ __forceinline__ uint32_t token_bits(const Codes &C, const uint8_t *db, uint32_t m, int pos) {
    return m ? match_bits(C, (int)(m >> 16), (int)(m & 0xffff)) : literal_bits(C, db[pos]);
}

// One CTA per BGZF member.  match: BLOCK words of scratch per block; slots: MAX_MEMBER bytes per block; sizes: member bytes.
__global__ void __launch_bounds__(CTA, 2) deflate_blocks_kernel(const uint8_t *__restrict__ in, int64_t n_in, uint32_t *__restrict__ match,
                                                                uint32_t *__restrict__ slots, uint32_t *__restrict__ sizes) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    Smem &S = *reinterpret_cast<Smem *>(smem_raw);
    const int t = threadIdx.x;
    const int64_t base = (int64_t)blockIdx.x * BLOCK;
    const int n = (int)(n_in - base < BLOCK ? n_in - base : BLOCK);
    uint32_t *slot = slots + (size_t)blockIdx.x * SLOT_WORDS;
    uint32_t *mt = match + (size_t)blockIdx.x * BLOCK;
    const uint8_t *db = reinterpret_cast<const uint8_t *>(S.data);

    // ---- stage ----
    const uint8_t *src = in + base;                    // 4-byte aligned: BLOCK is a multiple of 4
    for (int w = t; w < (BLOCK + 16) / 4; w += CTA) {
        uint32_t v = 0;
        if (4 * w + 4 <= n) v = reinterpret_cast<const uint32_t *>(src)[w];
        else for (int k = 0; k < 4 && 4 * w + k < n; ++k) v |= (uint32_t)src[4 * w + k] << (8 * k);
        S.data[w] = v;
    }
    for (int w = t; w < SLOT_WORDS; w += CTA) slot[w] = 0;
    for (int w = t; w < HASH_SIZE * WAYS / 2; w += CTA) reinterpret_cast<uint32_t *>(S.u.table)[w] = 0xffffffffu;
    S.crc_t[t] = crc_table_entry((uint32_t)t);
    __syncthreads();

    // ---- 1. match finding, CTA positions per round ----
    for (int r0 = 0; r0 < n; r0 += CTA) {
        const int p = r0 + t;
        uint32_t key[1] = {(p + 4 <= n ? (ld32(S.data, p) * 2654435761u) >> (32 - HASH_BITS) : NO_HASH) << 8 | (uint32_t)t};
        Sort(S.cub.sort).Sort(key, 0, HASH_BITS + 1 + 8);
        S.keys[t] = key[0];
        __syncthreads();
        const uint32_t h = key[0] >> 8;
        const int q = r0 + (int)(key[0] & 255u);      // the position this thread now evaluates
        if (h != NO_HASH) {
            const int maxl = min(MAX_MATCH, n - q);
            int best = 0, bd = 0, nc = 0;
            auto consider = [&](int c) {
                const int d = q - c;
                if (d > WINDOW || best >= maxl) return false;
                const int l = match_len(S.data, q, c, maxl);
                if (l > best) { best = l; bd = d; }
                return true;
            };
            for (int j = t - 1; j >= 0 && nc < WAYS && (S.keys[j] >> 8) == h; --j, ++nc)
                if (!consider(r0 + (int)(S.keys[j] & 255u))) break;
            for (int w = 0; nc < WAYS; ++w, ++nc) {
                const uint16_t c = S.u.table[h][w];
                if (c == EMPTY || !consider(c)) break;
            }
            mt[q] = best >= MIN_MATCH ? (uint32_t)best << 16 | (uint32_t)bd : 0u;
        } else if (q < n) mt[q] = 0;
        __syncthreads();
        // the last position of each hash in the round pushes the round's positions of that hash into its table entry
        if (h != NO_HASH && (t == CTA - 1 || (S.keys[t + 1] >> 8) != h)) {
            int m = 1;
            while (m < WAYS && m <= t && (S.keys[t - m] >> 8) == h) ++m;
            for (int w = WAYS - 1; w >= m; --w) S.u.table[h][w] = S.u.table[h][w - m];
            for (int i = 0; i < m; ++i) S.u.table[h][i] = (uint16_t)(r0 + (int)(S.keys[t - i] & 255u));
        }
        __syncthreads();
    }

    // ---- 2. greedy parse ----
    Encode &E = S.u.e;
    for (int s = t; s < LCODES + DCODES; s += CTA) (s < LCODES ? E.lf[s] : E.df[s - LCODES]) = 0;
    const int lo = t * SEG, hi = min(lo + SEG, n);
    int entry = lo;
    bool dirty = lo < n;
    for (;;) {
        if (dirty) {
            for (int w = 0; w < SEG / 32; ++w) E.vis[t * (SEG / 32) + w] = 0;
            int pos = entry;
            while (pos < hi) { E.vis[pos >> 5] |= 1u << (pos & 31); const uint32_t m = mt[pos]; pos += m ? (int)(m >> 16) : 1; }
            S.exitp[t] = (uint32_t)pos;
            dirty = false;
        }
        __syncthreads();
        if (t > 0 && lo < n) {
            const int ne = (int)S.exitp[t - 1];
            if (ne != entry) {
                if (ne < hi && (E.vis[ne >> 5] >> (ne & 31) & 1u)) {   // on this thread's path: drop the positions before it
                    for (int w = lo >> 5; w < (ne >> 5); ++w) E.vis[w] = 0;
                    if (ne & 31) E.vis[ne >> 5] &= ~0u << (ne & 31);
                } else dirty = true;
                entry = ne;
            }
        }
        if (!__syncthreads_or(dirty)) break;
    }

    // ---- 3. histogram, codes, mode ----
    for (int pos = entry; pos < hi;) {
        const uint32_t m = mt[pos];
        int e, v;
        if (m) { atomicAdd(&E.lf[len_sym((int)(m >> 16), e, v)], 1u); atomicAdd(&E.df[dist_sym((int)(m & 0xffff), e, v)], 1u); pos += (int)(m >> 16); }
        else { atomicAdd(&E.lf[db[pos]], 1u); ++pos; }
    }
    if (t == 0) atomicAdd(&E.lf[256], 1u);             // end of block
    __syncthreads();
    if (t == 0) {
        build_lengths(E.lf, LCODES, MAXBITS, E.C.llen, E.W);
        build_lengths(E.df, DCODES, MAXBITS, E.C.dlen, E.W);
        E.C.llen[286] = E.C.llen[287] = 0; E.C.dlen[30] = E.C.dlen[31] = 0;
        canonical(E.C.llen, 288, E.C.lcode, E.W.blc);
        canonical(E.C.dlen, 32, E.C.dcode, E.W.blc);
        dyn_header(E.C, E.H, E.W);
        fixed_codes(E.F, E.W.blc);
        const uint64_t dyn = (3 + E.H.bits + payload_bits(E.C, E.lf, E.df) + 7) / 8;
        const uint64_t fix = (3 + payload_bits(E.F, E.lf, E.df) + 7) / 8;
        const uint64_t sto = (uint64_t)n + STORED_OVERHEAD;
        S.mode = dyn < fix && dyn < sto ? DYNAMIC : fix < sto ? FIXED : STORED;
        S.dbytes = (uint32_t)(S.mode == DYNAMIC ? dyn : S.mode == FIXED ? fix : sto);
        S.start_bits = HDR * 8 + 3 + (S.mode == DYNAMIC ? E.H.bits : 0);
        Sink s;
        sink_init(s, slot, HDR * 8);
        if (S.mode == STORED) put_stored_header(s, n);
        else { sink_put(s, S.mode == DYNAMIC ? 5u : 3u, 3); if (S.mode == DYNAMIC) put_dyn_header(s, E.H); }
        sink_flush(s);
    }
    __syncthreads();

    // ---- 4. the payload ----
    const int mode = S.mode;
    if (mode == STORED) {
        if (lo < n) {
            Sink s;
            sink_init(s, slot, (uint64_t)(HDR + STORED_OVERHEAD + lo) * 8);
            for (int pos = lo; pos < hi; ++pos) sink_put(s, db[pos], 8);
            sink_flush(s);
        }
    } else {
        const Codes &C = mode == DYNAMIC ? E.C : E.F;
        uint32_t bits = 0;
        for (int pos = entry; pos < hi;) { const uint32_t m = mt[pos]; bits += token_bits(C, db, m, pos); pos += m ? (int)(m >> 16) : 1; }
        uint32_t off, total;
        Scan(S.cub.scan).ExclusiveSum(bits, off, total);
        Sink s;
        sink_init(s, slot, S.start_bits + off);
        for (int pos = entry; pos < hi;) {
            const uint32_t m = mt[pos];
            if (m) { put_match(s, C, (int)(m >> 16), (int)(m & 0xffff)); pos += (int)(m >> 16); }
            else { put_literal(s, C, db[pos]); ++pos; }
        }
        sink_flush(s);
        if (t == 0) { sink_init(s, slot, S.start_bits + total); put_eob(s, C); sink_flush(s); }
    }

    // ---- CRC32 and the framing ----
    uint32_t crc = lo < n ? crc_shift(crc_update(S.crc_t, 0, db + lo, hi - lo), (uint64_t)(n - hi)) : 0u;
    for (int o = 16; o; o >>= 1) crc ^= __shfl_xor_sync(0xffffffffu, crc, o);
    if ((t & 31) == 0) S.red[t >> 5] = crc;
    __syncthreads();
    if (t == 0) {
        for (int w = 1; w < CTA / 32; ++w) crc ^= S.red[w];
        const uint32_t member = HDR + S.dbytes + TRAILER;
        Sink s;
        sink_init(s, slot, 0);
        put_member_header(s, member);
        sink_flush(s);
        sink_init(s, slot, (uint64_t)(HDR + S.dbytes) * 8);
        put_member_trailer(s, crc, (uint32_t)n);
        sink_flush(s);
        sizes[blockIdx.x] = member;
    }
}

// The members of a chunk back to back at their scanned offsets, written straight into page-locked host memory.
__global__ void __launch_bounds__(256) pack_members_kernel(const uint32_t *__restrict__ slots, const uint32_t *__restrict__ sizes,
                                                           const uint64_t *__restrict__ off, uint8_t *__restrict__ out) {
    const uint8_t *src = reinterpret_cast<const uint8_t *>(slots + (size_t)blockIdx.x * SLOT_WORDS);
    uint8_t *dst = out + off[blockIdx.x];
    const uint32_t n = sizes[blockIdx.x];
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

}  // namespace deflate
}  // namespace brc

using namespace brc::deflate;

// Two staging sets: the host fills one while the device compresses the other.  Device buffers are shared, the stream
// orders their use; the output of each set is page-locked, mapped memory that the pack kernel fills.
struct brc_bgzf_writer {
    int fd = -1, device = 0;
    int status = BRC_OK, saved_errno = 0;              // the first failure; returned by every later call
    bool touched = false, ready = false;               // allocation begun / completed (at the first write)
    cudaStream_t stream = nullptr;
    uint8_t *h_in[2] = {nullptr, nullptr}, *h_out[2] = {nullptr, nullptr};
    uint64_t *h_off[2] = {nullptr, nullptr};           // per set: the members' offsets, [n_blocks] = the chunk's bytes
    cudaEvent_t done[2] = {nullptr, nullptr}, k0[2] = {nullptr, nullptr};
    int n_blocks[2] = {0, 0};
    bool pending[2] = {false, false};
    int cur = 0; int64_t fill = 0;
    uint8_t *d_in = nullptr; uint32_t *d_match = nullptr, *d_slots = nullptr, *d_sizes = nullptr; unsigned long long *d_partial = nullptr;
    double kernel_ms = 0; int64_t bytes_in = 0, bytes_out = 0;
};

namespace {

int cuda_fail(brc_bgzf_writer *w) { cudaGetLastError(); if (w->status == BRC_OK) w->status = BRC_E_CUDA; return w->status; }

// The writer's first failure, with errno set back to the failed write()'s when it was one.
int result(const brc_bgzf_writer *w) {
    if (w->status == BRC_E_IO) errno = w->saved_errno;
    return w->status;
}

// The writer's device is current while a call works on it; the caller's current device is restored afterwards.
struct DeviceScope {
    int prev = -1;
    explicit DeviceScope(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; }
        if (prev != dev) cudaSetDevice(dev);
    }
    DeviceScope(const DeviceScope &) = delete;
    ~DeviceScope() {
        int cur = -1;
        if (prev >= 0 && cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
        cudaGetLastError();
    }
};

bool write_fd(brc_bgzf_writer *w, const uint8_t *p, size_t n) {
    while (n > 0) {
        const ssize_t k = ::write(w->fd, p, n);
        if (k < 0) {
            if (errno == EINTR) continue;
            if (w->status == BRC_OK) { w->status = BRC_E_IO; w->saved_errno = errno; }
            return false;
        }
        p += k; n -= (size_t)k;
    }
    return true;
}

int setup(brc_bgzf_writer *w) {
    w->touched = true;
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != w->device) return cuda_fail(w);
    const size_t smem = sizeof(Smem);
    bool ok = cudaFuncSetAttribute(deflate_blocks_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) == cudaSuccess &&
              cudaStreamCreateWithFlags(&w->stream, cudaStreamNonBlocking) == cudaSuccess &&
              cudaMalloc(&w->d_in, CHUNK_BYTES + 16) == cudaSuccess &&
              cudaMalloc(&w->d_match, (size_t)CHUNK_BLOCKS * BLOCK * sizeof(uint32_t)) == cudaSuccess &&
              cudaMalloc(&w->d_slots, (size_t)CHUNK_BLOCKS * MAX_MEMBER) == cudaSuccess &&
              cudaMalloc(&w->d_sizes, CHUNK_BLOCKS * sizeof(uint32_t)) == cudaSuccess &&
              cudaMalloc(&w->d_partial, 64 * sizeof(unsigned long long)) == cudaSuccess;
    for (int k = 0; k < 2 && ok; ++k)
        ok = cudaHostAlloc(&w->h_in[k], CHUNK_BYTES, cudaHostAllocDefault) == cudaSuccess &&
             cudaHostAlloc(&w->h_out[k], (size_t)CHUNK_BLOCKS * MAX_MEMBER, cudaHostAllocMapped) == cudaSuccess &&
             cudaHostAlloc(&w->h_off[k], (CHUNK_BLOCKS + 1) * sizeof(uint64_t), cudaHostAllocMapped) == cudaSuccess &&
             cudaEventCreate(&w->done[k]) == cudaSuccess && cudaEventCreate(&w->k0[k]) == cudaSuccess;
    if (!ok) return cuda_fail(w);
    w->ready = true;
    return BRC_OK;
}

// The chunk of set k is done on the device: its members go to the file descriptor.
void retire(brc_bgzf_writer *w, int k) {
    if (!w->pending[k]) return;
    w->pending[k] = false;
    if (cudaEventSynchronize(w->done[k]) != cudaSuccess) { cuda_fail(w); return; }
    float ms = 0;
    if (cudaEventElapsedTime(&ms, w->k0[k], w->done[k]) == cudaSuccess) w->kernel_ms += ms;
    const uint64_t n = w->h_off[k][w->n_blocks[k]];
    w->bytes_out += (int64_t)n;
    if (w->status == BRC_OK) write_fd(w, w->h_out[k], (size_t)n);
}

// Compresses the filled set on the device, then retires the other set (the older chunk) so the host can fill it.
void submit(brc_bgzf_writer *w) {
    if (w->fill == 0 || w->status != BRC_OK) return;
    const int k = w->cur, nb = (int)((w->fill + BLOCK - 1) / BLOCK);
    uint8_t *out_dev = nullptr; uint64_t *off_dev = nullptr;
    bool ok = cudaHostGetDevicePointer((void **)&out_dev, w->h_out[k], 0) == cudaSuccess &&
              cudaHostGetDevicePointer((void **)&off_dev, w->h_off[k], 0) == cudaSuccess &&
              cudaMemcpyAsync(w->d_in, w->h_in[k], (size_t)w->fill, cudaMemcpyHostToDevice, w->stream) == cudaSuccess &&
              cudaEventRecord(w->k0[k], w->stream) == cudaSuccess;
    if (ok) {
        deflate_blocks_kernel<<<nb, CTA, sizeof(Smem), w->stream>>>(w->d_in, w->fill, w->d_match, w->d_slots, w->d_sizes);
        const int64_t ns = (nb + brc::scan::SCAN_CTA - 1) / brc::scan::SCAN_CTA;
        brc::scan::scan_partial_kernel<<<dim3((unsigned)ns, 1), brc::scan::SCAN_CTA, 0, w->stream>>>(w->d_sizes, nb, w->d_partial, ns);
        brc::scan::scan_top_kernel<<<1, 1024, 0, w->stream>>>(w->d_partial, ns);
        brc::scan::scan_apply_kernel<<<dim3((unsigned)ns, 1), brc::scan::SCAN_CTA, 0, w->stream>>>(w->d_sizes, nb, w->d_partial, ns, off_dev, nullptr, nullptr);
        pack_members_kernel<<<nb, 256, 0, w->stream>>>(w->d_slots, w->d_sizes, off_dev, out_dev);
        ok = cudaGetLastError() == cudaSuccess && cudaEventRecord(w->done[k], w->stream) == cudaSuccess;
    }
    if (!ok) { cuda_fail(w); return; }
    w->bytes_in += w->fill;
    w->n_blocks[k] = nb; w->pending[k] = true;
    w->cur ^= 1; w->fill = 0;
    retire(w, w->cur);
}

void release(brc_bgzf_writer *w) {
    if (w->stream) cudaStreamSynchronize(w->stream);
    for (int k = 0; k < 2; ++k) {
        if (w->h_in[k]) cudaFreeHost(w->h_in[k]);
        if (w->h_out[k]) cudaFreeHost(w->h_out[k]);
        if (w->h_off[k]) cudaFreeHost(w->h_off[k]);
        if (w->done[k]) cudaEventDestroy(w->done[k]);
        if (w->k0[k]) cudaEventDestroy(w->k0[k]);
    }
    cudaFree(w->d_in); cudaFree(w->d_match); cudaFree(w->d_slots); cudaFree(w->d_sizes); cudaFree(w->d_partial);
    if (w->stream) cudaStreamDestroy(w->stream);
    cudaGetLastError();
}

}  // namespace

extern "C" {

int brc_set_device(int device) {
    int n_dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || device < 0 || device >= n_dev || cudaSetDevice(device) != cudaSuccess) {
        cudaGetLastError();
        return BRC_E_NO_DEVICE;
    }
    return BRC_OK;
}

int brc_bgzf_open(int fd, brc_bgzf_writer **out) {
    if (!out || fd < 0) return BRC_E_INVALID;
    *out = nullptr;
    int n_dev = 0, dev = 0;
    if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev <= 0 || cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return BRC_E_NO_DEVICE; }
    brc_bgzf_writer *w = new (std::nothrow) brc_bgzf_writer();
    if (!w) return BRC_E_NOMEM;
    w->fd = fd; w->device = dev;
    *out = w;
    return BRC_OK;
}

int brc_bgzf_write(brc_bgzf_writer *w, const void *buf, size_t n) {
    if (!w || (!buf && n)) return BRC_E_INVALID;
    if (w->status != BRC_OK) return result(w);
    if (n == 0) return BRC_OK;
    DeviceScope scope(w->device);
    if (!w->ready && setup(w) != BRC_OK) return result(w);
    const uint8_t *p = static_cast<const uint8_t *>(buf);
    while (n > 0 && w->status == BRC_OK) {
        const size_t k = (size_t)std::min<int64_t>((int64_t)n, CHUNK_BYTES - w->fill);
        std::memcpy(w->h_in[w->cur] + w->fill, p, k);
        w->fill += (int64_t)k; p += k; n -= k;
        if (w->fill == CHUNK_BYTES) submit(w);
    }
    return result(w);
}

int brc_bgzf_close(brc_bgzf_writer *w) {
    if (!w) return BRC_E_INVALID;
    if (w->touched) {                                  // whatever setup allocated, also when it failed part-way
        DeviceScope scope(w->device);
        if (w->ready) {
            submit(w);
            retire(w, w->cur);
            retire(w, w->cur ^ 1);
        }
        release(w);
    }
    if (w->status == BRC_OK) {
        uint8_t eof[28];
        for (int i = 0; i < 28; ++i) eof[i] = eof_byte(i);
        write_fd(w, eof, sizeof eof);
    }
    const int rc = w->status, e = w->saved_errno;
    delete w;
    if (rc == BRC_E_IO) errno = e;
    return rc;
}

int brc_bgzf_stats(const brc_bgzf_writer *w, int64_t *bytes_in, int64_t *bytes_out, double *kernel_ms) {
    if (!w) return BRC_E_INVALID;
    if (bytes_in) *bytes_in = w->bytes_in;
    if (bytes_out) *bytes_out = w->bytes_out;
    if (kernel_ms) *kernel_ms = w->kernel_ms;
    return BRC_OK;
}

}  // extern "C"
