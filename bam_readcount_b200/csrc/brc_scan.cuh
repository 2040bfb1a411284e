// brc_scan.cuh — hand-written exclusive scan of u32 counts into u64 offsets, shared by the BGZF framing (brc_bgzf.cu: CIGAR,
// base and quality pool offsets) and the site selection (brc_select.cu: compact indices of the shipped sites).
//
// Three kernels, SCAN_CTA elements per CTA; blockIdx.y picks one of up to three arrays laid out back to back (array k starts
// at sz + k * n):
//   scan_partial_kernel  per-CTA sums                         partial[k * (nb + 1) + b]
//   scan_top_kernel      one CTA per array: exclusive scan of the partials in place; partial[k * (nb + 1) + nb] = total
//   scan_apply_kernel    out_k[i] = exclusive prefix of element i; out_k[n] = total
// Internal linkage (static): every translation unit that includes this header gets its own copy of the kernels.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace brc {
namespace scan {

constexpr int SCAN_CTA = 256;

static __global__ void __launch_bounds__(SCAN_CTA) scan_partial_kernel(const uint32_t *sz, int64_t n, unsigned long long *partial, int64_t nb) {
    __shared__ unsigned long long red[SCAN_CTA / 32];
    const int arr = blockIdx.y;
    const int64_t i = (int64_t)blockIdx.x * SCAN_CTA + threadIdx.x;
    unsigned long long v = i < n ? sz[(int64_t)arr * n + i] : 0ull;
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) { unsigned long long t = 0; for (int w = 0; w < SCAN_CTA / 32; ++w) t += red[w]; partial[(int64_t)arr * (nb + 1) + blockIdx.x] = t; }
}
static __global__ void __launch_bounds__(1024) scan_top_kernel(unsigned long long *partial, int64_t nb) {      // exclusive, in place; [nb] = total
    __shared__ unsigned long long part[1024];
    unsigned long long *v = partial + (int64_t)blockIdx.x * (nb + 1);
    const int t = threadIdx.x;
    const int64_t per = (nb + 1023) / 1024, lo = min(nb, per * t), hi = min(nb, lo + per);
    unsigned long long s = 0;
    for (int64_t i = lo; i < hi; ++i) s += v[i];
    part[t] = s;
    __syncthreads();
    if (t == 0) { unsigned long long acc = 0; for (int i = 0; i < 1024; ++i) { const unsigned long long x = part[i]; part[i] = acc; acc += x; } v[nb] = acc; }
    __syncthreads();
    unsigned long long acc = part[t];
    for (int64_t i = lo; i < hi; ++i) { const unsigned long long x = v[i]; v[i] = acc; acc += x; }
}
static __global__ void __launch_bounds__(SCAN_CTA) scan_apply_kernel(const uint32_t *sz, int64_t n, const unsigned long long *partial, int64_t nb, uint64_t *off0, uint64_t *off1, uint64_t *off2) {
    __shared__ unsigned long long sh[SCAN_CTA];
    const int arr = blockIdx.y;
    uint64_t *out = arr == 0 ? off0 : (arr == 1 ? off1 : off2);
    const int64_t i = (int64_t)blockIdx.x * SCAN_CTA + threadIdx.x;
    const unsigned long long v = i < n ? sz[(int64_t)arr * n + i] : 0ull;
    sh[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < SCAN_CTA; o <<= 1) { const unsigned long long a = threadIdx.x >= o ? sh[threadIdx.x - o] : 0ull; __syncthreads(); sh[threadIdx.x] += a; __syncthreads(); }
    const unsigned long long base = partial[(int64_t)arr * (nb + 1) + blockIdx.x];
    if (i < n) out[i] = base + sh[threadIdx.x] - v;
    if (i == n - 1) out[n] = base + sh[threadIdx.x];
}

}  // namespace scan
}  // namespace brc
