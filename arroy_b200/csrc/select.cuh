// select.cuh — CTA-wide selection primitives of the re-rank kernels: the estimate keys, an exclusive scan, the histogram
// narrowing to the k-th smallest key and a bitonic sort in shared memory. frerank_kernel (frerank.cuh), xf_select_kernel
// (xrerank.cuh) and topk_kernel (kernels.cuh) use them.
#pragma once
#include <stdint.h>

namespace ab {

// monotone float -> uint32 key for finite estimates; NaN / infinite estimates are "unknown" = max
__device__ __forceinline__ uint32_t xf_key(float a) {
    const uint32_t b = __float_as_uint(a);
    return fabsf(a) <= 3.0e38f ? (b ^ ((b & 0x80000000u) ? 0xffffffffu : 0x80000000u)) : 0xffffffffu;
}
__device__ __forceinline__ float xf_unkey(uint32_t k) {   // inverse of xf_key for finite values
    return __uint_as_float(k ^ ((k & 0x80000000u) ? 0x80000000u : 0xffffffffu));
}
__device__ __forceinline__ bool xf_unknown(float a) { return !(fabsf(a) <= 3.0e38f); }
__device__ __forceinline__ uint32_t xf_widen(uint32_t key, float two_e) {   // key of (value + 2E), max if not finite
    if (key == 0xffffffffu) return key;
    return xf_key(__fadd_rn(xf_unkey(key), two_e));
}

// exclusive scan of one value per thread over a CTA of THREADS threads; returns the exclusive prefix, *total = the sum.
// sm: THREADS / 32 words.
template <int THREADS>
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* sm, uint32_t* total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) { const uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
    __syncthreads();
    if (lane == 31) sm[warp] = inc;
    __syncthreads();
    uint32_t base = 0, tot = 0;
#pragma unroll
    for (int i = 0; i < THREADS / 32; ++i) { const uint32_t y = sm[i]; if (i < warp) base += y; tot += y; }
    *total = tot;
    return base + inc - v;
}

// Linear-range histograms over the keys in [rlo, rhi]: up to three levels, each spreading the current range over BINS bins
// (bin = (key - rlo) >> shift, the smallest shift that keeps every key below BINS) and keeping the smallest bin whose cumulative
// count reaches `want`. Stops once that bin holds at most `stop` keys or is one key wide. Returns the bin's upper edge: at least
// `want` of the visited keys are <= it (all of them if there are fewer). visit(f) calls f(key) for every key this thread owns.
// hist: BINS words; sm: what block_exclusive_scan<THREADS> takes; sh: 2 words.
template <int THREADS, int BINS, class Visit>
__device__ __forceinline__ uint32_t hist_narrow(uint32_t rlo, uint32_t rhi, uint32_t want, uint32_t stop, Visit visit,
                                                uint32_t* hist, uint32_t* sm, uint32_t* sh) {
    static_assert(BINS % THREADS == 0 && (BINS & (BINS - 1)) == 0, "bins per thread");
    constexpr int PER = BINS / THREADS;
    int log_bins = 0;
    while ((1 << log_bins) < BINS) ++log_bins;
    for (int level = 0; level < 3 && rhi > rlo; ++level) {
        for (int i = threadIdx.x; i < BINS; i += THREADS) hist[i] = 0;
        __syncthreads();
        const uint32_t span = rhi - rlo;
        const int shift = span < (uint32_t)BINS ? 0 : (32 - __clz(span)) - log_bins;
        visit([&](uint32_t key) { if (key >= rlo && key <= rhi) atomicAdd(&hist[(key - rlo) >> shift], 1u); });
        __syncthreads();
        // smallest bin whose cumulative count reaches `want` (the last bin if fewer keys were visited)
        uint32_t local = 0;
#pragma unroll
        for (int i = 0; i < PER; ++i) local += hist[threadIdx.x * PER + i];
        uint32_t total;
        const uint32_t ex = block_exclusive_scan<THREADS>(local, sm, &total);
        if (threadIdx.x == 0) { sh[0] = BINS - 1; sh[1] = total; }
        __syncthreads();
        if (ex < want && ex + local >= want) {
            uint32_t cum = ex;
            for (int i = 0; i < PER; ++i) { const uint32_t h = hist[threadIdx.x * PER + i]; if (cum + h >= want) { sh[0] = threadIdx.x * PER + i; sh[1] = cum; break; } cum += h; }
        }
        __syncthreads();
        const uint32_t b = sh[0], in_bin = hist[b];
        const uint32_t top = (uint32_t)min((unsigned long long)rhi, (unsigned long long)rlo + (((unsigned long long)b + 1ull) << shift) - 1ull);
        want -= sh[1]; rlo = rlo + (b << shift); rhi = top;
        __syncthreads();
        if (in_bin <= stop || shift == 0) break;
    }
    return rhi;
}

// ascending bitonic sort of n (a power of two) keys in shared memory by the whole CTA
template <class K>
__device__ __forceinline__ void bitonic_sort_shared(K* buf, int n) {
    for (int size = 2; size <= n; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
                const int i = 2 * t - (t & (stride - 1)), j = i + stride;
                const bool up = (i & size) == 0;
                const K a = buf[i], b = buf[j];
                if ((a > b) == up) { buf[i] = b; buf[j] = a; }
            }
        }
    }
    __syncthreads();
}

}  // namespace ab
