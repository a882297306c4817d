// ssl_unique_ids: the sorted distinct ids of an index vector, on the device and without a host sync -- the graph-safe form
// of HCCF's t.unique(ancs) / t.unique(poss) (hccf.py:80-81 of the reference).
//
// The ids live in [0, n_range).  One bit per possible id:
//   1. clear the bitmap                               (this launch sequence owns its scratch: a replay starts clean)
//   2. mark:      atomicOr of bit id into word id / 32
//   3. popcount:  per block of kWordsPerBlock words, the number of set bits
//   4. scan:      one CTA turns the block counts into exclusive offsets, writes the count and finds the largest id
//   5. compact:   every block writes the ids of its set bits, in ascending order, from its offset on;
//                 all blocks together fill out[count, n) with the largest id
// O(n + n_range / 32) work; the result is a pure function of the set of ids (no atomics decide an order).
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kThreads = 256, kWordsPerThread = 4, kWordsPerBlock = kThreads * kWordsPerThread;

struct Scratch {
    uint32_t *bits;        // [n_words]
    uint32_t *block_off;   // [n_blocks]: popcount per block, then its exclusive prefix
    int64_t *last;         // the largest id (or -1 when there is none)
};

int64_t n_words_of(int64_t n_range) { return (n_range + 31) / 32; }
int64_t n_blocks_of(int64_t n_range) { return (n_words_of(n_range) + kWordsPerBlock - 1) / kWordsPerBlock; }
// uint32 words of scratch: bitmap padded to whole blocks, block offsets, an aligned int64
int64_t scratch_words(int64_t n_range) {
    const int64_t nb = n_blocks_of(n_range);
    return nb * kWordsPerBlock + (nb + 1) / 2 * 2 + 2;
}
Scratch carve(uint32_t *scratch, int64_t n_range) {
    const int64_t nb = n_blocks_of(n_range);
    Scratch s;
    s.bits = scratch;
    s.block_off = scratch + nb * kWordsPerBlock;
    s.last = reinterpret_cast<int64_t *>(s.block_off + (nb + 1) / 2 * 2);
    return s;
}

__global__ void clear_kernel(uint32_t *__restrict__ bits, int64_t n_words) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_words; i += (int64_t)gridDim.x * blockDim.x) bits[i] = 0u;
}

__global__ void mark_kernel(const int64_t *__restrict__ idx, int64_t n, int64_t n_range, uint32_t *__restrict__ bits) {
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
        const int64_t id = idx[i];
        if (id >= 0 && id < n_range) atomicOr(bits + (id >> 5), 1u << (id & 31));   // out-of-range ids are not counted
    }
}

__device__ __forceinline__ uint4 load_words(const uint32_t *bits, int64_t block) {
    return reinterpret_cast<const uint4 *>(bits + block * kWordsPerBlock)[threadIdx.x];
}

// exclusive prefix of v over the CTA (kThreads threads); *total gets the CTA's sum
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t *total) {
    __shared__ uint32_t warp_sums[kThreads / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t x = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    uint32_t before = 0, all = 0;
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) {
        const uint32_t ws = warp_sums[w];
        before += (w < warp) ? ws : 0u;
        all += ws;
    }
    *total = all;
    return before + x - v;
}

__global__ void __launch_bounds__(kThreads) popcount_kernel(const uint32_t *__restrict__ bits, uint32_t *__restrict__ block_off) {
    const uint4 w = load_words(bits, blockIdx.x);
    uint32_t total;
    block_exclusive_scan(__popc(w.x) + __popc(w.y) + __popc(w.z) + __popc(w.w), &total);
    if (threadIdx.x == 0) block_off[blockIdx.x] = total;
}

// one CTA: block counts -> exclusive offsets (in place), *count, and the largest marked id
__global__ void __launch_bounds__(kThreads) scan_kernel(const uint32_t *__restrict__ bits, uint32_t *__restrict__ block_off, int64_t n_blocks,
                                                        int64_t *__restrict__ count, int64_t *__restrict__ last) {
    __shared__ unsigned long long s_last_block, s_last_word;      // 1 + the index, 0 = none
    if (threadIdx.x == 0) s_last_block = s_last_word = 0ull;
    __syncthreads();
    int64_t carry = 0, my_last = -1;
    for (int64_t base = 0; base < n_blocks; base += kThreads) {
        const int64_t b = base + threadIdx.x;
        const uint32_t c = (b < n_blocks) ? block_off[b] : 0u;
        if (c != 0u) my_last = b;
        uint32_t total;
        const uint32_t ex = block_exclusive_scan(c, &total);
        if (b < n_blocks) block_off[b] = (uint32_t)(carry + ex);
        carry += total;
        __syncthreads();                                  // warp_sums is reused by the next round
    }
    if (my_last >= 0) atomicMax(&s_last_block, (unsigned long long)(my_last + 1));
    __syncthreads();
    const int64_t lb = (int64_t)s_last_block - 1;
    if (lb >= 0) {
        const uint4 w = load_words(bits, lb);
        const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
        int64_t mine = -1;
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (ws[k] != 0u) mine = lb * kWordsPerBlock + threadIdx.x * kWordsPerThread + k;
        if (mine >= 0) atomicMax(&s_last_word, (unsigned long long)(mine + 1));
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        *count = carry;
        const int64_t lw = (int64_t)s_last_word - 1;
        *last = (lw < 0) ? -1 : lw * 32 + (31 - __clz(bits[lw]));
    }
}

__global__ void __launch_bounds__(kThreads) compact_kernel(const uint32_t *__restrict__ bits, const uint32_t *__restrict__ block_off,
                                                           const int64_t *__restrict__ count, const int64_t *__restrict__ last, int64_t n,
                                                           int64_t *__restrict__ out) {
    const uint4 w = load_words(bits, blockIdx.x);
    const uint32_t ws[4] = {w.x, w.y, w.z, w.w};
    uint32_t total;
    int64_t pos = block_off[blockIdx.x] + block_exclusive_scan(__popc(w.x) + __popc(w.y) + __popc(w.z) + __popc(w.w), &total);
    const int64_t id0 = ((int64_t)blockIdx.x * kWordsPerBlock + threadIdx.x * kWordsPerThread) * 32;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        uint32_t m = ws[k];
        while (m != 0u) {
            const int bit = __ffs(m) - 1;
            out[pos++] = id0 + 32 * k + bit;
            m &= m - 1;
        }
    }
    // padding: a gather through out[0, n) stays in bounds
    const int64_t c = *count, l = *last;
    for (int64_t i = c + (int64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (int64_t)gridDim.x * kThreads) out[i] = l;
}

}  // namespace

#define STREAM ((cudaStream_t)stream)

extern "C" int ssl_unique_ids_scratch(int64_t n_range, int64_t *words) {
    SSL_CHECK_ARG(words != nullptr, "ssl_unique_ids_scratch: null argument");
    SSL_CHECK_ARG(n_range >= 1, "ssl_unique_ids_scratch: n_range %lld < 1", (long long)n_range);
    *words = scratch_words(n_range);
    return SSL_OK;
}

extern "C" int ssl_unique_ids(const int64_t *idx, int64_t n, int64_t n_range, uint32_t *scratch, int64_t scratch_n_words,
                              int64_t *out, int64_t *count, void *stream) {
    SSL_CHECK_ARG(idx && scratch && out && count, "ssl_unique_ids: null argument");
    SSL_CHECK_ARG(n >= 0, "ssl_unique_ids: n %lld < 0", (long long)n);
    SSL_CHECK_ARG(n_range >= 1, "ssl_unique_ids: n_range %lld < 1", (long long)n_range);
    SSL_CHECK_ARG(scratch_n_words >= scratch_words(n_range), "ssl_unique_ids: scratch has %lld words, %lld needed",
                  (long long)scratch_n_words, (long long)scratch_words(n_range));
    SSL_CHECK_ARG((reinterpret_cast<uintptr_t>(scratch) & 15) == 0, "ssl_unique_ids: scratch must be 16-byte aligned");
    const Scratch s = carve(scratch, n_range);
    const int64_t nb = n_blocks_of(n_range), n_bits_words = nb * kWordsPerBlock;
    const unsigned grid_clear = (unsigned)std::min<int64_t>((n_bits_words + kThreads - 1) / kThreads, 4 * ssl::kNumSM);
    clear_kernel<<<grid_clear, kThreads, 0, STREAM>>>(s.bits, n_bits_words);
    SSL_LAUNCH_CHECK("clear_kernel");
    if (n > 0) {
        const unsigned grid_mark = (unsigned)std::min<int64_t>((n + kThreads - 1) / kThreads, 8 * ssl::kNumSM);
        mark_kernel<<<grid_mark, kThreads, 0, STREAM>>>(idx, n, n_range, s.bits);
        SSL_LAUNCH_CHECK("mark_kernel");
    }
    popcount_kernel<<<(unsigned)nb, kThreads, 0, STREAM>>>(s.bits, s.block_off);
    SSL_LAUNCH_CHECK("popcount_kernel");
    scan_kernel<<<1, kThreads, 0, STREAM>>>(s.bits, s.block_off, nb, count, s.last);
    SSL_LAUNCH_CHECK("scan_kernel");
    compact_kernel<<<(unsigned)nb, kThreads, 0, STREAM>>>(s.bits, s.block_off, count, s.last, n, out);
    SSL_LAUNCH_CHECK("compact_kernel");
    return SSL_OK;
}

extern "C" int ssl_row_bitmap(const int64_t *idx, int64_t n, int64_t n_range, uint32_t *bits, int64_t n_words, void *stream) {
    SSL_CHECK_ARG(bits && (idx || n == 0), "ssl_row_bitmap: null argument");
    SSL_CHECK_ARG(n >= 0 && n_range >= 1, "ssl_row_bitmap: bad sizes");
    SSL_CHECK_ARG(n_words >= (n_range + 31) / 32, "ssl_row_bitmap: %lld words, %lld needed", (long long)n_words, (long long)((n_range + 31) / 32));
    const unsigned grid_clear = (unsigned)std::max<int64_t>(1, std::min<int64_t>((n_words + kThreads - 1) / kThreads, 4 * ssl::kNumSM));
    clear_kernel<<<grid_clear, kThreads, 0, STREAM>>>(bits, n_words);
    SSL_LAUNCH_CHECK("clear_kernel");
    if (n > 0) {
        const unsigned grid_mark = (unsigned)std::min<int64_t>((n + kThreads - 1) / kThreads, 8 * ssl::kNumSM);
        mark_kernel<<<grid_mark, kThreads, 0, STREAM>>>(idx, n, n_range, bits);
        SSL_LAUNCH_CHECK("mark_kernel");
    }
    return SSL_OK;
}
