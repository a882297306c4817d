// Fused evaluation ranking: the top k items of every user of a batch straight from the embedding tables,
//   ssl_predict_mask (predict_tile.cuh) followed by ssl_topk (topk.cu), without the [n_b, n_item] score matrix between them.
//
// Chunk kernel, grid (item chunk, 128-user tile): the CTA walks its chunk's 128-item tiles with predict_tile_kernel's register
// tiling (tile_product: same staging, same sequential fp32 FMA chain per score), applies the mask with ssl_predict_mask's formulas,
// and turns every score into the total order key of ssl_topk,
//     key = okey(score) << 32 | (0xffffffff - item)      (value descending, then item ascending; every key of a row is distinct),
// Warp w owns the 16 rows 2w + h + 16 i (h = 0, 1; i = 0 .. 7) entirely: lanes 0-15 hold row 2w + 16 i, lanes 16-31 row 2w + 1 + 16 i,
// 8 columns each.  Each row keeps a threshold (initially 0, below every key) and a candidate list of `cap` keys in the caller's
// workspace.  Keys above the threshold are appended (ballot + popc compaction); when a tile's survivors would overflow the list,
// the warp selects the list's k largest keys in place (select_top: 8-bit radix select on the 64-bit key, warp-private histogram)
// and raises the threshold to the k-th of them.  At the end of the chunk every row keeps at most k keys and writes their count.
// The CSR mask keeps a cursor per row into the sorted training row, so each tile reads only the entries that fall inside it.
//
// Merge kernel, one CTA per user: radix select of the k largest keys over the row's chunk lists, bitonic sort, write ids and values.
// Because the keys are distinct, the k largest are one set whatever order candidates arrive in: the result is exact, independent of
// scheduling and of the chunking, and equal to ssl_topk on ssl_predict_mask's scores (ties, masked -1e8 entries, +-0 and NaN).
//
// Kernel-only header, as predict_tile.cuh, so that tests/emu runs the same source on the host.
#pragma once
#include <stdint.h>

#include "predict_tile.cuh"

namespace ssl_predict {

constexpr int kTopkMaxK = 256;
constexpr int kTopkMaxChunks = 1024;
constexpr int kMergeThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

// ssl_topk's order-preserving map of a float onto uint32 (topk.cu) and its inverse
__device__ __forceinline__ uint32_t okey(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float okey_inv(uint32_t k) {
    const uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(u);
}
__device__ __forceinline__ uint64_t rank_key(float v, uint32_t item) {
    return ((uint64_t)okey(v) << 32) | (uint64_t)(0xffffffffu - item);
}

// predict_tile_kernel's product, restated (that kernel is left as it is, the reference this one is tested against):
// acc[i][j] = U[u_s[ty + 16 i]] . I[n0 + tx + 16 j], each one sequential fp32 FMA chain over k = 0 .. dim-1 (padding rows,
// columns and inner values read as zeros).  All NT threads call it; it ends on a barrier, so a_s / b_s are free afterwards.
__device__ __forceinline__ void tile_product(float (&acc)[8][8], float (&a_s)[TK][TM + PAD], float (&b_s)[TK][TN + PAD],
                                             const int64_t *u_s, const float *__restrict__ ut, int64_t us,
                                             const float *__restrict__ itab, int64_t is, int64_t n0, int64_t n_item, int dim,
                                             int tid) {
    const int tx = tid & 15, ty = tid >> 4;
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    for (int k0 = 0; k0 < dim; k0 += TK) {
#pragma unroll 4
        for (int q = 0; q < TM * TK / NT; ++q) {
            const int idx = tid + NT * q;
            const int r = idx / TK, k = idx % TK;
            const int64_t u = u_s[r];
            a_s[k][r] = (u >= 0 && k0 + k < dim) ? ut[u * us + k0 + k] : 0.f;
        }
#pragma unroll 4
        for (int q = 0; q < TN * TK / NT; ++q) {
            const int idx = tid + NT * q;
            const int r = idx / TK, k = idx % TK;
            const int64_t it = n0 + r;
            b_s[k][r] = (it < n_item && k0 + k < dim) ? itab[it * is + k0 + k] : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int k = 0; k < TK; ++k) {
            float a[8], b[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = a_s[k][ty + 16 * i];
#pragma unroll
            for (int j = 0; j < 8; ++j) b[j] = b_s[k][tx + 16 * j];
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        __syncthreads();
    }
}

// One warp, warp-uniform arguments, n > k distinct keys in list[0, n): moves the k largest to list[0, k) (order kept) and returns the
// k-th largest.  hist: 256 words of shared memory private to the warp.
__device__ __forceinline__ uint64_t select_top(uint64_t *list, int n, int k, uint32_t *hist, int lane) {
    uint64_t prefix = 0;
    uint32_t need = (uint32_t)k;
    for (int shift = 56; shift >= 0; shift -= 8) {
        const uint64_t hi = (shift == 56) ? 0ull : (~0ull << (shift + 8));
        for (int q = lane; q < 256; q += 32) hist[q] = 0;
        __syncwarp();
        for (int e = lane; e < n; e += 32) {
            const uint64_t key = list[e];
            if ((key & hi) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1u);
        }
        __syncwarp();
        // lane l sums digits 255 - 8 l down to 248 - 8 l; an inclusive scan over the lanes counts the keys at or above each lane's digits
        uint32_t own = 0;
#pragma unroll
        for (int q = 0; q < 8; ++q) own += hist[255 - 8 * lane - q];
        uint32_t incl = own;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t v = __shfl_up_sync(kFull, incl, o);
            if (lane >= o) incl += v;
        }
        const int src = __ffs(__ballot_sync(kFull, incl >= need)) - 1;      // the keys matching prefix number >= need
        int digit = 0;
        uint32_t above = 0;
        if (lane == src) {
            above = incl - own;
            int q = 0;
            for (; q < 7; ++q) {
                const uint32_t h = hist[255 - 8 * lane - q];
                if (above + h >= need) break;
                above += h;
            }
            digit = 255 - 8 * lane - q;
        }
        digit = __shfl_sync(kFull, digit, src);
        above = __shfl_sync(kFull, above, src);
        prefix |= (uint64_t)digit << shift;
        need -= above;
        __syncwarp();
    }
    // prefix is the k-th largest key: keep the keys >= prefix, in place (a write never passes an unread entry)
    int out = 0;
    for (int base = 0; base < n; base += 32) {
        const int e = base + lane;
        const uint64_t key = e < n ? list[e] : 0ull;
        const bool keep = e < n && key >= prefix;
        const unsigned bal = __ballot_sync(kFull, keep);
        if (keep) list[out + __popc(bal & ((1u << lane) - 1u))] = key;
        out += __popc(bal);
    }
    __syncwarp();
    return prefix;
}

// ws_keys: [n_b][n_chunks][cap] keys, ws_cnt: [n_b][n_chunks] counts (cap >= k + TN; neither needs to be initialised).
// trn_cols: every training row sorted ascending.
static __global__ void __launch_bounds__(NT, 2)
predict_topk_chunk_kernel(const float *__restrict__ ut, int64_t us, const float *__restrict__ itab, int64_t is,
                          const int64_t *__restrict__ users, int64_t n_b, int64_t n_item, int dim,
                          const int64_t *__restrict__ mask_dense, const int32_t *__restrict__ trn_rowptr,
                          const int32_t *__restrict__ trn_cols, int k, int n_chunks, int cap, uint64_t *__restrict__ ws_keys,
                          int32_t *__restrict__ ws_cnt) {
    __shared__ float a_s[TK][TM + PAD];
    __shared__ float b_s[TK][TN + PAD];
    __shared__ int64_t u_s[TM];
    __shared__ uint64_t thr_s[TM];
    __shared__ int cnt_s[TM];
    __shared__ int cur_s[TM], end_s[TM], nxt_s[TM];
    __shared__ uint32_t bits_s[TM][TN / 32];
    __shared__ uint32_t hist_s[NT / 32][256];
    const int tid = (int)threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5;
    const int tx = tid & 15, ty = tid >> 4;
    const int64_t m0 = (int64_t)blockIdx.y * TM;
    const int64_t chunk = blockIdx.x;
    const int64_t n_tiles = (n_item + TN - 1) / TN;
    const int64_t t0 = n_tiles * chunk / n_chunks, t1 = n_tiles * (chunk + 1) / n_chunks;
    const bool csr = mask_dense == nullptr && trn_rowptr != nullptr;
    if (tid < TM) {
        const int64_t u = (m0 + tid < n_b) ? users[m0 + tid] : (int64_t)-1;
        u_s[tid] = u;
        thr_s[tid] = 0;
        cnt_s[tid] = 0;
        cur_s[tid] = end_s[tid] = nxt_s[tid] = 0;
        if (csr && u >= 0) {       // the first training item at or after the chunk's first item
            int lo = trn_rowptr[u], hi = trn_rowptr[u + 1];
            end_s[tid] = hi;
            while (lo < hi) {
                const int mid = lo + (hi - lo) / 2;
                if ((int64_t)trn_cols[mid] < t0 * TN) lo = mid + 1;
                else hi = mid;
            }
            cur_s[tid] = lo;
            if (lo < end_s[tid]) nxt_s[tid] = trn_cols[lo];
        }
    }
    __syncthreads();

    const unsigned half = (lane < 16) ? 0x0000ffffu : 0xffff0000u;
    const unsigned below = (1u << lane) - 1u;
    for (int64_t t = t0; t < t1; ++t) {
        const int64_t n0 = t * TN, n1 = n0 + TN;
        float acc[8][8];
        tile_product(acc, a_s, b_s, u_s, ut, us, itab, is, n0, n_item, dim, tid);

        if (csr && lane < 16) {
            // this tile's training items of row r as bits, one lane per row; the cursor stops at the first item >= n1, and the item it
            // points at is kept in nxt_s, so a tile without training items of the row reads no global memory
            const int r = 2 * warp + (lane & 1) + 16 * (lane >> 1);
#pragma unroll
            for (int q = 0; q < TN / 32; ++q) bits_s[r][q] = 0u;
            int e = cur_s[r];
            const int e1 = end_s[r];
            int64_t col = nxt_s[r];
            while (e < e1 && col < n1) {
                if (col >= n0) bits_s[r][(col - n0) >> 5] |= 1u << ((col - n0) & 31);
                ++e;
                col = e < e1 ? (int64_t)trn_cols[e] : 0;
            }
            cur_s[r] = e;
            nxt_s[r] = (int32_t)col;
        }
        __syncwarp();

        const uint32_t c0 = (uint32_t)n0 + tx, n_valid = (uint32_t)(n_item - n0);     // item of column j: c0 + 16 j; valid: tx + 16 j < n_valid
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = ty + 16 * i;
            const int64_t b = m0 + r;
            const bool row_ok = b < n_b;
            uint64_t thr = thr_s[r];
            int cnt = cnt_s[r];
            unsigned pass = 0;
            // the masked score, exactly as predict_tile_kernel writes it (and as its CSR pass rewrites it)
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (!row_ok || (uint32_t)(tx + 16 * j) >= n_valid) continue;
                float m = 0.f;
                if (mask_dense) m = (float)mask_dense[b * n_item + c0 + 16 * j];
                float v = acc[i][j] * (1.f - m) - 1e8f * m;
                if (csr && ((bits_s[r][j >> 1] >> (tx + 16 * (j & 1))) & 1u)) v = v * 0.f - 1e8f;
                acc[i][j] = v;
                if (rank_key(v, c0 + 16 * j) > thr) pass |= 1u << j;
            }
            int np = __popc(pass);       // survivors of the half-warp's row
#pragma unroll
            for (int o = 8; o > 0; o >>= 1) np += __shfl_xor_sync(kFull, np, o);
            const unsigned over = __ballot_sync(kFull, cnt + np > cap);
            if (over) {
                for (int h = 0; h < 2; ++h) {
                    if (!(over & (1u << (16 * h)))) continue;
                    const int rr = 2 * warp + h + 16 * i;
                    uint64_t *list = ws_keys + ((m0 + rr) * n_chunks + chunk) * cap;
                    const uint64_t kth = select_top(list, cnt_s[rr], k, hist_s[warp], lane);
                    if (lane == 0) {
                        thr_s[rr] = kth;
                        cnt_s[rr] = k;
                    }
                    __syncwarp();
                }
                thr = thr_s[r];
                cnt = cnt_s[r];
#pragma unroll
                for (int j = 0; j < 8; ++j)
                    if (((pass >> j) & 1u) && rank_key(acc[i][j], c0 + 16 * j) <= thr) pass &= ~(1u << j);
            }
            uint64_t *list = ws_keys + (b * n_chunks + chunk) * cap;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const bool p = (pass >> j) & 1u;
                const unsigned bal = __ballot_sync(kFull, p) & half;
                if (p) list[cnt + __popc(bal & below)] = rank_key(acc[i][j], c0 + 16 * j);
                cnt += __popc(bal);
            }
            if (tx == 0 && row_ok) cnt_s[r] = cnt;
            __syncwarp();
        }
    }

    for (int q = 0; q < 16; ++q) {
        const int r = 2 * warp + (q & 1) + 16 * (q >> 1);
        const int64_t b = m0 + r;
        if (b >= n_b) continue;
        int cnt = cnt_s[r];
        if (cnt > k) {
            select_top(ws_keys + (b * n_chunks + chunk) * cap, cnt, k, hist_s[warp], lane);
            cnt = k;
        }
        if (lane == 0) ws_cnt[b * n_chunks + chunk] = cnt;
    }
}

// One CTA per user: the k largest of the row's chunk lists, sorted (value descending, item ascending).
static __global__ void __launch_bounds__(kMergeThreads)
predict_topk_merge_kernel(const uint64_t *__restrict__ ws_keys, const int32_t *__restrict__ ws_cnt, int n_chunks, int cap, int k,
                          int64_t *__restrict__ out_idx, float *__restrict__ out_val) {
    __shared__ int cnt_s[kTopkMaxChunks];
    __shared__ uint32_t hist[256];
    __shared__ uint64_t cand[kTopkMaxK];
    __shared__ uint64_t s_prefix;
    __shared__ uint32_t s_need, s_n;
    const int tid = (int)threadIdx.x;
    const int64_t b = blockIdx.x;
    const uint64_t *keys = ws_keys + b * n_chunks * cap;
    for (int c = tid; c < n_chunks; c += kMergeThreads) cnt_s[c] = ws_cnt[b * n_chunks + c];
    for (int i = tid; i < kTopkMaxK; i += kMergeThreads) cand[i] = 0ull;
    if (tid == 0) {
        s_prefix = 0;
        s_need = (uint32_t)k;
        s_n = 0;
    }
    __syncthreads();
    const int slots = n_chunks * k;      // slot s: entry s % k of chunk s / k
    for (int shift = 56; shift >= 0; shift -= 8) {
        for (int i = tid; i < 256; i += kMergeThreads) hist[i] = 0;
        __syncthreads();
        const uint64_t prefix = s_prefix;
        const uint64_t hi = (shift == 56) ? 0ull : (~0ull << (shift + 8));
        for (int s = tid; s < slots; s += kMergeThreads) {
            const int c = s / k, e = s - c * k;
            if (e >= cnt_s[c]) continue;
            const uint64_t key = keys[(int64_t)c * cap + e];
            if ((key & hi) == prefix) atomicAdd(&hist[(key >> shift) & 255], 1u);
        }
        __syncthreads();
        if (tid == 0) {
            uint32_t need = s_need, above = 0;
            int d = 255;
            for (; d > 0; --d) {
                if (above + hist[d] >= need) break;
                above += hist[d];
            }
            s_need = need - above;
            s_prefix = prefix | ((uint64_t)d << shift);
        }
        __syncthreads();
    }
    const uint64_t kth = s_prefix;         // the keys are distinct: exactly k of them are >= kth
    for (int s = tid; s < slots; s += kMergeThreads) {
        const int c = s / k, e = s - c * k;
        if (e >= cnt_s[c]) continue;
        const uint64_t key = keys[(int64_t)c * cap + e];
        if (key >= kth) cand[atomicAdd(&s_n, 1u)] = key;
    }
    __syncthreads();
    int P = 1;      // bitonic sort, descending, on the next power of two >= k (unused slots are 0 = smallest)
    while (P < k) P <<= 1;
    for (int size = 2; size <= P; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int i = tid; i < P; i += kMergeThreads) {
                const int j = i ^ stride;
                if (j > i) {
                    const bool desc = (i & size) == 0;
                    const uint64_t x = cand[i], y = cand[j];
                    if ((x < y) == desc) {
                        cand[i] = y;
                        cand[j] = x;
                    }
                }
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < k; i += kMergeThreads) {
        const uint64_t c = cand[i];
        out_idx[b * k + i] = (int64_t)(0xffffffffu - (uint32_t)(c & 0xffffffffull));
        if (out_val) out_val[b * k + i] = okey_inv((uint32_t)(c >> 32));
    }
}

}  // namespace ssl_predict
