// Ordered scatter of staged batch rows into a gradient sink (ssl_scatter_rows_ordered; train.deterministic).
//
// Input: P staged rows stage[P, dim] (row p is the contribution c_p of batch position p), their destination ids[P] and
// order[P], the STABLE ascending argsort of ids.  For every sink row r that some position addresses:
//
//     sink[r] = sink[r] + (((c_p1 + c_p2) + c_p3) + ...)        p1 < p2 < ... the positions with ids[p] == r
//
// with plain fp32 adds, sequentially in position order: the result is a pure function of the inputs, whatever the
// scheduling.  Positions with a negative id are skipped (the count-bounded callers give dead positions id -1), so a row
// addressed by dead positions only is left bit-unchanged.
//
// Work split: one unit per (sorted position q, 32-column group).  The unit at the first position of an id's run in
// ``order`` (its segment) owns that segment: its lane l walks the segment's positions in order for column 32 g + l, reads
// the sink element once and writes it once (no atomics: the segments of one launch address distinct rows).  Every other
// unit returns after two id loads.  A popular id's long segment therefore occupies one warp per column group while the
// other warps move on; it cannot be split further without changing the summation order above.  The kernel is
// grid-agnostic (grid-stride over the units), so the host emulation runs it on a small grid.
//
// Kernel source only (no runtime API): tests/emu compiles this file for the host.
#pragma once
#include <stdint.h>

namespace ssl_scatter {

constexpr int kWarpsPerBlock = 8;

static __global__ void __launch_bounds__(kWarpsPerBlock * 32)
    ordered_scatter_kernel(const float *__restrict__ stage, const int64_t *__restrict__ ids, const int64_t *__restrict__ order,
                           int64_t n_pos, int dim, float *__restrict__ sink, int64_t stride) {
    const int lane = (int)threadIdx.x & 31;
    const int n_groups = (dim + 31) / 32;
    const int64_t n_units = n_pos * n_groups;
    const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
    for (int64_t u = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); u < n_units; u += n_warps) {
        const int64_t q = u / n_groups;
        const int col = (int)(u % n_groups) * 32 + lane;
        const int64_t r = ids[order[q]];
        if (r < 0 || (q > 0 && ids[order[q - 1]] == r)) continue;      // a dead position, or not the first of its segment
        float acc = 0.f;
        bool first = true;
        for (int64_t q0 = q;; q0 += 32) {
            // the segment's positions in [q0, q0 + 32) are a prefix of that window: ids ascend along order
            const int64_t qq = q0 + lane;
            const unsigned in_seg = __ballot_sync(0xffffffffu, qq < n_pos && ids[order[qq]] == r);
            const int n = __popc(in_seg);
            if (col < dim) {
#pragma unroll 4
                for (int j = 0; j < n; ++j) {
                    const float c = stage[order[q0 + j] * dim + col];
                    acc = first ? c : acc + c;           // no multiply anywhere: nothing can contract into an FMA
                    first = false;
                }
            }
            if (n < 32) break;
        }
        if (col < dim) {
            float *dst = sink + r * stride + col;
            *dst = *dst + acc;
        }
    }
}

}  // namespace ssl_scatter
