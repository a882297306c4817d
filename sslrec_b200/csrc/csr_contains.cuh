// Membership test in a sorted training-CSR row: the rejection test of the negative samplers (sample_negs_kernel,
// neg_candidates_kernel, neg_candidates_pop_kernel; common.cuh includes it).
//
// Kernel source only (no runtime API): tests/emu compiles this file for the host.
#pragma once
#include <stdint.h>

namespace ssl {

// key in the sorted int32 column list cols[lo, hi) (a training-CSR row)?  Binary search.
__device__ __forceinline__ bool csr_contains(const int32_t *__restrict__ cols, int lo, int hi, int key) {
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const int v = __ldg(cols + mid);
        if (v == key) return true;
        if (v < key) lo = mid + 1; else hi = mid;
    }
    return false;
}

}  // namespace ssl
