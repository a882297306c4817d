// Multi-view CSR SpMM propagation layer with in-kernel augmentation (include/sslrec_b200.h,
// ssl_propagate_layer).  HBM/L2-bound gather: no tensor cores (there is no dense contraction).
//
// Mapping.  A "group" of G = pow2(dim/4) lanes owns one work item (a CSR row, or a <= seg_len
// slice of a long row); each lane owns one float4 column slot of every view, so a neighbour row
// of view v is fetched by one coalesced 16 B x G request (256 B for dim = 64).  32/G items per
// warp.  The group's lanes first load G (col, val) pairs coalesced, evaluate the edge keep test
// once per edge (not once per lane), then broadcast them with shuffles while the row gathers are
// issued four edges deep.  Items are sorted by length (split segments first, then rows by
// descending degree) so the groups of a warp run equal trip counts and the heavy items start
// first.  Long rows are split into segments whose partial sums go to a plan-owned scratch; the
// last segment to finish (atomic ticket) adds the partials in segment order -- the summation
// order of every output element is fixed, so results are bit-reproducible run to run.
//
// Row-sharded multi-GPU (SURVEY.md 8e): a plan may own two global row ranges (its share of the user
// rows and of the item rows); every per-row pointer is a FULL [N, ...] table addressed by the global
// row.  The epilogue stores a finished row to this GPU's table and to the same row of every peer's
// table (pointers into the peers' HBM mapped over NVLink: x_out_peers / sum_out_peers), so the
// all-gather of the layer output is fused into the SpMM and its NVLink traffic overlaps the gathers.
//
// View-major variant (VM): with per-view inputs the grid's y dimension is the view and a thread
// keeps one accumulator.  CTAs are scheduled x-fastest, so all rows of view 0 run before view 1:
// the gathered working set is one view's rows (41 MB at the amazon shape) instead of the interleaved
// [N, V, d] table (123 MB, more than twice the 50 MB L2).
#include <algorithm>
#include <cmath>
#include <string>
#include <vector>

#include "common.cuh"

struct ssl_plan {
    int64_t n_rows, n_cols, nnz, row_offset;
    int64_t split_local, off_a, off_b;   // global row = local + (local < split_local ? off_a : off_b)
    const int32_t *colidx;
    const float *vals;
    const int32_t *rev;
    int4 *items;        // {local row, edge begin, edge end, long-row id or -1}
    int2 *long_info;    // per long row: {first slot, n segments}
    int32_t *counters;  // per long row: arrival ticket
    float *partial;     // [n_slots, SSL_MAX_VIEWS * SSL_MAX_DIM]
    int64_t n_items, n_long, n_slots, max_deg;
};

namespace {

constexpr int kMinSeg = 128;       // rows up to this many entries are never split
constexpr int kThreads = 256;
constexpr int kPartialStride = SSL_MAX_VIEWS * SSL_MAX_DIM;
// ssl_set_option("prop_view_major", 1): one view per thread, grid.y = view -- DRAM traffic at 1.03x compulsory instead of 1.3x,
// at the cost of less work per thread (the kernel is issue / latency bound, not DRAM bound).  Default off.
bool g_view_major = false;

struct PlanDev {
    const int32_t *colidx;
    const float *vals;
    const int32_t *rev;
    const int4 *items;
    const int2 *long_info;
    int32_t *counters;
    float *partial;
    int64_t n_items, n_long;
    int32_t split_local;
    uint32_t off_a, off_b;
};

// the view's RNG seed: a launch argument, or -- CUDA-graph replay -- a word the host rewrites on the device
__device__ __forceinline__ uint64_t view_seed(const ssl_prop_args &a, int v) { return a.seed_ptr[v] != nullptr ? __ldg(a.seed_ptr[v]) : a.seed[v]; }

__device__ __forceinline__ float sgnf(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }

// MODE 0: all views read the same input row and no view masks edges -> one accumulator, perturbed per view in the
//         epilogue (SimGCL layer 1);  MODE 1: per-view inputs, no edge masks -> V accumulators, ONE weight per entry;
// MODE 2: per-view edge masks -> V accumulators, V weights per entry.
// VM (view-major): V is 1 here, the thread serves view blockIdx.y of a.n_views; MODE 1 / 2 only.
template <int G, int V, int MODE, bool VM>
__device__ __forceinline__ void prop_item(const PlanDev &p, const ssl_prop_args &a, const int64_t item_idx, const int4 it) {
    constexpr bool SHARED = MODE == 0;
    constexpr int NA = SHARED ? 1 : V;
    constexpr int NW = (MODE == 2) ? V : 1;        // distinct weights per entry
    constexpr int UNR = (NA == 1 && G >= 8) ? 8 : 4;   // entries whose row gathers are in flight together (single view: 8)
    static_assert(!VM || (V == 1 && MODE != 0), "view-major serves one view per thread");
    const int lane = threadIdx.x & 31;
    const int gl = lane % G;
    const int grp = lane / G;
    const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (grp * G));
    const int dim = a.dim;
    const int col = gl * 4;
    const bool lane_on = col < dim;
    const int vbase = VM ? (int)blockIdx.y : 0;    // first (only) view of this thread
    const int nv = VM ? a.n_views : V;             // views interleaved in the row-wise tables
    const int r = it.x;
    const uint32_t grow = (uint32_t)r + ((r < p.split_local) ? p.off_a : p.off_b);    // global row

    // row-restricted views (row_bits): decided once per item; an inactive view issues no gathers (its partial stays zero)
    // and stores nothing.  At active rows the arithmetic and its order are those of an unrestricted launch.
    uint32_t act = 0u;                 // bit vi: view vbase + vi is computed at this row
#pragma unroll
    for (int vi = 0; vi < V; ++vi) {
        const uint32_t *bits = a.row_bits[vbase + vi];
        if (bits == nullptr || (r >= 0 && ((__ldg(bits + (grow >> 5)) >> (grow & 31)) & 1u) != 0u)) act |= 1u << vi;
    }
    // accumulators that gather: per view, or -- one shared accumulator -- when any view is computed; 0 on idle lanes
    const uint32_t gather = lane_on ? (SHARED ? (act != 0u ? 1u : 0u) : act) : 0u;

    float4 acc[NA];
#pragma unroll
    for (int v = 0; v < NA; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);

    const size_t in_row = (size_t)a.in_views * dim;
    const float *xin = a.x_in + ((VM && a.in_views != 1) ? vbase * dim : 0);
    for (int base = it.y; base < it.z; base += G) {
        const int pe = base + gl;
        const bool valid = pe < it.z;
        const int c = valid ? __ldg(p.colidx + pe) : 0;
        const float w = valid ? __ldg(p.vals + pe) : 0.f;
        float wv[NW];
#pragma unroll
        for (int v = 0; v < NW; ++v) {
            float f = w;
            if (MODE == 2) {
                const int mode = a.edge_mode[vbase + v];
                if (mode == 1) {
                    const uint32_t kr = a.transpose ? (uint32_t)c : grow;
                    const uint32_t kc = a.transpose ? grow : (uint32_t)c;
                    f = (valid && ssl::edge_keep_rng(view_seed(a, vbase + v), a.edge_stream_id, kr, kc, a.edge_keep[vbase + v])) ? w * a.edge_scale[vbase + v] : 0.f;
                } else if (mode == 2) {
                    const int q = valid ? (a.transpose ? __ldg(p.rev + pe) : pe) : 0;
                    f = (valid && a.edge_mask[vbase + v][q]) ? w * a.edge_scale[vbase + v] : 0.f;
                }
            }
            wv[v] = f;
        }
        const int cnt = min(G, it.z - base);
        for (int j = 0; j < cnt; j += UNR) {
            int cj[UNR];
            float wj[UNR][NW];
            float4 x[UNR][NA];
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                cj[u] = __shfl_sync(gmask, c, j + u, G);
#pragma unroll
                for (int v = 0; v < NW; ++v) wj[u][v] = __shfl_sync(gmask, wv[v], j + u, G);
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u) {
                const float *xr = xin + (size_t)cj[u] * in_row + col;
#pragma unroll
                for (int v = 0; v < NA; ++v) {
                    x[u][v] = make_float4(0.f, 0.f, 0.f, 0.f);
                    if (((gather >> v) & 1u) && wj[u][NW == 1 ? 0 : v] != 0.f) x[u][v] = ssl::ldg4(xr + ((VM || a.in_views == 1) ? 0 : v * dim));
                }
            }
#pragma unroll
            for (int u = 0; u < UNR; ++u)
#pragma unroll
                for (int v = 0; v < NA; ++v) ssl::fma4(acc[v], wj[u][NW == 1 ? 0 : v], x[u][v]);
        }
    }
    if (r < 0) return;

    // ---- split rows: publish the partial, the last arrival reduces in segment order ----
    if (it.w >= 0) {
        const int2 li = p.long_info[it.w];
        // split items are items [0, n_slots); a slot holds every view's partial (view v at v * dim); a view-major launch
        // keeps one arrival ticket per (view, long row)
        int32_t *ticket = p.counters + (size_t)vbase * p.n_long + it.w;
        float *mine = p.partial + (size_t)item_idx * kPartialStride + vbase * dim;
        if (lane_on) {
#pragma unroll
            for (int v = 0; v < NA; ++v) *reinterpret_cast<float4 *>(mine + v * dim + col) = acc[v];
        }
        __threadfence();
        int last = 0;
        if (gl == 0) last = (atomicAdd(ticket, 1) == li.y - 1);
        last = __shfl_sync(gmask, last, 0, G);
        if (!last) return;
        __threadfence();
#pragma unroll
        for (int v = 0; v < NA; ++v) acc[v] = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int s = 0; s < li.y; ++s) {
            const float *ps = p.partial + (size_t)(li.x + s) * kPartialStride + vbase * dim;
            if (lane_on) {
#pragma unroll
                for (int v = 0; v < NA; ++v) ssl::add4(acc[v], __ldcg(reinterpret_cast<const float4 *>(ps + v * dim + col)));
            }
        }
        if (gl == 0) *ticket = 0;   // ready for the next launch (stream ordered)
    }

    // ---- epilogue: residual, perturbation, layer output (own table + peers' tables), layer sum ----
    float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
    const size_t out_row = (size_t)grow * nv * dim;
#pragma unroll
    for (int vi = 0; vi < V; ++vi) {
        if (!((act >> vi) & 1u)) continue;            // the whole group skips (one row per group): the noise shuffle stays convergent
        const int v = vbase + vi;
        float4 x = acc[SHARED ? 0 : vi];
        if (a.residual != nullptr && lane_on) ssl::add4(x, ssl::ldg4(a.residual + out_row + v * dim + col));
        const int nm = a.noise_mode[v];
        if (nm != 0) {
            float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
            if (lane_on) {
                if (nm == 1) u = ssl::noise_u4_rng(view_seed(a, v), a.noise_stream_id, grow, (uint32_t)gl);
                else u = ssl::ldg4(a.noise_u[v] + (size_t)grow * dim + col);
            }
            float ss = u.x * u.x + u.y * u.y + u.z * u.z + u.w * u.w;
#pragma unroll
            for (int o = G / 2; o > 0; o >>= 1) ss += __shfl_xor_sync(gmask, ss, o, G);
            const float sc = a.noise_eps / fmaxf(sqrtf(ss), 1e-12f);   // F.normalize(p=2, eps=1e-12) * eps
            x.x += sgnf(x.x) * (u.x * sc);
            x.y += sgnf(x.y) * (u.y * sc);
            x.z += sgnf(x.z) * (u.z * sc);
            x.w += sgnf(x.w) * (u.w * sc);
        }
        if (!lane_on) continue;
        const size_t o = out_row + v * dim + col;
        if (a.x_out != nullptr) {
            *reinterpret_cast<float4 *>(a.x_out + o) = x;
            for (int q = 0; q < a.n_peers; ++q) *reinterpret_cast<float4 *>(a.x_out_peers[q] + o) = x;   // NVLink stores
        }
        if (a.sum_out != nullptr) {
            for (int i = 0; i < a.n_sum_src; ++i) {
                const int sv = a.sum_src_views[i];
                ssl::add4(x, ssl::ldg4(a.sum_src[i] + ((size_t)grow * sv + (sv == 1 ? 0 : v)) * dim + col));
            }
            if (a.reduce_views) ssl::add4(tot, x);
            else {
                *reinterpret_cast<float4 *>(a.sum_out + o) = x;
                for (int q = 0; q < a.n_peers; ++q) *reinterpret_cast<float4 *>(a.sum_out_peers[q] + o) = x;
            }
        }
    }
    if (a.sum_out != nullptr && a.reduce_views && lane_on) {
        if (a.reg_src != nullptr) {
            const float c = (a.reg_coef_dev != nullptr) ? a.reg_coef * __ldg(a.reg_coef_dev) : a.reg_coef;
            ssl::fma4(tot, c, ssl::ldg4(a.reg_src + (size_t)grow * dim + col));
        }
        if (a.reg_src2 != nullptr) ssl::add4(tot, ssl::ldg4(a.reg_src2 + (size_t)grow * dim + col));
        const size_t o = (size_t)grow * dim + col;
        *reinterpret_cast<float4 *>(a.sum_out + o) = tot;
        for (int q = 0; q < a.n_peers; ++q) *reinterpret_cast<float4 *>(a.sum_out_peers[q] + o) = tot;
    }
}

// One work item per group; the grid covers the list (blockIdx.y = view when view-major).  Tried and dropped (profiles/
// r02_prop_variants.md): a resident grid striding over the list with the next header prefetched (1.2-1.5x slower: the hardware CTA
// scheduler balances the uneven items better than a static stride) and a 2-deep / 6-CTA variant (1.05-1.4x slower).
template <int G, int V, int MODE, bool VM>
__global__ void __launch_bounds__(kThreads, (V <= 3) ? 4 : 3) prop_kernel(PlanDev p, ssl_prop_args a) {
    constexpr int RPW = 32 / G;
    const int grp = (threadIdx.x & 31) / G;
    const int64_t warp = (int64_t)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
    const int64_t item_idx = warp * RPW + grp;
    int4 it = make_int4(-1, 0, 0, -1);
    if (item_idx < p.n_items) it = p.items[item_idx];
    prop_item<G, V, MODE, VM>(p, a, item_idx, it);
}

template <int G, int V, int MODE, bool VM>
int launch_variant(const PlanDev &p, const ssl_prop_args &a, int64_t n_items, cudaStream_t st) {
    constexpr int RPW = 32 / G;
    const int64_t items_per_block = (int64_t)(kThreads / 32) * RPW;
    const dim3 grid((unsigned)((n_items + items_per_block - 1) / items_per_block), VM ? (unsigned)a.n_views : 1u);
    prop_kernel<G, V, MODE, VM><<<grid, kThreads, 0, st>>>(p, a);
    SSL_LAUNCH_CHECK("prop_kernel");
    return SSL_OK;
}

template <int G, int V>
int launch_gv(const ssl_plan *plan, const ssl_prop_args &a, int mode, bool view_major, cudaStream_t st) {
    PlanDev p{plan->colidx, plan->vals, plan->rev, plan->items, plan->long_info, plan->counters, plan->partial,
              plan->n_items, plan->n_long, (int32_t)plan->split_local, (uint32_t)plan->off_a, (uint32_t)plan->off_b};
    if (plan->n_items == 0) return SSL_OK;
    if (view_major) {
        if (mode == 1) return launch_variant<G, 1, 1, true>(p, a, plan->n_items, st);
        return launch_variant<G, 1, 2, true>(p, a, plan->n_items, st);
    }
    if (mode == 0) return launch_variant<G, V, 0, false>(p, a, plan->n_items, st);
    if (mode == 1) return launch_variant<G, V, 1, false>(p, a, plan->n_items, st);
    return launch_variant<G, V, 2, false>(p, a, plan->n_items, st);
}

template <int G>
int launch_g(const ssl_plan *plan, const ssl_prop_args &a, int mode, bool view_major, cudaStream_t st) {
    if (view_major) return launch_gv<G, 1>(plan, a, mode, true, st);
    switch (a.n_views) {
        case 1: return launch_gv<G, 1>(plan, a, mode, false, st);
        case 2: return launch_gv<G, 2>(plan, a, mode, false, st);
        case 3: return launch_gv<G, 3>(plan, a, mode, false, st);
        case 4: return launch_gv<G, 4>(plan, a, mode, false, st);
    }
    return SSL_E_ARG;
}

}  // namespace

extern "C" int ssl_plan_create(ssl_plan **out, const int32_t *h_rowptr, const int32_t *d_colidx, const float *d_vals,
                               const int32_t *d_rev, int64_t n_rows, int64_t n_cols, int64_t nnz, int64_t row_offset,
                               int64_t side_split, void *stream) {
    return ssl_plan_create_ranges(out, h_rowptr, d_colidx, d_vals, d_rev, n_rows, n_cols, nnz, row_offset, row_offset + n_rows, 0, 0,
                                  side_split, stream);
}

extern "C" int ssl_plan_create_ranges(ssl_plan **out, const int32_t *h_rowptr, const int32_t *d_colidx, const float *d_vals,
                                      const int32_t *d_rev, int64_t n_rows, int64_t n_cols, int64_t nnz, int64_t a0, int64_t a1,
                                      int64_t b0, int64_t b1, int64_t side_split, void *stream) {
    SSL_CHECK_ARG(out && h_rowptr, "ssl_plan_create: null argument");
    SSL_CHECK_ARG(nnz == 0 || (d_colidx && d_vals), "ssl_plan_create: null CSR arrays");
    SSL_CHECK_ARG(n_rows >= 0 && n_cols > 0 && nnz >= 0 && nnz < (int64_t)INT32_MAX, "ssl_plan_create: bad sizes");
    SSL_CHECK_ARG(0 <= a0 && a0 <= a1 && 0 <= b0 && b0 <= b1 && (a1 - a0) + (b1 - b0) == n_rows && a1 <= n_cols && b1 <= n_cols &&
                      (b1 == b0 || a1 <= b0),
                  "ssl_plan_create: the row ranges [%lld,%lld) + [%lld,%lld) must be ascending, disjoint and cover n_rows = %lld",
                  (long long)a0, (long long)a1, (long long)b0, (long long)b1, (long long)n_rows);
    SSL_CHECK_ARG(h_rowptr[0] == 0 && h_rowptr[n_rows] == nnz, "ssl_plan_create: rowptr does not span nnz");
    const int64_t split_range = a1 - a0;                     // local rows [0, split_range) are range a
    auto global_row = [&](int64_t r) { return r < split_range ? a0 + r : b0 + (r - split_range); };
    cudaStream_t st = (cudaStream_t)stream;

    // ---- host work list: split long rows, then whole rows by descending degree (counting sort) ----
    std::vector<int4> items;
    std::vector<int2> longs;
    // two sides (rows before / from side_split), each ordered by descending degree: bucket index = side * (kMinSeg+1) + (kMinSeg - deg)
    const int n_bucket = 2 * (kMinSeg + 1);
    std::vector<int64_t> bucket(n_bucket + 1, 0);
    auto bucket_of = [&](int64_t r, int64_t deg) { return (int)((global_row(r) < side_split ? 0 : 1) * (kMinSeg + 1) + (kMinSeg - deg)); };
    int64_t max_deg = 0;
    for (int64_t r = 0; r < n_rows; ++r) {
        const int64_t deg = (int64_t)h_rowptr[r + 1] - h_rowptr[r];
        SSL_CHECK_ARG(deg >= 0, "ssl_plan_create: rowptr not monotone at row %lld", (long long)r);
        max_deg = std::max(max_deg, deg);
        if (deg > kMinSeg) {
            // segment length ~ 2 sqrt(deg): the serial segment walk and the serial fix-up stay balanced
            int64_t seg = (int64_t)std::ceil(2.0 * std::sqrt((double)deg));
            seg = std::max<int64_t>(kMinSeg, (seg + kMinSeg - 1) / kMinSeg * kMinSeg);
            const int64_t nseg = (deg + seg - 1) / seg;
            longs.push_back(make_int2((int)items.size(), (int)nseg));
            for (int64_t s = 0; s < nseg; ++s) {
                const int64_t b = h_rowptr[r] + s * seg;
                items.push_back(make_int4((int)r, (int)b, (int)std::min<int64_t>(b + seg, h_rowptr[r + 1]), (int)longs.size() - 1));
            }
        } else {
            bucket[bucket_of(r, deg)]++;
        }
    }
    const int64_t n_slots = (int64_t)items.size();
    // counting-sort placement of the whole rows: side 0 by descending degree, then side 1 by descending degree
    std::vector<int64_t> start(n_bucket, 0);
    {
        int64_t pos = n_slots;
        for (int b = 0; b < n_bucket; ++b) {
            start[b] = pos;
            pos += bucket[b];
        }
        items.resize(pos);
    }
    for (int64_t r = 0; r < n_rows; ++r) {
        const int64_t deg = (int64_t)h_rowptr[r + 1] - h_rowptr[r];
        if (deg <= kMinSeg) items[start[bucket_of(r, deg)]++] = make_int4((int)r, h_rowptr[r], h_rowptr[r + 1], -1);
    }

    ssl_plan *p = new (std::nothrow) ssl_plan();
    if (!p) {
        ssl::set_error("ssl_plan_create: out of host memory");
        return SSL_E_ALLOC;
    }
    *p = ssl_plan{};
    p->n_rows = n_rows; p->n_cols = n_cols; p->nnz = nnz; p->row_offset = a0;
    p->split_local = split_range; p->off_a = a0; p->off_b = b0 - split_range;
    p->colidx = d_colidx; p->vals = d_vals; p->rev = d_rev;
    p->n_items = (int64_t)items.size(); p->n_long = (int64_t)longs.size(); p->n_slots = n_slots; p->max_deg = max_deg;
    auto fail = [&](cudaError_t e, const char *what) {
        ssl::set_error("ssl_plan_create: %s: %s", what, cudaGetErrorString(e));
        ssl_plan_destroy(p);
        return SSL_E_CUDA;
    };
    cudaError_t e;
    if (p->n_items) {
        if ((e = cudaMalloc(&p->items, sizeof(int4) * p->n_items)) != cudaSuccess) return fail(e, "cudaMalloc items");
        if ((e = cudaMemcpyAsync(p->items, items.data(), sizeof(int4) * p->n_items, cudaMemcpyHostToDevice, st)) != cudaSuccess)
            return fail(e, "copy items");
    }
    if (p->n_long) {
        if ((e = cudaMalloc(&p->long_info, sizeof(int2) * p->n_long)) != cudaSuccess) return fail(e, "cudaMalloc long_info");
        if ((e = cudaMalloc(&p->counters, sizeof(int32_t) * p->n_long * SSL_MAX_VIEWS)) != cudaSuccess) return fail(e, "cudaMalloc counters");
        if ((e = cudaMalloc(&p->partial, sizeof(float) * kPartialStride * p->n_slots)) != cudaSuccess) return fail(e, "cudaMalloc partial");
        if ((e = cudaMemcpyAsync(p->long_info, longs.data(), sizeof(int2) * p->n_long, cudaMemcpyHostToDevice, st)) != cudaSuccess)
            return fail(e, "copy long_info");
        if ((e = cudaMemsetAsync(p->counters, 0, sizeof(int32_t) * p->n_long * SSL_MAX_VIEWS, st)) != cudaSuccess) return fail(e, "memset counters");
    }
    if ((e = cudaStreamSynchronize(st)) != cudaSuccess) return fail(e, "synchronize");   // host vectors die here
    *out = p;
    return SSL_OK;
}

extern "C" int ssl_set_option(const char *name, int64_t value) {
    SSL_CHECK_ARG(name != nullptr, "ssl_set_option: null name");
    const std::string n(name);
    if (n == "prop_view_major") {
        g_view_major = value != 0;
        return SSL_OK;
    }
    if (n == "prop_interleaved") {          // round-2a name: 1 = not view-major
        g_view_major = value == 0;
        return SSL_OK;
    }
    if (n == "kmeans_rows_per_round") {     // 1: kmeans_assign_kernel<1> (one row per warp and round); anything else: the default <4>
        ssl::g_kmeans_rows_per_round = value == 1 ? 1 : 4;
        return SSL_OK;
    }
    if (n == "predict_tiled") {             // 0: the warp-per-item score kernel instead of the tiled one (ssl_predict_mask)
        ssl::g_predict_tiled = value != 0;
        return SSL_OK;
    }
    ssl::set_error("ssl_set_option: unknown option '%s'", name);
    return SSL_E_ARG;
}

extern "C" int ssl_plan_destroy(ssl_plan *p) {
    if (!p) return SSL_OK;
    cudaFree(p->items);
    cudaFree(p->long_info);
    cudaFree(p->counters);
    cudaFree(p->partial);
    delete p;
    return SSL_OK;
}

extern "C" int ssl_plan_stats(const ssl_plan *p, int64_t out[4]) {
    SSL_CHECK_ARG(p && out, "ssl_plan_stats: null argument");
    out[0] = p->n_items; out[1] = p->n_long; out[2] = p->n_slots; out[3] = p->max_deg;
    return SSL_OK;
}

extern "C" int ssl_propagate_layer(const ssl_plan *plan, const ssl_prop_args *args, void *stream) {
    SSL_CHECK_ARG(plan && args, "ssl_propagate_layer: null argument");
    const ssl_prop_args &a = *args;
    SSL_CHECK_ARG(a.dim >= 4 && a.dim <= SSL_MAX_DIM && a.dim % 4 == 0, "ssl_propagate_layer: dim %d must be a multiple of 4 in [4, %d]", a.dim, SSL_MAX_DIM);
    SSL_CHECK_ARG(a.n_views >= 1 && a.n_views <= SSL_MAX_VIEWS, "ssl_propagate_layer: n_views %d out of range", a.n_views);
    SSL_CHECK_ARG(a.in_views == 1 || a.in_views == a.n_views, "ssl_propagate_layer: in_views must be 1 or n_views");
    SSL_CHECK_ARG(a.x_in != nullptr, "ssl_propagate_layer: x_in is null");
    SSL_CHECK_ARG(a.x_out != nullptr || a.sum_out != nullptr, "ssl_propagate_layer: no output requested");
    SSL_CHECK_ARG(a.n_sum_src >= 0 && a.n_sum_src <= SSL_MAX_SUM_SRC, "ssl_propagate_layer: n_sum_src out of range");
    SSL_CHECK_ARG((a.reg_src == nullptr && a.reg_src2 == nullptr) || a.reduce_views, "ssl_propagate_layer: reg_src / reg_src2 need reduce_views");
    SSL_CHECK_ARG(a.reg_coef_dev == nullptr || a.reg_src != nullptr, "ssl_propagate_layer: reg_coef_dev without reg_src");
    for (int v = 0; v < a.n_views; ++v)
        SSL_CHECK_ARG(a.row_bits[v] == nullptr || (a.sum_out != nullptr && a.x_out == nullptr && !a.reduce_views),
                      "ssl_propagate_layer: a row-restricted view (row_bits[%d]) needs a launch that writes sum_out only, without x_out or reduce_views", v);
    bool any_edge = false;
    for (int v = 0; v < a.n_views; ++v) {
        SSL_CHECK_ARG(a.edge_mode[v] >= 0 && a.edge_mode[v] <= 2 && a.noise_mode[v] >= 0 && a.noise_mode[v] <= 2, "ssl_propagate_layer: bad mode for view %d", v);
        SSL_CHECK_ARG(a.edge_mode[v] != 2 || a.edge_mask[v] != nullptr, "ssl_propagate_layer: injected edge mask missing for view %d", v);
        SSL_CHECK_ARG(a.edge_mode[v] != 2 || !a.transpose || plan->rev != nullptr, "ssl_propagate_layer: injected mask with transpose needs the plan's rev array");
        SSL_CHECK_ARG(a.noise_mode[v] != 2 || a.noise_u[v] != nullptr, "ssl_propagate_layer: injected noise missing for view %d", v);
        any_edge |= a.edge_mode[v] != 0;
    }
    for (int i = 0; i < a.n_sum_src; ++i)
        SSL_CHECK_ARG(a.sum_src[i] && (a.sum_src_views[i] == 1 || a.sum_src_views[i] == a.n_views), "ssl_propagate_layer: bad sum_src %d", i);
    SSL_CHECK_ARG(a.n_peers >= 0 && a.n_peers <= SSL_MAX_PEERS, "ssl_propagate_layer: n_peers %d out of range", a.n_peers);
    for (int q = 0; q < a.n_peers; ++q) {
        SSL_CHECK_ARG(a.x_out == nullptr || a.x_out_peers[q] != nullptr, "ssl_propagate_layer: x_out_peers[%d] is null", q);
        SSL_CHECK_ARG(a.sum_out == nullptr || a.sum_out_peers[q] != nullptr, "ssl_propagate_layer: sum_out_peers[%d] is null", q);
    }
    SSL_CHECK_ARG(plan->n_cols + (int64_t)1 < ((int64_t)1 << 32), "ssl_propagate_layer: node ids must fit 32 bits");
    const int mode = any_edge ? 2 : ((a.in_views == 1) ? 0 : 1);
    // view-major: per-view inputs (mode 1 / 2 with more than one view) and no cross-view reduction in the epilogue
    const bool view_major = a.n_views > 1 && !a.reduce_views && (mode == 2 || a.in_views == a.n_views) && g_view_major;
    cudaStream_t st = (cudaStream_t)stream;
    const int quads = a.dim / 4;
    if (quads <= 4) return launch_g<4>(plan, a, mode, view_major, st);
    if (quads <= 8) return launch_g<8>(plan, a, mode, view_major, st);
    if (quads <= 16) return launch_g<16>(plan, a, mode, view_major, st);
    return launch_g<32>(plan, a, mode, view_major, st);
}

// ---------------------------------------------------------------------------------------------
// NodeDrop
// ---------------------------------------------------------------------------------------------
namespace {
struct NodeArgs {
    int32_t mode[SSL_MAX_VIEWS];
    float keep[SSL_MAX_VIEWS];
    const uint8_t *mask[SSL_MAX_VIEWS];
    uint64_t seed[SSL_MAX_VIEWS];
    const uint64_t *seed_ptr[SSL_MAX_VIEWS];
};

__global__ void node_drop_kernel(const float *__restrict__ x, float *__restrict__ out, int64_t n, int dim, int n_views,
                                 int backward, NodeArgs na, uint32_t row_offset) {
    const int quads = dim / 4;
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n * quads) return;
    const int64_t r = i / quads;
    const int q = (int)(i % quads);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 xin = make_float4(0.f, 0.f, 0.f, 0.f);
    if (!backward) xin = ssl::ldg4(x + r * dim + q * 4);
    for (int v = 0; v < n_views; ++v) {
        bool keep = true;
        if (na.mode[v] == 1) keep = ssl::node_keep_rng(na.seed_ptr[v] != nullptr ? __ldg(na.seed_ptr[v]) : na.seed[v], row_offset + (uint32_t)r, na.keep[v]);
        else if (na.mode[v] == 2) keep = na.mask[v][r] != 0;
        if (!backward) {
            *reinterpret_cast<float4 *>(out + ((size_t)r * n_views + v) * dim + q * 4) = keep ? xin : make_float4(0.f, 0.f, 0.f, 0.f);
        } else if (keep) {
            ssl::add4(acc, ssl::ldg4(x + ((size_t)r * n_views + v) * dim + q * 4));
        }
    }
    if (backward) {
        float4 *o = reinterpret_cast<float4 *>(out + r * dim + q * 4);
        float4 cur = *o;
        ssl::add4(cur, acc);
        *o = cur;
    }
}
}  // namespace

extern "C" int ssl_node_drop(const float *x, float *out, int64_t n, int32_t dim, int32_t n_views, int32_t backward,
                             const int32_t *mode, const float *keep, const uint8_t *const *mask, const uint64_t *seed,
                             int64_t row_offset, void *stream) {
    return ssl_node_drop_dev(x, out, n, dim, n_views, backward, mode, keep, mask, seed, nullptr, row_offset, stream);
}

extern "C" int ssl_node_drop_dev(const float *x, float *out, int64_t n, int32_t dim, int32_t n_views, int32_t backward,
                                 const int32_t *mode, const float *keep, const uint8_t *const *mask, const uint64_t *seed,
                                 const uint64_t *const *seed_ptr, int64_t row_offset, void *stream) {
    SSL_CHECK_ARG(x && out && mode && keep && seed, "ssl_node_drop: null argument");
    SSL_CHECK_ARG(dim >= 4 && dim % 4 == 0 && n_views >= 1 && n_views <= SSL_MAX_VIEWS, "ssl_node_drop: bad shape");
    NodeArgs na{};
    for (int v = 0; v < n_views; ++v) {
        na.mode[v] = mode[v]; na.keep[v] = keep[v]; na.seed[v] = seed[v];
        na.seed_ptr[v] = seed_ptr ? seed_ptr[v] : nullptr;
        na.mask[v] = mask ? mask[v] : nullptr;
        SSL_CHECK_ARG(mode[v] != 2 || na.mask[v], "ssl_node_drop: injected mask missing for view %d", v);
    }
    const int64_t total = n * (dim / 4);
    if (total == 0) return SSL_OK;
    node_drop_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, out, n, dim, n_views, backward, na, (uint32_t)row_offset);
    SSL_LAUNCH_CHECK("node_drop_kernel");
    return SSL_OK;
}
