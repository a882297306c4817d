/*
 * sslrec_b200 -- C ABI of the H100 (sm_90a) general_cf training hot path.
 *
 * The reference (HKUDS/SSLRec) has no FFI: its "operator interface" for this path is the set of
 * PyTorch calls made by models/general_cf/*.py, models/loss_utils.py, models/aug_utils.py and
 * trainer/trainer.py.  Each entry point below names the reference call site(s) it replaces
 * (file:line, relative to the reference checkout).  INTEGRATION.md shows the ctypes binding a
 * maintainer adds on the reference side.
 *
 * Conventions
 *   - plain C: raw device pointers, sizes, a cudaStream_t passed as void*; no torch types.
 *   - every function returns 0 on success, a negative SSL_E_* code otherwise; the message is
 *     available from ssl_last_error() (thread-local).  No C++ exception crosses the boundary.
 *   - the caller owns every buffer it passes; the library owns only what lives inside an
 *     ssl_plan (work lists + split-row scratch).  Kernels are enqueued on the given stream and
 *     never synchronise it (ssl_plan_create synchronises once, for its uploads).
 *   - all floating point is fp32; node / item ids inside batches are int64 (trainer.py:64),
 *     CSR indices are int32.
 *   - "table view": a [rows, dim] fp32 matrix addressed as base + row * stride (stride in
 *     floats), so one view of the interleaved [N, V, dim] propagation output is
 *     (E + v*dim, V*dim) without a copy.
 */
#ifndef SSLREC_B200_H
#define SSLREC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SSL_API __attribute__((visibility("default")))
#else
#define SSL_API
#endif

#define SSL_OK 0
#define SSL_E_ARG (-1)     /* bad argument (shape, null pointer, unsupported dim) */
#define SSL_E_CUDA (-2)    /* a CUDA runtime call or kernel launch failed */
#define SSL_E_ALLOC (-3)

#define SSL_MAX_VIEWS 4
#define SSL_MAX_CANDIDATES 256   /* negative candidates per BPR pair (train.dns_candidates) */
#define SSL_MAX_SUM_SRC 6
#define SSL_MAX_DIM 128    /* embedding_size must be a multiple of 4 and <= 128 */
#define SSL_MAX_PEERS 7    /* other GPUs of the node whose tables a kernel stores to over NVLink (8-GPU NVSwitch domain) */

SSL_API int ssl_version(void);
SSL_API const char *ssl_last_error(void);
/* number of kernel launches issued by this library since load (bench.py's gpu_launches) */
SSL_API int64_t ssl_launch_count(void);
/* process-wide switches for tests and A/B profiling (value 0 / 1):
 *   "prop_view_major"  propagation with grid.y = view and one accumulator per thread: DRAM traffic at 1.03x compulsory instead of
 *                      1.3x, at the cost of less work per thread (the kernel is issue / latency bound); default 0
 *   "kmeans_rows_per_round"  1 selects kmeans_assign_kernel<1> (one row per warp and round, the round-1 form); default 4 rows per round --
 *                      same arithmetic per (row, centroid), same summation order: bit-identical results (csrc/kmeans_assign.cuh)
 *   "predict_tiled"    ssl_predict_mask as a register-tiled product (128 x 128 score tiles, csrc/predict_tile.cuh); 0 selects the
 *                      round-1 warp-per-item kernel (4 % of the FFMA rate, profiles/r02_ncu_kernels.md), kept as the cross-check; default 1 */
SSL_API int ssl_set_option(const char *name, int64_t value);

/* ------------------------------------------------------------------------------------------
 * a1/a2  adjacency plan -- replaces the torch sparse COO tensor built by
 * data_utils/data_handler_general_cf.py:53-73 as the operand of t.spmm (lightgcn.py:28-29).
 * CSR of the (row block of the) normalised adjacency; the structure and values are symmetric,
 * so the same plan serves A and A^T.
 *   h_rowptr  host  int32 [n_rows+1]   (read during create only)
 *   d_colidx  device int32 [nnz]       global column (node) ids, ascending inside a row
 *   d_vals    device fp32  [nnz]
 *   d_rev     device int32 [nnz] or NULL: position of the reverse entry (col,row); only needed
 *             when an *injected* edge mask is used together with transpose = 1
 *   row_offset  global id of local row 0 (row-sharded multi-GPU; 0 on one GPU)
 *   side_split  global row id where the second side of the bipartite graph starts (|U|), or 0: the work list
 *               then runs all rows of one side before the other, so concurrently running CTAs gather from one
 *               half of the table only (user rows read item rows and vice versa) -- halves the L2 working set
 * ------------------------------------------------------------------------------------------ */
typedef struct ssl_plan ssl_plan;

SSL_API int ssl_plan_create(ssl_plan **out, const int32_t *h_rowptr, const int32_t *d_colidx, const float *d_vals,
                    const int32_t *d_rev, int64_t n_rows, int64_t n_cols, int64_t nnz, int64_t row_offset,
                    int64_t side_split, void *stream);
/* Row-sharded multi-GPU (SURVEY.md 8e): the plan owns the global rows [a0, a1) followed by [b0, b1) -- a GPU's share
 * of the user rows and of the item rows, so every GPU gets the same mix of both sides; h_rowptr runs over the
 * n_rows = (a1-a0) + (b1-b0) local rows in that order, column ids stay global.  ssl_plan_create is the single-range
 * case [row_offset, row_offset + n_rows). */
SSL_API int ssl_plan_create_ranges(ssl_plan **out, const int32_t *h_rowptr, const int32_t *d_colidx, const float *d_vals,
                           const int32_t *d_rev, int64_t n_rows, int64_t n_cols, int64_t nnz, int64_t a0, int64_t a1,
                           int64_t b0, int64_t b1, int64_t side_split, void *stream);
SSL_API int ssl_plan_destroy(ssl_plan *plan);
/* work-list statistics: out[0]=items, out[1]=split rows, out[2]=segments, out[3]=max row nnz */
SSL_API int ssl_plan_stats(const ssl_plan *plan, int64_t out[4]);

/* ------------------------------------------------------------------------------------------
 * a2-a10  one propagation layer for up to SSL_MAX_VIEWS augmented views at once.
 *
 *   acc_v[r]  = sum_p  m_v(p) * s_v * val[p] * x_in[col[p], v]          (CSR row r)
 *   x_v[r]    = acc_v[r] + residual[r, v]                                 (residual optional)
 *   x_v[r]   += eps * sign(x_v[r]) * u / max(|u|_2, 1e-12)                (noise_mode != 0)
 *   x_out[r, v]   = x_v[r]                                                (x_out optional)
 *   sum_out[r, v] = x_v[r] + sum_i sum_src[i][r, v]                       (sum_out optional;
 *                   reduce_views: sum_out[r] = sum_v of the above, + reg_coef * [*reg_coef_dev] * reg_src[r] + reg_src2[r])
 *
 * replaces: t.spmm (lightgcn.py:29, hccf.py:36), the layer sum (lightgcn.py:41, simgcl.py:29,
 * sgl.py:34, ncl.py:41), EdgeDrop (aug_utils.py:18-31) as an in-kernel keep test so no second
 * adjacency is built, EmbedPerturb (aug_utils.py:125-132) as an epilogue, and -- with
 * transpose = 1 and residual = upstream gradient -- the autograd backward of all of them
 * (dX = A_v^T dY evaluated on the same CSR with the mask key swapped).
 *
 * Layouts: x_in [n_cols, in_views, dim] (in_views = 1: all views read the same rows, or
 * = n_views); x_out, residual [n_cols, n_views, dim]; sum_src[i] [n_cols, sum_src_views[i], dim]
 * with sum_src_views[i] in {1, n_views}; sum_out [n_cols, n_views, dim] or [n_cols, dim].
 * Every table is FULL height (n_cols = N rows) and addressed by the GLOBAL row id; a row-sharded
 * plan reads and writes only the rows it owns.
 *
 * Fused all-gather (row-sharded multi-GPU, one NVSwitch domain): with n_peers > 0 every finished
 * row of x_out / sum_out is also stored to the same row of x_out_peers[q] / sum_out_peers[q] --
 * the other GPUs' tables, mapped into this process (CUDA IPC / symmetric memory) -- so after the
 * launches of all ranks have completed (cross-GPU barrier, caller's job) every GPU holds the
 * whole layer output; the NVLink stores overlap the gathers of the rows still being computed.
 * This replaces "one NCCL allgather of the d-wide layer output per layer".
 *
 * edge_mode[v]: 0 keep all; 1 counter-based RNG: keep iff U(seed[v], edge_stream_id, row, col) >= 1-keep
 *               (floor(U + keep), aug_utils.py:28); 2 injected: edge_mask[v][p] != 0, p = CSR
 *               position (rev[p] when transpose).  edge_scale[v] multiplies kept values
 *               (1, or 1/keep for EdgeDrop(resize_val=True), hccf.py:33).
 * noise_mode[v]: 0 none; 1 RNG uniform(seed[v], noise_stream_id, row, elem);
 *               2 injected: noise_u[v] is a [n_cols, dim] U[0,1) tensor (global row).
 * ------------------------------------------------------------------------------------------ */
typedef struct ssl_prop_args {
    int32_t dim, n_views, in_views, transpose;
    const float *x_in;
    float *x_out;
    float *sum_out;
    const float *residual;
    int32_t reduce_views;
    int32_t n_sum_src;
    const float *sum_src[SSL_MAX_SUM_SRC];
    int32_t sum_src_views[SSL_MAX_SUM_SRC];
    float reg_coef;
    const float *reg_src;             /* [n_rows, dim]; only with reduce_views */
    int32_t edge_mode[SSL_MAX_VIEWS];
    float edge_keep[SSL_MAX_VIEWS];
    float edge_scale[SSL_MAX_VIEWS];
    const uint8_t *edge_mask[SSL_MAX_VIEWS];
    int32_t noise_mode[SSL_MAX_VIEWS];
    const float *noise_u[SSL_MAX_VIEWS];
    float noise_eps;
    uint64_t seed[SSL_MAX_VIEWS];
    uint32_t edge_stream_id;          /* RNG sub-stream of the edge mask: constant over the layers of one forward
                                         (lightgcn.py:36-37, sgl.py:27-28) or the layer index (hccf.py:47) */
    uint32_t noise_stream_id;         /* RNG sub-stream of the perturbation: the layer index (simgcl.py:26-27) */
    int32_t n_peers;                  /* 0 on one GPU */
    float *x_out_peers[SSL_MAX_PEERS];    /* peers' copies of the x_out table (same shape, same row addressing) */
    float *sum_out_peers[SSL_MAX_PEERS];  /* peers' copies of the sum_out table */
    const float *reg_coef_dev;        /* optional device scalar multiplied into reg_coef (the upstream gradient of the
                                         regulariser term: d loss / d reg_params is only known on the device) */
    const float *reg_src2;            /* optional second [n_cols, dim] row source added with coefficient 1 (with reduce_views):
                                         gradient rows that losses wrote for layer 0 (ncl.py:75) */
    const uint64_t *seed_ptr[SSL_MAX_VIEWS];  /* optional: the view's seed is READ FROM THE DEVICE (overrides seed[v]) -- a step captured
                                         in a CUDA graph draws fresh masks / noise at every replay because the host rewrites these
                                         words, not the launch arguments */
    const uint32_t *row_bits[SSL_MAX_VIEWS];  /* optional per-view bitmap over the global rows (bit r of word r / 32; NULL = every
                                         row): a view whose bit is clear for a row gathers nothing there and stores nothing.
                                         Only a launch that writes sum_out without x_out and without reduce_views may restrict
                                         a view (the last summed layer, read by the losses at batch rows only) */
} ssl_prop_args;

SSL_API int ssl_propagate_layer(const ssl_plan *plan, const ssl_prop_args *args, void *stream);

/* ------------------------------------------------------------------------------------------
 * a9  NodeDrop (aug_utils.py:40-50, sgl.py:24-25).
 * forward : out[r, v] = x[r] * m_v(r)            x [n, dim] -> out [n, n_views, dim]
 * backward: out[r]   += sum_v g[r, v] * m_v(r)   g [n, n_views, dim] -> out [n, dim]  (accumulate)
 * mode[v]: 0 keep all; 1 RNG keep iff U(seed[v], row) >= 1-keep; 2 injected mask[v][r] != 0.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_node_drop(const float *x, float *out, int64_t n, int32_t dim, int32_t n_views, int32_t backward,
                  const int32_t *mode, const float *keep, const uint8_t *const *mask, const uint64_t *seed,
                  int64_t row_offset, void *stream);
/* the same with per-view seeds read from the device (seed_ptr[v] may be NULL: then seed[v] is used) */
SSL_API int ssl_node_drop_dev(const float *x, float *out, int64_t n, int32_t dim, int32_t n_views, int32_t backward,
                      const int32_t *mode, const float *keep, const uint8_t *const *mask, const uint64_t *seed,
                      const uint64_t *const *seed_ptr, int64_t row_offset, void *stream);

/* ------------------------------------------------------------------------------------------
 * a11+a12  gathers + BPR  (lightgcn.py:48-52, loss_utils.py:7-10; hccf.py:70-74 is the same
 * function written as -log sigmoid).  loss_b = softplus(a.n - a.p), coef_b = sigmoid(a.n - a.p).
 * users / items are table views; ancs index the user view, poss/negs the item view.
 * ssl_bpr_bwd adds scale * (*gscale) * d loss_b into the gradient views (atomicAdd: batch
 * indices repeat; the reference's index_put_(accumulate) does the same).
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_bpr_fwd(const float *users, int64_t u_stride, const float *items, int64_t i_stride,
                const int64_t *ancs, const int64_t *poss, const int64_t *negs, int64_t batch, int32_t dim,
                float *loss_b, float *coef_b, void *stream);
SSL_API int ssl_bpr_bwd(const float *users, int64_t u_stride, const float *items, int64_t i_stride,
                const int64_t *ancs, const int64_t *poss, const int64_t *negs, int64_t batch, int32_t dim,
                const float *coef_b, const float *gscale, float scale,
                float *g_users, int64_t gu_stride, float *g_items, int64_t gi_stride, void *stream);

/* ------------------------------------------------------------------------------------------
 * a13/a14  InfoNCE, never materialising the [B, N_side] logits
 * (loss_utils.py:30-39 cal_infonce_loss; :42-51 cal_infonce_loss_spec_nodes with norm_mode 1).
 *
 * ssl_rows_normalize  x^ = x / sqrt(1e-8 + |x|^2)  (norm_mode 0, loss_utils.py:33-35) or
 *                     F.normalize(x + 1e-8)        (norm_mode 1, loss_utils.py:45-46) or
 *                     F.normalize(x)               (norm_mode 2, loss_utils.py:78,85) or
 *                     x itself                     (norm_mode 3: LightGCL contracts raw rows, lightgcl.py:112);
 *   optional gather (idx != NULL: row i of the output is x[idx[i]]), optional scale of the
 *   output (alpha), writes row-major out [n, dim], the K-major tile copy out_t
 *   [ceil(n/64), dim, 64] the streaming side of ssl_softmax_gemm reads (may be NULL),
 *   rinv [n] (the 1/norm used, needed by the backward), and optionally the tf32 split
 *   out_hi = tf32(out), out_lo = out - out_hi, row-major [n, dim] each, plus their transposes
 *   out_thi / out_tlo [dim, t_pitch] (t_pitch >= ceil64(n), multiple of 4) that
 *   ssl_softmax_gemm_tf32x3 reads through TMA, with the columns of every aligned group of 8 stored
 *   in the order 0 2 4 6 1 3 5 7 (row 8j + 2t + c at column 8j + t + 4c) and rows n .. ceil64(n) zero.
 * ssl_softmax_gemm    for every row r of R [n_r, dim] over the rows c of C (row-major C
 *   [n_c, dim] and its K-major tile copy C_t):   e = exp2(R_r . C_c - offset) * colscale[c]
 *   rowsum_part[s, r] = sum_c e   (optional)     o_part[s, r, :] = sum_c e * C_c
 *   for the s-th of n_split contiguous chunks of C.  One launch does the forward of a term
 *   (R = scaled anchors, C = normalised table: log-sum-exp and the softmax-weighted table
 *   average that is the anchor gradient) and, with the roles swapped, its backward
 *   (R = table tile, C = anchors, colscale = g/rowsum: the dense table gradient).
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_rows_normalize(const float *x, int64_t stride, const int64_t *idx, int64_t n, int32_t dim, int32_t norm_mode,
                       float alpha, float *out, float *out_t, float *rinv, float *out_hi, float *out_lo,
                       float *out_thi, float *out_tlo, int64_t t_pitch, void *stream);
SSL_API int ssl_softmax_gemm(const float *R, int64_t n_r, const float *C, const float *C_t, int64_t n_c, int32_t dim,
                     const float *colscale, float offset, int32_t n_split, float *rowsum_part, float *o_part,
                     void *stream);
/* The same contraction on the Hopper tensor cores (wgmma) with 3xTF32 error compensation (fp32-grade
 * accuracy): operands are the hi / lo splits written by ssl_rows_normalize, row-major [n, dim],
 * and for the streamed operand also the transposed splits CT_hi / CT_lo [dim, ct_pitch] in
 * ssl_rows_normalize's column order (ct_pitch >= ceil8(n_c), columns n_c .. ceil8(n_c) zero);
 * dim must be 32 or 64.  colscale, when given, must be readable up to ceil64(n_c) floats (the
 * padded tail is loaded with the tile and masked).  Outputs and semantics are those of
 * ssl_softmax_gemm. */
SSL_API int ssl_softmax_gemm_tf32x3(const float *R_hi, const float *R_lo, int64_t n_r, const float *C_hi, const float *C_lo,
                            const float *CT_hi, const float *CT_lo, int64_t ct_pitch, int64_t n_c, int32_t dim,
                            const float *colscale, float offset, int32_t n_split, float *rowsum_part, float *o_part,
                            void *stream);
/* The same contraction at the FP16 tensor-core rate with 3xFP16 error compensation (fp32-grade accuracy, the grade of
 * ssl_softmax_gemm_tf32x3).  Operands are the fp16 bit patterns written by ssl_rows_normalize_f16x3: for each operand
 * x = hi + 2^-12 lo, hi = fp16(x) (0 below 2^-14), lo = fp16((x - hi) 2^12), row-major [n, dim].  No transposed copy.
 * The split's bounds (derived in csrc/f16x3.cuh) need rows of norm <= 1 scaled by |alpha| <= 16 and
 * R_r . C_c <= offset, with 0 <= offset <= 16 (tau >= 0.0902 in the InfoNCE roles); an offset outside [0, 16] is
 * rejected.  colscale may take any magnitude: the kernel rescales it by a power of two found on the device.
 * dim must be 32 or 64.  Outputs and semantics are those of ssl_softmax_gemm. */
SSL_API int ssl_softmax_gemm_f16x3(const uint16_t *R_hi, const uint16_t *R_lo, int64_t n_r, const uint16_t *C_hi, const uint16_t *C_lo,
                           int64_t n_c, int32_t dim, const float *colscale, float offset, int32_t n_split, float *rowsum_part,
                           float *o_part, void *stream);
/* ssl_rows_normalize (norm_mode 0, 1 or 2, |alpha| <= 16, dim 32 or 64) writing out [n, dim] and rinv [n] as it does,
 * plus the operands of ssl_softmax_gemm_f16x3: out_hi / out_lo, fp16 [ceil64(n), dim] each, rows n .. ceil64(n) zero
 * (out must hold ceil64(n) rows as well). */
SSL_API int ssl_rows_normalize_f16x3(const float *x, int64_t stride, const int64_t *idx, int64_t n, int32_t dim, int32_t norm_mode,
                             float alpha, float *out, float *rinv, uint16_t *out_hi, uint16_t *out_lo, void *stream);
/* forward epilogue of one term: reduces the split partials and produces, per anchor b,
 *   rowsum[b] (+ deno_eps), obar[b,:] = o[b,:]/rowsum[b] and
 *   loss_b[b] = -(a^_b . p^_b)/tau + 1/tau + ln(rowsum[b])          */
SSL_API int ssl_nce_finalize(const float *rowsum_part, const float *o_part, int32_t n_split, int64_t batch, int32_t dim,
                     const float *a_hat, const float *p_hat, float tau, float deno_eps,
                     float *rowsum, float *obar, float *loss_b, void *stream);
/* backward w.r.t. the gathered rows: d a^ = g/tau (obar - p^), d p^ = -g/tau a^, pushed through
 * the normalisation (de = rinv (dx^ - x^ (x^ . dx^))) and atomically added to the gradient views.
 * g = scale * (*gscale).  g1 / g2 may be NULL (NCL prototypes, HCCF's detached side). */
SSL_API int ssl_nce_bwd_rows(const float *a_hat, const float *p_hat, const float *obar, const float *rinv1, const float *rinv2,
                     const int64_t *idx, int64_t batch, int32_t dim, float tau, const float *gscale, float scale,
                     float *g1, int64_t g1_stride, float *g2, int64_t g2_stride, void *stream);
/* backward w.r.t. the table: dt^ = sum of the split partials of the swapped ssl_softmax_gemm;
 * g_table[j] (+)= rinv_j (dt^_j - t^_j (t^_j . dt^_j)) */
SSL_API int ssl_nce_bwd_table(const float *dt_part, int32_t n_split, const float *t_hat, const float *rinv, int64_t n,
                      int32_t dim, float *g_table, int64_t g_stride, int32_t accumulate, void *stream);
/* the epilogue of a term without a positive pair, log(sum_j exp(a_b . t_j / temp) + eps) (lightgcl.py:112-113):
 * rowsum[b] = sum of the partials + eps, obar = o / rowsum, loss_b[b] = ln(rowsum[b]) */
SSL_API int ssl_lse_finalize(const float *rowsum_part, const float *o_part, int32_t n_split, int64_t batch, int32_t dim, float eps,
                     float *rowsum, float *obar, float *loss_b, void *stream);
/* colscale[b] = scale * (*gscale) * ln2 / rowsum[b] for the swapped gemm */
SSL_API int ssl_nce_colscale(const float *rowsum, int64_t batch, const float *gscale, float scale, float *colscale, void *stream);

/* ------------------------------------------------------------------------------------------
 * a13b  the InfoNCE pieces bounded by a DEVICE row count: a term over a padded anchor list whose
 * live length only the device knows (HCCF's spec-node term under CUDA-graph capture, fed by
 * ssl_unique_ids).  n_live points to an int64 on the device, clamped to [0, capacity]; the host
 * passes the capacity, so buffer shapes, tensor maps and n_split depend on host-known sizes only.
 *
 * ssl_softmax_gemm_live / ssl_softmax_gemm_tf32x3_live / ssl_softmax_gemm_f16x3_live: the contractions above, with
 *   live_role SSL_LIVE_ROWS: only rows r < *n_live of R are live (the forward, R = anchors).  Their
 *     outputs equal those of the plain call at n_r = *n_live bit for bit; rows >= *n_live of
 *     o_part / rowsum_part are not written (the row pitch stays n_r).  Units whose R tile starts
 *     at or past the count are skipped.
 *   live_role SSL_LIVE_COLS: only rows c < *n_live of C are live (the backward, C = anchors).
 *     The chunks are cut from the live tile count, columns past it are masked (colscale there is
 *     never read), and a chunk left empty writes zero partials.  Outputs equal the plain call at
 *     n_c = *n_live bit for bit, for every n_split that call accepts; C rows past the count must
 *     be finite.
 * ssl_sum_live: out[0] = alpha / live * sum_{b < live} x[b]  (0 when live = 0).
 * ssl_nce_bwd_rows_live: ssl_nce_bwd_rows over the rows b < live only, with g = scale / live * (*gscale).
 * ssl_nce_colscale_live: colscale[b] = scale / live * (*gscale) * ln2 / rowsum[b] for b < live, 0 past it.
 * ------------------------------------------------------------------------------------------ */
#define SSL_LIVE_ROWS 1
#define SSL_LIVE_COLS 2
SSL_API int ssl_softmax_gemm_live(const float *R, int64_t n_r, const float *C, const float *C_t, int64_t n_c, int32_t dim,
                          const float *colscale, float offset, int32_t n_split, float *rowsum_part, float *o_part,
                          const int64_t *n_live, int32_t live_role, void *stream);
SSL_API int ssl_softmax_gemm_tf32x3_live(const float *R_hi, const float *R_lo, int64_t n_r, const float *C_hi, const float *C_lo,
                                 const float *CT_hi, const float *CT_lo, int64_t ct_pitch, int64_t n_c, int32_t dim,
                                 const float *colscale, float offset, int32_t n_split, float *rowsum_part, float *o_part,
                                 const int64_t *n_live, int32_t live_role, void *stream);
SSL_API int ssl_softmax_gemm_f16x3_live(const uint16_t *R_hi, const uint16_t *R_lo, int64_t n_r, const uint16_t *C_hi,
                                const uint16_t *C_lo, int64_t n_c, int32_t dim, const float *colscale, float offset,
                                int32_t n_split, float *rowsum_part, float *o_part, const int64_t *n_live, int32_t live_role,
                                void *stream);
SSL_API int ssl_sum_live(const float *x, int64_t n, const int64_t *n_live, float alpha, float *out, void *stream);
SSL_API int ssl_nce_bwd_rows_live(const float *a_hat, const float *p_hat, const float *obar, const float *rinv1, const float *rinv2,
                          const int64_t *idx, int64_t batch, const int64_t *n_live, int32_t dim, float tau, const float *gscale,
                          float scale, float *g1, int64_t g1_stride, float *g2, int64_t g2_stride, void *stream);
SSL_API int ssl_nce_colscale_live(const float *rowsum, int64_t batch, const int64_t *n_live, const float *gscale, float scale,
                          float *colscale, void *stream);

/* ------------------------------------------------------------------------------------------
 * a13c  ssl_unique_ids: sorted de-duplication on the device, the graph-safe form of HCCF's
 * t.unique(ancs) / t.unique(poss) (hccf.py:80-81 of the reference).
 *   idx [n] int64, every id in [0, n_range) (a precondition; ids outside are not counted).
 *   out [n] int64: out[0, *count) = the distinct ids ascending (torch.unique(idx, sorted=True));
 *     out[*count, n) repeat the largest id, so a gather through the whole padded list stays in bounds.
 *   count: an int64 on the DEVICE.
 *   scratch: caller-owned, 16-byte aligned, scratch_n_words uint32 words (ssl_unique_ids_scratch):
 *     a bitmap of ceil(n_range / 32) words padded to whole 1024-word blocks, plus the block sums.
 *     The launch sequence clears it itself, so a CUDA-graph replay with new indices is correct.
 * Five launches (clear, mark, per-block popcount, scan, compact + padding); O(n + n_range / 32);
 * the result does not depend on scheduling.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_unique_ids_scratch(int64_t n_range, int64_t *words);
/* bits[0, ceil(n_range / 32)) = the bitmap of the ids idx[0, n) in [0, n_range) (ids outside are ignored): the row_bits of
 * ssl_prop_args built on the device, with no host read (CUDA-graph safe) */
SSL_API int ssl_row_bitmap(const int64_t *idx, int64_t n, int64_t n_range, uint32_t *bits, int64_t n_words, void *stream);
SSL_API int ssl_unique_ids(const int64_t *idx, int64_t n, int64_t n_range, uint32_t *scratch, int64_t scratch_n_words,
                   int64_t *out, int64_t *count, void *stream);

/* ------------------------------------------------------------------------------------------
 * a15  reg_params (loss_utils.py:20-24): out[0] = sum x^2, deterministic two-stage reduction.
 * ssl_sum: out[0] = alpha * sum x (same reduction; used for the per-sample loss vectors).
 * ssl_axpy: y += alpha * (*gscale) * x  (gradient of the regulariser, 2 * reg_weight * W).
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_sumsq(const float *x, int64_t n, float *out, void *stream);
SSL_API int ssl_sum(const float *x, int64_t n, float alpha, float *out, void *stream);
SSL_API int ssl_axpy(const float *x, float *y, int64_t n, const float *gscale, float alpha, void *stream);

/* ------------------------------------------------------------------------------------------
 * a20  Adam (trainer.py:45-49,68 -> torch.optim.Adam, amsgrad off): one fused pass over
 * p, g, m, v.  step is 1-based; weight_decay is folded into g as torch does.  Hyper-parameters are
 * doubles (Python floats): 1 - beta and the bias corrections are formed in double, then rounded once.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_adam_step(float *p, const float *g, float *m, float *v, int64_t n, int64_t step, double lr, double beta1,
                  double beta2, double eps, double weight_decay, void *stream);
/* Row-sharded Adam: the same update on the n elements p[0..n) this GPU owns (p, g, m, v already point at the owned
 * range), with every new parameter value also stored to the same position of p_peers[q] (the other GPUs' replicas of
 * the table, mapped over NVLink) -- the all-gather of the updated table fused into the optimizer kernel. */
SSL_API int ssl_adam_step_peers(float *p, float *const *p_peers, int32_t n_peers, const float *g, float *m, float *v, int64_t n,
                        int64_t step, double lr, double beta1, double beta2, double eps, double weight_decay, void *stream);
/* The step count read from the device: *step_dev (>= 1) is the 1-based step of THIS update; the bias corrections are formed on the
 * device (double precision, as the host path) into scratch2 (2 floats) by a one-thread launch, so that a CUDA graph holding the
 * optimizer step replays with a counter the graph itself increments. */
SSL_API int ssl_adam_step_dev(float *p, float *const *p_peers, int32_t n_peers, const float *g, float *m, float *v, int64_t n,
                      const int64_t *step_dev, float *scratch2, double lr, double beta1, double beta2, double eps, double weight_decay,
                      void *stream);

/* ------------------------------------------------------------------------------------------
 * a18  full_predict + _mask_predict (lightgcn.py:58-66, base_model.py:35-36) and the top-k that
 * consumes it (metrics.py:108).
 * ssl_predict_mask: preds[b, i] = (U[users[b]] . I[i]) * (1 - M[b,i]) - 1e8 * M[b,i]; the mask is
 *   either the dense int64 [n_b, n_item] tensor the reference passes (mask_dense) or, when that
 *   is NULL, the training CSR (trn_rowptr int32 [n_user+1], trn_cols int32) read on device.  Every score is one
 *   sequential fp32 FMA chain over k = 0 .. dim-1; masked positions read exactly -1e8.
 * ssl_topk: the k largest entries of every row, descending, ties broken by the lower index.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_predict_mask(const float *users_tab, int64_t u_stride, const float *items_tab, int64_t i_stride,
                     const int64_t *users, int64_t n_b, int64_t n_item, int32_t dim, const int64_t *mask_dense,
                     const int32_t *trn_rowptr, const int32_t *trn_cols, float *preds, void *stream);
/* Opt-in evaluation mode (test.exact_order): Y = A X with the accumulation order of the reference's CPU t.spmm (lightgcn.py:29) -- every output
 * element one sequential fp32 FMA chain over the CSR row in ascending column order, no row splitting -- so that, with the layer sum formed in
 * the reference's order and ssl_predict_mask's sequential score chains, full_predict reproduces the reference's CPU full_predict bit for bit.
 * rowptr: DEVICE int32 [n_rows + 1]; x [*, dim] / y [n_rows, dim] with row strides in floats.  Not on the training path (csrc/spmm_exact.cuh). */
SSL_API int ssl_spmm_exact(const int32_t *rowptr, const int32_t *colidx, const float *vals, int64_t n_rows, const float *x, int64_t x_stride,
                   int32_t dim, float *y, int64_t y_stride, void *stream);
SSL_API int ssl_topk(const float *preds, int64_t n_b, int64_t n_item, int32_t k, int64_t *out_idx, float *out_val, void *stream);
/* ssl_predict_topk: ssl_predict_mask followed by ssl_topk in one call, without the [n_b, n_item] score matrix: out_idx int64 [n_b, k]
 *   and, when out_val is not NULL, out_val fp32 [n_b, k] are bit-identical to that pair on the same inputs.  Each score is formed by the
 *   same FMA chain and masked by the same formula, and rows are ranked by the same total key (value descending, then item ascending),
 *   so the result does not depend on scheduling.  Arguments as ssl_predict_mask; the training CSR rows must be sorted ascending.
 *   1 <= k <= min(256, n_item), n_b <= 65535.  workspace: ws_bytes >= what ssl_predict_topk_workspace reports for (n_b, n_item, k),
 *   16-byte aligned, owned by the caller and not required to be initialised (it is O(n_b * (2k + 128)) bytes per item chunk, at most
 *   264 / ceil(n_b / 128) chunks).  Bad arguments return SSL_E_ARG before anything is written. */
SSL_API int ssl_predict_topk_workspace(int64_t n_b, int64_t n_item, int32_t k, int64_t *bytes);
SSL_API int ssl_predict_topk(const float *users_tab, int64_t u_stride, const float *items_tab, int64_t i_stride, const int64_t *users,
                     int64_t n_b, int64_t n_item, int32_t dim, const int64_t *mask_dense, const int32_t *trn_rowptr,
                     const int32_t *trn_cols, int32_t k, void *workspace, int64_t ws_bytes, int64_t *out_idx, float *out_val,
                     void *stream);

/* ------------------------------------------------------------------------------------------
 * SURVEY 8(f) row 4  DirectAU's losses (loss_utils.py:75-86) on unit rows x^ = F.normalize(x)
 * (ssl_rows_normalize with norm_mode 2).
 * ssl_align_fwd: loss_b[b] = |x^_b - y^_b|^2 (alignment, alpha = 2; the caller averages).
 * uniformity(x) = log mean_{i<j} exp(-2 |x^_i - x^_j|^2): the pair sum is ssl_softmax_gemm[_tf32x3]
 *   with R = 4 log2(e) x^, C = x^, offset = 4 log2(e); ssl_uniform_finalize reduces its split partials
 *   and removes the i == j term: pair_sum[i] = sum_{j!=i} e_ij, w[i,:] = sum_{j!=i} e_ij x^_j.
 * ssl_uniform_pairs: the same pair_sum / w computed directly, e_ij = exp(-2 |x^_i - x^_j|^2) from the
 *   difference vector over j != i, one warp per row, O(B^2 d).  Used below 256 rows, where rowsum_i - e_ii
 *   above loses most of its digits to cancellation.
 * ssl_unit_rows_bwd: dx^_b = scale * (*gscale) * (c1 d1_b + c2 d2_b) pushed through the normalisation,
 *   g_out[idx[b]] += rinv_b (dx^_b - x^_b (x^_b . dx^_b))   (d2 may be NULL; idx NULL = identity).
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_align_fwd(const float *xhat, const float *yhat, int64_t batch, int32_t dim, float *loss_b, void *stream);
SSL_API int ssl_uniform_finalize(const float *rowsum_part, const float *o_part, int32_t n_split, int64_t batch, int32_t dim,
                         const float *r_scaled, const float *xhat, float offset, float *pair_sum, float *w, void *stream);
SSL_API int ssl_uniform_pairs(const float *xhat, int64_t batch, int32_t dim, float *pair_sum, float *w, void *stream);
SSL_API int ssl_unit_rows_bwd(const float *xhat, const float *rinv, const int64_t *idx, int64_t batch, int32_t dim, const float *d1,
                      float c1, const float *d2, float c2, const float *gscale, float scale, float *g_out, int64_t g_stride,
                      void *stream);

/* ------------------------------------------------------------------------------------------
 * a7  HCCF's hyper-graph branch (hccf.py:43-49 + HGNNLayer :100-108) and its autograd backward without library GEMMs.
 * All products are skinny (n rows x {dim, hyper_num} <= 128), so two kernel shapes cover them:
 * ssl_rowgemm   out[r, :n_out] (+)= leaky( scale * ( in1[r, :k1] M1 + in2[r, :k2] M2 ), slope )     row-local
 *     M1 [k1, n_out] row-major (m1_trans: given as [n_out, k1]); the second product is optional (in2 = NULL);
 *     pre_ref: in1[r, j] is multiplied by act'(pre_ref[r, j]) = (pre_ref > 0 ? 1 : pre_slope) while it is loaded
 *     (dZ = dY * act'(Y): with slope >= 0 LeakyReLU keeps the sign, so the saved OUTPUT tells the derivative; a negative
 *     slope maps both branches to Y > 0 and would need the pre-activation, so engine.hyper_layer rejects it);
 *     slope = 1: no activation.
 *     replaces  E_side @ W * mult (:43-44), adj @ hids (:106) and, in the backward, dZ @ lat^T + X @ dlat^T, H @ dlat, dA @ W^T.
 * ssl_colgemm   out[k1, k2] = post( scale * sum_r in1[r, :k1]^T (x) in2[r, :k2] )                   reduction over rows
 *     per-CTA partials part[ssl_colgemm_parts(n_rows), k1, k2] are reduced in a fixed order (bit-reproducible);
 *     pre_ref acts on in2 as above; mode 0: out_act (optional) = leaky(out); mode 1: out *= act'(ref).
 *     replaces  adj.T @ embeds (:105) and, in the backward, H^T dZ and E^T dA.
 * ssl_hyper_dropout  F.dropout(A, p = 1 - keep) (:48-49): out = x * m / keep (accumulate: out += ..., the backward);
 *     mode 1: m = floor(U + keep) from the in-kernel counter-based generator keyed (seed, stream_id; row, 4-column group);
 *     mode 2: m = mask [n, h] fp32 of 0 / 1 (injected draws).
 * n_rows = 0 (n = 0) is accepted with null row pointers (in1, in2, pre_ref, out; x, out, mask), as torch gives for an empty
 *     side: ssl_rowgemm and ssl_hyper_dropout write nothing, ssl_colgemm writes out = 0 and out_act = leaky(0) = 0.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_rowgemm(const float *in1, int64_t in1_stride, int32_t k1, const float *m1, int32_t m1_trans, const float *in2,
                int64_t in2_stride, int32_t k2, const float *m2, int32_t m2_trans, const float *pre_ref, int64_t pre_stride,
                float pre_slope, float *out, int64_t out_stride, int32_t n_out, float scale, float slope, int32_t accumulate, int64_t n_rows,
                void *stream);
SSL_API int ssl_colgemm_parts(int64_t n_rows);
SSL_API int ssl_colgemm(const float *in1, int64_t in1_stride, int32_t k1, const float *in2, int64_t in2_stride, int32_t k2,
                const float *pre_ref, int64_t pre_stride, float slope, int64_t n_rows, float *part, float scale, int32_t mode,
                const float *ref, float *out, float *out_act, void *stream);
SSL_API int ssl_hyper_dropout(const float *x, float *out, int64_t n, int32_t h, float keep, int32_t mode, const float *mask, uint64_t seed,
                      uint32_t stream_id, int32_t accumulate, void *stream);
/* seed read from the device (CUDA-graph replay, see ssl_prop_args.seed_ptr) */
SSL_API int ssl_hyper_dropout_dev(const float *x, float *out, int64_t n, int32_t h, float keep, int32_t mode, const float *mask,
                          const uint64_t *seed_ptr, uint32_t stream_id, int32_t accumulate, void *stream);

/* ------------------------------------------------------------------------------------------
 * a17  KMeansClustering (aug_utils.py:142-157, NCL): one Lloyd iteration = assignment
 *   idx[r] = argmin_k sum_j (x_rj - c_kj)^2 (ties -> lowest k) and the centroid update
 *   c_k = sum_{idx[r]=k} x_r / (count_k + 1e-6), in place.  Deterministic (static row partition,
 *   ordered partial sums, no floating-point atomics).  ssl_kmeans_workspace gives the launch
 *   shape: part_sum must hold n_cta * k * dim floats and part_cnt n_cta * k.  *changed is
 *   incremented by the number of rows whose assignment changed (initialise assign to -1).
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_kmeans_workspace(int64_t n, int32_t dim, int32_t k, int32_t *n_cta, int32_t *n_warps);
SSL_API int ssl_kmeans_iter(const float *x, int64_t stride, int64_t n, int32_t dim, int32_t k, float *centroids, int64_t *assign,
                    float *part_sum, float *part_cnt, float *counts, int32_t *changed, void *stream);

/* ------------------------------------------------------------------------------------------
 * a21  PairwiseTrnData.sample_negs (datasets_general_cf.py:13-26): negs[e] = an item drawn uniformly
 *   until users[e] has no training interaction with it (membership by binary search in the sorted
 *   training CSR, int32).  Counter-based: a pure function of (seed, epoch, e).
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_sample_negs(const int64_t *users, int64_t n_pairs, const int32_t *trn_rowptr, const int32_t *trn_cols,
                    int64_t n_item, uint64_t seed, uint32_t epoch, int64_t *negs, void *stream);

/* ------------------------------------------------------------------------------------------
 * a22  Ordered scatter of batch rows into a gradient sink (optional key train.deterministic): the
 *   backward of the batch-row gathers of loss_utils.py:7-10 (BPR), :30-51 (InfoNCE rows) and :75-86
 *   (alignment / uniformity), and of the torch indexing users[ancs] / items[poss] / items[negs] of
 *   hccf.py:94 and users[ancs], G_u[ancs], G_i[poss] of lightgcl.py:117-121, in a fixed order.
 *   stage [n_pos, dim] contiguous: row p = the contribution of batch position p; ids [n_pos] the sink
 *   row of each position (a negative id: the position is skipped); order [n_pos] the stable ascending
 *   argsort of ids.  For every row r addressed by some position p1 < p2 < ... (in position order):
 *     sink[r * stride + k] = sink[r * stride + k] + (((c_p1[k] + c_p2[k]) + c_p3[k]) + ...)
 *   with plain fp32 adds, each sink row read and written once (no atomics): bit-reproducible
 *   (csrc/ordered_scatter.cuh).  stride >= dim (a view of an interleaved [N, V, dim] sink has stride V * dim);
 *   n_pos = 0 is a no-op (stage, ids and order may then be NULL).
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_scatter_rows_ordered(const float *stage, const int64_t *ids, const int64_t *order, int64_t n_pos, int32_t dim,
                             float *sink, int64_t stride, void *stream);

/* ------------------------------------------------------------------------------------------
 * a24  (no counterpart: dynamic negative sampling, optional key train.dns_candidates = M)
 *   ssl_neg_candidates: cands [n_pairs, M] int64.  cands[b, 0] = negs[b]; cands[b, j >= 1] an item
 *   drawn uniformly until users[b] has no training interaction with it, with ssl_sample_negs's
 *   rejection rule and 64-block cap on Philox4x32-10 blocks keyed (seed; b, j, block, "DNSC").  The
 *   seed is *seed_ptr when seed_ptr is non-null (CUDA-graph replay), else seed.  2 <= M <= 256.
 *   ssl_neg_select: negs_out[b] = cands[b, j*], j* the candidate with the largest score
 *   s_j = U[ancs[b]] . I[cands[b, j]], each one sequential fp32 FMA chain over k = 0 .. dim-1; ties
 *   go to the lowest j, a NaN score never wins, all NaN gives j* = 0 (csrc/hard_negs.cuh).  Rows are
 *   u_tbl + id * u_stride and i_tbl + id * i_stride (elements; i_tbl is item 0's row).  One writer
 *   per output, no atomics.  dim <= SSL_MAX_DIM, 2 <= M <= 256.  n_pairs = 0 is a no-op for both.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_neg_candidates(const int64_t *users, const int64_t *negs, int64_t n_pairs, int32_t M, const int32_t *trn_rowptr,
                               const int32_t *trn_cols, int64_t n_item, uint64_t seed, const uint64_t *seed_ptr, int64_t *cands,
                               void *stream);
SSL_API int ssl_neg_select(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                           const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, int64_t *negs_out, void *stream);

/* ------------------------------------------------------------------------------------------
 * a25  (no counterpart: MixGCF negatives, Huang et al. KDD 2021, optional key train.mixgcf)
 *   ssl_mixgcf_bpr_fwd, for every pair b with u = U[ancs[b]], pbar = I[poss[b]] (rows of the summed
 *   table the BPR term reads), X_l the item rows of layer l = 0 .. n_layers-1 (layer 0 = E0) and
 *   candidates c_j = cands[b, j], j < M:
 *     alpha_l = u01(Philox4x32-10(ctr (b, l, 0, "MIXA"), key seed_key(seed)).x), or alpha_in[b, l]
 *     m_jl[k] = fmaf(alpha_l, X_l[p][k], (1 - alpha_l) * X_l[c_j][k])          (1 - alpha_l in fp32)
 *     s_jl    = one sequential fp32 FMA chain over k of u[k] * m_jl[k]
 *     j*_l    = argmax_j s_jl: lowest j on ties, NaN never wins, all NaN -> 0 (ssl_neg_select's rule)
 *     nhat    = ((m_{j*_0,0} + m_{j*_1,1}) + m_{j*_2,2}) + ...                  (sum pooling, layer order)
 *     z       = chain(u . nhat) - chain(u . pbar);  loss_b = softplus(z) (threshold-20 tail),
 *     coef_b  = sigmoid(z);  picks[b, l] = c_{j*_l};  alpha_out[b, l] = alpha_l;  nhat [n_pairs, dim].
 *   The seed is *seed_ptr when seed_ptr is non-null (CUDA-graph replay), else seed.  layer_tbls /
 *   layer_strides are HOST arrays of n_layers entries (item 0's row, row stride in elements).
 *   ssl_mixgcf_bpr_bwd, g = scale * (*gscale) * coef_b[b], gu = g * u (atomicAdd):
 *     g_users[ancs[b]] += g (nhat - pbar);   g_items[poss[b]] += -gu;
 *     g_layers[l][poss[b]] += alpha_l gu;    g_layers[l][picks[b, l]] += (1 - alpha_l) gu
 *   (g_layers / gl_strides host arrays).  Identity ids into -0.0 stages give the per-position
 *   contributions train.deterministic scatters in order; the numbering is in csrc/mixgcf.cuh.
 *   1 <= M <= 256, 1 <= n_layers <= 8, dim <= SSL_MAX_DIM; n_pairs = 0 is a no-op for both.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_mixgcf_bpr_fwd(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride,
                               const float *const *layer_tbls, const int64_t *layer_strides, int32_t n_layers, const int64_t *ancs,
                               const int64_t *poss, const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, uint64_t seed,
                               const uint64_t *seed_ptr, const float *alpha_in, float *loss_b, float *coef_b, int64_t *picks,
                               float *alpha_out, float *nhat, void *stream);
SSL_API int ssl_mixgcf_bpr_bwd(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                               const int64_t *poss, const int64_t *picks, int64_t n_pairs, int32_t n_layers, int32_t dim,
                               const float *nhat, const float *alpha, const float *coef_b, const float *gscale, float scale,
                               float *g_users, int64_t gu_stride, float *g_items, int64_t gi_stride, float *const *g_layers,
                               const int64_t *gl_strides, void *stream);

/* ------------------------------------------------------------------------------------------
 * a26  (no counterpart: sampled softmax loss, Wu et al. TOIS 2023, optional key
 *   train.ssm_temperature = tau; the reference's data handler leaves room for a non-pairwise
 *   loss, data_handler_general_cf.py:84-88)
 *   ssl_ssm_fwd, for every pair b with u = U[ancs[b]], c_0 = I[poss[b]], c_q = I[cands[b, q-1]]
 *   (q = 1 .. M; column q of every [n_pairs, M+1] array), x^ = x / sqrt(1e-8 + |x|^2) as in the
 *   InfoNCE terms (loss_utils.py:30-39):
 *     s_q    = (u^ . c^_q) / tau;   loss_b = lse_q(s_q) - s_0 (max-shifted, fp32; a NaN score makes
 *              loss_b NaN);   w_q = softmax(s)_q - [q = 0];   nrm[b] = (n_u, n_0 .. n_M)
 *   in the fp32 order of csrc/ssm.cuh: per float4 slot a 4-term FMA chain, the slots summed by a
 *   fixed xor-butterfly tree, s_q = dot / ((n_u * n_q) * tau), the exp sum per lane over
 *   q = t (mod G) then the same tree.  Outputs loss_b [n_pairs], s, w [n_pairs, M+1], nrm [n_pairs, M+2].
 *   ssl_ssm_bwd, g = scale * (*gscale) (gscale may be NULL), with float atomics:
 *     g_items[c_q] += g w_q (u^ / tau - s_q c^_q) / n_q        (each q as it comes)
 *     g_users[ancs[b]] += g sum_q w_q (c^_q / tau - s_q u^) / n_u  (summed in q order, added once)
 *   Duplicate candidates are separate terms adding into one row (no de-duplication; the logQ
 *   correction of popularity-drawn candidates is ssl_ssm_fwd_logq, a27).  Identity ids into -0.0 stages give the per-position
 *   contributions train.deterministic scatters in order; the numbering is in csrc/ssm.cuh.
 *   1 <= M <= 256; dim a multiple of 4, <= SSL_MAX_DIM; tau finite and > 0; every table and sink
 *   16-byte aligned with a stride (elements) that is a multiple of 4 and >= dim.  n_pairs = 0 is
 *   a no-op for both; rejected arguments write nothing.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_ssm_fwd(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                        const int64_t *poss, const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, float tau, float *loss_b,
                        float *s, float *w, float *nrm, void *stream);
SSL_API int ssl_ssm_bwd(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                        const int64_t *poss, const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, float tau, const float *s,
                        const float *w, const float *nrm, const float *gscale, float scale, float *g_users, int64_t gu_stride,
                        float *g_items, int64_t gi_stride, void *stream);

/* ------------------------------------------------------------------------------------------
 * a27  (no counterpart: popularity-proportional negative candidates with the logQ-corrected
 *   sampled softmax, optional key train.neg_popularity = beta with train.dns_candidates = M >= 2)
 *   Host tables (engine.pop_tables, float64 then fp32 once): w_i = (deg_i + 1)^beta, deg_i the
 *   count of item i in the training CSR's columns; V_i >= 1 the largest-remainder rounding of
 *   n_item 2^32 w_i / sum w (sum V = n_item 2^32 exactly); table [n_item] uint2 {thr, alias}, the
 *   Walker / Vose alias table of V in exact integers (column capacity 2^32; a column its own item
 *   fills alone has alias = itself); lp[i] = log(V_i / (n_item 2^32));
 *   lz_pop[u] = log(1 - sum_{i in P_u} V_i / (n_item 2^32)) (the subtraction in integers);
 *   lz_uni[u] = log(n_item - deg_u); both 0 for a user who has every item; ln_m = fp32(log M).
 *   ssl_neg_candidates_pop: cands [n_pairs, M] int64.  cands[b, 0] = negs[b]; cands[b, j >= 1]
 *   from the Philox4x32-10 blocks keyed (seed; b, j, blk, "DNSP"), blk < 64, two draws
 *   (x, y) = (r.x, r.y), (r.z, r.w) per block: c = (x * n_item) >> 32; item = c if alias[c] == c
 *   or y < thr[c], else alias[c]; rejected while in users[b]'s sorted training-CSR row; after 128
 *   draws the last is kept.  bias (nullable) [n_pairs, M] fp32, in this order:
 *     bias[b, 0] = ln_m - lz_uni[u]          bias[b, j] = (ln_m + lp[cands[b, j]]) - lz_pop[u]
 *   = ln(M q_j(c_j)), q_j candidate j's proposal restricted to u's non-positives, so
 *   sum_{q >= 1} exp(s_q - bias[b, q-1]) estimates sum_{i not in P_u} exp(s_i) without bias
 *   (ignoring the 128-draw cap).  The seed is *seed_ptr when seed_ptr is non-null, else seed.
 *   2 <= M <= 256; table 8-byte aligned; lp, lz_pop, lz_uni may be NULL when bias is.
 *   ssl_ssm_fwd_logq: ssl_ssm_fwd on s^_0 = s_0, s^_q = s_q - bias[b, q-1] (q >= 1, one fp32
 *   subtraction): m, S, loss_b = (m + logf(S)) - s^_0 and w in ssl_ssm_fwd's order on s^; s is
 *   stored raw, so ssl_ssm_bwd is its backward unchanged (csrc/ssm.cuh).  Arguments and checks as
 *   ssl_ssm_fwd, bias [n_pairs, M] non-null.  n_pairs = 0 is a no-op for both; rejected
 *   arguments write nothing.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_neg_candidates_pop(const int64_t *users, const int64_t *negs, int64_t n_pairs, int32_t M, const int32_t *trn_rowptr,
                                   const int32_t *trn_cols, int64_t n_item, const uint32_t *table, const float *lp,
                                   const float *lz_pop, const float *lz_uni, float ln_m, uint64_t seed, const uint64_t *seed_ptr,
                                   int64_t *cands, float *bias, void *stream);
SSL_API int ssl_ssm_fwd_logq(const float *u_tbl, int64_t u_stride, const float *i_tbl, int64_t i_stride, const int64_t *ancs,
                             const int64_t *poss, const int64_t *cands, int64_t n_pairs, int32_t M, int32_t dim, float tau,
                             float *loss_b, float *s, float *w, float *nrm, const float *bias, void *stream);

/* ------------------------------------------------------------------------------------------
 * a28  (no counterpart: in-batch negatives for the sampled softmax, mixed negative sampling of
 *   Yang et al. WWW 2020 with the logQ correction of Yi et al. RecSys 2019; optional key
 *   train.ssm_in_batch with train.ssm_temperature = tau)
 *   For every pair b with u = U[ancs[b]] and the 2B columns id_c = poss[c] (c < B), negs[c - B]
 *   (B <= c < 2B), shared by every pair, duplicates kept, x^ = x / sqrt(1e-8 + |x|^2):
 *     s_bc = (u^ . i^_{id_c}) / tau;   w_c = v[id_c] / B (fp32 division);
 *     loss_b = ln(sum_c w_c exp(s_bc)) - s_bb
 *   v [n_item] fp32 (engine.in_batch_weights, float64 then fp32 once): v_i = 1 / (p_i + r_i), 0
 *   when p_i + r_i = 0, with p_i = deg_i / |E| and r_i = sum_u (deg_u / |E|) [i not in P_u] /
 *   (n_item - deg_u): the probability that one positive / negative slot of the loaders holds i.
 *   The term is the InfoNCE pieces of a13/a14, no new forward:
 *     ssl_rows_normalize[_f16x3] (norm_mode 0) of U[ancs] scaled by log2(e) / tau and of the
 *       columns at alpha 1, both with the copies of either role; rows 0 .. B-1 of the column
 *       operand are the positives' p^;
 *     the contraction of users against columns with colscale = w, offset log2(e) / tau, row sums:
 *       rowsum_b = sum_c w_c exp(s_bc - 1/tau);
 *     ssl_nce_finalize with deno_eps 0: loss_b = -(u^ . p^_b)/tau + 1/tau + ln(rowsum_b);
 *     backward: ssl_nce_bwd_rows (user rows by ancs, positive rows by poss), ssl_nce_colscale,
 *       the swapped contraction (R = columns, C = users) and ssl_nce_bwd_cols.
 *   The 3xFP16 kernel serves the weighted forward only when its E' = exp2(S - offset) w_c 2^14 / M
 *   (M = 2^e >= max w, so w_c / M > 2^-1 min w / max w) cannot fall below the flush threshold
 *   2^-14: E' >= 2^(13 - 2 offset) min w / max w >= 2^-13 needs offset + (1 + log2(max w / min w)) / 2
 *   <= 13.5 (csrc/f16x3.cuh's kF16NoFlushOffset).  Past it an E' below 2^-14 is carried by its lo
 *   part alone, at 2^-11 relative instead of 2^-22, and a row whose sum is made of such entries
 *   (every cosine low against popular, low-weight columns; at tau = 0.1 the offset alone is
 *   14.4) gets its loss and softmax weights at 2^-11: not fp32 grade.  The engine then takes
 *   3xTF32 (engine.contraction_kind, from the weight table's range, known on the host).
 *   Every kernel forms a term as ex2(S - offset) * w_c, and ex2 is ex2.approx.ftz: a result below
 *   2^-126 is 0.  S - offset = log2(e) (cos - 1) / tau >= -2 log2(e) / tau and w_c >= min v / B
 *   (min over v > 0), so both ex2(S - offset) and the term are normal fp32 numbers when
 *     2 log2(e) / tau + max(0, log2(B / min v)) <= 126.
 *   Past it a row whose columns all sit near cos = -1 has rowsum 0 (loss -inf, colscale inf, then
 *   NaN), and a row whose largest term is small loses its terms below the flush: its rowsum is
 *   not fp32 grade.  engine.ssm_in_batch_sum refuses such a (B, tau, min v) with ValueError, on
 *   the host, at 125 rather than 126: one binade for the rounding of S - offset, so a column
 *   exactly opposite its row is not flushed by an ulp.  At B = 4096 and min v = 1 the smallest
 *   tau is 0.0256; the sampled softmax's tau = 0.1 spans 40.9 binades.
 *   ssl_nce_bwd_cols: the column gradient.  For c < n (= 2B), in the fp32 order of
 *   csrc/ssm_in_batch.cuh:  d = (sum_s dt_part[s, c]) * colw[c];
 *     sink[ids[c]] += rinv_c (d - t^_c (t^_c . d))   (float atomics; ids NULL: row c, into a -0.0
 *   stage whose rows train.deterministic scatters in order).  t_hat [n, dim] row-major, rinv [n],
 *   colw [n], dt_part [n_split, n, dim].  dim <= SSL_MAX_DIM, stride >= dim, n_split >= 1; n = 0 is
 *   a no-op; rejected arguments write nothing.
 * ------------------------------------------------------------------------------------------ */
SSL_API int ssl_nce_bwd_cols(const float *dt_part, int32_t n_split, const float *t_hat, const float *rinv, const float *colw,
                             const int64_t *ids, int64_t n, int32_t dim, float *sink, int64_t stride, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* SSLREC_B200_H */
