"""ctypes binding of ``libsslrec_b200.so`` (C ABI declared in ``include/sslrec_b200.h``).

The library is the product: if it is missing or cannot be loaded this module raises -- there is
no CPU or eager-PyTorch fallback anywhere in the package.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'lib', 'libsslrec_b200.so')

MAX_VIEWS = 4
MAX_CANDIDATES = 256
MAX_SUM_SRC = 6
MAX_DIM = 128
MAX_PEERS = 7

c_f32p = C.POINTER(C.c_float)
c_i32p = C.POINTER(C.c_int32)
c_i64p = C.POINTER(C.c_int64)
c_u8p = C.POINTER(C.c_uint8)
vp = C.c_void_p


class PropArgs(C.Structure):
    """Mirror of ``ssl_prop_args`` (include/sslrec_b200.h)."""
    _fields_ = [
        ('dim', C.c_int32), ('n_views', C.c_int32), ('in_views', C.c_int32), ('transpose', C.c_int32),
        ('x_in', vp), ('x_out', vp), ('sum_out', vp), ('residual', vp),
        ('reduce_views', C.c_int32), ('n_sum_src', C.c_int32),
        ('sum_src', vp * MAX_SUM_SRC), ('sum_src_views', C.c_int32 * MAX_SUM_SRC),
        ('reg_coef', C.c_float), ('reg_src', vp),
        ('edge_mode', C.c_int32 * MAX_VIEWS), ('edge_keep', C.c_float * MAX_VIEWS),
        ('edge_scale', C.c_float * MAX_VIEWS), ('edge_mask', vp * MAX_VIEWS),
        ('noise_mode', C.c_int32 * MAX_VIEWS), ('noise_u', vp * MAX_VIEWS),
        ('noise_eps', C.c_float), ('seed', C.c_uint64 * MAX_VIEWS),
        ('edge_stream_id', C.c_uint32), ('noise_stream_id', C.c_uint32),
        ('n_peers', C.c_int32), ('x_out_peers', vp * MAX_PEERS), ('sum_out_peers', vp * MAX_PEERS),
        ('reg_coef_dev', vp), ('reg_src2', vp), ('seed_ptr', vp * MAX_VIEWS), ('row_bits', vp * MAX_VIEWS),
    ]


class LibraryMissing(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(
            f'{LIB_PATH} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
            '(or `make -C sslrec_b200/csrc`). sslrec_b200 has no CPU fallback.')
    lib = C.CDLL(LIB_PATH)
    i32, i64, f32 = C.c_int32, C.c_int64, C.c_float
    sig = {
        'ssl_version': (C.c_int, []),
        'ssl_last_error': (C.c_char_p, []),
        'ssl_launch_count': (i64, []),
        'ssl_plan_create': (C.c_int, [C.POINTER(vp), vp, vp, vp, vp, i64, i64, i64, i64, i64, vp]),
        'ssl_plan_create_ranges': (C.c_int, [C.POINTER(vp), vp, vp, vp, vp, i64, i64, i64, i64, i64, i64, i64, i64, vp]),
        'ssl_set_option': (C.c_int, [C.c_char_p, i64]),
        'ssl_plan_destroy': (C.c_int, [vp]),
        'ssl_plan_stats': (C.c_int, [vp, c_i64p]),
        'ssl_propagate_layer': (C.c_int, [vp, C.POINTER(PropArgs), vp]),
        'ssl_node_drop': (C.c_int, [vp, vp, i64, i32, i32, i32, c_i32p, c_f32p, C.POINTER(vp), C.POINTER(C.c_uint64), i64, vp]),
        'ssl_node_drop_dev': (C.c_int, [vp, vp, i64, i32, i32, i32, c_i32p, c_f32p, C.POINTER(vp), C.POINTER(C.c_uint64), C.POINTER(vp), i64, vp]),
        'ssl_bpr_fwd': (C.c_int, [vp, i64, vp, i64, vp, vp, vp, i64, i32, vp, vp, vp]),
        'ssl_bpr_bwd': (C.c_int, [vp, i64, vp, i64, vp, vp, vp, i64, i32, vp, vp, f32, vp, i64, vp, i64, vp]),
        'ssl_rows_normalize': (C.c_int, [vp, i64, vp, i64, i32, i32, f32, vp, vp, vp, vp, vp, vp, vp, i64, vp]),
        'ssl_softmax_gemm_tf32x3': (C.c_int, [vp, vp, i64, vp, vp, vp, vp, i64, i64, i32, vp, f32, i32, vp, vp, vp]),
        'ssl_rows_normalize_f16x3': (C.c_int, [vp, i64, vp, i64, i32, i32, f32, vp, vp, vp, vp, vp]),
        'ssl_softmax_gemm_f16x3': (C.c_int, [vp, vp, i64, vp, vp, i64, i32, vp, f32, i32, vp, vp, vp]),
        'ssl_softmax_gemm_f16x3_live': (C.c_int, [vp, vp, i64, vp, vp, i64, i32, vp, f32, i32, vp, vp, vp, i32, vp]),
        'ssl_softmax_gemm': (C.c_int, [vp, i64, vp, vp, i64, i32, vp, f32, i32, vp, vp, vp]),
        'ssl_nce_finalize': (C.c_int, [vp, vp, i32, i64, i32, vp, vp, f32, f32, vp, vp, vp, vp]),
        'ssl_lse_finalize': (C.c_int, [vp, vp, i32, i64, i32, f32, vp, vp, vp, vp]),
        'ssl_nce_bwd_rows': (C.c_int, [vp, vp, vp, vp, vp, vp, i64, i32, f32, vp, f32, vp, i64, vp, i64, vp]),
        'ssl_nce_bwd_table': (C.c_int, [vp, i32, vp, vp, i64, i32, vp, i64, i32, vp]),
        'ssl_nce_colscale': (C.c_int, [vp, i64, vp, f32, vp, vp]),
        'ssl_softmax_gemm_live': (C.c_int, [vp, i64, vp, vp, i64, i32, vp, f32, i32, vp, vp, vp, i32, vp]),
        'ssl_softmax_gemm_tf32x3_live': (C.c_int, [vp, vp, i64, vp, vp, vp, vp, i64, i64, i32, vp, f32, i32, vp, vp, vp, i32, vp]),
        'ssl_sum_live': (C.c_int, [vp, i64, vp, f32, vp, vp]),
        'ssl_nce_bwd_rows_live': (C.c_int, [vp, vp, vp, vp, vp, vp, i64, vp, i32, f32, vp, f32, vp, i64, vp, i64, vp]),
        'ssl_nce_colscale_live': (C.c_int, [vp, i64, vp, vp, f32, vp, vp]),
        'ssl_unique_ids_scratch': (C.c_int, [i64, c_i64p]),
        'ssl_unique_ids': (C.c_int, [vp, i64, i64, vp, i64, vp, vp, vp]),
        'ssl_row_bitmap': (C.c_int, [vp, i64, i64, vp, i64, vp]),
        'ssl_sumsq': (C.c_int, [vp, i64, vp, vp]),
        'ssl_sum': (C.c_int, [vp, i64, f32, vp, vp]),
        'ssl_axpy': (C.c_int, [vp, vp, i64, vp, f32, vp]),
        'ssl_adam_step': (C.c_int, [vp, vp, vp, vp, i64, i64, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, vp]),
        'ssl_adam_step_peers': (C.c_int, [vp, C.POINTER(vp), i32, vp, vp, vp, i64, i64, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, vp]),
        'ssl_rowgemm': (C.c_int, [vp, i64, i32, vp, i32, vp, i64, i32, vp, i32, vp, i64, f32, vp, i64, i32, f32, f32, i32, i64, vp]),
        'ssl_colgemm_parts': (C.c_int, [i64]),
        'ssl_colgemm': (C.c_int, [vp, i64, i32, vp, i64, i32, vp, i64, f32, i64, vp, f32, i32, vp, vp, vp, vp]),
        'ssl_hyper_dropout': (C.c_int, [vp, vp, i64, i32, f32, i32, vp, C.c_uint64, C.c_uint32, i32, vp]),
        'ssl_adam_step_dev': (C.c_int, [vp, C.POINTER(vp), i32, vp, vp, vp, i64, vp, vp, C.c_double, C.c_double, C.c_double, C.c_double, C.c_double, vp]),
        'ssl_hyper_dropout_dev': (C.c_int, [vp, vp, i64, i32, f32, i32, vp, vp, C.c_uint32, i32, vp]),
        'ssl_predict_mask': (C.c_int, [vp, i64, vp, i64, vp, i64, i64, i32, vp, vp, vp, vp, vp]),
        'ssl_topk': (C.c_int, [vp, i64, i64, i32, vp, vp, vp]),
        'ssl_predict_topk_workspace': (C.c_int, [i64, i64, i32, c_i64p]),
        'ssl_predict_topk': (C.c_int, [vp, i64, vp, i64, vp, i64, i64, i32, vp, vp, vp, i32, vp, i64, vp, vp, vp]),
        'ssl_spmm_exact': (C.c_int, [vp, vp, vp, i64, vp, i64, i32, vp, i64, vp]),
        'ssl_align_fwd': (C.c_int, [vp, vp, i64, i32, vp, vp]),
        'ssl_uniform_finalize': (C.c_int, [vp, vp, i32, i64, i32, vp, vp, f32, vp, vp, vp]),
        'ssl_uniform_pairs': (C.c_int, [vp, i64, i32, vp, vp, vp]),
        'ssl_unit_rows_bwd': (C.c_int, [vp, vp, vp, i64, i32, vp, f32, vp, f32, vp, f32, vp, i64, vp]),
        'ssl_kmeans_workspace': (C.c_int, [i64, i32, i32, c_i32p, c_i32p]),
        'ssl_kmeans_iter': (C.c_int, [vp, i64, i64, i32, i32, vp, vp, vp, vp, vp, vp, vp]),
        'ssl_sample_negs': (C.c_int, [vp, i64, vp, vp, i64, C.c_uint64, C.c_uint32, vp, vp]),
        'ssl_scatter_rows_ordered': (C.c_int, [vp, vp, vp, i64, i32, vp, i64, vp]),
        'ssl_neg_candidates': (C.c_int, [vp, vp, i64, i32, vp, vp, i64, C.c_uint64, vp, vp, vp]),
        'ssl_neg_select': (C.c_int, [vp, i64, vp, i64, vp, vp, i64, i32, i32, vp, vp]),
        'ssl_mixgcf_bpr_fwd': (C.c_int, [vp, i64, vp, i64, C.POINTER(vp), c_i64p, i32, vp, vp, vp, i64, i32, i32, C.c_uint64, vp, vp,
                                         vp, vp, vp, vp, vp, vp]),
        'ssl_mixgcf_bpr_bwd': (C.c_int, [vp, i64, vp, i64, vp, vp, vp, i64, i32, i32, vp, vp, vp, vp, f32, vp, i64, vp, i64,
                                         C.POINTER(vp), c_i64p, vp]),
        'ssl_ssm_fwd': (C.c_int, [vp, i64, vp, i64, vp, vp, vp, i64, i32, i32, f32, vp, vp, vp, vp, vp]),
        'ssl_ssm_bwd': (C.c_int, [vp, i64, vp, i64, vp, vp, vp, i64, i32, i32, f32, vp, vp, vp, vp, f32, vp, i64, vp, i64, vp]),
        'ssl_neg_candidates_pop': (C.c_int, [vp, vp, i64, i32, vp, vp, i64, vp, vp, vp, vp, f32, C.c_uint64, vp, vp, vp, vp]),
        'ssl_ssm_fwd_logq': (C.c_int, [vp, i64, vp, i64, vp, vp, vp, i64, i32, i32, f32, vp, vp, vp, vp, vp, vp]),
        'ssl_nce_bwd_cols': (C.c_int, [vp, i32, vp, vp, vp, vp, i64, i32, vp, i64, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)          # AttributeError here = the .so does not export what the header declares
        fn.restype = res
        fn.argtypes = args
    return lib, tuple(sig)


lib, EXPORTS = _load()


class SslError(RuntimeError):
    pass


def check(rc: int, what: str = '') -> None:
    if rc != 0:
        msg = lib.ssl_last_error()
        raise SslError(f'{what or "sslrec_b200"} failed (code {rc}): {msg.decode() if msg else "?"}')


def launch_count() -> int:
    return int(lib.ssl_launch_count())
