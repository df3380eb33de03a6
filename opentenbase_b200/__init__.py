"""opentenbase_b200 — H100-native (sm_90a) executor hot path for OpenTenBase.

The product is ``libgpuexec.so`` (hand-written CUDA behind the C ABI of
``include/gpuexec.h``) plus the C CustomScan provider under ``provider/``.
This module is only the ctypes binding that tests and ``bench.py`` drive the
C ABI through.  There is no CPU fallback: if the library cannot be loaded, or
no GPU is present, every call fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgpuexec.so")
INCLUDE_DIR = os.path.join(os.path.dirname(_HERE), "include")

# --- enums of include/gpuexec.h ---------------------------------------------
GX_OK, GX_ERR_CUDA, GX_ERR_ARG, GX_ERR_NOMEM, GX_ERR_NCCL, GX_ERR_STATE, GX_ERR_OVERFLOW, GX_ERR_NODEVICE = range(8)
GX_INT4, GX_INT8, GX_FLOAT8, GX_DATE, GX_CHAR = 1, 2, 3, 4, 5
GX_LT, GX_LE, GX_EQ, GX_GE, GX_GT, GX_NE = 1, 2, 3, 4, 5, 6
(GX_AGG_COUNT_STAR, GX_AGG_COUNT, GX_AGG_SUM_F8, GX_AGG_AVG_F8, GX_AGG_SUM_I4,
 GX_AGG_MIN_F8, GX_AGG_MAX_F8, GX_AGG_SUM_I8, GX_AGG_COUNT_DISTINCT) = 1, 2, 3, 4, 5, 6, 7, 8, 9
(GX_AGG_VAR_POP_F8, GX_AGG_VAR_SAMP_F8, GX_AGG_STDDEV_POP_F8, GX_AGG_STDDEV_SAMP_F8) = 10, 11, 12, 13
(GX_AGG_REGR_COUNT, GX_AGG_REGR_SXX_F8, GX_AGG_REGR_SYY_F8, GX_AGG_REGR_SXY_F8, GX_AGG_REGR_AVGX_F8,
 GX_AGG_REGR_AVGY_F8, GX_AGG_REGR_R2_F8, GX_AGG_REGR_SLOPE_F8, GX_AGG_REGR_INTERCEPT_F8, GX_AGG_COVAR_POP_F8,
 GX_AGG_COVAR_SAMP_F8, GX_AGG_CORR_F8) = range(14, 26)
GX_OP_COL, GX_OP_CONST, GX_OP_ADD, GX_OP_SUB, GX_OP_MUL, GX_OP_ARG2 = 1, 2, 3, 4, 5, 6
GX_JOIN_INNER, GX_JOIN_LEFT, GX_JOIN_SEMI, GX_JOIN_ANTI = 0, 1, 4, 5
GX_JOIN_SEMI_RIGHT, GX_JOIN_ANTI_RIGHT = 8, 9      # gx_hash_agg_right only: the build side is the preserved relation
T_ORDERS, T_LINEITEM, T_CUSTOMER = 1, 2, 3
# fixed schemas of include/gx_tpch_gen.h
O_ORDERKEY, O_CUSTKEY, O_ORDERDATE, O_SHIPPRIORITY = 0, 1, 2, 3
(L_ORDERKEY, L_QUANTITY, L_EXTENDEDPRICE, L_DISCOUNT, L_TAX, L_SHIPDATE,
 L_RETURNFLAG, L_LINESTATUS) = range(8)
C_CUSTKEY, C_MKTSEGMENT = 0, 1
SCHEMAS = {
    T_ORDERS: [GX_INT8, GX_INT4, GX_DATE, GX_INT4],
    T_LINEITEM: [GX_INT8, GX_FLOAT8, GX_FLOAT8, GX_FLOAT8, GX_FLOAT8, GX_DATE, GX_CHAR, GX_CHAR],
    T_CUSTOMER: [GX_INT4, GX_CHAR],
}
NP_DTYPES = {GX_INT4: np.int32, GX_INT8: np.int64, GX_FLOAT8: np.float64, GX_DATE: np.int32, GX_CHAR: np.int8}


class GxError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(f"libgpuexec status {status}: {msg}")
        self.status = status


class GxPred(C.Structure):
    _fields_ = [("col", C.c_int32), ("op", C.c_int32), ("ival", C.c_int64), ("fval", C.c_double)]


class GxExprOp(C.Structure):
    _fields_ = [("op", C.c_int32), ("col", C.c_int32), ("k", C.c_double)]


class GxExpr(C.Structure):
    _fields_ = [("nops", C.c_int32), ("_pad", C.c_int32), ("ops", GxExprOp * 12)]


class GxAgg(C.Structure):
    _fields_ = [("fn", C.c_int32), ("_pad", C.c_int32), ("arg", GxExpr)]


class GxColRef(C.Structure):
    _fields_ = [("side", C.c_int32), ("col", C.c_int32)]


class GxAggPlan(C.Structure):
    _fields_ = [("n_preds", C.c_int32), ("outer_key_col", C.c_int32),
                ("preds", GxPred * 4),
                ("n_group_cols", C.c_int32), ("n_aggs", C.c_int32),
                ("group_cols", GxColRef * 4),
                ("aggs", GxAgg * 8),
                ("est_groups", C.c_int64),
                ("strategy", C.c_int32), ("join_type", C.c_int32)]


class GxJoinStep(C.Structure):
    _fields_ = [("h", C.c_void_p), ("key", GxColRef), ("join_type", C.c_int32), ("_pad", C.c_int32)]


GX_MAX_JOINS = 3


class GxHeapDesc(C.Structure):
    _fields_ = [("natts", C.c_int32), ("ncols", C.c_int32),
                ("att_len", C.c_int16 * 64), ("att_align", C.c_int8 * 64),
                ("attnums", C.c_int32 * 16), ("att_notnull", C.c_int8 * 64)]


class GxFnPageId(C.Structure):
    """FNQueryId + fragment / node / worker ids that FnPageInit stamps on every page (forward/fnbufpage.h:54-65)"""
    _fields_ = [("qid_timestamp_nodeid", C.c_int64), ("qid_sequence", C.c_int64), ("fid", C.c_uint16), ("nodeid", C.c_uint16),
                ("workerid", C.c_uint16), ("virtualid", C.c_uint8), ("_pad", C.c_uint8)]


class GxHostTable(C.Structure):
    _fields_ = [("ncols", C.c_int32), ("_pad", C.c_int32), ("nrows", C.c_int64),
                ("types", C.POINTER(C.c_int32)), ("cols", C.POINTER(C.c_void_p)),
                ("nulls", C.POINTER(C.c_void_p))]


def build(force: bool = False) -> str:
    """Compile libgpuexec.so for sm_90a with nvcc (cross-compiles without a GPU)."""
    subprocess.check_call(["make", "-C", os.path.join(_HERE, "csrc"), "-s"] + (["-B"] if force else []))
    return LIB_PATH


_lib = None


def lib() -> C.CDLL:
    """Load libgpuexec.so; fails loudly when it is missing (no fallback)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise GxError(-1, f"{LIB_PATH} is missing: run __graft_entry__.build() / make -C opentenbase_b200/csrc")
        _lib = C.CDLL(LIB_PATH)
        _declare(_lib)
    return _lib


def _declare(L):
    vp, i32, i64, dbl, sz = C.c_void_p, C.c_int32, C.c_int64, C.c_double, C.c_size_t
    pp = C.POINTER(vp)
    sig = {
        "gx_abi_version": (C.c_int, []),
        "gx_init": (C.c_int, [C.c_int, pp]),
        "gx_shutdown": (None, [vp]),
        "gx_last_error": (C.c_char_p, [vp]),
        "gx_device_info": (C.c_int, [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(i64)]),
        "gx_sync": (C.c_int, [vp]),
        "gx_pool_reserve": (C.c_int, [vp, sz]),
        "gx_launch_count": (i64, [vp]),
        "gx_timer_start": (C.c_int, [vp]),
        "gx_timer_stop": (C.c_int, [vp, C.POINTER(dbl)]),
        "gx_profile": (C.c_int, [vp, C.c_int]),
        "gx_profile_get": (C.c_int, [vp, C.c_char_p, C.POINTER(dbl), C.POINTER(i64)]),
        "gx_l2_flush": (C.c_int, [vp]),
        "gx_host_alloc": (C.c_int, [vp, sz, pp]),
        "gx_host_free": (C.c_int, [vp, vp]),
        "gx_h2d_probe": (C.c_int, [vp, vp, sz, C.c_int, C.POINTER(dbl)]),
        "gx_table_create": (C.c_int, [vp, C.c_int, C.POINTER(i32), i64, pp]),
        "gx_table_append_columns": (C.c_int, [vp, pp, pp, i64]),
        "gx_table_append_heap_pages": (C.c_int, [vp, vp, i64, C.POINTER(GxHeapDesc), vp, vp, i32]),
        "gx_stage_acquire": (C.c_int, [vp, sz, pp]),
        "gx_table_reserve": (C.c_int, [vp, i64]),
        "gx_table_load_finish": (C.c_int, [vp]),
        "gx_table_nrows": (i64, [vp]),
        "gx_table_ncols": (C.c_int, [vp]),
        "gx_table_read_column": (C.c_int, [vp, C.c_int, i64, i64, vp, vp]),
        "gx_table_truncate": (C.c_int, [vp]),
        "gx_table_drop_column": (C.c_int, [vp, C.c_int]),
        "gx_table_free": (None, [vp]),
        "gx_table_column_devptr": (C.c_int, [vp, C.c_int, pp]),
        "gx_table_permute": (C.c_int, [vp, vp, i64, pp]),
        "gx_table_generate": (C.c_int, [vp, C.c_int, C.c_int, i64, i64, C.c_int, C.c_int]),
        "gx_table_generate_cols": (C.c_int, [vp, C.c_int, C.c_int, i64, i64, C.c_int, C.c_int, C.POINTER(i32)]),
        "gx_scan_filter": (C.c_int, [vp, vp, C.c_int, C.POINTER(GxPred), C.c_int, C.POINTER(i32), pp]),
        "gx_hash_build": (C.c_int, [vp, vp, C.c_int, C.c_int, C.POINTER(GxPred), C.c_int, C.POINTER(i32), C.c_int, pp]),
        "gx_hash_nentries": (i64, [vp]),
        "gx_hash_nslots": (i64, [vp]),
        "gx_hash_info": (C.c_int, [vp, C.POINTER(C.c_int), C.POINTER(dbl)]),
        "gx_hash_free": (None, [vp]),
        "gx_fnpage_pack": (C.c_int, [vp, vp, C.POINTER(GxHeapDesc), C.POINTER(GxFnPageId), C.c_int, vp, i64, C.POINTER(i64)]),
        "gx_fnpage_unpack": (C.c_int, [vp, vp, i64, C.POINTER(GxHeapDesc), vp, pp]),
        "gx_bloom_build": (C.c_int, [vp, vp, C.c_int, C.c_int, C.POINTER(GxPred), pp]),
        "gx_bloom_log_num_buckets": (C.c_int, [vp]),
        "gx_bloom_read_words": (C.c_int, [vp, vp]),
        "gx_bloom_test": (C.c_int, [vp, vp, vp, C.c_int, vp]),
        "gx_bloom_free": (None, [vp]),
        "gx_hash_probe": (C.c_int, [vp, vp, C.c_int, C.c_int, C.POINTER(GxPred), vp, C.c_int, C.POINTER(i32), pp]),
        "gx_hash_probe_ex": (C.c_int, [vp, vp, C.c_int, C.c_int, C.POINTER(GxPred), vp, C.c_int, C.c_int, C.POINTER(i32), pp]),
        "gx_hash_agg": (C.c_int, [vp, vp, vp, C.POINTER(GxAggPlan), pp]),
        "gx_hash_agg_joins": (C.c_int, [vp, vp, C.c_int, C.POINTER(GxJoinStep), C.POINTER(GxAggPlan), pp]),
        "gx_hash_agg_right": (C.c_int, [vp, vp, C.c_int, C.c_int, C.POINTER(GxPred), vp, vp, C.c_int, C.POINTER(GxAggPlan), pp]),
        "gx_result_combine": (C.c_int, [vp, vp]),
        "gx_result_ngroups": (i64, [vp]),
        "gx_result_fetch": (C.c_int, [vp, i64, vp, vp, vp]),
        "gx_result_fetch_states": (C.c_int, [vp, i64, vp, vp, vp, vp]),
        "gx_result_fetch_sxx": (C.c_int, [vp, i64, vp]),
        "gx_result_fetch_regr": (C.c_int, [vp, i64, vp]),
        "gx_result_free": (None, [vp]),
        "gx_exec_host": (C.c_int, [vp, C.POINTER(GxHostTable), C.POINTER(GxHostTable), C.c_int, C.c_int,
                                   C.POINTER(GxPred), C.c_int, C.POINTER(i32), C.c_int, C.POINTER(GxAggPlan), pp]),
        "gx_comm_unique_id": (C.c_int, [vp]),
        "gx_comm_init": (C.c_int, [vp, C.c_int, C.c_int, vp]),
        "gx_comm_rank": (C.c_int, [vp, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
        "gx_comm_destroy": (None, [vp]),
        "gx_set_shardmap": (C.c_int, [vp, vp, C.c_int]),
        "gx_route": (C.c_int, [vp, vp, C.c_int, vp]),
        "gx_redistribute": (C.c_int, [vp, vp, C.c_int, pp]),
        "gx_partition_by_node": (C.c_int, [vp, vp, C.c_int, pp, vp]),
        "gx_debug_hash": (C.c_int, [vp, C.c_int, vp, i64, vp]),
        "gx_debug_combine": (C.c_int, [vp, C.c_int, pp, C.c_int]),
        "gx_debug_redistribute": (C.c_int, [vp, C.c_int, pp, C.c_int, C.c_int, sz, pp, C.POINTER(C.c_int)]),
    }
    for name, (res, args) in sig.items():
        f = getattr(L, name)
        f.restype = res
        f.argtypes = args


EXPORTED_SYMBOLS = None  # filled lazily by exported_symbols()


def mk_pred(col, op, const, is_float=False) -> GxPred:
    q = GxPred()
    q.col, q.op = col, op
    if is_float:
        q.fval = float(const)
    else:
        q.ival = int(const)
    return q


def make_plan(preds=(), outer_key_col=-1, group_cols=(), aggs=(), est_groups=0, strategy=0, join_type=0) -> GxAggPlan:
    """preds: (col, op, const[, is_float]); group_cols: (side, col);
    aggs: (fn, [(op, col, k), ...])  — postfix argument program."""
    p = GxAggPlan()
    p.n_preds = len(preds)
    p.outer_key_col = outer_key_col
    for i, pr in enumerate(preds):
        p.preds[i] = mk_pred(*pr)
    p.n_group_cols = len(group_cols)
    for i, (side, col) in enumerate(group_cols):
        p.group_cols[i].side, p.group_cols[i].col = side, col
    p.n_aggs = len(aggs)
    for i, (fn, ops) in enumerate(aggs):
        p.aggs[i].fn = fn
        p.aggs[i].arg.nops = len(ops)
        for j, (op, col, k) in enumerate(ops):
            p.aggs[i].arg.ops[j].op, p.aggs[i].arg.ops[j].col, p.aggs[i].arg.ops[j].k = op, col, float(k)
    p.est_groups = est_groups
    p.strategy = strategy
    p.join_type = join_type
    return p


class Table:
    def __init__(self, ctx: "Context", handle, types):
        self.ctx, self.h, self.types = ctx, handle, list(types)

    @property
    def nrows(self):
        return lib().gx_table_nrows(self.h)

    def append(self, cols, nulls=None):
        keep = [np.ascontiguousarray(c, NP_DTYPES[t]) for c, t in zip(cols, self.types)]
        n = len(keep[0]) if keep else 0
        cp = (C.c_void_p * len(keep))(*[c.ctypes.data for c in keep])
        npp = None
        kn = None
        if nulls is not None:
            kn = [None if x is None else np.ascontiguousarray(x, np.uint8) for x in nulls]
            npp = (C.c_void_p * len(kn))(*[None if x is None else x.ctypes.data for x in kn])
        self.ctx._chk(lib().gx_table_append_columns(self.h, cp, npp, n))
        self.ctx.sync()
        return self

    def append_heap_pages(self, pages: np.ndarray, att_len, att_align, attnums, vis=None, vis_counts=None, notnull=None):
        d = GxHeapDesc()
        d.natts, d.ncols = len(att_len), len(attnums)
        for i, nn in enumerate(notnull or ()):
            d.att_notnull[i] = 1 if nn else 0
        for i, (l, a) in enumerate(zip(att_len, att_align)):
            d.att_len[i], d.att_align[i] = l, a
        for i, a in enumerate(attnums):
            d.attnums[i] = a
        pages = np.ascontiguousarray(pages, np.uint8)
        npages = pages.size // 8192
        vo = vc = None
        stride = 0
        if vis is not None:
            vis = np.ascontiguousarray(vis, np.uint16)
            vis_counts = np.ascontiguousarray(vis_counts, np.int32)
            stride = vis.shape[1]
            vo, vc = vis.ctypes.data, vis_counts.ctypes.data
        self.ctx._chk(lib().gx_table_append_heap_pages(self.h, pages.ctypes.data, npages, C.byref(d), vo, vc, stride))
        self.ctx._chk(lib().gx_table_load_finish(self.h))
        return self

    def generate(self, table_id, sf, o0, o1, node=0, nnodes=1, colmap=None):
        if colmap is None:
            self.ctx._chk(lib().gx_table_generate(self.h, table_id, sf, o0, o1, node, nnodes))
        else:
            cm = (C.c_int32 * len(colmap))(*colmap)
            self.ctx._chk(lib().gx_table_generate_cols(self.h, table_id, sf, o0, o1, node, nnodes, cm))
        return self

    def read(self, col, with_nulls=False):
        n = self.nrows
        out = np.empty(n, NP_DTYPES[self.types[col]])
        nl = np.zeros(n, np.uint8) if with_nulls else None
        self.ctx._chk(lib().gx_table_read_column(self.h, col, 0, n, out.ctypes.data, None if nl is None else nl.ctypes.data))
        return (out, nl) if with_nulls else out

    def permuted(self, seed=1) -> "Table":
        h = C.c_void_p()
        self.ctx._chk(lib().gx_table_permute(self.ctx.h, self.h, seed, C.byref(h)))
        return Table(self.ctx, h, self.types)

    def truncate(self):
        self.ctx._chk(lib().gx_table_truncate(self.h))
        return self

    def drop_column(self, col):
        self.ctx._chk(lib().gx_table_drop_column(self.h, col))
        del self.types[col]
        return self

    def free(self):
        if self.h and self.ctx.h:          # handles die with their context (stream-ordered frees need its stream)
            lib().gx_table_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class HashTable:
    def __init__(self, ctx, handle):
        self.ctx, self.h = ctx, handle

    @property
    def nentries(self):
        return lib().gx_hash_nentries(self.h)

    @property
    def nslots(self):
        return lib().gx_hash_nslots(self.h)

    def info(self):
        m, c = C.c_int(), C.c_double()
        lib().gx_hash_info(self.h, C.byref(m), C.byref(c))
        return {"slot_mode": m.value, "avg_chain": c.value}

    def free(self):
        if self.h and self.ctx.h:          # handles die with their context (stream-ordered frees need its stream)
            lib().gx_hash_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Result:
    def __init__(self, ctx, handle, plan: GxAggPlan):
        self.ctx, self.h, self.plan = ctx, handle, plan

    @property
    def ngroups(self):
        return lib().gx_result_ngroups(self.h)

    def combine(self):
        self.ctx._chk(lib().gx_result_combine(self.ctx.h, self.h))
        return self

    def fetch(self, pinned=False):
        """keys int64[n, ng], aggs float64[n, na] (int results bit-cast), nulls uint8[n, ng+na].
        pinned=True: the arrays are views of the context's reusable pinned result buffers (valid until the
        next pinned fetch) — what a caller that fetches large results repeatedly would hand in."""
        n, ng, na = self.ngroups, self.plan.n_group_cols, self.plan.n_aggs
        if pinned:
            keys = self.ctx.pinned_array("keys", (n, ng), np.int64)
            aggs = self.ctx.pinned_array("aggs", (n, na), np.float64)
            nulls = self.ctx.pinned_array("nulls", (n, ng + na), np.uint8)
        else:
            keys = np.zeros((n, ng), np.int64)
            aggs = np.zeros((n, na), np.float64)
            nulls = np.zeros((n, ng + na), np.uint8)
        self.ctx._chk(lib().gx_result_fetch(self.h, n, keys.ctypes.data, aggs.ctypes.data, nulls.ctypes.data))
        return keys, aggs, nulls

    def fetch_states(self):
        """partial states: keys int64[n, ng], vals float64[n, na], cnts int64[n, na], nulls uint8[n, ng+na]"""
        n, ng, na = self.ngroups, self.plan.n_group_cols, self.plan.n_aggs
        keys = np.zeros((n, ng), np.int64); vals = np.zeros((n, na), np.float64)
        cnts = np.zeros((n, na), np.int64); nulls = np.zeros((n, ng + na), np.uint8)
        self.ctx._chk(lib().gx_result_fetch_states(self.h, n, keys.ctypes.data, vals.ctypes.data, cnts.ctypes.data, nulls.ctypes.data))
        return keys, vals, cnts, nulls

    def fetch_sxx(self):
        """Sxx of each variance aggregate's {N, Sx, Sxx} state, float64[n, na] (0 for other aggregates), groups in
        the order of fetch_states"""
        n, na = self.ngroups, self.plan.n_aggs
        sxx = np.zeros((n, na), np.float64)
        self.ctx._chk(lib().gx_result_fetch_sxx(self.h, n, sxx.ctypes.data))
        return sxx

    def fetch_regr(self):
        """float8_regr_accum's {N, Sx, Sxx, Sy, Syy, Sxy} of each regression aggregate, float64[n, na, 6] (zeros for
        other aggregates and regr_count), groups in the order of fetch_states"""
        n, na = self.ngroups, self.plan.n_aggs
        st = np.zeros((n, na, 6), np.float64)
        self.ctx._chk(lib().gx_result_fetch_regr(self.h, n, st.ctypes.data))
        return st

    def free(self):
        if self.h and self.ctx.h:          # handles die with their context (stream-ordered frees need its stream)
            lib().gx_result_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Context:
    """One per process and GPU (gx_init creates the CUDA context lazily)."""

    def __init__(self, device: int = 0):
        h = C.c_void_p()
        st = lib().gx_init(device, C.byref(h))
        if st != GX_OK:
            raise GxError(st, (lib().gx_last_error(None) or b"").decode())
        self.h = h

    def _chk(self, st):
        if st != GX_OK:
            raise GxError(st, (lib().gx_last_error(self.h) or b"").decode())

    def pinned_array(self, name, shape, dtype):
        """numpy view of a cached pinned host buffer (gx_host_alloc), grown on demand"""
        if not hasattr(self, "_pinned"):
            self._pinned = {}
        nbytes = max(int(np.prod(shape)) * np.dtype(dtype).itemsize, 8)
        ptr, cap = self._pinned.get(name, (None, 0))
        if cap < nbytes:
            if ptr:
                self.host_free(ptr)
            cap = int(nbytes * 1.25) + 4096
            ptr = self.host_alloc(cap)
            self._pinned[name] = (ptr, cap)
        buf = (C.c_uint8 * nbytes).from_address(ptr)
        return np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)

    def close(self):
        if self.h:
            for ptr, _ in getattr(self, "_pinned", {}).values():
                lib().gx_host_free(self.h, ptr)
            self._pinned = {}
            lib().gx_shutdown(self.h)
            self.h = None

    def sync(self):
        self._chk(lib().gx_sync(self.h))

    def stage_acquire(self, nbytes) -> int:
        p = C.c_void_p()
        self._chk(lib().gx_stage_acquire(self.h, nbytes, C.byref(p)))
        return p.value

    def pool_reserve(self, nbytes=0):
        self._chk(lib().gx_pool_reserve(self.h, nbytes))

    def device_info(self):
        sm, ma, mi, hbm = C.c_int(), C.c_int(), C.c_int(), C.c_int64()
        self._chk(lib().gx_device_info(self.h, C.byref(sm), C.byref(ma), C.byref(mi), C.byref(hbm)))
        return {"sm_count": sm.value, "cc": (ma.value, mi.value), "hbm_bytes": hbm.value}

    @property
    def launches(self):
        return lib().gx_launch_count(self.h)

    def timer_start(self):
        self._chk(lib().gx_timer_start(self.h))

    def timer_stop(self) -> float:
        ms = C.c_double()
        self._chk(lib().gx_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def profile(self, on=True):
        self._chk(lib().gx_profile(self.h, 1 if on else 0))

    def profile_get(self, name):
        ms, n = C.c_double(), C.c_int64()
        self._chk(lib().gx_profile_get(self.h, name.encode(), C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def l2_flush(self):
        self._chk(lib().gx_l2_flush(self.h))

    def host_alloc(self, nbytes) -> int:
        p = C.c_void_p()
        self._chk(lib().gx_host_alloc(self.h, nbytes, C.byref(p)))
        return p.value

    def host_free(self, p):
        self._chk(lib().gx_host_free(self.h, p))

    def h2d_probe(self, host_ptr, nbytes, nstreams=1) -> float:
        r = C.c_double()
        self._chk(lib().gx_h2d_probe(self.h, host_ptr, nbytes, nstreams, C.byref(r)))
        return r.value

    # ---- tables
    def table(self, types, capacity) -> Table:
        arr = (C.c_int32 * len(types))(*types)
        h = C.c_void_p()
        self._chk(lib().gx_table_create(self.h, len(types), arr, capacity, C.byref(h)))
        return Table(self, h, types)

    def table_from(self, types, cols, nulls=None) -> Table:
        n = len(cols[0]) if cols else 0
        return self.table(types, max(n, 1)).append(cols, nulls)

    def scan_filter(self, t: Table, preds, out_cols) -> Table:
        pr = (GxPred * max(len(preds), 1))(*[mk_pred(*p) for p in preds])
        oc = (C.c_int32 * len(out_cols))(*out_cols)
        h = C.c_void_p()
        self._chk(lib().gx_scan_filter(self.h, t.h, len(preds), pr, len(out_cols), oc, C.byref(h)))
        return Table(self, h, [t.types[c] for c in out_cols])

    # ---- join
    def hash_build(self, inner: Table, key_col, payload_cols=(), unique=False, preds=()) -> HashTable:
        pr = (GxPred * max(len(preds), 1))(*[mk_pred(*p) for p in preds])
        pc = (C.c_int32 * max(len(payload_cols), 1))(*payload_cols)
        h = C.c_void_p()
        self._chk(lib().gx_hash_build(self.h, inner.h, key_col, len(preds), pr, len(payload_cols), pc, 1 if unique else 0, C.byref(h)))
        ht = HashTable(self, h)
        ht.payload_types = [inner.types[c] for c in payload_cols] or [GX_INT8]
        return ht

    def hash_probe(self, outer: Table, key_col, ht: HashTable, out_outer_cols, preds=(), join_type=0) -> Table:
        pr = (GxPred * max(len(preds), 1))(*[mk_pred(*p) for p in preds])
        oc = (C.c_int32 * max(len(out_outer_cols), 1))(*out_outer_cols)
        h = C.c_void_p()
        self._chk(lib().gx_hash_probe_ex(self.h, outer.h, key_col, len(preds), pr, ht.h, join_type, len(out_outer_cols), oc, C.byref(h)))
        inner = [] if join_type in (GX_JOIN_SEMI, GX_JOIN_ANTI) else ht.payload_types
        return Table(self, h, [outer.types[c] for c in out_outer_cols] + inner)

    # ---- forward-node pages (the reference's redistribute wire format)
    @staticmethod
    def _wire_desc(att_len, att_align, attnums, notnull=None):
        d = GxHeapDesc()
        d.natts, d.ncols = len(att_len), len(attnums)
        for i, (l, a) in enumerate(zip(att_len, att_align)):
            d.att_len[i], d.att_align[i] = l, a
        for i, a in enumerate(attnums):
            d.attnums[i] = a
        for i, nn in enumerate(notnull or ()):
            d.att_notnull[i] = 1 if nn else 0
        return d

    def fnpage_pack(self, t: Table, att_len, att_align, page_id: GxFnPageId = None, end_marker=True) -> np.ndarray:
        """table -> (npages, 8192) uint8 array of FnPages as the reference's sender would hand them to the forwarder"""
        d = self._wire_desc(att_len, att_align, list(range(len(att_len))))
        pid = page_id or GxFnPageId()
        n = C.c_int64()
        self._chk(lib().gx_fnpage_pack(self.h, t.h, C.byref(d), C.byref(pid), int(bool(end_marker)), None, 0, C.byref(n)))
        out = np.empty((n.value, 8192), np.uint8)
        if n.value:
            self._chk(lib().gx_fnpage_pack(self.h, t.h, C.byref(d), C.byref(pid), int(bool(end_marker)), out.ctypes.data, n.value, C.byref(n)))
        return out

    def fnpage_unpack(self, pages: np.ndarray, att_len, att_align, attnums, col_types, notnull=None) -> Table:
        """FnPages of one stream -> a new table (columns attnums of the tuple)"""
        d = self._wire_desc(att_len, att_align, attnums, notnull)
        pages = np.ascontiguousarray(pages, np.uint8)
        tarr = (C.c_int32 * len(col_types))(*col_types)
        h = C.c_void_p()
        self._chk(lib().gx_fnpage_unpack(self.h, pages.ctypes.data if pages.size else None, pages.size // 8192, C.byref(d), tarr, C.byref(h)))
        return Table(self, h, list(col_types))

    # ---- bloom filter of the hash join
    def bloom_build(self, inner: Table, key_col, preds=()):
        """returns an opaque handle (int) or None when the reference would give up (> 2^20 buckets)"""
        pr = (GxPred * max(len(preds), 1))(*[mk_pred(*p) for p in preds])
        h = C.c_void_p()
        self._chk(lib().gx_bloom_build(self.h, inner.h, key_col, len(preds), pr, C.byref(h)))
        return h if h.value else None

    def bloom_words(self, b) -> np.ndarray:
        out = np.empty(8 << lib().gx_bloom_log_num_buckets(b), np.uint32)
        self._chk(lib().gx_bloom_read_words(b, out.ctypes.data))
        return out

    def bloom_test(self, b, outer: Table, key_col) -> np.ndarray:
        out = np.zeros(outer.nrows, np.uint8)
        self._chk(lib().gx_bloom_test(self.h, b, outer.h, key_col, out.ctypes.data))
        return out

    # ---- aggregate
    def hash_agg(self, outer: Table, plan: GxAggPlan, ht: HashTable | None = None) -> Result:
        h = C.c_void_p()
        self._chk(lib().gx_hash_agg(self.h, outer.h, ht.h if ht else None, C.byref(plan), C.byref(h)))
        return Result(self, h, plan)

    def hash_agg_joins(self, outer: Table, steps, plan: GxAggPlan) -> Result:
        """steps: (HashTable, (side, col)[, join_type]) per join of the chain, in probe order"""
        arr = (GxJoinStep * max(len(steps), 1))()
        for i, st in enumerate(steps):
            ht, (side, col) = st[0], st[1]
            arr[i].h = ht.h if ht is not None else None
            arr[i].key.side, arr[i].key.col = side, col
            arr[i].join_type = st[2] if len(st) > 2 else GX_JOIN_INNER
        h = C.c_void_p()
        self._chk(lib().gx_hash_agg_joins(self.h, outer.h, len(steps), arr, C.byref(plan), C.byref(h)))
        return Result(self, h, plan)

    def hash_agg_right(self, probe: Table, probe_key_col, build: Table, ht: HashTable, join_type, plan: GxAggPlan,
                       probe_preds=()) -> Result:
        """gx_hash_agg_right: the plan aggregates build's rows that a right semi (GX_JOIN_SEMI_RIGHT) or right anti
        (GX_JOIN_ANTI_RIGHT) join with the probe side consumes; ht = hash_build(build, key, preds=build quals) without
        payload columns"""
        pr = (GxPred * max(len(probe_preds), 1))(*[mk_pred(*p) for p in probe_preds])
        h = C.c_void_p()
        self._chk(lib().gx_hash_agg_right(self.h, probe.h, probe_key_col, len(probe_preds), pr, build.h, ht.h if ht else None,
                                          join_type, C.byref(plan), C.byref(h)))
        return Result(self, h, plan)

    # ---- communicator / routing
    @staticmethod
    def unique_id() -> bytes:
        buf = C.create_string_buffer(128)
        st = lib().gx_comm_unique_id(buf)
        if st != GX_OK:
            raise GxError(st, (lib().gx_last_error(None) or b"").decode())
        return buf.raw

    def comm_init(self, rank, nranks, uid: bytes):
        self._chk(lib().gx_comm_init(self.h, rank, nranks, uid))

    def set_shardmap(self, nnodes, shardmap=None):
        p = None if shardmap is None else np.ascontiguousarray(shardmap, np.int32).ctypes.data
        self._chk(lib().gx_set_shardmap(self.h, p, nnodes))

    def route(self, t: Table, key_col) -> np.ndarray:
        out = np.empty(t.nrows, np.int32)
        self._chk(lib().gx_route(self.h, t.h, key_col, out.ctypes.data))
        return out

    def partition_by_node(self, t: Table, key_col, nnodes):
        counts = np.zeros(nnodes, np.int64)
        h = C.c_void_p()
        self._chk(lib().gx_partition_by_node(self.h, t.h, key_col, C.byref(h), counts.ctypes.data))
        return Table(self, h, t.types), counts

    def redistribute(self, t: Table, key_col) -> Table:
        h = C.c_void_p()
        self._chk(lib().gx_redistribute(self.h, t.h, key_col, C.byref(h)))
        return Table(self, h, t.types)

    def debug_hash(self, which, values) -> np.ndarray:
        v = np.ascontiguousarray(values, np.int64)
        out = np.empty(len(v), np.uint32)
        self._chk(lib().gx_debug_hash(self.h, which, v.ctypes.data, len(v), out.ctypes.data))
        return out

    def debug_combine(self, parts, rank) -> Result:
        """gx_debug_combine: combine parts[rank] in place as rank `rank` of len(parts) datanodes would, the other
        parts standing for the other datanodes' partial results; returns parts[rank]"""
        arr = (C.c_void_p * max(len(parts), 1))(*[p.h for p in parts])
        self._chk(lib().gx_debug_combine(self.h, len(parts), arr, rank))
        return parts[rank]

    def debug_redistribute(self, parts, key_col, rank, window_bytes=0):
        """gx_debug_redistribute: the rows rank `rank` of len(parts) datanodes would receive from gx_redistribute, the
        parts standing for the datanodes' input tables; window_bytes > 0 takes the peer-window path with windows of
        that size, 0 the NCCL path.  Returns (Table, path): 0 peer windows, 1 one-pass regions, 2 two-pass partition."""
        arr = (C.c_void_p * max(len(parts), 1))(*[p.h for p in parts])
        h, path = C.c_void_p(), C.c_int(-1)
        self._chk(lib().gx_debug_redistribute(self.h, len(parts), arr, key_col, rank, window_bytes, C.byref(h), C.byref(path)))
        return Table(self, h, parts[rank].types), path.value


def _exec_host(self, outer_types, outer_ptrs, outer_nrows, plan, inner_types=None, inner_ptrs=None, inner_nrows=0,
               inner_key_col=0, payload_cols=(), inner_unique=False, inner_preds=()) -> Result:
    """HOST buffers in, partial result handle out (gx_exec_host).
    *_ptrs: host addresses (int) or numpy arrays, one per column."""
    keep = []

    def mk(types, ptrs, nrows):
        ht = GxHostTable()
        ht.ncols, ht.nrows = len(types), nrows
        tarr = (C.c_int32 * len(types))(*types)
        carr = (C.c_void_p * len(types))(*[p if isinstance(p, int) else p.ctypes.data for p in ptrs])
        ht.types = C.cast(tarr, C.POINTER(C.c_int32))
        ht.cols = C.cast(carr, C.POINTER(C.c_void_p))
        ht.nulls = None
        keep.extend([tarr, carr])
        return ht
    o = mk(outer_types, outer_ptrs, outer_nrows)
    i = mk(inner_types, inner_ptrs, inner_nrows) if inner_types is not None else None
    pr = (GxPred * max(len(inner_preds), 1))(*[mk_pred(*p) for p in inner_preds])
    pc = (C.c_int32 * max(len(payload_cols), 1))(*payload_cols)
    h = C.c_void_p()
    self._chk(lib().gx_exec_host(self.h, C.byref(o), C.byref(i) if i is not None else None, inner_key_col,
                                 len(inner_preds), pr, len(payload_cols), pc, 1 if inner_unique else 0,
                                 C.byref(plan), C.byref(h)))
    return Result(self, h, plan)


Context.exec_host = _exec_host


def declared_symbols() -> list[str]:
    """Every function include/gpuexec.h declares (parsed from the header)."""
    import re
    txt = open(os.path.join(INCLUDE_DIR, "gpuexec.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(gx_[a-z0-9_]+)\s*\(", txt)))
