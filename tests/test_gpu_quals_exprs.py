"""Scan quals and aggregate argument expressions at type, value and shape edges, on every kernel that evaluates them,
against exact references: tests/qual_ref.py for the quals (pinned to the oracle by tests/test_qual_ref_cpu.py),
tests/exact_ref.py for the aggregates, tests/join_ref.py and tests/exists_ref.py for the joins.

Quals (`col op const`, ANDed) are evaluated by gx_eval_pred row by row, by pred_tile (with its own int4 / date and
float8 fast paths for columns without NULLs), by pred_vec4 in the run-aggregate kernel, by the one-pass filter and by
the join build and bloom filter.  Every qual column holds its type's edge values and their neighbours (and NULLs in the
nullable variants), and every edge value is also a constant; int4 / date columns also meet constants outside int32.

Aggregate arguments are compiled into a chain of at most four terms (gx_agg.cu: compile_expr) and evaluated by three
separate interpreters: gx_eval_term (gx_k_agg), lpt_term (gx_k_agg_lptile) and slot_term over shared column registers
(gx_k_fewgroups, gx_k_runagg).  Every term kind runs first and later, in chains of up to four terms, with folded
constants, non-finite and signed-zero constants, int4 / int8 columns, NULL operands and shared column slots.

Each kernel family is forced by shape, estimate or switch, and its profile name proves it answered."""
import ctypes

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import exists_ref as E
import join_ref as J
import qual_ref as Q
from helpers import to_gpu_plan

pytestmark = pytest.mark.gpu

I32, I64 = Q.I32, Q.I64
NAN, INF = np.nan, np.inf
C, K = g.GX_OP_COL, g.GX_OP_CONST
ADD, SUB, MUL = (g.GX_OP_ADD, 0, 0), (g.GX_OP_SUB, 0, 0), (g.GX_OP_MUL, 0, 0)
LT, LE, EQ, GE, GT, NE = g.GX_LT, g.GX_LE, g.GX_EQ, g.GX_GE, g.GX_GT, g.GX_NE
SUM, AVG, MIN, MAX = g.GX_AGG_SUM_F8, g.GX_AGG_AVG_F8, g.GX_AGG_MIN_F8, g.GX_AGG_MAX_F8
CNT = (g.GX_AGG_COUNT_STAR, [])
SEEN = set()                     # profile names that answered somewhere in this module


def cl(c):
    return (C, c, 0)


def kn(v):
    return (K, 0, v)


def profiled(gx, fn, names):
    """fn() with profiling on; returns (fn's result or the GxError it raised, profile names of `names` that ran)"""
    gx.profile(True)
    try:
        out = fn()
    except g.GxError as e:
        out = e
    ran = {p for p in names if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    SEEN.update(ran)
    return out, ran


def bits(v):
    v = np.ascontiguousarray(v)
    return v.view({1: np.uint8, 4: np.uint32, 8: np.uint64}[v.dtype.itemsize])


def fetch(res):
    out = res.fetch()
    res.free()
    return out


# ================================================================ gx_scan_filter (one-pass filter)
FTYPES = Q.TYPES + [g.GX_FLOAT8, g.GX_INT4]     # qual columns 0..4, then 5: no qual (arbitrary float8 bits), 6: 0, 1, 2


def filter_table(rng, n, null_frac):
    cols, nulls = [], []
    for t in Q.TYPES:
        v, nl = Q.column(rng, t, n, null_frac)
        cols.append(v); nulls.append(nl)
    cols.append(rng.integers(I64.min, I64.max, n, endpoint=True, dtype=np.int64).view(np.float64)); nulls.append(None)
    cols.append((np.arange(n) % 3).astype(np.int32)); nulls.append(None)
    return cols, nulls


def fpred(c, op, k, t):
    return (c, op, k, True) if t == g.GX_FLOAT8 else (c, op, k)


def check_filter(gx, t, cols, nulls, preds, out_cols):
    """the filter's output is input[keep] in input order, bit for bit (NaN payloads, -0, "char" bytes), with the
    NULL flags of the input; returns the output table"""
    n = len(cols[0])
    keep = Q.quals(cols, nulls, preds, n, FTYPES)
    got = gx.scan_filter(t, preds, out_cols)
    m = int(keep.sum())
    assert got.nrows == m, f"{preds}: {got.nrows} rows, want {m}"
    for j, c in enumerate(out_cols):
        v, nl = got.read(j, with_nulls=True)
        want_nl = np.zeros(m, bool) if nulls[c] is None else nulls[c][keep] != 0
        np.testing.assert_array_equal(nl != 0, want_nl, err_msg=f"{preds}: NULL flags of output column {j}")
        np.testing.assert_array_equal(bits(v)[~want_nl], bits(cols[c][keep])[~want_nl], err_msg=f"{preds}: output column {j}")
    return got


def has_null_array(gx, t, c, gcol):
    """whether column c of t carries a NULL array: count(c) over a column without one is the row count and fits the
    register kernel gx_k_fewgroups; with one it needs a counter word, which only the general kernels keep"""
    plan = g.make_plan(group_cols=[(0, gcol)], aggs=[(g.GX_AGG_COUNT, [cl(c)])], est_groups=4)
    res, ran = profiled(gx, lambda: gx.hash_agg(t, plan), ["agg_fewgroups", "agg_smem_lp"])
    res.free()
    assert len(ran) == 1, ran
    return "agg_smem_lp" in ran


@pytest.mark.parametrize("null_frac", [0.0, 0.1])
def test_filter_every_operator_and_constant(gx, null_frac):
    """one qual per call: every type, operator and edge constant, on columns without NULLs (pred_tile's fast paths for
    int4 / date / float8) and with them (gx_eval_pred)"""
    rng = np.random.default_rng(1 + int(null_frac * 10))
    cols, nulls = filter_table(rng, 5000, null_frac)
    t = gx.table_from(FTYPES, cols, nulls)
    gx.profile(True)
    for c, typ in enumerate(Q.TYPES):
        for op in Q.OPS:
            for k in Q.consts(typ):
                check_filter(gx, t, cols, nulls, [fpred(c, op, k, typ)], [c, 5]).free()
    assert gx.profile_get("filter")[1] > 0
    gx.profile(False)
    SEEN.add("filter")
    t.free()


FILTER_SETS = [
    [(0, GE, -1), (1, LT, 2**32), (3, GT, 127), (4, LT, NAN, True)],        # four ANDed quals over mixed types
    [(1, GT, -2**31), (1, LE, 2**32)],                                       # a range over one column
    [(2, GE, -36_525), (2, LT, 2**31)],                                      # an int4 range with a constant outside int32
    [(4, GE, -INF, True), (4, LE, 0.0, True)],
    [(0, LT, I64.min)],                                                      # no row passes
    [],                                                                      # every row passes
]


@pytest.mark.parametrize("k16", ["1", "0"])
@pytest.mark.parametrize("n", [0, 1, 2047, 2048, 2049, 4095, 4096, 4097, 33 * 4096 + 5])
def test_filter_tile_edges_and_projection(gx, monkeypatch, n, k16):
    """row counts 0, 1, each tile size +-1 (4096-row tiles, 2048 with GX_FILTER_K16=0) and more than 32 tiles (the
    look-back takes more than one round); every column projected, one twice; a column has a NULL array in the output
    exactly when it has one in the input"""
    monkeypatch.setenv("GX_FILTER_K16", k16)
    rng = np.random.default_rng(n + int(k16))
    out = [3, 5, 0, 4, 5, 1, 2, 6]
    for null_frac in (0.0, 0.1):
        cols, nulls = filter_table(rng, n, null_frac)
        t = gx.table_from(FTYPES, cols, nulls)
        for i, preds in enumerate(FILTER_SETS):
            got, ran = profiled(gx, lambda: check_filter(gx, t, cols, nulls, preds, out), ["filter"])
            assert n == 0 or ran == {"filter"}
            if i == 0 and got.nrows:
                for j, c in enumerate(out[:-1]):
                    assert has_null_array(gx, got, j, len(out) - 1) == (nulls[c] is not None), (j, c)
            got.free()
        t.free()


def test_filter_several_tiles_per_cta(gx):
    """more tiles than the grid has CTAs (sm_count x 8): every CTA takes several tickets"""
    n = gx.device_info()["sm_count"] * 8 * 4096 + 3 * 4096 + 17
    rng = np.random.default_rng(5)
    cols, nulls = filter_table(rng, n, 0.05)
    t = gx.table_from(FTYPES, cols, nulls)
    for preds in FILTER_SETS[:2]:
        check_filter(gx, t, cols, nulls, preds, [0, 1, 2, 3, 4, 5]).free()
    t.free()


# ================================================================ quals in the aggregate kernels
# columns: 0 group column (scan: int4) or join key (int8), 1 x, 2 y (float8 arguments), 3..7 one qual column per type
# (int4, int8, date, char, float8), 8 an int4 group column for the SEMI / ANTI plans
def atypes(kind):
    return [g.GX_INT4 if kind == "scan" else g.GX_INT8, g.GX_FLOAT8, g.GX_FLOAT8] + Q.TYPES + [g.GX_INT4]


SX, SY, SXY = (SUM, [cl(1)]), (SUM, [cl(2)]), (SUM, [cl(1), cl(2), MUL])
REG = [SX, CNT, SXY]
GEN = [SX, CNT, SXY, (MIN, [cl(1)]), (MAX, [cl(2), kn(1.0), SUB]), (g.GX_AGG_SUM_I4, [cl(3)]), (g.GX_AGG_COUNT, [cl(7)])]
FMT = {"wide": "probe_agg_exist_wide", "compact": "probe_agg_exist_compact", "narrow": "probe_agg_exist_narrow"}

# family: (input kind, est_groups, strategy, switches, aggregates, profile name)
QUAL_FAMILIES = {
    "agg_fewgroups":     ("scan", 4, 0, {}, REG, "agg_fewgroups"),
    "agg_fewgroups_512": ("scan", 4, 0, {"GX_FG_VARIANT": "0"}, REG, "agg_fewgroups"),
    "agg_lptile8":       ("scan", 16, 0, {"GX_NO_FEWGROUPS": "1"}, REG, "agg_lptile8"),
    "agg_lptile4":       ("scan", 16, 0, {"GX_NO_FEWGROUPS": "1", "GX_LPTILE_K4": "1"}, REG, "agg_lptile4"),
    "agg_smem_lp":       ("scan", 16, 0, {}, GEN, "agg_smem_lp"),
    "agg_smem":          ("scan", 1000, 1, {}, GEN, "agg_smem"),
    "agg_global":        ("scan", 1000, 3, {}, GEN, "agg_global"),
    "radix":             ("scan", 1000, 2, {}, GEN, "scan_records"),
    "runagg_dense":      ("runagg", 0, 0, {"GX_RUNAGG_DENSE": "1"}, [SX, CNT], "runagg_dense"),
    "runagg_small1":     ("runagg", 0, 0, {"GX_RUNAGG_DENSE": "0"}, [SX, CNT], "runagg_small1"),
    "runagg_small2":     ("runagg", 0, 0, {}, [SX, SXY], "runagg_small2"),
    "runagg_wide":       ("runagg", 0, 0, {}, [SX, SXY, SY], "runagg_wide"),
    "probe_agg":         ("join", 1000, 1, {}, GEN, "probe_agg"),
}
for _f in FMT:
    for _jt in ("semi", "anti"):
        QUAL_FAMILIES[f"exist_{_f}_{_jt}"] = ("exist", 5, 0, {}, GEN, FMT[_f])

# quals over columns 3..7; the last set removes every row
AGG_QUALS = [
    [(3, EQ, 2**32 + 5)],                                   # nothing: a narrowed constant would take x = 5
    [(3, LT, 2**31)],                                       # every non-NULL row: narrowed, nothing
    [(3, GE, -2**31 - 1), (3, LE, 5)],                      # a range over one column
    [(5, GT, -2**32 + 5)],
    [(6, GT, 127)],                                         # "char" bytes 128..255
    [(6, LE, 1)],
    [(7, LT, INF, True)],                                   # drops NaN and +inf
    [(7, EQ, NAN, True)],                                   # NaN of either sign
    [(7, GE, -0.0, True), (7, LE, 5e-324, True)],
    [(4, GT, 2**31), (4, LE, I64.max - 1)],
    [(3, GE, -1), (7, LT, NAN, True), (6, NE, 200), (4, NE, 2**32)],      # four ANDed quals over mixed types
    [(3, LT, I64.min)],
]
WHOLE_GROUP = [(3, GT, I32.min)]                           # the victim group's rows all hold INT32_MIN (or NULL)
EXIST_NAMES = set(FMT.values()) | {"probe_agg"}


def bunched(n):
    i = np.arange(n, dtype=np.int64)
    return (i // 8) * 32 + (i % 8) + 1


class QualFamily:
    """one family's input (quals on columns 3..7, NULLs in them when null_frac > 0) and its join table"""

    def __init__(self, gx, name, null_frac):
        self.gx, self.name = gx, name
        self.kind, self.est, self.strategy, _, self.aggs, self.profile = QUAL_FAMILIES[name]
        rng = np.random.default_rng(sum(map(ord, name)) + int(null_frac * 100))
        n = 128 * 157 + 77                               # full 128-row tiles of the run-aggregate kernel, then a ragged one
        q = [Q.column(rng, t, n, null_frac) for t in Q.TYPES]
        x, y = rng.uniform(-4, 4, n), rng.uniform(-4, 4, n)
        g2 = rng.integers(0, 5, n).astype(np.int32)
        self.ht = self.inner = None
        self.jt = 0
        if self.kind == "scan":
            keys = np.array([I32.min, -1, I32.max], np.int64)
            self.gi = rng.integers(0, 3, n)
            key = keys[self.gi].astype(np.int32)
            self.gkeys = [(int(k),) for k in keys]
        elif self.kind in ("runagg", "join"):
            M = 3000
            key = rng.integers(1, M + 1, n).astype(np.int64)
            if self.kind == "runagg":
                key = np.sort(key)                         # a run of equal keys is a group
                self.gi, self.gkeys = key - 1, [(k,) for k in range(1, M + 1)]
                ipay = np.zeros(M, np.int32)
            else:
                self.gi, self.gkeys = key % 5, [(int(p) * 1000 - 2000,) for p in range(5)]
                ipay = (np.arange(1, M + 1) % 5 * 1000 - 2000).astype(np.int32)
            self.inner = gx.table_from([g.GX_INT8, g.GX_INT4], [np.arange(1, M + 1, dtype=np.int64), ipay])
            self.ht = gx.hash_build(self.inner, 0, [1], unique=True)
        else:
            _, fmt, jt = name.split("_")
            self.jt = g.GX_JOIN_SEMI if jt == "semi" else g.GX_JOIN_ANTI
            bk = bunched(100_000)
            bk = np.sort(np.concatenate([bk, bk[::3]]))
            if fmt == "wide":
                bk = rng.permutation(bk)
            self.inner = gx.table_from([g.GX_INT8, g.GX_INT4], [bk, (bk % 2406 - 2922).astype(np.int32)])
            self.ht = gx.hash_build(self.inner, 0, [] if fmt == "compact" else [1], unique=False)
            self.bkeys = bk
            key = np.concatenate([rng.choice(bk, n // 2), rng.choice(bk, n - n // 2) + 2]).astype(np.int64)
            self.gi, self.gkeys = g2, [(v,) for v in range(5)]
        q4 = q[0][0]
        q4[self.gi == 1] = I32.min                         # the victim group of WHOLE_GROUP
        self.types = atypes(self.kind)
        self.cols = [key, x, y] + [v for v, _ in q] + [g2]
        self.nulls = [None, None, None] + [nl for _, nl in q] + [None]
        self.t = gx.table_from(self.types, self.cols, self.nulls)

    def plan(self, preds, grouped=True):
        gc = [] if not grouped else [(0, 8)] if self.kind == "exist" else [(1, 0)] if self.kind == "join" else [(0, 0)]
        return g.make_plan(preds=preds, outer_key_col=-1 if self.kind == "scan" else 0, group_cols=gc, aggs=self.aggs,
                           est_groups=self.est, strategy=self.strategy, join_type=self.jt)

    def want(self, plan):
        preds = [(plan.preds[p].col, plan.preds[p].op, plan.preds[p].fval if self.types[plan.preds[p].col] == g.GX_FLOAT8
                  else plan.preds[p].ival) for p in range(plan.n_preds)]
        if self.kind == "exist":
            return E.expect_exists_groups(plan, self.jt, self.cols, self.types, self.bkeys, outer_nulls=self.nulls)
        keep = Q.quals(self.cols, self.nulls, preds, len(self.cols[0]), self.types)
        if plan.n_group_cols == 0:
            return X.expect_groups(plan, self.cols, nulls=self.nulls, types=self.types, keep=keep)
        return X.expect_groups(plan, self.cols, nulls=self.nulls, types=self.types, keep=keep, gindex=self.gi, gkeys=self.gkeys)

    def check(self, preds, grouped=True):
        plan = self.plan(preds, grouped)
        want = self.want(plan)
        got, ran = profiled(self.gx, lambda: fetch(self.gx.hash_agg(self.t, plan, self.ht)), {self.profile})
        assert not isinstance(got, g.GxError), f"{self.name} {preds}: {got}"
        if grouped:
            assert ran == {self.profile}, f"{self.name}: {self.profile} did not run"
        gt = [] if not grouped else [g.GX_INT4 if self.kind in ("scan", "exist", "join") else g.GX_INT8]
        X.check(plan, want, got, gt)
        return want, got

    def free(self):
        self.t.free()
        if self.ht is not None:
            self.ht.free(); self.inner.free()


@pytest.fixture(params=list(QUAL_FAMILIES))
def qfam(request, gx, monkeypatch):
    for k, v in QUAL_FAMILIES[request.param][3].items():
        monkeypatch.setenv(k, v)
    return request.param


@pytest.mark.parametrize("null_frac", [0.0, 0.1])
def test_quals_on_every_family(gx, qfam, null_frac):
    """every qual set on columns without NULLs (pred_tile / pred_vec4 fast paths) and with them (gx_eval_pred); a qual
    that removes one whole group leaves that group out (not present with count 0); no row: no group"""
    F = QualFamily(gx, qfam, null_frac)
    try:
        for preds in AGG_QUALS:
            F.check(preds)
        want, got = F.check(WHOLE_GROUP)
        assert F.gkeys[1] not in want and len(want) >= 2 and got[0].shape[0] == len(want), (F.gkeys[1], sorted(want)[:5])
        none, got = F.check(AGG_QUALS[-1])
        assert none == {} and got[0].shape[0] == 0
    finally:
        F.free()


@pytest.mark.parametrize("name", ["agg_lptile8", "agg_smem", "agg_global", "radix", "probe_agg", "exist_wide_semi", "exist_compact_anti"])
def test_plain_aggregate_when_every_row_is_removed(gx, name):
    """without GROUP BY one row comes back whatever the quals remove: count(*) 0, sums / min / max NULL"""
    F = QualFamily(gx, name, 0.1)
    try:
        for preds in (AGG_QUALS[-1], [(6, GT, 254), (6, LT, 1)], AGG_QUALS[-2]):
            _, got = F.check(preds, grouped=False)
            assert got[0].shape[0] == 1
        plan = F.plan(AGG_QUALS[-1], grouped=False)
        _, aggs, nulls = fetch(gx.hash_agg(F.t, plan, F.ht))
        assert int(aggs[0:1, 1].view(np.int64)[0]) == 0 and nulls[0, 0] == 1 and nulls[0, 1] == 0
    finally:
        F.free()


# ---------------------------------------------------------------- shapes whose kernel takes no quals
# family: (input kind, est_groups, strategy, switches, aggregates, profile without quals, profile that takes the quals)
REROUTE = {
    "agg_fast":       ("scan", 1000, 1, {}, [SX, CNT], "agg_fast", "agg_smem"),
    "agg_count_char": ("char", 3, 0, {}, [CNT], "agg_count_char", "agg_fewgroups"),
    "probe_agg_fast": ("join", 1000, 0, {"GX_NO_RUNJOIN": "1"}, [SX, CNT], "probe_agg_fast", "probe_agg"),
    "probe_agg_tma":  ("join", 1000, 0, {"GX_RUNJOIN_TMA": "1"}, [SX, CNT], "probe_agg_tma", "probe_agg"),
    "probe_agg_run":  ("join", 1000, 0, {"GX_RUNJOIN_TMA": "0", "GX_RUNJOIN_SEG": "0"}, [SX, CNT], "probe_agg_run", "probe_agg"),
    "probe_agg_seg":  ("join", 1000, 0, {"GX_RUNJOIN_TMA": "0", "GX_RUNJOIN_SEG": "1"}, [SX, CNT], "probe_agg_seg", "probe_agg"),
}
REROUTE_NAMES = {v[5] for v in REROUTE.values()} | {v[6] for v in REROUTE.values()}


@pytest.mark.parametrize("name", list(REROUTE))
def test_one_qual_routes_to_a_kernel_that_evaluates_it(gx, monkeypatch, name):
    kind, est, strategy, env, aggs, plain, qualed = REROUTE[name]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(len(name))
    n = 60_000
    q = [Q.column(rng, t, n) for t in Q.TYPES]
    x = rng.uniform(-4, 4, n)
    ht = inner = None
    if kind == "scan":
        G = 1000
        gi = rng.integers(0, G, n)
        key, gkeys, kt, gc = (gi * 7 - 3000).astype(np.int32), [(i * 7 - 3000,) for i in range(G)], g.GX_INT4, [(0, 0)]
    elif kind == "char":
        codes = np.array([65, 78, 200], np.uint8).view(np.int8)
        gi = rng.integers(0, 3, n)
        key, gkeys, kt, gc = codes[gi], [(int(c),) for c in codes], g.GX_CHAR, [(0, 0)]
    else:
        # a dense unique build side of 200k+ keys (the streamed-table kernels read its key-ordered compact form)
        G, M = 1000, 200_000
        ipay = (np.arange(M) % G * 7 - 3000).astype(np.int32)
        inner = gx.table_from([g.GX_INT8, g.GX_INT4], [np.arange(1, M + 1, dtype=np.int64), ipay])
        ht = gx.hash_build(inner, 0, [1], unique=True)
        key = np.sort(rng.integers(1, M + 1, n)).astype(np.int64)
        gi, gkeys, kt, gc = (key - 1) % G, [(i * 7 - 3000,) for i in range(G)], g.GX_INT8, [(1, 0)]
    types = [kt, g.GX_FLOAT8] + Q.TYPES
    cols = [key, x] + [v for v, _ in q]
    t = gx.table_from(types, cols)
    for preds in ([], [(6, LT, NAN, True)], [(5, GT, 127)], [(2, EQ, 2**32 + 5)], [(2, GE, 0), (3, LT, 2**32), (4, NE, 0), (6, GE, -0.0, True)]):
        plan = g.make_plan(preds=preds, outer_key_col=-1 if ht is None else 0, group_cols=gc, aggs=aggs, est_groups=est, strategy=strategy)
        keep = Q.quals(cols, None, preds, n, types)
        want = X.expect_groups(plan, cols, types=types, keep=keep, gindex=gi, gkeys=gkeys)
        got, ran = profiled(gx, lambda: fetch(gx.hash_agg(t, plan, ht)), REROUTE_NAMES)
        assert not isinstance(got, g.GxError), got
        if preds:
            assert plain not in ran and qualed in ran, (preds, sorted(ran))
        else:
            assert plain in ran, sorted(ran)
        X.check(plan, want, got, [g.GX_INT4 if kind != "char" else g.GX_CHAR])
    t.free()
    if ht is not None:
        ht.free(); inner.free()


# ---------------------------------------------------------------- build side: hash build, probe, bloom filter, exec_host
BUILD_PATHS = {          # rows, key-ordered, profile names of which one must run
    "direct":      (20_000, False, {"build_direct"}),
    "bucketed":    (200_000, False, {"build_bucket1"}),
    "key_ordered": (200_000, True, {"build_sorted_search", "build_sorted_pass"}),
}
BUILD_NAMES = {"build_direct", "build_bucket1", "build_bucket2", "build_sorted_search", "build_sorted_pass"}
BUILD_QUALS = [
    [(2, GE, -1), (6, LT, NAN, True)],
    [(5, GT, 127), (3, NE, 2**32)],
    [(2, LT, 2**31), (4, GE, -2**31 - 1), (4, LE, 0)],
    [(6, EQ, NAN, True)],
]


def read_rows(t):
    out = []
    for c in range(len(t.types)):
        v, nl = t.read(c, with_nulls=True)
        out.append(np.where(nl == 0, v.astype(np.int64), J.NULL))
    w = np.stack(out, 1) if out else np.zeros((t.nrows, 0), np.int64)
    return w[np.lexsort(w.T[::-1])] if len(w) else w


@pytest.mark.parametrize("null_frac", [0.0, 0.1])
@pytest.mark.parametrize("path", list(BUILD_PATHS))
def test_build_and_probe_quals(gx, path, null_frac):
    """build-side quals on each build path, outer quals of gx_hash_probe_ex for INNER, LEFT, SEMI and ANTI"""
    n, ordered, must = BUILD_PATHS[path]
    rng = np.random.default_rng(len(path) + int(null_frac * 10))
    bk = np.int64(-3 * n) + np.arange(n, dtype=np.int64) * 3
    if not ordered:
        bk = rng.permutation(bk)
    bpay = (np.arange(n) * 7 - 3).astype(np.int32)
    bq = [Q.column(rng, t, n, null_frac) for t in Q.TYPES]
    btypes = [g.GX_INT8, g.GX_INT4] + Q.TYPES
    bcols, bnulls = [bk, bpay] + [v for v, _ in bq], [None, None] + [nl for _, nl in bq]
    bt = gx.table_from(btypes, bcols, bnulls)
    no = 50_000
    ok = np.concatenate([rng.choice(bk, no // 2), rng.choice(bk, no - no // 2) + 1]).astype(np.int64)
    oq = [Q.column(rng, t, no, null_frac) for t in Q.TYPES]
    otypes = [g.GX_INT8, g.GX_INT4] + Q.TYPES
    oval = np.arange(no, dtype=np.int32)
    ocols, onulls = [ok, oval] + [v for v, _ in oq], [None, None] + [nl for _, nl in oq]
    ot = gx.table_from(otypes, ocols, onulls)
    for i, bpreds in enumerate(BUILD_QUALS):
        ht, ran = profiled(gx, lambda: gx.hash_build(bt, 0, [1], unique=True, preds=bpreds), BUILD_NAMES)
        assert ran & must, (path, sorted(ran))
        ikeep = Q.quals(bcols, bnulls, bpreds, n, btypes)
        assert ht.nentries == int(ikeep.sum())
        opreds = BUILD_QUALS[(i + 1) % len(BUILD_QUALS)]
        okeep = Q.quals(ocols, onulls, opreds, no, otypes)
        for jt in (g.GX_JOIN_INNER, g.GX_JOIN_LEFT, g.GX_JOIN_SEMI, g.GX_JOIN_ANTI):
            semi = jt in (g.GX_JOIN_SEMI, g.GX_JOIN_ANTI)
            got = gx.hash_probe(ot, 0, ht, [0, 1], preds=opreds, join_type=jt)
            want = J.rows(J.join(jt, ok, bk, okeep=okeep, ikeep=ikeep), [ok, oval], [] if semi else [bpay])
            rows = read_rows(got)
            got.free()
            np.testing.assert_array_equal(rows, want, err_msg=f"{path}: join type {jt}, build quals {bpreds}, outer quals {opreds}")
        ht.free()
    ot.free(); bt.free()


@pytest.mark.parametrize("null_frac", [0.0, 0.1])
def test_bloom_filter_quals(gx, null_frac):
    """gx_bloom_build's quals: the directory words are the oracle's bit for bit over the rows that pass"""
    L = O.lib()
    rng = np.random.default_rng(17 + int(null_frac * 10))
    n = 40_000
    keys = rng.integers(-2**40, 2**40, n).astype(np.int64)
    knull = (rng.random(n) < null_frac).astype(np.uint8) if null_frac else None
    q = [Q.column(rng, t, n, null_frac) for t in Q.TYPES]
    types = [g.GX_INT8] + Q.TYPES
    cols, nulls = [keys] + [v for v, _ in q], [knull] + [nl for _, nl in q]
    t = gx.table_from(types, cols, nulls)
    for preds in [[]] + [[(p[0] - 1,) + tuple(p[1:]) for p in s] for s in BUILD_QUALS]:     # the qual columns start at 1 here
        keep = Q.quals(cols, nulls, preds, n, types)
        if knull is not None:
            keep &= knull == 0
        b = gx.bloom_build(t, 0, preds)
        ob = L.orc_bloom_create(n)
        assert g.lib().gx_bloom_log_num_buckets(b) == L.orc_bloom_log_num_buckets(ob)
        for k in keys[keep].tolist():
            L.orc_bloom_insert(ob, L.orc_hashint8new(k))
        nw = ctypes.c_int64()
        want = np.ctypeslib.as_array(ctypes.cast(L.orc_bloom_words(ob, ctypes.byref(nw)), ctypes.POINTER(ctypes.c_uint32)), (nw.value,)).copy()
        np.testing.assert_array_equal(gx.bloom_words(b), want, err_msg=str(preds))
        g.lib().gx_bloom_free(b); L.orc_bloom_free(ob)
    t.free()


def test_exec_host_with_inner_and_outer_quals(gx):
    """gx_exec_host (host buffers in) and the resident path give the exact reference's groups under both sides' quals"""
    rng = np.random.default_rng(23)
    M, n = 100_000, 300_000
    ik = np.arange(1, M + 1, dtype=np.int64)
    ipay = (ik % 50 * 3 - 70).astype(np.int32)
    iq = [Q.column(rng, t, M) for t in Q.TYPES]
    itypes = [g.GX_INT8, g.GX_INT4] + Q.TYPES
    icols = [ik, ipay] + [v for v, _ in iq]
    ok = rng.integers(-100, M + 100, n).astype(np.int64)
    oq = [Q.column(rng, t, n) for t in Q.TYPES]
    otypes = [g.GX_INT8, g.GX_FLOAT8] + Q.TYPES
    ocols = [ok, rng.uniform(-4, 4, n)] + [v for v, _ in oq]
    ipreds = [(5, GT, 127), (2, LT, 2**31)]
    opreds = [(6, LT, NAN, True), (2, NE, 2**32 + 5), (4, GE, -36_525)]
    plan = g.make_plan(preds=opreds, outer_key_col=0, group_cols=[(1, 0)], aggs=[SX, CNT, (MIN, [cl(1)]), (AVG, [kn(1.0), cl(1), SUB])], est_groups=50)
    bt, ot = gx.table_from(itypes, icols), gx.table_from(otypes, ocols)
    ht = gx.hash_build(bt, 0, [1], unique=True, preds=ipreds)
    a = fetch(gx.hash_agg(ot, plan, ht))
    b = fetch(gx.exec_host(otypes, ocols, n, plan, inner_types=itypes, inner_ptrs=icols, inner_nrows=M, inner_key_col=0,
                           payload_cols=[1], inner_unique=True, inner_preds=ipreds))
    ikeep = Q.quals(icols, None, ipreds, M, itypes)
    want = J.expect_groups(plan, J.join(g.GX_JOIN_INNER, ok, ik, ikeep=ikeep), ocols, otypes, [ipay], [g.GX_INT4])
    X.check(plan, want, a, [g.GX_INT4])
    X.check(plan, want, b, [g.GX_INT4])
    ht.free(); bt.free(); ot.free()


# ---------------------------------------------------------------- declines
BAD_QUALS = {"operator 0": [(0, 0, 1)], "operator 7": [(0, 7, 1)], "column 99": [(99, EQ, 1)], "column -1": [(-1, EQ, 1)],
             "five quals": [(0, GE, -5)] * 5}


def test_bad_quals_are_argument_errors(gx):
    """operator 0 / 7, a column out of range and five quals are GX_ERR_ARG in every entry point that takes quals; the
    context answers the next call"""
    rng = np.random.default_rng(31)
    cols, nulls = filter_table(rng, 3000, 0.1)
    t = gx.table_from(FTYPES, cols, nulls)
    keys = np.arange(3000, dtype=np.int64)
    kt = gx.table_from([g.GX_INT8, g.GX_INT4], [keys, cols[0]])
    ht = gx.hash_build(kt, 0, [], unique=True)
    good = [(0, GE, -1), (4, LT, NAN, True)]

    def agg(preds):
        plan = g.make_plan(preds=preds[:4], group_cols=[(0, 6)], aggs=[CNT], est_groups=4)
        plan.n_preds = len(preds)
        return fetch(gx.hash_agg(t, plan))

    calls = {
        "scan_filter": lambda p: gx.scan_filter(t, p, [0]),
        "hash_build": lambda p: gx.hash_build(kt, 0, [], unique=True, preds=[(1 if c == 0 else c, op, k) for c, op, k, *_ in p]),
        "bloom_build": lambda p: gx.bloom_build(kt, 0, [(1 if c == 0 else c, op, k) for c, op, k, *_ in p]),
        "hash_probe": lambda p: gx.hash_probe(kt, 0, ht, [0], preds=[(1 if c == 0 else c, op, k) for c, op, k, *_ in p]),
        "hash_agg": agg,
    }
    for what, preds in BAD_QUALS.items():
        for name, call in calls.items():
            with pytest.raises(g.GxError) as ei:
                call(preds)
            assert ei.value.status == g.GX_ERR_ARG, (what, name, ei.value)
            check_filter(gx, t, cols, nulls, good, [0, 4]).free()
    want = Q.quals(cols, nulls, good, 3000, FTYPES)
    _, aggs, _ = agg(good)
    assert int(aggs[:, 0].view(np.int64).sum()) == int(want.sum())
    ht.free(); kt.free(); t.free()


BAD_EXPRS = {
    "compound right operand": [cl(1), cl(2), cl(3), ADD, MUL],
    "five terms": [cl(1), cl(2), ADD, cl(3), ADD, cl(4), ADD, cl(1), ADD],
    "stack underflow": [cl(1), ADD],
    "malformed program": [cl(1), cl(2)],
    "unknown opcode": [(9, 1, 0)],
    "no operand": [],
}


def test_bad_expressions_are_argument_errors(gx):
    """shapes compile_expr cannot represent, and nops 0 or 13, are GX_ERR_ARG for every value aggregate; the context
    answers the next call"""
    d = ExprData(gx, "scan", 3)
    for fn in (SUM, AVG, MIN, MAX):
        for what, ops in list(BAD_EXPRS.items()) + [("nops 13", [cl(1)] * 12)]:
            plan = g.make_plan(group_cols=[(0, 0)], aggs=[CNT, (fn, ops)], est_groups=1000, strategy=1)
            if what == "nops 13":
                plan.aggs[1].arg.nops = 13
            with pytest.raises(g.GxError) as ei:
                gx.hash_agg(d.t, plan)
            assert ei.value.status == g.GX_ERR_ARG, (fn, what, ei.value)
            d.check([CNT, (fn, [cl(1), cl(2), MUL, cl(3), ADD, cl(4), SUB])], 1000, 1, "agg_smem")
    d.free()


# ================================================================ aggregate argument expressions
# columns: 0 group column (scan: int4) or key (runagg: int8), 1 x, 2 y, 3 z, 4 w (float8), 5 int4, 6 int8 (near
# +-2^53 and the int64 limits), 7 / 8 float8 with NULLs.  x is -0 in every row of group 0 (scan) or of every third key.
ETYPES = [g.GX_FLOAT8] * 4 + [g.GX_INT4, g.GX_INT8, g.GX_FLOAT8, g.GX_FLOAT8]
P53 = float(2**53)


class ExprData:
    def __init__(self, gx, kind, seed):
        self.gx, self.kind = gx, kind
        rng = np.random.default_rng(seed)
        n = 128 * 100 + 33
        self.ht = self.inner = None
        if kind == "scan":
            keys = np.array([5, -1, I32.max], np.int64)
            self.gi = rng.integers(0, 3, n)
            key, self.gkeys, zero = keys[self.gi].astype(np.int32), [(int(k),) for k in keys], self.gi == 0
        else:
            M = 1500
            key = np.sort(rng.integers(1, M + 1, n)).astype(np.int64)
            self.gi, self.gkeys, zero = key - 1, [(k,) for k in range(1, M + 1)], key % 3 == 0
            self.inner = gx.table_from([g.GX_INT8, g.GX_INT4], [np.arange(1, M + 1, dtype=np.int64), np.zeros(M, np.int32)])
            self.ht = gx.hash_build(self.inner, 0, [1], unique=True)
        x, y, z, w = rng.uniform(-4, 4, (4, n))
        x[zero] = -0.0
        i4 = rng.choice(np.array([I32.min, I32.max, -1, 0, 7], np.int32), n)
        part = self.gi % 3
        i8 = np.where(part == 0, rng.choice(np.array([2**53 + 1, 2**53 + 3, 2**53 - 1], np.int64), n),
                      np.where(part == 1, rng.choice(np.array([-(2**53 + 1), -(2**53 + 3), 7], np.int64), n),
                               rng.choice(np.array([I64.min, I64.max, -7], np.int64), n)))
        xn, yn = rng.uniform(-4, 4, (2, n))
        self.types = [g.GX_INT4 if kind == "scan" else g.GX_INT8] + ETYPES
        self.cols = [key, x, y, z, w, i4, i8, xn, yn]
        self.nulls = [None] * 7 + [(rng.random(n) < 0.2).astype(np.uint8), (rng.random(n) < 0.2).astype(np.uint8)]
        self.t = gx.table_from(self.types, self.cols, self.nulls)

    def check(self, aggs, est, strategy, profile):
        plan = g.make_plan(outer_key_col=-1 if self.ht is None else 0, group_cols=[(0, 0)], aggs=aggs, est_groups=est, strategy=strategy)
        want = X.expect_groups(plan, self.cols, nulls=self.nulls, types=self.types, gindex=self.gi, gkeys=self.gkeys)
        names = {profile} | {"runagg_dense", "runagg_small1", "runagg_small2", "runagg_wide"}
        got, ran = profiled(self.gx, lambda: fetch(self.gx.hash_agg(self.t, plan, self.ht)), names)
        assert not isinstance(got, g.GxError), got
        assert profile in ran, f"{profile} did not run ({sorted(ran)})"
        X.check(plan, want, got, [self.types[0]])
        return want, got

    def free(self):
        self.t.free()
        if self.ht is not None:
            self.ht.free(); self.inner.free()


EXPRS = {
    # every term kind as the first term: k - x, x - k, k + x, x + k, k * x, x * k
    "first_a": [(SUM, [kn(2.5), cl(1), SUB]), (SUM, [cl(1), kn(2.5), SUB]), (SUM, [kn(-1.5), cl(1), ADD]), CNT],
    "first_b": [(SUM, [cl(1), kn(-1.5), ADD]), (SUM, [kn(3.0), cl(1), MUL]), (SUM, [cl(1), kn(3.0), MUL]), CNT],
    # ... and as a later term: y * (k - x), y + (x - k), y - (k + x), y * (x + k), y - (k * x), y + (x * k)
    "later_a": [(SUM, [cl(2), kn(2.5), cl(1), SUB, MUL]), (SUM, [cl(2), cl(1), kn(2.5), SUB, ADD]), (SUM, [cl(2), kn(-1.5), cl(1), ADD, SUB])],
    "later_b": [(SUM, [cl(2), cl(1), kn(-1.5), ADD, MUL]), (SUM, [cl(2), kn(3.0), cl(1), MUL, SUB]), (SUM, [cl(2), cl(1), kn(3.0), MUL, ADD])],
    # 2-, 3- and 4-term chains; Q1's x * (1 - y) * (1 + z)
    "chains": [(SUM, [cl(1), cl(2), SUB]), (SUM, [cl(1), cl(2), ADD, cl(3), MUL]),
               (SUM, [cl(1), kn(1.0), cl(2), SUB, MUL, kn(1.0), cl(3), ADD, MUL]), (SUM, [cl(1), cl(2), MUL, cl(3), SUB, cl(4), ADD])],
    # four terms: x * (2 - y) + z * 3 - w and (x - 0.5) * y - (1.5 + z) + w
    "four_terms": [(SUM, [cl(1), kn(2.0), cl(2), SUB, MUL, cl(3), kn(3.0), MUL, ADD, cl(4), SUB]),
                   (AVG, [cl(1), kn(2.0), cl(2), SUB, MUL, cl(3), kn(3.0), MUL, ADD, cl(4), SUB]),
                   (SUM, [cl(1), kn(0.5), SUB, cl(2), MUL, kn(1.5), cl(3), ADD, SUB, cl(4), ADD]), CNT],
    # constants folded on the host: x * (1 + 2), 2 * 3 - x, 1.5 - 0.25, x + (1 + 2) * 0.5
    "folding": [(SUM, [cl(1), kn(1.0), kn(2.0), ADD, MUL]), (SUM, [kn(2.0), kn(3.0), MUL, cl(1), SUB]), (SUM, [kn(1.5), kn(0.25), SUB]),
                (SUM, [cl(1), kn(1.0), kn(2.0), ADD, kn(0.5), MUL, ADD])],
    "non_finite": [(SUM, [cl(1), kn(NAN), ADD]), (SUM, [cl(1), kn(INF), MUL]), (SUM, [kn(-INF), cl(1), SUB]), (SUM, [cl(2), kn(-0.0), MUL])],
    # over x = -0: -0 + 0.0 = +0, -0 - 0.0 = -0, 0.0 - -0 = +0, -0 + -0 = -0
    "zero_signs": [(SUM, [cl(1), kn(0.0), ADD]), (SUM, [cl(1), kn(0.0), SUB]), (SUM, [kn(0.0), cl(1), SUB]), (SUM, [kn(-0.0), cl(1), ADD])],
    # sum / avg pairs share a running sum only when their programs match bit for bit, constants included
    "twins_zero": [(AVG, [cl(1), kn(0.0), ADD]), (SUM, [cl(1), kn(-0.0), ADD]), (SUM, [cl(1), kn(0.0), ADD]), (AVG, [cl(1), kn(-0.0), ADD])],
    "twins_value": [(SUM, [cl(1), kn(1.0), ADD]), (AVG, [cl(1), kn(2.0), ADD]), (AVG, [cl(1), kn(1.0), ADD]), (SUM, [cl(1), kn(2.0), ADD])],
    # one column in several aggregates (a shared register slot), and FG_NC = 4 distinct columns
    "shared_slot": [SX, (SUM, [cl(1), cl(2), MUL]), (AVG, [cl(1), kn(1.0), SUB]), (SUM, [cl(2), cl(1), MUL]), CNT],
    "four_columns": [(SUM, [cl(1), cl(2), MUL]), (SUM, [cl(3), cl(4), MUL]), (SUM, [cl(1), cl(4), ADD]), (SUM, [cl(3), cl(2), SUB])],
    "four_columns_five_values": [(SUM, [cl(1), cl(2), MUL]), (SUM, [cl(3), cl(4), MUL]), (SUM, [cl(1), cl(4), ADD]), (SUM, [cl(3), cl(2), SUB]),
                                 (SUM, [cl(4)])],
    # int4 / int8 columns converted to float8 (i8tod rounds 2^53 + 3 to 2^53 + 4), min / max, NULL operands
    "int_columns": [(SUM, [cl(5), kn(0.5), MUL]), (MIN, [cl(5), kn(0.5), SUB]), (MAX, [cl(6), kn(P53), SUB]), (MIN, [cl(6), kn(P53), ADD]),
                    (AVG, [cl(6), kn(1.0), MUL]), (MAX, [cl(6)]), (MIN, [kn(0.0), cl(6), SUB]), (SUM, [cl(5), cl(6), ADD, kn(P53), SUB])],
    "null_operands": [(SUM, [cl(7), cl(2), MUL]), (AVG, [cl(1), cl(8), ADD]), (MIN, [cl(7), cl(8), SUB]), (MAX, [cl(8), kn(2.0), MUL, cl(1), SUB]),
                      (g.GX_AGG_COUNT, [cl(7)]), (g.GX_AGG_COUNT, [cl(8)]), (SUM, [kn(1.0), cl(7), SUB, cl(8), MUL]), CNT],
}

# family: (input kind, est_groups, strategy, switches, profile name)
EXPR_FAMILIES = {
    "general":   ("scan", 1000, 1, {}, "agg_smem"),
    "lptile":    ("scan", 16, 0, {"GX_NO_FEWGROUPS": "1"}, "agg_lptile8"),
    "fewgroups": ("scan", 4, 0, {}, "agg_fewgroups"),
    "runagg":    ("runagg", 0, 0, {}, "runagg"),
}


def admits(aggs, fam):
    """does the family's kernel take this aggregate list (the host's shape checks in hash_agg_run)?"""
    if fam == "general":
        return True
    vals = [a for a in aggs if a[0] != g.GX_AGG_COUNT_STAR]
    if any(fn not in (SUM, AVG) for fn, _ in vals):
        return False
    cols = {c for _, ops in vals for op, c, _ in ops if op == C}
    if not cols <= {1, 2, 3, 4}:
        return False
    if fam == "fewgroups":
        return len(vals) <= 5 and len(cols) <= 4
    if fam == "runagg":
        return len(vals) <= 4 and len(cols) <= 4
    return True


EXPR_CASES = [(f, s) for f in EXPR_FAMILIES for s in EXPRS if admits(EXPRS[s], f)]


@pytest.mark.parametrize("fam,shape", EXPR_CASES)
def test_expression(gx, monkeypatch, fam, shape):
    kind, est, strategy, env, profile = EXPR_FAMILIES[fam]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    d = ExprData(gx, kind, len(shape))
    try:
        want, got = d.check(EXPRS[shape], est, strategy, profile)
        if shape in ("zero_signs", "twins_zero") and kind == "scan":
            a = got[1][list(X.result_keys(g.make_plan(group_cols=[(0, 0)]), [g.GX_INT4], got[0], got[2])).index((5,))]
            signs = np.signbit(a[:4]).tolist()
            # group 0 (x = -0): +0, -0, +0, -0 for zero_signs; sum(x + -0.0) = -0 next to sum(x + 0.0) = +0 for twins_zero
            assert signs == ([False, True, False, True] if shape == "zero_signs" else [False, True, False, False]), (shape, a[:4])
    finally:
        d.free()


def test_zz_every_family_answered_somewhere(request):
    """runs last: every kernel family this module forces answered at least one case.  Judged only when the whole
    module was selected (not under -k or a partial selection)."""
    ids = [it.nodeid.split("::")[-1] for it in request.session.items]
    need = {"test_quals_on_every_family": 2 * len(QUAL_FAMILIES), "test_expression": len(EXPR_CASES),
            "test_one_qual_routes_to_a_kernel_that_evaluates_it": len(REROUTE), "test_build_and_probe_quals": 2 * len(BUILD_PATHS),
            "test_filter_every_operator_and_constant": 2}
    if any(sum(i.startswith(t + "[") for i in ids) < n for t, n in need.items()):
        pytest.skip("not every case of this module was selected")
    want = {v[5] for v in QUAL_FAMILIES.values()} | {v[4] for v in EXPR_FAMILIES.values()} | REROUTE_NAMES
    want |= {"filter", "probe_agg", "build_direct", "build_bucket1", "runagg_dense", "runagg_small2", "runagg_wide"}
    assert SEEN >= want, f"families that never ran: {sorted(want - SEEN)}"
