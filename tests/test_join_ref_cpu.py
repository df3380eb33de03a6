"""tests/join_ref.py pinned to the oracle's ExecHashJoinImpl restatement (exec_join / exec_agg), without a GPU, on
small inputs carrying every key edge the GPU join tests use: negative keys and keys crossing zero, INT32 and INT64
limits, INT64_MIN on both sides (an ordinary value), NULL keys, duplicates, keys that differ by 2^31 or 2^32, int4
outer keys against int8 build keys, and quals on both sides."""
import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import join_ref as J

I64, I32 = np.iinfo(np.int64), np.iinfo(np.int32)
JOIN_TYPES = [g.GX_JOIN_INNER, g.GX_JOIN_LEFT, g.GX_JOIN_SEMI, g.GX_JOIN_ANTI]


def _build_keys(rng, unique):
    base = np.array([I64.min, I64.min + 1, I64.max, I64.max - 1, I32.min, I32.max, I32.min - 1, I32.max + 1,
                     -1, 0, 1, -(2**31), 2**31, 2**32, -(2**32), 5, 5 + 2**32, 9 * 10**18, -9 * 10**18], np.int64)
    k = np.concatenate([base, rng.integers(-300, 300, 60)])
    k = np.unique(k)
    if not unique:
        k = np.concatenate([k, k[rng.integers(0, len(k), 80)], [I64.min] * 3])
    return rng.permutation(k)


def _outer_keys(rng, bk, int4):
    near = np.concatenate([bk, bk + 1, bk - 1, bk + 2**31, bk - 2**31, bk + 2**32, bk - 2**32])
    k = np.concatenate([rng.choice(near, 400), rng.integers(-400, 400, 200), [I64.min, I64.max, 0]])
    if int4:
        k = k[(k >= I32.min) & (k <= I32.max)]
    return k


@pytest.mark.parametrize("unique", [True, False])
@pytest.mark.parametrize("int4_outer", [False, True])
def test_rows_match_the_oracle(unique, int4_outer):
    rng = np.random.default_rng(7 + unique + 2 * int4_outer)
    bk = _build_keys(rng, unique)
    nb = len(bk)
    bnull = (rng.random(nb) < 0.05).astype(np.uint8)
    bpay = rng.integers(-1000, 1000, nb).astype(np.int32)
    bq = rng.integers(0, 10, nb).astype(np.int32)
    ok = _outer_keys(rng, bk, int4_outer)
    no = len(ok)
    onull = (rng.random(no) < 0.05).astype(np.uint8)
    oval = np.arange(no, dtype=np.int32)
    ox = rng.standard_normal(no)
    okt = g.GX_INT4 if int4_outer else g.GX_INT8
    ot, it = [okt, g.GX_INT4, g.GX_FLOAT8], [g.GX_INT8, g.GX_INT4, g.GX_INT4]
    ocols, icols = [ok.astype(np.int32) if int4_outer else ok, oval, ox], [bk, bpay, bq]
    orel, irel = O.Rel(ot, ocols, [onull, None, None]), O.Rel(it, icols, [bnull, None, None])
    opreds, ipreds = [(2, g.GX_LT, 1.0, True)], [(2, g.GX_GE, 2)]
    okeep, ikeep = J.quals(ocols, None, opreds, no), J.quals(icols, None, ipreds, nb)
    for jt in JOIN_TYPES:
        join = O.make_join(0, payload_cols=[1], inner_unique=int(unique), inner_preds=ipreds, jointype=jt)
        w = O.exec_join(orel, 0, irel, join, [0, 1], outer_preds=opreds)
        semi = jt in (g.GX_JOIN_SEMI, g.GX_JOIN_ANTI)
        want = np.stack(w[:2] if semi else w, 1)
        want = want[np.lexsort(want.T[::-1])]
        pairs = J.join(jt, ocols[0], bk, onull, bnull, okeep, ikeep)
        got = J.rows(pairs, [ocols[0], oval], [] if semi else [bpay], [onull, None])
        np.testing.assert_array_equal(got, want, err_msg=f"join type {jt}")
    assert len(J.join(g.GX_JOIN_INNER, ocols[0], bk, onull, bnull)[0]) > 50


@pytest.mark.parametrize("unique", [True, False])
def test_groups_match_the_oracle(unique):
    """count(*), sum(int4) and an exact float8 sum over an INNER join, grouped by a payload column and by the key"""
    rng = np.random.default_rng(11 + unique)
    bk = _build_keys(rng, unique)
    nb = len(bk)
    bpay = rng.integers(-3, 3, nb).astype(np.int32)
    ok = _outer_keys(rng, bk, False)
    no = len(ok)
    onull = (rng.random(no) < 0.05).astype(np.uint8)
    ov = rng.integers(I32.min, I32.max, no, endpoint=True).astype(np.int32)
    ox = rng.standard_normal(no) * 10.0 ** rng.integers(-5, 5, no)
    ot, it = [g.GX_INT8, g.GX_INT4, g.GX_FLOAT8], [g.GX_INT8, g.GX_INT4]
    ocols = [ok, ov, ox]
    aggs = [(g.GX_AGG_COUNT_STAR, []), (g.GX_AGG_SUM_I4, [(g.GX_OP_COL, 1, 0)]), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 2, 0)])]
    join = O.make_join(0, payload_cols=[1], inner_unique=int(unique))
    pairs = J.join(g.GX_JOIN_INNER, ok, bk, onull)
    for gc in ([(1, 0)], [(0, 0)], [(0, 0), (1, 0)]):
        plan = O.make_plan(outer_key_col=0, group_cols=gc, aggs=aggs, est_groups=100, preds=[(2, g.GX_GT, -5.0, True)])
        r = O.exec_agg(O.Rel(ot, ocols, [onull, None, None]), plan, O.Rel(it, [bk, bpay]), join)
        want = J.expect_groups(plan, pairs, ocols, ot, [bpay], [g.GX_INT4], outer_nulls=[onull, None, None])
        X.check(plan, want, (r.keys, r.aggs, r.nulls), [g.GX_INT8 if s == 0 else g.GX_INT4 for s, _ in gc])
