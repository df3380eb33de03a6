"""The narrow 4-byte join-table slot: w = tag | (payload - pbase) << tbits, chosen by the key-ordered build of an int8 key
with one int4/date payload column whose sampled range fits the 32 - tbits payload bits (TPC-H orders: o_orderkey,
o_orderdate).  tbits is the smallest width with 2^(tbits-1) >= 4 (keys_per_slot 2048 + 64).

Every table is checked by joining against it (INNER, LEFT, SEMI, ANTI through hash_probe, the first-match probe that
reads the narrow slots directly, and INNER on a non-unique build, which probes the expanded 16-byte slots) and by
count(*) / sum(x) grouped by the payload through hash_agg, against the exact references of tests/join_ref.py and
tests/exact_ref.py.  The profile names build_narrow / build_narrow_refill / build_compact prove which form answered."""
import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import join_ref as J
from helpers import to_gpu_plan

pytestmark = pytest.mark.gpu

I64 = np.iinfo(np.int64)
SUB = 2048
NSAMPLE = 65536
NAMES = {"build_narrow", "build_narrow_refill", "build_compact", "build_fill_staged", "build_fill_rows",
         "build_sorted_search", "build_expand", "probe_agg_tma", "probe_agg_run", "probe_agg_seg", "probe_agg_fast",
         "probe_agg_run2", "probe_agg_run3", "agg_smem", "probe_records", "agg_global"}
# avg_chain of the bunched 3 M-row key set, as pinned in tests/test_gpu_sorted_build.py for the 8-byte form: the narrow
# form places every row where the 8-byte form does
BUNCHED_AVG_CHAIN = 1.2740106666666666


def bunched(n):
    i = np.arange(n, dtype=np.int64)
    return (i // 8) * 32 + (i % 8) + 1


def nslots_of(n):
    s = 1
    while s < n + n // 2 + 16:
        s *= 2
    return s


def tbits_of(keys):
    """the tag width the build derives from the exact key span"""
    n = len(keys)
    kps = (float(keys[-1]) - float(keys[0]) + 1.0) / float(nslots_of(n) - SUB)
    need, t = 4.0 * (kps * SUB + 64.0), 2
    while t < 32 and float(1 << (t - 1)) < need:
        t += 1
    return t


def sampled_rows(n):
    """rows the build's strided sample reads"""
    return np.arange(0, n, max(1, n // NSAMPLE))


def build(gx, keys, pay, ptype=g.GX_INT4, unique=True):
    t = gx.table_from([g.GX_INT8, ptype], [keys, pay])
    gx.profile(True)
    ht = gx.hash_build(t, 0, [1], unique=unique)
    ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    return ht, t, ran


def read_rows(t):
    out = []
    for c in range(len(t.types)):
        v, nl = t.read(c, with_nulls=True)
        out.append(np.where(nl == 0, v.astype(np.int64), J.NULL))
    w = np.stack(out, 1) if out else np.zeros((t.nrows, 0), np.int64)
    return w[np.lexsort(w.T[::-1])] if len(w) else w


def probe_side(rng, keys, n):
    """hits, misses next to hits, keys k +- 2^j (j = 12..20) inside the span, the span's ends and just outside"""
    lo, hi = int(keys[0]), int(keys[-1])
    parts = [rng.choice(keys, n // 2), rng.choice(keys, n // 8) + 1, rng.choice(keys, n // 8) - 1]
    for j in range(12, 21):
        d = np.int64(1 << j)
        parts += [rng.choice(keys, n // 64) + d, rng.choice(keys, n // 64) - d]
    ends = [v for v in (lo, hi, lo - 1, hi + 1, lo - 2, hi + 2, 0, I64.max) if I64.min < v <= I64.max]
    k = np.concatenate(parts + [np.array(ends, np.int64)]).astype(np.int64)
    return rng.permutation(k)


def check_probes(gx, ht, ht_multi, keys, pay, seed, nprobe=100_000):
    rng = np.random.default_rng(seed)
    ok = probe_side(rng, keys, nprobe)
    oval = np.arange(len(ok), dtype=np.int32)
    ot = gx.table_from([g.GX_INT8, g.GX_INT4], [ok, oval])
    cases = [(ht, jt) for jt in (g.GX_JOIN_INNER, g.GX_JOIN_LEFT, g.GX_JOIN_SEMI, g.GX_JOIN_ANTI)]
    if ht_multi is not None:
        cases.append((ht_multi, g.GX_JOIN_INNER))       # every match: the 16-byte slots expanded from the narrow ones
    for h, jt in cases:
        got = gx.hash_probe(ot, 0, h, [0, 1], join_type=jt)
        semi = jt in (g.GX_JOIN_SEMI, g.GX_JOIN_ANTI)
        want = J.rows(J.join(jt, ok, keys), [ok, oval], [] if semi else [pay])
        rows = read_rows(got)
        got.free()
        assert rows.shape == want.shape, f"join type {jt}: {rows.shape[0]} rows, want {want.shape[0]}"
        np.testing.assert_array_equal(rows, want, err_msg=f"join type {jt}")
    ot.free()


def check_agg(gx, ht, keys, pay, ptype, seed, strategy=0, nprobe=300_000):
    """count(*), sum(x) grouped by the payload over an INNER join, the outer side clustered on the key; returns the
    profile names that ran"""
    rng = np.random.default_rng(seed)
    ok = np.sort(probe_side(rng, keys, nprobe))
    x = rng.standard_normal(len(ok)) * 10.0 ** rng.integers(-3, 4, len(ok))
    ot = gx.table_from([g.GX_INT8, g.GX_FLOAT8], [ok, x])
    aggs = [(g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 1, 0)]), (g.GX_AGG_COUNT_STAR, [])]
    if strategy:
        aggs.append((g.GX_AGG_MIN_F8, [(g.GX_OP_COL, 1, 0)]))     # not the fast kernels' shape
    plan = O.make_plan(outer_key_col=0, group_cols=[(1, 0)], aggs=aggs, est_groups=2500, strategy=strategy)
    want = J.expect_groups(plan, J.join(g.GX_JOIN_INNER, ok, keys), [ok, x], [g.GX_INT8, g.GX_FLOAT8], [pay], [ptype])
    gx.profile(True)
    got = gx.hash_agg(ot, to_gpu_plan(plan), ht).fetch()
    ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    X.check(plan, want, got, [ptype])
    ot.free()
    return ran


def check_all(gx, keys, pay, ptype, seed, must, must_not=frozenset()):
    ht, t, ran = build(gx, keys, pay, ptype)
    assert must <= ran and not (must_not & ran), (sorted(ran), ht.info())
    assert ht.info()["slot_mode"] == 2 and ht.nentries == len(keys), ht.info()
    htm, tm, _ = build(gx, keys, pay, ptype, unique=False)
    check_probes(gx, ht, htm, keys, pay, seed)
    assert "probe_agg_tma" in check_agg(gx, ht, keys, pay, ptype, seed)
    htm.free(); tm.free()
    return ht, t, ran


# ---------------------------------------------------------------- TPC-H-shaped tables
@pytest.mark.parametrize("ptype", [g.GX_INT4, g.GX_DATE])
@pytest.mark.parametrize("n", [200_000, 3_000_000])
def test_tpch_shaped(gx, ptype, n):
    """bunched keys (8 of every 32) with a payload of 2406 values (o_orderdate's days, before 2000: negative): narrow,
    staged, and the chain statistics of the 8-byte build of the same keys"""
    keys = bunched(n)
    i = np.arange(n, dtype=np.int64)
    pay = (-2922 + (i * 7919) % 2406).astype(np.int32)
    ht, t, ran = check_all(gx, keys, pay, ptype, n + ptype, {"build_narrow", "build_compact", "build_fill_staged"},
                           {"build_narrow_refill", "build_fill_rows"})
    wide_pay = np.random.default_rng(n).integers(-2**31, 2**31, n).astype(np.int32)     # too wide: the 8-byte form
    h8, t8, ran8 = build(gx, keys, wide_pay)
    assert "build_compact" in ran8 and "build_narrow" not in ran8, sorted(ran8)
    assert ht.info()["avg_chain"] == h8.info()["avg_chain"] and ht.nentries == h8.nentries, (ht.info(), h8.info())
    if n == 3_000_000:
        assert ht.info()["avg_chain"] == BUNCHED_AVG_CHAIN
    h8.free(); t8.free(); ht.free(); t.free()


# ---------------------------------------------------------------- payload edges
@pytest.mark.parametrize("extra", [-1, 0])
@pytest.mark.parametrize("base", [-70_000, -20_000, 0])
def test_payload_span_at_the_window(gx, base, extra):
    """max - min = 2^pbits - 1 fills the window exactly (narrow); 2^pbits does not fit (the 8-byte form).  Both
    extremes sit in rows the strided sample reads; negative and zero-crossing payloads"""
    n = 200_000
    keys = bunched(n)
    pbits = 32 - tbits_of(keys)
    span = (1 << pbits) + extra
    seed = abs(base) + extra + 1
    rng = np.random.default_rng(seed)
    pay = (base + rng.integers(0, span + 1, n)).astype(np.int64)
    rows = sampled_rows(n)
    pay[rows[3]], pay[rows[-5]] = base, base + span
    pay = pay.astype(np.int32)
    if extra < 0:
        ht, t, ran = check_all(gx, keys, pay, g.GX_INT4, seed, {"build_narrow"}, {"build_narrow_refill"})
    else:
        ht, t, ran = build(gx, keys, pay)
        assert "build_compact" in ran and ("build_narrow" not in ran or "build_narrow_refill" in ran), sorted(ran)
        check_probes(gx, ht, None, keys, pay, seed)
        check_agg(gx, ht, keys, pay, g.GX_INT4, seed)
    ht.free(); t.free()


@pytest.mark.parametrize("where", ["above", "below"])
def test_outlier_payload_takes_the_refill(gx, where):
    """one payload far outside the sampled range, in a row the strided sample skips: the fill notices and the table is
    rebuilt in the 8-byte form (build_narrow_refill); answers stay exact"""
    n = 200_000
    keys = bunched(n)
    pay = (np.arange(n) % 2406 - 2922).astype(np.int32)
    r = int(sampled_rows(n)[1000]) + 1
    assert r not in set(sampled_rows(n).tolist())
    pay[r] = 2_000_000_000 if where == "above" else -2_000_000_000
    ht, t, ran = build(gx, keys, pay)
    assert {"build_narrow", "build_narrow_refill", "build_compact"} <= ran, sorted(ran)
    assert ht.info()["slot_mode"] == 2 and ht.nentries == n, ht.info()
    check_probes(gx, ht, None, keys, pay, len(where))
    check_agg(gx, ht, keys, pay, g.GX_INT4, len(where))
    ht.free(); t.free()


# ---------------------------------------------------------------- key edges
def spread(k0, n, span):
    """n sorted distinct keys from k0 to k0 + span - 1, both ends included"""
    return np.int64(k0) + (np.arange(n, dtype=np.int64) * np.int64(span - 1)) // np.int64(n - 1)


@pytest.mark.parametrize("over", [0, 1])
def test_key_span_at_the_tag_boundary(gx, over):
    """key span per sub-table S with 4 (S + 64) = 2^15 exactly: tbits 16 leaves 16 payload bits, which a payload span
    of 2^16 - 1 just fits.  One more key unit per sub-table needs tbits 17, and the same payloads are refused"""
    n = 200_000
    nsub = nslots_of(n) // SUB
    span = ((1 << 13) - 64 + over) * (nsub - 1)
    keys = spread(10**9, n, span)
    assert tbits_of(keys) == 16 + over
    pay = (np.arange(n) * 40503 % 65536 - 30000).astype(np.int32)
    rows = sampled_rows(n)
    pay[rows[7]], pay[rows[-7]] = -30000, 65535 - 30000
    if over:
        ht, t, ran = build(gx, keys, pay)
        assert "build_compact" in ran and "build_narrow" not in ran, sorted(ran)
        check_probes(gx, ht, None, keys, pay, 7)
    else:
        ht, t, ran = check_all(gx, keys, pay, g.GX_INT4, 7, {"build_narrow"}, {"build_narrow_refill"})
    ht.free(); t.free()


@pytest.mark.parametrize("keyset", ["cross0", "guard_in", "guard_in_neg"])
def test_key_edges(gx, keyset):
    """keys crossing zero and dense blocks just inside the +-9e18 interpolation guard"""
    n = 200_000
    start = {"cross0": -(n // 2) * 5, "guard_in": 9 * 10**18 - 4 * n - 2**22, "guard_in_neg": -9 * 10**18 + 2**22}[keyset]
    step = 5 if keyset == "cross0" else 4
    keys = np.int64(start) + np.arange(n, dtype=np.int64) * np.int64(step)
    pay = (np.arange(n) % 997 * 13 - 6000).astype(np.int32)
    ht, t, ran = check_all(gx, keys, pay, g.GX_INT4, len(keyset), {"build_narrow"}, {"build_narrow_refill"})
    ht.free(); t.free()


# ---------------------------------------------------------------- consumers of the expanded 16-byte slots
WIDE = {
    "no_runjoin":     ({"GX_NO_RUNJOIN": "1"}, 0, "probe_agg_fast", True),
    "records_smem":   ({}, 1, "agg_smem", True),
    "records_radix":  ({}, 2, "probe_records", True),
    "records_global": ({}, 3, "agg_global", True),
    "seg":            ({"GX_RUNJOIN_TMA": "0", "GX_RUNJOIN_SEG": "1"}, 0, "probe_agg_seg", False),
    "run":            ({"GX_RUNJOIN_TMA": "0", "GX_RUNJOIN_SEG": "0"}, 0, "probe_agg_run", False),
    "tma2":           ({"GX_RUNJOIN_TMA": "2"}, 0, "probe_agg_tma", False),
    "tma3":           ({"GX_RUNJOIN_TMA": "3"}, 0, "probe_agg_tma", False),
    "run2":           ({"GX_RUNJOIN_V2": "1"}, 0, "probe_agg_run2", False),
    "run3":           ({"GX_RUNJOIN_CARRY": "1"}, 0, "probe_agg_run3", False),
}


@pytest.mark.parametrize("family", list(WIDE))
def test_every_consumer(gx, monkeypatch, family):
    """each aggregate family against a narrow table: the ones that read 16-byte slots get them expanded (every key
    rebuilt from its tag), the run-join kernels read the narrow slots"""
    env, strategy, prof, expands = WIDE[family]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    n = 3_000_000
    keys = bunched(n)
    pay = (-2922 + (np.arange(n) * 7919) % 2406).astype(np.int32)
    ht, t, ran = build(gx, keys, pay, g.GX_DATE)
    assert "build_narrow" in ran, sorted(ran)
    ran = check_agg(gx, ht, keys, pay, g.GX_DATE, len(family), strategy)
    assert prof in ran and ("build_expand" in ran) == expands, sorted(ran)
    ht.free(); t.free()
