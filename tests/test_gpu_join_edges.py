"""Every join-table build path and the kernels that probe it, at key-value and key-multiplicity edges, against the
exact numpy join of tests/join_ref.py (itself pinned to the oracle by tests/test_join_ref_cpu.py).

gx_hash_build picks its path from the data: direct CAS insertion (small build sides, and the fallback after a
sub-table overflows), one-pass or two-level bucketing, or the key-ordered build with bounds from a pass over the
column or from a search; slots come from the mixing hash or a 32-bit / 64-bit interpolation, in 16-byte or compact
8-byte form.  Each path is forced here by size, layout and switch, and its profile name (and slot_mode) proves it
ran.  Key sets: negative and zero-crossing keys, INT32 and INT64 limits, INT64_MIN rows, dense blocks on both sides
of the interpolation guard (+-9e18), key spans across the compact form's 2^31 offset and the 32-bit / 64-bit switch
at 2^32, outliers the key sample misses.  Probe sides mix hits, misses, NULL keys, keys just outside the build span,
build keys +- 2^31 / 2^32 (the same home slot and stored bits in the compact form: they must not match) and int4
keys against int8 build keys.  Build sides with one key repeated up to and past what a 2048-slot sub-table holds
must either match the reference or be declined with GX_ERR_ARG."""
import zlib

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O
import exact_ref as X
import join_ref as J
from helpers import to_gpu_plan

pytestmark = pytest.mark.gpu

I64, I32 = np.iinfo(np.int64), np.iinfo(np.int32)
SUB = 2048
SEEN = set()                        # profile names that answered somewhere in this module
ALL_JT = [g.GX_JOIN_INNER, g.GX_JOIN_LEFT, g.GX_JOIN_SEMI, g.GX_JOIN_ANTI]


def dense(start, n, step):
    return np.int64(start) + np.arange(n, dtype=np.int64) * np.int64(step)


# key set: (sorted keys of n rows, fits int4, slot function the sample must choose: True interpolation, False the
# mixing hash, None either)
KEYSETS = {
    "negative":  (lambda n: dense(-3 * n - 17, n, 3), True, True),
    "cross0":    (lambda n: dense(-(n // 2) * 5, n, 5), True, True),
    "i32min":    (lambda n: dense(I32.min, n, 3), True, True),
    "i32max":    (lambda n: dense(I32.max - 3 * (n - 1), n, 3), True, True),
    "i64max":    (lambda n: dense(I64.max - 2 * (n - 1), n, 2), False, False),
    "i64min1":   (lambda n: dense(I64.min + 1, n, 2), False, False),
    "guard_in":  (lambda n: dense(9 * 10**18 - 4 * n - 2**22, n, 4), False, True),
    "guard_in_neg": (lambda n: dense(-9 * 10**18 + 2**22, n, 4), False, True),
    "guard_out": (lambda n: dense(9 * 10**18 + 2**12, n, 4), False, False),
    "guard_out_neg": (lambda n: dense(-9 * 10**18 - 4 * n - 2**12, n, 4), False, False),
    "with_min":  (lambda n: np.concatenate([[I64.min], dense(1, n - 1, 4)]), False, None),
    "outliers":  (lambda n: np.sort(np.concatenate([dense(10**6, n - 4, 4), [-10**15, -10**12, 10**12, 10**15]])), False, None),
}

# build path: (rows, shuffled, int4 key column, NULL keys, switches, profile names that must run, names that must not,
# slot_mode when the sample chooses interpolation, slot_mode under the mixing hash)
PATHS = {
    "direct":          (20_000, True, False, False, {}, {"build_direct"}, set(), 0, 0),
    "direct_forced":   (200_000, False, False, False, {"GX_BUILD_DIRECT": "1"}, {"build_direct"}, {"build_sorted_search"}, 1, 0),
    "bucket1_hash":    (200_000, True, False, False, {"GX_SLOT_MODE": "0"}, {"build_bucket1"}, {"build_direct"}, 0, 0),
    "bucket1":         (200_000, True, False, False, {}, {"build_bucket1"}, {"build_direct"}, 1, 0),
    "bucket1_nulls":   (200_000, False, False, True, {}, {"build_bucket1"}, {"build_direct"}, 1, 0),
    "bucket1_nosort":  (200_000, False, False, False, {"GX_BUILD_NOSORTED": "1"}, {"build_bucket1"}, {"build_sorted_search"}, 1, 0),
    "bucket2":         (3_000_000, True, False, False, {}, {"build_bucket2"}, {"build_bucket1", "build_direct"}, 1, 0),
    "bucket2_onepass": (3_000_000, True, False, False, {"GX_BUILD_ONEPASS": "1"}, {"build_bucket1"}, {"build_bucket2"}, 1, 0),
    "sorted_search":   (200_000, False, False, False, {}, {"build_sorted_search", "build_compact"}, {"build_bucket1"}, 2, 0),
    "sorted_wide":     (200_000, False, False, False, {"GX_NO_COMPACT": "1"}, {"build_sorted_search"}, {"build_compact"}, 2, 0),
    "sorted_pass":     (200_000, False, False, False, {"GX_NO_BOUNDS_SEARCH": "1"}, {"build_sorted_pass", "build_compact"}, {"build_sorted_search"}, 2, 0),
    "sorted_slot64":   (200_000, False, False, False, {"GX_SLOT_WIDE": "1"}, {"build_sorted_search", "build_compact"}, set(), 2, 0),
    "sorted_int4":     (200_000, False, True, False, {}, {"build_sorted_pass"}, {"build_compact"}, 2, 0),
}
BIG_KEYSETS = ["cross0", "i64max", "guard_in"]          # the 3 M-row paths run these only
PATH_NAMES = {"build_direct", "build_bucket1", "build_bucket2", "build_sorted_pass", "build_sorted_search", "build_compact", "build_expand"}


def probe_keys(rng, bk, n, int4):
    """hits, misses, the span's ends and just outside, build keys +- 2^31 / 2^32, INT64_MIN, INT64_MAX"""
    real = bk[bk != I64.min]
    lo, hi = int(real.min()), int(real.max())
    with np.errstate(over="ignore"):
        parts = [rng.choice(bk, n // 2), rng.choice(real, n // 8) + 1, rng.choice(real, n // 8) - 1]
        for d in (2**31, 2**32):
            parts += [rng.choice(real, n // 16) + np.int64(d), rng.choice(real, n // 16) - np.int64(d)]
    ends = [lo, hi, I64.min, I64.max, 0, -1]
    ends += [v for v in (lo - 1, hi + 1) if I64.min < v <= I64.max]
    k = np.concatenate(parts + [np.array(ends, np.int64)]).astype(np.int64)
    if int4:
        k = k[(k >= I32.min) & (k <= I32.max)]
    return rng.permutation(k)


def read_rows(t):
    out = []
    for c in range(len(t.types)):
        v, nl = t.read(c, with_nulls=True)
        out.append(np.where(nl == 0, v.astype(np.int64), J.NULL))
    w = np.stack(out, 1) if out else np.zeros((t.nrows, 0), np.int64)
    return w[np.lexsort(w.T[::-1])] if len(w) else w


def build(gx, keys, nulls=None, int4=False, unique=True, pay=None):
    """build with payload = an int4 column; returns (ht, payload column, profile names that ran, build table)"""
    n = len(keys)
    pay = (np.arange(n, dtype=np.int64) * 7 - 3).astype(np.int32) if pay is None else pay
    kt = g.GX_INT4 if int4 else g.GX_INT8
    t = gx.table_from([kt, g.GX_INT4], [keys.astype(np.int32) if int4 else keys, pay], [nulls, None])
    gx.profile(True)
    ht = gx.hash_build(t, 0, [1], unique=unique)
    ran = {p for p in PATH_NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    SEEN.update(ran)
    return ht, pay, ran, t


def check_probes(gx, rng, ht, bkeys, bnull, pay, unique, nprobe, jts=ALL_JT, int4_outer=(False, True)):
    for int4 in int4_outer:
        ok = probe_keys(rng, bkeys[bnull == 0] if bnull is not None else bkeys, nprobe, int4)
        if len(ok) == 0:
            continue
        onull = (rng.random(len(ok)) < 0.03).astype(np.uint8)
        oval = np.arange(len(ok), dtype=np.int32)
        ot = gx.table_from([g.GX_INT4 if int4 else g.GX_INT8, g.GX_INT4], [ok.astype(np.int32) if int4 else ok, oval], [onull, None])
        for jt in jts:
            if jt == g.GX_JOIN_LEFT and not unique:
                continue
            semi = jt in (g.GX_JOIN_SEMI, g.GX_JOIN_ANTI)
            gx.profile(True)
            got = gx.hash_probe(ot, 0, ht, [0, 1], join_type=jt)
            if gx.profile_get("build_expand")[1] > 0:
                SEEN.add("build_expand")
            gx.profile(False)
            want = J.rows(J.join(jt, ok, bkeys, onull, bnull), [ok, oval], [] if semi else [pay], [onull, None])
            rows = read_rows(got)
            got.free()
            assert rows.shape == want.shape, f"join type {jt}, int4 outer {int4}: {rows.shape[0]} rows, want {want.shape[0]}"
            np.testing.assert_array_equal(rows, want, err_msg=f"join type {jt}, int4 outer {int4}")
        ot.free()


def _path_cases():
    out = []
    for p, spec in PATHS.items():
        for k, (gen, fits4, interp) in KEYSETS.items():
            if spec[2] and not fits4:
                continue
            if spec[0] > 1_000_000 and k not in BIG_KEYSETS:
                continue
            out.append((p, k))
    return out


@pytest.mark.parametrize("unique", [True, False])
@pytest.mark.parametrize("path,keyset", _path_cases())
def test_build_path_and_probe(gx, monkeypatch, path, keyset, unique):
    n, shuffled, int4, has_nulls, env, must, must_not, mode_interp, mode_hash = PATHS[path]
    gen, _, interp = KEYSETS[keyset]
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(zlib.crc32(f"{path}/{keyset}/{unique}".encode()))
    keys = gen(n)
    if not unique:                                       # every 5th key twice, every 50th three times; more INT64_MIN rows
        extra = [keys[::5], keys[::50]] + ([np.full(3, I64.min)] if keyset == "with_min" else [])
        keys = np.sort(np.concatenate([keys] + extra))
    if shuffled:
        keys = rng.permutation(keys)
    bnull = (rng.random(len(keys)) < 0.02).astype(np.uint8) if has_nulls else None
    ht, pay, ran, bt = build(gx, keys, bnull, int4, unique)
    info = ht.info()
    if interp is not None:
        # a clean key-ordered build keeps the sampled choice; a unique key-ordered side could also be refused only
        # for long chains, which dense keys do not produce
        want_mode = mode_interp if interp else mode_hash
        assert info["slot_mode"] == want_mode, f"{path}/{keyset}: slot_mode {info['slot_mode']}, want {want_mode} ({sorted(ran)})"
        if interp or not (must & {"build_sorted_search", "build_sorted_pass", "build_compact"}):
            assert must <= ran, f"{path}/{keyset}: {sorted(must - ran)} did not run ({sorted(ran)})"
            assert not (must_not & ran), f"{path}/{keyset}: {sorted(must_not & ran)} ran"
    assert ht.nentries == (len(keys) if bnull is None else int((bnull == 0).sum()))
    check_probes(gx, rng, ht, keys, bnull, pay, unique, min(len(keys), 100_000))
    ht.free(); bt.free()


# ---------------------------------------------------------------- aggregates over the join
C = g.GX_OP_COL
SX, CNT = (g.GX_AGG_SUM_F8, [(C, 1, 0)]), (g.GX_AGG_COUNT_STAR, [])
# family: (switches, strategy, group by the key (runagg) or the payload, profile name)
AGG_FAMILIES = {
    "probe_agg_fast": ({"GX_NO_RUNJOIN": "1"}, 0, False, "probe_agg_fast"),
    "probe_agg_run":  ({"GX_RUNJOIN_TMA": "0", "GX_RUNJOIN_SEG": "0"}, 0, False, "probe_agg_run"),
    "probe_agg_tma1": ({"GX_RUNJOIN_TMA": "1"}, 0, False, "probe_agg_tma"),
    "probe_agg_tma2": ({"GX_RUNJOIN_TMA": "2"}, 0, False, "probe_agg_tma"),
    "probe_agg_tma3": ({"GX_RUNJOIN_TMA": "3"}, 0, False, "probe_agg_tma"),
    "probe_agg_seg":  ({"GX_RUNJOIN_TMA": "0", "GX_RUNJOIN_SEG": "1"}, 0, False, "probe_agg_seg"),
    "probe_agg_run2": ({"GX_RUNJOIN_V2": "1"}, 0, False, "probe_agg_run2"),
    "probe_agg_run3": ({"GX_RUNJOIN_CARRY": "1"}, 0, False, "probe_agg_run3"),
    "runagg":         ({}, 0, True, "runagg"),
    "records_smem":   ({}, 1, False, "agg_smem"),
    "records_radix":  ({}, 2, False, "probe_records"),
    "records_global": ({}, 3, False, "agg_global"),
}
AGG_KEYSETS = ["negative", "cross0", "i32max", "guard_in", "i64max"]


@pytest.mark.parametrize("keyset", AGG_KEYSETS)
@pytest.mark.parametrize("family", list(AGG_FAMILIES))
def test_join_aggregate(gx, monkeypatch, family, keyset):
    """sum(x), count(*) over an INNER join with a unique key-ordered build side (compact where the keys allow), the
    outer side clustered on the key; its aliases (+-2^31, +-2^32) and misses must fall out of every group"""
    env, strategy, by_key, prof = AGG_FAMILIES[family]
    if family == "probe_agg_seg" and not KEYSETS[keyset][2]:
        pytest.skip("the streamed-table kernel reads compact tables, which need order-preserving slots")
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(len(family) * 31 + len(keyset))
    n = 200_000
    keys = KEYSETS[keyset][0](n)
    G = 997
    pay = (np.arange(n) % G * 13 - 6000).astype(np.int32)
    ht, pay, ran, bt = build(gx, keys, pay=pay)
    no = 60_000 if by_key else 300_000
    ok = probe_keys(rng, keys, no, False)
    ok = np.sort(ok[ok != I64.min])                       # clustered on the key, as lineitem is
    x = rng.standard_normal(len(ok)) * 10.0 ** rng.integers(-3, 4, len(ok))
    ot = gx.table_from([g.GX_INT8, g.GX_FLOAT8], [ok, x])
    # the records families get a min() too: with sum + count(*) alone the plan has the fast kernels' shape
    aggs = [SX, CNT] + ([(g.GX_AGG_MIN_F8, [(C, 1, 0)])] if strategy else [])
    plan = O.make_plan(outer_key_col=0, group_cols=[(0, 0)] if by_key else [(1, 0)], aggs=aggs, est_groups=1000, strategy=strategy)
    want = J.expect_groups(plan, J.join(g.GX_JOIN_INNER, ok, keys), [ok, x], [g.GX_INT8, g.GX_FLOAT8], [pay], [g.GX_INT4])
    gx.profile(True)
    got = gx.hash_agg(ot, to_gpu_plan(plan), ht).fetch()
    used = gx.profile_get(prof)[1]
    if gx.profile_get("build_expand")[1] > 0:
        SEEN.add("build_expand")
    gx.profile(False)
    assert used > 0, f"{family}/{keyset}: {prof} did not run"
    SEEN.add(prof)
    X.check(plan, want, got, [g.GX_INT8 if by_key else g.GX_INT4])
    ot.free(); ht.free(); bt.free()


# ---------------------------------------------------------------- key multiplicity
def mix64(k):
    h = np.asarray(k, np.int64).view(np.uint64).copy()
    with np.errstate(over="ignore"):
        h ^= h >> np.uint64(33); h *= np.uint64(0xff51afd7ed558ccd)
        h ^= h >> np.uint64(33); h *= np.uint64(0xc4ceb9fe1a85ec53)
        h ^= h >> np.uint64(33)
    return h


def hash_sub(keys, nslots):
    """sub-table of each key under the mixing hash (gx_slot_index mode 0)"""
    return (mix64(keys) & np.uint64(nslots - 1)) >> np.uint64(11)


def skewed_side(rng, m, nfill, hot=123456789):
    """one key repeated m times + nfill distinct filler keys that hash into other sub-tables than the hot key's: the
    hot key's sub-table gets exactly m rows"""
    n = m + nfill
    nslots = 1
    while nslots < n + n // 2 + 16:
        nslots *= 2
    cand = rng.integers(-2**60, 2**60, 3 * nfill + 1000)
    cand = np.unique(cand[cand != hot])
    cand = cand[hash_sub(cand, nslots) != hash_sub([hot], nslots)[0]]
    keys = rng.permutation(np.concatenate([np.full(m, hot, np.int64), rng.choice(cand, nfill, replace=False)]))
    return keys, hot


def assert_declined(gx, err, m=None):
    """declined as too skewed (m: the row count the message must give); the context is still usable"""
    assert err.status == g.GX_ERR_ARG, err
    assert "sub-table" in str(err) and (m is None or f" {m} build rows" in str(err)), str(err)
    t = gx.table_from([g.GX_INT8, g.GX_INT4], [np.arange(100, dtype=np.int64), np.arange(100, dtype=np.int32)])
    ht = gx.hash_build(t, 0, [1], unique=True)
    o = gx.table_from([g.GX_INT8, g.GX_INT4], [np.arange(-5, 5, dtype=np.int64), np.zeros(10, np.int32)])
    r = gx.hash_probe(o, 0, ht, [0])
    assert r.nrows == 5
    for x in (r, o, ht, t):
        x.free()


@pytest.mark.parametrize("m", [2046, 2047, 2048, 5000])
@pytest.mark.parametrize("size,path", [(3000, "build_direct"), (60_000, "build_bucket1")])
def test_heavy_duplicates(gx, m, size, path):
    """a sub-table holds at most 2047 rows: up to there the join matches the reference, past it the build is
    declined (the direct build after the bucketed one overflowed, too) and the context stays usable"""
    rng = np.random.default_rng(m + size)
    keys, hot = skewed_side(rng, m, size)
    t_keys = keys
    if m <= SUB - 1:
        ht, pay, ran, bt = build(gx, t_keys, unique=False)
        assert path in ran, sorted(ran)
        if path != "build_direct":
            assert "build_direct" not in ran, sorted(ran)
        assert ht.nentries == len(keys)
        check_probes(gx, rng, ht, keys, None, pay, False, 4_000, jts=[g.GX_JOIN_INNER, g.GX_JOIN_SEMI, g.GX_JOIN_ANTI],
                     int4_outer=(False,))
        # the hot key itself, many times
        ot = gx.table_from([g.GX_INT8, g.GX_INT4], [np.full(7, hot, np.int64), np.arange(7, dtype=np.int32)])
        got = gx.hash_probe(ot, 0, ht, [0, 1])
        assert got.nrows == 7 * m
        got.free(); ot.free(); ht.free(); bt.free()
    else:
        t = gx.table_from([g.GX_INT8, g.GX_INT4], [t_keys, np.zeros(len(keys), np.int32)])
        gx.profile(True)
        with pytest.raises(g.GxError) as ei:
            gx.hash_build(t, 0, [1], unique=False)
        ran = {p for p in PATH_NAMES if gx.profile_get(p)[1] > 0}
        gx.profile(False)
        assert path in ran and "build_direct" in ran, sorted(ran)
        t.free()
        assert_declined(gx, ei.value, m)


@pytest.mark.parametrize("m", [SUB - 1, SUB])
def test_key_ordered_duplicates_fill_one_sub_table(gx, m):
    """a key-ordered non-unique side whose one key fills a whole sub-table's row range (no other key within several
    sub-tables' key spans): 2047 copies are built key-ordered and compact, 2048 are declined"""
    n = 1_500_000
    keys = dense(0, n, 4)
    hot = int(keys[n // 2])
    keys = keys[np.abs(keys - hot) > 200_000]
    keys = np.sort(np.concatenate([keys, np.full(m, hot, np.int64)]))
    t = gx.table_from([g.GX_INT8], [keys])
    gx.profile(True)
    try:
        ht = gx.hash_build(t, 0, [], unique=False)
    except g.GxError as e:
        gx.profile(False)
        assert m == SUB, f"{m} copies declined: {e}"
        t.free()
        assert_declined(gx, e)          # the mixing-hash rebuild adds the hot sub-table's other rows to the count
        return
    ran = {p for p in PATH_NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    SEEN.update(ran)
    assert m < SUB, "a full sub-table was accepted"
    assert ht.info()["slot_mode"] == 2 and {"build_sorted_search", "build_compact"} <= ran, (ht.info(), sorted(ran))
    rng = np.random.default_rng(m)
    check_probes(gx, rng, ht, keys, None, np.arange(len(keys), dtype=np.int64), False, 200_000,
                 jts=[g.GX_JOIN_INNER, g.GX_JOIN_SEMI, g.GX_JOIN_ANTI], int4_outer=(False,))
    ht.free(); t.free()


# ---------------------------------------------------------------- spans of the compact form and the slot functions
@pytest.mark.parametrize("case", ["offset_2_31", "span_below_2_32", "span_above_2_32", "shuffled_above_2_32"])
def test_wide_key_spans(gx, case):
    """compact tables whose key offsets pass 2^31 (the expanded 16-byte form must rebuild every key: its wrap
    correction), and spans just below / above 2^32 where the interpolation switches from 32-bit to 64-bit
    arithmetic; the shuffled one is built by two-level bucketing with the sampled slot function"""
    rng = np.random.default_rng(len(case))
    span = {"offset_2_31": 2**31 + 2**24, "span_below_2_32": 2**32 - 2**20 - 256, "span_above_2_32": 2**32 + 2**20,
            "shuffled_above_2_32": 2**32 + 2**20}[case]
    kmin = -(2**31) - 12345
    n = span // 256 + 1
    keys = dense(kmin, n, 256)
    keys[-1] = kmin + span - 1                            # the exact span
    keys = np.sort(np.concatenate([keys, keys[::97]]))    # non-unique: INNER reads the expanded form
    if case.startswith("shuffled"):
        keys = rng.permutation(keys)
    t = gx.table_from([g.GX_INT8], [keys])
    gx.profile(True)
    ht = gx.hash_build(t, 0, [], unique=False)
    ran = {p for p in PATH_NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    SEEN.update(ran)
    if case.startswith("shuffled"):
        assert "build_bucket2" in ran and ht.info()["slot_mode"] == 1, (ht.info(), sorted(ran))
    else:
        assert ht.info()["slot_mode"] == 2 and "build_compact" in ran, (ht.info(), sorted(ran))
    check_probes(gx, rng, ht, keys, None, np.arange(len(keys), dtype=np.int64), False, 2_000_000,
                 jts=[g.GX_JOIN_INNER, g.GX_JOIN_SEMI, g.GX_JOIN_ANTI], int4_outer=(False,))
    ht.free(); t.free()


def test_zz_every_path_and_family_ran(request):
    """runs last: a dispatch change that silently reroutes shows up as a build path or probe family nobody reached.
    Judged only when the whole module was selected."""
    ids = {it.nodeid.split("::")[-1] for it in request.session.items}
    if not all(any(i.startswith(f"test_join_aggregate[{f}-") for i in ids) for f in AGG_FAMILIES) or \
            not any(i.startswith("test_build_path_and_probe[") for i in ids) or "test_heavy_duplicates[3000-build_direct-2047]" not in ids:
        pytest.skip("not every case of this module was selected")
    want = PATH_NAMES | {f[3] for f in AGG_FAMILIES.values()}
    assert SEEN >= want, f"never ran: {sorted(want - SEEN)}"
