"""The key-ordered join-table build for a plain int8 key (gx_k_sorted_fill_staged): one 4-byte payload column (PK 1) or
none (PK 2, the payload is the row number), compact or 16-byte slots, bounds by search or by a pass over the column.
Every table is checked by joining against it and comparing with the exact numpy join of tests/join_ref.py; the second
profile names build_fill_staged / build_fill_rows tell whether the staged kernel or the generic row loader answered.

Most cases use a controlled key layout: keys K0 + d with d in [0, 4095 * 4096) over 2.8 M - 5.6 M rows give a table
of 2^23 slots whose order-preserving slot function is exactly slot = d / 2, so sub-table c holds the rows with
d in [4096 c, 4096 (c + 1)).  That puts any row count (0, 1, 2046, 2047, 2048) into a chosen sub-table, at a chosen
first row (lo mod 4 for the 16-byte aligned stage copies of 8-byte keys and 4-byte payloads), and a descending pair
of rows exactly at the boundary between two sub-tables that one CTA builds one after the other, or between two CTAs'
blocks of sub-tables."""
import numpy as np
import pytest

import opentenbase_b200 as g
import join_ref as J

pytestmark = pytest.mark.gpu

K0 = 1_000_000
SPAN = 4096                      # key units per sub-table in the controlled layout
NSUB = 4096                      # 2^23 slots / 2048
BG = 732                         # background rows per sub-table: 4095 x 732 = 3.0 M rows
# resident CTAs per SM of gx_k_sorted_fill_staged<1, compact, ..> on an H100 (74 KB of shared memory each)
STAGED_CTAS_PER_SM = 3
NAMES = {"build_fill_staged", "build_fill_rows", "build_sorted_search", "build_sorted_pass", "build_compact",
         "build_bucket1", "build_bucket2", "build_direct"}

# avg_chain and nentries of the bunched 3 M-row key set below (TPC-H order keys: 8 used of every 32), as the fill that
# gx_k_sorted_fill_staged replaced (gx_k_sorted_fill<1, true, true>) reported them on an H100.  Linear probing's total
# displacement does not depend on the insertion order, so the staged fill must give the same numbers.
BUNCHED_AVG_CHAIN = 1.2740106666666666
BUNCHED_NENTRIES = 3_000_000


def layout(counts):
    """sorted keys for per-sub-table row counts (len NSUB - 1; the last sub-table is never a home under interpolation).
    Sub-tables of up to 819 rows use offsets 5 j, fuller ones 2 j; the first key is K0 and the last K0 + 4095 * 4096 - 1,
    so the build's exact key span is 4095 * 4096 and slot = d / 2 exactly."""
    counts = np.asarray(counts, np.int64)
    assert len(counts) == NSUB - 1 and counts[0] > 0 and counts[-1] > 0 and counts.max() <= SPAN // 2
    c = np.repeat(np.arange(NSUB - 1, dtype=np.int64), counts)
    j = np.arange(len(c), dtype=np.int64) - np.repeat(np.cumsum(counts) - counts, counts)
    step = np.where(counts[c] <= 819, 5, 2)
    d = c * SPAN + j * step
    d[-1] = (NSUB - 1) * SPAN - 1
    assert np.all(np.diff(d) > 0)
    return K0 + d


def starts(counts):
    return np.concatenate([[0], np.cumsum(counts)])


def align_to(counts, special, a):
    """add 0-3 rows to the background sub-table before each non-empty special one so that it starts at lo = a (mod 4)"""
    for c in sorted(special):
        if counts[c] == 0:
            continue
        k = c - 1
        while k in special:
            k -= 1
        counts[k] += (a - int(np.sum(counts[:c]))) % 4


def bunched(n):
    i = np.arange(n, dtype=np.int64)
    return (i // 8) * 32 + (i % 8) + 1


def build(gx, keys, pk, unique=True):
    n = len(keys)
    pay = (np.arange(n, dtype=np.int64) * 7 - 3).astype(np.int32)
    if pk == 1:
        t = gx.table_from([g.GX_INT8, g.GX_INT4], [keys, pay])
        cols = [1]
    else:
        t = gx.table_from([g.GX_INT8], [keys])
        cols = []
        pay = np.arange(n, dtype=np.int64)
    gx.profile(True)
    ht = gx.hash_build(t, 0, cols, unique=unique)
    ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    return ht, t, pay, ran


def read_rows(t):
    out = []
    for c in range(len(t.types)):
        v, nl = t.read(c, with_nulls=True)
        out.append(np.where(nl == 0, v.astype(np.int64), J.NULL))
    w = np.stack(out, 1) if out else np.zeros((t.nrows, 0), np.int64)
    return w[np.lexsort(w.T[::-1])] if len(w) else w


def check_join(gx, ht, bkeys, pay, seed, jts=(g.GX_JOIN_INNER, g.GX_JOIN_ANTI)):
    """every build key, its neighbours and keys outside the span, against the reference join"""
    rng = np.random.default_rng(seed)
    ok = np.concatenate([bkeys, rng.choice(bkeys, len(bkeys) // 4) + 1, rng.choice(bkeys, len(bkeys) // 4) - 1,
                         [bkeys.min() - 1, bkeys.max() + 1, 0, np.iinfo(np.int64).max]]).astype(np.int64)
    ok = rng.permutation(ok)
    oval = np.arange(len(ok), dtype=np.int32)
    ot = gx.table_from([g.GX_INT8, g.GX_INT4], [ok, oval])
    for jt in jts:
        got = gx.hash_probe(ot, 0, ht, [0, 1], join_type=jt)
        semi = jt in (g.GX_JOIN_SEMI, g.GX_JOIN_ANTI)
        want = J.rows(J.join(jt, ok, bkeys), [ok, oval], [] if semi else [pay])
        rows = read_rows(got)
        got.free()
        assert rows.shape == want.shape, f"join type {jt}: {rows.shape[0]} rows, want {want.shape[0]}"
        np.testing.assert_array_equal(rows, want, err_msg=f"join type {jt}")
    ot.free()


def assert_staged(ht, ran, n, compact=True, searched=True):
    assert ht.info()["slot_mode"] == 2, (ht.info(), sorted(ran))
    assert "build_fill_staged" in ran and "build_fill_rows" not in ran, sorted(ran)
    assert ("build_sorted_search" if searched else "build_sorted_pass") in ran, sorted(ran)
    assert ("build_compact" in ran) == compact, sorted(ran)
    assert ht.nentries == n


# ---------------------------------------------------------------- range sizes and alignments
@pytest.mark.parametrize("a", [0, 1, 2, 3])
@pytest.mark.parametrize("pk", [1, 2])
def test_range_sizes_at_every_alignment(gx, pk, a):
    """sub-tables of 0, 1, 2, 2046 and 2047 rows, empty ones between full ones, each starting at lo = a (mod 4)"""
    counts = np.full(NSUB - 1, BG, np.int64)
    special = {1000: 0, 1001: 1, 1003: 0, 1004: 2046, 1005: 0, 1007: 2047, 1009: 2, 2000: 2047, 2001: 0, 4093: 1}
    for c, m in special.items():
        counts[c] = m
    align_to(counts, special, a)
    keys = layout(counts)
    st = starts(counts)
    assert all(st[c] % 4 == a for c in special if counts[c])
    ht, t, pay, ran = build(gx, keys, pk)
    assert_staged(ht, ran, len(keys))
    check_join(gx, ht, keys, pay, seed=10 * pk + a)
    ht.free(); t.free()


@pytest.mark.parametrize("pk", [1, 2])
def test_range_of_2048_rows_overflows(gx, pk):
    """2048 rows cannot share a sub-table: the staged build raises the overflow flag and the table is rebuilt with the
    mixing hash by bucketing, as for the generic loader"""
    counts = np.full(NSUB - 1, BG, np.int64)
    counts[1500] = 2048
    keys = layout(counts)
    ht, t, pay, ran = build(gx, keys, pk)
    assert "build_fill_staged" in ran and "build_sorted_search" in ran, sorted(ran)
    assert ht.info()["slot_mode"] == 0 and ran & {"build_bucket1", "build_bucket2"}, (ht.info(), sorted(ran))
    assert ht.nentries == len(keys)
    check_join(gx, ht, keys, pay, seed=pk, jts=(g.GX_JOIN_INNER,))
    ht.free(); t.free()


# ---------------------------------------------------------------- order check at stage and CTA boundaries
@pytest.mark.parametrize("where", ["stage", "cta", "cta_last"])
def test_descending_pair_at_a_boundary(gx, where):
    """one descending pair of rows whose first row ends a sub-table's range and whose second starts the next: inside
    one CTA's block (two consecutive stages), at the first sub-table of a CTA's block, or at the first sub-table of the
    last CTA's block.  The fill must notice, the build fall back to bucketing, and the join still be right."""
    counts = np.full(NSUB - 1, BG, np.int64)
    keys = layout(counts)
    st = starts(counts)
    import torch
    grid = STAGED_CTAS_PER_SM * torch.cuda.get_device_properties(0).multi_processor_count
    s = {"cta": NSUB * (grid // 2) // grid, "stage": NSUB * (grid // 2) // grid + 1, "cta_last": NSUB * (grid - 1) // grid}[where]
    r = int(st[s])
    keys[r - 1], keys[r] = keys[r], keys[r - 1]
    ht, t, pay, ran = build(gx, keys, 1)
    assert {"build_sorted_search", "build_fill_staged"} <= ran, sorted(ran)
    assert ht.info()["slot_mode"] != 2 and ran & {"build_bucket1", "build_bucket2"}, (ht.info(), sorted(ran))
    assert ht.nentries == len(keys)
    check_join(gx, ht, keys, pay, seed=len(where), jts=(g.GX_JOIN_INNER,))
    ht.free(); t.free()


# ---------------------------------------------------------------- every instantiation
@pytest.mark.parametrize("n", [200_000, 3_000_000])
@pytest.mark.parametrize("searched", [True, False])
@pytest.mark.parametrize("compact", [True, False])
@pytest.mark.parametrize("pk", [1, 2])
def test_every_instantiation(gx, monkeypatch, pk, compact, searched, n):
    """PK 1 / 2 x compact / 16-byte x searched / passed bounds; at 3 M rows every CTA builds several sub-tables, so
    every boundary between two CTAs' blocks and the last CTA's block are inside the checked table"""
    if not compact:
        monkeypatch.setenv("GX_NO_COMPACT", "1")
    if not searched:
        monkeypatch.setenv("GX_NO_BOUNDS_SEARCH", "1")
    keys = bunched(n)
    ht, t, pay, ran = build(gx, keys, pk)
    assert_staged(ht, ran, n, compact, searched)
    check_join(gx, ht, keys, pay, seed=n + pk)
    ht.free(); t.free()


def test_generic_loader_answers_other_shapes(gx):
    """an 8-byte payload is not a staged shape: gx_k_sorted_fill (the generic row loader) builds it"""
    n = 200_000
    keys = bunched(n)
    pay8 = np.arange(n, dtype=np.int64) * 3 - 5
    t = gx.table_from([g.GX_INT8, g.GX_INT8], [keys, pay8])
    gx.profile(True)
    ht = gx.hash_build(t, 0, [1], unique=True)
    ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    assert "build_fill_rows" in ran and "build_fill_staged" not in ran and ht.info()["slot_mode"] == 2, sorted(ran)
    check_join(gx, ht, keys, pay8, seed=5)
    ht.free(); t.free()


# ---------------------------------------------------------------- chain statistics
def test_chain_statistics_unchanged(gx):
    n = 3_000_000
    keys = bunched(n)
    pay = np.random.default_rng(20261015).integers(-2**31, 2**31, n).astype(np.int32)
    t = gx.table_from([g.GX_INT8, g.GX_INT4], [keys, pay])
    gx.profile(True)
    ht = gx.hash_build(t, 0, [1], unique=True)
    ran = {p for p in NAMES if gx.profile_get(p)[1] > 0}
    gx.profile(False)
    assert_staged(ht, ran, n)
    assert ht.info()["avg_chain"] == BUNCHED_AVG_CHAIN
    assert ht.nentries == BUNCHED_NENTRIES
    ht.free(); t.free()
