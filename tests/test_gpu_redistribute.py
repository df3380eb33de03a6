"""The redistribute of table rows (gx_route, gx_partition_by_node, gx_redistribute) on one GPU, against the reference's
routing rule.

The destination of every row is orc_route_node(map, type, key, isnull) of the oracle, which test_oracle_vs_ref.py pins
to the reference's own hashint4 / hashint8 (a NULL key hashes to 0: shard 0).  gx_debug_redistribute runs the
redistribute's own code for one rank of N, with an in-process transport standing in for the peer windows and NCCL: it
routes or partitions every other rank's part with the same device steps that rank would run and delivers what would
have arrived.  Every row carries a unique int8 row id; every output row is matched back to its input row and compared
as a whole tuple (every column, float8 by bit pattern, and every NULL flag), so a column travelling with another row's
columns is caught, not only a lost or duplicated value."""
import ctypes

import numpy as np
import pytest

import opentenbase_b200 as g
import oracle as O

pytestmark = pytest.mark.gpu

I4, I8, F8, DT, CH = g.GX_INT4, g.GX_INT8, g.GX_FLOAT8, g.GX_DATE, g.GX_CHAR
RID0 = 1 << 40                   # row ids: RID0 + index of the row in its Rows
I32, I64 = np.iinfo(np.int32), np.iinfo(np.int64)
NSHARD = 4096                    # GX_SHARD_MAP_SHARD_NUM
_IDENT = np.arange(NSHARD, dtype=np.int32)


@pytest.fixture(scope="module", autouse=True)
def _one_node_map_after(gx):
    yield
    gx.set_shardmap(1)


# ---- the reference's routing rule ----------------------------------------------------------------------------------
def shards(keys, nulls, gx_type):
    """shard index of every row: orc_route_node over the identity map (one oracle call per distinct key)"""
    L, mp = O.lib(), _IDENT.ctypes.data_as(ctypes.c_void_p)
    uniq, inv = np.unique(np.asarray(keys).astype(np.int64), return_inverse=True)
    su = np.array([L.orc_route_node(mp, gx_type, k, 0) for k in uniq.tolist()], np.int32)
    out = su[inv.reshape(-1)] if len(uniq) else np.zeros(0, np.int32)
    if nulls is not None and np.any(nulls):
        out[np.asarray(nulls) != 0] = L.orc_route_node(mp, gx_type, 0, 1)
    return out


def shard_map(kind, n, rng):
    """the 4096-entry map of a map kind: default (i % n), one (every shard on the last node), random, skip (random,
    never node n // 2)"""
    if kind == "default":
        return np.arange(NSHARD, dtype=np.int32) % n
    if kind == "one":
        return np.full(NSHARD, n - 1, np.int32)
    if kind == "random":
        return rng.integers(0, n, NSHARD).astype(np.int32)
    assert kind == "skip" and n > 1
    m = rng.integers(0, n - 1, NSHARD).astype(np.int32)
    return np.where(m >= n // 2, m + 1, m).astype(np.int32)


def install(gx, kind, n, rng):
    m = shard_map(kind, n, rng)
    gx.set_shardmap(n, None if kind == "default" else m)
    return m


# ---- rows -----------------------------------------------------------------------------------------------------------
F8_EDGES = np.array([0x7FF8000000000001, 0xFFF0000000000ABC, 0x8000000000000000, 0x7FF0000000000000,
                     0xFFF0000000000000, 0x0000000000000001, 0x7FEFFFFFFFFFFFFF, 0x3FF0000000000000],
                    np.uint64).view(np.float64)          # NaN payloads, -0.0, +-Inf, the least denormal, DBL_MAX, 1


def key_values(gx_type, n, rng):
    """edge keys of the type, then random ones"""
    if gx_type == I8:
        edges = [0, 1, -1, I32.min, I32.max, I64.min, I64.max, I64.min + 1, I64.max - 1]
        rnd = rng.integers(I64.min, I64.max, n, dtype=np.int64, endpoint=True)
    else:
        edges = [0, 1, -1, I32.min, I32.max, I32.min + 1, I32.max - 1]
        rnd = rng.integers(I32.min, I32.max, n, dtype=np.int64, endpoint=True)
    v = np.concatenate([np.array(edges, np.int64), rnd])[:n]
    return v.astype(g.NP_DTYPES[gx_type])


def column_values(t, n, rng):
    if t == F8:
        v = rng.standard_normal(n) * 10.0 ** rng.integers(-300, 300, n)
        k = min(n, len(F8_EDGES))
        v[:k] = F8_EDGES[:k]
        return rng.permutation(v)
    if t == CH:
        return rng.integers(-128, 128, n).astype(np.int8)
    if t == I8:
        return rng.integers(I64.min, I64.max, n, dtype=np.int64, endpoint=True)
    return rng.integers(I32.min, I32.max, n, dtype=np.int64, endpoint=True).astype(np.int32)


class Rows:
    """rows of one relation: column 0 the row id, column key_col the distribution key; nulls[c] None or uint8"""

    def __init__(self, types, key_col, n, rng, null_cols=(), null_frac=0.2, key_null_frac=0.0):
        self.types, self.key_col, self.n = list(types), key_col, n
        self.cols, self.nulls = [], []
        for c, t in enumerate(types):
            if c == 0:
                v = np.arange(n, dtype=np.int64) + RID0
            elif c == key_col:
                v = rng.permutation(key_values(t, n, rng))
            else:
                v = column_values(t, n, rng)
            self.cols.append(v)
            frac = key_null_frac if c == key_col else null_frac
            self.nulls.append((rng.random(n) < frac).astype(np.uint8) if c in null_cols else None)

    def shards(self):
        return shards(self.cols[self.key_col], self.nulls[self.key_col], self.types[self.key_col])

    def table(self, gx, rows=None, bare=()):
        """a device table of the rows `rows` (all by default); columns in `bare` get no NULL array (their rows must
        hold no NULL there)"""
        rows = np.arange(self.n) if rows is None else rows
        cols = [c[rows] for c in self.cols]
        nulls = [None if (nl is None or c in bare) else nl[rows] for c, nl in enumerate(self.nulls)]
        for c in bare:
            assert self.nulls[c] is None or not self.nulls[c][rows].any()
        return gx.table_from(self.types, cols, nulls if any(x is not None for x in nulls) else None)

    def check(self, got_cols, got_nulls, want_rows, what=""):
        """the output rows (columns, NULL flags) are exactly the rows want_rows, each once, as whole tuples"""
        idx = got_cols[0] - RID0
        assert len(idx) == len(want_rows), f"{what}: {len(idx)} rows, want {len(want_rows)}"
        np.testing.assert_array_equal(np.sort(idx), np.sort(np.asarray(want_rows, np.int64)), err_msg=f"{what}: row ids")
        for c, t in enumerate(self.types):
            wn = np.zeros(len(idx), np.uint8) if self.nulls[c] is None else self.nulls[c][idx]
            np.testing.assert_array_equal(got_nulls[c], wn, err_msg=f"{what}: NULL flags of column {c}")
            live = wn == 0
            gv, wv = got_cols[c][live], self.cols[c][idx][live]
            if t == F8:
                gv, wv = gv.view(np.int64), wv.view(np.int64)
            np.testing.assert_array_equal(gv, wv, err_msg=f"{what}: column {c} (type {t})")


def read_all(t):
    cols, nulls = [], []
    for c in range(len(t.types)):
        v, nl = t.read(c, with_nulls=True)
        cols.append(v); nulls.append(nl)
    return cols, nulls


def sliced(cols, nulls, a, b):
    return [c[a:b] for c in cols], [nl[a:b] for nl in nulls]


# ---- gx_route and gx_partition_by_node: the public two-pass path ----------------------------------------------------
def check_partition(gx, rows, t, m, n, what):
    dest = m[rows.shards()]
    np.testing.assert_array_equal(gx.route(t, rows.key_col), dest, err_msg=f"{what}: gx_route")
    part, counts = gx.partition_by_node(t, rows.key_col, n)
    np.testing.assert_array_equal(counts, np.bincount(dest, minlength=n), err_msg=f"{what}: counts")
    assert part.nrows == rows.n
    cols, nulls = read_all(part)
    off = 0
    for d in range(n):
        rows.check(*sliced(cols, nulls, off, off + counts[d]), np.flatnonzero(dest == d), f"{what}: node {d}")
        off += counts[d]
    part.free()


KEY_TYPES = [I4, I8, DT]
NODES = [1, 2, 3, 7, 8, 64]
MAPS = ["default", "one", "random", "skip"]


@pytest.mark.parametrize("kind", MAPS)
@pytest.mark.parametrize("n", NODES)
@pytest.mark.parametrize("key_type", KEY_TYPES, ids=["int4", "int8", "date"])
def test_route_and_partition_keys_maps(gx, key_type, n, kind):
    if kind == "skip" and n == 1:
        pytest.skip("one node cannot be left out of a one-node map")
    rng = np.random.default_rng([key_type, n, MAPS.index(kind)])
    rows = Rows([I8, key_type, F8, CH, I4, DT, I8], 1, 3000, rng, null_cols=(1, 2, 3, 6), key_null_frac=0.05)
    m = install(gx, kind, n, rng)
    t = rows.table(gx)
    check_partition(gx, rows, t, m, n, f"{kind} map, {n} nodes")
    if kind == "skip":
        assert (gx.route(t, 1) != n // 2).all()
    t.free()


def test_null_keys_go_to_shard_zero(gx):
    """rows whose key is NULL all land on the node of shard 0, whatever datum lies under the NULL flag"""
    rng = np.random.default_rng(5)
    m = install(gx, "random", 7, rng)
    for key_type in KEY_TYPES:
        rows = Rows([I8, key_type], 1, 1000, rng, null_cols=(1,), key_null_frac=1.0)
        t = rows.table(gx)
        np.testing.assert_array_equal(gx.route(t, 1), np.full(1000, m[0], np.int32))
        check_partition(gx, rows, t, m, 7, f"NULL keys of type {key_type}")
        t.free()


@pytest.mark.parametrize("size", [(0, 0), (0, 1), (0, 255), (0, 256), (0, 257), (1, -1), (1, 0), (1, 1)],
                         ids=["0", "1", "255", "256", "257", "S-1", "S", "S+1"])
def test_partition_row_counts(gx, size):
    """row counts at the edges of the route kernels' grid: 256 rows per block, up to sm_count * 4 blocks; size is
    (multiple of sm_count * 4 * 256, rows more)"""
    n = size[0] * gx.device_info()["sm_count"] * 4 * 256 + size[1]
    rng = np.random.default_rng(n)
    m = install(gx, "random", 7, rng)
    rows = Rows([I8, I8, I4, F8, CH], 1, n, rng, null_cols=(1, 3), key_null_frac=0.01)
    t = rows.table(gx)
    check_partition(gx, rows, t, m, 7, f"{n} rows")
    t.free()


ALL16 = [I8, I4, F8, CH, DT, I8, F8, CH, I4, DT, F8, I8, CH, I4, F8, DT]


@pytest.mark.parametrize("nulls", ["none", "all", "some"])
def test_partition_every_column_type(gx, nulls):
    """GX_MAX_COLS columns of every type pass through, with NULL arrays on none, all or some of them"""
    assert len(ALL16) == 16
    rng = np.random.default_rng(len(nulls))
    null_cols = {"none": (), "all": range(1, 16), "some": (2, 3, 7, 9, 14, 15)}[nulls]
    rows = Rows(ALL16, 5, 20000, rng, null_cols=null_cols, key_null_frac=0.02)
    m = install(gx, "skip", 8, rng)
    t = rows.table(gx)
    check_partition(gx, rows, t, m, 8, f"16 columns, NULL arrays on {nulls}")
    t.free()


# ---- gx_redistribute on one node ------------------------------------------------------------------------------------
@pytest.mark.parametrize("two_pass", [False, True])
@pytest.mark.parametrize("n", [0, 1, 5000])
def test_redistribute_one_node(gx, monkeypatch, two_pass, n):
    """without a communicator the redistribute keeps every row: the output is the input as a multiset of tuples"""
    if two_pass:
        monkeypatch.setenv("GX_PARTITION_TWO_PASS", "1")
    rng = np.random.default_rng(n)
    gx.set_shardmap(1)
    rows = Rows([I8, CH, I4, F8, I8, DT], 4, n, rng, null_cols=(1, 3, 4), key_null_frac=0.1)
    t = rows.table(gx)
    out = gx.redistribute(t, 4)
    rows.check(*read_all(out), np.arange(n), f"{n} rows")
    out.free(); t.free()


# ---- gx_debug_redistribute: every rank of N on all three paths ------------------------------------------------------
PATHS = ["windows", "regions", "two_pass"]
WANT_PATH = {"windows": 0, "regions": 1, "two_pass": 2}
# the row id, CHAR and INT4 columns between 8-byte ones (every column of a window region starts at a 256-byte boundary)
DEBUG_TYPES = [I8, CH, F8, I4, None, DT, CH, I8, F8]


@pytest.fixture(params=PATHS)
def path(request, monkeypatch):
    if request.param == "two_pass":
        monkeypatch.setenv("GX_PARTITION_TWO_PASS", "1")
    return request.param


def region_bytes(nrows, n, types, null_cols):
    """bytes of one writer's window region (peer_layout): every column, then every NULL array, 256-byte aligned"""
    cap = nrows // n + nrows // (4 * n) + 4096
    al = lambda b: (b + 255) & ~255
    return sum(al(cap * np.dtype(g.NP_DTYPES[t]).itemsize) for t in types) + sum(al(cap) for _ in null_cols)


def window_for(sizes, n, types, null_cols):
    """a window in which every part's region fits"""
    return n * ((max(region_bytes(s, n, types, null_cols) for s in sizes) + 255) & ~255)


def run_ranks(gx, rows, part_of, n, window, bare=None, want_path=None):
    """redistribute every rank 0..n-1 over the parts; each rank receives exactly the rows routed to it"""
    bare = bare or {}
    tables = [rows.table(gx, np.flatnonzero(part_of == p), bare.get(p, ())) for p in range(n)]
    dest = rows.map[rows.shards()]
    paths = []
    for r in range(n):
        out, got_path = gx.debug_redistribute(tables, rows.key_col, r, window)
        rows.check(*read_all(out), np.flatnonzero(dest == r), f"rank {r} of {n}")
        out.free()
        paths.append(got_path)
    for t in tables:
        t.free()
    if want_path is not None:
        assert paths == [want_path(r) for r in range(n)], paths
    return paths


def debug_rows(gx, n, nrows, rng, key_type=I8):
    types = [key_type if t is None else t for t in DEBUG_TYPES]
    rows = Rows(types, 4, nrows, rng, null_cols=(1, 2, 3, 4, 7), key_null_frac=0.03)
    rows.map = install(gx, "random", n, rng)
    return rows


def uneven_parts(n, nrows, rng):
    """parts of very different sizes, among them an empty one and a one-row one"""
    w = np.array([1.0, 30.0, 1e-9, 0.2, 5.0, 0.01, 12.0, 0.0])[np.arange(n) % 8]
    part_of = rng.choice(n, nrows, p=w / w.sum())
    part_of[:1] = 2 % n                                    # part 2 gets at least one row, part 7 none
    return part_of


DEBUG_N = {2: (I4, 60000), 3: (DT, 60000), 8: (I8, 120000), 64: (I8, 200000)}


@pytest.mark.parametrize("n", sorted(DEBUG_N))
def test_debug_redistribute_every_rank(gx, path, n):
    """parts of very different sizes (each writer chooses its own cap), mixed NULL arrays (some parts have none for
    a column that others have), CHAR and INT4 columns between 8-byte ones; every rank on every path"""
    key_type, nrows = DEBUG_N[n]
    rng = np.random.default_rng([n, PATHS.index(path)])
    rows = debug_rows(gx, n, nrows, rng, key_type)
    part_of = uneven_parts(n, nrows, rng)
    # parts 1, 4, 7, ... carry no NULL array for columns 2 and 7: their rows come back not NULL there
    bare = {p: (2, 7) for p in range(1, n, 3)}
    for p, cols in bare.items():
        for c in cols:
            rows.nulls[c][part_of == p] = 0
    sizes = np.bincount(part_of, minlength=n)
    window = window_for(sizes, n, rows.types, (1, 2, 3, 4, 7)) if path == "windows" else 0
    run_ranks(gx, rows, part_of, n, window, bare, lambda r: WANT_PATH[path])


@pytest.mark.parametrize("n", [2, 3, 8, 64])
def test_debug_redistribute_all_parts_empty(gx, path, n):
    rows = debug_rows(gx, n, 0, np.random.default_rng(n))
    window = window_for([0], n, rows.types, (1, 2, 3, 4, 7)) if path == "windows" else 0
    run_ranks(gx, rows, np.zeros(0, np.int64), n, window, None, lambda r: WANT_PATH[path])


@pytest.mark.parametrize("n", [2, 8])
def test_debug_redistribute_window_too_small(gx, n):
    """a window in which one part's region does not fit: that writer says so in its header and every rank takes the
    NCCL path (one-pass regions)"""
    rng = np.random.default_rng(n + 100)
    rows = debug_rows(gx, n, 50000, rng)
    part_of = uneven_parts(n, 50000, rng)
    sizes = np.bincount(part_of, minlength=n)
    small = sorted(sizes)[-2]                                  # fits every part but the largest
    window = window_for([small], n, rows.types, (1, 2, 3, 4, 7))
    assert region_bytes(sizes.max(), n, rows.types, (1, 2, 3, 4, 7)) > window // n
    run_ranks(gx, rows, part_of, n, window, None, lambda r: 1)


@pytest.mark.parametrize("n", [2, 8])
def test_debug_redistribute_skewed_map_overflows(gx, n):
    """every shard on node 0 and one part larger than its cap (rows/N + rows/(4N) + 4096): that part's window regions
    overflow, so every rank takes the NCCL path, and its one-pass regions overflow as well, so it falls back to the
    two-pass partition; the parts that fit stay on the one-pass regions"""
    rng = np.random.default_rng(n + 200)
    types = [I8, CH, F8, I4, I8, DT, CH, I8, F8]
    big, small = 40000, 300
    rows = Rows(types, 4, big + small * (n - 1), rng, null_cols=(2, 3, 4), key_null_frac=0.03)
    rows.map = np.zeros(NSHARD, np.int32)
    gx.set_shardmap(n, rows.map)
    part_of = np.concatenate([np.zeros(big, np.int64), np.repeat(np.arange(1, n), small)])
    assert big > big // n + big // (4 * n) + 4096
    window = window_for([big], n, types, (2, 3, 4))
    run_ranks(gx, rows, part_of, n, window, None, lambda r: 2 if r == 0 else 1)


# ---- argument errors: GX_ERR_ARG, and the context stays usable -----------------------------------------------------
def test_debug_redistribute_argument_errors(gx):
    rng = np.random.default_rng(7)
    gx.set_shardmap(2)
    rows = Rows([I8, I4, F8, CH, I8], 1, 100, rng, null_cols=(1,))
    a, b = rows.table(gx, np.arange(50)), rows.table(gx, np.arange(50, 100))
    other = gx.table_from([I8, I4, F8, CH], [c[:10] for c in rows.cols[:4]])
    other_types = gx.table_from([I8, I4, F8, I8, I8], [c[:10] for c in rows.cols[:3]] + [rows.cols[4][:10]] * 2)
    lib, h, path = g.lib(), ctypes.c_void_p(), ctypes.c_int()

    def call(parts, key_col=1, rank=0, window=0):
        arr = (ctypes.c_void_p * max(len(parts), 1))(*[p.h for p in parts])
        return lib.gx_debug_redistribute(gx.h, len(parts), arr, key_col, rank, window, ctypes.byref(h), ctypes.byref(path))

    cases = {
        "no parts": lambda: call([]),
        "65 parts": lambda: call([a] * 65),
        "rank -1": lambda: call([a, b], rank=-1),
        "rank 2 of 2": lambda: call([a, b], rank=2),
        "fewer columns": lambda: call([a, other]),
        "other types": lambda: call([a, other_types], rank=1),
        "key column -1": lambda: call([a, b], key_col=-1),
        "key column 5": lambda: call([a, b], key_col=5),
        "float8 key": lambda: call([a, b], key_col=2),
        "char key": lambda: call([a, b], key_col=3),
        "map of 3 nodes": lambda: (gx.set_shardmap(3), call([a, b]))[1],
        "windows over 4 GiB": lambda: (gx.set_shardmap(2), call([a, b], window=(2 << 30) + 256))[1],
    }
    for what, f in cases.items():
        st = f()
        assert st == g.GX_ERR_ARG, f"{what}: status {st}"
    gx.set_shardmap(2)
    assert call([a, b], window=2 << 30) == g.GX_OK             # exactly the limit is accepted
    g.Table(gx, h.value, rows.types).free()
    rows.map = np.arange(NSHARD, dtype=np.int32) % 2
    dest = rows.map[rows.shards()]
    for window in (0, 1 << 22):
        for r in range(2):
            out, p = gx.debug_redistribute([a, b], 1, r, window)
            assert p == (0 if window else 1)
            rows.check(*read_all(out), np.flatnonzero(dest == r), f"after the errors, rank {r}")
            out.free()
    for t in (a, b, other, other_types):
        t.free()
