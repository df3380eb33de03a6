"""Pins the oracle's restatement against the REFERENCE'S OWN OBJECT CODE.

oracle/ref/Makefile compiles a few of the reference's leaf source files into
oracle/_ref/libotbref.so (hashfunc.c, pg_crc32c_sb8.c, bloomfilter.c,
heaptuple.c, bufpage.c, float.c, int8.c, locator.c, fnbufpage.c).  What that
object code computes on the seeded inputs below is stored in
tests/golden/oracle_vs_ref.npz, so every test here compares the oracle with the
reference on any machine.  Where libotbref.so has been built, the stored values
are also checked against it (test_stored_vectors_match_the_reference_objects).
To regenerate the file after changing an input:

    python tests/test_oracle_vs_ref.py        # needs oracle/_ref/libotbref.so"""
import ctypes as C
import hashlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import oracle as O  # noqa: E402

REF_PATH = os.path.join(ROOT, "oracle", "_ref", "libotbref.so")
GOLDEN = os.path.join(ROOT, "tests", "golden", "oracle_vs_ref.npz")
HAVE_REF = os.path.exists(REF_PATH)


def load_ref():
    L = C.CDLL(REF_PATH)
    u32, i32, i64, dbl = C.c_uint32, C.c_int32, C.c_int64, C.c_double
    for n, res, args in [("ref_hash_any", u32, [C.c_char_p, C.c_int]), ("ref_hash_uint32", u32, [u32]),
                         ("ref_hashint4", u32, [i32]), ("ref_hashint8", u32, [i64]), ("ref_hashchar", u32, [C.c_int8]),
                         ("ref_hashfloat8", u32, [dbl]), ("ref_hash_any_new", u32, [C.c_char_p, C.c_int]),
                         ("ref_hashint4new", u32, [i32]), ("ref_hashint8new", u32, [i64]), ("ref_hashcharnew", u32, [C.c_int8]),
                         ("ref_hashfloat8new", u32, [dbl]), ("ref_murmurhash32", u32, [u32]), ("ref_hash_combine", u32, [u32, u32]),
                         ("ref_evaluate_hashkey1", u32, [C.c_int, i64, C.c_int]), ("ref_evaluate_hashkey2", u32, [i64, i32]),
                         ("ref_bloom_init", C.c_void_p, [dbl, dbl]), ("ref_bloom_insert", None, [C.c_void_p, u32]),
                         ("ref_bloom_find", C.c_int, [C.c_void_p, u32]), ("ref_bloom_log_num_buckets", C.c_int, [C.c_void_p]),
                         ("ref_bloom_words", C.c_void_p, [C.c_void_p]),
                         ("ref_float8pl", dbl, [dbl, dbl]), ("ref_float8mul", dbl, [dbl, dbl]), ("ref_float8mi", dbl, [dbl, dbl]),
                         ("ref_float8_accum", None, [C.c_void_p, dbl]), ("ref_float8_combine", None, [C.c_void_p, C.c_void_p]),
                         ("ref_float8_avg", C.c_int, [C.c_void_p, C.c_void_p]), ("ref_int8inc", i64, [i64]),
                         ("ref_heap_form_tuple", C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
                         ("ref_heap_deform_tuple", None, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
                         ("ref_page_build", C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
                         ("ref_page_offsets", None, [C.c_void_p]),
                         ("ref_fnpage_pack", C.c_int64, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int64,
                                                         C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int64]),
                         ("ref_fnpage_unpack", C.c_int64, [C.c_void_p, C.c_int64, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                           C.c_void_p, C.c_int64])]:
        f = getattr(L, n); f.restype = res; f.argtypes = args
    return L


def digest(a) -> np.ndarray:
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


# ------------------------------------------------------------------ seeded inputs
def hash_inputs():
    rng = np.random.default_rng(42)
    i4 = [0, 1, -1, 17, 42, 2**31 - 1, -2**31] + rng.integers(-2**31, 2**31, 3000).tolist()
    i8 = [0, 1, -1, 2**32 + 1, -2**32, 2**63 - 1, -2**63] + rng.integers(-2**63, 2**63 - 1, 3000).tolist()
    f8 = [0.0, -0.0, 1.0, -1.5, 1e300, float("inf")] + rng.normal(0, 1e6, 500).tolist()
    blobs = [bytes(rng.integers(0, 256, n).astype(np.uint8)) for n in list(range(0, 40)) + [63, 64, 65, 255]]
    pairs = rng.integers(0, 2**32, (200, 2)).tolist()
    return i4, i8, f8, blobs, pairs


BLOOM_ROWS = (10, 1000, 100000, 3000000)


def bloom_keys(nrows):
    L = O.lib()
    return [L.orc_hashint8new(i * 7919) for i in range(min(nrows, 5000))], [L.orc_hashint8new(i) for i in range(2000)]


def float8_inputs():
    rng = np.random.default_rng(9)
    # (1e300 would make Sxx overflow: the reference raises ERROR there, the oracle reports status 6)
    return np.concatenate([rng.normal(1000, 300, 4000), [0.0, -0.0, 1e-300, 1e150, -1e150]])


def float8_plan():
    import opentenbase_b200 as g
    return O.make_plan(aggs=[(g.GX_AGG_AVG_F8, [(g.GX_OP_COL, 0, 0)]), (g.GX_AGG_SUM_F8, [(g.GX_OP_COL, 0, 0)])])


ATT = {O.GX_INT8: (8, 8), O.GX_INT4: (4, 4), O.GX_FLOAT8: (8, 8), O.GX_DATE: (4, 4), O.GX_CHAR: (1, 1), O.ORC_BPCHAR1: (-1, 4)}
HEAP_TYPES = [O.GX_INT8, O.GX_INT4, O.ORC_BPCHAR1, O.ORC_BPCHAR1, O.GX_FLOAT8, O.GX_CHAR, O.GX_DATE, O.GX_INT8]


def heap_inputs():
    rng = np.random.default_rng(13)
    n = 400
    cols = [rng.integers(-2**62, 2**62, n), rng.integers(-2**31, 2**31, n).astype(np.int32),
            rng.integers(65, 90, n).astype(np.int8), rng.integers(65, 90, n).astype(np.int8), rng.normal(size=n),
            rng.integers(32, 127, n).astype(np.int8), rng.integers(-3000, 0, n).astype(np.int32), rng.integers(0, 2**40, n)]
    nulls = [None] + [(rng.random(n) < 0.25).astype(np.uint8) for _ in range(7)]
    nulls[4][:50] = 0
    for k in range(1, 8):
        nulls[k][:20] = 0                               # some tuples without any NULL (t_hoff 48)
    return cols, nulls


def heap_tuple_args(cols, nulls, i):
    t = len(HEAP_TYPES)
    vals = (C.c_int64 * t)(*[int(np.asarray(c)[i].view(np.int64)) if np.asarray(c).dtype == np.float64 else int(np.asarray(c)[i]) for c in cols])
    isn = (C.c_uint8 * t)(*[0 if x is None else int(x[i]) for x in nulls])
    return vals, isn


def att_arrays(types):
    return (C.c_int16 * len(types))(*[ATT[t][0] for t in types]), (C.c_int8 * len(types))(*[ATT[t][1] for t in types])


def oracle_first_page():
    """The oracle's first heap page of heap_inputs(): the page, pd_lower, the line count and every tuple's bytes."""
    cols, nulls = heap_inputs()
    pages = O.Rel(HEAP_TYPES, cols, nulls).pages().reshape(-1, 8192)
    pg = pages[0]
    lower = int(pg[16:20].copy().view(np.uint32)[0])
    nlines = (lower - 44) // 4
    tuples = []
    for i in range(nlines):
        lp = int(pg[44 + 4 * i: 48 + 4 * i].copy().view(np.uint32)[0])
        off, ln = lp & 0x7FFF, lp >> 17
        tuples.append(pg[off: off + ln])
    return pages, lower, nlines, tuples


FNPAGE_CASES = [([O.GX_INT8, O.GX_INT8, O.GX_DATE, O.GX_INT4], 5000, 0.0),
                ([O.GX_INT8, O.GX_INT4, O.ORC_BPCHAR1, O.GX_FLOAT8, O.GX_CHAR, O.GX_DATE, O.ORC_BPCHAR1, O.GX_INT8, O.GX_INT4], 3000, 0.2),
                ([O.GX_CHAR], 700, 0.5), ([O.GX_FLOAT8] * 12, 900, 0.1)]


def fnpage_inputs():
    rng = np.random.default_rng(99)
    out = []
    for types, n, frac in FNPAGE_CASES:
        vals = np.zeros((n, len(types)), np.int64)
        for i, t in enumerate(types):
            vals[:, i] = (rng.integers(-2**62, 2**62, n) if t in (O.GX_INT8, O.GX_FLOAT8) else
                          rng.integers(-2**31, 2**31 - 1, n) if t in (O.GX_INT4, O.GX_DATE) else rng.integers(-128, 127, n))
        isn = (rng.random((n, len(types))) < frac).astype(np.uint8)
        isn[:40] = 0
        out.append((types, n, frac, vals, isn))
    return out


# ------------------------------------------------------------------ what the reference computes
def reference_values(R) -> dict:
    """Every value the tests compare the oracle with, computed by the reference's object code on the inputs above."""
    out = {}
    a = (C.c_int * 10)()
    R.ref_page_offsets(a)
    out["layout"] = np.array(list(a) + [R.ref_sizeof_heap_header(), R.ref_offsetof_hoff(), R.ref_offsetof_infomask(),
                                        R.ref_sizeof_minimal_header(), R.ref_minimal_tuple_offset(),
                                        R.ref_sizeof_fnpage_header(), R.ref_invalid_shardid()], np.int64)
    # hashes
    i4, i8, f8, blobs, pairs = hash_inputs()
    out["hash_i4"] = np.array([[R.ref_hashint4(v), R.ref_hashint4new(v), R.ref_hash_uint32(v & 0xFFFFFFFF),
                                R.ref_murmurhash32(v & 0xFFFFFFFF), R.ref_evaluate_hashkey1(0, v, 0)] for v in i4], np.uint32)
    out["hash_i8"] = np.array([[R.ref_hashint8(v), R.ref_hashint8new(v), R.ref_evaluate_hashkey1(1, v, 0)] for v in i8], np.uint32)
    out["hash_char"] = np.array([[R.ref_hashchar(v), R.ref_hashcharnew(v)] for v in range(-128, 128)], np.uint32)
    out["hash_f8"] = np.array([[R.ref_hashfloat8(v), R.ref_hashfloat8new(v)] for v in f8], np.uint32)
    out["hash_any"] = np.array([[R.ref_hash_any(b, len(b)), R.ref_hash_any_new(b, len(b))] for b in blobs], np.uint32)
    out["hash_combine"] = np.array([R.ref_hash_combine(x, y) for x, y in pairs], np.uint32)
    out["hashkey2"] = np.array([R.ref_evaluate_hashkey2(x, y) for x, y in zip(i8[:200], i4[:200])], np.uint32)
    out["hashkey_null"] = np.array([R.ref_evaluate_hashkey1(1, 12345, 1)], np.uint32)
    # bloom filters: bucket count, a digest of the bit pattern, and the answers to 2000 probes; -1 = the filter gave up
    logs, words, finds = [], [], []
    L = O.lib()
    for nrows in BLOOM_ROWS + (1_000_000_000,):
        rb = R.ref_bloom_init(float(nrows), 0.05)
        if rb is None:
            logs.append(-1); words.append(np.zeros(32, np.uint8)); finds.append(np.zeros(2000, np.uint8))
            continue
        logs.append(R.ref_bloom_log_num_buckets(rb))
        keys, probes = bloom_keys(nrows)
        for k in keys:
            R.ref_bloom_insert(rb, k)
        ob = L.orc_bloom_create(nrows)                       # the word count only: the reference does not export it
        nw = C.c_int64()
        L.orc_bloom_words(ob, C.byref(nw))
        L.orc_bloom_free(ob)
        words.append(digest(np.ctypeslib.as_array(C.cast(R.ref_bloom_words(rb), C.POINTER(C.c_uint32)), (nw.value,))))
        finds.append(np.array([R.ref_bloom_find(rb, p) for p in probes], np.uint8))
    out["bloom_log"], out["bloom_words_sha256"], out["bloom_find"] = np.array(logs, np.int64), np.array(words), np.array(finds)
    # float8 transition functions
    vals = float8_inputs()
    state = (C.c_double * 3)(0.0, 0.0, 0.0)
    s = None
    for x in vals.tolist():
        R.ref_float8_accum(state, x)
        s = x if s is None else R.ref_float8pl(s, x)
    avg = C.c_double()
    st = R.ref_float8_avg(state, C.byref(avg))
    st0 = R.ref_float8_avg((C.c_double * 3)(0, 0, 0), C.byref(C.c_double()))
    h = len(vals) // 2
    plan = float8_plan()
    r1, _ = O.exec_agg(O.Rel([O.GX_FLOAT8], [vals[:h]]), plan, keep_raw=True)
    r2, _ = O.exec_agg(O.Rel([O.GX_FLOAT8], [vals[h:]]), plan, keep_raw=True)
    s1 = (C.c_double * 3)(*r1.states[0, 0]); s2 = (C.c_double * 3)(*r2.states[0, 0])
    R.ref_float8_combine(s1, s2)
    out["f8_state"], out["f8_sum"], out["f8_avg"] = np.array(list(state)), np.array([s]), np.array([avg.value])
    out["f8_avg_status"] = np.array([st, st0], np.int64)
    out["f8_split_states"] = np.array([list(r1.states[0, 0]), list(r2.states[0, 0])])
    out["f8_combined"] = np.array(list(s1))
    out["f8_misc"] = np.array([R.ref_float8mul(1.1, 3.3), R.ref_float8mi(1.0, 0.07)])
    out["int8inc"] = np.array([R.ref_int8inc(41)], np.int64)
    # heap tuples: the reference's heap_form_tuple of every input row of the oracle's first page, its deform of the
    # oracle's tuple bytes, and the page PageAddItem builds from those bytes
    cols, nulls = heap_inputs()
    _, _, nlines, tuples = oracle_first_page()
    attlen, attalign = att_arrays(HEAP_TYPES)
    buf = (C.c_uint8 * 1024)()
    formed, lens, dvals, dnulls = b"", [], [], []
    for i in range(nlines):
        v, isn = heap_tuple_args(cols, nulls, i)
        rl = R.ref_heap_form_tuple(len(HEAP_TYPES), attlen, attalign, v, isn, buf, 1024)
        formed += bytes(buf)[:rl]; lens.append(rl)
        mine = tuples[i]
        vo, no = (C.c_int64 * len(HEAP_TYPES))(), (C.c_uint8 * len(HEAP_TYPES))()
        R.ref_heap_deform_tuple(len(HEAP_TYPES), attlen, attalign, mine.ctypes.data, len(mine), vo, no)
        dvals.append(list(vo)); dnulls.append(list(no))
    rpage = (C.c_uint8 * 8192)()
    items = b"".join(t.tobytes() for t in tuples)
    added = R.ref_page_build(rpage, items, (C.c_int * nlines)(*[len(t) for t in tuples]), nlines)
    out["heap_formed"] = np.frombuffer(formed, np.uint8).copy()
    out["heap_formed_len"] = np.array(lens, np.int64)
    out["heap_deform_vals"], out["heap_deform_nulls"] = np.array(dvals, np.int64), np.array(dnulls, np.uint8)
    out["heap_page"], out["heap_page_added"] = np.frombuffer(bytes(rpage), np.uint8).copy(), np.array([added], np.int64)
    # forward-node pages: page count and digest of the reference sender's pages; its receiver's output on those pages
    npg, pdig, rgot, rdig = [], [], [], []
    for types, n, frac, vals8, isn in fnpage_inputs():
        attlen, attalign = att_arrays(types)
        cap = n // 20 + 4
        ref = np.zeros((cap, 8192), np.uint8)
        k = R.ref_fnpage_pack(len(types), attlen, attalign, vals8.ctypes.data, isn.ctypes.data, n, 123456789012345, -7, 12, 3, 1, 2, 1,
                              ref.ctypes.data, cap)
        npg.append(k); pdig.append(digest(ref[:max(k, 0)]))
        vo = np.zeros((n, len(types)), np.int64); no = np.zeros((n, len(types)), np.uint8)
        got = R.ref_fnpage_unpack(ref.ctypes.data, k, len(types), attlen, attalign, vo.ctypes.data, no.ctypes.data, n)
        rgot.append(got); rdig.append(np.concatenate([digest(no), digest(vo[no == 0])]))
    out["fnpage_npages"], out["fnpage_sha256"] = np.array(npg, np.int64), np.array(pdig)
    out["fnpage_unpacked_rows"], out["fnpage_unpacked_sha256"] = np.array(rgot, np.int64), np.array(rdig)
    return out


@pytest.fixture(scope="module")
def ref():
    return dict(np.load(GOLDEN))


# ------------------------------------------------------------------ the oracle against it
def test_struct_layout_constants(ref):
    flags, lower, upper, special, psv, linp, itemid, ctid, im2, bits, hdr, hoff, infomask, minhdr, minoff, fnhdr, noshard = ref["layout"].tolist()
    assert (flags, lower, upper, special, psv, linp, itemid) == (10, 16, 20, 24, 28, 44, 4)     # orc_heap.c PD_* / ORC_PAGE_HDR
    assert (ctid, im2, bits) == (32, 38, 47)                                                      # orc_internal.h HTH_*
    assert (hdr, hoff, infomask) == (47, 46, 40)
    assert (minhdr, minoff) == (15, 32)
    assert (fnhdr, noshard) == (32, 4096)                                                         # orc_fnpage.c header, InvalidShardId


def test_hash_functions_against_reference_objects(ref):
    L = O.lib()
    i4, i8, f8, blobs, pairs = hash_inputs()
    got = np.array([[L.orc_hashint4(v), L.orc_hashint4new(v), L.orc_hash_uint32(v & 0xFFFFFFFF), L.orc_murmurhash32(v & 0xFFFFFFFF),
                     L.orc_evaluate_hashkey((C.c_int * 1)(O.GX_INT4), None, (C.c_int64 * 1)(v), 1)] for v in i4], np.uint32)
    np.testing.assert_array_equal(got, ref["hash_i4"])
    got = np.array([[L.orc_hashint8(v), L.orc_hashint8new(v),
                     L.orc_evaluate_hashkey((C.c_int * 1)(O.GX_INT8), None, (C.c_int64 * 1)(v), 1)] for v in i8], np.uint32)
    np.testing.assert_array_equal(got, ref["hash_i8"])
    np.testing.assert_array_equal(np.array([[L.orc_hashchar(v), L.orc_hashcharnew(v)] for v in range(-128, 128)], np.uint32), ref["hash_char"])
    np.testing.assert_array_equal(np.array([[L.orc_hashfloat8(v), L.orc_hashfloat8new(v)] for v in f8], np.uint32), ref["hash_f8"])
    np.testing.assert_array_equal(np.array([[L.orc_hash_any(b, len(b)), L.orc_hash_any_new(b, len(b))] for b in blobs], np.uint32), ref["hash_any"])
    np.testing.assert_array_equal(np.array([L.orc_hash_combine(a, b) for a, b in pairs], np.uint32), ref["hash_combine"])
    # two-column distribution key: rotate-then-xor order (locator.c:1611-1628)
    got = [L.orc_evaluate_hashkey((C.c_int * 2)(O.GX_INT8, O.GX_INT4), None, (C.c_int64 * 2)(a, b), 2) for a, b in zip(i8[:200], i4[:200])]
    np.testing.assert_array_equal(np.array(got, np.uint32), ref["hashkey2"])
    # NULL distribution value hashes to 0 -> shard 0
    assert ref["hashkey_null"][0] == 0 == L.orc_evaluate_hashkey((C.c_int * 1)(O.GX_INT8), (C.c_uint8 * 1)(1), (C.c_int64 * 1)(12345), 1)


def test_bloom_filter_against_reference_object(ref):
    L = O.lib()
    for i, nrows in enumerate(BLOOM_ROWS):
        ob = L.orc_bloom_create(nrows)
        assert (ref["bloom_log"][i] < 0) == (not ob)
        if not ob:
            continue
        assert ref["bloom_log"][i] == L.orc_bloom_log_num_buckets(ob)
        keys, probes = bloom_keys(nrows)
        for k in keys:
            L.orc_bloom_insert(ob, k)
        nw = C.c_int64()
        ow = np.ctypeslib.as_array(C.cast(L.orc_bloom_words(ob, C.byref(nw)), C.POINTER(C.c_uint32)), (nw.value,))
        np.testing.assert_array_equal(digest(ow), ref["bloom_words_sha256"][i])               # identical bit patterns
        np.testing.assert_array_equal(np.array([L.orc_bloom_find(ob, p) for p in probes], np.uint8), ref["bloom_find"][i])
        L.orc_bloom_free(ob)
    assert ref["bloom_log"][len(BLOOM_ROWS)] == -1                                             # logNumBuckets > 20: gives up


def test_float8_transition_functions_against_reference_objects(ref):
    """float8_accum / float8_combine / float8_avg / float8pl from float.o versus the oracle's
    aggregate states on the same input order."""
    vals = float8_inputs()
    plan = float8_plan()
    r, raw = O.exec_agg(O.Rel([O.GX_FLOAT8], [vals]), plan, keep_raw=True)
    np.testing.assert_array_equal(r.states[0, 0], ref["f8_state"])                 # {N, Sx, Sxx} bit-identical
    assert r.aggs[0, 1] == ref["f8_sum"][0]
    assert ref["f8_avg_status"][0] == 0 and ref["f8_avg"][0] == r.aggs[0, 0]
    assert ref["f8_avg_status"][1] == 1                                            # N == 0 -> NULL
    # combine: split the input in two, states must merge exactly like float8_combine
    h = len(vals) // 2
    r1, raw1 = O.exec_agg(O.Rel([O.GX_FLOAT8], [vals[:h]]), plan, keep_raw=True)
    r2, raw2 = O.exec_agg(O.Rel([O.GX_FLOAT8], [vals[h:]]), plan, keep_raw=True)
    np.testing.assert_array_equal(np.array([r1.states[0, 0], r2.states[0, 0]]), ref["f8_split_states"])
    comb = O.combine(plan, [raw1, raw2])
    np.testing.assert_array_equal(comb.states[0, 0], ref["f8_combined"])
    assert ref["f8_misc"][0] == 1.1 * 3.3 and ref["f8_misc"][1] == 1.0 - 0.07
    assert ref["int8inc"][0] == 42


def test_heap_tuples_and_pages_against_reference_objects(ref):
    """The oracle's heap_form_tuple / PageAddItem restatement produces the bytes the
    reference's heaptuple.o / bufpage.o produce; its deform agrees with heap_deform_tuple."""
    cols, nulls = heap_inputs()
    pages, lower, nlines, tuples = oracle_first_page()
    pg = pages[0]
    lens = ref["heap_formed_len"]
    assert nlines == len(lens)
    ends = np.cumsum(lens)
    for i in range(nlines):
        mine, rl = tuples[i], int(lens[i])
        r = ref["heap_formed"][ends[i] - rl: ends[i]]
        vals, isn = heap_tuple_args(cols, nulls, i)
        assert rl == len(mine), f"tuple {i}: oracle length {len(mine)} vs reference {rl}"
        assert mine[46] == r[46]                                              # t_hoff
        assert (int(mine[38]) | int(mine[39]) << 8) & 0x07FF == (int(r[38]) | int(r[39]) << 8) & 0x07FF   # natts
        assert (int(mine[40]) & 0x03) == (int(r[40]) & 0x03)                 # HEAP_HASNULL | HEAP_HASVARWIDTH
        np.testing.assert_array_equal(mine[47:], r[47:])                     # null bitmap + padding + attribute data
        # the reference's deform of the oracle's tuple bytes gives back the inputs
        vo, no = ref["heap_deform_vals"][i], ref["heap_deform_nulls"][i]
        assert list(no) == list(isn)
        assert [v for v, z in zip(vo, no) if not z] == [v for v, z in zip(vals, isn) if not z]
    # page assembly: same line pointers, pd_lower, pd_upper
    assert ref["heap_page_added"][0] == nlines
    rp = ref["heap_page"]
    np.testing.assert_array_equal(rp[16:30], pg[16:30])                       # pd_lower, pd_upper, pd_special, pagesize_version
    np.testing.assert_array_equal(rp[44:lower], pg[44:lower])                 # ItemIdData array
    upper = int(pg[20:24].copy().view(np.uint32)[0])
    np.testing.assert_array_equal(rp[upper:], pg[upper:])                     # tuple area
    # and the next tuple really does not fit (heap_insert's fill rule)
    lp = int(pages[1][44:48].copy().view(np.uint32)[0])
    assert ((lp >> 17) + 7) // 8 * 8 > upper - lower - 4


def test_fnpages_against_reference_objects(ref):
    """Forward-node pages (the redistribute wire format): the oracle's sender writes the bytes that heaptuple.o's
    heap_form_minimal_tuple_ptr + fnbufpage.o's FnPageInit write under FragmentSendAttrs' control flow, and each side's
    receiver reads the other side's pages (iterator macros of fnbufpage.h + heap_deform_tuple)."""
    for c, (types, n, frac, vals, isn) in enumerate(fnpage_inputs()):
        k = int(ref["fnpage_npages"][c])
        assert k > 0
        cols = [vals[:, i].astype(O.NP_DTYPES[t]) if t != O.GX_FLOAT8 else vals[:, i].copy().view(np.float64) for i, t in enumerate(types)]
        nulls = [isn[:, i].copy() for i in range(len(types))] if frac else None
        mine = O.fnpage_pack(types, cols, nulls, O.OrcFnPageId(123456789012345, -7, 12, 3, 1, 2, 0), True)
        assert len(mine) == k
        np.testing.assert_array_equal(digest(mine), ref["fnpage_sha256"][c])          # the reference's pages, byte for byte
        # the reference's receiver on those pages gives back the inputs
        assert ref["fnpage_unpacked_rows"][c] == n
        np.testing.assert_array_equal(ref["fnpage_unpacked_sha256"][c], np.concatenate([digest(isn), digest(vals[isn == 0])]))
        # the oracle's receiver on the same bytes
        c2, n2 = O.fnpage_unpack(mine, types)
        for i in range(len(types)):
            np.testing.assert_array_equal(n2[i], isn[:, i])
            keep = isn[:, i] == 0
            np.testing.assert_array_equal(np.asarray(c2[i])[keep].view(np.uint8), np.asarray(cols[i])[keep].view(np.uint8))


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref/libotbref.so is built only where the reference sources are present")
def test_stored_vectors_match_the_reference_objects(ref):
    """The stored values are what the reference's object code computes today."""
    live = reference_values(load_ref())
    assert sorted(live) == sorted(ref)
    for k in ref:
        np.testing.assert_array_equal(live[k], ref[k], err_msg=k)


if __name__ == "__main__":
    np.savez_compressed(GOLDEN, **reference_values(load_ref()))
    print("wrote", GOLDEN, os.path.getsize(GOLDEN), "bytes")
