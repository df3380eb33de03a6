"""Float8 edge datasets shared by the exact-reference CPU test and the GPU family matrix.

A dataset is (group index per row, x, y): x carries the edge values, y is a benign second column for
expressions (x * y stays normal).  Rows are interleaved across groups unless sorted=True."""
import numpy as np

# ragged group sizes around warp (32), tile (128 = 32 x 4), warp-chunk (3968 = 31 x 128) and CTA edges
CANCEL_SIZES = [1, 31, 33, 127, 128, 129, 3967, 3968, 3971, 1_000_003]
SMALL_CANCEL_SIZES = [33, 129, 3971, 1_000_003]

SPECIAL_GROUPS = [
    [1.0, np.inf, 2.0],            # inf input: sum / avg inf, not an overflow
    [-np.inf, 3.0],
    [np.inf, -np.inf, 1.0],        # +inf + -inf = NaN
    [np.nan, 1.0, 2.0],
    [-0.0, -0.0],                  # sum of only -0 is -0
    [-0.0, 0.0, -0.0],             # mixed zeros sum to +0
    [np.nan],                      # min = max = NaN
    [5.0, np.nan, -3.0],           # max NaN, min -3
    [-0.0],
    [4.9e-324, -4.9e-324, 2.5e-320],
    [np.inf, 7.0, np.nan],
    [-np.inf, -1e300],
]


def _order(gidx, rng, sorted_rows):
    return np.argsort(gidx, kind="stable") if sorted_rows else rng.permutation(len(gidx))


def cancel(rng, sizes, sorted_rows=False, top=300):
    """mixed signs; group i lives in its own decade between 1e-300 and 1e<top>; half the rows are near-cancelling
    pairs x, -x(1 + d).  avg() needs top <= 100: float8_accum squares (x N - Sx) on the way, which overflows above ~1e150."""
    G = len(sizes)
    dec = np.round(np.linspace(-300, top, G)).astype(int) if G > 1 else np.array([0])
    gi, xs = [], []
    for i, n in enumerate(sizes):
        m = rng.random(n) * 9 + 1
        x = m * 10.0 ** int(dec[i]) * rng.choice([-1.0, 1.0], n)
        npair = n // 4
        if npair:
            x[1:2 * npair:2] = -x[0:2 * npair:2] * (1 + rng.integers(1, 1 << 20, npair) * 2.0 ** -40)
        gi.append(np.full(n, i)); xs.append(x)
    gi, x = np.concatenate(gi), np.concatenate(xs)
    o = _order(gi, rng, sorted_rows)
    return gi[o], x[o], (0.5 + rng.random(len(x)) * 1.5)[o]


def subnormal(rng, G, n_per=300, sorted_rows=False):
    """subnormal inputs, and groups whose exact sum cancels down to a subnormal"""
    gi, xs = [], []
    for i in range(G):
        k = rng.integers(-1000, 1000, n_per).astype(np.float64) * 2.0 ** -1074
        if i % 2:
            big = rng.random(n_per // 2) * 1e-300
            k[: n_per // 2] = big
            k[n_per // 2: 2 * (n_per // 2)] = -big                  # exact cancellation, leaves the subnormal tail
        gi.append(np.full(n_per, i)); xs.append(k)
    gi, x = np.concatenate(gi), np.concatenate(xs)
    o = _order(gi, rng, sorted_rows)
    return gi[o], x[o], (0.5 + rng.random(len(x)) * 1.5)[o]


def special(rng, groups=SPECIAL_GROUPS, sorted_rows=False, repeat=1):
    gi = np.concatenate([np.full(len(v) * repeat, i) for i, v in enumerate(groups)])
    x = np.concatenate([np.tile(np.array(v, np.float64), repeat) for v in groups])
    o = _order(gi, rng, sorted_rows)
    return gi[o], x[o], (0.5 + rng.random(len(x)) * 1.5)[o]


def batches(groups, limit):
    """a list of groups cut into runs of at most `limit` (kernels that hold a handful of groups)"""
    return [groups[i:i + limit] for i in range(0, len(groups), limit)]
