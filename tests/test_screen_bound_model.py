"""CPU model of DESIGN.md §4's screening argument: K1 drops a candidate when the bound computed from its 8-bit codes exceeds the
distance of the furthest key of a full `nearest`, and that is exact only if the bound never exceeds the CANONICAL (rounded) distance.

  table:  x~_i = fmaf(code_i, scale_i, offset_i) (round to nearest),  E_i = max over rows of (|x_i - x~_i| rounded up)
  bound:  a_i = max(0, |q_i - x~_i|_rz - E_i)_rd,  LB = sum_rd a_i^2,  b = LB * (1 - 2^-16)_rd,  bound = b if b > 2^-100 else 0

The argument: LB <= T = sum (q_i - x_i)^2 exactly (every step rounds down); the canonical distance D rounds each term at most CH + 9
times (the subtraction twice in the square, CH fma steps, two lane-sum adds, five butterfly adds), all on non-negative values, so
D >= T (1 - u)^(CH + 9) - err with u = 2^-24 and err <= 2^-139 from underflowing fma results; 1 - 2^-16 < (1 - u)^17 leaves at
least T 2^-17 of room, which exceeds err once T > 2^-100.  The model below restates both computations with numpy (directed rounding
emulated through float64) on data with ties, quantisation-boundary values and extreme magnitudes."""
import numpy as np

U = 2.0 ** -24
KEEP = np.float32(1 - 2.0 ** -16)
FLOOR = np.float32(2.0 ** -100)


def rd(x):  # float64 -> float32 rounded toward -inf
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) > x, np.nextafter(f, np.float32(-np.inf)), f)


def ru(x):
    f = x.astype(np.float32)
    return np.where(f.astype(np.float64) < x, np.nextafter(f, np.float32(np.inf)), f)


def rz(x):
    return np.where(x >= 0, rd(x), ru(x))


def fma_rn(a, b, c):  # float32 fma through float64 (the product of two floats is exact in float64)
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def canonical(q, x):
    """The canonical order of DESIGN §3 for rows (vectorised over the leading axis): 128 fma chains, lane sums, butterfly."""
    dim = q.shape[-1]
    pad = (-dim) % 128
    q = np.pad(q, [(0, 0), (0, pad)])
    x = np.pad(x, [(0, 0), (0, pad)])
    d = (q - x).astype(np.float32)
    acc = np.zeros((len(q), 128), dtype=np.float32)
    for j in range(0, d.shape[1], 128):
        acc = fma_rn(d[:, j:j + 128], d[:, j:j + 128], acc)
    s = ((acc[:, 0::4] + acc[:, 1::4]) + (acc[:, 2::4] + acc[:, 3::4])).astype(np.float32)  # lane l: acc[4l..4l+3]
    for off in (1, 2, 4, 8, 16):
        s = (s + s[:, np.arange(32) ^ off]).astype(np.float32)
    return s[:, 0]


def table(rows):
    lo, hi = rows.min(axis=0), rows.max(axis=0)
    scale = (hi / np.float32(255) - lo / np.float32(255)).astype(np.float32)
    scale = np.where(scale > 0, scale, np.float32(0))
    with np.errstate(divide="ignore", invalid="ignore"):
        c = np.where(scale > 0, np.clip(np.rint((rows - lo) / scale), 0, 255), 0).astype(np.float32)
    xt = fma_rn(c, np.broadcast_to(scale, c.shape), np.broadcast_to(lo, c.shape))
    err = ru(np.abs(rows.astype(np.float64) - xt.astype(np.float64))).max(axis=0)
    return c, scale, lo, err


def bound(q, c, scale, offset, err):
    xt = fma_rn(c, np.broadcast_to(scale, c.shape), np.broadcast_to(offset, c.shape))
    d = np.abs(rz(q.astype(np.float64) - xt.astype(np.float64)))
    a = np.maximum(rd(d.astype(np.float64) - err.astype(np.float64)), np.float32(0))
    lb = np.zeros(len(q), dtype=np.float32)
    for i in range(q.shape[1]):  # any order of round-down adds is a lower bound
        lb = rd(a[:, i].astype(np.float64) ** 2 + lb.astype(np.float64))
    b = rd(lb.astype(np.float64) * np.float64(KEEP))
    return np.where(b > FLOOR, b, np.float32(0))


def test_margin_covers_the_canonical_roundings():
    for ch in range(1, 9):
        assert float(KEEP) < (1 - U) ** (ch + 9) - 2.0 ** -17
    fma_per_distance = 1024  # at most 4 * 32 * CH fma results, each off by at most 2^-150 when it underflows
    err = fma_per_distance * 2.0 ** -150 * 2
    assert float(FLOOR) * 2.0 ** -17 > err


def test_bound_never_exceeds_the_canonical_distance():
    rng = np.random.default_rng(7)
    for dim in (4, 37, 128, 300):
        n = 2000
        rows = rng.standard_normal((n, dim)).astype(np.float32)
        cols = np.arange(dim)
        rows[:, cols % 5 == 1] *= np.float32(1e-21)
        rows[:, cols % 5 == 2] *= np.float32(1e17)
        rows[:, cols % 5 == 3] = (rng.integers(0, 256, (n, (cols % 5 == 3).sum())) / 255 * 2 - 1).astype(np.float32)
        rows[:50] = rows[50:100]
        c, scale, offset, err = table(rows)
        xt = fma_rn(c, np.broadcast_to(scale, c.shape), np.broadcast_to(offset, c.shape))
        assert (np.abs(rows.astype(np.float64) - xt.astype(np.float64)) <= err.astype(np.float64)).all()
        pick = rng.integers(0, n, 4000)
        q = np.concatenate([rows[pick[:1000]], np.nextafter(rows[pick[1000:2000]], np.float32(1)),
                            rng.standard_normal((1000, dim)).astype(np.float32) * np.float32(1e-25),
                            rows[pick[3000:]] * np.float32(1.001)])
        other = rng.integers(0, n, len(q))
        other[:1000] = pick[:1000]  # exact ties: distance 0
        b = bound(q, c[other], scale, offset, err)
        d = canonical(q, rows[other])
        assert not (b > d).any()
        assert (b[1000:] > 0).mean() > 0.5  # not vacuous
