"""CPU model of K1's integer screening bound (DESIGN.md §4 "screen") and of the table it reads (DESIGN.md §2):

  table:  S = max_i (hi_i / 255 rounded up - lo_i / 255 rounded down) rounded up, offset_i = lo_i,
          c_i = clamp(rint((x_i - offset_i) / S), 0, 255),  R >= max over the rows of ||x - x~||,  x~_i = offset_i + c_i S (real)
  query:  qc_i = clamp(rint((q_i - offset_i) / S), 0, 255) (NaN -> 0),  r_q >= ||q - q^||,  q^_i = offset_i + qc_i S (real)
  bound:  D = sum (qc_i - c_i)^2 (exact),  t = ((S sqrt(D))_rd - (r_q + R)_ru)_+,  b = (t^2)_rd (1 - 2^-16)_rd,  0 unless b > 2^-100

The triangle inequality gives ||q - x|| >= ||q^ - x~|| - r_q - R and ||q^ - x~|| = S sqrt(D) exactly; the factor and the floor are
§4's margin for the canonical order's roundings.  The device brackets x~ and q^ between fmaf_rd and fmaf_ru; numpy has no directed
rounding, so the model rounds through float64 and widens every directed step by one more float32 ulp, which only loosens the bound."""
import numpy as np

from tests import datagen
from tests.test_screen_bound_model import FLOOR, KEEP, canonical, rd, ru

INF = np.float32(np.inf)


def down(x):  # float64 -> a float32 certainly <= x
    return np.nextafter(rd(np.asarray(x, dtype=np.float64)), -INF)


def up(x):  # float64 -> a float32 certainly >= x
    return np.nextafter(ru(np.asarray(x, dtype=np.float64)), INF)


def codes_of(v, offset, step):
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        c = np.rint(((v - offset).astype(np.float32) / step).astype(np.float32)) if step > 0 else np.zeros_like(v)
    c = np.where(np.isnan(c), 0, np.clip(c, 0, 255))  # fmaxf(NaN, 0) = 0 on the device
    return c.astype(np.int64)


def coding_error(v, c, offset, step):
    """An upper bound of ||v - (offset + c S)|| per row, the way the device brackets it."""
    exact = c.astype(np.float64) * np.float64(step) + offset.astype(np.float64)
    lo, hi = down(exact), up(exact)
    with np.errstate(invalid="ignore", over="ignore"):
        d = np.maximum(up(v.astype(np.float64) - lo), up(hi.astype(np.float64) - v))
        ss = (d.astype(np.float64) ** 2).sum(axis=-1) * (1 + 2.0 ** -40)
        return up(np.sqrt(up(ss).astype(np.float64)))


def table(rows):
    lo, hi = rows.min(axis=0), rows.max(axis=0)
    per = up(up(hi / np.float64(255)).astype(np.float64) - down(lo / np.float64(255)).astype(np.float64))
    step = np.float32(max(float(per.max()), 0.0))
    c = codes_of(rows, lo, step)
    R = np.float32(coding_error(rows, c, lo, step).max())
    return c, lo, step, R


def bound(q, c_rows, offset, step, R):
    qc = codes_of(q, offset, step)
    with np.errstate(invalid="ignore", over="ignore"):
        slack = up(coding_error(q, qc, offset, step).astype(np.float64) + np.float64(R))
        D = ((qc - c_rows) ** 2).sum(axis=-1)
        a = down(np.float64(step) * down(np.sqrt(D.astype(np.float64))).astype(np.float64))
        t = np.maximum(down(a.astype(np.float64) - slack.astype(np.float64)), np.float32(0))  # NaN slack -> 0
        t = np.where(np.isnan(t), np.float32(0), t)
        b = down(down(t.astype(np.float64) ** 2).astype(np.float64) * np.float64(KEEP))
    return np.where(b > FLOOR, b, np.float32(0))


def adversarial_rows(rng, n, dim):
    rows = rng.standard_normal((n, dim)).astype(np.float32)
    cols = np.arange(dim)
    rows[:, cols % 7 == 1] *= np.float32(1e-20)
    rows[:, cols % 7 == 2] *= np.float32(1e-40 / 3)  # subnormal
    rows[:, cols % 7 == 3] *= np.float32(1e17)
    rows[:, cols % 7 == 4] = (rng.integers(0, 256, (n, (cols % 7 == 4).sum())) / 255 * 3 - 1.5).astype(np.float32)  # code boundaries
    rows[:, cols % 7 == 5] = np.float32(0.25)  # constant
    rows[:50] = rows[50:100]  # duplicates
    return rows


def test_coding_error_bounds_every_row():
    rng = np.random.default_rng(5)
    rows = adversarial_rows(rng, 1000, 37)
    c, offset, step, R = table(rows)
    assert (c >= 0).all() and (c <= 255).all()
    xt = c.astype(np.float64) * np.float64(step) + offset.astype(np.float64)
    assert (np.sqrt(((rows.astype(np.float64) - xt) ** 2).sum(axis=1)) <= np.float64(R)).all()


def test_bound_never_exceeds_the_canonical_distance():
    rng = np.random.default_rng(11)
    for dim in (4, 37, 128, 300):
        n = 1500
        rows = adversarial_rows(rng, n, dim)
        c, offset, step, R = table(rows)
        pick = rng.integers(0, n, 3000)
        outside = rows[pick[2000:2500]].copy()
        outside[:, ::3] += np.float32(50)
        outside[:, 1::3] -= np.float32(3e17)
        nonfinite = rows[pick[2500:]].copy()
        nonfinite[np.arange(500), rng.integers(0, dim, 500)] = np.where(np.arange(500) % 3 == 0, np.nan,
                                                                         np.where(np.arange(500) % 3 == 1, np.inf, -np.inf))
        q = np.concatenate([rows[pick[:500]], np.nextafter(rows[pick[500:1000]], INF),
                            rng.standard_normal((500, dim)).astype(np.float32),
                            rng.standard_normal((500, dim)).astype(np.float32) * np.float32(1e18), outside, nonfinite])
        other = rng.integers(0, n, len(q))
        other[:500] = pick[:500]  # exact ties: distance 0
        b = bound(q, c[other], offset, step, R)
        with np.errstate(invalid="ignore", over="ignore"):
            d = canonical(q, rows[other])
        assert (b >= 0).all()
        assert (b[2500:] == 0).all()  # NaN / infinite query elements: nothing is dropped
        ok = ~np.isnan(d)
        assert not (b[ok] > d[ok]).any()
        assert (b[500:1500] > 0).mean() > 0.5  # not vacuous


def test_bound_is_not_vacuous_on_sift_shaped_rows():
    rows, q = datagen.sift_shaped(20_000, 128, 1), datagen.sift_shaped(100, 128, 2)
    c, offset, step, R = table(rows)
    rng = np.random.default_rng(0)
    other = rng.integers(0, len(rows), (len(q), 50))
    qq = np.repeat(q, 50, axis=0)
    b = bound(qq, c[other.ravel()], offset, step, R)
    d = canonical(qq, rows[other.ravel()])
    assert not (b > d).any()
    assert np.median(b / d) > 0.5
