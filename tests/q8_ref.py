"""numpy / f64 statement of the q8 quantiser (DESIGN.md §3c), the reference the q8 tests compare the device against.

For a row x of dim finite f32 values: A = max |x_i|; A == 0 gives e = -149, b = 0, c = 0.  Otherwise e_lo = max(-149, ilogb(A) - 23)
and e is the smallest integer >= e_lo with ceil(max x / 2^e) - floor(min x / 2^e) <= 255; b = floor(min x / 2^e) and
c_i = rint(x_i / 2^e) - b (ties to even).  The dequantised row is (b + c_i) 2^e, an exact f32.  Every step is exact in f64: x / 2^e is
a power-of-two scaling of an f32.  A row is refused when an element is not finite, or when its header o = b 2^e or a dequantised
element would overflow f32.
"""
import numpy as np

E_MIN = -149


def _ilogb(a):
    return np.frexp(a)[1].astype(np.int64) - 1  # a > 0 (f64, so f32 subnormals are normal here)


def grid(rows):
    """rows: (n, dim) f32, finite.  Returns (e, b, c): e and b int64 per row, c uint8 (n, dim)."""
    x = np.ascontiguousarray(rows, np.float32).astype(np.float64)
    n = x.shape[0]
    mn, mx = x.min(axis=1), x.max(axis=1)
    A = np.maximum(np.abs(mn), np.abs(mx))
    zero = A == 0
    e = np.full(n, E_MIN, np.int64)
    e[~zero] = np.maximum(E_MIN, _ilogb(A[~zero]) - 23)
    while True:
        wide = np.ceil(np.ldexp(mx, -e)) - np.floor(np.ldexp(mn, -e)) > 255
        if not wide.any():
            break
        e[wide] += 1
    b = np.floor(np.ldexp(mn, -e))
    c = np.rint(np.ldexp(x, -e[:, None])) - b[:, None]
    assert (c >= 0).all() and (c <= 255).all()
    return e, b.astype(np.int64), c.astype(np.uint8)


def header(e, b):
    """(o, s) per row as f32: o = b 2^e, s = 2^e (inf where o overflows)."""
    with np.errstate(over="ignore"):
        return np.ldexp(b.astype(np.float64), e).astype(np.float32), np.ldexp(1.0, e).astype(np.float32)


def dequantize(e, b, c):
    """(b + c) 2^e as f32 (exact for rows that are not refused); -0 comes out as +0."""
    with np.errstate(over="ignore"):
        return np.ldexp(b[:, None].astype(np.float64) + c, e[:, None]).astype(np.float32) + np.float32(0.0)


def refused(rows):
    """Per row: True when the q8 storage refuses it (a NaN / inf element, or a header or dequantised value beyond f32)."""
    x = np.ascontiguousarray(rows, np.float32)
    bad = ~np.isfinite(x).all(axis=1)
    ok = ~bad
    if ok.any():
        e, b, c = grid(x[ok])
        big = np.ldexp(1.0, 128)
        hi = np.maximum(np.abs(b), np.abs(b[:, None] + c.astype(np.int64)).max(axis=1))
        bad[ok] = np.ldexp(hi.astype(np.float64), e) >= big
    return bad


def quantize(rows):
    """(e, b, c, dequantised rows) of rows none of which is refused."""
    e, b, c = grid(rows)
    return e, b, c, dequantize(e, b, c)


def roundtrip(rows):
    """The rows a q8 index stores (and exports) for these f32 rows."""
    return quantize(rows)[3]


def boundary_rows(dim=8):
    """Rows at the quantiser's edges: spans at exactly 255 steps and one ulp either side, rint ties, powers of two, constant rows,
    subnormals, +-0, tiny negative minima, mixed signs and extreme scales.  All accepted (finite, no overflow)."""
    f = np.float32
    out = []

    def add(v):
        r = np.zeros(dim, f)
        v = np.asarray(v, f)[:dim]  # (a row narrower than the case keeps its first elements)
        r[: len(v)] = v
        out.append(r)

    for e in (-140, -20, -3, 0, 5, 60, 100):
        s = np.ldexp(1.0, e)
        for lo in (0.0, -7.0, 3.0, -255.0):
            top = f((lo + 255) * s)
            add([lo * s, top])
            add([lo * s, np.nextafter(top, f(np.inf))])
            add([lo * s, np.nextafter(top, f(-np.inf))])
        for k in range(8):  # x / 2^e at .5: ties to even
            add([0.0, (k + 0.5) * s, 255 * s])
    for p in (-149, -126, -100, -1, 0, 1, 23, 24, 100, 127):
        a = np.ldexp(1.0, p)
        add([a])
        add([a, -a])
        add([a] * dim)
        add([-a] * dim)
        add([a, np.nextafter(f(a), f(0))])
    for v in (1000.0, 1e-3, 3.14159, -2.5e-40, 1e-45):
        add([v] * dim)
        add([v])
    add(np.float32(1000.0) + np.float32(1e-3) * np.linspace(-1, 1, dim, dtype=f))
    add([-0.0, 0.0, -0.0])
    add([-1e-45, 1e-45])
    add([-1e-45, 0.0, 3.0])
    add([-2e-45, 7e-45, 1.5e-44])
    add([np.ldexp(1.0, -149), -np.ldexp(1.0, -130)])
    add([-1e-40, 1e30])
    add([3.3e38, 1.0])
    add([1e38, -1e38])
    add([np.ldexp(1.0, 60), -np.ldexp(1.0, -60)])
    return np.stack(out)


def overflow_rows(dim=4):
    """Finite rows the q8 storage refuses, and the accepted rows right below them."""
    f = np.float32
    fmax = np.finfo(f).max
    refused_rows = [[fmax, -fmax], [fmax, 0.0], [-fmax, 0.0], [fmax], [-fmax]]
    accepted = [[3.3e38, 1.0], [np.ldexp(f(255), 119), 0.0], [-np.ldexp(f(255), 119), 0.0], [np.ldexp(f(1), 127)]]

    def pad(rows):
        a = np.zeros((len(rows), dim), f)
        for i, r in enumerate(rows):
            a[i, : len(r)] = r
        return a

    return pad(refused_rows), pad(accepted)
