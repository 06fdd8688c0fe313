"""fp16 rounding as the library states it (DESIGN.md §3b): f32 -> fp16 round to nearest even, subnormals kept, a finite value that
rounds to infinity (|x| >= 65520) refused.  `rne_bits` is an integer statement of that rounding; tests/test_f16_cpu.py pins numpy's
`astype(np.float16)` against it on `boundary_values()`, so the GPU tests can use numpy as the rounding reference."""
import numpy as np

F16_MAX = 65504.0
F16_REFUSED = 65520.0  # the midpoint between 65504 and 2^16: ties to even round it to infinity


def f16_round(x):
    """The f32 rows an fp16 index stores for x, widened back to f32 (numpy's rounding)."""
    return np.ascontiguousarray(x, dtype=np.float32).astype(np.float16).astype(np.float32)


def rne_bits(x):
    """fp16 bit patterns of the non-NaN f32 values x by integer arithmetic alone: round to nearest, ties to even."""
    u = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32).astype(np.int64)
    sign = (u >> 16) & 0x8000
    a = u & 0x7FFFFFFF
    exp = a >> 23
    out = np.zeros_like(a)
    # normal fp16 results: rebias the exponent (127 -> 15) and round away 13 mantissa bits; a carry moves into the exponent
    nrm = a >= 0x38800000  # 2^-14, the smallest normal fp16
    r = a - (112 << 23)
    out = np.where(nrm, (r + 0xFFF + ((r >> 13) & 1)) >> 13, out)
    # subnormal fp16 results: the value in units of 2^-24, rounded to an integer
    m = np.where(exp > 0, (a & 0x7FFFFF) | 0x800000, 0)  # f32 subnormals are far below 2^-25: they round to 0
    s = np.clip(126 - exp, 1, 40)                         # value * 2^24 = m * 2^-(126 - exp)
    half = np.left_shift(np.int64(1), s - 1)
    sub = (m + half - 1 + ((m >> s) & 1)) >> s
    out = np.where(nrm, out, np.where(exp > 0, sub, 0))
    out = np.where(a >= 0x477FF000, 0x7C00, out)          # |x| >= 65520 (and inf): infinity
    return (out | sign).astype(np.uint16)


def boundary_values():
    """Every positive finite fp16 value (0 and the subnormals included) as f32, every midpoint between neighbours and one f32 ulp
    either side of each, 65519.996 (the largest f32 below 65520), all with both signs.  Every one of them is accepted by fp16
    storage; the midpoint above 65504 (65520) is not in the set."""
    v = np.arange(0x7C00, dtype=np.uint16).view(np.float16).astype(np.float32)
    mid = ((v[:-1].astype(np.float64) + v[1:]) / 2).astype(np.float32)  # 12 significant bits: exact in f32
    assert ((mid.astype(np.float64) * 2) == (v[:-1].astype(np.float64) + v[1:])).all()
    up, down = np.nextafter(mid, np.float32(np.inf)), np.nextafter(mid, np.float32(0))
    top = np.nextafter(np.float32(F16_REFUSED), np.float32(0))
    pos = np.concatenate([v, mid, up, down, [top]]).astype(np.float32)
    return np.concatenate([pos, -pos]).astype(np.float32)
