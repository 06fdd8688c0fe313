"""K1's integer screening bound (DESIGN.md §4 "screen"): every element shares one code step S, so a candidate's bound is the triangle
inequality in code space, ((S sqrt(D))_rd - (r_q + R)_ru)_+^2 with D the exact squared code distance.  On the device it must never
exceed the canonical distance, including for queries outside the code range and queries with NaN or infinite elements, and searching
with it must give byte-identical results and counters to searching without a table (IDB_SCREEN=0), through every visited flavour
and the retry pass."""
import numpy as np
import pytest

from tests import datagen

pytestmark = pytest.mark.gpu

INVALID = 0xFFFFFFFF


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _adopt(abi, pts, storage="f32"):
    zero = np.full((len(pts), 4), INVALID, dtype=np.uint32)  # no edges: only the points matter here
    return abi.Index.from_graph(pts, zero, [], 2, storage=storage)


def _adversarial_rows(rng, n, dim):
    pts = rng.standard_normal((n, dim)).astype(np.float32)
    cols = np.arange(dim)
    pts[:, cols % 7 == 1] *= np.float32(1e-20)
    pts[:, cols % 7 == 2] *= np.float32(1e-40 / 3)  # subnormal
    pts[:, cols % 7 == 3] *= np.float32(1e17)
    grid = rng.integers(0, 256, size=(n, dim)).astype(np.float32) / np.float32(255) * np.float32(3) - np.float32(1.5)
    pts[:, cols % 7 == 4] = grid[:, cols % 7 == 4]  # codes on quantisation boundaries
    pts[:, cols % 7 == 5] = np.float32(0.25)  # constant elements
    pts[:100] = pts[100:200]  # exact duplicates
    return pts


@pytest.mark.parametrize("storage", ["f32", "bf16"])
@pytest.mark.parametrize("dim", [37, 128, 300, 1024])
def test_integer_bound_never_exceeds_the_canonical_distance(abi, monkeypatch, storage, dim):
    monkeypatch.setenv("IDB_SCREEN", "1")
    rng = np.random.default_rng(1000 + dim)
    n = 2000
    ix = _adopt(abi, _adversarial_rows(rng, n, dim), storage)
    stored = ix.export_graph()[0]
    fresh = rng.standard_normal((100, dim)).astype(np.float32)
    outside = stored[300:400].copy()
    outside[:, ::3] += np.float32(50)  # far above every element's code range
    outside[:, 1::3] -= np.float32(3e17)  # far below the largest element's range
    nan_q = stored[400:450].copy()
    nan_q[np.arange(50), rng.integers(0, dim, 50)] = np.nan
    inf_q = stored[450:500].copy()
    inf_q[np.arange(50), rng.integers(0, dim, 50)] = np.where(np.arange(50) % 2, np.inf, -np.inf).astype(np.float32)
    qs = [stored[:100], np.nextafter(stored[100:200], np.float32(np.inf)), (stored[200:300] + stored[500:600]) / np.float32(2),
          outside, fresh, fresh * np.float32(1e-30), fresh * np.float32(1e18), nan_q, inf_q]
    q = np.ascontiguousarray(np.concatenate(qs).astype(np.float32))
    nonfinite = ~np.isfinite(q).all(axis=1)
    qi = np.repeat(np.arange(len(q), dtype=np.uint32), 30)
    pid = rng.integers(0, n, size=len(qi)).astype(np.uint32)
    pid[::30] = np.arange(len(q), dtype=np.uint32) % n  # each stored-row query meets its own row
    bound, dist = ix.screen_bound(q, np.stack([qi, pid], axis=1))
    ix.close()
    assert (bound >= 0).all()
    assert (bound[nonfinite[qi]] == 0).all()  # a NaN or infinite query element: nothing is dropped
    ok = ~np.isnan(dist)
    assert not (bound[ok] > dist[ok]).any(), np.argwhere(ok & (bound > dist))[:5]
    assert (bound[ok] > 0.5 * dist[ok]).mean() > 0.3  # the bound is not vacuous


def test_integer_bound_is_tight_on_sift_rows(abi, monkeypatch):
    monkeypatch.setenv("IDB_SCREEN", "1")
    pts, q = datagen.sift_shaped(20_000, 128, 41), datagen.sift_shaped(200, 128, 42)
    ix = _adopt(abi, pts)
    rng = np.random.default_rng(3)
    qi = np.repeat(np.arange(len(q), dtype=np.uint32), 50)
    pid = rng.integers(0, len(pts), size=len(qi)).astype(np.uint32)
    bound, dist = ix.screen_bound(q, np.stack([qi, pid], axis=1))
    ix.close()
    assert not (bound > dist).any()
    assert np.median(bound / dist) > 0.5


def _graph(abi, pts, metric="l2sq"):
    built, _ = abi.Index.build(pts, metric=metric, seed=3, ef_construction=64)
    g = built.export_graph()
    built.close()
    return g


def _search(abi, monkeypatch, screen, g, q, ef, storage="f32", metric="l2sq", env=()):
    monkeypatch.setenv("IDB_SCREEN", str(screen))
    for k, v in env:
        monkeypatch.setenv(k, v)
    ix = abi.Index.from_graph(g[0], g[1], g[2], 32, storage=storage, metric=metric)
    ids, dist, lens = ix.search(q, ef_search=ef, k=10)
    out = (ids, dist, lens, ix.last_counters(len(q)), ix.last_full_fetches(), ix.last_retried(0xFFFFFFFF))
    ix.close()
    return out


def _same(on, off):
    assert (on[0] == off[0]).all()
    assert on[1].tobytes() == off[1].tobytes()
    assert (on[2] == off[2]).all()
    assert (on[3] == off[3]).all()
    n_dist = int(off[3][:, 1].sum() + off[3][:, 3].sum())
    assert off[4] >= n_dist  # every candidate fetched in full (the retry pass adds the aborted first attempts' rows)
    assert on[4] < off[4], "screening dropped no row"


FLAVOURS = {
    "b16": (),
    "hash": (("IDB_VIS_TIER", "0"),),
    "bitmap": (("IDB_VIS_TIER", "1"),),
    "retry": (("IDB_VIS_TIER", "0"), ("IDB_VIS_SLOTS", "1024")),
}


@pytest.mark.parametrize("flavour", sorted(FLAVOURS))
def test_every_visited_flavour_and_the_retry_pass_match_unscreened(abi, monkeypatch, flavour):
    g = _graph(abi, datagen.sift_shaped(8000, 128, 51))
    q = datagen.sift_shaped(300, 128, 52)
    env = FLAVOURS[flavour]
    off = _search(abi, monkeypatch, 0, g, q, 100, env=env)
    on = _search(abi, monkeypatch, 1, g, q, 100, env=env)
    _same(on, off)
    if flavour == "retry":
        assert on[5] > 0 and off[5] > 0


def test_queries_with_non_finite_elements_match_unscreened(abi, monkeypatch):
    g = _graph(abi, datagen.sift_shaped(6000, 128, 61))
    q = datagen.sift_shaped(200, 128, 62)
    q[::4, 5] = np.nan
    q[1::4, 7] = np.inf
    q[2::4] *= np.float32(100)  # far outside the code range
    off = _search(abi, monkeypatch, 0, g, q, 64)
    on = _search(abi, monkeypatch, 1, g, q, 64)
    assert (on[0] == off[0]).all()
    assert on[1].tobytes() == off[1].tobytes()
    assert (on[2] == off[2]).all()
    assert (on[3] == off[3]).all()
