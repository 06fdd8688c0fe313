"""K1's screening pass (DESIGN.md §4 "screen"): a candidate whose 8-bit-code lower bound already exceeds the furthest distance of a
full `nearest` is not fetched in full.  It must never change a result: searches with IDB_SCREEN=0 and =1 give byte-identical ids,
distances, lengths and per-layer counters, and the bound never exceeds the canonical distance.  The full-fetch tally shows that
screening actually happened."""
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


def _search(abi, monkeypatch, screen, g, q, ef, storage, metric):
    monkeypatch.setenv("IDB_SCREEN", str(screen))
    ix = abi.Index.from_graph(g[0], g[1], g[2], 32, storage=storage, metric=metric)
    ids, dist, lens = ix.search(q, ef_search=ef, k=10)
    counters = ix.last_counters(len(q))
    full = ix.last_full_fetches()
    ix.close()
    return ids, dist, lens, counters, full


CASES = {
    "sift": (lambda: datagen.sift_shaped(20_000, 128, 1), lambda: datagen.sift_shaped(500, 128, 2), "f32", "l2sq", 0.5),
    "uniform": (lambda: datagen.uniform(20_000, 128, 3), lambda: datagen.uniform(500, 128, 4), "f32", "l2sq", 1.0),
    "grid_ties": (lambda: datagen.grid_ties(6000, 8, 5), lambda: datagen.grid_ties(300, 8, 6), "f32", "l2sq", 1.0),
    "cosine": (lambda: datagen.sift_shaped(20_000, 128, 7), lambda: datagen.sift_shaped(500, 128, 8), "f32", "cosine", 0.5),
    "bf16": (lambda: datagen.sift_shaped(20_000, 128, 9), lambda: datagen.sift_shaped(500, 128, 10), "bf16", "l2sq", 0.5),
    "dim300": (lambda: datagen.sift_shaped(8000, 300, 11), lambda: datagen.sift_shaped(300, 300, 12), "f32", "l2sq", 1.0),
    "bf16_dim768": (lambda: datagen.sift_shaped(4000, 768, 13), lambda: datagen.sift_shaped(200, 768, 14), "bf16", "l2sq", 1.0),
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_screen_on_and_off_give_identical_results(abi, monkeypatch, case):
    make_pts, make_q, storage, metric, max_share = CASES[case]
    pts, q = make_pts(), make_q()
    built, _ = abi.Index.build(pts, metric=metric, seed=3, ef_construction=64)
    g = built.export_graph()
    built.close()
    ef = 100
    off = _search(abi, monkeypatch, 0, g, q, ef, storage, metric)
    on = _search(abi, monkeypatch, 1, g, q, ef, storage, metric)
    assert (on[0] == off[0]).all()
    assert on[1].tobytes() == off[1].tobytes()
    assert (on[2] == off[2]).all()
    assert (on[3] == off[3]).all()  # every fresh candidate is still counted as a distance evaluation
    n_dist = int(off[3][:, 1].sum() + off[3][:, 3].sum())
    assert off[4] == n_dist  # unscreened: every candidate is fetched in full
    assert on[4] <= n_dist
    assert on[4] <= max_share * n_dist, f"{case}: {on[4]} of {n_dist} rows fetched in full"


def test_sift_fetches_far_fewer_rows(abi, monkeypatch):
    pts, q = datagen.sift_shaped(50_000, 128, 21), datagen.sift_shaped(1000, 128, 22)
    built, _ = abi.Index.build(pts, seed=1)
    g = built.export_graph()
    built.close()
    on = _search(abi, monkeypatch, 1, g, q, 100, "f32", "l2sq")
    n_dist = int(on[3][:, 1].sum() + on[3][:, 3].sum())
    assert on[4] < 0.3 * n_dist, f"{on[4]} of {n_dist} rows fetched in full"


def _adopt(abi, pts, storage="f32"):
    n = len(pts)
    zero = np.full((n, 4), INVALID, dtype=np.uint32)  # no edges: only the points matter here
    return abi.Index.from_graph(pts, zero, [], 2, storage=storage)


@pytest.mark.parametrize("storage", ["f32", "bf16"])
@pytest.mark.parametrize("dim", [128, 37, 300, 1024])
def test_bound_never_exceeds_the_canonical_distance(abi, monkeypatch, storage, dim):
    monkeypatch.setenv("IDB_SCREEN", "1")
    rng = np.random.default_rng(dim)
    n = 3000
    pts = rng.standard_normal((n, dim)).astype(np.float32)
    cols = np.arange(dim)
    # elements of very different magnitudes: squares that underflow, squares near the top of the range
    pts[:, cols % 7 == 1] *= np.float32(1e-20)
    pts[:, cols % 7 == 2] *= np.float32(1e-40 / 3)  # subnormal
    pts[:, cols % 7 == 3] *= np.float32(1e17)
    # elements on an exact 255-step grid (codes at quantisation boundaries), and constant elements
    grid = rng.integers(0, 256, size=(n, dim)).astype(np.float32) / np.float32(255) * np.float32(3) - np.float32(1.5)
    pts[:, cols % 7 == 4] = grid[:, cols % 7 == 4]
    pts[:, cols % 7 == 5] = np.float32(0.25)
    pts[:100] = pts[100:200]  # exact duplicates
    ix = _adopt(abi, pts, storage)
    stored = ix.export_graph()[0]
    # queries: stored rows (exact ties: distance 0), stored rows one ulp away, half-way between two rows, fresh rows, scaled rows
    qs = [stored[:200], np.nextafter(stored[200:400], np.float32(np.inf)), (stored[400:600] + stored[600:800]) / np.float32(2)]
    fresh = rng.standard_normal((200, dim)).astype(np.float32)
    qs += [fresh, fresh * np.float32(1e-30), fresh * np.float32(1e18), stored[800:1000] * np.float32(1.0000001)]
    q = np.ascontiguousarray(np.concatenate(qs).astype(np.float32))
    nq = len(q)
    qi = np.repeat(np.arange(nq, dtype=np.uint32), 40)
    pid = rng.integers(0, n, size=len(qi)).astype(np.uint32)
    pid[::40] = np.arange(nq, dtype=np.uint32) % n  # includes each stored-row query's own row
    bound, dist = ix.screen_bound(q, np.stack([qi, pid], axis=1))
    ix.close()
    ok = ~np.isnan(dist)
    assert ok.mean() > 0.9
    assert not (bound[ok] > dist[ok]).any(), np.argwhere(bound > dist)[:5]
    assert (bound >= 0).all()
    assert (bound[ok] > 0.5 * dist[ok]).mean() > 0.3  # the bound is not vacuous


def test_no_table_for_non_finite_rows(abi, monkeypatch):
    monkeypatch.setenv("IDB_SCREEN", "1")
    pts = datagen.sift_shaped(500, 16, 31)
    pts[7, 3] = np.inf
    ix = _adopt(abi, pts)
    with pytest.raises(abi.IdbError) as e:
        ix.screen_bound(pts[:2], np.array([[0, 1]], dtype=np.uint32))
    assert e.value.status == abi.ERR_UNSUPPORTED
    ix.close()
    monkeypatch.setenv("IDB_SCREEN", "0")
    ix = _adopt(abi, datagen.sift_shaped(500, 16, 31))
    with pytest.raises(abi.IdbError):
        ix.screen_bound(pts[:2], np.array([[0, 1]], dtype=np.uint32))
    ix.close()
