"""K1's screen in its eight-lanes-per-row layout (DESIGN.md §4 "screen") on tables whose rows are padded to 16 bytes (DESIGN.md §2:
dim % 16 != 0): searches with IDB_SCREEN=0 and =1 give byte-identical ids, distances, lengths and per-layer counters, equal to the
oracle's, for f32, bf16 and fp16 rows and both metrics.  M = 64 gives up to 128 fresh candidates per expansion, so the screen runs
several batches per expansion.  The retry pass re-runs the screen from a fresh layer.  The bound K1 compares never exceeds the canonical distance at these widths, and it is not vacuous."""
import numpy as np
import pytest

from tests.test_gpu_k1_instantiations import _graph, _run, _same, _want

pytestmark = pytest.mark.gpu

PADDED_DIMS = (20, 37, 100, 300, 700)  # nchunks 5, 10, 25, 75, 175: CH = 1, 1, 1, 3, 6
M = 64
EF = 64


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _search(abi, monkeypatch, screen, g, storage, metric, env=()):
    monkeypatch.setenv("IDB_SCREEN", str(screen))
    for k, v in env:
        monkeypatch.setenv(k, v)
    ix = abi.Index.from_graph(g[0], g[1], g[2], M, storage=storage, metric=metric)
    got = _run(ix, g[3], EF)
    out = got, ix.last_full_fetches(), ix.last_retried(0xFFFFFFFF), ix.export_graph()[0]
    ix.close()
    return out


def _oracle_results(oracle, g, rows, metric):
    ox = oracle.from_graph(oracle.Graph(rows, g[1], g[2], M, 100))
    return _want(oracle, ox, g[3], EF, metric)


@pytest.mark.parametrize("metric", ["l2sq", "cosine"])
@pytest.mark.parametrize("storage", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("dim", PADDED_DIMS)
def test_screened_search_matches_unscreened_and_the_oracle(abi, oracle, monkeypatch, dim, storage, metric):
    g = _graph("sift", dim, M, metric=metric)
    on, full_on, _, rows = _search(abi, monkeypatch, 1, g, storage, metric)
    off, full_off, _, _ = _search(abi, monkeypatch, 0, g, storage, metric)
    what = f"dim {dim} {storage} {metric}"
    want = _oracle_results(oracle, g, rows, metric)
    _same(off, want, what + " unscreened")
    _same(on, want, what + " screened")
    assert on[4] == off[4]
    assert full_on < full_off, f"{what}: screening dropped no row"


@pytest.mark.parametrize("dim", [37, 300])
def test_retry_pass_screens_the_same(abi, oracle, monkeypatch, dim):
    g = _graph("sift", dim, M)
    env = (("IDB_VIS_TIER", "0"), ("IDB_VIS_SLOTS", "1024"))
    on, full_on, retried_on, rows = _search(abi, monkeypatch, 1, g, "f32", "l2sq", env)
    off, full_off, retried_off, _ = _search(abi, monkeypatch, 0, g, "f32", "l2sq", env)
    assert retried_on > 0 and retried_off > 0
    want = _oracle_results(oracle, g, rows, "l2sq")
    _same(off, want, f"dim {dim} retry unscreened")
    _same(on, want, f"dim {dim} retry screened")
    assert full_on < full_off


@pytest.mark.parametrize("storage", ["f32", "bf16", "f16"])
@pytest.mark.parametrize("dim", PADDED_DIMS)
def test_bound_at_padded_widths(abi, monkeypatch, dim, storage):
    monkeypatch.setenv("IDB_SCREEN", "1")
    from tests import datagen

    pts, q = datagen.sift_shaped(4000, dim, 70 + dim), datagen.sift_shaped(100, dim, 80 + dim)
    zero = np.full((len(pts), 4), 0xFFFFFFFF, dtype=np.uint32)
    ix = abi.Index.from_graph(pts, zero, [], 2, storage=storage)
    rows = ix.export_graph()[0]
    q = np.concatenate([q, rows[:50]])  # stored rows meet themselves: bound 0
    rng = np.random.default_rng(dim)
    qi = np.repeat(np.arange(len(q), dtype=np.uint32), 40)
    pid = rng.integers(0, len(pts), size=len(qi)).astype(np.uint32)
    pid[(qi >= 100) & (np.arange(len(qi)) % 40 == 0)] = np.arange(50, dtype=np.uint32)
    bound, dist = ix.screen_bound(q, np.stack([qi, pid], axis=1))
    ix.close()
    assert (bound >= 0).all()
    assert not (bound > dist).any(), np.argwhere(bound > dist)[:5]
    assert (bound[dist == 0] == 0).all()
    assert np.median(bound[qi < 100] / dist[qi < 100]) > 0.2
