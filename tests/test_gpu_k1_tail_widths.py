"""K1's distance batches at every width of the ladder (hnsw_device.cuh batch_width), against the oracle, bit for bit: ids, distance
bytes, lengths and per-layer counters.

An expansion's fresh rows (n_new, up to 2M) go through full batches of NB rows and one narrower last batch; screening shrinks n_new
further.  M = 4, 8, 32 and 64 make n_new reach every remainder 1 .. 2M and every width boundary; dims 20, 37, 128 (FULL), 300 and
1000 put the batches in the CH = 1, 3 and 8 cells; every row storage, both metrics, screening off and on, and the retry pass.
"""
import pytest

from tests.test_gpu_k1_instantiations import _graph, _run, _same, _want

pytestmark = pytest.mark.gpu

DIMS = (20, 37, 128, 300, 1000)
MS = (4, 8, 32, 64)
STORAGES = ("f32", "bf16", "f16", "q8")
EF = 64


@pytest.fixture(scope="module")
def abi():
    from instant_distance_b200 import _abi

    assert _abi.lib().idb_device_count() >= 1
    return _abi


def _indexes(abi, oracle, g, M, storage, metric):
    """A GPU index of the graph with this row storage, and the oracle on the rows the GPU index holds."""
    p, zero, upper, _ = g
    ix = abi.Index.from_graph(p, zero, upper, M, storage=storage, metric=metric)
    rows = ix.export_graph()[0]
    return ix, oracle.from_graph(oracle.Graph(rows, zero, upper, M, 100))


@pytest.mark.parametrize("metric", ["l2sq", "cosine"])
@pytest.mark.parametrize("M", MS)
@pytest.mark.parametrize("dim", DIMS)
def test_every_width_matches_the_oracle(abi, oracle, monkeypatch, dim, M, metric):
    g = _graph("sift", dim, M, metric=metric)
    for storage in STORAGES:
        for screen in (0, 1):
            monkeypatch.setenv("IDB_SCREEN", str(screen))
            ix, ox = _indexes(abi, oracle, g, M, storage, metric)
            _same(_run(ix, g[3], EF), _want(oracle, ox, g[3], EF, metric), f"{storage} {metric} dim {dim} M {M} IDB_SCREEN={screen}")
            ix.close()


@pytest.mark.parametrize("storage", STORAGES)
@pytest.mark.parametrize("dim", DIMS)
def test_retry_pass(abi, oracle, monkeypatch, dim, storage):
    """1024-slot hash sets overflow in every query: the retry pass re-runs them through the same batches."""
    g = _graph("sift", dim, 32, n=4000)
    monkeypatch.setenv("IDB_VIS_TIER", "0")
    monkeypatch.setenv("IDB_VIS_SLOTS", "1024")
    ix, ox = _indexes(abi, oracle, g, 32, storage, "l2sq")
    _same(_run(ix, g[3], 100), _want(oracle, ox, g[3], 100), f"retry {storage} dim {dim}")
    assert ix.last_retried(0xFFFFFFFF) > 0
    ix.close()
