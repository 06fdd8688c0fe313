"""The cosine metric on the CPU (DESIGN.md §3a): its CPU statement (tests/cosine_ref.py over the oracle's canonical squared L2) —
normalisation and cosine search against float64 numpy — the new binding surface, and the no-device behaviour of the new entry
points."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from tests import cosine_ref as cref
from tests import datagen
from tests.conftest import ROOT, _has_gpu


def _abi():
    from instant_distance_b200 import _abi

    return _abi


def _cos_dist64(q, p):
    """float64 0.5 * |q^ - p^|^2 for every (query, point) pair: 1 - cos for non-zero rows; a zero row stays zero when normalised, so
    it is at 0.5 from every non-zero row."""
    q, p = q.astype(np.float64), p.astype(np.float64)
    qn = np.linalg.norm(q, axis=1, keepdims=True)
    pn = np.linalg.norm(p, axis=1, keepdims=True)
    qh = np.divide(q, qn, out=np.zeros_like(q), where=qn > 0)
    ph = np.divide(p, pn, out=np.zeros_like(p), where=pn > 0)
    return 0.5 * ((qh * qh).sum(1)[:, None] + (ph * ph).sum(1)[None, :]) - qh @ ph.T


def test_normalised_rows_are_unit_for_every_dim(oracle):
    rng = np.random.default_rng(1)
    for dim in list(range(1, 140)) + [255, 256, 257, 300, 511, 768, 1023, 1024, 1025, 1100, 1536, 2049, 4099, 4100]:
        x = (rng.standard_normal((6, dim)) * rng.choice([1e-3, 1.0, 1e3], (6, 1))).astype(np.float32)
        y = cref.normalize(oracle, x).astype(np.float64)
        assert np.abs((y * y).sum(1) - 1.0).max() < 1e-5, dim


def test_zero_and_non_finite_rows(oracle):
    z = cref.normalize(oracle, np.zeros((2, 37), np.float32))
    assert z.tobytes() == np.zeros((2, 37), np.float32).tobytes()  # +0.0 everywhere
    big = cref.normalize(oracle, np.full((1, 8), 1e20, np.float32))  # the sum of squares overflows: x / inf = 0
    assert (big == 0).all()
    inf = cref.normalize(oracle, np.array([[np.inf, 1.0, 0.0]], np.float32))  # inf / inf = NaN, written canonically
    assert inf.view(np.uint32).tolist() == [[0x7FC00000, 0, 0]]
    nan = cref.normalize(oracle, np.array([[np.nan, 1.0]], np.float32))
    assert (nan.view(np.uint32) == 0x7FC00000).all()


def test_cosine_distances_match_float64(oracle):
    pts = datagen.uniform(3000, 96, 2) * 2 - 1
    pts[17] = 0.0
    q = datagen.uniform(50, 96, 3) * 2 - 1
    ids, dist = cref.bruteforce(oracle, pts, q, 10)
    ref = _cos_dist64(q, pts)
    assert np.abs(dist - np.take_along_axis(ref, ids.astype(np.int64), 1)).max() < 1e-6
    zq = np.zeros((1, 96), np.float32)  # a zero query: 0 from the zero row, 0.5 * |p^|^2 = 0.5 from every other point
    zi, zd = cref.bruteforce(oracle, pts, zq, 5)
    assert zi[0, 0] == 17 and zd[0, 0] == 0.0 and np.abs(zd[0, 1:] - 0.5).max() < 1e-6


def test_cosine_bruteforce_top10_matches_numpy(oracle):
    pts = datagen.sift_shaped(5000, 64, 4)
    q = datagen.sift_shaped(200, 64, 5)
    ids, _ = cref.bruteforce(oracle, pts, q, 10, threads=4)
    ref = _cos_dist64(q, pts)
    order = np.argsort(ref, axis=1, kind="stable")
    checked = 0
    for i in range(len(q)):
        d = np.sort(ref[i])
        if d[10] - d[9] < 1e-6:  # exact near-tie at the cut: either id is a correct 10th neighbour
            continue
        assert set(ids[i].tolist()) == set(order[i, :10].tolist()), i
        checked += 1
    assert checked > 150


def test_cosine_hnsw_recall_on_the_cpu(oracle):
    pts = datagen.sift_shaped(20000, 128, 6)
    q = datagen.sift_shaped(300, 128, 7)
    ix, ids = cref.build(oracle, pts, seed=3, threads=8)
    g = ix.export()
    inv = np.empty(len(ids), np.int64)
    inv[ids] = np.arange(len(ids))
    assert np.abs((g.points.astype(np.float64) ** 2).sum(1) - 1).max() < 1e-5  # the index stores unit rows
    got, dist, _ = cref.search(oracle, ix, q, ef_search=100, k=10, threads=8)
    truth, _ = cref.bruteforce(oracle, pts, q, 10, threads=8)
    rec = np.mean([len(set(inv[a].tolist()) & set(b.tolist())) / 10 for a, b in zip(got, truth)])
    assert rec > 0.95, rec
    assert (dist >= 0).all() and (dist <= 2).all()


def test_metric_constants_and_struct_layouts():
    abi = _abi()
    header = open(os.path.join(ROOT, "include", "instant_distance_b200.h")).read()
    consts = dict(re.findall(r"#define IDB_METRIC_(\w+) (\d+)u", header))
    assert {k.lower(): int(v) for k, v in consts.items()} == abi.METRIC
    # the metric travels as an argument and through idb_index_metric: both public structs keep their size
    assert C.sizeof(abi.Params) == 64 and C.sizeof(abi.Info) == 288
    with pytest.raises(ValueError):
        abi.Index.build(np.ones((4, 4), np.float32), metric="dot")


def test_from_graph_ex_rejects_non_unit_rows_without_a_device():
    abi = _abi()
    pts = np.array([[0.6, 0.8], [0.0, 0.0], [3.0, 4.0]], np.float32)
    zero = np.full((3, 4), 0xFFFFFFFF, np.uint32)
    with pytest.raises(abi.IdbError) as e:
        abi.Index.from_graph(pts, zero, [], 2, metric="cosine")
    assert e.value.status == abi.ERR_INVALID_ARG and "row 2" in str(e.value)
    h = C.c_void_p()
    st = abi.lib().idb_index_from_graph_ex(abi.ptr(pts, C.c_float), 3, 2, 2, 10, abi.ptr(zero, C.c_uint32), 0, None, None, 0, 7, 0,
                                           C.byref(h))
    assert st == abi.ERR_INVALID_ARG and b"metric" in abi.lib().idb_last_error()


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device behaviour")
def test_new_calls_fail_loudly_without_a_device():
    abi = _abi()
    with pytest.raises(abi.IdbError) as e:
        abi.normalize(np.ones((3, 5), np.float32))
    assert e.value.status == abi.ERR_CUDA and "no CPU fallback" in str(e.value)
    unit = np.array([[0.6, 0.8], [0.0, 0.0]], np.float32)
    with pytest.raises(abi.IdbError) as e:
        abi.Index.from_graph(unit, np.full((2, 4), 0xFFFFFFFF, np.uint32), [], 2, metric="cosine")
    assert e.value.status == abi.ERR_CUDA
    with pytest.raises(abi.IdbError) as e:
        abi.Index.build(np.ones((8, 4), np.float32), metric="cosine")
    assert e.value.status == abi.ERR_CUDA
