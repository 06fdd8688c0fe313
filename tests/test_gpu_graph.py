"""Calls that change an index hold it exclusively: idb_index_set_id_map waits for the searches already enqueued on every lane, so a
search reports every id through the map it was enqueued with, never partly through the next one."""
import os

import numpy as np
import pytest

from tests import datagen

pytestmark = pytest.mark.gpu

INVALID = 0xFFFFFFFF


def test_set_id_map_waits_for_an_exact_search_on_another_lane(oracle):
    import torch

    from instant_distance_b200 import _abi

    n, dim, nq, k = 200_000, 128, 4096, 10  # an exact search of tens of ms: still running when set_id_map is called
    pts = datagen.sift_shaped(n, dim, 41)
    q = datagen.sift_shaped(nq, dim, 42)
    zero = np.full((n, 4), INVALID, dtype=np.uint32)
    ix = _abi.Index.from_graph(pts, zero, [], 2)  # an empty graph: the exact search reads the rows only
    pid = np.arange(n, dtype=np.uint32)
    map_a, map_b = pid + 10**6, pid + 2 * 10**6
    ix.set_id_map(map_a)
    d_q = torch.from_numpy(q).cuda()
    ids = torch.empty(nq * k, dtype=torch.int32, device="cuda")
    dist = torch.empty(nq * k, dtype=torch.float32, device="cuda")
    lens = torch.empty(nq, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()

    def search():
        ix.exact_search_device(d_q.data_ptr(), nq, k, ids.data_ptr(), dist.data_ptr(), lens.data_ptr(), lane=1)

    search()  # once to load its kernels and grow the lane's scratch: the next call only enqueues
    ix.sync()
    search()
    ix.set_id_map(map_b)  # a map of the same size replaces A; none is ever freed while the search runs
    ix.sync()
    got_ids = ids.cpu().numpy().view(np.uint32).reshape(nq, k)
    got_dist = dist.cpu().numpy().reshape(nq, k)
    assert ((got_ids >= map_a[0]) & (got_ids <= map_a[-1])).all(), f"{int((got_ids >= map_b[0]).sum())} ids through map B"
    want_ids, want_dist = oracle.bruteforce(pts, q, k, threads=os.cpu_count() or 1)
    assert (got_ids - map_a[0] == want_ids).all()
    assert got_dist.tobytes() == want_dist.tobytes()
    assert (lens.cpu().numpy() == k).all()
