"""CPU model of the layout K1's screen reads code rows in (DESIGN.md §4 "screen"; hnsw_device.cuh screen_candidates), lane by lane:

  table:  rows of cwords = round_up(nchunks, 4) u32, zero past nchunks, laid end to end (a word read past cwords is the next row's);
  lanes:  group grp = lane >> 3 takes rows b0 + NSL grp + i in its slots i < NSL (NSL = 8, 4, 2, 2, 1, 1 at CH = 1, 2, 3, 4, 6, 8),
          lane l loads the 16-byte words 4 (l & 7) + 32 j (j < CH) of each, unless that word lies at or past cwords;
  query:  lane l holds word l + 32 j (the canonical layout) and gathers its slice 4 (l & 7) + 32 j .. +3 from lanes 4 (l & 7) + k;
  reduce: batch_butterfly<NSL, ..., W = 8> over the eight lanes of a group, then lane l holds row b0 + NSL (l >> 3) + (l & (NSL - 1));
  vote:   lanes with l & 7 < NSL vote, and the survivors are compacted by their ballot bit.

For every CH, padded table widths and every n_new of a K1 row (1..128) it checks that each row's reduced value is
D = sum (qc - c)^2 over its real words, that the padding words add 0, and that the survivors come out in row order."""
import numpy as np
import pytest

INVALID = 0xFFFFFFFF
DIMS = (20, 37, 100, 128, 300, 700, 1000, 1024)
SLOTS = {1: 8, 2: 4, 3: 2, 4: 2, 6: 1, 8: 1}
LANE = np.arange(32)


def code_words(nchunks):
    return (nchunks + 3) & ~3


def sq_dist(a, b):
    """Per row (first axis) of two u32 word arrays, sum over their bytes of (a - b)^2, as VABSDIFF4 + IDP.4A add them."""
    a, b = np.broadcast_arrays(a, b)
    sh = 8 * np.arange(4, dtype=np.uint64)
    d = (a[..., None] >> sh & 0xFF).astype(np.int64) - (b[..., None] >> sh & 0xFF).astype(np.int64)
    return (d * d).reshape(len(d), -1).sum(axis=1)


def batch_butterfly(p, width):
    """hnsw_device.cuh batch_butterfly on u32 partials: p is (32 lanes, NB); returns what each lane holds."""
    p = p.copy()
    nb = p.shape[1]
    off, m = 1, nb
    while m > 1:
        up = (LANE & off) != 0
        q = p.copy()
        for i in range(m // 2):
            send = np.where(up, p[:, 2 * i], p[:, 2 * i + 1])
            keep = np.where(up, p[:, 2 * i + 1], p[:, 2 * i])
            q[:, i] = keep + send[LANE ^ off]
        p, off, m = q, off << 1, m >> 1
    o = nb
    while o < width:
        p[:, 0] = p[:, 0] + p[LANE ^ o, 0]
        o <<= 1
    return p[:, 0]


def screen(flat, cwords, ch, qwords, cpid, n_new, keep_row):
    """The warp's screen over cpid[0, n_new): (D per row, survivors in compaction order)."""
    nsl = SLOTS[ch]
    ns = 4 * nsl
    grp, sub = LANE >> 3, LANE & 7
    first = nsl * grp
    # query slice: word 4 sub + k + 32 j comes from lane 4 sub + k, which holds word (4 sub + k) + 32 j
    qc = np.stack([np.stack([qwords[(4 * sub + k) + 32 * j] for k in range(4)], axis=-1) for j in range(ch)], axis=1)  # (32, CH, 4)
    cok = np.stack([4 * sub + 32 * j < cwords for j in range(ch)], axis=1)  # (32, CH)
    seen = {}
    out = []
    kept = 0
    cpid = cpid.copy()
    for b0 in range(0, n_new, ns):
        p = np.zeros((32, nsl), dtype=np.int64)
        for i in range(nsl):
            r = b0 + first + i
            ok = r < n_new
            pid = cpid[np.minimum(r, len(cpid) - 1)]
            w = np.zeros((32, ch, 4), dtype=np.uint64)
            for j in range(ch):
                lane_ok = ok & cok[:, j]
                at = pid.astype(np.int64) * cwords + 4 * sub + 32 * j
                for k in range(4):
                    w[:, j, k] = np.where(lane_ok, flat[np.where(lane_ok, at + k, 0)], 0)
            p[:, i] = sq_dist(w.reshape(32, -1), qc.reshape(32, -1))
        d = batch_butterfly(p, 8)
        mine_row = b0 + first + sub
        votes = (sub < nsl) & (mine_row < n_new)
        mine = np.where(votes, cpid[np.minimum(mine_row, len(cpid) - 1)], INVALID)
        for lane in np.flatnonzero(votes):
            seen.setdefault(int(mine_row[lane]), set()).add(int(d[lane]))
        keep = votes & np.array([keep_row(int(m)) if v else False for m, v in zip(mine, votes)])
        # ballot + compaction (lanes in order); writes go to [kept, b0 + NS), reads of later batches come from [b0 + NS, ...)
        for lane in np.flatnonzero(keep):
            cpid[kept] = mine[lane]
            kept += 1
        out = list(cpid[:kept])
    return seen, out


@pytest.mark.parametrize("ch", sorted(SLOTS))
def test_rows_reduce_to_their_code_distance_and_survive_in_row_order(ch):
    rng = np.random.default_rng(100 + ch)
    dims = [d for d in DIMS if 32 * (ch - 1) < (d + 3) // 4 <= 32 * ch] or [d for d in DIMS if (d + 3) // 4 <= 32 * ch][-1:]
    dims += [4 * (32 * ch) - 3 - 4 * int(rng.integers(0, 4))]  # a table width just below the CH's full width
    for dim in dims:
        nchunks = (dim + 3) // 4
        assert nchunks <= 32 * ch
        cwords = code_words(nchunks)
        n = 300
        real = rng.integers(0, 1 << 32, size=(n, nchunks), dtype=np.uint64)
        if dim % 4:  # the padding elements of the last chunk code to 0 (zero rows, zero offset)
            real[:, -1] &= (1 << (8 * (dim % 4))) - 1
        table = np.zeros((n, cwords), dtype=np.uint64)
        table[:, :nchunks] = real
        assert (table[:, nchunks:] == 0).all()
        flat = np.concatenate([table.ravel(), rng.integers(0, 1 << 32, size=32 * ch, dtype=np.uint64)])  # a row's tail reads run on
        q = np.zeros(32 * ch, dtype=np.uint64)
        q[:nchunks] = rng.integers(0, 1 << 32, size=nchunks, dtype=np.uint64)
        want_d = sq_dist(real, q[None, :nchunks])
        for n_new in range(1, 129):
            ids = rng.choice(n, size=128, replace=False).astype(np.uint64)
            thr = np.median(want_d[ids[:n_new]])
            seen, out = screen(flat, cwords, ch, q, ids, n_new, lambda pid: want_d[pid] <= thr)
            assert sorted(seen) == list(range(n_new)), (dim, n_new)
            for r, ds in seen.items():
                assert ds == {int(want_d[ids[r]])}, (dim, n_new, r)
            assert out == [ids[r] for r in range(n_new) if want_d[ids[r]] <= thr], (dim, n_new)


@pytest.mark.parametrize("dim", DIMS)
def test_padding_words_add_nothing(dim):
    nchunks = (dim + 3) // 4
    ch = next(c for c in sorted(SLOTS) if nchunks <= 32 * c)
    cwords = code_words(nchunks)
    assert cwords % 4 == 0 and nchunks <= cwords < nchunks + 4
    assert cwords == nchunks or dim % 16 != 0  # at dim % 16 == 0 the table is the unpadded one
    rng = np.random.default_rng(dim)
    row = np.zeros(cwords, dtype=np.uint64)
    row[:nchunks] = rng.integers(0, 1 << 32, size=nchunks, dtype=np.uint64)
    q = np.zeros(32 * ch, dtype=np.uint64)
    q[:nchunks] = rng.integers(0, 1 << 32, size=nchunks, dtype=np.uint64)
    assert sq_dist(row[None, nchunks:], q[None, nchunks:cwords])[0] == 0  # both sides zero there
    flat = np.concatenate([row, np.full(32 * ch, 0xFFFFFFFF, dtype=np.uint64)])  # a word read past cwords would add a lot
    seen, _ = screen(flat, cwords, ch, q, np.zeros(128, dtype=np.uint64), 1, lambda pid: True)
    assert seen == {0: {int(sq_dist(row[None, :nchunks], q[None, :nchunks])[0])}}
