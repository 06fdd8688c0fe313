"""The width ladder of K1's distance batches (hnsw_device.cuh batch_width / batch_floor), compiled for the host from the header the
kernels use: for every n_new <= 128 at every (CH, NB) the kernels instantiate, the batches cover rows [0, n_new) exactly once and in
order, every batch but the last is NB wide, and the last is the narrowest rung of NB, NB/2, ..., batch_floor<CH> that holds its rows."""
import os
import shutil
import subprocess

import pytest

from tests.conftest import ROOT

CSRC = os.path.join(ROOT, "instant-distance_b200", "csrc")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
CHS = (1, 2, 3, 4, 6, 8)
NBS = (2, 4, 8, 16, 32)  # K1 (f32 and packed rows, the tuning variants), the build, remove
MAX_N = 128              # cpid holds at most 128 ids (2M <= 128)

PROGRAM = r"""
#include <cstdio>
#include "hnsw_device.cuh"
template <int CH, int NB>
static void widths() {
    constexpr int F = idb::batch_floor<CH>();
    for (unsigned n = 1; n <= %d; ++n) {
        std::printf("%%d %%d %%d %%u", CH, NB, F, n);
        for (unsigned b0 = 0, w; b0 < n; b0 += w) std::printf(" %%u", w = (unsigned)idb::batch_width<NB, F>(n - b0));
        std::printf("\n");
    }
}
template <int CH>
static void all_nb() { widths<CH, 2>(); widths<CH, 4>(); widths<CH, 8>(); widths<CH, 16>(); widths<CH, 32>(); }
int main() { all_nb<1>(); all_nb<2>(); all_nb<3>(); all_nb<4>(); all_nb<6>(); all_nb<8>(); }
""" % MAX_N


@pytest.fixture(scope="module")
def ladder(tmp_path_factory):
    if not os.path.exists(NVCC) and not shutil.which("nvcc"):
        pytest.fail(f"nvcc not found at {NVCC}")
    d = tmp_path_factory.mktemp("ladder")
    src, exe = d / "ladder.cu", d / "ladder"
    src.write_text(PROGRAM)
    nvcc = NVCC if os.path.exists(NVCC) else shutil.which("nvcc")
    subprocess.check_call([nvcc, "-std=c++17", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a",
                           "-I", CSRC, "-o", str(exe), str(src)])
    rows = {}
    for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        ch, nb, floor, n, *w = map(int, line.split())
        rows[(ch, nb, n)] = (floor, w)
    return rows


def test_floor_keeps_four_chunk_loads_and_two_rows(ladder):
    floors = {ch: ladder[(ch, 16, 1)][0] for ch in CHS}
    assert floors == {1: 4, 2: 2, 3: 2, 4: 2, 6: 2, 8: 2}


@pytest.mark.parametrize("nb", NBS)
@pytest.mark.parametrize("ch", CHS)
def test_batches_cover_every_row_once_in_order(ladder, ch, nb):
    rungs = [nb >> k for k in range(6) if nb >> k >= 1]
    for n in range(1, MAX_N + 1):
        floor, widths = ladder[(ch, nb, n)]
        rungs_here = [w for w in rungs if w == nb or w >= floor]
        covered, b0 = [], 0
        for i, w in enumerate(widths):
            assert w in rungs_here, (ch, nb, n, widths)
            rest = n - b0
            if i < len(widths) - 1:
                assert w == nb and rest > nb, (ch, nb, n, widths)  # a full batch
            else:
                assert rest <= w, (ch, nb, n, widths)  # the last batch holds every row left ...
                assert w == min(r for r in rungs_here if r >= rest), (ch, nb, n, widths)  # ... in the narrowest rung that does
            covered += range(b0, b0 + min(w, rest))
            b0 += w
        assert covered == list(range(n)), (ch, nb, n, widths)
