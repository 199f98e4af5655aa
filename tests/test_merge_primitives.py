"""-m gpu: the comparator sort of cook_b200/csrc/sort.cuh and the merge comparator LessMerge of fold.cuh,
driven through tests/fold_probe.cu.  The sort against numpy's stable argsort at every tile and merge-pass
edge; LessMerge against the emission order of dru/sorted-merge (merge_ref.py) on tables with runs of equal
scores, as the whole pair relation and as the order the sort makes of it."""
import ctypes as C
import os

import numpy as np
import pytest

import merge_ref as M

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
PROBE = os.path.join(HERE, "libfoldprobe.so")
TILE = 2048


@pytest.fixture(scope="module")
def probe():
    if not os.path.exists(PROBE):
        raise FileNotFoundError(f"{PROBE} not built: run __graft_entry__.build() (nvcc, sm_90a)")
    lib = C.CDLL(PROBE)
    for name in ("fp_sort_tile", "fp_sort_indices", "fp_less_merge"):
        getattr(lib, name).restype = C.c_int
    assert lib.fp_sort_tile() == TILE
    return lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _ok(rc):
    assert rc == 0, f"CUDA error {rc}"


def _keys(kind, n, seed):
    rng = np.random.default_rng(seed)
    if kind == "equal":
        return np.full(n, 3.0)
    if kind == "few":
        return rng.integers(0, 4, n).astype(np.float64)
    if kind == "descending":
        return np.arange(n, 0, -1, dtype=np.float64)
    return rng.random(n)


def _sort(probe, key, by_index):
    n = len(key)
    out = np.full(max(n, 1), -5, np.int32)
    launches = C.c_int(-1)
    _ok(probe.fp_sort_indices(_p(key), n, by_index, _p(out), C.byref(launches)))
    return out[:n], launches.value


# tile edges (2047 / 2048 / 2049, 4095 / 4096 / 4097), an odd number of runs so that the last one has no
# partner in a merge pass (3 and 5 tiles), and ten merge passes
SORT_N = [0, 1, 2047, 2048, 2049, 4095, 4096, 4097, 3 * TILE + 1, 5 * TILE + 3, 2 ** 20 + 1]


@pytest.mark.parametrize("n", SORT_N)
@pytest.mark.parametrize("kind", ["equal", "few", "descending", "random"])
def test_sort_indices_by_key_and_index(probe, n, kind):
    key = _keys(kind, n, n)
    out, launches = _sort(probe, key, 1)
    assert np.array_equal(out, np.argsort(key, kind="stable"))
    tiles = -(-n // TILE)
    assert launches == (0 if n == 0 else 1 + (tiles - 1).bit_length())   # 1 + ceil(log2(tiles))


@pytest.mark.parametrize("n", [2049, 4097, 3 * TILE + 1, 5 * TILE + 3, 70001])
@pytest.mark.parametrize("kind", ["equal", "few"])
def test_sort_indices_merges_ties_stably(probe, n, kind):
    """By key alone: the tile sort may reorder equal keys inside its tile, but every merge pass takes the
    left run on a tie, so equal keys stay in tile order."""
    key = _keys(kind, n, n + 1)
    out, _ = _sort(probe, key, 0)
    assert np.array_equal(np.sort(out), np.arange(n))
    k = key[out]
    assert np.all(np.diff(k) >= 0)
    tie = k[1:] == k[:-1]
    assert np.all(np.diff(out // TILE)[tie] >= 0)


TABLES = M.tie_tables()


def _less_merge(probe, t, matrix=True):
    n, U = len(t["dru"]), len(t["seg_start"])
    less = np.zeros((n, n), np.uint8) if matrix else None
    order = np.full(n, -1, np.int32)
    _ok(probe.fp_less_merge(_p(t["dru"]), _p(t["user_at"]), _p(t["seg_start"]), _p(t["name_rank"]), n, U,
                            _p(less) if matrix else None, _p(order)))
    return less, order


@pytest.mark.parametrize("name", list(TABLES))
def test_less_merge_is_the_merge_order(probe, name):
    """less(i, j) <=> i comes before j in the merge (cut tasks last, in position order).  One comparison of
    the whole relation covers irreflexivity, asymmetry and transitivity."""
    t = TABLES[name]
    n = len(t["dru"])
    assert n <= 256
    want = M.expected_positions(t)
    pos = np.empty(n, np.int64)
    pos[want] = np.arange(n)
    less, order = _less_merge(probe, t)
    bad = np.argwhere(less.astype(bool) != (pos[:, None] < pos[None, :]))
    assert len(bad) == 0, f"{len(bad)} pairs differ, first less{tuple(bad[0])} = {less[tuple(bad[0])]}"
    assert np.array_equal(order, want)


def test_hand_case_order(probe):
    """Users A < B, two tasks each, all scores equal: a1 a2 b1 b2."""
    _, order = _less_merge(probe, M.hand_case())
    assert order.tolist() == [0, 1, 2, 3]


@pytest.mark.parametrize("seed,nu,ml,fz", [(1, 300, 40, 0.5), (2, 40, 400, 0.3), (3, 8, 1500, 0.9),
                                           (4, 500, 12, 1.0), (5, 200, 60, 0.0)])
def test_less_merge_sorts_large_tables(probe, seed, nu, ml, fz):
    """Past one sort tile: the merge passes order the runs as the merge does."""
    t = M.random_gpu_table(seed, nu, ml, fz)
    assert len(t["dru"]) > TILE
    assert t["merge"] == M.heap_merge(t["lists"], lambda p: t["dru"][p])
    _, order = _less_merge(probe, t, matrix=False)
    assert np.array_equal(order, M.expected_positions(t))
