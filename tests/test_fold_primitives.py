"""-m gpu: each primitive of cook_b200/csrc/fold.cuh, driven through tests/fold_probe.cu, against the
plain references of fold_ref.py.  With `exact` off a fold must give the Python left fold's bits
whatever the addends; with `exact` on and grid-valued addends it must give the exact sum."""
import ctypes as C
import os
import struct

import numpy as np
import pytest

import fold_ref as R

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
PROBE = os.path.join(HERE, "libfoldprobe.so")


@pytest.fixture(scope="module")
def probe():
    if not os.path.exists(PROBE):
        raise FileNotFoundError(f"{PROBE} not built: run __graft_entry__.build() (nvcc, sm_90a)")
    lib = C.CDLL(PROBE)
    for name in ("fp_warp_fold_prefix", "fp_warp_fold_sum", "fp_order_scan_f64", "fp_order_scan_i32",
                 "fp_grid_check", "fp_grid_value_ok", "fp_seg_bounds", "fp_compact", "fp_order_scan_tile",
                 "fp_compact_block"):
        getattr(lib, name).restype = C.c_int
    assert lib.fp_order_scan_tile() == R.OS_TILE and lib.fp_compact_block() == R.CP_BLOCK
    return lib


def _ok(rc):
    assert rc == 0, f"CUDA error {rc}"


def _offsets(lengths):
    return np.concatenate([[0], np.cumsum(lengths)]).astype(np.int32)


# chunk edges of one warp: 1, 31/32/33, 127/128/129 (four chunks), plus empty and long segments
SEG_LENGTHS = [1, 31, 32, 33, 0, 127, 128, 129, 2, 64, 300, 1]


def _values(rng, kind, n):
    if kind == "grid":
        return GRIDV[rng.integers(0, len(GRIDV), n)]
    if kind == "off":
        return rng.integers(1, 100000, n) / 7.0 + 0.1
    # magnitudes that round at every step: the order of the additions shows in the bits
    return rng.choice(np.array([1e16, 1.0, -1e16, 3.3, 2.0 ** 53, 0.1, 7.0, 1e-3]), n) * rng.random(n)


GRIDV = np.array([0.5, 1.0, 2.0, 4.0, 512.0, 3 * 2.0 ** -10, 1024.0 + 2.0 ** -10, 0.0])


@pytest.mark.parametrize("K", [1, 2, 3, 4])
@pytest.mark.parametrize("kind,exact", [("grid", 1), ("grid", 0), ("off", 0), ("wild", 0)])
def test_warp_fold_prefix(probe, K, kind, exact):
    rng = np.random.default_rng(100 * K + len(kind) + exact)
    lens = SEG_LENGTHS
    off = _offsets(lens)
    n, nseg = int(off[-1]), len(lens)
    x = np.ascontiguousarray(np.stack([_values(rng, kind, n) for _ in range(K)]))
    start = (GRIDV[rng.integers(0, 5, (nseg, K))] if kind == "grid" else rng.random((nseg, K)) * 3.0).copy()
    out = np.full((K, n), -7.0)
    carry = np.zeros((nseg, K))
    for pad in (0.0, float("nan")):   # lanes past a chunk's count must not leak in
        _ok(probe.fp_warp_fold_prefix(K, x.ctypes.data_as(C.c_void_p), n, off.ctypes.data_as(C.c_void_p), nseg,
                                      start.ctypes.data_as(C.c_void_p), exact, C.c_double(pad),
                                      out.ctypes.data_as(C.c_void_p), carry.ctypes.data_as(C.c_void_p)))
        for g in range(nseg):
            s, e = off[g], off[g + 1]
            for k in range(K):
                want = R.left_fold(x[k, s:e], start[g, k])
                assert R.same_bits(out[k, s:e], want), (pad, g, k)
                assert R.same_bits([carry[g, k]], [want[-1] if e > s else start[g, k]]), (pad, g, k)
                if exact and e > s:
                    assert carry[g, k] == R.exact_sum(x[k, s:e], start[g, k])


MASKS = {
    "none": lambda i: False,
    "all": lambda i: True,
    "third": lambda i: i % 3 == 0,
    "lane31": lambda i: i % 32 == 31,
    "lane0": lambda i: i % 32 == 0,
}


@pytest.mark.parametrize("K,D", [(1, 1), (3, 4), (4, 1), (4, 4), (2, 4)])
@pytest.mark.parametrize("mask", list(MASKS))
@pytest.mark.parametrize("kind,exact", [("grid", 1), ("off", 0), ("wild", 0)])
def test_warp_fold_sum(probe, K, D, mask, kind, exact):
    rng = np.random.default_rng(K * 7 + D + len(mask) * 13 + exact)
    lens = SEG_LENGTHS + [4 * 32 * 3 + 5]
    off = _offsets(lens)
    n, nseg = int(off[-1]), len(lens)
    x = np.ascontiguousarray(np.stack([_values(rng, kind, n) for _ in range(K)]))
    on = np.zeros(n, np.uint8)
    for g in range(nseg):
        for i in range(lens[g]):
            on[off[g] + i] = MASKS[mask](i)
    start = (GRIDV[rng.integers(0, 5, (nseg, K))] if kind == "grid" else rng.random((nseg, K)) * 3.0).copy()
    carry = np.zeros((nseg, K, 32))
    _ok(probe.fp_warp_fold_sum(K, D, x.ctypes.data_as(C.c_void_p), on.ctypes.data_as(C.c_void_p), n,
                               off.ctypes.data_as(C.c_void_p), nseg, start.ctypes.data_as(C.c_void_p), exact,
                               carry.ctypes.data_as(C.c_void_p)))
    for g in range(nseg):
        s, e = off[g], off[g + 1]
        for k in range(K):
            items = [x[k, i] for i in range(s, e) if on[i]]
            want = R.left_total(items, start[g, k])
            assert R.same_bits(carry[g, k], np.full(32, want)), (g, k)   # every lane holds the total
            if exact:
                assert carry[g, k, 0] == R.exact_sum(items, start[g, k])


def _order_scan_f64(probe, x, flag, qp, qs, read=1):
    n = x.shape[1]
    nb = (n + R.OS_TILE - 1) // R.OS_TILE
    part = np.full((3, n), -5.0)
    tile = np.full((3, nb), -5.0)
    at = np.zeros((3, n))
    seg = np.zeros((3, max(len(qp), 1)))
    _ok(probe.fp_order_scan_f64(x.ctypes.data_as(C.c_void_p), n, flag[0], C.c_ulonglong(flag[1]),
                                qp.ctypes.data_as(C.c_void_p), qs.ctypes.data_as(C.c_void_p), len(qp), read,
                                part.ctypes.data_as(C.c_void_p), tile.ctypes.data_as(C.c_void_p),
                                at.ctypes.data_as(C.c_void_p), seg.ctypes.data_as(C.c_void_p)))
    return part, tile, at, seg


def _queries(rng, n):
    """(p, s) pairs: segments from position 0, at and around tile edges, single positions, the last one."""
    T = R.OS_TILE
    qs = [0, 0, n - 1, 1]
    qp = [0, n - 1, n - 1, min(n - 1, 2)]
    for edge in range(T, n, T):
        for s in (edge - 1, edge, edge + 1):
            if 0 <= s < n:
                qs.append(s)
                qp.append(min(n - 1, s + int(rng.integers(0, 3 * T))))
    for _ in range(40):
        s = int(rng.integers(0, n))
        qs.append(s)
        qp.append(int(rng.integers(s, n)))
    return np.array(qp, np.int32), np.array(qs, np.int32)


@pytest.mark.parametrize("n", [1, R.OS_TILE - 1, R.OS_TILE, R.OS_TILE + 1, 33 * R.OS_TILE + 17, 70 * R.OS_TILE])
def test_order_scan_f64_on_the_grid(probe, n):
    """Grid-valued columns with the flag open: every position's scan and every segment_sum is exact;
    more than 32 tiles makes order_scan_totals loop."""
    rng = np.random.default_rng(n)
    x = np.ascontiguousarray(np.stack([GRIDV[rng.integers(0, len(GRIDV), n)] for _ in range(3)]))
    flag = R.grid_flag(x[0], x[1], x[2])
    assert R.grid_exact(flag, n)
    qp, qs = _queries(rng, n)
    _, _, at, seg = _order_scan_f64(probe, x, flag, qp, qs)
    for k in range(3):
        c = np.cumsum(x[k])    # exact: every partial sum is on the grid and below 2^43
        assert R.same_bits(at[k], c)
        want = [c[p] - (c[s - 1] if s > 0 else 0.0) for p, s in zip(qp, qs)]
        assert R.same_bits(seg[k, :len(qp)], want)
        for i, (p, s) in enumerate(zip(qp[:20], qs[:20])):
            assert seg[k, i] == R.exact_sum(x[k, s:p + 1])


@pytest.mark.parametrize("flag", [(1, 0), (0, struct.unpack("<Q", struct.pack("<d", 2.0 ** 40))[0])])
def test_order_scan_writes_nothing_when_the_gate_is_closed(probe, flag):
    """A flag that is not exact (an off-grid addend; or n * max past 2^43): both launches return early,
    the sentinels in part and tile survive."""
    n = 3 * R.OS_TILE + 5
    x = np.ascontiguousarray(np.ones((3, n)))
    assert not R.grid_exact(flag, n)
    qp, qs = np.zeros(1, np.int32), np.zeros(1, np.int32)
    part, tile, _, _ = _order_scan_f64(probe, x, flag, qp, qs, read=0)
    assert (part == -5.0).all() and (tile == -5.0).all()
    xi = np.ones(n, np.int32)
    parti = np.full(n, -5, np.int32)
    tilei = np.full(4, -5, np.int32)
    _ok(probe.fp_order_scan_i32(xi.ctypes.data_as(C.c_void_p), n, flag[0], C.c_ulonglong(flag[1]),
                                qp.ctypes.data_as(C.c_void_p), qs.ctypes.data_as(C.c_void_p), 1, 0,
                                parti.ctypes.data_as(C.c_void_p), tilei.ctypes.data_as(C.c_void_p),
                                np.zeros(n, np.int32).ctypes.data_as(C.c_void_p),
                                np.zeros(1, np.int32).ctypes.data_as(C.c_void_p)))
    assert (parti == -5).all() and (tilei == -5).all()


@pytest.mark.parametrize("n", [1, R.OS_TILE, R.OS_TILE + 1, 40 * R.OS_TILE + 3])
def test_order_scan_i32(probe, n):
    rng = np.random.default_rng(n + 1)
    x = rng.integers(0, 3, n).astype(np.int32)
    nb = (n + R.OS_TILE - 1) // R.OS_TILE
    qp, qs = _queries(rng, n)
    part, tile = np.full(n, -5, np.int32), np.full(nb, -5, np.int32)
    at, seg = np.zeros(n, np.int32), np.zeros(len(qp), np.int32)
    _ok(probe.fp_order_scan_i32(x.ctypes.data_as(C.c_void_p), n, 0, C.c_ulonglong(R.bits(2.0)),
                                qp.ctypes.data_as(C.c_void_p), qs.ctypes.data_as(C.c_void_p), len(qp), 1,
                                part.ctypes.data_as(C.c_void_p), tile.ctypes.data_as(C.c_void_p),
                                at.ctypes.data_as(C.c_void_p), seg.ctypes.data_as(C.c_void_p)))
    c = np.cumsum(x.astype(np.int64))
    assert np.array_equal(at, c)
    assert np.array_equal(seg, [c[p] - (c[s - 1] if s > 0 else 0) for p, s in zip(qp, qs)])


def _flag_and_queries(probe, cols, queries):
    n = max(len(c) for c in cols if c is not None)
    ptr = [None if c is None else np.ascontiguousarray(c, np.float64) for c in cols]
    qn = np.array([q[0] for q in queries], np.int64)
    qst = np.array([q[1] for q in queries], np.float64)
    ok = np.zeros(len(queries), np.uint8)
    bad, mb = C.c_int(0), C.c_ulonglong(0)
    _ok(probe.fp_grid_check(*[None if p is None else p.ctypes.data_as(C.c_void_p) for p in ptr], n,
                            qn.ctypes.data_as(C.c_void_p), qst.ctypes.data_as(C.c_void_p), len(queries),
                            C.byref(bad), C.byref(mb), ok.ctypes.data_as(C.c_void_p)))
    return (bad.value, mb.value), ok


BOUNDARY_VALUES = [0.0, -0.0, 2.0 ** -10, 2.0 ** -11, 3 * 2.0 ** -11, 2.0 ** 40, np.nextafter(2.0 ** 40, np.inf),
                   float("nan"), float("inf"), -(2.0 ** -10), 0.1, 0.5, 1023.0 + 2.0 ** -10, 2.0 ** 40 - 2.0 ** -10]


def test_grid_value_ok_boundary_table(probe):
    x = np.array(BOUNDARY_VALUES)
    ok = np.zeros(len(x), np.uint8)
    _ok(probe.fp_grid_value_ok(x.ctypes.data_as(C.c_void_p), len(x), ok.ctypes.data_as(C.c_void_p)))
    want = [R.grid_value_ok(v) for v in x]
    assert list(ok.astype(bool)) == want
    assert want[:7] == [True, True, True, False, False, True, False] and not any(want[7:11])


def _n_queries(m):
    """(n, start) at and one step below the 2^43 bound for the largest addend m, and start values."""
    mm = max(m, 1.0)
    q = []
    n0 = int(R.LIMIT // mm) - 1                       # (n0 + 1) * mm <= 2^43
    for n in (n0 - 2, n0 - 1, n0, n0 + 1, 0, 1):
        if n >= 0:
            q.append((n, 0.0))
    for st in (0.0, 2.0 ** -10, 2.0 ** -11, 0.1, -(2.0 ** -10), float("nan"), float("inf"), 2.0 ** 40,
               np.nextafter(2.0 ** 40, np.inf)):
        q.append((0, st))
        q.append((max(n0 - 3, 0), st))
    # (n + 1) * mm + start == 2^43 exactly, and one grid step below
    n1 = max(n0 - 5, 0)
    rest = R.LIMIT - (n1 + 1) * mm
    if 0 <= rest <= 2.0 ** 40:
        q += [(n1, rest), (n1, rest - 2.0 ** -10)]
    return q


@pytest.mark.parametrize("col", [
    [0.5, 1.0, 3.0],                             # m = 3
    [2.0 ** 40, 1.0],                            # the largest addend allowed
    [0.25, 0.5],                                 # m < 1: the bound uses max(m, 1)
    [0.0, -0.0],                                 # no positive addend: max_bits stays 0
    [2.0 ** -10, 7.0 * 2.0 ** 20],
    [1.0, 2.0 ** -11],                           # off the grid
    [1.0, 3 * 2.0 ** -11],
    [1.0, float("nan")],
    [1.0, float("inf")],
    [1.0, -(2.0 ** -10)],
    [1.0, 0.1],
    [1.0, float(np.nextafter(2.0 ** 40, np.inf))],
])
def test_grid_exact_boundary_table(probe, col):
    """grid_check_kernel + grid_exact on the device agree with the Python rule, value by value and query
    by query, at the boundary of the rule."""
    col = np.array(col, np.float64)
    want_flag = R.grid_flag(col, None, col[::-1].copy())
    m = struct.unpack("<d", struct.pack("<Q", want_flag[1]))[0]
    queries = _n_queries(m)
    flag, ok = _flag_and_queries(probe, [col, None, col[::-1].copy()], queries)
    assert (bool(flag[0]), flag[1]) == (bool(want_flag[0]), want_flag[1])
    want = [R.grid_exact(want_flag, n, st) for n, st in queries]
    assert list(ok.astype(bool)) == want, [(q, w) for q, w, o in zip(queries, want, ok) if bool(o) != w]
    if not want_flag[0]:
        assert any(want) and not all(want)   # the table reaches both sides of the bound


def test_grid_check_over_many_blocks(probe):
    """The flag is a reduction over every block: one bad value or one large one anywhere decides it."""
    n = 70_001
    a = np.full(n, 0.5)
    b = np.zeros(n)
    c = np.full(n, 2.0)
    b[n - 1] = 12345.0
    flag, _ = _flag_and_queries(probe, [a, b, c], [(1, 0.0)])
    assert flag == (0, R.bits(12345.0))
    c[40_000] = 0.3
    flag, _ = _flag_and_queries(probe, [a, b, c], [(1, 0.0)])
    assert flag[0] == 1


def _seg_bounds(probe, ord_, key, nseg, map_=None):
    n = len(ord_)
    ss, se, at = np.full(nseg, -9, np.int32), np.full(nseg, -9, np.int32), np.zeros(n, np.int32)
    ord_ = np.ascontiguousarray(ord_, np.int32)
    key = np.ascontiguousarray(key, np.int32)
    mp = None if map_ is None else np.ascontiguousarray(map_, np.int32)
    _ok(probe.fp_seg_bounds(ord_.ctypes.data_as(C.c_void_p), None if mp is None else mp.ctypes.data_as(C.c_void_p),
                            0 if mp is None else len(mp), key.ctypes.data_as(C.c_void_p), len(key), n, nseg,
                            ss.ctypes.data_as(C.c_void_p), se.ctypes.data_as(C.c_void_p), at.ctypes.data_as(C.c_void_p)))
    return ss, se, at


@pytest.mark.parametrize("lens", [[1], [1, 0, 3, 0, 0, 1], [0, 1, 5, 1], [300, 0, 1, 1, 257], [0, 0, 2]])
def test_seg_bounds(probe, lens):
    """Segment bounds of a sorted order: empty keys keep the sentinel, one-element segments at position 0
    and at n-1, n = 1; through a permutation and a map, as rank and the rebalancer call it."""
    rng = np.random.default_rng(len(lens))
    nseg = len(lens)
    keys_sorted = np.repeat(np.arange(nseg), lens).astype(np.int32)
    n = len(keys_sorted)
    ord_ = rng.permutation(n).astype(np.int32)
    key = np.empty(n, np.int32)
    key[ord_] = keys_sorted                       # key[ord[p]] is sorted
    off = _offsets(lens)
    want_s = np.where(np.array(lens) > 0, off[:-1], -9)
    want_e = np.where(np.array(lens) > 0, off[1:], -9)
    ss, se, at = _seg_bounds(probe, ord_, key, nseg)
    assert np.array_equal(ss, want_s) and np.array_equal(se, want_e) and np.array_equal(at, keys_sorted)
    mp = rng.permutation(n).astype(np.int32)
    key2 = np.empty(n, np.int32)
    key2[mp] = key                                # key2[map[i]] == key[i]
    ss, se, at = _seg_bounds(probe, ord_, key2, nseg, mp)
    assert np.array_equal(ss, want_s) and np.array_equal(se, want_e) and np.array_equal(at, keys_sorted)


def _compact(probe, keep, cap, n_dev=-1, extra=40):
    keep = np.ascontiguousarray(keep, np.uint8)
    out = np.full(cap + extra, -3, np.int32)
    out_n = np.zeros(1, np.int32)
    _ok(probe.fp_compact(keep.ctypes.data_as(C.c_void_p), len(keep), n_dev, cap, out.ctypes.data_as(C.c_void_p),
                         len(out), out_n.ctypes.data_as(C.c_void_p)))
    return out, int(out_n[0])


B = R.CP_BLOCK


@pytest.mark.parametrize("n", [1, 5, B - 1, B, B + 1, 33 * B + 7, 40 * B])
@pytest.mark.parametrize("pattern", ["all", "none", "third", "random", "tail"])
def test_compact(probe, n, pattern):
    """Stable compaction: slots 0.. get the kept items in order, up to the cap; out_n = min(count, cap);
    nothing is written past the cap.  More than 32 blocks makes compact_scan_kernel loop."""
    rng = np.random.default_rng(n * 7 + len(pattern))
    keep = {"all": np.ones(n), "none": np.zeros(n), "third": np.arange(n) % 3 == 1,
            "random": rng.random(n) < 0.4, "tail": np.arange(n) >= n - 2}[pattern].astype(np.uint8)
    idx = np.flatnonzero(keep)
    for cap in sorted({len(idx), max(len(idx) - 1, 0), len(idx) // 2, 1, 0, n}):
        out, out_n = _compact(probe, keep, cap)
        assert out_n == min(len(idx), cap)
        assert np.array_equal(out[:out_n], idx[:cap])
        assert (out[out_n:] == -3).all()


@pytest.mark.parametrize("n_max,n_dev", [(3 * B + 5, 2 * B + 1), (3 * B + 5, 0), (3 * B + 5, B), (50 * B, 33 * B + 1),
                                         (10, 99)])
def test_compact_with_a_device_count(probe, n_max, n_dev):
    """n read from the device (at most n_max): items at or past it never count, whatever keep says."""
    rng = np.random.default_rng(n_max + n_dev)
    keep = (rng.random(n_max) < 0.6).astype(np.uint8)
    n = min(n_dev, n_max)
    idx = np.flatnonzero(keep[:n])
    for cap in (len(idx), len(idx) // 3, n_max):
        out, out_n = _compact(probe, keep, cap, n_dev)
        assert out_n == min(len(idx), cap)
        assert np.array_equal(out[:out_n], idx[:cap])
        assert (out[out_n:] == -3).all()
