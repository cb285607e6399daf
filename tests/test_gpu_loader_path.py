"""The loader's device path: each data kernel against an exact reference, and the bulk-load path against the SQL path.

Kernels (bigru_chunk_minmax, bigru_window_gather_norm, bigru_window_targets).  Min, max, float32 subtraction and IEEE
division are exact in numpy float32, so every comparison is np.array_equal with NaN equal to NaN, and there is no
tolerance.  Signed zero is compared by value: fminf / fmaxf may return either zero of a (+0, -0) pair, and SQL's MIN /
MAX, which the kernel stands in for, compare them equal.  Every output buffer sits between sentinel guards that must come
back untouched, and rows a kernel must not read hold +-1e30.

End to end.  For every table shape of tests/golden/loader_edges.npz (the unmodified reference loader over
fake_db tables with NULLs at chunk edges, in runs longer than the window and in shared rows),
MySQLChunkLoader.from_table and MySQLBatchLoader.from_tensors on the table with NaN for NULL must give the SQL path's
(FakeCursor's) norm params, batches, ``x`` and per-sample windows bit for bit, and those of the reference.  The model's
window entry points on NULL rows must be finite and equal the ordinary calls on the SQL path's collated batch.

Sensitivity: each mutation below, applied alone to the library, fails this file.  The tests that caught it, measured
on an H100 80GB HBM3 (the file passes 116 tests in 26 s there):
  - the gather multiplies by the reciprocal of (max - min): test_gather_matches_exact_reference (all 14 cases),
    test_device_path_matches_sql_path (all 5 shapes), test_short_table_fetches_the_reference_rows;
  - the float4 gather uses feature group 0's bounds for every group: test_gather_matches_exact_reference (the 7 cases
    with F % 4 == 0), test_device_path_matches_sql_path at F = 8 and 16 ("divisible", "exact_fill");
  - chunk_minmax starts its minimum at 0: test_chunk_minmax_matches_nanmin_nanmax (all 64 cases),
    test_device_path_matches_sql_path, test_short_table_fetches_the_reference_rows,
    test_from_table_refuses_an_all_null_chunk_column;
  - chunk_minmax folds 7 of its 8 row lanes: test_chunk_minmax_matches_nanmin_nanmax (the 40 cases with 8 rows or more),
    test_device_path_matches_sql_path;
  - window_targets reads class C - 1 - c: test_window_targets_match_reference (the 12 cases with C > 1),
    test_collate_pairs_x_and_y, test_device_path_matches_sql_path;
  - the gather reads NaN as NaN (the IFNULL fix reverted): test_gather_matches_exact_reference,
    test_device_path_matches_sql_path and test_window_entry_points_on_null_rows (all 5 shapes each),
    test_short_table_fetches_the_reference_rows.
"""
import json
import os
import pickle
import warnings

import numpy as np
import pytest
import torch
import torch.nn as nn

import fake_db

pytestmark = pytest.mark.gpu

SENT = 0x7FC0BEEF                                   # a NaN payload no kernel computes: the guards' bit pattern
G = 64                                              # guard floats on each side (256 bytes keeps the payload aligned)
POISON = np.float32(1e30)


def _pkg():
    import financial_market_data_analysis_b200 as pkg
    return pkg


def _lib():
    return _pkg()._lib.load()


def _p(t):
    return _pkg()._lib.ptr(t)


def _stream():
    return torch.cuda.current_stream().cuda_stream


class Guarded:
    """A device output of ``shape`` starting ``off`` floats past a 256-byte boundary, inside sentinel guards."""

    def __init__(self, shape, off=0):
        n = int(np.prod(shape))
        self.buf = torch.empty(G + off + n + G, device="cuda", dtype=torch.float32)
        self.buf.view(torch.int32).fill_(SENT)
        self.lo, self.hi = G + off, G + off + n
        self.t = self.buf[self.lo:self.hi].view(*shape)

    def bits(self):
        torch.cuda.synchronize()
        return self.buf.view(torch.int32).cpu().numpy()

    def guards_intact(self):
        b = self.bits()
        return bool((b[:self.lo] == SENT).all() and (b[self.hi:] == SENT).all())

    def untouched(self):
        return bool((self.bits() == SENT).all())

    def numpy(self):
        assert self.guards_intact(), "a kernel wrote outside its output"
        return self.t.cpu().numpy()


def _dev(a, off=0):
    """float32 device copy of ``a`` starting ``off`` floats past an aligned allocation (a storage-offset view)."""
    a = np.ascontiguousarray(a, np.float32)
    base = torch.empty(off + a.size, device="cuda", dtype=torch.float32)
    base[off:] = torch.from_numpy(a.ravel()).cuda()
    return base[off:].view(*a.shape)


def _equal(a, b):
    return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def _bitwise(a, b):
    a, b = np.ascontiguousarray(a, np.float32), np.ascontiguousarray(b, np.float32)
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


def _poison(shape):
    r, f = np.indices(shape)
    return np.where((r + f) % 2 == 0, POISON, -POISON).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# bigru_chunk_minmax against np.nanmin / np.nanmax
# ---------------------------------------------------------------------------------------------------------------------
def _ref_minmax(x):
    allnan = np.isnan(x).all(0)
    with warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)            # all-NaN slices: nanmin says NaN, the kernel +-inf
        a, b = np.nanmin(x, 0), np.nanmax(x, 0)
    return np.where(allnan, np.float32(np.inf), a).astype(np.float32), np.where(allnan, np.float32(-np.inf), b).astype(np.float32)


def _minmax_patterns(rows, F, rng):
    """(name, data[rows, F]) for the row range; NaN is SQL NULL."""
    def rand():
        x = (rng.standard_normal((rows, F)) * 10.0 ** rng.integers(-3, 4, (1, F))).astype(np.float32)
        x[rng.random((rows, F)) < 0.05] = 0.0
        x[rng.random((rows, F)) < 0.05] = -0.0
        return x
    out = []
    x = rand()
    x[rng.random((rows, F)) < 0.15] = np.nan
    out.append(("sporadic_nan", x))
    x = rand()
    x[:min(rows - 1, 9)] = np.nan                                   # NaN in the leading rows (every lane's first read)
    out.append(("leading_nan", x))
    out.append(("positive", rng.uniform(1.0, 2.0, (rows, F)).astype(np.float32)))     # a minimum started at 0 shows
    out.append(("negative", rng.uniform(-2.0, -1.0, (rows, F)).astype(np.float32)))
    for lane in range(min(8, rows)):                                # one finite value per column, in each row lane in turn
        x = np.full((rows, F), np.nan, np.float32)
        x[lane] = rng.uniform(1.0, 2.0, F)
        out.append((f"one_value_lane{lane}", x))
    x = rand()
    x[rng.random((rows, F)) < 0.1] = np.inf
    x[rng.random((rows, F)) < 0.1] = -np.inf
    x[rng.random((rows, F)) < 0.1] = np.nan
    out.append(("inf", x))
    x = rng.uniform(-1, 1, (rows, F)).astype(np.float32)
    x[0], x[-1] = -5.0, 5.0
    out.append(("extrema_first_last", x))
    x = rng.uniform(-1, 1, (rows, F)).astype(np.float32)
    x[0], x[-1] = 5.0, -5.0
    out.append(("extrema_last_first", x))
    x = rand()
    x[:, ::3] = np.nan                                             # all-NaN columns: pinned at +inf / -inf
    out.append(("all_nan_columns", x))
    return out


@pytest.mark.parametrize("F", [1, 7, 31, 32, 33, 64, 65, 200])
@pytest.mark.parametrize("rows", [1, 2, 7, 8, 9, 16, 17, 1000])
def test_chunk_minmax_matches_nanmin_nanmax(F, rows):
    """Every feature block (one partial, full, ragged) and row count (fewer rows than the 8 row lanes, exactly 8, more),
    with the range at row 0, at an odd offset and ending at the table's last row, over poisoned neighbours."""
    lib = _lib()
    rng = np.random.default_rng(1000 * F + rows)
    for name, x in _minmax_patterns(rows, F, rng):
        want_mn, want_mx = _ref_minmax(x)
        for lo, after in ((0, 3), (3, 2), (5, 0)):                  # row_lo = 0 / odd / row_hi = N
            tab = np.concatenate([_poison((lo, F)), x, _poison((after, F))])
            N = tab.shape[0]
            t = _dev(tab)
            mn, mx = Guarded((F,)), Guarded((F,))
            assert lib.bigru_chunk_minmax(_p(t), N, F, lo, lo + rows, _p(mn.t), _p(mx.t), _stream()) == 0
            got_mn, got_mx = mn.numpy(), mx.numpy()
            assert _equal(got_mn, want_mn), (name, lo, np.flatnonzero(got_mn != want_mn)[:8])
            assert _equal(got_mx, want_mx), (name, lo, np.flatnonzero(got_mx != want_mx)[:8])
            if name == "all_nan_columns":
                assert (got_mn[::3] == np.inf).all() and (got_mx[::3] == -np.inf).all()


def test_chunk_minmax_refusals():
    """Bad arguments return BIGRU_ERR_ARG before any launch: both outputs keep every sentinel."""
    pkg, lib = _pkg(), _lib()
    N, F = 20, 5
    t = _dev(np.ones((N, F)))
    for lo, hi, f, tab, null_mn, null_mx in [(4, 4, F, t, 0, 0), (5, 4, F, t, 0, 0), (0, N + 1, F, t, 0, 0),
                                             (-1, 3, F, t, 0, 0), (0, 3, 0, t, 0, 0), (0, 3, -1, t, 0, 0),
                                             (0, 3, F, None, 0, 0), (0, 3, F, t, 1, 0), (0, 3, F, t, 0, 1)]:
        mn, mx = Guarded((F,)), Guarded((F,))
        rc = lib.bigru_chunk_minmax(_p(tab), N, f, lo, hi, None if null_mn else _p(mn.t), None if null_mx else _p(mx.t),
                                    _stream())
        assert rc == pkg._lib.ERR_ARG, (lo, hi, f)
        assert mn.untouched() and mx.untouched(), (lo, hi, f)


# ---------------------------------------------------------------------------------------------------------------------
# bigru_window_gather_norm against (ifnull(x) - min) / (max - min) in numpy float32
# ---------------------------------------------------------------------------------------------------------------------
def _gather_data(N, F, rng):
    """Rows [N, F] and bounds [F] by column family: wide normals, subnormals, large values where x - min rounds, and
    signed zeros; NaN (NULL) in every family."""
    x = np.empty((N, F), np.float32)
    mn = np.empty(F, np.float32)
    mx = np.empty(F, np.float32)
    for f in range(F):
        k = f % 4
        if k == 0:
            x[:, f] = rng.standard_normal(N) * 100
            mn[f], mx[f] = -317.3 - f, 291.7 + f
        elif k == 1:
            x[:, f] = rng.uniform(0, 1, N) * 1e-39                  # subnormal operands and differences
            mn[f], mx[f] = 3e-41, 1.1e-39
        elif k == 2:
            x[:, f] = 1.0e7 + rng.uniform(0, 1e3, N)                 # x - min rounds
            mn[f], mx[f] = -0.3171 - f * 1e-3, 2.3e7
        else:
            x[:, f] = rng.choice(np.array([0.0, -0.0, 1e-3, -2.5], np.float32), N)
            mn[f], mx[f] = -2.5, 1.5 + f
    x[rng.random((N, F)) < 0.07] = np.nan
    return x, mn, mx


def _gather_ref(src, mn, mx, start, B, T):
    s = np.where(np.isnan(src), np.float32(0), src).astype(np.float32)
    rows = s[start + np.arange(B)[:, None] + np.arange(T)[None, :]]
    if mn is None:
        return rows
    with np.errstate(all="ignore"):
        return (rows - mn) / (mx - mn)


def _gather(src, mn, mx, start, N, B, T, F, off_out=0):
    out = Guarded((B, T, F), off_out)
    rc = _lib().bigru_window_gather_norm(_p(src), _p(mn), _p(mx), start, N, B, T, F, _p(out.t), _stream())
    return rc, out


GATHER_CASES = [  # (F, B, T, N, start)
    (8, 5, 7, 24, 3), (12, 3, 4, 9, 0), (64, 9, 5, 20, 6), (1, 5, 7, 24, 3), (5, 6, 3, 15, 2), (13, 4, 6, 12, 0),
    (8, 4, 6, 30, 30 - 9), (13, 4, 6, 30, 30 - 9),                                         # the last legal start
    (8, 1, 11, 11, 0), (7, 1, 11, 11, 0),                                                  # B = 1, T = N
    (8, 17, 1, 40, 5), (7, 17, 1, 40, 5),                                                  # T = 1
    (8, 600, 512, 1200, 7), (5, 300, 400, 720, 9),                        # B*T*F/VEC beyond the 132*16*256 capped grid
]


@pytest.mark.parametrize("F,B,T,N,start", GATHER_CASES)
def test_gather_matches_exact_reference(F, B, T, N, start):
    """Both instantiations; for F % 4 == 0 also src, out or the bounds one float off 16 bytes (the scalar fall-back,
    same bits); no bounds (a plain gather, NULL still 0); rows outside the windows poisoned."""
    rng = np.random.default_rng(F * 7919 + B * 31 + T)
    x, mn, mx = _gather_data(N, F, rng)
    want = _gather_ref(x, mn, mx, start, B, T)
    with np.errstate(all="ignore"):
        rows = np.where(np.isnan(x), np.float32(0), x)[start + np.arange(B)[:, None] + np.arange(T)[None, :]]
        recip = (rows - mn) * (np.float32(1) / (mx - mn))
    assert not _equal(recip, want)                  # the data tells a division from a reciprocal multiply
    src = x.copy()
    used = np.zeros(N, bool)
    used[start:start + B + T - 1] = True
    src[~used] = _poison((N, F))[~used]
    layouts = {"aligned": (0, 0, 0), "src+1": (1, 0, 0), "out+1": (0, 1, 0), "bounds+1": (0, 0, 1)}
    for layout, (o_src, o_out, o_b) in layouts.items():
        rc, out = _gather(_dev(src, o_src), _dev(mn, o_b), _dev(mx, o_b), start, N, B, T, F, o_out)
        assert rc == 0
        got = out.numpy()
        bad = ~((got == want) | (np.isnan(got) & np.isnan(want)))
        assert _equal(got, want), (layout, np.argwhere(bad)[:5], got[bad][:5], want[bad][:5])
    rc, out = _gather(_dev(src), None, None, start, N, B, T, F)
    assert rc == 0 and _equal(out.numpy(), _gather_ref(x, None, None, start, B, T))


def test_gather_refusals_and_empty_batch():
    """B = 0 writes nothing; a start one past the end, a negative start, one null bound, a null src or out, T <= 0 and
    F <= 0 return BIGRU_ERR_ARG and write nothing."""
    pkg, lib = _pkg(), _lib()
    N, F, B, T = 20, 8, 3, 5
    x, mn, mx = _gather_data(N, F, np.random.default_rng(3))
    src, dmn, dmx = _dev(x), _dev(mn), _dev(mx)
    rc, out = _gather(src, dmn, dmx, 0, N, 0, T, F)
    assert rc == 0 and out.untouched()
    last = N - (B + T - 1)
    rc, out = _gather(src, dmn, dmx, last, N, B, T, F)
    assert rc == 0 and out.guards_intact()
    for args in [(src, dmn, dmx, last + 1, B, T, F), (src, dmn, dmx, -1, B, T, F), (src, dmn, None, 0, B, T, F),
                 (src, None, dmx, 0, B, T, F), (None, dmn, dmx, 0, B, T, F), (src, dmn, dmx, 0, -1, T, F),
                 (src, dmn, dmx, 0, B, 0, F), (src, dmn, dmx, 0, B, T, 0)]:
        s, a, b, start, bb, tt, ff = args
        out = Guarded((max(bb, 1), max(tt, 1), F))
        assert lib.bigru_window_gather_norm(_p(s), _p(a), _p(b), start, N, bb, tt, ff, _p(out.t), _stream()) == \
            pkg._lib.ERR_ARG, args[3:]
        assert out.untouched(), args[3:]
    out = Guarded((B, T, F))
    assert lib.bigru_window_gather_norm(_p(src), _p(dmn), _p(dmx), 0, N, B, T, F, None, _stream()) == pkg._lib.ERR_ARG


# ---------------------------------------------------------------------------------------------------------------------
# bigru_window_targets against y[start + b + T - 1]
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C", [1, 3, 4, 5])
@pytest.mark.parametrize("B,T,N,start", [(5, 7, 20, 2), (6, 1, 9, 0), (4, 6, 30, 30 - 9), (300, 4, 320, 11)])
def test_window_targets_match_reference(C, B, T, N, start):
    """The last row of each window, over rows poisoned outside the target rows; B = 300 spans several blocks."""
    pkg, lib = _pkg(), _lib()
    rng = np.random.default_rng(C * 100 + B)
    y = rng.standard_normal((N, C)).astype(np.float32)
    want = y[start + np.arange(B) + T - 1][:, None, :]
    used = np.zeros(N, bool)
    used[start + T - 1:start + T - 1 + B] = True
    y[~used] = _poison((N, C))[~used]
    d = _dev(y)
    out = Guarded((B, 1, C))
    assert lib.bigru_window_targets(_p(d), start, N, B, T, C, _p(out.t), _stream()) == 0
    assert _bitwise(out.numpy(), want)
    out = Guarded((1, 1, C))
    assert lib.bigru_window_targets(_p(d), start, N, 0, T, C, _p(out.t), _stream()) == 0 and out.untouched()
    for args in [(d, N - (B + T - 1) + 1, B, T, C), (d, -1, B, T, C), (None, start, B, T, C), (d, start, -1, T, C),
                 (d, start, B, 0, C), (d, start, B, T, 0)]:
        out = Guarded((B, 1, C))
        assert lib.bigru_window_targets(_p(args[0]), args[1], N, args[2], args[3], args[4], _p(out.t), _stream()) == \
            pkg._lib.ERR_ARG, args[1:]
        assert out.untouched(), args[1:]
    assert lib.bigru_window_targets(_p(d), start, N, B, T, C, None, _stream()) == pkg._lib.ERR_ARG


def test_collate_pairs_x_and_y():
    """collate(start, count): window b's inputs are rows start+b .. start+b+T-1, its target is row start+b+T-1's."""
    pkg = _pkg()
    N, F, C, T = 50, 6, 3, 7
    x = np.repeat(np.arange(N, dtype=np.float32)[:, None], F, 1)
    y = np.arange(N, dtype=np.float32)[:, None] * 8 + np.arange(C, dtype=np.float32)
    norm = (torch.zeros(1, F), torch.ones(1, F))                   # (x - 0) / (1 - 0) = x exactly
    ds = pkg.MySQLBatchLoader.from_tensors(torch.from_numpy(x).cuda(), torch.from_numpy(y).cuda(), norm, window=T)
    for start, count in ((0, 1), (5, 13), (N - T - 9, 10)):
        xb, yb = (a.cpu().numpy() for a in ds.collate(start, count))
        rows = start + np.arange(count)
        assert np.array_equal(xb[:, :, 0], rows[:, None] + np.arange(T))
        assert np.array_equal(yb[:, 0, :], xb[:, T - 1, :1] * 8 + np.arange(C))


# ---------------------------------------------------------------------------------------------------------------------
# The device path against the SQL path and the reference, over tests/golden/loader_edges.npz
# ---------------------------------------------------------------------------------------------------------------------
EDGE_SHAPES = ["current", "divisible", "window1", "one_window", "exact_fill"]


@pytest.fixture(scope="module")
def edges(golden_dir):
    return np.load(os.path.join(golden_dir, "loader_edges.npz"))


class Shape:
    """One table shape of loader_edges.npz: the table (NaN = NULL) on the device, and the SQL path's cursor."""

    def __init__(self, z, name, monkeypatch):
        import financial_market_data_analysis_b200.sql_pytorch_dataloader as L
        self.L, self.z, self.p = L, z, name + "__"
        self.spec = json.loads(str(z[self.p + "spec"]))
        self.window, self.chunk_size = self.spec["window"], self.spec["chunk_size"]
        levels = self.spec["table"].get("levels", 2)
        monkeypatch.setattr(L, "bid_levels", levels)
        monkeypatch.setattr(L, "ask_levels", levels)
        self.cols, targets, self.fields, self.query = fake_db.make_table(**self.spec["table"])
        assert self.fields == list(z[self.p + "fields"])
        self.cur = fake_db.FakeCursor(self.cols, targets)
        self.y_fields = ", ".join(targets)
        self.table = torch.tensor(np.stack([self.cols[f] for f in self.fields], 1), dtype=torch.float32).cuda()
        self.ytab = torch.tensor(np.stack([targets[t] for t in targets], 1), dtype=torch.float32).cuda()

    def g(self, key):
        return self.z[self.p + key]

    def loaders(self, tmp_path):
        dev = self.L.MySQLChunkLoader.from_table(self.table, self.fields, self.chunk_size, self.window,
                                                 norm_params_path=str(tmp_path / "np_dev"))
        sql = self.L.MySQLChunkLoader(self.cur, "stock_data_joined", self.query, self.chunk_size, self.window,
                                      norm_params_path=str(tmp_path / "np_sql"))
        return dev, sql

    def datasets(self, ids, norm):
        rows = torch.tensor(np.asarray(ids) - 1, device="cuda")
        dev = self.L.MySQLBatchLoader.from_tensors(self.table[rows], self.ytab[rows], norm, self.window)
        sql = self.L.MySQLBatchLoader(ids, norm, self.cur, "stock_data_joined", self.query, self.y_fields, self.window)
        return dev, sql


@pytest.mark.parametrize("name", EDGE_SHAPES)
def test_device_path_matches_sql_path(name, edges, tmp_path, monkeypatch):
    """from_table / from_tensors (NaN = NULL) against the SQL path and the reference: chunk ids, norm params, the pickled
    norm_params, batches(bs) both ways, ``x`` and the per-sample DataLoader route, bit for bit."""
    s = Shape(edges, name, monkeypatch)
    cl_dev, cl_sql = s.loaders(tmp_path)
    assert len(cl_dev) == len(cl_sql) == int(s.g("n_chunks"))
    assert [len(list(part)) for part in s.L.TrainValTestSplit(cl_dev, 0.1, 0.1).get_sets()] == list(s.g("split"))
    pd, ps = (pickle.load(open(tmp_path / f, "rb")) for f in ("np_dev", "np_sql"))
    assert list(pd) == list(ps) == s.fields
    for k, f in enumerate(s.fields):
        for key, want in (("MIN", s.g("pickle_min")[k]), ("MAX", s.g("pickle_max")[k])):
            assert _bitwise(pd[f][key].numpy(), ps[f][key].numpy()) and _bitwise(pd[f][key].numpy(), want), (f, key)
    n_nulls = 0
    for i in range(len(cl_dev)):
        ids, (mn, mx) = cl_dev[i]
        ids_s, (mn_s, mx_s) = cl_sql[i]
        c = f"chunk{i}_"
        assert ids == ids_s and np.array_equal(np.array(ids), s.g(c + "ids")), i
        for got, sql, key in ((mn, mn_s, "min"), (mx, mx_s, "max")):
            assert _bitwise(got.numpy(), sql.numpy()) and _bitwise(got.numpy(), s.g(c + key)), (i, key)
        norm = (mn, mx)
        n_nulls += int(torch.isnan(s.table[np.asarray(ids) - 1]).sum())
        for bs in s.spec["batch_sizes"]:
            for drop in (True, False):
                d, q = s.datasets(ids, norm)
                got = [(x.cpu().numpy(), y.cpu().numpy()) for x, y in d.batches(bs, drop_incomplete=drop)]
                want = [(x.cpu().numpy(), y.cpu().numpy()) for x, y in q.batches(bs, drop_incomplete=drop)]
                assert len(got) == len(want), (i, bs, drop)
                for j, ((gx, gy), (wx, wy)) in enumerate(zip(got, want)):
                    assert _bitwise(gx, wx), (f"{name} chunk {i} bs {bs} drop_incomplete={drop} batch {j}: x differs from "
                                              f"the SQL path at {np.argwhere(gx != wx)[:3].tolist()}, "
                                              f"NaN in the device batch: {int(np.isnan(gx).sum())}")
                    assert _bitwise(gy, wy), (name, i, bs, drop, j)
                if drop:
                    assert len(got) == int(s.g(c + f"bs{bs}_nbatches")), (i, bs)
                    gx = np.concatenate([x for x, _ in got]) if got else np.zeros((0, s.window, len(s.fields)), np.float32)
                    gy = np.concatenate([y for _, y in got]) if got else np.zeros((0, 1, s.ytab.shape[1]), np.float32)
                    assert _bitwise(gx, s.g(c + f"bs{bs}_x")) and _bitwise(gy, s.g(c + f"bs{bs}_y")), (i, bs)
            d, q = s.datasets(ids, norm)                         # the drop-in route: per-sample windows through DataLoader
            got = list(torch.utils.data.DataLoader(d, batch_size=bs))
            want = list(torch.utils.data.DataLoader(q, batch_size=bs))
            assert len(got) == len(want) == int(s.g(c + f"bs{bs}_nbatches")), (i, bs)
            for (gx, gy), (wx, wy) in zip(got, want):
                assert _bitwise(gx.cpu().numpy(), wx.cpu().numpy()) and _bitwise(gy.cpu().numpy(), wy.cpu().numpy()), (i, bs)
            if got:
                assert _bitwise(torch.cat([x for x, _ in got]).cpu().numpy(), s.g(c + f"bs{bs}_x")), (i, bs)
            assert _bitwise(d.x.cpu().numpy(), q.x.cpu().numpy()), (i, bs)           # the normalised chunk, ``x``
            assert _bitwise(d.x.cpu().numpy(), s.g(c + "xnorm")), (i, bs)
    assert n_nulls > 0


def _precisions():
    pkg = _pkg()
    lib, out, h = pkg._lib.load(), ["fp32"], pkg._lib.C.c_void_p()
    for name, code in (("bf16x3", pkg._lib.PREC_BF16X3), ("bf16", pkg._lib.PREC_BF16)):
        if lib.bigru_plan_create(128, 16, 64, 256, 1, 3, 1, code, pkg._lib.C.byref(h)) == 0:
            lib.bigru_plan_destroy(h)
            out.append(name)
    return out


def _rel_l2(a, b):
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-30))


@pytest.mark.parametrize("name", EDGE_SHAPES)
def test_window_entry_points_on_null_rows(name, edges, tmp_path, monkeypatch):
    """forward_windows / infer_windows / train_step_windows on windows of a bulk-loaded chunk that hold NULL rows are
    finite and equal forward / infer / train_step on the SQL path's collate of the same windows (the fp32 step up to its
    atomic summation order, as in test_zero_copy_windows_match_collated_batches)."""
    pkg = _pkg()
    s = Shape(edges, name, monkeypatch)
    cl_dev, _ = s.loaders(tmp_path)
    ids, norm = cl_dev[0]
    d, q = s.datasets(ids, norm)
    count = min(d.n_rows - s.window + 1, 16)
    assert torch.isnan(d.x_raw[:count + s.window - 1]).any()       # the windows hold NULLs
    x, y = q.collate(0, count)
    F, C = len(s.fields), s.ytab.shape[1]
    for precision in _precisions():
        H = 32 if precision == "fp32" else 128
        torch.manual_seed(0)
        m = pkg.BiGRU(H, F, C, 2, 1, 0.0, False, True, precision=precision).cuda()
        m.eval()
        with torch.no_grad():
            want = m(x)
        got = m.forward_windows(d, 0, count)
        assert torch.isfinite(got).all() and torch.equal(got, want), precision
        got = m.infer_windows(d, 0, count)
        assert torch.isfinite(got).all() and torch.equal(got, m.infer(x)), precision
        outs = []
        for mode in ("sql", "windows"):
            torch.manual_seed(0)
            mm = pkg.BiGRU(H, F, C, 2, 1, 0.0, False, True, precision=precision).cuda()
            mm.add_loss_fn(nn.BCEWithLogitsLoss()); mm.add_optimizer(torch.optim.Adam(mm.parameters(), lr=1e-2)); mm.train()
            loss, _ = mm.train_step(x, y.reshape(count, C)) if mode == "sql" else mm.train_step_windows(d, 0, count)
            assert torch.isfinite(loss).all(), (precision, mode)
            outs.append(mm.flat_parameters().detach().cpu().numpy().copy())
        assert np.isfinite(outs[1]).all(), precision
        if precision == "fp32":
            assert _rel_l2(outs[1], outs[0]) < 1e-6
        else:
            assert np.array_equal(outs[1], outs[0]), precision


def test_short_table_fetches_the_reference_rows(edges, tmp_path, monkeypatch):
    """db_length < chunk_size: the reference's chunk is IDs range(window, chunk_size), chunk_id_ranges' is
    range(window, db_length + 1).  The rows fetched, the norm params and the normalised chunk agree."""
    s = Shape(edges, "short", monkeypatch)
    cl_dev, cl_sql = s.loaders(tmp_path)
    ref_ids = s.g("chunk0_ids")
    n = len(s.cols[s.fields[0]])
    assert len(cl_dev) == len(cl_sql) == int(s.g("n_chunks")) == 1
    ids, (mn, mx) = cl_dev[0]
    assert ids == cl_sql[0][0] == tuple(range(s.window, n + 1)) == tuple(int(i) for i in ref_ids if i <= n)
    assert len(ref_ids) > len(ids)
    for norm in (cl_dev[0][1], cl_sql[0][1]):
        assert _bitwise(norm[0].numpy(), s.g("chunk0_min")) and _bitwise(norm[1].numpy(), s.g("chunk0_max"))
    d, q = s.datasets(ids, (mn, mx))
    qr = s.L.MySQLBatchLoader(tuple(int(i) for i in ref_ids), (mn, mx), s.cur, "stock_data_joined", s.query, s.y_fields,
                              s.window)                          # the reference's IDs through the SQL path
    d[0]
    for got in (d.x, q.x, qr.x):
        assert _bitwise(got.cpu().numpy(), s.g("chunk0_xnorm"))


def test_from_table_refuses_an_all_null_chunk_column(tmp_path, monkeypatch):
    """A column NULL in every row of one chunk: from_table names the column and the chunk (the SQL path cannot build that
    chunk either: MIN is NULL); NULL in every row but one is accepted."""
    import financial_market_data_analysis_b200.sql_pytorch_dataloader as L
    monkeypatch.setattr(L, "bid_levels", 2)
    monkeypatch.setattr(L, "ask_levels", 2)
    cols, _, fields, _ = fake_db.make_table(n_rows=250, null_rows={"sd.f2": range(170, 250)})       # chunk 2: IDs 171..250
    table = torch.tensor(np.stack([cols[f] for f in fields], 1), dtype=torch.float32).cuda()
    with pytest.raises(ValueError, match=r"'sd\.f2'.*chunk 2"):
        L.MySQLChunkLoader.from_table(table, fields, 100, 30, norm_params_path=None)
    table[200, fields.index("sd.f2")] = 1.5
    cl = L.MySQLChunkLoader.from_table(table, fields, 100, 30, norm_params_path=None)
    assert float(cl[2][1][0][0, fields.index("sd.f2")]) == 1.5


# ---------------------------------------------------------------------------------------------------------------------
# DevicePrefetcher
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("depth,sizes,int_targets", [
    (2, [8, 8, 8, 8, 8], False), (3, [8] * 7, True),            # depth 2 and 3
    (3, [8, 8], False), (2, [8], True),                         # fewer batches than the depth
    (2, [], False),                                             # no batches
    (2, [8, 8, 8, 5], True), (3, [8, 8, 8, 8, 3], False),       # a smaller last batch: its slot is reallocated
])
def test_device_prefetcher_yields_the_host_batches(depth, sizes, int_targets):
    """Every yielded pair, consumed before the next is asked for, is bitwise its host batch, in order."""
    from financial_market_data_analysis_b200.prefetch import DevicePrefetcher
    g = torch.Generator().manual_seed(depth * 100 + len(sizes))
    host = []
    for b in sizes:
        x = torch.randn(b, 6, 5, generator=g).pin_memory()
        t = (torch.randint(0, 4, (b,), generator=g) if int_targets else torch.rand(b, 3, generator=g)).pin_memory()
        host.append((x, t))
    got = []
    for x, t in DevicePrefetcher(iter(host), torch.device("cuda"), depth=depth):
        assert x.is_cuda and t.is_cuda
        got.append((x.cpu(), t.cpu()))
    assert len(got) == len(host)
    for (gx, gt), (hx, ht) in zip(got, host):
        assert gx.dtype == torch.float32 and gt.dtype == ht.dtype
        assert torch.equal(gx, hx) and torch.equal(gt, ht)
