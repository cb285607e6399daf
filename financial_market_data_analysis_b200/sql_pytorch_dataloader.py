"""H100-native drop-in for the reference's ``sql_pytorch_dataloader`` module.

Same public names and constructor signatures as /root/reference/sql_pytorch_dataloader.py
(``window_indices`` :8, ``MySQLChunkLoader`` :21, ``MySQLBatchLoader`` :162, ``TrainValTestSplit`` :251).
What changes is where the collation happens: a chunk's rows are uploaded to HBM once and every
batch ``x[B, W, F]`` / ``y[B, 1, C]`` is produced by the window-gather/normalise kernel of
libbigru_b200 (``bigru_window_gather_norm``), instead of B Python ``__getitem__`` calls plus
``default_collate``.  The SQL round trips (COUNT / MIN / MAX / SELECT ... WHERE ID IN) are the
reference's interface to MariaDB and are issued unchanged through the DB-API cursor.
"""
from __future__ import annotations

import pickle
from itertools import islice

import torch
from torch.utils.data import Dataset

if __package__:
    from . import _lib
else:                                   # drop-in route: this directory is on sys.path (see biGRU_model.py)
    import importlib as _importlib
    import os as _os
    import sys as _sys
    _here = _os.path.dirname(_os.path.abspath(__file__))
    if _os.path.dirname(_here) not in _sys.path:
        _sys.path.insert(0, _os.path.dirname(_here))
    _lib = _importlib.import_module(_os.path.basename(_here) + "._lib")

try:                                    # the reference reads these from its config.py (:5)
    from config import ask_levels, bid_levels
except Exception:                       # config.py needs pytz + credentials; default to its shipped values (config.py:36-37)
    bid_levels, ask_levels = 7, 7


def window_indices(seq, n=2):
    """Sliding window of width n (stride 1) over an iterable, as tuples."""
    it = iter(seq)
    win = tuple(islice(it, n))
    if len(win) == n:
        yield win
    for item in it:
        win = win[1:] + (item,)
        yield win


def _split_query(db_x_query: str):
    """-> (list of selected column expressions, "FROM ..." clause without the trailing ';')."""
    toks = [w.strip(",") for w in db_x_query.split()]
    s, f = toks.index("SELECT"), toks.index("FROM")
    return toks[s + 1:f], " ".join(toks[f:]).strip(";")


def chunk_id_ranges(db_length: int, chunk_size: int, window: int):
    """ID ranges of the chunks; neighbours overlap by window-1 rows so every window appears once."""
    n_full = db_length // chunk_size
    ranges = []
    for c in range(n_full + 1):
        lo = window if c == 0 else chunk_size * c - window + 1
        hi = chunk_size * (c + 1) if c < n_full else db_length + 1
        ranges.append(range(lo, hi))
    return ranges


def widen_degenerate(x_min: torch.Tensor, x_max: torch.Tensor):
    """Columns whose MIN equals MAX cannot be min-max scaled: push MAX up by 0.1 % (or 1e-3 at 0)."""
    same = x_min == x_max
    nonzero = same & (x_max != 0)
    x_max = torch.where(nonzero, x_max + x_max * 0.001, x_max)
    x_max = torch.where(same & ~nonzero, x_max + 0.001, x_max)
    return x_min, x_max


def share_book_levels(x_fields, x_min, x_max):
    """Order-book size columns of one side share a single MIN/MAX over all levels."""
    if "sd.bid_0_size" not in x_fields:
        return
    for side, levels in (("ask", ask_levels), ("bid", bid_levels)):
        cols = [x_fields.index(f"sd.{side}_{i}_size") for i in range(levels) if f"sd.{side}_{i}_size" in x_fields]
        if cols:
            x_min[0][cols] = x_min[0][cols].min()
            x_max[0][cols] = x_max[0][cols].max()


class MySQLChunkLoader(Dataset):
    """Chunk ID ranges + per-chunk normalisation parameters (MIN, MAX) of a MySQL/MariaDB table.

    ``loader[i]`` -> (tuple of row IDs of chunk i, (x_min[1,F], x_max[1,F])); slicing is supported
    (TrainValTestSplit uses it).  The last chunk's parameters are pickled to ``norm_params`` (a
    dict name -> {"MIN", "MAX"}), the file the live predictor loads.
    """

    def __init__(self, cursor, table, db_x_query, chunk_size, window, norm_params_path="norm_params"):
        cursor.execute("SELECT COUNT(ID) FROM {};".format(table))
        db_length = cursor.fetchone()[0]
        self.num_chunks = db_length // chunk_size
        self.chunk_indices = chunk_id_ranges(db_length, chunk_size, window)
        self.x_fields, from_clause = _split_query(db_x_query)

        mins = ", ".join("MIN({})".format(f) for f in self.x_fields)
        maxs = ", ".join("MAX({})".format(f) for f in self.x_fields)
        self.norm_params = []
        for ids in self.chunk_indices:
            cursor.execute("SELECT {} {} WHERE ID IN {};".format(mins, from_clause, tuple(ids)))
            x_min = torch.Tensor(cursor.fetchall())
            cursor.execute("SELECT {} {} WHERE ID IN {};".format(maxs, from_clause, tuple(ids)))
            x_max = torch.Tensor(cursor.fetchall())
            x_min[0], x_max[0] = widen_degenerate(x_min[0], x_max[0])
            self.norm_params.append((x_min, x_max))
        for x_min, x_max in self.norm_params:
            share_book_levels(self.x_fields, x_min, x_max)

        if norm_params_path:
            last_min, last_max = self.norm_params[-1]
            table_ = {name: {"MIN": last_min[0][i], "MAX": last_max[0][i]} for i, name in enumerate(self.x_fields)}
            with open(norm_params_path, "wb") as fh:
                pickle.dump(table_, fh)

    def __getitem__(self, idx):
        return tuple(self.chunk_indices[idx]), self.norm_params[idx]

    def __len__(self):
        return self.num_chunks + 1

    @classmethod
    def from_table(cls, table: torch.Tensor, x_fields, chunk_size, window, norm_params_path="norm_params"):
        """Same object, built from a bulk-loaded feature table resident in HBM instead of 2 SQL aggregates per chunk
        (SURVEY.md 8(f) N3): ``table[i]`` is the row with database ID ``i + 1``, NaN = SQL NULL.  Per-chunk MIN/MAX come
        from one reduction kernel (``bigru_chunk_minmax``); the min==max guard, order-book sharing and the
        ``norm_params`` pickle are the reference's host rules, unchanged."""
        if not table.is_cuda:
            raise RuntimeError("from_table needs the table on a CUDA device (no CPU fallback)")
        self = cls.__new__(cls)
        table = table.to(torch.float32).contiguous()
        db_length, F = table.shape
        self.num_chunks = db_length // chunk_size
        self.chunk_indices = chunk_id_ranges(db_length, chunk_size, window)
        self.x_fields = list(x_fields)
        self.norm_params = []
        lib = _lib.load()
        mn = torch.empty(F, device=table.device, dtype=torch.float32)
        mx = torch.empty(F, device=table.device, dtype=torch.float32)
        for ids in self.chunk_indices:
            with torch.cuda.device(table.device):
                _lib.check(lib.bigru_chunk_minmax(_lib.ptr(table), db_length, F, ids[0] - 1, ids[-1], _lib.ptr(mn), _lib.ptr(mx),
                                                  torch.cuda.current_stream(table.device).cuda_stream), "bigru_chunk_minmax")
            x_min, x_max = mn.cpu().reshape(1, F).clone(), mx.cpu().reshape(1, F).clone()
            x_min[0], x_max[0] = widen_degenerate(x_min[0], x_max[0])
            self.norm_params.append((x_min, x_max))
        for x_min, x_max in self.norm_params:
            share_book_levels(self.x_fields, x_min, x_max)
        if norm_params_path:
            last_min, last_max = self.norm_params[-1]
            table_ = {name: {"MIN": last_min[0][i], "MAX": last_max[0][i]} for i, name in enumerate(self.x_fields)}
            with open(norm_params_path, "wb") as fh:
                pickle.dump(table_, fh)
        return self


def delivered_window_batches(n_rows: int, window: int, batch_size: int):
    """(start, count) of every batch a ``DataLoader(dataset, batch_size)`` over the reference dataset
    delivers.  The reference dataset reports len == n_rows but can only produce n_rows-window+1
    windows; the batch that is in flight when its window generator is exhausted is lost
    (StopIteration ends the epoch).  Reproduced here so the fast path yields identical batches."""
    n_win = max(n_rows - window + 1, 0)
    out = [(s, min(batch_size, n_win - s)) for s in range(0, n_win, batch_size)]
    if out and out[-1][1] < batch_size and n_win < n_rows:
        out.pop()
    return out


class MySQLBatchLoader(Dataset):
    """Sliding-window dataset over one chunk, resident in HBM.

    Drop-in use (per-sample, as the reference): ``DataLoader(MySQLBatchLoader(...), batch_size)``.
    Fast path: ``for x, y in dataset.batches(batch_size)`` - one gather kernel per batch, yielding
    exactly the batches the DataLoader would (``drop_incomplete=False`` also returns the tail the
    reference loses).
    """

    def __init__(self, indices, norm_params, cursor, table, db_x_query, y_fields, window, device=None):
        super().__init__()
        indices = tuple(indices)
        x_fields, from_clause = _split_query(db_x_query)
        cols = ", ".join("IFNULL({}, 0)".format(f) for f in x_fields)
        cursor.execute("SELECT {} {} WHERE ID IN {};".format(cols, from_clause, indices))
        x_rows = torch.Tensor(cursor.fetchall())
        cursor.execute("SELECT {} FROM target WHERE ID IN {};".format(y_fields, indices))
        y_rows = torch.Tensor(cursor.fetchall())

        if device is None:
            if not torch.cuda.is_available():
                raise RuntimeError("MySQLBatchLoader (H100-native) keeps the chunk in HBM and collates with a CUDA "
                                   "kernel; no CUDA device is available and there is no CPU fallback")
            device = torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        self.window = int(window)
        self.n_rows, self.n_features = x_rows.shape[0], x_rows.shape[1] if x_rows.dim() == 2 else 0
        self.n_targets = y_rows.shape[1] if y_rows.dim() == 2 else 0
        self.x_raw = x_rows.to(self.device).contiguous()                    # one H2D copy per chunk
        self.y = y_rows.to(self.device).contiguous()
        self.x_min = norm_params[0][0].to(self.device, torch.float32).contiguous()
        self.x_max = norm_params[1][0].to(self.device, torch.float32).contiguous()
        # normalised chunk (reference attribute `x`, :239) = the gather kernel with one window of N rows
        self.x = self._gather(0, 1, self.n_rows)[0] if self.n_rows else self.x_raw
        self.indices_gen = window_indices(range(len(indices)), window)

    @classmethod
    def from_tensors(cls, x_rows, y_rows, norm_params, window, device=None):
        """The same dataset over a chunk that is already in memory (x_rows [N, F] raw features, y_rows [N, C] targets,
        norm_params = (min [1, F], max [1, F]) as MySQLChunkLoader yields them) - no cursor, no SQL.  Used when the table
        has been bulk-loaded (MySQLChunkLoader.from_table) and by the loader arm of bench.py."""
        self = cls.__new__(cls)
        Dataset.__init__(self)
        if device is None:
            device = x_rows.device if x_rows.is_cuda else torch.device("cuda", torch.cuda.current_device())
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("MySQLBatchLoader (H100-native) keeps the chunk in HBM; there is no CPU fallback")
        self.window = int(window)
        self.x_raw = x_rows.to(self.device, torch.float32).contiguous()
        self.y = y_rows.to(self.device, torch.float32).contiguous()
        self.n_rows, self.n_features = self.x_raw.shape
        self.n_targets = self.y.shape[1] if self.y.dim() == 2 else 0
        self.x_min = norm_params[0][0].to(self.device, torch.float32).contiguous()
        self.x_max = norm_params[1][0].to(self.device, torch.float32).contiguous()
        self.x = None                                   # the normalised copy is formed on demand by collate()/the fused forward
        self.indices_gen = window_indices(range(self.n_rows), window)
        return self

    def _gather(self, start, count, width):
        out = torch.empty(count, width, self.n_features, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):             # the C ABI launches on the current device: make it the chunk's
            _lib.check(_lib.load().bigru_window_gather_norm(
                _lib.ptr(self.x_raw), _lib.ptr(self.x_min), _lib.ptr(self.x_max), start, self.n_rows, count, width,
                self.n_features, _lib.ptr(out), torch.cuda.current_stream(self.device).cuda_stream),
                "bigru_window_gather_norm")
        return out

    def collate(self, start: int, count: int):
        """x[count, W, F] (normalised) and y[count, 1, C] for windows start .. start+count-1."""
        x = self._gather(start, count, self.window)
        y = torch.empty(count, 1, self.n_targets, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            _lib.check(_lib.load().bigru_window_targets(
                _lib.ptr(self.y), start, self.n_rows, count, self.window, self.n_targets, _lib.ptr(y),
                torch.cuda.current_stream(self.device).cuda_stream), "bigru_window_targets")
        return x, y

    def batches(self, batch_size: int, drop_incomplete: bool = True):
        n_win = max(self.n_rows - self.window + 1, 0)
        if drop_incomplete:
            plan = delivered_window_batches(self.n_rows, self.window, batch_size)
        else:
            plan = [(s, min(batch_size, n_win - s)) for s in range(0, n_win, batch_size)]
        for start, count in plan:
            yield self.collate(start, count)

    def __getitem__(self, idx):
        w = next(self.indices_gen)          # sequential by construction, like the reference (idx is ignored)
        if self.x is None:
            self.x = self._gather(0, 1, self.n_rows)[0]
        return self.x[w[0]:w[-1] + 1], self.y[w[-1]:w[-1] + 1]

    def __len__(self):
        return self.n_rows


class TrainValTestSplit:
    """Chunk-granular train / validation / test split (contiguous, in that order).

    train gets int((1 - val - test) * n_chunks) chunks, validation and test int(frac * n_chunks) + 1.
    """

    def __init__(self, dataset, val_size=0.1, test_size=0.1):
        assert (val_size + test_size) < 1, 'Validation size and test size sum is greater or equal 1'
        assert val_size >= 0 and test_size >= 0, 'Negative size is not accepted'
        self.dataset = dataset
        self.val_size, self.test_size = val_size, test_size
        self.train_size = 1 - val_size - test_size
        self.dataset_len = len(dataset)

    def _take(self, lo, hi):
        ids, norms = self.dataset[lo:hi]
        return zip(ids, norms)

    def get_train(self):
        self.train_end_idx = int(self.train_size * self.dataset_len)
        return self._take(0, self.train_end_idx)

    def get_val(self):
        self.val_start_idx = self.train_end_idx
        self.val_end_idx = self.val_start_idx + int(self.val_size * self.dataset_len) + 1
        return self._take(self.val_start_idx, self.val_end_idx)

    def get_test(self):
        self.test_start_idx = self.val_end_idx
        self.test_end_idx = self.test_start_idx + int(self.test_size * self.dataset_len) + 1
        return self._take(self.test_start_idx, self.test_end_idx)

    def get_sets(self):
        return self.get_train(), self.get_val(), self.get_test()
