"""In-memory stand-ins for the reference's process boundaries (MariaDB cursor, `config`, `pytz`).

The reference's loader talks to MariaDB through a DB-API cursor (sql_pytorch_dataloader.py:65-66,
96-105, 227-236).  FakeCursor answers exactly the five statement shapes it issues from a table
held as numpy columns, so both the unmodified reference loader (tests/golden/make_golden.py)
and the product loader can be driven without a database.
"""
from __future__ import annotations

import re
import sys
import types

import numpy as np


class FakeCursor:
    def __init__(self, columns: dict, targets: dict):
        """columns: {"sd.open": array[N], ...}; targets: {"up1": array[N], ...}; row i has ID i+1."""
        self.columns = {k: np.asarray(v, np.float64) for k, v in columns.items()}
        self.targets = {k: np.asarray(v, np.float64) for k, v in targets.items()}
        self.n = len(next(iter(self.columns.values())))
        self._rows = []
        self.statements = []

    @staticmethod
    def _ids(sql):
        inside = sql[sql.rindex("ID IN") + 5:]
        return [int(v) for v in re.findall(r"-?\d+", inside)]

    def execute(self, sql):
        self.statements.append(sql)
        s = sql.strip()
        if s.startswith("SELECT COUNT(ID)"):
            self._rows = [(self.n,)]
            return
        rows = np.array(self._ids(s), dtype=np.int64) - 1
        rows = rows[(rows >= 0) & (rows < self.n)]          # WHERE ID IN (...) skips IDs the table does not have
        head = s[len("SELECT"):s.index(" FROM ")]
        if "FROM target" in s:
            names = [w.strip() for w in head.split(",")]
            self._rows = [tuple(float(self.targets[n][r]) for n in names) for r in rows]
        elif head.lstrip().startswith("MIN(") or head.lstrip().startswith("MAX("):
            fn = np.nanmin if head.lstrip().startswith("MIN(") else np.nanmax
            names = re.findall(r"M(?:IN|AX)\(([^)]+)\)", head)
            self._rows = [tuple(float(fn(self.columns[n][rows])) for n in names)]
        elif "IFNULL(" in head:
            names = re.findall(r"IFNULL\(([^,]+), 0\)", head)
            mat = np.stack([np.nan_to_num(self.columns[n][rows], nan=0.0) for n in names], 1)
            self._rows = [tuple(float(v) for v in r) for r in mat]
        else:
            raise ValueError("FakeCursor: unexpected statement: " + s[:80])

    def fetchone(self):
        return self._rows[0]

    def fetchall(self):
        return list(self._rows)


def make_table(n_rows=250, n_plain=3, levels=2, n_targets=4, seed=7, with_nulls=True, const_col=True, null_rows=None):
    """A small synthetic joined table with order-book size columns, a constant column and NULLs.

    Columns: ``levels`` bid/ask size pairs, ``n_plain`` normal columns ``sd.f<i>``, then (``const_col``) a constant
    non-zero and a constant zero column.  ``with_nulls`` puts NULL (NaN) in about 5 % of ``sd.f0``; ``null_rows``
    ({field: 0-based row numbers}) adds NULLs at chosen rows, e.g. at chunk edges.  The defaults reproduce
    tests/golden/loader.npz's table bit for bit."""
    rng = np.random.default_rng(seed)
    cols = {}
    for i in range(levels):
        cols[f"sd.bid_{i}_size"] = rng.integers(100, 900 + 100 * i, n_rows).astype(np.float64)
        cols[f"sd.ask_{i}_size"] = rng.integers(50, 700 + 150 * i, n_rows).astype(np.float64)
    for i in range(n_plain):
        cols[f"sd.f{i}"] = rng.normal(10 * i, 1 + i, n_rows)
    if const_col:
        cols["sd.const_nz"] = np.full(n_rows, 3.5)
        cols["sd.const_zero"] = np.zeros(n_rows)
    if with_nulls:
        nul = rng.random(n_rows) < 0.05
        cols["sd.f0"] = np.where(nul, np.nan, cols["sd.f0"])
    targets = {f"t{i}": (rng.random(n_rows) < 0.3).astype(np.float64) for i in range(n_targets)}
    for name, rows in (null_rows or {}).items():
        cols[name][list(rows)] = np.nan
    fields = list(cols.keys())
    query = "SELECT " + ", ".join(fields) + " FROM stock_data_joined sd JOIN other o ON sd.ID = o.ID;"
    return cols, targets, fields, query


def install_reference_stubs(bid_levels=2, ask_levels=2):
    """`config.py` of the reference imports pytz (absent here) and holds credentials; the loader only
    needs config.bid_levels / config.ask_levels (sql_pytorch_dataloader.py:5)."""
    cfg = types.ModuleType("config")
    cfg.bid_levels, cfg.ask_levels = bid_levels, ask_levels
    sys.modules["config"] = cfg
    if "pytz" not in sys.modules:
        sys.modules["pytz"] = types.ModuleType("pytz")
