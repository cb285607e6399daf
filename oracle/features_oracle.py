"""TEST INFRASTRUCTURE ONLY - CPU restatement of the reference's SQL window-function features (SURVEY.md 8(f) N4).

Follows /root/reference/create_database.py:76-190 (the CREATE VIEW statements) and :239-256 (column order of the join):
  vol_MA / price_MA / delta_MA  :76-118   AVG(col) OVER (ORDER BY Timestamp ROWS BETWEEN p-1 PRECEDING AND CURRENT ROW)
  bollinger_bands               :120-135  (avg + k*std) - close, close - (avg - k*std); MariaDB STD = population std
  stochastic_oscillator         :137-147  (close - min) / (max - min) over ROWS BETWEEN 14 PRECEDING AND CURRENT ROW; x/0 = NULL
  price_change                  :150-154  close - LAG(close, 1): NULL on the first row
  ATR                           :156-161  AVG(high - low) over ROWS BETWEEN 14 PRECEDING AND CURRENT ROW
  target                        :163-185  LEAD(close, 8 / 15) vs close +- n1 / n2 * ATR; a comparison with NULL is not true -> 0
Frames at the head of the table are shorter (SQL window frames clip at the partition start).  NULL is NaN.

PINNED to the reference's own SQL: tests/golden/make_features_golden.py imports the UNMODIFIED create_database.py with a
`mysql.connector` stub that forwards its statements to sqlite3 (window functions; MariaDB's STD registered as a window
aggregate), fills the table with a seed-fixed synthetic market and stores what the reference's views return in
tests/golden/features.npz; tests/test_oracle_cpu.py checks this restatement against it (exact) and, independently,
against pandas.rolling and hand-computed rows.  tests/golden/features_ties.npz is the same check on a quarter-point tick
grid, where the move to row i + 8 / i + 15 often equals n1 / n2 * ATR exactly.

Exactness: every frame is summed on its own with math.fsum (the correctly rounded sum; a running cumsum loses its low bits
on long tables) and then divided by the row count, as SQL's AVG does.  The targets compare close[i + h] with
close[i] +- n * ATR in double, in the SQL's order of operations.  So on a tick grid, where the sums are exact, the labels
equal the SQL's at ties as well."""
from __future__ import annotations

import math

import numpy as np
from numpy.lib.stride_tricks import sliding_window_view


def _frames(n, w):
    i = np.arange(n)
    return np.maximum(0, i - w + 1), i


def _head_and_body(x, w):
    """The clipped frames of the first min(w - 1, n) rows as lists, and the full frames after them as a [n - w + 1, w] view."""
    x = np.asarray(x, dtype=np.float64)
    h = min(w - 1, len(x))
    head = [x[:i + 1] for i in range(h)]
    body = sliding_window_view(x, w) if len(x) >= w else np.zeros((0, w))
    return head, body


def _chunks(body, elems=1 << 20):
    """(first row, rows) of the [n - w + 1, w] frame view in pieces of about `elems` values, so that no list or
    temporary of the whole view is built (w = 4096 over 20,000 rows would be 65M values)."""
    step = max(1, elems // max(1, body.shape[1]))
    for r in range(0, len(body), step):
        yield r, body[r:r + step]


def rolling_sum(x, w):
    """Correctly rounded sum of every frame [max(0, i - w + 1), i]."""
    head, body = _head_and_body(x, w)
    out = [math.fsum(f.tolist()) for f in head]
    for _, rows in _chunks(body):
        out += [math.fsum(f) for f in rows.tolist()]
    return np.array(out, dtype=np.float64)


def rolling_mean(x, w):
    lo, hi = _frames(len(x), w)
    return rolling_sum(x, w) / (hi - lo + 1)


def rolling_std_pop(x, w):
    """Population standard deviation of every frame, two-pass around the frame's exact mean: no cancellation."""
    x = np.asarray(x, dtype=np.float64)
    m = rolling_mean(x, w)
    head, body = _head_and_body(x, w)
    out = np.empty(len(x))
    for i, f in enumerate(head):
        out[i] = np.sqrt(np.mean((f - m[i]) ** 2))
    for r, rows in _chunks(body):
        i = len(head) + r
        out[i:i + len(rows)] = np.sqrt(np.mean((rows - m[i:i + len(rows), None]) ** 2, axis=1))
    return out


def rolling_minmax(x, w):
    x = np.asarray(x, dtype=np.float64)
    head, body = _head_and_body(x, w)
    mn = np.array([f.min() for f in head] + [v for _, rows in _chunks(body) for v in rows.min(axis=1)], dtype=np.float64)
    mx = np.array([f.max() for f in head] + [v for _, rows in _chunks(body) for v in rows.max(axis=1)], dtype=np.float64)
    return mn, mx


def window_features(close, high, low, volume=None, delta=None, volume_MA_periods=(6, 20), price_MA_periods=(20,),
                    delta_MA_periods=(12,), bollinger_bands_period=20, bollinger_bands_std=2, stochastic_oscillator=True,
                    n1=1.5, n2=3.0):
    """Returns (features [n, n_out] float64, targets [n, 4] float64), columns as create_database.py:239-240."""
    close = np.asarray(close, dtype=np.float64)
    n = len(close)
    cols = []
    if bollinger_bands_period and bollinger_bands_std:
        avg, sd = rolling_mean(close, bollinger_bands_period), rolling_std_pop(close, bollinger_bands_period)
        cols += [(avg + bollinger_bands_std * sd) - close, close - (avg - bollinger_bands_std * sd)]
    cols += [rolling_mean(volume, p) for p in (volume_MA_periods or [])]
    cols += [rolling_mean(close, p) for p in (price_MA_periods or [])]
    cols += [rolling_mean(delta, p) for p in (delta_MA_periods or [])]
    if stochastic_oscillator:
        mn, mx = rolling_minmax(close, 15)
        with np.errstate(divide="ignore", invalid="ignore"):
            cols.append(np.where(mx > mn, (close - mn) / (mx - mn), np.nan))
    atr = rolling_mean(np.asarray(high, dtype=np.float64) - np.asarray(low, dtype=np.float64), 15)
    cols.append(atr)
    pc = np.full(n, np.nan)
    if n > 1:
        pc[1:] = close[1:] - close[:-1]
    cols.append(pc)
    feats = np.stack(cols, axis=1) if n else np.zeros((0, len(cols)))
    tgt = np.zeros((n, 4))
    n1, n2 = float(n1), float(n2)
    for h, n_atr, up, down in ((8, n1, 0, 2), (15, n2, 1, 3)):       # p_h >= p0 + (n * ATR), p_h <= p0 - (n * ATR); NULL -> 0
        if n > h:
            p0, ph, a = close[:-h], close[h:], n_atr * atr[:-h]
            tgt[:-h, up] = ph >= p0 + a
            tgt[:-h, down] = ph <= p0 - a
    return feats, tgt
