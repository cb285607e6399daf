"""Window-function features of the reference's database layer on the GPU (SURVEY.md 8(f) N4).

The reference builds its technical-indicator columns and the four target labels as MariaDB window-function VIEWs over the
joined table (``create_database.py:76-190``) and joins them back in a fixed column order (``create_database.py:239-256``).
``window_features`` computes the same columns from device tensors with one row-parallel CUDA kernel
(``bigru_window_features``), for bulk back-fills where the table already lives on the GPU.  SQL ``NULL`` is ``NaN``.
A NULL inside an input column differs from SQL: AVG skips it, while the kernel's NaN propagates into every frame holding it.
Argument names follow ``config.py:40-49`` of the reference.  There is no CPU fallback."""
from __future__ import annotations

import ctypes as C

import torch

from . import _lib


def feature_names(volume_MA_periods=(6, 20), price_MA_periods=(20,), delta_MA_periods=(12,), bollinger_bands_period=20,
                  bollinger_bands_std=2, stochastic_oscillator=True):
    """Column names in the order of the reference's join statement (``create_database.py:239-240``)."""
    names = []
    if bollinger_bands_period and bollinger_bands_std:
        names += ["upper_BB_dist", "lower_BB_dist"]
    names += [f"vol_MA{p}" for p in (volume_MA_periods or [])]
    names += [f"price_MA{p}" for p in (price_MA_periods or [])]
    names += [f"delta_MA{p}" for p in (delta_MA_periods or [])]
    if stochastic_oscillator:
        names.append("stoch")
    return names + ["ATR", "price_change"]


def window_features(close, high, low, volume=None, delta=None, volume_MA_periods=(6, 20), price_MA_periods=(20,),
                    delta_MA_periods=(12,), bollinger_bands_period=20, bollinger_bands_std=2, stochastic_oscillator=True,
                    n1=1.5, n2=3.0, with_targets=True):
    """close/high/low/volume/delta: 1-D float32 CUDA tensors of the table's ``4_close, 2_high, 3_low, 5_volume, delta``
    columns in Timestamp order.  Returns ``(features[n, n_out], targets[n, 4] or None)``; targets are
    ``up1, up2, down1, down2`` of the reference's ``target`` view."""
    cols = [close, high, low, volume, delta]
    if not close.is_cuda:
        raise RuntimeError("window_features runs on the GPU only (no CPU fallback): pass CUDA tensors")
    vol_p = list(volume_MA_periods or [])
    price_p = list(price_MA_periods or [])
    delta_p = list(delta_MA_periods or [])
    if vol_p and volume is None:
        raise ValueError("volume_MA_periods needs the volume column")
    if delta_p and delta is None:
        raise ValueError("delta_MA_periods needs the delta column")
    n = close.numel()
    cols = [None if c is None else c.contiguous().float() for c in cols]
    for c in cols:
        if c is not None and (c.numel() != n or c.device != close.device):
            raise ValueError("all columns must have the same length and device")
    bb = int(bollinger_bands_period) if (bollinger_bands_period and bollinger_bands_std) else 0
    n_out = len(feature_names(vol_p, price_p, delta_p, bb, bollinger_bands_std, stochastic_oscillator))
    out = torch.empty((n, n_out), dtype=torch.float32, device=close.device)
    tgt = torch.empty((n, 4), dtype=torch.float32, device=close.device) if with_targets else None
    lib = _lib.load()

    def arr(v):
        return (C.c_int * max(1, len(v)))(*v) if v else None

    got = C.c_int(0)
    with torch.cuda.device(close.device):
        _lib.check(lib.bigru_window_features(*[_lib.ptr(c) if c is not None else None for c in cols], n, arr(vol_p), len(vol_p),
                                             arr(price_p), len(price_p), arr(delta_p), len(delta_p), bb, float(bollinger_bands_std or 0),
                                             1 if stochastic_oscillator else 0, float(n1), float(n2), _lib.ptr(out) if n else None,
                                             _lib.ptr(tgt) if (tgt is not None and n) else None, C.byref(got),
                                             torch.cuda.current_stream(close.device).cuda_stream), "bigru_window_features")
    assert got.value == n_out, (got.value, n_out)
    return out, tgt
