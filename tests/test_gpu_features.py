"""window_features_kernel (csrc/features.cuh) per column against the exact oracle (oracle/features_oracle.py), at its tile,
halo and grid-stride edges, and its target labels against the reference's own SQL at exact ties.

Per-column bounds, row by row (u = 2^-24, ulp(x) = np.spacing(float32(x))):
  stoch, price_change   bitwise equal to the fp32 rounding of the exact value.  Both are formed from fp32 differences of
                        prices that are exact by Sterbenz's lemma when every price is positive (p/2 <= q <= 2p), so the
                        only rounding is that of the final division (stoch) or of nothing at all (price_change).
  vol_MA / price_MA /   |got - ref| <= A_MA ulp(ref) + B_MA u max_k |c_k - c_i| over the frame: the kernel sums the
  delta_MA              differences to the current row, so the error scales with the frame's spread, not its level.
                        With integer inputs every difference and partial sum is exact, leaving the rounding of s / cnt and
                        of ref + s / cnt: |got - ref| <= ulp(ref) + u max_k |c_k - c_i|.  A plain 1-ulp bound does not
                        hold: fl(s / cnt) is off by up to u |s / cnt|, more than an ulp of the mean when the frame's
                        spread is comparable to its level.
  upper / lower_BB_dist <= B_BB u max_k |c_k - c_i| over the BB frame.
  ATR                   <= C_ATR u mean(|high - low|) over the 15-row frame.
Labels are exact: against the oracle, against tests/golden/features_ties.npz (the reference's SQL on a quarter-point grid,
where the move often equals n * ATR exactly) and against tests/golden/features.npz.

Measured on an H100 80GB HBM3 (700 W power limit), worst value over every case of this file and both goldens:
  MA (rounding sums)   (|got - ref| - ulp(ref)) / (u spread) = 2.89  ->  A_MA = 1, B_MA = 12
  MA (integer inputs)  |got - ref| / (ulp(ref) + u spread)   = 0.503 ->  held to 1 (the derived bound, not a fit)
  BB                   |got - ref| / (u spread)              = 7.67  ->  B_BB = 32
  ATR                  |got - ref| / (u mean|high - low|)    = 1.87  ->  C_ATR = 8
stoch and price_change were bitwise equal to the rounded exact value everywhere, and the labels had no difference from
the oracle or either golden.  The feature columns are bit for bit those of the kernel before the tie-aware labels, on
every table here.  That kernel got 36 labels of features_ties.npz wrong, 257 of the 60,000-row tick table (FAST; the
generic path got them right, so the two paths disagreed), 1,155 of the one-pass-plus-one tick table and 1 of the
continuous one-pass-plus-257 table.

Mutations, one at a time, each value-only (no indexing that can leave an allocation), and the tests that fail (H100):
  mutation                                        this file                                  test_gpu_parity window_features
  frame_mean over levels (s = ref + sum c[k])     4 generic cases (halo14, halo255/257,      none
                                                  eight_periods)
  halo staged from blockIdx.x, not tile           the 3 one-pass-plus cases, the 2M sample   properties_large
  generic ATR as sa * (1 / cnt)                   16 cases on the tick grid, FAST against    none
                                                  generic, features_ties.npz
  fp64 label >= turned into >                     7 tie-heavy cases, FAST against generic,   none
                                                  features_ties.npz, the 2M sample
  tie bound 2^-30 instead of 2^-19 (fp32 decides  3 FAST cases (past one grid pass, or    none
  near ties)                                      dyadic n), FAST against generic,
                                                  features_ties.npz, the 2M sample
  FAST BB variance / 19 instead of / 20           7 FAST cases, FAST against generic, both   match_reference_sql,
                                                  goldens, the 2M sample                     match_oracle[500, 20000]
"""
import os

import numpy as np
import pytest
import torch

from oracle import features_oracle as fo

U = 2.0 ** -24
A_MA, B_MA, B_BB, C_ATR = 1.0, 12.0, 32.0, 8.0
PASS = 132 * 8 * 256                         # rows one grid-stride pass covers (the grid is capped at 132 * 8 blocks)
DEFAULT = dict(volume_MA_periods=[6, 20], price_MA_periods=[20], delta_MA_periods=[12], bollinger_bands_period=20,
               bollinger_bands_std=2, stochastic_oscillator=True)


# ---- tables ----------------------------------------------------------------------------------------------------------
def tick_table(n, seed=11, tick=0.25):
    """Quarter-point steps from 3000, high / low 1-5 ticks either side, integer volume and delta, flat stretches: every
    value exact in fp32, and the move to row i + 8 / i + 15 often equals n * ATR exactly."""
    rng = np.random.default_rng(seed)
    close = 3000 + tick * np.cumsum(np.round(rng.normal(0, 3, n)))
    for s in range(500, n, 5000):
        close[s:s + 30] = close[s]
    high = close + tick * rng.integers(1, 6, n)
    low = close - tick * rng.integers(1, 6, n)
    return [np.float32(c) for c in (close, high, low, rng.integers(1, 5000, n), rng.integers(-2000, 2000, n))]


def market_table(n, seed=5):
    """A continuous price near 2900 (not on a grid) with real-valued delta: the frame sums round."""
    rng = np.random.default_rng(seed)
    close = 2900 + np.cumsum(rng.normal(0, 2.0, n))
    if n > 200:
        close[100:140] = close[100]
    cols = [close, close + rng.uniform(0.1, 3.0, n), close - rng.uniform(0.1, 3.0, n),
            rng.integers(100, 50000, n).astype(np.float64), rng.normal(0, 300, n)]
    return [np.float32(c) for c in cols]


TABLES = {"tick": tick_table, "market": market_table}


def halo_of(kw):
    ps = list(kw.get("volume_MA_periods") or []) + list(kw.get("price_MA_periods") or []) + list(kw.get("delta_MA_periods") or [])
    bb = kw.get("bollinger_bands_period") if kw.get("bollinger_bands_std") else 0
    return max([14] + [p - 1 for p in ps] + [(bb or 0) - 1])


def is_fast(kw):
    return (list(kw.get("volume_MA_periods") or []) == [6, 20] and list(kw.get("price_MA_periods") or []) == [20]
            and list(kw.get("delta_MA_periods") or []) == [12] and kw.get("bollinger_bands_period") == 20
            and bool(kw.get("bollinger_bands_std")) and bool(kw.get("stochastic_oscillator")))


# ---- cases and the regimes they cover ---------------------------------------------------------------------------------
def _k(**kw):
    return dict(DEFAULT, **kw)


CASES = {
    "tick_n1": dict(table="tick", n=1, kw=DEFAULT),
    "tick_n7": dict(table="tick", n=7, kw=DEFAULT),
    "tick_n8": dict(table="tick", n=8, kw=DEFAULT),
    "tick_n9": dict(table="tick", n=9, kw=DEFAULT),
    "tick_n15": dict(table="tick", n=15, kw=DEFAULT),
    "tick_n16": dict(table="tick", n=16, kw=DEFAULT),
    "tick_n19": dict(table="tick", n=19, kw=DEFAULT),
    "tick_n20": dict(table="tick", n=20, kw=DEFAULT),
    "tick_n21": dict(table="tick", n=21, kw=DEFAULT),
    "market_n255": dict(table="market", n=255, kw=DEFAULT),
    "market_n256": dict(table="market", n=256, kw=_k(volume_MA_periods=[20, 6])),
    "tick_n257": dict(table="tick", n=257, kw=DEFAULT),
    "tick_60k": dict(table="tick", n=60_000, kw=DEFAULT),
    "tick_60k_generic": dict(table="tick", n=60_000, kw=_k(volume_MA_periods=[20, 6])),
    "tick_pass_plus_1": dict(table="tick", n=PASS + 1, kw=DEFAULT),
    "tick_pass_plus_257_generic": dict(table="tick", n=PASS + 257, kw=_k(volume_MA_periods=[20, 6])),
    "market_pass_plus_257": dict(table="market", n=PASS + 257, kw=DEFAULT),
    "halo255_price_eq_bb": dict(table="market", n=5000, kw=_k(volume_MA_periods=[3, 256], price_MA_periods=[10, 40],
                                                            delta_MA_periods=[5], bollinger_bands_period=40,
                                                            bollinger_bands_std=1.5, stochastic_oscillator=False)),
    "halo256_no_bb": dict(table="tick", n=5000, kw=_k(volume_MA_periods=[], price_MA_periods=[257, 20], delta_MA_periods=[],
                                                      bollinger_bands_period=False)),
    "halo257_period1": dict(table="market", n=3000, kw=_k(volume_MA_periods=[1, 6], price_MA_periods=[1, 258], delta_MA_periods=[1],
                                                          bollinger_bands_period=2)),
    "halo4095": dict(table="tick", n=20_000, kw=_k(volume_MA_periods=[4096], price_MA_periods=[7, 31], delta_MA_periods=[12],
                                                   bollinger_bands_period=10, bollinger_bands_std=1.5)),
    "eight_periods": dict(table="market", n=4000, kw=_k(volume_MA_periods=[1, 2, 3, 5, 8, 13, 21, 34],
                                                        price_MA_periods=[2, 4, 6, 8, 10, 12, 14, 16],
                                                        delta_MA_periods=[3, 6, 9, 12, 15, 18, 21, 24])),
    "no_volume_no_targets": dict(table="tick", n=3000, kw=_k(volume_MA_periods=[], price_MA_periods=[15], bollinger_bands_period=15),
                                 volume=False, targets=False),
    "halo14": dict(table="market", n=3000, kw=_k(volume_MA_periods=[6, 15], price_MA_periods=[3], delta_MA_periods=[12],
                                                 bollinger_bands_period=15)),
    "no_delta": dict(table="market", n=3000, kw=_k(delta_MA_periods=[]), delta=False),
    "dyadic_n": dict(table="tick", n=20_000, kw=_k(n1=0.75, n2=2.5)),
    "n1_zero": dict(table="tick", n=20_000, kw=_k(volume_MA_periods=[20, 6], n1=0.0, n2=0.5)),
}

REGIMES = {
    "n = 1, 7, 8, 9: no label, or the first 8-step label": ["tick_n1", "tick_n7", "tick_n8", "tick_n9"],
    "n = 15, 16: no 15-step label, or the first": ["tick_n15", "tick_n16"],
    "n = 19, 20, 21: row 19 is the first FAST row": ["tick_n19", "tick_n20", "tick_n21"],
    "n = 255, 256, 257: one tile, and one row past it": ["market_n255", "market_n256", "tick_n257"],
    "one grid pass + 1 and + 257, in full": ["tick_pass_plus_1", "tick_pass_plus_257_generic", "market_pass_plus_257"],
    "halo 14 (every period <= 15)": ["halo14", "no_volume_no_targets"],
    "halo 255, 256, 257 (a whole tile of halo)": ["halo255_price_eq_bb", "halo256_no_bb", "halo257_period1"],
    "halo 4095 (period 4096)": ["halo4095"],
    "period 1: each MA equals its input": ["halo257_period1"],
    "generic price_MA equal to the BB period, and not": ["halo255_price_eq_bb"],
    "BB off": ["halo256_no_bb"],
    "stochastic off": ["halo255_price_eq_bb"],
    "volume absent": ["no_volume_no_targets"],
    "delta absent": ["no_delta"],
    "with_targets=False": ["no_volume_no_targets"],
    "8 periods in every list (n_out = 29)": ["eight_periods"],
    "dyadic n1 / n2 other than 1.5 / 3": ["dyadic_n", "n1_zero"],
    "n1 = 0: a flat 8-step move sets up1 and down1": ["n1_zero"],
    "FAST and generic on the same tie-heavy table": ["tick_60k", "tick_60k_generic"],
}
# test_fast_and_generic_agree_at_ties runs this pair (one table through both paths); the per-case test skips it.
PAIR = ("tick_60k", "tick_60k_generic")


def case_regimes(c):
    """The regimes a case is in, derived from its parameters (what REGIMES claims must be true of the case)."""
    n, kw, h = c["n"], c["kw"], halo_of(c["kw"])
    ps = list(kw.get("volume_MA_periods") or []) + list(kw.get("price_MA_periods") or []) + list(kw.get("delta_MA_periods") or [])
    lists = [kw.get("volume_MA_periods") or [], kw.get("price_MA_periods") or [], kw.get("delta_MA_periods") or []]
    bb = kw.get("bollinger_bands_period") if kw.get("bollinger_bands_std") else 0
    r = set()
    if n in (1, 7, 8, 9):
        r.add("n = 1, 7, 8, 9: no label, or the first 8-step label")
    if n in (15, 16):
        r.add("n = 15, 16: no 15-step label, or the first")
    if n in (19, 20, 21) and is_fast(kw):
        r.add("n = 19, 20, 21: row 19 is the first FAST row")
    if n in (255, 256, 257):
        r.add("n = 255, 256, 257: one tile, and one row past it")
    if n - PASS in (1, 257):
        r.add("one grid pass + 1 and + 257, in full")
    if h == 14:
        r.add("halo 14 (every period <= 15)")
    if h in (255, 256, 257):
        r.add("halo 255, 256, 257 (a whole tile of halo)")
    if h == 4095:
        r.add("halo 4095 (period 4096)")
    if 1 in ps:
        r.add("period 1: each MA equals its input")
    if not is_fast(kw) and bb and bb in (kw.get("price_MA_periods") or []) and any(p != bb for p in kw["price_MA_periods"]):
        r.add("generic price_MA equal to the BB period, and not")
    if not bb:
        r.add("BB off")
    if not kw.get("stochastic_oscillator"):
        r.add("stochastic off")
    if c.get("volume", True) is False:
        r.add("volume absent")
    if c.get("delta", True) is False:
        r.add("delta absent")
    if c.get("targets", True) is False:
        r.add("with_targets=False")
    if all(len(x) == 8 for x in lists):
        r.add("8 periods in every list (n_out = 29)")
    if (kw.get("n1", 1.5), kw.get("n2", 3.0)) != (1.5, 3.0):
        r.add("dyadic n1 / n2 other than 1.5 / 3")
    if kw.get("n1", 1.5) == 0:
        r.add("n1 = 0: a flat 8-step move sets up1 and down1")
    if c["table"] == "tick" and n >= 60_000 and c["kw"]["volume_MA_periods"] in ([6, 20], [20, 6]):
        r.add("FAST and generic on the same tie-heavy table")
    return r


def test_regimes_are_covered_and_claims_hold():
    for regime, names in REGIMES.items():
        assert names, regime
        for name in names:
            assert regime in case_regimes(CASES[name]), (regime, name)
    for name, c in CASES.items():
        for v in ("n1", "n2"):
            x = c["kw"].get(v, 1.5)
            assert float(np.float32(x)) == x, (name, v)        # the factors are dyadic: exact in the fp32 C ABI
    claimed = {n for names in REGIMES.values() for n in names}
    assert claimed == set(CASES), set(CASES) ^ claimed
    fast, gen = (CASES[k] for k in PAIR)
    assert (fast["table"], fast["n"]) == (gen["table"], gen["n"]) and is_fast(fast["kw"]) and not is_fast(gen["kw"])
    assert dict(fast["kw"], volume_MA_periods=fast["kw"]["volume_MA_periods"][::-1]) == gen["kw"]


# ---- running the kernel and the oracle --------------------------------------------------------------------------------
def table_of(c):
    cols = TABLES[c["table"]](c["n"])
    if c.get("volume", True) is False:
        cols[3] = None
    if c.get("delta", True) is False:
        cols[4] = None
    return cols


def gpu(cols, kw, with_targets=True):
    from financial_market_data_analysis_b200.features import window_features
    f, t = window_features(*[None if x is None else torch.from_numpy(x).cuda() for x in cols], with_targets=with_targets, **kw)
    return f.cpu().numpy(), None if t is None else t.cpu().numpy()


def oracle(cols, kw):
    return fo.window_features(*[None if x is None else x.astype(np.float64) for x in cols], **kw)


def names_of(kw):
    from financial_market_data_analysis_b200.features import feature_names
    kw = {k: v for k, v in kw.items() if k not in ("n1", "n2")}
    return feature_names(**kw)


def _spread(x, w):
    """max_k |x_k - x_i| over every frame [max(0, i - w + 1), i]."""
    mn, mx = fo.rolling_minmax(x, w)
    x = np.asarray(x, np.float64)
    return np.maximum(mx - x, x - mn)


def column_errors(cols, kw, got, ref, rows=None):
    """{column: (error / bound scale) row by row} for the bounded columns; asserts the bitwise ones.  `rows` picks the
    rows of got / ref that are compared when the oracle ran on a slice."""
    close, high, low, volume, delta = [None if x is None else x.astype(np.float64) for x in cols]
    sel = slice(None) if rows is None else rows
    assert np.array_equal(np.isnan(got), np.isnan(ref)), "SQL NULLs in other places"
    out = {}
    src = {"vol": volume, "price": close, "delta": delta}
    bb = kw.get("bollinger_bands_period") if kw.get("bollinger_bands_std") else 0
    for k, name in enumerate(names_of(kw)):
        g, r = got[:, k].astype(np.float64), ref[:, k]
        if name in ("stoch", "price_change"):
            assert np.array_equal(got[:, k], np.float32(r), equal_nan=True), name
            continue
        e = np.abs(np.nan_to_num(g) - np.nan_to_num(r))
        if name.endswith("BB_dist"):
            out[name] = ("BB", e, _spread(close, bb)[sel])
        elif name == "ATR":
            out[name] = ("ATR", e, fo.rolling_mean(np.abs(high - low), 15)[sel])
        else:
            kind, p = name.split("_MA")
            x = src[kind]
            sp = _spread(x, int(p))
            exact = bool(np.all(x == np.round(x)) and sp.max() * int(p) < 2 ** 24)     # every partial sum is an exact integer
            out[name] = ("MA", e, sp[sel], np.spacing(np.abs(np.float32(r))).astype(np.float64), exact)
    return out


def check_columns(cols, kw, got, ref, rows=None):
    for name, v in column_errors(cols, kw, got, ref, rows).items():
        kind, e, scale = v[0], v[1], v[2]
        if kind == "MA":
            ulp, integer = v[3], v[4]
            bound = ulp + U * scale if integer else A_MA * ulp + B_MA * U * scale
        else:
            bound = (B_BB if kind == "BB" else C_ATR) * U * scale
        bad = np.flatnonzero(e > bound)
        assert bad.size == 0, (name, int(bad[0]), float(e[bad[0]]), float(bound[bad[0]]))
    # On a quarter-point grid the 15-row sum of high - low is exact in fp32, so the generic path's sa / cnt is the fp32
    # rounding of the exact ATR (the FAST path's sa * (1/15.f) rounds twice: its rows from 19 on are held to the bound).
    hl = cols[1].astype(np.float64) - cols[2].astype(np.float64)
    if np.all(hl * 4 == np.round(hl * 4)) and np.abs(hl).max() * 60 < 2 ** 24:
        k = names_of(kw).index("ATR")
        idx = np.arange(len(cols[0])) if rows is None else rows
        gen = idx < 19 if is_fast(kw) else np.ones(len(idx), bool)
        assert np.array_equal(got[gen, k], np.float32(ref[gen, k])), "generic ATR is not the rounded exact mean"


def check_labels(tgt, ref_t):
    bad = np.argwhere(tgt != ref_t)
    assert bad.size == 0, (len(bad), bad[:8].tolist())


# ---- per column and labels, every case --------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(set(CASES) - set(PAIR)))
def test_case_against_exact_oracle(name):
    c = CASES[name]
    cols, kw = table_of(c), c["kw"]
    got, tgt = gpu(cols, kw, with_targets=c.get("targets", True))
    assert got.shape == (c["n"], len(names_of(kw)))
    ref, ref_t = oracle(cols, kw)
    check_columns(cols, kw, got, ref)
    if 1 in (kw.get("volume_MA_periods") or []) + (kw.get("price_MA_periods") or []) + (kw.get("delta_MA_periods") or []):
        nm = names_of(kw)
        for col, x in (("vol_MA1", cols[3]), ("price_MA1", cols[0]), ("delta_MA1", cols[4])):
            if col in nm:
                assert np.array_equal(got[:, nm.index(col)], x), col
    if c.get("targets", True):
        check_labels(tgt, ref_t)
    else:
        assert tgt is None
    if kw.get("n1") == 0:
        flat = np.flatnonzero(cols[0][8:] == cols[0][:-8])
        assert flat.size and np.all(tgt[flat, 0] == 1) and np.all(tgt[flat, 2] == 1)


@pytest.mark.gpu
def test_fast_and_generic_agree_at_ties():
    """volume_MA_periods=[20, 6] takes the generic path and only swaps two columns: both are within the bounds, and the
    labels agree bit for bit (one label routine, decided as the SQL decides at ties)."""
    fast, gen = (CASES[k] for k in PAIR)
    cols, kw = table_of(fast), gen["kw"]
    f_fast, t_fast = gpu(cols, fast["kw"])
    f_gen, t_gen = gpu(cols, kw)
    ref, ref_t = oracle(cols, kw)
    check_columns(cols, kw, f_gen, ref)
    swap = [0, 1, 3, 2, 4, 5, 6, 7, 8]
    check_columns(cols, fast["kw"], f_fast, ref[:, swap])
    assert np.array_equal(t_fast, t_gen)
    check_labels(t_gen, ref_t)


@pytest.mark.gpu
@pytest.mark.parametrize("golden", ["features.npz", "features_ties.npz"])
def test_against_reference_sql(golden_dir, golden):
    """The reference's own CREATE VIEW statements, run through sqlite (tests/golden/make_features_golden.py): NULLs,
    every column within its bound, and the labels exactly, also where the move equals n * ATR."""
    z = np.load(os.path.join(golden_dir, golden))
    cols = [z[k].astype(np.float32) for k in ("close", "high", "low", "volume", "delta")]
    kw = dict(volume_MA_periods=[int(v) for v in z["volume_MA_periods"]], price_MA_periods=[int(v) for v in z["price_MA_periods"]],
              delta_MA_periods=[int(v) for v in z["delta_MA_periods"]], bollinger_bands_period=int(z["bollinger_bands_period"]),
              bollinger_bands_std=float(z["bollinger_bands_std"]), stochastic_oscillator=True)
    got, tgt = gpu(cols, kw)
    check_columns(cols, kw, got, z["features"])
    check_labels(tgt, z["targets"])


def _oracle_rows(cols, kw, rows, h):
    """The oracle at the given (sorted, contiguous-run) rows of a long table, from slices of [row - h, row + 15]."""
    n = len(cols[0])
    f, t = [], []
    runs = np.split(rows, np.flatnonzero(np.diff(rows) != 1) + 1)
    for run in runs:
        lo, hi = max(0, run[0] - h), min(n, run[-1] + 16)
        rf, rt = oracle([x[lo:hi] for x in cols], kw)
        f.append(rf[run - lo])
        t.append(rt[run - lo])
    return np.concatenate(f), np.concatenate(t)


@pytest.mark.gpu
def test_two_million_rows_strided_sample():
    """Eight grid-stride passes: 64-row runs every 25,000 rows, the tile boundaries past each pass and the last tile,
    against the oracle on slices that hold each run's frames and leads."""
    n = 2_000_000
    cols = tick_table(n, seed=3)
    got, tgt = gpu(cols, DEFAULT)
    starts = list(range(19, n - 64, 25_000)) + [k * PASS - 32 for k in range(1, n // PASS + 1)] + [n - 300]
    rows = np.unique(np.concatenate([np.arange(s, min(n, s + 64)) for s in starts] + [np.arange(n - 256, n)]))
    ref, ref_t = _oracle_rows(cols, DEFAULT, rows, halo_of(DEFAULT))
    check_columns(cols, DEFAULT, got[rows], ref, rows=rows)
    check_labels(tgt[rows], ref_t)


@pytest.mark.gpu
def test_period_4097_is_refused():
    from financial_market_data_analysis_b200.features import window_features
    x = torch.ones(5000, device="cuda")
    with pytest.raises(ValueError, match=r"code -4"):
        window_features(x, x, x, x, x, volume_MA_periods=[4097])
    with pytest.raises(ValueError, match=r"code -4"):
        window_features(x, x, x, x, x, bollinger_bands_period=4097)
