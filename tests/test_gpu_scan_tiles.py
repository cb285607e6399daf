"""Scan geometry: at bf16x3 a cluster of the tensor-core forward scan takes one or two 16-row batch tiles, and the backward
scan runs a short last round of 16-row tiles as 8-row clusters.  Both follow from how many clusters the device holds at
once (bigru_scan_geometry reports the numbers).

1. The rules, with n = D*B/16 tiles and R resident clusters.  Forward: rounds = ceil(n / 2R) and n2 = n - rounds*R
   clusters (rounded up to a multiple of D) take two tiles; n <= R gives none, and so does bf16 at any n.  Backward:
   rounds = ceil(n / R), and the L = n - (rounds-1)*R tiles of the last round are split when rounds > 1 and 2L <= R.
2. No bit depends on the geometry.  At shapes read off R, one with two-tile and one-tile clusters mixed and one with only
   two-tile clusters, with and without an initial state, reversing the batch moves rows between kinds of clusters (and a
   small batch runs every row in a one-tile cluster).  Per row, the forward's Y, G, Y planes and h_n, the logits and the
   backward's dgi, dgh, their planes and dh_{-1} must be bitwise equal.
3. Lengths and infer at the mixed shapes: infer is bitwise the eval-mode forward, and reversing the batch changes no bit of
   any row's logits, at T = 1 and T = 5."""
import ctypes as C

import numpy as np
import pytest
import torch

from gru_driver import CODE, abi_names, kernel


def _pkg():
    import financial_market_data_analysis_b200 as pkg
    return pkg


def _geometry(prec, B, H, D, scan=0, T=2, F=16, L=1, C_=3):
    """(R, n_split) of bigru_scan_geometry for a plan of this shape; scan 0 forward, 1 backward."""
    pkg = _pkg()
    lib = pkg._lib.load()
    plan = C.c_void_p()
    pkg._lib.check(lib.bigru_plan_create(B, T, F, H, L, C_, int(D == 2), CODE[prec], C.byref(plan)), "plan_create")
    try:
        R, n2 = C.c_int(), C.c_int()
        pkg._lib.check(lib.bigru_scan_geometry(plan, scan, C.byref(R), C.byref(n2)), "scan_geometry")
        return R.value, n2.value
    finally:
        lib.bigru_plan_destroy(plan)


def _rule(R, n, D):
    rounds = -(-n // (2 * R))
    n2 = max(0, n - rounds * R)
    return min(-(-n2 // D) * D, D * (n // D // 2))


def _bwd_rule(R, n):
    rounds = -(-n // R)
    L = n - (rounds - 1) * R
    return L if rounds > 1 and 2 * L <= R else 0


def _batch(H, D, kind, prec="bf16x3"):
    """A batch whose forward scan has two-tile and one-tile clusters ("mixed") or only two-tile clusters ("two"), or whose
    backward scan splits the tiles of its last round ("split")."""
    if kind == "split":
        R, _ = _geometry(prec, 32, H, D, 1)
        n = (2 * R // (2 * D) + 1) * 2 * D          # just above two full rounds (B % 32 == 0)
        B = 16 * n // D
        R2, L8 = _geometry(prec, B, H, D, 1)
        assert R2 == R and 0 < L8 == n - 2 * R, (R, n, L8)
        return B
    R, _ = _geometry(prec, 32, H, D)
    if kind == "mixed":
        n = (R // (2 * D) + 1) * 2 * D             # the least multiple of 2D above R (B % 32 == 0)
    else:
        n = 2 * R // (2 * D) * (2 * D)             # the most tiles that one round of two-tile clusters holds
    B = 16 * n // D
    R2, n2 = _geometry(prec, B, H, D)
    assert R2 == R
    if kind == "mixed":
        assert 0 < n2 < n - n2, (R, n, n2)
    else:
        assert 2 * n2 == n, (R, n, n2)
    return B


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ("bf16x3", "bf16"))
@pytest.mark.parametrize("H", (128, 256, 512))
@pytest.mark.parametrize("D", (1, 2))
def test_geometry_follows_residency(prec, H, D):
    if H == 512 and prec == "bf16x3":
        pytest.skip("hidden 512 runs at bf16 only")
    R, n2 = _geometry(prec, 32, H, D)
    assert R >= 1 and n2 == 0
    for n in sorted({D, R // D * D, (R // D + 1) * D, 2 * R // D * D, (2 * R // D + 1) * D, 3 * R // D * D}):
        if n < D:
            continue
        B = 16 * n // D
        if (H == 512 or prec == "bf16x3") and B % 32:
            continue
        R2, n2 = _geometry(prec, B, H, D)
        assert R2 == R
        assert n2 == (0 if prec == "bf16" else _rule(R, n, D)), (n, R, n2)
        assert n2 % D == 0 and 0 <= n2 <= n // 2


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ("bf16x3", "bf16"))
@pytest.mark.parametrize("H", (128, 256, 512))
@pytest.mark.parametrize("D", (1, 2))
def test_backward_geometry_follows_residency(prec, H, D):
    if H == 512 and prec == "bf16x3":
        pytest.skip("hidden 512 runs at bf16 only")
    R, L8 = _geometry(prec, 32, H, D, 1)
    assert R >= 1 and L8 == 0
    for n in sorted({D, R // D * D, (R // D + 1) * D, (2 * R // D + 1) * D, (3 * R // D - 1) * D, 5 * R // (2 * D) * D}):
        B = 16 * n // D
        if n < D or ((H == 512 or prec == "bf16x3") and B % 32):
            continue
        R2, L8 = _geometry(prec, B, H, D, 1)
        assert R2 == R
        assert L8 == _bwd_rule(R, n), (n, R, L8)


def _per_row(out, perm):
    """Every per-row tensor of a kernel() result with regions, batch rows reordered by perm."""
    ws = out["ws"]
    r = dict(logits=out["logits"][perm], hn=out["hn"][:, perm], dhc=ws["DHC"][:, perm])
    for l, y in enumerate(out["ys"]):
        r[f"y{l}"] = y[perm]
        r[f"g{l}"] = ws["G"][l][:, perm]
        r[f"yp{l}"] = [None if p is None else p[perm] for p in ws["YP"][l]]
    for k in ("DGI", "DGH"):
        r[k] = ws[k][:, perm]
    for k in ("DGIP", "DGHP"):
        r[k] = [None if p is None else p[:, perm] for p in ws[k]]
    return r


def _assert_bitwise(a, b, what):
    for k in a:
        for i, (x, y) in enumerate(zip(*((v if isinstance(v, list) else [v]) for v in (a[k], b[k])))):
            if x is None:
                assert y is None
                continue
            assert np.array_equal(np.asarray(x), np.asarray(y)), f"{what}: {k}[{i}] differs"


@pytest.mark.gpu
@pytest.mark.parametrize("H", (128, 256))
@pytest.mark.parametrize("D", (1, 2))
@pytest.mark.parametrize("kind", ("mixed", "two", "split"))
@pytest.mark.parametrize("prec,h0", (("bf16x3", False), ("bf16x3", True), ("bf16", False)))
def test_rows_do_not_depend_on_the_tile(H, D, kind, prec, h0):
    if prec == "bf16" and kind != "split":
        pytest.skip("bf16 forward clusters take one tile")
    B = _batch(H, D, kind, prec)
    s = dict(B=B, T=2, F=16, H=H, L=2, C=3, D=D, h0=h0)
    rng = np.random.default_rng(7)
    n = sum(v[1] for v in abi_names(s).values())
    flat = (rng.standard_normal(n) * 0.08).astype(np.float32)
    x = rng.standard_normal((B, s["T"], s["F"])).astype(np.float32)
    h0 = (rng.standard_normal((s["L"] * D, B, H)) * 0.5).astype(np.float32) if s["h0"] else None
    dl = rng.standard_normal((B, s["C"])).astype(np.float32)
    base, _ = kernel(s, prec, flat, x, h0, dl, regions=True)
    want = _per_row(base, np.arange(B))
    rev = np.arange(B)[::-1].copy()
    got, _ = kernel(s, prec, flat, np.ascontiguousarray(x[rev]), None if h0 is None else np.ascontiguousarray(h0[:, rev]),
                    np.ascontiguousarray(dl[rev]), regions=True)
    _assert_bitwise(want, _per_row(got, rev), "reversed batch")
    # the first 64 rows as a batch of their own: every cluster takes one 16-row tile
    bs = 64
    assert _geometry(prec, bs, H, D)[1] == 0 and _geometry(prec, bs, H, D, 1)[1] == 0
    ss = dict(s, B=bs)
    small, _ = kernel(ss, prec, flat, np.ascontiguousarray(x[:bs]), None if h0 is None else np.ascontiguousarray(h0[:, :bs]),
                      np.ascontiguousarray(dl[:bs]), regions=True)
    _assert_bitwise(_per_row(base, np.arange(bs)), _per_row(small, np.arange(bs)), "one-tile batch")


@pytest.mark.gpu
@pytest.mark.parametrize("H", (128, 256))
@pytest.mark.parametrize("T", (1, 5))
def test_lengths_and_infer_at_mixed_tiles(H, T):
    prec, D, F, C_, L = "bf16x3", 2, 16, 3, 2
    B = _batch(H, D, "mixed")
    torch.manual_seed(3)
    m = _pkg().BiGRU(H, F, C_, L, 50, 0.0, False, True, precision=prec).cuda().eval()
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, T, F, generator=g).cuda()
    lens = torch.randint(1, T + 1, (B,), generator=g)
    lens[0] = T
    rev = torch.arange(B - 1, -1, -1)
    with torch.no_grad():
        for ln in (None, lens):
            y = m(x, lengths=ln)
            yi = m.infer(x, lengths=ln)
            yr = m(x[rev.cuda()], lengths=None if ln is None else ln[rev])
            torch.cuda.synchronize()
            assert torch.equal(y, yi)
            assert torch.equal(y, yr[rev.cuda()])
