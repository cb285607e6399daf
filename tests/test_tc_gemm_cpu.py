"""Host-side checks of tests/test_gpu_tc_gemm.py and of bigru_tc_gemm: the exact-operand generator (its split is exact, its
partial sums stay below the bound, fp32 sums of its products in any order are the fp64 sum), the plans' output jobs
that file relies on being staged, and the argument checks bigru_tc_gemm makes before it touches the device."""
import ctypes as C

import numpy as np
import pytest

from gru_driver import CODE, split
from test_gpu_tc_gemm import (JOBS, LIMIT, PAD, PLAN, UNIT, exact_bound, exact_parts, job, n_splits, operands, staged)
from test_gpu_tc_steps import cdiv, wg_splits, wg_staged


@pytest.mark.parametrize("name", list(JOBS))
def test_exact_operands(name):
    j = JOBS[name]
    ops = operands(j, "exact")
    assert exact_bound(ops, j) < LIMIT
    rng = np.random.default_rng(7)
    for key in ("a", "b"):
        v = ops[key]
        hi, lo = exact_parts(v)
        # hi an integer in [-3, 3]; lo = q * 2^-11 with |q| <= 3, 0 where hi is 0; both parts take part
        assert np.abs(hi).max() <= 3 and np.array_equal(lo / UNIT, np.round(lo / UNIT)) and np.abs(lo).max() <= 3 * UNIT
        assert not lo[hi == 0].any() and lo.any() and hi.any()
        # split_bf16 gives back the parts, at both precisions
        sh, sl = split(v, "bf16x3")
        assert np.array_equal(sh, hi) and np.array_equal(sl, lo)
        assert np.array_equal(split(v, "bf16")[0], hi)
    # fp32 sums of one output's products (the three bf16x3 terms per k, the bias, beta's C) in random orders: every
    # partial sum is the fp64 one
    for _ in range(4):
        z, m, n = (int(rng.integers(0, s)) for s in (j["batch"], j["M"], j["N"]))
        ah, al = exact_parts(ops["a"][z, m].astype(np.float64))
        bh, bl = exact_parts(ops["b"][z, n].astype(np.float64))
        terms = [ah * bh, ah * bl, al * bh]
        if ops["bias"] is not None:
            terms.append(ops["bias"][z * j["zbias"] + n: z * j["zbias"] + n + 1].astype(np.float64))
        if ops["c0"] is not None:
            terms.append(ops["c0"][z, m, n: n + 1].astype(np.float64))
        t = np.concatenate(terms)
        t = t[t != 0]
        for _ in range(3):
            p = rng.permutation(t)
            assert np.array_equal(np.cumsum(p.astype(np.float32), dtype=np.float32).astype(np.float64), np.cumsum(p))


def test_plan_output_jobs_are_staged_when_aligned():
    """The end-to-end check of test_gpu_tc_gemm.py compares each output of its plan aligned and one float off.  That
    compares the staged with the direct epilogue only if every output job is staged when aligned: restate the jobs."""
    B, T, F, H, L, C_, D = (PLAN[k] for k in "BTFHLCD")
    BT, H3 = B * T, 3 * H
    I = [F] + [D * H] * (L - 1)
    ld_block = [H3 * i + H3 * H + 2 * H3 for i in I]
    off_wih = [sum(D * b for b in ld_block[:l]) for l in range(L)]
    jobs = [("logits", B, C_, 1, 0, C_, B * C_), ("dx", BT, F, 1, 0, F, BT * F),
            ("dlin_w", C_, H3, 1, off_wih[-1] + D * ld_block[-1], H3, C_ * H3)]
    for l in range(L):
        jobs.append((f"dW_ih[{l}]", H3, I[l], D, off_wih[l], I[l], ld_block[l]))
        jobs.append((f"dW_hh[{l}]", H3, H, D, off_wih[l] + H3 * I[l], H, ld_block[l]))
    for name, M, N, batch, base, ldc, zc in jobs:
        if name.startswith("dW"):
            assert wg_splits(cdiv(M, 128) * cdiv(N, 128) * batch, cdiv(BT, 64)) == 1, name
        assert wg_staged(1, 0, 4 * (PAD + base), ldc, zc if batch > 1 else M * ldc, N) == 1, name
        assert wg_staged(1, 0, 4 * (PAD + 1 + base), ldc, zc if batch > 1 else M * ldc, N) == 0, name


def test_staging_rule_of_the_jobs():
    """Split jobs write their partials: C's alignment does not change their epilogue; N = 13 partials are direct."""
    assert staged(JOBS["split8_beta_batch"], 0) == staged(JOBS["split8_beta_batch"], 1) == 1
    assert staged(JOBS["split_n13"], 0) == staged(JOBS["split_n13"], 1) == 0
    assert staged(JOBS["n12_pitch16_gaps"], 0) == 1 and staged(JOBS["n12_pitch16_gaps"], 1) == 0
    # N = 13 at pitch 16: aligned, but the rows end inside a 16-byte chunk
    assert staged(JOBS["n13_pitch16"], 0) == 0
    assert staged(JOBS["beta_bias"], 0) == 0


# ---- bigru_tc_gemm's argument checks, before the device --------------------------------------------------------------
def _lib():
    import financial_market_data_analysis_b200 as pkg
    return pkg._lib


def _ws_floats(prec, mn, M, N, K, batch, splits):
    """The workspace layout of api.cu restated (floats): A's planes, B's planes (offsets rounded to 64 floats), partials."""
    x = 2 if prec == "bf16x3" else 1
    r = lambda v, m: -(-v // m) * m                                             # noqa: E731
    planes = (lambda rows: r(x * batch * K * r(rows, 8), 128) // 2) if mn else \
        (lambda rows: r(x * batch * r(rows, 128) * r(K, 64), 128) // 2)
    return planes(M) + planes(N) + (splits * batch * M * N if splits > 1 else 0)


@pytest.mark.parametrize("prec", ["bf16", "bf16x3"])
@pytest.mark.parametrize("mn", [0, 1])
def test_workspace_bytes(prec, mn):
    lib = _lib().load()
    nb = C.c_size_t()
    for M, N, K, batch, splits in ((1, 4, 1, 1, 0), (200, 13, 100, 3, 0), (768, 256, 65536, 2, 0), (384, 256, 4160, 2, 8),
                                   (150, 13, 1100, 1, 0)):
        s = splits or wg_splits(cdiv(M, 128) * cdiv(N, 128) * batch, cdiv(K, 64))
        assert lib.bigru_tc_gemm_workspace_bytes(CODE[prec], mn, M, N, K, batch, splits, C.byref(nb)) == 0
        assert nb.value == 4 * _ws_floats(prec, mn, M, N, K, batch, s), (M, N, K, batch, splits)


def test_argument_checks():
    """Every refusal happens before any device work (no pointer below is dereferenced)."""
    L_ = _lib()
    lib = L_.load()
    p = C.c_void_p(4096)                       # never dereferenced: each call below is refused first
    st = C.c_int(-1)

    def call(prec=1, mn=0, M=256, N=128, K=640, batch=2, a=p, b=p, bias=None, zbias=0, c=p, ldc=128, zc=256 * 128,
             beta=0, splits=0, ws=p, staged=C.byref(st)):
        return lib.bigru_tc_gemm(prec, mn, M, N, K, batch, a, b, bias, zbias, c, ldc, zc, beta, splits, ws, staged, None)

    refused = [dict(prec=0), dict(prec=3), dict(mn=2), dict(M=0), dict(N=0), dict(K=0), dict(batch=0), dict(splits=-1),
               dict(a=None), dict(b=None), dict(c=None), dict(ws=None), dict(staged=None),
               dict(ldc=127), dict(zc=255 * 128 + 127), dict(bias=p, zbias=-1),
               dict(splits=6), dict(splits=11),                         # 10 k-blocks: 6 or 11 splits leave one empty
               dict(bias=p, splits=2), dict(bias=p, K=4096)]            # a bias with split-K, forced or from wg_splits
    assert n_splits(job(256, 128, 4096, batch=2)) > 1
    for kw in refused:
        st.value = -1
        assert call(**kw) == L_.ERR_ARG, kw
        assert lib.bigru_last_error(), kw
        assert st.value == -1, kw
    nb = C.c_size_t()
    assert lib.bigru_tc_gemm_workspace_bytes(1, 0, 256, 128, 640, 1, 6, C.byref(nb)) == L_.ERR_ARG
    assert lib.bigru_tc_gemm_workspace_bytes(0, 0, 256, 128, 640, 1, 0, C.byref(nb)) == L_.ERR_ARG
    assert lib.bigru_tc_gemm_workspace_bytes(1, 0, 256, 128, 640, 1, 0, None) == L_.ERR_ARG
