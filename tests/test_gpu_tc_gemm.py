"""The tensor-core GEMM (wg_gemm_kernel, tc_hopper.cuh) one job at a time, through bigru_tc_gemm: the same wg_gemm host code
the plans run, on operands, output pitches and alignments the plans never produce.

A job that overwrites a 16-byte-aligned output goes out through shared memory and bulk tensor stores (the staged epilogue,
clipped by TMA at the map's bounds); every other job stores element by element (the direct epilogue).  The plans reach
both only at the shapes their B, H and T rules make, always with ldc == N, so a map with the wrong column extent or batch
stride, a box written to the wrong place or a dropped partial box could pass them.  Here every job of JOBS runs at bf16
and bf16x3, with K-major and MN-major operands (the four instantiations of wg_gemm_kernel), and
  1. staged against direct, bitwise: the same job with C 16-byte aligned, then one float off.  *staged must follow
     wg_staged (test_gpu_tc_steps.py, the library's rule restated), and both whole buffers, with NaN canaries in the gaps
     between rows and batches and on both sides, must be equal bit for bit, the canaries untouched;
  2. exact jobs: operands whose bf16 split is exact (hi an integer, lo a multiple of 2^-11) and whose products and
     partial sums are integer multiples of 2^-11 below 2^20 of them, so that every summation order, every split and the
     split-K reduction give the fp64 result bit for bit: C must equal pmm(split(A), split(B)^T) + bias (+ C) exactly;
  3. random fp32 operands against that fp64 rounding model (class gemm_job), within TOL.
Jobs too large to model whole are modelled on three row tiles (the first, a middle one, the last); checks 1 and the
canaries always cover the whole buffer.  The plans' own output jobs are checked the same way end to end: their logits,
dx and grads, written 16-byte aligned and one float off, must be bitwise equal.
Run on an H100:  python -m pytest tests/test_gpu_tc_gemm.py -m gpu -q
(BIGRU_TC_GEMM_REPORT=path.jsonl appends every measured distance to that file.)  Measurements and mutations:
tests/ROUNDING_MODEL.md, section "One GEMM job at a time"."""
import ctypes as C
import json
import os
import resource

import numpy as np
import pytest

from gru_driver import CODE, dist, pmm, split, tr
from test_gpu_tc_steps import NSM, cdiv, wg_splits, wg_staged

PAD = 8                    # canary floats before and after every output buffer
CANARY = 0x7FC5A3E1        # a quiet NaN whose payload no arithmetic produces
UNIT = 2.0 ** -11          # the exact jobs' unit: lo parts are multiples of it, hi parts integers (2048 units)
LIMIT = 2 ** 20            # bound, in units, on every partial sum of an exact job (with its bias and beta's C)


def job(M, N, K, batch=1, ldc=None, zc=None, beta=False, bias=False, zbias=None, splits=0, sample=False, regimes=()):
    """A bigru_tc_gemm job.  ldc / zc: C's row pitch and batch stride (N, M * ldc by default); zbias: the bias's batch
    stride; splits: forced split count (0: wg_splits); sample: model three row tiles only."""
    ldc = N if ldc is None else ldc
    return dict(M=M, N=N, K=K, batch=batch, ldc=ldc, zc=M * ldc if zc is None else zc, beta=beta, bias=bias,
                zbias=N if zbias is None else zbias, splits=splits, sample=sample, regimes=regimes)


def n_splits(j):
    return j["splits"] or wg_splits(cdiv(j["M"], 128) * cdiv(j["N"], 128) * j["batch"], cdiv(j["K"], 64))


def units(j):
    """(tile, split) units of the persistent kernel: at most NSM CTAs stride over them."""
    return cdiv(j["M"], 128) * cdiv(j["N"], 128) * j["batch"] * n_splits(j)


def short_last_split(j):
    kb, s = cdiv(j["K"], 64), n_splits(j)
    return s > 1 and kb % cdiv(kb, s) != 0


def staged(j, off):
    """The epilogue of job j with C at PAD + off floats past a 16-byte-aligned allocation.  With splits > 1 the kernel
    writes the partials, which the workspace keeps 16-byte aligned at pitch N: C's alignment does not matter then."""
    s = n_splits(j)
    if s > 1:
        return wg_staged(s, j["beta"], 0, j["N"], j["M"] * j["N"], j["N"])
    return wg_staged(1, j["beta"], 4 * (PAD + off), j["ldc"], j["zc"] if j["batch"] > 1 else j["M"] * j["ldc"], j["N"])


def direct_because(j):
    """Why the aligned run of a one-split job stores element by element (None: it is staged)."""
    if n_splits(j) > 1 or staged(j, 0):
        return None
    return "beta" if j["beta"] else "ldc" if j["ldc"] % 4 else "N" if j["N"] % 4 else "zc"


# the regimes where the epilogues go wrong, and how a job proves it is in one
REGIMES = {
    # epilogue: staged, and direct for each of its reasons (the base one float off is every staged one-split job's second run)
    "staged": lambda j: staged(j, 0) == 1,
    "direct_beta": lambda j: direct_because(j) == "beta",
    "direct_base_off_by_one": lambda j: n_splits(j) == 1 and staged(j, 0) == 1 and staged(j, 1) == 0,
    "direct_odd_ldc": lambda j: direct_because(j) == "ldc",
    "direct_odd_zc": lambda j: direct_because(j) == "zc" and j["batch"] > 1 and j["zc"] % 4 != 0,
    # a row ending inside a 16-byte chunk at an aligned pitch: the bulk store would overrun it into the gap
    "direct_n_mod4": lambda j: direct_because(j) == "N" and j["ldc"] > j["N"],
    "direct_split_n_mod4": lambda j: n_splits(j) > 1 and j["N"] % 4 != 0 and staged(j, 0) == 0,
    # columns: one partial box (boxes 1-3 skipped), a ragged last box, whole tiles, a ragged last n-tile, N = 4
    "N_lt_32": lambda j: j["N"] < 32 and staged(j, 0) == 1,
    "N_ragged_box": lambda j: j["N"] % 32 != 0 and j["N"] % 4 == 0 and j["N"] > 32,
    "N_mult_128": lambda j: j["N"] % 128 == 0,
    "N_gt_128_ragged_tile": lambda j: j["N"] > 128 and j["N"] % 128 != 0,
    "N_4": lambda j: j["N"] == 4,
    # rows: one row; the second warpgroup's rows wholly outside the map; partly outside; whole tiles
    "M_1": lambda j: j["M"] == 1,
    "M_wg1_outside": lambda j: 0 < j["M"] % 128 <= 64 and staged(j, 0) == 1,
    "M_wg1_partial": lambda j: 64 < j["M"] % 128 < 128,
    "M_mult_128": lambda j: j["M"] % 128 == 0,
    # gaps between rows and between batches, where canaries sit
    "gaps": lambda j: j["ldc"] > j["N"] and j["batch"] > 1 and j["zc"] > j["M"] * j["ldc"],
    "gaps_staged": lambda j: j["ldc"] > j["N"] and j["batch"] > 1 and j["zc"] > j["M"] * j["ldc"] and staged(j, 0) == 1,
    # batches and splits: the partials' index s * batch + zb
    "batch_gt_1": lambda j: j["batch"] > 1,
    "split_staged": lambda j: n_splits(j) > 1 and staged(j, 0) == 1,
    "split_direct": lambda j: n_splits(j) > 1 and staged(j, 0) == 0,
    "split_short_last": short_last_split,
    "split_batch": lambda j: n_splits(j) > 1 and j["batch"] > 1,
    "split_beta": lambda j: n_splits(j) > 1 and j["beta"],
    # staging-slot reuse: a CTA's next unit rewrites the slots its last stores read (four per warpgroup at bf16, two at
    # bf16x3, so already within a unit there); at least three units per CTA
    "units_gt_sms": lambda j: units(j) > NSM and staged(j, 0) == 1,
    "units_3_per_cta": lambda j: units(j) >= 3 * NSM and staged(j, 0) == 1,
    # K: one element, ragged against the 64-deep k-block, configs[1]'s dW_hh depth
    "K_1": lambda j: j["K"] == 1,
    "K_ragged_64": lambda j: j["K"] % 64 != 0,
    "K_65536": lambda j: j["K"] == 65536,
    # bias
    "bias": lambda j: j["bias"] and not j["beta"],
    "no_bias": lambda j: not j["bias"],
    "beta_bias": lambda j: j["bias"] and j["beta"],
}

JOBS = {
    "m1_n4_k1": job(1, 4, 1, bias=True, regimes=("staged", "direct_base_off_by_one", "N_lt_32", "N_4", "M_1",
                                                  "M_wg1_outside", "K_1", "K_ragged_64", "bias")),
    "n12_pitch16_gaps": job(200, 12, 100, batch=3, ldc=16, zc=200 * 16 + 20, bias=True, zbias=12,
                            regimes=("staged", "direct_base_off_by_one", "N_lt_32", "M_wg1_partial", "gaps", "gaps_staged",
                                     "batch_gt_1", "K_ragged_64", "bias")),
    "n13_pitch16": job(70, 13, 64, batch=2, ldc=16, zc=70 * 16 + 4, bias=True, zbias=16,
                       regimes=("direct_n_mod4", "M_wg1_partial", "gaps", "batch_gt_1", "bias")),
    "odd_ldc": job(130, 40, 64, batch=2, ldc=41, zc=130 * 41 + 3,
                   regimes=("direct_odd_ldc", "N_ragged_box", "gaps", "batch_gt_1", "no_bias")),
    "odd_zc": job(64, 84, 200, batch=2, ldc=88, zc=64 * 88 + 2, bias=True, zbias=88,
                  regimes=("direct_odd_zc", "N_ragged_box", "gaps", "K_ragged_64", "bias")),
    "beta_bias": job(256, 256, 192, batch=2, beta=True, bias=True, zbias=256,
                     regimes=("direct_beta", "N_mult_128", "M_mult_128", "beta_bias", "batch_gt_1")),
    "wide_ragged": job(300, 300, 257, ldc=304,
                       regimes=("staged", "direct_base_off_by_one", "N_ragged_box", "N_gt_128_ragged_tile", "M_wg1_outside",
                                "K_ragged_64", "no_bias")),
    "split8_beta_batch": job(384, 256, 4160, batch=2, beta=True, splits=8,
                             regimes=("split_staged", "split_short_last", "split_batch", "split_beta", "N_mult_128",
                                      "M_mult_128", "no_bias")),
    "split_n13": job(150, 13, 1100, regimes=("split_direct", "direct_split_n_mod4", "no_bias")),
    "slots_gaps": job(640, 512, 64, batch=20, ldc=516, zc=640 * 516 + 8, bias=True, zbias=512, sample=True,
                      regimes=("staged", "direct_base_off_by_one", "units_gt_sms", "units_3_per_cta", "gaps", "gaps_staged",
                               "N_mult_128", "M_mult_128", "bias")),
    "k65536": job(768, 256, 65536, batch=2, sample=True,
                  regimes=("split_staged", "split_short_last", "split_batch", "units_gt_sms", "units_3_per_cta", "K_65536",
                           "no_bias")),
}

# Kernel-vs-model tolerances of gemm_job (rel-L2, max-abs over max |model|): about 4x the worst value measured on an
# H100 80GB HBM3 (SXM, 700 W power limit) over JOBS; the measurements are in tests/ROUNDING_MODEL.md.
TOL = {"bf16": (1.3e-5, 1.4e-5), "bf16x3": (4e-5, 4.2e-5)}


def test_jobs_are_in_the_regimes_they_claim():
    covered = set()
    for name, j in JOBS.items():
        for r in j["regimes"]:
            assert REGIMES[r](j), (name, r)
        covered |= set(j["regimes"])
        # the library's own argument rules: rows and batches do not overlap, and no bias with split-K
        assert j["ldc"] >= j["N"] and (j["batch"] == 1 or j["zc"] >= (j["M"] - 1) * j["ldc"] + j["N"]), name
        assert not (j["bias"] and n_splits(j) > 1), name
    assert covered == set(REGIMES), set(REGIMES) - covered
    # the split counts the regimes rest on: 8 forced (65 k-blocks, 9 per split, 2 in the last); configs[1]'s dW_hh rule
    assert n_splits(JOBS["split8_beta_batch"]) == 8 and n_splits(JOBS["split_n13"]) == 2
    assert n_splits(JOBS["k65536"]) == 22 and units(JOBS["k65536"]) == 528


# ---- operands -------------------------------------------------------------------------------------------------------
def exact_operand(rng, shape, density):
    """fp32 values hi + lo: hi an integer in [-3, 3], nonzero with probability `density`; lo = q * 2^-11, q in [-3, 3],
    and 0 where hi is 0.  |lo| < 2^-9, less than half a bf16 ulp on either side of any nonzero hi (just below |hi| = 1 the
    ulp is 2^-8), so split_bf16 gives back (hi, lo) exactly."""
    hi = rng.integers(-3, 4, shape, dtype=np.int8).astype(np.float32)
    hi *= rng.random(shape, dtype=np.float32) < density
    lo = rng.integers(-3, 4, shape, dtype=np.int8).astype(np.float32) * np.float32(UNIT)
    lo *= hi != 0
    return hi + lo


def exact_parts(v):
    """The (hi, lo) an exact operand was built from: the nearest integer and the rest."""
    hi = np.round(v)
    return hi, v - hi


def bias_len(j):
    return (j["batch"] - 1) * j["zbias"] + j["N"]


def exact_bound(ops, j):
    """Largest sum, over one output, of |hi_a hi_b| + |hi_a lo_b| + |lo_a hi_b| + |bias| + |C|, in units: it bounds every
    partial sum in every order."""
    def mag(v):
        hi, lo = exact_parts(v.astype(np.float64))
        return np.abs(hi) + np.abs(lo)
    s = np.matmul(mag(ops["a"]), mag(ops["b"]).transpose(0, 2, 1))
    if ops["bias"] is not None:
        s += np.stack([np.abs(ops["bias"][z * j["zbias"]: z * j["zbias"] + j["N"]]) for z in range(j["batch"])])[:, None, :]
    if ops["c0"] is not None:
        s += np.abs(ops["c0"])
    return s.max() / UNIT


def operands(j, kind, seed=0):
    """A [batch][M][K], B [batch][N][K], bias, and C's prior values (beta), float32.  exact: exact_operand at a density
    that keeps the partial sums below LIMIT units (lowered until exact_bound says so), bias and C integers plus multiples
    of 2^-11; random: standard normal."""
    M, N, K, b = j["M"], j["N"], j["K"], j["batch"]
    rng = np.random.default_rng([seed, M, N, K, b, kind == "exact"])
    if kind == "random":
        f = lambda *s: rng.standard_normal(s, dtype=np.float32)                 # noqa: E731
        return dict(a=f(b, M, K), b=f(b, N, K), bias=f(bias_len(j)) if j["bias"] else None,
                    c0=f(b, M, N) if j["beta"] else None)
    small = lambda *s: (rng.integers(-20, 21, s) + rng.integers(-3, 4, s) * UNIT).astype(np.float32)   # noqa: E731
    density = min(1.0, float(np.sqrt(60.0 / K)))
    while True:
        ops = dict(a=exact_operand(rng, (b, M, K), density), b=exact_operand(rng, (b, N, K), density),
                   bias=small(bias_len(j)) if j["bias"] else None, c0=small(b, M, N) if j["beta"] else None)
        if exact_bound(ops, j) < LIMIT:
            return ops
        density *= 0.8


def model_rows(j):
    """Rows the model computes: all, or for a sampled job the first, a middle and the last 128-row tile."""
    M = j["M"]
    if not j["sample"]:
        return np.arange(M)
    tm = cdiv(M, 128)
    return np.concatenate([np.arange(t * 128, min(M, t * 128 + 128)) for t in sorted({0, tm // 2, tm - 1})])


def model(j, ops, prec, rows):
    """C [batch][rows][N] in float64: pmm of the operands split as the kernels split them (prec "exact": unsplit), plus
    the bias and, for beta, C's prior values."""
    out = np.empty((j["batch"], len(rows), j["N"]))
    for z in range(j["batch"]):
        out[z] = pmm(split(ops["a"][z][rows], prec), tr(split(ops["b"][z], prec)))
        if ops["bias"] is not None:
            out[z] += ops["bias"][z * j["zbias"]: z * j["zbias"] + j["N"]].astype(np.float64)
        if ops["c0"] is not None:
            out[z] += ops["c0"][z][rows].astype(np.float64)
    return out


def c_index(j):
    """Positions of C's elements [batch][M][N] in the canaried buffer, and the buffer's length."""
    z, m, n = np.ix_(np.arange(j["batch"]), np.arange(j["M"]), np.arange(j["N"]))
    idx = PAD + z * j["zc"] + m * j["ldc"] + n
    span = (j["batch"] - 1) * j["zc"] + (j["M"] - 1) * j["ldc"] + j["N"]
    return idx, span + 2 * PAD


# ---- the library --------------------------------------------------------------------------------------------------
def _lib():
    import financial_market_data_analysis_b200 as pkg
    return pkg._lib


def tc_gemm(prec, mn, j, a, b, bias, c, ws):
    """bigru_tc_gemm on device pointers (ints or None) for job j; returns (rc, *staged)."""
    import torch
    st = C.c_int(-1)
    rc = _lib().load().bigru_tc_gemm(CODE[prec], int(mn), j["M"], j["N"], j["K"], j["batch"], a, b, bias, j["zbias"], c,
                                     j["ldc"], j["zc"], int(j["beta"]), j["splits"], ws, C.byref(st),
                                     C.c_void_p(torch.cuda.current_stream().cuda_stream))
    return rc, st.value


def run_job(j, prec, mn, ops):
    """The job with C 16-byte aligned (off 0) and one float off (off 1), each in a canaried buffer.  Returns
    [(staged, int32 bits of the whole buffer)] for the two runs."""
    import torch
    L_ = _lib()
    lib = L_.load()
    dev = torch.device("cuda")
    a = ops["a"] if not mn else np.ascontiguousarray(ops["a"].transpose(0, 2, 1))
    b = ops["b"] if not mn else np.ascontiguousarray(ops["b"].transpose(0, 2, 1))
    ad, bd = torch.from_numpy(a).to(dev), torch.from_numpy(b).to(dev)
    del a, b
    biasd = None if ops["bias"] is None else torch.from_numpy(ops["bias"]).to(dev)
    nb = C.c_size_t()
    L_.check(lib.bigru_tc_gemm_workspace_bytes(CODE[prec], int(mn), j["M"], j["N"], j["K"], j["batch"], j["splits"],
                                               C.byref(nb)), "tc_gemm_workspace_bytes")
    ws = torch.empty(max(nb.value, 16) // 4, dtype=torch.float32, device=dev)
    idx, n = c_index(j)
    init = np.full(n, CANARY, np.int32)
    if ops["c0"] is not None:
        init[idx] = ops["c0"].view(np.int32)
    out = []
    for off in (0, 1):
        buf = torch.empty(n + 1, dtype=torch.int32, device=dev)
        assert buf.data_ptr() % 16 == 0
        view = buf[off:off + n]
        view.copy_(torch.from_numpy(init))
        rc, st = tc_gemm(prec, mn, j, ad.data_ptr(), bd.data_ptr(), None if biasd is None else biasd.data_ptr(),
                         view.data_ptr() + 4 * PAD, ws.data_ptr())
        L_.check(rc, "tc_gemm")
        torch.cuda.synchronize()
        out.append((st, view.cpu().numpy()))
    return out


_CACHE = {}


def _cached(name, key, make):
    """Operands and models of one job, kept while the parameters of that job run (JOB_CASES is job-major)."""
    if _CACHE.get("job") != name:
        _CACHE.clear()
        _CACHE["job"] = name
    if key not in _CACHE:
        _CACHE[key] = make()
    return _CACHE[key]


JOB_CASES = [(n, p, mn) for n in JOBS for p in ("bf16", "bf16x3") for mn in (0, 1)]


def _need_gpu():
    lib = _lib().load()
    if lib.bigru_device_check(0) != 0:
        pytest.fail("no H100: " + lib.bigru_last_error().decode())


@pytest.mark.gpu
@pytest.mark.parametrize("name,prec,mn", JOB_CASES, ids=[f"{n}-{p}-{'mn' if m else 'k'}major" for n, p, m in JOB_CASES])
def test_gemm_job(name, prec, mn):
    _need_gpu()
    j = JOBS[name]
    idx, n = c_index(j)
    canary = np.ones(n, bool)
    canary[idx.ravel()] = False
    rows = model_rows(j)
    bad, report = [], []
    for kind in ("exact", "random"):
        ops = _cached(name, kind, lambda: operands(j, kind))
        runs = run_job(j, prec, mn, ops)
        for off, (st, _) in zip((0, 1), runs):
            if st != staged(j, off):
                bad.append((kind, "staged", off, st))
        if not np.array_equal(runs[0][1], runs[1][1]):
            diff = np.flatnonzero(runs[0][1] != runs[1][1])
            bad.append((kind, "staged != direct", len(diff), diff[:8].tolist()))
        for off, (_, bits) in zip((0, 1), runs):
            hit = np.flatnonzero(bits[canary] != CANARY)
            if len(hit):
                bad.append((kind, "canaries overwritten", off, len(hit), np.flatnonzero(canary)[hit[:8]].tolist()))
        got = runs[0][1][idx[:, rows]].view(np.float32).astype(np.float64)
        want = _cached(name, (kind, prec), lambda: model(j, ops, prec, rows))
        if kind == "exact":
            wrong = np.argwhere(got != want)
            if len(wrong):
                bad.append((kind, "not exact", len(wrong), [(tuple(w), got[tuple(w)], want[tuple(w)]) for w in wrong[:4]]))
        else:
            km = dist(got, want)
            me = dist(want, _cached(name, ("random", "exact"), lambda: model(j, ops, "exact", rows)))
            report.append(dict(job=name, prec=prec, major="mn" if mn else "k", cls="gemm_job", km_l2=km[0], km_max=km[1],
                               me_l2=me[0], me_max=me[1], staged=int(staged(j, 0)), splits=n_splits(j), units=units(j)))
            tol = TOL[prec]
            if not (km[0] <= tol[0] and km[1] <= tol[1]):
                bad.append((kind, "gemm_job", km, tol))
    peak_gb = resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 2 ** 20
    out = os.environ.get("BIGRU_TC_GEMM_REPORT")
    if out:
        with open(out, "a") as f:
            for r in report:
                f.write(json.dumps(dict(r, peak_host_gb=peak_gb)) + "\n")
    print(f"\n{name} {prec} {'mn' if mn else 'k'}-major peak host {peak_gb:.1f} GB " +
          " ".join(f"km {r['km_l2']:.1e}/{r['km_max']:.1e} me {r['me_l2']:.1e}" for r in report))
    assert not bad, bad


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "bf16x3"])
def test_bias_with_split_k_is_refused(prec):
    """A bias with more than one split, forced or from wg_splits, is refused, and C is left as it was."""
    import torch
    _need_gpu()
    L_ = _lib()
    dev = torch.device("cuda")
    for j in (job(256, 128, 4096, bias=True, splits=4), job(256, 128, 4096, bias=True)):
        assert n_splits(j) > 1
        a = torch.ones(j["M"] * j["K"], device=dev)
        b = torch.ones(j["N"] * j["K"], device=dev)
        bias = torch.ones(j["N"], device=dev)
        c = torch.full((j["M"] * j["N"],), CANARY, dtype=torch.int32, device=dev)
        ws = torch.empty(1 << 22, device=dev)
        rc, _ = tc_gemm(prec, 0, j, a.data_ptr(), b.data_ptr(), bias.data_ptr(), c.data_ptr(), ws.data_ptr())
        assert rc == L_.ERR_ARG, rc
        assert b"split-K" in L_.load().bigru_last_error()
        torch.cuda.synchronize()
        assert (c.cpu().numpy() == CANARY).all()


# ---- the plans' own output jobs, aligned and one float off ---------------------------------------------------------
# B32 T9 F20 H128 L2 D2 C4: every output job of these calls is staged when its buffer is aligned (the logits N = 4; dx
# N = 20; dW_ih of layer 0 has one split, K = 288 being 5 k-blocks, and writes grads at pitch 20 and block stride 57,600;
# dW_hh, layer 1 and dlin_w at pitches 128, 256 and 384), and direct one float off.
PLAN = dict(B=32, T=9, F=20, H=128, L=2, C=4, D=2)


def _canaried(n, off):
    """An int32 buffer of n elements with PAD canaries on both sides, off floats past 16-byte alignment: (whole view,
    device pointer of the n elements)."""
    import torch
    buf = torch.full((n + 2 * PAD + 1,), CANARY, dtype=torch.int32, device=torch.device("cuda"))
    view = buf[off:off + n + 2 * PAD]
    return view, view.data_ptr() + 4 * PAD


def _plan_outputs(prec, head, off):
    import torch
    L_ = _lib()
    lib = L_.load()
    B, T, F, H, L, C_, D = (PLAN[k] for k in "BTFHLCD")
    dev = torch.device("cuda")
    plan = C.c_void_p()
    if head:
        L_.check(lib.bigru_plan_create(B, T, F, H, L, C_, 1, CODE[prec], C.byref(plan)), "plan_create")
    else:
        L_.check(lib.bigru_gru_plan_create(B, T, F, H, L, 1, CODE[prec], C.byref(plan)), "gru_plan_create")
    try:
        n = lib.bigru_param_count(plan)
        rng = np.random.default_rng([B, T, F, H, int(head)])
        pd = torch.from_numpy(rng.uniform(-H ** -0.5, H ** -0.5, n).astype(np.float32)).to(dev)
        xd = torch.from_numpy(rng.standard_normal((B, T, F), dtype=np.float32)).to(dev)
        sb, cb, ib = C.c_size_t(), C.c_size_t(), C.c_size_t()
        L_.check(lib.bigru_workspace_bytes(plan, C.byref(sb), C.byref(cb)), "workspace_bytes")
        L_.check(lib.bigru_infer_workspace_bytes(plan, C.byref(ib)), "infer_workspace_bytes")
        stash = torch.zeros(sb.value // 4, device=dev)
        scratch = torch.zeros(cb.value // 4, device=dev)
        st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        ptr = L_.ptr
        grads, gp = _canaried(n, off)
        dx, xp = _canaried(B * T * F, off)
        out = dict(grads=grads, dx=dx)
        if head:
            dl = torch.from_numpy(rng.standard_normal((B, C_), dtype=np.float32)).to(dev)
            logits, lp = _canaried(B * C_, off)
            L_.check(lib.bigru_forward(plan, ptr(pd), ptr(xd), None, 0.0, 0, 0, 0, ptr(stash), ptr(scratch), lp, None, st),
                     "forward")
            L_.check(lib.bigru_backward(plan, ptr(pd), ptr(xd), None, 0.0, 0, 0, 0, ptr(stash), ptr(scratch), ptr(dl), gp, xp,
                                        None, st), "backward")
            ws = torch.zeros(ib.value // 4, device=dev)
            inf, ip = _canaried(B * C_, off)
            L_.check(lib.bigru_infer(plan, ptr(pd), ptr(xd), None, ptr(ws), ip, st), "infer")
            out.update(logits=logits, infer_logits=inf)
        else:
            y = torch.zeros(B, T, D * H, device=dev)
            dy = torch.from_numpy(rng.standard_normal((B, T, D * H), dtype=np.float32)).to(dev)
            L_.check(lib.bigru_gru_forward(plan, ptr(pd), ptr(xd), None, 0.0, 0, 0, ptr(stash), ptr(scratch), ptr(y), None,
                                           None, st), "gru_forward")
            L_.check(lib.bigru_gru_backward(plan, ptr(pd), ptr(xd), None, 0.0, 0, 0, ptr(stash), ptr(scratch), ptr(y), ptr(dy),
                                            None, gp, xp, None, None, st), "gru_backward")
        torch.cuda.synchronize()
        return {k: v.cpu().numpy() for k, v in out.items()}
    finally:
        lib.bigru_plan_destroy(plan)


@pytest.mark.gpu
@pytest.mark.parametrize("head", [True, False], ids=["bigru", "gru"])
@pytest.mark.parametrize("prec", ["bf16", "bf16x3"])
def test_plan_outputs_do_not_depend_on_their_alignment(prec, head):
    """bigru_forward / bigru_backward / bigru_infer (logits, dx, grads) and bigru_gru_backward (dx, grads) with their outputs
    16-byte aligned and one float off: bitwise the same, every element written, the canaries untouched."""
    _need_gpu()
    a, b = _plan_outputs(prec, head, 0), _plan_outputs(prec, head, 1)
    assert set(a) == ({"logits", "infer_logits", "grads", "dx"} if head else {"grads", "dx"})
    for k in a:
        assert (a[k][:PAD] == CANARY).all() and (a[k][-PAD:] == CANARY).all(), k
        assert (b[k][:PAD] == CANARY).all() and (b[k][-PAD:] == CANARY).all(), k
        body = a[k][PAD:-PAD].view(np.float32)
        assert np.isfinite(body).all(), k
        assert np.array_equal(a[k], b[k]), (k, int((a[k] != b[k]).sum()))
    if head:
        assert np.array_equal(a["logits"], a["infer_logits"])
