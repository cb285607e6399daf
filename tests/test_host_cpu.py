"""CPU-only tests: the C-ABI library loads and exports every declared symbol, host-side logic of the
model wrapper and the loader, and the data-parallel plumbing over gloo (world_size 2)."""
import os
import re
import sys

import numpy as np
import pytest
import torch
import torch.nn as nn

import fake_db
from oracle import bigru_oracle as bo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def pkg():
    import financial_market_data_analysis_b200 as p
    from financial_market_data_analysis_b200 import build as b
    if not os.path.exists(p._lib.LIB_PATH):
        b.build()
    return p


def header_functions():
    src = open(os.path.join(ROOT, "include", "bigru_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(bigru_[a-z_0-9]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(pkg):
    lib = pkg._lib.load()
    names = header_functions()
    assert len(names) >= 15
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/bigru_b200.h but not exported"
    assert sorted(pkg._lib.SIGNATURES) == names          # the ctypes mirror binds exactly the header
    assert lib.bigru_version() >= 100


def test_plan_bookkeeping_and_null_backward_input_without_gpu(pkg):
    """Plans are host objects: parameter layout and workspace sizes can be checked on CPU."""
    lib, C = pkg._lib.load(), pkg._lib.C
    h = C.c_void_p()
    assert lib.bigru_plan_create(512, 128, 64, 256, 2, 3, 1, pkg._lib.PREC_FP32, C.byref(h)) == 0
    assert lib.bigru_param_count(h) == 1_679_619            # SURVEY.md 8(a) A5
    off, rows, cols = C.c_int64(), C.c_int64(), C.c_int64()
    assert lib.bigru_param_offset(h, 1, 1, 1, C.byref(off), C.byref(rows), C.byref(cols)) == 0
    assert (rows.value, cols.value) == (768, 256)
    a, b = C.c_size_t(), C.c_size_t()
    assert lib.bigru_workspace_bytes(h, C.byref(a), C.byref(b)) == 0 and a.value > 0 and b.value > 0
    lib.bigru_plan_destroy(h)
    assert lib.bigru_plan_create(4, 4, 4, 4, 1, 2, 1, 7, C.byref(h)) == pkg._lib.ERR_ARG
    if not torch.cuda.is_available():
        assert lib.bigru_device_check(0) == pkg._lib.ERR_DEVICE      # fails loudly, no fallback
        assert b"no CPU fallback" in lib.bigru_last_error()
        # the backward needs the input the forward read: a null d_x is refused before anything is launched (a call that got
        # past the argument checks would fail here with ERR_CUDA at its first memset)
        assert lib.bigru_plan_create(32, 4, 8, 128, 1, 3, 1, pkg._lib.PREC_BF16X3, C.byref(h)) == 0
        dev = C.c_void_p(256)                                        # stands for a device pointer; never dereferenced
        assert lib.bigru_backward(h, dev, None, None, 0.0, 0, 0, 0, dev, dev, dev, dev, None, None, None) == pkg._lib.ERR_ARG
        assert b"null argument" in lib.bigru_last_error()
        lib.bigru_plan_destroy(h)


def test_model_surface_and_state_dict(pkg, golden_dir):
    z = np.load(os.path.join(golden_dir, "kat.npz"))
    m = pkg.BiGRU(8, 108, 4, 1, 50, 0.2, False, True)
    keys = [k[2:] for k in z.files if k.startswith("p:")]
    assert list(m.state_dict().keys()) == keys
    m.load_state_dict({k: torch.from_numpy(z["p:" + k]) for k in keys})
    assert m._is_flat()
    for a in ("hidden_size", "n_features", "output_size", "n_layers", "clip", "dropout_p", "spatial_dropout",
              "bidirectional", "n_directions"):
        assert hasattr(m, a)
    # flat vector is in C-ABI order and aliases the parameters
    m.linear.bias.data.fill_(7.0)
    assert torch.all(m.flat_parameters()[-4:] == 7.0)
    # same seed -> same initial weights as torch.nn.GRU / nn.Linear (what the reference constructs)
    torch.manual_seed(0); ref = bo.OracleBiGRU(16, 5, 3, 2, 50, 0.1, True, True)
    torch.manual_seed(0); mine = pkg.BiGRU(16, 5, 3, 2, 50, 0.1, True, True)
    for (k1, v1), (k2, v2) in zip(ref.state_dict().items(), mine.state_dict().items()):
        assert k1 == k2 and torch.equal(v1, v2)
    with pytest.raises(RuntimeError, match="no CPU path"):
        mine(torch.zeros(2, 3, 5))
    with pytest.raises(RuntimeError):
        mine.gru(torch.zeros(2, 3, 5))
    opt = torch.optim.Adam(mine.parameters(), lr=1e-3)
    mine.add_optimizer(opt); mine.add_loss_fn(nn.CrossEntropyLoss()); mine.add_device(torch.device("cpu"))
    assert mine.can_fuse_step()
    mine.add_loss_fn(nn.CrossEntropyLoss(label_smoothing=0.1))
    assert not mine.can_fuse_step()
    # precision="auto": the fp32-class tensor-core path for hidden sizes up to 256 (smaller models zero-padded to 128 / 256 hidden
    # units, other batch sizes to whole 32-row tiles), the exact FFMA path beyond
    auto = pkg.BiGRU(256, 64, 3, 2, precision="auto")
    assert auto.resolved_precision(512) == "bf16x3" and auto.resolved_precision(500) == "bf16x3"
    assert auto._padded_batch(512) == 512 and auto._padded_batch(500) == 512 and auto._padded_batch(1) == 32
    assert pkg.BiGRU(256, 64, 3, 2, precision="bf16")._padded_batch(500) == 512 and pkg.BiGRU(256, 64, 3, 2, precision="bf16")._padded_batch(17) == 32
    assert pkg.BiGRU(256, 64, 3, 2, precision="fp32")._padded_batch(500) == 500
    assert pkg.BiGRU(256, 108, 3, 2, precision="auto").resolved_precision(512) == "bf16x3"     # any feature count (padded K extent)
    small = pkg.BiGRU(8, 108, 4, 1, precision="auto")                                          # the shipped checkpoint's shape
    assert small.resolved_precision(64) == "bf16x3" and small.plan_hidden() == 128
    assert pkg.BiGRU(200, 16, 3, 2, precision="auto").plan_hidden() == 256
    assert pkg.BiGRU(300, 16, 3, 2, precision="auto").resolved_precision() == "fp32" and pkg.BiGRU(300, 16, 3, 2, precision="auto").plan_hidden() == 300
    assert pkg.BiGRU(300, 16, 3, 2, precision="bf16").plan_hidden() == 512 and pkg.BiGRU(8, 4, 2, 1, precision="fp32").plan_hidden() == 8
    assert pkg.BiGRU(256, 64, 3, 2, precision="bf16").resolved_precision(7) == "bf16"
    with pytest.raises(ValueError):
        pkg.BiGRU(8, 4, 2, 1, precision="fp64")


def test_bce_weight_fuses_only_when_it_broadcasts_per_class(pkg):
    """The fused BCE applies weight[c] / pos_weight[c] to every row.  A weight of C elements that broadcasts over rows
    instead ([C, 1] against logits [B, C] with B == C) must take the autograd path, or the fused step would compute a
    different loss than torch."""
    C = B = 4
    m = pkg.BiGRU(8, 5, C, 1, 50, 0.0, False, True)
    m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
    g = torch.Generator().manual_seed(3)
    logits, target = torch.randn(B, C, generator=g), (torch.rand(B, C, generator=g) < 0.5).float()
    w = torch.rand(C, generator=g) + 0.5
    # what torch computes with the [C, 1] weight is row-weighted: not the per-class loss the fused kernel would apply
    row_w = nn.BCEWithLogitsLoss(weight=w.reshape(C, 1))(logits, target)
    col_w = nn.BCEWithLogitsLoss(weight=w)(logits, target)
    assert not torch.allclose(row_w, col_w)
    for kw in ({"weight": w.reshape(C, 1)}, {"pos_weight": w.reshape(C, 1)}, {"weight": w.reshape(C, 1, 1)},
               {"weight": torch.rand(B, C, generator=g)}, {"weight": w.reshape(2, 2)}):
        m.add_loss_fn(nn.BCEWithLogitsLoss(**kw))
        assert m._loss_spec() is None and not m.can_fuse_step(), kw
    for kw in ({}, {"weight": w}, {"weight": w.reshape(1, C)}, {"weight": w.reshape(1, 1, C)}, {"pos_weight": w},
               {"weight": torch.tensor(2.0)}, {"weight": torch.tensor([2.0])}, {"pos_weight": torch.ones(1, 1)},
               {"weight": w.reshape(1, C), "pos_weight": w}):
        m.add_loss_fn(nn.BCEWithLogitsLoss(**kw))
        assert m._loss_spec() is not None and m.can_fuse_step(), kw


def test_hidden_padding_index_map(pkg):
    """BiGRU._plan_params / _plan_grads (real parameter -> position in the zero-padded plan's flat vector) against an independent construction:
    every weight tensor zero-padded by its own rule (gate rows g*H + j -> g*Hp + j, input columns of upper layers d*H + k ->
    d*Hp + k, head columns part*H + j -> part*Hp + j) and flattened in the C-ABI order."""
    import oracle_c
    for H, F, L, bidir, C, prec in ((8, 108, 1, True, 4, "auto"), (33, 5, 3, True, 3, "bf16x3"), (7, 3, 2, False, 2, "bf16"),
                                    (200, 16, 2, True, 3, "auto"), (300, 9, 2, True, 2, "bf16")):
        torch.manual_seed(H)
        m = pkg.BiGRU(H, F, C, L, 50, 0.0, False, bidir, precision=prec)
        D, Hp = (2 if bidir else 1), m.plan_hidden()
        assert Hp in (128, 256, 512) and Hp >= H
        sd = {k: v.detach().numpy() for k, v in m.state_dict().items()}
        padded = {}

        def pad_rows(w, cols_out, colmap):
            out = np.zeros((3 * Hp, cols_out), np.float32)
            for g in range(3):
                out[g * Hp:g * Hp + H][:, colmap] = w[g * H:(g + 1) * H]
            return out
        for l in range(L):
            I = F if l == 0 else D * H
            colmap = np.arange(F) if l == 0 else np.concatenate([d * Hp + np.arange(H) for d in range(D)])
            for d in range(D):
                sfx = f"l{l}" + ("_reverse" if d else "")
                padded[f"gru.weight_ih_{sfx}"] = pad_rows(sd[f"gru.weight_ih_{sfx}"], F if l == 0 else D * Hp, colmap)
                padded[f"gru.weight_hh_{sfx}"] = pad_rows(sd[f"gru.weight_hh_{sfx}"], Hp, np.arange(H))
                for b in ("bias_ih", "bias_hh"):
                    padded[f"gru.{b}_{sfx}"] = pad_rows(sd[f"gru.{b}_{sfx}"][:, None], 1, np.arange(1))[:, 0]
        lw = np.zeros((C, 3 * Hp), np.float32)
        for part in range(3):
            lw[:, part * Hp:part * Hp + H] = sd["linear.weight"][:, part * H:(part + 1) * H]
        padded["linear.weight"], padded["linear.bias"] = lw, sd["linear.bias"]
        want = oracle_c.flatten_params(padded, L, D)
        got = m._plan_params().numpy()
        assert got.shape == want.shape and np.array_equal(got, want), (H, F, L, bidir)
        back = m._plan_grads(torch.from_numpy(want)).numpy()                      # unpad = the original flat vector
        assert np.array_equal(back, m.flat_parameters().detach().numpy())


def test_chunk_loader_host_logic(pkg, golden_dir, tmp_path):
    """MySQLChunkLoader / TrainValTestSplit are host code: compare with the unmodified reference's output."""
    import pickle
    z = np.load(os.path.join(golden_dir, "loader.npz"))
    cols, targets, fields, query = fake_db.make_table(n_rows=250)
    cur = fake_db.FakeCursor(cols, targets)
    import financial_market_data_analysis_b200.sql_pytorch_dataloader as L
    L.bid_levels, L.ask_levels = 2, 2
    npath = str(tmp_path / "norm_params")
    cl = L.MySQLChunkLoader(cur, "stock_data_joined", query, chunk_size=100, window=30, norm_params_path=npath)
    assert len(cl) == int(z["n_chunks"])
    for i in range(len(cl)):
        ids, (mn, mx) = cl[i]
        assert np.array_equal(np.array(ids), z[f"chunk{i}_ids"])
        assert np.array_equal(mn.numpy(), z[f"chunk{i}_min"]) and np.array_equal(mx.numpy(), z[f"chunk{i}_max"])
    tr, va, te = L.TrainValTestSplit(cl, 0.1, 0.1).get_sets()
    assert [len(i) for i, _ in tr] == list(z["split_train"])
    assert [len(i) for i, _ in va] == list(z["split_val"])
    assert [len(i) for i, _ in te] == list(z["split_test"])
    saved = pickle.load(open(npath, "rb"))
    assert list(saved.keys()) == fields and float(saved[fields[0]]["MIN"]) == float(z["chunk2_min"][0][0])
    with pytest.raises(AssertionError):
        L.TrainValTestSplit(cl, 0.6, 0.5)
    assert list(L.window_indices(range(5), 3)) == [(0, 1, 2), (1, 2, 3), (2, 3, 4)]
    assert list(L.window_indices(range(2), 3)) == []
    assert L.delivered_window_batches(129, 30, 8) == [(s, 8) for s in range(0, 96, 8)]
    assert L.delivered_window_batches(129, 30, 2)[-1] == (98, 2)
    assert L.delivered_window_batches(10, 1, 4) == [(0, 4), (4, 4), (8, 2)]       # window 1: nothing is lost
    assert L.delivered_window_batches(3, 5, 2) == []
    if not torch.cuda.is_available():
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            ids, norm = cl[1]
            L.MySQLBatchLoader(ids, norm, cur, "stock_data_joined", query, "t0, t1, t2, t3", 30)


@pytest.mark.parametrize("name", ["current", "divisible", "window1", "one_window", "exact_fill", "short"])
def test_chunk_loader_host_logic_at_table_edges(pkg, golden_dir, tmp_path, monkeypatch, name):
    """The SQL-path MySQLChunkLoader over every table shape of loader_edges.npz (NULLs at chunk edges, 1-3 book levels,
    db_length % chunk_size == 0, window 1, one-window chunks): chunk IDs, norm params, the pickle and the split equal the
    unmodified reference's.  For db_length < chunk_size ("short") the reference's IDs run past the table: the ranges
    differ on purpose and select the same rows."""
    import json
    import pickle
    import financial_market_data_analysis_b200.sql_pytorch_dataloader as L
    z = np.load(os.path.join(golden_dir, "loader_edges.npz"))
    spec = json.loads(str(z[name + "__spec"]))
    g = lambda key: z[f"{name}__{key}"]                                        # noqa: E731
    monkeypatch.setattr(L, "bid_levels", spec["table"].get("levels", 2))
    monkeypatch.setattr(L, "ask_levels", spec["table"].get("levels", 2))
    cols, targets, fields, query = fake_db.make_table(**spec["table"])
    assert fields == list(g("fields"))
    npath = str(tmp_path / "norm_params")
    cl = L.MySQLChunkLoader(fake_db.FakeCursor(cols, targets), "stock_data_joined", query, spec["chunk_size"], spec["window"],
                            norm_params_path=npath)
    assert len(cl) == int(g("n_chunks"))
    n = len(cols[fields[0]])
    for i in range(len(cl)):
        ids, (mn, mx) = cl[i]
        ref_ids = g(f"chunk{i}_ids")
        if name == "short":
            assert n < spec["chunk_size"] and ids == tuple(range(spec["window"], n + 1)) and len(ref_ids) > len(ids)
            ref_ids = ref_ids[ref_ids <= n]
        assert np.array_equal(np.array(ids), ref_ids), i
        assert np.array_equal(mn.numpy(), g(f"chunk{i}_min")) and np.array_equal(mx.numpy(), g(f"chunk{i}_max")), i
    assert [len(list(s)) for s in L.TrainValTestSplit(cl, 0.1, 0.1).get_sets()] == list(g("split"))
    saved = pickle.load(open(npath, "rb"))
    assert list(saved) == fields
    assert np.array_equal(np.array([float(saved[f]["MIN"]) for f in fields], np.float32), g("pickle_min"))
    assert np.array_equal(np.array([float(saved[f]["MAX"]) for f in fields], np.float32), g("pickle_max"))


def test_metric_arithmetic_matches_sklearn(pkg):
    from sklearn.metrics import accuracy_score, fbeta_score, hamming_loss
    rng = np.random.default_rng(0)
    C, sizes, rows, acc, ham, fb = 4, [], [], [], [], []
    for B in (8, 8, 5):
        t = (rng.random((B, C)) < 0.4).astype(int)
        p = (rng.random((B, C)) < 0.4).astype(int)
        row = np.zeros(2 + 3 * C)
        row[0] = (t == p).all(1).sum(); row[1] = (t != p).sum()
        for c in range(C):
            row[2 + 3 * c] = ((p[:, c] == 1) & (t[:, c] == 1)).sum()
            row[3 + 3 * c] = ((p[:, c] == 1) & (t[:, c] == 0)).sum()
            row[4 + 3 * c] = ((p[:, c] == 0) & (t[:, c] == 1)).sum()
        rows.append(row); sizes.append(B)
        acc.append(accuracy_score(t, p)); ham.append(hamming_loss(t, p))
        fb.append(fbeta_score(t, p, beta=0.5, average=None, zero_division=0))
    a, h, f = pkg.BiGRU._scores(np.stack(rows), sizes, C)
    assert abs(a - np.mean(acc)) < 1e-12 and abs(h - np.mean(ham)) < 1e-12
    np.testing.assert_allclose(f, np.mean(fb, axis=0), atol=1e-12)


def _dp_worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    from financial_market_data_analysis_b200.parallel import allreduce_flat_, max_over_ranks, shard_batch
    torch.manual_seed(0)
    torch.set_num_threads(1)
    model = bo.OracleBiGRU(8, 4, 3, 2, 50, 0.0, False, True)          # replica (same seed on every rank)
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(8, 5, 4, generator=g)
    t = torch.randint(0, 3, (8,), generator=g)
    xs, ts = shard_batch(x, rank, world), shard_batch(t, rank, world)
    loss = nn.CrossEntropyLoss(reduction="sum")(model(xs), ts) / x.shape[0]     # global-mean normalisation
    loss.backward()
    flat = torch.cat([p.grad.reshape(-1) for p in model.parameters()])
    allreduce_flat_(flat)                                                       # the one collective per step
    mx = max_over_ranks(float(rank + 1), torch.device("cpu"))
    if rank == 0:
        q.put((flat.numpy(), mx))
    dist.destroy_process_group()


def test_data_parallel_allreduce_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_dp_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    got, mx = q.get(timeout=120)
    [p.join(60) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    torch.manual_seed(0)
    model = bo.OracleBiGRU(8, 4, 3, 2, 50, 0.0, False, True)
    g = torch.Generator().manual_seed(1234)
    x = torch.randn(8, 5, 4, generator=g)
    t = torch.randint(0, 3, (8,), generator=g)
    nn.CrossEntropyLoss()(model(x), t).backward()
    full = torch.cat([p.grad.reshape(-1) for p in model.parameters()]).numpy()
    np.testing.assert_allclose(got, full, atol=1e-6)
    assert mx == 2.0
    from financial_market_data_analysis_b200.parallel import shard_bounds
    assert shard_bounds(4096, 3, 8) == (1536, 2048)
    with pytest.raises(ValueError):
        shard_bounds(10, 0, 4)


def test_next_row_entry_points_refuse_the_cpu(pkg):
    """features.window_features / predict.LivePredictor (SURVEY 8(f) N4, N5): host-side argument logic, and no CPU fallback."""
    from financial_market_data_analysis_b200 import features, predict
    kw = dict(volume_MA_periods=[6, 20], price_MA_periods=[20], delta_MA_periods=[12], bollinger_bands_period=20,
              bollinger_bands_std=2, stochastic_oscillator=True)
    assert features.feature_names(**kw) == ["upper_BB_dist", "lower_BB_dist", "vol_MA6", "vol_MA20", "price_MA20", "delta_MA12",
                                            "stoch", "ATR", "price_change"]            # create_database.py:239-240 join order
    assert features.feature_names([], [], [], False, 2, False) == ["ATR", "price_change"]
    x = torch.ones(16)
    with pytest.raises(RuntimeError, match="GPU only"):
        features.window_features(x, x, x, x, x)
    with pytest.raises(RuntimeError, match="GPU only"):
        predict.LivePredictor({}, None, n_features=4, device="cpu")
    assert predict.Y_FIELDS == ["up1", "up2", "down1", "down2"]                          # predict.py:33
    # the n_out query of the C entry point needs no device
    lib, C = pkg._lib.load(), pkg._lib.C
    n_out = C.c_int(0)
    assert lib.bigru_window_features(None, None, None, None, None, 0, (C.c_int * 2)(6, 20), 2, (C.c_int * 1)(20), 1, (C.c_int * 1)(12), 1,
                                     20, 2.0, 1, 1.5, 3.0, None, None, C.byref(n_out), None) == 0
    assert n_out.value == 9
    assert lib.bigru_window_features(None, None, None, None, None, 0, None, 9, None, 0, None, 0, 0, 2.0, 0, 1.5, 3.0, None, None,
                                     C.byref(n_out), None) == pkg._lib.ERR_ARG


def test_drop_in_import_route(tmp_path):
    """INTEGRATION.md: with the package directory itself on sys.path the reference's own import lines
    (`from biGRU_model import BiGRU`, predict.py:16; `from sql_pytorch_dataloader import ...`, the notebook) resolve
    to the H100 implementation - checked in a fresh interpreter started outside the repo."""
    import subprocess
    code = (
        "import sys; sys.path.insert(0, %r)\n"
        "from biGRU_model import BiGRU\n"
        "from sql_pytorch_dataloader import MySQLBatchLoader, MySQLChunkLoader, TrainValTestSplit, window_indices\n"
        "m = BiGRU(8, 108, 4, 1, 50, 0.2, False, True)\n"
        "assert sorted(m.state_dict())[0] == 'gru.bias_hh_l0' and m.linear.weight.shape == (4, 24)\n"
        "assert list(window_indices(range(4), 2)) == [(0, 1), (1, 2), (2, 3)]\n"
        "print('ok')\n") % os.path.join(ROOT, "financial_market_data_analysis_b200")
    r = subprocess.run([sys.executable, "-c", code], cwd=str(tmp_path), capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and r.stdout.strip().endswith("ok"), r.stderr[-2000:]
