"""Generates tests/golden/*.npz by running the UNMODIFIED reference from /root/reference.

Run in the build container only (python tests/golden/make_golden.py); /root/reference does not
exist on the GPU box, so the fixtures are committed.  Nothing here is imported by the product.

  kat.npz          shipped model_params.pt (H=8,F=108,C=4,L=1) + two fixed inputs -> logits
  model_<case>.npz seed-fixed synthetic cases through reference BiGRU: inputs, state_dict,
                   logits, loss, every gradient, (dx, dh0), params after clip+Adam
  loader.npz       reference MySQLChunkLoader / MySQLBatchLoader / TrainValTestSplit driven by
                   tests/fake_db.FakeCursor: chunk ranges, norm params, delivered batches
  loader_edges.npz the same over the table shapes of LOADER_EDGES / LOADER_SHORT (NULLs at chunk edges, F % 4 == 0
                   and != 0, window 1, one-window chunks, db_length < chunk_size), every chunk
Usage: python tests/golden/make_golden.py [kat models loader loader_edges]   (no argument: all)
"""
import os
import pickle
import sys
import warnings

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, "/root/reference")
import fake_db  # noqa: E402

fake_db.install_reference_stubs(bid_levels=2, ask_levels=2)
from biGRU_model import BiGRU  # noqa: E402  (reference, unmodified)
import sql_pytorch_dataloader as ref_loader  # noqa: E402  (reference, unmodified)

torch.set_num_threads(4)


def sd_np(sd, prefix):
    return {prefix + k: v.detach().cpu().numpy().copy() for k, v in sd.items()}


def gen_kat():
    sd = torch.load("/root/reference/model_params.pt", map_location="cpu")
    m = BiGRU(8, 108, 4, 1, 50, 0.2, False, True)
    m.load_state_dict(sd)
    m.eval()
    x1 = torch.full((1, 5, 108), 0.5)
    x2 = (torch.arange(540).view(1, 5, 108) % 17).float() / 17
    g = torch.Generator().manual_seed(5)
    x3 = torch.rand(6, 5, 108, generator=g)
    with torch.no_grad():
        out = {"x1": x1.numpy(), "y1": m(x1).numpy(), "x2": x2.numpy(), "y2": m(x2).numpy(),
               "x3": x3.numpy(), "y3": m(x3).numpy()}
    out.update(sd_np(sd, "p:"))
    with open("/root/reference/norm_params", "rb") as f:
        npar = pickle.load(f)
    out["norm_min"] = np.array([float(v["MIN"]) for v in npar.values()], np.float32)
    out["norm_max"] = np.array([float(v["MAX"]) for v in npar.values()], np.float32)
    np.savez_compressed(os.path.join(HERE, "kat.npz"), **out)
    print("kat", out["y1"], out["y2"])


def gen_model(name, B, T, F, H, L, C, bidir, loss, with_h0=False, seed=1234):
    torch.manual_seed(0)
    m = BiGRU(H, F, C, L, 50, 0.0, False, bidir)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, T, F, generator=g)
    D = 2 if bidir else 1
    out = {}
    if loss == "ce":
        target = torch.randint(0, C, (B,), generator=g)
        loss_fn = nn.CrossEntropyLoss()
    else:
        target = (torch.rand(B, C, generator=g) < 0.25).float()
        if loss == "bce":
            w = torch.rand(C, generator=g) + 0.5
            pw = torch.rand(C, generator=g) * 3 + 0.5
            loss_fn = nn.BCEWithLogitsLoss(weight=w, pos_weight=pw)
            out["loss_weight"], out["loss_pos_weight"] = w.numpy(), pw.numpy()
        else:
            loss_fn = nn.MultiLabelSoftMarginLoss()
    h0 = None
    if with_h0:
        h0 = (torch.randn(L * D, B, H, generator=g) * 0.5).requires_grad_(True)
        out["h0"] = h0.detach().numpy()
    x.requires_grad_(True)
    m.train()                      # dropout p=0: identical to eval, exercises the training path
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    out.update(sd_np(m.state_dict(), "p:"))
    opt.zero_grad()
    pred = m.forward(x, h0)
    lv = loss_fn(pred, target)
    lv.backward()
    out.update({"x": x.detach().numpy(), "target": target.numpy(), "logits": pred.detach().numpy(),
                "loss": np.array(lv.item(), np.float64), "dx": x.grad.numpy()})
    if with_h0:
        out["dh0"] = h0.grad.numpy()
    for k, p in m.named_parameters():
        out["g:" + k] = p.grad.detach().numpy().copy()
    norm = nn.utils.clip_grad_norm_(m.parameters(), m.clip)
    out["grad_norm"] = np.array(float(norm), np.float64)
    opt.step()
    out.update(sd_np(m.state_dict(), "q:"))          # params after one clip+Adam step
    out["meta"] = np.array([B, T, F, H, L, C, int(bidir)], np.int64)
    out["loss_kind"] = np.array(loss)
    np.savez_compressed(os.path.join(HERE, f"model_{name}.npz"), **out)
    print(name, "loss", lv.item(), "norm", float(norm))


def gen_loader():
    warnings.simplefilter("ignore")
    cols, targets, fields, query = fake_db.make_table(n_rows=250)
    cur = fake_db.FakeCursor(cols, targets)
    cwd = os.getcwd()
    os.chdir("/tmp")               # the reference pickles ./norm_params as a side effect
    try:
        cl = ref_loader.MySQLChunkLoader(cur, "stock_data_joined", query, chunk_size=100, window=30)
    finally:
        os.chdir(cwd)
    out = {"n_chunks": np.array(len(cl))}
    for i in range(len(cl)):
        idx, (mn, mx) = cl[i]
        out[f"chunk{i}_ids"] = np.array(idx, np.int64)
        out[f"chunk{i}_min"] = mn.numpy()
        out[f"chunk{i}_max"] = mx.numpy()
    split = ref_loader.TrainValTestSplit(cl, 0.1, 0.1)
    tr, va, te = split.get_sets()
    out["split_train"] = np.array([len(i) for i, _ in tr], np.int64)
    out["split_val"] = np.array([len(i) for i, _ in va], np.int64)
    out["split_test"] = np.array([len(i) for i, _ in te], np.int64)
    for bs in (2, 8):
        idx, norm = cl[1]
        ds = ref_loader.MySQLBatchLoader(idx, norm, cur, "stock_data_joined", query, "t0, t1, t2, t3", 30)
        dl = torch.utils.data.DataLoader(ds, batch_size=bs)
        xs, ys = [], []
        for xb, yb in dl:
            xs.append(xb.numpy())
            ys.append(yb.numpy())
        out[f"bs{bs}_x"] = np.concatenate(xs)
        out[f"bs{bs}_y"] = np.concatenate(ys)
        out[f"bs{bs}_nbatches"] = np.array(len(xs))
        out[f"bs{bs}_xnorm"] = ds.x.numpy()
    out["fields"] = np.array(fields)
    np.savez_compressed(os.path.join(HERE, "loader.npz"), **out)
    print("loader chunks", len(cl), "bs2 windows", out["bs2_x"].shape, "bs8", out["bs8_x"].shape)


# Table shapes of loader_edges.npz.  Row numbers in "null_rows" are 0-based (ID - 1) and sit at the first and last row
# of chunks, in the rows two chunks share, in runs longer than the window and in constant and order-book columns.
# F = 2 * levels + n_plain + 2.
LOADER_EDGES = {
    # loader.npz's shape (F = 9), with NULLs at its chunk edges
    "current": dict(table=dict(n_rows=250, null_rows={"sd.f1": [29, 98, 70, 198, 170, 249], "sd.f2": list(range(100, 140)),
                                                      "sd.bid_1_size": [75, 76, 77, 180], "sd.const_nz": [29]}),
                    chunk_size=100, window=30, batch_sizes=[2, 8, 32]),
    # db_length % chunk_size == 0: the last chunk holds one window; F = 8 (float4 gather); middle chunks' 60 windows are
    # filled exactly by every batch size
    "divisible": dict(table=dict(n_rows=240, n_plain=4, levels=1, seed=11,
                                 null_rows={"sd.f1": [11, 58, 48, 118, 108, 228, 239], "sd.f3": list(range(120, 140)),
                                            "sd.ask_0_size": [50, 170, 230], "sd.const_zero": [229]}),
                      chunk_size=60, window=12, batch_sizes=[4, 12, 60]),
    # window 1: chunks share no rows; F = 13
    "window1": dict(table=dict(n_rows=130, n_plain=5, levels=3, seed=12,
                               null_rows={"sd.f1": [0, 48, 49, 98, 99, 129], "sd.f4": list(range(60, 75)),
                                          "sd.bid_2_size": [10, 120]}),
                    chunk_size=50, window=1, batch_sizes=[1, 7, 16]),
    # chunk 0 has exactly window rows (one window); F = 6
    "one_window": dict(table=dict(n_rows=130, n_plain=2, levels=1, seed=13,
                                  null_rows={"sd.f1": [19, 38, 20, 78, 60, 118, 100, 129], "sd.ask_0_size": list(range(40, 62))}),
                       chunk_size=40, window=20, batch_sizes=[1, 3, 8]),
    # middle chunks' 64 windows are filled exactly by 16, 32 and 64; F = 16 (float4 gather)
    "exact_fill": dict(table=dict(n_rows=200, n_plain=8, levels=3, seed=14,
                                  null_rows={"sd.f2": [7, 62, 56, 126, 120, 190, 184, 199], "sd.f5": list(range(70, 80)),
                                             "sd.bid_0_size": [58, 122, 186]}),
                       chunk_size=64, window=8, batch_sizes=[16, 32, 64]),
}
# db_length < chunk_size: the reference's only chunk is IDs range(window, chunk_size), past the table's end
LOADER_SHORT = dict(table=dict(n_rows=50, seed=15, null_rows={"sd.f1": [7, 49]}), chunk_size=64, window=8)


def _ref_chunk_loader(cur, query, spec):
    cwd = os.getcwd()
    os.chdir("/tmp")               # the reference pickles ./norm_params as a side effect
    try:
        cl = ref_loader.MySQLChunkLoader(cur, "stock_data_joined", query, chunk_size=spec["chunk_size"], window=spec["window"])
        with open("norm_params", "rb") as fh:
            pick = pickle.load(fh)
    finally:
        os.chdir(cwd)
    return cl, pick


def gen_loader_edges():
    """loader_edges.npz: the reference loader over LOADER_EDGES / LOADER_SHORT.  Keys are "<shape>__<name>"; "<shape>__spec"
    is the shape's JSON, from which the tests rebuild the same table with fake_db.make_table."""
    import json
    warnings.simplefilter("ignore")
    out = {}
    for name, spec in list(LOADER_EDGES.items()) + [("short", LOADER_SHORT)]:
        levels = spec["table"].get("levels", 2)
        ref_loader.bid_levels = ref_loader.ask_levels = levels
        cols, targets, fields, query = fake_db.make_table(**spec["table"])
        cur = fake_db.FakeCursor(cols, targets)
        cl, pick = _ref_chunk_loader(cur, query, spec)
        p = name + "__"
        out[p + "spec"] = np.array(json.dumps(spec))
        out[p + "fields"] = np.array(fields)
        out[p + "n_chunks"] = np.array(len(cl))
        out[p + "pickle_min"] = np.array([float(pick[f]["MIN"]) for f in fields], np.float32)
        out[p + "pickle_max"] = np.array([float(pick[f]["MAX"]) for f in fields], np.float32)
        y_fields = ", ".join(targets)
        for i in range(len(cl)):
            idx, (mn, mx) = cl[i]
            q = f"{p}chunk{i}_"
            out[q + "ids"] = np.array(idx, np.int64)
            out[q + "min"], out[q + "max"] = mn.numpy(), mx.numpy()
            ds = ref_loader.MySQLBatchLoader(idx, (mn, mx), cur, "stock_data_joined", query, y_fields, spec["window"])
            out[q + "xnorm"] = ds.x.numpy()
            for bs in spec.get("batch_sizes", []):        # the short table's windows run past its rows: no batches
                ds = ref_loader.MySQLBatchLoader(idx, (mn, mx), cur, "stock_data_joined", query, y_fields, spec["window"])
                xs, ys = [], []
                for xb, yb in torch.utils.data.DataLoader(ds, batch_size=bs):
                    xs.append(xb.numpy())
                    ys.append(yb.numpy())
                F, C = len(fields), len(targets)
                out[q + f"bs{bs}_nbatches"] = np.array(len(xs))
                out[q + f"bs{bs}_x"] = np.concatenate(xs) if xs else np.zeros((0, spec["window"], F), np.float32)
                out[q + f"bs{bs}_y"] = np.concatenate(ys) if ys else np.zeros((0, 1, C), np.float32)
        split = ref_loader.TrainValTestSplit(cl, 0.1, 0.1)
        out[p + "split"] = np.array([len(list(s)) for s in split.get_sets()], np.int64)     # chunks in train, val, test
        print("loader_edges", name, "F", len(fields), "chunks", len(cl))
    ref_loader.bid_levels = ref_loader.ask_levels = 2
    np.savez_compressed(os.path.join(HERE, "loader_edges.npz"), **out)


if __name__ == "__main__":
    GENERATORS = {
        "kat": gen_kat,
        "models": lambda: (
            gen_model("c0", 32, 64, 32, 128, 1, 3, True, "ce"),                 # BASELINE config 0
            gen_model("small_l2", 4, 7, 5, 8, 2, 3, True, "ce"),
            gen_model("small_uni_bce", 3, 6, 4, 8, 2, 4, False, "bce", with_h0=True),
            gen_model("small_bi_h0_mlsm", 5, 9, 12, 16, 2, 4, True, "mlsm", with_h0=True),
            gen_model("ragged", 3, 1, 7, 24, 1, 3, True, "ce")),                # T=1 edge, odd sizes
        "loader": gen_loader,
        "loader_edges": gen_loader_edges,
    }
    for g in sys.argv[1:] or GENERATORS:         # e.g. `make_golden.py loader loader_edges`; no argument: all of them
        GENERATORS[g]()
