"""Train-step time of the reference's OWN model shapes (notebook: F=108, H=32, window 30, batch 2; predict.py: H=8, window 5) on
the exact FFMA path vs precision="auto" (zero-padded onto the fp32-class tensor-core kernels).  Usage: python tools/small_shapes_bench.py [OUT.json]"""
import json, os, sys, time
import torch, torch.nn as nn
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import financial_market_data_analysis_b200 as pkg

out = []
for name, (B, T, F, H, L, C, drop) in {"notebook (B2 T30 F108 H32 L2, dropout 0.2)": (2, 30, 108, 32, 2, 4, 0.2),
                                          "notebook shape, batch 64, no dropout": (64, 30, 108, 32, 2, 4, 0.0),
                                          "predict.py shape (B1 T5 F108 H8 L1)": (1, 5, 108, 8, 1, 4, 0.0)}.items():
    row = {"case": name}
    for prec in ("fp32", "auto"):
        torch.manual_seed(0)
        m = pkg.BiGRU(H, F, C, L, 50, drop, True, True, precision=prec).cuda().train()
        m.add_loss_fn(nn.BCEWithLogitsLoss()); m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
        x = torch.randn(B, T, F, device="cuda"); y = (torch.rand(B, C, device="cuda") > 0.5).float()
        for _ in range(5):
            m.train_step(x, y)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = 50
        for _ in range(n):
            m.train_step(x, y)
        torch.cuda.synchronize()
        row[prec + "_us_per_step"] = (time.perf_counter() - t0) / n * 1e6
        row[prec + "_runs_as"] = m.resolved_precision(B) + (f" (hidden {m.plan_hidden(B)})" if m.plan_hidden(B) != H else "")
    out.append(row)
    print(row)
if len(sys.argv) > 1:                  # optional output path for the rows as JSON
    json.dump(out, open(sys.argv[1], "w"), indent=1)
