"""The cost of recurrent dropout at configs[1] (B512 T128 F64 H256 L2 C3, bidirectional): ``BiGRU.train_step`` with
recurrent_dropout 0 against 0.25 at bf16x3 and at bf16 (plain launches, no CUDA graph, so that both sides launch the same
way), and the PyTorch alternative at the same shape: a loop of fp32 ``nn.GRUCell`` per layer and direction with fixed masks
on the state, forward + backward of the same head and loss.

Per path: ms per call from CUDA events over windows of at least --window seconds, --repeats windows each, paths in rotating
order (median, min, max) and sequences/s of the median.  The card's name, power limit and maximum SM clock are read in the
same run.

    python tools/bench_recurrent_dropout.py [--out DIR] [--window 0.5] [--repeats 7]   (writes DIR/bench_recurrent_dropout.json)"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from financial_market_data_analysis_b200 import BiGRU   # noqa: E402
from bench_gru import measure                           # noqa: E402
from bench_lengths import card                          # noqa: E402

B, T, F, H, L, C, P = 512, 128, 64, 256, 2, 3, 0.25


def model(prec, p):
    torch.manual_seed(0)
    m = BiGRU(H, F, C, L, 50, 0.2, True, True, precision=prec, recurrent_dropout=p).cuda().train()
    m.use_cuda_graph = False
    m.add_loss_fn(nn.CrossEntropyLoss())
    m.add_optimizer(torch.optim.Adam(m.parameters(), lr=1e-3))
    return m


class CellLoop(nn.Module):
    """What a PyTorch user writes for recurrent dropout: one nn.GRUCell per layer and direction stepped in Python, the state
    multiplied by a mask drawn once per call, then BiGRU's pooling head."""

    def __init__(self):
        super().__init__()
        self.cells = nn.ModuleList([nn.GRUCell(F if l == 0 else 2 * H, H) for l in range(L) for _ in range(2)])
        self.linear = nn.Linear(3 * H, C)

    def forward(self, x):
        inp = x
        for l in range(L):
            outs = []
            for d in range(2):
                cell = self.cells[2 * l + d]
                m = torch.bernoulli(torch.full((B, H), 1 - P, device=x.device)) / (1 - P)
                h = x.new_zeros(B, H)
                ys = [None] * T
                for t in (range(T) if d == 0 else reversed(range(T))):
                    h = cell(inp[:, t], m * h)
                    ys[t] = h
                outs.append(torch.stack(ys, 1))
            inp = torch.cat(outs, -1)
        s = inp[..., :H] + inp[..., H:]
        last = inp[:, -1, :H] + inp[:, 0, H:]
        return self.linear(torch.cat([last, s.max(1).values, s.mean(1)], 1))


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--out", default="bench_recurrent_dropout_out")
    ap.add_argument("--window", type=float, default=0.5, help="seconds of work per timed window")
    ap.add_argument("--repeats", type=int, default=7, help="timed windows per path")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_recurrent_dropout needs a CUDA device (an H100); there is nothing to measure without one")
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, T, F, generator=g).cuda()
    tgt = torch.randint(0, C, (B,), generator=g).cuda()
    calls = {}
    for prec in ("bf16x3", "bf16"):
        for p in (0.0, P):
            m = model(prec, p)
            calls[f"{prec}_p{p}"] = lambda m=m: m.train_step(x, tgt)
    torch.manual_seed(0)
    loop = CellLoop().cuda()
    opt = torch.optim.Adam(loop.parameters(), lr=1e-3)
    loss_fn = nn.CrossEntropyLoss()

    def loop_step():
        opt.zero_grad()
        loss = loss_fn(loop(x), tgt)
        loss.backward()
        nn.utils.clip_grad_norm_(loop.parameters(), 50)
        opt.step()

    calls["torch_grucell_loop_fp32"] = loop_step
    info = {"card": card(), "torch": torch.__version__, "shape": dict(B=B, T=T, F=F, H=H, L=L, C=C, bidirectional=True),
            "recurrent_dropout": P, "window_s": a.window, "repeats": a.repeats,
            "train_step": measure(calls, a.window, a.repeats)}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "bench_recurrent_dropout.json"), "w") as f:
        json.dump(info, f, indent=1)
    print(json.dumps(info))


if __name__ == "__main__":
    main()
