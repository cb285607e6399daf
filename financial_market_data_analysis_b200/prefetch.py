"""Host -> device input pipeline for the training loop: batches that live in (pinned) host memory are copied to the
GPU on a side stream one step ahead of their use, so the H2D transfer of step i+1 overlaps the kernels of step i.
The reference feeds CPU tensors from a DataLoader straight into the model (biGRU_model.py:189-200); this is the
H100 counterpart for callers that keep their batches on the host."""
from __future__ import annotations

import torch


class DevicePrefetcher:
    """Iterate (x, target) host batches as device tensors, double-buffered through a copy stream."""

    def __init__(self, batches, device, depth: int = 2):
        self.batches, self.device, self.depth = batches, torch.device(device), max(2, depth)
        self.stream = torch.cuda.Stream(device=self.device)

    def __iter__(self):
        it = iter(self.batches)
        slots, ready, free = [None] * self.depth, [None] * self.depth, [None] * self.depth
        pending = []

        def issue(k):
            try:
                x, t = next(it)
            except StopIteration:
                return False
            with torch.cuda.stream(self.stream):
                if free[k] is not None:
                    self.stream.wait_event(free[k])              # the consumer is done with this slot
                if slots[k] is None or slots[k][0].shape != x.shape or slots[k][1].shape != t.shape:
                    slots[k] = (torch.empty(x.shape, dtype=torch.float32, device=self.device),
                                torch.empty(t.shape, dtype=t.dtype, device=self.device))
                slots[k][0].copy_(x, non_blocking=True)
                slots[k][1].copy_(t, non_blocking=True)
                ev = torch.cuda.Event()
                ev.record(self.stream)
                ready[k] = ev
            pending.append(k)
            return True

        for k in range(self.depth):
            if not issue(k):
                break
        while pending:
            k = pending.pop(0)
            cur = torch.cuda.current_stream(self.device)
            cur.wait_event(ready[k])
            yield slots[k]
            ev = torch.cuda.Event()
            ev.record(cur)
            free[k] = ev
            issue(k)
