"""CPU oracle for per-sequence lengths.  TEST INFRASTRUCTURE ONLY (see bigru_oracle.py for who may import oracle/).

The defining rule of ``BiGRU.forward(x, lengths=...)``, written in torch float64: every GRU layer is ``nn.GRU`` on
``pack_padded_sequence(x, lengths, batch_first=True, enforce_sorted=False)``, unpacked with ``pad_packed_sequence(...,
total_length=T)`` (layer outputs 0 at padded steps; ``h_n`` the state after each direction's last valid step), then the head
of biGRU_model.py:111-137 over the valid steps only: ``last`` = forward output at t = len - 1 plus reverse output at t = 0,
max and mean of ``s_t = y_t[:H] + y_t[H:]`` over t < len.  Gradients come from autograd.

Layers run one at a time so that dropout masks can be injected between them (the kernels' masks are a pure function of
(seed, element index); tests rebuild them on the host).
"""
from __future__ import annotations

import torch
import torch.nn as nn
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence


class LengthsOracle(nn.Module):
    """float64 restatement of the model with lengths, parameters taken from a BiGRU / OracleBiGRU state_dict."""

    def __init__(self, state_dict, hidden_size, n_features, n_layers, bidirectional=True):
        super().__init__()
        self.H, self.L, self.D = hidden_size, n_layers, 2 if bidirectional else 1
        sd = {k: v.detach().cpu().double() for k, v in state_dict.items()}
        self.layers = nn.ModuleList()
        for l in range(n_layers):
            g = nn.GRU(n_features if l == 0 else self.D * hidden_size, hidden_size, num_layers=1, batch_first=True,
                       bidirectional=bidirectional).double()
            g.load_state_dict({k.replace(f"_l{l}", "_l0")[len("gru."):]: v for k, v in sd.items()
                               if k.startswith("gru.") and f"_l{l}" in k})
            self.layers.append(g)
        self.linear = nn.Linear(3 * hidden_size, sd["linear.weight"].shape[0]).double()
        self.linear.load_state_dict({"weight": sd["linear.weight"], "bias": sd["linear.bias"]})

    def forward(self, x, lengths, masks=None, idx=None):
        """x [B, T, F] float64, lengths [B] integers in [1, T].  masks: None or one factor per layer (None or a tensor
        broadcasting against that layer's input [B, T, I_l]), multiplied into the layer's input before packing.  idx:
        None or [B, H] time indices at which the max-pool is read (the kernel's routing), else its arg-max over t < len.
        Returns (logits [B, C], h_n [L*D, B, H], s [B, T, H])."""
        B, T = x.shape[0], x.shape[1]
        lens = torch.as_tensor(lengths, dtype=torch.int64).cpu()
        inp, hns = x, []
        for l, g in enumerate(self.layers):
            if masks is not None and masks[l] is not None:
                inp = inp * masks[l]
            out, hn = g(pack_padded_sequence(inp, lens, batch_first=True, enforce_sorted=False))
            inp, _ = pad_packed_sequence(out, batch_first=True, total_length=T)
            hns.append(hn)
        H = self.H
        s = inp[..., :H] + inp[..., H:] if self.D == 2 else inp
        last = hns[-1].sum(0)                                     # forward at t = len - 1, reverse at t = 0
        valid = (torch.arange(T)[None, :] < lens[:, None])[..., None]
        if idx is None:
            mx = s.masked_fill(~valid, float("-inf")).max(dim=1).values
        else:
            mx = s.gather(1, torch.as_tensor(idx, dtype=torch.int64).unsqueeze(1)).squeeze(1)
        av = s.sum(dim=1) / lens[:, None].to(s.dtype)             # s is 0 at padded steps
        return self.linear(torch.cat([last, mx, av], dim=1)), torch.cat(hns), s

    def flat_grads(self):
        """Parameter gradients in the C-ABI order of the flat vector (per layer and direction w_ih, w_hh, b_ih, b_hh; then
        the Linear's weight and bias), as one float64 vector."""
        out = []
        for g in self.layers:
            for sfx in ("l0", "l0_reverse")[:self.D]:
                for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                    out.append(getattr(g, f"{n}_{sfx}").grad.reshape(-1))
        out += [self.linear.weight.grad.reshape(-1), self.linear.bias.grad.reshape(-1)]
        return torch.cat(out)
