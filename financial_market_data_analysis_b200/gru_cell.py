"""``GRUCell``: a drop-in ``torch.nn.GRUCell`` on the H100 kernels of libbigru_b200 (bigru_cell_forward / bigru_cell_backward):
one step at a time, for loops that choose their next input themselves (a decoder over a ``GRU`` encoder, scheduled sampling,
an attention step, one step per new bar in a live path)."""
from __future__ import annotations

from typing import Optional

import torch
import torch.nn as nn

from . import _lib
from ._modelbase import _PRECISIONS, _FlatModel, _resolve_precision, _stream_ptr
from .gru import GRU


class _CellFunction(torch.autograd.Function):
    """autograd boundary: forward and backward are single calls into the C ABI.  Output: h' [B][H]."""

    @staticmethod
    def forward(ctx, mod, x, h, *params):
        lib = _lib.load()
        B, I, H, prec = x.shape[0], mod.input_size, mod.hidden_size, mod._precision_code()
        stash_bytes, scratch_bytes = mod._workspace_bytes(B)
        flat = mod._flat
        with torch.cuda.device(x.device):                 # the C ABI launches on the CURRENT device: make it the model's
            hout = torch.empty(B, H, device=x.device, dtype=torch.float32)
            stash = torch.empty(stash_bytes, dtype=torch.uint8, device=x.device)
            _lib.check(lib.bigru_cell_forward(B, I, H, prec, _lib.ptr(flat), _lib.ptr(x), _lib.ptr(h), _lib.ptr(hout),
                                              _lib.ptr(stash), _stream_ptr(x.device)), "bigru_cell_forward")
        ctx.mod, ctx.prec, ctx.flat, ctx.has_h, ctx.scratch_bytes = mod, prec, flat, h is not None, scratch_bytes
        # the stash through save_for_backward, not a ctx attribute, as GRU keeps its y: a forward that no backward follows
        # frees it on refcount
        ctx.save_for_backward(x, h if h is not None else torch.empty(0, device=x.device), stash)
        return hout

    @staticmethod
    def backward(ctx, dhout):
        lib = _lib.load()
        x, h, stash = ctx.saved_tensors
        h = h if ctx.has_h else None
        B, I, H = x.shape[0], ctx.mod.input_size, ctx.mod.hidden_size
        dhout = dhout.float().contiguous()
        with torch.cuda.device(x.device):
            grads = torch.empty_like(ctx.flat)
            dx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
            dh = torch.empty_like(h) if (h is not None and ctx.needs_input_grad[2]) else None
            scratch = torch.empty(ctx.scratch_bytes, dtype=torch.uint8, device=x.device)
            _lib.check(lib.bigru_cell_backward(B, I, H, ctx.prec, _lib.ptr(ctx.flat), _lib.ptr(x), _lib.ptr(h), _lib.ptr(stash),
                                               _lib.ptr(dhout), _lib.ptr(grads), _lib.ptr(dx), _lib.ptr(dh), _lib.ptr(scratch),
                                               _stream_ptr(x.device)), "bigru_cell_backward")
        ctx.flat = None
        return (None, dx, dh) + ctx.mod._grad_views(grads)


class GRUCell(_FlatModel):
    """``torch.nn.GRUCell`` on libbigru_b200's CUDA kernels (sm_90a).

    The constructor is nn.GRUCell's, plus ``precision`` as in ``GRU`` ("fp32", "bf16x3", "bf16" or "auto"; default
    $BIGRU_B200_PRECISION or "auto", which picks what ``GRU`` picks at this hidden size: "bf16x3" up to 256 hidden units,
    "fp32" beyond).  Every precision takes every shape, an ``hx`` included, with nothing padded.  Parameter names
    (``weight_ih``, ``weight_hh``, ``bias_ih``, ``bias_hh``), registration order and initialisation are nn.GRUCell's, so a
    given ``torch.manual_seed`` gives nn.GRUCell's weights and ``load_state_dict`` works both ways.  The parameter vector is
    that of a ``GRU(input_size, hidden_size, 1)``.  ``bias=False`` and dtypes other than float32 raise ValueError.  There is
    no CPU path.
    """

    _kind = "GRUCell"

    def __init__(self, input_size, hidden_size, bias=True, device=None, dtype=None, precision: Optional[str] = None):
        if not bias:
            raise ValueError("GRUCell: bias=False is not supported (the kernels always add b_ih and b_hh)")
        if dtype is not None and dtype != torch.float32:
            raise ValueError(f"GRUCell: parameters are float32, got dtype={dtype}")
        super().__init__(precision)
        self.input_size, self.hidden_size, self.bias = input_size, hidden_size, True
        kw = {"device": device, "dtype": torch.float32}
        self.weight_ih = nn.Parameter(torch.empty(3 * hidden_size, input_size, **kw))
        self.weight_hh = nn.Parameter(torch.empty(3 * hidden_size, hidden_size, **kw))
        self.bias_ih = nn.Parameter(torch.empty(3 * hidden_size, **kw))
        self.bias_hh = nn.Parameter(torch.empty(3 * hidden_size, **kw))
        self.reset_parameters()
        self._flatten()

    reset_parameters = GRU.reset_parameters

    def _ordered_params(self):
        return [self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh]

    def _adopt(self, flat, views):
        # a cell runs its own shapes: no plans and no padding
        self._flat, self._views = flat, views
        self._ws = {}

    def _precision_code(self) -> int:
        return _PRECISIONS[_resolve_precision(self.precision, self.hidden_size)]

    def _workspace_bytes(self, B):
        """(stash, scratch) bytes of a B-row call, from the library."""
        key = (B, self._precision_code())
        if key not in self._ws:
            a, b = _lib.C.c_size_t(), _lib.C.c_size_t()
            _lib.check(_lib.load().bigru_cell_workspace_bytes(B, self.input_size, self.hidden_size, key[1], _lib.C.byref(a),
                                                              _lib.C.byref(b)), "bigru_cell_workspace_bytes")
            self._ws[key] = (a.value, b.value)
        return self._ws[key]

    def extra_repr(self):
        return f"{self.input_size}, {self.hidden_size}, precision={self.precision!r}"

    def forward(self, input, hx=None):
        """h' as nn.GRUCell: ``input`` [B, I] or unbatched [I], ``hx`` [B, H] / [H] or None (the zero state), at every
        precision.  A wrong number of dimensions raises ValueError, a wrong size RuntimeError, as in nn.GRUCell.

        With grad mode on and anything requiring grad, the call records one autograd node over bigru_cell_forward /
        bigru_cell_backward (gradients for ``input``, ``hx`` and every parameter).  Every other call runs the forward without a
        stash and allocates only h'."""
        if input.dim() not in (1, 2):
            raise ValueError(f"GRUCell: Expected input to be 1D or 2D, got {input.dim()}D instead")
        if hx is not None and hx.dim() not in (1, 2):
            raise ValueError(f"GRUCell: Expected hidden to be 1D or 2D, got {hx.dim()}D instead")
        unbatched = input.dim() == 1
        dev = self._cuda_device()
        x = input.unsqueeze(0) if unbatched else input
        if x.shape[1] != self.input_size:
            raise RuntimeError(f"input has inconsistent input_size: got {x.shape[1]} expected {self.input_size}")
        B = x.shape[0]
        if hx is not None:
            h = hx.unsqueeze(0) if unbatched else hx
            if h.dim() != 2 or h.shape[0] != B:
                raise RuntimeError(f"Input batch size {B} doesn't match hidden0 batch size {h.shape[0]}")
            if h.shape[1] != self.hidden_size:
                raise RuntimeError(f"hidden0 has inconsistent hidden_size: got {h.shape[1]}, expected {self.hidden_size}")
            h = h.to(device=dev, dtype=torch.float32).contiguous()
        else:
            h = None
        x = x.to(device=dev, dtype=torch.float32).contiguous()
        if B == 0:
            out = torch.empty(0, self.hidden_size, device=dev, dtype=torch.float32)
            return out.squeeze(0) if unbatched else out
        params = self._ordered_params()
        if torch.is_grad_enabled() and (x.requires_grad or (h is not None and h.requires_grad)
                                        or any(p.requires_grad for p in params)):
            out = _CellFunction.apply(self, x, h, *params)
        else:
            with torch.no_grad(), torch.cuda.device(dev):
                out = torch.empty(B, self.hidden_size, device=dev, dtype=torch.float32)
                _lib.check(_lib.load().bigru_cell_forward(B, self.input_size, self.hidden_size, self._precision_code(),
                                                          _lib.ptr(self._flat), _lib.ptr(x), _lib.ptr(h), _lib.ptr(out), None,
                                                          _stream_ptr(dev)), "bigru_cell_forward")
        return out.squeeze(0) if unbatched else out
