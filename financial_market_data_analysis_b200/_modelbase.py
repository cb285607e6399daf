"""What ``BiGRU``, ``GRU`` and ``GRUCell`` share: the zero padding between a model's shapes and its C plans' (``_Padding``),
the plans and their workspaces (``_Plan``), one C call's padded inputs, plan and dropout seed (``_PaddedCall``), and the
single flat fp32 parameter vector the C ABI reads (``_FlatModel``)."""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from . import _lib

_PRECISIONS = {"fp32": _lib.PREC_FP32, "bf16": _lib.PREC_BF16, "bf16x3": _lib.PREC_BF16X3}


def _resolve_precision(precision: str, hidden: int) -> str:
    """The precision a model of `hidden` units runs at: "auto" is "bf16x3" up to 256 hidden units, "fp32" beyond."""
    return precision if precision != "auto" else ("bf16x3" if hidden <= 256 else "fp32")


def _stream_ptr(device=None):
    """Raw cudaStream_t of torch's current stream ON THE MODEL'S DEVICE (not the process-wide current device)."""
    return torch.cuda.current_stream(device).cuda_stream


class _Padding:
    """What the C plans of one model run at, and the zero padding between the model's own shapes and the plan's.

    The tensor-core kernels exist for whole batch tiles (32 rows at "bf16x3" and at "bf16" with 512 hidden units, 16 rows
    otherwise at "bf16") and for 128 / 256 (/ 512 at "bf16") hidden units.  Other batch sizes run with zero rows appended:
    batch rows are independent and the padded rows receive a zero upstream gradient.  Smaller hidden sizes run with zero
    units appended (see BiGRU.plan_hidden).  Logits, loss and every gradient of the real rows and parameters are those of
    the unpadded model (up to summation order).  dims: (hidden, directions, layers, features, head outputs); a GRU has no
    head (0 outputs) and its parameter map is the recurrent prefix of BiGRU's."""

    def __init__(self, dims, precision, device):
        H = dims[0]
        prec = _resolve_precision(precision, H)
        sizes = {"bf16x3": (128, 256), "bf16": (128, 256, 512)}.get(prec, ())
        self.precision = prec
        self.hidden = next((hp for hp in sizes if H <= hp), H)
        self.tile = 32 if (prec == "bf16x3" or (prec == "bf16" and self.hidden == 512)) else (16 if prec == "bf16" else 1)
        self.padded = self.hidden != H
        self._dims = tuple(dims)
        self._device = device
        self._index = None

    def batch(self, B: int) -> int:
        """The batch size a plan runs for B real rows."""
        return (B + self.tile - 1) // self.tile * self.tile

    def pad(self, t, Bp, dim=0, units=False):
        """t with zero rows appended along `dim` up to Bp and, when `units`, zero hidden units up to the plan's (last dim),
        contiguous as the C ABI reads it."""
        if t is None:
            return None
        shape = list(t.shape)
        shape[dim] = Bp
        if units:
            shape[-1] = self.hidden
        if list(t.shape) == shape:
            return t.contiguous()
        out = t.new_zeros(shape)
        out[tuple(slice(0, n) for n in t.shape)] = t
        return out

    def lengths(self, lens, Bp, T):
        """Per-row lengths [Bp] of a plan: `lens` (None stays None) with the appended zero rows T steps long."""
        if lens is None or lens.shape[0] == Bp:
            return lens
        out = lens.new_full((Bp,), T)
        out[:lens.shape[0]] = lens
        return out

    def crop(self, t, B, dim=0, units=False):
        """The first B rows along `dim` of a plan-sized tensor and, when `units`, its real hidden units."""
        if t is None:
            return None
        if units and t.shape[-1] != self._dims[0]:
            t = t[..., :self._dims[0]]
        return t if t.shape[dim] == B else t.narrow(dim, 0, B)

    def crop_outputs(self, y, B):
        """The real rows and units of a plan's layer output [Bp][T][D*Hp]: direction d's units are plan columns d*Hp + j."""
        H, D = self._dims[0], self._dims[1]
        y = self.crop(y, B)
        if not self.padded:
            return y
        return y.view(B, y.shape[1], D, self.hidden)[..., :H].reshape(B, y.shape[1], D * H)

    def pad_outputs(self, dy, Bp):
        """A gradient of the real outputs [B][T][D*H] as the plan's [Bp][T][D*Hp], zero in the padded rows and units."""
        H, D = self._dims[0], self._dims[1]
        B, T = dy.shape[0], dy.shape[1]
        if not self.padded:
            return self.pad(dy, Bp)
        out = dy.new_zeros(Bp, T, D, self.hidden)
        out[:B, :, :, :H] = dy.reshape(B, T, D, H)
        return out.view(Bp, T, D * self.hidden)

    def _map(self):
        """(index tensor, padded parameter count): position of every real parameter inside the padded plan's flat vector."""
        if self._index is None:
            H, D, L, F, C = self._dims
            Hp = self.hidden
            idx, off_p = [], 0

            def rows(n_cols_pad, col_map):
                # a [3H][cols] block -> padded [3Hp][cols_pad]: row g*H + j -> g*Hp + j, column through col_map
                r = (np.arange(3)[:, None] * Hp + np.arange(H)[None, :]).reshape(-1)
                return (r[:, None] * n_cols_pad + col_map[None, :]).reshape(-1)

            for l in range(L):
                Ip = F if l == 0 else D * Hp
                cm = np.arange(F) if l == 0 else (np.arange(D)[:, None] * Hp + np.arange(H)[None, :]).reshape(-1)
                for d in range(D):
                    idx.append(off_p + rows(Ip, cm)); off_p += 3 * Hp * Ip                         # W_ih
                    idx.append(off_p + rows(Hp, np.arange(H))); off_p += 3 * Hp * Hp               # W_hh
                    b = (np.arange(3)[:, None] * Hp + np.arange(H)[None, :]).reshape(-1)
                    idx.append(off_p + b); off_p += 3 * Hp                                        # b_ih
                    idx.append(off_p + b); off_p += 3 * Hp                                        # b_hh
            cmh = (np.arange(3)[:, None] * Hp + np.arange(H)[None, :]).reshape(-1)                # head: last | max | avg, H wide each
            idx.append(off_p + (np.arange(C)[:, None] * 3 * Hp + cmh[None, :]).reshape(-1)); off_p += C * 3 * Hp
            idx.append(off_p + np.arange(C)); off_p += C
            self._index = (torch.from_numpy(np.concatenate(idx).astype(np.int64)).to(self._device), off_p)
        return self._index

    def params(self, flat, out=None):
        """The flat parameter vector as the plan sees it: `flat` itself, or its entries scattered into a zero-padded vector
        (`out` when given; its padded entries must be zero)."""
        if not self.padded:
            return flat
        index, n = self._map()
        assert index.numel() == flat.numel()
        if out is None:
            out = flat.new_zeros(n)
        return out.index_copy_(0, index, flat.detach())

    def grads(self, pgrad, out=None):
        """The real parameters' entries of a plan-sized gradient vector (into `out` when given)."""
        if not self.padded:
            return pgrad
        return torch.index_select(pgrad, 0, self._map()[0], out=out) if out is not None else torch.index_select(pgrad, 0, self._map()[0])


class _Plan:
    """A C plan plus its device workspaces for one (B, T) shape.  The model makes the create call (``_create_plan``:
    bigru_plan_create for BiGRU, bigru_gru_plan_create for GRU).  Each workspace is allocated on first use: a plan that only
    runs inference holds the inference workspace alone, not the stash and scratch of the training forward."""

    def __init__(self, model, B: int, T: int, device):
        lib = _lib.load()
        _lib.check(lib.bigru_device_check(device.index if device.index is not None else torch.cuda.current_device()),
                   "bigru_device_check")
        h = _lib.C.c_void_p()
        model._create_plan(lib, B, T, h)
        self.handle, self.B, self.T, self.device = h, B, T, device
        a, b, c = _lib.C.c_size_t(), _lib.C.c_size_t(), _lib.C.c_size_t()
        _lib.check(lib.bigru_workspace_bytes(h, _lib.C.byref(a), _lib.C.byref(b)), "bigru_workspace_bytes")
        _lib.check(lib.bigru_infer_workspace_bytes(h, _lib.C.byref(c)), "bigru_infer_workspace_bytes")
        self.stash_bytes, self.scratch_bytes, self.infer_bytes = a.value, b.value, c.value
        self._scratch = self._infer_ws = None
        self._free_stash = []

    @property
    def scratch(self):
        if self._scratch is None:
            self._scratch = torch.empty(max(self.scratch_bytes, 16), dtype=torch.uint8, device=self.device)
        return self._scratch

    def infer_workspace(self):
        if self._infer_ws is None:
            self._infer_ws = torch.empty(max(self.infer_bytes, 16), dtype=torch.uint8, device=self.device)
        return self._infer_ws

    def acquire_stash(self):
        if self._free_stash:
            return self._free_stash.pop()
        return torch.empty(max(self.stash_bytes, 16), dtype=torch.uint8, device=self.device)

    def release_stash(self, s):
        if len(self._free_stash) < 2:
            self._free_stash.append(s)

    def __del__(self):
        try:
            if self.handle:
                _lib.load().bigru_plan_destroy(self.handle)
        except Exception:
            pass


class _PaddedCall:
    """What one C call of a plan-running model gets from the real x [B][T][F], h0 [L*D][B][H] and lengths [B] (None: no
    initial state, every row T steps): the real batch ``B``, the plan's batch ``Bp`` (the model's _Padding rule unless
    given), ``x``, ``h0`` and ``lengths`` zero-padded to it, and the ``plan`` of Bp rows.

    A training forward passes ``training``, the dropout flag of its C call: it gets the dropout ``seed``, drawn from torch's
    host generator when the flag is set and 0 otherwise, and recorded as ``model._last_seed``.  Without ``training``
    (inference) no seed is drawn and ``_last_seed`` is left as it is."""

    def __init__(self, model, x, h0, lengths, training=None, Bp=None):
        pad = model._pad
        self.B = x.shape[0]
        self.Bp = Bp = pad.batch(self.B) if Bp is None else Bp
        self.x, self.h0 = pad.pad(x, Bp), pad.pad(h0, Bp, dim=1, units=True)
        self.lengths = pad.lengths(lengths, Bp, x.shape[1])
        self.plan = model._plan_for(self.x)
        self.training, self.seed = bool(training), 0
        if training is not None:
            if training:                                  # the dropout masks are a pure function of (seed, layer, element)
                self.seed = int(torch.randint(0, 2 ** 62, (1,)).item())
            model._last_seed = self.seed


class _FlatModel(nn.Module):
    """A module whose parameters are views of one contiguous fp32 vector in the C ABI's order (``_ordered_params``), with
    the plans that run it.  Subclasses give ``_dims()`` (hidden, directions, layers, features, head outputs),
    ``_create_plan`` and ``_ordered_params``, and pass ``precision`` to the constructor."""

    _kind = "model"

    def __init__(self, precision: Optional[str]):
        """``precision``: "fp32", "bf16x3", "bf16" or "auto"; None reads $BIGRU_B200_PRECISION (default "auto")."""
        super().__init__()
        self.precision = precision or os.environ.get("BIGRU_B200_PRECISION", "auto")
        if self.precision != "auto" and self.precision not in _PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_PRECISIONS) + ['auto']}")

    def _flatten(self):
        """(Re)pack every parameter into one contiguous vector and make the nn.Parameters views of it,
        keeping the Parameter objects (optimisers hold references to them)."""
        params = self._ordered_params()
        dev = params[0].device
        flat = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=dev)
        views, off = [], 0
        with torch.no_grad():
            for p in params:
                n = p.numel()
                flat[off:off + n].copy_(p.detach().reshape(-1).to(device=dev, dtype=torch.float32))
                p.data = flat[off:off + n].view(p.shape)
                views.append((off, n, tuple(p.shape)))
                off += n
        self._adopt(flat, views)

    def _adopt(self, flat, views):
        """`flat` (whose ranges `views` the parameters already are) becomes this model's flat vector; plans start afresh."""
        self._flat, self._views = flat, views
        self._pad = _Padding(self._dims(), self.precision, flat.device)
        self._plans = {}

    def _is_flat(self):
        f = getattr(self, "_flat", None)
        if f is None:
            return False
        base = f.data_ptr()
        for p, (off, n, _) in zip(self._ordered_params(), self._views):
            if p.device != f.device or p.dtype != torch.float32 or p.data_ptr() != base + 4 * off:
                return False
        return True

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)       # .cuda() / .to() create fresh tensors per parameter
        self._flatten()
        return out

    def flat_parameters(self) -> torch.Tensor:
        if not self._is_flat():
            self._flatten()
        return self._flat

    def _plan_params(self, out=None):
        """The flat parameter vector as the C plan sees it (zero-padded hidden units scattered in when the plan pads them)."""
        return self._pad.params(self._flat, out)

    def _plan_grads(self, pgrad, out=None):
        """The real parameters' entries of a plan-sized gradient vector."""
        return self._pad.grads(pgrad, out)

    def _grad_views(self, grads):
        """Each parameter's gradient as a view of a gradient vector in the flat vector's order."""
        return tuple(grads[o:o + n].view(shape) for (o, n, shape) in self._views)

    def _backward_result(self, pgrad, dx, dh0, B):
        """What the autograd backward of (model, x, h0, lengths, *params) returns from the plan-sized gradient vector and
        dx / dh0 of the padded batch: dx and dh0 cropped to the B real rows and units, and views of the real entries."""
        pad = self._pad
        return (None, pad.crop(dx, B), pad.crop(dh0, B, dim=1, units=True), None) + self._grad_views(self._plan_grads(pgrad))

    def _plan_for(self, x) -> _Plan:
        # plans are keyed by the recurrent dropout p too: assigning model.recurrent_dropout takes effect at the next call
        key = (int(x.shape[0]), int(x.shape[1]), self._pad.precision, x.device.index, float(getattr(self, "recurrent_dropout", 0.0)))
        plan = self._plans.get(key)
        if plan is None:
            if len(self._plans) > 8:
                self._plans.clear()
            plan = self._plans[key] = _Plan(self, key[0], key[1], x.device)
        return plan

    @staticmethod
    def _check_recurrent_dropout(p) -> float:
        """The recurrent dropout p as a float in [0, 1) (ValueError otherwise)."""
        p = float(p)
        if not 0.0 <= p < 1.0:
            raise ValueError(f"recurrent_dropout must be in [0, 1), got {p}")
        return p

    def _create_plan_c(self, lib, creator, args, out):
        """`creator`(*args, out), or its *_rd twin when the model has recurrent dropout (DESIGN.md §4.8)."""
        rd = self._check_recurrent_dropout(getattr(self, "recurrent_dropout", 0.0))
        if rd > 0:
            _lib.check(getattr(lib, creator + "_rd")(*args, rd, _lib.C.byref(out)), creator + "_rd")
        else:
            _lib.check(getattr(lib, creator)(*args, _lib.C.byref(out)), creator)

    def _cuda_device(self):
        """The device of the flat parameter vector (re-packed first if needed), which must be a CUDA device."""
        dev = self.flat_parameters().device
        if dev.type != "cuda":
            raise RuntimeError(f"{self._kind} (H100-native) has no CPU path: move the model to a CUDA device with .cuda() first")
        return dev

    def _prepare_input(self, input_seq, hidden):
        """input_seq [B, T, F] and hidden [L*D, B, H] (or None) as contiguous fp32 tensors on the model's device."""
        dev = self._cuda_device()
        H, D, L, F, _ = self._dims()
        if input_seq.dim() != 3 or input_seq.shape[2] != F:
            raise ValueError(f"input_seq must be [batch, seq_len, {F}], got {tuple(input_seq.shape)}")
        x = input_seq.to(device=dev, dtype=torch.float32, non_blocking=True).contiguous()
        h0 = None
        if hidden is not None:
            want = (L * D, x.shape[0], H)
            if tuple(hidden.shape) != want:
                raise RuntimeError(f"Expected hidden size {want}, got {tuple(hidden.shape)}")
            h0 = hidden.to(device=dev, dtype=torch.float32).contiguous()
        return x, h0

    @staticmethod
    def _prepare_lengths(lengths, x, hidden):
        """`lengths` (a list, a CPU or a CUDA tensor of integers) as an int32 tensor [B] on x's device, checked on the host:
        shape [B], every value in [1, T], and no initial state with it.  None stays None (every row T steps long)."""
        if lengths is None:
            return None
        if hidden is not None:
            raise ValueError("lengths together with an initial hidden state (hidden) are not supported")
        B, T = int(x.shape[0]), int(x.shape[1])
        host = lengths.detach().cpu() if isinstance(lengths, torch.Tensor) else torch.as_tensor(lengths)
        if host.dtype.is_floating_point or host.dtype.is_complex or host.dtype == torch.bool:
            raise ValueError(f"lengths must hold integers, got {host.dtype}")
        if tuple(host.shape) != (B,):
            raise ValueError(f"lengths must have shape [{B}] (one per batch row), got {tuple(host.shape)}")
        if B and (int(host.min()) < 1 or int(host.max()) > T):
            raise ValueError(f"every length must lie in [1, {T}], got values from {int(host.min())} to {int(host.max())}")
        # from pinned memory, so that the copy does not wait for the work already queued on the stream
        return host.to(torch.int32).pin_memory().to(x.device, non_blocking=True)
