"""``GRU``: a drop-in ``torch.nn.GRU`` on the H100 kernels of libbigru_b200 (bigru_gru_plan_create / bigru_gru_forward /
bigru_gru_infer / bigru_gru_backward): the recurrence of ``BiGRU`` without its pooling head, for any head or model built on
a GRU encoder."""
from __future__ import annotations

import math
from typing import Optional

import torch
import torch.nn as nn
from torch.nn.utils.rnn import PackedSequence, pack_padded_sequence, pad_packed_sequence

from . import _lib
from ._modelbase import _PRECISIONS, _FlatModel, _PaddedCall, _stream_ptr


class _TrainForward:
    """One bigru_gru_forward call (the training forward: dropout in training mode, a stash for the backward) on the plan of
    x's padded batch.  Keeps what the backward needs; ``outputs()`` are the real rows and units of y and h_n."""

    def __init__(self, mod, x, h0, lengths):
        lib = _lib.load()
        # the C call gets the module's own p (at one layer it drops nothing), except p = 1 at one layer, which the C ABI
        # refuses and nn.GRU ignores there; forward refuses p = 1 wherever it would drop
        self.drop = drop = float(mod.dropout) if mod.dropout < 1 else 0.0
        self.pad = pad = mod._pad
        self.c = c = _PaddedCall(mod, x, h0, lengths, training=mod.training and (drop > 0 or mod.recurrent_dropout > 0))
        plan, D, Hp = c.plan, mod._dims()[1], pad.hidden
        with torch.cuda.device(x.device):                 # the C ABI launches on the CURRENT device: make it the model's
            self.pflat = pflat = mod._plan_params()
            self.y = y = torch.empty(c.Bp, x.shape[1], D * Hp, device=x.device, dtype=torch.float32)
            self.hn = hn = torch.empty(mod.num_layers * D, c.Bp, Hp, device=x.device, dtype=torch.float32)
            self.stash = stash = plan.acquire_stash()
            _lib.check(lib.bigru_gru_forward(plan.handle, _lib.ptr(pflat), _lib.ptr(c.x), _lib.ptr(c.h0), drop,
                                             int(c.training), c.seed, _lib.ptr(stash), _lib.ptr(plan.scratch), _lib.ptr(y),
                                             _lib.ptr(hn), _lib.ptr(c.lengths), _stream_ptr(x.device)), "bigru_gru_forward")

    def outputs(self):
        return self.pad.crop_outputs(self.y, self.c.B), self.pad.crop(self.hn, self.c.B, dim=1, units=True)


class _GRUFunction(torch.autograd.Function):
    """autograd boundary: forward and backward are single calls into the C ABI.  Outputs: y [B][T][D*H] and h_n [L*D][B][H]."""

    @staticmethod
    def forward(ctx, mod, x, h0, lengths, *params):
        f = _TrainForward(mod, x, h0, lengths)
        c = f.c
        ctx.mod, ctx.plan, ctx.stash, ctx.seed, ctx.training, ctx.drop = mod, c.plan, f.stash, c.seed, c.training, f.drop
        ctx.pflat, ctx.real_batch, ctx.has_h0, ctx.lengths = f.pflat, c.B, c.h0 is not None, c.lengths
        # y through save_for_backward, not a ctx attribute: when nothing is padded the output IS y, and an attribute would
        # make output -> grad_fn -> ctx -> output a cycle that keeps the stash alive until the garbage collector runs when no
        # backward follows.  Saving it also checks that nobody modified it in place before the backward reads it.
        ctx.save_for_backward(c.x, c.h0 if c.h0 is not None else torch.empty(0, device=c.x.device), f.y)
        return f.outputs()

    @staticmethod
    def backward(ctx, dy, dhn):
        lib = _lib.load()
        mod, plan, pad = ctx.mod, ctx.plan, ctx.mod._pad
        x, h0, y = ctx.saved_tensors
        h0 = h0 if ctx.has_h0 else None
        Bp = x.shape[0]
        dy = pad.pad_outputs(dy.float(), Bp) if dy is not None else torch.zeros_like(y)
        dhn = None if dhn is None else pad.pad(dhn.float(), Bp, dim=1, units=True)
        grads = torch.empty_like(ctx.pflat)
        dx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        dh0 = torch.empty_like(h0) if (h0 is not None and ctx.needs_input_grad[2]) else None
        with torch.cuda.device(x.device):
            _lib.check(lib.bigru_gru_backward(plan.handle, _lib.ptr(ctx.pflat), _lib.ptr(x), _lib.ptr(h0), ctx.drop,
                                              int(ctx.training), ctx.seed, _lib.ptr(ctx.stash), _lib.ptr(plan.scratch),
                                              _lib.ptr(y), _lib.ptr(dy), _lib.ptr(dhn), _lib.ptr(grads), _lib.ptr(dx),
                                              _lib.ptr(dh0), _lib.ptr(ctx.lengths), _stream_ptr(x.device)), "bigru_gru_backward")
        plan.release_stash(ctx.stash)
        ctx.stash = ctx.pflat = ctx.lengths = None
        return mod._backward_result(grads, dx, dh0, ctx.real_batch)


class GRU(_FlatModel):
    """``torch.nn.GRU`` on libbigru_b200's CUDA kernels (sm_90a).

    The constructor is nn.GRU's, plus ``precision`` as in ``BiGRU`` ("fp32", "bf16x3", "bf16" or "auto"; default
    $BIGRU_B200_PRECISION or "auto": "bf16x3" up to 256 hidden units, zero-padded to 128 / 256, "fp32" beyond).  Attribute and
    parameter names (``weight_ih_l0[_reverse]``, ...), registration order and initialisation are nn.GRU's, so a given
    ``torch.manual_seed`` gives nn.GRU's weights and ``load_state_dict(nn_gru.state_dict())`` works.  ``bias=False``,
    ``proj_size != 0`` and dtypes other than float32 raise ValueError.  There is no CPU path.

    The parameters are views of one flat fp32 vector (``flat_parameters()``), which ``.cuda()`` / ``.to()`` re-pack and
    ``flatten_parameters()`` re-packs on request; a call copies no parameters.  ``BiGRU.gru`` is a GRU whose vector is the
    leading part of the BiGRU's own.

    ``recurrent_dropout`` (p in [0, 1), default 0): variational dropout of the recurrent state, as in ``BiGRU``: in training
    mode one mask per layer, direction, batch row and hidden unit, the same at every step, multiplies the state entering each
    valid step, ``h_t = GRUCell(x_t, m * h_{t-1})``; ``output`` and ``h_n`` are unmasked, and eval mode never masks.  Not a
    parameter; assigning the attribute takes effect at the next call.
    """

    _kind = "GRU"

    def __init__(self, input_size, hidden_size, num_layers=1, bias=True, batch_first=False, dropout=0.0,
                 bidirectional=False, device=None, dtype=None, precision: Optional[str] = None, proj_size=0,
                 recurrent_dropout: float = 0.0):
        if not bias:
            raise ValueError("GRU: bias=False is not supported (the kernels always add b_ih and b_hh)")
        if proj_size != 0:
            raise ValueError("GRU: proj_size is an LSTM option; nn.GRU does not take it either")
        if dtype is not None and dtype != torch.float32:
            raise ValueError(f"GRU: parameters are float32, got dtype={dtype}")
        if not 0 <= float(dropout) <= 1:
            raise ValueError("dropout should be a number in range [0, 1]")
        rd = self._check_recurrent_dropout(recurrent_dropout)
        super().__init__(precision)
        self.recurrent_dropout = rd
        self.mode, self.input_size, self.hidden_size, self.num_layers = "GRU", input_size, hidden_size, num_layers
        self.bias, self.batch_first, self.dropout, self.bidirectional = True, batch_first, float(dropout), bidirectional
        self.proj_size = 0
        dirs = 2 if bidirectional else 1
        kw = {"device": device, "dtype": torch.float32}
        for layer in range(num_layers):
            fan = input_size if layer == 0 else hidden_size * dirs
            for d in range(dirs):
                sfx = f"l{layer}" + ("_reverse" if d else "")
                self.register_parameter(f"weight_ih_{sfx}", nn.Parameter(torch.empty(3 * hidden_size, fan, **kw)))
                self.register_parameter(f"weight_hh_{sfx}", nn.Parameter(torch.empty(3 * hidden_size, hidden_size, **kw)))
                self.register_parameter(f"bias_ih_{sfx}", nn.Parameter(torch.empty(3 * hidden_size, **kw)))
                self.register_parameter(f"bias_hh_{sfx}", nn.Parameter(torch.empty(3 * hidden_size, **kw)))
        self.reset_parameters()
        self._last_seed = 0
        self._flatten()

    def reset_parameters(self):
        """nn.GRU's and nn.GRUCell's initialisation: U(-1/sqrt(H), 1/sqrt(H)), drawn in registration order."""
        bound = 1.0 / math.sqrt(self.hidden_size) if self.hidden_size > 0 else 0.0
        with torch.no_grad():
            for p in self.parameters():
                p.uniform_(-bound, bound)

    @property
    def _flat_weights_names(self):
        return [f"{n}_l{layer}{'_reverse' if d else ''}" for layer in range(self.num_layers)
                for d in range(2 if self.bidirectional else 1) for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]

    @property
    def all_weights(self):
        """Per layer and direction [w_ih, w_hh, b_ih, b_hh], as nn.GRU.all_weights."""
        return [[getattr(self, n) for n in self._flat_weights_names[i:i + 4]] for i in range(0, len(self._flat_weights_names), 4)]

    def _ordered_params(self):
        return [getattr(self, n) for n in self._flat_weights_names]

    def _dims(self):
        return self.hidden_size, 2 if self.bidirectional else 1, self.num_layers, self.input_size, 0

    def _create_plan(self, lib, B, T, out):
        self._create_plan_c(lib, "bigru_gru_plan_create", (B, T, self.input_size, self._pad.hidden, self.num_layers,
                                                           int(self.bidirectional), _PRECISIONS[self._pad.precision]), out)

    def flatten_parameters(self):
        """Re-pack the parameters into one flat vector when they are not views of it any more (nn.GRU's name for it)."""
        if not self._is_flat():
            self._flatten()

    def extra_repr(self):
        s = f"{self.input_size}, {self.hidden_size}"
        if self.num_layers != 1:
            s += f", num_layers={self.num_layers}"
        if self.batch_first:
            s += ", batch_first=True"
        if self.dropout:
            s += f", dropout={self.dropout}"
        if self.bidirectional:
            s += ", bidirectional=True"
        if self.recurrent_dropout:
            s += f", recurrent_dropout={self.recurrent_dropout}"
        return s + f", precision={self.precision!r}"

    def forward(self, input, hx=None, lengths=None):
        """(output, h_n) as nn.GRU.

        ``input``: [T, B, F], [B, T, F] with ``batch_first``, unbatched [T, F], or a ``PackedSequence`` (then ``output`` is
        packed the same way).  The kernels read batch-major rows: ``batch_first=True`` passes the input as it is, while
        ``batch_first=False`` costs a transposing copy of the input and of the output.  ``hx``: [L*D, B, H] (or [L*D, H]
        unbatched); a wrong shape raises RuntimeError.  ``lengths`` ([B] integers in [1, T]): row b is that many steps long, as
        in ``BiGRU.forward``; ``output`` is 0 at later steps and ``h_n`` holds each direction's state after its last valid step.
        ``hx`` together with ``lengths`` (or a PackedSequence), and ``hx`` at precision "bf16", raise ValueError.

        With grad mode on and anything requiring grad, the call records one autograd node over bigru_gru_forward /
        bigru_gru_backward (gradients for the parameters, ``input`` and ``hx``).  In training mode, ``dropout`` drops each
        layer's output but the last's, as nn.GRU does, with or without grad mode; ``dropout = 1`` cannot be run there
        (ValueError).  Every other call runs bigru_gru_infer, and the plan holds only its inference workspace."""
        packed = isinstance(input, PackedSequence)
        if packed:
            if lengths is not None:
                raise ValueError("GRU: a PackedSequence carries its own lengths; do not pass lengths as well")
            x, lens = pad_packed_sequence(input, batch_first=True)           # rows in the caller's order
            lengths = lens
            unbatched = False
        else:
            if input.dim() not in (2, 3):
                raise ValueError(f"GRU: Expected input to be 2D or 3D, got {input.dim()}D instead")
            unbatched = input.dim() == 2
            x = input.unsqueeze(0) if unbatched else (input if self.batch_first else input.transpose(0, 1))
        if x.shape[-1] != self.input_size:
            raise RuntimeError(f"input.size(-1) must be equal to input_size. Expected {self.input_size}, got {x.shape[-1]}")
        if hx is not None:
            if unbatched:
                if hx.dim() != 2:
                    raise RuntimeError(f"For unbatched 2-D input, hx should also be 2-D but got {hx.dim()}-D tensor")
                hx = hx.unsqueeze(1)
            elif hx.dim() != 3:
                raise RuntimeError(f"For batched 3-D input, hx should also be 3-D but got {hx.dim()}-D tensor")
            if self._pad.precision == "bf16":
                raise ValueError("GRU: an initial hidden state is not supported at precision 'bf16'; use 'bf16x3' or 'fp32'")
        xs, h0 = self._prepare_input(x, hx)
        lens = self._prepare_lengths(lengths, xs, hx)
        if self._drops() and self.dropout >= 1:
            raise ValueError("GRU: dropout = 1 in training mode is not supported (the kernels take p in [0, 1))")
        params = self._ordered_params()
        if torch.is_grad_enabled() and (xs.requires_grad or (h0 is not None and h0.requires_grad)
                                        or any(p.requires_grad for p in params)):
            y, hn = _GRUFunction.apply(self, xs, h0, lens, *params)
        elif self._drops() or self._masks():              # nn.GRU drops in training mode without grad mode too
            with torch.no_grad():
                f = _TrainForward(self, xs, h0, lens)
                f.c.plan.release_stash(f.stash)
                y, hn = f.outputs()
        else:
            y, hn = self._infer(xs, h0, lens)
        if packed:
            return self._repack(y, lengths, input), hn
        if unbatched:
            return y.squeeze(0), hn.squeeze(1)
        return (y if self.batch_first else y.transpose(0, 1).contiguous()), hn

    def _drops(self) -> bool:
        """Whether a call drops anything: training mode, dropout > 0 and a layer above the first."""
        return bool(self.training and self.dropout > 0 and self.num_layers > 1)

    def _masks(self) -> bool:
        """Whether a call masks the recurrent state: training mode and recurrent_dropout > 0."""
        return bool(self.training and self.recurrent_dropout > 0)

    def _infer(self, x, h0, lengths):
        """(y, h_n) of the real rows through bigru_gru_infer, without an autograd record."""
        pad, c = self._pad, _PaddedCall(self, x, h0, lengths)
        D, Hp = self._dims()[1], pad.hidden
        with torch.no_grad(), torch.cuda.device(x.device):
            pflat = self._plan_params()               # held until the call has been queued: padded plans get a fresh vector
            y = torch.empty(c.Bp, x.shape[1], D * Hp, device=x.device, dtype=torch.float32)
            hn = torch.empty(self.num_layers * D, c.Bp, Hp, device=x.device, dtype=torch.float32)
            _lib.check(_lib.load().bigru_gru_infer(c.plan.handle, _lib.ptr(pflat), _lib.ptr(c.x), _lib.ptr(c.h0),
                                                   _lib.ptr(c.plan.infer_workspace()), _lib.ptr(y), _lib.ptr(hn),
                                                   _lib.ptr(c.lengths), _stream_ptr(x.device)), "bigru_gru_infer")
        return pad.crop_outputs(y, c.B), pad.crop(hn, c.B, dim=1, units=True)

    @staticmethod
    def _repack(y, lens, like):
        """y [B][T][D*H] (rows in the caller's order) packed as `like`: its sorting, batch sizes and index tensors.  lens:
        the host lengths pad_packed_sequence returned, in the caller's order."""
        idx = like.sorted_indices
        ys = y if idx is None else y.index_select(0, idx.to(y.device))
        p = pack_padded_sequence(ys, torch.sort(lens, descending=True).values, batch_first=True, enforce_sorted=True)
        return PackedSequence(p.data, p.batch_sizes, like.sorted_indices, like.unsorted_indices)
