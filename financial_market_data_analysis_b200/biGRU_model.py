"""H100-native drop-in for the reference's ``biGRU_model`` module.

``BiGRU`` keeps the class surface of /root/reference/biGRU_model.py:8-286 - constructor
argument order (:32-33), attribute names (:39-47), submodule names ``dropout`` /
``spatial_dropout1d`` / ``gru`` / ``linear`` (so ``model_params.pt`` loads unchanged),
``forward(input_seq, hidden=None)`` (:63), ``add_loss_fn`` / ``add_optimizer`` / ``add_device``
(:141-159), ``train_model`` (:162) and ``evaluate_model`` (:227) with the same return tuples -
but every floating-point operation of forward/backward, the loss, gradient clipping and the
Adam update run in hand-written sm_90a CUDA kernels behind the C ABI of
``libbigru_b200.so`` (include/bigru_b200.h).  PyTorch only owns device memory, streams and the
process group.  There is no CPU path: parameters must live on a CUDA device.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch
import torch.nn as nn

if __package__:
    from . import _lib
    from ._modelbase import _PRECISIONS, _FlatModel, _PaddedCall, _stream_ptr
    from .gru import GRU
    from .parallel import allreduce_flat_
else:
    # drop-in route of the reference's callers (`predict.py:16`, the notebook): this directory itself is on sys.path and
    # the module is imported top-level as `biGRU_model`; bind the sibling modules through the package
    import importlib as _importlib
    import sys as _sys
    _here = os.path.dirname(os.path.abspath(__file__))
    if os.path.dirname(_here) not in _sys.path:
        _sys.path.insert(0, os.path.dirname(_here))
    _lib = _importlib.import_module(os.path.basename(_here) + "._lib")
    _base = _importlib.import_module(os.path.basename(_here) + "._modelbase")
    _PRECISIONS, _FlatModel, _PaddedCall, _stream_ptr = _base._PRECISIONS, _base._FlatModel, _base._PaddedCall, _base._stream_ptr
    GRU = _importlib.import_module(os.path.basename(_here) + ".gru").GRU
    allreduce_flat_ = _importlib.import_module(os.path.basename(_here) + ".parallel").allreduce_flat_

class _AdamState:
    """Optimiser state of the fused step.  The flat gradient and the scalar loss share one buffer (``gext`` = P gradients + 1
    loss), so that data parallelism needs exactly one all-reduce per step.  Adam's step count lives on the device too
    (``dstep``), so that a captured CUDA graph of the step stays valid from one step to the next; ``step`` counts on the host.
    So do the hyperparameters of each parameter group (``hyper``, bigru_adam_group rows) and the group of each parameter
    tensor (``segs``, bigru_adam_segment rows over the flat vector): a learning-rate schedule changes a table entry, not
    the captured graph."""

    def __init__(self, flat, pad, n_tensors):
        P, dev = flat.numel(), flat.device
        self.gext = torch.empty(P + 1, device=dev, dtype=torch.float32)
        self.grad, self.loss = self.gext[:P], self.gext[P:P + 1]
        self.m, self.v = torch.zeros_like(flat), torch.zeros_like(flat)
        self.step, self.dstep = 0, torch.zeros(1, device=dev, dtype=torch.int32)
        self.scal = torch.zeros(2, device=dev, dtype=torch.float32)
        self.sqws = torch.empty(_lib.SQNORM_WS, device=dev, dtype=torch.float32)
        # the plan's own parameter / gradient vectors: zero-padded ones when the plan pads hidden units, else the flat ones
        self.pflat = pad.params(flat)
        self.pgrad = torch.empty_like(self.pflat) if pad.padded else self.grad
        self.mirror_steps = []           # optimizer.state[p]["step"] tensors, kept equal to `step`
        self.hyper = torch.zeros(_lib.ADAM_MAX_GROUPS, _lib.ADAM_GROUP_FIELDS, device=dev, dtype=torch.float32)
        self.segs = torch.zeros(n_tensors, 3, device=dev, dtype=torch.int64)
        self.hyper_rows = self.seg_rows = None   # what the last load_tables enqueued

    def load_tables(self, hyper_rows, seg_rows):
        """Enqueue on the current stream a copy of each table that differs from what the previous call enqueued.  The
        host rows go through pinned memory, which torch keeps alive until the asynchronous copy has read it: no host
        synchronisation, and the copy runs before whatever the stream runs next (the step, or its graph replay)."""
        for rows, dst, dt, attr in ((hyper_rows, self.hyper, torch.float32, "hyper_rows"),
                                    (seg_rows, self.segs, torch.int64, "seg_rows")):
            if rows != getattr(self, attr):
                dst[:len(rows)].copy_(torch.tensor(rows, dtype=dt).pin_memory(), non_blocking=True)
                setattr(self, attr, rows)

    def __getitem__(self, name):
        """Read access by name (``st["grad"]``) for callers that index the state like a dict."""
        return getattr(self, name)

    def advance(self):
        """Host-side bookkeeping of one executed step (the device counter advances inside bigru_adam_tick)."""
        self.step += 1
        if self.mirror_steps:
            torch._foreach_add_(self.mirror_steps, 1.0)


class _StepBuffers:
    """What one fused train step reads and writes: its padded call `c` (plan, padded inputs and lengths, dropout seed) and a
    stash of the plan's pool, the targets of the real rows, the loss arguments and logits / dlogits of the padded batch."""

    def __init__(self, c, tgt, loss, C):
        self.c, self.stash, self.tgt, self.loss = c, c.plan.acquire_stash(), tgt, loss
        self.logits = torch.empty(c.Bp, C, device=c.x.device, dtype=torch.float32)
        # the loss writes dlogits of the real rows only: the padded rows stay zero
        self.dlogits = (torch.zeros if c.Bp != tgt.shape[0] else torch.empty)(c.Bp, C, device=c.x.device, dtype=torch.float32)


class _BiGRUFunction(torch.autograd.Function):
    """autograd boundary: forward/backward are single calls into the C ABI."""

    @staticmethod
    def forward(ctx, model, x, h0, lengths, *params):
        pad = model._pad
        c = _PaddedCall(model, x, h0, lengths, training=model._draws_masks())
        with torch.cuda.device(x.device):                 # the C ABI launches on the CURRENT device: make it the model's
            pflat = model._plan_params()
            logits = torch.empty(c.Bp, model.output_size, device=x.device, dtype=torch.float32)
            hn = torch.empty(model.n_layers * model.n_directions, c.Bp, pad.hidden, device=x.device, dtype=torch.float32)
            stash = c.plan.acquire_stash()
            model._forward_c(c.plan, pflat, c.x, c.h0, c.lengths, c.training, c.seed, stash, logits, hn, _stream_ptr(x.device))
            model._last_hidden = pad.crop(hn, c.B, dim=1, units=True)
            model._last_forward = (c.plan, stash, c.B)
            if any(ctx.needs_input_grad):                 # grad mode is off inside Function.forward; ask the ctx
                ctx.model, ctx.plan, ctx.stash, ctx.seed, ctx.training = model, c.plan, stash, c.seed, c.training
                ctx.pflat, ctx.real_batch, ctx.has_h0, ctx.lengths = pflat, c.B, c.h0 is not None, c.lengths
                ctx.save_for_backward(c.x, c.h0 if c.h0 is not None else torch.empty(0, device=x.device))
            else:
                c.plan.release_stash(stash)
            return pad.crop(logits, c.B)

    @staticmethod
    def backward(ctx, dlogits):
        model, plan = ctx.model, ctx.plan
        x, h0 = ctx.saved_tensors
        h0 = h0 if ctx.has_h0 else None
        dlogits = model._pad.pad(dlogits.float(), x.shape[0])             # padded rows: zero upstream gradient
        grads = torch.empty_like(ctx.pflat)
        dx = torch.empty_like(x) if ctx.needs_input_grad[1] else None
        dh0 = torch.empty_like(h0) if (h0 is not None and ctx.needs_input_grad[2]) else None
        with torch.cuda.device(x.device):
            model._backward_c(plan, ctx.pflat, x, h0, ctx.lengths, ctx.training, ctx.seed, ctx.stash, dlogits, grads, dx, dh0,
                              _stream_ptr(x.device))
        plan.release_stash(ctx.stash)
        ctx.stash = ctx.pflat = ctx.lengths = None
        return model._backward_result(grads, dx, dh0, ctx.real_batch)


class BiGRU(_FlatModel):
    """Bidirectional GRU classifier (reference: biGRU_model.py:8).

    Parameters (same order and defaults as the reference, :32-33): hidden_size, n_features,
    output_size, n_layers=1, clip=50, dropout=0.2, spatial_dropout=True, bidirectional=True.
    Extra keyword ``precision``:
      "fp32"    FFMA kernels, exact transcendental functions; any shape (the exact path),
      "bf16x3"  fp32-class on tensor cores (every operand a (hi, lo) bf16 pair, fp32 accumulation / state /
                gradients): meets the reference's 1e-4 logits tolerance; H in {128, 256} (other batch sizes than whole 32-row tiles
                run zero-padded, any feature count),
      "bf16"    single bf16 operands on tensor cores, fp32 accumulation and state (fastest, ~3e-3 on logits); H in {128, 256, 512},
      "auto"    "bf16x3" for hidden sizes up to 256 (smaller models run zero-padded to 128 / 256 hidden units), "fp32" beyond.
    Default: $BIGRU_B200_PRECISION or "auto" (the reference tolerance at tensor-core speed wherever the kernels apply).
    Extra keyword ``recurrent_dropout`` (p in [0, 1), default 0): variational dropout of the recurrent state (Gal &
    Ghahramani, 2016; Keras' ``recurrent_dropout``).  In a training-mode forward every layer and direction draws one mask
    m[b, j] in {0, 1/(1-p)} per batch row and hidden unit, the same at every step, and each valid step runs
    ``h_t = GRUCell(x_t, m * h_{t-1})``; layer outputs and the final state are unmasked, padded steps are not masked, and
    eval mode and ``infer`` never mask.  It is not a parameter (state_dict is unchanged); assigning the attribute takes
    effect at the next call.
    """

    def __init__(self, hidden_size, n_features, output_size, n_layers=1, clip=50, dropout=0.2,
                 spatial_dropout=True, bidirectional=True, precision: Optional[str] = None, recurrent_dropout: float = 0.0):
        rd = self._check_recurrent_dropout(recurrent_dropout)
        super().__init__(precision)
        self.recurrent_dropout = rd
        self.hidden_size = hidden_size
        self.n_features = n_features
        self.output_size = output_size
        self.n_layers = n_layers
        self.clip = clip
        self.dropout_p = dropout
        self.spatial_dropout = spatial_dropout
        self.bidirectional = bidirectional
        self.n_directions = 2 if bidirectional else 1

        # same submodule names and construction order as the reference (:50-60) so that a given
        # torch.manual_seed produces the same initial weights and state_dict keys
        self.dropout = nn.Dropout(self.dropout_p)
        if self.spatial_dropout:
            self.spatial_dropout1d = nn.Dropout2d(self.dropout_p)
        self.gru = GRU(n_features, hidden_size, n_layers, batch_first=True, dropout=0 if n_layers == 1 else dropout,
                       bidirectional=bidirectional, precision=self.precision)
        self.linear = nn.Linear(hidden_size * 3, output_size)

        self.device = torch.device("cpu")
        self.loss_fn = None
        self.optimizer = None
        self._flat = None            # all parameters, one contiguous fp32 vector (C-ABI order)
        self._views = []             # (offset, numel, shape) per parameter in C-ABI order
        self._plans = {}
        self._adam = None            # fused-step optimiser state (_AdamState)
        self._dp_group = None
        self._dp_world = 1
        self._last_hidden = None
        self._last_forward = None    # (plan, stash, real batch) of the last forward
        self._last_seed = 0
        self._graphs = {}
        self.use_cuda_graph = os.environ.get("BIGRU_B200_CUDA_GRAPH", "1") != "0"
        self._loss_cache = {}
        self._flatten()

    # ------------------------------------------------------------------ parameter storage
    def _ordered_params(self):
        out = []
        for layer in range(self.n_layers):
            for d in range(self.n_directions):
                sfx = f"l{layer}" + ("_reverse" if d else "")
                for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh"):
                    out.append(getattr(self.gru, f"{n}_{sfx}"))
        out += [self.linear.weight, self.linear.bias]
        return out

    _kind = "BiGRU"

    def _dims(self):
        return self.hidden_size, self.n_directions, self.n_layers, self.n_features, self.output_size

    def _create_plan(self, lib, B, T, out):
        self._create_plan_c(lib, "bigru_plan_create", (B, T, self.n_features, self.plan_hidden(B), self.n_layers, self.output_size,
                                                       int(self.bidirectional), _PRECISIONS[self.resolved_precision(B)]), out)

    def _draws_masks(self) -> bool:
        """Whether a forward draws dropout noise (and a seed): training mode with input, spatial, inter-layer or recurrent
        dropout."""
        return bool(self.training and (self.dropout_p > 0 or self.recurrent_dropout > 0))

    def extra_repr(self):
        return f"recurrent_dropout={self.recurrent_dropout}" if self.recurrent_dropout else ""

    def _flatten(self):
        """(Re)pack every parameter into one contiguous vector (the recurrent prefix of which is also ``self.gru``'s), keeping
        the Parameter objects and the fused step's Adam moments."""
        super()._flatten()
        self.gru._adopt(self._flat[:self.gru_param_count()], self._views[:4 * self.n_layers * self.n_directions])
        total = self._flat.numel()
        old = getattr(self, "_adam", None)
        self._graphs = {}
        self._adam = None
        if old is not None and old.m.numel() == total:          # keep the Adam moments across a re-flatten (.to() / .cuda())
            st = self._fused_state()
            st.m.copy_(old.m.to(self._flat.device)); st.v.copy_(old.v.to(self._flat.device))
            st.step = old.step
            st.dstep.fill_(old.step)
            self._mirror_optimizer_state()

    def gru_param_count(self) -> int:
        """Entries of the flat vector that belong to ``self.gru`` (its leading part, in nn.GRU's order)."""
        return self._flat.numel() - self.linear.weight.numel() - self.linear.bias.numel()

    # ------------------------------------------------------------------ plans
    def resolved_precision(self, batch: int = 0) -> str:
        """The precision a batch runs at ("auto": the fp32-class tensor-core path wherever it applies, i.e. hidden_size <= 256)."""
        return self._pad.precision

    def plan_hidden(self, batch: int = 0) -> int:
        """Hidden size of the C plan.  The tensor-core kernels exist for 128 / 256 (/ 512 at "bf16") hidden units; smaller models run
        ZERO-PADDED to the next of these: a padded unit has zero weights and biases, so r = z = 1/2, n = 0 and its state stays 0
        from h0 = 0 on; it feeds zero columns of W_hh / W_ih / the head.  Logits, loss and the gradients of the real parameters are
        exactly those of the unpadded model (up to summation order); the padded gradient entries are dropped."""
        return self._pad.hidden

    def _padded_batch(self, batch: int) -> int:
        """The batch size a plan runs for `batch` real rows (whole batch tiles on the tensor-core paths, _Padding)."""
        return self._pad.batch(batch)

    def pooled_argmax(self) -> torch.Tensor:
        """argmax_t of the max-pooled direction sum [batch, hidden] as taken by the last ``forward`` (the routing of the
        max-pool gradient, biGRU_model.py:125).  Valid until the next forward of the same shape."""
        plan, stash, B = self._last_forward
        off = _lib.C.c_size_t()
        _lib.check(_lib.load().bigru_stash_argmax_offset(plan.handle, _lib.C.byref(off)), "bigru_stash_argmax_offset")
        Hp = self._pad.hidden
        arg = stash[off.value:off.value + plan.B * Hp * 4].view(torch.int32).view(plan.B, Hp)
        return self._pad.crop(arg, B, units=True).clone()

    # ------------------------------------------------------------------ reference surface
    def forward(self, input_seq, hidden=None, lengths=None):
        """Logits [batch, output_size] (biGRU_model.py:63-138).

        ``lengths`` ([batch] integers, each in [1, seq_len]; a list, a CPU or a CUDA tensor): row b is ``lengths[b]`` steps
        long and its inputs at later steps are ignored.  Each GRU layer then runs as ``nn.GRU`` on
        ``pack_padded_sequence(input_seq, lengths, batch_first=True, enforce_sorted=False)``, the head pools over the valid
        steps only (``last`` at t = lengths[b] - 1 forward, t = 0 reverse) and the input gradient is 0 at padded steps.
        Not with ``hidden`` (ValueError)."""
        x, h0 = self._prepare_input(input_seq, hidden)
        lens = self._prepare_lengths(lengths, x, hidden)
        self.batch_size, self.input_length = x.size(0), x.size(1)          # as the reference sets (:82-85)
        return _BiGRUFunction.apply(self, x, h0, lens, *self._ordered_params())

    def infer(self, input_seq, hidden=None, max_batch: Optional[int] = None, lengths=None):
        """Eval-mode logits [batch, output_size] (bigru_infer), bit-identical to ``self.eval()(input_seq, hidden)`` under
        ``torch.no_grad()``: no dropout whatever ``self.training`` says, no autograd record, and nothing kept for a backward, so
        the plan allocates only its inference workspace (about a sixth of the training forward's stash + scratch at
        configs[1]).  ``max_batch`` runs the batch in slices of at most that many rows, all on one plan (the last slice
        zero-padded), which bounds the memory whatever the batch size.  ``pooled_argmax()`` and the last hidden state stay
        those of the last ``forward``.  ``lengths``: per-row lengths as in ``forward``."""
        x, h0 = self._prepare_input(input_seq, hidden)
        lens = self._prepare_lengths(lengths, x, hidden)
        B = x.shape[0]
        k = self._slice_rows(max_batch, B)
        pflat = self._plan_params()
        outs = [self._infer_slice(pflat, x[s:s + k], None if h0 is None else h0[:, s:s + k], self._pad.batch(k),
                                  None if lens is None else lens[s:s + k])
                for s in range(0, B, k)]
        return outs[0] if len(outs) == 1 else torch.cat(outs)

    @staticmethod
    def _slice_rows(max_batch, n):
        """Rows per slice when `infer` splits n rows by max_batch."""
        if max_batch is None:
            return n
        if int(max_batch) <= 0:
            raise ValueError(f"max_batch must be positive, got {max_batch}")
        return min(int(max_batch), n)

    def _infer_slice(self, pflat, x, h0, Bp, lengths=None):
        """Logits of the rows of x (at most Bp) through bigru_infer on the plan of Bp rows; pflat: _plan_params()."""
        c = _PaddedCall(self, x, h0, lengths, Bp=Bp)
        with torch.no_grad(), torch.cuda.device(x.device):    # the C ABI launches on the CURRENT device: make it the model's
            logits = torch.empty(Bp, self.output_size, device=x.device, dtype=torch.float32)
            _lib.check(_lib.load().bigru_infer_lengths(c.plan.handle, _lib.ptr(pflat), _lib.ptr(c.x), _lib.ptr(c.h0),
                                                       _lib.ptr(c.plan.infer_workspace()), _lib.ptr(logits),
                                                       _lib.ptr(c.lengths), _stream_ptr(x.device)), "bigru_infer_lengths")
        return self._pad.crop(logits, c.B)

    def add_loss_fn(self, loss_fn):
        self.loss_fn = loss_fn

    def add_optimizer(self, optimizer):
        self.optimizer = optimizer
        self._adam = None
        self._graphs = {}

    def add_device(self, device=torch.device("cpu")):
        self.device = device

    def enable_data_parallel(self, process_group=None):
        """Batch data parallelism: one process per GPU, every rank holds a replica and a batch shard;
        train_step/train_model all-reduce the flat gradient once per step (NCCL over NVLink)."""
        import torch.distributed as dist
        self._dp_group = process_group if process_group is not None else dist.group.WORLD
        self._dp_world = dist.get_world_size(self._dp_group)

    # ------------------------------------------------------------------ fused training step
    def _loss_spec(self):
        """(loss kind, weight, pos_weight, scalar parameter) of a loss the fused step computes, else None."""
        fn = self.loss_fn
        if getattr(fn, "reduction", None) != "mean":
            return None
        if isinstance(fn, nn.CrossEntropyLoss):
            if getattr(fn, "label_smoothing", 0.0) == 0.0 and fn.ignore_index == -100:
                if fn.weight is None:
                    return _lib.LOSS_CE, None, None, 0.0
                if fn.weight.dim() == 1 and fn.weight.numel() == self.output_size:
                    return _lib.LOSS_CE_WEIGHTED, fn.weight, None, 0.0
        elif isinstance(fn, nn.BCEWithLogitsLoss):
            if self._per_class(fn.weight) and self._per_class(fn.pos_weight):
                return _lib.LOSS_BCE, fn.weight, fn.pos_weight, 0.0
        elif isinstance(fn, nn.MultiLabelSoftMarginLoss):
            if fn.weight is None:
                return _lib.LOSS_MLSM, None, None, 0.0
        elif type(fn) in (nn.MSELoss, nn.L1Loss):
            return (_lib.LOSS_MSE if type(fn) is nn.MSELoss else _lib.LOSS_L1), None, None, 0.0
        elif type(fn) is nn.SmoothL1Loss and fn.beta >= 0:
            return _lib.LOSS_SMOOTH_L1, None, None, float(fn.beta)
        elif type(fn) is nn.HuberLoss and fn.delta > 0:
            return _lib.LOSS_HUBER, None, None, float(fn.delta)
        return None

    def _per_class(self, w):
        """Whether a BCE weight broadcasts over [B, C] logits as one value per class: a single element, or C values along the
        last dimension with every leading dimension 1.  Anything else ([C, 1], per-row, per-element) weighs rows, which the
        fused loss cannot express, even when its element count happens to be C."""
        if w is None or w.numel() == 1:
            return True
        return w.dim() >= 1 and w.shape[-1] == self.output_size and all(s == 1 for s in w.shape[:-1])

    def _adam_spec(self):
        """The param_groups of a torch.optim.Adam / AdamW (AdamW is Adam with decoupled weight decay) whose groups hold
        exactly this model's parameters, each once, else None."""
        opt = self.optimizer
        if not isinstance(opt, torch.optim.Adam) or not 1 <= len(opt.param_groups) <= _lib.ADAM_MAX_GROUPS:
            return None
        groups = opt.param_groups
        if any(g.get("amsgrad", False) or g.get("maximize", False) for g in groups):
            return None
        mine = {id(p) for p in self._ordered_params()}
        theirs = [id(p) for g in groups for p in g["params"]]
        if len(theirs) != len(mine) or set(theirs) != mine:
            return None
        return groups

    def _adam_tables(self, groups):
        """(bigru_adam_group rows, bigru_adam_segment rows) of the optimizer's current param_groups: one row per group, and
        (offset, count, group) per parameter tensor in the flat vector's order (``_views``)."""
        hyper = tuple((float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"]),
                       float(g.get("weight_decay", 0.0)), float(bool(g.get("decoupled_weight_decay", False))))
                      for g in groups)
        group_of = {id(p): k for k, g in enumerate(groups) for p in g["params"]}
        segs = tuple((off, n, group_of[id(p)]) for p, (off, n, _) in zip(self._ordered_params(), self._views))
        return hyper, segs

    def can_fuse_step(self) -> bool:
        return self._loss_spec() is not None and self._adam_spec() is not None

    def _loss_vec(self, w, C):
        """Per-class loss weight as a device vector.  Cached (and kept alive across the asynchronous C
        calls) until the source tensor changes."""
        if w is None:
            return None
        key = (id(w), w._version, C)
        hit = self._loss_cache.get(key)
        if hit is None:
            v = w.detach().to(device=self._flat.device, dtype=torch.float32).reshape(-1)
            if v.numel() == 1:
                v = v.expand(C)
            if v.numel() != C:
                raise ValueError("loss weight must have one entry per class")
            if len(self._loss_cache) > 8:
                self._loss_cache.clear()
            hit = self._loss_cache[key] = v.contiguous()
        return hit

    def _fused_state(self):
        if self._adam is None:
            self._adam = _AdamState(self._flat, self._pad, len(self._views))
            self._import_optimizer_state(self._adam)
            self._mirror_optimizer_state()
        return self._adam

    def _import_optimizer_state(self, st):
        """Moments the user's torch.optim.Adam / AdamW already holds (generic steps taken before, or a loaded optimizer.state_dict())
        become the fused step's flat moments."""
        opt = getattr(self, "optimizer", None)
        if opt is None:
            return
        steps = []
        for p, (off, n, _) in zip(self._ordered_params(), self._views):
            ps = opt.state.get(p)
            if not ps or "exp_avg" not in ps:
                return
            steps.append(int(float(ps["step"])) if "step" in ps else 0)
        if len(set(steps)) != 1:
            return
        with torch.no_grad():
            for p, (off, n, _) in zip(self._ordered_params(), self._views):
                ps = opt.state[p]
                st.m[off:off + n].copy_(ps["exp_avg"].reshape(-1).to(st.m.device))
                st.v[off:off + n].copy_(ps["exp_avg_sq"].reshape(-1).to(st.v.device))
        st.step = steps[0]
        st.dstep.fill_(steps[0])

    def _mirror_optimizer_state(self):
        """optimizer.state[p] = views of the flat moments + a step tensor, in torch.optim.Adam's (and AdamW's) own format: optimizer.state_dict()
        checkpoints carry the fused step's moments, and a later generic optimizer.step() continues from them (in place)."""
        opt, st = getattr(self, "optimizer", None), self._adam
        if opt is None or st is None or self._adam_spec() is None:
            return
        for p, (off, n, shape) in zip(self._ordered_params(), self._views):
            opt.state[p] = {"step": torch.tensor(float(st.step)), "exp_avg": st.m[off:off + n].view(shape),
                            "exp_avg_sq": st.v[off:off + n].view(shape)}
        st.mirror_steps = [opt.state[p]["step"] for p in self._ordered_params()]

    def _launch_compute(self, buf, st, s):
        """Forward, loss and backward of one step on stream `s`: the loss into st.loss and the gradient of the real parameters
        into st.grad."""
        lib = _lib.load()
        c, (kind, wv, pwv, denom, param) = buf.c, buf.loss
        pflat = self._plan_params(st.pflat)
        # the loss sees the real batch rows (tgt's); logits / dlogits may carry zero-padded rows behind them
        B, C = buf.tgt.shape[0], buf.logits.shape[1]
        self._forward_c(c.plan, pflat, c.x, c.h0, c.lengths, c.training, c.seed, buf.stash, buf.logits, None, s)
        _lib.check(lib.bigru_loss_param(kind, _lib.ptr(buf.logits), _lib.ptr(buf.tgt), _lib.ptr(wv), _lib.ptr(pwv), B, C, denom,
                                        param, _lib.ptr(st.loss), _lib.ptr(buf.dlogits), s), "bigru_loss_param")
        self._backward_c(c.plan, pflat, c.x, c.h0, c.lengths, c.training, c.seed, buf.stash, buf.dlogits, st.pgrad, None, None, s)
        self._plan_grads(st.pgrad, st.grad)

    def _forward_c(self, plan, pflat, x, h0, lengths, training, seed, stash, logits, hn, s):
        """bigru_forward_lengths of a padded batch on `plan` and stream `s`, with this model's dropout."""
        _lib.check(_lib.load().bigru_forward_lengths(plan.handle, _lib.ptr(pflat), _lib.ptr(x), _lib.ptr(h0),
                                                     float(self.dropout_p), int(bool(self.spatial_dropout)), int(training),
                                                     seed, _lib.ptr(stash), _lib.ptr(plan.scratch), _lib.ptr(logits),
                                                     _lib.ptr(hn), _lib.ptr(lengths), s), "bigru_forward_lengths")

    def _backward_c(self, plan, pflat, x, h0, lengths, training, seed, stash, dlogits, grads, dx, dh0, s):
        """bigru_backward_lengths of the forward `_forward_c` ran with the same arguments."""
        _lib.check(_lib.load().bigru_backward_lengths(plan.handle, _lib.ptr(pflat), _lib.ptr(x), _lib.ptr(h0),
                                                      float(self.dropout_p), int(bool(self.spatial_dropout)), int(training),
                                                      seed, _lib.ptr(stash), _lib.ptr(plan.scratch), _lib.ptr(dlogits),
                                                      _lib.ptr(grads), _lib.ptr(dx), _lib.ptr(dh0), _lib.ptr(lengths), s),
                   "bigru_backward_lengths")

    def _launch_update(self, g, st, s):
        """clip_grad_norm_(clip) + Adam / AdamW of the param_groups `g` on the flat buffers on stream `s`, with each group's
        hyperparameters read from st.hyper on the device; Adam's step counter is incremented on the device."""
        lib = _lib.load()
        sq = st.scal[1:2]
        _lib.check(lib.bigru_adam_tick(_lib.ptr(st.dstep), _lib.ptr(sq), s), "bigru_adam_tick")
        _lib.check(lib.bigru_sqnorm(_lib.ptr(st.grad), st.grad.numel(), _lib.ptr(sq), _lib.ptr(st.sqws), s), "bigru_sqnorm")
        _lib.check(lib.bigru_clip_adam_groups_dev(_lib.ptr(self._flat), _lib.ptr(st.grad), _lib.ptr(st.m), _lib.ptr(st.v),
                                                  self._flat.numel(), _lib.ptr(sq), float(self.clip), _lib.ptr(st.hyper),
                                                  len(g), _lib.ptr(st.segs), st.segs.shape[0], _lib.ptr(st.dstep), 1.0, s),
                   "bigru_clip_adam_groups_dev")

    def _graph_key(self, B, T, loss, n_groups, dev, has_lengths):
        """Key of the captured step graph.  It holds no optimizer hyperparameter: the update reads those from the device
        table (_AdamState.hyper), so a schedule replays one graph.  clip stays a kernel argument, as the model's own
        attribute (the reference's constructor argument) that no scheduler touches.  The last element is whether the step
        has per-row lengths."""
        kind, wv, pwv, denom, param = loss
        return (B, T, self.precision, kind, id(wv), id(pwv), denom, param, n_groups, float(self.clip), self._dp_world,
                dev.index, has_lengths)

    def _capture(self, key, buf, st, g):
        """CUDA graph(s) of the step on the static buffers `buf` (SURVEY.md 8(f) N5): one graph at world size 1; with data
        parallelism two (compute | update), replayed with the gradient all-reduce between them."""
        lib = _lib.load()
        dev = buf.c.x.device
        torch.cuda.current_stream(dev).synchronize()
        n0 = lib.bigru_launch_count()
        # an explicit capture stream ON THE MODEL'S DEVICE: torch's default capture stream is created once per process, on whichever
        # device was current then
        cap = torch.cuda.Stream(device=dev)
        try:
            ga, gb = torch.cuda.CUDAGraph(), None
            with torch.cuda.graph(ga, stream=cap, capture_error_mode="thread_local"):
                self._launch_compute(buf, st, _stream_ptr(dev))
                if self._dp_world == 1:
                    self._launch_update(g, st, _stream_ptr(dev))
            if self._dp_world > 1:
                gb = torch.cuda.CUDAGraph()
                with torch.cuda.graph(gb, stream=cap, capture_error_mode="thread_local"):
                    self._launch_update(g, st, _stream_ptr(dev))
        except Exception as e:                            # capture is an optimisation: fall back to plain launches
            import warnings
            warnings.warn(f"BiGRU.train_step: CUDA-graph capture failed ({e}); using plain launches")
            self.use_cuda_graph = False
            ga = None
        launches = int(lib.bigru_launch_count() - n0)
        lib.bigru_launch_count_add(-launches)             # captured, not executed
        if ga is None:
            buf.c.plan.release_stash(buf.stash)
            return
        if len(self._graphs) > 4:
            self._graphs.clear()
        self._graphs[key] = (buf, ga, gb, launches)

    def train_step(self, input_seq, target, hidden=None, lengths=None):
        """One optimisation step = the body of the reference loop (biGRU_model.py:198-210):
        zero_grad, forward, loss, backward, clip_grad_norm_(clip), Adam step - C-ABI calls with no autograd graph, replayed
        from a captured CUDA graph when the step is replayable (no dropout noise to draw, no initial state).  ``lengths``:
        per-row lengths as in ``forward``.
        Returns (loss, logits) as device tensors (no host sync, except that lengths given as a CUDA tensor are copied back to
        be checked on the host)."""
        spec, g = self._loss_spec(), self._adam_spec()
        if spec is None or g is None:
            raise RuntimeError("train_step needs add_loss_fn(CrossEntropyLoss [weight=] | BCEWithLogitsLoss | "
                               "MultiLabelSoftMarginLoss | MSELoss | L1Loss | SmoothL1Loss | HuberLoss, mean reduction) and "
                               "add_optimizer(torch.optim.Adam or AdamW over model.parameters(), any parameter groups, "
                               "no amsgrad / maximize)")
        lib = _lib.load()
        x, h0 = self._prepare_input(input_seq, hidden)
        lens = self._prepare_lengths(lengths, x, hidden)
        dev = x.device
        kind, w, pw, param = spec
        B, C = x.shape[0], self.output_size
        if kind in (_lib.LOSS_CE, _lib.LOSS_CE_WEIGHTED):
            tgt = target.to(device=dev, dtype=torch.int64, non_blocking=True).contiguous()
            if tgt.shape != (B,):
                raise ValueError(f"CrossEntropyLoss target must be [{B}] class indices")
            # weighted CE: each rank's weighted mean (the kernel divides by its own weight sum), averaged over the ranks
            denom = float((B if kind == _lib.LOSS_CE else 1) * self._dp_world)
        else:
            tgt = target.to(device=dev, dtype=torch.float32, non_blocking=True).contiguous()
            if tuple(tgt.shape) != (B, C):
                raise ValueError(f"target must be [{B}, {C}]")
            denom = float(B * C * self._dp_world)
        training = self._draws_masks()
        with torch.cuda.device(dev):
            graphed = self.use_cuda_graph and not training and h0 is None and not torch.cuda.is_current_stream_capturing()
            wv, pwv = self._loss_vec(w, C), self._loss_vec(pw, C)
            st = self._fused_state()
            st.load_tables(*self._adam_tables(g))
            s = _stream_ptr(dev)
            key = ent = None
            if graphed:
                key = self._graph_key(B, int(x.shape[1]), (kind, wv, pwv, denom, param), len(g), dev, lens is not None)
                ent = self._graphs.get(key)
            if ent is not None:
                buf, ga, gb, launches = ent
                buf.c.x[:B].copy_(x, non_blocking=True)    # rows >= B of the static buffer stay zero
                buf.tgt.copy_(tgt, non_blocking=True)
                if lens is not None:
                    buf.c.lengths[:B].copy_(lens, non_blocking=True)   # rows >= B stay T steps long
                compute, update = ga.replay, (gb.replay if gb is not None else lambda: None)
                lib.bigru_launch_count_add(launches)
            else:
                c = _PaddedCall(self, x, h0, lens, training=training)
                if graphed:                               # a new graph key: this step runs on the graph's static buffers
                    c.x, tgt = c.x.clone(), tgt.clone()
                    c.lengths = None if c.lengths is None else c.lengths.clone()
                buf = _StepBuffers(c, tgt, (kind, wv, pwv, denom, param), C)
                compute, update = (lambda: self._launch_compute(buf, st, s)), (lambda: self._launch_update(g, st, s))
            compute()
            if self._dp_world > 1:
                allreduce_flat_(st.gext, self._dp_group)  # ONE all-reduce: shard gradients of the global-mean loss + the loss
            update()
            st.advance()
            self.optimizer._opt_called = True                 # torch's mark of a stepped optimizer, which lr schedulers check
            if not graphed:
                buf.c.plan.release_stash(buf.stash)
            elif ent is None:
                self._capture(key, buf, st, g)
            logits = self._pad.crop(buf.logits, B)
            return st.loss.clone(), (logits.clone() if graphed else logits)

    # ------------------------------------------------------------------ windows of a chunk-resident dataset (SURVEY.md 8(f) N1)
    def _window_args(self, dataset, start, count):
        if dataset.device != self.flat_parameters().device:
            raise RuntimeError("dataset and model live on different devices")
        if dataset.n_features != self.n_features:
            raise ValueError(f"dataset has {dataset.n_features} features, the model expects {self.n_features}")
        if count <= 0 or start < 0 or start + count + dataset.window - 1 > dataset.n_rows:
            raise ValueError(f"windows [{start}, {start + count}) of width {dataset.window} exceed the {dataset.n_rows}-row chunk")

    def forward_windows(self, dataset, start: int, count: int):
        """Logits (no autograd graph) for windows start .. start+count-1 of a chunk-resident ``MySQLBatchLoader``: only the
        chunk's rows cross the host link; the windows are collated and normalised on the device (one gather kernel), then
        ``forward`` runs on them."""
        self._window_args(dataset, start, count)
        with torch.no_grad():
            return self.forward(dataset.collate(start, count)[0])

    def infer_windows(self, dataset, start: int, count: int, max_batch: Optional[int] = None):
        """``infer`` on windows start .. start+count-1 of a chunk-resident ``MySQLBatchLoader``: eval-mode logits, bit-identical
        to ``forward_windows`` in eval mode.  The windows are collated one slice of at most ``max_batch`` at a time, so the
        whole [count, window, F] input never exists at once."""
        self._window_args(dataset, start, count)
        k = self._slice_rows(max_batch, count)
        pflat, Bp = self._plan_params(), self._pad.batch(k)
        outs = []
        for s in range(start, start + count, k):
            x, _ = self._prepare_input(dataset.collate(s, min(k, start + count - s))[0], None)
            outs.append(self._infer_slice(pflat, x, None, Bp))
        return outs[0] if len(outs) == 1 else torch.cat(outs)

    def train_step_windows(self, dataset, start: int, count: int):
        """``train_step`` on windows of a chunk-resident dataset, inputs and targets collated on the device.
        Returns (loss, logits)."""
        spec = self._loss_spec()
        if spec is None or self._adam_spec() is None:
            raise RuntimeError("train_step_windows needs a fusable loss and torch.optim.Adam or AdamW (see train_step)")
        self._window_args(dataset, start, count)
        x, y = dataset.collate(start, count)
        ce = spec[0] in (_lib.LOSS_CE, _lib.LOSS_CE_WEIGHTED)
        tgt = y.reshape(count, -1)[:, 0].to(torch.int64) if ce else y.reshape(count, self.output_size)
        return self.train_step(x, tgt)

    def _generic_step(self, x, target):
        """Any loss / optimiser: autograd drives the same CUDA forward/backward kernels."""
        self.optimizer.zero_grad()
        pred = self.forward(x)
        if isinstance(self.loss_fn, nn.Module):
            self.loss_fn.to(pred.device)                 # class weights follow the logits
        loss = self.loss_fn(pred, target.to(pred.device))
        loss.backward()
        if self._dp_world > 1:                            # ONE all-reduce of all gradients (flattened), then scattered back
            ps = [p for p in self.parameters() if p.grad is not None]
            flat = torch.cat([p.grad.reshape(-1) for p in ps])
            allreduce_flat_(flat, self._dp_group)
            flat.div_(self._dp_world)
            off = 0
            for p in ps:
                p.grad.copy_(flat[off:off + p.grad.numel()].view_as(p.grad))
                off += p.grad.numel()
        nn.utils.clip_grad_norm_(self.parameters(), self.clip)
        self.optimizer.step()
        return loss.detach().reshape(1), pred.detach()

    # ------------------------------------------------------------------ epoch loops
    def _metric_counts(self, logits, target, counts_row):
        if target.dim() != 2 or target.shape != logits.shape:
            raise ValueError("multilabel metrics need a [batch, n_classes] indicator target "
                             "(biGRU_model.py:213-221 feeds sigmoid(pred) > 0.5 to sklearn)")
        tgt = target.to(device=logits.device, dtype=torch.float32).contiguous()
        with torch.cuda.device(logits.device):
            _lib.check(_lib.load().bigru_multilabel_counts(_lib.ptr(logits), _lib.ptr(tgt), logits.shape[0],
                                                           logits.shape[1], _lib.ptr(counts_row), _stream_ptr(logits.device)),
                       "bigru_multilabel_counts")

    @staticmethod
    def _scores(counts: np.ndarray, sizes, C, beta=0.5):
        """Per-batch accuracy / Hamming loss / F-beta from the device counters, then the mean over
        batches (the reference averages per-batch sklearn scores, :224 / :286)."""
        acc, ham, fb = [], [], []
        b2 = beta * beta
        for row, B in zip(counts, sizes):
            acc.append(row[0] / B)
            ham.append(row[1] / (B * C))
            tp, fp, fn = row[2::3][:C], row[3::3][:C], row[4::3][:C]
            den = (1 + b2) * tp + b2 * fn + fp
            fb.append(np.where(den > 0, (1 + b2) * tp / np.maximum(den, 1), 0.0))
        return float(np.mean(acc)), float(np.mean(ham)), np.mean(np.stack(fb), axis=0)

    def train_model(self, train_iterator):
        """One training epoch (biGRU_model.py:162-224).  Returns
        (mean accuracy, mean Hamming loss, mean loss, mean F-beta(0.5) per class)."""
        self.train()
        fused = self.can_fuse_step()
        losses, sizes, rows = [], [], []
        C = self.output_size
        for input_seq, target in train_iterator:
            target = target.squeeze(1)                                   # [B,1,C] -> [B,C]  (:193)
            if fused:
                loss, logits = self.train_step(input_seq, target)
            else:
                x, _ = self._prepare_input(input_seq, None)
                loss, logits = self._generic_step(x, target)
            row = torch.zeros(2 + 3 * C, dtype=torch.int64, device=logits.device)
            self._metric_counts(logits, target, row)
            losses.append(loss.reshape(1))
            rows.append(row)
            sizes.append(logits.shape[0])
        if not rows:
            return float("nan"), float("nan"), float("nan"), np.full(C, np.nan)
        counts = torch.stack(rows).cpu().numpy().astype(np.float64)      # one host sync per epoch
        acc, ham, fb = self._scores(counts, sizes, C)
        return acc, ham, float(torch.cat(losses).float().mean().item()), fb

    def evaluate_model(self, eval_iterator):
        """One evaluation epoch (biGRU_model.py:227-286).  Returns (mean accuracy, mean Hamming loss,
        mean F-beta(0.5) per class, pred_total LongTensor, target_total LongTensor)."""
        self.eval()
        C = self.output_size
        rows, sizes, preds, targets = [], [], [], []
        with torch.no_grad():
            for input_seq, target in eval_iterator:
                target = target.squeeze(1)
                logits = self.forward(input_seq)
                row = torch.zeros(2 + 3 * C, dtype=torch.int64, device=logits.device)
                self._metric_counts(logits, target, row)
                rows.append(row)
                sizes.append(logits.shape[0])
                preds.append(logits > 0)                                  # sigmoid(x) > 0.5
                targets.append(target)
        if not rows:
            return float("nan"), float("nan"), np.full(C, np.nan), torch.LongTensor(), torch.LongTensor()
        counts = torch.stack(rows).cpu().numpy().astype(np.float64)
        acc, ham, fb = self._scores(counts, sizes, C)
        pred_total = torch.cat(preds).cpu().type(torch.LongTensor)
        target_total = torch.cat([t.cpu() for t in targets]).type(torch.LongTensor)
        return acc, ham, fb, pred_total, target_total
