"""Drop-in replacements for VideoPose3D's temporal-convolution models.

Mirrors ``common/model.py`` of the reference (TemporalModelBase :10-77, TemporalModel :79-138,
TemporalModelOptimized1f :140-197): same constructor signatures, attribute names and
``state_dict`` keys/shapes, so ``run.py`` and published checkpoints work unchanged.  Parameters
live in ordinary ``nn.Conv1d`` / ``nn.BatchNorm1d`` containers (never called); ``forward`` hands raw
device pointers to the sm_90a kernels behind the C ABI (``include/vp3d_b200.h``).

There is no PyTorch/CPU execution path here: without the CUDA library or with CPU tensors
``forward`` raises.
"""
import copy
import os
import weakref

import torch
import torch.nn as nn

from . import _capi

_PRECISIONS = {"bf16": _capi.VP3D_PRECISION_BF16, "bf16x3": _capi.VP3D_PRECISION_BF16X3,
               "mixed": _capi.VP3D_PRECISION_MIXED, "fp16": _capi.VP3D_PRECISION_FP16,
               "int8": _capi.VP3D_PRECISION_INT8}
_CALIB_METHODS = {"amax": _capi.VP3D_INT8_CALIB_AMAX,
                  "percentile": _capi.VP3D_INT8_CALIB_PERCENTILE, "mse": _capi.VP3D_INT8_CALIB_MSE}


# id(parameter) -> weakref(owning model): lets optim.FusedAdam find the model whose packed bf16
# weights it can refresh while it updates the parameter (no API change for run.py, which builds the
# optimizer from `model.parameters()` alone)
_PARAM_OWNER = {}


def owner_of(param):
    """The live TemporalModel* that owns `param`, or None."""
    ref = _PARAM_OWNER.get(id(param))
    m = ref() if ref is not None else None
    if m is None or not any(param is q for q in m.parameters()):
        return None
    return m


class _Plan:
    """A plan handle and the parameter versions (``TemporalModelBase._versions``) each kind of its
    weight packs was made from, None while never packed: ``eval`` (VP3D_PACK_CONV |
    VP3D_PACK_BN_EVAL), ``train`` (VP3D_PACK_CONV | VP3D_PACK_CONV_T) and ``expand_t``
    (VP3D_PACK_EXPAND_T, the expand conv weight's entry only).  ``bn_sync`` is (reducer, ctypes
    exchange callback) while the plan's synchronized BatchNorm is on (vp3d_set_bn_sync): the plan
    holds the callback as long as it may call it.  ``int8`` is the calibration (the module's
    ``_int8`` tuple) whose scales an int8 plan holds, None before any; ``int8_mask`` the block
    mask (vp3d_set_int8_blocks) it was last given, None before any."""

    __slots__ = ("handle", "precision", "eval", "train", "expand_t", "bn_sync", "int8",
                 "int8_mask")

    def __init__(self, handle, precision):
        self.handle = handle
        self.precision = precision
        self.eval = self.train = self.expand_t = None
        self.bn_sync = None
        self.int8 = None
        self.int8_mask = None

    @property
    def _as_parameter_(self):
        # ctypes passes a _Plan to the C ABI as its handle
        return self.handle


class _EngineState:
    """A module's engine state: its plans by (device index, precision), the plan of its last call
    (what ``_plan`` and ``last_launch_count`` report), the plan each host-pipeline slot was submitted
    on, and the eval workspace.  Owns the handles: they are destroyed exactly once, when the state
    itself is collected (weakref.finalize), never by a module that merely shares or copies the
    reference.  Copies of a module start with an empty state of their own."""

    def __init__(self):
        self.plans = {}
        self.last = None
        self.host_slots = {}
        self.workspace = None
        self._handles = []
        self._finalizer = weakref.finalize(self, _EngineState._destroy, self._handles)

    def add(self, key, handle):
        self.plans[key] = plan = _Plan(handle, key[1])
        self._handles.append(handle)
        return plan

    def __deepcopy__(self, memo):
        return _EngineState()

    def __copy__(self):
        return _EngineState()

    def __reduce__(self):
        return (_EngineState, ())

    @staticmethod
    def _destroy(handles):
        try:
            lib = _capi.load()
        except Exception:  # pragma: no cover - interpreter shutdown / library gone
            return
        for h in handles:
            try:
                lib.vp3d_plan_destroy(h)
            except Exception:  # pragma: no cover
                pass
        del handles[:]


def _default_precision():
    p = os.environ.get("VP3D_PRECISION", "fp16")
    if p not in _PRECISIONS:
        raise ValueError(f"VP3D_PRECISION must be one of {sorted(_PRECISIONS)}, got {p!r}")
    return p


class TemporalModelBase(nn.Module):
    """
    Do not instantiate this class.  (reference: common/model.py:10-77)
    """

    _variant = None  # set by subclasses

    def __init__(self, num_joints_in, in_features, num_joints_out,
                 filter_widths, causal, dropout, channels):
        super().__init__()

        # Validate input (model.py:20-21)
        for fw in filter_widths:
            assert fw % 2 != 0, 'Only odd filter widths are supported'

        self.num_joints_in = num_joints_in
        self.in_features = in_features
        self.num_joints_out = num_joints_out
        self.filter_widths = filter_widths

        self.drop = nn.Dropout(dropout)
        self.relu = nn.ReLU(inplace=True)

        self.pad = [filter_widths[0] // 2]
        self.expand_bn = nn.BatchNorm1d(channels, momentum=0.1)
        self.shrink = nn.Conv1d(channels, num_joints_out * 3, 1)

        # engine state (not part of the state_dict)
        self._channels = channels
        self._causal = bool(causal)
        self._dense = False
        self._precision = _default_precision()
        self._train_precision = os.environ.get("VP3D_TRAIN_PRECISION", "bf16")
        self._engine = _EngineState()
        self._stats_epoch = 0      # bumped by every training forward (running stats changed)
        self._fwd_token = 0        # identifies the most recent training forward
        self._grad_reducer = None  # data_parallel.GradientReducer, set by its attach()
        # int8 calibration: (amax CPU float tensor [2B], parameter versions it belongs to), or None
        self._int8 = None
        # blocks (1..B) the 'int8' precision runs u8 x s8, None = all (set_int8_blocks)
        self._int8_blocks = None
        self.last_predict_launches = 0   # kernels the last predict() launched

    def _build_layers(self, strided):
        """Create the parameter containers with the reference's names, shapes and default init.

        Per block i >= 1 with width w_i and dilation d_i = prod(w_0..w_{i-1}) (model.py:107-121,
        172-184): pad_i = (w_i - 1) * d_i // 2; the first conv is Conv1d(C, C, w_i, dilation=d_i)
        for the dilated model (kernel 2*pad_i+1, dilation 1 when dense) or Conv1d(C, C, w_i,
        stride=w_i) for the strided one; the second is a 1x1 conv; each is followed by a
        BatchNorm1d(momentum=0.1).  causal_shift is in frames for the dilated model and in strided
        units for the strided one.
        """
        fw, C = self.filter_widths, self._channels
        c_in = self.num_joints_in * self.in_features
        half0 = fw[0] // 2
        if strided:
            self.expand_conv = nn.Conv1d(c_in, C, fw[0], stride=fw[0], bias=False)
        else:
            self.expand_conv = nn.Conv1d(c_in, C, fw[0], bias=False)
        self.causal_shift = [half0 if self._causal else 0]
        convs, bns = [], []
        dilation = fw[0]
        for w in fw[1:]:
            pad = (w - 1) * dilation // 2
            self.pad.append(pad)
            if strided:
                self.causal_shift.append(w // 2 if self._causal else 0)
                convs.append(nn.Conv1d(C, C, w, stride=w, bias=False))
            else:
                self.causal_shift.append((w // 2) * dilation if self._causal else 0)
                if self._dense:
                    convs.append(nn.Conv1d(C, C, 2 * pad + 1, dilation=1, bias=False))
                else:
                    convs.append(nn.Conv1d(C, C, w, dilation=dilation, bias=False))
            bns.append(nn.BatchNorm1d(C, momentum=0.1))
            convs.append(nn.Conv1d(C, C, 1, dilation=1, bias=False))
            bns.append(nn.BatchNorm1d(C, momentum=0.1))
            dilation *= w
        self.layers_conv = nn.ModuleList(convs)
        self.layers_bn = nn.ModuleList(bns)
        self._register_params()

    def _register_params(self):
        ref = weakref.ref(self)
        for prm in self.parameters():
            _PARAM_OWNER[id(prm)] = ref

    # ------------------------------------------------------------------ reference API
    def set_bn_momentum(self, momentum):
        # model.py:36-39 — read at call time by the training kernels, never cached
        self.expand_bn.momentum = momentum
        for bn in self.layers_bn:
            bn.momentum = momentum

    def receptive_field(self):
        """
        Return the total receptive field of this model as # of frames.  (model.py:41-48)
        """
        frames = 0
        for f in self.pad:
            frames += f
        return 1 + 2 * frames

    def total_causal_shift(self):
        """
        Return the asymmetric offset for sequence padding.  (model.py:50-61)
        """
        frames = self.causal_shift[0]
        next_dilation = self.filter_widths[0]
        for i in range(1, len(self.filter_widths)):
            frames += self.causal_shift[i] * next_dilation
            next_dilation *= self.filter_widths[i]
        return frames

    # ------------------------------------------------------------------ engine controls
    def set_precision(self, precision):
        """Eval-mode operand format.  'fp16' (default): IEEE fp16 operands and activations, fp32
        accumulate -- ~4e-4 of the fp32 reference at the tensor rate of bf16; 'bf16x3': every GEMM
        split-bf16 (fp32-faithful, ~1e-5); 'mixed': bf16 residual blocks on a hi+lo residual
        stream, split-bf16 expand / shrink (~1e-3); 'bf16': every GEMM plain bf16 (~3e-3);
        'int8': the residual blocks' convs on u8 activations times s8 weights (exact int32 sums),
        the rest as 'fp16' -- about 0.73x the fp16 forward time on the bench model (H100), at
        ~5e-3 of fp32 on a random-init model (ten times fp16's error; trained checkpoints not
        measured).  Needs ``calibrate_int8`` or ``load_int8_calibration`` first;
        ``set_int8_blocks`` keeps chosen blocks in fp16.  Not in the reference."""
        if precision not in _PRECISIONS:
            raise ValueError(f"precision must be one of {sorted(_PRECISIONS)}")
        self._precision = precision
        return self

    @property
    def precision(self):
        return self._precision

    def invalidate(self):
        """Force a re-pack of every parameter on the next forward.  Needed only after edits that
        bypass torch's version counters (``p.data.mul_()``, ``p.data.copy_()``, raw-pointer
        writes): ordinary in-place ops, ``optimizer.step`` and ``load_state_dict`` are detected
        automatically through ``tensor._version``.  Not in the reference."""
        for plan in self._engine.plans.values():
            plan.eval = plan.train = plan.expand_t = None
        if self._int8 is not None:
            self._int8 = (self._int8[0], None)   # stale: recalibrate or load a calibration
        return self

    # ------------------------------------------------------------------ int8 calibration
    def calibrate_int8(self, inputs, method="amax", percentile=99.99):
        """Measure the activation ranges of the 'int8' eval mode: runs the fp16 eval forward
        (without shrink) on `inputs` -- one CUDA float32 (N, T, J, F) tensor, a list of them, or an
        ``UnchunkedGenerator`` on the device (every batch of one epoch) -- and keeps, for every
        residual-block conv, a clipping threshold of its input over all of them (the int8 scale is
        threshold / 255; larger values saturate at 255).  `method`:

        - "amax": the maximum;
        - "percentile": the smallest value at or above `percentile` percent (in (0, 100]) of the
          values, zeros included, from an exact histogram with one bin per fp16 value;
        - "mse": the fp16 value between max / 256 and max that minimises the squared quantisation
          error over that histogram.

        The last two keep one outlier (a glitch frame of a 2-D detector, a long-tailed activation)
        from coarsening the scale of every ordinary value.  Recorded with the current parameter
        versions: after any parameter change an int8 forward raises until the model is recalibrated
        or a calibration is loaded.  Not in the reference."""
        if method not in _CALIB_METHODS:
            raise ValueError(f"method must be one of {sorted(_CALIB_METHODS)} (got {method!r})")
        if method == "percentile" and not 0.0 < float(percentile) <= 100.0:
            raise ValueError(f"percentile must be in (0, 100] (got {percentile})")
        if hasattr(inputs, "next_epoch"):
            inputs = [batch[-1] for batch in inputs.next_epoch()]
        elif torch.is_tensor(inputs):
            inputs = [inputs]
        inputs = list(inputs)
        if not inputs:
            raise ValueError("calibrate_int8 needs at least one input batch")
        lib = _capi.load()
        device = self.expand_conv.weight.device
        if device.type != "cuda":
            raise RuntimeError("module parameters must be on a CUDA device")
        layers = len(self.layers_conv)
        hist = None   # "amax" (and a model without residual blocks): the maxima alone
        with torch.cuda.device(device):
            plan = self._get_plan(device, "fp16")
            stream = torch.cuda.current_stream(device).cuda_stream
            self._sync_weights(plan, stream)
            if method == "amax" or layers == 0:
                amax = torch.zeros(layers, dtype=torch.float32, device=device)
            else:
                hist = torch.zeros(lib.vp3d_int8_hist_bytes(plan) // 8, dtype=torch.int64,
                                   device=device)
            for x in inputs:
                if not (torch.is_tensor(x) and x.is_cuda and x.device == device
                        and x.dtype == torch.float32 and x.dim() == 4
                        and x.shape[-2] == self.num_joints_in and x.shape[-1] == self.in_features):
                    raise ValueError("calibrate_int8 takes CUDA float32 (N, T, J, F) tensors on the "
                                     "model's device")
                x = x.contiguous()
                N, T = int(x.shape[0]), int(x.shape[1])
                nbytes = lib.vp3d_workspace_bytes(plan, N, T)
                if nbytes == 0:
                    raise ValueError(f"input of {T} frames is shorter than the receptive field "
                                     f"({self.receptive_field()})")
                ws = self._get_workspace(nbytes, device)
                if hist is None:
                    _capi.check(lib.vp3d_calibrate_int8(plan, x.data_ptr(), N, T, ws.data_ptr(),
                                                        ws.numel(), amax.data_ptr(), stream),
                                "vp3d_calibrate_int8")
                else:
                    _capi.check(lib.vp3d_calibrate_int8_hist(plan, x.data_ptr(), N, T,
                                                             ws.data_ptr(), ws.numel(),
                                                             hist.data_ptr(), stream),
                                "vp3d_calibrate_int8_hist")
            if hist is not None:
                scratch = torch.empty(lib.vp3d_int8_thresholds_scratch_bytes(layers),
                                      dtype=torch.uint8, device=device)
                amax = torch.empty(layers, dtype=torch.float32, device=device)
                _capi.check(lib.vp3d_int8_thresholds(hist.data_ptr(), layers, _CALIB_METHODS[method],
                                                     float(percentile), amax.data_ptr(),
                                                     scratch.data_ptr(), scratch.numel(), stream),
                            "vp3d_int8_thresholds")
        amax = amax.cpu()
        if hist is not None and not bool(torch.isfinite(amax).all()):   # (NaN: invalid values)
            raise ValueError("calibrate_int8: inf or NaN values in the calibration inputs or their "
                             "activations")
        self._int8 = (amax, self._versions())
        return self

    def int8_calibration(self):
        """The activation maxima of the last calibration as a CPU float32 tensor of 2B values
        (block i's first-conv input, then its 1x1-conv input, for i = 1..B); None before any.  Kept
        out of the state_dict: checkpoints keep the reference's layout.  Not in the reference."""
        return None if self._int8 is None else self._int8[0].clone()

    def load_int8_calibration(self, amax):
        """Use a calibration saved with ``int8_calibration`` for the current parameters.  Not in the
        reference."""
        amax = torch.as_tensor(amax, dtype=torch.float32).detach().cpu().contiguous()
        if amax.shape != (len(self.layers_conv),):
            raise ValueError(f"expected {len(self.layers_conv)} amax values, got shape "
                             f"{tuple(amax.shape)}")
        if not bool(torch.isfinite(amax).all()) or bool((amax < 0).any()):
            raise ValueError("amax values must be finite and >= 0")
        self._int8 = (amax.clone(), self._versions())
        return self

    def set_int8_blocks(self, blocks=None):
        """Which residual blocks (numbered 1..B) the 'int8' precision runs on u8 x s8: an iterable
        of block numbers, ``[]`` for none, or None (the default) for all.  Every other block runs
        exactly as in 'fp16'; expand and shrink are fp16 either way.  Keeping the blocks whose
        quantisation costs the most accuracy in fp16 trades some of int8's speed for accuracy;
        measure each block's error as in the README.  One calibration serves every set.  Kept out
        of the state_dict, like the calibration; copies and pickles carry it.  Returns self.  Not in
        the reference."""
        nb = len(self.filter_widths) - 1
        if blocks is not None:
            blocks = list(blocks)
            for b in blocks:
                if isinstance(b, bool) or not isinstance(b, int):
                    raise ValueError(f"int8 blocks are ints in 1..{nb} (got {b!r})")
                if not 1 <= b <= nb:
                    raise ValueError(f"int8 block {b} is outside 1..{nb}")
            blocks = tuple(sorted(set(blocks)))
        self._int8_blocks = blocks
        return self

    @property
    def int8_blocks(self):
        """The blocks (1..B) the 'int8' precision runs on u8 x s8, as a sorted tuple."""
        if self._int8_blocks is None:
            return tuple(range(1, len(self.filter_widths)))
        return self._int8_blocks

    def _sync_int8(self, plan):
        """Give an int8 plan the block set and the scales of the current calibration (its next
        weight sync re-packs and folds them); raises when there is no calibration or the parameters
        changed since it was taken."""
        mask = sum(1 << (b - 1) for b in self.int8_blocks)
        if plan.int8_mask != mask:
            _capi.check(_capi.load().vp3d_set_int8_blocks(plan, mask), "vp3d_set_int8_blocks")
            plan.int8_mask = mask
            plan.eval = None   # the next sync re-packs in the new formats
        if self._int8 is None:
            raise RuntimeError("precision 'int8' needs calibrate_int8(inputs) or "
                               "load_int8_calibration(amax) first")
        amax, versions = self._int8
        if versions != self._versions():
            raise RuntimeError("the int8 calibration is stale: the parameters changed since it was "
                               "taken; call calibrate_int8 again or load_int8_calibration")
        if plan.int8 is self._int8:
            return
        vals = (_capi.ctypes.c_float * amax.numel())(*amax.tolist())
        _capi.check(_capi.load().vp3d_set_int8_scales(plan, vals, amax.numel()),
                    "vp3d_set_int8_scales")
        plan.eval = None   # the next sync re-packs and folds the scales in
        plan.int8 = self._int8

    # copies / replicas never share engine state with the original (the handles point into one
    # device allocation each; sharing them made a collected copy free the original's plans)
    def __deepcopy__(self, memo):
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        new.__setstate__(copy.deepcopy(self.__getstate__(), memo))
        return new

    def __copy__(self):
        cls = self.__class__
        new = cls.__new__(cls)
        new.__dict__.update(self.__dict__)
        # nn.Module.__copy__-style shallow copy of the registries
        for k in ("_parameters", "_buffers", "_modules"):
            new.__dict__[k] = self.__dict__[k].copy()
        new._engine = _EngineState()
        return new

    def __getstate__(self):
        state = self.__dict__.copy()
        state.pop("_engine", None)
        state.pop("_grad_reducer", None)
        return state

    def __setstate__(self, state):
        super().__setstate__(state)
        self._engine = _EngineState()
        self._grad_reducer = None
        self._register_params()

    def _replicate_for_data_parallel(self):
        replica = super()._replicate_for_data_parallel()
        replica._engine = _EngineState()
        return replica

    def _config(self, precision):
        cfg = _capi.Config()
        cfg.num_joints_in = self.num_joints_in
        cfg.in_features = self.in_features
        cfg.num_joints_out = self.num_joints_out
        cfg.num_widths = len(self.filter_widths)
        if cfg.num_widths > _capi.VP3D_MAX_WIDTHS:
            raise NotImplementedError(f"at most {_capi.VP3D_MAX_WIDTHS} filter widths are supported")
        for i, w in enumerate(self.filter_widths):
            cfg.filter_widths[i] = int(w)
        cfg.causal = int(self._causal)
        cfg.channels = self._channels
        cfg.dense = int(self._dense)
        cfg.variant = self._variant
        cfg.precision = _PRECISIONS[precision]
        return cfg

    def _get_plan(self, device, precision=None):
        """The _Plan of `precision` (default: the eval precision) on `device`, created on first use.
        A lookup: which plan ``_plan`` reports does not change."""
        key = (device.index, precision or self._precision)
        plan = self._engine.plans.get(key)
        if plan is None:
            lib = _capi.load()
            handle = _capi.ctypes.c_void_p()
            cfg = self._config(key[1])
            with torch.cuda.device(device):
                _capi.check(lib.vp3d_plan_create(_capi.ctypes.byref(cfg), _capi.ctypes.byref(handle)),
                            "vp3d_plan_create")
            plan = self._engine.add(key, handle)
        return plan

    def _use_plan(self, device, precision):
        """_get_plan for a call that runs on the plan: it becomes the plan ``_plan`` and
        ``last_launch_count`` report."""
        plan = self._engine.last = self._get_plan(device, precision)
        return plan

    @property
    def _plan(self):
        """Handle of the plan of the module's last forward, eval-mode backward or fused optimizer
        step (None before the first)."""
        last = self._engine.last
        return None if last is None else last.handle

    def _param_tensors(self):
        """All fp32 tensors of the state_dict in the order of ``vp3d_weights``."""
        conv = [self.expand_conv.weight] + [c.weight for c in self.layers_conv] + \
               [self.shrink.weight]
        bn = []
        for m in [self.expand_bn] + list(self.layers_bn):
            bn += [m.weight, m.bias, m.running_mean, m.running_var]
        bn.append(self.shrink.bias)
        return conv, bn

    def _weights_struct(self):
        w = _capi.Weights()
        w.expand_conv_weight = self.expand_conv.weight.data_ptr()
        for k, t in enumerate((self.expand_bn.weight, self.expand_bn.bias,
                               self.expand_bn.running_mean, self.expand_bn.running_var)):
            w.expand_bn[k] = t.data_ptr()
        for i, c in enumerate(self.layers_conv):
            w.layers_conv_weight[i] = c.weight.data_ptr()
        for i, m in enumerate(self.layers_bn):
            for k, t in enumerate((m.weight, m.bias, m.running_mean, m.running_var)):
                w.layers_bn[i][k] = t.data_ptr()
        w.shrink_weight = self.shrink.weight.data_ptr()
        w.shrink_bias = self.shrink.bias.data_ptr()
        return w

    def _versions(self):
        """What the packs are made from: ((data pointer, ``_version``) of every conv weight, the
        same of every BatchNorm / bias tensor followed by ``_stats_epoch``), tensors in the order of
        ``_param_tensors``.  The training kernels' running-stat updates are tracked through
        ``_stats_epoch`` because they bypass torch's version counters."""
        conv, bn = self._param_tensors()
        return (tuple((t.data_ptr(), t._version) for t in conv),
                tuple((t.data_ptr(), t._version) for t in bn) + (self._stats_epoch,))

    def _sync_weights(self, plan, stream, training=False):
        """Re-pack whatever changed since `plan`'s eval (or training) packs last saw the parameters
        (optimizer.step, load_state_dict, in-place edits).  Returns whether it packed."""
        if not training and plan.precision == "int8":
            self._sync_int8(plan)
        versions = self._versions()
        seen = plan.train if training else plan.eval
        what = 0
        if seen is None or seen[0] != versions[0]:
            what |= _capi.VP3D_PACK_CONV
            if training:
                what |= _capi.VP3D_PACK_CONV_T
        if not training and (seen is None or seen[1] != versions[1]):
            what |= _capi.VP3D_PACK_BN_EVAL
        if not what:
            return False
        conv, bn = self._param_tensors()
        for t in conv + bn:
            if t.dtype != torch.float32 or not t.is_contiguous():
                raise RuntimeError("parameters must be contiguous float32 tensors")
        w = self._weights_struct()
        _capi.check(_capi.load().vp3d_set_weights(plan, _capi.ctypes.byref(w), what, stream),
                    "vp3d_set_weights")
        if training:
            plan.train = versions
        else:
            plan.eval = versions
        return True

    # -- hooks for optim.FusedAdam (update + re-pack in one kernel) -----------------------------------
    def _packed_train_plan(self, device):
        """The training plan on `device` if it already holds packed weights (i.e. a training forward
        has run), else None: only such a plan can the fused optimizer keep current."""
        plan = self._engine.plans.get((device.index, self._train_precision))
        return plan if plan is not None and plan.train is not None else None

    def _mark_train_packs_current(self, plan, repacked):
        """The fused optimizer step has just re-packed the conv weights in `repacked` (the parameters
        it updated) on the training plan `plan`: record their new versions so that the next forward
        does not pack again.  Every other conv weight keeps the version its packs were made from, so
        a change that did not go through this step (another optimizer, an in-place edit of a frozen
        weight) still forces the full re-pack.  The step ran on the plan, so it is the one
        ``last_launch_count`` reports."""
        ids = {id(t) for t in repacked}
        conv, _ = self._param_tensors()
        now = self._versions()
        plan.train = (tuple(v if id(t) in ids else old
                            for t, v, old in zip(conv, now[0], plan.train[0])), now[1])
        self._engine.last = plan

    def _sync_expand_t(self, plan, stream):
        """Pack the transposed expand conv for the input gradient when expand_conv.weight changed
        since `plan` last packed it.  Only input-gradient backwards call this, and nothing else
        marks the pack current (the fused optimizer step does not refresh it), so a version bump
        of the weight always leads to a re-pack here."""
        seen = self._versions()[0][0]   # expand_conv.weight
        if plan.expand_t == seen:
            return
        w = self._weights_struct()
        _capi.check(_capi.load().vp3d_set_weights(plan, _capi.ctypes.byref(w),
                                                   _capi.VP3D_PACK_EXPAND_T, stream),
                    "vp3d_set_weights")
        plan.expand_t = seen

    def _grads_struct(self, grads):
        """vp3d_grads over `grads`, tensors in the order of ``_learnable_tensors``."""
        nb2 = len(self.layers_conv)
        g = _capi.Grads()
        g.expand_conv_weight = grads[0].data_ptr()
        g.expand_bn[0] = grads[1].data_ptr()
        g.expand_bn[1] = grads[2].data_ptr()
        for i in range(nb2):
            g.layers_conv_weight[i] = grads[3 + i].data_ptr()
            g.layers_bn[i][0] = grads[3 + nb2 + 2 * i].data_ptr()
            g.layers_bn[i][1] = grads[3 + nb2 + 2 * i + 1].data_ptr()
        g.shrink_weight = grads[3 + 3 * nb2].data_ptr()
        g.shrink_bias = grads[3 + 3 * nb2 + 1].data_ptr()
        return g

    def _get_workspace(self, nbytes, device):
        ws = self._engine.workspace
        if ws is None or ws.device != device or ws.numel() < nbytes:
            self._engine.workspace = None
            ws = torch.empty(nbytes, dtype=torch.uint8, device=device)
            self._engine.workspace = ws
        return ws

    # ------------------------------------------------------------------ forward
    def forward(self, x):
        assert len(x.shape) == 4
        assert x.shape[-2] == self.num_joints_in
        assert x.shape[-1] == self.in_features

        if not x.is_cuda:
            raise RuntimeError("videopose3d_b200 models run on CUDA (sm_90a) tensors only; "
                               "there is no CPU fallback")
        if x.dtype != torch.float32:
            raise TypeError(f"expected a float32 input, got {x.dtype}")
        if self.expand_conv.weight.device != x.device:
            raise RuntimeError("input and parameters are on different devices")
        if self.training:
            return self._forward_train(x)
        return self._forward_eval(x)

    def _forward_eval(self, x):
        params = self._learnable_tensors()
        if torch.is_grad_enabled() and (x.requires_grad or any(p.requires_grad for p in params)):
            reducer = getattr(self, "_grad_reducer", None)
            if reducer is not None and reducer.world > 1:
                raise NotImplementedError("eval-mode gradients are not all-reduced across ranks; "
                                          "detach the data-parallel reducer or run under no_grad")
            return _EvalFunction.apply(self, x.contiguous(), *params)
        return self._eval_launch(x)

    def _eval_launch(self, x):
        lib = _capi.load()
        x = x.contiguous()
        device = x.device
        N, T = int(x.shape[0]), int(x.shape[1])
        with torch.cuda.device(device):
            plan = self._use_plan(device, self._precision)
            stream = torch.cuda.current_stream(device).cuda_stream
            self._sync_weights(plan, stream)
            t_out = lib.vp3d_output_frames(plan, T)
            if t_out < 1:
                raise ValueError(f"input of {T} frames is shorter than the receptive field "
                                 f"({self.receptive_field()})")
            nbytes = lib.vp3d_workspace_bytes(plan, N, T)
            ws = self._get_workspace(nbytes, device)
            y = torch.empty((N, t_out, self.num_joints_out, 3), dtype=torch.float32, device=device)
            _capi.check(lib.vp3d_forward_eval(plan, x.data_ptr(), y.data_ptr(), N, T, ws.data_ptr(),
                                              ws.numel(), stream), "vp3d_forward_eval")
        return y

    def _forward_train(self, x):
        params = self._learnable_tensors()
        return _TrainFunction.apply(self, x.contiguous(), *params)

    def _learnable_tensors(self):
        """Learnable tensors in the order of ``vp3d_grads``."""
        out = [self.expand_conv.weight, self.expand_bn.weight, self.expand_bn.bias]
        out += [c.weight for c in self.layers_conv]
        for m in self.layers_bn:
            out += [m.weight, m.bias]
        out += [self.shrink.weight, self.shrink.bias]
        return out

    def _learnable_names(self):
        out = ["expand_conv.weight", "expand_bn.weight", "expand_bn.bias"]
        out += [f"layers_conv.{i}.weight" for i in range(len(self.layers_conv))]
        for i in range(len(self.layers_bn)):
            out += [f"layers_bn.{i}.weight", f"layers_bn.{i}.bias"]
        out += ["shrink.weight", "shrink.bias"]
        return out

    def set_train_precision(self, precision):
        """'bf16' (default) or 'bf16x3' (fp32-faithful gradients) for the training kernels."""
        if precision not in ("bf16", "bf16x3"):
            raise ValueError("train precision must be 'bf16' or 'bf16x3'")
        self._train_precision = precision
        return self

    def forward_host(self, x_host, out=None):
        """Eval forward from a HOST float32 tensor/array (pinned for full PCIe speed): copies the
        batch to the device, runs the kernels and copies the result back (the .cuda()/.cpu() round
        trip of run.py:663-672 in one call).  Used by bench.py for the end-to-end number."""
        lib = _capi.load()
        if self.training:
            raise RuntimeError("forward_host is an eval-mode call")
        x_host = torch.as_tensor(x_host)
        assert x_host.dim() == 4 and x_host.shape[-2] == self.num_joints_in \
            and x_host.shape[-1] == self.in_features
        if x_host.is_cuda or x_host.dtype != torch.float32 or not x_host.is_contiguous():
            raise ValueError("forward_host expects a contiguous float32 CPU tensor")
        device = self.expand_conv.weight.device
        if device.type != "cuda":
            raise RuntimeError("module parameters must be on a CUDA device")
        N, T = int(x_host.shape[0]), int(x_host.shape[1])
        with torch.cuda.device(device):
            plan = self._use_plan(device, self._precision)
            stream = torch.cuda.current_stream(device)
            self._sync_weights(plan, stream.cuda_stream)
            stream.synchronize()  # packed weights are read by the plan's own stream
            t_out = lib.vp3d_output_frames(plan, T)
            if t_out < 1:
                raise ValueError("input shorter than the receptive field")
            if out is None:
                out = torch.empty((N, t_out, self.num_joints_out, 3), dtype=torch.float32,
                                  pin_memory=True)
            _capi.check(lib.vp3d_forward_eval_host(plan, x_host.data_ptr(), out.data_ptr(), N, T),
                        "vp3d_forward_eval_host")
        return out

    def forward_host_submit(self, x_host, out, slot):
        """Pipelined form of forward_host: enqueue copy-in -> kernels -> copy-out for one batch on
        `slot` (0 or 1) and return immediately; `forward_host_wait(slot)` completes it.  Alternating
        the slots overlaps the PCIe copy of the next batch with the kernels of the current one.
        `x_host` and `out` must be pinned CPU float32 tensors that stay alive until the wait."""
        lib = _capi.load()
        if self.training:
            raise RuntimeError("forward_host_submit is an eval-mode call")
        if x_host.is_cuda or x_host.dtype != torch.float32 or not x_host.is_contiguous():
            raise ValueError("forward_host_submit expects a contiguous float32 CPU tensor")
        assert x_host.dim() == 4 and x_host.shape[-2] == self.num_joints_in \
            and x_host.shape[-1] == self.in_features
        device = self.expand_conv.weight.device
        N, T = int(x_host.shape[0]), int(x_host.shape[1])
        with torch.cuda.device(device):
            plan = self._use_plan(device, self._precision)
            stream = torch.cuda.current_stream(device)
            if self._sync_weights(plan, stream.cuda_stream):
                stream.synchronize()  # freshly packed weights are read by the plan's own stream
            _capi.check(lib.vp3d_forward_eval_host_submit(plan, x_host.data_ptr(), out.data_ptr(), N,
                                                          T, int(slot)),
                        "vp3d_forward_eval_host_submit")
        self._engine.host_slots[int(slot)] = plan
        return out

    def forward_host_wait(self, slot):
        """Block until the batch submitted on `slot` is in its `out`, on the plan it was submitted
        on (calls at other precisions in between do not matter)."""
        plan = self._engine.host_slots.pop(int(slot), self._engine.last)
        _capi.check(_capi.load().vp3d_forward_eval_host_wait(plan, int(slot)),
                    "vp3d_forward_eval_host_wait")

    def last_launch_count(self):
        return 0 if self._plan is None else _capi.load().vp3d_last_launch_count(self._plan)

    def streaming(self, streams, max_frames=1, augment=False, kps_left=None, kps_right=None,
                  joints_left=None, joints_right=None, provisional=False, int8=False,
                  detections=False, max_gap=None):
        """A StreamingSession (videopose3d_b200.streaming) of `streams` slots that takes up to
        `max_frames` new frames per slot and push, and returns each output frame as soon as its
        input has arrived.  `augment=True` with UnchunkedGenerator's left / right lists returns
        run.py's test-time flip average (run.py:674-680).  `provisional=True` (non-causal models
        only, ValueError otherwise) lets push(..., provisional=True) also return provisional
        poses for the frames still inside the look-ahead.  `int8=True` streams a model in
        precision 'int8' (ValueError in any other precision; an int8 model needs it), bit for bit
        its offline int8 forward.  `detections=True` (in_features == 2) makes a session fed by
        push_detections: a 2-D detector's pixel keypoints, a host per-frame detection flag and
        the camera resolution, with missed frames interpolated and screen-normalised on the device
        as the reference's in-the-wild pipeline does; `max_gap` bounds how many missed frames wait
        for the next detection.  Not in the reference."""
        from .streaming import StreamingSession
        return StreamingSession(self, streams, max_frames, augment=augment, kps_left=kps_left,
                                kps_right=kps_right, joints_left=joints_left,
                                joints_right=joints_right, provisional=provisional, int8=int8,
                                detections=detections, max_gap=max_gap)

    def predict(self, sequences, augment=False, kps_left=None, kps_right=None, joints_left=None,
                joints_right=None, max_rows=None):
        """Offline inference on a list of whole clips (videopose3d_b200.clips): CUDA fp32
        (T_i, J_in, F) tensors, T_i >= 1, in; their (T_i, J_out, 3) outputs (views into one
        buffer) out, in input order.  Each clip's output is the eval forward on the clip
        edge-padded as UnchunkedGenerator pads it, bit for bit (with `augment=True` and its left /
        right lists: run.py's flip average, run.py:674-680), computed by a few GEMM chains over
        the concatenated padded clips of at most `max_rows` packed rows each.  TemporalModel in
        eval() mode, any precision but 'mixed'; inference only (run it under torch.no_grad()).
        Not in the reference."""
        from .clips import predict
        return predict(self, sequences, augment=augment, kps_left=kps_left, kps_right=kps_right,
                       joints_left=joints_left, joints_right=joints_right, max_rows=max_rows)


def _train_forward(module, plan, x, stream, momenta=None, p_drop=0.0, seed=0, flags=0):
    """vp3d_forward_train_ex of `module` on `plan` (training packs current); returns y and the
    workspace that holds the activations its backward reads."""
    lib = _capi.load()
    N, T = int(x.shape[0]), int(x.shape[1])
    t_out = lib.vp3d_output_frames(plan, T)
    nbytes = lib.vp3d_train_workspace_bytes(plan, N, T)
    if t_out < 1 or nbytes == 0:
        raise ValueError(f"input of {T} frames is shorter than the receptive field "
                         f"({module.receptive_field()})")
    ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
    y = torch.empty((N, t_out, module.num_joints_out, 3), dtype=torch.float32, device=x.device)
    w = module._weights_struct()
    _capi.check(lib.vp3d_forward_train_ex(plan, x.data_ptr(), y.data_ptr(), N, T,
                                          _capi.ctypes.byref(w), momenta, p_drop, seed, flags,
                                          ws.data_ptr(), ws.numel(), stream),
                "vp3d_forward_train_ex")
    return y, ws


def _backward(module, plan, ws, dy, stream, want_x, dx_shape, want_p, shapes, reducer=None):
    """The vp3d_backward_ex call of both autograd functions, after a _train_forward on `plan`.

    Parameter gradients, when any is wanted, go to one tensor each, or with a data-parallel
    `reducer` to its flat buffer, whose stages the stage callback all-reduces while the later
    stages still compute; dL/dx, when wanted, to a new `dx_shape` tensor.  Returns dx (or None) and
    the gradients in the order of ``_learnable_tensors``, None for those not wanted."""
    device = dy.device
    grads = flat = cb = g = None
    errors = []
    if any(want_p):
        if reducer is not None:
            # one flat buffer laid out in backward-completion order: each stage is a contiguous
            # slice that is all-reduced on a side stream while later stages are still computing
            _, spans, stage_spans, total = reducer.plan_layout(module)
            flat = torch.empty(total, dtype=torch.float32, device=device)
            grads = [flat[spans[n][0]: spans[n][0] + spans[n][1]].view(s)
                     for n, s in zip(module._learnable_names(), shapes)]

            def _stage(stage, _user):
                try:
                    lo, hi = stage_spans[stage]
                    reducer.stage_ready(flat, lo, hi)
                except Exception as e:  # never raise through the C frame
                    errors.append(e)

            cb = _capi.STAGE_FN(_stage)
        else:
            grads = [torch.empty(s, dtype=torch.float32, device=device) for s in shapes]
        g = module._grads_struct(grads)
    dx = torch.empty(dx_shape, dtype=torch.float32, device=device) if want_x else None
    _capi.check(_capi.load().vp3d_backward_ex(
        plan, dy.data_ptr(), None if g is None else _capi.ctypes.byref(g),
        None if dx is None else dx.data_ptr(), ws.data_ptr(), ws.numel(), stream,
        None if cb is None else _capi.ctypes.cast(cb, _capi.ctypes.c_void_p), None),
        "vp3d_backward_ex")
    if errors:
        raise errors[0]
    if flat is not None:
        reducer.finish(flat)
    if grads is None:
        return dx, (None,) * len(want_p)
    return dx, tuple(gr if w else None for gr, w in zip(grads, want_p))


def _configure_bn_sync(module, plan):
    """Point `plan`'s synchronized BatchNorm at the module's reducer when it has sync_bn on, and
    switch it off otherwise; returns that reducer or None."""
    reducer = getattr(module, "_grad_reducer", None)
    want = reducer if reducer is not None and reducer.sync_bn else None
    have = plan.bn_sync[0] if plan.bn_sync is not None else None
    if want is have:
        return want
    lib = _capi.load()
    if want is None:
        _capi.check(lib.vp3d_set_bn_sync(plan, 0, 0, None, None), "vp3d_set_bn_sync")
        plan.bn_sync = None
        return None
    cb = want.bn_exchange_fn()
    _capi.check(lib.vp3d_set_bn_sync(plan, want.world, want.rank,
                                      _capi.ctypes.cast(cb, _capi.ctypes.c_void_p), None),
                "vp3d_set_bn_sync")
    plan.bn_sync = (want, cb)
    return want


class _TrainFunction(torch.autograd.Function):
    """Training-mode forward/backward through the C ABI (vp3d_forward_train_ex with flags 0 /
    vp3d_backward_ex).

    The learnable tensors are passed as inputs so that autograd accumulates the returned
    gradients into ``.grad`` exactly as it does for the reference's nn modules.  dL/dx is computed
    when x requires grad (the expand conv's data gradient); parameter gradients are skipped when no
    learnable tensor requires grad.  With a data-parallel reducer of more than one rank attached,
    the backward's stage callback all-reduces the gradients while it runs; with one that has
    sync_bn on (any number of ranks), forward and backward exchange every BatchNorm's statistics
    and sums with the other ranks."""

    @staticmethod
    def forward(ctx, module, x, *params):
        device = x.device
        momenta = [module.expand_bn.momentum] + [bn.momentum for bn in module.layers_bn]
        if any(m is None for m in momenta):
            raise NotImplementedError("BatchNorm momentum=None (cumulative average) is not supported")
        p_drop = float(module.drop.p)
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())  # CPU generator: torch.manual_seed applies
        with torch.cuda.device(device):
            plan = module._use_plan(device, module._train_precision)
            stream = torch.cuda.current_stream(device).cuda_stream
            module._sync_weights(plan, stream, training=True)
            sync = _configure_bn_sync(module, plan)
            mom = (_capi.ctypes.c_float * len(momenta))(*[float(m) for m in momenta])
            y, ws = _train_forward(module, plan, x, stream, mom, p_drop, seed)
        if sync is not None:
            sync.raise_errors()
        # nn.BatchNorm1d bookkeeping that lives outside the kernels
        with torch.no_grad():
            module.expand_bn.num_batches_tracked += 1
            for bn in module.layers_bn:
                bn.num_batches_tracked += 1
        module._stats_epoch += 1
        module._fwd_token += 1
        ctx.module = module
        ctx.plan = plan
        ctx.ws = ws
        ctx.token = module._fwd_token
        ctx.shapes = [tuple(p.shape) for p in params]
        ctx.x_shape = tuple(x.shape)
        ctx.device = device
        ctx.bn_sync = sync     # the C backward keeps this forward's setting
        return y

    @staticmethod
    def backward(ctx, dy):
        module = ctx.module
        if ctx.token != module._fwd_token:
            raise RuntimeError("only the most recent training forward of a module can be "
                               "back-propagated (one forward per backward, as in run.py)")
        dy = dy.contiguous().float()
        want_x = ctx.needs_input_grad[1]
        sync = ctx.bn_sync
        if sync is not None and sync.step_scale != 1.0:
            # the ragged-shard weight (set_step_rows) on dY: the BatchNorm backward sums mix every
            # rank's dY, so scaling this rank's gradients afterwards would miss its share in theirs
            dy = dy * sync.step_scale
        reducer = getattr(module, "_grad_reducer", None)
        if reducer is not None and reducer.world <= 1:
            reducer = None
        with torch.cuda.device(ctx.device):
            stream = torch.cuda.current_stream(ctx.device).cuda_stream
            if want_x:
                module._sync_expand_t(ctx.plan, stream)
            dx, grads = _backward(module, ctx.plan, ctx.ws, dy, stream, want_x,
                                  ctx.x_shape, ctx.needs_input_grad[2:], ctx.shapes, reducer)
        if sync is not None:
            sync.raise_errors()
        ctx.ws = None
        return (None, dx) + grads


class _EvalFunction(torch.autograd.Function):
    """Eval-mode forward inside autograd (model.eval() with x or parameters requiring grad).

    The forward is the plain eval forward (``vp3d_forward_eval``: same kernels, same bits as under
    ``no_grad``, no workspace kept).  The backward recomputes: a training-geometry forward with
    BatchNorm frozen to its running statistics (``VP3D_TRAIN_FROZEN_BN``) in the module's train
    precision, then ``vp3d_backward_ex``.  The gradient is therefore that of the train-precision
    forward ('bf16' or the fp32-faithful 'bf16x3', ``set_train_precision``), which is the reference's
    eval-mode backward: BatchNorm is a fixed affine, no dropout, running statistics untouched."""

    @staticmethod
    def forward(ctx, module, x, *params):
        y = module._eval_launch(x)
        ctx.module = module
        ctx.save_for_backward(x, *params)
        return y

    @staticmethod
    def backward(ctx, dy):
        module = ctx.module
        x = ctx.saved_tensors[0]     # (raises if x or a parameter was modified in place since)
        want_x = ctx.needs_input_grad[1]
        dy = dy.contiguous().float()
        device = x.device
        T = int(x.shape[1])
        with torch.cuda.device(device):
            plan = module._use_plan(device, module._train_precision)
            stream = torch.cuda.current_stream(device).cuda_stream
            module._sync_weights(plan, stream, training=True)
            if want_x:
                module._sync_expand_t(plan, stream)
            t_used = T
            if module._variant == _capi.VP3D_VARIANT_STRIDED:
                # the strided convs ignore trailing frames: recompute on the prefix the output
                # depends on (exact under frozen BatchNorm, whose affine does not see the batch)
                t_used = _capi.load().vp3d_output_frames(plan, T)
                for w in module.filter_widths:
                    t_used *= int(w)
            xs = x if t_used == T else x[:, :t_used].contiguous()
            _, ws = _train_forward(module, plan, xs, stream, flags=_capi.VP3D_TRAIN_FROZEN_BN)
            # the recompute replaced the plan's saved training state: a pending train-mode
            # backward of this module must now fail instead of reading it
            module._fwd_token += 1
            dx, grads = _backward(module, plan, ws, dy, stream, want_x,
                                  tuple(xs.shape), ctx.needs_input_grad[2:],
                                  [p.shape for p in ctx.saved_tensors[1:]])
        if dx is not None and t_used != T:
            full = torch.zeros(x.shape, dtype=torch.float32, device=device)
            full[:, :t_used] = dx
            dx = full
        return (None, dx) + grads


class TemporalModel(TemporalModelBase):
    """Dilated-convolution model, usable for every use-case (reference: common/model.py:79-138).

    Constructor signature identical to model.py:85-86:
    num_joints_in, in_features, num_joints_out, filter_widths, causal=False, dropout=0.25,
    channels=1024, dense=False (dense = ablation with regular convolutions of width 2*pad+1).
    """

    _variant = _capi.VP3D_VARIANT_DILATED

    def __init__(self, num_joints_in, in_features, num_joints_out,
                 filter_widths, causal=False, dropout=0.25, channels=1024, dense=False):
        super().__init__(num_joints_in, in_features, num_joints_out, filter_widths, causal, dropout,
                         channels)
        self._dense = bool(dense)
        self._build_layers(strided=False)


class TemporalModelOptimized1f(TemporalModelBase):
    """Strided model for single-frame batches: input length == receptive field, one output frame
    (reference: common/model.py:140-197).  Same parameters as TemporalModel, interchangeable
    weights; constructor signature identical to model.py:151-152.
    """

    _variant = _capi.VP3D_VARIANT_STRIDED

    def __init__(self, num_joints_in, in_features, num_joints_out,
                 filter_widths, causal=False, dropout=0.25, channels=1024):
        super().__init__(num_joints_in, in_features, num_joints_out, filter_widths, causal, dropout,
                         channels)
        self._build_layers(strided=True)
