"""Single-launch Adam / AMSGrad (SURVEY §8 row f4).

Drop-in for the optimiser the reference constructs with
`optim.Adam(model.parameters(), lr=lr, amsgrad=True)` (run.py:252, 264) and drives with
`optimizer.zero_grad()` / `optimizer.step()` (run.py:347, 396, 409, 420) and
`param_group['lr'] *= lr_decay` (run.py:583-586): same constructor arguments, same update rule,
same `state_dict()` layout (`step`, `exp_avg`, `exp_avg_sq`, `max_exp_avg_sq` per parameter), so
checkpoints written by either optimiser load into the other (run.py:295-296, 600-608).

`step()` hands every parameter of a group to `vp3d_adam_step` (csrc/step_ops.cu): one kernel launch
reads p, g, m, v, vmax and writes p, m, v, vmax once (36 B per element) instead of the eight
multi-tensor launches of torch's implementation.  CUDA float32 contiguous tensors only; anything
else raises -- there is no fallback path.

The bf16 re-pack of the conv weights is fused into the update: parameters that belong to a
`TemporalModel*` of this package (found automatically; `attach(model)` registers one explicitly)
go through `vp3d_adam_step_packed`, whose kernel writes the updated value straight into the
forward and transposed bf16 packs of the model's training plan, so the next training forward finds
them current (no pack kernels, no second read of the fp32 masters).  `fuse_repack = False` restores
the plain update + separate re-pack.
"""
import ctypes
import weakref

import torch

from . import _capi
from . import temporal_model as _tm

__all__ = ["FusedAdam"]


class FusedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False):
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, amsgrad=amsgrad)
        super().__init__(params, defaults)
        self._owners = {}     # id(param) -> weakref(model) for explicitly attached models
        self.fuse_repack = True   # parameters of TemporalModel* instances are found automatically
        self.last_launches = 0

    def attach(self, *models):
        """Fuse the conv-weight re-pack of these models into `step()` (see module docstring)."""
        for m in models:
            ref = weakref.ref(m)
            for prm in m.parameters():
                self._owners[id(prm)] = ref
        return self

    def __setstate__(self, state):
        super().__setstate__(state)
        for group in self.param_groups:
            group.setdefault("amsgrad", False)
        for st in self.state.values():  # checkpoints from old torch versions keep `step` as an int
            if "step" in st and not torch.is_tensor(st["step"]):
                st["step"] = torch.tensor(float(st["step"]), dtype=torch.float32)

    @staticmethod
    def _check(t, what):
        if not (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()):
            raise RuntimeError(f"FusedAdam: {what} must be a contiguous CUDA float32 tensor "
                               f"(got {t.device}, {t.dtype}, contiguous={t.is_contiguous()}); "
                               "there is no fallback path")

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        lib = _capi.load()
        self.last_launches = 0   # over every group of this step
        for group in self.param_groups:
            beta1, beta2 = group["betas"]
            by_step = {}  # parameters that share a step count share a launch
            for p in group["params"]:
                if p.grad is None:
                    continue
                if p.grad.is_sparse:
                    raise RuntimeError("FusedAdam does not support sparse gradients")
                self._check(p, "parameter")
                self._check(p.grad, "gradient")
                st = self.state[p]
                if len(st) == 0:
                    st["step"] = torch.tensor(0.0, dtype=torch.float32)
                    st["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    if group["amsgrad"]:
                        st["max_exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                elif group["amsgrad"] and "max_exp_avg_sq" not in st:
                    st["max_exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                for key in ("exp_avg", "exp_avg_sq") + (("max_exp_avg_sq",) if group["amsgrad"] else ()):
                    self._check(st[key], key)
                st["step"] += 1
                by_step.setdefault(int(st["step"].item()), []).append((p, st))
            for step, items in by_step.items():
                dev = items[0][0].device
                if any(p.device != dev for p, _ in items):
                    raise RuntimeError("FusedAdam: parameters of one group must share a device")
                # parameters of attached models whose training plan already holds packed weights go
                # through the fused update + re-pack entry, model by model; the rest the plain way
                by_model, plain = {}, []
                for p, st in items:
                    ref = self._owners.get(id(p))
                    m = ref() if ref is not None else _tm.owner_of(p)
                    plan = m._packed_train_plan(dev) if m is not None and self.fuse_repack else None
                    if plan is not None:
                        by_model.setdefault(id(m), (m, plan, []))[2].append((p, st))
                    else:
                        plain.append((p, st))

                def table_of(rows):
                    table = (_capi.AdamTensor * len(rows))()
                    for row, (p, st) in zip(table, rows):
                        row.param = p.data_ptr()
                        row.grad = p.grad.data_ptr()
                        row.exp_avg = st["exp_avg"].data_ptr()
                        row.exp_avg_sq = st["exp_avg_sq"].data_ptr()
                        row.max_exp_avg_sq = st["max_exp_avg_sq"].data_ptr() if group["amsgrad"] else None
                        row.numel = p.numel()
                    return table
                hyper = (step, float(group["lr"]), float(beta1), float(beta2), float(group["eps"]),
                         float(group["weight_decay"]))
                with torch.cuda.device(dev):
                    stream = torch.cuda.current_stream(dev).cuda_stream
                    if plain:
                        _capi.check(lib.vp3d_adam_step(table_of(plain), len(plain), *hyper, stream),
                                    "vp3d_adam_step")
                        self.last_launches += 1
                    for m, plan, rows in by_model.values():
                        w = m._weights_struct()
                        _capi.check(lib.vp3d_adam_step_packed(plan, ctypes.byref(w), table_of(rows),
                                                              len(rows), *hyper, stream),
                                    "vp3d_adam_step_packed")
                        self.last_launches += lib.vp3d_last_launch_count(plan)
                for p, _ in items:
                    # the kernel wrote through raw pointers: tell autograd / the weight-pack cache
                    torch.autograd.graph.increment_version(p)
                for m, plan, rows in by_model.values():   # after the version bumps above
                    m._mark_train_packs_current(plan, [p for p, _ in rows])
        return loss
