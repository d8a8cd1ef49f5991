"""The optimizer step on libb200kge's kernels: `install_native_step(optimizer)` replaces `step` of one
torch.optim.Adagrad or torch.optim.SparseAdam instance by a step that runs engine.adagrad_step /
engine.sparse_adam_step per parameter (one fused pass over the elements each updates).

Only `step` changes.  param_groups, state, state_dict() / load_state_dict() and whatever writes group["lr"] (LR
schedulers, warm-up) keep working on the same object, and the state has torch's layout, so a checkpoint written with
the native step resumes with torch's and the reverse.  Each call reads its scalars from the groups and forms them in
double precision as torch 2.11 does (adagrad.py, _functional.sparse_adam); the kernels round every operation in
torch's order, but torch's own kernels may contract some of them into FMAs, so tables can differ at the ulp level.
"""
from __future__ import annotations

import math
import types
import weakref

import torch

from . import engine


def _on_cuda(p: torch.Tensor) -> bool:
    return p.is_cuda


def _param_reason(p: torch.Tensor):
    if not _on_cuda(p):
        return f"a parameter on {p.device} (the kernels run on CUDA)"
    if p.is_complex():
        return "a complex parameter"
    if p.dtype != torch.float32:
        return f"a {p.dtype} parameter (the kernels update float32)"
    if p.layout != torch.strided or not p.is_contiguous():
        return "a non-contiguous parameter"
    return None


def _group_reason(optimizer, group):
    if optimizer.__class__ is torch.optim.Adagrad:
        for key in ("maximize", "differentiable", "fused"):
            if group.get(key):
                return f"Adagrad with {key}=True"
    elif group.get("maximize"):
        return "SparseAdam with maximize=True"
    return None


def unsupported_reason(optimizer):
    """Why the native step cannot serve `optimizer`, or None if it can."""
    if optimizer.__class__ not in (torch.optim.Adagrad, torch.optim.SparseAdam):
        return f"{optimizer.__class__.__name__} (served: torch.optim.Adagrad and torch.optim.SparseAdam)"
    for group in optimizer.param_groups:
        reason = _group_reason(optimizer, group)
        for p in group["params"]:
            reason = reason or _param_reason(p)
        if reason:
            return reason
    return None


def _check(optimizer):
    reason = unsupported_reason(optimizer)
    if reason is not None:
        raise NotImplementedError(f"the native optimizer step does not serve {reason}")


def _adagrad_step(self, closure=None):
    """torch.optim.Adagrad.step on libb200kge: per group, the dense gradients of a group without a sparse one take
    the order of _multi_tensor_adagrad unless `foreach` is False (torch's default on CUDA is foreach); every other
    gradient takes _single_tensor_adagrad's."""
    loss = None
    if closure is not None:
        with torch.enable_grad():
            loss = closure()
    _check(self)
    self._opt_called = True         # what torch's LR schedulers' wrapper of `step` records
    for group in self.param_groups:
        params = [p for p in group["params"] if p.grad is not None]
        if not params:
            continue
        lr = float(group["lr"])
        lr_decay, wd, eps = group["lr_decay"], group["weight_decay"], group["eps"]
        # one device per group (torch groups by device and dtype; every parameter here is float32)
        sparse_devices = {p.device for p in params if p.grad.is_sparse}
        for p in params:
            state = self.state[p]
            step_t = state["step"]
            step_t += 1
            step = step_t.item()
            if wd != 0 and p.grad.is_sparse:
                raise RuntimeError("weight_decay option is not compatible with sparse gradients")
            clr = lr / (1 + (step - 1) * lr_decay)
            foreach_order = group["foreach"] is not False and p.device not in sparse_devices
            engine.adagrad_step(p, state["sum"], p.grad, clr, eps, wd, foreach_order)
    return loss


def _sparse_adam_step(self, closure=None):
    """torch.optim.SparseAdam.step on libb200kge, with torch's state initialisation and step count."""
    loss = None
    if closure is not None:
        with torch.enable_grad():
            loss = closure()
    _check(self)
    self._opt_called = True
    for group in self.param_groups:
        beta1, beta2 = group["betas"]
        todo = []
        for p in group["params"]:
            if p.grad is None:
                continue
            if not p.grad.is_sparse:
                raise RuntimeError("SparseAdam does not support dense gradients, please consider Adam instead")
            state = self.state[p]
            if len(state) == 0:
                state["step"] = 0
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            state["step"] += 1
            todo.append((p, state))
        lr = float(group["lr"])
        for p, state in todo:
            step = state["step"]
            step_size = lr * math.sqrt(1 - beta2 ** step) / (1 - beta1 ** step)
            engine.sparse_adam_step(p, state["exp_avg"], state["exp_avg_sq"], p.grad, beta1, beta2, group["eps"],
                                    step_size)
    return loss


def install_native_step(optimizer):
    """Bind the native `step(closure=None)` to this optimizer instance (torch's optimizer hooks and profiler label
    still apply).  Raises NotImplementedError naming the reason if the optimizer type, a group option (maximize,
    differentiable, fused) or a parameter (not a contiguous float32 CUDA tensor) is not served."""
    _check(optimizer)
    fn = _adagrad_step if optimizer.__class__ is torch.optim.Adagrad else _sparse_adam_step
    # bound to a weak proxy: the instance attribute must not keep the optimizer (and its state) alive in a cycle
    step = types.MethodType(torch.optim.Optimizer.profile_hook_step(fn), weakref.proxy(optimizer))
    step.__func__._b200_native = True
    optimizer.step = step
    return optimizer


def is_native(optimizer) -> bool:
    """True if `optimizer.step` is the native step (possibly wrapped by a torch LR scheduler)."""
    return bool(getattr(optimizer.step, "_b200_native", False))
