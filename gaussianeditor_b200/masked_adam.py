"""``MaskedAdam``: torch's Adam restricted to the Gaussians under edit, one fused CUDA launch per step.

A GaussianEditor edit trains under a Gaussian mask: with ``render(..., grad_mask=mask)`` (or GaussianEditor's gradient
hooks) every unedited row's gradient is +0.0, and since the optimizer is created before the mask is applied and
densification appends rows with zero moments, an unedited row also has zero moments on every step. On such a row
``torch.optim.Adam`` writes back exactly the bits it read (``lerp(0, 0) = 0``, ``0 * beta2 + 0 = 0``,
``p - step_size * 0 / (0 + eps) = p``), yet still streams it through HBM. ``MaskedAdam`` skips those rows inside the
kernel (``gsr_adam_masked``, ``csrc/masked_adam.cu``): it neither reads nor writes them, and updates the edited rows
with Adam's arithmetic in fp32.
"""
from __future__ import annotations

import math

import torch

from . import _lib

# torch.optim.Adam's param-group options that MaskedAdam does not implement, at the values that leave Adam unchanged:
# groups carry them so that state dicts move between the two optimizers in both directions
_NEUTRAL = {"weight_decay": 0.0, "amsgrad": False, "maximize": False, "foreach": None, "fused": None,
            "differentiable": False, "decoupled_weight_decay": False}


def _check_options(group):
    for key, neutral in _NEUTRAL.items():
        val = group.get(key, neutral)
        if val != neutral and not (neutral is None and val is False):
            raise ValueError(f"MaskedAdam does not support {key}={val!r}")
    lr = group["lr"]
    if torch.is_tensor(lr):
        raise ValueError("MaskedAdam takes a float lr, not a tensor")
    if not 0.0 <= lr:
        raise ValueError(f"invalid lr: {lr}")
    b1, b2 = group["betas"]
    if not (0.0 <= b1 < 1.0 and 0.0 <= b2 < 1.0):
        raise ValueError(f"invalid betas: {group['betas']}")
    if not 0.0 <= group["eps"]:
        raise ValueError(f"invalid eps: {group['eps']}")


def _check_param(p, device=False):
    """dtype, layout and (`device`: at step time, so that state can be held and edited on the CPU) the device."""
    if p.dtype != torch.float32 or not p.is_contiguous() or p.dim() < 1:
        raise ValueError("MaskedAdam takes contiguous float32 tensors of at least one dimension, got "
                         f"{p.dtype} {tuple(p.shape)}" + ("" if p.is_contiguous() else " (non-contiguous)"))
    if device and not p.is_cuda:
        raise ValueError(f"MaskedAdam steps CUDA tensors only, got one on {p.device}")


class MaskedAdam(torch.optim.Optimizer):
    """``torch.optim.Adam`` (no weight decay, amsgrad or maximize) over the rows of a Gaussian cloud selected by a mask.

    Param groups follow ``optim_surgery``'s contract: each holds exactly one row-aligned float32, contiguous CUDA tensor,
    all with the same first dimension P (the Gaussian index). The state has ``torch.optim.Adam``'s layout for the same
    ``capturable`` flag (``step``: a CPU float32 tensor, or a device one when capturable; ``exp_avg``; ``exp_avg_sq``),
    created at the first step with a gradient, so ``optim_surgery``, ``shard_rebalance.rebalance``, GaussianEditor's
    ``_prune_optimizer`` / ``cat_tensors_to_optimizer`` and ``state_dict`` / ``load_state_dict`` with
    ``torch.optim.Adam`` (both directions) work on it unchanged.

    ``step()`` updates every group with a gradient in one kernel launch. Rows with ``mask[i] != 0`` get Adam's update;
    the other rows are neither read nor written. ``lr`` is read from each group at every step; with
    ``capturable=True`` the step is capturable in a CUDA graph (the float lr, the mask and the tensors are baked into
    the graph, as for torch's capturable Adam).

    ``set_mask(mask)`` takes a bool or uint8 CUDA tensor [P] (a bool mask is viewed, not copied); it must be called
    again whenever P changes (densification), otherwise ``step()`` raises ``ValueError``.

    Semantic difference from ``torch.optim.Adam``: the two agree bit for bit on an unedited row only while its gradient
    and moments are zero (the edit invariant). A row that leaves the mask while its moments are non-zero (for example
    when a mask is flipped) is frozen here, where torch's Adam would keep moving it on momentum.
    """

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, capturable=False, mask=None, **options):
        for key in options:
            if key not in _NEUTRAL:
                raise TypeError(f"MaskedAdam() got an unexpected keyword argument {key!r}")
        defaults = dict(lr=lr, betas=tuple(betas), eps=eps, capturable=bool(capturable), **_NEUTRAL)
        defaults.update(options)
        _check_options(defaults)
        self._mask = None
        super().__init__(params, defaults)
        if mask is not None:
            self.set_mask(mask)

    def add_param_group(self, param_group):
        super().add_param_group(param_group)
        group = self.param_groups[-1]
        _check_options(group)
        if len(group["params"]) != 1:
            raise ValueError("each MaskedAdam param group must hold exactly one tensor")
        _check_param(group["params"][0])

    def set_mask(self, mask: torch.Tensor):
        """The rows to update: a bool or uint8 CUDA tensor [P], kept by reference (not copied)."""
        if not torch.is_tensor(mask) or mask.dtype not in (torch.bool, torch.uint8):
            raise ValueError("mask must be a bool or uint8 tensor")
        if mask.dim() != 1:
            raise ValueError(f"mask must be 1-D [P], got shape {tuple(mask.shape)}")
        if not mask.is_cuda or not mask.is_contiguous():
            raise ValueError("mask must be a contiguous CUDA tensor")
        self._mask = mask.view(torch.uint8) if mask.dtype == torch.bool else mask

    @property
    def mask(self):
        return self._mask

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        mask = self._mask
        if mask is None:
            raise RuntimeError("MaskedAdam.step() needs a mask: call set_mask(mask) first")
        P, descs = None, []
        for group in self.param_groups:
            _check_options(group)
            p = group["params"][0]
            _check_param(p, device=True)
            if P is None:
                P = p.shape[0]
            elif p.shape[0] != P:
                raise ValueError(f"param groups have {P} and {p.shape[0]} rows: every group must have the same P")
            if p.grad is None:
                continue
            grad = p.grad
            if grad.is_sparse or grad.dtype != torch.float32 or grad.shape != p.shape or not grad.is_contiguous():
                raise ValueError("MaskedAdam needs dense contiguous float32 gradients shaped like their parameters")
            descs.append((group, p, grad))
        if mask.numel() != P:
            raise ValueError(f"the mask has {mask.numel()} rows but the param groups have P = {P}: "
                             "call set_mask after every densification")
        if not descs:
            return loss
        dev = descs[0][1].device
        if mask.device != dev or any(p.device != dev for _, p, _ in descs):
            raise ValueError("the mask and every parameter must be on one device")
        capturing = torch.cuda.is_current_stream_capturing()
        arr = (_lib.AdamGroup * len(descs))()
        for i, (group, p, grad) in enumerate(descs):
            capturable = group["capturable"]
            if capturing and not capturable:
                raise RuntimeError("MaskedAdam must be created with capturable=True to be captured in a CUDA graph")
            state = self.state[p]
            if len(state) == 0:   # torch.optim.Adam._init_group
                state["step"] = (torch.zeros((), dtype=torch.float32, device=p.device) if capturable
                                 else torch.tensor(0.0, dtype=torch.float32))
                state["exp_avg"] = torch.zeros_like(p, memory_format=torch.preserve_format)
                state["exp_avg_sq"] = torch.zeros_like(p, memory_format=torch.preserve_format)
            step, m, v = state["step"], state["exp_avg"], state["exp_avg_sq"]
            for t in (m, v):
                if t.shape != p.shape or t.dtype != torch.float32 or not t.is_contiguous() or t.device != p.device:
                    raise ValueError("exp_avg / exp_avg_sq must be contiguous float32 tensors shaped like the parameter")
            d = arr[i]
            d.p, d.g, d.m, d.v = p.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr()
            d.D = math.prod(p.shape[1:])
            d.lr, (d.beta1, d.beta2), d.eps = group["lr"], group["betas"], group["eps"]
            if capturable:
                if step.device != p.device or step.dtype != torch.float32:
                    raise ValueError("capturable=True needs a float32 step on the parameter's device")
                d.step_dev = step.data_ptr()   # advanced on the device by the call
            else:
                step += 1
                d.step = float(step)
        lib = _lib.load()
        with torch.cuda.device(dev):
            _lib.check(lib.gsr_adam_masked(arr, len(descs), P, mask.data_ptr(),
                                           torch.cuda.current_stream(dev).cuda_stream), "gsr_adam_masked")
        return loss
