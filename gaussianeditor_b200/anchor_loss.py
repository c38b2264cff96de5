"""``anchor_loss``: GaussianEditor's per-step anchor regularizer (``GaussianModel.anchor_loss``) on two CUDA launches
forward and one backward, without a host synchronisation.

GaussianEditor pulls every Gaussian under edit back towards a snapshot of its parameters (``model.anchor``), weighted
by the Gaussian's densification generation (``model._anchor_loss_schedule[model._generation]``). The reference body
boolean-indexes each of the six parameters and anchors with the mask, which waits on the host for the size of every
``nonzero`` and so cannot be captured in a CUDA graph. Here the mask is applied inside the kernels
(``gsr_anchor_loss_forward`` / ``gsr_anchor_loss_backward``, ``csrc/anchor_loss.cu``): the loss is reduced in fp64 in a
fixed order and rounded to fp32, and the backward writes the six gradients in one launch.

Switch GaussianEditor over with one line: ``GaussianModel.anchor_loss = gaussianeditor_b200.anchor_loss``.
"""
from __future__ import annotations

import math

import torch
from torch.autograd.function import once_differentiable

from . import _lib

# GaussianModel.update_anchor's keys, in the order of the C ABI's terms
TERMS = ("_xyz", "_features_dc", "_features_rest", "_scaling", "_rotation", "_opacity")
# the reference's output dict, in its order (the order of the kernel's out4)
KEYS = ("loss_anchor_color", "loss_anchor_geo", "loss_anchor_opacity", "loss_anchor_scale")
_MAX_D = 1 << 24   # GSR_ADAM_MAX_D


def _terms(params, anchors, grads=None):
    arr = (_lib.AnchorTerm * _lib.ANCHOR_TERMS)()
    for i, (p, a) in enumerate(zip(params, anchors)):
        d = arr[i]
        d.p, d.a, d.D = p.data_ptr(), a.data_ptr(), math.prod(p.shape[1:])
        d.g = grads[i].data_ptr() if grads is not None else None
    return arr


class _AnchorLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mask, generation, schedule, *tensors):
        params, anchors = tensors[:6], tensors[6:]
        lib = _lib.load()
        P, dev = mask.numel(), mask.device
        nbytes = lib.gsr_anchor_loss_scratch_bytes(P)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=dev)
        out = torch.empty(4, dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            _lib.check(lib.gsr_anchor_loss_forward(_terms(params, anchors), P, mask.data_ptr(), generation.data_ptr(),
                                                   schedule.data_ptr(), schedule.numel(), scratch.data_ptr(), nbytes,
                                                   out.data_ptr(), torch.cuda.current_stream(dev).cuda_stream),
                       "gsr_anchor_loss_forward")
        ctx.save_for_backward(mask, generation, schedule, scratch, *params, *anchors)
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_out):
        mask, generation, schedule, scratch, *tensors = ctx.saved_tensors
        params, anchors = tensors[:6], tensors[6:]
        lib = _lib.load()
        P, dev = mask.numel(), mask.device
        grads = [torch.empty_like(p) for p in params]   # every element is written
        go = grad_out.to(torch.float32).contiguous()
        with torch.cuda.device(dev):
            _lib.check(lib.gsr_anchor_loss_backward(_terms(params, anchors, grads), P, mask.data_ptr(),
                                                    generation.data_ptr(), schedule.data_ptr(), schedule.numel(),
                                                    scratch.data_ptr(), scratch.numel(), go.data_ptr(),
                                                    torch.cuda.current_stream(dev).cuda_stream),
                       "gsr_anchor_loss_backward")
        return (None, None, None, *grads) + (None,) * len(anchors)


def _check_tensor(name, t, dtype, shape=None):
    if not torch.is_tensor(t):
        raise ValueError(f"anchor_loss: {name} must be a tensor, got {type(t).__name__}")
    if t.dtype != dtype:
        raise ValueError(f"anchor_loss: {name} must be {dtype}, got {t.dtype}")
    if not t.is_contiguous():
        raise ValueError(f"anchor_loss: {name} must be contiguous")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise ValueError(f"anchor_loss: {name} has shape {tuple(t.shape)}, expected {tuple(shape)}")


def anchor_loss(model) -> dict:
    """``GaussianModel.anchor_loss`` of GaussianEditor (``scene/gaussian_model.py``) on this repository's kernels.

    Reads ``model._xyz``, ``_features_dc``, ``_features_rest``, ``_scaling``, ``_rotation``, ``_opacity`` (contiguous
    float32 CUDA tensors [P, ...]), ``model.anchor`` (their snapshots, same shapes), ``model.mask`` (bool [P]),
    ``model._generation`` (int64 [P]) and ``model._anchor_loss_schedule`` (float32 [G], G >= 1), all on one device.
    Returns ``{"loss_anchor_color", "loss_anchor_geo", "loss_anchor_opacity", "loss_anchor_scale"}``: 0-dim views of one
    [4] output, differentiable with respect to the six parameters. An empty ``model.anchor`` returns the reference's
    integer zeros without a launch. Only shapes, dtypes and devices are checked, so the call never synchronises and can
    be captured in a CUDA graph; the mask and the generations must still hold the same values when the backward runs.

    The values are the reference's: each term is the mean over the edited rows of ``w * (p - a)^2``, summed in fp64
    and rounded to fp32, and the groups (color = dc + rest, geo = xyz + rotation) add in fp32. As with torch, a term
    without elements (no edited row, or ``_features_rest`` at SH degree 0) is NaN and its gradient +0.0. One
    difference: a generation outside ``[0, len(schedule))`` gives its row a NaN weight, where ``torch.gather`` would
    trap. Raises ``ValueError`` on any other input, including an anchor dict that lacks or adds a key."""
    anchor = model.anchor
    if len(anchor) == 0:
        return {k: 0 for k in KEYS}
    if set(anchor) != set(TERMS):
        raise ValueError(f"anchor_loss: model.anchor must hold exactly {TERMS}, got {tuple(anchor)}")
    mask = model.mask
    if not torch.is_tensor(mask) or mask.dtype != torch.bool or mask.dim() != 1:
        raise ValueError("anchor_loss: model.mask must be a 1-D bool tensor")
    _check_tensor("model.mask", mask, torch.bool)
    P = mask.numel()
    if P >= 2 ** 31:
        raise ValueError(f"anchor_loss: P = {P} does not fit in int32")
    params = [getattr(model, key) for key in TERMS]
    anchors = [anchor[key] for key in TERMS]
    for key, p, a in zip(TERMS, params, anchors):
        _check_tensor(f"model.{key}", p, torch.float32)
        if p.dim() < 1 or p.shape[0] != P:
            raise ValueError(f"anchor_loss: model.{key} has shape {tuple(p.shape)}, expected [{P}, ...]")
        if math.prod(p.shape[1:]) > _MAX_D:
            raise ValueError(f"anchor_loss: model.{key} has more than {_MAX_D} floats per row")
        _check_tensor(f"model.anchor[{key!r}]", a, torch.float32, p.shape)
    generation, schedule = model._generation, model._anchor_loss_schedule
    _check_tensor("model._generation", generation, torch.int64, (P,))
    _check_tensor("model._anchor_loss_schedule", schedule, torch.float32)
    if schedule.dim() != 1 or schedule.numel() < 1:
        raise ValueError(f"anchor_loss: model._anchor_loss_schedule must be 1-D with at least one weight, "
                         f"got shape {tuple(schedule.shape)}")
    dev = mask.device
    if not mask.is_cuda:
        raise ValueError(f"anchor_loss: the tensors must be on a CUDA device, the mask is on {dev}")
    for t in (*params, *anchors, generation, schedule):
        if t.device != dev:
            raise ValueError(f"anchor_loss: every tensor must be on the mask's device {dev}, one is on {t.device}")
    out = _AnchorLoss.apply(mask.view(torch.uint8), generation, schedule, *params, *anchors)
    return {k: out[i] for i, k in enumerate(KEYS)}
