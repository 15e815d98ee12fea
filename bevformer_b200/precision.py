"""Which storage type the encoder path computes in, and entering it once at a public entry point.

Two mixed-precision mechanisms reach the kernels:
  * ``torch.autocast(device_type="cuda", dtype=torch.bfloat16 | torch.float16)`` -- PyTorch's own; the autocast dtype
    wins;
  * ``fp16_enabled = True`` on the module, which mmcv's ``wrap_fp16_model`` sets and its ``auto_fp16`` decorator
    answers by casting the inputs to half: the module computes in fp16 even outside autocast.
Otherwise the module computes in the dtype of its floating inputs.  The entry point casts the floating activations
once and runs its body with autocast off, so the glue's own torch ops are not re-cast op by op; parameters stay in
their own dtype (each projection casts its weight per call and autograd returns the gradient in the parameter's
dtype), and the result comes back in the compute dtype.
"""
from __future__ import annotations

import contextlib
import functools
import inspect

import torch


def compute_dtype(module, *tensors) -> torch.dtype:
    """The storage type ``module`` computes in for these inputs (first floating tensor decides the fallback)."""
    if torch.is_autocast_enabled("cuda"):
        return torch.get_autocast_dtype("cuda")
    if getattr(module, "fp16_enabled", False):
        return torch.float16
    for t in tensors:
        if torch.is_tensor(t) and t.is_floating_point():
            return t.dtype
    return torch.float32


def cast(x, dtype):
    """``x`` in ``dtype`` if it is a floating tensor (lists / tuples element-wise); anything else unchanged."""
    if torch.is_tensor(x):
        return x.to(dtype) if x.is_floating_point() and x.dtype != dtype else x
    if isinstance(x, (list, tuple)):
        return type(x)(cast(v, dtype) for v in x)
    return x


def entered(module, *tensors):
    """(dtype, context): the compute dtype, and a context that switches autocast off for the body when it was on."""
    dt = compute_dtype(module, *tensors)
    ctx = (torch.autocast(device_type="cuda", enabled=False) if torch.is_autocast_enabled("cuda")
           else contextlib.nullcontext())
    return dt, ctx


def entry(*activations):
    """Decorator for a module's public ``forward``: the arguments named in ``activations`` (tensors, or lists of
    tensors) are the floating activations cast to the compute dtype; every other argument (reference points,
    shapes, masks, ...) is passed unchanged.  Without autocast and without ``fp16_enabled`` the call goes straight
    through, so a module nested inside another entry point (whose body runs with autocast off) costs nothing."""
    def deco(fwd):
        sig = inspect.signature(fwd)

        @functools.wraps(fwd)
        def wrapper(self, *args, **kwargs):
            if not (torch.is_autocast_enabled("cuda") or getattr(self, "fp16_enabled", False)):
                return fwd(self, *args, **kwargs)
            bound = sig.bind(self, *args, **kwargs)
            acts = [bound.arguments.get(n) for n in activations]
            first = next((t for a in acts for t in (a if isinstance(a, (list, tuple)) else (a,))
                          if torch.is_tensor(t)), None)
            dt, amp_off = entered(self, first)
            done = {}      # an activation passed under several names (self-attention: key is query) stays one tensor
            for n in activations:
                if n in bound.arguments:
                    a = bound.arguments[n]
                    if torch.is_tensor(a):
                        if id(a) not in done:
                            done[id(a)] = (a, cast(a, dt))
                        bound.arguments[n] = done[id(a)][1]
                    else:
                        bound.arguments[n] = cast(a, dt)
            with amp_off:
                return fwd(*bound.args, **bound.kwargs)
        return wrapper
    return deco
