"""The autograd boundary of the trainable modules.

A trainable module runs its inference launch sequence once more, keeping the operands its backward reads (split
activations, fp16 qkv, the DCN head, ...) instead of recomputing them.  ``KeptLaunches`` is the one place that holds
those operands between forward and backward; ``tracked`` is the one test of whether a call needs it.
"""
import itertools

import torch


def tracked(inputs, params):
    """Grad mode is on and a tensor in ``inputs`` or a parameter in ``params`` requires grad: the call gets a
    ``grad_fn``.  ``None`` and non-tensor entries are skipped."""
    return torch.is_grad_enabled() and any(isinstance(t, torch.Tensor) and t.requires_grad
                                           for t in itertools.chain(inputs, params))


class KeptLaunches(torch.autograd.Function):
    """``KeptLaunches.apply(name, run, back, *args)``: a launch sequence with a backward pass.

    forward: ``out, saved = run(keep, *args)`` with ``keep`` an empty dict that ``run`` fills with what ``back`` reads;
    ``out`` is a tensor or a tuple of tensors, ``saved`` the tensors (``None`` allowed) handed to ``save_for_backward``,
    so that changing one in place between forward and backward (an ``optimizer.step()``) raises autograd's usual error
    instead of giving the gradient of the new values.

    backward: ``back(keep, saved, needs, *grads)`` returns one gradient (or ``None``) per entry of ``args``; ``needs``
    is ``needs_input_grad`` of ``args`` (False for non-tensor and ``None`` entries).  The backward frees ``keep``, so a
    second backward through the same output raises."""

    @staticmethod
    def forward(ctx, name, run, back, *args):
        keep = {}
        out, saved = run(keep, *args)
        ctx.name, ctx.back, ctx.keep = name, back, keep
        ctx.save_for_backward(*saved)
        return out

    @staticmethod
    def backward(ctx, *grads):
        if ctx.keep is None:
            raise RuntimeError(f"{ctx.name}: the backward frees the operands it keeps, so the output cannot be "
                               "backpropagated a second time (retain_graph=True is not supported); run the forward again")
        saved = ctx.saved_tensors           # raises if a saved tensor was modified in place since the forward
        keep, ctx.keep = ctx.keep, None
        return (None, None, None) + tuple(ctx.back(keep, saved, ctx.needs_input_grad[3:], *grads))
