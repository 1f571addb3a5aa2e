"""`conv2d` / `conv_transpose2d` with arbitrarily high order gradients and an opt-out for weight gradients.

Surface of the reference's torch_utils/ops/conv2d_gradfix.py (:23 `enabled`, :26-33 `no_weight_gradients`,
:37-45 entry points). The forward / data-gradient / weight-gradient convolutions are ATen calls, exactly as in the reference
(:128-129, :169) -- except inside `native_conv.first_order()` regions (the generator's training passes), where the fp32
stride-1, strided (down=2) and transposed (up=2) convolutions run forward, input gradient and weight gradient on libp3d's wgmma
kernels (native_conv.py). The inference path does not go
through this module (engine.py drives the same kernels directly).
"""
import contextlib

import torch

enabled = False                     # training_loop.py:281 turns this on
weight_gradients_disabled = False   # set by no_weight_gradients() around the R1 penalty (loss.py:873)


@contextlib.contextmanager
def no_weight_gradients(disable=True):
    global weight_gradients_disabled
    old = weight_gradients_disabled
    if disable:
        weight_gradients_disabled = True
    yield
    weight_gradients_disabled = old


def _pair(v):
    return tuple(v) if isinstance(v, (tuple, list)) else (v, v)


def _use_custom(x):
    return enabled and isinstance(x, torch.Tensor) and x.device.type == 'cuda'


def conv2d(input, weight, bias=None, stride=1, padding=0, dilation=1, groups=1):
    from . import native_conv
    if native_conv.applies(input, weight, bias, _pair(stride), _pair(padding), _pair(dilation), groups):
        # fp32 training convolutions of the generator / label-map encoder: forward + input gradient on p3d_conv_gemm
        return native_conv.conv2d(input, weight)
    if native_conv.applies_strided(input, weight, bias, _pair(stride), _pair(padding), _pair(dilation), groups):
        # the label-map Encoder's down=2 layers: stride-2 'valid' convolution forward, phase GEMMs for the input gradient
        return native_conv.conv2d_stride2(input, weight)
    if _use_custom(input):
        return _make_op(False, weight.shape, _pair(stride), _pair(padding), (0, 0), _pair(dilation), groups).apply(
            input, weight, bias)
    return torch.nn.functional.conv2d(input=input, weight=weight, bias=bias, stride=stride, padding=padding,
                                      dilation=dilation, groups=groups)


def conv_transpose2d(input, weight, bias=None, stride=1, padding=0, output_padding=0, groups=1, dilation=1):
    from . import native_conv
    if native_conv.applies_transposed(input, weight, bias, _pair(stride), _pair(padding), _pair(output_padding), _pair(dilation), groups):
        # fp32 up=2 layers of the generator's training passes: phase GEMMs forward, stride-2 convolution for the input gradient
        return native_conv.conv_transpose2d(input, weight)
    if _use_custom(input):
        return _make_op(True, weight.shape, _pair(stride), _pair(padding), _pair(output_padding), _pair(dilation),
                        groups).apply(input, weight, bias)
    return torch.nn.functional.conv_transpose2d(input=input, weight=weight, bias=bias, stride=stride, padding=padding,
                                                output_padding=output_padding, groups=groups, dilation=dilation)


_op_cache = {}


def _make_op(transpose, weight_shape, stride, padding, output_padding, dilation, groups):
    """Autograd node whose backward is expressed with the same family of nodes, so double backward
    (R1 through the discriminator) works, and which skips the weight gradient on request."""
    key = (transpose, tuple(weight_shape), stride, padding, output_padding, dilation, groups)
    if key in _op_cache:
        return _op_cache[key]
    kw = dict(stride=stride, padding=padding, dilation=dilation, groups=groups)

    def adjoint_output_padding(in_shape, out_shape):
        if transpose:
            return (0, 0)
        return tuple(
            in_shape[i + 2] - (out_shape[i + 2] - 1) * stride[i] - (1 - 2 * padding[i]) - dilation[i] * (weight_shape[i + 2] - 1)
            for i in range(2))

    class Conv(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, w, b):
            assert w.shape == weight_shape
            ctx.save_for_backward(x if w.requires_grad else None, w if x.requires_grad else None)
            ctx.x_shape = x.shape
            ctx.has_bias = b is not None
            if transpose:
                return torch.nn.functional.conv_transpose2d(x, w, b, output_padding=output_padding, **kw)
            return torch.nn.functional.conv2d(x, w, b, **kw)

        @staticmethod
        def backward(ctx, dy):
            x, w = ctx.saved_tensors
            dx = dw = db = None
            if ctx.needs_input_grad[0]:
                op = _make_op(not transpose, weight_shape, stride, padding,
                              adjoint_output_padding(ctx.x_shape, dy.shape), dilation, groups)
                dx = op.apply(dy, w, None)
            if ctx.needs_input_grad[1] and not weight_gradients_disabled:
                dw = WeightGrad.apply(dy, x)
            if ctx.has_bias and ctx.needs_input_grad[2]:
                db = dy.sum([0, 2, 3])
            return dx, dw, db

    class WeightGrad(torch.autograd.Function):
        @staticmethod
        def forward(ctx, dy, x):
            ctx.save_for_backward(dy if x.requires_grad else None, x if dy.requires_grad else None)
            ctx.dy_shape, ctx.x_shape = dy.shape, x.shape
            # ATen's convolution_backward takes (grad_output, input) of the op described by `transposed`; no operand
            # swap for the transposed op (conv2d_gradfix.py:166-169 of the reference does the same)
            grads = torch.ops.aten.convolution_backward(
                dy, x, torch.empty(weight_shape, dtype=x.dtype, device=x.device), None,
                list(stride), list(padding), list(dilation), transpose, list(output_padding), groups,
                [False, True, False])
            return grads[1]

        @staticmethod
        def backward(ctx, d2w):
            dy, x = ctx.saved_tensors
            d_dy = d_x = None
            if ctx.needs_input_grad[0]:
                d_dy = Conv.apply(x, d2w, None)
            if ctx.needs_input_grad[1]:
                op = _make_op(not transpose, weight_shape, stride, padding,
                              adjoint_output_padding(ctx.x_shape, ctx.dy_shape), dilation, groups)
                d_x = op.apply(dy, d2w, None)
            return d_dy, d_x

    _op_cache[key] = Conv
    return Conv
