"""fp32 convolutions of the training path on libp3d's wgmma kernels (three-pass fp16 split = fp32 accuracy) instead of cuDNN's
fp32 SIMT kernels (TF32 is off during training, training_loop.py:278-279, which leaves cuDNN on its fp32 CUDA-core kernels).

Scope: what `conv2d_gradfix.conv2d` receives from the non-fused modulated convolutions of the generator and from the label-map
Encoder when gradients are required (`networks_stylegan2.py:68-75`, `conv2d_resample.py:134-136`): 3x3 (padding 1) and 1x1
(padding 0), stride 1, dilation 1, groups 1, no bias, fp32 NCHW; the Encoder's down=2 3x3 convolutions (`conv2d_resample.py:54-56`:
stride 2, padding 0 on the FIR-filtered (2H+1) x (2W+1) grid); and what `conv2d_gradfix.conv_transpose2d` receives from the
up=2 layers (`conv2d_resample.py:114-128`: 3x3, stride 2, padding 0 -> the (2H+1) x (2W+1) grid the FIR then filters).

Each node runs all three of its computations on libp3d:
- stride 1: forward and input gradient on `p3d_conv_gemm` (the input gradient is the same convolution with the kernel flipped
  and its channel axes swapped);
- transposed stride 2: forward as its four phase GEMMs in one launch, input gradient as a stride-2 'valid' convolution of the
  incoming gradient with the same weight tensor;
- strided stride 2: the reverse pair (forward = the stride-2 'valid' convolution, input gradient = the phase GEMMs);
- the weight gradient of every node on `p3d_conv_wgrad` (tcconv.conv_wgrad): one GEMM over pixels with both operands in
  NCHW order (pixels contiguous: the K-major tiles wgmma takes, no MN-major tiles needed), the second operand stored once per
  horizontal tap shift so that each tap is a whole-row offset.
First-order only: the nodes are used where no double backward can follow (inside `first_order()`, which the generator's
`mapping` / `synthesis` / `sample_mixed` enter; the discriminators, whose R1 penalty differentiates twice, never do).
"""
import contextlib

import torch

_depth = 0
enabled = True             # module switch (tests flip it for A/B)
min_pixels = 256           # below this the launch is latency-bound either way: leave it to cuDNN


@contextlib.contextmanager
def first_order():
    """Region in which convolutions are differentiated at most once."""
    global _depth
    _depth += 1
    try:
        yield
    finally:
        _depth -= 1


def applies(x, w, bias, stride, padding, dilation, groups):
    if not (enabled and _depth > 0 and bias is None and isinstance(x, torch.Tensor) and x.is_cuda):
        return False
    if x.dtype != torch.float32 or w.dtype != torch.float32 or x.ndim != 4:
        return False
    k = w.shape[2]
    if w.shape[2] != w.shape[3] or k not in (1, 3) or groups != 1:
        return False
    if tuple(stride) != (1, 1) or tuple(dilation) != (1, 1) or tuple(padding) != (k // 2, k // 2):
        return False
    if x.shape[2] * x.shape[3] < min_pixels or x.shape[0] > 4096:
        return False
    if w.shape[0] > 128 and w.shape[0] % 128:          # beyond one 128-channel tile the kernel wants whole tiles (256, 512, ...)
        return False
    if w.shape[1] > 128 and w.shape[1] % 128:          # (the input gradient swaps the channel roles)
        return False
    return torch.is_grad_enabled() and (x.requires_grad or w.requires_grad)


def _conv(x, w):
    """x [B,I,H,W] fp32, w [O,I,k,k] fp32 -> [B,O,H,W] fp32 (stride 1, 'same' padding), three tensor-core passes."""
    from ... import tcconv
    b, i, h, wd = x.shape
    o, _, k, _ = w.shape
    ip = tcconv.pad_to(i, 64)
    xh = tcconv.to_nhwc_f16(x.contiguous(), c_padded=ip, planes=2)                      # hi/lo split, channels padded
    ones = torch.ones(1, i, device=x.device, dtype=torch.float32)
    wk = tcconv.modulate_weights(w, ones, demodulate=False, pre_scale=1.0, planes=2, cin_padded=ip)   # K-major hi/lo, x WEIGHT_SCALE
    y = torch.empty(b, h, wd, o, device=x.device, dtype=torch.float32)
    taps = tcconv.TAPS_3X3 if k == 3 else tcconv.TAPS_1X1
    tcconv.conv_gemm(xh, wk, o, taps, (h, wd), y, out_mode=2, split=True, act=1, gain=1.0)
    return tcconv.nhwc_to_nchw_f32(y)


class _Conv2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w):
        ctx.save_for_backward(x, w)
        return _conv(x, w)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        from . import conv2d_gradfix
        from ... import tcconv
        x, w = ctx.saved_tensors
        dx = dw = None
        # gradients sit far below fp16's normal range (1e-6 and less), where the hi/lo split has no bits left: bring the
        # tensor's largest magnitude to ~2^10 with a power-of-two scale (exact), undo it on the result. The scale stays on
        # the device (no host read-back).
        scale = tcconv.pow2_scale(dy)
        if ctx.needs_input_grad[0]:
            dx = _conv(dy * scale, w.flip([2, 3]).transpose(0, 1).contiguous()) / scale
        if ctx.needs_input_grad[1] and not conv2d_gradfix.weight_gradients_disabled:
            dw = tcconv.conv_wgrad(dy, x, w.shape[2], 1, p_scale=scale)
        return dx, dw


def conv2d(x, w):
    return _Conv2d.apply(x, w)


# ----------------------------------------------------------------------------------------------
# stride-2 transposed 3x3 convolution (the up=2 layers)
# ----------------------------------------------------------------------------------------------
_TAPS_3X3_VALID = [(ky, kx, ky * 3 + kx) for ky in range(3) for kx in range(3)]


def applies_transposed(x, w, bias, stride, padding, output_padding, dilation, groups):
    """conv_transpose2d(x [B,I,H,W], w [I,O,3,3], stride 2, padding 0) inside a first_order() region."""
    if not (enabled and _depth > 0 and bias is None and isinstance(x, torch.Tensor) and x.is_cuda):
        return False
    if x.dtype != torch.float32 or w.dtype != torch.float32 or x.ndim != 4 or tuple(w.shape[2:]) != (3, 3) or groups != 1:
        return False
    if tuple(stride) != (2, 2) or tuple(padding) != (0, 0) or tuple(output_padding) != (0, 0) or tuple(dilation) != (1, 1):
        return False
    if x.shape[2] * x.shape[3] < min_pixels or x.shape[0] > 4096 or w.shape[0] != x.shape[1]:
        return False
    for ch in (w.shape[0], w.shape[1]):                # channel-tile rule of the kernel, for both roles (forward / input gradient)
        if ch > 128 and ch % 128:
            return False
    return torch.is_grad_enabled() and (x.requires_grad or w.requires_grad)


def _conv_transpose(x, wt):
    """x [B,I,H,W], wt [I,O,3,3] -> [B,O,2H+1,2W+1]: the four phases of the transposed convolution as one launch."""
    from ... import tcconv
    b, i, h, wd = x.shape
    o = wt.shape[1]
    ip = tcconv.pad_to(i, 64)
    xh = tcconv.to_nhwc_f16(x.contiguous(), c_padded=ip, planes=2)
    ones = torch.ones(1, i, device=x.device, dtype=torch.float32)
    wk = tcconv.modulate_weights(wt.transpose(0, 1).contiguous(), ones, demodulate=False, pre_scale=1.0, planes=2, cin_padded=ip)
    y = torch.empty(b, 2 * h + 1, 2 * wd + 1, o, device=x.device, dtype=torch.float32)
    tcconv.conv_transpose3x3_s2(xh, wk, o, y, split=True)
    return tcconv.nhwc_to_nchw_f32(y)


def _conv_stride2_valid(g, wt):
    """g [B,O,2H+1,2W+1], wt [I,O,3,3] -> [B,I,H,W]: dx[i,y,x] = sum g[o,2y+ky,2x+kx] wt[i,o,ky,kx] (adjoint of _conv_transpose)."""
    from ... import tcconv
    b, o, hh, ww = g.shape
    i = wt.shape[0]
    h, wd = (hh - 1) // 2, (ww - 1) // 2
    op = tcconv.pad_to(o, 64)
    gh = tcconv.to_nhwc_f16(g.contiguous(), c_padded=op, planes=2)
    ones = torch.ones(1, o, device=g.device, dtype=torch.float32)
    wk = tcconv.modulate_weights(wt.contiguous(), ones, demodulate=False, pre_scale=1.0, planes=2, cin_padded=op)
    y = torch.empty(b, h, wd, i, device=g.device, dtype=torch.float32)
    tcconv.conv_gemm(gh, wk, i, _TAPS_3X3_VALID, (h, wd), y, out_mode=2, split=True, act=1, gain=1.0, stride=2)
    return tcconv.nhwc_to_nchw_f32(y)


class _ConvTranspose2d(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, wt):
        ctx.save_for_backward(x, wt)
        return _conv_transpose(x, wt)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        from . import conv2d_gradfix
        from ... import tcconv
        x, wt = ctx.saved_tensors
        dx = dw = None
        scale = tcconv.pow2_scale(dy)          # power-of-two scaling before the fp16 split, as in _Conv2d
        if ctx.needs_input_grad[0]:
            dx = _conv_stride2_valid(dy * scale, wt) / scale
        if ctx.needs_input_grad[1] and not conv2d_gradfix.weight_gradients_disabled:
            dw = tcconv.conv_wgrad(x, dy, 3, 2, q_scale=scale)      # [in, out, 3, 3]: P = x, Q = the four phases of dy
        return dx, dw


def conv_transpose2d(x, wt):
    return _ConvTranspose2d.apply(x, wt)


# ----------------------------------------------------------------------------------------------
# stride-2 3x3 convolution, padding 0 (the label-map Encoder's down=2 layers after their FIR)
# ----------------------------------------------------------------------------------------------
def applies_strided(x, w, bias, stride, padding, dilation, groups):
    """conv2d(x [B,I,2H+1,2W+1], w [O,I,3,3], stride 2, padding 0) -> [B,O,H,W] inside a first_order() region."""
    if not (enabled and _depth > 0 and bias is None and isinstance(x, torch.Tensor) and x.is_cuda):
        return False
    if x.dtype != torch.float32 or w.dtype != torch.float32 or x.ndim != 4 or tuple(w.shape[2:]) != (3, 3) or groups != 1:
        return False
    if tuple(stride) != (2, 2) or tuple(padding) != (0, 0) or tuple(dilation) != (1, 1) or w.shape[1] != x.shape[1]:
        return False
    hh, ww = x.shape[2], x.shape[3]
    if hh % 2 == 0 or ww % 2 == 0 or (hh // 2) * (ww // 2) < min_pixels or x.shape[0] > 4096:
        return False
    for ch in (w.shape[0], w.shape[1]):                # channel-tile rule of the kernel, for both roles (forward / input gradient)
        if ch > 128 and ch % 128:
            return False
    return torch.is_grad_enabled() and (x.requires_grad or w.requires_grad)


class _Conv2dStride2(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w):
        ctx.save_for_backward(x, w)
        return _conv_stride2_valid(x, w)

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dy):
        from . import conv2d_gradfix
        from ... import tcconv
        x, w = ctx.saved_tensors
        dx = dw = None
        scale = tcconv.pow2_scale(dy)
        if ctx.needs_input_grad[0]:
            dx = _conv_transpose(dy * scale, w) / scale          # adjoint of the stride-2 'valid' convolution
        if ctx.needs_input_grad[1] and not conv2d_gradfix.weight_gradients_disabled:
            dw = tcconv.conv_wgrad(dy, x, 3, 2, p_scale=scale)   # [out, in, 3, 3]: P = dy, Q = the four phases of x
        return dx, dw


def conv2d_stride2(x, w):
    return _Conv2dStride2.apply(x, w)
