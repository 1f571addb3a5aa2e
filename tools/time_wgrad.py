"""Weight gradients of the training generator's fp32 convolutions: ATen (cuDNN fp32, TF32 off as in training) against
p3d_conv_wgrad (tcconv.conv_wgrad), per layer shape of the afhq / seg2cat_512 training configuration at batch 4.

    python tools/time_wgrad.py [--batch 4] [--iters 20] [--warmup 5]

The two are timed alternately with CUDA events after a warm-up of both. Each row gives the median time of each, the
algorithmic TFLOP/s (2 * M * N * taps * pixels, one pass) and the max relative difference |new - ATen| / max|ATen|. The
p3d time includes the operand conversion (hi/lo planes on the padded grid) and the split-K reduction.
"""
import argparse
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from pix2pix3d_b200 import tcconv  # noqa: E402

# name, P channels (dY; x for the transposed up layers), Q channels, H, W (P's spatial size), k, stride
LAYERS = [
    ('backbone 3x3 4^2', 512, 512, 4, 4, 3, 1), ('backbone 3x3 8^2', 512, 512, 8, 8, 3, 1),
    ('backbone 3x3 16^2', 512, 512, 16, 16, 3, 1), ('backbone 3x3 32^2', 512, 512, 32, 32, 3, 1),
    ('backbone 3x3 64^2', 256, 256, 64, 64, 3, 1), ('backbone 3x3 128^2', 128, 128, 128, 128, 3, 1),
    ('backbone 3x3 256^2', 64, 64, 256, 256, 3, 1),
    ('ToRGB 1x1 64^2', 96, 256, 64, 64, 1, 1), ('ToRGB 1x1 256^2', 96, 64, 256, 256, 1, 1),
    ('up 3x3 s2 16->33', 512, 512, 16, 16, 3, 2), ('up 3x3 s2 32->65', 512, 512, 32, 32, 3, 2),
    ('up 3x3 s2 64->129', 256, 256, 64, 64, 3, 2), ('up 3x3 s2 128->257', 128, 128, 128, 128, 3, 2),
    ('Encoder fromrgb 1x1 512^2', 64, 19, 512, 512, 1, 1), ('Encoder conv0 3x3 512^2', 64, 64, 512, 512, 3, 1),
    ('Encoder conv0 3x3 256^2', 128, 128, 256, 256, 3, 1), ('Encoder conv0 3x3 128^2', 256, 256, 128, 128, 3, 1),
    ('Encoder skip 1x1 256^2', 128, 64, 256, 256, 1, 1), ('Encoder conv1 s2 513->256', 128, 64, 256, 256, 3, 2),
    ('Encoder conv1 s2 257->128', 256, 128, 128, 128, 3, 2), ('Encoder conv1 s2 129->64', 512, 256, 64, 64, 3, 2),
    ('Encoder conv1 s2 65->32', 512, 512, 32, 32, 3, 2),
]


def aten_wgrad(p, q, k, stride):
    m, n = p.shape[1], q.shape[1]
    w = torch.empty(m, n, k, k, device=p.device)
    if stride == 1:
        return torch.ops.aten.convolution_backward(p, q, w, None, [1, 1], [k // 2, k // 2], [1, 1], False, [0, 0], 1,
                                                   [False, True, False])[1]
    return torch.ops.aten.convolution_backward(p, q, w, None, [2, 2], [0, 0], [1, 1], False, [0, 0], 1, [False, True, False])[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_wgrad.py measures on a GPU; none is visible')
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    dev = torch.device('cuda')
    prop = torch.cuda.get_device_properties(dev)
    print(f'# {prop.name}, {prop.multi_processor_count} SMs, batch {args.batch}')
    print(f'{"layer":<28} {"splits":>6} {"ATen ms":>9} {"p3d ms":>9} {"ATen TF/s":>9} {"p3d TF/s":>9} {"speed-up":>8} {"max rel diff":>12}')
    tot_a = tot_p = 0.0
    for name, m, n, h, w, k, s in LAYERS:
        g = torch.Generator(device=dev).manual_seed(m + n + h)
        p = torch.randn(args.batch, m, h, w, device=dev, generator=g) * 1e-6
        qh, qw = (h, w) if s == 1 else (2 * h + 1, 2 * w + 1)
        q = torch.randn(args.batch, n, qh, qw, device=dev, generator=g)
        fns = (lambda: aten_wgrad(p, q, k, s), lambda: tcconv.conv_wgrad(p, q, k, s))
        for _ in range(args.warmup):
            for f in fns:
                f()
        times = ([], [])
        for _ in range(args.iters):
            for i, f in enumerate(fns):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                f()
                e1.record()
                torch.cuda.synchronize()
                times[i].append(e0.elapsed_time(e1))
        ta, tp = statistics.median(times[0]), statistics.median(times[1])
        ref, new = fns[0](), fns[1]()
        diff = float((new - ref).abs().max() / ref.abs().max().clamp_min(1e-30))
        flops = 2.0 * args.batch * h * w * m * n * k * k
        plan = tcconv.wgrad_plan(args.batch, m, n, (h, w), k, s, prop.multi_processor_count)
        tot_a += ta
        tot_p += tp
        print(f'{name:<28} {plan["splits"]:>6} {ta:9.3f} {tp:9.3f} {flops / ta / 1e9:9.1f} {flops / tp / 1e9:9.1f} '
              f'{ta / tp:8.2f} {diff:12.3g}')
    print(f'{"sum":<28} {"":>6} {tot_a:9.3f} {tot_p:9.3f} {"":>9} {"":>9} {tot_a / tot_p:8.2f}')


if __name__ == '__main__':
    main()
