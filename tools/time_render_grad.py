"""Time ImportanceRenderer.forward + backward under autograd at BASELINE config-5 shapes (4 images, 128^2 rays, 48 + 48
samples, OSGDecoder_semantic_lateSeparate): the fused path (_FusedRender: p3d_render_fwd + p3d_render_bwd) against the
staged chain, alternating the two, with CUDA events; prints per-call times (min / median / max) and the peak memory rise."""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from pix2pix3d_b200.training import triplane_cond as tc  # noqa: E402
from pix2pix3d_b200.training.volumetric_rendering import renderer as rmod  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=4)
    ap.add_argument('--res', type=int, default=128)
    ap.add_argument('--reps', type=int, default=10)
    args = ap.parse_args()
    dev = torch.device('cuda')
    torch.manual_seed(0)
    dec = tc.OSGDecoder_semantic_lateSeparate(32, {'decoder_lr_mul': 1.0, 'decoder_output_dim': 32, 'sigmoid': False}).to(dev)
    planes = (0.5 * torch.randn(args.batch, 3, 32, 256, 256, device=dev)).requires_grad_(True)
    R = args.res * args.res
    o = torch.randn(args.batch, R, 3, device=dev)
    o = o / o.norm(dim=-1, keepdim=True) * 2.7
    d = -o + 0.3 * torch.randn_like(o)
    d = d / d.norm(dim=-1, keepdim=True)
    opts = dict(depth_resolution=48, depth_resolution_importance=48, ray_start=2.25, ray_end=3.3, box_warp=1.0,
                disparity_space_sampling=False, clamp_mode='softplus', white_back=False)
    r = rmod.ImportanceRenderer().to(dev)

    def step():
        feat, depth, wsum = r(planes, dec, o, d, opts)
        loss = feat.sum() + depth.sum() + wsum.sum()
        torch.autograd.grad(loss, [planes] + list(dec.parameters()))

    times = {'fused': [], 'staged': []}
    peaks = {}
    for name, flag in (('fused', True), ('staged', False)):      # warm-up and peak memory
        rmod.fused_grad = flag
        step()
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        step()
        torch.cuda.synchronize()
        peaks[name] = (torch.cuda.max_memory_allocated() - base) / 1e9
    for _ in range(args.reps):
        for name, flag in (('fused', True), ('staged', False)):
            rmod.fused_grad = flag
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1))
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    out = {'gpu': gpu, 'shape': [args.batch, R, 48, 48]}
    for name in times:
        t = times[name]
        out[name] = {'ms_min': min(t), 'ms_median': statistics.median(t), 'ms_max': max(t), 'peak_rise_gb': peaks[name]}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
