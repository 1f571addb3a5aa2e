"""Per-launch timing of the implicit-GEMM convolutions in one G.synthesis step (eager, CUDA events around every launch).

    python tools/time_conv.py [--workload seg2cat_512] [--steps 12] [--warmup 3] [--json FILE]

Prints one row per conv launch of a step: layer shape (B, computed grid, Cin, Cout, taps, phases, precision passes), the
tiling the library picks for it (BN, 128-pixel tiles, k-steps per tile, split-K factor, work units, and which epilogue:
`tma` on the accumulator fragments with TMA stores, or `staged` through shared memory), the median time over
the timed steps and the executed TFLOP/s (the fp32 layers execute three fp16 passes). The tiling columns mirror the host
rules of conv_launch in csrc/conv_gemm.cu.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from pix2pix3d_b200 import _lib, configs, native  # noqa: E402


def ceil_div(a, b):
    return -(-a // b)


def tiling(phases, sms):
    """BN, spatial tiles, channel tiles, k-steps per tile (per phase) and split-K factor of one launch (see conv_launch)."""
    p = phases[0]
    passes = 3 if p.split else 1
    bn = 128 if p.Cout_padded > 64 else 64 if p.Cout_padded > 32 else 32
    stride = max(p.stride, 1)
    bw, best = 1, -1
    for cand in (1, 2, 4, 8, 16, 32, 64):
        bh = 128 // cand
        if cand * stride > 256 or bh * stride > 256:
            continue
        area = sum(ceil_div(r.gW, cand) * cand * ceil_div(r.gH, bh) * bh for r in phases)
        if best < 0 or area <= best:
            best, bw = area, cand
    bh = 128 // bw
    tiles_m = sum(ceil_div(r.gW, bw) * ceil_div(r.gH, bh) for r in phases)
    tiles_n = ceil_div(p.Cout_padded, bn)
    ksteps = [r.n_taps * passes * p.C // 64 for r in phases]
    base = tiles_m * tiles_n * p.B
    splits = 1
    if p.splitk_scratch and not p.up_prev and not p.residual and not p.rgb_w and base * 2 <= sms and min(ksteps) >= 8:
        s = (2 * sms if len(phases) > 1 else sms) // base
        s = min(s, min(ksteps) // 4, 16)
        per_split = sum(p.B * r.gH * r.gW * p.Cout_padded * 4 for r in phases)
        while s > 1 and per_split * s > p.splitk_scratch_bytes:
            s -= 1
        if s > 1 and p.splitk_scratch % 32 == 0:
            splits = s
    # epilogue: on the accumulator fragments with TMA stores, or staged through shared memory as fp32
    tma = (p.out_mode <= 1 and not p.residual and not p.up_prev and splits == 1 and bn >= 64 and p.y_coff % 8 == 0
           and p.y_cstride % 8 == 0 and ((p.y or 0) | ((p.y_lo or 0) if p.out_mode == 1 else 0)) % 16 == 0)
    return dict(BN=bn, tile=f'{bw}x{bh}', tiles=tiles_m * tiles_n, ksteps=ksteps, splits=splits, units=base * splits,
                epi='tma' if tma else 'staged')


class _Recorder:
    """Forwards to the libp3d handle; remembers the arguments of every conv launch that the library accepted."""

    def __init__(self, handle):
        self._h = handle
        self.calls = []

    def __getattr__(self, name):
        return getattr(self._h, name)

    def p3d_conv_gemm(self, a, stream):
        st = self._h.p3d_conv_gemm(a, stream)
        if st == 0:
            src = a._obj
            self.calls.append([_lib.ConvArgs.from_buffer_copy(src)])
        return st

    def p3d_conv_gemm_phases(self, arr, n, stream):
        st = self._h.p3d_conv_gemm_phases(arr, n, stream)
        if st == 0:
            self.calls.append([_lib.ConvArgs.from_buffer_copy(arr[k]) for k in range(n)])
        return st


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--workload', default='seg2cat_512')
    ap.add_argument('--steps', type=int, default=12)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--json', default=None, help='also write the rows as JSON')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('time_conv.py needs a CUDA device')
    dev = torch.device('cuda', 0)
    w = configs.WORKLOADS[args.workload]
    G = configs.build_generator(args.workload, seed=0, device=dev, with_mapping=False)
    ws = configs.synthetic_ws(w['batch'], G.backbone.num_ws, 1).to(dev)
    c = configs.camera_labels(w['batch'], 2, w['preset']).to(dev)
    kw = dict(noise_mode='const', neural_rendering_resolution=w['nrr'])
    torch.manual_seed(0)
    with torch.no_grad():
        for _ in range(args.warmup):
            G.synthesis(ws, c, **kw)
    torch.cuda.synchronize()

    rec = _Recorder(_lib.lib())
    _lib._lib = rec
    per_step = None
    times, calls = [], None
    try:
        for _ in range(args.steps):
            rec.calls = []
            native.kernel_events = []
            with torch.no_grad():
                G.synthesis(ws, c, **kw)
            torch.cuda.synchronize()
            ev = [e for e in native.kernel_events if e[0] == 'conv_gemm']
            native.kernel_events = None
            assert len(ev) == len(rec.calls), (len(ev), len(rec.calls))
            if per_step is None:
                per_step, calls = len(ev), rec.calls
                flops = [(e[3], e[4]) for e in ev]
            assert len(ev) == per_step
            times.append([e[1].elapsed_time(e[2]) * 1e3 for e in ev])
    finally:
        _lib._lib = rec._h
        native.kernel_events = None

    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    rows = []
    for i, ph in enumerate(calls):
        p = ph[0]
        us = statistics.median(t[i] for t in times)
        t = tiling(ph, sms)
        rows.append(dict(i=i, B=p.B, grid='+'.join(f'{r.gH}x{r.gW}' for r in ph), Cin=p.C, Cout=p.Cout,
                         taps=sum(r.n_taps for r in ph), phases=len(ph), passes=3 if p.split else 1, rgb=bool(p.rgb_w), **t,
                         us=us, alg_gflop=flops[i][0] / 1e9, exec_gflop=flops[i][1] / 1e9, exec_tflops=flops[i][1] / us / 1e6))
    name = torch.cuda.get_device_name(dev)
    print(f'# {name}, {sms} SMs; {args.workload}, median of {args.steps} eager steps after {args.warmup} warm-up')
    print(f'{"#":>3} {"B":>2} {"grid":>23} {"Cin":>4} {"Cout":>4} {"taps":>4} {"ph":>2} {"pass":>4} {"BN":>3} {"tile":>6} '
          f'{"tiles":>6} {"k/tile":>11} {"split":>5} {"units":>6} {"epi":>6} {"us":>8} {"execTF/s":>8}')
    for r in rows:
        ks = '/'.join(str(k) for k in r['ksteps'])
        print(f'{r["i"]:>3} {r["B"]:>2} {r["grid"]:>23} {r["Cin"]:>4} {r["Cout"]:>4}{"+rgb" if r["rgb"] else "    "}'
              f'{r["taps"]:>4} {r["phases"]:>2} {r["passes"]:>4} {r["BN"]:>3} {r["tile"]:>6} {r["tiles"]:>6} {ks:>11} '
              f'{r["splits"]:>5} {r["units"]:>6} {r["epi"]:>6} {r["us"]:>8.1f} {r["exec_tflops"]:>8.1f}')
    tot_us = sum(r['us'] for r in rows)
    print(f'# {len(rows)} launches, {tot_us / 1e3:.3f} ms per step (sum of medians), '
          f'{sum(r["alg_gflop"] for r in rows) / tot_us * 1e3:.1f} TFLOP/s algorithmic, '
          f'{sum(r["exec_gflop"] for r in rows) / tot_us * 1e3:.1f} TFLOP/s executed')
    if args.json:
        with open(args.json, 'w') as fh:
            json.dump({'device': name, 'workload': args.workload, 'steps': args.steps, 'rows': rows}, fh, indent=1)


if __name__ == '__main__':
    main()
