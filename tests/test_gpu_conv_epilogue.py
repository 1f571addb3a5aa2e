"""The two epilogues of the persistent conv kernel: on the accumulator fragments with fp16 TMA stores (`tma`), and staged
through shared memory as fp32 (`staged`).

conv_launch sends fp16 NHWC outputs with 8-channel-aligned offsets and strides (and no residual, ToRGB tail or split-K) to the
`tma` epilogue; `tools/time_conv.py`'s `tiling()` mirrors that rule. The same launch at channel offset 4 of a wider tensor takes
the staged epilogue, which must give the same bits. The TMA store clips ragged tiles and channels past Cout by itself, so the
model checks below run on grids and channel counts that leave partial boxes, with NaN sentinels around the written region.
"""
import types

import pytest
import torch

from test_gpu_conv_persistent import SQRT2, _inputs, _launch, _rgb_args, _sms, _tiling

gpu = pytest.mark.gpu


def _epi(args, kw, phases=None):
    return _tiling(args, kw, phases)['epi']


def _bw_of(gh, gw):
    """The tile width conv_launch picks for one phase of grid gh x gw (time_conv.tiling on a stand-in argument struct)."""
    from tools.time_conv import tiling
    p = types.SimpleNamespace(split=0, Cout_padded=64, stride=1, gH=gh, gW=gw, n_taps=1, C=64, B=1, splitk_scratch=0,
                              up_prev=None, residual=None, rgb_w=None, out_mode=0, y_coff=0, y_cstride=64, y=0, y_lo=None)
    return int(tiling([p], 132)['tile'].split('x')[0])


def _ragged_grid(bw):
    """The smallest grid for which the host picks tile width bw, with a full tile and a partial one in x (where bw > 1) and
    in y (where bh > 1)."""
    bh = 128 // bw
    best = None
    for gh in range(1, 300):
        for gw in range(1, 300):
            if (bw > 1 and (gw % bw == 0 or gw < bw)) or (bh > 1 and (gh % bh == 0 or gh < bh)) or gh * gw > 4 * 128 * 9:
                continue
            if (best is None or gh * gw < best[0] * best[1]) and _bw_of(gh, gw) == bw:
                best = (gh, gw)
    assert best is not None, bw
    return best


def test_ragged_grids_pick_every_tile_width():
    """The grids of test_every_tile_width_ragged do reach every tile width, ragged where the tile allows it (CPU)."""
    for bw in (1, 2, 4, 8, 16, 32, 64):
        gh, gw = _ragged_grid(bw)
        assert _bw_of(gh, gw) == bw and (bw == 1 or (gw % bw and gw > bw)) and gh % (128 // bw) and gh > 128 // bw


# ---------------------------------------------------------------------------------------------------------------------
# the two epilogues give the same bits
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('cout', [64, 128, 256])
@pytest.mark.parametrize('out_mode', [0, 1])
@pytest.mark.parametrize('act,alpha,gain,clamp', [(1, 0.2, 1.0, -1.0), (3, 0.2, SQRT2, -1.0), (3, 0.2, SQRT2, 0.5),
                                                  (3, -0.3, -0.7, 1.0)])
def test_tma_and_staged_epilogues_bit_identical(cout, out_mode, act, alpha, gain, clamp):
    """The same fp16 launch at channel offset 0 (tma) and at offset 4 of a wider tensor (staged): identical bits in every
    written element, for both output modes, linear / leaky-relu (max and select forms), with and without the clamp, BN 64
    and 128 (with two channel tiles at 256)."""
    from pix2pix3d_b200 import tcconv
    b, hw = 3, (21, 37)
    d = _inputs(b, 64, cout, hw, seed=cout + out_mode)
    outs = {}
    for y_coff, cs in ((0, cout), (4, cout + 8)):
        y = torch.full((b, hw[0], hw[1], cs), float('nan'), device='cuda', dtype=torch.float16)
        lo = torch.full_like(y, float('nan')) if out_mode == 1 else None
        kw = dict(out_mode=out_mode, out_lo=lo, y_coff=y_coff, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=act,
                  alpha=alpha, gain=gain, clamp=clamp, split_k=False)
        args = (d['x'], d['w'], cout, tcconv.TAPS_3X3, hw, y)
        assert _epi(args, kw) == ('tma' if y_coff == 0 else 'staged')
        _launch(args, kw)
        outs[y_coff] = [t[..., y_coff:y_coff + cout] for t in (y, lo) if t is not None]
    for t0, t4 in zip(outs[0], outs[4]):
        assert torch.equal(t0.view(torch.int16), t4.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------------------
# the tma epilogue against the float64 model, sentinels intact
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize('bw', [1, 2, 4, 8, 16, 32, 64])
def test_every_tile_width_ragged(bw):
    """Every tile width the host picks, on a grid with partial tiles in both directions: the store clips at the grid."""
    from pix2pix3d_b200 import tcconv
    hw = _ragged_grid(bw)
    d = _inputs(2, 64, 96, hw, seed=bw)
    y = torch.full((2, hw[0], hw[1], 96), float('nan'), device='cuda', dtype=torch.float16)
    kw = dict(out_mode=0, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2, split_k=False)
    args = (d['x'], d['w'], 96, tcconv.TAPS_3X3, hw, y)
    assert _epi(args, kw) == 'tma'
    r, t = _launch(args, kw)
    assert t['tile'] == f'{bw}x{128 // bw}'
    print(f'BW {bw}, grid {hw}: worst err / tol {r:.3g}')


@gpu
@pytest.mark.parametrize('cout', [64, 96, 128, 160, 256])
@pytest.mark.parametrize('out_mode', [0, 1])
def test_channel_counts(cout, out_mode):
    """Partial 64-channel halves (96, 160) and channel tiles past Cout (160: the second tile's upper half is empty)."""
    from pix2pix3d_b200 import tcconv
    b, hw = 2, (19, 23)
    d = _inputs(b, 64, cout, hw, seed=cout)
    y = torch.full((b, hw[0], hw[1], cout), float('nan'), device='cuda', dtype=torch.float16)
    lo = torch.full_like(y, float('nan')) if out_mode == 1 else None
    kw = dict(out_mode=out_mode, out_lo=lo, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2,
              clamp=2.0, split_k=False)
    args = (d['x'], d['w'], cout, tcconv.TAPS_3X3, hw, y)
    assert _epi(args, kw) == 'tma'
    r, _ = _launch(args, kw)
    print(f'Cout {cout}, out_mode {out_mode}: worst err / tol {r:.3g}')


@gpu
@pytest.mark.parametrize('y_coff,cs', [(8, 136), (64, 200)])
def test_concatenated_outputs(y_coff, cs):
    """Channels [y_coff, y_coff + 96) of a wider tensor: the other channels of each pixel keep their sentinels."""
    from pix2pix3d_b200 import tcconv
    b, hw = 3, (17, 29)
    d = _inputs(b, 64, 96, hw, seed=y_coff)
    y = torch.full((b, hw[0], hw[1], cs), float('nan'), device='cuda', dtype=torch.float16)
    kw = dict(out_mode=0, y_coff=y_coff, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2,
              split_k=False)
    args = (d['x'], d['w'], 96, tcconv.TAPS_3X3, hw, y)
    assert _epi(args, kw) == 'tma'
    r, _ = _launch(args, kw)
    print(f'y_coff {y_coff} of {cs}: worst err / tol {r:.3g}')


@gpu
@pytest.mark.parametrize('h,cout', [(16, 64), (64, 128), (128, 128)])
def test_merged_transposed_phases_odd_grids(h, cout):
    """The four phases of a stride-2 transposed convolution into a (2h+1)^2 grid (33^2, 129^2, 257^2): one output map per
    phase, each a strided view of the output; the phases interleave without overwriting each other."""
    from pix2pix3d_b200 import tcconv
    from test_gpu_conv_persistent import worst_ratio, snapshot
    b = 2
    d = _inputs(b, 64, cout, (h, h), per_sample=False, seed=h)
    out = torch.full((b, 2 * h + 1, 2 * h + 1, cout), float('nan'), device='cuda', dtype=torch.float16)
    phases = [(tcconv.tconv_phase_taps(py, px), (h + 1 - py, h + 1 - px), (2, py, 2, px)) for py in (0, 1) for px in (0, 1)]
    kw = dict(out_mode=0)
    args = (d['x'], d['w'], cout, None, None, out)
    assert _epi(args, kw, phases) == 'tma'
    snap = snapshot(out, kw)
    tcconv.conv_transpose3x3_s2(d['x'], d['w'], cout, out)
    torch.cuda.synchronize()
    r = worst_ratio(snap, args, kw, phases=phases)
    assert r <= 1.0, f'worst err / tol = {r:.3g}'
    print(f'{2 * h + 1}^2, Cout {cout}: worst err / tol {r:.3g}')


@gpu
def test_per_sample_weights_many_units():
    """Per-sample weights, dscale and noise with more samples than SMs, two channel tiles: every unit stores its own sample."""
    from pix2pix3d_b200 import tcconv
    b = _sms() + 3
    hw = (16, 8)
    d = _inputs(b, 64, 256, hw, seed=5)
    y = torch.full((b, hw[0], hw[1], 256), float('nan'), device='cuda', dtype=torch.float16)
    kw = dict(out_mode=0, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2, split_k=False)
    args = (d['x'], d['w'], 256, tcconv.TAPS_3X3, hw, y)
    assert _epi(args, kw) == 'tma'
    r, t = _launch(args, kw)
    assert t['units'] == 2 * b
    print(f'{b} samples: worst err / tol {r:.3g}')


@gpu
@pytest.mark.parametrize('rgb_cout', [1, 3, 6, 8])
@pytest.mark.parametrize('cout,skip_x', [(64, False), (96, True), (128, False), (128, True)])
def test_fused_torgb(rgb_cout, cout, skip_x):
    """The fused ToRGB reads its pixel's fp16 outputs back from the tile: 1 to 8 ToRGB channels, a partial second half
    (Cout 96), the activation stored or kept to the launch (skip_x)."""
    from pix2pix3d_b200 import tcconv
    b, hw = 3, (18, 26)
    d = _inputs(b, 64, cout, hw, seed=rgb_cout)
    y = torch.full((b, hw[0], hw[1], cout), float('nan'), device='cuda', dtype=torch.float16)
    rgb = _rgb_args(b, cout, hw, skip_x=skip_x, ci=rgb_cout)
    kw = dict(out_mode=0, bias=d['bias'], noise=d['noise'], dscale=d['dscale'], act=3, alpha=0.2, gain=SQRT2, clamp=256.0, rgb=rgb,
              split_k=False)
    args = (d['x'], d['w'], cout, tcconv.TAPS_3X3, hw, y)
    assert _epi(args, kw) == 'tma'
    r, _ = _launch(args, kw, fn='conv_gemm_try')
    if skip_x:
        assert torch.isnan(y).all()
    print(f'ToRGB {rgb_cout} of {cout}, skip_x {skip_x}: worst err / tol {r:.3g}')
