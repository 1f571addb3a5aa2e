"""The streaming kernels of the discriminators and the fp16 super-resolution layers -- p3d_bias_act, p3d_upfirdn2d and p3d_fma
-- against a float64 model of each launch, element by element.

Under autograd these three run every activation and FIR filter of both discriminators, forward, backward and in the R1 double
backward, in fp16 on the blocks at 64^2 and above. Each model takes the operands and scalars exactly as the Python wrapper passes
them to the C ABI and returns, per element, the float64 value `ref` and a bound `tol` on what the kernel may return.

Arithmetic. `u` is the unit roundoff of the kernel's compute type: 2^-24 (fp32, also for fp16 storage, whose operands widen
exactly) or, for fp64, 2^-52 -- two units of 2^-53, because the model is itself evaluated in float64. Every bound is a sum of
`k u` times the magnitudes the kernel forms on the way (so that cancellation is paid for), plus a floor of a few smallest normal
numbers of the compute type for underflow. fp16 outputs add half an fp16 ulp of |ref| + tol (the final __float2half_rn) and
2^-25, the half-spacing of fp16 subnormals.

- bias_act (`bias_act_eval` in bias_act.cu). alpha, gain and clamp are fp32 (the ABI's C floats). The forward input v = x + b is
  one rounding (u|v|), which moves a transcendental's result by u|v| relative (e^v); the CUDA Math API bounds expf at 2 ulp
  (<= 4u relative) and logf at 1 ulp (<= 2u), and IEEE division, reciprocal, add and multiply at u each. Per activation, with
  a the activation value and c = e^(+-v):
    linear u|v|; relu u|a|; lrelu 2u|a|; tanh u(|v| + 8)(1 + |a|) (c - 1/c over c + 1/c: both sums carry the relative error of
    c, |v| u + 4u, and one rounding each); sigmoid u(|v| + 6)|a|; elu c u(|v| + 4) + u|a| (e^v - 1 cancels near 0); selu the
    same times lambda*alpha plus 4u|a| for the constants; softplus c/(1+c) u(|v| + 4) + u + 2u|a| (log of the rounded 1 + c);
    swish u(|v| + 7)|a|.
  Then y = a gain (u|y|) and the clamp, which is 1-Lipschitz and so carries the bound unchanged. The gradient forms (grad 1, 2)
  read yy = yref / gain (u): each factor's relative error is summed over the magnitude of the product with every difference
  replaced by the sum of its terms' magnitudes, e.g. tanh grad 1: 4u |x| (yy^2 + |1 - yy^2|); swish recomputes e^(x+b) and
  pays u(4|x+b| + 24) (grad 1) or u(6|x+b| + 40) (grad 2) on |x| c (|x+b| + d) / d^2 (resp. its grad-2 analogue over d^3),
  d = c + 1. Then * (gain * dy): 2u|y|.
  Branches. Those taken on a stored value -- yref's sign, the clamp gate |yref| < clamp on the stored yref (so a forward output
  clamped to 181.0193 and stored in fp16 as 181.0 lets its gradient through, as the reference plugin does) -- are modelled
  exactly and must match. Those taken on a value the kernel computes in fp32 -- the saturation tests of x + b at +-80 and +-40,
  swish's recomputed yref against the clamp, and the overflow of d^3 in fp32 (which makes the kernel return 0 for swish
  grad 2 above x + b ~ 29.6) -- may go either way within their own bound of the threshold; there either branch is accepted
  and the elements are counted as margin elements.
- upfirdn2d: the direct polyphase sum, tap (ty, tx) of the mirrored filter (unless flip) reading the zero-inserted, padded input
  at (o * down - pad0 + t) / up. The accumulation is a chain of fmaf: (taps + 1) u S with S = |gain| sum |f||x| (taps = fh fw;
  the generic fp32 / fp64 kernels write `acc += f * x`, which may or may not be contracted: 2 taps + 1).
- fma: fp32 (fp64) fma of the widened operands, one rounding: u|ref|, plus 2^-53 (|ab| + |c|) for the model's own float64 sum.

The grid rules and path choices of the three launchers are mirrored here (`ba_grid`, `fir_grid`, `fma_grid`, ...) so that the
sweep's shapes can be shown, without a GPU, to reach every edge they are meant to for any SM count.
"""
import math

import numpy as np
import pytest
import torch

from test_gpu_synth_aux import _ulp16, f32, rn16

gpu = pytest.mark.gpu

U32 = 2.0 ** -24
U64 = 2.0 ** -52              # two units of 2^-53: the kernel's rounding and the model's own
H16 = 2.0 ** -25              # half the fp16 subnormal spacing
FLOOR = {torch.float64: 8 * 2.0 ** -1022}
SELU_L = 1.0507009873554804934193349852946
SELU_A = 1.6732632423543772848170429916717
ACTS = ['linear', 'relu', 'lrelu', 'tanh', 'sigmoid', 'elu', 'selu', 'softplus', 'swish']
ACT_IDX = {a: i + 1 for i, a in enumerate(ACTS)}
HAS_2ND = {'tanh', 'sigmoid', 'elu', 'selu', 'softplus', 'swish'}
REF = {'linear': '', 'swish': 'x'}                      # the others save y
CLAMP_D = f32(256 * math.sqrt(0.5))                      # D's resnet conv1: conv_clamp 256 times the skip gain sqrt(1/2)


def _u(dtype):
    return U64 if dtype == torch.float64 else U32


def _floor(dtype):
    return FLOOR.get(dtype, 8 * 2.0 ** -126)


def _ceil(a, b):
    return -(-a // b)


def _vec(dtype):
    return 16 // torch.empty((), dtype=dtype).element_size()


def _flat(t):
    """The elements of a dense tensor in memory order (what the kernel indexes)."""
    return t.as_strided((t.numel(),), (1,))


def _out_tol(y, e, dtype):
    if dtype == torch.float16:
        return e + 0.5 * _ulp16(y.abs() + e) + H16
    return e


# ---------------------------------------------------------------------------------------------------------------------
# grid rules and path choices, mirrored
# ---------------------------------------------------------------------------------------------------------------------
def ba_grid(size_x, V, sms):
    """launch_bias_act_g: ~4 vectors per thread; past one wave of 8 CTAs / SM, whole waves, at most 4."""
    blocks = _ceil(_ceil(size_x, 4 * V), 256)
    wave = 8 * sms
    if blocks > wave:
        k = _ceil(blocks, wave)
        blocks = 4 * wave if k > 4 else k * wave
    return max(blocks, 1)


def ba_vec_path(ptrs, has_b, step_b, V):
    """(vector loop runs, bias shared by a whole vector): every non-null operand and y 16-byte aligned; step_b % V == 0."""
    aligned = all(p % 16 == 0 for p in ptrs if p)
    return aligned, (not has_b) or step_b % V == 0


def ba_sizes(V, sms):
    """The sweep's sizes: below one vector, the size % V tails, one wave of CTAs -1 / exact / +1, the 4-wave cap and twice it."""
    wave, per_cta = 8 * sms, 256 * 4 * V
    return {'lt_V': V - 1, 'mod_0': 96 * V, 'mod_1': 96 * V + 1, 'mod_V-1': 96 * V + V - 1,
            'wave-1': (wave - 1) * per_cta, 'wave': wave * per_cta, 'wave+1': (wave + 1) * per_cta,
            'cap': 4 * wave * per_cta, '2x_cap': 8 * wave * per_cta + V + 1}


def fir_grid(items, sms):
    """grid_for: one item per thread up to one wave of 8 CTAs / SM, then whole waves, at most 8."""
    blocks = _ceil(items, 256)
    wave = 8 * sms
    if blocks > wave:
        blocks = min(_ceil(blocks, wave), 8) * wave
    return max(blocks, 1)


STRIP_TX = {(1, 1): 4, (2, 1): 4, (1, 2): 2}


def _contig_nchw(shape, stride):
    s = 1
    for d in (3, 2, 1, 0):
        if shape[d] != 1 and stride[d] != s:
            return False
        s *= shape[d]
    return True


def fir_route(dtype, xs, xst, ys, yst, fw, fh, upx, upy, downx, downy):
    """p3d_upfirdn2d's choice: a strip instance 'strip u{up}d{down}' or 'generic'."""
    if (dtype != torch.float64 and upx == upy and downx == downy and _contig_nchw(xs, xst) and _contig_nchw(ys, yst)
            and fw == 4 and fh == 4 and (upx, downx) in STRIP_TX):
        return f'strip u{upx}d{downx}'
    return 'generic'


def fir_items(route, ys):
    n, c, oh, ow = ys
    if route == 'generic':
        return n * c * oh * ow
    tx = STRIP_TX[(int(route[7]), int(route[9]))]
    return n * c * oh * _ceil(ow, tx)


def fir_cap(sms):
    return 8 * 8 * sms * 256


def fma_grid(n, sms):
    return min(_ceil(n, 256), 16 * sms)


def fma_vec_path(dtype, shape4, ptrs, strides, y_ptr):
    es = torch.empty((), dtype=dtype).element_size()
    vec = 16 // es
    if shape4[3] % vec or y_ptr % 16:
        return False
    for p, s in zip(ptrs, strides):
        if s[3] == 0:
            continue
        if s[3] != 1 or p % 16 or any((s[i] * es) % 16 for i in range(3)):
            return False
    return True


def fma_cap(sms):
    return 16 * sms * 256


# ---------------------------------------------------------------------------------------------------------------------
# bias_act model
# ---------------------------------------------------------------------------------------------------------------------
def bias_act_model(x, b, xref, yref, dy, dtype, grad, act_idx, alpha, gain, clamp, size_b, step_b, fault=None):
    """One p3d_bias_act launch: x, xref, yref, dy flat in memory order (None = null pointer), b [size_b].
    Returns dict(ref, tol, alts=[(value, mask)], margin): `alts` are the other side of branches decided on fp32 values."""
    u, fl = _u(dtype), _floor(dtype)
    alpha, gain, clamp = f32(alpha), f32(gain), f32(clamp)
    act = ACTS[act_idx - 1]
    X = x.double()
    zero = torch.zeros_like(X)
    if b is not None:
        idx = torch.div(torch.arange(X.numel(), device=X.device), step_b, rounding_mode='floor') % size_b
        if fault == 'bias_shift':
            idx = (idx + 1) % size_b
        B = b.double()[idx]
    else:
        B = zero
    XR = zero if xref is None else xref.double()
    YR = zero if yref is None else yref.double()
    DY = torch.ones_like(X) if dy is None else dy.double()
    yy = YR / gain if gain != 0 else zero
    la = SELU_L * SELU_A
    alts = []

    def near(v, thr, rel=1.0):
        return (v - thr).abs() <= rel * u * v.abs() + fl

    def branch(cond, nr, ra, ea, rb, eb):
        alts.append((torch.where(cond, rb, ra), nr))
        e = torch.where(cond, ea, eb)
        return torch.where(cond, ra, rb), torch.where(nr, torch.maximum(ea, eb), e)

    if grad == 0:
        v = X + B
        if fault == 'round16_xb':
            v = rn16(v)
        av = v.abs()
        if act == 'linear':
            r, e = v, u * av
        elif act == 'relu':
            r = v.clamp(min=0)
            e = u * r.abs()
        elif act == 'lrelu':
            r = torch.where(v > 0, v, alpha * v)
            e = 2 * u * r.abs() + fl
        elif act == 'tanh':
            t = torch.tanh(v)
            r, e = branch(av > 80, near(av, 80), torch.sign(v), zero + fl, t, u * (av + 8) * (1 + t.abs()) + fl)
        elif act == 'sigmoid':
            s = torch.sigmoid(v)
            r, e = branch(v < -80, near(v, -80), zero, zero + fl, s, u * (av + 6) * s + fl)
        elif act == 'elu':
            c, em = torch.exp(v.clamp(max=0)), torch.expm1(v.clamp(max=0))
            r = torch.where(v >= 0, v, em)
            e = torch.where(v >= 0, u * av, c * u * (av + 4) + u * em.abs() + fl)
        elif act == 'selu':
            c, em = torch.exp(v.clamp(max=0)), torch.expm1(v.clamp(max=0))
            r = torch.where(v >= 0, SELU_L * v, la * em)
            e = torch.where(v >= 0, 3 * u * r.abs(), la * (c * u * (av + 4) + u * em.abs()) + 4 * u * r.abs() + fl)
        elif act == 'softplus':
            c = torch.exp(v.clamp(max=700))
            sp = torch.log1p(c)
            r, e = branch(v > 80, near(v, 80), v, u * av, sp, c / (1 + c) * u * (av + 4) + u + 2 * u * sp + fl)
        else:  # swish
            w = v * torch.sigmoid(v)
            r, e = branch(v < -80, near(v, -80), zero, zero + fl, w, u * (av + 7) * w.abs() + fl)
        y = r * gain
        e = gain * e + u * y.abs() + fl
        alts = [(a * gain, m) for a, m in alts]
        if clamp >= 0:
            y = y.clamp(-clamp, clamp)
            alts = [(a.clamp(-clamp, clamp), m) for a, m in alts]
    else:
        xr = XR + B
        axr = xr.abs()
        ax = X.abs()
        if act == 'linear':
            r, e = (X, zero) if grad == 1 else (zero, zero)
        elif act == 'relu':
            r, e = (torch.where(yy > 0, X, zero), zero) if grad == 1 else (zero, zero)
        elif act == 'lrelu':
            if grad == 1:
                r = torch.where((X if fault == 'slope_from_x' else yy) > 0, X, alpha * X)
                e = u * r.abs() + fl
            else:
                r, e = zero, zero
        elif act == 'tanh':
            m = ax * (yy * yy + (1 - yy * yy).abs())
            if grad == 1:
                r, e = X * (1 - yy * yy), 4 * u * m
            else:
                r, e = X * (1 - yy * yy) * (-2 * yy), 12 * u * m * yy.abs()
        elif act == 'sigmoid':
            m = ax * yy.abs() * (yy.abs() + (1 - yy).abs())
            if grad == 1:
                r, e = X * yy * (1 - yy), 5 * u * m
            else:
                r, e = X * yy * (1 - yy) * (1 - 2 * yy), 8 * u * m * (2 * yy.abs() + (1 - 2 * yy).abs())
        elif act in ('elu', 'selu'):
            k = 1.0 if act == 'elu' else la
            neg = X * (yy + k)
            eneg = 5 * u * ax * (yy.abs() + k)
            if grad == 1:
                pos, epos = (X, zero) if act == 'elu' else (X * SELU_L, 2 * u * ax * SELU_L)
            else:
                pos, epos = zero, zero
            r, e = torch.where(yy >= 0, pos, neg), torch.where(yy >= 0, epos, eneg)
        elif act == 'softplus':
            c = torch.exp(-yy)
            if grad == 1:
                r = X * (1 - c)
                e = ax * (c * u * (yy.abs() + 5) + 2 * u * (1 - c).abs())
            else:
                r = X * c * (1 - c)
                e = u * (yy.abs() + 8) * ax * c * (c + (1 - c).abs())
        else:  # swish
            c = torch.exp(xr.clamp(max=700))
            d = c + 1
            lo_floor = fl * (1 + ax) * (1 + axr)
            if grad == 1:
                inner = X * c * (xr + d) / (d * d)
                ein = u * (4 * axr + 24) * ax * c * (axr + d) / (d * d) + lo_floor
                r, e = branch(xr > 40, near(xr, 40), X, zero, inner, ein)
            else:
                d3 = d * d * d
                inner = X * c * (xr * (2 - d) + 2 * d) / d3
                ein = u * (6 * axr + 40) * ax * c * (axr * (2 + d) + 2 * d) / d3 + lo_floor
                if dtype != torch.float64:      # (d * d) * d overflows fp32 above x + b ~ 29.6: the kernel returns +-0
                    big = 2.0 ** 128
                    r0, e0 = branch(d3 >= big, (d3 / big - 1).abs() <= u * (3 * axr + 20), zero, lo_floor, inner, ein)
                    inner, ein = r0, e0
                r, e = branch(xr > 40, near(xr, 40), zero, zero, inner, ein)
        g = gain * DY
        y = r * g
        e = g.abs() * e + 2 * u * y.abs() + fl
        alts = [(a * g, m) for a, m in alts]
        if clamp >= 0 and fault != 'no_clamp_gate':
            gate_alt = None
            if act == 'swish':     # the kernel recomputes yref from x + b in fp32
                ys = torch.where(xr < -80, zero, xr * torch.sigmoid(xr) * gain)
                es = u * (axr + 8) * ys.abs() + fl
                gate = ys.abs() < clamp
                gate_alt = (torch.where(gate, zero, y), (ys.abs() - clamp).abs() <= es)
            else:
                gate = (YR > -clamp) & (YR < clamp)
            y = torch.where(gate, y, zero)
            alts = [(torch.where(gate, a, zero), m) for a, m in alts]
            if gate_alt is not None:
                alts.append(gate_alt)
    margin = torch.zeros_like(X, dtype=torch.bool)
    for _, m in alts:
        margin |= m
    return dict(ref=y, tol=_out_tol(y, e, dtype), alts=alts, margin=margin)


def ba_launch_model(x, b, xref, yref, dy, grad, dim, act_idx, alpha, gain, clamp, fault=None):
    """The model of `bias_act._launch(x, b, xref, yref, dy, grad, dim, act_idx, alpha, gain, clamp)`."""
    fl = lambda t: None if t is None else _flat(t)     # noqa: E731
    step_b = x.stride(dim) if b is not None else 1
    return bias_act_model(_flat(x), b, fl(xref), fl(yref), fl(dy), x.dtype, grad, act_idx, alpha, gain, clamp,
                          0 if b is None else b.numel(), step_b, fault)


# ---------------------------------------------------------------------------------------------------------------------
# upfirdn2d model
# ---------------------------------------------------------------------------------------------------------------------
def upfirdn2d_model(x, f2d, y_hw, upx, upy, downx, downy, padx0, pady0, flip, gain, generic=False, fault=None):
    """One p3d_upfirdn2d launch: x [N,C,H,W] (any strides), f2d [fh,fw] fp32, output size y_hw (taken from y)."""
    X = x.double()
    _, _, H, W = X.shape
    oh, ow = y_hw
    fh, fw = f2d.shape
    F = f2d.double().to(X.device)
    if not flip:
        F = F.flip([0, 1])
    dev = X.device
    by = torch.arange(oh, device=dev) * downy - pady0
    bx = torch.arange(ow, device=dev) * downx - padx0 + (1 if fault == 'pad_shift' else 0)
    ref = torch.zeros(X.shape[0], X.shape[1], oh, ow, dtype=torch.float64, device=dev)
    S = torch.zeros_like(ref)
    for ty in range(fh):
        py = by + ty
        vy = (py >= 0) & (py % upy == 0) & (torch.div(py, upy, rounding_mode='floor') < H)
        iy = torch.where(vy, torch.div(py, upy, rounding_mode='floor'), torch.zeros_like(py))
        rows = X[:, :, iy, :] * vy[:, None].double()
        for tx in range(fw):
            if fault == 'drop_tap' and (ty, tx) == (fh // 2, fw // 2):
                continue
            px = bx + tx
            vx = (px >= 0) & (px % upx == 0) & (torch.div(px, upx, rounding_mode='floor') < W)
            ix = torch.where(vx, torch.div(px, upx, rounding_mode='floor'), torch.zeros_like(px))
            cols = rows[..., ix] * vx.double()
            ref += F[ty, tx] * cols
            S += F[ty, tx].abs() * cols.abs()
    g = f32(gain)
    ref, S = ref * g, S * abs(g)
    taps = fh * fw
    if x.dtype == torch.float64:
        e = (2 * taps + 1) * U64 * S
    else:
        e = ((2 * taps + 1) if (generic and x.dtype == torch.float32) else (taps + 1)) * U32 * S
    return dict(ref=ref, tol=_out_tol(ref, e, x.dtype) + _floor(x.dtype), alts=[], margin=None)


# ---------------------------------------------------------------------------------------------------------------------
# fma model
# ---------------------------------------------------------------------------------------------------------------------
def fma_model(a, b, c, fault=None):
    A, B, C = a.double(), b.double(), c.double()
    ab = A * B
    if fault == 'mul16_add':
        ab = rn16(ab)
    ref = ab + C
    mag = (A * B).abs() + C.abs()
    e = _u(a.dtype) * ref.abs() + 2.0 ** -53 * mag + _floor(a.dtype)
    if a.dtype == torch.float64:
        e = U64 * mag + _floor(a.dtype)
    return dict(ref=ref, tol=_out_tol(ref, e, a.dtype), alts=[], margin=None)


# ---------------------------------------------------------------------------------------------------------------------
# scoring
# ---------------------------------------------------------------------------------------------------------------------
def score(got, m):
    """(worst err / tol, elements over 1, elements, margin elements) of one launch's output against its model."""
    got = got.double().reshape(m['ref'].shape)
    ref = m['ref']
    err = (got - ref).abs()
    err = torch.where(torch.isinf(got) & (got == ref), torch.zeros_like(err), err)
    for alt, mask in m['alts']:
        err = torch.where(mask, torch.minimum(err, (got - alt).abs()), err)
    r = torch.nan_to_num(err / m['tol'], nan=math.inf)
    marg = 0 if m.get('margin') is None else int(m['margin'].sum())
    return (float(r.max()) if r.numel() else 0.0), int((r > 1).sum()), r.numel(), marg


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the models against the oracle and the wrappers' impl='ref' compositions (float64, ops.npz fixtures)
# ---------------------------------------------------------------------------------------------------------------------
def _fixture():
    from conftest import load_golden
    return load_golden('ops')


@pytest.mark.parametrize('act', ACTS)
def test_bias_act_model_reproduces_the_oracle(act):
    import p3d_oracle as O
    from pix2pix3d_b200.torch_utils.ops import bias_act as BA
    g = _fixture()
    x64, b64 = g['ba_x'].astype(np.float64), g['ba_b'].astype(np.float64)
    spec = BA.activation_funcs[act]
    for kw in (dict(alpha=spec.def_alpha, gain=spec.def_gain, clamp=-1.0), dict(alpha=0.3, gain=1.7, clamp=0.9)):
        kw = {k: f32(v) for k, v in kw.items()}
        okw = dict(kw, clamp=None if kw['clamp'] < 0 else kw['clamp'])
        x, b = torch.from_numpy(x64), torch.from_numpy(b64)
        st = x.stride(1)
        m = bias_act_model(_flat(x), b, None, None, None, torch.float64, 0, ACT_IDX[act], size_b=5, step_b=st, **kw)
        y_or = O.ops.bias_act(x64, b64, act=act, **okw)
        y_ref = BA._bias_act_ref(x, b, act=act, **okw).numpy()
        assert np.abs(m['ref'].numpy().reshape(x64.shape) - y_or).max() <= 1e-12 * max(1, np.abs(y_or).max()), act
        assert np.abs(m['ref'].numpy().reshape(x64.shape) - y_ref).max() <= 1e-12 * max(1, np.abs(y_ref).max()), act
        y = torch.from_numpy(y_or)
        gy = torch.from_numpy(g[f'ba_{act}_{"d" if kw["clamp"] < 0 else "c"}_gy'])
        xref = x if (REF.get(act, 'y') == 'x' or act in HAS_2ND) else None
        yref = y if 'y' in REF.get(act, 'y') else None
        m1 = bias_act_model(_flat(gy), b if xref is not None else None, None if xref is None else _flat(xref),
                            None if yref is None else _flat(yref), None, torch.float64, 1, ACT_IDX[act], size_b=5, step_b=st, **kw)
        g1 = O.ops.bias_act_grad(gy.numpy(), x64, b64, y_or, act=act, order=1, plugin_semantics=True, **okw)
        assert np.abs(m1['ref'].numpy().reshape(x64.shape) - g1).max() <= 1e-12 * max(1, np.abs(g1).max()), act
        if act in HAS_2ND:
            ggx = torch.from_numpy(g[f'ba_{act}_{"d" if kw["clamp"] < 0 else "c"}_ggx'])
            m2 = bias_act_model(_flat(ggx), b, _flat(x), None if yref is None else _flat(yref), _flat(gy), torch.float64, 2,
                                ACT_IDX[act], size_b=5, step_b=st, **kw)
            g2 = O.ops.bias_act_grad(ggx.numpy(), x64, b64, y_or, act=act, order=2, dy1=gy.numpy(), plugin_semantics=True, **okw)
            assert np.abs(m2['ref'].numpy().reshape(x64.shape) - g2).max() <= 1e-12 * max(1, np.abs(g2).max()), act


UP_CFGS = {   # test_gpu_ops.UP_CFGS with the wrapper's padding
    'post_tconv': dict(f='f4', up=1, down=1, padding=[1, 1, 1, 1], gain=4),
    'skip_up': dict(f='f4', up=2, down=1, padding=[2, 1, 2, 1], gain=4),
    'down2': dict(f='f4', up=1, down=2, padding=[1, 1, 1, 1], gain=1),
    'pre_sconv': dict(f='f4', up=1, down=1, padding=[2, 2, 2, 2], gain=1),
    'odd': dict(f='f35', up=[3, 2], down=[2, 1], padding=[2, 0, -1, 3], gain=0.7, flip_filter=True),
    'crop': dict(f='f4', up=1, down=1, padding=[-1, 2, 0, -2], gain=1),
    'identity': dict(f=None, up=1, down=1, padding=0, gain=1),
}


def _pair(v):
    return (v, v) if isinstance(v, int) else tuple(v)


@pytest.mark.parametrize('name', list(UP_CFGS))
def test_upfirdn2d_model_reproduces_the_oracle(name):
    import p3d_oracle as O
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d as UF
    g = _fixture()
    kw = dict(UP_CFGS[name])
    fk = kw.pop('f')
    f = None if fk is None else torch.from_numpy(g['up_' + fk])
    x = torch.from_numpy(g['up_x'].astype(np.float64))
    y_or = O.ops.upfirdn2d(x.numpy(), None if f is None else f.numpy(), **kw)
    y_ref = UF._upfirdn2d_ref(x, f, **kw).numpy()
    upx, upy = _pair(kw['up'])
    downx, downy = _pair(kw['down'])
    px0, px1, py0, py1 = UF._parse_padding(kw['padding'])
    f2d = torch.ones(1, 1) if f is None else f
    m = upfirdn2d_model(x, f2d, y_or.shape[2:], upx, upy, downx, downy, px0, py0, kw.get('flip_filter', False), kw['gain'])
    for want in (y_or, y_ref, g[f'up_{name}_y']):
        # the compositions scale the filter by gain in fp32 before filtering; the kernels scale the sum
        exact = math.frexp(kw['gain'])[0] == 0.5
        tol = (1e-12 if exact else 2 * U32) if want.dtype == np.float64 else 2e-6
        assert np.abs(m['ref'].numpy() - want).max() <= tol * max(1, np.abs(want).max()), name
    # the output size the wrapper computes is the model's
    oh = (x.shape[2] * upy + py0 + py1 - f2d.shape[0] + downy) // downy
    ow = (x.shape[3] * upx + px0 + px1 - f2d.shape[1] + downx) // downx
    assert (oh, ow) == tuple(y_or.shape[2:])


def test_separable_and_adjoint_models_reproduce_the_compositions():
    """The separable two-pass launches compose to the 8-tap reference, and the backward's launch (up / down swapped, filter
    mirrored, _Upfirdn2d.backward's padding) is the adjoint of the forward's: <A x, g> = <x, A^T g> in float64."""
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d as UF
    g = _fixture()
    x = torch.from_numpy(g['up_x'].astype(np.float64))
    f8 = torch.from_numpy(g['up_f8'])
    h = upfirdn2d_model(x, f8[None], (x.shape[2], 2 * x.shape[3]), 2, 1, 1, 1, 4, 0, False, 1.0)['ref']
    v = upfirdn2d_model(h, f8[:, None], (2 * x.shape[2], 2 * x.shape[3]), 1, 2, 1, 1, 0, 4, False, 4.0)['ref']
    assert np.abs(v.numpy() - g['up_sep8_up2_y']).max() < 2e-6 * np.abs(g['up_sep8_up2_y']).max()
    gen = torch.Generator().manual_seed(0)
    f4 = torch.from_numpy(g['up_f4'])
    for (up, down), pads, flip in (((1, 1), (1, 2, 2, 1), False), ((2, 1), (2, 1, 2, 1), True), ((1, 2), (1, 1, 0, 2), False),
                                   ((1, 1), (-1, 2, 0, -2), True)):
        xs = torch.randn(2, 3, 9, 11, dtype=torch.float64, generator=gen)
        px0, px1, py0, py1 = pads
        oh = (9 * up + py0 + py1 - 4 + down) // down
        ow = (11 * up + px0 + px1 - 4 + down) // down
        y = upfirdn2d_model(xs, f4, (oh, ow), up, up, down, down, px0, py0, flip, 2.0)['ref']
        gy = torch.randn(y.shape, dtype=torch.float64, generator=gen)
        bp = adjoint_pads(f4.shape, pads, (up, up), (down, down), xs.shape, y.shape)
        gx = upfirdn2d_model(gy, f4, (9, 11), down, down, up, up, bp[0], bp[2], not flip, 2.0)['ref']
        assert gx.shape == xs.shape
        lhs, rhs = float((y * gy).sum()), float((xs * gx).sum())
        assert abs(lhs - rhs) <= 1e-12 * (y.abs() * gy.abs()).sum(), (up, down, pads)


def adjoint_pads(fshape, pads, up, down, xshape, yshape):
    """_Upfirdn2d.backward's padding of the adjoint launch."""
    fh, fw = fshape
    px0, _, py0, _ = pads
    (upx, upy), (downx, downy) = up, down
    ih, iw = xshape[2:]
    oh, ow = yshape[2:]
    return (fw - px0 - 1, iw * upx - ow * downx + px0 - upx + 1, fh - py0 - 1, ih * upy - oh * downy + py0 - upy + 1)


def test_fma_model_is_addcmul():
    gen = torch.Generator().manual_seed(3)
    a, b, c = (torch.randn(s, dtype=torch.float64, generator=gen) for s in ((2, 4, 6, 8), (2, 4, 1, 1), (2, 1, 6, 8)))
    m = fma_model(a, b, c)
    assert torch.allclose(m['ref'], torch.addcmul(c, a, b), rtol=1e-15, atol=1e-15)


def test_grid_mirrors_reach_the_sweep_edges():
    """For 132 SMs (H100 SXM) and another count, the sweep's shapes land on every grid edge they are named for."""
    for sms in (132, 114):
        wave = 8 * sms
        for V in (8, 4, 2):
            s = ba_sizes(V, sms)
            assert s['lt_V'] < V and s['mod_0'] % V == 0 and s['mod_1'] % V == 1 and s['mod_V-1'] % V == V - 1
            assert ba_grid(s['wave-1'], V, sms) == wave - 1 and ba_grid(s['wave'], V, sms) == wave
            assert _ceil(_ceil(s['wave+1'], 4 * V), 256) == wave + 1 and ba_grid(s['wave+1'], V, sms) == 2 * wave
            assert ba_grid(s['cap'], V, sms) == 4 * wave and _ceil(s['cap'] // V, 4 * wave * 256) == 4
            assert ba_grid(s['cap'] + 1, V, sms) == 4 * wave            # one element past the cap: a 5th vector for some threads
            assert ba_grid(s['2x_cap'], V, sms) == 4 * wave and s['2x_cap'] // V >= 2 * 4 * 4 * wave * 256
        # vector / scalar selection
        assert ba_vec_path([256, 0, 512, 0, 768], True, 64, 8) == (True, True)
        assert ba_vec_path([258, 0, 0, 0, 512], True, 64, 8) == (False, True)
        assert ba_vec_path([256, 0, 0, 0, 512], True, 63, 8) == (True, False)
        # FIR: the 8-wave cap +-1 and past it
        cap = fir_cap(sms)
        for d in (-1, 0, 1):
            assert fir_grid(cap + d, sms) == (8 * wave if d >= 0 else 8 * wave)
        assert fir_grid(cap - 256 * wave, sms) == 7 * wave and fir_grid(wave * 256 + 1, sms) == 2 * wave
        for route, ys in FIR_PAST_CAP:
            assert fir_items(route, ys) > 2 * cap, (route, ys)
        # fma: the 16-CTA cap +-1
        fc = fma_cap(sms)
        assert fma_grid(fc - 256, sms) == 16 * sms - 1 and fma_grid(fc, sms) == 16 * sms and fma_grid(fc + 1, sms) == 16 * sms
    # the routes the sweep means to reach
    c = (1, 1, 1, 1)
    assert fir_route(torch.float16, (2, 3, 8, 8), (192, 64, 8, 1), (2, 3, 8, 8), (192, 64, 8, 1), 4, 4, 2, 2, 1, 1) == 'strip u2d1'
    assert fir_route(torch.float64, (2, 3, 8, 8), (192, 64, 8, 1), (2, 3, 8, 8), (192, 64, 8, 1), 4, 4, 1, 1, 1, 1) == 'generic'
    assert fir_route(torch.float32, (2, 3, 8, 8), (192, 1, 24, 3), (2, 3, 8, 8), (192, 64, 8, 1), 4, 4, 1, 1, 1, 1) == 'generic'
    assert fir_route(torch.float32, (2, 3, 8, 8), (192, 64, 8, 1), (2, 3, 8, 8), (192, 64, 8, 1), 1, 1, 1, 1, 1, 1) == 'generic'
    assert fma_vec_path(torch.float16, (2, 4, 6, 8), [0, 16, 32], [(192, 48, 8, 1), (4, 1, 0, 0), (0, 0, 0, 0)], 64)
    assert not fma_vec_path(torch.float16, (2, 4, 6, 8), [2, 16, 32], [(192, 48, 8, 1), (4, 1, 0, 0), c], 64)
    assert not fma_vec_path(torch.float16, (2, 4, 6, 8), [0, 16, 32], [(216, 54, 9, 1), (4, 1, 0, 0), c], 64)
    assert not fma_vec_path(torch.float16, (2, 4, 6, 12), [0, 16, 32], [(288, 72, 12, 1), (4, 1, 0, 0), c], 64)


# D's first fp16 FIRs at 512^2, batch 4, 64 channels: conv1's pre-filter (pads 2) and the skip's down=2 filter; an up=2 FIR
# 256 -> 512 (output sizes)
FIR_PAST_CAP = [('strip u1d1', (4, 64, 513, 513)), ('strip u1d2', (4, 64, 256, 256)), ('strip u2d1', (4, 64, 512, 512))]


def test_bounds_reject_planted_faults_cpu():
    """Each planted model fault moves values well outside the bound of a clean model (here against the clean model's own
    value as a stand-in for the kernel; the GPU variant below uses the kernels' outputs)."""
    gen = torch.Generator().manual_seed(5)
    for fault, ratio in planted_fault_ratios(lambda *a, **k: None, gen, 'cpu').items():
        assert ratio > 2, (fault, ratio)


def _fault_cases(gen, dev):
    """(name, model(fault) -> dict, output) for each planted fault; output None = the clean model's own value."""
    cases = []
    x = (torch.randn(4, 6, 16, 16, generator=gen) * 3).to(dev)
    b = torch.randn(6, generator=gen).to(dev)
    for dt, fault in ((torch.float32, 'bias_shift'), (torch.float16, 'round16_xb')):
        xd, bd = x.to(dt), b.to(dt)
        cases.append((fault, dt, 'ba0', (xd, bd, None, None, None, 0, 1, ACT_IDX['lrelu'], 0.2, math.sqrt(2), -1.0)))
    y16 = x.half()
    xs = torch.where(x.abs() > 1.5, x.sign() * 300, x).half().to(dev)
    gy = torch.randn(4, 6, 16, 16, generator=gen).half().to(dev)
    cases.append(('slope_from_x', torch.float16, 'ba1', (gy, None, None, y16, None, 1, 1, ACT_IDX['lrelu'], 0.2, math.sqrt(2), -1.0)))
    cases.append(('no_clamp_gate', torch.float16, 'ba1', (gy, None, None, xs, None, 1, 1, ACT_IDX['lrelu'], 0.2, math.sqrt(2), CLAMP_D)))
    f = torch.tensor([1., 3., 3., 1.]).outer(torch.tensor([1., 3., 3., 1.])) / 64
    xf = torch.randn(2, 3, 17, 19, generator=gen).to(dev)
    for fault in ('drop_tap', 'pad_shift'):
        cases.append((fault, torch.float32, 'fir', (xf, f.to(dev), (18, 20), 1, 1, 1, 1, 2, 2, False, 4.0)))
    a, bb, c = (torch.randn(64, 1024, generator=gen).half().to(dev) * 4 for _ in range(3))
    cases.append(('mul16_add', torch.float16, 'fma', (a, bb, c)))
    return cases


def planted_fault_ratios(run, gen, dev):
    """{fault: worst err / tol of the launch's output against the faulty model}. `run(kind, args)` returns the kernel's
    output for the clean arguments or None, in which case the clean model's value stands in (CPU)."""
    out = {}
    for fault, dt, kind, args in _fault_cases(gen, dev):
        if kind.startswith('ba'):
            got = run(kind, args)
            clean = ba_launch_model(*args)
            bad = ba_launch_model(*args, fault=fault)
            got = clean['ref'] if got is None else _flat(got).double()
            if fault in ('slope_from_x', 'no_clamp_gate'):
                assert score(got, clean)[0] <= 1
        elif kind == 'fir':
            x, f, hw, *rest = args
            got = run(kind, args)
            clean = upfirdn2d_model(x, f, hw, *rest)
            bad = upfirdn2d_model(x, f, hw, *rest, fault=fault)
            got = clean['ref'] if got is None else got
        else:
            got = run(kind, args)
            clean = fma_model(*args)
            bad = fma_model(*args, fault=fault)
            got = clean['ref'] if got is None else got
        if dt == torch.float16 and got is clean['ref']:
            got = rn16(got)
        out[fault] = score(got, bad)[0]
    return out


# ---------------------------------------------------------------------------------------------------------------------
# checking wrappers: every launch of the three ops against its model, while its inputs are alive
# ---------------------------------------------------------------------------------------------------------------------
_DT = {torch.float16: 'fp16', torch.float32: 'fp32', torch.float64: 'fp64'}


def _acc(stats, key, res):
    st = stats.setdefault(key, dict(launches=0, elements=0, bad=0, margin=0, worst=0.0))
    st['launches'] += 1
    st['worst'] = max(st['worst'], res[0])
    st['bad'] += res[1]
    st['elements'] += res[2]
    st['margin'] += res[3]


def install_stream_checks(stats):
    """Wraps bias_act._launch, upfirdn2d._launch and fma._addcmul so that each launch is scored against its model into
    `stats` {'<op> <dtype> <mode> <path>': {launches, elements, bad, margin, worst}}. Returns a function that unwraps."""
    from pix2pix3d_b200.torch_utils.ops import bias_act as BA
    from pix2pix3d_b200.torch_utils.ops import fma as FM
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d as UF
    real = (BA._launch, UF._launch, FM._addcmul)

    def ba_launch(x, b, xref, yref, dy, grad, dim, act_idx, alpha, gain, clamp):
        y = real[0](x, b, xref, yref, dy, grad, dim, act_idx, alpha, gain, clamp)
        if x.numel():
            m = ba_launch_model(x, b, xref, yref, dy, grad, dim, act_idx, alpha, gain, clamp)
            V = _vec(x.dtype)
            vec, _ = ba_vec_path([t.data_ptr() for t in (x, xref, yref, dy, y) if t is not None], b is not None,
                                 x.stride(dim) if b is not None else 1, V)
            _acc(stats, f'bias_act {_DT[x.dtype]} grad{grad} {"vec" if vec else "scalar"}', score(_flat(y), m))
        return y

    def uf_launch(x, f2d, upx, upy, downx, downy, px0, px1, py0, py1, flip, gain):
        y = real[1](x, f2d, upx, upy, downx, downy, px0, px1, py0, py1, flip, gain)
        fh, fw = f2d.shape
        route = fir_route(x.dtype, x.shape, x.stride(), y.shape, y.stride(), fw, fh, upx, upy, downx, downy)
        m = upfirdn2d_model(x, f2d, y.shape[2:], upx, upy, downx, downy, px0, py0, flip, gain, generic=route == 'generic')
        _acc(stats, f'upfirdn2d {_DT[x.dtype]} {route}', score(y, m))
        return y

    def addcmul(a, b, c):
        out = real[2](a, b, c)
        if out.is_cuda and a.dtype == b.dtype == c.dtype and out.numel():
            form = 'bwd' if (c.ndim == 0 and not bool(c.any())) else 'fwd'
            _acc(stats, f'fma {_DT[a.dtype]} {form}', score(out, fma_model(*torch.broadcast_tensors(a, b, c))))
        return out

    BA._launch, UF._launch, FM._addcmul = ba_launch, uf_launch, addcmul

    def restore():
        BA._launch, UF._launch, FM._addcmul = real
    return restore


# ---------------------------------------------------------------------------------------------------------------------
# GPU sweeps
# ---------------------------------------------------------------------------------------------------------------------
REPORT = {}


@pytest.fixture(scope='module', autouse=True)
def _report():
    yield
    if REPORT:
        print('\nworst err / tol per case (elements over 1 must be 0; margin = elements on an fp32-decided branch edge):')
        for k in sorted(REPORT):
            print(f'  {k:64s} {REPORT[k]}')


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _check(case, got, m, grid=''):
    torch.cuda.synchronize()
    w, bad, n, marg = score(got, m)
    REPORT[case] = f'worst {w:.3g}  elements {n}  margin {marg}' + (f'  grid {grid}' if grid else '')
    assert bad == 0, f'{case}: {bad} of {n} elements over their bound (worst err/tol {w:.3g})'
    return w


def _alloc(shape, dtype, misalign=False, channels_last=False, gen=None, scale=1.0):
    """A dense tensor of `shape` (channels_last if asked), its base 16-byte aligned or one element past it."""
    n = int(np.prod(shape))
    buf = torch.empty(n + 8, dtype=torch.float64 if dtype == torch.float64 else torch.float32, device='cuda')
    buf.normal_(generator=gen).mul_(scale)
    buf = buf.to(dtype)
    off = 1 if misalign else 0
    if channels_last:
        nn, c, h, w = shape
        return buf[off:off + n].view(nn, h, w, c).permute(0, 3, 1, 2)
    return buf[off:off + n].view(shape)


def _edge_values(dtype, clamp):
    """Values on the activations' branch edges: the saturation thresholds and beyond, and +-clamp with its neighbours."""
    vals = [0.0, 40.0, 40.5, 80.0, 85.0, 100.0, 200.0, 29.5, 30.0]
    vals += [-v for v in vals]
    if clamp >= 0:
        if dtype == torch.float16:
            c16 = float(rn16(torch.tensor(clamp, dtype=torch.float64)))
            step = float(_ulp16(torch.tensor(c16, dtype=torch.float64)))
            near = [c16 - step, c16, c16 + step]
        else:
            t = np.float32 if dtype == torch.float32 else np.float64
            c = t(clamp)
            near = [float(np.nextafter(c, t(0))), float(c), float(np.nextafter(c, t(np.inf)))]
        vals += near + [-v for v in near]
    return torch.tensor(vals, dtype=torch.float64, device='cuda').to(dtype)


def _plant(t, vals, stride):
    f = _flat(t)
    pos = torch.arange(0, f.numel(), stride, device='cuda')
    f[pos] = vals[torch.arange(pos.numel(), device='cuda') % vals.numel()]


def ba_case(case, dtype, grad, act, shape, dim=1, clamp=-1.0, bias=True, channels_last=False, misalign=(), edges=True, seed=0,
            big=False):
    """Builds operands as autograd would hand them to bias_act._launch for `grad`, runs the launch and checks it."""
    from pix2pix3d_b200.torch_utils.ops import bias_act as BA
    gen = torch.Generator(device='cuda').manual_seed(seed)
    spec = BA.activation_funcs[act]
    alpha, gain = float(spec.def_alpha), float(spec.def_gain)
    C = shape[dim]
    b = _alloc((C,), dtype, gen=gen) if bias else None
    x = _alloc(shape, dtype, 'x' in misalign and grad == 0, channels_last, gen, 3.0)
    if edges:
        _plant(x, _edge_values(dtype, clamp), 59)
        if b is not None:            # x + b == 0
            xf = _flat(x)
            step_b = x.stride(dim)
            pos = torch.arange(7, xf.numel(), 53, device='cuda')
            xf[pos] = -b[torch.div(pos, step_b, rounding_mode='floor') % C]
    y = BA._launch(x, b, None, None, None, 0, dim, ACT_IDX[act], alpha, gain, clamp)
    if grad == 0:
        V = _vec(dtype)
        grid = ba_grid(x.numel(), V, _sms())
        info = f'{grid} CTAs, {grid / (8 * _sms()):.3g} waves, {_ceil(x.numel() // V, grid * 256)} vectors/thread'
        return _check(case, _flat(y), ba_launch_model(x, b, None, None, None, 0, dim, ACT_IDX[act], alpha, gain, clamp),
                      info if big or not edges else '')
    if edges and 'y' in spec.ref:
        yv = _edge_values(dtype, clamp)
        if act in ('softplus', 'sigmoid', 'tanh'):
            yv = yv.abs().clamp(max=1.0 if act != 'softplus' else 80.0) * (1 if act == 'softplus' else gain)
        _plant(y, yv, 61)
    need_x = 'x' in spec.ref or spec.has_2nd_grad
    xref, bref = (x, b) if need_x else (None, None)
    yref = y if 'y' in spec.ref else None

    def re(t, name):       # the same values at a misaligned address
        if t is None or name not in misalign:
            return t
        u = _alloc(t.shape, dtype, True, channels_last)
        u.copy_(t)
        return u
    xref, yref = re(xref, 'xref'), re(yref, 'yref')
    g1 = _alloc(shape, dtype, 'x' in misalign, channels_last, gen, 1.0)
    if grad == 1:
        dx = BA._launch(g1, bref, xref, yref, None, 1, dim, ACT_IDX[act], alpha, gain, clamp)
        return _check(case, _flat(dx), ba_launch_model(g1, bref, xref, yref, None, 1, dim, ACT_IDX[act], alpha, gain, clamp))
    dy = _alloc(shape, dtype, 'dy' in misalign, channels_last, gen, 1.0)
    d_x = BA._launch(g1, b, xref, yref, dy, 2, dim, ACT_IDX[act], alpha, gain, clamp)
    return _check(case, _flat(d_x), ba_launch_model(g1, b, xref, yref, dy, 2, dim, ACT_IDX[act], alpha, gain, clamp))


def _clamp_for(act):
    return 0.75 if act in ('tanh', 'sigmoid') else CLAMP_D


@gpu
@pytest.mark.parametrize('grad', [0, 1, 2])
@pytest.mark.parametrize('dtype', [torch.float16, torch.float32, torch.float64])
def test_bias_act_sweep(dtype, grad):
    from pix2pix3d_b200.torch_utils.ops import bias_act as BA
    dn = _DT[dtype]
    acts = [a for a in ACTS if grad < 2 or a in HAS_2ND]
    for act in acts:
        for clamp in (-1.0, _clamp_for(act)):
            ba_case(f'bias_act {dn} g{grad} {act} clamp={clamp:g}', dtype, grad, act, (2, 6, 9, 13), clamp=clamp, seed=ACT_IDX[act])
    a1 = 'lrelu' if grad < 2 else 'tanh'
    c1 = _clamp_for(a1)
    lay = {'nchw hw%V==0': dict(shape=(2, 6, 8, 8)), 'channels_last': dict(shape=(2, 6, 9, 13), channels_last=True),
           'dim=3': dict(shape=(2, 3, 5, 6), dim=3), '2d [B,C]': dict(shape=(5, 24))}
    for name, kw in lay.items():
        ba_case(f'bias_act {dn} g{grad} {a1} {name}', dtype, grad, a1, clamp=c1, **kw)
    ops = {0: ['x'], 1: ['x', 'xref', 'yref'], 2: ['x', 'xref', 'yref', 'dy']}[grad]
    for a in ((a1, 'swish') if grad else (a1,)):
        spec = BA.activation_funcs[a]
        passed = {'x', 'dy', 'xref' if ('x' in spec.ref or spec.has_2nd_grad) else '', 'yref' if 'y' in spec.ref else ''}
        for op in (o for o in ops if o in passed):
            ba_case(f'bias_act {dn} g{grad} {a} misaligned {op}', dtype, grad, a, (2, 6, 9, 13), clamp=_clamp_for(a), misalign=(op,))
    V = _vec(dtype)
    for name, n in ba_sizes(V, _sms()).items():
        ba_case(f'bias_act {dn} g{grad} {a1} size {name} ({n})', dtype, grad, a1, (n,), dim=0, clamp=c1, edges=n > 1000,
                big=True, bias=n < 1_000_000 or grad == 0)


@gpu
@pytest.mark.parametrize('dtype', [torch.float16, torch.float32])
def test_upfirdn2d_strip_sweep(dtype):
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d as UF
    sms = _sms()
    gen = torch.Generator(device='cuda').manual_seed(1)
    f = UF.setup_filter([1, 3, 3, 1]).cuda()
    fa = (torch.rand(4, 4, generator=gen, device='cuda') - 0.3)         # an asymmetric filter: mirroring matters
    pads = {(1, 1): [(1, 2, 2, 1), (-1, 2, 0, -2)], (2, 1): [(2, 1, 2, 1), (2, 2, 2, 1), (-1, 2, 1, -1)],
            (1, 2): [(1, 1, 1, 1), (-1, 3, 0, 1)]}
    for (up, down), plist in pads.items():
        inst = f'strip u{up}d{down}'
        res = set()
        for pd in plist:
            for flip in (False, True):
                worst = 0.0
                for ih in (1, 3, 7):
                    for iw in range(1, 10):
                        px0, px1, py0, py1 = pd
                        oh = (ih * up + py0 + py1 - 4 + down) // down
                        ow = (iw * up + px0 + px1 - 4 + down) // down
                        if oh < 1 or ow < 1:
                            continue
                        x = _alloc((2, 3, ih, iw), dtype, gen=gen)
                        y = UF._launch(x, fa, up, up, down, down, px0, px1, py0, py1, flip, 2.0)
                        # a 1x1 input has stride(1) == 1, so the wrapper writes a channels_last output: the generic kernel
                        route = fir_route(dtype, x.shape, x.stride(), y.shape, y.stride(), 4, 4, up, up, down, down)
                        assert route == ('generic' if ih == iw == 1 and (oh, ow) != (1, 1) else inst), (ih, iw, route)
                        torch.cuda.synchronize()
                        w, bad, n, _ = score(y, upfirdn2d_model(x, fa, (oh, ow), up, up, down, down, px0, py0, flip, 2.0))
                        assert bad == 0, (inst, pd, flip, ih, iw, w)
                        worst = max(worst, w)
                        if route == inst:
                            res.add(ow % STRIP_TX[(up, down)])
                REPORT[f'upfirdn2d {_DT[dtype]} {inst} pads {pd} flip={flip} small shapes'] = f'worst {worst:.3g}'
        assert res == set(range(STRIP_TX[(up, down)])), res             # every residue of outW % TX
        # the 8-wave cap -1 / at / +1: one output per plane
        cap = fir_cap(sms)
        p1 = {(1, 1): (2, 1, 2, 1), (2, 1): (1, 1, 1, 1), (1, 2): (2, 1, 2, 1)}[(up, down)]
        for d in (-1, 0, 1):
            x = _alloc((1, cap + d, 1, 1), dtype, gen=gen)
            y = UF._launch(x, f, up, up, down, down, *p1, False, 4.0)
            assert tuple(y.shape[2:]) == (1, 1)
            assert fir_route(dtype, x.shape, x.stride(), y.shape, y.stride(), 4, 4, up, up, down, down) == inst
            _check(f'upfirdn2d {_DT[dtype]} {inst} items cap{d:+d}', y,
                   upfirdn2d_model(x, f, (1, 1), up, up, down, down, p1[0], p1[2], False, 4.0),
                   f'{fir_grid(cap + d, sms)} CTAs, {_ceil(cap + d, fir_grid(cap + d, sms) * 256)} items/thread')
    # past the cap, at training sizes
    for (inst, ys), (xs, pd) in zip(FIR_PAST_CAP, (((4, 64, 512, 512), (2, 2, 2, 2)), ((4, 64, 512, 512), (1, 1, 1, 1)),
                                                   ((4, 64, 256, 256), (2, 1, 2, 1)))):
        up, down = int(inst[7]), int(inst[9])
        x = _alloc(xs, dtype, gen=gen, scale=2.0)
        y = UF._launch(x, f, up, up, down, down, *pd, False, float(up * up))
        assert tuple(y.shape) == ys
        items = fir_items(inst, ys)
        g = fir_grid(items, sms)
        _check(f'upfirdn2d {_DT[dtype]} {inst} training size {ys}', y,
               upfirdn2d_model(x, f, ys[2:], up, up, down, down, pd[0], pd[2], False, float(up * up)),
               f'{g} CTAs, {_ceil(items, g * 256)} strips/thread')
        del x, y


@gpu
def test_upfirdn2d_generic_and_adjoint():
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d as UF
    gen = torch.Generator(device='cuda').manual_seed(2)
    f = UF.setup_filter([1, 3, 3, 1]).cuda()
    f35 = torch.rand(3, 5, generator=gen, device='cuda')
    cases = [('fp64 up2', torch.float64, (2, 5, 33, 47), f, (2, 2), (1, 1), (2, 1, 2, 1), False, False),
             ('fp64 down2 flip', torch.float64, (2, 5, 33, 47), f, (1, 1), (2, 2), (1, 1, 1, 1), True, False),
             ('fp32 channels_last', torch.float32, (2, 8, 33, 47), f, (1, 1), (1, 1), (2, 2, 2, 2), False, True),
             ('fp16 channels_last up2', torch.float16, (2, 8, 33, 47), f, (2, 2), (1, 1), (2, 1, 2, 1), False, True),
             ('fp32 up (3,2) down (2,1)', torch.float32, (2, 3, 19, 23), f35, (3, 2), (2, 1), (2, 0, -1, 3), True, False),
             ('fp16 up (3,2) down (2,1)', torch.float16, (2, 3, 19, 23), f35, (3, 2), (2, 1), (2, 0, -1, 3), False, False),
             ('fp32 1x1 pad-only', torch.float32, (4, 16, 64, 64), torch.ones(1, 1, device='cuda'), (1, 1), (1, 1), (1, 1, 1, 1), False,
              False),
             ('fp16 1x1 pad-only', torch.float16, (4, 16, 64, 64), torch.ones(1, 1, device='cuda'), (1, 1), (1, 1), (1, 1, 1, 1), False,
              False)]
    for name, dt, shape, ff, up, down, pd, flip, cl in cases:
        x = _alloc(shape, dt, channels_last=cl, gen=gen)
        y = UF._launch(x, ff, up[0], up[1], down[0], down[1], *pd, flip, 1.5)
        assert fir_route(dt, x.shape, x.stride(), y.shape, y.stride(), ff.shape[1], ff.shape[0], *up, *down) == 'generic'
        _check(f'upfirdn2d generic {name}', y,
               upfirdn2d_model(x, ff, y.shape[2:], up[0], up[1], down[0], down[1], pd[0], pd[2], flip, 1.5, generic=True))
    # the separable 8-tap path (two launches) and the autograd adjoint of every strip configuration, each launch checked
    stats = {}
    restore = install_stream_checks(stats)
    try:
        f8 = UF.setup_filter([1, 3, 3, 1, 1, 3, 3, 1]).cuda()
        for dt in (torch.float16, torch.float32):
            x = _alloc((2, 6, 32, 32), dt, gen=gen)
            UF.upsample2d(x, f8)
            for (up, down), pd in (((1, 1), [1, 2, 2, 1]), ((2, 1), [2, 1, 2, 1]), ((1, 2), [1, 1, 1, 1])):
                xg = _alloc((2, 6, 33, 35), dt, gen=gen).clone().requires_grad_(True)
                y = UF.upfirdn2d(xg, f, up=up, down=down, padding=pd, gain=up * up)
                y.backward(torch.randn_like(y))
    finally:
        restore()
    torch.cuda.synchronize()
    for k, v in stats.items():
        REPORT[f'{k} (separable / autograd)'] = v
        assert v['bad'] == 0, (k, v)
    for k in ('strip u1d1', 'strip u2d1', 'strip u1d2', 'generic'):
        assert any(k in s for s in stats), k
    # adjointness in float64 through _Upfirdn2d.backward's padding: <A x, g> = <x, A^T g>
    for (up, down), pd, flip in (((1, 1), [1, 2, 2, 1], False), ((2, 1), [2, 1, 2, 1], True), ((1, 2), [1, 1, 0, 2], False)):
        x = torch.randn(2, 3, 17, 19, dtype=torch.float64, device='cuda', generator=gen).requires_grad_(True)
        y = UF.upfirdn2d(x, f, up=up, down=down, padding=pd, flip_filter=flip, gain=2)
        g = torch.randn_like(y)
        gx, = torch.autograd.grad(y, x, g)
        lhs, rhs = float((y * g).sum()), float((x * gx).sum())
        assert abs(lhs - rhs) <= 1e-12 * float((y.abs() * g.abs()).sum() + (x.abs() * gx.abs()).sum()), (up, down)


def fma_case(case, dtype, shapes, misalign=None, pad_outer=None, gen=None, grid=False):
    from pix2pix3d_b200.torch_utils.ops import fma as FM
    ops = []
    for i, s in enumerate(shapes):
        if s == ():
            ops.append(torch.zeros((), dtype=dtype, device='cuda'))
            continue
        if pad_outer == i:         # a row stride one element longer than the row
            big = _alloc(tuple(s[:-1]) + (s[-1] + 1,), dtype, gen=gen)
            ops.append(big[..., :s[-1]])
            continue
        ops.append(_alloc(s, dtype, misalign == i, gen=gen))
    a, b, c = ops
    out = FM._addcmul(a, b, c)
    shape = out.shape
    pad = (1,) * (4 - len(shape))
    strides = [(0,) * len(pad) + tuple(0 if shape[j] == 1 else t.expand(shape).stride(j) for j in range(len(shape))) for t in ops]
    vec = fma_vec_path(dtype, pad + tuple(shape), [t.data_ptr() for t in ops], strides, out.data_ptr())
    n = out.numel() // (_vec(dtype) if vec else 1)
    info = f'{"vec" if vec else "scalar"} path' + (f', {fma_grid(n, _sms())} CTAs' if grid else '')
    _check(f'fma {_DT[dtype]} {case}', out, fma_model(*torch.broadcast_tensors(a, b, c)), info)
    return vec


@gpu
@pytest.mark.parametrize('dtype', [torch.float16, torch.float32, torch.float64])
def test_fma_sweep(dtype):
    gen = torch.Generator(device='cuda').manual_seed(3)
    V = _vec(dtype)
    W = 2 * V
    assert fma_case('dense', dtype, [(2, 4, 6, W)] * 3, gen=gen)
    assert fma_case('modconv x*dcoef+noise', dtype, [(2, 4, 6, W), (2, 4, 1, 1), (2, 1, 6, W)], gen=gen)
    assert fma_case('a broadcast along W', dtype, [(2, 4, 6, 1), (2, 4, 6, W), (2, 4, 6, W)], gen=gen)
    assert fma_case('broadcast operand misaligned', dtype, [(2, 4, 6, W), (2, 4, 1, 1), (2, 1, 6, W)], misalign=1, gen=gen)
    assert not fma_case('dense a misaligned', dtype, [(2, 4, 6, W), (2, 4, 1, 1), (2, 1, 6, W)], misalign=0, gen=gen)
    assert not fma_case('dense c misaligned', dtype, [(2, 4, 6, W), (2, 4, 1, 1), (2, 1, 6, W)], misalign=2, gen=gen)
    assert not fma_case('outer stride not 16B', dtype, [(2, 4, 6, W), (2, 4, 1, 1), (2, 1, 6, W)], pad_outer=0, gen=gen)
    assert not fma_case('W % vec != 0', dtype, [(2, 4, 6, W + 1), (2, 4, 1, 1), (2, 1, 6, W + 1)], gen=gen)
    fma_case('backward form (c 0-dim zero)', dtype, [(2, 4, 6, W), (2, 4, 6, W), ()], gen=gen)
    fma_case('backward form, odd W', dtype, [(2, 4, 6, 9), (2, 4, 1, 1), ()], gen=gen)
    fma_case('lower rank', dtype, [(5, 12), (12,), (5, 1)], gen=gen)
    cap = fma_cap(_sms())
    for name, g in (('cap-256', cap - 256), ('cap', cap), ('cap+1', cap + 1), ('4x cap', 4 * cap + 3)):
        assert fma_case(f'vec groups {name}', dtype, [(1, 1, g, V), (1, 1, g, 1), (1, 1, g, V)], gen=gen, grid=True)
        assert not fma_case(f'scalar elements {name}', dtype, [(1, 1, g, 1), (1, 1, 1, 1), (1, 1, g, 1)], gen=gen, grid=True)


@gpu
def test_planted_faults_are_rejected():
    """Each fault planted in a model (never in a kernel) puts the kernels' own outputs more than 2x outside the bound,
    while the clean models hold them within it."""
    from pix2pix3d_b200.torch_utils.ops import bias_act as BA
    from pix2pix3d_b200.torch_utils.ops import fma as FM
    from pix2pix3d_b200.torch_utils.ops import upfirdn2d as UF

    def run(kind, args):
        if kind.startswith('ba'):
            got = BA._launch(*args)
            m = ba_launch_model(*args)
        elif kind == 'fir':
            x, f, hw, *rest = args
            upx, upy, downx, downy, px0, py0, flip, gain = rest      # up = down = 1 here: px1 from the output width
            got = UF._launch(x, f, upx, upy, downx, downy, px0, hw[1] + 3 - x.shape[3] - px0, py0, hw[0] + 3 - x.shape[2] - py0,
                             flip, gain)
            assert tuple(got.shape[2:]) == hw
            m = upfirdn2d_model(x, f, hw, *rest)
        else:
            got = FM._addcmul(*args)
            m = fma_model(*args)
        torch.cuda.synchronize()
        assert score(got if kind in ('fir', 'fma') else _flat(got), m)[0] <= 1, kind
        return got
    gen = torch.Generator().manual_seed(5)
    ratios = planted_fault_ratios(run, gen, 'cuda')
    for k, v in ratios.items():
        REPORT[f'planted fault {k}'] = f'worst err/tol {v:.3g}'
    for k, v in ratios.items():
        assert v > 2, (k, v)


def _report_stats(title, stats):
    print(f'\n{title}:')
    for k in sorted(stats):
        v = stats[k]
        print(f"  {k:36s} {v['launches']:>5d} launches {v['elements']:>12d} elements  worst err/tol {v['worst']:.3g}  "
              f"margin {v['margin']}  over {v['bad']}")


@gpu
def test_discriminator_fullsize_pass():
    """Config 4's D and D_semantic (512^2, batch 4, fp16 blocks at 512..64 with conv_clamp 256): forward, a softplus loss
    backward and the R1 double backward on real images, every bias_act / upfirdn2d / fma launch checked against its model."""
    from pix2pix3d_b200 import train_step as ts
    from pix2pix3d_b200.training.dual_discriminator import DualDiscriminator
    kw = ts.discriminator_kwargs(ts.AFHQ_TRAIN)
    kw.pop('class_name')
    assert kw['num_fp16_res'] == 4 and kw['conv_clamp'] == 256 and kw['epilogue_kwargs']['mbstd_group_size'] == 4
    stats = {}
    torch.manual_seed(0)
    restore = install_stream_checks(stats)
    try:
        for ch in (3, 3 + ts.AFHQ_TRAIN['semantic_channels']):
            D = DualDiscriminator(c_dim=25, img_resolution=512, img_channels=ch, **kw).train().cuda()
            img = (torch.rand(4, ch, 512, 512, device='cuda') * 2 - 1)
            raw = (torch.rand(4, ch, 128, 128, device='cuda') * 2 - 1)
            c = torch.randn(4, 25, device='cuda')
            logits = D({'image': img, 'image_raw': raw}, c)
            torch.nn.functional.softplus(logits).sum().backward()
            D.zero_grad(set_to_none=True)
            ir, rr = img.detach().requires_grad_(True), raw.detach().requires_grad_(True)
            logits = D({'image': ir, 'image_raw': rr}, c)
            gi, gr = torch.autograd.grad(logits.sum(), [ir, rr], create_graph=True)
            (gi.square().sum() + gr.square().sum()).mul(2.5).backward()
            torch.cuda.synchronize()
            del D, logits, gi, gr
    finally:
        restore()
    _report_stats('full-size D / D_semantic pass, per (op, dtype, mode, path)', stats)
    for k, v in stats.items():
        REPORT[f'D pass {k}'] = f"worst {v['worst']:.3g}  launches {v['launches']}  elements {v['elements']}"
    bad = {k: v['bad'] for k, v in stats.items() if v['bad']}
    assert not bad, bad
    assert any(k.startswith('bias_act fp16 grad1') for k in stats), sorted(stats)
    assert any(k.startswith('upfirdn2d fp16 strip u2d1') for k in stats), sorted(stats)


REPLAY = """
import json, sys
sys.path[:0] = [{root!r}, {root!r} + '/baseline', {root!r} + '/tests', {root!r} + '/oracle']
import torch
import pix2pix3d_b200
pix2pix3d_b200.install(reference_root={ref!r})
from pix2pix3d_b200 import train_step as ts
import test_gpu_stream_ops_model as T
dev = torch.device('cuda')
stats = {{}}
T.install_stream_checks(stats)
cfg = dict(ts.TINY_TRAIN, d_num_fp16_res=4, sr_num_fp16_res=4)
st = ts.build(cfg, dev)
batch = ts.synthetic_batch(cfg, dev, 5)
torch.manual_seed(2)
st.batch_idx = 0                       # every phase runs
ts.run_iteration(st, batch)
torch.cuda.synchronize()
print('RESULT ' + json.dumps(stats))
"""


@gpu
def test_replay_training_iteration_fp16_blocks():
    """One run_iteration of the tiny recipe with D, D_semantic and SR blocks in fp16 (conv_clamp 256), batch_idx 0 so that
    Gmain, Greg, Dmain, Dreg, D_semanticmain and D_semanticreg all run; every launch of the three ops is checked against its
    model. Runs in a subprocess because install() re-maps module names. (The iteration makes no generic-kernel upfirdn2d
    launch; test_upfirdn2d_generic_and_adjoint covers that kernel.)"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    ref = os.path.join(root, 'oracle', '_ref')
    if not os.path.isdir(os.path.join(ref, 'training')):
        pytest.skip('the reference copy under oracle/_ref is made by build()')
    p = subprocess.run([sys.executable, '-c', REPLAY.format(root=root, ref=ref)], capture_output=True, text=True, timeout=1200)
    line = [ln for ln in p.stdout.splitlines() if ln.startswith('RESULT ')]
    assert p.returncode == 0 and line, p.stdout[-3000:] + p.stderr[-3000:]
    stats = json.loads(line[0][7:])
    _report_stats('replayed training iteration (fp16 D / SR blocks), per (op, dtype, mode, path)', stats)
    for k, v in stats.items():
        REPORT[f'replay {k}'] = f"worst {v['worst']:.3g}  launches {v['launches']}  elements {v['elements']}"
    bad = {k: v['bad'] for k, v in stats.items() if v['bad']}
    assert not bad, bad
    must = ['bias_act fp16 grad0', 'bias_act fp16 grad1', 'bias_act fp32 grad0', 'bias_act fp32 grad1',
            'upfirdn2d fp16 strip u1d1', 'upfirdn2d fp16 strip u2d1', 'upfirdn2d fp16 strip u1d2', 'fma fp32 fwd', 'fma fp32 bwd']
    missing = [m for m in must if not any(k.startswith(m) for k in stats)]
    assert not missing, (missing, sorted(stats))
