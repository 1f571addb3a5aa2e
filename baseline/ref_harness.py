"""Drive the UNMODIFIED reference (oracle/_ref, the byte-identical copy of pix2pix3D that build() makes) through its own public API:
`TriPlaneSemanticEntangleGenerator.synthesis` (training/triplane_cond.py:1020-1061) built with the kwargs train.py assembles
(`pix2pix3d_b200.configs.generator_kwargs`, pure data) and the same seeds as the product arm, so both arms hold identical
weights and see identical inputs.

  device 'cpu'  -> the reference's CPU path: every custom op takes its `_ref` branch (bias_act.py:86-88, upfirdn2d.py:162-164),
                   fp32 everywhere (networks_stylegan2.py:423-425)                     [BASELINE.md plan item 1]
  device 'cuda' -> the reference's stock CUDA path: plugins JIT-built by its own torch_utils/custom_ops.py:61 on first use,
                   cuDNN convolutions, SR in fp16 as shipped (or force_fp32)           [BASELINE.md plan item 2]

Nothing from the product package's kernels or modules is on this path (only `configs`, a table of constructor arguments
and input generators). Used by bench.py (`--impl reference`, `--impl reference-cuda`, the `cpu_baseline` /
`stock_cuda` legs) and tests/test_gpu_vs_reference.py.
"""
import atexit
import contextlib
import os
import shutil
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF_ROOT = os.path.join(ROOT, 'oracle', '_ref')


def available():
    return os.path.isdir(os.path.join(REF_ROOT, 'training'))


def import_reference():
    """Put oracle/_ref first on sys.path and return its `training.triplane_cond` module. The reference's CUDA plugins, JIT-built
    on first use, go to a temporary directory (removed at exit) unless TORCH_EXTENSIONS_DIR names one."""
    if not available():
        raise RuntimeError('oracle/_ref is missing: __graft_entry__.build() copies the reference there (oracle/vendor_reference.py)')
    if 'TORCH_EXTENSIONS_DIR' not in os.environ:
        d = tempfile.mkdtemp(prefix='p3d_torch_extensions_')
        atexit.register(shutil.rmtree, d, True)
        os.environ['TORCH_EXTENSIONS_DIR'] = d
    if REF_ROOT not in sys.path:
        sys.path.insert(0, REF_ROOT)
    if ROOT not in sys.path:
        sys.path.append(ROOT)
    import training.triplane_cond as tc
    assert os.path.abspath(tc.__file__).startswith(REF_ROOT), f'`training` resolved to {tc.__file__}, not the vendored reference'
    _torch2_plugin_loader_compat()
    import torch_utils.custom_ops as co
    co.verbosity = 'none'          # as train.py:54 does; keeps stdout to the one JSON line
    return tc


def _torch2_plugin_loader_compat():
    """Environment shim, not a change to the reference: its loader (torch_utils/custom_ops.py:137-144) calls
    `torch.utils.cpp_extension.load(name=...)` and then `importlib.import_module(name)`. torch 1.11 (the reference's pin,
    environment.yml:21) registered the built module in `sys.modules`; torch 2.x returns it without registering, so the second
    call raises ModuleNotFoundError. Registering the module `load` returns restores
    the behaviour the reference was written against; sources, flags and kernels are the reference's own."""
    import torch.utils.cpp_extension as ce
    if getattr(ce.load, '_p3d_registers_module', False):
        return
    orig = ce.load

    def load(*args, **kwargs):
        mod = orig(*args, **kwargs)
        name = kwargs.get('name', args[0] if args else None)
        if mod is not None and name and name not in sys.modules:
            sys.modules[name] = mod
        return mod
    load._p3d_registers_module = True
    ce.load = load


def build_generator(workload, seed=0, device='cpu', with_mapping=False):
    """Reference generator with the product arm's weights: same constructor kwargs, same torch seed, same noise-strength
    draw (pix2pix3d_b200.configs.build_generator), so state dicts agree bit for bit (tests/test_mirror_cpu.py digest)."""
    import torch
    tc = import_reference()
    from pix2pix3d_b200 import configs
    kw = configs.generator_kwargs(workload)
    if not with_mapping:
        kw['mapping_kwargs'] = dict(class_name='training.networks_stylegan2.MappingNetwork', num_layers=2)
    torch.manual_seed(seed)
    G = tc.TriPlaneSemanticEntangleGenerator(**kw).eval().requires_grad_(False)
    g = torch.Generator().manual_seed(seed + 1)
    with torch.no_grad():
        for pname, p in G.named_parameters():
            if pname.endswith('noise_strength'):
                p.copy_(torch.randn([], generator=g) * 0.1)
    return G.to(device)


def inputs(workload, batch, num_ws, rank=0):
    from pix2pix3d_b200 import configs
    preset = configs.WORKLOADS[workload]['preset']
    return configs.synthetic_ws(batch, num_ws, 1 + rank), configs.camera_labels(batch, 2 + rank, preset)


@contextlib.contextmanager
def replay_rand(jitter, u):
    """Feed the renderer's two draws (renderer.py:190 rand_like, :237 rand) from given tensors."""
    import torch
    it = iter([jitter, u])
    o_like, o_rand = torch.rand_like, torch.rand
    torch.rand_like = lambda x, *a, **k: next(it).to(x.device)
    torch.rand = lambda *a, **k: next(it).to(k.get('device', 'cpu'))
    try:
        yield
    finally:
        torch.rand_like, torch.rand = o_like, o_rand


class StageTimer:
    """Per-stage wall (CPU) or CUDA-event (GPU) time of backbone / renderer / SR stacks via forward hooks (BASELINE.md 3.1)."""

    def __init__(self, G, cuda):
        import torch
        self.cuda = cuda
        self.spans = {}
        self.handles = []
        stages = {'backbone': G.backbone.synthesis, 'renderer': G.renderer, 'sr_rgb': G.superresolution}
        if hasattr(G, 'superresolution_semantic'):
            stages['sr_semantic'] = G.superresolution_semantic
        for name, mod in stages.items():
            self.handles.append(mod.register_forward_pre_hook(lambda m, a, n=name: self._begin(n)))
            self.handles.append(mod.register_forward_hook(lambda m, a, o, n=name: self._end(n)))
        self._torch = torch

    def _mark(self):
        if self.cuda:
            e = self._torch.cuda.Event(enable_timing=True)
            e.record()
            return e
        return time.perf_counter()

    def _begin(self, n):
        self.spans.setdefault(n, []).append([self._mark(), None])

    def _end(self, n):
        self.spans[n][-1][1] = self._mark()

    def reset(self):
        self.spans = {}

    def totals_ms(self):
        if self.cuda:
            self._torch.cuda.synchronize()
            return {n: sum(a.elapsed_time(b) for a, b in v) for n, v in self.spans.items()}
        return {n: 1000 * sum(b - a for a, b in v) for n, v in self.spans.items()}

    def close(self):
        for h in self.handles:
            h.remove()


def usable_cores():
    """Cores this process may run on: the affinity mask, further limited by a cgroup CPU quota if one is set."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, 'sched_getaffinity') else (os.cpu_count() or 1)
    try:
        with open('/sys/fs/cgroup/cpu.max') as fh:
            quota, period = fh.read().split()[:2]
        if quota != 'max':
            n = max(1, min(n, int(float(quota) / float(period) + 0.5)))
    except (OSError, ValueError):
        pass
    return n


_thread_choice = {}


def pick_cpu_threads(G, ws1, c1, kw, log=None):
    """The CPU arm should be the reference at its best, not at `os.cpu_count()` threads: on a many-core host the
    reference's many small ATen ops run several times slower with 128 intra-op threads than with a few dozen. One image is timed at a few thread counts and the fastest kept."""
    import torch
    cores = usable_cores()
    key = (cores, tuple(ws1.shape))
    if key in _thread_choice:
        torch.set_num_threads(_thread_choice[key])
        return _thread_choice[key]
    cands = sorted({t for t in (cores, cores // 2, cores // 4, 32, 16, 8) if 1 <= t <= cores})
    best, best_t = None, None
    for t in cands:                                      # ascending; stop once more threads clearly stop paying
        if best is not None and t > 8 and last > 1.25 * best:
            break
        torch.set_num_threads(t)
        with torch.no_grad():
            G.synthesis(ws1, c1, **kw)                  # warm (allocator, oneDNN primitive cache)
            t0 = time.perf_counter()
            G.synthesis(ws1, c1, **kw)
            dt = time.perf_counter() - t0
        last = dt
        if log:
            log(f'reference cpu: {t} threads -> {dt:.2f} s per image')
        if best is None or dt < best:
            best, best_t = dt, t
    torch.set_num_threads(best_t)
    _thread_choice[key] = best_t
    return best_t


def time_synthesis(workload, device, batch, steps, warmup, force_fp32=False, budget_s=None, stage_split=True, log=None):
    """Time `G.synthesis(ws, c, noise_mode='const', neural_rendering_resolution=nrr)` of the reference. Returns a dict with
    ms per step (wall clock on CPU, CUDA events on GPU), the steps / warm-up actually run (bounded by `budget_s` seconds of
    run time) and the per-stage split."""
    import torch
    from pix2pix3d_b200 import configs
    cuda = str(device).startswith('cuda')
    w = configs.WORKLOADS[workload]
    G = build_generator(workload, seed=0, device=device)
    ws, c = inputs(workload, batch, G.backbone.num_ws)
    ws, c = ws.to(device), c.to(device)
    kw = dict(noise_mode='const', neural_rendering_resolution=w['nrr'])
    if force_fp32:
        kw['force_fp32'] = True
    threads = None
    if not cuda:
        threads = pick_cpu_threads(G, ws[:1], c[:1], kw, log)

    def step():
        with torch.no_grad():
            return G.synthesis(ws, c, **kw)

    def sync():
        if cuda:
            torch.cuda.synchronize()

    t0 = time.perf_counter()
    step(); sync()
    t_first = time.perf_counter() - t0
    if log:
        log(f'reference {device} first step (incl. plugin JIT / warm caches): {t_first:.1f} s')
    t0 = time.perf_counter()
    step(); sync()
    t_step = max(time.perf_counter() - t0, 1e-4)
    if budget_s is not None:
        warm = max(2, min(warmup, int(0.2 * budget_s / t_step)))
        steps = max(1, min(steps, int(0.8 * budget_s / t_step)))
    else:
        warm = max(2, warmup)
    for _ in range(warm - 2):
        step()
    sync()
    timer = StageTimer(G, cuda) if stage_split else None
    if cuda:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            out = step()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1)
    else:
        t0 = time.perf_counter()
        for _ in range(steps):
            out = step()
        ms = 1000 * (time.perf_counter() - t0)
    stages = None
    if timer is not None:
        tot = timer.totals_ms()
        stages = {k: v / steps for k, v in tot.items()}
        stages['other'] = ms / steps - sum(stages.values())
        timer.close()
    return {'threads': threads, 'ms_per_step': ms / steps, 'steps': steps, 'warmup': warm, 'batch': batch, 'images_per_s': batch * steps / (ms / 1000),
            'first_step_s': t_first, 'stage_ms_per_step': stages, 'out_shapes': {k: list(v.shape) for k, v in out.items()},
            'dtype': 'f32' if (force_fp32 or not cuda) else 'f32 backbone/renderer + f16 super-resolution (as shipped)'}
