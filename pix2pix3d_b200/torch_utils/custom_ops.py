"""Plugin loader with the reference's surface (torch_utils/custom_ops.py:26 `verbosity`, :61 `get_plugin`).

The reference JIT-compiles a pybind module per op on first use and hands it to `torch_utils/ops/*.py`, whose autograd
classes call `_plugin.bias_act(...)`, `_plugin.upfirdn2d(...)`, `_plugin.filtered_lrelu(...)`,
`_plugin.filtered_lrelu_act_(...)` (bias_act.cpp:36, upfirdn2d.cpp:20, filtered_lrelu.cpp:20,217). Here the plugins are
ahead-of-time objects over libp3d.so's C-ABI (include/p3d.h) with those very call signatures, so the REFERENCE's own
`torch_utils/ops/{bias_act,upfirdn2d,filtered_lrelu}.py` run unmodified on the sm_90a kernels when this module stands in
for the reference's (`tests/test_gpu_vs_reference.py::test_reference_op_wrappers_run_on_libp3d_plugins` and
`::test_reference_filtered_lrelu_wrapper_runs_on_libp3d_plugin` do exactly that). Nothing is compiled at import or call time;
`sources`, `headers`, `source_dir` and build kwargs are accepted and ignored.
"""
import torch

verbosity = 'brief'            # 'none' | 'brief' | 'full' (train.py:54 sets it); no build output exists to be verbose about


def _opt(t):
    """The pybind plugins take an empty tensor for "absent" (bias_act.cpp:47-52)."""
    return None if t is None or t.numel() == 0 else t


class _BiasActPlugin:
    plugin_name = 'bias_act_plugin'

    @staticmethod
    def bias_act(x, b, xref, yref, dy, grad, dim, act, alpha, gain, clamp):
        from .ops import bias_act as impl
        return impl._launch(x, _opt(b), _opt(xref), _opt(yref), _opt(dy), int(grad), int(dim), int(act), float(alpha),
                            float(gain), float(clamp))


class _Upfirdn2dPlugin:
    plugin_name = 'upfirdn2d_plugin'

    @staticmethod
    def upfirdn2d(x, f, upx, upy, downx, downy, padx0, padx1, pady0, pady1, flip, gain):
        from .ops import upfirdn2d as impl
        return impl._launch(x, f, int(upx), int(upy), int(downx), int(downy), int(padx0), int(padx1), int(pady0), int(pady1),
                            bool(flip), float(gain))


class _FilteredLReluPlugin:
    plugin_name = 'filtered_lrelu_plugin'

    @staticmethod
    def filtered_lrelu(x, fu, fd, b, si, up, down, px0, px1, py0, py1, sx, sy, gain, slope, clamp, flip_filter, write_signs):
        from .ops import filtered_lrelu as impl
        return impl._plugin_filtered_lrelu(x, fu, fd, b, si, int(up), int(down), int(px0), int(px1), int(py0), int(py1), int(sx),
                                           int(sy), float(gain), float(slope), float(clamp), bool(flip_filter), bool(write_signs))

    @staticmethod
    def filtered_lrelu_act_(x, si, sx, sy, gain, slope, clamp, write_signs):
        from .ops import filtered_lrelu as impl
        return impl._plugin_filtered_lrelu_act_(x, si, int(sx), int(sy), float(gain), float(slope), float(clamp), bool(write_signs))


_PLUGINS = {p.plugin_name: p for p in (_BiasActPlugin, _Upfirdn2dPlugin, _FilteredLReluPlugin)}


def get_plugin(module_name, sources=None, headers=None, source_dir=None, **build_kwargs):
    assert verbosity in ('none', 'brief', 'full')
    if module_name not in _PLUGINS:
        raise RuntimeError(f'no ahead-of-time plugin named {module_name!r} in libp3d.so (known: {sorted(_PLUGINS)})')
    from .. import _lib
    _lib.lib()                 # fail here, loudly, if the native library has not been built
    return _PLUGINS[module_name]
