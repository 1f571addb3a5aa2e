"""pix2pix3d_b200 -- sm_90a (H100) implementation of pix2pix3D's volumetric-rendering + StyleGAN2-op hot path.

Layout
  csrc/            CUDA kernels and the C-ABI (include/p3d.h) -> libp3d.so (built by `pix2pix3d_b200.build`)
  _lib.py          ctypes binding of the C-ABI
  native.py        tensor-level wrappers (allocate outputs, pass raw pointers)
  torch_utils/, training/, dnnlib/
                   host-side mirror of the reference's operator surface (same import paths below the package
                   root, same class / function names and signatures)

`install()` makes the mirror answer to the reference's top-level module names (`training.*`, `torch_utils.*`,
`dnnlib`, `camera_utils`, `legacy`), so reference callers (applications/generate_samples.py, train.py) and pickles that
refer to those paths resolve to this package.
"""
import importlib
import importlib.abc
import importlib.util
import os
import sys

__version__ = '0.2.0'

_ALIASED_ROOTS = ('training', 'torch_utils', 'dnnlib', 'camera_utils', 'legacy')
_PKG_DIR = os.path.dirname(os.path.abspath(__file__))


class _AliasFinder(importlib.abc.MetaPathFinder, importlib.abc.Loader):
    """Resolves `training.x.y` to the already-imported (or importable) `pix2pix3d_b200.training.x.y`, returning
    the very same module object so that classes are not duplicated under two names.

    Modules of an aliased root that this package does NOT own -- the reference's host-side siblings
    (`training.training_loop`, `training.dataset`, `training.augment`, `training.utils`, `training.crosssection_utils`,
    `training.networks_stylegan3`, `training.loss`) -- keep resolving to the reference checkout: they are looked up
    under `reference_root` (if given) and then along `sys.path`, exactly where the plain import system would have found
    them, and are executed under their reference names. Their own `from torch_utils import ...` / `from training.x import
    ...` statements come back through this finder, so they run on the mirror's operators."""

    def __init__(self, reference_root=None):
        self.reference_root = reference_root

    def _sibling_spec(self, fullname):
        parts = fullname.split('.')
        bases = ([self.reference_root] if self.reference_root else []) + [p or os.getcwd() for p in sys.path]
        for base in bases:
            if not isinstance(base, str) or os.path.abspath(base).startswith(_PKG_DIR):
                continue
            cand = os.path.join(base, *parts)
            if os.path.isfile(cand + '.py'):
                return importlib.util.spec_from_file_location(fullname, cand + '.py')
            init = os.path.join(cand, '__init__.py')
            if os.path.isfile(init):
                return importlib.util.spec_from_file_location(fullname, init, submodule_search_locations=[cand])
        return None

    @staticmethod
    def _mirror_owns(short):
        cand = os.path.join(_PKG_DIR, *short.split('.'))
        return os.path.isfile(cand + '.py') or os.path.isfile(os.path.join(cand, '__init__.py'))

    def find_spec(self, fullname, path=None, target=None):
        prefix = __name__ + '.'
        if fullname.startswith(prefix):
            # `from training import training_loop` asks for `pix2pix3d_b200.training.training_loop` (the alias module keeps
            # its real __name__): hand out the reference-side sibling `training.training_loop` for names the mirror lacks
            short = fullname[len(prefix):]
            if short.split('.', 1)[0] in _ALIASED_ROOTS and '.' in short and not self._mirror_owns(short) \
                    and self._sibling_spec(short) is not None:
                return importlib.util.spec_from_loader(fullname, self, origin=short)
            return None
        root = fullname.split('.', 1)[0]
        if root not in _ALIASED_ROOTS:
            return None
        if self._mirror_owns(fullname):
            return importlib.util.spec_from_loader(fullname, self, origin=f'{__name__}.{fullname}')
        return self._sibling_spec(fullname)

    def create_module(self, spec):
        return importlib.import_module(spec.origin)

    def exec_module(self, module):
        pass


_finder = None


def install(reference_root=None):
    """Register the alias finder (idempotent). Call before importing `training`, `torch_utils` or `dnnlib`.
    `reference_root`: a checkout of the reference whose host-side modules (training loop, datasets, metrics glue) should
    stay importable next to the mirror; without it they are searched along `sys.path`."""
    global _finder
    if _finder is None:
        _finder = _AliasFinder(reference_root)
        sys.meta_path.insert(0, _finder)
    elif reference_root is not None:
        _finder.reference_root = reference_root
    return _finder


def uninstall():
    global _finder
    if _finder is not None:
        sys.meta_path.remove(_finder)
        _finder = None
    for name in list(sys.modules):
        if name.split('.', 1)[0] in _ALIASED_ROOTS:
            mod = sys.modules[name]
            if getattr(mod, '__name__', '').startswith(__name__ + '.') or getattr(mod, '__name__', '') == name:
                del sys.modules[name]
