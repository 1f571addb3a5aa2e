"""Every module of the package (and the repo-root entry points) imports on a machine without a GPU: a missing import in a module
the CPU suite does not otherwise touch (engine.py, graphs.py, train_step.py ...) would only show up on a GPU machine."""
import importlib
import os
import pkgutil


def test_every_module_imports():
    import pix2pix3d_b200
    names = ['pix2pix3d_b200']
    for m in pkgutil.walk_packages(pix2pix3d_b200.__path__, 'pix2pix3d_b200.'):
        if not m.name.endswith('.libp3d'):          # the C-ABI library sits in the package directory; it is loaded with ctypes
            names.append(m.name)
    for n in names:
        importlib.import_module(n)
    for n in ('bench', '__graft_entry__'):
        spec = importlib.util.spec_from_file_location(n + '_probe', os.path.join(os.path.dirname(os.path.dirname(__file__)), n + '.py'))
        spec.loader.exec_module(importlib.util.module_from_spec(spec))
