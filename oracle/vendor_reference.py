"""Copy the UNMODIFIED reference (pix2pix3D) into the git-ignored oracle/_ref/.

The reference is a script tree without setup.py / pyproject.toml, so `pip install --target <dir> <checkout>` has nothing to
install (DESIGN.md section 2); the build of a script tree is a verbatim copy of its importable modules. `__graft_entry__.build()`
runs this recipe, so that the CPU tests that drive the reference's own loss class, training loop and pickle writer
(test_train_step_cpu, test_train_step_gloo_cpu, test_install_boundary, test_checkpoint_compat), the GPU tests that run the
reference's op wrappers on this package's plugins, and the reference arms and legs of bench.py (baseline/ref_harness.py)
find it under oracle/_ref/. The copy is byte-identical and never part of this repository's history; it imports under its own
module names (`training`, `torch_utils`, `dnnlib`), never mixed into the product path.

    python oracle/vendor_reference.py

The checkout is read from $P3D_REFERENCE_ROOT, by default from where the reference is mounted read-only next to this
repository's working copy; without a checkout nothing is copied.
"""
import filecmp
import os
import shutil
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.environ.get('P3D_REFERENCE_ROOT', '/root/reference')
DST = os.path.join(HERE, '_ref')
# importable code + the three CUDA plugins' sources (JIT-built on first use by the reference's own custom_ops.get_plugin)
TREES = ('training', 'torch_utils', 'dnnlib', 'metrics')
FILES = ('camera_utils.py', 'legacy.py', 'train.py', 'LICENSE', 'applications/generate_samples.py',
         'applications/generate_video.py', 'applications/extract_mesh.py')
SUFFIXES = ('.py', '.cu', '.cpp', '.h', '.txt')


def vendor(verbose=False):
    if not SRC or not os.path.isdir(os.path.join(SRC, 'training')):
        return available()
    n = 0
    for tree in TREES:
        for root, dirs, files in os.walk(os.path.join(SRC, tree)):
            dirs[:] = [d for d in dirs if d != '__pycache__']
            for f in files:
                if f.endswith(SUFFIXES):
                    rel = os.path.relpath(os.path.join(root, f), SRC)
                    n += _copy(rel)
    for rel in FILES:
        if os.path.exists(os.path.join(SRC, rel)):
            n += _copy(rel)
    if verbose:
        print(f'vendored reference -> {DST} ({n} files updated)')
    return True


def _copy(rel):
    s, d = os.path.join(SRC, rel), os.path.join(DST, rel)
    if os.path.exists(d) and filecmp.cmp(s, d, shallow=False):
        return 0
    os.makedirs(os.path.dirname(d), exist_ok=True)
    shutil.copyfile(s, d)
    return 1


def available():
    return os.path.isdir(os.path.join(DST, 'training'))


if __name__ == '__main__':
    ok = vendor(verbose=True)
    sys.exit(0 if ok else 1)
