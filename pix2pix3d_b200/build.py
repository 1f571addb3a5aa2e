"""Ahead-of-time build of libp3d.so (sm_90a only) with nvcc.

Unlike the reference's JIT loader (torch_utils/custom_ops.py:61-157 in the reference repo) nothing is
compiled at first call: `python -m pix2pix3d_b200.build` (or __graft_entry__.build()) produces
pix2pix3d_b200/libp3d.so in-tree, and the library is then loaded through ctypes.
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OUT = os.path.join(HERE, 'libp3d.so')
STAMP = os.path.join(HERE, 'csrc', '.build_stamp')

NVCC_FLAGS = [
    '-gencode', 'arch=compute_90a,code=sm_90a',
    '-O3', '-lineinfo', '-std=c++17',
    '-Xcompiler', '-fPIC', '-Xcompiler', '-O3',
    '--expt-relaxed-constexpr',
    '-Xptxas', '-v',
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _digest():
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, '..', 'include')):
        for f in sorted(os.listdir(root)):
            if f.endswith(('.cu', '.cuh', '.h')):
                with open(os.path.join(root, f), 'rb') as fh:
                    h.update(f.encode())
                    h.update(fh.read())
    h.update(' '.join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ into objects and link libp3d.so. Returns the library path."""
    digest = _digest()
    if not force and os.path.exists(OUT) and os.path.exists(STAMP):
        with open(STAMP) as fh:
            if fh.read().strip() == digest:
                return OUT
    nvcc = os.environ.get('NVCC', 'nvcc')
    objs = []
    procs = []
    hdr = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, '..', 'include')):
        for f in sorted(os.listdir(root)):
            if f.endswith(('.cuh', '.h')):
                with open(os.path.join(root, f), 'rb') as fh:
                    hdr.update(fh.read())
    hdr.update(' '.join(NVCC_FLAGS).encode())
    for src in sources():
        obj = src[:-3] + '.o'
        objs.append(obj)
        with open(src, 'rb') as fh:
            src_digest = hashlib.sha256(hdr.digest() + fh.read()).hexdigest()
        tag = obj + '.sha'
        if not force and os.path.exists(obj) and os.path.exists(tag) and open(tag).read().strip() == src_digest:
            continue       # object is up to date (per-file incremental build)
        cmd = [nvcc] + NVCC_FLAGS + ['-c', src, '-o', obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True), tag, src_digest))
    log = []
    for src, p, tag, src_digest in procs:
        out, _ = p.communicate()
        log.append(out)
        if p.returncode != 0:
            sys.stderr.write(out)
            raise RuntimeError(f'nvcc failed for {src}')
        with open(tag, 'w') as fh:
            fh.write(src_digest)
        with open(src[:-3] + '.ptxas.log', 'w') as fh:
            fh.write(out)
    cmd = [nvcc, '-shared', '-gencode', 'arch=compute_90a,code=sm_90a', '-o', OUT] + objs
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError('link failed')
    with open(STAMP, 'w') as fh:
        fh.write(digest)
    if verbose:
        sys.stdout.write('\n'.join(log))
    return OUT


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='-v' in sys.argv))
