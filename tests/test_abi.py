"""The C-ABI: include/p3d.h, its ctypes declaration in _lib.py and the library agree; _lib.launch issues a call as declared
(no compute: runs without a GPU)."""
import contextlib
import ctypes
import os
import re
import subprocess
import tempfile

import pytest
import torch

from conftest import ROOT
from pix2pix3d_b200 import _lib

HEADER = os.path.join(ROOT, 'include', 'p3d.h')

# the ctypes mirror of each struct of the header
MIRRORS = {'p3d_decoder_t': _lib.DecoderDesc, 'p3d_render_args_t': _lib.RenderArgs, 'p3d_render_bwd_args_t': _lib.RenderBwdArgs,
           'p3d_filtered_lrelu_args_t': _lib.FilteredLReluArgs, 'p3d_conv_args_t': _lib.ConvArgs,
           'p3d_wgrad_args_t': _lib.WgradArgs, 'p3d_modw_desc_t': _lib.ModwDesc}
# (kind, bytes) of the scalar types the header uses: i signed integer, u unsigned integer, f floating point, p pointer
C_SCALARS = {'int': ('i', 4), 'int8_t': ('i', 1), 'int32_t': ('i', 4), 'int64_t': ('i', 8), 'uint32_t': ('u', 4),
             'float': ('f', 4), 'p3d_stream_t': ('p', 8)}


def header_source():
    return re.sub(r'/\*.*?\*/', '', open(HEADER).read(), flags=re.S)


def declared_symbols():
    return sorted(set(re.findall(r'\b(p3d_[a-z0-9_]+)\s*\(', header_source())))


def c_decl(text):
    """'const int64_t x_stride[4]' -> (name, base type, pointer?, array length or None)."""
    m = re.fullmatch(r'(?:const\s+)?(unsigned char|\w+)\s*(\*?)\s*(\w+)\s*(?:\[(\d+)\])?', text.strip())
    assert m, text
    return m[3], m[1], bool(m[2]), None if m[4] is None else int(m[4])


def header_structs():
    """{struct name: [(field, base type, pointer?, array length or None), ...]} in declaration order."""
    structs = {}
    for body, name in re.findall(r'typedef struct \{(.*?)\}\s*(\w+);', header_source(), flags=re.S):
        fields = []
        for stmt in filter(None, (s.strip() for s in body.split(';'))):
            first, *more = stmt.split(',')
            fields.append(c_decl(first))
            base = fields[-1][1]
            for d in more:      # further declarators share the base type; a pointer says so itself
                m = re.fullmatch(r'(\*?)\s*(\w+)\s*(?:\[(\d+)\])?', d.strip())
                fields.append((m[2], base, bool(m[1]), None if m[3] is None else int(m[3])))
        structs[name] = fields
    return structs


def header_prototypes():
    """{entry point: (return declaration, [parameter declarations])}."""
    protos = {}
    for ret, name, params in re.findall(r'^((?:const\s+)?\w+\s*\*?)\s*(p3d_\w+)\s*\(([^)]*)\)\s*;', header_source(), flags=re.M):
        params = ' '.join(params.split())
        protos[name] = (c_decl(ret + ' ret'), [] if params == 'void' else [c_decl(p) for p in params.split(',')])
    return protos


def ctypes_kind(t):
    if issubclass(t, ctypes._Pointer):
        return 'p', ctypes.sizeof(t)
    code = t._type_
    return ('f' if code in 'fd' else 'p' if code in 'Pz' else 'u' if code.isupper() else 'i'), ctypes.sizeof(t)


def c_kind(base, pointer):
    return ('p', ctypes.sizeof(ctypes.c_void_p)) if pointer else C_SCALARS.get(base)


def argument_matches(decl, t):
    """A C pointer or array takes c_void_p or a POINTER to the same type; a scalar a ctypes type of its kind and width."""
    _, base, pointer, length = decl
    if pointer or length is not None:
        if t is ctypes.c_void_p:
            return True
        if t is ctypes.c_char_p:
            return base == 'char'
        if not issubclass(t, ctypes._Pointer):
            return False
        return t._type_ is MIRRORS[base] if base in MIRRORS else ctypes_kind(t._type_) == C_SCALARS.get(base)
    return ctypes_kind(t) == c_kind(base, False)


def test_header_declares_entry_points():
    syms = declared_symbols()
    for must in ('p3d_render_fwd', 'p3d_bias_act', 'p3d_upfirdn2d', 'p3d_ray_sampler', 'p3d_run_model'):
        assert must in syms


def test_library_exports_all_declared_symbols():
    if not _lib.available():
        pytest.skip('libp3d.so not built (run python -m pix2pix3d_b200.build)')
    handle = ctypes.CDLL(_lib.LIB_PATH)
    missing = [s for s in declared_symbols() if not hasattr(handle, s)]
    assert not missing, missing
    assert handle.p3d_abi_version() == _lib.ABI_VERSION


def test_ctypes_table_covers_header():
    assert sorted(_lib.EXPORTED_SYMBOLS) == declared_symbols()


def test_signatures_match_header_prototypes():
    """Every _SIGNATURES row has its prototype's arity, and each argument and the return value its kind and width: a c_int where
    the header says int64_t, or a dropped argument, would marshal garbage without an error."""
    protos = header_prototypes()
    bad = []
    for name, (res, args) in _lib._SIGNATURES.items():
        ret, params = protos[name]
        if len(params) != len(args):
            bad.append((name, f'{len(args)} arguments, the header has {len(params)}'))
            continue
        if not argument_matches(ret, res):
            bad.append((name, 'return type'))
        bad += [(name, p[0]) for p, t in zip(params, args) if not argument_matches(p, t)]
    assert not bad, bad


def c_layouts(structs):
    """{struct: (sizeof, {field: (offsetof, sizeof)})} as gcc lays out the header's `structs`."""
    lines = []
    for s, fields in structs.items():
        lines.append(f'printf("{s} - %zu 0\\n", sizeof({s}));')
        lines += [f'printf("{s} {f[0]} %zu %zu\\n", offsetof({s}, {f[0]}), sizeof((({s}*)0)->{f[0]}));' for f in fields]
    prog = '#include <stdio.h>\n#include <stddef.h>\n#include "p3d.h"\nint main(void) {\n' + '\n'.join(lines) + '\nreturn 0;\n}\n'
    with tempfile.TemporaryDirectory() as td:
        src, exe = os.path.join(td, 'layout.c'), os.path.join(td, 'layout')
        with open(src, 'w') as fh:
            fh.write(prog)
        subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), src, '-o', exe])
        out = subprocess.check_output([exe], text=True)
    layouts = {s: [0, {}] for s in structs}
    for ln in out.splitlines():
        s, f, a, b = ln.split()
        if f == '-':
            layouts[s][0] = int(a)
        else:
            layouts[s][1][f] = (int(a), int(b))
    return layouts


def test_struct_mirrors_match_header():
    """Each of the seven mirrors has its struct's fields in the header's order, its gcc sizeof, and each field gcc's offset and
    size and the header's kind."""
    structs = header_structs()
    layouts = c_layouts(structs)
    bad = []
    for struct, mirror in MIRRORS.items():
        fields, (size, offsets) = structs[struct], layouts[struct]
        if [n for n, _ in mirror._fields_] != [f[0] for f in fields]:
            bad.append((struct, 'field names or order'))
            continue
        if ctypes.sizeof(mirror) != size:
            bad.append((struct, 'sizeof'))
        types = dict(mirror._fields_)
        for name, base, pointer, length in fields:
            t = types[name]
            if (getattr(mirror, name).offset, getattr(mirror, name).size) != offsets[name]:
                bad.append((struct, name, 'offset or size'))
            if length is not None:
                if not (issubclass(t, ctypes.Array) and t._length_ == length):
                    bad.append((struct, name, 'array length'))
                    continue
                t = t._type_
            if ctypes_kind(t) != c_kind(base, pointer):
                bad.append((struct, name, 'kind'))
    assert not bad, bad


def test_cuda_ops_fail_loudly_without_library(monkeypatch):
    monkeypatch.setattr(_lib, 'LIB_PATH', '/nonexistent/libp3d.so')
    monkeypatch.setattr(_lib, '_lib', None)
    with pytest.raises(RuntimeError, match='missing'):
        _lib.lib()


def test_library_exports_nothing_undeclared():
    """Every `p3d_*` symbol the shared library exports is declared in include/p3d.h (no entry points outside the documented ABI)."""
    import shutil
    if not _lib.available() or not shutil.which('nm'):
        pytest.skip('needs the built library and nm')
    out = subprocess.check_output(['nm', '-D', '--defined-only', _lib.LIB_PATH], text=True)
    exported = sorted({ln.split()[-1] for ln in out.splitlines() if ln.split() and re.fullmatch(r'p3d_[a-z0-9_]+', ln.split()[-1])})
    assert exported == declared_symbols()


class _FakeLibrary:
    """Stands in for the libp3d handle: records each call's arguments and returns a fixed status."""

    def __init__(self, status):
        self.status, self.calls = status, []

    def p3d_status_string(self, status):
        return b'fake status'

    def __getattr__(self, name):
        def call(*args):
            self.calls.append((name, args))
            return self.status
        return call


@pytest.fixture
def fake_library(monkeypatch):
    def install(status):
        fake = _FakeLibrary(status)
        monkeypatch.setattr(_lib, '_lib', fake)
        monkeypatch.setattr(_lib, 'stream_ptr', lambda device=None: 'stream')
        monkeypatch.setattr(torch.cuda, 'device', lambda device: contextlib.nullcontext())
        monkeypatch.setattr(_lib, 'launch_count', 0)
        return fake
    return install


def test_launch_passes_pointers_scalars_and_the_stream(fake_library):
    fake = fake_library(0)
    t, u = torch.zeros(16), torch.zeros(4)
    assert _lib.launch('p3d_sample_importance', t, u, None, 3, 4, 5, t, None, device='cuda:0') is True
    (name, args), = fake.calls
    assert name == 'p3d_sample_importance' and args[-1] == 'stream'
    assert [a.value for a in args[:2]] == [t.data_ptr(), u.data_ptr()] and all(isinstance(a, ctypes.c_void_p) for a in args[:2])
    assert args[2] is None and args[7] is None
    assert args[3:6] == (3, 4, 5)
    assert _lib.launch_count == 1
    _lib.launch('p3d_decoder_mlp_bwd', *([t] * 3), 1, 1, *([t] * 4), 0, *([t] * 5), 16, device='cuda:0', launches=2)
    assert _lib.launch_count == 3


def test_launch_rejects_a_tensor_in_a_scalar_slot(fake_library):
    fake = fake_library(0)
    t = torch.zeros(4)
    with pytest.raises(TypeError, match='p3d_ray_sampler: argument 2'):
        _lib.launch('p3d_ray_sampler', t, t, torch.tensor(2), 4, t, t, device='cuda:0')
    assert fake.calls == [] and _lib.launch_count == 0


def test_launch_raises_on_a_failing_status_naming_the_entry_point(fake_library):
    fake_library(-2)
    with pytest.raises(RuntimeError, match=r'^p3d_render_fwd_tc failed: fake status \(status -2\)$'):
        _lib.launch('p3d_render_fwd_tc', None, device='cuda:0')
    with pytest.raises(RuntimeError, match='p3d_conv_gemm failed'):
        _lib.launch('p3d_conv_gemm', None, device='cuda:0', unsupported_ok=True)       # only P3D_UNSUPPORTED is tolerated
    assert _lib.launch_count == 0


def test_launch_reports_unsupported_when_asked(fake_library):
    fake_library(_lib.P3D_UNSUPPORTED)
    assert _lib.launch('p3d_conv_gemm', None, device='cuda:0', unsupported_ok=True) is False
    with pytest.raises(RuntimeError, match='p3d_conv_gemm failed'):
        _lib.launch('p3d_conv_gemm', None, device='cuda:0')
    assert _lib.launch_count == 0
