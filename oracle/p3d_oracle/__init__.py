"""CPU oracle for the pix2pix3D render + StyleGAN2-op hot path.

TEST INFRASTRUCTURE ONLY. This package is a numpy restatement of the reference's algorithms, each function citing
the reference file:line it follows. It may be imported by tests/, by __graft_entry__.smoke() and by the
cpu_baseline / --impl reference legs of bench.py -- never by pix2pix3d_b200 (the product), which must fail loudly
when its CUDA library is missing.

Pinning: the reference ships no tests or golden vectors (SURVEY.md section 4). The oracle is pinned against the
reference's own Python implementation, imported from a reference checkout and run on CPU by
oracle/make_golden.py; the resulting fixtures live in tests/golden/ and tests/test_oracle_golden.py checks the
oracle against them. Dense-convolution arithmetic that the reference itself delegates to ATen
(F.conv2d / F.conv_transpose2d, torch_utils/ops/conv2d_gradfix.py:40-45) is available both ways: ATen's CPU
convolution (default; keeps the CPU baseline at the reference's own CPU speed) and an explicit im2col + matmul
restatement in numpy (P3D_ORACLE_NUMPY_CONV=1); the tests check that the two agree.
"""
from . import ops, renderer, networks  # noqa: F401
