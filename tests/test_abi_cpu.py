"""CPU-only checks of the drop-in boundary: the C-ABI library loads, exports every symbol include/fqb200.h declares,
its struct layout matches the ctypes mirror, argument validation works without a GPU, and the product has no CPU
fallback."""
import ctypes
import os
import re
import subprocess

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


def _header_symbols():
    src = open(os.path.join(ROOT, "include", "fqb200.h")).read()
    return sorted(set(re.findall(r"\b(fqb200_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol(lib):
    from cnn_quantization_b200 import _lib
    declared = _header_symbols()
    assert sorted(_lib.SYMBOLS) == declared
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    exported = set(line.split()[-1] for line in out.splitlines() if line.strip())
    for sym in declared:
        assert sym in exported, sym
        assert getattr(lib, sym) is not None
    # ... and nothing else: no undeclared hooks ride along in the shipped library (round-1 VERDICT, boundary hygiene)
    ours = sorted(s for s in exported if s.startswith("fqb"))
    assert ours == declared, sorted(set(ours) - set(declared))
    assert lib.fqb200_abi_version() == _lib.ABI_VERSION == 3


def test_desc_struct_layout_matches_header():
    from cnn_quantization_b200 import _lib
    # compile a one-liner against the header and compare sizeof / offsetof with the ctypes mirror
    code = ('#include <stdio.h>\n#include <stddef.h>\n#include "fqb200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu %zu\\n", '
            'sizeof(fqb200_desc), offsetof(fqb200_desc, clip_k), offsetof(fqb200_desc, mt_target), '
            'offsetof(fqb200_desc, out_stats), offsetof(fqb200_desc, channels_last), offsetof(fqb200_desc, residual_stats), '
            'offsetof(fqb200_desc, debug_stamps));'
            'return 0;}\n')
    exe = os.path.join(ROOT, "oracle", "_build", "abi_probe")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    subprocess.run(["gcc", "-x", "c", "-", "-I", os.path.join(ROOT, "include"), "-o", exe], input=code, text=True, check=True)
    got = [int(v) for v in subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()]
    D = _lib.Desc
    assert got == [ctypes.sizeof(D), D.clip_k.offset, D.mt_target.offset, D.out_stats.offset, D.channels_last.offset,
                   D.residual_stats.offset, D.debug_stamps.offset]


def test_argument_validation_without_gpu(lib):
    from cnn_quantization_b200 import _lib
    d = _lib.Desc()
    d.outer, d.groups, d.inner, d.num_bits = 4, 16, 196, 4
    assert lib.fqb200_workspace_bytes(ctypes.byref(d)) > 0
    d.num_bits = 0
    assert lib.fqb200_workspace_bytes(ctypes.byref(d)) == 0
    d.num_bits, d.scope = 4, 7
    assert lib.fqb200_workspace_bytes(ctypes.byref(d)) == 0
    assert b"scope" in lib.fqb200_last_error()
    assert lib.fqb200_float2gemmlowp(None, None, -1, 1.0, 0.0, 8, 0, 1, None, None) == _lib.ERR_INVALID
    assert lib.fqb200_float2gemmlowp(None, None, 0, 1.0, 0.0, 8, 0, 1, None, None) == _lib.OK  # empty tensor: no-op
    assert lib.fqb200_quantize1(None, None, None, 1, 4, 4, None, None, None, 1, 4, None, 0, None) == _lib.ERR_INVALID
    # the plan query works without a device (it assumes an H100, 132 SMs): channels-last ResNet-50 layer, 3 phases on the
    # bulk ring
    d = _lib.Desc()
    d.outer, d.groups, d.inner, d.num_bits, d.range_mode, d.channels_last = 512, 256, 196, 4, _lib.RANGE_LAPLACE, 1
    out = (ctypes.c_int64 * 8)()
    assert lib.fqb200_plan_info(ctypes.byref(d), out) == _lib.OK
    assert out[0] == 2 and 1 <= out[1] <= 264 and out[5] == 512 and out[7] == 3
    d.groups = 96   # C/4 = 24 does not divide 512: 504 consumer threads take part
    assert lib.fqb200_plan_info(ctypes.byref(d), out) == _lib.OK and out[5] == 504
    d.groups = 6
    assert lib.fqb200_plan_info(ctypes.byref(d), out) == _lib.ERR_UNSUPPORTED


def test_no_cpu_fallback():
    import cnn_quantization_b200 as fq
    p = dict(clipping="no", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=False, bit_alloc_act=False,
             bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    q = fq.int_quantizer("int8", p)
    with pytest.raises(fq._lib.FqError):
        q(torch.zeros(2, 3, 4, 4), "id", "activation")
    with pytest.raises(fq._lib.FqError):
        fq.int_quantization.float2gemmlowp(torch.zeros(8), 1.0, -0.5, 8, False, True, None)


def test_product_never_imports_the_oracle():
    pkg = os.path.join(ROOT, "cnn-quantization_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                text = open(os.path.join(dirpath, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", text, re.M), f
                assert "fq_oracle" not in text.replace("oracle/fq_oracle.py", ""), f
