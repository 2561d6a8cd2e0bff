"""a1 against the REFERENCE's own CUDA extension (kernels/int_quantization.cpp + gemmlowp.cu, unmodified).

What that kernel computes on these inputs is stored under tests/golden/ (tests/golden/make_ref_ext_golden.py: SHA-256
digests of its float2gemmlowp outputs, the levels and indices of its min/max outputs), so the comparison needs no
reference binary.  Where oracle/build_oracle.py has built the extension for this GPU architecture (oracle/_ref/sm_90a/),
the same calls also run live and are compared as well.  This is the strongest pin for the compiled leaf: same inputs, the
reference's kernel vs ours, bit for bit (including the FFMA contraction of the non-true-zero form)."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import golden_inputs as G

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def ref_ext():
    """The reference's compiled extension when it is built for this architecture, else None (golden data only)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import ref_live
    return ref_live.load_extension() if ref_live.ext_path() else None


@pytest.fixture(scope="module")
def f2g_golden():
    with open(os.path.join(GOLD, "ref_ext_float2gemmlowp.json")) as f:
        return json.load(f)


def _digest(t):
    return hashlib.sha256(t.contiguous().cpu().numpy().tobytes()).hexdigest()


@pytest.mark.parametrize("n", G.F2G_SIZES)
@pytest.mark.parametrize("bits", G.F2G_BITS)
def test_float2gemmlowp_bit_exact_vs_reference_kernel(ref_ext, f2g_golden, n, bits):
    import cnn_quantization_b200 as fq
    xn, nn = G.f2g_inputs(n, bits)
    x, noise = torch.from_numpy(xn).cuda(), torch.from_numpy(nn).cuda()
    zeros = torch.zeros_like(x)
    for call in G.F2G_CALLS:
        tz, rng, off = call
        for nz in (zeros, noise):
            got = fq.int_quantization.float2gemmlowp(x, rng, off, bits, False, tz, None if nz is zeros else nz)
            torch.cuda.synchronize()
            assert _digest(got) == f2g_golden[G.f2g_key(n, bits, call, nz is noise)], (tz, rng, off, nz is noise)
            if ref_ext is not None:
                assert torch.equal(got, ref_ext.float2gemmlowp(x, rng, off, bits, False, tz, nz)), (tz, rng, off, nz is noise)
    got = fq.int_quantization.float2gemmlowp(x, 7.3, -3.1, bits, True, True, None)   # int_exp
    assert _digest(got) == f2g_golden[G.f2g_key(n, bits, (True, 7.3, -3.1), False, int_exp=True)]
    if ref_ext is not None:
        assert torch.equal(got, ref_ext.float2gemmlowp(x, 7.3, -3.1, bits, True, True, zeros))
        assert ref_ext.float2gemmlowp(x, 0.0, 0.0, bits, False, True, zeros) is not None  # range <= 0: input returned


def test_minmax_path_vs_reference_kernel_with_reference_host_logic(ref_ext):
    """gemmlowpMinMaxQuantize (int_quantizer.py:361-379, 605-614) with the reference's own kernel as the leaf vs our fused
    launch: the range comes from torch reductions there and from our statistics phase here."""
    import cnn_quantization_b200 as fq
    from test_gpu_parity import params
    gold = np.load(os.path.join(GOLD, "ref_ext_minmax.npz"))
    for i, (shape, tag, positive) in enumerate(G.MINMAX_CASES):
        x = torch.from_numpy(G.minmax_input(i)).cuda()
        want = torch.from_numpy(gold["levels_%d" % i][gold["codes_%d" % i].astype(np.int64)]).cuda()
        delta = float(gold["delta_%d" % i])
        if ref_ext is not None:   # the reference's host logic around its kernel, live
            avg = "activation" in tag and "classifier" not in tag
            t = x.view(x.shape[0], -1) if avg else x.view(-1)
            mn = t.min(-1)[0].mean() if avg else t.min()
            mx = t.max(-1)[0].mean() if avg else t.max()
            if positive:
                mn = 0
            d = mx - mn
            preserve_zero = bool((mn + d) > 0 and mn < 0)
            live = ref_ext.float2gemmlowp(x.contiguous(), float(d), float(mn), 8, False, preserve_zero, torch.zeros_like(x))
            assert torch.equal(live, want), i
        q = fq.int_quantizer("int8", params())
        q.half_range = positive
        got = q(x, "id", tag)
        step = delta / 255
        bad = (got - want).abs() > 1e-5 * want.abs() + 1e-9
        assert float(bad.float().mean()) <= 2e-4
        assert float((got - want).abs().max()) <= step * 1.01
