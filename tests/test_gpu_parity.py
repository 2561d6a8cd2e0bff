"""GPU parity: the sm_90a kernels (through the C ABI / the drop-in Python API) against the CPU oracle and the
golden fixtures generated from the real reference.

Two-tier protocol (SURVEY.md section 7, "hard parts"):
  (i)  given identical parameters the integer grid and the dequantised output are BIT-EXACT;
  (ii) end to end with on-device statistics: parameters within 1e-5 relative of the reference's (bit widths
       exact), outputs within 1e-5 relative except a bounded fraction of elements that sit on a rounding
       boundary and land one quantization step away.
"""
import json
import os

import numpy as np
import pytest
import torch

from conftest import fq_mismatch
from golden_inputs import regen

pytestmark = pytest.mark.gpu

FLIP_FRAC = 2e-4   # tier (ii): at most this fraction of elements may differ ...
FLIP_STEPS = 1.01  # ... and by at most one quantization step


@pytest.fixture(scope="module")
def fq():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import cnn_quantization_b200 as m
    m._lib.load()
    return m


@pytest.fixture(scope="module")
def O():
    from oracle import fq_oracle
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    return fq_oracle


def params(**over):
    p = dict(clipping="no", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=False, bit_alloc_act=False,
             bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    p.update(over)
    return p


def cuda(x):
    return torch.as_tensor(x).cuda()


def assert_tier2(y, y_ref, step, what):
    frac, worst = fq_mismatch(y, y_ref, step)
    assert frac <= FLIP_FRAC, "%s: %.3g of the elements differ" % (what, frac)
    assert worst <= FLIP_STEPS, "%s: a difference of %.3f steps" % (what, worst)


def _meta():
    with open(os.path.join(os.path.dirname(__file__), "golden", "ref_cpu_meta.json")) as f:
        return json.load(f)


def _names(prefixes):
    return sorted(n for n in _meta() if n.startswith(prefixes))


# ---------------------------------------------------------------------------------------------------
# the exact-division building block
# ---------------------------------------------------------------------------------------------------
def test_division_is_ieee(fq):
    g = torch.Generator(device="cuda").manual_seed(1)
    n = 1 << 24
    for rep in range(8):
        a = torch.randn(n, device="cuda", generator=g) * (10.0 ** torch.randint(-6, 7, (n,), device="cuda", generator=g))
        b = torch.exp(torch.rand(n, device="cuda", generator=g) * 27.6 - 18.4)  # 1e-8 .. 1e4, log-uniform
        if rep % 2:
            # adversarial significands: all-ones / one / near-one mantissas
            bits = b.view(torch.int32)
            pat = torch.tensor([0x7FFFFF, 0x000000, 0x000001, 0x7FFFFE, 0x400000, 0x3FFFFF], device="cuda", dtype=torch.int32)
            sel = pat[torch.randint(0, 6, (n,), device="cuda", generator=g)]
            b = ((bits & ~0x7FFFFF) | sel).view(torch.float32)
        if rep == 7:
            a[:1000] = float("inf")
            a[1000:2000] = float("nan")
            a[2000:3000] = 3e38
            a[3000:4000] = 1e-42
        fast, ieee = fq.ops._test_division(a.contiguous(), b.contiguous())
        # exact wherever a quotient can influence a grid point; below 1e-30 it rounds to zero whatever its last bit
        sane = (ieee.abs() < 1e30) & ((ieee.abs() > 1e-30) | (ieee == 0))
        assert torch.equal(fast[sane], ieee[sane])
        tiny = ieee.abs() <= 1e-30
        assert bool((fast[tiny].abs() <= 2e-30).all())
        big = ~sane & ~torch.isnan(ieee)
        # outside the exact window only sign / hugeness matter (the caller clamps)
        assert bool(((fast[big] > 1e29) == (ieee[big] > 1e29)).all())
        assert bool((torch.isnan(fast) == torch.isnan(ieee)).all())


# ---------------------------------------------------------------------------------------------------
# a1: compiled leaf
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 3, 4, 1023, 4096, 100003, 1 << 20, 1500004, 5000001, 6291456 + 8])
@pytest.mark.parametrize("bits", [2, 4, 8])
def test_a1_float2gemmlowp_matches_oracle(fq, O, n, bits):
    # from 2^20 elements (16-byte aligned, a multiple of 4) the bulk-copy ring kernel runs, the noise tensor through pair
    # stages; 1500004 and 6291464 end on a ragged stage, 5000001 takes the scalar kernel
    rs = np.random.RandomState(n % 100000 + bits)
    x = (rs.standard_normal(n) * 2 + 0.3).astype(np.float32)
    if n >= 4096:
        x[rs.randint(0, n, 6)] = np.array([np.inf, -np.inf, 1e38, -1e38, 0.0, -0.0], np.float32)
    for tz, rng, off in ((True, 7.3, -3.1), (False, 5.0, 0.0), (False, 6.0, 0.5), (True, 9.0, -0.0001), (False, 4.0, -1.0)):
        want = O.float2gemmlowp(x, rng, off, bits, False, tz, None)
        got = fq.int_quantization.float2gemmlowp(cuda(x), rng, off, bits, False, tz, None)
        assert np.array_equal(got.cpu().numpy(), want), (tz, rng, off)
    noise = rs.uniform(-0.5, 0.5, n).astype(np.float32)
    want = O.float2gemmlowp(x, 7.3, -3.1, bits, False, True, noise)
    got = fq.int_quantization.float2gemmlowp(cuda(x), 7.3, -3.1, bits, False, True, cuda(noise))
    assert np.array_equal(got.cpu().numpy(), want)
    want = O.float2gemmlowp(x, 7.3, -3.1, bits, True, True, None)  # int_exp: power-of-two scale
    got = fq.int_quantization.float2gemmlowp(cuda(x), 7.3, -3.1, bits, True, True, None)
    assert np.array_equal(got.cpu().numpy(), want)


def test_a1_edge_cases(fq, O):
    x = cuda(np.array([0.0, -0.0, 1.5, 2.5, -1.5, np.inf, -np.inf, np.nan, 1e38, -1e38, 0.49999997, 0.5], np.float32))
    # range <= 0: the reference returns its input object
    assert fq.int_quantization.float2gemmlowp(x, 0.0, -1.0, 8, False, True, None) is x
    assert fq.int_quantization.float2gemmlowp(x, -2.0, -1.0, 8, False, True, None) is x
    for tz in (True, False):
        want = O.float2gemmlowp(x.cpu().numpy(), 15.0, -7.0 if tz else 0.25, 4, False, tz, None)
        got = fq.int_quantization.float2gemmlowp(x, 15.0, -7.0 if tz else 0.25, 4, False, tz, None).cpu().numpy()
        assert np.array_equal(got, want, equal_nan=True)
    # 0-d tensor scalars, like the reference's callers pass
    y = fq.int_quantization.float2gemmlowp(x, torch.tensor(15.0).cuda(), torch.tensor(-7.0).cuda(), 4, False, True, None)
    assert np.array_equal(y.cpu().numpy(), O.float2gemmlowp(x.cpu().numpy(), 15.0, -7.0, 4, False, True, None), equal_nan=True)
    # empty
    e = torch.empty(0, device="cuda")
    assert fq.int_quantization.float2gemmlowp(e, 1.0, 0.0, 8, False, True, None).numel() == 0
    with pytest.raises(Exception):
        fq.int_quantization.float2gemmlowp(torch.zeros(4), 1.0, 0.0, 8, False, True, None)  # CPU tensor: no fallback


# ---------------------------------------------------------------------------------------------------
# a3: leaf with given parameters - tier (i), bit-exact
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", _names(("leaf_",)))
def test_a3_golden_bit_exact(fq, golden, name):
    arrays, meta = golden
    info = meta[name]
    x = cuda(regen(info["input"]))
    q = fq.int_quantizer("int%d" % info["num_bits"], params())
    delta, offset = cuda(arrays[name + ".delta"]), cuda(arrays[name + ".offset"])
    bits = cuda(arrays[name + ".bits"]) if name + ".bits" in arrays else None
    if info["kind"] == "leaf":
        delta, offset = delta.reshape(()), offset.reshape(())
    y = q.__gemmlowpQuantize1__(x, delta, offset, bit_alloc=bits)
    assert np.array_equal(y.cpu().numpy(), arrays[name + ".y"])


@pytest.mark.parametrize("shape,rows", [((7, 1000), True), ((64, 49), True), ((5, 3, 7, 7), False), ((33, 12544), True),
                                        ((1, 64, 56, 56), False), ((2049,), False)])
def test_a3_random_bit_exact_with_grid(fq, O, shape, rows):
    rs = np.random.RandomState(len(shape) * 17 + shape[0])
    x = (rs.laplace(size=shape) * 1.7).astype(np.float32)
    xt = torch.from_numpy(x)
    for nb in (2, 4, 8):
        if rows:
            t = xt.view(shape[0], -1)
            mn, mx = t.min(-1)[0], t.max(-1)[0]
            bits = torch.from_numpy(rs.randint(0, 9, size=shape[0]).astype(np.float32))
            for b in (None, bits):
                want, wgrid = O.gemmlowp_quantize1(t, mx - mn, mn, nb, bit_alloc=b, return_grid=True)
                got, ggrid = fq.ops.quantize1(cuda(x).view(shape[0], -1), cuda(mx - mn), cuda(mn), nb,
                                              bits=None if b is None else cuda(b), want_grid=True)
                assert np.array_equal(ggrid.cpu().numpy(), wgrid.numpy())  # the integer grid
                assert np.array_equal(got.cpu().numpy(), want.numpy())
        else:
            mn, mx = xt.min(), xt.max()
            want = O.gemmlowp_quantize1(xt, mx - mn, mn, nb)
            got = fq.ops.quantize1(cuda(x), cuda(mx - mn), cuda(mn), nb)
            assert np.array_equal(got.cpu().numpy(), want.numpy())


def test_a3_nchw_layout_given_params(fq, O):
    """Per-channel parameters applied directly on NCHW (no transpose) == the reference's [C, N*HW] formulation."""
    rs = np.random.RandomState(3)
    for shape in ((3, 8, 7, 7), (2, 12, 14, 14), (4, 5, 3, 5)):
        x = rs.standard_normal(shape).astype(np.float32)
        xt = torch.from_numpy(x)
        n, c, h, w = shape
        t = xt.transpose(0, 1).contiguous().view(c, -1)
        mn, mx = t.min(-1)[0], t.max(-1)[0]
        bits = torch.from_numpy(rs.randint(1, 7, size=c).astype(np.float32))
        want = O.gemmlowp_quantize1(t, mx - mn, mn, 4, bit_alloc=bits).view(c, n, h, w).transpose(0, 1).contiguous()
        got = fq.ops.quantize1(cuda(x), cuda(mx - mn), cuda(mn), 4, bits=cuda(bits), layout=(n, c, h * w))
        assert np.array_equal(got.cpu().numpy(), want.numpy())


# ---------------------------------------------------------------------------------------------------
# fused statistics -> parameters -> apply, against the fixtures of the real reference - tier (ii)
# ---------------------------------------------------------------------------------------------------
def _quantizer_for(fq, info):
    p = params(**info["params"])
    q = fq.int_quantizer("int%d" % info["num_bits"], p)
    q.half_range = bool(info.get("half_range"))
    q.force_positive = bool(info.get("force_positive"))
    return q


@pytest.mark.parametrize("name", _names(("act_", "mt_act")))
def test_fused_activation_vs_reference_fixture(fq, golden, name):
    arrays, meta = golden
    info = meta[name]
    x = cuda(regen(info["input"]))
    q = _quantizer_for(fq, info)
    q.pcq_w = False
    y = q(x, "conv1_activation", "activation").cpu().numpy()
    ref = arrays[name + ".y"]
    if name + ".delta" in arrays:
        step = float(np.max(arrays[name + ".delta"])) / 1.0  # >= any per-channel scale
        qmax = 2 ** info["num_bits"] - 1
        step = step / max(qmax, 1) * (2 ** 4 if name + ".bits" in arrays else 1)
    else:
        step = float(np.abs(ref).max()) + 1.0
    assert_tier2(y, ref, step, name)
    assert y.shape == ref.shape


@pytest.mark.parametrize("name", _names(("act_",)))
def test_fused_parameters_vs_reference_fixture(fq, golden, name):
    """The on-device solve (statistics, bit allocation, ACIQ alpha, delta/offset) against what the reference's leaf
    received: delta / offset within 1e-5, bit widths identical."""
    arrays, meta = golden
    info = meta[name]
    p = info["params"]
    x = cuda(regen(info["input"]))
    from cnn_quantization_b200 import _lib as L
    q = _quantizer_for(fq, info)
    positive = q._positive()
    clip = p.get("clipping", "no")
    pc = q._pc_act(x) and x.shape[1] > 1
    kw = dict(leaf=L.LEAF_TORCH, num_bits=info["num_bits"], positive=positive, want_stats=True)
    if clip != "no":
        mode, k = q._range_mode(clip)
        kw.update(range_mode=mode, clip_k=k)
    if pc:
        kw.update(bit_alloc=p.get("bit_alloc_act", False), bit_alloc_prior=q._prior(), bit_alloc_round=q.bit_alloc_round,
                  bit_alloc_target=q.bit_alloc_target_act)
        layout = (x.shape[0], x.shape[1], x.numel() // (x.shape[0] * x.shape[1]))
    else:
        kw.update(solve_f64=True)
        layout = (1, 1, x.numel())
    _, st = fq.ops.fused(x, layout, **kw)
    st = st.cpu().numpy()
    want_delta, want_off = arrays[name + ".delta"], arrays[name + ".offset"]
    assert np.allclose(st[:, 5], np.broadcast_to(want_delta, st[:, 5].shape), rtol=1e-5, atol=1e-7), name
    assert np.allclose(st[:, 6], np.broadcast_to(want_off, st[:, 6].shape), rtol=1e-5, atol=1e-6), name
    if name + ".bits" in arrays:
        assert np.array_equal(st[:, 7], arrays[name + ".bits"]), name


@pytest.mark.parametrize("name", _names(("w_", "mt_w")))
def test_fused_weights_vs_reference_fixture(fq, golden, name):
    arrays, meta = golden
    info = meta[name]
    w = cuda(regen(info["input"]))
    q = _quantizer_for(fq, info)
    q.pcq_a = False
    q.clipping = "no"
    ov = ("num_bits", info["override_num_bits"]) if info.get("override_num_bits") else None
    y = q(w, "w", "weight", override_att=ov).cpu().numpy()
    ref = arrays[name + ".y"]
    step = float(np.abs(ref).max())
    assert_tier2(y, ref, step, name)
    assert q.num_bits == info["num_bits"]  # override restored


def test_statistics_helpers_vs_reference_fixture(fq, golden):
    arrays, _ = golden
    x = cuda(regen(dict(seed=4000, shape=(6, 10, 5, 7))))
    names = ["min", "max", "mean", "b", "std"]
    IQ = fq.IntQuantizer
    for pre, st in (("tensor", IQ.__act_stats__(x, names)), ("sampleavg", IQ.__act_stats__(x, names, True)),
                    ("pc", IQ.__act_stats_perchannel__(x, names)), ("pcavg", IQ.__act_stats_perchannel__(x, names, True))):
        for k in names:
            got = st[k].cpu().numpy().reshape(-1)
            want = arrays["stats.%s.%s" % (pre, k)].reshape(-1)
            assert np.allclose(got, want, rtol=2e-6, atol=1e-7), (pre, k, np.abs(got - want).max())


# ---------------------------------------------------------------------------------------------------
# a11: per-tensor min/max through the compiled leaf (W8A8 config; pooling / classifier tensors everywhere)
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(4, 16, 14, 14), (8, 1000), (3, 5, 7, 7), (2, 64, 56, 56)])
@pytest.mark.parametrize("tag,positive,relu", [("activation", False, False), ("activation", True, True),
                                               ("activation_pooling", False, True), ("activation_classifier", False, False),
                                               ("weight", False, False)])
def test_a11_minmax_vs_oracle(fq, O, shape, tag, positive, relu):
    x = regen(dict(seed=sum(shape), shape=shape, relu=relu))
    for nb in (8, 4):
        want, parts = O.minmax_quantize(torch.from_numpy(x), nb, tag, positive, return_parts=True)
        q = fq.int_quantizer("int%d" % nb, params())
        q.half_range = positive
        got = q(cuda(x), "id", tag).cpu().numpy()
        step = float(parts["delta"]) / (2 ** nb - 1)
        assert_tier2(got, want.numpy(), step, "%s %s" % (tag, shape))


def test_a11_degenerate_range_passes_input_through(fq):
    x = torch.full((2, 3, 4, 4), 1.25, device="cuda")
    q = fq.int_quantizer("int8", params())
    assert torch.equal(q(x, "id", "weight"), x)           # max == min -> range 0 -> input returned
    z = torch.zeros(2, 3, 4, 4, device="cuda")
    q.half_range = True
    assert torch.equal(q(z, "id", "activation"), z)


# ---------------------------------------------------------------------------------------------------
# a13: weight bias / variance correction fused into the weight launch
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(16, 8, 3, 3), (10, 64), (8, 3, 7, 7), (64, 147)])
@pytest.mark.parametrize("bc,vc", [(True, False), (True, True), (False, True)])
@pytest.mark.parametrize("pcq", [True, False])
def test_a13_weight_correction_vs_oracle(fq, O, shape, bc, vc, pcq):
    w = (regen(dict(seed=shape[0] * 3 + shape[1], shape=shape)) * 0.05).astype(np.float32)
    wt = torch.from_numpy(w)
    if pcq:
        wq = O.quantize_weights_per_channel(wt, 4, bit_alloc_weight=True)
    else:
        wq = O.minmax_quantize(wt, 4, "weight", False)
    want = O.weight_correction(wt, wq, bc, vc).numpy()
    q = fq.int_quantizer("int4", params(pcq_weights=pcq, bit_alloc_weight=True, bcorr_weight=bc, vcorr_weight=vc))
    q.pcq_a = False
    got = q(cuda(w), "w", "weight", weight_correction=(bc, vc)).cpu().numpy()
    step = float(np.abs(w).max())
    # corrected weights are differences of nearly equal numbers: 1e-5 relative to the weight scale
    frac, worst = fq_mismatch(got, want, step, atol=1e-5 * step)
    assert frac <= 5e-3 and worst <= 1.01, (frac, worst)
    # property: the corrected rows have the original row means
    if bc:
        assert np.allclose(got.reshape(shape[0], -1).mean(-1), w.reshape(shape[0], -1).mean(-1), atol=2e-7)


# ---------------------------------------------------------------------------------------------------
# layout / size coverage and size-independent properties
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(1, 1, 2, 2), (1, 3, 1, 5), (2, 4, 1, 1), (5, 7, 3, 3), (3, 2, 49, 1), (16, 64, 7, 7),
                                   (8, 32, 28, 28), (2, 3, 225, 225)])
def test_fused_laplace_vs_oracle_shapes(fq, O, shape):
    x = regen(dict(seed=sum(shape) + 1, shape=shape, dist="laplace"))
    for hr in (False, True):
        kw = dict(clipping="laplace", pcq_act=True, bit_alloc_act=True)
        q = fq.int_quantizer("int4", params(**kw))
        q.pcq_w = False
        q.half_range = hr
        got = q(cuda(x), "c", "activation").cpu().numpy()
        want, parts = O.clipping_quantize(torch.from_numpy(x), 4, "laplace", True, hr, True, "gaus", None, True,
                                          return_parts=True)
        step = float(torch.as_tensor(parts["delta"]).max()) + 1e-6
        frac, worst = fq_mismatch(got, want.numpy(), step)
        assert frac <= max(FLIP_FRAC, 2.0 / x.size) and worst <= 1.01, (shape, hr, frac, worst)


def test_fused_noncontiguous_and_inplace_and_determinism(fq):
    torch.manual_seed(0)
    base = torch.randn(6, 20, 14, 14, device="cuda")
    q = fq.int_quantizer("int4", params(clipping="laplace", pcq_act=True, bit_alloc_act=True))
    q.pcq_w = False
    nc = base.transpose(2, 3)  # non-contiguous view: the wrapper makes it contiguous like the reference (:352)
    y1 = q(nc, "c", "activation")
    y2 = q(nc.contiguous(), "c", "activation")
    assert torch.equal(y1, y2)
    y3 = q(nc.contiguous(), "c", "activation")
    assert torch.equal(y2, y3)  # deterministic: fixed reduction order
    from cnn_quantization_b200 import _lib as L
    xin = base.clone()
    out = fq.ops.fused(xin, (6, 20, 196), range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True, out=xin)
    assert out.data_ptr() == xin.data_ptr()
    assert torch.equal(out, q(base, "c", "activation"))


@pytest.mark.parametrize("shape", [(16, 64, 7, 7), (5, 12, 7, 7), (9, 8, 3, 3), (4, 6, 5, 5), (7, 16, 9, 5), (3, 4, 11, 2), (64, 256, 7, 7)])
def test_bundled_layout_matches_scalar_path_and_oracle(fq, O, shape):
    """H*W not a multiple of 4: channels are walked in bundles of 2/4 with 128-bit accesses.  Same results as the
    scalar walk of the same data (forced by a 4-byte-misaligned view) and as the oracle."""
    from cnn_quantization_b200 import _lib as L
    x = regen(dict(seed=sum(shape) + 5, shape=shape, dist="laplace"))
    xt = torch.from_numpy(x)
    n, c = shape[0], shape[1]
    hw = x.size // (n * c)
    lay = (n, c, hw)
    xa = cuda(x)
    pad = torch.empty(x.size + 1, device="cuda")
    xm = pad[1:].view(shape)  # same values, base pointer off by 4 bytes -> scalar mode
    xm.copy_(xa)
    bias = torch.randn(c, device="cuda")
    for kw in (dict(range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True), dict(range_mode=L.RANGE_LAPLACE, num_bits=4, positive=True),
               dict(range_mode=L.RANGE_MINMAX, num_bits=4), dict(range_mode=L.RANGE_GAUS, num_bits=3),
               dict(leaf=L.LEAF_MIDTREAD, mt_target=4.0, mt_clip=True)):
        for b in (None, bias):
            y4, s4 = fq.ops.fused(xa, lay, want_stats=True, bias=b, **kw)
            y1, s1 = fq.ops.fused(xm, lay, want_stats=True, bias=b, **kw)
            assert torch.allclose(s4[:, :7], s1[:, :7], rtol=2e-6, atol=1e-6), (shape, kw)
            assert torch.equal(s4[:, 7], s1[:, 7])  # bit widths
            step = float(s4[:, 8].max()) + 1e-9
            frac, worst = fq_mismatch(y4.cpu().numpy(), y1.cpu().numpy(), step)
            assert frac <= max(FLIP_FRAC, 2.0 / x.size) and worst <= 1.01, (shape, kw, frac, worst)
    want, parts = O.clipping_quantize(xt, 4, "laplace", True, False, True, "gaus", None, True, return_parts=True)
    got = fq.ops.fused(xa, lay, range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True)
    step = float(torch.as_tensor(parts["delta"]).max()) + 1e-6
    frac, worst = fq_mismatch(got.cpu().numpy(), want.numpy(), step)
    assert frac <= max(FLIP_FRAC, 2.0 / x.size) and worst <= 1.01, (shape, frac, worst)


@pytest.mark.parametrize("shape", [(6, 64, 14, 14), (3, 16, 7, 7), (5, 8, 3, 5), (2, 256, 6, 6), (4, 2048, 2, 2), (9, 4, 5, 5), (16, 128, 28, 28)])
def test_channels_last_matches_nchw(fq, shape):
    """The same activation stored NHWC goes through the channels-last kernels: same statistics, same grid."""
    from cnn_quantization_b200 import _lib as L
    x = cuda(regen(dict(seed=sum(shape) + 9, shape=shape, dist="laplace")))
    xcl = x.contiguous(memory_format=torch.channels_last)
    n, c = shape[0], shape[1]
    lay = (n, c, shape[2] * shape[3])
    bias = torch.randn(c, device="cuda")
    for kw in (dict(range_mode=L.RANGE_LAPLACE, num_bits=4, bit_alloc=True), dict(range_mode=L.RANGE_LAPLACE, num_bits=4, positive=True, bit_alloc=True),
               dict(range_mode=L.RANGE_MINMAX, num_bits=4), dict(range_mode=L.RANGE_GAUS, num_bits=3),
               dict(leaf=L.LEAF_MIDTREAD, mt_target=4.0, mt_clip=True)):
        for b in (None, bias):
            y0, s0 = fq.ops.fused(x, lay, want_stats=True, bias=b, **kw)
            y1, s1 = fq.ops.fused(xcl, lay, want_stats=True, bias=b, channels_last=True, **kw)
            assert y1.is_contiguous(memory_format=torch.channels_last) and y1.shape == x.shape
            # min, max, mean, delta, offset always; b / std where the range mode consumes them (the NCHW kernel leaves them
            # at 0 when it skips its second pass, the channels-last kernel gets the std out of the first one)
            cols = [0, 1, 2, 5, 6] + ([3, 4] if kw.get("range_mode") in (L.RANGE_LAPLACE, L.RANGE_GAUS) or "leaf" in kw else [])
            assert torch.allclose(s0[:, cols], s1[:, cols], rtol=2e-6, atol=1e-6), (shape, kw)
            assert torch.equal(s0[:, 7], s1[:, 7])
            step = float(s0[:, 8].max()) + 1e-9
            frac, worst = fq_mismatch(y1.cpu().numpy(), y0.cpu().numpy(), step)
            assert frac <= max(FLIP_FRAC, 2.0 / x.numel()) and worst <= 1.01, (shape, kw, frac, worst)
    # through the quantizer: dispatch on the memory format, in place, entropy histogram, back-to-back launches (the
    # per-channel atomic accumulators must be left zeroed)
    q = fq.int_quantizer("int4", params(clipping="laplace", pcq_act=True, bit_alloc_act=True, measure_entropy=True))
    q.pcq_w = False
    a = q(x, "c", "activation")
    e0 = float(q.last_entropy)
    for _ in range(3):
        b_ = q(xcl.clone(), "c", "activation")
    assert b_.is_contiguous(memory_format=torch.channels_last)
    frac, worst = fq_mismatch(b_.cpu().numpy(), a.cpu().numpy(), float(a.abs().max()))
    assert frac <= max(FLIP_FRAC, 2.0 / x.numel())
    assert abs(float(q.last_entropy) - e0) < 2e-3
    q8 = fq.int_quantizer("int8", params())  # per-sample min/max: any dense format, no copy
    q8.inplace = True
    buf = xcl.clone()
    r = q8(buf, "p", "activation_pooling")
    assert r.data_ptr() == buf.data_ptr()
    assert torch.allclose(r, fq.int_quantizer("int8", params())(x, "p", "activation_pooling"), atol=1e-6)


def test_fused_bias_operand_and_inplace_flag(fq):
    """x + bias[c] inside the kernel == quantizing the tensor the convolution would have produced with its bias,
    bit for bit, for every per-channel path; the in-place flag returns the same values in the caller's buffer."""
    torch.manual_seed(3)
    for shape in ((6, 20, 14, 14), (5, 12, 7, 7), (3, 8, 5, 6)):
        x = torch.randn(*shape, device="cuda") * 1.5
        b = torch.randn(shape[1], device="cuda")
        for kw in (dict(clipping="laplace", pcq_act=True, bit_alloc_act=True), dict(pcq_act=True),
                   dict(clipping="gaus", pcq_act=True), dict(clipping="laplace", pcq_act=True, mtd_quant=True)):
            for hr in (False, True):
                q = fq.int_quantizer("int4", params(**kw))
                q.pcq_w = False
                q.half_range = hr
                want = q(x + b.view(1, -1, 1, 1), "c", "activation")
                got = q(x, "c", "activation", bias=b)
                assert torch.equal(got, want), (shape, kw, hr)
                q.inplace = True
                buf = x.clone()
                got2 = q(buf, "c", "activation", bias=b)
                assert got2.data_ptr() == buf.data_ptr() and torch.equal(got2, want)
    # per-tensor / per-sample min-max layouts: the bias is indexed by the channel inside the row (bias_period = H*W) ...
    q = fq.int_quantizer("int8", params())
    for shape in ((4, 6, 4, 4), (3, 64, 14, 14), (2, 5, 6, 2)):
        x = torch.randn(*shape, device="cuda")
        b = torch.randn(shape[1], device="cuda")
        for tag, hr in (("activation", False), ("activation", True), ("activation_classifier", False)):
            q.half_range = hr
            assert torch.equal(q(x, "c", tag, bias=b), q(x + b.view(1, -1, 1, 1), "c", tag)), (shape, tag, hr)
    q.half_range = False
    # ... and where H*W is not a multiple of 4 the bias is added first
    x = torch.randn(4, 6, 5, 5, device="cuda")
    b = torch.randn(6, device="cuda")
    assert torch.equal(q(x, "c", "activation", bias=b), q(x + b.view(1, -1, 1, 1), "c", "activation"))


def test_entropy_measurement_matches_reference_definition(fq, O):
    """`-me`: Shannon entropy of the integer grid (utils/entropy.py:6-17 on output.int()), here from the fused 256-bin
    histogram instead of torch.unique over the tensor."""
    class Log(object):
        def __init__(self):
            self.rows = []

        def log_metric(self, name, value, step=None, meterId=None, weight=None):
            self.rows.append((name, value, meterId, weight))

    def shannon(grid):
        pk = torch.unique(grid.flatten().int(), return_counts=True)[1].float()
        p = pk / pk.sum()
        return float(-(p * torch.log2(p)).sum())

    for shape in ((6, 16, 14, 14), (5, 8, 7, 7)):
        x = regen(dict(seed=sum(shape), shape=shape, dist="laplace"))
        xt = torch.from_numpy(x)
        log = Log()
        q = fq.int_quantizer("int4", params(clipping="laplace", pcq_act=True, bit_alloc_act=True, measure_entropy=True, logger=log))
        q.pcq_w = False
        y = q(cuda(x), "conv3_activation", "activation")
        _, parts = O.clipping_quantize(xt, 4, "laplace", True, False, True, "gaus", None, True, return_parts=True)
        n, c = shape[0], shape[1]
        t = xt.transpose(0, 1).contiguous().view(c, -1)
        _, grid = O.gemmlowp_quantize1(t, parts["delta"], parts["offset"], 4, bit_alloc=parts["bits"], return_grid=True)
        want = shannon(grid)
        assert len(log.rows) == 1 and log.rows[0][0] == "conv3_activation.entropy" and log.rows[0][2] == "avg.entropy.act"
        assert log.rows[0][3] == x.size and abs(log.rows[0][1] - want) < 2e-3, (log.rows, want)
        assert 0 < want < 4.5
    # weights, and the compatibility path of the leaf itself
    w = (regen(dict(seed=9, shape=(16, 8, 3, 3))) * 0.05).astype(np.float32)
    log = Log()
    q = fq.int_quantizer("int4", params(pcq_weights=True, bit_alloc_weight=True, measure_entropy=True, logger=log))
    q.pcq_a = False
    q(cuda(w), "layer1.0.conv1.weight", "weight")
    wt = torch.from_numpy(w).view(16, -1)
    _, parts = O.quantize_weights_per_channel(torch.from_numpy(w), 4, True, return_parts=True)
    _, grid = O.gemmlowp_quantize1(wt, parts["delta"], parts["offset"], 4, bit_alloc=parts["bits"], return_grid=True)
    assert abs(log.rows[0][1] - shannon(grid)) < 2e-3 and log.rows[0][2] == "avg.entropy.weight"
    out, ent = q.__gemmlowpQuantize1__(cuda(w).view(16, -1), cuda(parts["delta"]), cuda(parts["offset"]), bit_alloc=cuda(parts["bits"]),
                                       measure_entropy=True)
    assert abs(float(ent) - shannon(grid)) < 1e-5


def test_full_size_properties(fq):
    """ResNet-50 sized activation (config 3, batch 64 slice): per-channel level count, range, idempotence of the grid."""
    torch.manual_seed(1)
    n, c, h = 64, 256, 56
    x = torch.randn(n, c, h, h, device="cuda") * torch.linspace(0.2, 3.0, c, device="cuda").view(1, c, 1, 1)
    x = torch.relu(x)
    from cnn_quantization_b200 import _lib as L
    y, st = fq.ops.fused(x, (n, c, h * h), range_mode=L.RANGE_LAPLACE, num_bits=4, positive=True, bit_alloc=True,
                         want_stats=True)
    bits, delta, offset = st[:, 7], st[:, 5], st[:, 6]
    assert abs(float(bits.mean()) - 4.0) < 0.05 and bits.min() >= 0 and bits.max() <= 8
    yc = y.transpose(0, 1).reshape(c, -1)
    assert bool((yc.min(-1)[0] >= offset - 1e-6).all())
    assert bool((yc.max(-1)[0] <= offset + delta * (1 + 1e-5)).all())
    for ch in (0, 17, 255):
        assert torch.unique(yc[ch]).numel() <= 2 ** int(bits[ch])
    # re-quantizing the output with the same parameters reproduces it bit for bit
    y2 = fq.ops.quantize1(y, delta.contiguous(), offset.contiguous(), 4, bits=bits.contiguous(), layout=(n, c, h * h))
    assert torch.equal(y, y2)
    # error is bounded by half a step inside the clipping range
    scale = st[:, 8].view(1, c, 1, 1)
    inside = (x >= offset.view(1, c, 1, 1)) & (x <= (offset + delta).view(1, c, 1, 1))
    assert bool((((y - x).abs() <= 0.5 * scale * 1.0001 + 1e-7) | ~inside).all())


def test_api_surface_matches_reference(fq):
    q = fq.int_quantizer("int4", params(clipping="laplace", pcq_act=True))
    assert q.num_bits == 4 and repr(q).startswith("IntQuantizer - [bits: 4, clipping: laplace")
    for attr in ("num_bits", "clipping", "kld", "pcq_w", "pcq_a", "sm", "stats_kind", "measure_entropy", "force_positive",
                 "half_range", "bit_alloc_act", "bit_alloc_weight", "alpha_laplace", "alpha_gaus"):
        assert hasattr(q, attr)
    for meth in ("gemmlowpClippingQuantize", "gemmlowpMinMaxQuantize", "gemmlowpQuantizeActivationPerChannel",
                 "gemmlowpQuantizeWeightsPerChannel", "mid_tread_quantization", "get_alpha", "alpha2DeltaOffset",
                 "get_bits_alloc", "get_bits_alloc_fixed_target", "get_omega", "get_alpha_mult",
                 "__gemmlowpQuantize1__", "__gemmlowpQuantize__", "__act_stats__", "__act_stats_perchannel__"):
        assert hasattr(q, meth), meth
    with pytest.raises(RuntimeError):  # offline statistics need a statistics manager on the quantizer
        q(torch.zeros(1, 2, 3, 3, device="cuda"), "id", "activation", stat_id="conv0_activation")
    with pytest.raises(KeyError):
        fq.int_quantizer("int4", {"clipping": "no"})  # the reference requires the other 14 keys too
