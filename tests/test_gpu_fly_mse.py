"""`-c mse` on the fly (`-sm no`) on the GPU.

* ops.clip_mse_select against ops.clip_mse on seeded tensors - NCHW and channels-last per channel (among them
  512x2048x7x7 and the 512x64x112x112 ResNet-50 stem) and per tensor; signed and positive; 4 and 8 bits; with and
  without `-baa`; priors laplace and gaus: the sums bit for bit, the choice equal to statistics.best_columns, the given
  parameters and the table equal to clip_mse's parameters at the chosen column bit for bit, crafted ties (repeated
  multipliers, a constant channel) and a NaN channel included; the same bits on every run and for every max_ctas.
* The quantizer: with one multiplier at the ACIQ Laplace factor it is on-the-fly `-c laplace`, bit for bit; on every
  launch route (plain, block epilogue, deferred shortcut, 2x2 and 3x3 pooling, Inception slice write, `-bca`) its output
  is the use-mode apply of the chosen parameters, and every fused route equals its unfused composition.
* Seeded ResNet-50 and Inception-v3 W4A4 forwards: the same logits with every fusion on and off, no host
  synchronisation inside a forward, and nothing cached per forward."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import __graft_entry__
    __graft_entry__.build()


def _bits(t):
    view = {torch.float32: torch.int32, torch.float64: torch.int64}.get(t.dtype)
    return t.contiguous().view(view) if view is not None else t.contiguous()


def _same(a, b):
    """bit-identical (NaN included)"""
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(_bits(a), _bits(b))


def _tensor(shape, seed, cl=False, positive=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    n, c = shape[0], shape[1]
    scale = torch.linspace(0.2, 3.0, c, device="cuda").view(1, c, *([1] * (len(shape) - 2)))
    x = torch.empty(shape, device="cuda").exponential_(generator=g) * scale
    x = x - (0.0 if positive else 0.9 * scale)
    x.view(-1)[:: 997] *= 9.0   # outliers
    return x.contiguous(memory_format=torch.channels_last) if cl else x


def _mults(k, seed=0):
    if k == 125:
        from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
        return torch.tensor(MSE_MULTIPLIERS, dtype=torch.float32, device="cuda")
    g = torch.Generator().manual_seed(seed)
    return (1.0 + 10.0 * torch.rand(k, generator=g)).cuda()


def _table(x, per_channel, cl, bits, positive, baa, prior_b=True):
    from cnn_quantization_b200 import _lib as L, ops
    if not per_channel:
        layout = (1, 1, x.numel())
        return layout, ops.fused(x, layout, stats_only=True, num_bits=bits, positive=positive, any_dense_format=True)
    layout = (x.shape[0], x.shape[1], x.numel() // (x.shape[0] * x.shape[1]))
    return layout, ops.fused(x, layout, stats_only=True, channels_last=cl, num_bits=bits, positive=positive, bit_alloc=baa,
                             bit_alloc_prior=L.PRIOR_B if prior_b else L.PRIOR_STD, bit_alloc_round=True,
                             bit_alloc_target=bits)


def _check_select(x, per_channel, cl, bits, positive, baa, prior, mult, max_ctas=0):
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.statistics import best_columns
    cl = cl and per_channel   # one group reads any dense memory order
    x = x if (cl or not per_channel) else x.contiguous()
    layout, table = _table(x, per_channel, cl, bits, positive, baa)
    alloc = baa and per_channel and bits <= 4
    kw = dict(prior=prior, bit_alloc=alloc, solve_f64=not per_channel)
    sums, params = ops.clip_mse(x, table, layout, cl, bits, positive, mult, want_params=True, **kw)
    got = ops.clip_mse_select(x, table, layout, cl, bits, positive, mult, max_ctas=max_ctas, **kw)
    s, choice, given, chosen = got
    assert _same(s, sums)
    want = torch.from_numpy(best_columns(mult.cpu().numpy(), sums[:, 1:].cpu().numpy()).astype(np.int32))
    assert torch.equal(choice.cpu(), want)
    g = torch.arange(layout[1], device="cuda")
    p = params[g, choice.long()]                    # [G, 6]: delta, offset, bits, scale, zero point, qmax
    assert _same(given, p[:, :3].t().contiguous())
    assert _same(chosen[:, :5], table[:, :5]) and _same(chosen[:, 5:11], p)
    assert torch.all(chosen[:, 11] == 2.0)          # FLAG_TRUE_ZERO of the torch leaf
    return got


# (shape, per channel, channels-last); the large shapes run fewer flag sets
SMALL = [((8, 32, 14, 14), True, False), ((8, 64, 28, 28), True, True), ((6, 24, 9, 11), True, True),
         ((4, 16, 20, 20), False, False), ((4, 16, 20, 20), False, True), ((3, 7, 5, 5), True, False)]
FLAGS = [dict(bits=b, positive=p, baa=a, prior=r) for b in (4, 8) for p in (False, True) for a in (False, True)
         for r in ("laplace", "gaus") if not (a and b == 8)]


@pytest.mark.parametrize("shape,pc,cl", SMALL, ids=["nchw", "cl", "cl-odd", "tensor", "tensor-cl", "nchw-c7"])
def test_select_matches_clip_mse(shape, pc, cl):
    for i, f in enumerate(FLAGS):
        x = _tensor(shape, seed=11 + i, cl=cl, positive=f["positive"])
        _check_select(x, pc, cl, f["bits"], f["positive"], f["baa"], f["prior"], _mults(125 if i % 3 == 0 else 17, seed=i))


@pytest.mark.parametrize("shape,cl,flags", [
    ((512, 2048, 7, 7), True, dict(bits=4, positive=True, baa=True, prior="laplace")),
    ((512, 2048, 7, 7), False, dict(bits=4, positive=False, baa=False, prior="gaus")),
    ((512, 64, 112, 112), True, dict(bits=4, positive=True, baa=True, prior="laplace")),
], ids=["2048-cl", "2048-nchw", "stem-cl"])
def test_select_matches_clip_mse_at_model_sizes(shape, cl, flags):
    x = _tensor(shape, seed=3, cl=cl, positive=flags["positive"])
    _check_select(x, True, cl, flags["bits"], flags["positive"], flags["baa"], flags["prior"], _mults(125))


def test_ties_constant_and_nan_channels():
    x = _tensor((4, 8, 6, 6), seed=5)
    x[:, 2] = 1.5                                    # constant: every candidate has the same error
    x[1, 5, 2, 3] = float("nan")                     # NaN: every sum is NaN, the smallest multiplier wins
    mult = torch.tensor([4.0, 2.0, 4.0, 2.0, 3.0, 9.0], device="cuda")   # repeated multipliers: exact ties
    for cl in (False, True):
        for prior in ("laplace", "gaus"):
            xx = x.contiguous(memory_format=torch.channels_last) if cl else x
            _, choice, _, _ = _check_select(xx, True, cl, 4, False, False, prior, mult)
            assert int(choice[2]) == 1 and int(choice[5]) == 1
            assert all(int(c) not in (2, 3) for c in choice.cpu())   # a repeat never beats its first column
    xt = x.clone()
    xt.view(-1)[7] = float("nan")
    _, choice, _, _ = _check_select(xt, False, False, 4, False, False, "laplace", mult)
    assert int(choice[0]) == 1


def test_deterministic_over_runs_and_ctas():
    for shape, pc, cl in SMALL[:2] + SMALL[3:4]:
        x = _tensor(shape, seed=8, cl=cl)
        ref = _check_select(x, pc, cl, 4, False, True, "laplace", _mults(33))
        for ctas in (0, 1, 7, 300):
            got = _check_select(x, pc, cl, 4, False, True, "laplace", _mults(33), max_ctas=ctas)
            assert all(_same(a, b) for a, b in zip(ref, got))


# ---- the quantizer ---------------------------------------------------------------------------------------------------------
def _q(clipping="mse", pcq=True, bits=4, baa=False, positive=False, bca=False, mult=None, prior="laplace"):
    import cnn_quantization_b200 as fq
    from cnn_quantization_b200.int_quantizer import MseCandidates
    p = dict(clipping=clipping, stats_kind="mean", kld=False, pcq_weights=False, pcq_act=pcq, bit_alloc_act=baa,
             bit_alloc_weight=False, bcorr_act=bca, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="laplace", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    q = fq.int_quantizer("int%d" % bits, p)
    q.half_range = positive
    if mult is not None:
        q.mse_candidates = MseCandidates(mult, prior)
    return q


@pytest.mark.parametrize("bits", [4, 8])
def test_one_multiplier_at_the_laplace_factor_is_aciq(bits):
    from cnn_quantization_b200.int_quantizer import ALPHA_LAPLACE, ALPHA_LAPLACE_POSITIVE
    for positive in (False, True):
        factor = (ALPHA_LAPLACE_POSITIVE if positive else ALPHA_LAPLACE)[bits]
        for shape, pc, cl in SMALL:
            x = _tensor(shape, seed=21, cl=cl, positive=positive)
            lap = _q("laplace", pcq=pc, bits=bits, positive=positive)(x.clone(), "c", "activation")
            mse = _q("mse", pcq=pc, bits=bits, positive=positive, mult=[factor])(x.clone(), "c", "activation")
            assert _same(lap, mse), (shape, pc, cl, positive)


def _use_ref(q_fly, flags, x_seen):
    """A `-sm use` quantizer whose resolved parameters are the ones the on-the-fly call chose (its exported table)."""
    from cnn_quantization_b200.int_quantizer import _UseParams
    t = q_fly.last_stats
    qr = _q("mse", **flags)
    qr.sm = lambda: None
    if q_fly._pc_act(x_seen) and x_seen.shape[1] > 1:
        p = _UseParams(True, t[:, 5].contiguous(), t[:, 6].contiguous(), t[:, 7].contiguous() if flags.get("baa") else None,
                       None)
    else:
        p = _UseParams(False, t[0, 5], t[0, 6], None, None)
    qr._use_params = lambda tensor, stat_id, route: p
    return qr


def _fly(flags, mult):
    q = _q("mse", mult=mult, **flags)
    q.export_stats = True
    return q


@pytest.mark.parametrize("flags", [dict(), dict(positive=True, baa=True), dict(bits=8, positive=True)],
                         ids=["signed", "positive-baa", "int8-positive"])
def test_routes_equal_use_mode_apply_and_unfused(flags):
    mult = _mults(33).cpu().numpy()
    n, c, h, w = 4, 32, 16, 16
    x = _tensor((n, c, h, w), seed=31, cl=True, positive=flags.get("positive", False))
    bias = torch.linspace(-0.5, 0.5, c, device="cuda")
    r = _tensor((n, c, h, w), seed=32, cl=True)

    # plain, with the convolution bias (added first on this route, fused in use mode)
    q = _fly(flags, mult)
    y = q(x.clone(), "c", "activation", bias=bias)
    assert q.last_clip_choice is not None and q._stat_cache == {}
    ref = _use_ref(q, flags, x)(x.clone(), "c", "activation", stat_id="s", bias=bias)
    assert _same(y, ref)
    plain = y

    # block epilogue
    q = _fly(flags, mult)
    y = q(x.clone(), "c", "activation", bias=bias, residual=r)
    assert getattr(y, "_fq_residual_fused", False)
    assert _same(y, _use_ref(q, flags, x)(x.clone(), "c", "activation", stat_id="s", bias=bias, residual=r))
    assert _same(y, torch.relu(plain + r))

    # deferred shortcut, consumed by the block epilogue of another call
    s = _tensor((n, c, h, w), seed=33, cl=True)
    qs = _fly(flags, mult)
    d = qs(s.clone(), "s", "activation", defer=True)
    assert getattr(d, "_fq_deferred", None) is not None and d._fq_deferred[0] is qs.last_stats and qs._stat_cache == {}
    q = _fly(flags, mult)
    y = q(x.clone(), "c", "activation", residual=d)
    assert getattr(y, "_fq_residual_fused", False)
    qs_plain = _fly(flags, mult)(s.clone(), "s", "activation")
    x_plain = _fly(flags, mult)(x.clone(), "c", "activation")
    assert _same(y, torch.relu(x_plain + qs_plain))
    qrs = _use_ref(qs, flags, s)
    dr = qrs(s.clone(), "s", "activation", stat_id="s", defer=True)
    assert _same(y, _use_ref(q, flags, x)(x.clone(), "c", "activation", stat_id="s", residual=dr))

    # pooling inside the launch: 2x2 directly, 3x3 behind a ReLU the caller skips (positive ranges only)
    for pool, ref_pool in (((2, 2, "direct"), lambda t: F.max_pool2d(t, 2)), ((3, 3), lambda t: F.max_pool2d(t, 3, 2, 1))):
        if len(pool) == 2 and not flags.get("positive"):
            continue
        q = _fly(flags, mult)
        y = q(x.clone(), "c", "activation", bias=bias, pool=pool, relu_follows=True)
        assert getattr(y, "_fq_pooled", None) == pool[0]
        assert _same(y, ref_pool(plain))
        yr = _use_ref(q, flags, x)(x.clone(), "c", "activation", stat_id="s", bias=bias, pool=pool, relu_follows=True)
        assert _same(y, yr)

    # an Inception branch writing its channel slice of the block's output
    wide = torch.full((n, c + 8, h, w), float("nan"), device="cuda").contiguous(memory_format=torch.channels_last)
    sl = wide[:, 4:4 + c]
    q = _fly(flags, mult)
    y = q(x.clone(), "c", "activation", bias=bias, out=sl)
    assert y.data_ptr() == sl.data_ptr()
    assert _same(sl.contiguous(), plain.contiguous())
    wide2 = torch.full_like(wide, float("nan"))
    _use_ref(q, flags, x)(x.clone(), "c", "activation", stat_id="s", bias=bias, out=wide2[:, 4:4 + c])
    assert _same(wide, wide2)

    # -bca
    for relu_first in (False, True):
        q = _fly(dict(flags, bca=True), mult)
        y = q(x.clone(), "c", "activation", bias=bias, bias_correct=relu_first)
        ref = _use_ref(q, dict(flags, bca=True), x)(x.clone(), "c", "activation", stat_id="s", bias=bias,
                                                    bias_correct=relu_first)
        assert _same(y, ref)


def test_per_tensor_and_nchw_equal_use_mode_apply():
    mult = _mults(17).cpu().numpy()
    for pcq, cl in ((False, True), (False, False), (True, False)):
        for positive in (False, True):
            flags = dict(pcq=pcq, positive=positive)
            x = _tensor((4, 12, 10, 10), seed=41, cl=cl, positive=positive)
            q = _fly(flags, mult)
            y = q(x.clone(), "c", "activation")
            assert _same(y, _use_ref(q, flags, x)(x.clone(), "c", "activation", stat_id="s"))
            q = _fly(dict(flags, bca=True), mult)
            y = q(x.clone(), "c", "activation", bias_correct=True)
            ref = _use_ref(q, dict(flags, bca=True), x)(x.clone(), "c", "activation", stat_id="s", bias_correct=True)
            assert _same(y, ref)


# ---- whole networks -----------------------------------------------------------------------------------------------------------
def _model(config, hw, fused=True):
    from cnn_quantization_b200 import pipeline
    cfg = dict(pipeline.CONFIGS[config], clipping="mse")
    model, qm = pipeline.build_quantized_model(cfg, "cuda", channels_last=True)
    if not fused:
        qm.fuse_residual_into_quant = qm.defer_shortcut = qm.fuse_pool_into_quant = qm.fuse_inception_concat = False
    x, _ = pipeline.synthetic_batch(2, seed=7, hw=hw, device="cuda", channels_last=True)
    return model, qm, x


def _quantizers(qm):
    return [q for q in list(qm.quantizers.values()) + [qm.quantizer_default] if hasattr(q, "_stat_cache")]


@pytest.mark.parametrize("config,hw", [("resnet50_w4a4", 224), ("inception_v3_w4a4", 299)], ids=["resnet50", "inception_v3"])
def test_network_fused_equals_unfused(config, hw):
    from cnn_quantization_b200 import ops
    outs = []
    for fused in (True, False):
        model, qm, x = _model(config, hw, fused)
        ops.profile_reset(enable=True)
        with torch.no_grad():
            outs.append(model(x))
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
        assert prof["modes"]["R"]["launches"] > 0
        if fused:
            assert sum(v["launches"] for k, v in prof["modes"].items() if k.endswith(("r", "p", "i"))) > 0
        qm.detach()
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1])


def test_forward_without_host_sync_and_without_cache_growth():
    model, qm, x = _model("resnet50_w4a4", 224)
    with torch.no_grad():
        model(x)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            model(x)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        model(x)
    torch.cuda.synchronize()
    qs = [q for q in _quantizers(qm) if q.clipping == "mse"]
    assert qs and all(q.mse_candidates is qm.fly_mse for q in qs)
    assert all(q._stat_cache == {} for q in _quantizers(qm))
    qm.detach()
