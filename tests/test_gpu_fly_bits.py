"""`-baa -bap mse` on the fly (`-sm no`, fly_bits) on the GPU.

* The allocator: fqb200_allocate_widths and fqb200_allocate_select (M = 1) give bit_alloc.allocate's widths bit for bit
  on random, tied and constant tables, G in {1, 3, 64, 2048, 4096}, targets {0, 0.5, 2, 4, 5.3, 8} (budgets under 8
  channels among them); the status flag on NaN / inf.
* ops.allocate_select: with M = 1 the widths are allocate(sums[:, 1:]) and given / table the gathered clip_mse
  parameters; with M > 1 (clip_mse_grid) each width's column is statistics.best_columns' and the widths allocate's over
  the per-width least sums; the same bits on every run.
* The quantizer: on every launch route (plain, block epilogue, deferred shortcut, pooling, Inception slice write), NCHW
  and channels-last, up to the 512x64x112x112 stem, the output equals ops.quantize1 at the gathered parameters and the
  unfused composition, on every run and for every max_ctas; the measured error at the fly_bits widths is never above the
  error at the analytic alpha^(2/3) widths.
* Seeded ResNet-50 and Inception-v3 W4A4 forwards under fly_bits (`-c laplace`, and `-c mse` with a few multipliers): the
  same logits with every fusion on and off, no host synchronisation inside a forward, nothing cached per forward."""
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


def _tables(g, seed):
    rs = np.random.RandomState(seed)
    rand = np.sort(rs.gamma(0.5, 1.0, (g, 9)), 1)[:, ::-1] * rs.uniform(0.1, 10.0, (g, 1))
    tied = rs.randint(0, 4, (g, 9)).astype(np.float64)
    const = np.ones((g, 9))
    return {"random": np.ascontiguousarray(rand), "tied": tied, "constant": const}


def _select_m1(sse, target):
    """fqb200_allocate_select over a [G, 9] table, as the M = 1 sums of clip_mse with widths 0..8."""
    from cnn_quantization_b200 import ops
    g = sse.shape[0]
    sums = torch.cat([torch.zeros(g, 1, dtype=torch.float64, device="cuda"), sse], 1)
    params = torch.arange(g * 9 * 6, dtype=torch.float32, device="cuda").view(g, 9, 6)
    return ops.allocate_select(sums, params, torch.zeros(g, 12, device="cuda"), target)


TARGETS = [0, 0.5, 2, 4, 5.3, 8]


@pytest.mark.parametrize("g", [1, 3, 64, 2048, 4096])
def test_both_entries_match_allocate(g):
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.bit_alloc import allocate
    targets = TARGETS if g <= 2048 else [0.5, 4, 5.3]
    for name, t in _tables(g, seed=g).items():
        td = torch.from_numpy(t).cuda()
        for target in targets:
            want = allocate(t, target).astype(np.float32)
            got = ops.allocate_widths(td, target).cpu().numpy()
            np.testing.assert_array_equal(got, want, err_msg="%s G=%d target=%r" % (name, g, target))
            got = _select_m1(td, target)[0].cpu().numpy()
            np.testing.assert_array_equal(got, want, err_msg="select %s G=%d target=%r" % (name, g, target))


def test_budgets_under_eight():
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.bit_alloc import allocate
    for g in (1, 2, 3, 5, 7):
        for name, t in _tables(g, seed=100 + g).items():
            for target in (0.2, 0.5, 1.0, 1.5, 2.9):
                want = allocate(t, target).astype(np.float32)
                td = torch.from_numpy(t).cuda()
                np.testing.assert_array_equal(ops.allocate_widths(td, target).cpu().numpy(), want, err_msg=name)
                np.testing.assert_array_equal(_select_m1(td, target)[0].cpu().numpy(), want, err_msg=name)


def test_status_on_non_finite():
    from cnn_quantization_b200 import ops
    for bad in (float("nan"), float("inf")):
        t = torch.from_numpy(_tables(16, seed=3)["random"]).cuda()
        t[5, 3] = bad
        status = torch.zeros(1, dtype=torch.int32, device="cuda")
        ops.allocate_widths(t, 4, status)
        assert int(status) == 1
        sums = torch.cat([torch.zeros(16, 1, dtype=torch.float64, device="cuda"), t], 1)
        status.zero_()
        ops.allocate_select(sums, torch.zeros(16, 9, 6, device="cuda"), torch.zeros(16, 12, device="cuda"), 4,
                            status=status)
        assert int(status) == 1
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    ops.allocate_widths(torch.from_numpy(_tables(16, seed=3)["random"]).cuda(), 4, status)
    assert int(status) == 0


# ---- allocate_select on real candidate tables ------------------------------------------------------------------------------
def _tensor(shape, seed, cl=False, positive=False):
    g = torch.Generator(device="cuda").manual_seed(seed)
    n, c = shape[0], shape[1]
    scale = torch.linspace(0.2, 3.0, c, device="cuda").view(1, c, *([1] * (len(shape) - 2)))
    x = torch.empty(shape, device="cuda").exponential_(generator=g) * scale
    x = x - (0.0 if positive else 0.9 * scale)
    x.view(-1)[:: 997] *= 9.0   # outliers
    return x.contiguous(memory_format=torch.channels_last) if cl else x


def _stats(x, cl):
    from cnn_quantization_b200 import ops
    layout = (x.shape[0], x.shape[1], x.numel() // (x.shape[0] * x.shape[1]))
    return layout, ops.fused(x, layout, stats_only=True, channels_last=cl, num_bits=8)


def _check_m1(x, cl, rule, positive, target):
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.statistics import bit_candidates
    layout, table = _stats(x, cl)
    mult, prior = bit_candidates(rule, positive, 4)
    sums, params = ops.clip_mse(x, table, layout, cl, 4, positive, mult, prior=prior, widths=range(9), solve_f64=False,
                                want_params=True)
    got = ops.allocate_select(sums, params, table, target)
    widths, choice, given, chosen = got
    assert choice is None
    want = allocate(sums[:, 1:].cpu().numpy(), target)
    np.testing.assert_array_equal(widths.cpu().numpy(), want.astype(np.float32))
    p = params[torch.arange(layout[1], device="cuda"), torch.from_numpy(want).cuda()]
    assert _same(given, p[:, :3].t().contiguous())
    assert _same(chosen[:, :5], table[:, :5]) and _same(chosen[:, 5:11], p)
    assert torch.all(chosen[:, 11] == 2.0)   # FLAG_TRUE_ZERO of the torch leaf
    return got


@pytest.mark.parametrize("rule", ["laplace", "gaus", "no"])
@pytest.mark.parametrize("positive", [False, True])
def test_select_m1(rule, positive):
    for shape, cl in (((8, 32, 14, 14), False), ((8, 64, 28, 28), True), ((4, 12, 9, 11), False)):
        x = _tensor(shape, seed=7, cl=cl, positive=positive)
        for target in (2, 4, 5.3):
            _check_m1(x, cl, rule, positive, target)


def test_select_grid():
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.statistics import best_columns
    mult = torch.tensor([4.0, 2.0, 4.0, 2.5, 3.0, 9.0, 1.5], device="cuda")   # a repeat: exact ties
    for shape, cl, positive in (((8, 32, 14, 14), False, False), ((8, 64, 28, 28), True, True)):
        x = _tensor(shape, seed=9, cl=cl, positive=positive)
        x[:, 3] = 1.5   # a constant channel: every candidate ties
        layout, table = _stats(x, cl)
        sums, params = ops.clip_mse_grid(x, table, layout, cl, 4, positive, mult, range(9), solve_f64=False,
                                         want_params=True)
        widths, choice, given, chosen = ops.allocate_select(sums, params, table, 4, multipliers=mult)
        grid = sums[:, 1:].cpu().numpy().reshape(layout[1], 9, -1)
        cols = np.stack([best_columns(mult.cpu().numpy(), grid[:, w]) for w in range(9)], 1)
        least = np.take_along_axis(grid, cols[:, :, None], 2)[:, :, 0]
        want = allocate(least, 4)
        np.testing.assert_array_equal(widths.cpu().numpy(), want.astype(np.float32))
        g = np.arange(layout[1])
        np.testing.assert_array_equal(choice.cpu().numpy(), cols[g, want])
        p = params[torch.from_numpy(g).cuda(), torch.from_numpy(want * mult.numel() + cols[g, want]).cuda()]
        assert _same(given, p[:, :3].t().contiguous()) and _same(chosen[:, 5:11], p)
        again = ops.allocate_select(sums, params, table, 4, multipliers=mult)
        assert all(_same(a, b) for a, b in zip((widths, choice, given, chosen), again))


def test_select_deterministic():
    x = _tensor((8, 64, 28, 28), seed=4, cl=True)
    ref = _check_m1(x, True, "laplace", False, 4)
    for _ in range(3):
        got = _check_m1(x, True, "laplace", False, 4)
        assert all(_same(a, b) for a, b in zip(ref[::2] + ref[3:], got[::2] + got[3:]))


# ---- the quantizer ---------------------------------------------------------------------------------------------------------
def _q(clipping="laplace", positive=False, bca=False, mult=None, target=None):
    import cnn_quantization_b200 as fq
    from cnn_quantization_b200.int_quantizer import MseCandidates
    p = dict(clipping=clipping, stats_kind="mean", kld=False, pcq_weights=False, pcq_act=True, bit_alloc_act=True,
             bit_alloc_weight=False, bcorr_act=bca, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="mse", bit_alloc_target_act=target, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    q = fq.int_quantizer("int4", p)
    q.half_range = positive
    q.fly_bits = True
    q.export_stats = True
    if mult is not None:
        q.mse_candidates = MseCandidates(mult, "laplace")
    return q


def _applied(q, x, bias=None):
    """ops.quantize1 at the parameters the quantizer's last call gathered (its exported table)."""
    from cnn_quantization_b200 import ops
    t = q.last_stats
    xb = x if bias is None else x + bias.view(1, -1, 1, 1)
    return ops.quantize1(xb, t[:, 5].contiguous(), t[:, 6].contiguous(), 4, bits=t[:, 7].contiguous(),
                         layout=(x.shape[0], x.shape[1], x.numel() // (x.shape[0] * x.shape[1])))


@pytest.mark.parametrize("clipping", ["laplace", "gaus", "no", "mse"])
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "cl"])
def test_routes_equal_quantize1_and_unfused(clipping, cl):
    mult = [2.0, 3.0, 4.5] if clipping == "mse" else None
    positive = clipping != "gaus"
    n, c, h, w = 4, 32, 16, 16
    x = _tensor((n, c, h, w), seed=31, cl=cl, positive=positive)
    bias = torch.linspace(-0.5, 0.5, c, device="cuda")
    r = _tensor((n, c, h, w), seed=32, cl=cl)

    q = _q(clipping, positive, mult=mult)
    plain = q(x.clone(), "c", "activation", bias=bias)
    assert q._stat_cache == {} and (q.last_clip_choice is not None) == (clipping == "mse")
    assert _same(plain, _applied(q, x, bias))
    widths = q.last_stats[:, 7].clone()
    assert float(widths.sum()) <= 4 * c

    # block epilogue
    y = _q(clipping, positive, mult=mult)(x.clone(), "c", "activation", bias=bias, residual=r)
    assert getattr(y, "_fq_residual_fused", False) == cl
    if not cl:   # NCHW launches leave the block's add and ReLU to the caller
        y = torch.relu(y + r)
    assert _same(y, torch.relu(plain + r))

    # deferred shortcut, consumed by the block epilogue of another call
    s = _tensor((n, c, h, w), seed=33, cl=cl)
    qs = _q(clipping, positive, mult=mult)
    d = qs(s.clone(), "s", "activation", defer=True)
    if cl:
        assert d._fq_deferred[0] is qs.last_stats and qs._stat_cache == {}
    y = _q(clipping, positive, mult=mult)(x.clone(), "c", "activation", residual=d)
    if not getattr(y, "_fq_residual_fused", False):
        d = qs(d, "s", "activation") if getattr(d, "_fq_deferred", None) is not None else d
        y = torch.relu(y + d)
    s_plain = _q(clipping, positive, mult=mult)(s.clone(), "s", "activation")
    x_plain = _q(clipping, positive, mult=mult)(x.clone(), "c", "activation")
    assert _same(y, torch.relu(x_plain + s_plain))

    # pooling inside the launch
    if positive:
        for pool, ref_pool in (((2, 2, "direct"), lambda t: F.max_pool2d(t, 2)), ((3, 3), lambda t: F.max_pool2d(t, 3, 2, 1))):
            y = _q(clipping, positive, mult=mult)(x.clone(), "c", "activation", bias=bias, pool=pool, relu_follows=True)
            if getattr(y, "_fq_pooled", None) is None:
                y = ref_pool(y)
            assert _same(y, ref_pool(plain))

    # an Inception branch writing its channel slice of the block's output
    if cl:
        wide = torch.full((n, c + 8, h, w), float("nan"), device="cuda").contiguous(memory_format=torch.channels_last)
        sl = wide[:, 4:4 + c]
        y = _q(clipping, positive, mult=mult)(x.clone(), "c", "activation", bias=bias, out=sl)
        assert y.data_ptr() == sl.data_ptr()
        assert _same(sl.contiguous(), plain.contiguous())


@pytest.mark.parametrize("shape", [(512, 2048, 7, 7), (512, 64, 112, 112)], ids=["2048", "stem"])
def test_model_sizes_equal_quantize1(shape):
    x = _tensor(shape, seed=3, cl=True, positive=True)
    q = _q("laplace", True)
    y = q(x, "c", "activation")   # the manager's activations are quantized in place; the input is kept here
    assert _same(y, _applied(q, x))
    first = q.last_stats.clone()
    del y
    q(x, "c", "activation")
    assert _same(q.last_stats, first)


def test_deterministic_over_runs_and_ctas():
    x = _tensor((8, 64, 28, 28), seed=8, cl=True)
    q = _q("laplace")
    ref = q._fly_bits(x.clone(), None, "laplace")
    t = q.last_stats.clone()
    for ctas in (0, 1, 7, 300):
        y = q._fly_bits(x.clone(), None, "laplace", max_ctas=ctas)
        assert _same(y, ref) and _same(q.last_stats, t)


@pytest.mark.parametrize("positive", [False, True])
def test_never_worse_than_the_analytic_widths(positive):
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    from cnn_quantization_b200.statistics import bit_candidates
    for shape, cl in (((8, 64, 28, 28), True), ((8, 32, 14, 14), False)):
        x = _tensor(shape, seed=12, cl=cl, positive=positive)
        layout, table = _stats(x, cl)
        mult, prior = bit_candidates("laplace", positive, 4)
        sums, params = ops.clip_mse(x, table, layout, cl, 4, positive, mult, prior=prior, widths=range(9),
                                    solve_f64=False, want_params=True)
        widths = ops.allocate_select(sums, params, table, 4)[0].long()
        analytic = IntQuantizer.get_bits_alloc_fixed_target(table[:, 3].contiguous(), 4, True).long()
        g = torch.arange(layout[1], device="cuda")
        got = float(sums[g, 1 + widths].sum())
        if int(analytic.sum()) <= 4 * layout[1]:
            assert got <= float(sums[g, 1 + analytic].sum())


# ---- whole networks -----------------------------------------------------------------------------------------------------------
def _model(config, hw, clipping, fused=True):
    from cnn_quantization_b200 import pipeline
    extra = dict(mse_multipliers=[2.0, 3.0, 4.0, 6.0]) if clipping == "mse" else {}
    cfg = dict(pipeline.CONFIGS[config], clipping=clipping, bit_alloc_prior="mse", fly_bits=True, **extra)
    model, qm = pipeline.build_quantized_model(cfg, "cuda", channels_last=True)
    if not fused:
        qm.fuse_residual_into_quant = qm.defer_shortcut = qm.fuse_pool_into_quant = qm.fuse_inception_concat = False
    x, _ = pipeline.synthetic_batch(2, seed=7, hw=hw, device="cuda", channels_last=True)
    return model, qm, x


def _quantizers(qm):
    return [q for q in list(qm.quantizers.values()) + [qm.quantizer_default] if hasattr(q, "_stat_cache")]


@pytest.mark.parametrize("clipping", ["laplace", "mse"])
@pytest.mark.parametrize("config,hw", [("resnet50_w4a4", 224), ("inception_v3_w4a4", 299)], ids=["resnet50", "inception_v3"])
def test_network_fused_equals_unfused(config, hw, clipping):
    from cnn_quantization_b200 import ops
    outs = []
    for fused in (True, False):
        model, qm, x = _model(config, hw, clipping, fused)
        ops.profile_reset(enable=True)
        with torch.no_grad():
            outs.append(model(x))
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
        assert prof["modes"]["L"]["launches"] > 0 and prof["modes"]["R"]["launches"] > 0
        qm.detach()
    assert torch.isfinite(outs[0]).all()
    assert torch.equal(outs[0], outs[1])


def test_forward_without_host_sync_and_without_cache_growth():
    model, qm, x = _model("resnet50_w4a4", 224, "laplace")
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
    assert all(q.fly_bits for q in _quantizers(qm))
    assert all(q._stat_cache == {} for q in _quantizers(qm))
    qm.detach()


def test_ops_argument_checks():
    from cnn_quantization_b200 import ops
    sums = torch.zeros(4, 1 + 9 * 3, dtype=torch.float64, device="cuda")
    params = torch.zeros(4, 27, 6, device="cuda")
    stats = torch.zeros(4, 12, device="cuda")
    mult = torch.tensor([1.0, 2.0, 3.0], device="cuda")
    with pytest.raises(ValueError, match="params"):
        ops.allocate_select(sums, params[:, :9], stats, 4, multipliers=mult)
    with pytest.raises(ValueError, match="params"):
        ops.allocate_select(sums, params.double(), stats, 4, multipliers=mult)
    with pytest.raises(ValueError, match="stats"):
        ops.allocate_select(sums, params, stats[:, :5], 4, multipliers=mult)
    with pytest.raises(ValueError, match="stats"):
        ops.allocate_select(sums, params, stats.cpu(), 4, multipliers=mult)
    for bad in (None, mult[:2], mult.double(), mult.cpu()):
        with pytest.raises(ValueError, match="multipliers"):
            ops.allocate_select(sums, params, stats, 4, multipliers=bad)
    for bad in (torch.zeros(1, dtype=torch.int64, device="cuda"), torch.zeros(1, dtype=torch.int32)):
        with pytest.raises(ValueError, match="status"):
            ops.allocate_select(sums, params, stats, 4, multipliers=mult, status=bad)
    widths, choice, _, _ = ops.allocate_select(sums, params, stats, 4, multipliers=mult)
    assert widths.shape == (4,) and choice.dtype == torch.int32


# ---- consistency with use mode: the tables collect_bits writes for the same tensors ----------------------------------------------
def test_resnet18_consistent_with_use_mode(tmp_path):
    """A seeded channels-last ResNet-18 W4A4 batch under `-c laplace` with fly_bits; each call site is also quantized
    plainly (no pooling, epilogue, deferral or slice write: those routes equal the plain one, tests above).  For every allocated call site, the tensor it quantized goes through
    collect_bits (BitMseStatistics.save_table) and the per-channel statistics collect, then a `-sm use -bap mse` quantizer:
    the collected table is the route's own sums divided by the element count, bit for bit; the fly_bits widths are
    allocate's on the sums, the use-mode widths allocate's on the table; where they agree the outputs agree bit for bit."""
    from cnn_quantization_b200 import _lib as L, ops, pipeline, statistics as S
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.int_quantizer import IntQuantizer, int_quantizer
    torch.backends.cudnn.allow_tf32 = False
    cfg = dict(pipeline.CONFIGS["resnet18_w4a4"], bit_alloc_prior="mse", fly_bits=True)
    model, qm = pipeline.build_quantized_model(cfg, "cuda", channels_last=True)
    for q in _quantizers(qm):
        q.export_stats = True
    x, _ = pipeline.synthetic_batch(2, seed=11, hw=224, device="cuda", channels_last=True)
    seen, sums_of = [], []
    orig_fly, orig_select = IntQuantizer._fly_bits, ops.allocate_select

    def select(sums, *a, **k):
        sums_of.append(sums.clone())
        return orig_select(sums, *a, **k)

    def fly(self, tensor, bias, rule, max_ctas=0):
        t = tensor.clone()   # before an in-place apply overwrites it
        routes = self._pool, self._residual, self._defer, self._into
        self._pool, self._residual, self._defer, self._into = None, None, False, None
        try:
            plain = orig_fly(self, t.clone(), bias, rule, max_ctas)
        finally:
            self._pool, self._residual, self._defer, self._into = routes
        seen.append((t, self._positive(), plain, self.last_stats.clone(), rule))
        return orig_fly(self, tensor, bias, rule, max_ctas)

    mp = pytest.MonkeyPatch()
    mp.setattr(IntQuantizer, "_fly_bits", fly)
    mp.setattr(ops, "allocate_select", select)
    try:
        with torch.no_grad():
            model(x)
    finally:
        mp.undo()
        qm.detach()
    assert 2 * len(seen) == len(sums_of) and len(seen) > 10
    assert all(_same(a, b) for a, b in zip(sums_of[0::2], sums_of[1::2]))   # the plain and the network's call
    sums_of = sums_of[0::2]

    base = str(tmp_path)
    sm = S.StatisticManagerPerChannel("r18", load_stats=False, base_dir=base)
    bm = S.BitMseStatistics("r18", "laplace", base_dir=base)
    for i, (t, positive, _, _, rule) in enumerate(seen):
        assert rule == "laplace"
        c = S.ClipErrConfig(num_bits=4, positive=positive, per_channel=True, bit_alloc=True, bit_alloc_prior=L.PRIOR_B,
                            bit_alloc_round=True, bit_alloc_target=4)
        for _ in range(2):   # one batch collected twice: the per-channel summary keeps channels only over batches
            sm.save_tensor_stats(t, "conv", "site%d" % i)
            bm.save_table(t, "conv", "site%d" % i, c)
    sm.__exit__()
    bm.__exit__()
    loaded = S.StatisticManagerPerChannel("r18", load_stats=True, base_dir=base)
    tables = S.BitMseStatistics("r18", base_dir=base, load=True)
    agree, differ = [], []
    stats_differ = []
    for i, ((t, positive, y, chosen, _), sums) in enumerate(zip(seen, sums_of)):
        w_fly = chosen[:, 7]
        sid = "site%d" % i
        mse, rule = tables.table(sid)
        count = float(t.numel() // t.shape[1])   # (2 s / 2 n is s / n exactly)
        fly_sums = sums[:, 1:].cpu().numpy()
        assert rule == "laplace" and np.array_equal(mse, fly_sums / count), sid
        w_fly = w_fly.cpu().numpy()
        np.testing.assert_array_equal(w_fly, allocate(fly_sums, 4).astype(np.float32), err_msg=sid)
        p = dict(clipping="laplace", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=True, bit_alloc_act=True,
                 bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
                 bit_alloc_prior="mse", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
                 logger=None, mtd_quant=False)
        q = int_quantizer("int4", p)
        q.half_range = positive
        q.sm = lambda: loaded
        q.bit_tables = tables
        w_use = q._stat_bits(sid, "cuda", 4).cpu().numpy()
        np.testing.assert_array_equal(w_use, allocate(mse, 4).astype(np.float32), err_msg=sid)
        if np.array_equal(w_use, w_fly):
            agree.append(sid)
            y_use = q(t.clone(), sid, "activation", stat_id=sid)
            # use mode solves from the collected statistics (min, max, mean, b of the NCHW statistics launch); the route
            # from its own launch's table.  Where they are the same numbers the outputs are the same bits.
            same_stats = all(np.array_equal(np.asarray(loaded.get_tensor_stat(sid, k, "mean"), dtype=np.float32),
                                            chosen[:, j].cpu().numpy()) for j, k in enumerate(("min", "max", "mean", "b")))
            if same_stats:
                assert _same(y, y_use), sid
            else:
                # the same use-mode quantizer reading the route's own statistics: the same bits
                own = {k: chosen[:, j].cpu().numpy() for j, k in enumerate(("min", "max", "mean", "b", "std"))}
                q.sm = lambda: type("Own", (), {"get_tensor_stat": staticmethod(lambda id, stat, kind: own[stat])})()
                q._stat_cache.clear()
                assert _same(y, q(t.clone(), sid, "activation", stat_id=sid)), sid
                b_use = np.asarray(loaded.get_tensor_stat(sid, "b", "mean"), dtype=np.float32)
                b_fly = chosen[:, 3].cpu().numpy()
                stats_differ.append((sid, float(np.abs(b_use / b_fly - 1).max()), int((y != y_use).sum()), y.numel()))
        else:
            # the same measurement, allocated on sums instead of per-element errors: the additions of the programme
            # round differently, so nearly equal totals may compare the other way
            differ.append((sid, int((w_use != w_fly).sum()), t.shape[1]))
    print("fly_bits vs -sm use -bap mse on ResNet-18: %d call sites with the same widths (%d of them with other "
          "statistics: (site, max rel. b difference, differing elements, elements) %r), %d with other widths "
          "(site, channels that differ, channels) %r" % (len(agree), len(stats_differ), stats_differ, len(differ), differ))
