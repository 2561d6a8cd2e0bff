"""Measured bit allocation on the GPU: ops.clip_mse with per-candidate widths against float64 numpy sums over
ops.quantize1 at each width with the kernel's own parameters, the Laplace columns bit for bit against the launch without
widths, determinism, NaN propagation, a model-size channels-last tensor, `-baw -bap mse` on every ResNet-18 weight, the
`-bap mse` use-mode quantizer against its own tables, and `-sm collect` with collect_bits followed by `-sm use -baa
-bap mse` on the seeded ResNet-18."""
import math
import os
import pickle

import numpy as np
import pandas as pd
import pytest
import torch

pytestmark = pytest.mark.gpu

WIDTHS = list(range(9))
REL = 1e-12   # every (x - q)^2 is formed and added in float64; only the order of the additions differs from numpy's


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def stats_table(x, layout, channels_last=False):
    from cnn_quantization_b200 import ops
    return ops.fused(x, layout, stats_only=True, channels_last=channels_last, num_bits=8)


def candidate_sums(x, params, layout, on_gpu=False):
    """[G, K + 1] float64 sums: sum x^2 and sum (x - q_k)^2, q_k = ops.quantize1 with candidate k's parameters and width."""
    from cnn_quantization_b200 import ops
    outer, groups, inner = layout
    xs = x.contiguous().view(outer, groups, inner)
    xd = xs.double() if on_gpu else xs.cpu().numpy().astype(np.float64)
    red = (lambda t: t.sum((0, 2))) if on_gpu else (lambda t: t.sum(axis=(0, 2)))
    cols = [red(xd * xd)]
    for k in range(params.shape[1]):
        q = ops.quantize1(xs, params[:, k, 0].contiguous(), params[:, k, 1].contiguous(), 4, bits=params[:, k, 2].contiguous(),
                          layout=layout).view(outer, groups, inner)
        d = xd - (q.double() if on_gpu else q.cpu().numpy().astype(np.float64))
        cols.append(red(d * d))
    return torch.stack(cols, 1).cpu().numpy() if on_gpu else np.stack(cols, 1)


def check(x, layout, rule, positive, channels_last=False, on_gpu=False):
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.statistics import bit_candidates
    table = stats_table(x, layout, channels_last)
    mults, prior = bit_candidates(rule, positive, 4)
    got, params = ops.clip_mse(x, table, layout, channels_last, 4, positive, mults, prior=prior, widths=WIDTHS,
                               want_params=True, solve_f64=False)
    assert got.shape == (layout[1], 10)
    p = params.cpu().numpy()
    np.testing.assert_array_equal(p[:, :, 2], np.tile(np.float32(WIDTHS), (layout[1], 1)))
    if rule == "no":   # the min/max range: offset = min (0 when positive), delta = max - offset
        t = table.cpu().numpy()
        off = np.zeros_like(t[:, 0]) if positive else t[:, 0]
        np.testing.assert_array_equal(p[:, :, 1], np.tile(off[:, None], (1, 9)))
        np.testing.assert_array_equal(p[:, :, 0], np.tile((t[:, 1] - off)[:, None], (1, 9)))
    want = candidate_sums(x, params, layout, on_gpu)
    got = got.cpu().numpy()
    err = (np.abs(got - want) / np.maximum(np.abs(want), 1e-300)).max()
    assert err < REL, err
    return got


@pytest.mark.parametrize("rule", ["laplace", "gaus", "no"])
@pytest.mark.parametrize("positive", [False, True])
@pytest.mark.parametrize("shape", [(4, 96, 14, 14), (2, 7, 9, 11)])
def test_per_channel_nchw(shape, rule, positive):
    g = torch.Generator(device="cuda").manual_seed(sum(shape) * 5 + len(rule))
    x = torch.randn(shape, device="cuda", generator=g) * torch.linspace(0.1, 3, shape[1], device="cuda").view(1, -1, 1, 1)
    if positive:
        x = torch.relu(x)
    n, c = shape[:2]
    check(x, (n, c, x.numel() // (n * c)), rule, positive)


@pytest.mark.parametrize("rule", ["laplace", "gaus", "no"])
@pytest.mark.parametrize("positive", [False, True])
@pytest.mark.parametrize("shape", [(8, 96, 10, 12), (2, 2048, 7, 7)])
def test_per_channel_channels_last(shape, rule, positive):
    from cnn_quantization_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(sum(shape) * 3 + len(rule))
    x = (torch.randn(shape, device="cuda", generator=g) + 0.5).contiguous(memory_format=torch.channels_last)
    assert ops.cl_eligible(x)
    n, c = shape[:2]
    check(x, (n, c, x.numel() // (n * c)), rule, positive, channels_last=True)


@pytest.mark.parametrize("shape", [(64, 3, 7, 7), (128, 64, 3, 3), (512, 256, 1, 1), (1000, 512)])
def test_weight_rows(shape):
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    w = torch.randn(shape, device="cuda", generator=g) * 0.05
    rows = shape[0]
    check(w, (1, rows, w.numel() // rows), "no", False)


def test_view_at_storage_offset_one():
    base = torch.randn(2 * 3 * 32 * 32 + 1, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    x = base[1:].view(2, 3, 32, 32)
    assert x.data_ptr() % 16 != 0
    for rule in ("laplace", "no"):
        check(x, (2, 3, 32 * 32), rule, False)


@pytest.mark.parametrize("positive", [False, True])
@pytest.mark.parametrize("cl", [False, True])
def test_laplace_column_is_the_launch_without_widths(positive, cl):
    """Column w is, bit for bit, fqb200_clip_mse with multiplier alpha_laplace[w] and bit_alloc on a table whose column 7
    is w: the candidate sums are independent per tile slot."""
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.statistics import bit_candidates
    x = torch.randn(4, 64, 20, 20, device="cuda", generator=torch.Generator(device="cuda").manual_seed(3)) + 0.2
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    layout = (4, 64, 400)
    table = stats_table(x, layout, cl)
    mults, prior = bit_candidates("laplace", positive, 4)
    got, p = ops.clip_mse(x, table, layout, cl, 4, positive, mults, prior=prior, widths=WIDTHS, want_params=True,
                          solve_f64=False)
    for w in WIDTHS:
        t = table.clone()
        t[:, 7] = float(w)
        one, p1 = ops.clip_mse(x, t, layout, cl, 4, positive, [mults[w]], bit_alloc=True, want_params=True, solve_f64=False)
        assert torch.equal(one[:, 0], got[:, 0])
        assert torch.equal(one[:, 1], got[:, 1 + w]), w
        assert torch.equal(p1[:, 0], p[:, w])


def test_nan_propagates():
    from cnn_quantization_b200 import ops
    x = torch.randn(2, 4, 8, 8, device="cuda")
    x[1, 2, 3, 4] = float("nan")
    layout = (2, 4, 64)
    for t, cl in ((x, False), (x.contiguous(memory_format=torch.channels_last), True)):
        for prior, mults in (("laplace", [1.05] * 9), ("minmax", [0.0] * 9)):
            got = ops.clip_mse(t, stats_table(t, layout, cl), layout, cl, 4, False, mults, prior=prior, widths=WIDTHS).cpu()
            assert torch.isnan(got[2]).all() and torch.isfinite(got[[0, 1, 3]]).all()


def test_deterministic_across_runs_and_grids():
    from cnn_quantization_b200 import ops
    x = torch.randn(16, 64, 28, 28, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    xcl = x.contiguous(memory_format=torch.channels_last)
    for t, cl in ((x, False), (xcl, True)):
        layout = (16, 64, 784)
        table = stats_table(t, layout, cl)
        runs = [ops.clip_mse(t, table, layout, cl, 4, False, [0.0] * 9, prior="minmax", widths=WIDTHS, max_ctas=m)
                for m in (0, 0, 7, 1)]
        for r in runs[1:]:
            assert torch.equal(r, runs[0])


def test_model_size_channels_last():
    """The shape of ResNet-50's first stage at batch 128 (103 M elements)."""
    g = torch.Generator(device="cuda").manual_seed(50)
    x = torch.relu(torch.randn(128, 256, 56, 56, device="cuda", generator=g)).contiguous(memory_format=torch.channels_last)
    check(x, (128, 256, 56 * 56), "laplace", True, channels_last=True, on_gpu=True)


# ---- weights: `-baw -bap mse` ----------------------------------------------------------------------------------------------------
def weight_quantizer(prior):
    from cnn_quantization_b200 import int_quantizer
    p = dict(clipping="no", stats_kind="mean", kld=False, pcq_weights=True, pcq_act=False, bit_alloc_act=False,
             bit_alloc_weight=True, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior=prior, bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    return int_quantizer("int4", p)


def test_resnet18_weights():
    """Every 4-bit ResNet-18 weight: the quantized weight is ops.quantize1 at allocate's widths bit for bit, its float64
    SSE is the table's sum at those widths, and no more than the table's (and the directly measured) SSE of the analytic
    allocation for the same budget."""
    import torchvision
    from cnn_quantization_b200 import _lib as L, ops
    from cnn_quantization_b200.bit_alloc import allocate
    torch.manual_seed(0)
    model = torchvision.models.resnet18().cuda()
    q, qa = weight_quantizer("mse"), weight_quantizer("gaus")
    seen = 0
    for name, m in model.named_modules():
        if not isinstance(m, torch.nn.Conv2d) or m.weight.shape[1] == 3:   # the stem stays at 8 bits
            continue
        w = m.weight.data
        rows = w.shape[0]
        layout = (1, rows, w.numel() // rows)
        got = q(w.clone(), name + ".weight", "weight")
        table = ops.fused(w, layout, num_bits=8, stats_only=True)
        sse = ops.clip_mse(w, table, layout, False, 4, False, [0.0] * 9, prior="minmax", widths=WIDTHS)[:, 1:].cpu().numpy()
        bits = allocate(sse, 4)
        assert bits.sum() <= 4 * rows
        want = ops.quantize1(w, table[:, 1] - table[:, 0], table[:, 0].contiguous(), 4,
                             bits=torch.from_numpy(bits).float().cuda(), layout=layout)
        assert torch.equal(got, want), name
        direct = float(((w.double() - got.double()) ** 2).sum())
        mine = sse[np.arange(rows), bits].sum()
        assert direct == pytest.approx(mine, rel=REL, abs=0)
        # the analytic allocation (widths ∝ log2 std^(2/3)) of the same launch: from the table and measured directly
        abits = ops.fused(w, layout, num_bits=4, stats_only=True, bit_alloc=True, bit_alloc_prior=L.PRIOR_STD,
                          bit_alloc_round=True, bit_alloc_target=4)[:, 7].long().cpu().numpy()
        ana = qa(w.clone(), name + ".weight", "weight")
        ana_direct = float(((w.double() - ana.double()) ** 2).sum())
        assert ana_direct == pytest.approx(sse[np.arange(rows), abits].sum(), rel=REL, abs=0)
        assert mine <= sse[np.arange(rows), abits].sum() and direct <= ana_direct, (name, bits.sum(), abits.sum())
        seen += 1
    assert seen == 19


# ---- the use-mode quantizer on the tensor its tables were measured on --------------------------------------------------------------
@pytest.mark.parametrize("rule", ["laplace", "gaus", "no"])
def test_use_mode_quantizer_reaches_the_table_sum(tmp_path, rule):
    """Statistics and tables collected twice on one tensor, then `-baa -bap mse` on that tensor: its SSE is the sum of
    the table at the allocated widths within 1e-6 relative, and no more than with the analytic `-bap gaus` / `laplace`."""
    from cnn_quantization_b200 import _lib as L, int_quantizer, statistics as S
    base = str(tmp_path)
    g = torch.Generator(device="cuda").manual_seed(78)
    x = torch.randn(4, 64, 16, 16, device="cuda", generator=g) * torch.linspace(0.05, 3, 64, device="cuda").view(1, -1, 1, 1)
    x[:, 5] = 0.25   # a constant channel
    sm = S.StatisticManagerPerChannel("t", load_stats=False, base_dir=base)
    for _ in range(2):
        sm.save_tensor_stats(x, "conv", "conv1_activation")
    sm.__exit__()
    cfg = S.ClipErrConfig(num_bits=4, positive=False, per_channel=True, bit_alloc=True, bit_alloc_prior=L.PRIOR_STD,
                          bit_alloc_round=True, bit_alloc_target=4)
    bm = S.BitMseStatistics("t", rule, base_dir=base)
    for _ in range(2):
        bm.save_table(x, "conv", "conv1_activation", cfg)
    bm.__exit__()
    loaded = S.StatisticManagerPerChannel("t", load_stats=True, base_dir=base)

    def sse_of(prior):
        p = dict(clipping=rule, stats_kind="mean", kld=False, pcq_weights=False, pcq_act=True, bit_alloc_act=True,
                 bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
                 bit_alloc_prior=prior, bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
                 logger=None, mtd_quant=False)
        q = int_quantizer("int4", p)
        q.sm = lambda: loaded
        q.bit_tables = S.BitMseStatistics("t", base_dir=base, load=True)
        y = q(x.clone(), "conv1_activation", "activation", stat_id="conv1_activation")
        return float(((x.double() - y.double()) ** 2).sum()), q

    got, q = sse_of("mse")
    mse, _ = q.bit_tables.table("conv1_activation")
    bits = q._stat_bits("conv1_activation", "cpu", 4).long().numpy()
    assert bits[5] == 0 and bits.sum() <= 256
    want = mse[np.arange(64), bits].sum() * x.numel() / 64
    assert abs(got - want) <= 1e-6 * want, (got, want)
    for prior in ("gaus", "laplace"):
        other = sse_of(prior)[0]
        assert got <= other, (prior, got, other)


# ---- ResNet-18: collect_bits, then `-sm use -baa -bap mse` --------------------------------------------------------------------------
W4A4 = dict(qtype="int4", qweight="int4", per_channel_quant_weights=True, bit_alloc_weight=True, bias_corr_weight=True,
            per_channel_quant_act=True, bit_alloc_act=True, clipping="laplace")


def batches():
    rs = np.random.RandomState(2024)
    return [torch.from_numpy(rs.standard_normal((2, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


def run(cfg, xs):
    from cnn_quantization_b200 import pipeline
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, qm = pipeline.build_quantized_model(dict(arch="resnet18", stats_folder="resnet18", **cfg), "cuda")
    with torch.no_grad():
        for x in xs:
            model(x.cuda())
    qm.__exit__()


def test_resnet18_collect_then_use(tmp_path):
    """The widths every activation launch of `-sm use -baa -bap mse` receives (captured at the launch entry points, per
    call site) are allocate's on the written table, within the budget; alloc.csv shows measured <= analytic."""
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    base = str(tmp_path)
    xs = batches()
    no_pc = {k: v for k, v in W4A4.items() if k not in ("per_channel_quant_act", "bit_alloc_act")}
    run(dict(stats_mode="collect", stats_base_dir=base, **no_pc), xs)   # the per-tensor statistics every use run reads
    run(dict(stats_mode="collect", stats_base_dir=base, collect_bits=True, **W4A4), xs)
    folder = os.path.join(base, "bit_mse", "resnet18")
    with open(os.path.join(folder, "bit_mse.pkl"), "rb") as f:
        tables = pickle.load(f)
    assert tables["rule"] == "laplace" and len(tables) > 10
    launched = {}   # stat_id -> the per-channel widths of each launch of that call site
    current = [None]
    mp = pytest.MonkeyPatch()

    def call(orig):
        def wrapped(self, tensor, id, tag="", stat_id=None, *a, **k):
            current[0] = stat_id
            try:
                return orig(self, tensor, id, tag, stat_id, *a, **k)
            finally:
                current[0] = None
        return wrapped

    def record(orig, bits_of):
        def wrapped(*a, **k):
            bits = bits_of(k)
            if current[0] is not None and bits is not None:
                launched.setdefault(current[0], []).append(bits.detach().cpu().numpy().copy())
            return orig(*a, **k)
        return wrapped

    mp.setattr(IntQuantizer, "__call__", call(IntQuantizer.__call__))
    mp.setattr(ops, "quantize1", record(ops.quantize1, lambda k: k.get("bits")))
    mp.setattr(ops, "quantize1_bca", record(ops.quantize1_bca, lambda k: k.get("bits")))
    mp.setattr(ops, "fused", record(ops.fused, lambda k: (k.get("given") or (None, None, None))[2]))
    try:
        run(dict(stats_mode="use", stats_base_dir=base, bit_alloc_prior="mse", **W4A4), xs)
    finally:
        mp.undo()
    assert set(launched) == {k for k in tables if k != "rule"}
    for stat_id, calls in launched.items():
        mse = tables[stat_id][["mse_w%d" % w for w in WIDTHS]].to_numpy()
        want = allocate(mse, 4)
        assert len(calls) == len(xs)
        for bits in calls:
            np.testing.assert_array_equal(bits, want.astype(np.float32), err_msg=stat_id)
        assert want.sum() <= 4 * len(want)
    csv = pd.read_csv(os.path.join(folder, "alloc.csv"))
    assert set(csv.id) == {k for k in tables if k != "rule"}
    print(csv[["id", "groups", "bits_uniform", "mse_uniform", "bits_analytic", "mse_analytic", "bits_measured",
               "mse_measured"]].to_string())
    assert (csv.mse_measured <= csv.mse_analytic).all()
    assert (csv.bits_measured <= np.floor(csv.target * csv.groups)).all()


@pytest.mark.parametrize("corr", [(True, False), (False, True), (True, True)])
def test_channels_last_weights_with_correction(corr):
    """`-baw -bap mse` with `-bcw` / `-vcw` on a channels-last weight: the same values as on its NCHW copy, which are the
    corrections of _weight_correction_torch applied to the allocated quantization."""
    from cnn_quantization_b200.manager import QuantizationManagerInference as Q
    q = weight_quantizer("mse")
    g = torch.Generator(device="cuda").manual_seed(11)
    w = torch.randn(64, 64, 3, 3, device="cuda", generator=g) * torch.linspace(0.01, 0.2, 64, device="cuda").view(-1, 1, 1, 1)
    w_cl = w.contiguous(memory_format=torch.channels_last)
    got = q(w_cl.clone(), "w", "weight", weight_correction=corr)
    plain = q(w.clone(), "w", "weight")
    want = Q._weight_correction_torch(w, plain, *corr)
    assert torch.equal(got, want)
    assert torch.equal(q(w.clone(), "w", "weight", weight_correction=corr), want)


@pytest.mark.parametrize("vcw", [False, True])
def test_channels_last_resnet18_model(vcw):
    """The channels-last ResNet-18 with `-baw -bap mse -bcw` (and `-vcw`) gets the weights of the NCHW one."""
    from cnn_quantization_b200 import pipeline
    cfg = dict(arch="resnet18", qtype="int4", qweight="int4", per_channel_quant_weights=True, bit_alloc_weight=True,
               bias_corr_weight=True, var_corr_weight=vcw, bit_alloc_prior="mse")
    m_cl, qm_cl = pipeline.build_quantized_model(cfg, "cuda", channels_last=True)
    m_n, qm_n = pipeline.build_quantized_model(cfg, "cuda")
    qm_cl.detach()
    qm_n.detach()
    convs = 0
    for (name, a), (_, b) in zip(m_cl.named_modules(), m_n.named_modules()):
        if isinstance(a, (torch.nn.Conv2d, torch.nn.Linear)):
            assert torch.equal(a.weight, b.weight), name
            convs += 1
    assert convs == 21


def test_weight_entropy_is_measured():
    """`-me` with `-baw -bap mse`: the entropy of the allocated weight's integer grid."""
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.bit_alloc import allocate
    q = weight_quantizer("mse")
    q.measure_entropy = True
    w = torch.randn(128, 64, 3, 3, device="cuda", generator=torch.Generator(device="cuda").manual_seed(4)) * 0.05
    layout = (1, 128, 576)
    got = q(w.clone(), "w", "weight")
    table = ops.fused(w, layout, num_bits=8, stats_only=True)
    sse = ops.clip_mse(w, table, layout, False, 4, False, [0.0] * 9, prior="minmax", widths=WIDTHS)[:, 1:]
    bits = torch.from_numpy(allocate(sse, 4)).float().cuda()
    want, grid = ops.quantize1(w, table[:, 1] - table[:, 0], table[:, 0].contiguous(), 4, bits=bits, layout=layout,
                               want_grid=True)
    assert torch.equal(got, want)
    hist = torch.bincount(grid.flatten().long(), minlength=256)
    assert q.last_entropy is not None and torch.equal(q.last_entropy, q.entropy_from_hist(hist))
