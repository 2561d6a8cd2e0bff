"""The joint width-and-clip search on the GPU: ops.clip_mse_grid against float64 sums over ops.quantize1 with each
candidate's own parameters, every column bit for bit against ops.clip_mse(widths=...) on the same (width, multiplier)
pair, determinism, NaN propagation, a model-size channels-last tensor, the `-c mse -baa -bap mse` quantizer against its
own tables, and a seeded channels-last ResNet-18: joint collect no worse than the Laplace tables, then use mode."""
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


def pairwise(x, table, layout, cl, positive, mults, widths, prior, **kw):
    """The grid's columns from ops.clip_mse(widths=...) launches of at most 256 candidates each: [G, 1 + W * M]."""
    from cnn_quantization_b200 import ops
    pairs = [(w, m) for w in widths for m in mults]
    cols = []
    for i in range(0, len(pairs), 256):
        part = pairs[i:i + 256]
        got = ops.clip_mse(x, table, layout, cl, 4, positive, [m for _, m in part], prior=prior,
                           widths=[w for w, _ in part], solve_f64=False, **kw)
        cols.append(got[:, :1] if i == 0 else None)
        cols.append(got[:, 1:])
    return torch.cat([c for c in cols if c is not None], 1)


def check(x, layout, positive, prior, mults, widths=WIDTHS, channels_last=False, on_gpu=False, sample=None):
    """Sums against float64 over ops.quantize1 with the reported parameters (all candidates, or ``sample`` of them), and
    every column bit for bit against the per-candidate-width launch."""
    from cnn_quantization_b200 import ops
    outer, groups, inner = layout
    table = stats_table(x, layout, channels_last)
    got, params = ops.clip_mse_grid(x, table, layout, channels_last, 4, positive, mults, widths, prior=prior,
                                    want_params=True, solve_f64=False)
    n = len(widths) * len(mults)
    assert got.shape == (groups, 1 + n) and params.shape == (groups, n, 6)
    np.testing.assert_array_equal(params[:, :, 2].cpu().numpy(),
                                  np.tile(np.repeat(np.float32(widths), len(mults)), (groups, 1)))
    assert torch.equal(got, pairwise(x, table, layout, channels_last, positive, mults, widths, prior))
    xs = x.contiguous().view(outer, groups, inner)
    xd = xs.double() if on_gpu else xs.cpu().numpy().astype(np.float64)
    red = (lambda t: t.sum((0, 2)).cpu().numpy()) if on_gpu else (lambda t: t.sum(axis=(0, 2)))
    cols = range(n) if sample is None else sample
    want = [red(xd * xd)]
    for j in cols:
        q = ops.quantize1(xs, params[:, j, 0].contiguous(), params[:, j, 1].contiguous(), 4, bits=params[:, j, 2].contiguous(),
                          layout=layout).view(outer, groups, inner)
        d = xd - (q.double() if on_gpu else q.cpu().numpy().astype(np.float64))
        want.append(red(d * d))
    want = np.stack(want, 1)
    g = got.cpu().numpy()[:, [0] + [1 + j for j in cols]]
    err = (np.abs(g - want) / np.maximum(np.abs(want), 1e-300)).max()
    assert err < REL, err
    return got


M13 = [0.5 + 0.75 * k for k in range(13)]   # not a multiple of the 8-candidate tile
M30 = [0.25 + 0.5 * k for k in range(30)]   # 9 x 30 = 270 > 256 candidates


@pytest.mark.parametrize("prior", ["laplace", "gaus"])
@pytest.mark.parametrize("positive", [False, True])
@pytest.mark.parametrize("shape", [(4, 96, 14, 14), (2, 7, 9, 11)])
def test_per_channel_nchw(shape, positive, prior):
    g = torch.Generator(device="cuda").manual_seed(sum(shape) + len(prior))
    x = torch.randn(shape, device="cuda", generator=g) * torch.linspace(0.1, 3, shape[1], device="cuda").view(1, -1, 1, 1)
    if positive:
        x = torch.relu(x)
    n, c = shape[:2]
    check(x, (n, c, x.numel() // (n * c)), positive, prior, M13)


@pytest.mark.parametrize("prior", ["laplace", "gaus"])
@pytest.mark.parametrize("positive", [False, True])
def test_per_channel_channels_last(positive, prior):
    from cnn_quantization_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(31 + len(prior))
    x = (torch.randn(8, 96, 10, 12, device="cuda", generator=g) + 0.5).contiguous(memory_format=torch.channels_last)
    assert ops.cl_eligible(x)
    check(x, (8, 96, 120), positive, prior, M30, channels_last=True, sample=range(0, 270, 7))


@pytest.mark.parametrize("positive", [False, True])
def test_per_tensor(positive):
    g = torch.Generator(device="cuda").manual_seed(8)
    x = torch.randn(3, 17, 33, 5, device="cuda", generator=g)
    if positive:
        x = torch.relu(x)
    check(x, (1, 1, x.numel()), positive, "laplace", M30, widths=[8, 2, 5, 0], sample=range(0, 120, 3))


def test_deterministic_across_runs_and_grids():
    from cnn_quantization_b200 import ops
    x = torch.randn(16, 64, 28, 28, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    for t, cl in ((x, False), (x.contiguous(memory_format=torch.channels_last), True)):
        layout = (16, 64, 784)
        table = stats_table(t, layout, cl)
        runs = [ops.clip_mse_grid(t, table, layout, cl, 4, False, M30, WIDTHS, max_ctas=m) for m in (0, 0, 7, 1)]
        for r in runs[1:]:
            assert torch.equal(r, runs[0])


def test_nan_propagates():
    from cnn_quantization_b200 import ops
    x = torch.randn(2, 4, 8, 8, device="cuda")
    x[1, 2, 3, 4] = float("nan")
    layout = (2, 4, 64)
    for t, cl in ((x, False), (x.contiguous(memory_format=torch.channels_last), True)):
        got = ops.clip_mse_grid(t, stats_table(t, layout, cl), layout, cl, 4, False, M13, WIDTHS).cpu()
        assert torch.isnan(got[2]).all() and torch.isfinite(got[[0, 1, 3]]).all()


def test_model_size_channels_last():
    """The shape of ResNet-50's first stage at batch 128 (103 M elements) at the default 9 x 125 candidates."""
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    g = torch.Generator(device="cuda").manual_seed(50)
    x = torch.relu(torch.randn(128, 256, 56, 56, device="cuda", generator=g)).contiguous(memory_format=torch.channels_last)
    check(x, (128, 256, 56 * 56), True, "laplace", list(MSE_MULTIPLIERS), channels_last=True, on_gpu=True,
          sample=[0, 300, 562, 1124])


# ---- the use-mode quantizer on the tensor its tables were measured on --------------------------------------------------------------
def joint_sse(x, stat_id, base, mults):
    """Statistics and joint tables collected on ``x`` (twice), then `-c mse -baa -bap mse` on ``x``: (float64 SSE of the
    quantizer, the tables' sum at the allocated widths, widths)."""
    from cnn_quantization_b200 import _lib as L, int_quantizer, statistics as S
    from cnn_quantization_b200.bit_alloc import allocate
    sm = S.StatisticManagerPerChannel("t", load_stats=False, base_dir=base)
    for _ in range(2):
        sm.save_tensor_stats(x, "conv", stat_id)
    sm.__exit__()
    cfg = S.ClipErrConfig(num_bits=4, positive=False, per_channel=True, bit_alloc=True, bit_alloc_prior=L.PRIOR_STD,
                          bit_alloc_round=True, bit_alloc_target=4)
    bm = S.BitMseStatistics("t", "mse", base_dir=base, multipliers=mults)
    for _ in range(2):
        bm.save_table(x, "conv", stat_id, cfg)
    bm.__exit__()
    loaded = S.StatisticManagerPerChannel("t", load_stats=True, base_dir=base)
    p = dict(clipping="mse", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=True, bit_alloc_act=True,
             bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="mse", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    q = int_quantizer("int4", p)
    q.sm = lambda: loaded
    q.bit_tables = S.BitMseStatistics("t", base_dir=base, load=True)
    y = q(x.clone(), stat_id, "activation", stat_id=stat_id)
    mse, _ = q.bit_tables.table(stat_id)
    c = x.shape[1]
    bits = allocate(mse, 4)
    return float(((x.double() - y.double()) ** 2).sum()), mse[np.arange(c), bits].sum() * x.numel() / c, bits


def test_use_mode_quantizer_reaches_the_table_sum(tmp_path):
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    g = torch.Generator(device="cuda").manual_seed(78)
    x = torch.randn(4, 64, 16, 16, device="cuda", generator=g) * torch.linspace(0.05, 3, 64, device="cuda").view(1, -1, 1, 1)
    x[:, 5] = 0.25   # a constant channel
    got, want, bits = joint_sse(x, "conv1_activation", str(tmp_path), MSE_MULTIPLIERS[::3])
    assert bits[5] == 0 and bits.sum() <= 256
    assert abs(got - want) <= 1e-6 * want, (got, want)


# ---- ResNet-18 W4A4, channels-last: joint collect against the Laplace tables, then `-sm use -c mse -baa -bap mse` --------------------
W4A4 = dict(qtype="int4", qweight="int4", per_channel_quant_weights=True, bit_alloc_weight=True, bias_corr_weight=True,
            per_channel_quant_act=True, bit_alloc_act=True)


def batches():
    rs = np.random.RandomState(2024)
    return [torch.from_numpy(rs.standard_normal((2, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


def run(cfg, xs):
    from cnn_quantization_b200 import pipeline
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, qm = pipeline.build_quantized_model(dict(arch="resnet18", stats_folder="resnet18", **cfg), "cuda",
                                               channels_last=True)
    with torch.no_grad():
        out = [model(x.cuda().contiguous(memory_format=torch.channels_last)) for x in xs]
    qm.__exit__()
    return out


def joint_grid():
    """Every Laplace ACIQ factor (plain and positive) and the default sweep's every fourth value, as float32."""
    from cnn_quantization_b200.int_quantizer import ALPHA_LAPLACE, ALPHA_LAPLACE_POSITIVE
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    vals = [ALPHA_LAPLACE[w] for w in WIDTHS] + [ALPHA_LAPLACE_POSITIVE[w] for w in WIDTHS] + list(MSE_MULTIPLIERS[::4])
    return sorted(set(np.float32(vals).tolist()))


def test_resnet18_joint_collect_then_use(tmp_path):
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    from cnn_quantization_b200.bit_alloc import allocate
    x = batches()
    mults = joint_grid()
    assert len(mults) <= 256
    no_pc = {k: v for k, v in W4A4.items() if k not in ("per_channel_quant_act", "bit_alloc_act")}
    lap, joint = str(tmp_path / "laplace"), str(tmp_path / "mse")
    for base, clip, extra in ((lap, "laplace", {}), (joint, "mse", dict(collect_mse=True, mse_multipliers=mults))):
        run(dict(stats_mode="collect", stats_base_dir=base, clipping=clip, **no_pc), x)   # the per-tensor statistics
        run(dict(stats_mode="collect", stats_base_dir=base, clipping=clip, collect_bits=True, **W4A4, **extra), x)

    def load(base):
        folder = os.path.join(base, "bit_mse", "resnet18")
        with open(os.path.join(folder, "bit_mse.pkl"), "rb") as f:
            return pickle.load(f), pd.read_csv(os.path.join(folder, "alloc.csv"), float_precision="round_trip")

    (t_lap, c_lap), (t_joint, c_joint) = load(lap), load(joint)
    assert t_lap["rule"] == "laplace" and t_joint["rule"] == "mse" and t_joint["prior"] == "laplace"
    ids = [k for k in t_lap if k not in ("rule",)]
    assert len(ids) > 10 and set(ids) == {k for k in t_joint if k not in ("rule", "multipliers", "prior")}
    both = c_lap.merge(c_joint, on="id", suffixes=("_lap", "_joint"))
    assert len(both) == len(ids)
    print(both[["id", "groups_lap", "mse_measured_lap", "mse_measured_joint"]].to_string())
    # the Laplace candidates are in the grid with the same sums: no width, and so no allocation, is worse
    assert (both.mse_measured_joint <= both.mse_measured_lap).all()
    for id in ids:
        cols = ["mse_w%d" % w for w in WIDTHS]
        assert (t_joint[id][cols].to_numpy() <= t_lap[id][cols].to_numpy()).all(), id
    # use mode on the collect batches: every bit-allocated launch gets allocate's widths; the first one's tensor and result
    first = {}
    launched = {}
    orig = IntQuantizer.__call__

    def wrapped(self, tensor, id, tag="", stat_id=None, *a, **k):
        if stat_id in ids and stat_id not in first:
            first[stat_id] = tensor.detach().clone()
        return orig(self, tensor, id, tag, stat_id, *a, **k)

    orig_params = IntQuantizer._joint_alpha_from_stats

    def params(self, stat_id, dev):
        res = orig_params(self, stat_id, dev)
        launched[stat_id] = res[1].cpu().numpy()
        return res

    mp = pytest.MonkeyPatch()
    mp.setattr(IntQuantizer, "__call__", wrapped)
    mp.setattr(IntQuantizer, "_joint_alpha_from_stats", params)
    try:
        logits = run(dict(stats_mode="use", stats_base_dir=joint, clipping="mse", bit_alloc_prior="mse", **W4A4), x)
    finally:
        mp.undo()
    assert all(torch.isfinite(v).all() for v in logits)
    assert set(launched) == set(ids)
    for id, bits in launched.items():
        want = allocate(t_joint[id][["mse_w%d" % w for w in WIDTHS]].to_numpy(), 4)
        np.testing.assert_array_equal(bits, want.astype(np.float32), err_msg=id)
    # the first bit-allocated layer's use-mode tensor: the quantizer reaches its own tables' minimum
    stat_id = next(k for k in ids if k in first)
    got, want, _ = joint_sse(first[stat_id], stat_id, str(tmp_path / "first"), mults)
    assert abs(got - want) <= 1e-6 * want, (stat_id, got, want)
