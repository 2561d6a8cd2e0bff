"""Quantization-noise measurement on the GPU: ops.sample_noise against a float64 two-pass restatement (layouts, both bias
conventions, short and long rows, no q, no rows, NaN / Inf), its determinism, and the manager end to end on ResNet-18,
ResNet-50, Inception-v3 and VGG-16-BN."""
import os
import warnings

import numpy as np
import pandas as pd
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_noise")
W4A4 = dict(qtype="int4", qweight="int4", clipping="laplace", per_channel_quant_weights=True, per_channel_quant_act=True,
            bit_alloc_act=True, bit_alloc_weight=True, bias_corr_weight=True)
CONFIGS = {
    "w4a4": W4A4,
    "w8a8": dict(qtype="int8", qweight="int8"),
    "q_off_int8": dict(qtype="int8", qweight="int8", q_off=True),
}
# Largest relative deviation from the reference's files of the variances and the input / output norms of the run without
# quantization (the weight norm is left out: the reference's fp32 torch.norm is off by up to 3.4e-4 on large weights).
# Only the convolutions separate them: cuDNN's on the GPU, which torch lets use TF32, against the CPU's fp32 ones
# (4.3e-4 measured on an H100).  Where activations are quantized, such a difference can move an element across a grid
# step (test_gpu_angle.py), so those configs are only reported.
REF_BOUND_Q_OFF = 2e-3


def rows(t, like):
    if like.dim() == 4 and not like.is_contiguous() and like.is_contiguous(memory_format=torch.channels_last):
        t = t.permute(0, 2, 3, 1)
    return t.reshape(t.shape[0], -1)


def restate(y, q=None, bias=None, bias_period=0):
    """float64 two-pass restatement: {column: float32 numpy [N]} of the eps_* and y_* columns (y_* only without q)."""
    yr = rows(y, y)
    if bias is not None:
        i = torch.arange(yr.shape[1], device=y.device)
        yr = yr + bias[i // bias_period if bias_period > 0 else i % -bias_period]   # one fp32 add
    yd = yr.double()
    n = yd.shape[1]
    m = yd.mean(1)
    out = {"y_mean": m, "y_var": ((yd - m[:, None]) ** 2).mean(1), "y_norm": yd.norm(dim=1)}
    if q is not None:
        qd = rows(q, y).double()
        e = yd - qd
        em = e.mean(1)
        cos = (yd * qd).sum(1) / ((yd * yd).sum(1) * (qd * qd).sum(1)).sqrt()   # exactly 1 where q == y
        out.update(eps_norm=e.norm(dim=1), eps_mse=(e * e).sum(1) / n, eps_cos_sim=cos,
                   eps_ang_dist=torch.nan_to_num(torch.acos(cos.clamp(-1, 1))) / np.pi, eps_mean=em,
                   eps_var=((e - em[:, None]) ** 2).mean(1))
    return {k: v.float().cpu().numpy() for k, v in out.items()}


def columns(sums, n):
    """The eps_* / y_* columns noise_columns derives from ops.sample_noise sums."""
    from cnn_quantization_b200.statistics import NOISE_COLUMNS, noise_columns
    s = sums.cpu().numpy()
    yq = s if s.shape[1] == 7 else np.concatenate([s, np.full((s.shape[0], 5), np.nan)], 1)
    t = noise_columns(yq, s[:, :2], s[:, :2], n, n, n, 1).astype(np.float32)
    return {c: t[:, i] for i, c in enumerate(NOISE_COLUMNS)}


def assert_ulp(got, want, what=""):
    """equal (NaN included) or one float32 ulp apart"""
    for k, w in want.items():
        g = got[k]
        same = (g == w) | (np.isnan(g) & np.isnan(w))
        near = np.abs(g.astype(np.float64) - w) <= np.spacing(np.abs(w))
        assert np.all(same | near), (what, k, g[~(same | near)][:4], w[~(same | near)][:4])


def check(y, q=None, bias=None, bias_period=0, **kw):
    from cnn_quantization_b200 import ops
    s = ops.sample_noise(y, q, bias, bias_period, **kw)
    assert s.dtype == torch.float64 and s.shape == (y.shape[0], 7 if q is not None else 2)
    assert_ulp(columns(s, y[0].numel()), restate(y, q, bias, bias_period), (tuple(y.shape), bias_period))
    return s


def quantized(y, step=0.25):
    return torch.round(y / step) * step


@pytest.mark.parametrize("shape", [(8, 16, 56, 56), (16, 2048, 7, 7), (8, 3, 5, 7), (6, 1000), (4, 40000), (3, 1, 1, 1)])
def test_layouts_against_the_restatement(shape):
    torch.manual_seed(1)
    y = torch.randn(shape, device="cuda") * 2 + 0.3
    q = quantized(y)
    check(y, q)
    check(y)
    if len(shape) == 4:
        cl = lambda t: t.contiguous(memory_format=torch.channels_last)
        check(cl(y), cl(q))


@pytest.mark.parametrize("hw", [7, 56])
def test_both_bias_conventions(hw):
    torch.manual_seed(2)
    c = 12
    y = torch.randn(5, c, hw, hw, device="cuda")
    b = torch.randn(c, device="cuda") * 3
    q = quantized(y + b.view(1, -1, 1, 1))
    check(y, q, b, hw * hw)
    ycl, qcl = (t.contiguous(memory_format=torch.channels_last) for t in (y, q))
    check(ycl, qcl, b, -c)
    # the fp32 sum the quantization launch forms: the bias-free tensor plus the bias is the biased tensor, bit for bit
    from cnn_quantization_b200 import ops
    assert torch.equal(ops.sample_noise(y, q, b, hw * hw), ops.sample_noise(y + b.view(1, -1, 1, 1), q))
    # a row that is not a multiple of four (scalar path) and a misaligned one
    y3 = torch.randn(4, 3, 7, 7, device="cuda")
    check(y3, quantized(y3), torch.randn(3, device="cuda"), 49)
    flat = torch.randn(4 * 12 * 49 + 1, device="cuda")[1:].view(4, 12, 7, 7)
    check(flat, quantized(flat), torch.randn(12, device="cuda"), 49)


def test_short_and_long_rows_and_determinism():
    from cnn_quantization_b200 import ops
    torch.manual_seed(3)
    y = torch.randn(16, 64, 112, 112, device="cuda").contiguous(memory_format=torch.channels_last)   # 49 chunks per row
    b = torch.randn(64, device="cuda")
    q = quantized(y + b.view(1, -1, 1, 1)).contiguous(memory_format=torch.channels_last)
    s = check(y, q, b, -64)
    for max_ctas in (0, 1, 7):
        assert torch.equal(ops.sample_noise(y, q, b, -64, max_ctas=max_ctas), s), max_ctas
    assert torch.equal(ops.sample_noise(y, q, b, -64), s)
    z = torch.randn(512, 3, device="cuda")   # rows far shorter than one unit
    check(z, quantized(z), max_ctas=7)


def test_special_values_and_empty():
    from cnn_quantization_b200 import ops
    y = torch.randn(5, 3, 4, 4, device="cuda")
    q = quantized(y)
    y[1, 0, 0, 0] = float("nan")
    y[2, 1, 1, 1] = float("inf")
    q[3, 2, 2, 2] = float("-inf")
    y[4] = 0
    q[4] = 0
    s = ops.sample_noise(y, q).cpu()
    assert torch.isnan(s[1, [0, 1, 4, 5, 6]]).all() and torch.isfinite(s[1, [2, 3]]).all()
    assert torch.isinf(s[2, [0, 1, 5, 6]]).all()
    assert torch.isinf(s[3, 3]) and torch.isfinite(s[3, :2]).all()
    assert (s[4] == 0).all() and torch.isfinite(s[0]).all()
    cols = columns(s.cuda(), 48)
    assert np.isnan(cols["eps_cos_sim"][4]) and cols["eps_ang_dist"][4] == 0
    assert ops.sample_noise(torch.empty(0, 3, 4, 4, device="cuda"), torch.empty(0, 3, 4, 4, device="cuda")).shape == (0, 7)


def test_profile_mode():
    from cnn_quantization_b200 import ops
    y = torch.randn(4, 8, 16, 16, device="cuda")
    ops.profile_reset(enable=True)
    ops.sample_noise(y, y)
    ops.sample_noise(y)
    prof = ops.profile_collect()
    ops.profile_reset(enable=False)
    assert set(prof["modes"]) == {"N"} and prof["modes"]["N"]["bytes"] == 12 * y.numel()
    assert prof["modes"]["N"]["launches"] == 2


def test_sum_of_squares_is_the_activation_norm():
    """The activation norm (`-ms`, ops.sample_sumsq: the one-sum instance of fq_sample_sums.cuh) and column 1 of these sums
    without q add the same float64 squares in the same order: bit for bit equal on the vector and the scalar path
    (DESIGN.md §4.6)."""
    from cnn_quantization_b200 import ops
    torch.manual_seed(4)
    x = torch.randn(8, 64, 56, 56, device="cuda") * 3 + 0.5   # 13 chunks per row
    misaligned = torch.randn(9 * 40000 + 1, device="cuda")[1:].view(9, 40000)
    assert misaligned.data_ptr() % 16 != 0
    for t in (x, x.contiguous(memory_format=torch.channels_last), misaligned):
        assert torch.equal(ops.sample_sumsq(t), ops.sample_noise(t)[:, 1])


# ---- the manager end to end -------------------------------------------------------------------------------------------------
def batches():
    rs = np.random.RandomState(2026)   # make_noise_golden.py's batches
    return [torch.from_numpy(rs.standard_normal((4, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


def run_model(cfg, base_dir, channels_last, xs, arch="resnet18"):
    """The model with the noise kind; returns ({id: our CSV}, {id: [restatement of each call's tensors]})."""
    from cnn_quantization_b200 import pipeline
    cfg = dict(cfg, arch=arch, stats_base_dir=base_dir, measure_stats=True, measure_stats_kind="noise")
    model, qm = pipeline.build_quantized_model(cfg, "cuda", channels_last=channels_last)
    seen = {}
    orig = qm.measure_stats.save_measure

    def spy(y, q, x, w, id, bias=None, bias_period=0):   # the restatement of this call's tensors, before any later write
        r = restate(y, q, bias, bias_period)
        r.update({k.replace("y_", "x_"): v for k, v in restate(x).items()})
        if w is not None:
            r.update({k.replace("y_", "w_"): v for k, v in restate(w.reshape(1, -1)).items()})
        seen.setdefault(id, []).append(r)
        return orig(y, q, x, w, id, bias, bias_period)

    qm.measure_stats.save_measure = spy
    with torch.no_grad():
        for x in xs:
            x = x.cuda()
            model(x.contiguous(memory_format=torch.channels_last) if channels_last else x)
    qm.__exit__()
    folder = os.path.join(base_dir, "noise", arch)
    return {f[:-4]: pd.read_csv(os.path.join(folder, f), float_precision="round_trip") for f in os.listdir(folder)}, seen


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_resnet18_end_to_end(tmp_path, name, channels_last):
    ours, seen = run_model(CONFIGS[name], str(tmp_path), channels_last, batches())
    z = np.load(os.path.join(GOLD, name + ".npz"))
    ids = [str(i) for i in z["ids"]]
    assert sorted(ours) == sorted(ids) == sorted(seen)
    worst, worst_unq = 0.0, 0.0
    for k in ids:
        got = ours[k]
        assert got.shape == (8, 19)
        for b, r in enumerate(seen[k]):
            part = {c: got[c].to_numpy()[4 * b:4 * b + 4].astype(np.float32) for c in got.columns}
            assert_ulp(part, {c: (np.repeat(v, 4) if c.startswith("w_") else v) for c, v in r.items()}, (name, k, b))
        ref = z["id%03d" % ids.index(k)]
        g = got.to_numpy(dtype=np.float64)
        with np.errstate(all="ignore"):
            rel = np.abs(g - ref) / np.maximum(np.abs(ref), 1e-30)
        worst = max(worst, float(np.nanmax(np.where(np.abs(ref) > 0, rel, np.abs(g - ref)))))
        unq = [list(got.columns).index(c) for c in ("x_var", "y_var", "w_var", "y_norm", "x_norm")]
        worst_unq = max(worst_unq, float(np.nanmax(rel[:, unq])))
    print("%s channels_last=%s: largest relative deviation from the reference %.3g (variances and norms %.3g)"
          % (name, channels_last, worst, worst_unq))
    if name == "q_off_int8":
        assert worst_unq < REF_BOUND_Q_OFF, worst_unq
        assert all((ours[k][["eps_norm", "eps_mse", "eps_mean", "eps_var", "eps_ang_dist"]].to_numpy() == 0).all()
                   for k in ids)


def test_resnet50_logits_ids_and_no_host_synchronisation(tmp_path):
    """ResNet-50 W4A4 channels-last at batch 32."""
    from cnn_quantization_b200 import pipeline
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    x, _ = pipeline.synthetic_batch(32, seed=3, device="cuda", channels_last=True)
    outs, counts = [], []
    for ms in (False, True):
        model, qm = pipeline.build_quantized_model(dict(pipeline.CONFIGS["resnet50_w4a4"], measure_stats=ms,
                                                        measure_stats_kind="noise", stats_base_dir=str(tmp_path)),
                                                   "cuda", channels_last=True)
        with torch.no_grad():
            outs.append(model(x.clone()))   # also the warm-up: workspaces, library load
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                with torch.no_grad():
                    model(x.clone())
            finally:
                torch.cuda.set_sync_debug_mode("default")
        counts.append(sum("synchroniz" in str(r.message) for r in w))
        if ms:
            assert len(qm.measure_stats.stats) == 54   # 53 convolutions + the classifier
            assert all(len(v) == 2 and v[0][0].shape == (32, 7) for v in qm.measure_stats.stats.values())
        qm.detach()
    assert torch.equal(outs[0], outs[1])
    assert counts[1] <= counts[0], counts


@pytest.mark.parametrize("arch,hw", [("inception_v3", 299), ("vgg16_bn", 64)])
def test_paper_nets_write_one_finite_file_per_site(tmp_path, arch, hw):
    from cnn_quantization_b200 import pipeline
    x, _ = pipeline.synthetic_batch(2, seed=4, hw=hw, channels_last=True)
    ours, seen = run_model(W4A4, str(tmp_path), True, [x], arch=arch)
    assert sorted(ours) == sorted(seen) and len(ours) > 10
    for k, df in ours.items():
        assert df.shape == (2, 19)
        v = df.drop(columns=["eps_cos_sim"]).to_numpy()
        assert np.isfinite(v).all(), k
