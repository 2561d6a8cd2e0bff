"""Sample-angle measurement (`-ms` with measure_stats_kind="angle") on the GPU: ops.sample_angles against the float64
oracle X.double() @ X.double().T, its exact special cases and determinism, the manager end to end on ResNet-18 (against
the hooked tensors and the reference's angle.pkl, tests/golden/make_angle_golden.py), unchanged ResNet-50 logits and no
added host synchronisation."""
import os
import pickle
import warnings

import numpy as np
import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_angle")
W4A4 = dict(qtype="int4", qweight="int4", clipping="laplace", per_channel_quant_weights=True, per_channel_quant_act=True,
            bit_alloc_act=True, bit_alloc_weight=True, bias_corr_weight=True)
CONFIGS = {
    "w4a4": W4A4,
    "w8a8": dict(qtype="int8", qweight="int8"),
    "q_off_int8": dict(qtype="int8", qweight="int8", q_off=True),
    "collect": dict(stats_mode="collect", qtype="int4", qweight="int4"),
}
# q_off_int8 against the reference's CPU run: no activation is quantized, so only convolution numerics (cuDNN against the
# CPU, fp32) and the reference's fp32 cosine differ; the largest deviation measured was 1.4e-6 rad.  Where activations are
# quantized, cuDNN-vs-CPU last-ulp differences flip single grid steps (0.035 rad W4A4, 0.0049 rad W8A8 measured): those
# runs are checked against the float64 oracle on the hooked tensors only.
REF_BOUND_Q_OFF = 1e-5


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False


def oracle(x):
    """float64 Gram matrix, float64 cosine and angle of the samples of x (on x's device)."""
    t = x.reshape(x.shape[0], -1).double()
    g = t @ t.T
    d = g.diagonal()
    c = g / (d[:, None] * d[None, :]).sqrt()
    return g, c, torch.acos(c.clamp(-1.0, 1.0))


def assert_gram(got, g):
    d = g.diagonal()
    scale = (d[:, None] * d[None, :]).sqrt()
    up = torch.triu(torch.ones_like(g, dtype=torch.bool))
    err = ((got - g).abs() - 1e-11 * scale)[up]
    assert float(err.max()) <= 0, float(((got - g).abs() / scale)[up].max())


def assert_angles(got, c, th):
    """Within one float32 ulp of the oracle's angle rounded to float32, or within 1e-6 rad where |cos| > 1 - 1e-9; 0 on
    and below the diagonal."""
    n = got.shape[0]
    got, c, th = got.cpu(), c.cpu(), th.cpu()
    low = ~torch.triu(torch.ones(n, n, dtype=torch.bool), diagonal=1)
    assert torch.equal(got[low], torch.zeros_like(got[low]))
    want32 = th.float()
    ulp = torch.from_numpy(np.spacing(want32.abs().numpy()))
    ok = ((got - want32).abs() <= ulp) | ((c.abs() > 1 - 1e-9) & ((got.double() - th).abs() <= 1e-6))
    assert bool(ok[~low].all()), float(((got - want32).abs() / ulp)[~low].max())


def sample_matrix(rows, row_len, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(rows, row_len, device="cuda", generator=g) * 2 + 0.25
    if rows > 2:   # nearly parallel pairs, the regime where the angle is ill-conditioned
        x[1] = x[0] + 1e-3 * x[1]
        x[-1] = x[0] * 3 + 1e-6 * x[-1]
    return x


# ---- the kernel ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 2, 7, 63, 64, 65, 512])
@pytest.mark.parametrize("row_len", [1, 3, 4, 5, 49, 4097, 100352])
def test_sample_angles_against_float64_oracle(rows, row_len):
    from cnn_quantization_b200 import ops
    x = sample_matrix(rows, row_len, rows * 1000003 + row_len)
    ang, gram = ops.sample_angles(x, return_gram=True)
    assert ang.dtype == torch.float32 and ang.shape == (rows, rows) and ang.is_cuda
    assert gram.dtype == torch.float64 and gram.shape == (rows, rows)
    g, c, th = oracle(x)
    assert_gram(gram, g)
    assert_angles(ang, c, th)
    assert torch.equal(ops.sample_angles(x), ang)


@pytest.mark.parametrize("row_len", [4, 49, 4096, 40001])
def test_sample_angles_unaligned_view(row_len):
    from cnn_quantization_b200 import ops
    rows = 70
    base = sample_matrix(1, rows * row_len + 1, row_len).view(-1)
    x = base[1:].view(rows, row_len)   # storage offset 1: 4 bytes off 16-byte alignment
    assert x.data_ptr() % 16 != 0
    ang, gram = ops.sample_angles(x, return_gram=True)
    g, c, th = oracle(x)
    assert_gram(gram, g)
    assert_angles(ang, c, th)


def test_sample_angles_resnet50_stem_at_batch_512():
    """One model-size case: the ResNet-50 stem output at batch 512, 512 x 802816 (1.6 GB)."""
    from cnn_quantization_b200 import ops
    x = torch.empty(512, 64, 112, 112, device="cuda")
    x.normal_(generator=torch.Generator(device="cuda").manual_seed(11))
    x = x.relu_().contiguous(memory_format=torch.channels_last)
    ang, gram = ops.sample_angles(x, return_gram=True)
    g, c, th = oracle(x.contiguous())
    assert_gram(gram, g)
    assert_angles(ang, c, th)


@pytest.mark.parametrize("row_len", [5, 4096, 40001])
def test_sample_angles_exact_special_cases(row_len):
    from cnn_quantization_b200 import ops
    rows = 70
    x = sample_matrix(rows, row_len, 5 + row_len)
    x[65] = x[3]             # a duplicate in another tile
    x[66] = -x[3]            # a negated copy
    x[4] = x[3]              # a duplicate in the same tile
    x[10] = 0                # a zero sample
    x[20, row_len // 2] = float("nan")
    x[30, 0] = float("inf")
    x[40, -1] = float("-inf")
    ang = ops.sample_angles(x).cpu()
    pi32 = float(np.float32(np.pi))
    assert float(ang[3, 65]) == 0.0 and float(ang[3, 4]) == 0.0 and float(ang[4, 65]) == 0.0
    assert float(ang[3, 66]) == pi32 and float(ang[4, 66]) == pi32 and float(ang[65, 66]) == pi32
    bad = {10, 20, 30, 40}
    for r in bad:
        assert torch.isnan(ang[:r, r]).all() and torch.isnan(ang[r, r + 1:]).all(), r
    keep = [i for i in range(rows) if i not in bad]
    sub = ang[keep][:, keep]
    assert not torch.isnan(sub).any()
    assert torch.equal(torch.tril(ang), torch.zeros(rows, rows))   # the lower triangle and the diagonal, NaN rows too
    _, c, th = oracle(x[keep])
    assert_angles(sub, c, th)


@pytest.mark.parametrize("shape", [(6, 96, 12, 10), (5, 3, 7, 7), (130, 64, 28, 28), (33, 2048, 7, 7)])
def test_sample_angles_nchw_and_channels_last(shape):
    from cnn_quantization_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(sum(shape))
    x = torch.randn(shape, device="cuda", generator=g).relu_()
    xcl = x.contiguous(memory_format=torch.channels_last)
    _, c, th = oracle(x)
    for y in (x, xcl, x.transpose(2, 3)):   # any other layout is made contiguous first
        assert_angles(ops.sample_angles(y), c, th)


def test_sample_angles_is_deterministic_across_runs_and_grids():
    from cnn_quantization_b200 import ops
    x = torch.randn(512, 2048, 7, 7, device="cuda").relu_().contiguous(memory_format=torch.channels_last)
    a, g = ops.sample_angles(x, return_gram=True)
    for max_ctas in (0, 1, 3):
        b, h = ops.sample_angles(x, return_gram=True, max_ctas=max_ctas)
        assert torch.equal(a, b) and torch.equal(torch.triu(g), torch.triu(h)), max_ctas


def test_sample_angles_profile_mode_and_empty():
    from cnn_quantization_b200 import ops
    x = torch.randn(4, 8, 16, 16, device="cuda")
    ops.profile_reset(enable=True)
    ops.sample_angles(x)
    prof = ops.profile_collect()
    ops.profile_reset(enable=False)
    assert set(prof["modes"]) == {"G"} and prof["modes"]["G"]["bytes"] == 4 * x.numel()
    assert ops.sample_angles(torch.empty(0, 3, 4, 4, device="cuda")).shape == (0, 0)


# ---- the manager end to end -------------------------------------------------------------------------------------------------
def batches():
    rs = np.random.RandomState(2025)   # make_angle_golden.py's batches
    return [torch.from_numpy(rs.standard_normal((6, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


def run_resnet18(flags, base_dir, channels_last):
    """ResNet-18 with the angle kind; returns (our angle.pkl, {id: [(cos, angle) of the oracle on what the call site
    handed on]})."""
    from cnn_quantization_b200 import pipeline
    cfg = dict(arch="resnet18", stats_folder="resnet18", stats_base_dir=base_dir, measure_stats=True,
               measure_stats_kind="angle", **flags)
    model, qm = pipeline.build_quantized_model(cfg, "cuda", channels_last=channels_last)
    seen = {}

    def capture(m, i, o):   # registered after the manager's hook; computed now, before any later in-place write
        prefix = "conv" if isinstance(m, nn.Conv2d) else "linear"
        seen.setdefault("%s%d_activation" % (prefix, m._fq_id), []).append(oracle(o)[1:])

    handles = [m.register_forward_hook(capture) for m in model.modules() if type(m) in (nn.Conv2d, nn.Linear)]
    with torch.no_grad():
        for x in batches():
            x = x.cuda()
            model(x.contiguous(memory_format=torch.channels_last) if channels_last else x)
    for h in handles:
        h.remove()
    qm.__exit__()
    with open(os.path.join(base_dir, "angle", "resnet18", "angle.pkl"), "rb") as f:
        return pickle.load(f), seen


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_resnet18_end_to_end(tmp_path, name, channels_last):
    ours, seen = run_resnet18(CONFIGS[name], str(tmp_path), channels_last)
    z = np.load(os.path.join(GOLD, name + ".npz"))
    ids = [str(i) for i in z["ids"]]
    assert list(ours) == ids + ["target"] and ours["target"] == []
    worst = 0.0
    for k in ids:
        got = torch.from_numpy(ours[k].to_numpy().copy())
        assert got.shape == (12, 6)
        for b, (c, th) in enumerate(seen[k]):
            assert_angles(got[6 * b:6 * b + 6].float(), c, th)
        worst = max(worst, float(np.max(np.abs(ours[k].to_numpy() - z["id%03d" % ids.index(k)]))))
    if name == "q_off_int8":
        assert worst < REF_BOUND_Q_OFF, worst
    print("%s channels_last=%s: largest deviation from the reference %.3g rad" % (name, channels_last, worst))


def test_logits_unchanged_by_the_angle_kind():
    """ResNet-50 W4A4 channels-last at batch 32."""
    from cnn_quantization_b200 import pipeline
    torch.backends.cudnn.benchmark = False
    torch.backends.cudnn.deterministic = True
    x, _ = pipeline.synthetic_batch(32, seed=3, device="cuda", channels_last=True)
    outs = []
    for ms in (False, True):
        model, qm = pipeline.build_quantized_model(dict(pipeline.CONFIGS["resnet50_w4a4"], measure_stats=ms,
                                                        measure_stats_kind="angle"), "cuda", channels_last=True)
        with torch.no_grad():
            outs.append(model(x.clone()))
        if ms:
            assert len(qm.measure_stats.stats) == 54   # 53 convolutions + the classifier
            assert all(v[0].shape == (32, 32) for v in qm.measure_stats.stats.values())
        qm.detach()
    assert torch.equal(outs[0], outs[1])


def test_angle_kind_adds_no_host_synchronisation(tmp_path):
    from cnn_quantization_b200 import pipeline
    x, _ = pipeline.synthetic_batch(4, seed=1, device="cuda", hw=64, channels_last=True)
    counts = []
    for ms in (False, True):
        model, qm = pipeline.build_quantized_model(dict(pipeline.CONFIGS["resnet50_w4a4"], measure_stats=ms,
                                                        measure_stats_kind="angle", stats_base_dir=str(tmp_path)),
                                                   "cuda", channels_last=True)
        with torch.no_grad():
            model(x)   # warm-up: workspaces, library load
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                with torch.no_grad():
                    model(x)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        counts.append(sum("synchroniz" in str(r.message) for r in w))
        qm.detach()
    assert counts[1] <= counts[0], counts
