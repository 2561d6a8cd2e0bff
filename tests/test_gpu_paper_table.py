"""The paper's results table (``pipeline.PAPER_TABLE``) on the GPU: the per-sample / per-tensor min-max ("rows") launch
writing a channel slice of a wider channels-last tensor, bit for bit the unfused launch plus a copy; the 8W4A and 4W8A rows
layer by layer against the live reference; Inception-v3's 4W8A rows with every branch output written in place; and every
quantized cell end to end."""
import numpy as np
import pytest
import torch

import test_gpu_ref_live as RL
from test_gpu_paper_nets import _layerwise_vs_reference, _run_counting

pytestmark = pytest.mark.gpu

ROWS = {
    "8W4A": ["baseline", "aciq", "bit_alloc", "aciq_bit_alloc"],
    "4W8A": ["baseline", "bias_corr", "bit_alloc", "bias_corr_bit_alloc"],
    "4W4A": ["baseline", "all"],
}
NETS = ["vgg16", "vgg16_bn", "inception_v3", "resnet18", "resnet50", "resnet101"]
QUANTIZED = [(net, s, m) for net in NETS for s, methods in ROWS.items() for m in methods]


@pytest.fixture(scope="module", autouse=True)
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _id(cell):
    return "-".join(cell)


# ---- the rows launch into a channel slice, at the op level ----------------------------------------------------------------
# (C, Ctot, c0): the branch widths of Inception-v3 that 4W8A quantizes per tensor, at several slice offsets and pitches
SLICES = [(32, 256, 224), (32, 64, 0), (48, 288, 64), (48, 52, 4), (192, 768, 0), (192, 768, 576), (192, 200, 8),
          (320, 1280, 0), (320, 2048, 1728), (320, 324, 4)]


def _nan_buffer(n, ctot, h, w):
    return torch.full((n, ctot, h, w), float("nan"), device="cuda").contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("variant", ["plain", "positive", "relu_passthrough", "empty_range_passthrough"])
@pytest.mark.parametrize("scope", ["per_sample", "per_tensor"])
def test_rows_slice_write_equals_dense_launch_then_copy(scope, variant):
    from cnn_quantization_b200 import _lib as L, ops
    n, h = 8, 17
    for c, ctot, c0 in SLICES:
        g = torch.Generator(device="cuda").manual_seed(c * 1000 + c0)
        x = torch.randn(n, c, h, h, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
        bias = torch.randn(c, device="cuda", generator=g)
        if variant == "empty_range_passthrough":   # nothing above 0 under a positive range: the leaf passes max(x, 0) on
            x, bias = -x.abs(), -bias.abs()
        kw = dict(scope=L.SCOPE_GROUP_MEAN if scope == "per_sample" else L.SCOPE_TENSOR, range_mode=L.RANGE_MINMAX,
                  leaf=L.LEAF_COMPILED, num_bits=8, positive=variant != "plain",
                  relu_passthrough=variant in ("relu_passthrough", "empty_range_passthrough"),
                  bias=bias, bias_period=-c, any_dense_format=True)
        lay = (1, n, c * h * h)
        ops.profile_reset(enable=True)
        dense = ops.fused(x, lay, **kw)
        buf = _nan_buffer(n, ctot, h, h)
        sl = buf[:, c0:c0 + c]
        assert ops.slice_eligible(x, sl, channels_last=False, bias_period=-c)
        res = ops.fused(x, lay, out=sl, **kw)
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
        assert res is sl and prof["modes"]["Bi"]["launches"] == 1 and prof["modes"]["B"]["launches"] == 1, prof["modes"]
        assert torch.equal(sl, dense), (c, ctot, c0)
        rest = torch.cat([buf[:, :c0], buf[:, c0 + c:]], 1)
        assert torch.isnan(rest).all(), (c, ctot, c0)
        if variant == "empty_range_passthrough":
            assert torch.equal(sl, torch.relu(x + bias.view(1, -1, 1, 1)))


def test_rows_slice_write_through_the_quantizer():
    """IntQuantizer.gemmlowpMinMaxQuantize hands ``out`` to its rows launch: the slice comes back written."""
    from cnn_quantization_b200 import manager as M, ops, pipeline
    args = M.make_args(**pipeline.PAPER_TABLE[("inception_v3", "4W8A", "baseline")])
    qm = M.QuantizationManagerInference(args, M.get_params(args))
    q = qm.get_quantizer("activation")
    q.half_range = False
    n, c, h = 32, 192, 17
    x = torch.randn(n, c, h, h, device="cuda").contiguous(memory_format=torch.channels_last)
    bias = torch.randn(c, device="cuda")
    buf = _nan_buffer(n, 768, h, h)
    sl = buf[:, 384:576]
    want = q(x.clone(), "conv0_activation", "activation", bias=bias)
    ops.profile_reset(enable=True)
    got = q(x.clone(), "conv0_activation", "activation", bias=bias, out=sl)
    prof = ops.profile_collect()
    ops.profile_reset(enable=False)
    assert got is sl and list(prof["modes"]) == ["Bi"], prof["modes"]
    assert torch.equal(sl, want)
    assert torch.isnan(torch.cat([buf[:, :384], buf[:, 576:]], 1)).all()


# ---- layer by layer against the live reference --------------------------------------------------------------------------
def _layerwise(monkeypatch, cell, batch):
    """test_gpu_paper_nets._layerwise_vs_reference on a PAPER_TABLE cell (the helper reads a named config; it follows the
    fusions of Inception-v3 and VGG-16-BN)."""
    from cnn_quantization_b200 import pipeline
    name = "paper_" + _id(cell)
    monkeypatch.setitem(pipeline.CONFIGS, name, pipeline.PAPER_TABLE[cell])
    monkeypatch.setitem(pipeline.INPUT_SIZE, name, pipeline.paper_cell_input_size(cell))
    return _layerwise_vs_reference(name, batch, channels_last=True)


@pytest.mark.parametrize("cell", [("resnet18", s, m) for s, ms in ROWS.items() for m in ms], ids=_id)
def test_resnet18_layerwise_vs_live_reference(monkeypatch, cell):
    """test_gpu_ref_live.test_layerwise_differential_vs_live_reference (which follows the ResNet fusions: the block
    epilogue, the shortcut quantized inside the launch that consumes it, the stem's pooling) on a PAPER_TABLE cell."""
    from cnn_quantization_b200 import pipeline
    from oracle import ref_live
    import cnn_quantization_b200 as fq
    if not ref_live.available():
        pytest.skip("oracle/_ref (staged reference + its compiled extension) not built")
    name = "paper_" + _id(cell)
    monkeypatch.setitem(pipeline.CONFIGS, name, pipeline.PAPER_TABLE[cell])
    RL.test_layerwise_differential_vs_live_reference(ref_live.load(), fq, name, 32, True)


@pytest.mark.parametrize("cell", [(net, s, m) for net in ("inception_v3", "vgg16_bn") for s in ("8W4A", "4W8A") for m in ROWS[s]],
                         ids=_id)
def test_paper_nets_layerwise_vs_live_reference(monkeypatch, cell):
    net = cell[0]
    rows, pooled, into = _layerwise(monkeypatch, cell, 32 if net == "inception_v3" else 16)
    if net == "inception_v3":
        assert len(rows) == 97 and len(into) == 44   # every branch convolution writes its slice, 4W8A's rows launches too
    else:
        assert len(rows) == 21 and len(pooled) == 5


# ---- Inception-v3, 4W8A: every branch output in place --------------------------------------------------------------------
def _build(cell, concat=True):
    """pipeline.build_paper_cell, channels-last; ``concat=False``: with ``fuse_inception_concat`` off"""
    from cnn_quantization_b200 import pipeline
    model, qm = pipeline.build_paper_cell(cell, "cuda", channels_last=True)
    if not concat:
        qm.detach()
        qm.fuse_inception_concat = False
        qm.attach(model)
    return model, qm


@pytest.mark.parametrize("method", ROWS["4W8A"])
def test_inception_4w8a_concat_fusion_is_exact_and_complete(method):
    cell = ("inception_v3", "4W8A", method)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(4, 3, 299, 299, generator=g).cuda().contiguous(memory_format=torch.channels_last)
    a, qa = _build(cell, concat=True)
    qa.record = True
    ya, ba, pa, cats_a = _run_counting(a, x)
    b, qb = _build(cell, concat=False)
    yb, bb, pb, cats_b = _run_counting(b, x)
    assert torch.equal(ya, yb)
    assert len(ba) == len(bb) == 11
    for u, v in zip(ba, bb):
        assert torch.equal(u, v)
    assert len(qa.calls) == 97
    # 44 branch convolutions (per-tensor int8: rows launches) and 2 max-pool branches write their slice; no fallback copy
    assert pa["modes"]["Bi"]["launches"] == 44 and pa["modes"]["Pi"]["launches"] == 2, pa["modes"]
    assert sum(v["launches"] for k, v in pa["modes"].items() if k.endswith("i")) == 46
    assert not any(k.endswith("i") for k in pb["modes"]), pb["modes"]
    assert cats_a == 1 and cats_b == 1 + 11 + 4
    qa.detach()
    qb.detach()


# ---- every quantized cell, end to end ------------------------------------------------------------------------------------
@pytest.mark.parametrize("cell", QUANTIZED, ids=_id)
def test_every_cell_end_to_end(cell):
    from cnn_quantization_b200 import pipeline
    model, qm = pipeline.build_paper_cell(cell, "cuda", channels_last=True)
    x, _ = pipeline.synthetic_batch(8, seed=1, device="cuda", hw=pipeline.paper_cell_input_size(cell), channels_last=True)
    with torch.no_grad():
        y = model(x)
    torch.cuda.synchronize()
    qm.detach()
    assert tuple(y.shape) == (8, 1000)
    assert torch.isfinite(y).all()
    assert float(y.float().std()) > 0 and np.isfinite(float(y.abs().max()))
