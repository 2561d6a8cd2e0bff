"""Inception-v3 and VGG-16-BN on the GPU: call sites and logits against the reference census, and the launch fusions these
two networks add - Inception branches writing straight into their block's output, the functional ReLU of BasicConv2d
skipped, VGG-16-BN's poolings inside the quantization launches - bit-identical to the same forward without them."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


@pytest.fixture(scope="module", autouse=True)
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def build(config, fused=True, channels_last=True, **over):
    from cnn_quantization_b200 import manager as M, pipeline
    import torchvision.models as models
    flags = dict(pipeline.CONFIGS[config], **over)
    args = M.make_args(**flags)
    qm = M.QuantizationManagerInference(args, M.get_params(args))
    if not fused:
        qm.fuse_inception_concat = qm.skip_redundant_relu = qm.fuse_pool_into_quant = False
    qm.enable()
    try:
        torch.manual_seed(12345)
        model = models.__dict__[args.arch](weights=None, **pipeline.ARCH_KWARGS.get(args.arch, {}))
    finally:
        qm.stop_stamping()
    M.set_node_names(model)
    M.search_absorbe_bn(model)
    qm.bn_folding = True
    model.eval().cuda()
    if channels_last:
        model.to(memory_format=torch.channels_last)
    qm.quantize_model(model)
    qm.attach(model)
    return model, qm


def batch(n, hw, channels_last=True, seed=5):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, 3, hw, hw, generator=g).cuda()
    return x.contiguous(memory_format=torch.channels_last) if channels_last else x


@pytest.mark.parametrize("channels_last", [False, True])
@pytest.mark.parametrize("name", ["inception_v3_w4a4", "vgg16_bn_w4a4"])
def test_call_sites_and_logits(name, channels_last):
    """The reference census (tests/golden/make_census_paper_nets.py) on the CUDA path, tolerances of
    test_cuda_pipeline_call_sites_and_logits."""
    with open(os.path.join(GOLD, "ref_census_paper_nets.json")) as f:
        info = json.load(f)[name]
    ref = np.load(os.path.join(GOLD, "ref_pipeline_paper_nets.npz"))[name]
    model, qm = build(name, channels_last=channels_last)
    qm.record = True
    rs = np.random.RandomState(12345)
    x = torch.from_numpy(rs.standard_normal((info["batch"], 3, info["hw"], info["hw"])).astype(np.float32)).cuda()
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    with torch.no_grad():
        y = model(x).cpu().numpy()
    qm.detach()
    assert [[c[0], c[1], c[2], list(c[3])] for c in qm.calls] == info["act_calls"]
    cos = float((y * ref).sum() / (np.linalg.norm(y) * np.linalg.norm(ref)))
    assert cos > 0.95, cos
    assert abs(np.linalg.norm(y) / np.linalg.norm(ref) - 1) < 0.1


def _run_counting(model, x):
    """logits, the output of every Inception block, the profile, and the number of torch.cat calls of one forward"""
    from cnn_quantization_b200 import ops
    from torchvision.models import inception as I
    blocks, hooks = [], []
    for m in model.modules():
        if type(m) in (I.InceptionA, I.InceptionB, I.InceptionC, I.InceptionD, I.InceptionE):
            hooks.append(m.register_forward_hook(lambda mod, i, o: blocks.append(o.clone())))
    cats = [0]
    orig_cat = torch.cat

    def counting_cat(*a, **k):
        cats[0] += 1
        return orig_cat(*a, **k)

    torch.cat = counting_cat
    ops.profile_reset(enable=True)
    try:
        with torch.no_grad():
            y = model(x.clone())
        prof = ops.profile_collect()
    finally:
        torch.cat = orig_cat
        ops.profile_reset(enable=False)
        for h in hooks:
            h.remove()
    return y, blocks, prof, cats[0]


def _quant_launches(prof):
    return sum(v["launches"] for k, v in prof["modes"].items() if not k.startswith(("E", "P")))


def test_inception_fused_equals_unfused():
    x = batch(4, 299)
    a, qa = build("inception_v3_w4a4", fused=True)
    qa.record = True
    ya, ba, pa, cats_a = _run_counting(a, x)
    b, qb = build("inception_v3_w4a4", fused=False)
    yb, bb, pb, cats_b = _run_counting(b, x)
    assert torch.equal(ya, yb)
    assert len(ba) == len(bb) == 11
    for u, v in zip(ba, bb):
        assert torch.equal(u, v)
    hooked = len(qa.calls)
    assert hooked == 97
    assert _quant_launches(pa) == hooked and _quant_launches(pb) == hooked   # one launch per hooked tensor
    # 44 branch convolutions and 2 max-pool branches write their slice in place; only transform_input's cat is left
    written = sum(v["launches"] for k, v in pa["modes"].items() if k.endswith("i"))
    assert written == 46, pa["modes"]
    assert pa["modes"]["Pi"]["launches"] == 2
    assert cats_a == 1 and cats_b == 1 + 11 + 4   # + every block's cat and InceptionE's two inner ones
    qa.detach()
    qb.detach()


def test_vgg16_bn_pooling_inside_launches_is_exact():
    x = batch(4, 64)
    from cnn_quantization_b200 import ops
    ys = []
    for fused in (True, False):
        model, qm = build("vgg16_bn_w4a4", fused=fused)
        ops.profile_reset(enable=True)
        with torch.no_grad():
            ys.append(model(x.clone()))
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
        qm.detach()
        pooled = sum(v["launches"] for k, v in prof["modes"].items() if "p" in k)
        assert pooled == (5 if fused else 0), prof["modes"]
    assert torch.equal(ys[0], ys[1])


def test_inception_collect_use_round_trip_writes_slices(tmp_path):
    from cnn_quantization_b200 import ops
    x = batch(4, 107)
    base = dict(stats_folder="inc", stats_base_dir=str(tmp_path))
    for pcq in (False, True):
        model, qm = build("inception_v3_w4a4", stats_mode="collect", per_channel_quant_act=pcq, **base)
        with torch.no_grad():   # two batches: a single one collapses the per-channel summary (see bench.py)
            model(x[:2].clone())
            model(x[2:].clone())
        qm.__exit__()
    ys = []
    for fused in (True, False):
        model, qm = build("inception_v3_w4a4", fused=fused, stats_mode="use", **base)
        ops.profile_reset(enable=True)
        with torch.no_grad():
            ys.append(model(x.clone()))
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
        qm.detach()
        if fused:
            assert prof["modes"].get("Ai", {"launches": 0})["launches"] == 44, prof["modes"]
    assert torch.equal(ys[0], ys[1])


# ---- the slice write at the op level, for every branch geometry of Inception-v3 at 299x299 ------------------------------
# (C, H, W, Ctot, c0) of every branch output
BRANCHES = sorted({(c, h, h, tot, c0) for h, parts in (
    (35, [(64, 64, 96, 32)]), (35, [(64, 64, 96, 64)]),
    (17, [(384, 96, 288)]), (17, [(192, 192, 192, 192)]), (8, [(320, 192, 768)]),
    (8, [(320, 384, 384, 384, 384, 192)])) for ws in parts for tot in [sum(ws)]
    for c, c0 in zip(ws, np.cumsum([0] + list(ws[:-1])).tolist())})


def _nan_buffer(n, ctot, h, w):
    return torch.full((n, ctot, h, w), float("nan"), device="cuda").contiguous(memory_format=torch.channels_last)


@pytest.mark.parametrize("kind", ["D", "A", "midtread"])
def test_slice_write_equals_dense_launch_then_copy(kind):
    from cnn_quantization_b200 import _lib as L, ops
    n = 8
    for c, h, w, ctot, c0 in BRANCHES:
        g = torch.Generator(device="cuda").manual_seed(c * 1000 + c0)
        x = torch.randn(n, c, h, w, device="cuda", generator=g).contiguous(memory_format=torch.channels_last)
        lay = (n, c, h * w)
        if kind == "D":
            kw = dict(range_mode=L.RANGE_LAPLACE, num_bits=4, positive=True, bit_alloc=True)
        elif kind == "A":
            kw = dict(range_mode=L.RANGE_GIVEN, num_bits=4, given=(torch.rand(c, device="cuda") + 0.5,
                                                                  torch.zeros(c, device="cuda"), None))
        else:
            kw = dict(leaf=L.LEAF_MIDTREAD, positive=True, mt_target=4.0, mt_clip=True)
        bias = torch.randn(c, device="cuda", generator=g)
        dense = ops.fused(x, lay, channels_last=True, bias=bias, **kw)
        buf = _nan_buffer(n, ctot, h, w)
        sl = buf[:, c0:c0 + c]
        assert ops.slice_eligible(x, sl)
        ops.profile_reset(enable=True)
        res = ops.fused(x, lay, channels_last=True, bias=bias, out=sl, **kw)
        prof = ops.profile_collect()
        ops.profile_reset(enable=False)
        assert res is sl and all(k.endswith("i") for k in prof["modes"]), prof["modes"]
        assert torch.equal(sl, dense), (c, h, ctot, c0)
        rest = torch.cat([buf[:, :c0], buf[:, c0 + c:]], 1)
        assert torch.isnan(rest).all(), (c, h, ctot, c0)


def test_maxpool_slice_write_equals_torch():
    from cnn_quantization_b200 import ops
    for c, h, ctot, c0 in ((288, 35, 768, 480), (768, 17, 1280, 512), (64, 9, 128, 64)):
        x = torch.randn(4, c, h, h, device="cuda").contiguous(memory_format=torch.channels_last)
        oh = (h - 3) // 2 + 1
        buf = _nan_buffer(4, ctot, oh, oh)
        sl = buf[:, c0:c0 + c]
        ops.maxpool2d_cl(x, 3, 2, 0, out=sl)
        assert torch.equal(sl, F.max_pool2d(x, 3, 2))
        assert torch.isnan(torch.cat([buf[:, :c0], buf[:, c0 + c:]], 1)).all()


# ---- layer-wise differential against the live reference ---------------------------------------------------------------
FLIP_FRAC_MODEL = 5e-5   # the bound of test_gpu_ref_live.py::test_layerwise_differential_vs_live_reference


def _layerwise_vs_reference(config, batch, channels_last):
    """The method of test_layerwise_differential_vs_live_reference: the hooked model runs a batch at the config's input
    size; at every quantize_instant call the same GPU input (conv bias added, as the reference's convolution would have)
    also goes through the reference's quantizer for that tag, and the two outputs are compared - with the slice writes,
    the skipped ReLUs and the in-launch poolings of these networks in place (a pooled result is compared with the
    reference's result pooled by torch; a result written into a block's channel slice is compared where it was written).
    Channels whose allocated bit width sits on a rounding boundary (reference fp32 std vs our float64) may differ by one
    bit, at most 2 per layer; they are reported and left out.  Returns the per-layer rows."""
    from oracle import ref_live
    from oracle.ref_live import LeafSpy
    from cnn_quantization_b200 import manager as M, pipeline
    if not ref_live.available():
        pytest.skip("oracle/_ref (staged reference + its compiled extension) not built")
    ref = ref_live.load()
    flags = dict(pipeline.CONFIGS[config])
    args = M.make_args(**flags)
    ref_ops = ref.iqm.TruncationOpManagerInference(args, M.get_params(args))   # the reference's tag -> quantizer table
    model, qm = pipeline.build_quantized_model(flags, "cuda", channels_last=channels_last)
    x, _ = pipeline.synthetic_batch(batch, seed=3, channels_last=channels_last, config=config)
    x = x.cuda()
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    rows, boundary, pooled, into = [], [], [], []
    orig = qm.quantize_instant

    def spy(tensor, id, tag="", stat_id=None, half_range=False, override_att=None, verbose=False, **extra):
        bias = extra.get("bias")
        ref_in = tensor.contiguous().clone() if bias is None else (tensor + bias.view(1, -1, 1, 1)).contiguous()
        q = qm.get_quantizer(tag)
        q.export_stats, q.last_stats = True, None
        out = orig(tensor, id, tag, stat_id, half_range, override_att, verbose, **extra)
        rq = ref_ops.get_quantizer(tag)
        rq.half_range = half_range
        with LeafSpy(rq) as leaf:
            want = rq(ref_in, id, tag)
        if getattr(out, "_fq_pooled", False):
            pooled.append(id)
            want = F.max_pool2d(want, 2) if out._fq_pooled == 2 else F.max_pool2d(want, 3, 2, 1)
        if extra.get("out") is not None and out is extra["out"]:
            into.append(id)
        tol = 1e-5 * torch.maximum(out.abs(), want.abs()) + 1e-9
        diff = (out - want).abs()
        bad = diff > tol
        r_bits = leaf.calls[-1][3] if leaf.calls and leaf.calls[-1][0] == "torch" else None
        if r_bits is not None and q.last_stats is not None and out.dim() == 4 and q.last_stats.shape[0] == r_bits.numel():
            o_bits = q.last_stats[:, 7]
            off = (o_bits != r_bits).nonzero().flatten().tolist()
            assert len(off) <= 2, (id, "bit widths differ in %d channels" % len(off))
            for c in off:
                assert abs(float(o_bits[c]) - float(r_bits[c])) == 1.0, (id, c, float(o_bits[c]), float(r_bits[c]))
                boundary.append((id, c))
                bad[:, c] = False
                diff[:, c] = 0
        rows.append((id, tag, tuple(tensor.shape), float(bad.float().mean()), float(diff.max()), float(want.max() - want.min())))
        return out

    qm.quantize_instant = spy
    with torch.no_grad():
        y = model(x)
    qm.detach()
    assert torch.isfinite(y).all()
    for id, tag, shape, frac, dmax, span in rows:
        assert frac <= FLIP_FRAC_MODEL, (id, tag, shape, frac)
        assert dmax <= span / 2 + 1e-6, (id, tag, shape, dmax, span)   # flips are single grid steps, never garbage
    print("[layerwise] %s batch %d: %d tensors, worst flip fraction %.2e, %d pooled in launch, %d written into a block slice, "
          "%d bit-boundary channels" % (config, batch, len(rows), max(r[3] for r in rows), len(pooled), len(into), len(boundary)))
    return rows, pooled, into


def test_inception_v3_layerwise_vs_live_reference():
    rows, pooled, into = _layerwise_vs_reference("inception_v3_w4a4", 32, channels_last=True)
    assert len(rows) == 97 and len(into) == 44


def test_vgg16_bn_layerwise_vs_live_reference():
    rows, pooled, into = _layerwise_vs_reference("vgg16_bn_w4a4", 16, channels_last=True)
    assert len(rows) == 21 and len(pooled) == 5
