"""Inception-v3 and VGG-16-BN, the two networks of the paper's table beyond ResNet-18/50/101 and VGG-16, without a GPU:

* this package's manager with the CPU oracle reproduces the call list and the logits of the REAL reference manager
  (tests/golden/make_census_paper_nets.py) on both networks;
* the pitched-output rules of fqb200_fused_into / fqb200_maxpool2d_nhwc_into, and ops.slice_eligible against the library;
* attach / detach patch and restore exactly the Inception blocks and their BasicConv2d modules.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import fq_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
NAMES = ["inception_v3_w4a4", "vgg16_bn_w4a4"]


@pytest.fixture(scope="module")
def census():
    with open(os.path.join(GOLD, "ref_census_paper_nets.json")) as f:
        return json.load(f), np.load(os.path.join(GOLD, "ref_pipeline_paper_nets.npz"))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


def build(config, factory=None):
    """(model, manager) as pipeline.build_quantized_model builds them, on the CPU, before quantize_model / attach."""
    from cnn_quantization_b200 import manager as M, pipeline
    import torchvision.models as models
    args = M.make_args(**pipeline.CONFIGS[config])
    qm = M.QuantizationManagerInference(args, M.get_params(args), quantizer_factory=factory)
    qm.enable()
    try:
        torch.manual_seed(12345)
        model = models.__dict__[args.arch](weights=None, **pipeline.ARCH_KWARGS.get(args.arch, {}))
    finally:
        qm.stop_stamping()
    M.set_node_names(model)
    M.search_absorbe_bn(model)
    qm.bn_folding = True
    return model.eval(), qm


@pytest.mark.parametrize("name", NAMES)
def test_call_sites_and_logits_match_reference(census, name):
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    meta, logits = census
    info = meta[name]
    model, qm = build(name, O.oracle_int_quantizer)
    qm.record = True
    qm.quantize_model(model)
    n_w = len(qm.calls)
    qm.attach(model)
    rs = np.random.RandomState(12345)
    x = torch.from_numpy(rs.standard_normal((info["batch"], 3, info["hw"], info["hw"])).astype(np.float32))
    with torch.no_grad():
        y = model(x).numpy()
    qm.detach()
    calls = [[c[0], c[1], c[2], list(c[3])] for c in qm.calls]
    assert calls[:n_w] == info["weight_calls"]
    assert calls[n_w:] == info["act_calls"]
    ref = logits[name]
    assert y.shape == ref.shape
    assert np.allclose(y, ref, rtol=1e-4, atol=1e-5 * float(np.abs(ref).max())), float(np.abs(y - ref).max())


def test_census_counts(census):
    meta, _ = census
    inc = meta["inception_v3_w4a4"]
    assert len(inc["weight_calls"]) == 98   # 94 + the auxiliary head's 2 convolutions, fc and the auxiliary fc
    acts = [c[0] for c in inc["act_calls"]]
    assert len(acts) == 97
    assert sum(a.startswith("conv") for a in acts) == 94
    assert sum(a.startswith("maxpool") for a in acts) == 2
    assert sum(a.startswith("linear") for a in acts) == 1
    vgg = meta["vgg16_bn_w4a4"]
    assert len(vgg["weight_calls"]) == 16 and len(vgg["act_calls"]) == 21


def test_configs_and_input_sizes():
    from cnn_quantization_b200 import pipeline
    assert pipeline.INPUT_SIZE["inception_v3_w4a4"] == 299 and pipeline.INPUT_SIZE["vgg16_bn_w4a4"] == 224
    assert pipeline.INPUT_SIZE["resnet50_w4a4"] == 224
    for name in NAMES:
        assert "bit_alloc_target_act" not in pipeline.CONFIGS[name]
    x, _ = pipeline.synthetic_batch(1, seed=0, config="inception_v3_w4a4")
    assert tuple(x.shape) == (1, 3, 299, 299)
    assert tuple(pipeline.synthetic_batch(1, seed=0)[0].shape) == (1, 3, 224, 224)


# ---- pitched output -------------------------------------------------------------------------------------------------------
def _desc(x, **kw):
    from cnn_quantization_b200 import _lib as L
    d = L.Desc()
    d.outer, d.groups, d.inner = x.shape[0], x.shape[1], x.shape[2] * x.shape[3]
    d.num_bits, d.bit_alloc_target, d.channels_last = 4, 4.0, 1
    d.range_mode = L.RANGE_LAPLACE
    for k, v in kw.items():
        setattr(d, k, v)
    return d


def _fused_into(lib, x, out, pitch, **kw):
    """Return code of fqb200_fused_into on host memory without a workspace: whatever the pitch rules accept stops at the
    device (ERR_CUDA without one) or at the missing workspace (ERR_WORKSPACE), never at a kernel."""
    d = _desc(x, **kw)
    return lib.fqb200_fused_into(ctypes.byref(d), x.data_ptr(), out.data_ptr(), pitch, None, 0, None)


def _cl(n, c, h, w, offset_floats=0):
    """A channels-last [n, c, h, w] view whose storage starts ``offset_floats`` floats into a 16-byte aligned buffer."""
    buf = torch.zeros(n * c * h * w + 64)
    base = (16 - buf.data_ptr() % 16) % 16 // 4
    flat = buf[base + offset_floats: base + offset_floats + n * c * h * w]
    return flat.view(n, h, w, c).permute(0, 3, 1, 2)


def test_fused_into_rules_and_slice_predicate_agree(lib):
    from cnn_quantization_b200 import _lib as L, ops
    n, h, w = 2, 5, 5
    refused = (L.ERR_INVALID, L.ERR_UNSUPPORTED)
    cases = 0
    for c in (8, 12, 64):
        x = _cl(n, c, h, w)
        for ctot_extra in (0, 4, 6, 32):
            for c0 in (0, 2, 4, 8):
                ctot = c + c0 + ctot_extra
                big = _cl(n, ctot, h, w)
                sl = big[:, c0:c0 + c]
                pitch = ops.slice_pitch(sl)
                assert pitch == ctot
                for kind in ("apply", "stats_only", "pool", "nchw"):
                    kw = {"stats_only": dict(stats_only=1, out_stats=16), "pool": dict(pool=2, pool_h=h, pool_w=w, pool_out=16),
                          "nchw": dict(channels_last=0)}.get(kind, {})
                    want = ops.slice_eligible(x, sl, channels_last=kind != "nchw", stats_only=kind == "stats_only",
                                              pool=(2, 2) if kind == "pool" else None)
                    rc = _fused_into(lib, x, sl, pitch, **kw)
                    # no case of the grid overlaps: every refusal (launch kind, pitch, misaligned slice) is UNSUPPORTED
                    assert rc not in refused if want else rc == L.ERR_UNSUPPORTED, (c, ctot, c0, kind, rc,
                                                                                     lib.fqb200_last_error())
                    cases += 1
                    if kind == "apply":
                        want_ok = ctot % 4 == 0 and c0 % 4 == 0
                        assert want == want_ok, (c, ctot, c0)
    assert cases > 100
    # an output overlapping its input, and a pitch below C / not a multiple of 4, with the codes the header documents
    x = _cl(n, 8, h, w)
    assert _fused_into(lib, x, x, 8) not in refused   # the dense in-place case stays fqb200_fused's
    assert _fused_into(lib, x, x, 12) == L.ERR_INVALID and "overlaps" in lib.fqb200_last_error().decode()
    assert _fused_into(lib, x, _cl(n, 8, h, w), 4) == L.ERR_UNSUPPORTED
    assert _fused_into(lib, x, _cl(n, 12, h, w), 10) == L.ERR_UNSUPPORTED
    assert _fused_into(lib, x, _cl(n, 16, h, w, offset_floats=2), 16) == L.ERR_UNSUPPORTED   # misaligned out
    assert "aligned" in lib.fqb200_last_error().decode()
    assert not ops.slice_eligible(x, x)


def test_maxpool_into_rules(lib):
    from cnn_quantization_b200 import _lib as L
    x = _cl(2, 8, 7, 7)
    out = _cl(2, 16, 3, 3)

    def rc(dst, pitch, c=8):
        return lib.fqb200_maxpool2d_nhwc_into(x.data_ptr(), dst.data_ptr(), 2, 7, 7, c, 3, 3, 2, 2, 0, 0, pitch, None)

    assert rc(out, 4) == L.ERR_UNSUPPORTED        # pitch below C
    assert rc(out, 14) == L.ERR_UNSUPPORTED       # not a multiple of 4
    assert rc(_cl(2, 16, 3, 3, offset_floats=2), 16) == L.ERR_UNSUPPORTED   # misaligned
    assert rc(x, 16) == L.ERR_INVALID and "overlaps" in lib.fqb200_last_error().decode()
    assert rc(out, 16, c=6) == L.ERR_UNSUPPORTED  # C % 4


def test_attach_detach_patch_exactly_the_inception_modules():
    from torchvision.models import inception as I
    model, qm = build("inception_v3_w4a4")
    qm.attach(model)
    blocks = {m for m in model.modules() if type(m) in (I.InceptionA, I.InceptionB, I.InceptionC, I.InceptionD, I.InceptionE)}
    basics = {m for m in model.modules() if type(m) is I.BasicConv2d}
    patched = {m for m in model.modules() if "forward" in m.__dict__}
    assert len(blocks) == 11 and len(basics) == 96
    for m in blocks | basics:
        assert m in patched
    others = patched - blocks - basics
    assert all(type(m) in (torch.nn.BatchNorm2d, torch.nn.MaxPool2d) for m in others)   # the existing patches
    qm.detach()
    assert not any("forward" in m.__dict__ for m in model.modules())
    assert not any("_fq_out" in m.__dict__ for m in model.modules())


@pytest.mark.parametrize("flags", [dict(stats_mode="collect"), dict(measure_stats=True), dict(q_off=True)])
def test_inception_patches_stay_off(flags, tmp_path):
    from cnn_quantization_b200 import manager as M, pipeline
    from torchvision.models import inception as I
    args = M.make_args(**dict(pipeline.CONFIGS["inception_v3_w4a4"], stats_base_dir=str(tmp_path), **flags))
    qm = M.QuantizationManagerInference(args, M.get_params(args))
    qm.enable()
    try:
        torch.manual_seed(0)
        model = I.inception_v3(weights=None, **pipeline.ARCH_KWARGS["inception_v3"])
    finally:
        qm.stop_stamping()
    qm.attach(model)
    assert not any("forward" in m.__dict__ for m in model.modules() if isinstance(m, (I.BasicConv2d, I.InceptionA, I.InceptionE)))
    qm.detach()


def test_vgg16_bn_pooling_scan_steps_over_folded_bn():
    model, qm = build("vgg16_bn_w4a4")
    qm.attach(model)
    marked = [m for m in model.modules() if "_fq_pool_module" in m.__dict__]
    assert len(marked) == 5 and all(m.__dict__["_fq_pool_module"][1] is False for m in marked)   # behind the ReLU
    qm.detach()
    assert not any("_fq_pool_module" in m.__dict__ for m in model.modules())
