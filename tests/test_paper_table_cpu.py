"""The paper's whole results table (``pipeline.PAPER_TABLE``) without a GPU:

* the 66 cells and their flags, and the "4W4A all" cells that ``pipeline.CONFIGS`` already holds;
* this package's manager with the CPU oracle reproduces, cell by cell, the call list (ids, tags, half_range, shapes, the
  8-bit override of the first layers' weights) and the leading logits of the REAL reference manager
  (tests/golden/make_census_paper_table.py);
* the pitched-output rules of fqb200_fused_into for the per-sample / per-tensor min-max ("rows") launch, against
  ops.slice_eligible.
"""
import ctypes
import json
import os

import numpy as np
import pytest
import torch

from oracle import fq_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden")
NETS = ["vgg16", "vgg16_bn", "inception_v3", "resnet18", "resnet50", "resnet101"]
ROWS = {
    "8W4A": ["baseline", "aciq", "bit_alloc", "aciq_bit_alloc"],
    "4W8A": ["baseline", "bias_corr", "bit_alloc", "bias_corr_bit_alloc"],
    "4W4A": ["baseline", "all"],
}
QUANTIZED = [(net, s, m) for net in NETS for s, methods in ROWS.items() for m in methods]


@pytest.fixture(scope="module")
def census():
    """(meta, logits): make_census_paper_table.py's compact census; the call lists of the networks that ref_census.json /
    ref_census_paper_nets.json already hold come from there (the generator checked that every cell reproduces them)."""
    with open(os.path.join(GOLD, "ref_census_paper_table.json")) as f:
        meta = json.load(f)
    for net, (fname, name) in meta["known"].items():
        with open(os.path.join(GOLD, fname)) as f:
            e = json.load(f)[name]
        meta["calls"][net] = [e["weight_calls"], e["act_calls"]]
    return meta, np.load(os.path.join(GOLD, "ref_pipeline_paper_table.npz"))


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


# ---- the table --------------------------------------------------------------------------------------------------------
def test_table_cells_and_flags():
    from cnn_quantization_b200 import pipeline as P
    T = P.PAPER_TABLE
    assert len(T) == 66
    assert set(T) == set(QUANTIZED) | {(net, "FP32", "fp32") for net in NETS}
    assert tuple(P.PAPER_NETS) == tuple(NETS)
    common = {
        "8W4A": dict(qtype="int4", qweight="int8", per_channel_quant_act=True),
        "4W8A": dict(qtype="int8", qweight="int4", per_channel_quant_weights=True),
        "4W4A": dict(qtype="int4", qweight="int4", per_channel_quant_weights=True, per_channel_quant_act=True),
        "FP32": dict(q_off=True),
    }
    added = {
        ("8W4A", "baseline"): {}, ("8W4A", "aciq"): dict(clipping="laplace"), ("8W4A", "bit_alloc"): dict(bit_alloc_act=True),
        ("8W4A", "aciq_bit_alloc"): dict(clipping="laplace", bit_alloc_act=True),
        ("4W8A", "baseline"): {}, ("4W8A", "bias_corr"): dict(bias_corr_weight=True),
        ("4W8A", "bit_alloc"): dict(bit_alloc_weight=True),
        ("4W8A", "bias_corr_bit_alloc"): dict(bit_alloc_weight=True, bias_corr_weight=True),
        ("4W4A", "baseline"): {},
        ("4W4A", "all"): dict(clipping="laplace", bit_alloc_act=True, bit_alloc_weight=True, bias_corr_weight=True),
        ("FP32", "fp32"): {},
    }
    for (net, s, m), flags in T.items():
        assert flags == dict(arch=net, **common[s], **added[(s, m)]), (net, s, m)
        assert "bit_alloc_target_act" not in flags and "bit_alloc_target_weight" not in flags
        from cnn_quantization_b200 import manager as M
        M.make_args(**flags)   # every key is a reference CLI flag
    assert P.paper_cell_input_size(("inception_v3", "4W8A", "baseline")) == 299
    assert all(P.paper_cell_input_size((net, "8W4A", "aciq")) == 224 for net in NETS if net != "inception_v3")


def test_4w4a_all_cells_equal_the_existing_configs():
    from cnn_quantization_b200 import pipeline as P
    for net in ("resnet18", "resnet50", "resnet101", "inception_v3", "vgg16_bn"):
        assert P.PAPER_TABLE[(net, "4W4A", "all")] == P.CONFIGS[net + "_w4a4"], net
    # vgg16_w4a4 is BASELINE's bin-allocation run at a 5.3-bit target; the paper's cell keeps the default target
    vgg = dict(P.CONFIGS["vgg16_w4a4"])
    assert vgg.pop("bit_alloc_target_act") == 5.3 and vgg.pop("bit_alloc_target_weight") == 5.3
    assert P.PAPER_TABLE[("vgg16", "4W4A", "all")] == vgg


def test_fp32_cell_builds_without_quantizing():
    from cnn_quantization_b200 import pipeline as P
    model, qm = P.build_paper_cell(("resnet18", "FP32", "fp32"), "cpu")
    qm.record = True
    with torch.no_grad():
        y = model(torch.randn(1, 3, 64, 64))
    qm.detach()
    assert y.shape == (1, 1000) and torch.isfinite(y).all()
    assert qm.disable_quantization and not qm.calls


# ---- the census, cell by cell ------------------------------------------------------------------------------------------
def _build(cell, factory):
    """(model, manager) as pipeline.build_paper_cell builds them, on the CPU, before quantize_model / attach."""
    from cnn_quantization_b200 import manager as M, pipeline
    import torchvision.models as models
    args = M.make_args(**pipeline.PAPER_TABLE[cell])
    qm = M.QuantizationManagerInference(args, M.get_params(args), quantizer_factory=factory)
    qm.enable()
    try:
        torch.manual_seed(12345)
        model = models.__dict__[args.arch](weights=None, **pipeline.ARCH_KWARGS.get(args.arch, {}))
    finally:
        qm.stop_stamping()
    M.set_node_names(model)
    if "resnet" in args.arch:
        M.resnet_mark_before_relu(model)
    if "resnet" in args.arch or args.arch in ("vgg16_bn", "inception_v3"):
        M.search_absorbe_bn(model)
        qm.bn_folding = True
    return model.eval(), qm


@pytest.mark.parametrize("cell", QUANTIZED, ids=["-".join(c) for c in QUANTIZED])
def test_call_lists_and_logits_match_reference(census, cell):
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    meta, logits = census
    net = cell[0]
    model, qm = _build(cell, O.oracle_int_quantizer)
    qm.record = True
    overrides = []
    orig = qm.quantize_instant

    def spy(tensor, id, tag="", stat_id=None, half_range=False, override_att=None, verbose=False, **extra):
        if override_att == ("num_bits", 8):
            overrides.append(id)
        return orig(tensor, id, tag, stat_id, half_range, override_att, verbose, **extra)

    qm.quantize_instant = spy
    qm.quantize_model(model)
    n_w = len(qm.calls)
    qm.attach(model)
    rs = np.random.RandomState(12345)
    hw = meta["hw"][net]
    x = torch.from_numpy(rs.standard_normal((meta["batch"], 3, hw, hw)).astype(np.float32))
    with torch.no_grad():
        y = model(x).numpy()
    qm.detach()
    calls = [[c[0], c[1], c[2], list(c[3])] for c in qm.calls]
    want_w, want_a = meta["calls"][net]
    assert calls[:n_w] == want_w
    assert calls[n_w:] == want_a
    # the 8-bit weights: the first layers by attribute override, the classifier by its own int8 quantizer (tag)
    assert overrides == meta["first8"][net] and len(overrides) == (2 if net == "inception_v3" else 1)
    assert sum(c[1] == "weight_classifier" for c in want_w) == (2 if net == "inception_v3" else 1)
    assert sum(c[1] == "activation_classifier" for c in want_a) == 1
    ref = logits["|".join(cell)]   # the first logits of each sample
    got = y[:, :ref.shape[1]]
    assert np.allclose(got, ref, rtol=1e-4, atol=1e-5 * float(np.abs(ref).max())), float(np.abs(got - ref).max())


def test_census_covers_every_quantized_cell(census):
    meta, logits = census
    assert sorted(logits.files) == sorted("|".join(c) for c in QUANTIZED)
    assert sorted(meta["calls"]) == sorted(meta["hw"]) == sorted(NETS)
    assert [len(v) for v in meta["calls"]["resnet101"]] == [105, 106]
    assert len(meta["calls"]["inception_v3"][1]) == 97


# ---- pitched output of the rows launch -------------------------------------------------------------------------------------
def _cl(n, c, h, w, offset_floats=0):
    """A channels-last [n, c, h, w] view whose storage starts ``offset_floats`` floats into a 16-byte aligned buffer."""
    buf = torch.zeros(n * c * h * w + 64)
    base = (16 - buf.data_ptr() % 16) % 16 // 4
    flat = buf[base + offset_floats: base + offset_floats + n * c * h * w]
    return flat.view(n, h, w, c).permute(0, 3, 1, 2)


def _rows_into(lib, x, out, pitch, bias=None, scope=None, **kw):
    """Return code of fqb200_fused_into for the rows launch IntQuantizer.gemmlowpMinMaxQuantize makes of the channels-last
    ``x`` (samples as rows, compiled leaf, min / max; C from the channel-fastest bias), on host memory without a workspace:
    whatever the rules accept stops at the device or at the missing workspace, never at a kernel."""
    from cnn_quantization_b200 import _lib as L
    n, c = x.shape[0], x.shape[1]
    d = L.Desc()
    d.outer, d.groups, d.inner = 1, n, x.numel() // n
    d.scope = L.SCOPE_GROUP_MEAN if scope is None else scope
    d.range_mode, d.leaf, d.num_bits, d.channels_last = L.RANGE_MINMAX, L.LEAF_COMPILED, 8, 0
    if bias is not None:
        d.bias, d.bias_period = bias.data_ptr(), -c
    for k, v in kw.items():
        setattr(d, k, v)
    return lib.fqb200_fused_into(ctypes.byref(d), x.data_ptr(), out.data_ptr(), pitch, None, 0, None)


def test_rows_fused_into_rules_and_slice_predicate_agree(lib):
    from cnn_quantization_b200 import _lib as L, ops
    n, h, w = 2, 5, 5
    refused = (L.ERR_INVALID, L.ERR_UNSUPPORTED)
    accepted = cases = 0
    for c in (8, 12, 64):
        x = _cl(n, c, h, w)
        bias = torch.zeros(c + 4)[:c]
        for ctot_extra in (0, 4, 6, 32):
            for c0 in (0, 2, 4, 8):
                ctot = c + c0 + ctot_extra
                sl = _cl(n, ctot, h, w)[:, c0:c0 + c]
                pitch = ops.slice_pitch(sl)
                assert pitch == ctot
                for with_bias in (True, False):
                    for scope in (L.SCOPE_GROUP_MEAN, L.SCOPE_TENSOR):
                        want = ops.slice_eligible(x, sl, channels_last=False, bias_period=-c if with_bias else 0)
                        rc = _rows_into(lib, x, sl, pitch, bias if with_bias else None, scope)
                        assert rc not in refused if want else rc == L.ERR_UNSUPPORTED, (c, ctot, c0, with_bias, rc,
                                                                                        lib.fqb200_last_error())
                        assert want == (with_bias and ctot % 4 == 0 and c0 % 4 == 0), (c, ctot, c0, with_bias)
                        accepted += want
                        cases += 1
    assert cases > 150 and accepted > 30
    x = _cl(n, 8, h, w)
    bias = torch.zeros(8)
    out = _cl(n, 16, h, w)
    assert _rows_into(lib, x, out, 16, bias) not in refused
    # histogram (-me), residual, pooling and statistics-only requests take no pitch
    hist = torch.zeros(256, dtype=torch.int64)
    assert _rows_into(lib, x, out, 16, bias, out_hist=hist.data_ptr()) == L.ERR_UNSUPPORTED
    assert _rows_into(lib, x, out, 16, bias, residual=x.data_ptr()) == L.ERR_UNSUPPORTED
    assert _rows_into(lib, x, out, 16, bias, pool=2, pool_h=h, pool_w=w, pool_out=out.data_ptr()) == L.ERR_UNSUPPORTED
    stats = torch.zeros(n * 12)
    assert _rows_into(lib, x, out, 16, bias, stats_only=1, out_stats=stats.data_ptr()) == L.ERR_UNSUPPORTED
    # other leaves / ranges with the same bias are no rows launch
    assert _rows_into(lib, x, out, 16, bias, leaf=L.LEAF_TORCH) == L.ERR_UNSUPPORTED
    assert _rows_into(lib, x, out, 16, bias, range_mode=L.RANGE_LAPLACE) == L.ERR_UNSUPPORTED
    # pitch below C (though >= the sample count), not a multiple of 4, misaligned, overlapping
    assert _rows_into(lib, _cl(2, 12, h, w), _cl(2, 12, h, w), 8, torch.zeros(12)) == L.ERR_UNSUPPORTED
    assert _rows_into(lib, x, _cl(n, 12, h, w), 10, bias) == L.ERR_UNSUPPORTED
    assert _rows_into(lib, x, _cl(n, 16, h, w, offset_floats=2), 16, bias) == L.ERR_UNSUPPORTED
    assert "aligned" in lib.fqb200_last_error().decode()
    assert _rows_into(lib, x, x, 12, bias) == L.ERR_INVALID and "overlaps" in lib.fqb200_last_error().decode()
    assert _rows_into(lib, x, x, 8, bias) not in refused   # pitch C: the dense (in-place) case
    # more than 4096 samples: no rows launch, no slice
    big = _cl(4100, 4, 1, 2)
    assert not ops.slice_eligible(big, _cl(4100, 8, 1, 2)[:, :4], channels_last=False, bias_period=-4)
    assert not ops.slice_eligible(x, out[:, :8], channels_last=False, bias_period=-4)   # the bias must have C elements
