"""Measured clipping of weights (`clip_weight="mse"`) on the GPU: the given-parameter weight launch against the
RANGE_MINMAX weight launch bit for bit, the device width allocation against bit_alloc.allocate exactly, the consistency
of the recorded errors with the launch output, never worse than min/max per channel and per layer, determinism, layout,
no host synchronisation inside quantize_model, and what the option changes on a seeded ResNet-18."""
import csv
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fq():
    import __graft_entry__
    __graft_entry__.build()
    import cnn_quantization_b200 as fq
    return fq


def _weights(arch):
    import torchvision.models as models
    torch.manual_seed(12345)
    return [(n, m.weight.data.cuda()) for n, m in models.__dict__[arch](weights=None).named_modules()
            if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear))]


def _shapes(*archs):
    seen = {}
    for arch in archs:
        for n, w in _weights(arch):
            seen.setdefault(tuple(w.shape), w)
    return list(seen.values())


CONFIGS = [(4, False, False, False, False), (4, True, False, False, False), (4, True, True, True, True),
           (4, False, True, False, True), (8, False, False, True, False), (8, False, True, True, True)]


def test_launch_parity_with_minmax_launch(fq):
    from cnn_quantization_b200 import _lib as L, ops
    for w in _shapes("resnet18", "resnet50"):
        rows = w.shape[0]
        layout = (1, rows, w.numel() // rows)
        for bits, alloc, bc, vc, me in CONFIGS:
            h0 = torch.zeros(256, dtype=torch.int64, device="cuda") if me else None
            h1 = torch.zeros(256, dtype=torch.int64, device="cuda") if me else None
            ref, st = ops.fused(w, layout, range_mode=L.RANGE_MINMAX, leaf=L.LEAF_TORCH, num_bits=bits, bit_alloc=alloc,
                                bit_alloc_prior=L.PRIOR_STD, bit_alloc_target=bits, bias_corr=bc, var_corr=vc, hist=h0,
                                want_stats=True)
            got = ops.quantize_weights_given(w, st[:, 5].contiguous(), st[:, 6].contiguous(), bits,
                                             bits=st[:, 7].contiguous() if alloc else None, bias_corr=bc, var_corr=vc,
                                             hist=h1)
            cfg = (tuple(w.shape), bits, alloc, bc, vc, me)
            assert torch.equal(got.view(-1), ref.contiguous().view(-1)), cfg
            if me:
                assert torch.equal(h0, h1), cfg


def _tables(rs):
    for g in (1, 2, 7, 64, 333, 2048):
        yield "random", rs.exponential(size=(g, 9)).cumsum(1)[:, ::-1].copy()      # decreasing in the width
        yield "noise", rs.standard_normal((g, 9)) ** 2
        t = rs.randint(0, 3, size=(g, 9)).astype(np.float64)                         # exact ties everywhere
        t[::3] = 5.0                                                                # constant channels
        yield "ties", t


def test_allocation_parity(fq):
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.bit_alloc import allocate
    rs = np.random.RandomState(7)
    for kind, t in _tables(rs):
        for target in (0, 0.5, 4, 7.9, 8):
            want = allocate(t, target)
            got = ops.allocate_widths(torch.from_numpy(t).cuda(), target).cpu().numpy()
            assert np.array_equal(got, want.astype(np.float32)), (kind, t.shape, target)


def test_allocation_parity_on_resnet50_tables(fq):
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.bit_alloc import allocate
    status = torch.zeros(1, dtype=torch.int32, device="cuda")
    for n, w in _weights("resnet50"):
        layout = (1, w.shape[0], w.numel() // w.shape[0])
        table = ops.fused(w, layout, num_bits=8, stats_only=True)
        sse = ops.clip_mse(w, table, layout, False, 4, False, [0.0] * 9, prior="minmax", widths=list(range(9)),
                           solve_f64=False)[:, 1:].contiguous()
        for target in (2, 4):
            got = ops.allocate_widths(sse, target, status).cpu().numpy()
            assert np.array_equal(got, allocate(sse, target).astype(np.float32)), (n, target)
    assert int(status.item()) == 0
    bad = torch.ones(5, 9, dtype=torch.float64, device="cuda")
    bad[2, 3] = math.nan
    ops.allocate_widths(bad, 4, status)
    assert int(status.item()) == 1


def _quantizer(fq, bits=4, baw=False, prior="gaus", mult=None, bcw=False, vcw=False):
    from cnn_quantization_b200.int_quantizer import WeightMse
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    p = dict(clipping="no", stats_kind="mean", kld=False, pcq_weights=True, pcq_act=False, bit_alloc_act=False,
             bit_alloc_weight=baw, bcorr_act=False, bcorr_weight=bcw, vcorr_weight=vcw, bit_alloc_rmode="round",
             bit_alloc_prior=prior, bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    q = fq.int_quantizer("int%d" % bits, p)
    q.clip_weight = "mse"
    q.weight_mse = WeightMse(MSE_MULTIPLIERS if mult is None else mult, "laplace")
    q.export_stats = True
    return q


@pytest.mark.parametrize("baw,prior", [(False, "gaus"), (True, "gaus"), (True, "mse")])
def test_consistency_and_never_worse(fq, baw, prior):
    q = _quantizer(fq, baw=baw, prior=prior)
    for arch in ("resnet18", "resnet50"):
        for n, w in _weights(arch):
            y = q(w, n)
            chosen, minmax, widths = q.last_weight_mse
            assert bool((chosen <= minmax).all()), (arch, n)
            if not baw:
                assert bool((widths == 4).all())
            e = ((w.double() - y.double()).reshape(w.shape[0], -1) ** 2).sum(1)
            assert torch.allclose(e, chosen, rtol=1e-9, atol=0), (arch, n, float((e - chosen).abs().max()))


def test_layer_totals_never_worse_than_minmax_allocation(fq, tmp_path):
    import torchvision.models as models
    import cnn_quantization_b200.manager as M
    for arch in ("resnet18", "resnet50"):
        report = str(tmp_path / ("%s.csv" % arch))
        args = M.make_args(arch=arch, qtype="int4", qweight="int4", per_channel_quant_weights=True, bit_alloc_weight=True,
                           bit_alloc_prior="mse", clip_weight="mse", weight_mse_report=report)
        qm = M.QuantizationManagerInference(args, M.get_params(args))
        torch.manual_seed(12345)
        model = models.__dict__[arch](weights=None).cuda()
        qm.quantize_model(model)
        with open(report) as f:
            rows = list(csv.DictReader(f))
        assert len(rows) == sum(1 for m in model.modules() if isinstance(m, (torch.nn.Conv2d, torch.nn.Linear)))
        red = []
        for r in rows:
            assert float(r["mse_chosen"]) <= float(r["mse_minmax"]), r
            if r["mse_minmax_alloc"]:   # the 4-bit, bit-allocated weights
                assert float(r["mse_chosen"]) <= float(r["mse_minmax_alloc"]), r
                assert int(r["bits"]) <= int(r["rows"]) * 4 and int(r["bits_minmax_alloc"]) <= int(r["rows"]) * 4
                red.append(1.0 - float(r["mse_chosen"]) / float(r["mse_minmax_alloc"]))
        print("%s: per-layer MSE reduction against the min/max allocation: min %.3f median %.3f max %.3f"
              % (arch, min(red), float(np.median(red)), max(red)))


def test_determinism_and_layout(fq):
    q = _quantizer(fq, baw=True, prior="mse", bcw=True, vcw=True)
    for n, w in _weights("resnet18")[::4]:
        layout = (1, w.shape[0], w.numel() // w.shape[0])
        ref = q._clip_mse_weights(w, n, layout, True, True)
        for max_ctas in (0, 0, 7, 33):
            assert torch.equal(q._clip_mse_weights(w, n, layout, True, True, max_ctas=max_ctas), ref), (n, max_ctas)
        if w.dim() == 4:
            cl = w.contiguous(memory_format=torch.channels_last)
            assert torch.equal(q(cl, n, weight_correction=(True, True)).contiguous(), ref.contiguous()), n


def _resnet18_cl(M, **flags):
    import torchvision.models as models
    args = M.make_args(arch="resnet18", qtype="int4", qweight="int4", per_channel_quant_weights=True,
                       per_channel_quant_act=True, bias_corr_weight=True, **flags)
    qm = M.QuantizationManagerInference(args, M.get_params(args))
    qm.enable()
    try:
        torch.manual_seed(12345)
        model = models.resnet18(weights=None)
    finally:
        qm.stop_stamping()
    M.set_node_names(model)
    M.resnet_mark_before_relu(model)
    M.search_absorbe_bn(model)
    qm.bn_folding = True
    return qm, model.eval().cuda().to(memory_format=torch.channels_last)


def test_no_host_sync_inside_quantize_model(fq, tmp_path):
    import cnn_quantization_b200.manager as M
    for flags in (dict(), dict(bit_alloc_weight=True), dict(bit_alloc_weight=True, bit_alloc_prior="mse")):
        qm, model = _resnet18_cl(M, clip_weight="mse", weight_mse_report=str(tmp_path / "r.csv"), **flags)
        qm.quantize_model(model)   # warm-up: library load, workspaces, pinned multipliers
        qm, model = _resnet18_cl(M, clip_weight="mse", weight_mse_report=str(tmp_path / "r.csv"), **flags)
        finish, calls = qm.weight_mse.finish, []
        qm.weight_mse.finish = lambda: calls.append(1)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            qm.quantize_model(model)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        assert calls == [1]
        finish()   # the one read-back


def test_model_level(fq):
    import cnn_quantization_b200.manager as M
    qa, ma = _resnet18_cl(M)
    qb, mb = _resnet18_cl(M, clip_weight="mse")
    qa.quantize_model(ma)
    qb.quantize_model(mb)
    changed = 0
    for (n, a), (_, b) in zip(ma.named_parameters(), mb.named_parameters()):
        if n.endswith(".weight") and a.dim() in (2, 4):
            changed += int(not torch.equal(a, b))
        else:
            assert torch.equal(a, b), n
    assert changed > 0
    # with the option off the weights are the default launch's
    qc, mc = _resnet18_cl(M)
    from cnn_quantization_b200 import _lib as L, ops
    for (n, m), (_, mq) in zip(mc.named_modules(), ma.named_modules()):
        if isinstance(m, torch.nn.Conv2d):
            w = m.weight.data
            want = ops.fused(w, (1, w.shape[0], w.numel() // w.shape[0]), num_bits=8 if w.shape[1] == 3 else 4,
                             bias_corr=True)
            assert torch.equal(mq.weight.data.contiguous().view(-1), want.view(-1)), n
    # activations run through the unchanged launches: the same weights give the same logits under either manager
    mb.load_state_dict(ma.state_dict())
    x = torch.randn(4, 3, 224, 224, generator=torch.Generator().manual_seed(3)).cuda().contiguous(
        memory_format=torch.channels_last)
    outs = []
    for qm, model in ((qa, ma), (qb, mb)):
        qm.attach(model)
        with torch.no_grad():
            outs.append(model(x.clone()))
        qm.detach()
    assert torch.equal(outs[0], outs[1])
