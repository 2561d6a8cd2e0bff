"""Measured clipping of weights (`clip_weight="mse"`) on the GPU: the given-parameter weight launch against the
RANGE_MINMAX weight launch bit for bit, the device width allocation against bit_alloc.allocate exactly, the consistency
of the recorded errors with the launch output, never worse than min/max per channel and per layer, determinism, layout,
no host synchronisation inside quantize_model, and what the option changes on a seeded ResNet-18.  Then every stage of
the chain - statistics, candidate parameters and errors, selection, widths, corrected output and report - against the
float64 restatement tests/golden/weight_mse_oracle.py on ResNet-18, ResNet-50 and VGG-16 fc6 weights and on edge rows."""
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


def _quantizer(fq, bits=4, baw=False, prior="gaus", mult=None, bcw=False, vcw=False, mse_prior="laplace", target=None):
    from cnn_quantization_b200.int_quantizer import WeightMse
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    p = dict(clipping="no", stats_kind="mean", kld=False, pcq_weights=True, pcq_act=False, bit_alloc_act=False,
             bit_alloc_weight=baw, bcorr_act=False, bcorr_weight=bcw, vcorr_weight=vcw, bit_alloc_rmode="round",
             bit_alloc_prior=prior, bit_alloc_target_act=None, bit_alloc_target_weight=target, measure_entropy=False,
             logger=None, mtd_quant=False)
    q = fq.int_quantizer("int%d" % bits, p)
    q.clip_weight = "mse"
    q.weight_mse = WeightMse(MSE_MULTIPLIERS if mult is None else mult, mse_prior)
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


# ---- every stage against the float64 restatement (tests/golden/weight_mse_oracle.py) -------------------------------------------
# A sum of the same float64 squares added in another order: the clipping-error tests' tolerance.
REL = 1e-12
# tests/test_gpu_parity.py's tolerance for the statistics columns mean, b and std
STAT_RTOL, STAT_ATOL = 2e-6, 1e-6


class _Spy(object):
    """Records the arguments and results of the ops calls `_clip_mse_weights` makes (it looks them up on the module)."""
    NAMES = ("fused", "clip_mse_grid", "clip_mse", "allocate_widths", "quantize_weights_given")

    def __init__(self, mp):
        from cnn_quantization_b200 import ops
        self.calls = {}
        for n in self.NAMES:
            mp.setattr(ops, n, self._wrap(n, getattr(ops, n)))

    def _wrap(self, name, f):
        def call(*a, **k):
            r = f(*a, **k)
            self.calls.setdefault(name, []).append((a, k, r))
            return r
        return call


def _f64(t):
    return t.detach().double().cpu().numpy()


def _edge_weights():
    """Synthetic weights at O in {1, 7, 1000, 2048, 4096}: [O, 1] and [O, 3] rows, and rows cycling through Gaussian,
    constant, all-zero, one 100x outlier and denormal scale (~1e-39, under the fp32 normal range: the 1e-8 scale floor)."""
    g = torch.Generator().manual_seed(2024)
    out = []
    for shape in ((1, 64), (7, 1), (7, 3), (1000, 3, 5, 5), (2048, 3), (4096, 1), (4096, 27)):
        w = torch.randn(shape, generator=g) * 0.05
        r = w.view(shape[0], -1)
        for i in range(1, shape[0], 5):
            r[i] = 0.0625 * (1 + i % 3)                               # constant
        r[2::5] = 0.0                                                   # all zero
        if r.shape[1] > 1:
            r[3::5, 7 % r.shape[1]] = 100 * r[3::5].abs().max(1)[0]    # one outlier per row
        r[4::5] *= 2e-38                                                # denormal scale
        out.append(("edge%s" % "x".join(map(str, shape)), w.cuda()))
    return out


def _vgg_fc6_rows(rows=64):
    """Rows of VGG-16's fc6 (25088 inputs) as torchvision initialises it, N(0, 0.01): sliced to keep the CPU reference
    affordable."""
    g = torch.Generator().manual_seed(16)
    return [("fc6", (torch.randn(rows, 25088, generator=g) * 0.01).cuda())]


def _check(fq, mp, tmp_path, name, w, bits=4, baw=False, prior="gaus", mult=None, bcw=False, vcw=False,
           mse_prior="laplace", target=None, channels_last=False):
    """Run one weight through `clip_weight="mse"` with a report and compare every stage with the restatement."""
    import weight_mse_oracle as W
    from conftest import fq_mismatch
    from cnn_quantization_b200 import _lib as L, ops
    from cnn_quantization_b200.bit_alloc import allocate
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    mult = list(MSE_MULTIPLIERS if mult is None else mult)
    cfg = (name, tuple(w.shape), bits, baw, prior, len(mult), bcw, vcw, mse_prior, target, channels_last)
    q = _quantizer(fq, bits, baw, prior, mult, bcw, vcw, mse_prior, target)
    q.weight_mse.report = str(tmp_path / "report.csv")
    spy = _Spy(mp)
    x = w.contiguous(memory_format=torch.channels_last) if channels_last else w
    y = q(x, name, weight_correction=(bcw, vcw)).contiguous()
    q.weight_mse.finish()
    with open(q.weight_mse.report) as f:
        rep = list(csv.DictReader(f))
    calls = spy.calls
    mp.undo()
    g = w.shape[0]
    n = w.numel()
    alloc = baw and bits <= 4
    bap = alloc and prior == "mse"
    tgt = bits if target is None else target
    table = calls["fused"][0][2]
    ta = table.cpu().numpy()

    # statistics (tier b): min and max exact, mean / b / std within rounding of their float64 values
    st = W.row_stats(w)
    assert np.array_equal(ta[:, :2], st[:, :2]), cfg
    for c in (2, 3, 4):
        both_nan = np.isnan(st[:, c]) & np.isnan(ta[:, c])
        ok = np.abs(ta[:, c] - st[:, c]) <= STAT_ATOL + STAT_RTOL * np.abs(st[:, c])
        assert (ok | both_nan).all(), (cfg, L.STAT_COLUMNS[c], np.nonzero(~(ok | both_nan))[0][:5])

    # the std prior's widths (-baw): the default weight launch's and get_bits_alloc_fixed_target's
    if alloc:
        _, ref = ops.fused(w, (1, g, n // g), range_mode=L.RANGE_MINMAX, leaf=L.LEAF_TORCH, num_bits=bits, bit_alloc=True,
                           bit_alloc_prior=L.PRIOR_STD, bit_alloc_target=tgt, want_stats=True)
        assert torch.equal(table[:, 7], ref[:, 7]), cfg
        sw = W.std_widths(ta, tgt)
        # a NaN std (one-element rows) gives NaN widths on the host; the launch clamps a NaN width to 0.  Otherwise a
        # channel whose log2(bins) sits within fp32 rounding of x.5 may land one bit away (float64 vs fp32 sum of the prior)
        sw = np.where(np.isnan(sw), 0, sw)
        off = np.nonzero(sw != ta[:, 7])[0]
        assert len(off) <= 1 and (np.abs(sw[off] - ta[off, 7]) == 1).all(), (cfg, off)

    h = W.restate(w, ta, mult, mse_prior, bits, baw=baw, bap_mse=bap, target=target, bcw=bcw, vcw=vcw)
    grid, gp = calls["clip_mse_grid"][0][2]
    mm, mpar = calls["clip_mse"][0][2]
    nw, c = len(h["widths"]), len(mult) + 1
    dev_err = np.concatenate([_f64(mm)[:, 1:].reshape(g, nw, 1), _f64(grid)[:, 1:].reshape(g, nw, c - 1)], 2)
    dev_par = torch.cat([mpar.reshape(g, nw, 1, 6), gp.reshape(g, nw, c - 1, 6)], 2).cpu().numpy()

    # candidate parameters (tier a), bit for bit.  A NaN alpha (the unbiased std of a one-element row under the gaus
    # prior) is NaN on the host; the launch's fmaxf keeps offset = min, so that candidate quantizes like min/max
    nan_a = np.isnan(h["delta"])
    hd = np.broadcast_to(h["delta"][:, None], (g, nw, c))
    ho = np.broadcast_to(h["offset"][:, None], (g, nw, c))
    nan_w = np.broadcast_to(nan_a[:, None], (g, nw, c))
    assert np.array_equal(dev_par[..., 0], hd, equal_nan=True), cfg
    assert np.array_equal(dev_par[..., 1][~nan_w], ho[~nan_w]), cfg
    assert (dev_par[..., 1][nan_w] == np.broadcast_to(ta[:, None, None, 0], (g, nw, c))[nan_w]).all(), cfg
    assert (dev_par[..., 2] == np.asarray(h["widths"], np.float32)[None, :, None]).all(), cfg

    # candidate errors within REL; NaN-alpha candidates NaN on the host and min/max's error on the device
    he = h["err"]
    assert np.isnan(he[nan_w]).all() and np.array_equal(dev_err[nan_w], np.broadcast_to(dev_err[..., :1], he.shape)[nan_w])
    fin = ~nan_w
    assert np.array_equal(np.isnan(dev_err[fin]), np.isnan(he[fin])), cfg
    with np.errstate(invalid="ignore"):
        rel = np.abs(dev_err - he) / np.maximum(np.abs(he), 1e-300)
    assert np.nanmax(np.where(fin, rel, 0)) <= REL, (cfg, np.nanmax(np.where(fin, rel, 0)))

    # widths: num_bits, the table's column 7, or under -bap mse allocate on the per-width best errors; the device's
    # allocation is allocate's on its own table exactly, and any other allocation on the host's table costs the same
    qa, qk, _ = calls["quantize_weights_given"][0]
    dbits = qk["bits"].cpu().numpy() if alloc else np.full(g, bits, np.float32)
    if not alloc:
        assert qk["bits"] is None and qa[3] == bits
    elif not bap:
        assert np.array_equal(dbits, ta[:, 7]), cfg
    else:
        _, dev_best = W.select(dev_err)
        assert np.array_equal(dbits, allocate(dev_best, tgt).astype(np.float32)), cfg
        assert dbits.sum() <= math.floor(tgt * g), cfg
        if not np.array_equal(dbits, h["chosen"][2]):
            gi = np.arange(g)
            a, b = h["best"][gi, dbits.astype(np.int64)].sum(), h["best"][gi, h["wi"]].sum()
            assert abs(a - b) <= REL * abs(b), (cfg, a, b)
            h = W.restate(w, ta, mult, mse_prior, bits, baw=baw, bap_mse=bap, target=target, bcw=bcw, vcw=vcw,
                          wi=dbits.astype(np.int64))
    assert qk["bias_corr"] == bcw and qk["var_corr"] == vcw, cfg

    # selection at the chosen width: the host's first minimum (NaN never wins), the device's parameters bit for bit;
    # where two distinct candidates' host errors are within REL of each other the device may take either
    gi = np.arange(g)
    e_w, b_w = h["err"][gi, h["wi"]], h["best"][gi, h["wi"]]
    acc = W.near_ties(e_w, b_w, REL)
    acc[gi, h["k"]] = True
    dd, do = qa[1].cpu().numpy(), qa[2].cpu().numpy()
    match = (h["delta"] == dd[:, None]) & (h["offset"] == do[:, None]) & acc
    assert match.any(1).all(), (cfg, np.nonzero(~match.any(1))[0][:5])

    # output: bit for bit without corrections; with -bcw / -vcw within test_a13's bound of the corrected host weights
    got = y.cpu().numpy()
    if not (bcw or vcw):
        assert np.array_equal(got, h["y0"], equal_nan=True), cfg
    else:
        assert np.array_equal(np.isnan(got), np.isnan(h["y"])), cfg
        step = float(np.abs(W.rows_of(w)).max())
        frac, worst = fq_mismatch(got, h["y"], step, atol=1e-5 * step)
        assert frac <= 5e-3 and worst <= 1.01, (cfg, frac, worst)

    # the report: every column against the host's row
    assert len(rep) == 1, cfg
    r, hr = rep[0], h["report"]
    assert r["id"] == name and int(r["rows"]) == g and int(r["bits"]) == hr["bits"], (cfg, r, hr)
    # mse_chosen is the error of the uncorrected quantizer - what the selection measures - also under -bcw / -vcw
    for col in ("mse_minmax", "mse_chosen"):
        assert abs(float(r[col]) - hr[col]) <= REL * abs(hr[col]), (cfg, col, r[col], hr[col])
    if not (bcw or vcw):
        sse = float((((w.double() - y.double().view(w.shape)) ** 2).sum()))
        assert abs(float(r["mse_chosen"]) * n - sse) <= REL * sse + 1e-300, (cfg, r["mse_chosen"], sse / n)
    lo = int(((acc.sum(1) == 1) & acc[:, 0]).sum())
    assert lo <= int(r["kept_minmax"]) <= int(acc[:, 0].sum()), (cfg, r["kept_minmax"], lo, hr["kept_minmax"])
    if not bap:
        assert r["bits_minmax_alloc"] == "" and r["mse_minmax_alloc"] == "", (cfg, r)
    else:
        wmm = allocate(_f64(mm)[:, 1:], tgt)
        assert int(r["bits_minmax_alloc"]) == int(wmm.sum()) <= math.floor(tgt * g), (cfg, r)
        ref = h["err"][gi, wmm, 0].sum() / n
        assert abs(float(r["mse_minmax_alloc"]) - ref) <= REL * ref, (cfg, r, ref)
        assert abs(hr["mse_minmax_alloc"] - ref) <= REL * ref, (cfg, hr, ref)


def _mults(step):
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    return list(MSE_MULTIPLIERS[::step])


# Each flag of the matrix - 4 / 8 bits; plain, -baw with the std prior, -baw -bap mse at targets 4 and 3.5; -bcw / -vcw off
# and on; the laplace and gaus clipping priors; NCHW and channels-last - on every input family, with the multiplier sweep
# thinned where nine widths multiply the host's work.
EDGE_CONFIGS = [dict(bits=4, mult=_mults(8)),
                dict(bits=4, baw=True, prior="gaus", mse_prior="gaus", bcw=True, mult=_mults(8)),
                dict(bits=4, baw=True, prior="mse", target=4, vcw=True, mult=_mults(8)),
                dict(bits=4, baw=True, prior="mse", target=3.5, mse_prior="gaus", bcw=True, vcw=True, channels_last=True,
                     mult=_mults(8)),
                dict(bits=8, mse_prior="gaus", bcw=True, mult=_mults(8))]


@pytest.mark.parametrize("cfg", range(len(EDGE_CONFIGS)))
def test_restatement_edge_rows(fq, monkeypatch, tmp_path, cfg):
    kw = dict(EDGE_CONFIGS[cfg])
    for name, w in _edge_weights():
        _check(fq, monkeypatch, tmp_path, name, w, **dict(kw, channels_last=kw.get("channels_last") and w.dim() == 4))


@pytest.mark.parametrize("kw", [dict(bits=4, bcw=True, channels_last=True, mult=_mults(8)),
                                dict(bits=8, mse_prior="gaus", mult=_mults(8)),
                                dict(bits=4, baw=True, prior="mse", target=4, mult=_mults(32))],
                         ids=["int4-bcw-cl", "int8-gaus", "int4-bap-mse"])
def test_restatement_resnet18(fq, monkeypatch, tmp_path, kw):
    for n, w in _weights("resnet18"):
        _check(fq, monkeypatch, tmp_path, n, w, **dict(kw, channels_last=kw.get("channels_last") and w.dim() == 4))


@pytest.mark.parametrize("kw", [dict(bits=4, baw=True, prior="gaus", mse_prior="gaus", vcw=True, mult=[2.0, 3.0]),
                                dict(bits=4, baw=True, prior="mse", target=3.5, bcw=True, vcw=True, mult=[3.0, 5.0])],
                         ids=["baw-std-vcw", "bap-mse-3.5"])
def test_restatement_resnet50_shapes(fq, monkeypatch, tmp_path, kw):
    for w in _shapes("resnet50"):
        _check(fq, monkeypatch, tmp_path, "x".join(map(str, w.shape)), w, **kw)


@pytest.mark.parametrize("kw", [dict(bits=4, baw=True, prior="mse", target=4, bcw=True, mult=_mults(8)),
                                dict(bits=8, mse_prior="gaus")], ids=["bap-mse-bcw", "int8-default-sweep"])
def test_restatement_vgg16_fc6_rows(fq, monkeypatch, tmp_path, kw):
    for n, w in _vgg_fc6_rows():
        _check(fq, monkeypatch, tmp_path, n, w, **kw)


def test_nan_row_keeps_minmax_and_raises(fq, monkeypatch, tmp_path):
    """A NaN in a row makes every candidate's error NaN: the row keeps min/max, the width allocation raises the device
    flag, and finish() raises the documented ValueError after writing the report."""
    w = (torch.randn(7, 27, generator=torch.Generator().manual_seed(3)) * 0.05).cuda()
    w[3, 5] = math.nan
    q = _quantizer(fq, 4, True, "mse", _mults(8), target=4)
    q.weight_mse.report = str(tmp_path / "report.csv")
    spy = _Spy(monkeypatch)
    q(w, "nan", weight_correction=(False, False))
    table = spy.calls["fused"][0][2]
    grid, _ = spy.calls["clip_mse_grid"][0][2]
    mm, _ = spy.calls["clip_mse"][0][2]
    qa, qk, _ = spy.calls["quantize_weights_given"][0]
    assert torch.isnan(grid[3, 1:]).all() and torch.isnan(mm[3, 1:]).all()
    assert torch.isfinite(grid[[0, 1, 2, 4, 5, 6], 1:]).all()
    assert np.array_equal([float(qa[1][3]), float(qa[2][3])], [float(table[3, 1] - table[3, 0]), float(table[3, 0])],
                          equal_nan=True)
    assert int(q.weight_mse.status(w.device).item()) == 1
    with pytest.raises(ValueError) as e:
        q.weight_mse.finish()
    assert str(e.value) == ("clip_weight='mse': a weight's error table holds NaN or Inf, so its width allocation is not "
                            "defined (bit_alloc.allocate refuses such tables)")
    with open(str(tmp_path / "report.csv")) as f:
        assert [r["id"] for r in csv.DictReader(f)] == ["nan"]
