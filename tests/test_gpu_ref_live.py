"""GPU parity against the REFERENCE ITSELF, live on the GPU, at BASELINE sizes.

oracle/build_oracle.py stages the reference's Python path (unmodified) and compiles its CUDA extension (unmodified)
under the git-ignored oracle/_ref/.  Here the reference's ``IntQuantizer``
(int_quantizer.py:56-632) runs on the same CUDA tensor as our kernels, for every distinct ResNet-50 / ResNet-101
activation layout at the BASELINE batch sizes (512 per GPU; 128 per GPU for the 8-GPU ResNet-101 config), in contiguous
NCHW **and** channels-last memory:

  tier (i)   the reference's own (delta, offset, bit_alloc) fed to our given-parameter kernels -> output BIT-EXACT;
  tier (ii)  end to end: our on-device statistics / parameters within 1e-5 relative of the reference's, allocated bit
             widths identical, outputs equal except a measured, bounded fraction of one-step flips.

The measured flip fractions and parameter errors are written to $FQB_REPORT_DIR/parity_live.json when that variable is set.
"""
import json
import os
import time

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FLIP_FRAC = 5e-6     # tier (ii) bound on the fraction of elements that may land one step away (measured on an H100: <= 3.2e-7)
FLIP_FRAC_MODEL = 5e-5  # ... layer by layer inside a model, incl. the compiled leaf's round-half-away grid (H100: <= 8.5e-6)
PARAM_RTOL = 1e-5    # north_star: parameters / outputs within 1e-5 relative
REPORT = {}


def _params(**over):
    p = dict(clipping="laplace", stats_kind="mean", kld=False, pcq_weights=True, pcq_act=True, bit_alloc_act=True,
             bit_alloc_weight=True, bcorr_act=False, bcorr_weight=True, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    p.update(over)
    return p


@pytest.fixture(scope="module")
def ref():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import ref_live
    if not ref_live.available():
        pytest.skip("oracle/_ref (staged reference + its compiled extension) not built")
    return ref_live.load()


@pytest.fixture(scope="module")
def fq():
    import cnn_quantization_b200 as m
    m._lib.load()
    return m


def _dump_report():
    out = os.environ.get("FQB_REPORT_DIR")
    if not out:
        return
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "parity_live.json"), "w") as f:
            json.dump(REPORT, f, indent=1, sort_keys=True)
    except OSError:
        pass


def _activation(n, c, hw, seed):
    """A conv-output-like tensor: per-channel scale U(0.1, 3) and shift N(0, 0.5) (SURVEY.md 8d)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, c, hw, hw, device="cuda", generator=g)
    scale = torch.rand(c, device="cuda", generator=g) * 2.9 + 0.1
    shift = torch.randn(c, device="cuda", generator=g) * 0.5
    return x.mul_(scale.view(1, c, 1, 1)).add_(shift.view(1, c, 1, 1))


def _rel(a, b, floor=None):
    """max |a - b| / max(|b|, floor): ``floor`` (scalar or per-channel tensor) is the magnitude that matters when b itself
    may be near zero (a mean is compared on the scale of the channel's std, an offset on the scale of its range)."""
    a, b = a.double().flatten(), b.double().flatten()
    den = b.abs().clamp_min(1e-30)
    if floor is not None:
        den = torch.maximum(den, floor.double().flatten() if torch.is_tensor(floor) else torch.full_like(den, floor))
    return float(((a - b).abs() / den).max())


def _flips(y, y_ref, step_per_channel):
    """(fraction of elements beyond 1e-5 relative, worst difference in quantization steps) - computed on the device."""
    tol = 1e-5 * torch.maximum(y.abs(), y_ref.abs()) + 1e-9
    diff = (y - y_ref).abs()
    bad = diff > tol
    nbad = int(bad.sum())
    if nbad == 0:
        return 0.0, 0.0
    steps = diff / step_per_channel.view(1, -1, 1, 1).clamp_min(1e-30)
    return nbad / y.numel(), float(steps[bad].max())


# every distinct (C, H) of the hooked conv outputs of ResNet-50 / ResNet-101 (SURVEY.md 8d census)
LAYOUTS = [(64, 112), (64, 56), (256, 56), (128, 56), (128, 28), (512, 28), (256, 28), (256, 14), (1024, 14), (512, 14),
           (512, 7), (2048, 7)]


@pytest.mark.parametrize("c,hw", LAYOUTS)
@pytest.mark.parametrize("n", [512, 128])
def test_w4a4_activation_layouts_vs_live_reference(ref, fq, n, c, hw):
    """BASELINE configs[2] / [3] activation path (-pcq_a -c laplace -baa, int4) on one layout: a6 -> a7 -> a8 -> a9 -> a4
    -> a3 of the reference next to ONE fused launch of ours, NCHW and channels-last."""
    from oracle.ref_live import LeafSpy
    from cnn_quantization_b200 import ops
    idx = LAYOUTS.index((c, hw))
    half_range = idx % 3 != 2                       # 2/3 of the hooked convs feed a ReLU (33 of 53 in ResNet-50)
    x = _activation(n, c, hw, seed=1000 * n + idx)
    rq = ref.int_quantizer("int4", _params())
    rq.pcq_w = False                                # the 'activation' entry of __fill_quantizers__ (:455-461)
    rq.half_range = half_range
    t0 = time.time()
    with LeafSpy(rq) as spy:
        want = rq(x, "conv%d_activation" % idx, "activation")
    torch.cuda.synchronize()
    t_ref = time.time() - t0
    kind, r_delta, r_offset, r_bits = spy.calls[-1]
    assert kind == "torch" and r_bits is not None and r_bits.numel() == c
    r_stats = rq.__act_stats_perchannel__(x, ["min", "max", "b", "std"], avg_over_batch=False)
    r_mean = rq.__act_stats_perchannel__(x, ["mean"], avg_over_batch=True)["mean"]
    r_offset = r_offset.reshape(-1).expand(c) if r_offset.numel() == 1 else r_offset.reshape(-1)
    qmax = 2.0 ** r_bits - 1
    r_scale = torch.where(qmax > 0, r_delta / qmax, torch.zeros_like(r_delta)).clamp_min(1e-8)

    q = fq.int_quantizer("int4", _params())
    q.pcq_w = False
    q.half_range = half_range
    q.export_stats = True
    rec = {"half_range": half_range, "elements": x.numel(), "reference_s": round(t_ref, 3)}
    for fmt in ("nchw", "nhwc"):
        xin = x if fmt == "nchw" else x.contiguous(memory_format=torch.channels_last)
        # ---- tier (i): the reference's parameters through our given-parameter kernel: bit-exact
        got_a = ops.quantize1(xin, r_delta.contiguous(), r_offset.contiguous(), 4, bits=r_bits.contiguous(),
                              layout=(n, c, hw * hw))
        assert torch.equal(got_a, want), "%s: given-parameter output differs from the reference" % fmt
        # ---- tier (ii): end to end
        got = q(xin, "conv%d_activation" % idx, "activation")
        st = q.last_stats
        errs = {"min": _rel(st[:, 0], r_stats["min"]) if not half_range else 0.0, "max": _rel(st[:, 1], r_stats["max"]),
                "mean": _rel(st[:, 2], r_mean, r_stats["std"]), "b": _rel(st[:, 3], r_stats["b"]),
                "std": _rel(st[:, 4], r_stats["std"]), "delta": _rel(st[:, 5], r_delta),
                "offset": _rel(st[:, 6], r_offset, r_delta)}
        # bit widths: identical, except that a channel whose log2(bins) sits within fp32 rounding of x.5 may land on the
        # other side (the reference's fp32 std vs our float64 accumulation): at most one such channel, off by exactly one
        # bit, reported, and left out of the element-wise comparison (its delta / offset follow its bit width)
        off = (st[:, 7] != r_bits).nonzero().flatten().tolist()
        bits_equal = not off
        assert len(off) <= 1 and all(abs(float(st[c_, 7]) - float(r_bits[c_])) == 1.0 for c_ in off), (fmt, off)
        keep = torch.ones(c, dtype=torch.bool, device=x.device)
        keep[off] = False
        errs["delta"], errs["offset"] = _rel(st[keep, 5], r_delta[keep]), _rel(st[keep, 6], r_offset[keep], r_delta[keep])
        frac, worst = _flips(got[:, keep], want[:, keep], r_scale[keep])
        rec[fmt] = {"flip_fraction": frac, "worst_steps": worst, "bits_identical": bits_equal, "bit_boundary_channels": off,
                    "max_rel_err": {k: float("%.3g" % v) for k, v in errs.items()},
                    "bit_widths": sorted(set(int(v) for v in r_bits.tolist()))}
        REPORT["act %dx%dx%dx%d" % (n, c, hw, hw)] = rec
        _dump_report()
        assert errs["max"] == 0.0 and errs["min"] == 0.0, errs
        for k in ("mean", "b", "std", "delta", "offset"):
            assert errs[k] <= PARAM_RTOL, (fmt, k, errs[k])
        assert frac <= FLIP_FRAC and worst <= 1.01, (fmt, frac, worst)
        del got, got_a
    print("[parity-live] %4dx%4dx%3dx%3d half_range=%d  flips nchw %.2e nhwc %.2e  (reference %.2fs)" % (
        n, c, hw, hw, half_range, rec["nchw"]["flip_fraction"], rec["nhwc"]["flip_fraction"], t_ref))


@pytest.mark.parametrize("case", ["maxpool", "fc"])
def test_int8_minmax_tensors_vs_live_reference(ref, fq, case):
    """The two mode-B tensors of every W4A4 forward and every tensor of configs[1]: gemmlowpMinMaxQuantize -> the
    reference's compiled kernel (a11 -> a2 -> a1) vs our fused launch, batch 512."""
    torch.manual_seed(7)
    if case == "maxpool":
        x = torch.relu(_activation(512, 64, 56, seed=77))
        tag, tid = "activation_pooling", "maxpool0_out"
    else:
        x = torch.randn(512, 1000, device="cuda") * 3
        tag, tid = "activation_classifier", "linear0_activation"
    for half_range in (False, True):
        if case == "fc" and half_range:
            continue
        rq = ref.int_quantizer("int8", _params(clipping="no", pcq_act=False, pcq_weights=False))
        rq.half_range = half_range
        want = rq(x, tid, tag)
        q = fq.int_quantizer("int8", _params(clipping="no", pcq_act=False, pcq_weights=False))
        q.half_range = half_range
        q.export_stats = True
        formats = ("nchw", "nhwc") if x.dim() == 4 else ("nchw",)
        for fmt in formats:
            xin = x if fmt == "nchw" else x.contiguous(memory_format=torch.channels_last)
            got = q(xin, tid, tag)
            step = q.last_stats[0, 8].reshape(1)
            tol = 1e-5 * torch.maximum(got.abs(), want.abs()) + 1e-9
            bad = (got - want).abs() > tol
            frac = float(bad.float().mean())
            worst = float(((got - want).abs() / step).max())
            REPORT["int8 %s %s half_range=%d" % (case, fmt, half_range)] = {"flip_fraction": frac, "worst_steps": worst}
            _dump_report()
            assert frac <= FLIP_FRAC_MODEL and worst <= 1.01, (case, fmt, frac, worst)


@pytest.mark.parametrize("arch", ["resnet50", "resnet101"])
def test_quantize_model_weights_vs_live_reference_manager(ref, fq, arch):
    """a5 + a9 + a13 at full model size: ``quantize_model`` of the reference's manager (per-out-channel int4 weights, bit
    allocation, its torch bias correction) vs ours (one fused launch per weight tensor)."""
    from oracle import ref_live
    from cnn_quantization_b200 import manager as M, pipeline
    flags = dict(pipeline.CONFIGS["%s_w4a4" % arch])
    args = M.make_args(**flags)
    model_ref, rqm = ref_live.build_reference_model(args, M.get_params(args), "cuda")
    rqm.__exit__()
    model, qm = pipeline.build_quantized_model(flags, "cuda")
    qm.detach()
    worst_frac, n_tensors, total = 0.0, 0, 0
    for (n1, p1), (n2, p2) in zip(model.named_parameters(), model_ref.named_parameters()):
        assert n1 == n2
        if p1.dim() < 2:
            assert torch.allclose(p1, p2, rtol=1e-6, atol=1e-7), n1      # folded-BN biases: same torch ops
            continue
        scale = p2.abs().amax(dim=tuple(range(1, p2.dim())), keepdim=True).clamp_min(1e-12)
        bad = (p1 - p2).abs() > 1e-5 * scale
        frac = float(bad.float().mean())
        worst_frac = max(worst_frac, frac)
        n_tensors += 1
        total += p1.numel()
        assert frac <= 2e-3, (n1, frac)
    REPORT["weights %s_w4a4" % arch] = {"tensors": n_tensors, "elements": total, "worst_flip_fraction": worst_frac}
    _dump_report()


@pytest.mark.parametrize("config,batch,channels_last", [("resnet50_w4a4", 64, True), ("resnet50_w4a4", 32, False),
                                                        ("resnet101_w4a4", 128, True), ("resnet50_w8a8", 64, True),
                                                        ("vgg16_w4a4", 16, True)])
def test_layerwise_differential_vs_live_reference(ref, fq, config, batch, channels_last):
    """Layer-wise differential on real activations: our hooked model runs a 224x224 batch; at EVERY quantize_instant call
    the same GPU input (conv bias added, as the reference's convolution would have) also goes through the reference's
    quantizer for that tag, and the two outputs are compared.  Replaces the loose logits cosine of round 1."""
    from cnn_quantization_b200 import manager as M, pipeline
    flags = dict(pipeline.CONFIGS[config])
    args = M.make_args(**flags)
    ref_ops = ref.iqm.TruncationOpManagerInference(args, M.get_params(args))   # the reference's tag -> quantizer table
    model, qm = pipeline.build_quantized_model(flags, "cuda", channels_last=channels_last)
    x, _ = pipeline.synthetic_batch(batch, seed=3, channels_last=channels_last)
    x = x.cuda()
    if channels_last:
        x = x.contiguous(memory_format=torch.channels_last)
    rows = []
    orig = qm.quantize_instant

    boundary = []   # (layer, channel, our bits, reference bits): bit-allocation rounding-boundary cases, see below
    fused_blocks = []   # layers whose launch also did the block's residual add + ReLU
    pooled_layers = []  # layers whose launch also did the max pooling behind them
    deferred, deferred_used = {}, []   # shortcut convolutions quantized inside the launch of the block's last convolution

    def spy(tensor, id, tag="", stat_id=None, half_range=False, override_att=None, verbose=False, **extra):
        from oracle.ref_live import LeafSpy
        bias = extra.get("bias")
        ref_in = tensor.contiguous().clone() if bias is None else (tensor + bias.view(1, -1, 1, 1)).contiguous()
        q = qm.get_quantizer(tag)
        q.export_stats, q.last_stats = True, None
        out = orig(tensor, id, tag, stat_id, half_range, override_att, verbose, **extra)
        rq = ref_ops.get_quantizer(tag)
        rq.half_range = half_range
        with LeafSpy(rq) as leaf:
            want = rq(ref_in, id, tag)
        if getattr(out, "_fq_deferred", None) is not None:
            # the shortcut of a down-sampling block: our launch stopped after the statistics and handed the raw tensor on;
            # the launch that takes it as `residual` quantizes it - compared there, against this reference result
            # (channels whose bit width sits on a rounding boundary, see below, are carried along)
            excl = []
            r_bits = leaf.calls[-1][3] if leaf.calls and leaf.calls[-1][0] == "torch" else None
            if r_bits is not None and q.last_stats is not None and q.last_stats.shape[0] == r_bits.numel():
                o_bits = q.last_stats[:, 7]
                excl = (o_bits != r_bits).nonzero().flatten().tolist()
                assert len(excl) <= 2, (id, "bit widths differ in %d channels" % len(excl))
                for c in excl:
                    assert abs(float(o_bits[c]) - float(r_bits[c])) == 1.0, (id, c, float(o_bits[c]), float(r_bits[c]))
                    boundary.append((id, c, float(o_bits[c]), float(r_bits[c])))
            deferred[id] = (out, want, excl)
            return out
        excl_res = []
        if getattr(out, "_fq_pooled", False):
            # the 2x2 max pooling behind this convolution ran inside our launch: pool the reference's quantized tensor
            pooled_layers.append(id)
            want = torch.nn.functional.max_pool2d(want, 2) if out._fq_pooled == 2 else torch.nn.functional.max_pool2d(want, 3, 2, 1)
        if getattr(out, "_fq_residual_fused", False):
            # the block's residual add + ReLU ran inside our quantization launch: apply the block's own two torch ops
            # (torchvision Bottleneck.forward: out += identity; out = relu(out)) to the reference's quantized tensor
            fused_blocks.append(id)
            res = extra["residual"]
            for did, (dt, dwant, dexcl) in deferred.items():
                if dt is res:
                    res = dwant   # the reference's quantized shortcut
                    excl_res = dexcl
                    deferred_used.append(did)
            mag = torch.maximum(want.abs(), res.abs())   # the sum cancels: tolerance on the operands' scale
            want = torch.relu(want + res)
        else:
            mag = want.abs()
        tol = 1e-5 * torch.maximum(out.abs(), mag) + 1e-9
        diff = (out - want).abs()
        bad = diff > tol
        for c in excl_res:
            bad[:, c] = False
            diff[:, c] = 0
        # Per-channel bit allocation rounds log2(bins): where the reference's value sits within fp32 rounding of x.5 its
        # own std (fp32 torch.std) and ours (float64 accumulation) can land on different sides - that channel then gets
        # the neighbouring bit width, a legitimate 1e-7 sensitivity of the reference algorithm, not an arithmetic error.
        # Such channels are identified by the captured bit widths (must differ by exactly one), counted, reported and
        # excluded from the element-wise comparison; at most 2 per layer are tolerated.
        r_bits = leaf.calls[-1][3] if leaf.calls and leaf.calls[-1][0] == "torch" else None
        if r_bits is not None and q.last_stats is not None and out.dim() == 4 and q.last_stats.shape[0] == r_bits.numel():
            o_bits = q.last_stats[:, 7]
            off = (o_bits != r_bits).nonzero().flatten().tolist()
            assert len(off) <= 2, (id, "bit widths differ in %d channels" % len(off))
            for c in off:
                assert abs(float(o_bits[c]) - float(r_bits[c])) == 1.0, (id, c, float(o_bits[c]), float(r_bits[c]))
                boundary.append((id, c, float(o_bits[c]), float(r_bits[c])))
                bad[:, c] = False
                diff[:, c] = 0
        levels = max(int(torch.unique(want[:1]).numel()), 2)
        span = float(want.max() - want.min())
        rows.append((id, tag, tuple(tensor.shape), float(bad.float().mean()), float(diff.max()), span, levels))
        return out

    qm.quantize_instant = spy
    with torch.no_grad():
        y = model(x)
    qm.detach()
    assert torch.isfinite(y).all()
    assert sorted(deferred_used) == sorted(deferred)   # every deferred shortcut was compared where it was consumed
    worst = max(r[3] for r in rows)
    REPORT["layerwise %s batch %d %s" % (config, batch, "nhwc" if channels_last else "nchw")] = {
        "hooked_tensors": len(rows), "worst_flip_fraction": worst,
        "mean_flip_fraction": sum(r[3] for r in rows) / len(rows),
        "worst_layer": max(rows, key=lambda r: r[3])[0],
        "launches_with_fused_block_epilogue": len(fused_blocks),
        "launches_with_fused_max_pooling": len(pooled_layers),
        "shortcuts_quantized_inside_that_launch": len(deferred_used),
        "bit_allocation_boundary_channels": ["%s ch %d: %g vs %g bits" % b for b in boundary]}
    _dump_report()
    for id, tag, shape, frac, dmax, span, levels in rows:
        assert frac <= FLIP_FRAC_MODEL, (id, tag, shape, frac)
        assert dmax <= span / 2 + 1e-6, (id, tag, shape, dmax, span)   # flips are single grid steps, never garbage


@pytest.mark.parametrize("config,min_cos", [("resnet50_w4a4", 0.95), ("resnet50_w8a8", 0.999)])
def test_dropin_alias_runs_the_unmodified_reference_manager(ref, config, min_cos, tmp_path):
    """SURVEY 8(b): the reference's OWN manager + model preparation, unmodified, in a fresh process, once as shipped and
    once after the zero-edit alias of INTEGRATION.md section 1.  In the aliased run every quantize_instant of the
    reference manager must have gone through libfqb200.so, and the logits must agree with the shipped reference."""
    import subprocess
    import sys
    import numpy as np
    runner = os.path.join(ROOT, "tests", "helpers", "dropin_runner.py")
    outs = {}
    for mode in ("reference", "dropin"):
        out = str(tmp_path / ("%s.npz" % mode))
        res = subprocess.run([sys.executable, runner, "--mode", mode, "--config", config, "--batch", "8", "--out", out],
                             capture_output=True, text=True, timeout=900)
        assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
        outs[mode] = np.load(out)
    assert str(outs["reference"]["quantizer_module"]) == "pytorch_quantizer.quantization.qtypes.int_quantizer"
    assert str(outs["dropin"]["quantizer_module"]).startswith("cnn_quantization_b200")
    # ResNet-50: 54 weight tensors + 55 hooked activations per forward, every one a launch of ours
    assert int(outs["dropin"]["launches"]) >= 109, int(outs["dropin"]["launches"])
    y, r = outs["dropin"]["logits"].astype(np.float64), outs["reference"]["logits"].astype(np.float64)
    assert np.isfinite(y).all() and y.shape == r.shape
    cos = float((y * r).sum() / (np.linalg.norm(y) * np.linalg.norm(r)))
    REPORT["dropin %s" % config] = {"cosine_vs_shipped_reference": cos, "launches": int(outs["dropin"]["launches"])}
    _dump_report()
    assert cos >= min_cos, cos
    assert abs(np.linalg.norm(y) / np.linalg.norm(r) - 1) < 0.1


class _Log(object):
    def __init__(self):
        self.rows = []

    def log_metric(self, name, value, **kw):
        self.rows.append((name, float(value), kw))


@pytest.mark.parametrize("positive", [True, False])
def test_mid_tread_entropy_vs_live_reference(ref, fq, positive):
    """SURVEY 8(f) rank 3 / README.md:135-140 (`-mtq -me`): the average activation entropy of the mid-tread grid.  The
    reference runs torch.unique over the float grid; ours histograms inside the apply phase (channels-last) or falls back
    to torch ops (NCHW).  Same tensor, same logger call, entropies within 2e-3 bit."""
    x = _activation(64, 64, 28, seed=4242)
    if positive:
        x = torch.relu(x)
    over = dict(mtd_quant=True, measure_entropy=True, bit_alloc_target_act=5.3, bit_alloc_target_weight=5.3)
    lr, lo = _Log(), _Log()
    rq = ref.int_quantizer("int4", _params(logger=lr, **over))
    rq.pcq_w, rq.force_positive = False, positive
    want = rq(x, "conv3_activation", "activation")
    q = fq.int_quantizer("int4", _params(logger=lo, **over))
    q.pcq_w, q.force_positive = False, positive
    got_cl = q(x.contiguous(memory_format=torch.channels_last), "conv3_activation", "activation")
    got_nchw = q(x, "conv3_activation", "activation")
    assert len(lr.rows) == 1 and len(lo.rows) == 2
    name, e_ref, kw = lr.rows[0]
    for (n2, e, kw2), got in zip(lo.rows, (got_cl, got_nchw)):
        assert n2 == name == "conv3_activation.entropy" and kw2["meterId"] == kw["meterId"] == "avg.entropy.act"
        assert kw2["weight"] == kw["weight"] == x.numel()
        assert abs(e - e_ref) <= 2e-3, (e, e_ref)
        bad = (got - want).abs() > 1e-5 * want.abs() + 1e-9
        assert float(bad.float().mean()) <= 1e-3
    REPORT["mid-tread entropy positive=%d" % positive] = {"reference_bits": e_ref, "ours_channels_last_bits": lo.rows[0][1],
                                                          "ours_nchw_bits": lo.rows[1][1]}
    _dump_report()
    # weights: per-output-channel symmetric grid, min/max range
    w = torch.randn(128, 64, 3, 3, device="cuda") * 0.05
    lr, lo = _Log(), _Log()
    rq = ref.int_quantizer("int4", _params(logger=lr, clipping="no", **over))
    wq_ref = rq(w, "layer.weight", "weight")
    q = fq.int_quantizer("int4", _params(logger=lo, clipping="no", **over))
    wq = q(w, "layer.weight", "weight")
    assert abs(lo.rows[0][1] - lr.rows[0][1]) <= 2e-3 and lo.rows[0][2]["meterId"] == "avg.entropy.weight"
    assert float(((wq - wq_ref).abs() > 1e-5 * wq_ref.abs() + 1e-9).float().mean()) <= 2e-3
