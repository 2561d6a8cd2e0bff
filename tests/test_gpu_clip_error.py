"""Clipping-error measurement on the GPU: ops.clip_error's candidate parameters against the host restatement of the same
rules, its sums against float64 torch sums over the candidate tensors (ops.quantize1 with those parameters), determinism,
the identity of the gaus / laplace candidates with the on-the-fly quantizers, and `-sm collect` with collect_err followed
by `-c mix -sm use` on the seeded ResNet-18."""
import numpy as np
import pandas as pd
import pytest
import torch

pytestmark = pytest.mark.gpu

GAUS = {1: 1.24, 2: 1.71, 3: 2.15, 4: 2.55, 5: 2.93, 6: 3.28, 7: 3.61, 8: 3.92}
GAUS_POS = {1: 1.71, 2: 2.15, 3: 2.55, 4: 2.93, 5: 3.28, 6: 3.61, 7: 3.92, 8: 4.2}
LAPLACE = {0: 1.05, 1: 1.86, 2: 2.83, 3: 3.89, 4: 5.03, 5: 6.2, 6: 7.41, 7: 8.64, 8: 9.89}
LAPLACE_POS = {0: 1.86, 1: 2.83, 2: 3.89, 3: 5.02, 4: 6.2, 5: 7.41, 6: 8.64, 7: 9.89, 8: 11.16}
# The kernel adds every x^2, (x - q)^2, x q, q^2 in float64 (products of two floats are exact there); only the order of
# the additions differs from torch's, so the sums agree to a few float64 roundings relative to the sum of magnitudes.
REL = 1e-12


@pytest.fixture(scope="module", autouse=True)
def need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def f32(v):
    return np.float32(v)


def host_params(table, num_bits, positive, bit_alloc, f64):
    """[G, 3, 6] (delta, offset, bits, scale, zero point, qmax) of the candidates lowp / gaus / laplace, by the rules of
    solve_range and make_leaf_param (torch leaf) in numpy float32 / float64."""
    T = table.cpu().numpy().astype(np.float32)
    out = np.zeros((T.shape[0], 3, 6), dtype=np.float32)
    with np.errstate(all="ignore"):
        for g in range(T.shape[0]):
            mn, mx, mean, b, sd = (f32(v) for v in T[g, :5])
            bits = f32(T[g, 7]) if bit_alloc else f32(num_bits)
            alphas = (f32((mx - mn) * f32(0.5)),
                      f32(sd * f32((GAUS_POS if positive else GAUS)[num_bits])),
                      f32(b * f32((LAPLACE_POS if positive else LAPLACE)[int(bits)])))
            for k, al in enumerate(alphas):
                if f64:
                    if positive:
                        dl, of = max(float(mean), 0.0) + float(al), 0.0
                    else:
                        dl, of = 2.0 * float(al), float(np.fmax(float(mn), float(mean) - float(al)))
                    delta, offset = f32(dl), f32(of)
                elif positive:
                    delta, offset = f32(np.fmax(mean, f32(0)) + al), f32(0)
                else:
                    rng = f32(f32(2) * al)
                    offset = f32(np.fmax(mn, f32(mean - al)))
                    delta = f32(f32(offset + rng) - offset)
                qmax = f32(2 ** int(bits) - 1)
                scale = f32(delta / qmax) if qmax > 0 else f32(0)
                scale = np.fmax(scale, f32(1e-8))
                zp = f32(np.rint(f32(f32(0) - f32(offset / scale))))
                out[g, k] = (delta, offset, bits, scale, zp, qmax)
    return out


def stats_table(x, layout, channels_last=False, num_bits=8, bit_alloc=False):
    from cnn_quantization_b200 import ops
    return ops.fused(x, layout, stats_only=True, channels_last=channels_last, num_bits=num_bits, bit_alloc=bit_alloc,
                     bit_alloc_round=True, bit_alloc_target=num_bits)


def torch_sums(x, params, layout, num_bits):
    """[G, 10] float64 sums over the candidate tensors quantize1 produces with ``params`` (the kernel's) on the NCHW
    order of ``x``, and the matching sums of magnitudes for the tolerance."""
    from cnn_quantization_b200 import ops
    outer, groups, inner = layout
    xs = x.contiguous().view(outer, groups, inner)
    xd = xs.double()
    p = params
    cols, mags = [xd.pow(2).sum((0, 2))], [xd.pow(2).sum((0, 2))]
    qs = []
    for k in range(3):
        if groups == 1:
            q = ops.quantize1(xs.view(-1), p[0, k, 0], p[0, k, 1], num_bits)
        else:
            q = ops.quantize1(xs, p[:, k, 0].contiguous(), p[:, k, 1].contiguous(), num_bits, bits=p[:, k, 2].contiguous(),
                              layout=layout)
        qs.append(q.view(outer, groups, inner).double())
    for q in qs:
        cols.append((xd - q).pow(2).sum((0, 2)))
        mags.append(cols[-1])
    for q in qs:
        cols.append((xd * q).sum((0, 2)))
        mags.append((xd * q).abs().sum((0, 2)))
    for q in qs:
        cols.append(q.pow(2).sum((0, 2)))
        mags.append(cols[-1])
    return torch.stack(cols, 1), torch.stack(mags, 1)


def check(x, layout, num_bits, positive, channels_last=False, bit_alloc=False):
    from cnn_quantization_b200 import ops
    f64 = layout[0] == 1 and layout[1] == 1
    table = stats_table(x, layout, channels_last, num_bits if bit_alloc else 8, bit_alloc)
    got, params = ops.clip_error(x, table, layout, channels_last, num_bits, positive, bit_alloc=bit_alloc, want_params=True)
    assert got.dtype == torch.float64 and got.shape == (layout[1], 10)
    want_p = host_params(table, num_bits, positive, bit_alloc, f64)
    np.testing.assert_array_equal(params.cpu().numpy(), want_p)   # bit for bit
    want, mag = torch_sums(x, params, layout, num_bits)
    err = ((got - want).abs() / mag.clamp_min(1e-300)).max().item()
    assert err < REL, err
    return got


@pytest.mark.parametrize("shape", [(2, 3, 64, 64), (3, 5, 7, 7), (1, 1, 1, 13)])
@pytest.mark.parametrize("num_bits,positive", [(4, False), (4, True), (8, False), (2, True)])
def test_per_tensor(shape, num_bits, positive):
    g = torch.Generator(device="cuda").manual_seed(sum(shape) + num_bits)
    x = torch.randn(shape, device="cuda", generator=g) * 2 + 0.3
    check(x, (1, 1, x.numel()), num_bits, positive)


@pytest.mark.parametrize("shape", [(4, 96, 14, 14), (3, 5, 7, 7), (2, 7, 9, 11), (8, 64, 28, 28)])
@pytest.mark.parametrize("num_bits,positive,bit_alloc", [(4, False, False), (4, True, True), (3, False, True), (8, True, False)])
def test_per_channel_nchw(shape, num_bits, positive, bit_alloc):
    g = torch.Generator(device="cuda").manual_seed(sum(shape) * 7 + num_bits)
    x = torch.randn(shape, device="cuda", generator=g) * torch.linspace(0.1, 3, shape[1], device="cuda").view(1, -1, 1, 1)
    n, c = shape[:2]
    check(x, (n, c, x.numel() // (n * c)), num_bits, positive, bit_alloc=bit_alloc)


@pytest.mark.parametrize("shape", [(8, 96, 10, 12), (2, 2048, 7, 7), (3, 36, 5, 5)])
@pytest.mark.parametrize("num_bits,positive,bit_alloc", [(4, False, True), (8, True, False)])
def test_per_channel_channels_last(shape, num_bits, positive, bit_alloc):
    from cnn_quantization_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(sum(shape) * 3 + num_bits)
    x = (torch.randn(shape, device="cuda", generator=g) + 0.5).contiguous(memory_format=torch.channels_last)
    assert ops.cl_eligible(x)
    n, c = shape[:2]
    check(x, (n, c, x.numel() // (n * c)), num_bits, positive, channels_last=True, bit_alloc=bit_alloc)


def test_view_at_storage_offset_one():
    base = torch.randn(2 * 3 * 32 * 32 + 1, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    x = base[1:].view(2, 3, 32, 32)
    assert x.data_ptr() % 16 != 0
    check(x, (1, 1, x.numel()), 4, False)
    check(x, (2, 3, 32 * 32), 4, False)


def test_nan_propagates():
    from cnn_quantization_b200 import ops
    x = torch.randn(2, 4, 8, 8, device="cuda")
    x[1, 2, 3, 4] = float("nan")
    layout = (2, 4, 64)
    got = ops.clip_error(x, stats_table(x, layout), layout, False, 4, False).cpu()
    assert torch.isnan(got[2]).all()
    assert torch.isfinite(got[[0, 1, 3]]).all()
    t = (1, 1, x.numel())
    assert torch.isnan(ops.clip_error(x, stats_table(x, t), t, False, 4, False)).all()


def test_deterministic_across_runs_and_grids():
    from cnn_quantization_b200 import ops
    x = torch.randn(16, 64, 28, 28, device="cuda", generator=torch.Generator(device="cuda").manual_seed(9))
    xcl = x.contiguous(memory_format=torch.channels_last)
    for t, layout, cl in ((x, (1, 1, x.numel()), False), (x, (16, 64, 784), False), (xcl, (16, 64, 784), True)):
        table = stats_table(t, layout, cl)
        runs = [ops.clip_error(t, table, layout, cl, 4, False, max_ctas=m) for m in (0, 0, 7, 1)]
        for r in runs[1:]:
            assert torch.equal(r, runs[0])


@pytest.mark.parametrize("per_channel,cl", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("num_bits,positive,bit_alloc", [(4, False, True), (4, True, False), (8, False, False)])
def test_candidates_are_the_on_the_fly_quantizers(per_channel, cl, num_bits, positive, bit_alloc):
    """Given the statistics table of a `-sm no -c gaus` / `-c laplace` launch, the gaus / laplace candidates' parameters
    equal the ones that launch solved and applied."""
    import cnn_quantization_b200 as fq
    from cnn_quantization_b200 import ops
    x = torch.randn(4, 32, 12, 12, device="cuda", generator=torch.Generator(device="cuda").manual_seed(num_bits)) * 1.5
    if cl:
        x = x.contiguous(memory_format=torch.channels_last)
    layout = (4, 32, 144) if per_channel else (1, 1, x.numel())
    ba = bit_alloc and per_channel
    for k, clip in ((1, "gaus"), (2, "laplace")):
        p = dict(clipping=clip, stats_kind="mean", kld=False, pcq_weights=False, pcq_act=per_channel, bit_alloc_act=bit_alloc,
                 bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
                 bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
                 logger=None, mtd_quant=False)
        q = fq.int_quantizer("int%d" % num_bits, p)
        q.half_range = positive
        q.export_stats = True
        q(x.clone(), "conv1_activation", "activation")
        table = q.last_stats
        _, params = ops.clip_error(x, table, layout, cl, num_bits, positive, bit_alloc=ba, want_params=True)
        exported = table[:, 5:11].cpu().numpy()   # delta offset bits scale zero_point qmax
        np.testing.assert_array_equal(params[:, k].cpu().numpy(), exported)


def test_vgg16_stem_at_n672():
    """2.16 G elements: 64-bit offsets per tensor and per channel (NCHW), against the sums over 24-sample slices."""
    from cnn_quantization_b200 import ops
    n, c, h, w = 672, 64, 224, 224
    x = torch.empty((n, c, h, w), device="cuda")
    g = torch.Generator(device="cuda").manual_seed(16)
    for i in range(0, n, 96):
        x[i:i + 96].normal_(generator=g)
    for layout in ((1, 1, x.numel()), (n, c, h * w)):
        table = stats_table(x, layout)
        got, params = ops.clip_error(x, table, layout, False, 4, True, want_params=True)
        want = torch.zeros_like(got)
        mag = torch.zeros_like(got)
        for i in range(0, n, 24):
            xs = x[i:i + 24]
            sl = (1, 1, xs.numel()) if layout[1] == 1 else (24, c, h * w)
            s, m = torch_sums(xs, params, sl, 4)
            want += s
            mag += m
        err = ((got - want).abs() / mag.clamp_min(1e-300)).max().item()
        assert err < 1e-11, err   # the slices add up in another order again
        del table, got


# ---- end to end against the reference: ResNet-18 collect with collect_err, then `-c mix -sm use` ------------------------------
# (tests/golden/make_clip_error_golden.py: the reference's collect with its quantized candidates wired in, per tensor and
# with -pcq_a -baa, and its `-c mix -sm use` logits on those statistics)
import os  # noqa: E402
import pickle  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
REF_ERR = os.path.join(GOLD, "ref_stats_err")
PCQ = dict(per_channel_quant_act=True, bit_alloc_act=True)
W4A4_MIX = dict(qtype="int4", qweight="int4", clipping="mix", per_channel_quant_weights=True, bit_alloc_weight=True,
                bias_corr_weight=True)
# The activations themselves come from GPU convolutions here and CPU ones in the reference (the other statistics agree
# to test_gpu_stats.py's 2e-3), so an element can sit on the other side of a grid boundary.  Per tensor that moves mse by
# far less than 1e-4 relative and cos by a few 1e-6 (4.6e-6 seen on conv15).  A per-channel row of the 64x64 fixture
# input can hold as few as 8 elements, where one such element moves its mse by percents: there at most 2 % of the rows
# may exceed the bounds.  The largest deviations are printed.
MSE_REL, COS_ABS, PC_OUTLIERS = 1e-4, 5e-5, 0.02
CANDS = ("lowp", "gaus", "laplace")


def batches():
    rs = np.random.RandomState(2024)
    return [torch.from_numpy(rs.standard_normal((2, 3, 64, 64)).astype(np.float32)) for _ in range(2)]


def run(cfg, device="cuda"):
    from cnn_quantization_b200 import pipeline
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    model, qm = pipeline.build_quantized_model(dict(arch="resnet18", stats_folder="resnet18", **cfg), device)
    outs = []
    with torch.no_grad():
        for x in batches():
            outs.append(model(x.to(device)).cpu().numpy())
    qm.__exit__()
    return np.stack(outs)


def mix_choice(lowp, gaus, laplace):
    c = np.where(np.asarray(gaus) < np.asarray(laplace), 1, 2)
    return np.where(np.asarray(lowp) < np.asarray(gaus), 0, c)


def decided(lowp, gaus, laplace, tol):
    """Where both comparisons of the rule are decided by more than ``tol`` relative."""
    lowp, gaus, laplace = (np.asarray(v, dtype=np.float64) for v in (lowp, gaus, laplace))
    gap = lambda a, b: np.abs(a - b) > tol * np.maximum(np.abs(a), np.abs(b))
    return gap(lowp, gaus) & gap(gaus, laplace)


def compare(ours, ref, what, worst, outliers=None):
    """mse within MSE_REL relative, cos within COS_ABS absolute; records the largest deviations in ``worst``.  With
    ``outliers`` (per channel) rows beyond the bounds are counted there instead of failing."""
    for k in CANDS:
        for kind in ("min", "mean", "max"):
            a = np.asarray(ours["%s_mse_%s" % (kind, k)], dtype=np.float64)
            b = np.asarray(ref["%s_mse_%s" % (kind, k)], dtype=np.float64)
            rel = np.atleast_1d(np.abs(a - b) / np.maximum(np.abs(b), 1e-30))
            a = np.asarray(ours["%s_cos_%s" % (kind, k)], dtype=np.float64)
            b = np.asarray(ref["%s_cos_%s" % (kind, k)], dtype=np.float64)
            dc = np.atleast_1d(np.abs(a - b))
            worst["mse"] = max(worst["mse"], float(rel.max()))
            worst["cos"] = max(worst["cos"], float(dc.max()))
            if outliers is None:
                assert (rel <= MSE_REL).all(), (what, kind, k, float(rel.max()))
                assert (dc <= COS_ABS).all(), (what, kind, k, float(dc.max()))
            else:
                outliers[0] += int((rel > MSE_REL).sum()) + int((dc > COS_ABS).sum())
                outliers[1] += 2 * rel.size


def test_resnet18_collect_err_against_the_reference(tmp_path):
    base = str(tmp_path)
    run(dict(stats_mode="collect", qtype="int4", qweight="int4", stats_base_dir=base, collect_err=True))
    run(dict(stats_mode="collect", qtype="int4", qweight="int4", stats_base_dir=base, collect_err=True, **PCQ))
    ref_choice = np.load(os.path.join(GOLD, "ref_stats_err_logits.npz"))
    worst = {"mse": 0.0, "cos": 0.0}
    ours = pd.read_csv(os.path.join(base, "statistics", "resnet18", "resnet18_summary.csv"), index_col=0)
    ref = pd.read_csv(os.path.join(REF_ERR, "statistics", "resnet18", "resnet18_summary.csv"), index_col=0)
    assert list(ours.columns) == list(ref.columns) and list(ours.index) == list(ref.index)
    for stat in ("min", "max", "mean", "std", "b", "mean_abs", "kurtosis", "dim"):   # test_gpu_stats.py's bounds
        for kind in ("min", "mean", "max"):
            col = "%s_%s" % (kind, stat)
            a, b = ours[col].to_numpy(dtype=np.float64), ref[col].to_numpy(dtype=np.float64)
            assert np.allclose(a, b, rtol=2e-3, atol=2e-4 * (np.abs(b).max() + 1e-12)), col
    for layer in ref.index:
        compare(ours.loc[layer], ref.loc[layer], layer, worst)
        mse = [ours.loc[layer, "mean_mse_" + k] for k in CANDS]
        if decided(*mse, tol=2 * MSE_REL):
            assert int(mix_choice(*mse)) == int(ref_choice["choice_tensor/" + layer]), layer
    path = os.path.join("statistics", "per_channel", "resnet18", "resnet18_statistics_perchannel_summary.pkl")
    with open(os.path.join(base, path), "rb") as f:
        mine = pickle.load(f)
    with open(os.path.join(REF_ERR, path), "rb") as f:
        theirs = pickle.load(f)
    assert sorted(mine) == sorted(theirs)
    worst_pc, outliers = {"mse": 0.0, "cos": 0.0}, [0, 0]
    for layer in theirs:
        assert list(mine[layer].columns) == list(theirs[layer].columns)
        compare({c: mine[layer][c].to_numpy() for c in mine[layer].columns},
                {c: theirs[layer][c].to_numpy() for c in theirs[layer].columns}, layer, worst_pc, outliers)
        mse = [mine[layer]["mean_mse_" + k].to_numpy() for k in CANDS]
        keep = decided(*mse, tol=2 * MSE_REL)
        np.testing.assert_array_equal(mix_choice(*mse)[keep], ref_choice["choice_channel/" + layer][keep])
    print("largest deviation from the reference: per tensor mse %.3g relative, cos %.3g absolute; per channel mse %.3g, "
          "cos %.3g, %d of %d entries beyond the bounds" % (worst["mse"], worst["cos"], worst_pc["mse"], worst_pc["cos"],
                                                             outliers[0], outliers[1]))
    assert outliers[0] <= PC_OUTLIERS * outliers[1], outliers


@pytest.mark.parametrize("name,flags", [("use_mix_w4a4", {}), ("use_mix_w4a4_pcq", PCQ)])
def test_mix_use_mode_against_the_reference(name, flags):
    """`-c mix -sm use` on the reference's statistics: logits under test_gpu_stats.py's use-mode bound, and the same
    run twice is bit-identical (parameters solved once per layer, then given-parameter launches)."""
    ref = np.load(os.path.join(GOLD, "ref_stats_err_logits.npz"))[name]
    got = run(dict(stats_mode="use", stats_base_dir=REF_ERR, **W4A4_MIX, **flags))
    assert got.shape == ref.shape
    cos = float((got * ref).sum() / (np.linalg.norm(got) * np.linalg.norm(ref)))
    assert cos > 0.97, cos
    assert abs(np.linalg.norm(got) / np.linalg.norm(ref) - 1) < 0.08
    np.testing.assert_array_equal(run(dict(stats_mode="use", stats_base_dir=REF_ERR, **W4A4_MIX, **flags)), got)
