"""Clipping-error columns (collect_err) and `-c mix` without a GPU: the C ABI's argument checks, the quantizer settings the
manager hands each collect call site, the flag's validation, the `mix` selection on crafted statistics, `mix` on the
reference's own per-tensor statistics (tests/golden/ref_stats, error columns NaN: exactly `-c laplace`) and the NaN
columns of a default collect."""
import ctypes
import os

import numpy as np
import pandas as pd
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---- C ABI ------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def lib():
    import __graft_entry__
    __graft_entry__.build()
    from cnn_quantization_b200 import _lib
    return _lib.load()


def test_abi_workspace_bytes(lib):
    ws = lib.fqb200_clip_error_workspace_bytes
    assert ws(1, 1, 16384, 0) == 10 * 8                    # 16384-element units
    assert ws(1, 1, 16385, 0) == 2 * 10 * 8
    assert ws(512, 64, 112 * 112, 0) == 64 * 392 * 10 * 8
    assert ws(8, 96, 10 * 12, 1) == 96 * 2 * 10 * 8        # channels-last: 512-pixel units per channel
    assert ws(0, 4, 4, 0) == 0 and b"> 0" in lib.fqb200_last_error()
    assert ws(2, 6, 4, 1) == 0 and b"C %" in lib.fqb200_last_error()
    assert ws(2, 4096, 4, 1) == 0
    assert ws(2, 3, 1 << 31, 0) == 0 and b"2^32" in lib.fqb200_last_error()
    assert ws(1, 1, 1 << 33, 0) == ((1 << 33) // 16384) * 80   # one group of one row: any length


def test_abi_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 12)
    need = lib.fqb200_clip_error_workspace_bytes(2, 4, 64, 0)

    def call(inp=buf, outer=2, groups=4, inner=64, cl=0, stats=buf, bits=4, bit_alloc=0, out=buf, ws=buf, nbytes=need,
             ctas=0):
        return lib.fqb200_clip_error(inp, outer, groups, inner, cl, stats, bits, 0, bit_alloc, 0, out, None, ws, nbytes,
                                     ctas, None)

    assert call(outer=0) == _lib.ERR_INVALID
    assert call(cl=1, groups=6) == _lib.ERR_INVALID
    assert call(inp=None) == _lib.ERR_INVALID and b"null" in lib.fqb200_last_error()
    assert call(stats=None) == _lib.ERR_INVALID
    assert call(out=None) == _lib.ERR_INVALID
    assert call(bits=0) == _lib.ERR_INVALID and b"num_bits" in lib.fqb200_last_error()
    assert call(bits=9) == _lib.ERR_INVALID
    assert call(bits=8, bit_alloc=1) == _lib.ERR_INVALID and b"bit_alloc" in lib.fqb200_last_error()
    assert call(ctas=-1) == _lib.ERR_INVALID
    assert call(ws=None) == _lib.ERR_WORKSPACE
    assert call(nbytes=need - 1) == _lib.ERR_WORKSPACE and b"workspace" in lib.fqb200_last_error()


# ---- the manager: which quantizer settings each collect call site hands over ---------------------------------------------------
def run_collect(arch, flags, base_dir, shape=(2, 3, 64, 64)):
    """A collect run on CPU with save_tensor_stats recorded; returns {id: (tag, clip_err)}."""
    from cnn_quantization_b200 import pipeline, statistics
    seen = {}

    def record(self, tensor, tag, id, tensors_q=None, force_global_min_max=False, clip_err=None):
        seen[id] = (tag, clip_err)

    mp = pytest.MonkeyPatch()
    mp.setattr(statistics.StatisticManager, "save_tensor_stats", record)
    mp.setattr(statistics.StatisticManagerPerChannel, "save_tensor_stats", record)
    try:
        cfg = dict(arch=arch, stats_folder=arch, stats_base_dir=base_dir, stats_mode="collect", **flags)
        model, qm = pipeline.build_quantized_model(cfg, "cpu")
        with torch.no_grad():
            model(torch.randn(shape))
        qm.detach()
    finally:
        mp.undo()
    return seen


def test_manager_passes_each_call_sites_use_mode_quantizer(tmp_path):
    from cnn_quantization_b200 import _lib as L
    seen = run_collect("resnet18", dict(qtype="int4", qweight="int4", collect_err=True), str(tmp_path))
    # conv0 is on the 8-bit `ignored` list of int4; it sits before a ReLU (half range)
    assert seen["conv0_activation"][1].num_bits == 8 and seen["conv0_activation"][1].positive
    assert seen["conv1_activation"][1].num_bits == 4 and seen["conv1_activation"][1].positive
    # the last convolution of a block is not before_relu (the ReLU follows the residual add)
    assert seen["conv2_activation"][1].num_bits == 4 and not seen["conv2_activation"][1].positive
    assert seen["linear0_activation"][0] == "activation_classifier"
    assert seen["linear0_activation"][1].num_bits == 8 and not seen["linear0_activation"][1].positive
    assert seen["maxpool0_out"][1].num_bits == 8 and not seen["maxpool0_out"][1].positive
    assert all(not c.bit_alloc and not c.per_channel for _, c in seen.values())
    # -baa without -pcq_a: the use-mode quantizers are per tensor, where bit allocation never applies
    seen = run_collect("resnet18", dict(qtype="int4", qweight="int4", collect_err=True, bit_alloc_act=True), str(tmp_path))
    assert all(not c.bit_alloc and not c.per_channel for _, c in seen.values())
    assert seen["conv1_activation"][1].num_bits == 4
    seen = run_collect("resnet18", dict(qtype="int4", qweight="int4", collect_err=True, per_channel_quant_act=True,
                                        bit_alloc_act=True, bit_alloc_prior="std", bit_alloc_rmode="ceil"), str(tmp_path))
    c = seen["conv1_activation"][1]
    assert c.per_channel and c.bit_alloc and c.bit_alloc_prior == L.PRIOR_B and not c.bit_alloc_round and c.bit_alloc_target == 4
    # the ignored stem and the poolings are quantized per tensor (pcq_a off) at 8 bits: no allocation
    assert not seen["conv0_activation"][1].per_channel and not seen["conv0_activation"][1].bit_alloc
    assert not seen["maxpool0_out"][1].per_channel and not seen["maxpool0_out"][1].bit_alloc
    assert not seen["linear0_activation"][1].per_channel


def test_manager_force_positive_on_vgg(tmp_path):
    seen = run_collect("vgg16", dict(qtype="int8", qweight="int8", collect_err=True), str(tmp_path), shape=(1, 3, 32, 32))
    convs = [c for k, (t, c) in seen.items() if k.startswith("conv")]
    assert convs and all(c.positive and c.num_bits == 8 for c in convs)
    assert not seen["linear2_activation"][1].positive   # the classifier


def test_manager_without_the_flag_passes_nothing(tmp_path):
    seen = run_collect("resnet18", dict(qtype="int4", qweight="int4"), str(tmp_path))
    assert seen and all(c is None for _, c in seen.values())


@pytest.mark.parametrize("flags", [dict(stats_mode="no", qtype="int4"), dict(stats_mode="use", qtype="int4"),
                                   dict(stats_mode="collect", qtype=None)])
def test_flag_validation(flags, tmp_path):
    from cnn_quantization_b200 import manager as M
    args = M.make_args(collect_err=True, stats_base_dir=str(tmp_path), **flags)
    with pytest.raises(ValueError, match="collect_err"):
        M.QuantizationManagerInference(args, M.get_params(args))


# ---- `-c mix` in use mode ----------------------------------------------------------------------------------------------------
class FakeStats(object):
    """get_tensor_stat over {id: {stat: value}} ('mean' kind only)."""

    def __init__(self, table):
        self.table = table

    def get_tensor_stat(self, id, stat, kind="mean"):
        return self.table[id]["%s_%s" % (kind, stat)]


def quantizer(sm, num_bits=4, pcq=False, bit_alloc=False, positive=False):
    import cnn_quantization_b200 as fq
    p = dict(clipping="mix", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=pcq, bit_alloc_act=bit_alloc,
             bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    q = fq.int_quantizer("int%d" % num_bits, p)
    q.sm = lambda: sm
    q.half_range = positive
    return q


def per_tensor_stats(lowp, gaus, laplace):
    return {"mean_min": -1.5, "mean_max": 4.0, "mean_mean": 0.25, "mean_b": 0.6, "mean_std": 0.8,
            "mean_mse_lowp": lowp, "mean_mse_gaus": gaus, "mean_mse_laplace": laplace}


def params(q, t, clip):
    d, o, b, pc = q._clipping_params_from_stats(t, "l", clip)
    return d.numpy(), o.numpy(), None if b is None else b.numpy()


@pytest.mark.parametrize("mse,want", [
    ((3.0, 1.0, 2.0), "gaus"),              # gaus < laplace, lowp worse than gaus
    ((0.5, 1.0, 0.1), "lowp"),              # lowp < gaus wins although laplace is best
    ((1.0, 1.0, 1.0), "laplace"),           # ties keep the earlier choice
    ((2.0, 1.0, 1.0), "laplace"),
    ((1.0, 1.0, 2.0), "gaus"),
    ((np.nan, np.nan, np.nan), "laplace"),  # statistics collected without error columns
    ((np.nan, 1.0, 2.0), "gaus"),
])
@pytest.mark.parametrize("positive", [False, True])
def test_mix_selection_per_tensor(mse, want, positive):
    t = torch.zeros(2, 3, 4, 4)
    q = quantizer(FakeStats({"l": per_tensor_stats(*mse)}), positive=positive)
    got = params(q, t, "mix")
    ref = params(q, t, want)
    for a, b in zip(got, ref):
        np.testing.assert_array_equal(a, b)
    assert np.asarray(q.get_alpha(t, stat_id="l", clip_type="mix")) == np.asarray(
        q._alpha_from_stats("l", want, False, t.device)[0], dtype=np.float64)


def per_channel_frame(mse=True):
    c = 5
    rs = np.random.RandomState(3)
    df = pd.DataFrame({"mean_min": -rs.rand(c).astype(np.float32) * 2, "mean_max": rs.rand(c).astype(np.float32) * 3 + 1,
                       "mean_mean": rs.randn(c).astype(np.float32) * 0.1, "mean_b": rs.rand(c).astype(np.float32) + 0.2,
                       "mean_std": rs.rand(c).astype(np.float32) + 0.3})
    if mse:
        df["mean_mse_lowp"] = np.array([3, 0.5, 1, 2, np.nan], dtype=np.float32)
        df["mean_mse_gaus"] = np.array([1, 1.0, 1, 1, np.nan], dtype=np.float32)
        df["mean_mse_laplace"] = np.array([2, 0.1, 1, 1, np.nan], dtype=np.float32)
    return df


@pytest.mark.parametrize("bit_alloc", [False, True])
def test_mix_selection_per_channel(bit_alloc):
    t = torch.zeros(2, 5, 4, 4)
    q = quantizer(FakeStats({"l": per_channel_frame()}), pcq=True, bit_alloc=bit_alloc)
    d, o, b = params(q, t, "mix")
    choice = ["gaus", "lowp", "laplace", "laplace", "laplace"]
    ref = {k: params(q, t, k) for k in ("lowp", "gaus", "laplace")}
    for ch, k in enumerate(choice):
        assert d[ch] == ref[k][0][ch] and o[ch] == ref[k][1][ch]
    if bit_alloc:
        np.testing.assert_array_equal(b, ref["laplace"][2])   # the allocated widths of the layer


def test_mix_per_channel_without_error_columns_names_collect_err():
    q = quantizer(FakeStats({"l": per_channel_frame(mse=False)}), pcq=True)
    with pytest.raises(KeyError, match="collect_err"):
        params(q, torch.zeros(2, 5, 4, 4), "mix")


def test_mix_needs_collected_statistics():
    q = quantizer(None)
    q.sm = None
    with pytest.raises(NotImplementedError):
        q.get_alpha(torch.zeros(2, 3), clip_type="mix")


def test_mix_on_reference_statistics_is_laplace():
    """The reference's collect leaves the error columns NaN: `-c mix -sm use` resolves to `-c laplace`, layer for layer."""
    from cnn_quantization_b200.statistics import StatisticManager
    sm = StatisticManager("resnet18", load_stats=True, base_dir=os.path.join(GOLD, "ref_stats"))
    assert sm.stats_df["mean_mse_laplace"].isna().all()
    for positive in (False, True):
        q = quantizer(sm, positive=positive)
        for layer in sm.stats_df.index:
            d, o, _, _ = q._clipping_params_from_stats(torch.zeros(2, 3, 4, 4), layer, "mix")
            dl, ol, _, _ = q._clipping_params_from_stats(torch.zeros(2, 3, 4, 4), layer, "laplace")
            assert torch.equal(d, dl) and torch.equal(o, ol), layer


# ---- default collect: NaN error columns -------------------------------------------------------------------------------------------
def test_default_collect_writes_nan_error_columns(monkeypatch, tmp_path):
    from cnn_quantization_b200 import ops
    from cnn_quantization_b200.statistics import StatisticManager

    def fused(x, layout, stats_only=False, **kw):
        return torch.ones((int(layout[1]), 12))

    def no_gpu(*a, **k):
        raise AssertionError("no error columns without a ClipErrConfig")

    monkeypatch.setattr(ops, "fused", fused)
    monkeypatch.setattr(ops, "clip_error", no_gpu)
    sm = StatisticManager("m", load_stats=False, base_dir=str(tmp_path))
    sm.save_tensor_stats(torch.randn(2, 3, 4, 4), "activation", "conv0_activation")
    sm.__exit__()
    df = pd.read_csv(tmp_path / "statistics" / "m" / "m_summary.csv", index_col=0)
    for c in ("mse_lowp", "mse_gaus", "mse_laplace", "cos_lowp", "cos_gaus", "cos_laplace"):
        assert df["mean_" + c].isna().all()


@pytest.mark.parametrize("per_channel,bit_alloc,channels_last", [
    (False, False, False), (True, False, False), (True, True, False), (False, False, True), (True, False, True),
    (True, True, True)], ids=["False-False", "True-False", "True-True", "False-False-cl", "True-False-cl", "True-True-cl"])
def test_managers_launch_the_configured_candidates(monkeypatch, tmp_path, per_channel, bit_alloc, channels_last):
    """What the collect measurements launch for a call site's quantizer.  collect_err (ops.clip_error): per tensor, one
    float64-solved group at the configured width and never a bit allocation; per channel (per-channel manager), the
    (sample, channel) groups of the NCHW tensor with the channel table repeated per sample and the allocation's widths
    only when configured; a per-tensor manager sums the same per-channel launch and runs its statistics launch once.
    collect_mse (ops.clip_mse) and collect_bits (ops.clip_mse or, under -c mse, ops.clip_mse_grid): per channel on a
    channels-last tensor the kernels take in place, per tensor on any dense memory order, else on the NCHW tensor."""
    from cnn_quantization_b200 import _lib as L, ops
    from cnn_quantization_b200.statistics import (BitMseStatistics, ClipErrConfig, ClipMseStatistics, StatisticManager,
                                                  StatisticManagerPerChannel, bit_candidates)
    launches, tables = [], []

    def fused(x, layout, stats_only=False, bit_alloc=False, num_bits=8, channels_last=False, any_dense_format=False, **kw):
        t = torch.arange(int(layout[1]) * 12, dtype=torch.float32).view(-1, 12)
        tables.append(dict(layout=tuple(layout), bit_alloc=bit_alloc, num_bits=num_bits, channels_last=channels_last,
                           any_dense_format=any_dense_format, kw=kw, table=t))
        return t

    def clip_error(x, table, layout, channels_last, num_bits, positive, bit_alloc=False, solve_f64=None, **kw):
        launches.append(dict(op="clip_error", layout=tuple(layout), num_bits=num_bits, positive=positive,
                             bit_alloc=bit_alloc, solve_f64=solve_f64, table=table.clone(), channels_last=channels_last,
                             nhwc=ops.nhwc(x)))
        return torch.ones((int(layout[1]), 10), dtype=torch.float64)

    def clip_mse(x, table, layout, channels_last, num_bits, positive, multipliers, prior="laplace", bit_alloc=False,
                 solve_f64=None, widths=None, **kw):
        launches.append(dict(op="clip_mse", layout=tuple(layout), num_bits=num_bits, positive=positive,
                             bit_alloc=bit_alloc, solve_f64=solve_f64, table=table, channels_last=channels_last,
                             nhwc=ops.nhwc(x), prior=prior, multipliers=torch.as_tensor(multipliers).tolist(),
                             widths=None if widths is None else list(widths)))
        return torch.ones((int(layout[1]), len(launches[-1]["multipliers"]) + 1), dtype=torch.float64)

    def clip_mse_grid(x, table, layout, channels_last, num_bits, positive, multipliers, widths, prior="laplace",
                      solve_f64=None, **kw):
        launches.append(dict(op="clip_mse_grid", layout=tuple(layout), num_bits=num_bits, positive=positive,
                             solve_f64=solve_f64, table=table, channels_last=channels_last, nhwc=ops.nhwc(x), prior=prior,
                             multipliers=torch.as_tensor(multipliers).tolist(), widths=list(widths)))
        return torch.ones((int(layout[1]), 1 + 9 * len(launches[-1]["multipliers"])), dtype=torch.float64)

    monkeypatch.setattr(ops, "fused", fused)
    monkeypatch.setattr(ops, "clip_error", clip_error)
    monkeypatch.setattr(ops, "clip_mse", clip_mse)
    monkeypatch.setattr(ops, "clip_mse_grid", clip_mse_grid)
    cfg = ClipErrConfig(num_bits=4, positive=True, per_channel=per_channel, bit_alloc=bit_alloc, bit_alloc_prior=L.PRIOR_STD,
                        bit_alloc_round=True, bit_alloc_target=4)
    x = torch.randn(2, 4, 4, 4)
    if channels_last:
        x = x.to(memory_format=torch.channels_last)
        assert ops.cl_eligible(x)
    chan_layout = (2, 4, 16) if per_channel else (1, 1, 128)
    cl = per_channel and channels_last

    def stats_launch(t, alloc):
        """The statistics-only launch of the quantizer ``cfg``, with its bit allocation when ``alloc``."""
        assert t["layout"] == chan_layout and t["bit_alloc"] == alloc and t["num_bits"] == (4 if alloc else 8)
        if alloc:
            assert t["kw"]["bit_alloc_prior"] == L.PRIOR_STD and t["kw"]["bit_alloc_round"] and t["kw"]["bit_alloc_target"] == 4
        assert per_channel or t["any_dense_format"]

    # -- collect_err ---------------------------------------------------------------------------------------------------------
    if not per_channel:
        StatisticManager("m", load_stats=False, base_dir=str(tmp_path)).save_tensor_stats(x, "a", "conv1_activation",
                                                                                         clip_err=cfg)
        (l,) = launches
        assert l["layout"] == (1, 1, 128) and l["num_bits"] == 4 and l["positive"] and not l["bit_alloc"] and l["solve_f64"]
        assert not l["channels_last"] and not l["nhwc"]
    else:
        sm = StatisticManagerPerChannel("m", load_stats=False, collect_err=True, base_dir=str(tmp_path))
        sm.save_tensor_stats(x, "a", "conv1_activation", clip_err=cfg)
        (l,) = launches
        assert l["layout"] == (1, 8, 16) and l["bit_alloc"] == bit_alloc and not l["solve_f64"]
        assert not l["channels_last"] and not l["nhwc"]
        chan = [t for t in tables if t["layout"] == (2, 4, 16) and t["bit_alloc"] == bit_alloc][-1]
        assert not chan["channels_last"]
        assert torch.equal(l["table"], chan["table"].repeat(2, 1))   # row n * C + c = channel c
        assert set(sm.stats["conv1_activation"]) >= {"mse_lowp", "cos_laplace"}
        # a per-channel quantizer under the per-tensor manager: all channels' errors together, one statistics launch
        del launches[:], tables[:]
        StatisticManager("m", load_stats=False, base_dir=str(tmp_path)).save_tensor_stats(x, "a", "conv1_activation",
                                                                                         clip_err=cfg)
        (l,) = launches
        assert l["layout"] == (1, 8, 16) and l["bit_alloc"] == bit_alloc and not l["solve_f64"] and not l["nhwc"]
        chan = [t for t in tables if t["layout"] == (2, 4, 16)]
        assert len(chan) == 1
        stats_launch(chan[0], bit_alloc)
        assert torch.equal(l["table"], chan[0]["table"].repeat(2, 1))

    # -- collect_mse ---------------------------------------------------------------------------------------------------------
    for prior in ("laplace", "gaus"):
        del launches[:], tables[:]
        ClipMseStatistics("m", multipliers=[1.0, 2.5, 4.0], prior=prior, base_dir=str(tmp_path)).save_curve(
            x, "a", "conv1_activation", cfg)
        (t,), (l,) = tables, launches
        stats_launch(t, bit_alloc)
        assert t["channels_last"] == cl
        assert l["op"] == "clip_mse" and l["table"] is t["table"] and l["layout"] == chan_layout
        assert l["channels_last"] == cl and l["nhwc"] == (channels_last and (cl or not per_channel))
        assert l["num_bits"] == 4 and l["positive"] and l["bit_alloc"] == bit_alloc and l["solve_f64"] == (not per_channel)
        assert l["prior"] == prior and l["multipliers"] == [1.0, 2.5, 4.0] and l["widths"] is None

    # -- collect_bits --------------------------------------------------------------------------------------------------------
    for rule in ("laplace", "gaus", "no", "mse"):
        del launches[:], tables[:]
        BitMseStatistics("m", rule, base_dir=str(tmp_path), multipliers=[1.0, 2.5], prior="gaus").save_table(
            x, "a", "conv1_activation", cfg)
        if not (per_channel and bit_alloc):
            assert not launches and not tables
            continue
        (t,), (l,) = tables, launches
        stats_launch(t, False)   # an 8-bit table without allocation: every width is a candidate of its own
        assert t["channels_last"] == cl
        assert l["table"] is t["table"] and l["layout"] == chan_layout and l["channels_last"] == cl and l["nhwc"] == cl
        assert l["num_bits"] == 4 and l["positive"] and not l["solve_f64"] and l["widths"] == list(range(9))
        if rule == "mse":
            assert l["op"] == "clip_mse_grid" and l["prior"] == "gaus" and l["multipliers"] == [1.0, 2.5]
        else:
            mults, p = bit_candidates(rule, True, 4)
            assert l["op"] == "clip_mse" and not l["bit_alloc"] and l["prior"] == p
            assert l["multipliers"] == torch.tensor(mults, dtype=torch.float32).tolist()


@pytest.mark.parametrize("channels_last", [False, True], ids=["nchw", "cl"])
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("baa", [False, True])
@pytest.mark.parametrize("positive", [False, True])
@pytest.mark.parametrize("pcq", [False, True])
def test_on_the_fly_routes_launch_what_collect_measures(monkeypatch, tmp_path, pcq, positive, baa, bits, channels_last):
    """One call site, measured in collect mode (the manager's _clip_err) and on the fly (its quantizer): the
    statistics-only launch and the candidate launch get the same arguments.  `-c mse -sm no` makes collect_mse's curve
    with ops.clip_mse_select in place of ops.clip_mse; fly_bits makes collect_bits' width tables under each rule, with
    want_params.  Collect runs -bap laplace: the prior fly_bits' -bap mse describes its call sites with."""
    import inspect
    import cnn_quantization_b200.manager as M
    from cnn_quantization_b200 import ops
    calls = []

    def sums(a, k):
        g = int(a["layout"][1])
        s = torch.zeros(g, k + 1, dtype=torch.float64)
        return (s, torch.zeros(g, k, 6)) if a.get("want_params") else s

    results = {
        "fused": lambda a: torch.zeros(int(a["layout"][1]), 12),
        "clip_mse": lambda a: sums(a, len(a["multipliers"])),
        "clip_mse_grid": lambda a: sums(a, 9 * len(a["multipliers"])),
        "clip_mse_select": lambda a: (sums(a, len(a["multipliers"])), torch.zeros(int(a["layout"][1]), dtype=torch.int32),
                                      torch.ones(3, int(a["layout"][1])), torch.ones(int(a["layout"][1]), 12)),
    }

    def recorder(name):
        sig = inspect.signature(getattr(ops, name))

        def rec(*args, **kw):
            bound = sig.bind(*args, **kw)
            bound.apply_defaults()
            a = dict(bound.arguments)
            a["nhwc"] = ops.nhwc(a.pop("x"))
            table = a.pop("table", None)
            if "multipliers" in a:
                a["multipliers"] = torch.as_tensor(a["multipliers"]).tolist()
            if a.get("widths") is not None:
                a["widths"] = list(a["widths"])
            res = results[name](a)
            calls.append((name, a, table, res))
            return res
        return rec

    for name in results:
        monkeypatch.setattr(ops, name, recorder(name))
    monkeypatch.setattr(ops, "allocate_select", lambda s, p, stats, target, multipliers=None, status=None: (
        torch.full((s.shape[0],), 3.0), None, torch.ones(3, s.shape[0]), torch.ones(s.shape[0], 12)))
    monkeypatch.setattr(ops, "quantize1", lambda x, *a, **kw: x)
    x = torch.randn(2, 4, 4, 4)
    if channels_last:
        x = x.to(memory_format=torch.channels_last)
    flags = dict(qtype="int%d" % bits, per_channel_quant_act=pcq, bit_alloc_act=baa, mse_multipliers=[1.0, 2.5, 4.0],
                 mse_prior="gaus")

    def run(collect, **over):
        """[(op, arguments)] of the call site's measurement launches under a manager with ``flags`` and ``over``."""
        args = M.make_args(**dict(flags, **over))
        qm = M.QuantizationManagerInference(args, M.get_params(args))
        del calls[:]
        if collect:
            qm._clip_err(x, "activation", "conv1_activation", positive, "conv1")
        else:
            q = qm.quantizers["activation"]
            q.half_range = positive
            q(x.clone(), "conv1_activation", "activation")
        for i, (name, _, table, _) in enumerate(calls):   # each candidate launch reads the table of the launch before it
            assert table is None if name == "fused" else table is calls[i - 1][3]
        return [c[:2] for c in calls]

    allocates = pcq and baa and bits == 4
    fly_mse = run(False, clipping="mse", bit_alloc_prior="laplace")
    assert [n for n, _ in fly_mse] == ["fused", "clip_mse_select"]
    for rule in ("laplace", "gaus", "no", "mse"):
        collect = run(True, clipping=rule, bit_alloc_prior="laplace", stats_mode="collect", stats_base_dir=str(tmp_path),
                      collect_mse=True, collect_bits=pcq and baa)
        (_, stats), (op, curve) = collect[:2]
        assert op == "clip_mse" and stats["stats_only"] and stats["positive"] == positive
        assert stats["layout"] == ((2, 4, 16) if pcq else (1, 1, 128)) and stats["channels_last"] == (pcq and channels_last)
        assert curve["num_bits"] == bits and curve["bit_alloc"] == allocates and curve["multipliers"] == [1.0, 2.5, 4.0]
        assert fly_mse[0][1] == stats
        assert fly_mse[1][1] == {k: v for k, v in curve.items() if k not in ("want_params", "widths")}
        tables = collect[2:]
        if not allocates:
            assert not tables
            continue
        fly_bits = run(False, clipping=rule, bit_alloc_prior="mse", fly_bits=True)
        assert [n for n, _ in tables] == [n for n, _ in fly_bits] == ["fused", "clip_mse_grid" if rule == "mse" else "clip_mse"]
        assert not tables[0][1]["bit_alloc"] and tables[1][1]["widths"] == list(range(9))
        assert fly_bits[0][1] == tables[0][1]
        assert fly_bits[1][1] == dict(tables[1][1], want_params=True)
