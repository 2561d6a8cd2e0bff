"""Clipping-MSE curves (collect_mse) and `-c mse` without a GPU: the C ABI's workspace sizes and argument checks, the
manager's flag validation, the argmin and its tie rule, the clip_mse.pkl / curve.csv round trip into `-c mse`'s alpha, the
missing-curve errors, and the float64 port of the reference's mse_analysis.py against its own output
(tests/golden/ref_mse_analysis.npz)."""
import ctypes
import os
import pickle
import sys

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
    ws = lib.fqb200_clip_mse_workspace_bytes
    assert ws(1, 1, 1 << 18, 0, 125) == 126 * 8                  # 2^18-element units on NCHW / per tensor
    assert ws(1, 1, (1 << 18) + 1, 0, 125) == 2 * 126 * 8
    assert ws(512, 64, 112 * 112, 0, 125) == 64 * 25 * 126 * 8
    assert ws(512, 64, 112 * 112, 1, 125) == 64 * 784 * 126 * 8  # channels-last: 8192-pixel units per channel
    assert ws(8, 96, 10 * 12, 1, 1) == 96 * 1 * 2 * 8
    assert ws(1, 1, 4, 0, 256) == 257 * 8
    assert ws(1, 1, 4, 0, 0) == 0 and b"num_multipliers" in lib.fqb200_last_error()
    assert ws(1, 1, 4, 0, 257) == 0 and b"num_multipliers" in lib.fqb200_last_error()
    assert ws(0, 4, 4, 0, 8) == 0 and b"> 0" in lib.fqb200_last_error()
    assert ws(2, 6, 4, 1, 8) == 0 and b"C %" in lib.fqb200_last_error()
    assert ws(2, 3, 1 << 31, 0, 8) == 0 and b"2^32" in lib.fqb200_last_error()


def test_abi_rejects_bad_arguments(lib):
    from cnn_quantization_b200 import _lib
    buf = ctypes.create_string_buffer(1 << 14)
    need = lib.fqb200_clip_mse_workspace_bytes(2, 4, 64, 0, 8)

    def call(inp=buf, groups=4, cl=0, stats=buf, bits=4, bit_alloc=0, prior=0, mult=buf, k=8, out=buf, ws=buf, nbytes=need,
             ctas=0):
        return lib.fqb200_clip_mse(inp, 2, groups, 64, cl, stats, bits, 0, bit_alloc, 0, prior, mult, k, out, None, ws, nbytes,
                                   ctas, None)

    assert call(k=0) == _lib.ERR_INVALID and b"num_multipliers" in lib.fqb200_last_error()
    assert call(k=257) == _lib.ERR_INVALID
    assert call(prior=2) == _lib.ERR_INVALID and b"prior" in lib.fqb200_last_error()
    assert call(prior=-1) == _lib.ERR_INVALID
    assert call(cl=1, groups=6) == _lib.ERR_INVALID and b"C %" in lib.fqb200_last_error()
    for kw in ("inp", "stats", "mult", "out"):
        assert call(**{kw: None}) == _lib.ERR_INVALID and b"null" in lib.fqb200_last_error()
    assert call(bits=9) == _lib.ERR_INVALID and b"num_bits" in lib.fqb200_last_error()
    assert call(bits=8, bit_alloc=1) == _lib.ERR_INVALID and b"bit_alloc" in lib.fqb200_last_error()
    assert call(ctas=-1) == _lib.ERR_INVALID
    assert call(ws=None) == _lib.ERR_WORKSPACE
    assert call(nbytes=need - 1) == _lib.ERR_WORKSPACE and b"workspace" in lib.fqb200_last_error()


def test_ops_rejects_bad_arguments():
    from cnn_quantization_b200 import ops, _lib
    with pytest.raises(_lib.FqError):
        ops.clip_mse(torch.zeros(4), torch.zeros(1, 12), (1, 1, 4), False, 4, False, [1.0])   # CPU tensor


# ---- the manager ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flags", [dict(stats_mode="no", qtype="int4"), dict(stats_mode="use", qtype="int4"),
                                   dict(stats_mode="collect", qtype=None)])
def test_collect_mse_needs_collect_and_qtype(flags, tmp_path):
    from cnn_quantization_b200 import manager as M
    args = M.make_args(arch="resnet18", collect_mse=True, stats_base_dir=str(tmp_path), **flags)
    with pytest.raises(ValueError, match="collect_mse"):
        M.QuantizationManagerInference(args, M.get_params(args))


def test_bad_prior_and_multipliers(tmp_path):
    from cnn_quantization_b200.statistics import ClipMseStatistics
    with pytest.raises(ValueError, match="mse_prior"):
        ClipMseStatistics("x", prior="cauchy", base_dir=str(tmp_path))
    with pytest.raises(ValueError, match="mse_multipliers"):
        ClipMseStatistics("x", multipliers=[], base_dir=str(tmp_path))
    with pytest.raises(ValueError, match="mse_multipliers"):
        ClipMseStatistics("x", multipliers=np.ones(257), base_dir=str(tmp_path))


def test_default_multipliers():
    from cnn_quantization_b200.statistics import MSE_MULTIPLIERS
    assert len(MSE_MULTIPLIERS) == 125 and MSE_MULTIPLIERS[0] == 0.5 and MSE_MULTIPLIERS[-1] == 16.0
    assert np.all(np.diff(MSE_MULTIPLIERS) == 0.125)


# ---- argmin -------------------------------------------------------------------------------------------------------------------
def test_argmin_and_tie_rule():
    from cnn_quantization_b200.statistics import best_multipliers
    m = [1.0, 2.0, 3.0, 4.0]
    mse = np.array([[4.0, 3.0, 1.0, 2.0],          # clear minimum
                    [5.0, 1.0, 1.0, 1.0],          # ties: the smallest multiplier
                    [np.nan, 2.0, np.nan, 2.0],    # NaN never wins
                    [np.nan] * 4])                 # nothing measured: the smallest multiplier
    np.testing.assert_array_equal(best_multipliers(m, mse), np.float32([3, 2, 2, 1]))
    # unsorted multipliers: the tie still goes to the smaller multiplier, wherever its column is
    np.testing.assert_array_equal(best_multipliers([4.0, 2.0, 3.0], np.array([[1.0, 1.0, 5.0]])), np.float32([2]))
    assert best_multipliers(m, mse).dtype == np.float32


# ---- files and `-c mse` ---------------------------------------------------------------------------------------------------------
def fake_curves(tmp_path, positive=False, prior="laplace"):
    """A ClipMseStatistics with two batches' worth of accumulated sums for a per-channel (3 groups) and a per-tensor id,
    written to tmp_path; returns it with the sums."""
    from cnn_quantization_b200.statistics import ClipMseStatistics
    mults = [0.5, 1.0, 2.0, 4.0]
    cs = ClipMseStatistics("r18", multipliers=mults, prior=prior, base_dir=str(tmp_path))
    per_batch = 2 * 16   # N * HW of one batch
    sse_pc = np.array([[100.0, 9.0, 4.0, 4.0, 6.0],
                       [50.0, 1.0, 2.0, 3.0, 4.0],
                       [70.0, 8.0, 7.0, 6.0, 5.0]])
    bsd_pc = np.array([[1.0, 1.5, 4.0], [0.5, 0.7, 3.0], [2.0, 2.5, 2.0]]) * 2   # two batches of (b, std, bits)
    sse_pt = np.array([[300.0, 30.0, 10.0, 20.0, 40.0]])
    bsd_pt = np.array([[0.8, 1.1, 4.0]]) * 2
    cs.acc = {"conv1_activation": (torch.from_numpy(sse_pc), torch.from_numpy(bsd_pc), 2),
              "linear20_activation": (torch.from_numpy(sse_pt), torch.from_numpy(bsd_pt), 2)}
    cs.meta = {"conv1_activation": ("conv1", positive, per_batch), "linear20_activation": ("fc", False, 64)}
    cs.__exit__()
    return cs, mults, sse_pc, bsd_pc / 2, sse_pt


@pytest.mark.parametrize("positive,prior", [(False, "laplace"), (True, "gaus")])
def test_pickle_and_csv_round_trip(tmp_path, positive, prior):
    from cnn_quantization_b200 import mse_analysis as MA
    cs, mults, sse, bsd, sse_pt = fake_curves(tmp_path, positive, prior)
    folder = os.path.join(str(tmp_path), "clip_mse", "r18")
    with open(os.path.join(folder, "clip_mse.pkl"), "rb") as f:
        d = pickle.load(f)
    assert d["prior"] == prior
    np.testing.assert_array_equal(d["multipliers"], mults)
    df = d["conv1_activation"]
    assert list(df.columns) == ["count", "b", "std", "bits", "mse_0", "mse_1", "mse_2", "mse_3"]
    np.testing.assert_array_equal(df["count"], [64.0] * 3)
    np.testing.assert_array_equal(df[["b", "std", "bits"]].to_numpy(), bsd)
    np.testing.assert_array_equal(df[["mse_%d" % k for k in range(4)]].to_numpy(), sse[:, 1:] / 64)
    assert len(d["linear20_activation"]) == 1
    csv = pd.read_csv(os.path.join(folder, "curve.csv"), float_precision="round_trip")
    assert list(csv.columns) == ["id", "internal_name", "multiplier", "mse", "mse_laplace_analytic", "mse_gaus_analytic"]
    c1 = csv[csv.id == "conv1_activation"]
    assert (c1.internal_name == "conv1").all()
    np.testing.assert_allclose(c1.mse, sse[:, 1:].sum(0) / 192, rtol=1e-15)
    # analytic curves: per group at alpha = m * b (or std), width + 1 on a positive range, weighted by the group's count
    scale = bsd[:, 0] if prior == "laplace" else bsd[:, 1]
    width = bsd[:, 2] + (1 if positive else 0)
    lap = np.mean([[2 * b ** 2 * np.e ** (-(m * s) / b) + (m * s) ** 2 / (3 * 2 ** (2 * w)) for m in mults]
                   for b, s, w in zip(bsd[:, 0], scale, width)], axis=0)
    np.testing.assert_allclose(c1.mse_laplace_analytic, lap, rtol=1e-13)
    gau = np.mean([MA.GaussianClippingAnalysis(np.float64(mults) * s, sd, w).numpy() for sd, s, w in zip(bsd[:, 1], scale, width)],
                  axis=0)
    np.testing.assert_allclose(c1.mse_gaus_analytic, gau, rtol=1e-13)
    # read back: the argmin per group
    from cnn_quantization_b200.statistics import ClipMseStatistics
    back = ClipMseStatistics("r18", base_dir=str(tmp_path), load=True)
    m, p = back.best("conv1_activation")
    np.testing.assert_array_equal(m, np.float32([1.0, 0.5, 4.0]))    # group 0: tie between 1.0 and 2.0 -> 1.0
    assert p == prior
    np.testing.assert_array_equal(back.best("linear20_activation")[0], np.float32([1.0]))
    back.__exit__()   # a loaded instance writes nothing
    assert os.path.exists(os.path.join(folder, "clip_mse.pkl"))


class _Stats(object):
    def __init__(self, table):
        self.table = table

    def get_tensor_stat(self, id, stat, kind="mean"):
        return self.table[stat]


def quantizer(**over):
    from cnn_quantization_b200.int_quantizer import IntQuantizer
    p = dict(clipping="mse", stats_kind="mean", kld=False, pcq_weights=False, pcq_act=True, bit_alloc_act=False,
             bit_alloc_weight=False, bcorr_act=False, bcorr_weight=False, vcorr_weight=False, bit_alloc_rmode="round",
             bit_alloc_prior="gaus", bit_alloc_target_act=None, bit_alloc_target_weight=None, measure_entropy=False,
             logger=None, mtd_quant=False)
    p.update(over)
    return IntQuantizer(4, p)


@pytest.mark.parametrize("prior", ["laplace", "gaus"])
def test_use_mode_alpha_from_the_curves(tmp_path, prior):
    from cnn_quantization_b200.statistics import ClipMseStatistics
    fake_curves(tmp_path, prior=prior)
    q = quantizer()
    b = np.float32([0.3, 0.7, 1.1])
    sd = np.float32([0.4, 0.9, 1.3])
    q.sm = lambda: _Stats({"b": b, "std": sd})
    q.mse_curves = ClipMseStatistics("r18", base_dir=str(tmp_path), load=True)
    alpha, bits = q._mse_alpha_from_stats("conv1_activation", True, "cpu")
    assert alpha.dtype == np.float32 and bits is None
    np.testing.assert_array_equal(alpha, (b if prior == "laplace" else sd) * np.float32([1.0, 0.5, 4.0]))
    q.sm = lambda: _Stats({"b": 0.8125, "std": 1.25})
    alpha, _ = q._mse_alpha_from_stats("linear20_activation", False, "cpu")
    assert alpha == (0.8125 if prior == "laplace" else 1.25) * 1.0
    with pytest.raises(ValueError, match="per channel"):
        q._mse_alpha_from_stats("conv1_activation", False, "cpu")


def test_missing_curves_raise_keyerror(tmp_path):
    from cnn_quantization_b200.statistics import ClipMseStatistics
    q = quantizer()
    q.sm = lambda: _Stats({"b": np.float32([1.0])})
    with pytest.raises(KeyError, match="collect_mse"):
        q._mse_alpha_from_stats("conv1_activation", True, "cpu")    # no curves attached
    q.mse_curves = ClipMseStatistics("r18", base_dir=str(tmp_path), load=True)
    with pytest.raises(KeyError, match="collect_mse"):
        q._mse_alpha_from_stats("conv1_activation", True, "cpu")    # no file
    fake_curves(tmp_path)
    q.mse_curves = ClipMseStatistics("r18", base_dir=str(tmp_path), load=True)
    with pytest.raises(KeyError, match="collect_mse"):
        q._mse_alpha_from_stats("conv7_activation", True, "cpu")    # no curve for this layer


def test_mse_without_offline_statistics_is_not_implemented():
    q = quantizer()
    with pytest.raises(NotImplementedError):
        q._range_mode("mse")
    with pytest.raises(NotImplementedError, match="collect_mse"):
        q.get_alpha(torch.zeros(2, 4, 3, 3), clip_type="mse", per_channel=True)


# ---- mse_analysis.py --------------------------------------------------------------------------------------------------------------
def test_mse_analysis_against_the_reference():
    sys.path.insert(0, GOLD)
    try:
        import make_mse_analysis_golden as G
    finally:
        sys.path.remove(GOLD)
    from cnn_quantization_b200 import mse_analysis as MA
    d = np.load(os.path.join(GOLD, "ref_mse_analysis.npz"))
    for name, prior, _, _, _, _ in G.CASES:
        alpha = d[name + "_alpha"]
        scale, bits, seed, total = d[name + "_meta"]
        sample = G.draw(prior, scale, int(seed))
        assert sample.sum() == total
        lap = prior == "laplace"
        ana = (MA.LaplacianClippingAnalysis if lap else MA.GaussianClippingAnalysis)(alpha, scale, int(bits))
        sim = (MA.LaplacianClippingSimulation if lap else MA.GaussianClippingSimulation)(alpha, sample, int(bits))
        assert ana.dtype == torch.float64 and sim.dtype == torch.float64
        np.testing.assert_allclose(ana.numpy(), d[name + "_analysis"], rtol=1e-14, atol=0)
        np.testing.assert_allclose(sim.numpy(), d[name + "_simulation"], rtol=1e-12, atol=0)


def test_mse_analysis_script_writes_csv(tmp_path):
    from cnn_quantization_b200 import mse_analysis as MA
    out = os.path.join(str(tmp_path), "curves.csv")
    MA.main(["--prior", "gaus", "--seed", "3", "--out", out])
    df = pd.read_csv(out, float_precision="round_trip")
    assert list(df.columns) == ["alpha", "simulation", "analysis"] and len(df) == 150
    np.random.seed(3)
    x = np.random.normal(0, 2, size=100000)
    np.testing.assert_allclose(df.simulation, MA.GaussianClippingSimulation(np.arange(5, 20, 0.1), x, 4).numpy(), rtol=1e-15)
